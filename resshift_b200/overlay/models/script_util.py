"""Overlay of the reference's ``models.script_util``: the yaml ``diffusion.target`` factories."""
from resshift_b200.models.script_util import create_gaussian_diffusion, create_gaussian_diffusion_ddpm  # noqa: F401
