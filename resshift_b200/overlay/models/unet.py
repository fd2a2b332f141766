"""Overlay of the reference's ``models.unet``: ``UNetModelSwin`` runs on the sm_90a kernels.
(``models`` is a namespace package in the reference — no __init__.py — so every other ``models.*`` module
keeps resolving to the reference tree.)"""
from resshift_b200.models.unet import UNetModelSwin  # noqa: F401
