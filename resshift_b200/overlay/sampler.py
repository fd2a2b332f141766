"""Overlay of the reference's top-level ``sampler`` module: same names, H100-native hot path."""
from resshift_b200.sampler import BaseSampler, ResShiftSampler  # noqa: F401
