"""b200sd -- Hopper-native Stable Diffusion hot path (UNet denoising loop, CFG + scheduler
step, VAE decoder) behind the reference's model-call / pipeline interface.

The directory is named ``ml-stable-diffusion_b200`` (not importable as-is); import it as
``b200sd`` (``b200sd/__init__.py`` at the repo root forwards here).
"""
from . import config  # noqa: F401

__all__ = ["config"]
