"""Drop-in for the reference operator package ``models/stylegan2/op`` (op/__init__.py:1-2):
same three names, same signatures and defaults, backed by libhairfast_sm90.so."""
from .fused_act import FusedLeakyReLU, fused_leaky_relu
from .upfirdn2d import upfirdn2d

__all__ = ["FusedLeakyReLU", "fused_leaky_relu", "upfirdn2d"]
