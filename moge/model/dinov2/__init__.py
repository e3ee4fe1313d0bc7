"""Drop-in alias of the reference's moge.model.dinov2 package, backed by moge_b200.dinov2 (sm_90a encoder kernels)."""
__version__ = "0.0.1"

from moge_b200.dinov2 import DinoVisionTransformer  # noqa: F401
