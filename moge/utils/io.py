"""Drop-in for the writers of the reference's `moge.utils.io` that its CLI calls: `save_glb` and `save_ply` (moge_b200.export)."""
from moge_b200.export import save_glb, save_ply  # noqa: F401

__all__ = ["save_glb", "save_ply"]
