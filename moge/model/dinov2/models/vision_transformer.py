from moge_b200.dinov2 import DinoVisionTransformer, vit_small, vit_base, vit_large, vit_giant2  # noqa: F401
