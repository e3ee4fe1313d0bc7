from moge_b200.dinov2 import (dinov2_vits14, dinov2_vitb14, dinov2_vitl14, dinov2_vitg14, dinov2_vits14_reg,  # noqa: F401
                              dinov2_vitb14_reg, dinov2_vitl14_reg, dinov2_vitg14_reg)
