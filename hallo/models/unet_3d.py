"""hallo.models.unet_3d (scripts/inference.py:46) -> the H100 engine-backed class (hallo/models/unet_3d.py:59-839)."""
from hallo_b200.models.unet_3d import UNet3DConditionModel, UNet3DConditionOutput  # noqa: F401
