"""H100-native Wave-U-Net forward path (drop-in for haoxiangsnr/Wave-U-Net-for-Speech-Enhancement's
``model/unet_basic.py``). See DESIGN.md / INTEGRATION.md at the repo root."""
from .unet_basic import Model  # noqa: F401

__all__ = ["Model"]
