"""ConvTranspose2d(2, 2) up-sampling used by YoloNASUpStage (reference: modules/sampling.py:50-86)."""
from torch import nn

from .. import functional as SF


class ConvTranspose2x2(nn.ConvTranspose2d):
    """nn.ConvTranspose2d(c_in, c_out, kernel_size=2, stride=2) parameters; forward = GEMM + pixel-scatter store."""

    def __init__(self, in_channels: int, out_channels: int):
        super().__init__(in_channels, out_channels, kernel_size=2, stride=2)
        self._cache = {}

    def forward(self, x, output_size=None):
        return SF.conv_transpose2x2(x, self.weight, self.bias, self._cache)


def make_upsample_module_with_explicit_channels(in_channels: int, out_channels: int, scale_factor: int, upsample_mode="conv_transpose", align_corners=None) -> nn.Module:
    mode = getattr(upsample_mode, "value", upsample_mode)
    if str(mode).lower() not in ("conv_transpose",) or scale_factor != 2:
        raise NotImplementedError(f"upsample mode {upsample_mode} (x{scale_factor}) has no sm_90a kernel; YOLO-NAS uses conv_transpose x2")
    return ConvTranspose2x2(in_channels, out_channels)
