"""`Conv`, `ConvBNAct` with the reference's constructor signature and state-dict keys
(modules/conv_bn_act_block.py:9-104); forward is the fused sm_90a path (functional.conv_bn_act)."""
from typing import Tuple, Type, Union

from torch import nn

from .. import functional as SF
from ..common.factories import activation_code
from .utils import autopad


def _single(v):
    if isinstance(v, (tuple, list)):
        if len(set(v)) != 1:
            raise NotImplementedError(f"only square kernels / symmetric strides are implemented, got {v}")
        return int(v[0])
    return int(v)


def check_conv_supported(conv: nn.Conv2d):
    if conv.groups != 1:
        raise NotImplementedError("grouped convolutions have no sm_90a kernel in super_gradients_b200")
    if _single(conv.dilation) != 1:
        raise NotImplementedError("dilated convolutions have no sm_90a kernel in super_gradients_b200")
    if conv.padding_mode != "zeros":
        raise NotImplementedError("only zero padding is implemented")


class _FusedConvBN:
    """Mixin: runs conv -> bn -> act of sibling nn.Conv2d / nn.BatchNorm2d parameter containers through the fused path."""

    def _fused(self, x, conv: nn.Conv2d, bn, act_code: str, cache, residual=None, sample_scale=None):
        stride, pad = _single(conv.stride), _single(conv.padding)
        if bn is None:
            return SF.conv_bias(x, conv.weight, conv.bias, stride=stride, pad=pad, cache=cache, act=act_code)
        if conv.bias is not None:
            raise NotImplementedError("Conv2d(bias=True) followed by BatchNorm is not on the supported path")
        momentum = 0.1 if bn.momentum is None else bn.momentum
        return SF.conv_bn_act(
            x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked,
            stride=stride, pad=pad, eps=bn.eps, momentum=momentum, act=act_code, training=self.training and bn.training, cache=cache, residual=residual, sample_scale=sample_scale,
            sync=SF.bn_sync(bn),
        )  # fmt: skip


class ConvBNAct(nn.Module, _FusedConvBN):
    def __init__(
        self,
        in_channels: int,
        out_channels: int,
        kernel_size: Union[int, Tuple[int, int]],
        padding: Union[int, Tuple[int, int]],
        activation_type: Type[nn.Module],
        stride: Union[int, Tuple[int, int]] = 1,
        dilation: Union[int, Tuple[int, int]] = 1,
        groups: int = 1,
        bias: bool = True,
        padding_mode: str = "zeros",
        use_normalization: bool = True,
        eps: float = 1e-5,
        momentum: float = 0.1,
        affine: bool = True,
        track_running_stats: bool = True,
        device=None,
        dtype=None,
        activation_kwargs=None,
    ):
        super().__init__()
        activation_kwargs = activation_kwargs or {}
        self.seq = nn.Sequential()
        self.seq.add_module("conv", nn.Conv2d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding, dilation=dilation, groups=groups, bias=bias, padding_mode=padding_mode))
        if use_normalization:
            self.seq.add_module("bn", nn.BatchNorm2d(out_channels, eps=eps, momentum=momentum, affine=affine, track_running_stats=track_running_stats, device=device, dtype=dtype))
        if activation_type is not None:
            self.seq.add_module("act", activation_type(**activation_kwargs))
        self._act_code = activation_code(activation_type)
        check_conv_supported(self.seq.conv)
        self._cache = SF.WeightCache()

    def forward(self, x, residual=None):
        return self._fused(x, self.seq.conv, getattr(self.seq, "bn", None), self._act_code, self._cache, residual)

    def replace_input_channels(self, in_channels: int, compute_new_weights_fn=None):
        from .weight_replacement_utils import replace_conv2d_input_channels

        self.seq[0] = replace_conv2d_input_channels(conv=self.seq[0], in_channels=in_channels, fn=compute_new_weights_fn)
        check_conv_supported(self.seq[0])

    def get_input_channels(self) -> int:
        return self.seq[0].in_channels


class Conv(nn.Module, _FusedConvBN):
    def __init__(self, input_channels, output_channels, kernel, stride, activation_type: Type[nn.Module], padding: int = None, groups: int = None):
        super().__init__()
        self.conv = nn.Conv2d(input_channels, output_channels, kernel, stride, autopad(kernel, padding), groups=groups or 1, bias=False)
        self.bn = nn.BatchNorm2d(output_channels)
        self.act = activation_type()
        self._act_code = activation_code(activation_type)
        check_conv_supported(self.conv)
        self._cache = SF.WeightCache()

    def forward(self, x):
        return self._fused(x, self.conv, self.bn, self._act_code, self._cache)

    def replace_input_channels(self, in_channels: int, compute_new_weights_fn=None):
        from .weight_replacement_utils import replace_conv2d_input_channels

        self.conv = replace_conv2d_input_channels(conv=self.conv, in_channels=in_channels, fn=compute_new_weights_fn)
        check_conv_supported(self.conv)

    def get_input_channels(self) -> int:
        return self.conv.in_channels
