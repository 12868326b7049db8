"""YOLO-NAS stages with the reference's names, signatures and state-dict keys
(training/models/detection_models/yolo_nas/yolo_stages.py).  All arithmetic goes through the fused blocks."""
from functools import partial
from typing import Iterable, List, Type, Union

import torch
from torch import Tensor, nn

from ..... import functional as SF
from .....common.factories import resolve_activation
from .....common.registry import register_detection_module
from .....modules import BaseDetectionModule, Conv, QARepVGGBlock, Residual
from .....modules.sampling import make_upsample_module_with_explicit_channels
from .....modules.utils import width_multiplier

__all__ = ["YoloNASStage", "YoloNASUpStage", "YoloNASStem", "YoloNASDownStage", "YoloNASBottleneck", "YoloNASCSPLayer"]


class YoloNASBottleneck(nn.Module):
    def __init__(self, input_channels: int, output_channels: int, block_type: Type[nn.Module], activation_type: Type[nn.Module], shortcut: bool, use_alpha: bool, drop_path_rate: float = 0.0):
        super().__init__()
        if drop_path_rate > 0.0:
            raise NotImplementedError("drop_path_rate > 0 is not used by the shipped YOLO-NAS recipes and is not implemented")
        self.cv1 = block_type(input_channels, output_channels, activation_type=activation_type)
        self.cv2 = block_type(output_channels, output_channels, activation_type=activation_type)
        self.add = shortcut and input_channels == output_channels
        self.shortcut = Residual() if self.add else None
        self.drop_path = nn.Identity()
        if use_alpha:
            self.alpha = torch.nn.Parameter(torch.tensor([1.0]), requires_grad=True)
        else:
            self.alpha = 1.0

    def forward(self, x):
        learnable = self.add and isinstance(self.alpha, torch.Tensor)
        tok = SF.defer_shortcut_offer(x, self.alpha) if learnable and self.training else None
        h = self.cv1(x)
        tok = SF.defer_shortcut_withdraw(x, tok)  # not None: cv1's backward finishes the shortcut's input gradient (functional._defer_finish)
        if tok is not None and SF.FUSE_SHORTCUT[0] and getattr(self.cv2, "takes_shortcut", lambda: False)():
            # alpha * x joins cv2's own apply pass (one launch and two tensor passes fewer than a scale_add after it); cv2's backward
            # parks the shortcut's gradient for cv1's backward exactly as _ScaledAdd would
            return self.cv2(h, shortcut=(x, self.alpha, tok))
        y = self.cv2(h)
        if not self.add:
            return y
        if learnable:
            return _ScaledAdd.apply(x, y, self.alpha, tok)
        return SF.add(x, y, self.alpha, 1.0)


class _ScaledAdd(torch.autograd.Function):
    """alpha * x + y with a learnable scalar alpha read on the device (yolo_stages.py:61-63)."""

    @staticmethod
    def forward(ctx, x, y, alpha, defer=None):
        from ..... import kernels as K

        x, y = K.as_nhwc(x), K.as_nhwc(y)
        ctx.save_for_backward(x, alpha)
        ctx.slot = getattr(alpha, "main_grad", None)
        ctx.defer = defer if ctx.slot is not None else None
        return K.scale_add(x, alpha, y)

    @staticmethod
    def backward(ctx, dy):
        from ..... import kernels as K

        x, alpha = ctx.saved_tensors
        dy = K.as_nhwc(dy)
        if ctx.defer is not None:
            # the block that consumes x (cv1) adds alpha * dy into its own input gradient and accumulates d(alpha) in ONE pass after its
            # dgrad: no gradient tensor for x from here, no ATen add afterwards
            ctx.defer.pending = (dy, alpha, x, ctx.slot)
            return None, dy, None, None
        dx, dot = K.scale_add_dot(dy, alpha, x)  # alpha * dy and sum(dy * x) in one pass over dy
        dalpha = dot.sum().float().reshape(1)
        if ctx.slot is not None:
            ctx.slot.add_(dalpha)
            dalpha = None
        return dx, dy, dalpha, None


class SequentialWithIntermediates(nn.Sequential):
    def __init__(self, output_intermediates: bool, *args):
        super().__init__(*args)
        self.output_intermediates = output_intermediates

    def forward(self, input: Tensor) -> List[Tensor]:
        if self.output_intermediates:
            output = [input]
            for module in self:
                output.append(module(output[-1]))
            return output
        return [super().forward(input)]


class YoloNASCSPLayer(nn.Module):
    def __init__(
        self,
        in_channels: int,
        out_channels: int,
        num_bottlenecks: int,
        block_type: Type[nn.Module],
        activation_type: Type[nn.Module],
        shortcut: bool = True,
        use_alpha: bool = True,
        expansion: float = 0.5,
        hidden_channels: int = None,
        concat_intermediates: bool = False,
        drop_path_rates: Union[Iterable[float], None] = None,
        dropout_rate: float = 0.0,
    ):
        drop_path_rates = [0.0] * num_bottlenecks if drop_path_rates is None else tuple(drop_path_rates)
        if len(drop_path_rates) != num_bottlenecks:
            raise ValueError(f"Argument drop_path_rates ({drop_path_rates}, len {len(drop_path_rates)} must have the length equal to the num_bottlenecks ({num_bottlenecks}).")
        if dropout_rate > 0.0:
            raise NotImplementedError("dropout_rate > 0 is not used by the shipped YOLO-NAS recipes and is not implemented")
        super().__init__()
        if hidden_channels is None:
            hidden_channels = int(out_channels * expansion)
        self.conv1 = Conv(in_channels, hidden_channels, 1, stride=1, activation_type=activation_type)
        self.conv2 = Conv(in_channels, hidden_channels, 1, stride=1, activation_type=activation_type)
        self.conv3 = Conv(hidden_channels * (2 + concat_intermediates * num_bottlenecks), out_channels, 1, stride=1, activation_type=activation_type)
        module_list = [YoloNASBottleneck(hidden_channels, hidden_channels, block_type, activation_type, shortcut, use_alpha, drop_path_rate=drop_path_rates[i]) for i in range(num_bottlenecks)]
        self.bottlenecks = SequentialWithIntermediates(concat_intermediates, *module_list)
        self.dropout = nn.Identity()
        self._cache12 = SF.WeightCache()

    def sgb_adjacent_tensors(self):
        """conv1 and conv2 read the same tensor: in training they run as ONE GEMM + ONE BatchNorm launch over the concatenated channels
        (functional.dual_conv_bn_act), which needs the pair's BatchNorm parameters / statistics back to back in the flat buffers."""
        b1, b2 = self.conv1.bn, self.conv2.bn
        return [[b1.weight, b2.weight], [b1.bias, b2.bias], [b1.running_mean, b2.running_mean], [b1.running_var, b2.running_var]]

    def forward(self, x: Tensor) -> Tensor:
        if self.training and SF.dual_conv_bn_act_ready(self.conv1.conv, self.conv1.bn, self.conv2.conv, self.conv2.bn):
            h1, x_2 = SF.dual_conv_bn_act(x, self.conv1.conv, self.conv1.bn, self.conv2.conv, self.conv2.bn, act=self.conv1._act_code, cache=self._cache12)
            x_1 = self.bottlenecks(h1)
        else:
            x_1 = self.bottlenecks(self.conv1(x))
            x_2 = self.conv2(x)
        return self.conv3(SF.concat([*x_1, x_2]))


@register_detection_module()
class YoloNASStem(BaseDetectionModule):
    def __init__(self, in_channels: int, out_channels: int, stride: int = 2):
        super().__init__(in_channels)
        self._out_channels = out_channels
        self.conv = QARepVGGBlock(in_channels, out_channels, stride=stride, use_residual_connection=False)

    @property
    def out_channels(self):
        return self._out_channels

    def forward(self, x: Tensor) -> Tensor:
        return self.conv(x)

    def replace_input_channels(self, in_channels: int, compute_new_weights_fn=None):
        """A fresh QARepVGG block, as the reference does (yolo_stages.py:176-177): a three-branch block has no single filter to cut."""
        old = self.conv
        self.conv = QARepVGGBlock(in_channels, self._out_channels, stride=2, use_residual_connection=False)
        self.conv.to(next(old.parameters()).device)

    def get_input_channels(self) -> int:
        return self.conv.in_channels


@register_detection_module()
class YoloNASStage(BaseDetectionModule):
    def __init__(self, in_channels: int, out_channels: int, num_blocks: int, activation_type, hidden_channels: int = None, concat_intermediates: bool = False, drop_path_rates=None, dropout_rate: float = 0.0, stride: int = 2):
        super().__init__(in_channels)
        activation_type = resolve_activation(activation_type)
        self._out_channels = out_channels
        self.downsample = QARepVGGBlock(in_channels, out_channels, stride=stride, activation_type=activation_type, use_residual_connection=False)
        self.blocks = YoloNASCSPLayer(out_channels, out_channels, num_blocks, QARepVGGBlock, activation_type, True, hidden_channels=hidden_channels, concat_intermediates=concat_intermediates, drop_path_rates=drop_path_rates, dropout_rate=dropout_rate)

    @property
    def out_channels(self):
        return self._out_channels

    def forward(self, x):
        return self.blocks(self.downsample(x))


@register_detection_module()
class YoloNASUpStage(BaseDetectionModule):
    def __init__(
        self,
        in_channels: List[int],
        out_channels: int,
        width_mult: float,
        num_blocks: int,
        depth_mult: float,
        activation_type,
        hidden_channels: int = None,
        concat_intermediates: bool = False,
        reduce_channels: bool = False,
        drop_path_rates=None,
        dropout_rate: float = 0.0,
        upsample_mode="conv_transpose",
    ):
        super().__init__(in_channels)
        activation_type = resolve_activation(activation_type)
        num_inputs = len(in_channels)
        if num_inputs == 2:
            in_channels, skip_in_channels = in_channels
        else:
            in_channels, skip_in_channels1, skip_in_channels2 = in_channels
            skip_in_channels = skip_in_channels1 + out_channels
        out_channels = width_multiplier(out_channels, width_mult, 8)
        num_blocks = max(round(num_blocks * depth_mult), 1) if num_blocks > 1 else num_blocks
        if num_inputs == 2:
            self.reduce_skip = Conv(skip_in_channels, out_channels, 1, 1, activation_type) if reduce_channels else nn.Identity()
        else:
            self.reduce_skip1 = Conv(skip_in_channels1, out_channels, 1, 1, activation_type) if reduce_channels else nn.Identity()
            self.reduce_skip2 = Conv(skip_in_channels2, out_channels, 1, 1, activation_type) if reduce_channels else nn.Identity()
        self.conv = Conv(in_channels, out_channels, 1, 1, activation_type)
        self.upsample = make_upsample_module_with_explicit_channels(in_channels=out_channels, out_channels=out_channels, scale_factor=2, upsample_mode=upsample_mode, align_corners=True)
        if num_inputs == 3:
            self.downsample = Conv(out_channels if reduce_channels else skip_in_channels2, out_channels, kernel=3, stride=2, activation_type=activation_type)
        self.reduce_after_concat = Conv(num_inputs * out_channels, out_channels, 1, 1, activation_type) if reduce_channels else nn.Identity()
        after_concat_channels = out_channels if reduce_channels else out_channels + skip_in_channels
        self.blocks = YoloNASCSPLayer(after_concat_channels, out_channels, num_blocks, QARepVGGBlock, activation_type, hidden_channels=hidden_channels, concat_intermediates=concat_intermediates, drop_path_rates=drop_path_rates, dropout_rate=dropout_rate)
        self._out_channels = [out_channels, out_channels]

    @property
    def out_channels(self):
        return self._out_channels

    def forward(self, inputs):
        if len(inputs) == 2:
            x, skip_x = inputs
            skip_x = [self.reduce_skip(skip_x)]
        else:
            x, skip_x1, skip_x2 = inputs
            skip_x1, skip_x2 = self.reduce_skip1(skip_x1), self.reduce_skip2(skip_x2)
            skip_x = [skip_x1, self.downsample(skip_x2)]
        x_inter = self.conv(x)
        x = self.upsample(x_inter)
        x = SF.concat([x, *skip_x])
        x = self.reduce_after_concat(x)
        x = self.blocks(x)
        return x_inter, x


@register_detection_module()
class YoloNASDownStage(BaseDetectionModule):
    def __init__(self, in_channels: List[int], out_channels: int, width_mult: float, num_blocks: int, depth_mult: float, activation_type, hidden_channels: int = None, concat_intermediates: bool = False, drop_path_rates=None, dropout_rate: float = 0.0):
        super().__init__(in_channels)
        activation_type = resolve_activation(activation_type)
        in_channels, skip_in_channels = in_channels
        out_channels = width_multiplier(out_channels, width_mult, 8)
        num_blocks = max(round(num_blocks * depth_mult), 1) if num_blocks > 1 else num_blocks
        self.conv = Conv(in_channels, out_channels // 2, 3, 2, activation_type)
        after_concat_channels = out_channels // 2 + skip_in_channels
        self.blocks = YoloNASCSPLayer(in_channels=after_concat_channels, out_channels=out_channels, num_bottlenecks=num_blocks, block_type=partial(Conv, kernel=3, stride=1), activation_type=activation_type, hidden_channels=hidden_channels, concat_intermediates=concat_intermediates, drop_path_rates=drop_path_rates, dropout_rate=dropout_rate)
        self._out_channels = out_channels

    @property
    def out_channels(self):
        return self._out_channels

    def forward(self, inputs):
        x, skip_x = inputs
        x = self.conv(x)
        x = SF.concat([x, skip_x])
        return self.blocks(x)
