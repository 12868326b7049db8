"""ResNet / CifarResNet with the reference's constructors and state-dict keys
(training/models/classification_models/resnet.py:26-379).  Every conv-bn(-add)-relu group is one fused call:
GEMM with fused batch statistics + one normalise/add/ReLU pass (training) or a single GEMM (inference)."""
from typing import Dict

import torch
import torch.nn as nn

from .... import functional as SF
from ....common.registry import register_model
from ....modules.conv_bn_act_block import _FusedConvBN
from ....modules.utils import width_multiplier
from ...utils import get_param
from ...utils.regularization_utils import DropPath
from ..sg_module import SgModule


class _Block(nn.Module, _FusedConvBN):
    def _init_caches(self, n):
        self._caches = [SF.WeightCache() for _ in range(n)]

    def _shortcut(self, x):
        if len(self.shortcut) == 0:
            return x
        return self._fused(x, self.shortcut[0], self.shortcut[1], "none", self._caches[-1])


class BasicResNetBlock(_Block):
    def __init__(self, in_planes, planes, stride=1, expansion=1, final_relu=True, droppath_prob=0.0):
        super().__init__()
        self.expansion = expansion
        self.conv1 = nn.Conv2d(in_planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.final_relu = final_relu
        self.drop_path = DropPath(drop_prob=droppath_prob)  # draws the per-image mask; the multiply runs inside the fused bn + add kernel
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != self.expansion * planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, self.expansion * planes, kernel_size=1, stride=stride, bias=False), nn.BatchNorm2d(self.expansion * planes))
        self._init_caches(3)

    def forward(self, x):
        out = self._fused(x, self.conv1, self.bn1, "relu", self._caches[0])
        return self._fused(out, self.conv2, self.bn2, "relu" if self.final_relu else "none", self._caches[1], residual=self._shortcut(x), sample_scale=self.drop_path.sample_scale(x))


class Bottleneck(_Block):
    def __init__(self, in_planes, planes, stride=1, expansion=4, final_relu=True, droppath_prob=0.0):
        super().__init__()
        self.expansion = expansion
        self.conv1 = nn.Conv2d(in_planes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, self.expansion * planes, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(self.expansion * planes)
        self.final_relu = final_relu
        self.drop_path = DropPath(drop_prob=droppath_prob)  # draws the per-image mask; the multiply runs inside the fused bn + add kernel
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != self.expansion * planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, self.expansion * planes, kernel_size=1, stride=stride, bias=False), nn.BatchNorm2d(self.expansion * planes))
        self._init_caches(4)

    def forward(self, x):
        out = self._fused(x, self.conv1, self.bn1, "relu", self._caches[0])
        out = self._fused(out, self.conv2, self.bn2, "relu", self._caches[1])
        return self._fused(out, self.conv3, self.bn3, "relu" if self.final_relu else "none", self._caches[2], residual=self._shortcut(x), sample_scale=self.drop_path.sample_scale(x))


class _Classifier(SgModule, _FusedConvBN):
    def _head(self, out):
        """avgpool -> Linear (as a 1x1 GEMM) -> fp32 logits [N, num_classes]."""
        out = SF.global_avg_pool(out)
        logits = SF.conv_bias(out, self.linear.weight, self.linear.bias, stride=1, pad=0, cache=self._fc_cache)  # [K, C] == OIHW [K, C, 1, 1]
        return SF.from_nhwc(logits).flatten(1)

    def _make_layer(self, block, planes, num_blocks, stride, droppath_prob=0.0):
        strides = [stride] + [1] * (num_blocks - 1)
        layers = []
        if num_blocks == 0:
            raise NotImplementedError("zero-block stages are not implemented")
        for stride in strides:
            kw = {"droppath_prob": droppath_prob} if droppath_prob else {}
            layers.append(block(self.in_planes, planes, stride, **kw))
            self.in_planes = planes * self.expansion
        return nn.Sequential(*layers)

    def replace_input_channels(self, in_channels: int, compute_new_weights_fn=None):
        """resnet.py:249-255."""
        from ....modules.weight_replacement_utils import replace_conv2d_input_channels

        self.conv1 = replace_conv2d_input_channels(conv=self.conv1, in_channels=in_channels, fn=compute_new_weights_fn)

    def get_input_channels(self) -> int:
        return self.conv1.in_channels

    def get_finetune_lr_dict(self, lr: float) -> Dict[str, float]:
        return {"linear": lr, "default": 0}


class CifarResNet(_Classifier):
    def __init__(self, block, num_blocks, num_classes=10, width_mult=1, expansion=1, in_channels: int = 3):
        super().__init__()
        self.expansion = expansion
        self.structure = [num_blocks, width_mult]
        self.in_planes = width_multiplier(64, width_mult)
        self.conv1 = nn.Conv2d(in_channels, width_multiplier(64, width_mult), kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(width_multiplier(64, width_mult))
        self.layer1 = self._make_layer(block, width_multiplier(64, width_mult), num_blocks[0], stride=1)
        self.layer2 = self._make_layer(block, width_multiplier(128, width_mult), num_blocks[1], stride=2)
        self.layer3 = self._make_layer(block, width_multiplier(256, width_mult), num_blocks[2], stride=2)
        self.layer4 = self._make_layer(block, width_multiplier(512, width_mult), num_blocks[3], stride=2)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.linear = nn.Linear(width_multiplier(512, width_mult) * self.expansion, num_classes)
        self._stem_cache, self._fc_cache = SF.WeightCache(), SF.WeightCache()

    def forward(self, x):
        x = SF.to_nhwc(x)
        out = self._fused(x, self.conv1, self.bn1, "relu", self._stem_cache)
        out = self.layer4(self.layer3(self.layer2(self.layer1(out))))
        return self._head(out)


class ResNet(_Classifier):
    def __init__(self, block, num_blocks: list, num_classes: int = 10, width_mult: float = 1, expansion: int = 1, droppath_prob=0.0, input_batchnorm: bool = False, backbone_mode: bool = False, in_channels: int = 3):
        super().__init__()
        if input_batchnorm or backbone_mode:
            raise NotImplementedError("input_batchnorm / backbone_mode are not implemented on the fused path")
        self.expansion = expansion
        self.backbone_mode = backbone_mode
        self.structure = [num_blocks, width_mult]
        self.in_planes = width_multiplier(64, width_mult)
        self.input_batchnorm = input_batchnorm
        self.conv1 = nn.Conv2d(in_channels, width_multiplier(64, width_mult), kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(width_multiplier(64, width_mult))
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, width_multiplier(64, width_mult), num_blocks[0], stride=1, droppath_prob=droppath_prob)
        self.layer2 = self._make_layer(block, width_multiplier(128, width_mult), num_blocks[1], stride=2, droppath_prob=droppath_prob)
        self.layer3 = self._make_layer(block, width_multiplier(256, width_mult), num_blocks[2], stride=2, droppath_prob=droppath_prob)
        self.layer4 = self._make_layer(block, width_multiplier(512, width_mult), num_blocks[3], stride=2, droppath_prob=droppath_prob)
        self.linear = nn.Linear(width_multiplier(512, width_mult) * self.expansion, num_classes)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.width_mult = width_mult
        self._stem_cache, self._fc_cache = SF.WeightCache(), SF.WeightCache()
        self._stem_patch_cache = SF.StagedWeightCache()

    def forward(self, x):
        if SF.conv_stem_patches_supported(self.conv1, self.bn1, x, self.training and self.bn1.training):
            out = SF.conv_bn_act_stem(x, self.conv1, self.bn1, act="relu", cache=self._stem_patch_cache)  # 7x7 / s2 as a 1x1 GEMM over patches
        else:
            x = SF.to_nhwc(x)
            out = self._fused(x, self.conv1, self.bn1, "relu", self._stem_cache)
        out = SF.max_pool(out, 3, 2, 1)
        out = self.layer4(self.layer3(self.layer2(self.layer1(out))))
        return self._head(out)

    def replace_head(self, new_num_classes=None, new_head=None):
        if new_num_classes is None and new_head is None:
            raise ValueError("At least one of new_num_classes, new_head must be given to replace output layer.")
        self.linear = new_head if new_head is not None else nn.Linear(width_multiplier(512, self.width_mult) * self.expansion, new_num_classes)
        self._fc_cache = SF.WeightCache()


def _nc(arch_params, num_classes):
    return num_classes or get_param(arch_params, "num_classes", None)


@register_model("resnet18")
class ResNet18(ResNet):
    def __init__(self, arch_params, num_classes=None):
        super().__init__(BasicResNetBlock, [2, 2, 2, 2], num_classes=_nc(arch_params, num_classes), droppath_prob=get_param(arch_params, "droppath_prob", 0), backbone_mode=get_param(arch_params, "backbone_mode", False))


@register_model("resnet18_cifar")
class ResNet18Cifar(CifarResNet):
    def __init__(self, arch_params, num_classes=None):
        super().__init__(BasicResNetBlock, [2, 2, 2, 2], num_classes=_nc(arch_params, num_classes))


@register_model("resnet34")
class ResNet34(ResNet):
    def __init__(self, arch_params, num_classes=None):
        super().__init__(BasicResNetBlock, [3, 4, 6, 3], num_classes=_nc(arch_params, num_classes), droppath_prob=get_param(arch_params, "droppath_prob", 0), backbone_mode=get_param(arch_params, "backbone_mode", False))


@register_model("resnet50")
class ResNet50(ResNet):
    def __init__(self, arch_params, num_classes=None):
        super().__init__(Bottleneck, [3, 4, 6, 3], num_classes=_nc(arch_params, num_classes), droppath_prob=get_param(arch_params, "droppath_prob", 0), backbone_mode=get_param(arch_params, "backbone_mode", False), expansion=4)


@register_model("resnet101")
class ResNet101(ResNet):
    def __init__(self, arch_params, num_classes=None):
        super().__init__(Bottleneck, [3, 4, 23, 3], num_classes=_nc(arch_params, num_classes), droppath_prob=get_param(arch_params, "droppath_prob", 0), backbone_mode=get_param(arch_params, "backbone_mode", False), expansion=4)
