"""YoloNASDFLHead / NDFLHeads with the reference's names, signatures and state-dict keys
(training/models/detection_models/yolo_nas/dfl_heads.py).  The per-level convs are fused GEMMs; the softmax-integral
decode, sigmoid, anchor arithmetic and the [B, L, *] concatenation are ONE kernel per level (functional.dfl_decode)."""
import math
from typing import List, Optional, Tuple

import torch
from torch import Tensor, nn

from ..... import functional as SF
from .....common.factories import DetectionModulesFactory
from .....common.registry import register_detection_module
from .....modules import BaseDetectionModule, ConvBNReLU
from .....modules.utils import width_multiplier


@register_detection_module()
class YoloNASDFLHead(BaseDetectionModule):
    def __init__(self, in_channels: int, inter_channels: int, width_mult: float, first_conv_group_size: int, num_classes: int, stride: int, reg_max: int, cls_dropout_rate: float = 0.0, reg_dropout_rate: float = 0.0):
        super().__init__(in_channels)
        inter_channels = width_multiplier(inter_channels, width_mult, 8)
        if first_conv_group_size == 0:
            groups = 0
        elif first_conv_group_size == -1:
            groups = 1
        else:
            groups = inter_channels // first_conv_group_size
        if cls_dropout_rate > 0 or reg_dropout_rate > 0:
            raise NotImplementedError("head dropout is not used by the shipped YOLO-NAS recipes and is not implemented")
        self.num_classes = num_classes
        self.stem = ConvBNReLU(in_channels, inter_channels, kernel_size=1, stride=1, padding=0, bias=False)
        first_cls_conv = [ConvBNReLU(inter_channels, inter_channels, kernel_size=3, stride=1, padding=1, groups=groups, bias=False)] if groups else []
        self.cls_convs = nn.Sequential(*first_cls_conv, ConvBNReLU(inter_channels, inter_channels, kernel_size=3, stride=1, padding=1, bias=False))
        first_reg_conv = [ConvBNReLU(inter_channels, inter_channels, kernel_size=3, stride=1, padding=1, groups=groups, bias=False)] if groups else []
        self.reg_convs = nn.Sequential(*first_reg_conv, ConvBNReLU(inter_channels, inter_channels, kernel_size=3, stride=1, padding=1, bias=False))
        self.cls_pred = nn.Conv2d(inter_channels, self.num_classes, 1, 1, 0)
        self.reg_pred = nn.Conv2d(inter_channels, 4 * (reg_max + 1), 1, 1, 0)
        self.cls_dropout_rate = nn.Identity()
        self.reg_dropout_rate = nn.Identity()
        self.grid = torch.zeros(1)
        self.stride = stride
        self.prior_prob = 1e-2
        self._initialize_biases()
        self._cls_cache, self._reg_cache = SF.WeightCache(), SF.WeightCache()
        self._cache_pair = SF.WeightCache()

    def _first_pair(self):
        """The first cls / reg convolutions read the same tensor (the stem's output; training/models/detection_models/yolo_nas/dfl_heads.py:86-92
        of the reference): candidates for ONE GEMM (functional.dual_conv_bn_act)."""
        a, b = self.cls_convs[0], self.reg_convs[0]
        ok = all(hasattr(m.seq, "bn") and m.seq.conv.bias is None and m.seq.conv.groups == 1 and m._act_code == a._act_code for m in (a, b))
        return (a, b) if ok else None

    def sgb_adjacent_tensors(self):
        pair = self._first_pair()
        if pair is None:
            return []
        b1, b2 = pair[0].seq.bn, pair[1].seq.bn
        return [[b1.weight, b2.weight], [b1.bias, b2.bias], [b1.running_mean, b2.running_mean], [b1.running_var, b2.running_var]]

    def replace_num_classes(self, num_classes: int, compute_new_weights_fn=None):
        old = self.cls_pred
        self.cls_pred = nn.Conv2d(old.in_channels, num_classes, 1, 1, 0).to(old.weight.device)
        self.num_classes = num_classes
        self._initialize_biases()
        self._cls_cache = SF.WeightCache()

    @property
    def out_channels(self):
        return None

    def forward(self, x):
        """Returns (reg_output, cls_output) as bf16 NHWC maps [B, 4*(reg_max+1), H, W], [B, num_classes, H, W]."""
        x = self.stem(x)
        pair = self._first_pair() if self.training else None
        if pair is not None and SF.dual_conv_bn_act_ready(pair[0].seq.conv, pair[0].seq.bn, pair[1].seq.conv, pair[1].seq.bn):
            cls_feat, reg_feat = SF.dual_conv_bn_act(x, pair[0].seq.conv, pair[0].seq.bn, pair[1].seq.conv, pair[1].seq.bn, act=pair[0]._act_code, cache=self._cache_pair)
            for m in list(self.cls_convs)[1:]:
                cls_feat = m(cls_feat)
            for m in list(self.reg_convs)[1:]:
                reg_feat = m(reg_feat)
        else:
            cls_feat, reg_feat = self.cls_convs(x), None
        cls_output = SF.conv_bias(cls_feat, self.cls_pred.weight, self.cls_pred.bias, stride=1, pad=0, cache=self._cls_cache)
        if reg_feat is None:
            reg_feat = self.reg_convs(x)
        reg_output = SF.conv_bias(reg_feat, self.reg_pred.weight, self.reg_pred.bias, stride=1, pad=0, cache=self._reg_cache)
        return reg_output, cls_output

    def _initialize_biases(self):
        prior_bias = -math.log((1 - self.prior_prob) / self.prior_prob)
        torch.nn.init.constant_(self.cls_pred.bias, prior_bias)


def generate_anchors_for_grid_cell(shapes, fpn_strides, grid_cell_size: float = 5.0, grid_cell_offset: float = 0.5, device="cpu"):
    """anchors [L,4], anchor_points [L,2] (pixels), num_anchors_list, stride_tensor [L,1]
    (reference: pp_yolo_e/pp_yolo_head.py:21-76).  Tiny; cached per feature-map geometry instead of being rebuilt on
    the host every forward."""
    anchors, anchor_points, num_anchors_list, stride_tensor = [], [], [], []
    for (h, w), stride in zip(shapes, fpn_strides):
        cell_half_size = grid_cell_size * stride * 0.5
        shift_x = (torch.arange(end=w) + grid_cell_offset) * stride
        shift_y = (torch.arange(end=h) + grid_cell_offset) * stride
        shift_y, shift_x = torch.meshgrid(shift_y, shift_x, indexing="ij")
        anchor = torch.stack([shift_x - cell_half_size, shift_y - cell_half_size, shift_x + cell_half_size, shift_y + cell_half_size], dim=-1).to(dtype=torch.float)
        anchor_point = torch.stack([shift_x, shift_y], dim=-1).to(dtype=torch.float)
        anchors.append(anchor.reshape([-1, 4]))
        anchor_points.append(anchor_point.reshape([-1, 2]))
        num_anchors_list.append(len(anchors[-1]))
        stride_tensor.append(torch.full([num_anchors_list[-1], 1], stride, dtype=torch.float))
    return torch.cat(anchors).to(device), torch.cat(anchor_points).to(device), num_anchors_list, torch.cat(stride_tensor).to(device)


@register_detection_module()
class NDFLHeads(BaseDetectionModule):
    def __init__(self, num_classes: int, in_channels: Tuple[int, int, int], heads_list, grid_cell_scale: float = 5.0, grid_cell_offset: float = 0.5, reg_max: int = 16, eval_size: Optional[Tuple[int, int]] = None, width_mult: float = 1.0):
        super().__init__(in_channels)
        in_channels = [max(round(c * width_mult), 1) for c in in_channels]
        self.in_channels = tuple(in_channels)
        self.num_classes = num_classes
        self.grid_cell_scale = grid_cell_scale
        self.grid_cell_offset = grid_cell_offset
        self.reg_max = reg_max
        self.eval_size = eval_size
        proj = torch.linspace(0, self.reg_max, self.reg_max + 1).reshape([1, self.reg_max + 1, 1, 1])
        self.register_buffer("proj_conv", proj, persistent=False)
        factory = DetectionModulesFactory()
        for i in range(len(heads_list)):
            heads_list[i] = factory.insert_module_param(heads_list[i], "num_classes", num_classes)
            heads_list[i] = factory.insert_module_param(heads_list[i], "reg_max", reg_max)
        self.num_heads = len(heads_list)
        fpn_strides: List[int] = []
        for i in range(self.num_heads):
            new_head = factory.get(factory.insert_module_param(heads_list[i], "in_channels", in_channels[i]))
            fpn_strides.append(new_head.stride)
            setattr(self, f"head{i + 1}", new_head)
        self.fpn_strides = tuple(fpn_strides)
        self._anchor_cache = {}

    def replace_num_classes(self, num_classes: int, compute_new_weights_fn=None):
        for i in range(self.num_heads):
            getattr(self, f"head{i + 1}").replace_num_classes(num_classes, compute_new_weights_fn)
        self.num_classes = num_classes

    @property
    def out_channels(self):
        return None

    def _anchors(self, shapes, device):
        key = (tuple(shapes), str(device))
        if key not in self._anchor_cache:
            self._anchor_cache[key] = generate_anchors_for_grid_cell(shapes, self.fpn_strides, self.grid_cell_scale, self.grid_cell_offset, device)
        return self._anchor_cache[key]

    def forward(self, feats: Tuple[Tensor, ...]):
        feats = feats[: self.num_heads]
        regs, clss = [], []
        for i, feat in enumerate(feats):
            reg_distri, cls_logit = getattr(self, f"head{i + 1}")(feat)
            regs.append(reg_distri)
            clss.append(cls_logit)
        pred_bboxes, pred_scores, cls_score_list, reg_distri_list = SF.dfl_decode(regs, clss, self.fpn_strides, self.num_classes, self.reg_max, self.grid_cell_offset)
        decoded_predictions = pred_bboxes, pred_scores
        shapes = [(f.shape[2], f.shape[3]) for f in feats]
        anchors, anchor_points, num_anchors_list, stride_tensor = self._anchors(shapes, pred_bboxes.device)
        raw_predictions = cls_score_list, reg_distri_list, anchors, anchor_points, num_anchors_list, stride_tensor
        return decoded_predictions, raw_predictions
