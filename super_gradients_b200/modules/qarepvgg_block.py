"""QARepVGGBlock with the reference's constructor, sub-module names and state-dict keys
(modules/qarepvgg_block.py:10-338).  Train mode runs the fused branch algebra (functional._QARepVGG); eval /
fused modes run ONE 3x3 GEMM with the re-parameterised kernel and post_bn folded into its epilogue."""
from types import SimpleNamespace
from typing import Any, Mapping, Optional, Type, Union

import torch
from torch import nn

from .. import functional as SF
from .. import kernels as K
from ..common.factories import activation_code
from .skip_connections import Residual


class QARepVGGBlock(nn.Module):
    def __init__(
        self,
        in_channels: int,
        out_channels: int,
        stride: int = 1,
        dilation: int = 1,
        groups: int = 1,
        activation_type: Type[nn.Module] = nn.ReLU,
        activation_kwargs: Union[Mapping[str, Any], None] = None,
        se_type: Type[nn.Module] = nn.Identity,
        se_kwargs: Union[Mapping[str, Any], None] = None,
        build_residual_branches: bool = True,
        use_residual_connection: bool = True,
        use_alpha: bool = False,
        use_1x1_bias: bool = True,
        use_post_bn: bool = True,
    ):
        super().__init__()
        if groups != 1 or dilation != 1:
            raise NotImplementedError("QARepVGGBlock: groups/dilation != 1 have no sm_90a kernel")
        if se_type is not nn.Identity:
            raise NotImplementedError("QARepVGGBlock: SE blocks are not on the YOLO-NAS path (se_type must be nn.Identity)")
        activation_kwargs = activation_kwargs or {}
        self.groups, self.in_channels, self.out_channels = groups, in_channels, out_channels
        self.stride, self.dilation = stride, dilation
        self.activation_type, self.activation_kwargs = activation_type, activation_kwargs
        self.se_type, self.se_kwargs = se_type, se_kwargs or {}
        self.use_residual_connection, self.use_alpha = use_residual_connection, use_alpha
        self.use_1x1_bias, self.use_post_bn = use_1x1_bias, use_post_bn

        self.nonlinearity = activation_type(**activation_kwargs)
        self.se = se_type(**self.se_kwargs)
        self._act_code = activation_code(activation_type)

        self.branch_3x3 = nn.Sequential()
        self.branch_3x3.add_module("conv", nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=stride, padding=dilation, groups=groups, bias=False, dilation=dilation))
        self.branch_3x3.add_module("bn", nn.BatchNorm2d(num_features=out_channels))
        self.branch_1x1 = nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=stride, padding=0, groups=groups, bias=use_1x1_bias)

        if use_residual_connection:
            assert out_channels == in_channels and stride == 1
            self.identity = Residual()
            id_tensor = torch.zeros((in_channels, in_channels // groups, 3, 3))
            for i in range(in_channels):
                id_tensor[i, i % (in_channels // groups), 1, 1] = 1.0
            self.register_buffer("id_tensor", id_tensor, persistent=False)
        else:
            self.identity = None

        if use_alpha:
            noise = torch.randn((1,)) * 0.01
            self.alpha = torch.nn.Parameter(torch.tensor([1.0]) + noise, requires_grad=True)
        else:
            self.alpha = 1.0

        self.post_bn = nn.BatchNorm2d(num_features=out_channels) if use_post_bn else nn.Identity()

        # placeholder kept for checkpoint compatibility (never receives a gradient, SURVEY.md D7)
        self.rbr_reparam = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=stride, padding=dilation, dilation=dilation, groups=groups, bias=True)

        self.partially_fused = False
        self.fully_fused = False
        self._cache3, self._cache1, self._cache_eq = SF.WeightCache(), SF.WeightCache(), SF.WeightCache()
        self._cache_fold = SF.WeightCache()
        self._cache_stem = SF.StagedWeightCache()
        self._eq = None
        self._eval_fold = None  # (key, bf16 KRSC filter, scale, shift) of the on-the-fly eval fold
        if not build_residual_branches:
            self.fuse_block_residual_branches()

    # ------------------------------------------------------------------------------------------------ forward
    def takes_shortcut(self) -> bool:
        """True when forward(inputs, shortcut=...) can add a caller's `alpha * x` in its own apply pass (the unfused train-mode path)."""
        return self.training and not self.fully_fused and not self.partially_fused and self.in_channels % 8 == 0

    def forward(self, inputs, shortcut=None):
        K.require_cuda(inputs, "inputs")
        if shortcut is not None and not self.takes_shortcut():
            raise RuntimeError("QARepVGGBlock: a fused shortcut needs the train-mode branch path (takes_shortcut())")
        if self.fully_fused:
            return SF.conv_bias(inputs, self.rbr_reparam.weight, self.rbr_reparam.bias, stride=self.stride, pad=1, cache=self._cache_eq, act=self._act_code)
        if self.partially_fused:
            return self._forward_single_conv(inputs, self.rbr_reparam.weight, self.rbr_reparam.bias)
        if self.training:
            bn3 = self.branch_3x3.bn
            pbn = self.post_bn if self.use_post_bn else None
            if SF.stem_patches_supported(self, inputs):  # a raw fp32 image entering a first layer (the detector passes it through)
                cfg = SimpleNamespace(
                    stride=self.stride, act=self._act_code, eps=bn3.eps, momentum=0.1 if bn3.momentum is None else bn3.momentum, cache_stem=self._cache_stem,
                    rm3=bn3.running_mean, rv3=bn3.running_var, rmp=pbn.running_mean, rvp=pbn.running_var, nbt=(bn3.num_batches_tracked, pbn.num_batches_tracked),
                    sync=self._bn_sync(bn3, pbn),
                )  # fmt: skip
                if pbn.eps != bn3.eps:
                    raise NotImplementedError("branch and post BatchNorm must share eps")
                return SF.qarepvgg_stem_block(inputs, self.branch_3x3.conv.weight, bn3.weight, bn3.bias, self.branch_1x1.weight, self.branch_1x1.bias, pbn.weight, pbn.bias, cfg)
            if inputs.dtype == torch.float32 and inputs.shape[1] == self.in_channels and self.in_channels % 8 != 0:
                inputs = SF.to_nhwc(inputs)  # a raw image the patch path does not serve
            cfg = SimpleNamespace(
                stride=self.stride, residual=self.identity is not None, act=self._act_code, eps=bn3.eps, momentum=0.1 if bn3.momentum is None else bn3.momentum,
                use_post_bn=self.use_post_bn, cache3=self._cache3, cache1=self._cache1, cache_fold=self._cache_fold, rm3=bn3.running_mean, rv3=bn3.running_var,
                rmp=pbn.running_mean if pbn is not None else None, rvp=pbn.running_var if pbn is not None else None,
                nbt=(bn3.num_batches_tracked, pbn.num_batches_tracked if pbn is not None else None), sync=self._bn_sync(bn3, pbn), shortcut=shortcut,
            )  # fmt: skip
            if pbn is not None and pbn.eps != bn3.eps:
                raise NotImplementedError("branch and post BatchNorm must share eps")
            alpha = self.alpha if isinstance(self.alpha, torch.Tensor) else None
            return SF.qarepvgg_block(
                inputs, self.branch_3x3.conv.weight, bn3.weight, bn3.bias, self.branch_1x1.weight, self.branch_1x1.bias, alpha,
                pbn.weight if pbn is not None else None, pbn.bias if pbn is not None else None, cfg,
            )  # fmt: skip
        # eval with branches: fold them (numerically the reference's partial fusion, max abs err ~5e-6).  The folded bf16 filter
        # and the post_bn scale / shift are kept until one of their SOURCE tensors changes, so a steady-state inference forward of
        # the block is exactly one GEMM launch (predict() on an unfused model costs what the reference's fused model costs).
        with torch.no_grad():
            x = K.as_nhwc(inputs)
            key = (self._eval_source_key(), x.shape[1], SF.weight_epoch())
            if self._eval_fold is None or self._eval_fold[0] != key:
                k, b = self._get_equivalent_kernel_bias_for_branches()
                krsc, _ = K.weight_prepare(k, c_pad=x.shape[1], want_crsk=False)
                if self.use_post_bn:
                    pbn = self.post_bn
                    scale = pbn.weight * torch.rsqrt(pbn.running_var + pbn.eps)
                    shift = pbn.bias - pbn.running_mean * scale + b * scale
                else:
                    scale, shift = None, b
                self._eval_fold = (key, krsc, scale, shift)
            _, krsc, scale, shift = self._eval_fold
            return K.conv_fprop(x, krsc, self.out_channels, 3, 3, self.stride, 1, scale=scale, shift=shift, act=self._act_code)

    @staticmethod
    def _bn_sync(bn3, pbn):
        """Cross-rank statistics for the block: the branch BN and post_bn follow from the same five moments, so they are synced
        together (one collective per direction) and must agree on it."""
        sync = SF.bn_sync(bn3)
        if pbn is not None and (sync is None) != (SF.bn_sync(pbn) is None):
            raise NotImplementedError("QARepVGGBlock: branch BatchNorm and post_bn must both be SyncBatchNorm or both not")
        return sync

    def _eval_source_key(self):
        """Identity + version of every tensor the folded eval kernel is computed from.  The folded kernel itself is a temporary
        whose address the caching allocator reuses, so it cannot key a cache (load_state_dict / in-place edits would go unnoticed);
        optimizer steps that write parameters through raw pointers are covered by functional.weight_epoch()."""
        bn = self.branch_3x3.bn
        srcs = [self.branch_3x3.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, self.branch_1x1.weight, self.branch_1x1.bias]
        if isinstance(self.alpha, torch.Tensor):
            srcs.append(self.alpha)
        if self.use_post_bn:
            srcs += [self.post_bn.weight, self.post_bn.bias, self.post_bn.running_mean, self.post_bn.running_var]
        return tuple((t.data_ptr(), t._version) for t in srcs if t is not None)

    def _forward_single_conv(self, x, weight, bias):
        """act(post_bn_eval(conv3x3(x, weight) + bias)) in one GEMM launch."""
        x = K.as_nhwc(x)
        krsc, _ = self._cache_eq.get(weight, c_pad=x.shape[1])
        if self.use_post_bn and not self.fully_fused:
            pbn = self.post_bn
            if self.training:
                raise NotImplementedError("training a partially fused QARepVGGBlock is not supported; fuse for inference only")
            scale = pbn.weight * torch.rsqrt(pbn.running_var + pbn.eps)
            shift = pbn.bias - pbn.running_mean * scale + bias * scale
        else:
            scale, shift = None, bias
        return K.conv_fprop(x, krsc, self.out_channels, 3, 3, self.stride, 1, scale=scale, shift=shift, act=self._act_code)

    # ------------------------------------------------------------------------------------------------ re-parameterisation
    def _get_equivalent_kernel_bias_for_branches(self):
        """K = K3 * gamma/std + alpha * pad(K1) + I ;  b = beta - gamma*mu/std + alpha*b1  (qarepvgg_block.py:206-229)."""
        bn = self.branch_3x3.bn
        std = torch.sqrt(bn.running_var + bn.eps)
        a = bn.weight / std
        kernel3x3 = self.branch_3x3.conv.weight * a.reshape(-1, 1, 1, 1)
        bias3x3 = bn.bias - bn.weight * bn.running_mean / std
        kernel1x1 = torch.nn.functional.pad(self.branch_1x1.weight, [1, 1, 1, 1])
        bias1x1 = self.branch_1x1.bias if self.branch_1x1.bias is not None else 0
        kernelid = self.id_tensor if self.identity is not None else 0
        return kernel3x3 + self.alpha * kernel1x1 + kernelid, bias3x3 + self.alpha * bias1x1

    def partial_fusion(self):
        if self.partially_fused:
            return
        if self.fully_fused:
            raise NotImplementedError("QARepVGGBlock can't be converted to partially fused from fully fused")
        kernel, bias = self._get_equivalent_kernel_bias_for_branches()
        self.rbr_reparam.weight.data = kernel.detach()
        self.rbr_reparam.bias.data = bias.detach()
        for name in ("branch_3x3", "branch_1x1", "identity", "alpha", "id_tensor"):
            if hasattr(self, name):
                self.__delattr__(name)
        self.identity = None
        self.partially_fused, self.fully_fused = True, False

    def full_fusion(self):
        if self.fully_fused:
            return
        if not self.partially_fused:
            self.partial_fusion()
        if self.use_post_bn:
            pbn = self.post_bn
            std = torch.sqrt(pbn.running_var + pbn.eps)
            a = pbn.weight / std
            self.rbr_reparam.weight.data = (self.rbr_reparam.weight * a.reshape(-1, 1, 1, 1)).detach()
            self.rbr_reparam.bias.data = (self.rbr_reparam.bias * a + pbn.bias - pbn.weight * pbn.running_mean / std).detach()
        for para in self.parameters():
            para.detach_()
        if hasattr(self, "post_bn"):
            self.__delattr__("post_bn")
        self.partially_fused, self.fully_fused = False, True

    def fuse_block_residual_branches(self):
        self.partial_fusion()

    def prep_model_for_conversion(self, input_size: Optional[Union[tuple, list]] = None, full_fusion: bool = False, **kwargs):
        if full_fusion:
            self.full_fusion()
        else:
            self.partial_fusion()
