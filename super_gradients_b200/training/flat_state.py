"""Flat parameter / gradient / buffer storage.

All live parameters of a model are re-pointed to views of ONE contiguous fp32 buffer, and every parameter gets a
`main_grad` view of ONE contiguous fp32 gradient buffer that the backward kernels write into directly (no autograd
accumulation kernels).  That makes the optimizer step two kernel launches (decay / no-decay range), EMA one launch, and
the data-parallel exchange a single NCCL all-reduce over the live-gradient buffer -- the reference needs
DistributedDataParallel(find_unused_parameters=True) buckets because 32% of YOLO-NAS parameters (the `rbr_reparam`
placeholders) never receive a gradient (SURVEY.md D7, training/sg_trainer/sg_trainer.py:459).
"""
from typing import Dict, List, Tuple

import torch
from torch import nn


def _is_no_decay(name: str, p: torch.Tensor, bn_param_ids) -> bool:
    """zero_weight_decay_on_bias_and_bn grouping (reference: training/utils/optimizer_utils.py:32-85): normalisation weights and
    biases, and every module's `bias` parameter; everything else decays -- including the scalar `alpha` parameters of QARepVGG
    blocks and YOLO-NAS bottlenecks (pinned against the reference's grouping in tests/test_host_logic.py)."""
    return id(p) in bn_param_ids or name.endswith(".bias")


def _adjacency_groups(model: nn.Module):
    """Tensors that modules ask to be laid out back to back (`sgb_adjacent_tensors()` -> iterable of tensor lists): layers that share
    one GEMM (the two 1x1 convolutions of a CSP layer) then run their BatchNorm over the concatenated channels with ONE pointer per
    parameter / statistic, no gather."""
    groups = []
    for m in model.modules():
        fn = getattr(m, "sgb_adjacent_tensors", None)
        if callable(fn):
            groups.extend([t for t in g] for g in fn())
    return groups


def _apply_adjacency(items, groups):
    """items: [(name, tensor)] in layout order.  Every group whose members are ALL in `items` is moved so that its members follow its
    first member directly, in group order; everything else keeps its relative order."""
    pos = {id(t): i for i, (_, t) in enumerate(items)}
    followers = {}
    skip = set()
    for g in groups:
        if len(g) < 2 or any(id(t) not in pos for t in g) or any(id(t) in skip or id(t) in followers for t in g):
            continue
        followers[id(g[0])] = [items[pos[id(t)]] for t in g[1:]]
        skip.update(id(t) for t in g[1:])
    out = []
    for n, t in items:
        if id(t) in skip:
            continue
        out.append((n, t))
        out.extend(followers.get(id(t), ()))
    return out


class FlatState:
    def __init__(self, model: nn.Module, zero_wd_on_bias_and_bn: bool = True, dead_param_filter=lambda n: "rbr_reparam" in n):
        dev = next(model.parameters()).device
        bn_ids = set()
        for m in model.modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                bn_ids.update(id(p) for p in m.parameters(recurse=False))
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        self.dead = [(n, p) for n, p in named if dead_param_filter(n)]
        live = [(n, p) for n, p in named if not dead_param_filter(n)]
        decay = [(n, p) for n, p in live if not (zero_wd_on_bias_and_bn and _is_no_decay(n, p, bn_ids))]
        no_decay = [(n, p) for n, p in live if zero_wd_on_bias_and_bn and _is_no_decay(n, p, bn_ids)]
        groups = _adjacency_groups(model)
        decay, no_decay = _apply_adjacency(decay, groups), _apply_adjacency(no_decay, groups)
        self.order: List[Tuple[str, nn.Parameter]] = decay + no_decay
        self.n_decay = sum(p.numel() for _, p in decay)
        self.n_live = sum(p.numel() for _, p in self.order)
        self.params = torch.empty(self.n_live, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(self.n_live, dtype=torch.float32, device=dev)
        self.offsets: Dict[str, Tuple[int, int]] = {}
        off = 0
        with torch.no_grad():
            for n, p in self.order:
                k = p.numel()
                self.params[off : off + k].copy_(p.detach().reshape(-1))
                p.data = self.params[off : off + k].view(p.shape)
                p.main_grad = self.grads[off : off + k].view(p.shape)
                self.offsets[n] = (off, k)
                off += k
        # floating-point buffers (BN running statistics) -> one flat tensor so EMA covers them in one launch
        bufs = [(n, b) for n, b in model.named_buffers() if b is not None and b.dtype == torch.float32 and n.split(".")[-1] in ("running_mean", "running_var")]
        bufs = _apply_adjacency(bufs, groups)
        self.n_buf = sum(b.numel() for _, b in bufs)
        self.buffers = torch.empty(self.n_buf, dtype=torch.float32, device=dev)
        off = 0
        with torch.no_grad():
            for n, b in bufs:
                k = b.numel()
                self.buffers[off : off + k].copy_(b.reshape(-1))
                b.data = self.buffers[off : off + k].view(b.shape)
                off += k
        self.buffer_names = [n for n, _ in bufs]
        self._chunks = None

    @property
    def chunks(self) -> torch.Tensor:
        """Device int64 chunk table over the live parameters (fused_optimizers.lamb_chunk_table), built on first use: the fixed-order
        float64 gradient norms of Lamb and of clip_grad_norm reduce over it."""
        if self._chunks is None:
            from .fused_optimizers import lamb_chunk_table

            self._chunks = lamb_chunk_table([p.numel() for _, p in self.order]).to(self.params.device)
        return self._chunks

    def zero_grad(self):
        self.grads.zero_()

    def grad_of(self, name: str) -> torch.Tensor:
        off, k = self.offsets[name]
        return self.grads[off : off + k]

    def all_reduce_grads(self, world_size: int):
        """The single data-path collective of a training step: flat NCCL all-reduce (SUM) of the live gradients;
        the 1/world_size average is folded into the optimizer's grad_scale."""
        import torch.distributed as dist

        dist.all_reduce(self.grads, op=dist.ReduceOp.SUM)
