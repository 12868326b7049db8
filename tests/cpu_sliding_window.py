"""Test infrastructure: CPU stand-ins for the sliding-window kernel wrappers, so that SlidingWindowInferenceDetectionWrapper's glue
(tiling, chunking, the per-tile callback, buffer slices, the merge call) runs without a GPU.  The gather is torch slicing of the
zero-padded canvas, the per-tile NMS restates the reference callback on torchvision (pp_yolo_e/post_prediction_callback.py:42-98),
and the merge is the host build of the merge kernel's algorithm (tests/host_kernels/merge_nms_host.cpp over nms_math.cuh).
Only tests may import this module."""
import torch
import torchvision

import cpu_backend
from sliding_window_cases import merge_nms_host
from super_gradients_b200 import kernels as K


def sliding_window_gather(canvas, tiles_host, tiles, tile, out=None):
    B, C, H, W = canvas.shape
    padded = torch.zeros((B, C, H + tile, W + tile), dtype=canvas.dtype)
    padded[:, :, :H, :W] = canvas
    return torch.stack([padded[b, :, y : y + tile, x : x + tile] for b, y, x in tiles_host.tolist()]).contiguous(memory_format=torch.channels_last)


def batched_nms(boxes, scores, score_thr, iou_thr, top_k, max_out, multi_label=True, class_agnostic=False, thr_inclusive=None, out=None, out_idx=None, out_count=None):
    B, _, C = scores.shape
    rows = torch.zeros((B, max_out, 6)) if out is None else out
    cnt = torch.zeros((B,), dtype=torch.int32) if out_count is None else out_count
    idx = torch.full((B, max_out), -1, dtype=torch.int32) if out_idx is None else out_idx
    for b in range(B):
        bb, ss = boxes[b].float(), scores[b].float()
        if multi_label:
            i, j = (ss > score_thr).nonzero(as_tuple=False).T
            conf = ss[i, j]
        else:
            conf, j = ss.max(1)
            m = conf >= score_thr
            i, conf, j = m.nonzero().flatten(), conf[m], j[m]
        if conf.shape[0] > top_k:
            t = torch.topk(conf, k=top_k, largest=True).indices
            i, j, conf = i[t], j[t], conf[t]
        keep = torchvision.ops.nms(bb[i], conf, iou_thr) if class_agnostic else torchvision.ops.batched_nms(bb[i], conf, j, iou_thr)
        keep = keep[:max_out]
        n = keep.numel()
        cnt[b] = n
        rows[b, :n] = torch.cat([bb[i][keep], conf[keep, None], j[keep, None].float()], 1)
        idx[b, :n] = (i[keep] * C + j[keep]).int()
    return rows, idx, cnt


def sliding_window_merge(rows, counts, tiles, image_tiles_host, image_tiles, ncls, iou_thr):
    T, P, _ = rows.shape
    B = image_tiles_host.shape[0] - 1
    cap = P * int((image_tiles_host[1:] - image_tiles_host[:-1]).max())
    out = torch.zeros((B, cap, 6))
    cnt = torch.zeros((B,), dtype=torch.int32)
    for b in range(B):
        parts = []
        for t in range(int(image_tiles_host[b]), int(image_tiles_host[b + 1])):
            r = rows[t, : int(counts[t])].clone()
            _, y0, x0 = tiles[t].tolist()
            r[:, :4] += torch.tensor([x0, y0, x0, y0], dtype=torch.float32)
            parts.append(r)
        d = torch.cat(parts) if parts else torch.zeros((0, 6))
        keep = merge_nms_host(d[:, :4], d[:, 4], d[:, 5], iou_thr)
        out[b, : keep.numel()] = d[keep]
        cnt[b] = keep.numel()
    return out, cnt


def install(monkeypatch):
    cpu_backend.install(monkeypatch)
    for name, fn in (("sliding_window_gather", sliding_window_gather), ("batched_nms", batched_nms), ("sliding_window_merge", sliding_window_merge)):
        monkeypatch.setattr(K, name, fn)
