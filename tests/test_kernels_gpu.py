"""GPU parity tests of the raw C-ABI kernels against the CPU oracle (fp32 torch / numpy restatement).

Tolerances.  The kernels take bf16 operands and accumulate in fp32, so against an fp32 oracle fed the SAME
bf16-rounded operands the accumulators must agree to 1e-3 relative (north_star); they actually agree to ~1e-5.
bf16 *storage* of an output adds at most half a bf16 ulp (2^-9 relative), which no bf16 kernel can avoid.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import sg_oracle as O  # noqa: E402

DEV = "cuda"


def K():
    from super_gradients_b200 import kernels

    return kernels


def to_nhwc_bf16(x_nchw: torch.Tensor, pitch=None, off=0) -> torch.Tensor:
    """CPU NCHW fp32 -> CUDA NHWC bf16 view (optionally a channel slice of a wider buffer)."""
    n, c, h, w = x_nchw.shape
    pitch = pitch or ((c + 7) // 8) * 8
    buf = torch.zeros(n, pitch, h, w, dtype=torch.bfloat16, device=DEV).contiguous(memory_format=torch.channels_last)
    view = buf[:, off : off + c]
    view.copy_(x_nchw.to(DEV))
    return view


def _canon(rows):
    if rows.shape[0] == 0:
        return rows
    return rows[np.lexsort((rows[:, 5], rows[:, 3], rows[:, 2], rows[:, 1], rows[:, 0], -rows[:, 4]))]


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def test_layout_roundtrip():
    k = K()
    x = torch.randn(3, 3, 17, 19)
    y = k.nchw_f32_to_nhwc_bf16(x.to(DEV))
    assert y.shape == (3, 8, 17, 19)
    torch.testing.assert_close(y[:, :3].float().cpu(), x.bfloat16().float())
    assert float(y[:, 3:].abs().max()) == 0
    z = k.nhwc_bf16_to_nchw_f32(y[:, :3])
    torch.testing.assert_close(z.cpu(), x.bfloat16().float())


@pytest.mark.parametrize("act,with_res", [("relu", False), ("relu", True), ("none", False)])
def test_bn_act_fwd_bwd(act, with_res):
    k = K()
    g = torch.Generator().manual_seed(13)
    n, c, h, w = 4, 48, 9, 7
    x = (torch.randn(n, c, h, w, generator=g) * 2 + 0.5).bfloat16().float().requires_grad_(True)
    res = torch.randn(n, c, h, w, generator=g).bfloat16().float().requires_grad_(True) if with_res else None
    gamma = (torch.rand(c, generator=g) + 0.5).requires_grad_(True)
    beta = (torch.randn(c, generator=g) * 0.2).requires_grad_(True)
    rm, rv = torch.zeros(c), torch.ones(c)
    eps, mom = 1e-3, 0.03
    z = F.batch_norm(x, rm, rv, gamma, beta, True, mom, eps)
    if with_res:
        z = z + res
    ref = O.act_fn(z, act)
    dy = torch.randn(ref.shape, generator=g).bfloat16().float()
    ref.backward(dy)
    xg = to_nhwc_bf16(x.detach())
    stats = k.channel_stats(xg)
    rmg, rvg = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    resg = to_nhwc_bf16(res.detach()) if with_res else None
    y, mean, rstd = k.bn_act_fwd(xg, stats, gamma.detach().to(DEV), beta.detach().to(DEV), rmg, rvg, eps, mom, act, resg)
    assert ((y.float().cpu() - ref.detach()).abs() <= ref.detach().abs() * 2**-7 + 2e-3).all()
    torch.testing.assert_close(rmg.cpu(), rm, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(rvg.cpu(), rv, rtol=1e-4, atol=1e-5)
    # stats=None: ONE cooperative launch computes the sums itself (wide layers whose GEMM epilogue keeps no statistics): same results
    rmf, rvf = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    yf, meanf, rstdf = k.bn_act_fwd(xg, None, gamma.detach().to(DEV), beta.detach().to(DEV), rmf, rvf, eps, mom, act, resg)
    torch.testing.assert_close(meanf, mean, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(rstdf, rstd, rtol=1e-6, atol=1e-6)
    assert ((yf.float() - y.float()).abs() <= y.float().abs() * 2**-7 + 1e-6).all()
    torch.testing.assert_close(rmf, rmg, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(rvf, rvg, rtol=1e-6, atol=1e-7)
    # without a residual the activation mask is recomputed from x / gamma / beta instead of reading y
    dx, dres, dgamma, dbeta = k.bn_act_bwd(to_nhwc_bf16(dy), xg, y, gamma.detach().to(DEV), mean, rstd, eps, act, want_residual_grad=with_res, beta=beta.detach().to(DEV))
    assert rel_err(dx.float().cpu(), x.grad) < 2e-2
    assert rel_err(dgamma.cpu(), gamma.grad) < 5e-3
    assert rel_err(dbeta.cpu(), beta.grad) < 5e-3
    if with_res:
        assert rel_err(dres.float().cpu(), res.grad) < 1e-2
    # dy as a channel slice of a wider buffer (the gradient of a concat): read in place (SgbBnDesc.dy_pitch), identical results
    wide = torch.randn(n, c + 24, h, w, generator=g).to(DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wide[:, 16 : 16 + c].copy_(to_nhwc_bf16(dy))
    count = lambda: torch.cuda.memory_stats()["allocation.all.allocated"]  # noqa: E731
    dyg = to_nhwc_bf16(dy)
    n0 = count()
    k.bn_act_bwd(dyg, xg, y, gamma.detach().to(DEV), mean, rstd, eps, act, want_residual_grad=with_res, beta=beta.detach().to(DEV))
    n1 = count()
    dx2, dres2, dgamma2, dbeta2 = k.bn_act_bwd(wide[:, 16 : 16 + c], xg, y, gamma.detach().to(DEV), mean, rstd, eps, act, want_residual_grad=with_res, beta=beta.detach().to(DEV))
    assert count() - n1 == n1 - n0, "the sliced dy was copied instead of being read in place"
    assert torch.equal(dx2, dx) and torch.equal(dgamma2, dgamma) and torch.equal(dbeta2, dbeta)
    assert not with_res or torch.equal(dres2, dres)


@pytest.mark.parametrize("shape", [(8, 192, 40, 40), (3, 384, 20, 20), (2, 128, 80, 80)])
def test_bn_act_fwd_fused_statistics_many_ctas(shape):
    """sgb_bn_act_fwd_fused (sums, grid-wide barrier, apply) on shapes that span the whole grid: equal to channel_stats + bn_act_fwd."""
    k = K()
    g = torch.Generator().manual_seed(131)
    n, c, h, w = shape
    xg = to_nhwc_bf16(torch.randn(n, c, h, w, generator=g) * 1.5 + 0.25)
    gamma, beta = (torch.rand(c, generator=g) + 0.5).to(DEV), (torch.randn(c, generator=g) * 0.2).to(DEV)
    rm0, rv0, rm1, rv1 = torch.zeros(c, device=DEV), torch.ones(c, device=DEV), torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    y0, m0, r0 = k.bn_act_fwd(xg, k.channel_stats(xg), gamma, beta, rm0, rv0, 1e-3, 0.03, "relu")
    for _ in range(3):  # repeated launches: the grid barrier's state is reusable
        rm1.zero_(), rv1.fill_(1.0)
        y1, m1, r1 = k.bn_act_fwd(xg, None, gamma, beta, rm1, rv1, 1e-3, 0.03, "relu")
        torch.testing.assert_close(m1, m0, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(r1, r0, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(rv1, rv0, rtol=1e-6, atol=1e-7)
        assert ((y1.float() - y0.float()).abs() <= y0.float().abs() * 2**-7 + 1e-6).all()
    xr = xg.float()
    ref = F.relu(F.batch_norm(xr, None, None, gamma, beta, True, 0.0, 1e-3))
    assert ((y1.float() - ref).abs() <= ref.abs() * 2**-7 + 2e-3).all()


def test_maxpool_axpby_avgpool():
    k = K()
    g = torch.Generator().manual_seed(14)
    x = torch.randn(2, 16, 10, 10, generator=g).bfloat16().float().requires_grad_(True)
    xg = to_nhwc_bf16(x.detach())
    for ks, stride, pad in [(5, 1, 2), (9, 1, 4), (13, 1, 6), (3, 2, 1)]:
        ref = F.max_pool2d(x, ks, stride, pad)
        y, idx = k.maxpool_fwd(xg, ks, stride, pad)
        torch.testing.assert_close(y.float().cpu(), ref.detach())
        dy = torch.randn(ref.shape, generator=g).bfloat16().float()
        (gx,) = torch.autograd.grad(ref, x, dy)
        dx = k.maxpool_bwd(to_nhwc_bf16(dy), idx, x.shape, ks, stride, pad)
        if stride >= 2:  # gather form: bf16 output, one rounding of the (<= 4 term) fp32 sum
            assert dx.dtype == torch.bfloat16
            torch.testing.assert_close(dx.float().cpu(), gx, rtol=2**-8, atol=1e-6)
        else:
            torch.testing.assert_close(dx.cpu(), gx, rtol=1e-5, atol=1e-5)
    a = torch.randn(2, 16, 5, 5, generator=g).bfloat16().float()
    b = torch.randn(2, 16, 5, 5, generator=g).bfloat16().float()
    out = k.axpby(to_nhwc_bf16(a), 1.5, to_nhwc_bf16(b), -0.5)
    torch.testing.assert_close(out.float().cpu(), (1.5 * a - 0.5 * b).bfloat16().float(), rtol=2**-7, atol=1e-3)
    ap = k.avgpool_fwd(to_nhwc_bf16(a))
    torch.testing.assert_close(ap.float().cpu().flatten(1), a.mean((2, 3)).bfloat16().float(), rtol=2**-7, atol=1e-3)


def test_scale_add_and_channel_dot():
    k = K()
    g = torch.Generator().manual_seed(15)
    a = torch.randn(2, 24, 7, 5, generator=g).bfloat16().float()
    b = torch.randn(2, 24, 7, 5, generator=g).bfloat16().float()
    alpha = torch.tensor([0.75], device=DEV)
    out = k.scale_add(to_nhwc_bf16(a), alpha, to_nhwc_bf16(b))
    torch.testing.assert_close(out.float().cpu(), (0.75 * a + b).bfloat16().float(), rtol=2**-7, atol=1e-3)
    out = k.scale_add(to_nhwc_bf16(a, pitch=48, off=8), alpha)
    torch.testing.assert_close(out.float().cpu(), (0.75 * a).bfloat16().float(), rtol=2**-7, atol=1e-3)
    d = k.channel_dot(to_nhwc_bf16(a), to_nhwc_bf16(b, pitch=32, off=8))
    torch.testing.assert_close(d.cpu(), (a.double() * b.double()).sum((0, 2, 3)), rtol=1e-5, atol=1e-4)


def _loss_inputs(G, case):
    g = G[case]
    B = g["cls_logits"].shape[0]
    gt_class, gt_bbox, pad = g["gt_class"], g["gt_bbox"], g["pad_gt_mask"]
    n = gt_bbox.shape[1]
    return g, B, n, gt_class, gt_bbox, pad


@pytest.mark.parametrize("case", ["regular", "ragged_with_empty", "no_targets"])
@pytest.mark.parametrize("extra_pad", [0, 3])
def test_tal_and_loss_kernels_vs_reference_golden(golden, case, extra_pad):
    """Assigner + fused loss fwd/bwd against fixtures produced by the reference's PPYoloELoss (tests/golden/loss.pt)."""
    k = K()
    G = golden("loss")
    g, B, n, gt_class, gt_bbox, pad = _loss_inputs(G, case)
    L, C = g["cls_logits"].shape[1], g["cls_logits"].shape[2]
    n_max = n + extra_pad
    gb = torch.zeros(B, max(n_max, 1), 4)
    gl = torch.zeros(B, max(n_max, 1), dtype=torch.int32)
    gv = torch.zeros(B, max(n_max, 1), dtype=torch.uint8)
    if n > 0:
        gb[:, :n] = gt_bbox
        gl[:, :n] = gt_class.squeeze(-1).int()
        gv[:, :n] = pad.squeeze(-1).byte()
    d = k.loss_desc(B, L, C, 16, n_max)
    cls, reg = g["cls_logits"].to(DEV), g["reg_distri"].to(DEV)
    ap, st = G["anchor_points"].to(DEV), G["stride_tensor"].flatten().to(DEV)
    sums = torch.zeros(4, dtype=torch.float64, device=DEV)
    al, ab, asc = k.tal_assign(d, cls, reg, ap, st, gb.to(DEV), gl.to(DEV), gv.to(DEV), sums)
    assert torch.equal(al.cpu().long(), g["assigned_labels"])
    ref_sc = g["assigned_scores"].sum(-1)
    torch.testing.assert_close(asc.cpu(), ref_sc, rtol=1e-4, atol=1e-6)
    posm = g["assigned_labels"] != C
    torch.testing.assert_close(ab.cpu()[posm], g["assigned_bboxes"][posm])
    items, gc, gr = k.dfl_iou_loss(d, cls, reg, ap, st, al, ab, asc, sums)
    torch.testing.assert_close(items.cpu(), g["items"], rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(gc.cpu(), g["g_cls"], rtol=1e-3, atol=1e-7)
    torch.testing.assert_close(gr.cpu(), g["g_reg"], rtol=1e-3, atol=1e-7)


def test_loss_kernel_random_large():
    """Config-2 sized loss (B=8, L=8400, C=80) against the oracle restatement, TAL included."""
    k = K()
    g = torch.Generator().manual_seed(21)
    B, C, n = 8, 80, 8
    _, ap, nums, st = O.anchors_for_levels([(80, 80), (40, 40), (20, 20)], (8, 16, 32))
    L = sum(nums)
    cls = torch.randn(B, L, C, generator=g) * 1.5 - 2.0
    reg = torch.randn(B, L, 68, generator=g)
    rows = []
    for b in range(B):
        for _ in range(n if b != 3 else 2):
            cx, cy = (torch.rand(2, generator=g) * 440 + 100).tolist()
            w, h = (torch.rand(2, generator=g) * 150 + 30).tolist()
            rows.append([b, int(torch.randint(0, C, (1,), generator=g)), cx, cy, w, h])
    targets = torch.tensor(rows)
    cls_r, reg_r = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
    loss, items, (al_r, ab_r, asc_r) = O.ppyoloe_loss((cls_r, reg_r, None, ap, nums, st), targets, C, return_assignment=True)
    loss.backward()
    gt_class, gt_bbox, pad = O.pad_targets(targets, B)
    d = k.loss_desc(B, L, C, 16, gt_bbox.shape[1])
    sums = torch.zeros(4, dtype=torch.float64, device=DEV)
    clsg, regg, apg, stg = cls.to(DEV), reg.to(DEV), ap.to(DEV), st.flatten().to(DEV)
    al, ab, asc = k.tal_assign(d, clsg, regg, apg, stg, gt_bbox.to(DEV), gt_class.squeeze(-1).int().to(DEV), pad.squeeze(-1).byte().to(DEV), sums)
    mism = (al.cpu().long() != al_r).sum().item()
    assert mism == 0, f"{mism} anchors assigned differently"
    torch.testing.assert_close(asc.cpu(), asc_r.sum(-1), rtol=1e-3, atol=1e-6)
    out, gc, gr = k.dfl_iou_loss(d, clsg, regg, apg, stg, al, ab, asc, sums)
    torch.testing.assert_close(out.cpu(), items, rtol=1e-3, atol=1e-6)  # north_star: loss within 1e-3 rel
    assert rel_err(gc.cpu(), cls_r.grad) < 1e-3
    assert rel_err(gr.cpu(), reg_r.grad) < 1e-3


def test_dfl_decode_and_grad_scatter():
    k = K()
    g = torch.Generator().manual_seed(22)
    B, C = 2, 80
    shapes, strides = [(8, 8), (4, 4), (2, 2)], (8, 16, 32)
    regs = [torch.randn(B, 68, h, w, generator=g).bfloat16().float() for h, w in shapes]
    clss = [torch.randn(B, C, h, w, generator=g).bfloat16().float() for h, w in shapes]
    (pb, ps), raw = O.ndfl_decode(regs, clss, strides)
    L = pb.shape[1]
    pbg = torch.empty(B, L, 4, device=DEV)
    psg = torch.empty(B, L, C, device=DEV)
    clg = torch.empty(B, L, C, device=DEV)
    rdg = torch.empty(B, L, 68, device=DEV)
    base = 0
    for r, c, s in zip(regs, clss, strides):
        k.dfl_decode(to_nhwc_bf16(r), to_nhwc_bf16(c), L, base, C, 16, s, 0.5, pbg, psg, clg, rdg)
        base += r.shape[2] * r.shape[3]
    torch.testing.assert_close(pbg.cpu(), pb, rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(psg.cpu(), ps, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(clg.cpu(), raw[0])
    torch.testing.assert_close(rdg.cpu(), raw[1])
    gsrc = torch.randn(B, L, 68, generator=g)
    dy = k.empty_nhwc(B, 68, 4, 4, DEV)
    k.head_grad_scatter(gsrc.to(DEV), B, 16, L, 64, dy)
    ref = gsrc[:, 64:80].permute(0, 2, 1).reshape(B, 68, 4, 4).bfloat16().float()
    torch.testing.assert_close(dy.float().cpu(), ref)


@pytest.mark.parametrize("case", ["multi_small", "multi_topk", "multi_vanilla", "single_label", "class_agnostic", "nothing_passes"])
def test_nms_bit_exact_vs_oracle_and_reference_golden(golden, case):
    k = K()
    g = golden("nms")[case]
    p = g["params"]
    ref_rows, ref_idx = O.ppyoloe_postprocess(g["boxes"], g["scores"], **p)
    out, oidx, cnt = k.batched_nms(g["boxes"].to(DEV), g["scores"].to(DEV), p["score_threshold"], p["nms_threshold"], p["nms_top_k"], p["max_predictions"], p["multi_label_per_box"], p["class_agnostic_nms"])
    out, oidx, cnt = out.cpu().numpy(), oidx.cpu().numpy(), cnt.cpu().numpy()
    for b in range(len(ref_rows)):
        assert cnt[b] == ref_rows[b].shape[0], (cnt[b], ref_rows[b].shape)
        np.testing.assert_array_equal(oidx[b, : cnt[b]], ref_idx[b])  # bit-exact index selection (oracle tie rule)
        np.testing.assert_array_equal(out[b, : cnt[b]], ref_rows[b])
        # and the reference's own output, up to the order inside exactly tied scores
        rr = g["result"][b].numpy()
        np.testing.assert_array_equal(_canon(out[b, : cnt[b]]), _canon(rr))


@pytest.mark.parametrize("case", ["regular", "topk", "few_joints", "nothing_passes"])
def test_pose_post_prediction_callback_vs_oracle_and_reference_golden(golden, case):
    """Row N2: YoloNASPosePostPredictionCallback on the batched NMS kernel (single score, class-agnostic, >= threshold)."""
    from super_gradients_b200.training.models.pose_estimation_models import YoloNASPosePostPredictionCallback

    g = golden("pose_nms")[case]
    p = g["params"]
    ref, ref_idx = O.yolo_nas_pose_postprocess(g["boxes"], g["conf"], g["coords"], g["jscores"], **p)
    cb = YoloNASPosePostPredictionCallback(**p)
    dev = [g[k].to(DEV) for k in ("boxes", "conf", "coords", "jscores")]
    rows, poses, idx, cnt = cb.forward_batched((tuple(dev), None))
    preds = cb((tuple(dev), None))
    assert len(preds) == len(ref)
    for b, ((rposes, rscores, rboxes), kept) in enumerate(zip(ref, ref_idx)):
        n = int(cnt[b])
        assert n == kept.shape[0]
        np.testing.assert_array_equal(idx[b, :n].cpu().numpy(), kept)  # the same anchors in the same order
        np.testing.assert_array_equal(preds[b].scores.cpu().numpy(), rscores)
        np.testing.assert_array_equal(preds[b].bboxes_xyxy.cpu().numpy(), rboxes)
        np.testing.assert_array_equal(preds[b].poses.cpu().numpy(), rposes)
        # and the unmodified reference callback's own output
        gp, gs, gb = g["result"][b]
        np.testing.assert_array_equal(preds[b].poses.cpu().numpy(), gp.numpy())
        np.testing.assert_array_equal(preds[b].scores.cpu().numpy(), gs.numpy())
        np.testing.assert_array_equal(preds[b].bboxes_xyxy.cpu().numpy(), gb.numpy())
    with pytest.raises(ValueError):
        YoloNASPosePostPredictionCallback(0.5, 0.6, pre_nms_max_predictions=10, post_nms_max_predictions=20)


def test_nms_config2_shape():
    """B=32, 8400 anchors, 80 classes, thr 0.25 / top-k 1000 / IoU 0.7 / max 300 (BASELINE.md section 3)."""
    k = K()
    g = torch.Generator().manual_seed(31)
    B, L, C = 8, 8400, 80
    xy = torch.rand(B, L, 2, generator=g) * 540
    wh = torch.rand(B, L, 2, generator=g) * 100 + 5
    boxes = torch.cat([xy, xy + wh], -1)
    scores = torch.rand(B, L, C, generator=g) ** 8
    ref_rows, ref_idx = O.ppyoloe_postprocess(boxes, scores, 0.25, 0.7, 1000, 300)
    out, oidx, cnt = k.batched_nms(boxes.to(DEV), scores.to(DEV), 0.25, 0.7, 1000, 300)
    out, oidx, cnt = out.cpu().numpy(), oidx.cpu().numpy(), cnt.cpu().numpy()
    for b in range(B):
        assert cnt[b] == ref_rows[b].shape[0]
        np.testing.assert_array_equal(oidx[b, : cnt[b]], ref_idx[b])
        np.testing.assert_array_equal(out[b, : cnt[b]], ref_rows[b])


def test_optimizer_kernels():
    k = K()
    g = torch.Generator().manual_seed(41)
    p = torch.randn(1000, generator=g)
    gr = torch.randn(1000, generator=g)
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.SGD([pr], lr=0.1, momentum=0.9, weight_decay=1e-4)
    pg, mg = p.to(DEV), torch.zeros(1000, device=DEV)
    for _ in range(3):
        pr.grad = gr.clone()
        opt.step()
        k.sgd_step(pg, gr.to(DEV), mg, torch.tensor([0.1, 0.9, 1e-4, 1.0, 0.0], device=DEV))
    torch.testing.assert_close(pg.cpu(), pr.detach(), rtol=1e-5, atol=1e-6)
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=2e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5)
    pg, m, v = p.to(DEV), torch.zeros(1000, device=DEV), torch.zeros(1000, device=DEV)
    for step in range(1, 4):
        pr.grad = gr.clone()
        opt.step()
        k.adamw_step(pg, gr.to(DEV), m, v, torch.tensor([2e-4, 0.9, 0.999, 1e-8, 1e-5, 1 - 0.9**step, 1 - 0.999**step, 1.0], device=DEV))
    torch.testing.assert_close(pg.cpu(), pr.detach(), rtol=1e-5, atol=1e-6)
