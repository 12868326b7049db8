"""Generates tests/golden/pose_metrics.pt by running the UNMODIFIED reference (/root/reference) on CPU through
oracle/ref_shim.py: its PoseEstimationMetrics and compute_oks on synthetic validation batches.  Run once in the build container:

    python tests/golden/make_pose_goldens.py

The reference tree does not exist on the GPU box, so the output is committed.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402


def _pose_scene(gen, n_img, J, max_t, max_p, crowd_p, invisible_p, empty_images):
    """Synthetic post-NMS poses / ground truth of one validation batch: predictions are jittered copies of targets plus clutter,
    with distinct scores in no particular order.  Image 1 has no prediction and image 2 no target when `empty_images`; image 3 then
    has neither."""
    imgs = []
    for i in range(n_img):
        nt = int(torch.randint(1, max_t + 1, (1,), generator=gen))
        if empty_images and i in (2, 3):
            nt = 0
        xy = torch.rand(nt, 2, generator=gen) * 300 + 20
        wh = torch.rand(nt, 2, generator=gen) * 100 + 20
        joints = torch.cat([xy[:, None] + torch.rand(nt, J, 2, generator=gen) * wh[:, None], torch.randint(0, 3, (nt, J, 1), generator=gen).float()], -1)
        joints[..., 2][torch.rand(nt, J, generator=gen) < 0.15] = 0
        if nt:
            joints[0, :, 2] = torch.clamp_min(joints[0, :, 2], 1)  # at least one regular target
        allinv = torch.rand(nt, generator=gen) < invisible_p
        allinv[0:1] = False
        joints[allinv, :, 2] = 0
        crowd = torch.rand(nt, generator=gen) < crowd_p
        crowd[0:1] = False
        boxes = torch.cat([xy, wh], 1)
        areas = wh.prod(1) * (torch.rand(nt, generator=gen) * 0.5 + 0.4)
        poses = []
        for k in range(nt):
            for _ in range(int(torch.randint(0, 4, (1,), generator=gen))):
                noise = torch.randn(J, 2, generator=gen) * float(areas[k].sqrt()) * float(torch.rand(1, generator=gen)) * 0.15
                poses.append(torch.cat([joints[k, :, :2] + noise, torch.rand(J, 1, generator=gen)], -1))
        for _ in range(int(torch.randint(0, max_p + 1, (1,), generator=gen))):
            c = torch.rand(1, 2, generator=gen) * 340 + 10
            poses.append(torch.cat([c + torch.randn(J, 2, generator=gen) * 30, torch.rand(J, 1, generator=gen)], -1))
        p = torch.stack(poses) if poses and not (empty_images and i == 1) and not (empty_images and i == 3) else torch.zeros(0, J, 3)
        sc = torch.rand(len(p), generator=gen) * 0.99 + 0.005  # unordered; distinct across the whole case (ties would make AP depend on sort stability)
        imgs.append(dict(poses=p.numpy(), scores=sc.numpy(), joints=joints.numpy(), bboxes=boxes.numpy(), areas=areas.numpy(), is_crowd=crowd.numpy()))
    return imgs


def golden_pose_metrics():
    """PoseEstimationMetrics (pose_estimation_metrics.py:45-381, pose_estimation_utils.py:35-263) of the unmodified reference on
    synthetic validation batches: the compute_oks matrices, every image's ImageKeypointMatchingResult and compute()'s dictionary.
    Scenes with a reference OKS within 1e-5 of a threshold, or with two equal scores, are drawn again, so that equal flags are not
    luck.  Boxes are always
    given: the reference's compute_visible_bbox_xywh (the path without boxes) does not run on torch (torch.min has no where=)."""
    import numpy as np
    from super_gradients.training.metrics.pose_estimation_metrics import PoseEstimationMetrics
    from super_gradients.training.metrics.pose_estimation_utils import compute_oks

    gen = torch.Generator().manual_seed(88)
    specs = {
        "coco17_crowd": dict(J=17, kw=dict(), n_img=4, max_t=8, max_p=12, crowd_p=0.25, invisible_p=0.0),
        "invisible_targets": dict(J=17, kw=dict(max_objects_per_image=30), n_img=4, max_t=8, max_p=10, crowd_p=0.1, invisible_p=0.35),
        "empty_images": dict(J=17, kw=dict(), n_img=5, max_t=5, max_p=6, crowd_p=0.2, invisible_p=0.1, empty_images=True),
        "topk_small": dict(J=17, kw=dict(max_objects_per_image=5), n_img=3, max_t=6, max_p=15, crowd_p=0.2, invisible_p=0.0),
        "custom_joints": dict(J=5, kw=dict(), n_img=4, max_t=8, max_p=10, crowd_p=0.2, invisible_p=0.1),
        "report_thresholds": dict(J=17, kw=dict(iou_thresholds_to_report=[0.5, 0.75]), n_img=4, max_t=8, max_p=10, crowd_p=0.2, invisible_p=0.1),
        "no_areas": dict(J=17, kw=dict(), n_img=4, max_t=8, max_p=10, crowd_p=0.2, invisible_p=0.1, no_areas=True),
    }
    cases = {}
    for name, sp in specs.items():
        kw = dict(post_prediction_callback=None, num_joints=sp["J"], **sp["kw"])
        m = object.__new__(PoseEstimationMetrics)  # the shim's torchmetrics.Metric stub drops constructor arguments
        PoseEstimationMetrics.__init__(m, **kw)
        m.predictions = []
        thr, sig = m.iou_thresholds, m.oks_sigmas
        batches = []
        for _ in range(2):
            for attempt in range(200):
                imgs = _pose_scene(gen, sp["n_img"], sp["J"], sp["max_t"], sp["max_p"], sp["crowd_p"], sp["invisible_p"], sp.get("empty_images", False))
                recs, close = [], False
                for im in imgs:
                    gt = torch.from_numpy(im["joints"])
                    ign = gt[:, :, 2].eq(0).all(1) | torch.from_numpy(im["is_crowd"])
                    areas = torch.from_numpy(im["bboxes"][:, 2] * im["bboxes"][:, 3] if sp.get("no_areas") else im["areas"]).float()
                    boxes = torch.from_numpy(im["bboxes"]).float()
                    k = min(m.max_objects_per_image, len(im["scores"]))
                    use = torch.topk(torch.from_numpy(im["scores"]), k=k, sorted=True, largest=True).indices
                    p = torch.from_numpy(im["poses"])[use]
                    oks = compute_oks(p, gt[~ign][:, :, :2], gt[~ign][:, :, 2], sig, gt_areas=areas[~ign], gt_bboxes=boxes[~ign]) if len(p) else torch.zeros(0, int((~ign).sum()))
                    oks_c = compute_oks(p, gt[ign][:, :, :2], gt[ign][:, :, 2], sig, gt_areas=areas[ign], gt_bboxes=boxes[ign]) if len(p) else torch.zeros(0, int(ign.sum()))
                    for o in (oks, oks_c):
                        if o.numel() and float((o.reshape(-1, 1) - thr.reshape(1, -1)).abs().min()) < 1e-5:
                            close = True
                    recs.append(dict(oks=oks.clone(), oks_crowd=oks_c.clone(), use=use.clone()))
                all_scores = np.concatenate([im["scores"] for im in imgs] + [im["scores"] for b in batches for im in b["images"]])
                if not close and len(np.unique(all_scores)) == len(all_scores):
                    break
            else:
                raise RuntimeError("no scene without an OKS next to a threshold")
            results = []
            for im, rec in zip(imgs, recs):
                before = len(m.predictions)
                m.update_single_image(im["poses"], im["scores"], im["joints"], im["bboxes"], None if sp.get("no_areas") else im["areas"], im["is_crowd"])
                results.append(tuple(t.clone() if torch.is_tensor(t) else t for t in m.predictions[-1]) if len(m.predictions) > before else None)
            batches.append(dict(images=imgs, oks=[r["oks"] for r in recs], oks_crowd=[r["oks_crowd"] for r in recs], results=results))
        metrics = {k: float(v) for k, v in m.compute().items()}
        cases[name] = dict(kw={k: v for k, v in kw.items() if k != "post_prediction_callback"}, iou_thresholds=thr.clone(), sigmas=sig.clone(), recall_thresholds=m.recall_thresholds.clone(),
                           no_areas=bool(sp.get("no_areas")), batches=batches, metrics=metrics)  # fmt: skip
        print(name, metrics, "images", sum(len(b["images"]) for b in batches), "preds", sum(len(r[0]) for b in batches for r in b["results"] if r is not None))
    torch.save(cases, os.path.join(HERE, "pose_metrics.pt"))


if __name__ == "__main__":
    ref_shim.install()
    golden_pose_metrics()
    print("done")
