"""Generates distance_matching.pt: the UNMODIFIED reference's distance-based detection matching (compute_detection_matching with
DistanceMatching + EuclideanDistance / ManhattanDistance) and DetectionMetricsDistanceBased.compute(), on CPU in fp32 through
oracle/ref_shim.py.  Run once in the build container:

    python tests/golden/make_distance_matching_goldens.py

Per case: the inputs (NMS rows per image, flat targets / crowd targets), and per metric ("euclidean", "manhattan") the
per-image (preds_matched, preds_to_ignore) flags and the compute() dictionary (include_classwise_ap=True, so every key).
The hand-made scenes pin the edge cases: equal distances to two targets, a distance exactly equal to a threshold, class
mismatches, crowd targets (one around a matched prediction), a top_k cut, zero scores, images with no prediction / no target /
only crowd targets, boxes partly outside the image, pixel and normalised targets, one and several unsorted thresholds.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

HW = (100, 120)


def _t(img, cls, cx, cy, w, h):
    return [float(img), float(cls), float(cx), float(cy), float(w), float(h)]


def _p(cx, cy, w, h, score, cls):
    return [cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, score, float(cls)]


def edge_scene(normalized):
    """Six images, pixel (or normalised) targets on a 100 x 120 image; thresholds around 5 px make every edge below bite."""
    H, W = HW
    tg, cr = [], []
    out = []
    # image 0: two targets 5 px left and right of a prediction (equal distances: the lower index wins), a second prediction
    # between them takes the other one; a prediction exactly 5 px from a target (no match at thr 5: strict)
    tg += [_t(0, 0, 50, 50, 10, 10), _t(0, 0, 60, 50, 10, 10), _t(0, 1, 20, 20, 8, 8)]
    out.append(torch.tensor([_p(55, 50, 12, 12, 0.9, 0), _p(55, 50, 6, 6, 0.8, 0), _p(25, 20, 6, 6, 0.7, 1), _p(20, 21, 6, 6, 0.6, 0)]))
    # image 1: no prediction
    tg += [_t(1, 0, 30, 30, 10, 10)]
    out.append(None)
    # image 2: predictions, no target at all
    out.append(torch.tensor([_p(40, 40, 10, 10, 0.5, 0), _p(80, 60, 10, 10, 0.4, 1)]))
    # image 3: only crowd targets; one prediction inside the crowd radius, one of another class, one far away
    cr += [_t(3, 0, 70, 30, 30, 20), _t(3, 1, 10, 90, 20, 10)]
    out.append(torch.tensor([_p(72, 31, 10, 10, 0.9, 0), _p(71, 30, 10, 10, 0.8, 1), _p(20, 80, 10, 10, 0.7, 0)]))
    # image 4: a matched prediction that also sits inside a crowd radius; three same-class predictions with top_k = 2 (the third is
    # ignored everywhere); a zero score; boxes partly outside the image (clipped before the centre is taken)
    tg += [_t(4, 2, 30, 30, 10, 10), _t(4, 2, 5, 50, 10, 10), _t(4, 2, 115, 95, 10, 10)]
    cr += [_t(4, 2, 33, 31, 40, 40)]
    out.append(torch.tensor([_p(31, 30, 10, 10, 0.95, 2), _p(-2, 50, 20, 10, 0.9, 2), _p(118, 97, 16, 14, 0.85, 2), _p(30, 30, 10, 10, 0.0, 3),
                             _p(110, 10, 30, 30, 0.5, 3)]))  # fmt: skip
    # image 5: class mismatch only -- every prediction near a target of another class
    tg += [_t(5, 0, 60, 60, 10, 10), _t(5, 1, 20, 70, 10, 10)]
    out.append(torch.tensor([_p(60, 61, 10, 10, 0.9, 1), _p(21, 70, 10, 10, 0.8, 0)]))
    targets, crowds = torch.tensor(tg), torch.tensor(cr)
    if normalized:
        for t in (targets, crowds):
            t[:, [2, 4]] /= W
            t[:, [3, 5]] /= H
    return [None if o is None else o.float() for o in out], targets.float(), crowds.float()


def random_scene(gen, n_img, n_cls, hw, max_t, max_clutter, crowd, normalized, spread):
    """Predictions are copies of targets moved by a few pixels (spread), plus clutter across (and over) the image borders."""
    H, W = hw
    targets, crowds, output = [], [], []
    for i in range(n_img):
        nt = int(torch.randint(0, max_t + 1, (1,), generator=gen))
        cxcy = torch.rand(nt, 2, generator=gen) * torch.tensor([W, H])
        wh = torch.rand(nt, 2, generator=gen) * 20 + 2
        cls = torch.randint(0, n_cls, (nt, 1), generator=gen).float()
        t = torch.cat([torch.full((nt, 1), float(i)), cls, cxcy, wh], 1)
        is_crowd = (torch.rand(nt, generator=gen) < 0.15) if crowd else torch.zeros(nt, dtype=torch.bool)
        rows = []
        for k in range(nt):
            for _ in range(int(torch.randint(0, 4, (1,), generator=gen))):
                off = (torch.rand(2, generator=gen) - 0.5) * 2 * spread
                w, h = (t[k, 4:6] * (0.7 + 0.6 * torch.rand(2, generator=gen))).tolist()
                c = t[k, 1].item() if torch.rand(1, generator=gen) < 0.85 else float(torch.randint(0, n_cls, (1,), generator=gen))
                rows.append(_p(float(t[k, 2] + off[0]), float(t[k, 3] + off[1]), w, h, 0.0, c))
        for _ in range(int(torch.randint(0, max_clutter + 1, (1,), generator=gen))):
            cx, cy = (torch.rand(2, generator=gen) * torch.tensor([W + 40, H + 40]) - 20).tolist()
            w, h = (torch.rand(2, generator=gen) * 30 + 2).tolist()
            rows.append(_p(cx, cy, w, h, 0.0, float(torch.randint(0, n_cls, (1,), generator=gen))))
        p = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
        if len(p):
            sc = torch.rand(len(p), generator=gen)
            p[:, 4] = sc[torch.argsort(sc, descending=True)]  # NMS output is sorted by confidence
        if normalized:
            t[:, [2, 4]] /= W
            t[:, [3, 5]] /= H
        targets.append(t[~is_crowd])
        crowds.append(t[is_crowd])
        output.append(p if len(p) else None)
    return output, torch.cat(targets), torch.cat(crowds)


def main():
    ref_shim.install()
    from super_gradients.training.metrics import detection_metrics as RM
    from super_gradients.training.utils.detection_utils import DistanceMatching, EuclideanDistance, ManhattanDistance, compute_detection_matching

    # the reference metric is a torchmetrics.Metric, which the shim stubs: construct it without the stub's metaclass call and give
    # it the members of Metric it uses
    RM.DetectionMetrics.add_state = lambda self, name, default, dist_reduce_fx=None: setattr(self, name, list(default))
    RM.DetectionMetrics.device = "cpu"
    base = RM.DetectionMetrics.__mro__[1]
    base.__init__ = lambda self, *a, **k: None

    def new_metric(**kw):
        m = object.__new__(RM.DetectionMetricsDistanceBased)
        RM.DetectionMetricsDistanceBased.__init__(m, **kw)
        return m

    metrics = {"euclidean": EuclideanDistance, "manhattan": ManhattanDistance}
    recall_thresholds = torch.linspace(0, 1, 101)  # an input of the golden (its last bit depends on the CPU's SIMD width)

    gen = torch.Generator().manual_seed(2024)
    specs = {
        "edges_pixels_thr5": dict(scenes=[edge_scene(False)], normalized=False, thresholds=[5.0], top_k=2, n_cls=4, score_thres=0.1),
        "edges_normalized_unsorted": dict(scenes=[edge_scene(True)], normalized=True, thresholds=[8.0, 2.5, 5.0, 12.0], top_k=2, n_cls=4, score_thres=0.1),
        "random_crowd_unsorted": dict(scenes=[random_scene(gen, 5, 3, HW, 12, 10, True, True, 6.0) for _ in range(2)], normalized=True, thresholds=[10.0, 3.0, 6.0, 1.5, 20.0],
                                      top_k=5, n_cls=3, score_thres=0.2),
        "random_dense_pixels": dict(scenes=[random_scene(gen, 3, 2, (320, 416), 40, 60, True, False, 4.0) for _ in range(2)], normalized=False, thresholds=[1.0, 2.0, 4.0, 8.0],
                                    top_k=100, n_cls=2, score_thres=0.05),
    }
    cases = {}
    for name, sp in specs.items():
        hw = HW if name.startswith("edges") or name.startswith("random_crowd") else (320, 416)
        case = {"hw": hw, "top_k": sp["top_k"], "normalized": sp["normalized"], "thresholds": sp["thresholds"], "n_cls": sp["n_cls"], "score_thres": sp["score_thres"],
                "recall_thresholds": recall_thresholds, "batches": [{"output": o, "targets": t, "crowd_targets": c} for o, t, c in sp["scenes"]]}  # fmt: skip
        for mname, mcls in metrics.items():
            per_batch = []
            metric = new_metric(num_cls=sp["n_cls"], post_prediction_callback=lambda preds, device=None: preds, normalize_targets=not sp["normalized"],
                                                      distance_thresholds=list(sp["thresholds"]), distance_metric=mcls(), recall_thres=recall_thresholds,
                                                      score_thres=sp["score_thres"], top_k_predictions=sp["top_k"], include_classwise_ap=True)  # fmt: skip
            for batch in case["batches"]:
                res = compute_detection_matching(
                    [None if o is None else o.clone() for o in batch["output"]], batch["targets"].clone(), hw[0], hw[1], denormalize_targets=sp["normalized"], device="cpu",
                    crowd_targets=batch["crowd_targets"].clone(), top_k=sp["top_k"], matching_strategy=DistanceMatching(mcls(), list(sp["thresholds"])),
                )  # fmt: skip
                per_batch.append([(r[0].clone(), r[1].clone()) for r in res])
                inputs = torch.zeros(len(batch["output"]), 3, *hw)
                metric.update([None if o is None else o.clone() for o in batch["output"]], batch["targets"].clone(), device="cpu", inputs=inputs,
                              crowd_targets=batch["crowd_targets"].clone())  # fmt: skip
            out = metric.compute()
            case[mname] = {"matching": per_batch, "compute": out}
            n = sum(len(r[0]) for b in per_batch for r in b)
            m = sum(int(r[0].sum()) for b in per_batch for r in b)
            g = sum(int(r[1].sum()) for b in per_batch for r in b)
            print(name, mname, "preds", n, "matched", m, "ignored", g, {k: round(v, 4) for k, v in list(out.items())[:4]})
        cases[name] = case
    torch.save(cases, os.path.join(HERE, "distance_matching.pt"))


if __name__ == "__main__":
    main()
