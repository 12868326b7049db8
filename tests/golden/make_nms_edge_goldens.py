"""Generates nms_edges.pt: the UNMODIFIED reference's post-processing (on CPU, through oracle/ref_shim.py) on every case of
tests/nms_cases.py.  Run once in the build container:

    python tests/golden/make_nms_edge_goldens.py

Only the reference's outputs are stored; the inputs are rebuilt from their seeds.  Per case and image:
  count    rows per image (-1 where non_max_suppression returns None);
  idx      the outputs as indices into the inputs (int32: anchor * C + class for PPYoloEPostPredictionCallback and
           non_max_suppression rows, the anchor for the pose callback), concatenated over images, each checked here to gather the
           reference's output bit for bit (nms_cases.rows_from_idx);
  pre_nms  per image whose top_k cut falls inside a run of equal scores: the sorted scores the reference handed to torchvision's
           NMS (torch.topk's choice among the tied entries is implementation defined, their multiset is not); None elsewhere.
One tensor per field and case keeps the file small.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import nms_cases as N  # noqa: E402
from oracle import ref_shim  # noqa: E402


class _Capture:
    """Wraps torchvision.ops.boxes.nms / batched_nms and records the scores of each outermost call (batched_nms calls nms)."""

    def __init__(self, tvb):
        self.tvb, self.depth, self.scores = tvb, 0, []
        self.orig = {k: getattr(tvb, k) for k in ("nms", "batched_nms")}

    def __enter__(self):
        for k, f in self.orig.items():
            setattr(self.tvb, k, self._wrap(f))
        return self

    def __exit__(self, *exc):
        for k, f in self.orig.items():
            setattr(self.tvb, k, f)

    def _wrap(self, f):
        def g(*a, **kw):
            if self.depth == 0:
                s = kw["scores"] if "scores" in kw else a[1]
                self.scores.append(s.detach().clone())
            self.depth += 1
            try:
                return f(*a, **kw)
            finally:
                self.depth -= 1

        return g


def main():
    ref_shim.install()
    import torchvision.ops.boxes as tvb
    from super_gradients.training.models.detection_models.pp_yolo_e import PPYoloEPostPredictionCallback
    from super_gradients.training.models.pose_estimation_models.yolo_nas_pose.yolo_nas_pose_post_prediction_callback import YoloNASPosePostPredictionCallback
    from super_gradients.training.utils.detection_utils import non_max_suppression

    out = {}
    for name in N.CASES:
        c = N.build(name)
        p = c["params"]
        with _Capture(tvb) as cap:
            if c["kind"] == "ppyoloe":
                res = [r.clone() for r in PPYoloEPostPredictionCallback(**p)(((c["boxes"], c["scores"]), None))]
            elif c["kind"] == "yolox":
                res = [None if r is None else r.clone() for r in non_max_suppression(c["pred"].clone(), **p)]
            else:
                r = YoloNASPosePostPredictionCallback(**p)(((c["boxes"], c["conf"], c["coords"], c["jscores"]), None))
                res = [(x.poses.clone(), x.scores.clone(), x.bboxes_xyxy.clone()) for x in r]
        # one NMS call per image that has candidates (non_max_suppression skips images without any)
        cand = N.candidate_scores(c)
        calls = iter(cap.scores)
        pre = [next(calls) if cs.size else torch.zeros(0) for cs in cand]
        tied = N.tied_cut(c)
        idx = [torch.zeros(0, dtype=torch.int32) if r is None else N.idx_of_rows(c, b, r) for b, r in enumerate(res)]
        for b, r in enumerate(res):
            if r is not None:
                got = N.rows_from_idx(c, b, idx[b])
                for x, y in zip(got if isinstance(got, tuple) else (got,), r if isinstance(r, tuple) else (r,)):
                    assert torch.equal(N._bits(x), N._bits(y)), (name, b)
        entry = dict(count=[-1 if r is None else i.numel() for i, r in zip(idx, res)], idx=torch.cat(idx))
        entry["pre_nms"] = torch.cat([pre[b].sort(descending=True).values for b in range(len(cand)) if tied[b]] + [torch.zeros(0)]) if any(tied) else None
        out[name] = entry
        print(name, [(len(r[1]) if isinstance(r, tuple) else (0 if r is None else r.shape[0])) for r in res], "tied cut" if any(tied) else "")
    torch.save(out, os.path.join(HERE, "nms_edges.pt"))


if __name__ == "__main__":
    main()
