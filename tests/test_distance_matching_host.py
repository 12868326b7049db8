"""DetectionMetricsDistanceBased matching on the CPU: the kernel's arithmetic (csrc/detection_match_math.cuh, compiled with g++
behind a serial driver) against the reference's flags in tests/golden/distance_matching.pt, bit for bit."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import distance_matching_cases as DC  # noqa: E402
import host_distance_match as H  # noqa: E402


@pytest.mark.parametrize("name,metric", DC.CASES)
def test_host_flags_match_reference(name, metric):
    case = DC.GOLD[name]
    H_, W_ = case["hw"]
    for i, batch in enumerate(case["batches"]):
        rows, counts, t_pad, t_cnt, c_pad, c_cnt = DC.padded(batch)
        matched, ignore = H.detection_distance_matching(rows, counts, t_pad, t_cnt, c_pad, c_cnt, case["thresholds"], metric, H_, W_, case["top_k"], case["normalized"])
        DC.assert_flags_equal(matched, ignore, counts, case[metric]["matching"][i], (name, metric, i))


def test_fixture_covers_the_edges():
    """The hand-made scenes reach what they are there for (thresholds 8, 2.5, 5, 12 px in that column order): a prediction exactly
    5 px from its target matches at 8 and 12 but not at 5; two predictions tied at 5 px from two targets take one each; a matched
    prediction inside a crowd radius is ignored too; the third class-0 prediction falls outside top_k = 2."""
    e = DC.GOLD["edges_pixels_thr5"]["euclidean"]["matching"][0]
    assert e[0][0][2].tolist() == [False]  # 5 px == thr 5
    u = DC.GOLD["edges_normalized_unsorted"]["euclidean"]["matching"][0]
    assert u[0][0][:3].int().tolist() == [[1, 0, 0, 1]] * 3 and u[0][1][3].int().tolist() == [1, 1, 1, 1]
    assert u[4][0][0].int().tolist() == [1, 1, 1, 1] and u[4][1][0].int().tolist() == [1, 1, 1, 1]


@pytest.mark.parametrize("metric", sorted(DC.METRICS))
def test_lane_strided_search_equals_reference_order(metric):
    """nearest_free_target over 32 lanes + the nearer() butterfly = the reference's first free target in stable ascending order of
    its own distance expression (EuclideanDistance / ManhattanDistance.calculate_distance), distance bit-identical."""
    gen = torch.Generator().manual_seed(9)
    dist = DC.METRICS[metric]()
    for trial in range(300):
        n = int(torch.randint(1, 90, (1,), generator=gen))
        xy = (torch.rand(n, 2, generator=gen) * 50).round() if trial % 2 else torch.rand(n, 2, generator=gen) * 50
        tbox = torch.cat([xy, xy + (torch.rand(n, 2, generator=gen) * 10).round() * 2], 1)
        if trial % 3 == 0:  # duplicated targets: equal distances, the lowest index must win
            tbox[n // 2 :] = tbox[: n - n // 2].clone()
        tcls = torch.randint(0, 2, (n,), generator=gen).float()
        taken = (torch.rand(n, generator=gen) < 0.3).to(torch.uint8)
        pbox = tbox[int(torch.randint(0, n, (1,), generator=gen))] + (torch.rand(4, generator=gen) * 6).round()
        thr = float(torch.rand(1, generator=gen) * 15)
        t, v = H.nearest_free_target_lanes(metric, pbox.contiguous(), 1.0, thr, tbox.contiguous(), tcls.contiguous(), taken.contiguous())
        d = dist.calculate_distance(pbox[None], tbox)[0]
        d[(tcls != 1.0) | (taken != 0)] = float("inf")
        sd, order = d.sort(stable=True)
        want = int(order[0]) if float(sd[0]) < thr else -1
        assert t == want, (trial, t, want)
        if want >= 0:
            assert v == float(d[want])
