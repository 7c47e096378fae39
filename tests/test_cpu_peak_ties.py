"""not-gpu: the picking oracles (oracle/postprocess_ref.py, oracle/stream_ref.py) on traces with exact height ties,
plateaus and NaN (tests/peak_ties.py) against what the reference's own `_detect_peaks`, with a stable `np.argsort`,
returned for them (tests/golden/reference_peak_ties.pt, written by tests/golden/make_golden_peak_ties.py); runs and the
validation counters at their edges."""
import os
from functools import lru_cache

import numpy as np
import pytest
import torch

import peak_ties as PT
from oracle import postprocess_ref as PR
from oracle import stream_ref as SR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_peak_ties.pt")


@lru_cache(maxsize=None)
def _traces(mpd):
    return {seed: x for seed, _, _, x in PT.fixture_traces(mpd)}


def _cases():
    return torch.load(GOLD)["cases"]


def _smaller_index_first(x, mph, mpd):
    """detect_peaks_all with the opposite tie rule: equal heights, the smaller index ranks first."""
    ind = PT.candidates(x, mph)
    keep = np.zeros(ind.size, bool)
    for j in np.lexsort((-ind, x[ind]))[::-1]:
        if not keep[(ind >= ind[j] - mpd) & (ind <= ind[j] + mpd)].any():
            keep[j] = True
    return ind[keep]


def test_fixture_covers_every_case():
    cases = _cases()
    want = {(mph, mpd, topk, seed) for mph, mpd, topk in PT.FIXTURE_PARAMS for seed in range(PT.FIXTURE_SEEDS)}
    assert {(c["mph"], c["mpd"], c["topk"], c["seed"]) for c in cases} == want and len(cases) == len(want)
    for c in cases:
        x = _traces(c["mpd"])[c["seed"]]
        assert x.size == c["L"] and bool(np.isnan(x).any()) <= c["nan"]


def test_oracle_equals_reference_with_stable_sort():
    nan_cases = 0
    for c in _cases():
        x = _traces(c["mpd"])[c["seed"]]
        want = np.array(c["peaks"], dtype=np.int64)
        mph, mpd, topk = c["mph"], c["mpd"], c["topk"]
        if topk is None:
            got = SR.detect_peaks_all(x, mph, mpd)
            assert np.array_equal(got, want), (c["seed"], c["L"], mph, mpd)
            assert np.array_equal(PR.detect_peaks_topk(x, mph, mpd, None), want)
        else:
            got = PR.pick_phase(x[None], mph, mpd, topk)[0]
            assert np.array_equal(got[:want.size], want) and (got[want.size:] == PR.PAD_PHASE).all(), (c["seed"], c["L"], mph, mpd, topk)
        if np.isnan(x).any():
            nan_cases += 1
            assert not (np.isnan(x[want]).any() or np.isnan(x[np.maximum(want - 1, 0)]).any() or np.isnan(x[want + 1]).any())
    assert nan_cases >= 50


def test_ties_decide_the_fixture():
    """The fixture pins the tie rule: the opposite rule (smaller index first) gives other picks on many of its traces."""
    differ = 0
    for c in _cases():
        if c["topk"] is None:
            x = _traces(c["mpd"])[c["seed"]]
            differ += not np.array_equal(_smaller_index_first(x, c["mph"], c["mpd"]), np.array(c["peaks"], dtype=np.int64))
    assert differ >= 20, differ


@pytest.mark.parametrize("mpd", sorted({p[1] for p in PT.FIXTURE_PARAMS}))
def test_detect_peaks_all_equals_topk_infinity(mpd):
    for x in _traces(mpd).values():
        for mph in (0.0, *PT.THRESHOLDS, 0.9998, 1.0):
            assert np.array_equal(SR.detect_peaks_all(x, mph, mpd), PR.detect_peaks_topk(x, mph, mpd, x.size))


def test_long_rows_reach_the_kernel_boundaries():
    """The landmarks of tests/peak_ties.long_rows are where their docstring says (candidates at threshold 0.7)."""
    x, marks = PT.long_rows()
    c = [PT.candidates(r, 0.7) for r in x]
    assert {4090, 4095, 4097} <= set(c[0].tolist()) and 2 not in c[0] and x.shape[1] - 3 not in c[0]
    assert np.isnan(x[0, [0, 1, -2, -1]]).all()
    assert 4096 in c[2] and {8190, 8192, 8194} <= set(c[2].tolist())
    assert c[3].size == 0
    a = marks[1]["seg_cross"]
    assert c[1][PT.CL_SEG - 1] == a and c[1][PT.CL_SEG] == a + 2 and c[1][PT.CL_SEG - 2] < a - PT.GAP
    assert c[1][2 * PT.CL_SEG - 1] == marks[1]["cluster4097"]
    for mpd in (2, 7, 100):
        last = PT.cluster_last(x[1], 0.7, mpd)
        assert last[marks[1]["cluster4097"]] == marks[1]["cluster4097"] + 2 * PT.CL_SMEM
        assert last[marks[1]["cluster4096"]] == marks[1]["cluster4096"] + 2 * (PT.CL_SMEM - 1)
        last = PT.cluster_last(x[0], 0.7, mpd)
        assert last[marks[0]["cluster32"]] == marks[0]["cluster32"] + 2 * (PT.CL_SMALL - 1)
        assert last[marks[0]["cluster33"]] == marks[0]["cluster33"] + 2 * PT.CL_SMALL
    assert max(np.diff(PT.candidates(x[4], 0.3)).max(), 0) <= 100 and PT.candidates(x[4], 0.3).size > 30_000


def test_equal_chains_follow_the_tie_rule():
    """In an all-equal chain the answer depends only on the tie rule: from the last candidate back, every candidate more
    than mpd before the previous kept one."""
    for sp in (2, 3, 7, 8):
        for mpd in (2, 7):
            x = np.concatenate([[0.0], PT.chain(12, sp, 0.9998), [0.0]]).astype(np.float32)
            pos = 1 + sp * np.arange(12)
            step = sp * (mpd // sp + 1)
            want = np.sort(pos[-1] - step * np.arange((pos[-1] - pos[0]) // step + 1))
            assert np.array_equal(SR.detect_peaks_all(x, 0.7, mpd), want), (sp, mpd)
    x = np.array([0, 1, 1, 1, 0, 1, 0, 0.9998, 0.9998, 0], np.float32)             # plateaus: their first sample only
    assert SR.detect_peaks_all(x, 0.5, 2).tolist() == [1, 5] and SR.detect_peaks_all(x, 0.5, 3).tolist() == [1, 5]
    assert SR.detect_peaks_all(x, 0.5, 4).tolist() == [5]
    assert PR.detect_peaks_topk(x, 0.5, 2, 1).tolist() == [5] and PR.detect_peaks_topk(x, 0.99985, 2, 8).tolist() == [1, 5]


def test_runs_at_the_threshold():
    """Runs are samples > float32(thr): a value equal to float32(0.7) (< 0.7) ends a run; it is a pick (>=)."""
    t = np.float32(0.7)
    x = np.array([t, t, 0.70000005, 0.70000005, t, 0.9, np.nan, 0.9, t], np.float32)
    assert PR.trigger_runs(x, 0.7) == [[2, 3], [5, 5], [7, 7]]
    assert PR.detect_event(x[None], 0.7, 4)[0].tolist() == [2, 3, 5, 5, 7, 7, 1, 0]
    assert PR.trigger_runs(np.full(5, t), 0.7) == [] and PR.trigger_runs(np.full(5, t), 0.69999) == [[0, 4]]
    y = np.array([0, t, 0, t, t, 0], np.float32)
    assert SR.detect_peaks_all(y, 0.7, 2).tolist() == [3] and PR.trigger_runs(y, 0.7) == []


def test_pick_counters_at_their_edges():
    n, thr = 100, 5
    pad = PR.PAD_PHASE
    t = np.array([[99], [99], [50], [50], [pad], [10], [100], [0]])
    p = np.array([[99], [100], [55], [44], [10], [pad], [99], [-1]])
    c = PR.pick_counters(t, p, n, thr)
    # predp: 99, 55, 44, 10, 99 (100 and -1 are out of [0, n)); possp: 99, 99, 50, 50, 10, 0 (100 is not)
    # tp: (99, 99) and (50, 55) at |t - p| = t_thres; (50, 44) is 6 away
    assert (c["data_size"], c["tp"], c["predp"], c["possp"]) == (8, 2, 5, 6)
    assert (c["sum_res"], c["sum_squ_res"], c["sum_abs_res"]) == (-5.0, 25.0, 5.0)


def test_det_counters_at_their_edges():
    n = 32
    t = np.array([[0, 3, 10, 12], [1, 0, 1, 0], [5, 40, 1, 0]])                                  # k_targets = 2
    p = np.array([[2, 5, 4, 11, 1, 0], [0, 31, 1, 0, 1, 0], [-10, 6, 6, 6, 30, 31]])             # k_preds = 3
    d = PR.det_counters(t, p, n)
    # row 0: t covers {0..3, 10..12}, p covers {2..11} (overlapping runs once): tp {2, 3, 10, 11}
    # row 1: t covers nothing ([1, 0] padding), p covers 0..31; row 2: t covers 5..31, p covers 0..6, 30, 31
    assert (d["data_size"], d["tp"], d["predp"], d["possp"]) == (3, 4 + 0 + 4, 10 + 32 + 9, 7 + 0 + 27)
