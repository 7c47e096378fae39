"""not-gpu: the post-processing oracle (oracle/postprocess_ref.py) against what the reference's own `_detect_peaks`
(training/postprocess.py) returned for the same traces (tests/golden/reference_functions.pt, written by
tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import postprocess_ref as PR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_functions.pt")
CASES = [(1, 50), (3, 50), (5, 8), (2, 200)]
THRESHOLDS = (0.3, 0.05)


def _traces(rng, n, L):
    t = np.arange(L, dtype=np.float32)
    out = np.zeros((n, L), dtype=np.float32)
    for i in range(n):
        for _ in range(rng.integers(0, 6)):
            c, w, a = rng.integers(0, L), rng.uniform(3, 40), rng.uniform(0.1, 1.0)
            out[i] += a * np.exp(-((t - c) ** 2) / (2 * w * w)).astype(np.float32)
        out[i] = out[i] + 0.02 * rng.standard_normal(L).astype(np.float32)
        # no clipping: equal peak heights have no defined order in the reference (np.argsort's default sort is unstable)
        out[i] = (out[i] - out[i].min()) / max(1.0, float(out[i].max() - out[i].min()) * 1.01)
    return out


def peak_traces(topk, mpd):
    x = _traces(np.random.default_rng(topk * 100 + mpd), 48, 2048)
    x[0] = 0.0                          # no peak at all
    x[1, :] = 0.5                       # flat above the threshold: no rising edge
    x[2] = 0.0
    x[2, 100:110] = 0.8                 # flat-topped peak: rising edge only
    x[3] = 0.0
    x[3, 0], x[3, -1] = 0.9, 0.9        # first / last samples cannot be peaks
    return x


@pytest.mark.parametrize("topk,mpd", CASES)
def test_pick_phase_matches_reference_detect_peaks(topk, mpd):
    ref = torch.load(GOLD)["detect_peaks"]
    x = peak_traces(topk, mpd)
    for thr in THRESHOLDS:
        mine = PR.pick_phase(x, thr, mpd, topk)
        for i in range(x.shape[0]):
            want = np.array(ref[(topk, mpd, thr)][i], dtype=np.int64)
            got = mine[i][mine[i] != PR.PAD_PHASE]
            assert np.array_equal(got, want), (i, thr, got, want)
            assert (mine[i][got.size:] == PR.PAD_PHASE).all()


def test_detect_event_runs_and_padding():
    x = np.zeros((3, 64), dtype=np.float32)
    x[0, 5:9] = 0.9
    x[0, 20:40] = 0.7
    x[0, 63] = 0.9                      # run of one sample touching the end
    x[1, :] = 0.9                       # one run covering everything
    out = PR.detect_event(x, 0.5, 2)
    assert out[0].tolist() == [20, 39, 5, 8]
    assert out[1].tolist() == [0, 63, 1, 0]
    assert out[2].tolist() == [1, 0, 1, 0]
    assert PR.detect_event(x, 0.5, 1)[0].tolist() == [20, 39]
    x[2, 10:14] = 0.6
    x[2, 30:34] = 0.6                   # equal lengths: the earlier run first (stable sort)
    assert PR.detect_event(x, 0.5, 2)[2].tolist() == [10, 13, 30, 33]
    assert PR.detect_event(np.full((1, 8), 0.5, np.float32), 0.5, 1)[0].tolist() == [1, 0]     # strict >


def test_counters():
    t = np.array([[100], [200], [-10000000], [300]])
    p = np.array([[103], [260], [50], [-10000000]])
    c = PR.pick_counters(t, p, 8192, 5)
    assert (c["tp"], c["predp"], c["possp"], c["data_size"]) == (1, 3, 3, 4)
    assert c["sum_res"] == -3.0 and c["sum_abs_res"] == 3.0 and c["sum_squ_res"] == 9.0
    d = PR.det_counters(np.array([[10, 19], [1, 0]]), np.array([[15, 30], [5, 6]]), 64)
    assert (d["tp"], d["predp"], d["possp"]) == (5, 18, 10)
