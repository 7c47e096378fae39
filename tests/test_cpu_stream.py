"""not-gpu: the continuous-record oracle (oracle/stream_ref.py) — whole-trace `detect_peaks_all` against what the
reference's own `_detect_peaks(topk=None)` returned (tests/golden/reference_continuous.pt, written by
tests/golden/make_golden_continuous.py), window starts, stacking and event runs on hand-checked cases."""
import os

import numpy as np
import pytest
import torch

from oracle import stream_ref as SR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_continuous.pt")
CONT_L = 200_000
CONT_CASES = [(0.3, 100), (0.1, 20)]            # (mph, mpd)
SEED = 20261016


def long_traces(L: int = CONT_L, seed: int = SEED, n_bumps: int = 300, teeth: int = 6000) -> np.ndarray:
    """Four rows of L samples: Gaussian bumps plus noise (no exact height ties); the same with a sawtooth of `teeth`
    teeth of period 5 above every threshold (one cluster of `teeth` candidates chained within mpd); a flat-topped peak,
    peaks at samples 1 and L - 2 and a few bumps; a row without a peak."""
    rng = np.random.default_rng(seed)
    t = np.arange(L, dtype=np.float32)
    out = np.zeros((4, L), dtype=np.float32)
    for i in range(2):
        for _ in range(n_bumps):
            c, w, a = rng.integers(0, L), rng.uniform(3, 40), rng.uniform(0.1, 1.0)
            lo, hi = max(0, c - 200), min(L, c + 200)
            out[i, lo:hi] += a * np.exp(-((t[lo:hi] - c) ** 2) / (2 * w * w)).astype(np.float32)
        out[i] = out[i] + 0.02 * rng.standard_normal(L).astype(np.float32)
        out[i] = (out[i] - out[i].min()) / max(1.0, float(out[i].max() - out[i].min()) * 1.01)
    a = L // 4
    h = rng.uniform(0.5, 0.95, teeth).astype(np.float32)              # distinct tooth heights
    saw = (h[:, None] * (np.arange(1, 6, dtype=np.float32) / 5)[None, :]).reshape(-1)
    out[1, a:a + saw.size] = np.maximum(saw, 0.2)
    for _ in range(20):
        c, w, amp = rng.integers(0, L), rng.uniform(3, 40), rng.uniform(0.2, 0.9)
        lo, hi = max(0, c - 200), min(L, c + 200)
        out[2, lo:hi] += amp * np.exp(-((t[lo:hi] - c) ** 2) / (2 * w * w)).astype(np.float32)
    out[2, 1000:1010] = 0.8                                             # flat top: its rising edge only
    out[2, 0:3] = (0.0, 0.9, 0.0)                                       # a peak at sample 1
    out[2, L - 3:] = (0.0, 0.95, 0.0)                                   # a peak at sample L - 2
    out[3] = 0.05 * np.abs(rng.standard_normal(L)).astype(np.float32).clip(0, 1)
    out[3] = np.minimum(out[3], 0.09)                                   # below every threshold
    return out


@pytest.mark.parametrize("mph,mpd", CONT_CASES)
def test_detect_peaks_all_matches_reference(mph, mpd):
    ref = torch.load(GOLD)["detect_peaks"][(mph, mpd)]
    x = long_traces()
    for i, row in enumerate(x):
        got = SR.detect_peaks_all(row, mph, mpd)
        want = np.array(ref[i], dtype=np.int64)
        assert np.array_equal(got, want), (i, got.size, want.size)
    assert len(ref[3]) == 0 and ref[2][0] == 1 and ref[2][-1] == CONT_L - 2 and 1000 in ref[2]


def test_sawtooth_is_one_long_cluster():
    x = long_traces()[1]
    mph, mpd = CONT_CASES[0]
    cand = SR.detect_peaks_all(x, mph, 1 << 30)       # one survivor per cluster when mpd spans the whole trace
    assert cand.size == 1
    a = CONT_L // 4
    dx = x[1:] - x[:-1]
    ind = np.where((np.concatenate([dx, [0.0]]) <= 0) & (np.concatenate([[0.0], dx]) > 0))[0]
    ind = ind[(ind >= a) & (ind < a + 5 * 6000) & (x[ind] >= mph)]
    assert ind.size >= 5000 and np.diff(ind).max() <= mpd


@pytest.mark.parametrize("T,W,P,want", [
    (16, 16, 8, [0]),                    # T = W
    (32, 16, 8, [0, 8, 16]),             # (T - W) % P == 0
    (35, 16, 8, [0, 8, 16, 19]),         # (T - W) % P != 0: one more window ending at T
    (35, 16, 16, [0, 16, 19]),           # P = W
    (20, 16, 1, [0, 1, 2, 3, 4]),        # P = 1
    (17, 16, 16, [0, 1]),
])
def test_window_starts(T, W, P, want):
    assert SR.window_starts(T, W, P).tolist() == want


def test_windows_normalised_per_channel():
    rng = np.random.default_rng(0)
    rec = (rng.standard_normal((2, 3, 35)) * 5 + 3).astype(np.float32)
    x = SR.windows(rec, 16, 8, "std")
    assert x.shape == (8, 3, 16)
    np.testing.assert_array_equal(x[3], SR.PR.normalize(rec[0, :, 19:35], "std"))
    np.testing.assert_array_equal(x[4], SR.PR.normalize(rec[1, :, 0:16], "std"))


def test_stack_by_hand():
    # T = 7, W = 4, P = 2: starts 0, 2 and 3 (the tail window)
    out = np.zeros((3, 3, 4), dtype=np.float32)
    out[0, :] = [1, 2, 3, 4]
    out[1, :] = [10, 20, 30, 40]
    out[2, :] = [100, 200, 300, 400]
    mean = SR.stack(out, 1, 7, 4, 2, "mean")[0, 0]
    # t: 0 1 | 2: (3+10)/2 | 3: (4+20+100)/3 | 4: (30+200)/2 | 5: (40+300)/2 | 6: 400
    assert mean.tolist() == [1, 2, 6.5, np.float32(124) / np.float32(3), 115, 170, 400]
    mx = SR.stack(out, 1, 7, 4, 2, "max")[0, 0]
    assert mx.tolist() == [1, 2, 10, 100, 200, 300, 400]


def test_trigger_runs_touching_both_ends():
    p = np.zeros((2, 3, 12), dtype=np.float32)
    p[0, 0, 0:3] = 0.9
    p[0, 0, 5] = 0.6
    p[0, 0, 9:] = 0.7
    p[1, 0, 4:8] = 0.5                  # not above: strict >
    pairs, off = SR.detect_all(p, 0, 0.5)
    assert pairs.tolist() == [[0, 2], [5, 5], [9, 11]] and off.tolist() == [0, 3, 3]
