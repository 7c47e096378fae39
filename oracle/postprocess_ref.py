"""CPU oracle (TEST INFRASTRUCTURE) for the GPU post-processing of SURVEY §8f-1: phase picking and event detection on the
model's probability traces, and the precision/recall/residual counters built from them.

Restates, in numpy, for the reference's default configuration (mpd > 1, rising edges, no valley / kpsh / threshold):
  * `_detect_peaks`  — training/postprocess.py:15-111 (BMC detect_peaks + top-k), called by
  * `_pick_phase`    — :161-193 (pads to `topk` with -1e7),
  * `_detect_event`  — :114-158, which calls obspy.signal.trigger.trigger_onset(x, thr, thr).  obspy is a third-party
                       dependency absent from the reference (requirements.txt pins obspy==1.4.0);
                       with equal on/off thresholds its published algorithm returns the maximal runs of x > thr as
                       inclusive [on, off] index pairs.  PARITY UNPINNED for this one function (no obspy to run);
  * `Metrics.compute` counters for the tasks ppk / spk / det — utils/metrics.py:141-247.
`pick_phase` IS pinned: tests/test_cpu_postprocess.py executes the reference's own `_detect_peaks` source (extracted from
the file with `ast`, nothing else of that module imports here) on random and crafted traces and compares index for index.
Tie rule: the reference ranks candidates with `np.argsort(x[ind])[::-1]`, whose default sort is unstable (on x86 SIMD
either of two equal heights can win).  This restatement and the GPU kernels are the reference with a STABLE sort: equal
heights, the larger index first.  tests/test_cpu_peak_ties.py pins that against the reference's own `_detect_peaks` run
with `np.argsort(kind="stable")` on tie-rich traces (tests/golden/reference_peak_ties.pt).  Ties do occur: quantised
inputs, sigmoid outputs saturated at 1.0f, plateaus on the detection channel (SURVEY section 0.7).
NaN rule, pinned by the same fixture: NaN and its two neighbours are never peaks (the reference maps NaN to inf and
removes them; here every comparison with NaN is false, which gives the same candidates), and a NaN sample is in no run.
"""
import numpy as np

PAD_PHASE = int(-1e7)


def detect_peaks_topk(x: np.ndarray, mph: float, mpd: int, topk: int) -> np.ndarray:
    """postprocess.py:15-111 with edge='rising', threshold=0, kpsh=False, valley=False, mpd > 1 (topk None: all)."""
    x = np.asarray(x, dtype=np.float32)
    n = x.size
    if n < 3:
        return np.zeros(0, dtype=np.int64)
    dx = x[1:] - x[:-1]
    nxt = np.concatenate([dx, [0.0]])
    prv = np.concatenate([[0.0], dx])
    ind = np.where((nxt <= 0) & (prv > 0))[0]                 # :67-68
    ind = ind[(ind != 0) & (ind != n - 1)]                    # :82-85
    ind = ind[x[ind] >= np.float32(mph)]                      # :87-88
    if ind.size == 0:
        return ind.astype(np.int64)
    assert mpd > 1
    order = np.lexsort((ind, x[ind]))[::-1]                   # height descending, equal heights: larger index first
    ind = ind[order][:topk]                                   # :94-97
    keep = np.ones(ind.size, dtype=bool)
    for i in range(ind.size):                                 # :98-105
        if keep[i]:
            close = (ind >= ind[i] - mpd) & (ind <= ind[i] + mpd)
            keep &= ~close
            keep[i] = True
    return np.sort(ind[keep]).astype(np.int64)                # :107


def pick_phase(prob: np.ndarray, threshold: float, min_peak_dist: int, topk: int) -> np.ndarray:
    """(N, L) probabilities -> (N, topk) int64 sample indices, padded with -1e7 (postprocess.py:161-193)."""
    out = np.full((prob.shape[0], topk), PAD_PHASE, dtype=np.int64)
    for i, row in enumerate(prob):
        s = detect_peaks_topk(row, threshold, min_peak_dist, topk)
        out[i, :s.size] = s
    return out


def trigger_runs(x: np.ndarray, thr: float):
    """obspy trigger_onset(x, thr, thr): inclusive [start, end] of every maximal run of x > thr."""
    on = np.asarray(x, dtype=np.float32) > np.float32(thr)
    d = np.diff(np.concatenate([[0], on.astype(np.int8), [0]]))
    return [[int(a), int(b) - 1] for a, b in zip(np.where(d == 1)[0], np.where(d == -1)[0])]


def detect_event(prob: np.ndarray, threshold: float, topk: int) -> np.ndarray:
    """(N, L) -> (N, 2*topk) int64 [on, off] pairs, the `topk` longest runs first (stable: earlier run wins a tie), padded
    with [1, 0] (postprocess.py:114-158)."""
    out = np.zeros((prob.shape[0], 2 * topk), dtype=np.int64)
    for i, row in enumerate(prob):
        pairs = trigger_runs(row, threshold)
        pairs.sort(key=lambda v: v[1] - v[0], reverse=True)
        pairs = pairs[:topk] + [[1, 0]] * max(0, topk - len(pairs))
        out[i] = np.array(pairs, dtype=np.int64).reshape(-1)
    return out


def pick_counters(targets: np.ndarray, preds: np.ndarray, num_samples: int, t_thres: int) -> dict:
    """ppk / spk with one phase per waveform (max_detect_event_num = 1, the reference default): metrics.py:152-167 + residual
    sums :205-232 (mask = true positives)."""
    t = targets.astype(np.int64).reshape(-1)
    p = preds.astype(np.int64).reshape(-1)
    pb = (p >= 0) & (p < num_samples)
    tb = (t >= 0) & (t < num_samples)
    ae = np.abs(t - p)
    tp = pb & tb & (ae <= t_thres)
    res = (t - p).astype(np.float64) * tp
    return {"data_size": int(t.size), "tp": int(tp.sum()), "predp": int(pb.sum()), "possp": int(tb.sum()),
            "sum_res": float(res.sum()), "sum_squ_res": float((res ** 2).sum()), "sum_abs_res": float(np.abs(res).sum())}


def det_counters(targets: np.ndarray, preds: np.ndarray, num_samples: int) -> dict:
    """det: samples covered by any target interval / any predicted interval / both (metrics.py:169-193)."""
    n = targets.shape[0]
    t = targets.astype(np.int64).reshape(n, -1, 2)
    p = preds.astype(np.int64).reshape(n, -1, 2)
    idx = np.arange(num_samples)[None, None, :]
    tb = ((t[:, :, :1] <= idx) & (idx <= t[:, :, 1:])).any(1)
    pb = ((p[:, :, :1] <= idx) & (idx <= p[:, :, 1:])).any(1)
    return {"data_size": int(n), "tp": int((tb & pb).sum()), "predp": int(pb.sum()), "possp": int(tb.sum())}
