"""CPU oracle (TEST INFRASTRUCTURE) for phase picking on continuous records (seist_b200/stream.py, DESIGN §4.15).

The reference annotates one window only (demo_predict.py:75: `waveform_ndarray[:, :8192]`, then `normalize` :8-23); this
restates, in numpy, what running it window after window over a long record means:
  * `window_starts`    — k * P for k = 0 .. (T - W) // P, plus T - W when the last of those ends before T;
  * `windows`          — record[s, :, start:start + W] normalised per channel as `DataPreprocessor._normalize`
                         (training/preprocess.py:224-242, oracle/preprocess_ref.normalize), window id s * K + k;
  * `stack`            — the window outputs of every station stacked into (S, 3, T) float32: "mean" adds the covering
                         windows in ascending id order from 0.0f and divides once by their number; "max" is the maximum;
  * `detect_peaks_all` — `_detect_peaks(x, mph, mpd, topk=None)` (training/postprocess.py:15-111) with the restrictions
                         and the tie rule of oracle/postprocess_ref.detect_peaks_topk (rising edges, mpd > 1, equal heights:
                         the larger index ranks first), the suppression loop of :98-105 run over each candidate's
                         neighbours within mpd only (the same result: a candidate survives iff no higher-ranked kept one
                         lies within mpd);
  * `pick_all` / `detect_all` — per station, as CSR arrays (values, offsets); detections are `trigger_runs`
                         (oracle/postprocess_ref.py, obspy trigger_onset(p, thr, thr)) with every run in time order.
"""
import numpy as np

from oracle import postprocess_ref as PP
from oracle import preprocess_ref as PR


def window_starts(T: int, W: int, P: int) -> np.ndarray:
    assert 1 <= P <= W <= T
    starts = list(range(0, T - W + 1, P))
    if starts[-1] + W < T:
        starts.append(T - W)
    return np.array(starts, dtype=np.int64)


def windows(record: np.ndarray, W: int, P: int, norm_mode: str) -> np.ndarray:
    """(S, C, T) -> (S * K, C, W) float32 model inputs."""
    S, _, T = record.shape
    out = [PR.normalize(record[s, :, a:a + W].astype(np.float32), norm_mode) for s in range(S) for a in window_starts(T, W, P)]
    return np.stack(out).astype(np.float32)


def stack(outputs: np.ndarray, S: int, T: int, W: int, P: int, mode: str = "mean") -> np.ndarray:
    """(S * K, 3, W) window outputs -> (S, 3, T) float32."""
    starts = window_starts(T, W, P)
    K = starts.size
    assert outputs.shape[0] == S * K
    outputs = outputs.astype(np.float32)
    if mode == "mean":
        acc = np.zeros((S, outputs.shape[1], T), dtype=np.float32)
        cnt = np.zeros(T, dtype=np.float32)
        for a in starts:
            cnt[a:a + W] += np.float32(1)
    else:
        assert mode == "max"
        acc = np.full((S, outputs.shape[1], T), -np.inf, dtype=np.float32)
    for s in range(S):
        for k, a in enumerate(starts):
            seg = acc[s, :, a:a + W]
            if mode == "mean":
                seg += outputs[s * K + k]
            else:
                np.maximum(seg, outputs[s * K + k], out=seg)
    if mode == "mean":
        acc /= cnt
    return acc


def detect_peaks_all(x: np.ndarray, mph: float, mpd: int) -> np.ndarray:
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
    lo = np.searchsorted(ind, ind - mpd, "left")
    hi = np.searchsorted(ind, ind + mpd, "right")
    keep = np.zeros(ind.size, dtype=bool)
    for j in order:                                           # :98-105
        if not keep[lo[j]:hi[j]].any():
            keep[j] = True
    return ind[keep].astype(np.int64)                         # :107 (ind is in index order)


def pick_all(probs: np.ndarray, channel: int, mph: float, mpd: int):
    """(S, C, T) -> (index int64, prob float32, offsets int64)."""
    idx = [detect_peaks_all(row[channel], mph, mpd) for row in probs]
    off = np.concatenate([[0], np.cumsum([i.size for i in idx])]).astype(np.int64)
    index = np.concatenate(idx).astype(np.int64)
    prob = np.concatenate([row[channel][i] for row, i in zip(probs, idx)]).astype(np.float32)
    return index, prob, off


def detect_all(probs: np.ndarray, channel: int, thr: float):
    """(S, C, T) -> (pairs (E, 2) int64, offsets int64)."""
    runs = [PP.trigger_runs(row[channel], thr) for row in probs]
    off = np.concatenate([[0], np.cumsum([len(r) for r in runs])]).astype(np.int64)
    pairs = np.array([p for r in runs for p in r], dtype=np.int64).reshape(-1, 2)
    return pairs, off
