"""CPU oracle (TEST INFRASTRUCTURE) for whole records with data gaps (seist_b200/stream.py `gap_segments`, `segment_plan`,
`annotate(record, segments=...)`, DESIGN §4.21), composed from oracle/stream_ref.py and oracle/event_ref.py:
  * `segments`   — per station, every maximal run of samples whose channels are all finite, inclusive [on, off];
  * `plan`       — window counts, their prefix and the segments each batch spans, window by window;
  * `annotate`   — each segment of at least W samples as a record of its own (`SR.windows` + `SR.stack` of the slice),
                   NaN everywhere else;
  * `packed`     — the device algorithm restated: all segments' windows packed back to back `batch` at a time, each
                   sample accumulating its covering windows in ascending order from 0.0f (the max from -inf), then one
                   division by the count;
  * `pick` / `detect` — `SR.detect_peaks_all` / `SR.detect_all` of each annotated segment's slice, indices shifted by on;
  * `event_windows` — `ER.window` of the pick's own annotated segment, zeros for a pick outside every one.
"""
import numpy as np

from oracle import event_ref as ER
from oracle import stream_ref as SR


def segments(record: np.ndarray):
    """(S, C, T) -> per station an (n, 2) int64 array of inclusive [on, off]."""
    ok = np.isfinite(record).all(axis=1)
    out = []
    for row in ok:
        d = np.diff(np.concatenate([[0], row.astype(np.int8), [0]]))
        on, off = np.nonzero(d == 1)[0], np.nonzero(d == -1)[0] - 1
        out.append(np.stack([on, off], 1).astype(np.int64).reshape(-1, 2))
    return out


def table(record: np.ndarray):
    """(pairs (G, 2), offsets (S + 1,)) int64."""
    segs = segments(record)
    return np.concatenate(segs).reshape(-1, 2), np.concatenate([[0], np.cumsum([len(s) for s in segs])]).astype(np.int64)


def plan(pairs: np.ndarray, W: int, P: int, B: int):
    """K (G,), win_off (G + 1,), first / last segment of each batch, and the packed windows as (segment, start in it)."""
    K = [SR.window_starts(int(b - a + 1), W, P).size if b - a + 1 >= W else 0 for a, b in pairs]
    ids = [(g, int(a)) for g, (on, off) in enumerate(pairs) if off - on + 1 >= W for a in SR.window_starts(int(off - on + 1), W, P)]
    first = [ids[j][0] for j in range(0, len(ids), B)]
    last = [ids[min(j + B, len(ids)) - 1][0] for j in range(0, len(ids), B)]
    return np.array(K, np.int64), np.concatenate([[0], np.cumsum(K)]).astype(np.int64), first, last, ids


def annotate(record: np.ndarray, W: int, P: int, mode: str, norm: str, fn) -> np.ndarray:
    """(S, 3, T) float32: each annotated segment's `SR.stack` of fn(its windows), NaN elsewhere."""
    S, _, T = record.shape
    probs = np.full((S, 3, T), np.nan, np.float32)
    for s, segs in enumerate(segments(record)):
        for on, off in segs:
            n = int(off - on + 1)
            if n >= W:
                sl = record[s:s + 1, :, on:off + 1]
                probs[s, :, on:off + 1] = SR.stack(fn(SR.windows(sl, W, P, norm)), 1, n, W, P, mode)[0]
    return probs


def packed(record: np.ndarray, W: int, P: int, B: int, mode: str, norm: str, fn) -> np.ndarray:
    """The device algorithm: packed windows through fn one batch at a time, stacked per sample in window order."""
    S, _, T = record.shape
    pairs, off_s = table(record)
    station = np.repeat(np.arange(S), np.diff(off_s))
    _, _, _, _, ids = plan(pairs, W, P, B)
    acc = np.full((S, 3, T), np.nan, np.float32)
    cnt = np.zeros((S, T), np.int64)
    for j0 in range(0, len(ids), B):
        batch = ids[j0:j0 + B]
        x = np.stack([SR.windows(record[station[g]:station[g] + 1, :, pairs[g, 0] + a:pairs[g, 0] + a + W], W, W, norm)[0]
                      for g, a in batch])
        y = fn(x)
        for (g, a), yk in zip(batch, y):
            s, t0 = station[g], int(pairs[g, 0] + a)
            seg = acc[s, :, t0:t0 + W]
            fresh = cnt[s, t0:t0 + W] == 0
            seg[:, fresh] = np.float32(0) if mode == "mean" else np.float32(-np.inf)
            if mode == "mean":
                seg += yk
            else:
                np.maximum(seg, yk, out=seg)
            cnt[s, t0:t0 + W] += 1
    if mode == "mean":
        acc = np.where(cnt[:, None] > 0, acc / np.maximum(cnt[:, None], 1).astype(np.float32), np.nan).astype(np.float32)
    return acc


def _annotated(record, W):
    return [[(int(a), int(b)) for a, b in segs if b - a + 1 >= W] for segs in segments(record)]


def pick(probs: np.ndarray, record: np.ndarray, W: int, channel: int, mph: float, mpd: int):
    """Per-station CSR (index, prob, offsets) of `SR.detect_peaks_all` on each annotated segment's slice, shifted by on."""
    idx, val = [], []
    for s, segs in enumerate(_annotated(record, W)):
        row = [SR.detect_peaks_all(probs[s, channel, a:b + 1], mph, mpd) + a for a, b in segs]
        row = np.concatenate(row).astype(np.int64) if row else np.zeros(0, np.int64)
        idx.append(row)
        val.append(probs[s, channel, row])
    off = np.concatenate([[0], np.cumsum([i.size for i in idx])]).astype(np.int64)
    return np.concatenate(idx).astype(np.int64), np.concatenate(val).astype(np.float32), off


def detect(probs: np.ndarray, record: np.ndarray, W: int, channel: int, thr: float):
    """(pairs, offsets) of `SR.detect_all` on each annotated segment's slice, shifted by on."""
    runs = []
    for s, segs in enumerate(_annotated(record, W)):
        r = [SR.detect_all(probs[s:s + 1, :, a:b + 1], channel, thr)[0] + a for a, b in segs]
        runs.append(np.concatenate(r).reshape(-1, 2) if r else np.zeros((0, 2), np.int64))
    off = np.concatenate([[0], np.cumsum([len(r) for r in runs])]).astype(np.int64)
    return np.concatenate(runs).astype(np.int64).reshape(-1, 2), off


def event_windows(record: np.ndarray, W_ann: int, index, offsets, window: int, ratio: float, mode: str) -> np.ndarray:
    """(M, C, window): each pick cut from its own annotated segment (`ER.window` of the slice), zeros outside every one."""
    C = record.shape[1]
    out = np.zeros((len(index), C, window), np.float32)
    segs = _annotated(record, W_ann)
    for s in range(record.shape[0]):
        for e in range(int(offsets[s]), int(offsets[s + 1])):
            p = int(index[e])
            for a, b in segs[s]:
                if a <= p <= b:
                    out[e] = ER.window(record[s, :, a:b + 1], p - a, window, ratio, mode)
    return out
