"""CPU oracle (TEST INFRASTRUCTURE) for continuous records streamed chunk by chunk (seist_b200/stream.py ContinuousStream /
PickStream, DESIGN §4.16): a numpy restatement of the streaming state machine and its finality rules, built on the
whole-record oracle (oracle/stream_ref.py), which it leaves unchanged.

  * `PickStreamRef` takes final (S, 3, m) probabilities stretch by stretch.  A rising-edge candidate t is decided once
    t + 1 < F (F: final samples so far); at the close samples 0 and T - 1 are excluded as in `detect_peaks_all`.  A
    cluster (consecutive candidate gaps <= mpd) whose last candidate c has c + mpd <= F - 2 is resolved by the greedy
    rule and its kept candidates are emitted; the open cluster stays pending.  A run of det > thr closes once the sample
    after its end is final, or at the close.
  * `StreamRef` runs regular window k (start kP) in the first push after which kP + W <= R, the tail window only at the
    close, stacks them in ascending window order from 0.0f (-inf for max) and emits the samples t < F = max(0, R - W)
    (T at the close), the mean divided once by the number of covering windows.  Window outputs come from a callable
    `outputs(x (n, C, W) normalised windows, ids [(station, start)]) -> (n, 3, W)`.
Every call returns (t0, probs, ppk, spk, det) with picks as (index, prob, offsets) and runs as (pairs, offsets).
"""
import numpy as np

from oracle import preprocess_ref as PR


def _csr(rows):
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return rows, off


class PickStreamRef:
    def __init__(self, S: int, mpd: int, thresholds=(0.5, 0.3, 0.3), t0: int = 0):
        assert mpd > 1
        self.S, self.mpd, self.thr = S, int(mpd), tuple(np.float32(t) for t in thresholds)
        self.t0 = self.F = int(t0)
        self.look = np.full((S, 3, 2), -np.inf, dtype=np.float32)
        self.pend = {ch: [[] for _ in range(S)] for ch in (1, 2)}      # (index, value) of undecided clusters
        self.open = [-1] * S
        self.closed = False

    def push(self, probs: np.ndarray):
        return self._step(probs, False)

    def close(self, probs: np.ndarray | None = None):
        return self._step(np.zeros((self.S, 3, 0), np.float32) if probs is None else probs, True)

    def _resolve(self, cand):
        if not cand:
            return []
        idx = np.array([c[0] for c in cand], dtype=np.int64)
        val = np.array([c[1] for c in cand], dtype=np.float32)
        order = np.lexsort((idx, val))[::-1]
        lo = np.searchsorted(idx, idx - self.mpd, "left")
        hi = np.searchsorted(idx, idx + self.mpd, "right")
        keep = np.zeros(idx.size, dtype=bool)
        for j in order:
            if not keep[lo[j]:hi[j]].any():
                keep[j] = True
        return [cand[j] for j in np.nonzero(keep)[0]]

    def _step(self, probs: np.ndarray, last: bool):
        assert not self.closed
        probs = np.asarray(probs, dtype=np.float32)
        S, m = self.S, probs.shape[2]
        f0, f1 = self.F, self.F + m
        parts = [self.look, probs] + ([np.full((S, 3, 1), -np.inf, np.float32)] if last else [])
        ext = np.concatenate(parts, axis=2)
        g0 = f0 - 2
        picks = []
        for ch in (1, 2):
            rows = []
            for s in range(S):
                x = ext[s, ch]
                cand = self.pend[ch][s]
                for i in range(max(1, 3 - (f0 - self.t0)), m + 1):       # global f0 - 1 .. f1 - 2
                    v = x[i]
                    if v - x[i - 1] > 0 and x[i + 1] - v <= 0 and v >= self.thr[ch]:
                        cand.append((g0 + i, v))
                nc = len(cand)
                if cand and not last and cand[-1][0] + self.mpd > f1 - 2:
                    nc = 0                                                # the start of the open (last) cluster
                    for j in range(len(cand) - 1, 0, -1):
                        if cand[j][0] - cand[j - 1][0] > self.mpd:
                            nc = j
                            break
                rows.append(self._resolve(cand[:nc]))
                self.pend[ch][s] = cand[nc:]
            index = np.array([c[0] for r in rows for c in r], dtype=np.int64)
            value = np.array([c[1] for r in rows for c in r], dtype=np.float32)
            picks.append((index, value, _csr(rows)[1]))
        runs = []
        thr = self.thr[0]
        for s in range(S):
            x, r = ext[s, 0], []
            for p in range(2, m + (3 if last else 2)):
                if x[p - 1] > thr and not x[p] > thr:
                    r.append((self.open[s], g0 + p - 1))
                    self.open[s] = -1
                elif x[p] > thr and not x[p - 1] > thr:
                    self.open[s] = g0 + p
            runs.append(r)
        pairs = np.array([p for r in runs for p in r], dtype=np.int64).reshape(-1, 2)
        self.look = ext[:, :, m:m + 2].copy()
        self.F = f1
        self.closed = last
        return picks[0], picks[1], (pairs, _csr(runs)[1])


class StreamRef:
    def __init__(self, S: int, C: int, W: int, P: int, outputs, mpd: int, thresholds=(0.5, 0.3, 0.3), norm_mode: str = "std",
                 stack: str = "mean"):
        assert 1 <= P <= W and stack in ("mean", "max")
        self.S, self.C, self.W, self.P, self.outputs = S, C, W, P, outputs
        self.norm_mode, self.mode = norm_mode, stack
        self.rec = np.zeros((S, C, 0), np.float32)
        self.acc = np.zeros((S, 3, 0), np.float32)
        self.cnt = np.zeros(0, np.float32)
        self.started = np.zeros(0, bool)
        self.R = self.F = self.k = 0
        self.picker = PickStreamRef(S, mpd, thresholds)

    def _grow(self, r1):
        n = r1 - self.acc.shape[2]
        self.acc = np.concatenate([self.acc, np.zeros((self.S, 3, n), np.float32)], axis=2)
        self.cnt = np.concatenate([self.cnt, np.zeros(n, np.float32)])
        self.started = np.concatenate([self.started, np.zeros(n, bool)])

    def _run(self, starts):
        if not starts:
            return
        W = self.W
        ids = [(s, a) for s in range(self.S) for a in starts]
        x = np.stack([PR.normalize(self.rec[s, :, a:a + W].astype(np.float32), self.norm_mode) for s, a in ids]).astype(np.float32)
        y = np.asarray(self.outputs(x, ids), dtype=np.float32)
        for a in starts:
            st = self.started[a:a + W]
            seg = self.acc[:, :, a:a + W]
            init = np.float32(0) if self.mode == "mean" else np.float32(-np.inf)
            seg[:, :, ~st] = init
            self.cnt[a:a + W] += np.float32(1)
            st[:] = True
        for j, (s, a) in enumerate(ids):
            seg = self.acc[s, :, a:a + W]
            if self.mode == "mean":
                seg += y[j]
            else:
                np.maximum(seg, y[j], out=seg)

    def _emit(self, f1):
        out = self.acc[:, :, self.F:f1].copy()
        if self.mode == "mean":
            out /= self.cnt[self.F:f1]
        t0 = self.F
        self.F = f1
        return t0, out

    def push(self, chunk: np.ndarray):
        assert not self.picker.closed
        chunk = np.asarray(chunk, dtype=np.float32)
        self.rec = np.concatenate([self.rec, chunk], axis=2)
        r1 = self.rec.shape[2]
        self._grow(r1)
        k1 = (r1 - self.W) // self.P + 1 if r1 >= self.W else 0
        self._run([k * self.P for k in range(self.k, k1)])
        self.k, self.R = max(self.k, k1), r1
        t0, probs = self._emit(max(0, r1 - self.W))
        return (t0, probs) + self.picker.push(probs)

    def close(self):
        T, W, P = self.R, self.W, self.P
        if T < W:
            raise ValueError("shorter than one window")
        kr = (T - W) // P + 1
        if (kr - 1) * P + W < T:
            self._run([T - W])
        t0, probs = self._emit(T)
        return (t0, probs) + self.picker.close(probs)


def concat(outs, S: int):
    """Call-by-call outputs -> (probs, ppk, spk, det) of the whole record, per station in call order."""
    probs = np.concatenate([o[1] for o in outs], axis=2)

    def cat_picks(k):
        idx, val = [], []
        for s in range(S):
            for o in outs:
                i, v, off = o[k]
                idx.append(np.asarray(i)[off[s]:off[s + 1]])
                val.append(np.asarray(v)[off[s]:off[s + 1]])
        counts = [sum(int(o[k][2][s + 1] - o[k][2][s]) for o in outs) for s in range(S)]
        return np.concatenate(idx).astype(np.int64), np.concatenate(val).astype(np.float32), \
            np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)

    pairs = []
    counts = []
    for s in range(S):
        n = 0
        for o in outs:
            p, off = o[4]
            pairs.append(np.asarray(p)[off[s]:off[s + 1]].reshape(-1, 2))
            n += int(off[s + 1] - off[s])
        counts.append(n)
    det = (np.concatenate(pairs).astype(np.int64).reshape(-1, 2), np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
    return probs, cat_picks(2), cat_picks(3), det
