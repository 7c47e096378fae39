"""CPU oracle (TEST INFRASTRUCTURE) for the P picks of a streamed record characterised as they close
(seist_b200/events.py CharacterizedStream, DESIGN §4.18): `StreamRef` (tests/stream_chunks_ref.py, which keeps the whole
record) composed with the event cut of oracle/event_ref.py, plus the raw history the device keeps.

  * After every call the retention bound is keep = max(keep, min(first pending P candidate, F - 1) - a), read from
    `StreamRef.picker` (`pend[1]`, `F`), a = anchor(W_ch, p_position_ratio).  A push of n > 0 samples replaces the history
    by the samples [keep, R) of the previous call's bound, so h0 (the history's first global sample) lags keep by one call;
    a push of 0 samples and the close keep the history as it is.
  * Each P pick p the call emits is cut from the history alone, at p - h0 (`event_ref.cut`: zero outside the history),
    and the call records the global range [p - a, p - a + W_ch) it reads, with h0 and R at that moment.
Every call returns (stream output, windows (m, C, W_ch) normalised, reads [(station, lo, hi, h0, R, closed)]).
"""
import numpy as np

from oracle import event_ref as ER
from oracle.preprocess_ref import normalize
from stream_chunks_ref import StreamRef


class CharacterizedStreamRef:
    def __init__(self, S, C, W, P, outputs, mpd, thresholds, window, p_position_ratio, norm_mode="std", stack="mean",
                 ch_norm_mode="std"):
        self.a = ER.anchor(window, p_position_ratio)
        assert window - self.a <= W
        self.ref = StreamRef(S, C, W, P, outputs, mpd, thresholds, norm_mode, stack)
        self.S, self.C, self.window, self.mode = S, C, window, ch_norm_mode
        self.history = np.zeros((S, C, 0), np.float32)
        self.h0 = self.R = self.keep = 0
        self.span = 0            # F - 1 - first pending candidate at the last bound, 0 when none is before F - 1

    @property
    def held_samples(self):
        return self.R - self.h0

    def push(self, chunk):
        out = self.ref.push(chunk)
        n = chunk.shape[2]
        if n:
            full = np.concatenate([self.history, np.asarray(chunk, np.float32)], axis=2)
            assert self.keep >= self.h0
            self.history = full[:, :, self.keep - self.h0:].copy()
            self.h0, self.R = self.keep, self.R + n
        return self._finish(out)

    def close(self):
        return self._finish(self.ref.close())

    def _finish(self, out):
        pk = self.ref.picker
        first = min((p[0][0] for p in pk.pend[1] if p), default=np.iinfo(np.int64).max)
        self.keep = max(self.keep, min(first, pk.F - 1) - self.a)
        self.span = max(0, pk.F - 1 - first)
        index, _, off = out[2]
        x = np.zeros((len(index), self.C, self.window), np.float32)
        reads = []
        for s in range(self.S):
            for e in range(int(off[s]), int(off[s + 1])):
                p = int(index[e])
                x[e] = normalize(ER.cut(self.history[s], p - self.h0, self.window, self.a), self.mode)
                reads.append((s, p - self.a, p - self.a + self.window, self.h0, self.R, pk.closed))
        return out, x, reads


def concat_windows(calls, S):
    """Per station in call order -> (M, C, W_ch), the order of the whole-record pick CSR."""
    rows = []
    for s in range(S):
        for out, x, _ in calls:
            off = out[2][2]
            rows.append(x[int(off[s]):int(off[s + 1])])
    return np.concatenate(rows)
