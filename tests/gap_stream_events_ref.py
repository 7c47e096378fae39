"""CPU oracle (TEST INFRASTRUCTURE) for the P picks of a stream with data gaps characterised as they close
(seist_b200/events.py GapCharacterizedStream, DESIGN §4.23): per station and per segment one `CharacterizedStreamRef`
(tests/stream_events_ref.py) with S = 1, fed that segment's slice of each push (a call without samples for the station
is a 0-sample push of its open segment) and closed in the call that delivers the gap after the segment, or at the close.
A segment that closes with fewer than W samples has no windows and emits nothing, as in tests/gap_stream_ref.py.

Every call returns a dict:
  * ppk (index, prob, offsets): the call's P picks of all stations packed in station then time order, station indices;
  * windows (m, C, W_ch): their normalised event windows in the same order, each cut from its segment's own history;
  * reads [(station, lo, hi, on, end)]: the station range [lo, hi) each cut reads and its segment [on, end] so far;
  * segments: per station the [(on, picks)] of the segments that emitted picks in the call, in time order;
  * held (S,): the open segment's held samples R - h0 after the call, -1 for a station in a gap;
  * seg_on, first_pend, F, span (S,): the open segment's first sample, first pending P candidate and final count in station
    indices (-1, int64 max and 0 in a gap), and its span F - 1 - first pending candidate (0 when none is before F - 1).
"""
import numpy as np

import gap_stream_ref as GSR
from stream_events_ref import CharacterizedStreamRef

_I64_MAX = np.iinfo(np.int64).max


class GapCharacterizedStreamRef:
    def __init__(self, S, C, W, P, outputs, mpd, thresholds, window, p_position_ratio, norm_mode="std", stack="mean",
                 ch_norm_mode="std"):
        """outputs(x, ids) as for StreamRef; the ids it gets are (0, start in the segment)."""
        self.args = (1, C, W, P, outputs, mpd, thresholds, window, p_position_ratio, norm_mode, stack, ch_norm_mode)
        self.S, self.C, self.W, self.window = S, C, W, window
        self.open = [None] * S                       # per station: (on, CharacterizedStreamRef) of its open segment
        self.R = np.zeros(S, np.int64)
        self.a = CharacterizedStreamRef(*self.args).a

    def push(self, chunks):
        """chunks: S arrays (C, n_s), NaN / Inf for gap samples."""
        assert len(chunks) == self.S
        return self._pack([self._station(s, np.asarray(c, np.float32)) for s, c in enumerate(chunks)])

    def close(self):
        calls = []
        for s in range(self.S):
            calls.append([self._end(s)] if self.open[s] else [])
        return self._pack(calls)

    def _end(self, s):
        on, ref = self.open[s]
        self.open[s] = None
        return (on, ref.close()) if ref.ref.R >= self.W else (on, None)

    def _station(self, s, block):
        """The calls of station s's segment refs for one push, in time order: [(on, (out, x, reads) or None)]."""
        n = block.shape[1]
        pieces = [(int(a), int(b)) for a, b in (GSR.segments(block) if n else [])]
        calls = []
        if self.open[s]:
            on, ref = self.open[s]
            if n == 0:
                calls.append((on, ref.push(block[None])))
            elif pieces and pieces[0][0] == 0:
                a, b = pieces.pop(0)
                calls.append((on, ref.push(block[None, :, :b + 1])))
                if b < n - 1:
                    calls.append(self._end(s))
            else:
                calls.append(self._end(s))
        for a, b in pieces:
            ref = CharacterizedStreamRef(*self.args)
            on = int(self.R[s]) + a
            calls.append((on, ref.push(block[None, :, a:b + 1])))
            self.open[s] = (on, ref)
            if b < n - 1:
                calls.append(self._end(s))
        self.R[s] += n
        return calls

    def _pack(self, calls):
        index, prob, counts, xs, reads, segs = [], [], [], [], [], []
        for s, station in enumerate(calls):
            k, mine = 0, []
            for on, call in station:
                if call is None:
                    continue
                out, x, rd = call
                i, p, _ = out[2]
                i = np.asarray(i, np.int64) + on
                index.append(i)
                prob.append(np.asarray(p, np.float32))
                xs.append(x)
                k += len(i)
                if len(i) and mine and mine[-1][0] == on:      # a segment's last push and its close in one call
                    mine[-1] = (on, mine[-1][1] + len(i))
                elif len(i):
                    mine.append((on, len(i)))
                end = on + rd[0][4] - 1 if rd else None
                reads += [(s, lo + on, hi + on, on, end) for _, lo, hi, _, _, _ in rd]
            counts.append(k)
            segs.append(mine)
        held = np.full(self.S, -1, np.int64)
        seg_on = np.full(self.S, -1, np.int64)
        first = np.full(self.S, _I64_MAX, np.int64)
        F = np.zeros(self.S, np.int64)
        span = np.zeros(self.S, np.int64)
        for s, o in enumerate(self.open):
            if o:
                on, ref = o
                pk = ref.ref.picker
                f = min((p[0][0] for p in pk.pend[1] if p), default=None)
                held[s], seg_on[s], F[s], span[s] = ref.held_samples, on, on + pk.F, ref.span
                first[s] = _I64_MAX if f is None else on + f
        ppk = (np.concatenate(index) if index else np.zeros(0, np.int64),
               np.concatenate(prob) if prob else np.zeros(0, np.float32),
               np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
        x = np.concatenate(xs).reshape(-1, self.C, self.window) if xs else np.zeros((0, self.C, self.window), np.float32)
        return dict(ppk=ppk, windows=x, reads=reads, segments=segs, held=held, seg_on=seg_on, first_pend=first, F=F, span=span)


def station_windows(calls, s):
    """Station s's windows over all calls, in call order."""
    return np.concatenate([c["windows"][int(c["ppk"][2][s]):int(c["ppk"][2][s + 1])] for c in calls])
