"""CPU oracle (TEST INFRASTRUCTURE) for the P picks of a ragged stream characterised as they close
(seist_b200/events.py RaggedCharacterizedStream, DESIGN §4.20): one `CharacterizedStreamRef` (tests/stream_events_ref.py)
with S = 1 per station, fed only that station's pushes (a call in which the station pushes nothing is a 0-sample push).

Every call returns (ppk, windows, reads, held):
  * ppk (index, prob, offsets): the call's P picks of all stations packed in station order, as the device stream emits them;
  * windows (m, C, W_ch): their normalised event windows in the same order;
  * reads [(station, lo, hi, h0, R, closed)]: the global range [lo, hi) each cut reads and the station's history then;
  * held (S,) int64: each station's held samples R - h0 after the call.
"""
import numpy as np

from stream_events_ref import CharacterizedStreamRef


class RaggedCharacterizedStreamRef:
    def __init__(self, S, C, W, P, outputs, mpd, thresholds, window, p_position_ratio, norm_mode="std", stack="mean",
                 ch_norm_mode="std"):
        """outputs(x, ids) as for StreamRef, ids (station, window start) with the station of this stream."""
        def station(s):
            return lambda x, ids: outputs(x, [(s, a) for _, a in ids])
        self.refs = [CharacterizedStreamRef(1, C, W, P, station(s), mpd, thresholds, window, p_position_ratio, norm_mode, stack,
                                            ch_norm_mode) for s in range(S)]
        self.S, self.C, self.window = S, C, window
        self.a = self.refs[0].a

    @property
    def held_samples(self):
        return np.array([r.held_samples for r in self.refs], np.int64)

    def push(self, chunks):
        """chunks: S arrays (C, n_s)."""
        assert len(chunks) == self.S
        return self._pack([r.push(np.asarray(c, np.float32)[None]) for r, c in zip(self.refs, chunks)])

    def close(self):
        return self._pack([r.close() for r in self.refs])

    def _pack(self, calls):
        index, prob, counts, xs, reads = [], [], [], [], []
        for s, (out, x, rd) in enumerate(calls):
            i, p, _ = out[2]
            index.append(np.asarray(i, np.int64))
            prob.append(np.asarray(p, np.float32))
            counts.append(len(i))
            xs.append(x)
            reads += [(s,) + r[1:] for r in rd]
        ppk = (np.concatenate(index), np.concatenate(prob), np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
        return ppk, np.concatenate(xs).reshape(-1, self.C, self.window), reads, self.held_samples


def station_windows(calls, s):
    """Station s's windows over all calls, in call order."""
    return np.concatenate([x[int(ppk[2][s]):int(ppk[2][s + 1])] for ppk, x, _, _ in calls])
