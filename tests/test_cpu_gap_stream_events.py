"""not-gpu: the characterised gapped stream's bookkeeping (seist_b200/events.py gap_history_keep, seist_b200/stream.py
gap_pick_positions, DESIGN §4.23) against the per-segment oracle (tests/gap_stream_events_ref.py), and that oracle against
the whole-record gapped cut of each station's own record (tests/gaps_ref.py): call by call a numpy mirror of the packed
histories, the position table and the gap cut rule reproduces the oracle's windows bit for bit; no cut reads outside its
station's history or its segment; the held samples stay within the §4.20 bound, equal the open segment's own count
inside a segment and drop to the push at the first non-empty push after a gap."""
import numpy as np
import pytest

import gaps_ref as GR
from gap_stream_events_ref import GapCharacterizedStreamRef, station_windows
from oracle import event_ref as ER
from oracle.preprocess_ref import normalize
from seist_b200 import events as EV
from seist_b200 import stream as ST
from test_cpu_gap_stream import _crafted, _pieces, _record, _schedules
from test_cpu_stream_chunks import _standin


class _Mirror:
    """The host and device state of a GapCharacterizedStream in numpy: the gapped stream's plan and row flips, the packed
    histories of `ragged_history_plan` on the `gap_history_keep` bounds, and the gap cut over the position table."""

    def __init__(self, S, C, W, P, window, a, mode="std"):
        self.S, self.C, self.W, self.P, self.window, self.a, self.mode = S, C, W, P, window, a, mode
        self.state = ST.gap_stream_state(S)
        self.flip = np.zeros(S, np.int64)
        self.buf = np.zeros(0, np.float32)
        self.h0 = np.zeros(S, np.int64)
        self.R = np.zeros(S, np.int64)
        self.off = np.zeros(S + 1, np.int64)
        self.keep = np.zeros(S, np.int64)

    def push(self, chunks):
        n = np.array([c.shape[1] for c in chunks], np.int64)
        hp = EV.ragged_history_plan(self.h0, self.R, n, self.keep)
        plan = ST.gap_stream_plan(self.state, n, _pieces(chunks), self.W, self.P)
        if n.any():
            C = self.C
            chunk = np.concatenate([np.asarray(c, np.float32).reshape(-1) for c in chunks])
            coff = np.concatenate([[0], np.cumsum(n)])
            out = np.zeros(C * int(hp["off"][-1]), np.float32)
            for s in range(self.S):
                nh = int(self.off[s + 1] - self.off[s])
                held = self.buf[C * self.off[s]:C * self.off[s + 1]].reshape(C, nh)
                new = chunk[C * coff[s]:C * coff[s + 1]].reshape(C, int(n[s]))
                full = np.concatenate([held, new], axis=1)
                L = int(hp["len"][s])
                out[C * hp["off"][s]:C * hp["off"][s + 1]] = full[:, int(hp["h0"][s] - self.h0[s]):][:, :L].reshape(-1)
            self.buf, self.h0, self.off = out, hp["h0"], hp["off"]
        self.R = hp["R"]
        return self._call(plan)

    def close(self):
        return self._call(ST.gap_stream_plan(self.state, None, None, self.W, self.P, close=True))

    def _call(self, plan):
        where = ST.gap_pick_positions(plan, self.flip)
        self.flip[plan["station"][plan["kind"] == ST._TRAILING]] ^= 1
        self.state = plan["state"]
        return where

    def finish(self, where, call):
        """The keep rule on the oracle's open segments, then the gap cut of the call's picks -> windows, the read ranges."""
        assert np.array_equal(self.state["seg_on"], call["seg_on"])
        self.keep = EV.gap_history_keep(self.keep, self.state["seg_on"], self.state["R"], call["first_pend"], call["F"], self.a)
        # each oracle segment with picks at its position: positions are station-contiguous, found by the segment's start
        counts = np.zeros(where["n_pos"], np.int64)
        for s, segs in enumerate(call["segments"]):
            for on, k in segs:
                q = [q for q in range(where["first"][s], where["first"][s + 1]) if where["on"][q] == on and where["end"][q] >= on]
                assert len(q) == 1, (s, on)
                counts[q[0]] = k
        pos_off = np.concatenate([[0], np.cumsum(counts)])
        assert np.array_equal(pos_off[where["first"]], call["ppk"][2])
        index = call["ppk"][0]
        x = np.zeros((len(index), self.C, self.window), np.float32)
        reads = []
        for e in range(len(index)):
            q = int(np.searchsorted(pos_off, e, "right") - 1)
            s, on, end = int(where["station"][q]), int(where["on"][q]), int(where["end"][q])
            L = int(self.off[s + 1] - self.off[s])
            row = self.buf[self.C * self.off[s]:self.C * self.off[s + 1]].reshape(self.C, L)
            lo, hi = max(on, int(self.h0[s])), min(end + 1, int(self.h0[s]) + L)
            p = int(index[e])
            assert lo <= p < hi
            t = p - self.a + np.arange(self.window)
            ok = (t >= lo) & (t < hi)
            w = np.zeros((self.C, self.window), np.float32)
            w[:, ok] = row[:, t[ok] - int(self.h0[s])]
            x[e] = normalize(w, self.mode)
            reads.append((s, on, end, int(self.h0[s]), int(self.h0[s]) + L))
        return x, reads


def _drive(rec, sched, W, P, window, ratio, fn, mpd, thr):
    """The oracle and the mirror over `sched`, checked call by call -> the oracle's calls."""
    S, C, T = rec.shape
    ref = GapCharacterizedStreamRef(S, C, W, P, fn, mpd, thr, window, ratio)
    mirror = _Mirror(S, C, W, P, window, ref.a)
    pos = np.zeros(S, np.int64)
    calls = []
    for n in list(sched) + [None]:
        if n is None:
            where, call = mirror.close(), ref.close()
        else:
            chunks = [rec[s, :, pos[s]:pos[s] + n[s]] for s in range(S)]
            before = mirror.state["seg_on"].copy()
            bound = np.where(n > 0, n + W + ref.a + 1 + (calls[-1]["span"] if calls else 0), mirror.R - mirror.h0)
            where, call = mirror.push(chunks), ref.push(chunks)
            held = mirror.R - mirror.h0
            assert (held <= bound).all(), (len(calls), held, bound)                 # the §4.20 bound
            after = mirror.state["seg_on"]
            inside = (n > 0) & (before >= 0) & (before == after)
            assert np.array_equal(held[inside], call["held"][inside]), len(calls)  # the open segment's own count
            assert np.array_equal(held[(n > 0) & (before < 0)], n[(n > 0) & (before < 0)]), len(calls)   # released in a gap
            pos += n
        got, reads = mirror.finish(where, call)
        assert got.shape == call["windows"].shape and np.array_equal(got, call["windows"]), len(calls)
        assert not np.isnan(got).any()
        for (s, lo, hi, on, end), (s2, m_on, m_end, h0, R) in zip(call["reads"], reads):
            assert s == s2 and (on, end) == (m_on, m_end), (s, on, end, m_on, m_end)
            assert max(lo, on) >= h0 and min(hi, end + 1) <= R, (s, lo, hi, on, end, h0, R)   # inside history and segment
        calls.append(call)
    assert pos.tolist() == [T] * S
    return calls


def _check_whole(rec, calls, W, P, window, ratio, fn, mpd, thr):
    """Each station's windows over the calls equal the whole-record gapped cut of its own record -> its pick count and
    how many of its windows a segment edge cuts."""
    total = edged = 0
    for s in range(rec.shape[0]):
        r = rec[s:s + 1]
        probs = GR.annotate(r, W, P, "mean", "std", fn)
        ppk = GR.pick(probs, r, W, 1, thr[1], mpd)
        want = GR.event_windows(r, W, ppk[0], ppk[2], window, ratio, "std")
        got = station_windows(calls, s)
        assert got.shape == want.shape and np.array_equal(got, want), s
        a = ER.anchor(window, ratio)
        for p in ppk[0]:
            on, off = next((a_, b_) for a_, b_ in GR.segments(r)[0] if a_ <= p <= b_)
            edged += p - a < on or p - a + window > off + 1
        total += len(ppk[0])
    return total, edged


@pytest.mark.parametrize("W,P", [(16, 16), (16, 8), (16, 5)])          # stride W, W / 2 and P not dividing W
@pytest.mark.parametrize("window,ratio", [(12, 0.0), (16, 0.3), (16, 1.0), (24, 0.5)])
def test_crafted_gaps_equal_each_stations_whole_record(W, P, window, ratio):
    assert window - ER.anchor(window, ratio) <= W
    rec = _crafted(W)                       # segments of W - 1, W, W + 1, NaN in one channel, +-Inf, an all-gap station, ...
    fn, thr, mpd = _standin(3), (0.5, 0.3, 0.3), 5
    total = edged = 0
    for sched in _schedules(rec.shape[0], rec.shape[2], W, 7):          # gaps at push edges, 0- and 1-sample pushes, ...
        calls = _drive(rec, [np.asarray(n, np.int64) for n in sched], W, P, window, ratio, fn, mpd, thr)
        t, e = _check_whole(rec, calls, W, P, window, ratio, fn, mpd, thr)
        total, edged = total + t, edged + e
    assert total > 0 and edged > 0


@pytest.mark.parametrize("seed", range(4))
def test_random_gaps_equal_each_stations_whole_record(seed):
    W, P = 12, [12, 6, 5, 7][seed]
    window, ratio = [(12, 0.3), (16, 0.5), (10, 0.0), (12, 1.0)][seed]
    rec = _record(5, 30 * W, W, seed)
    fn, thr, mpd = _standin(3), (0.5, 0.3, 0.3), 4
    total = 0
    for sched in _schedules(5, rec.shape[2], W, seed):
        calls = _drive(rec, [np.asarray(n, np.int64) for n in sched], W, P, window, ratio, fn, mpd, thr)
        total += _check_whole(rec, calls, W, P, window, ratio, fn, mpd, thr)[0]
    assert total > 0


def test_a_station_whose_feed_goes_down_releases_its_history():
    """A station in a long gap holds only its last push; its history drops at its first non-empty push in the gap."""
    W, P, window, ratio = 16, 8, 16, 0.3
    rec = np.random.default_rng(5).standard_normal((2, 3, 40 * W)).astype(np.float32)
    rec[1, :, 10 * W:30 * W] = np.nan
    sched = [np.array([W, W], np.int64)] * 40
    fn, thr, mpd = _standin(3), (0.5, 0.3, 0.3), 5
    ref = GapCharacterizedStreamRef(2, 3, W, P, fn, mpd, thr, window, ratio)
    mirror = _Mirror(2, 3, W, P, window, ref.a)
    held = []
    for i, n in enumerate(sched):
        chunks = [rec[s, :, i * W:(i + 1) * W] for s in range(2)]
        where, call = mirror.push(chunks), ref.push(chunks)
        mirror.finish(where, call)
        held.append((mirror.R - mirror.h0).tolist())
    assert all(h[1] == W for h in held[11:30])                      # only the push itself while the feed is down
    assert max(h[1] for h in held[:10]) > W                         # more while its segment was open
    mirror.finish(mirror.close(), ref.close())


def test_keep_rule():
    keep, seg_on, R = np.array([0, 5, 40, 7]), np.array([10, -1, 30, 7]), np.array([50, 60, 70, 9])
    first, F = np.array([20, 0, np.iinfo(np.int64).max, 8]), np.array([25, 0, 60, 7])
    got = EV.gap_history_keep(keep, seg_on, R, first, F, 4)
    assert got.tolist() == [16, 60, 55, 7]          # the pending candidate, the gap, F - 1 - a, the segment's start
    with pytest.raises(ValueError):
        EV.gap_history_keep(keep, seg_on[:2], R, first, F, 4)
