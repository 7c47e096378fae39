"""not-gpu: the ragged characterised stream's bookkeeping (seist_b200/events.py ragged_history_plan, DESIGN §4.20) against
the per-station oracle (tests/stream_ragged_events_ref.py), and that oracle against the whole-record cut of each station's
own record (oracle/event_ref.py on oracle/stream_ref.py's picks): call by call the plan's histories are the one-station
streams' histories; a numpy mirror of the packed buffers and of both kernels' rules cuts the oracle's windows; per station
the windows equal `event_ref.windows` bit for bit, no cut reads below h0_s or at or past R_s before the close, and the
held samples stay within the §4.18 bound; a station's open sawtooth cluster is held only by that station."""
import numpy as np
import pytest

from oracle import event_ref as ER
from oracle import stream_ref as SR
from oracle.preprocess_ref import normalize
from seist_b200 import events as EV
from stream_ragged_events_ref import RaggedCharacterizedStreamRef, station_windows
from test_cpu_stream import long_traces
from test_cpu_stream_chunks import _standin, _whole
from test_cpu_stream_ragged import _schedule


class _Packed:
    """The device state of a RaggedCharacterizedStream in numpy: histories packed back to back by `ragged_history_plan`,
    rebuilt as the history kernel does and cut as the ragged event-window kernel does."""

    def __init__(self, S, C, window, a, mode="std"):
        self.S, self.C, self.window, self.a, self.mode = S, C, window, a, mode
        self.buf = np.zeros(0, np.float32)
        self.h0 = np.zeros(S, np.int64)
        self.R = np.zeros(S, np.int64)
        self.off = np.zeros(S + 1, np.int64)

    def push(self, chunks, keep):
        n = np.array([c.shape[1] for c in chunks], np.int64)
        hp = EV.ragged_history_plan(self.h0, self.R, n, keep)
        if n.any():
            C = self.C
            chunk = np.concatenate([np.asarray(c, np.float32).reshape(-1) for c in chunks])
            coff = np.concatenate([[0], np.cumsum(n)])
            out = np.full(C * int(hp["off"][-1]), np.nan, np.float32)
            for s in range(self.S):
                nh = int(self.off[s + 1] - self.off[s])
                held = self.buf[C * self.off[s]:C * self.off[s + 1]].reshape(C, nh)
                new = chunk[C * coff[s]:C * coff[s + 1]].reshape(C, int(n[s]))
                full = np.concatenate([held, new], axis=1)
                L = int(hp["len"][s])
                out[C * hp["off"][s]:C * hp["off"][s + 1]] = full[:, int(hp["h0"][s] - self.h0[s]):][:, :L].reshape(-1)
            assert not np.isnan(out).any()
            self.buf, self.h0, self.off = out, hp["h0"], hp["off"]
        self.R = hp["R"]
        return hp

    def cut(self, ppk):
        index, _, offsets = ppk
        x = np.zeros((len(index), self.C, self.window), np.float32)
        for s in range(self.S):
            L = int(self.off[s + 1] - self.off[s])
            row = self.buf[self.C * self.off[s]:self.C * self.off[s + 1]].reshape(self.C, L)
            for e in range(int(offsets[s]), int(offsets[s + 1])):
                x[e] = normalize(ER.cut(row, int(index[e]) - int(self.h0[s]), self.window, self.a), self.mode)
        return x


def _drive(recs, W, P, fn, mpd, thr, window, ratio, sched):
    """Both the oracle and the packed mirror over `sched`; checks them call by call -> the oracle's calls, held per call."""
    S, C = len(recs), recs[0].shape[0]
    ref = RaggedCharacterizedStreamRef(S, C, W, P, fn, mpd, thr, window, ratio)
    mirror = _Packed(S, C, window, ref.a)
    pos = np.zeros(S, np.int64)
    calls, held = [], []
    for lengths in list(sched) + [None]:
        if lengths is None:
            call = ref.close()
        else:
            chunks = [recs[s][:, pos[s]:pos[s] + lengths[s]] for s in range(S)]
            keep = np.array([r.keep for r in ref.refs], np.int64)          # the bounds of the previous call
            bound = [h if n == 0 else n + W + ref.a + 1 + r.span for h, n, r in zip(ref.held_samples, lengths, ref.refs)]
            hp = mirror.push(chunks, keep)
            call = ref.push(chunks)
            for s, r in enumerate(ref.refs):                                # the plan is each one-station stream's history
                assert hp["h0"][s] == r.h0 and hp["R"][s] == r.R and hp["len"][s] == r.history.shape[2], (len(calls), s)
                assert hp["off"][s + 1] - hp["off"][s] == hp["len"][s]
                assert call[3][s] <= bound[s], (s, call[3][s], bound[s])   # the §4.18 bound, per station
            pos += lengths
        got = mirror.cut(call[0])
        assert got.shape == call[1].shape and np.array_equal(got, call[1]), len(calls)
        for s, lo, hi, h0, R, closed in call[2]:
            assert max(lo, 0) >= h0, (s, lo, h0)                           # nothing below the history that exists
            assert closed or hi <= R, (s, hi, R)                           # nothing not pushed yet before the close
        calls.append(call)
        held.append(call[3])
    assert pos.tolist() == [r.shape[1] for r in recs]
    return calls, np.array(held)


def _records(totals, C, seed):
    rng = np.random.default_rng(seed)
    return [(rng.standard_normal((C, T)) * rng.uniform(0.5, 10, (C, 1)) + rng.standard_normal((C, 1))).astype(np.float32)
            for T in totals]


@pytest.mark.parametrize("W,P", [(64, 64), (64, 32), (64, 24)])       # stride W, W / 2 and P not dividing W
@pytest.mark.parametrize("window,ratio", [(40, 0.0), (64, 0.3), (64, 1.0), (96, 0.5)])
def test_ragged_windows_equal_each_stations_whole_record(W, P, window, ratio):
    assert window - ER.anchor(window, ratio) <= W
    totals = [W, W + 1, 4 * W, 4 * W + 17, 5 * W + 9, 3 * W + P, 7 * W]   # T = W, T = W + 1, ...
    C = 3
    recs = _records(totals, C, W + P)
    fn = _standin(C)
    thr, mpd = (0.5, 0.3, 0.3), 5
    total = 0
    for seed in (0, 1):
        sched = _schedule(totals, W, P, seed)                              # 0- and 1-sample pushes, a silent station, ...
        assert any(all(c[s] == 0 for c in sched[:len(sched) // 2]) for s in range(len(totals)))
        calls, _ = _drive(recs, W, P, fn, mpd, thr, window, ratio, sched)
        for s, rec in enumerate(recs):
            _, ppk, _, _ = _whole(rec[None], W, P, "mean", "std", fn, mpd, thr)
            want = ER.windows(rec[None], ppk[0], ppk[2], window, ratio, "std")
            got = station_windows(calls, s)
            assert got.shape == want.shape and np.array_equal(got, want), (seed, s)
            total += len(ppk[0])
    assert total > 0


def test_plan_of_a_call_without_samples_keeps_every_history():
    h0, R, keep = np.array([0, 5, 9]), np.array([10, 20, 30]), np.array([3, 7, 12])
    hp = EV.ragged_history_plan(h0, R, [0, 0, 0], keep)
    assert hp["h0"].tolist() == [0, 5, 9] and hp["R"].tolist() == [10, 20, 30] and hp["off"].tolist() == [0, 10, 25, 46]
    hp = EV.ragged_history_plan(h0, R, [0, 4, 0], keep)
    assert hp["h0"].tolist() == [0, 7, 9] and hp["len"].tolist() == [10, 17, 21]
    with pytest.raises(ValueError):
        EV.ragged_history_plan(h0, R, [0, -1, 0], keep)
    with pytest.raises(ValueError):
        EV.ragged_history_plan(h0, R, [0, 1, 0], [3, 4, 12])               # a bound below the held samples
    with pytest.raises(ValueError):
        EV.ragged_history_plan(h0, R, [1, 1], keep)


def _injected(traces, W):
    def outputs(x, ids):
        return np.stack([np.repeat(traces[s, None, a:a + W], 3, axis=0) for s, a in ids]).astype(np.float32)
    return outputs


def test_an_open_sawtooth_cluster_is_held_by_its_own_station():
    """long_traces rows injected as the P trace: station 1 holds a 6000-candidate cluster spanning 30 000 samples; its
    history grows while the cluster is open and shrinks once it closes, and the other stations' histories stay small."""
    T, W, P, mpd, tp = 60_000, 256, 128, 100, 0.3
    tr = long_traces(T, seed=1, n_bumps=80)
    totals = [T - 5000, T, T - 777, 20_000]
    recs = _records(totals, 3, 4)
    fn = _injected(tr, W)
    thr = (0.5, tp, 0.3)
    rng = np.random.default_rng(3)
    rows = []
    for s, n in enumerate(totals):
        cuts = sorted(rng.integers(0, n, 60 if s != 3 else 8).tolist())
        rows.append(np.diff([0] + cuts + [n]).tolist())
    calls = max(len(r) for r in rows)
    rows = [r + [0] * (calls - len(r)) if s != 3 else [0] * (calls - len(r)) + r for s, r in enumerate(rows)]   # 3: silent, then late
    sched = [list(c) for c in zip(*rows)]
    biggest = max(max(r) for r in rows)
    for ratio, window in ((0.3, 256), (1.0, 200)):
        out, held = _drive(recs, W, P, fn, mpd, thr, window, ratio, sched)
        for s, rec in enumerate(recs):
            probs = SR.stack(fn(None, [(s, a) for a in SR.window_starts(totals[s], W, P)]), 1, totals[s], W, P, "mean")
            ppk = SR.pick_all(probs, 1, tp, mpd)
            assert np.array_equal(station_windows(out, s), ER.windows(rec[None], ppk[0], ppk[2], window, ratio, "std")), s
        assert held[:, 1].max() > 30_000 - W and held[-1, 1] < biggest + W + window + 1     # held while open, then released
        small = biggest + W + window + 1 + 2000
        assert held[:, [0, 2, 3]].max() < small, (held[:, [0, 2, 3]].max(), small)          # the others stay small
