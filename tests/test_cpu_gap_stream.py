"""not-gpu: streams with data gaps (DESIGN §4.22) on the CPU.  `gap_stream_plan` call by call against the per-station
oracle (tests/gap_stream_ref.py): each station's t0, final count and windows run, on schedules with gaps at the edges of
pushes, pushes that are all gap, many segments in one push, segments spanning many pushes, segments of W - 1, W and W + 1
samples, 0- and 1-sample pushes, a silent station, NaN in one channel, +-Inf, and closes inside short segments and gaps;
gap-free schedules against `ragged_plan`."""
import numpy as np
import pytest

import gap_stream_ref as GSR
from seist_b200 import stream as ST

NAN, INF = np.float32(np.nan), np.float32(np.inf)


def _pieces(blocks):
    """The (station, on, off) segment table of one push's blocks (C, n_s), as seist_gap_stream_scan writes it."""
    st, on, off = [], [], []
    for s, b in enumerate(blocks):
        for a, e in GSR.segments(b) if b.shape[1] else []:
            st.append(s), on.append(a), off.append(e)
    return tuple(np.array(x, np.int64) for x in (st, on, off))


def _record(S, T, W, seed):
    rng = np.random.default_rng(seed)
    rec = rng.standard_normal((S, 3, T)).astype(np.float32)
    for s in range(S):
        for _ in range(rng.integers(0, 8)):
            a = int(rng.integers(0, T))
            rec[s, rng.integers(0, 3) if rng.random() < 0.3 else slice(None), a:a + int(rng.integers(1, 2 * W))] = \
                rng.choice([NAN, INF, -INF])
    return rec


def _crafted(W):
    """Stations with the edge cases named above, and a schedule that puts gaps at push edges."""
    T = 8 * W + 5
    rec = np.random.default_rng(1).standard_normal((7, 3, T)).astype(np.float32)
    rec[0, :, [W - 1, 2 * W + 1, 3 * W + 1, 4 * W + 2]] = NAN           # segments of W - 1, W + 1, W - 1, W samples
    rec[1, 1, 3 * W:3 * W + 3] = NAN                                    # one channel only
    rec[2, 2, W] = INF
    rec[2, 0, W + 1] = -INF
    rec[3] = NAN                                                        # all gap
    rec[5, :, T - W // 2:] = NAN                                        # ends inside a gap
    rec[6, :, T - W - 3] = NAN                                          # ends inside a short segment
    return rec


def _schedules(S, T, W, seed):
    rng = np.random.default_rng(seed)
    yield _equal(S, T, W // 2 + 1)
    yield _equal(S, T, 3 * W + 7)
    sched, left = [], np.full(S, T)
    while left.any():
        n = np.minimum(left, rng.choice([0, 1, 2, W - 1, W, W + 1, 3 * W], size=S))
        n[4] = 0 if left[4] == T and len(sched) < 5 else n[4]           # a station silent for a while
        sched.append(n)
        left -= n
    yield sched


def _equal(S, T, n):
    out, r = [], 0
    while r < T:
        out.append(np.full(S, min(n, T - r)))
        r += n
    return out


def _drive(rec, sched, W, P, check=None):
    S, C, T = rec.shape
    state = ST.gap_stream_state(S)
    R = np.zeros(S, np.int64)
    for i, n in enumerate(sched + [None]):
        close = n is None
        blocks = [] if close else [rec[s, :, R[s]:R[s] + n[s]] for s in range(S)]
        plan = ST.gap_stream_plan(state, None if close else n, None if close else _pieces(blocks), W, P, close=close)
        R1 = R if close else R + n
        ids = GSR.window_ids(plan, P)
        for s in range(S):
            t0, m, win = GSR.call(rec[s, :, :R[s]], rec[s, :, :R1[s]], W, P, close)
            assert (plan["t0"][s], plan["m"][s]) == (t0, m), (i, s)
            got = [a for st, a in ids if st == s]
            assert sorted(got) == win, (i, s, got, win)
        # the rows: offsets are the prefix sums of their counts, windowed rows first, each row's final stretch inside its
        # station's output
        nw = plan["nk"] + (plan["tail"] >= 0)
        assert np.array_equal(np.diff(plan["win_off"]), nw) and (np.diff((nw == 0).astype(int)) >= 0).all()
        assert np.array_equal(np.diff(plan["out_off"]), plan["f1"] - plan["f0"])
        a = plan["on"] + plan["f0"] - plan["t0"][plan["station"]]
        assert (a >= 0).all() and (a + plan["f1"] - plan["f0"] <= plan["m"][plan["station"]]).all()
        assert ((plan["r1"] >= W) | ~plan["closes"]).all()
        if check:
            check(plan, R, n)
        state, R = plan["state"], R1


@pytest.mark.parametrize("W,P", [(16, 16), (16, 8), (16, 5)])
def test_plan_against_oracle_on_crafted_records(W, P):
    rec = _crafted(W)
    for sched in _schedules(rec.shape[0], rec.shape[2], W, 7):
        _drive(rec, sched, W, P)


@pytest.mark.parametrize("seed", range(4))
def test_plan_against_oracle_on_random_records(seed):
    W, P = 12, [12, 6, 5, 7][seed]
    rec = _record(5, 30 * W, W, seed)
    for sched in _schedules(5, rec.shape[2], W, seed):
        _drive(rec, sched, W, P)


def test_gap_free_rows_are_ragged_plan():
    W, P = 16, 5
    rec = np.random.default_rng(0).standard_normal((5, 3, 20 * W)).astype(np.float32)

    def check(plan, R, n):
        rp = ST.ragged_plan(R, np.zeros_like(R) if n is None else n, W, P, close=n is None)
        pushed = R > 0 if n is None else n > 0                         # stations that push nothing get no row
        assert np.array_equal(np.sort(plan["station"]), np.nonzero(pushed)[0])
        for r, s in enumerate(plan["station"]):
            for k in ST._RG_COUNTS:
                assert plan[k][r] == rp[k][s], (k, s)
        assert np.array_equal(plan["t0"], rp["f0"]) and np.array_equal(plan["m"], rp["f1"] - rp["f0"])
    for sched in _schedules(5, rec.shape[2], W, 3):
        _drive(rec, sched, W, P, check)


def test_plan_rejects_bad_lengths():
    st = ST.gap_stream_state(2)
    z = np.zeros(0, np.int64)
    with pytest.raises(ValueError):
        ST.gap_stream_plan(st, [1, -1], (z, z, z), 16, 8)
    with pytest.raises(ValueError):
        ST.gap_stream_plan(st, [1], (z, z, z), 16, 8)
