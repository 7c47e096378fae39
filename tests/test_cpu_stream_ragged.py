"""not-gpu: the per-call descriptors of a ragged stream (seist_b200/stream.py ragged_plan, DESIGN §4.19) against the
streaming oracle (tests/stream_chunks_ref.py StreamRef) run on each station alone: for ragged splits, every call's
windows, final range and offsets are those of the station's own one-station stream."""
import numpy as np
import pytest

from seist_b200 import stream as ST
from stream_chunks_ref import StreamRef


def _recording(W):
    """A StreamRef window-output stand-in that records which windows each call runs."""
    seen = []

    def outputs(x, ids):
        seen.extend(a for _, a in ids)
        return np.zeros((len(ids), 3, W), np.float32)
    return outputs, seen


def _schedule(totals, W, P, seed):
    """Per-station push lengths, one list per call, for stations of the given final lengths: 0-sample and 1-sample
    pushes, pushes ending on window ends and on R - W boundaries, a station silent for many calls."""
    rng = np.random.default_rng(seed)
    per = []
    for s, T in enumerate(totals):
        kind = 0 if s == len(totals) - 1 else s % 5
        if kind == 0:
            cuts = [T]
        elif kind == 1:
            cuts = list(range(1, min(T, 40) + 1)) + [T]                              # 1-sample pushes first
        elif kind == 2:
            cuts = [W] + [W + q * P for q in range(1, (T - W) // P + 1)] + [T]      # every push ends on a window end
        elif kind == 3:
            cuts = [c for c in (W - 1, W, W + 1, W + P - 1, T - W, T - 1) if 0 < c < T] + [T]   # around R - W boundaries
        else:
            cuts = sorted(set(rng.integers(0, T + 1, 6).tolist())) + [T]
        cuts = sorted(set(cuts))
        per.append(np.diff([0] + cuts).tolist())
    calls = max(len(p) for p in per) + 3
    out = []
    for s, p in enumerate(per):
        lead = calls - len(p) if s == len(per) - 1 else int(rng.integers(0, calls - len(p) + 1))   # the last: silent, then all
        row = [0] * lead + p
        for _ in range(2):                                                               # 0-sample pushes in between
            row.insert(int(rng.integers(0, len(row) + 1)), 0)
        out.append(row + [0] * (calls + 2 - len(row)))
    return [list(c) for c in zip(*out)]


def _check_ids(plan, P):
    ids = ST.ragged_window_ids(plan, P)
    off = plan["win_off"]
    assert len(ids) == off[-1]
    for j, (s, a) in enumerate(ids):
        assert int(np.searchsorted(off, j, "right") - 1) == s                   # the last station with win_off[s] <= j
        q = j - off[s]
        assert a == ((plan["k0"][s] + q) * P if q < plan["nk"][s] else plan["tail"][s])
    return ids


@pytest.mark.parametrize("W,P", [(64, 32), (64, 64), (64, 24)])
@pytest.mark.parametrize("seed", [0, 1])
def test_plan_equals_one_station_streams(W, P, seed):
    totals = [W, W + 1, 4 * W, 4 * W + 17, 5 * W + 9, 3 * W + P, 7 * W]
    S, C = len(totals), 1
    rng = np.random.default_rng(seed)
    recs = [rng.standard_normal((1, C, T)).astype(np.float32) for T in totals]
    refs, seen = [], []
    for _ in range(S):
        fn, log = _recording(W)
        refs.append(StreamRef(1, C, W, P, fn, 5))
        seen.append(log)
    sched = _schedule(totals, W, P, seed)
    R = np.zeros(S, np.int64)
    for lengths in sched + [None]:
        plan = ST.ragged_plan(R, lengths, W, P, close=lengths is None)
        ids = _check_ids(plan, P)
        for s in range(S):
            seen[s].clear()
            if lengths is None:
                o = refs[s].close()
            else:
                o = refs[s].push(recs[s][:, :, R[s]:R[s] + lengths[s]])
            assert plan["f0"][s] == o[0] and plan["f1"][s] - plan["f0"][s] == o[1].shape[2]
            assert plan["r0"][s] == R[s] and plan["r1"][s] == refs[s].R
            assert [a for t, a in ids if t == s] == seen[s]                     # the same windows, in the same order
            assert plan["chunk_off"][s + 1] - plan["chunk_off"][s] == plan["r1"][s] - plan["r0"][s]
            assert plan["acc_off"][s + 1] - plan["acc_off"][s] == plan["r1"][s] - plan["f0"][s]
            assert plan["out_off"][s + 1] - plan["out_off"][s] == plan["f1"][s] - plan["f0"][s]
            assert 0 <= plan["r0"][s] - plan["f0"][s] <= W and 0 <= plan["r1"][s] - plan["f1"][s] <= W
        R = plan["r1"]
    assert R.tolist() == totals
    assert any(((t - W) // P) * P + W < t for t in totals) and any(((t - W) // P) * P + W == t for t in totals)   # tails, and none


def test_plan_close_names_short_stations():
    R = np.array([100, 5, 64, 63])
    with pytest.raises(ValueError, match=r"\[1, 3\]"):
        ST.ragged_plan(R, None, 64, 32, close=True)
    with pytest.raises(ValueError):
        ST.ragged_plan(R, [1, -1, 0, 0], 64, 32)
    with pytest.raises(ValueError):
        ST.ragged_plan(R, [1, 1], 64, 32)


def test_plan_of_equal_lengths_is_the_equal_rate_step():
    """When every station pushes the same n, each station's counts are the equal-rate stream's step."""
    W, P, S = 64, 24, 3
    R = np.zeros(S, np.int64)
    k = 0
    for n in (10, 60, 0, 1, 100, 7, None):
        plan = ST.ragged_plan(R, None if n is None else [n] * S, W, P, close=n is None)
        r0 = int(R[0])
        if n is None:
            kr = (r0 - W) // P + 1
            want = dict(f0=r0 - W, r1=r0, f1=r0, nk=0, tail=r0 - W if (kr - 1) * P + W < r0 else -1, kr=kr)
        else:
            r1 = r0 + n
            k1 = (r1 - W) // P + 1 if r1 >= W else 0
            want = dict(f0=max(0, r0 - W), r1=r1, f1=max(0, r1 - W), nk=k1 - k, tail=-1, kr=-1)
            k = k1
        for key, v in want.items():
            assert (plan[key] == v).all(), (n, key)
        assert (plan["k0"] == plan["k0"][0]).all()
        R = plan["r1"]
