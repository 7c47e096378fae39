"""A network of mixed input rates in one Resampler on the host (seist_b200/resample.py, DESIGN §4.24): the stream plan over
per-station ratio arrays against the scalar plan of each station, the mixed stream's plan (identity stations at no
latency) against the float64 oracle's per-station streams, the oracle's per-station streams against their whole
records, the filter table, and the argument errors that need no device."""
import numpy as np
import pytest
import torch

from oracle import resample_ref as RR
from seist_b200 import resample as RS

OUT = 100
RATES = [100, 50, 40, 125, 1000, 100, 40]          # 1:1, 100 -> 50, 40 -> 100, 125 -> 100, 1000 -> 100 (at 100 Hz out)


def _schedules(totals, rng, silent):
    """Ragged pushes per station, an empty push and one of a few samples among them, station `silent` only at the end."""
    rows = []
    for s, T in enumerate(totals):
        if s == silent:
            rows.append([0] * 6 + [T])
            continue
        cuts = sorted(rng.integers(0, T + 1, 4).tolist() + [min(3, T)])
        n = np.diff([0] + cuts + [T]).tolist()
        rows.append(n[:1] + [0] + n[1:])
    calls = max(map(len, rows))
    return [r + [0] * (calls - len(r)) for r in rows]


def _run_plans(up, down, hl, sched):
    """The vectorised plans of every call and the close."""
    S = len(sched)
    N, K, plans = np.zeros(S, np.int64), np.zeros(S, np.int64), []
    for c in range(len(sched[0]) + 1):
        n = np.array([r[c] for r in sched]) if c < len(sched[0]) else None
        plans.append(RS.stream_plan(N, K, n, up, down, close=n is None, hl=hl))
        N, K = plans[-1]["N1"], plans[-1]["K1"]
    return plans


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_vectorised_plan_equals_the_scalar_plan_of_each_station(seed):
    rng = np.random.default_rng(seed)
    ratios = [RR.ratio(r, OUT) for r in RATES] + [RR.ratio(100, 50)]
    up, down = np.array([u for u, _ in ratios]), np.array([d for _, d in ratios])
    totals = [int(t) for t in rng.integers(1, 20000, len(ratios))]
    sched = _schedules(totals, rng, silent=2)
    plans = _run_plans(up, down, None, sched)
    for s in range(len(ratios)):
        one = _run_plans(int(up[s]), int(down[s]), None, [sched[s]])
        for c, (p, q) in enumerate(zip(plans, one)):
            for k in ("N0", "lo0", "K0", "lo1", "N1", "K1"):
                assert p[k][s] == q[k][0], (s, c, k)
            for k in ("chunk_off", "out_off"):
                assert np.diff(p[k])[s] == np.diff(q[k])[0], (s, c, k)
    scalar = RS.stream_plan([0, 7], [0, 0], [300, 5], 1, 2)                         # scalar ratios, as before
    assert scalar["K1"].tolist() == [140, 0] and scalar["lo1"].tolist() == [260, 0]


def test_network_plan_equals_the_oracle_stream_of_each_station():
    rng = np.random.default_rng(5)
    rs = RS.Resampler(RATES, OUT)
    totals = [12000, 5003, 1, 37, 20011, 0, 999]
    sched = _schedules(totals, rng, silent=3)
    plans = _run_plans(rs.up, rs.down, rs.half_len, sched)
    for s, fin in enumerate(RATES):
        up, down = RR.ratio(fin, OUT)
        ref = RR.StreamRef(1, 3, up, down)
        recs = rng.standard_normal((3, totals[s]))
        pos, got = 0, []
        for c, n in enumerate([r[s] for r in zip(*sched)] + [None]):
            got += ref.push([recs[:, pos:pos + n]]) if n is not None else ref.close()
            pos += n or 0
            for k, v in ref.calls[-1].items():
                assert plans[c][k][s] == v[0], (s, c, k)
            assert ref.held[0].shape[1] <= rs.held_bound
        # the oracle's per-station stream concatenates to its whole record
        assert np.array_equal(np.concatenate(got, axis=1), RR.resample(recs, up, down)), s
    ident = [s for s, r in enumerate(RATES) if r == OUT]                              # no latency at 1:1
    assert all((p["K1"][ident] == p["N1"][ident]).all() for p in plans)


def test_filter_table():
    rs = RS.Resampler([100, 40, 200, 50, 100, 1000], 50)
    assert rs.up.tolist() == [1, 5, 1, 1, 1, 1] and rs.down.tolist() == [2, 4, 4, 1, 2, 20]
    assert len(rs.table) == 5 and rs.filt[0] == rs.filt[4]
    for s in range(6):
        up, down, hl, nt, off, tile, ident, smem = rs.table[rs.filt[s]].tolist()
        assert (up, down) == (rs.up[s], rs.down[s]) or (ident and rs.up[s] == rs.down[s])
        if ident:
            assert (up, down, hl, nt, tile) == (1, 1, 0, 0, 1024)
            continue
        assert hl == rs.half_len[s] == 10 * max(up, down) and nt == 2 * hl // up + 1 and off % 4 == 0
        assert smem == 4 * (((up * nt + 3) & ~3) + ((tile - 1) * down + 2 * hl) // up + 1) <= rs.smem
    offs = sorted((r[4], r[0] * r[3]) for r in rs.table.tolist())
    assert all(a + n <= b for (a, n), (b, _) in zip(offs, offs[1:]))                  # taps do not overlap
    assert rs.output_lengths([360000, 144000, 1, 2, 3, 10007]).tolist() == [180000, 180000, 1, 2, 2, 501]
    single = RS.Resampler(100, 50)                                                    # the single-rate attributes as before
    assert (single.up, single.down, single.half_len, single.held_bound, single.identity, single.mixed) == (1, 2, 20, 43, False, False)


def test_argument_errors():
    with pytest.raises(ValueError, match="station 2"):
        RS.Resampler([100, 40, 44100], 100)                                          # 441 / 1 at station 2
    for bad in ([100, 0], [100, -40], [100, 50.0], [], [100, True]):
        with pytest.raises(ValueError):
            RS.Resampler(bad, 50)
    rs = RS.Resampler([100, 40, 50], 50)
    with pytest.raises(ValueError):
        rs(torch.zeros(3, 3, 100))                                                    # a tensor into a mixed Resampler
    for bad in ([torch.zeros(3, 10)] * 2, [torch.zeros(3, 10)] * 4, (torch.zeros(3, 10),)):
        with pytest.raises(ValueError):
            rs(bad)                                                                   # a list length other than S
    for S in (2, 4):
        with pytest.raises(ValueError):
            rs.open_stream(S)
