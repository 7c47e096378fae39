"""Polyphase resampling on the host (seist_b200/resample.py, oracle/resample_ref.py, DESIGN §4.24): the numpy taps against
scipy's firwin, the float64 oracle against scipy's resample_poly, the oracle's stream restatement against its whole-record
result under random ragged schedules (and the package's stream plan against the oracle's), and the argument errors that
need no device."""
import numpy as np
import pytest
import torch
from scipy import signal

from oracle import resample_ref as RR
from seist_b200 import resample as RS

PAIRS = [(100, 50), (200, 100), (500, 100), (1000, 100), (250, 100), (125, 100), (80, 100), (40, 100), (50, 100), (100, 100),
         (20, 100)]
EXTREME = [(1, 256), (256, 1), (3, 256)]                         # the largest ratios accepted


@pytest.mark.parametrize("fin,fout", [p for p in PAIRS + EXTREME if p[0] != p[1]])   # resample_poly designs no filter for 1:1
def test_taps_match_firwin(fin, fout):
    up, down = RR.ratio(fin, fout)
    L = max(up, down)
    want = signal.firwin(20 * L + 1, 1.0 / L, window=("kaiser", 5.0)) * up
    assert np.abs(RS.design_taps(up, down) - want).max() <= 1e-15 * max(1, up)
    assert np.abs(RR.taps(up, down) - want).max() <= 1e-15 * max(1, up)
    table = RS.polyphase_taps(up, down)                           # phase-major, ascending input index
    hl = 10 * L
    assert table.dtype == np.float32 and table.shape == (up, 2 * hl // up + 1)
    for phi in range(up):
        n = (2 * hl - phi) // up + 1
        assert np.array_equal(table[phi, :n], want[phi::up][::-1].astype(np.float32)) and not table[phi, n:].any()


@pytest.mark.parametrize("fin,fout", PAIRS)
def test_oracle_matches_resample_poly(fin, fout):
    up, down = RR.ratio(fin, fout)
    rng = np.random.default_rng(fin * 1000 + fout)
    hl = 10 * max(up, down)
    for T in (1, 2, hl // 3 + 1, 2 * hl - 1, 9999, 10001):
        x = rng.standard_normal((2, 3, T)) * 7 + 1
        want = signal.resample_poly(x, up, down, axis=-1)
        got = RR.resample(x, up, down)
        assert got.shape == want.shape == (2, 3, -(-T * up // down))
        assert np.abs(got - want).max() <= 1e-12 * np.abs(x).max(), (T, np.abs(got - want).max())


def _schedule(T, calls, rng):
    cuts = sorted(rng.integers(0, T + 1, max(0, calls - 3)).tolist() + [min(1, T), min(2, T)])
    n = np.diff([0] + cuts + [T]).tolist()
    n.insert(int(rng.integers(0, len(n) + 1)), 0)
    return n


@pytest.mark.parametrize("fin,fout", PAIRS)
def test_oracle_stream_concatenates_to_the_whole_record(fin, fout):
    up, down = RR.ratio(fin, fout)
    rng = np.random.default_rng(fin + 7 * fout)
    totals = [0, 1, 37, 5003, 12000]                              # a station silent throughout, one sample, short, long
    recs = [rng.standard_normal((3, T)) for T in totals]
    rows = [_schedule(T, 9, rng) for T in totals]
    calls = max(len(r) for r in rows)
    rows = [r + [0] * (calls - len(r)) for r in rows]
    ref = RR.StreamRef(len(totals), 3, up, down)
    got = [[] for _ in totals]
    N, K = np.zeros(len(totals), np.int64), np.zeros(len(totals), np.int64)
    for c in range(calls + 1):
        if c < calls:
            n = np.array([rows[s][c] for s in range(len(totals))])
            outs = ref.push([recs[s][:, N[s]:N[s] + n[s]] for s in range(len(totals))])
        else:
            n, outs = None, ref.close()
        if up != down:                                            # the package's plan is the oracle's call
            plan = RS.stream_plan(N, K, n, up, down, close=n is None)
            for k, v in ref.calls[-1].items():
                assert np.array_equal(plan[k], v), (c, k)
            assert np.array_equal(np.diff(plan["out_off"]), plan["K1"] - plan["K0"])
        for s, y in enumerate(outs):
            got[s].append(y)
        N, K = ref.N.copy(), ref.K.copy()
    for s, rec in enumerate(recs):
        whole = RR.resample(rec, up, down)
        assert np.array_equal(np.concatenate(got[s], axis=1), whole), s


def test_stream_finality_and_latency():
    up, down = 1, 2                                               # 100 -> 50 Hz: 20 input samples of latency
    plan = RS.stream_plan([0], [0], [100], up, down)
    assert plan["K1"].tolist() == [40] and 39 * down + 20 < 100 <= 40 * down + 20
    plan = RS.stream_plan([100], [40], [0], up, down, close=True)
    assert plan["K1"].tolist() == [50] and plan["lo0"].tolist() == [60]
    with pytest.raises(ValueError):
        RS.stream_plan([0, 0], [0, 0], [3, -1], up, down)


def test_argument_errors():
    for a, b in ((0, 50), (-100, 50), (100, 0), (100.0, 50), (True, 50), ("100", 50)):
        with pytest.raises(ValueError):
            RS.Resampler(a, b)
    for a, b in ((257, 256), (1, 300), (44100, 100), (48000, 100)):   # reduced ratio beyond 256
        with pytest.raises(ValueError):
            RS.Resampler(a, b)
    rs = RS.Resampler(200, 100)
    assert (rs.up, rs.down, rs.half_len, rs.held_bound) == (1, 2, 20, 43)
    assert (RS.Resampler(np.int64(25600), 100).down, RS.Resampler(1, 256).up) == (256, 256)
    with pytest.raises(ValueError):
        RS.Resampler(100, 50, device="cpu")
    for bad in (torch.zeros(2, 3, 10), torch.zeros(2, 3, 10, dtype=torch.float64), torch.zeros(3, 10), torch.zeros(2, 3, 0),
                torch.zeros(2, 3, 10).transpose(1, 2), np.zeros((2, 3, 10), np.float32)):
        with pytest.raises(ValueError):
            rs(bad)
