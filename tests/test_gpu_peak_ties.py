"""-m gpu: every device picker on traces with exact height ties, plateaus and NaN (tests/peak_ties.py) against the oracle
that tests/test_cpu_peak_ties.py pins to the reference's `_detect_peaks` with a stable sort, bit for bit (index, value and
offsets): `pick_phase` / `detect_event` (csrc/postproc.cu) up to L = 16384 and topk = 8, `pick_peaks` / `detect_runs` on
rows of 2^20 samples at the cluster kernels' size boundaries, `RaggedPickStream` with splits on tied clusters, and
`pick_segments` on records whose gaps cut through them."""
from functools import lru_cache

import numpy as np
import pytest
import torch

import peak_ties as PT
from oracle import postprocess_ref as PR
from oracle import stream_ref as SR
from seist_b200 import postprocess as PP
from seist_b200 import stream as ST

pytestmark = pytest.mark.gpu

MPDS = (2, 7, 100)
THR = {1: 0.7, 2: 0.3}        # pick channel -> threshold; detections at 0.7
DET = 0.7


@pytest.mark.parametrize("L", [3, 4096, 12289, 16384])       # 12289: the first pick row past 48 KB; 16384: the largest
def test_pick_phase_and_detect_event_with_ties(L):
    N = 24
    x = np.zeros((N, 3, L), np.float32)
    for mpd in (2, 7, 50):
        for i in range(N):
            x[i, 0] = PT.short_trace(1000 + i, L, mpd, i % 3 == 1)
            x[i, 1] = PT.short_trace(i, L, mpd, i % 3 == 2)
            x[i, 2] = PT.short_trace(2000 + i, L, mpd, i % 2 == 0)
        if L >= 4096:          # more equal-height candidates than the largest topk
            c = PT.candidates(x[0, 1], THR[1])
            assert (x[0, 1, c] == x[0, 1, c].max()).sum() > 8
        xg = torch.from_numpy(x).cuda()
        for topk in range(1, 9):
            for ch, thr in THR.items():
                got = PP.pick_phase(xg, ch, thr, mpd, topk).cpu().numpy()
                want = PR.pick_phase(x[:, ch], thr, mpd, topk)
                assert np.array_equal(got, want), (mpd, topk, ch, np.argwhere(got != want)[:4])
            for thr in (DET, 0.3):
                got = PP.detect_event(xg, 0, thr, topk).cpu().numpy()
                want = PR.detect_event(x[:, 0], thr, topk)
                assert np.array_equal(got, want), (topk, thr, np.argwhere(got != want)[:4])


def test_postprocess_argument_rejections():
    ok = torch.zeros(2, 3, 16384, device="cuda")
    PP.pick_phase(ok, 1, 0.5, 2, 8)
    PP.detect_event(ok, 0, 0.5, 8)
    long = torch.zeros(2, 3, 16385, device="cuda")
    for call in (lambda: PP.pick_phase(long, 1, 0.5, 2, 1), lambda: PP.pick_phase(ok, 1, 0.5, 2, 9),
                 lambda: PP.pick_phase(ok, 1, 0.5, 1, 1), lambda: PP.detect_event(long, 0, 0.5, 1),
                 lambda: PP.detect_event(ok, 0, 0.5, 9)):
        with pytest.raises(RuntimeError):
            call()


def test_counters_at_their_edges():
    pad = PR.PAD_PHASE
    t = torch.tensor([[99], [99], [50], [50], [pad], [10], [100], [0]])
    p = torch.tensor([[99], [100], [55], [44], [10], [pad], [99], [-1]])
    td = torch.tensor([[0, 3, 10, 12], [1, 0, 1, 0], [5, 40, 1, 0]])
    pd = torch.tensor([[2, 5, 4, 11, 1, 0], [0, 31, 1, 0, 1, 0], [-10, 6, 6, 6, 30, 31]])
    for n, thr in ((100, 5), (32, 0)):
        ctr = PP.StepCounters(["ppk", "det"], n, thr, "cuda")
        ctr.update("ppk", t.cuda(), p.cuda())
        ctr.update("det", td.cuda(), pd.cuda())
        got = ctr.result()
        for task, want in (("ppk", PR.pick_counters(t.numpy(), p.numpy(), n, thr)), ("det", PR.det_counters(td.numpy(), pd.numpy(), n))):
            for k, v in want.items():
                assert got[task][k] == v, (n, task, k, got[task][k], v)


# ---- rows of 2^20 samples ---------------------------------------------------------------------------------------------
@lru_cache(maxsize=1)
def _rows():
    x, marks = PT.long_rows()
    return np.ascontiguousarray(np.broadcast_to(x[:, None], (x.shape[0], 3, x.shape[1]))), marks


@lru_cache(maxsize=None)
def _want(s, n, ch, mpd):
    """The oracle's picks of row s's first n samples on channel ch, and each pick's cluster end."""
    row = _rows()[0][s, ch, :n]
    idx = SR.detect_peaks_all(row, THR[ch], mpd)
    last = PT.cluster_last(row, THR[ch], mpd)
    return idx, row[idx], np.array([last[int(i)] for i in idx], np.int64)


@lru_cache(maxsize=None)
def _want_runs(s, n):
    return np.array(PR.trigger_runs(_rows()[0][s, 0, :n], DET), np.int64).reshape(-1, 2)


@pytest.mark.parametrize("mpd", MPDS)
def test_whole_record_pickers(mpd):
    probs, _ = _rows()
    S, _, T = probs.shape
    pg = torch.from_numpy(probs).cuda()
    got = ST.pick_peaks(pg, (1, 2), (THR[1], THR[2]), mpd)
    for (index, value, off), ch in zip(got, (1, 2)):
        want = [_want(s, T, ch, mpd) for s in range(S)]
        assert off.tolist() == np.cumsum([0] + [w[0].size for w in want]).tolist(), (mpd, ch)
        assert np.array_equal(index.cpu().numpy(), np.concatenate([w[0] for w in want])), (mpd, ch)
        assert np.array_equal(value.cpu().numpy(), np.concatenate([w[1] for w in want])), (mpd, ch)
    pairs, off = ST.detect_runs(pg, 0, DET)
    want = [_want_runs(s, T) for s in range(S)]
    assert off.tolist() == np.cumsum([0] + [w.shape[0] for w in want]).tolist()
    assert np.array_equal(pairs.cpu().numpy(), np.concatenate(want))


def _splits(s, n, mpd, rng, marks):
    """Cut points of row s (n samples): on a tied candidate, inside a plateau, at c + mpd + 1 and c + mpd + 2 of a tied
    cluster's last candidate c, and random ones."""
    m = marks[s]
    cuts = set(rng.integers(1, n, 12).tolist())
    for name, a in m.items():
        cuts |= {a, a + 1, a + 2}                                     # on / just past a tied candidate or plateau start
    probs = _rows()[0]
    for ch in (1, 2):
        last = PT.cluster_last(probs[s, ch, :n], THR[ch], mpd)
        for name, a in m.items():
            if a in last:
                c = last[a]
                cuts |= {c + mpd + 1, c + mpd + 2}
    return sorted(c for c in cuts if 0 < c < n)


def _check_calls(outs, finals, lengths, t0, mpd):
    """The concatenated picks and runs of every row equal the whole-row oracle; after each call but the last, exactly
    the picks whose cluster ends at c with c + mpd <= F - 2 (F: the row's final count) have been returned."""
    for s, n in enumerate(lengths):
        for k, ch in ((0, 1), (1, 2)):
            idx = [o[k][0][o[k][2][s]:o[k][2][s + 1]] for o in outs]
            val = [o[k][1][o[k][2][s]:o[k][2][s + 1]] for o in outs]
            want, wval, wlast = _want(s, n, ch, mpd)
            assert np.array_equal(np.concatenate(idx), want + t0[s]), (mpd, s, ch)
            assert np.array_equal(np.concatenate(val), wval), (mpd, s, ch)
            done = np.cumsum([i.size for i in idx])
            for c, F in enumerate(finals[s][:-1]):
                assert done[c] == int((wlast + mpd <= F - 2).sum()), (mpd, s, ch, c, F)
        pairs = np.concatenate([o[2][0][o[2][1][s]:o[2][1][s + 1]] for o in outs]).reshape(-1, 2)
        assert np.array_equal(pairs, _want_runs(s, n) + t0[s]), (mpd, s)


def _np(out):
    return tuple(tuple(t.cpu().numpy() for t in csr) for csr in out)


@pytest.mark.parametrize("mpd", MPDS)
def test_ragged_pick_stream_dense_pushes(mpd):
    probs, marks = _rows()
    S, _, T = probs.shape
    pg = torch.from_numpy(probs).cuda()
    cuts = _splits(0, T, mpd, np.random.default_rng(mpd), marks) + [T]
    pk = ST.RaggedPickStream(S, "cuda", mpd, THR[1], THR[2], DET)
    outs, a = [], 0
    for b in cuts:
        outs.append(_np(pk.push(pg[:, :, a:b].contiguous())))
        a = b
    outs.append(_np(pk.close()))
    _check_calls(outs, [cuts + [T]] * S, [T] * S, [0] * S, mpd)


@pytest.mark.parametrize("mpd", MPDS)
def test_ragged_pick_stream_per_station_pushes(mpd):
    """Rows of different lengths, each cut at its own landmarks; row 3 silent for its first calls; row 2's global sample
    indices cross 2^31."""
    probs, marks = _rows()
    S, _, T = probs.shape
    lengths = [T, T - 1, 600_001, T - 4096, 300_000]
    t0 = [0, 5, (1 << 31) - 50_000, 0, 17]
    rng = np.random.default_rng(100 + mpd)
    cuts = [_splits(s, n, mpd, rng, marks) + [n] for s, n in enumerate(lengths)]
    cuts[3] = [0] * 6 + cuts[3]
    calls = max(len(c) for c in cuts)
    cuts = [c + [c[-1]] * (calls - len(c)) for c in cuts]
    pg = torch.from_numpy(probs).cuda()
    pk = ST.RaggedPickStream(S, "cuda", mpd, THR[1], THR[2], DET, t0=t0)
    outs, a = [], [0] * S
    for c in range(calls):
        outs.append(_np(pk.push([pg[s, :, a[s]:cuts[s][c]].contiguous() for s in range(S)])))
        a = [cuts[s][c] for s in range(S)]
    outs.append(_np(pk.close()))
    _check_calls(outs, [c + [c[-1]] for c in cuts], lengths, t0, mpd)
    last = np.concatenate([o[k][0][o[k][2][2]:o[k][2][3]] for o in outs for k in (0, 1)])
    assert (last >= 1 << 31).any() and (last < 1 << 31).any()


@pytest.mark.parametrize("mpd", MPDS)
def test_pick_segments_through_ties(mpd):
    """Segments from gap_segments of a record whose gaps cut through plateaus and tied clusters (and sit wherever the
    probabilities are NaN): each annotated segment's picks are `detect_peaks_all` of its own slice, shifted by its start."""
    probs, marks = _rows()
    probs = probs.copy()
    S, _, T = probs.shape
    gap = np.isnan(probs[:, 0])
    m0, m1 = marks[0], marks[1]
    for s, a, w in ((0, m0["plateau1.0_1"] + 1, 1), (0, m0["cluster33"] + 20, 3), (0, m0["chain7"] + 14, 2),
                    (1, m1["seg_cross"] + 10, 1), (1, m1["cluster4097"] + 4001, 5), (2, 8192, 1), (3, T // 2, 100),
                    (4, 50_000, 1), (4, 50_003, 1)):
        gap[s, a:a + w] = True
    rec = np.where(gap[:, None], np.float32(np.nan), np.float32(1.0)).repeat(3, 1)
    probs[np.broadcast_to(gap[:, None], probs.shape)] = np.nan
    segs = ST.gap_segments(torch.from_numpy(rec).cuda(), 3)
    got = ST.pick_segments(torch.from_numpy(probs).cuda(), segs, (THR[1], THR[2]), mpd)
    offs = segs.host_offsets
    for (index, value, off), ch in zip(got, (1, 2)):
        widx, wval, count = [], [], [0]
        for s in range(S):
            n = 0
            for on, e in zip(segs.on[offs[s]:offs[s + 1]], segs.off[offs[s]:offs[s + 1]]):
                if e - on + 1 >= 3:
                    i = SR.detect_peaks_all(probs[s, ch, on:e + 1], THR[ch], mpd)
                    widx.append(i + on)
                    wval.append(probs[s, ch, on + i])
                    n += i.size
            count.append(count[-1] + n)
        assert off.tolist() == count, (mpd, ch)
        assert np.array_equal(index.cpu().numpy(), np.concatenate(widx)), (mpd, ch)
        assert np.array_equal(value.cpu().numpy(), np.concatenate(wval)), (mpd, ch)
