"""-m gpu: streams with data gaps (seist_b200/stream.py GapStream, `gap_stream_segments`, csrc/stream.cu seist_gap_stream_*,
DESIGN §4.22).  The scan against numpy on packed blocks (empty and one-sample blocks, NaN in one channel, +-Inf, gaps at
both ends, more than 65 536 segments in one push); end to end with seist_s_dpk, every station's concatenated output
bit-identical to `annotate` with segments of its own record (NaN at the same samples), its picks to `pick_phases` with
segments (a gap shorter than min_peak_dist included) and its runs to `detect_events`, each call's finality and replays
against the oracle (tests/gap_stream_ref.py); gap-free input against RaggedStream call by call; the synchronisation
budgets, argument errors and the memory held over 50 pushes."""
import numpy as np
import pytest
import torch

import gap_stream_ref as GSR
from oracle import golden as G
from seist_b200 import _lib
from seist_b200 import stream as ST
from seist_b200.models import create_model
from test_cpu_gap_stream import _pieces
from test_gpu_gaps import _record, _syncs

pytestmark = pytest.mark.gpu

NAN = float("nan")
W = 8192


@pytest.fixture(scope="module")
def model():
    m = create_model("seist_s_dpk", in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict("seist_s_dpk", W), strict=True)
    return m.cuda().eval()


def _annotator(model, stride=4096, stack="mean", batch=3):
    ann = ST.ContinuousAnnotator(model, window=W, stride=stride, batch=batch, stack=stack)
    ann.min_peak_dist = 100
    ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
    return ann


def _gapped(seed=5):
    """Five stations: random gaps; gap free; all NaN; one 50-sample gap; gaps at 0 and T - 1 with segments of W - 1, W."""
    T = 5 * W + 1234
    rec = _record(5, 3, T, 31)
    rng = np.random.default_rng(seed)
    for _ in range(6):
        a = int(rng.integers(0, T))
        rec[0, :, a:a + int(rng.integers(1, 3000))] = NAN
    rec[2] = NAN
    rec[3, :, 20000:20050] = NAN
    rec[4, :, 0] = NAN
    rec[4, 2, T - 1] = NAN
    rec[4, 0, W] = NAN
    rec[4, 1, 2 * W + 1] = float("inf")
    return rec


def _schedule(S, T, kind, seed=0):
    if kind == "equal":
        return [np.full(S, min(6000, T - r)) for r in range(0, T, 6000)]
    rng = np.random.default_rng(seed)
    out, left = [], np.full(S, T)
    while left.any():
        n = np.minimum(left, rng.choice([0, 1, 777, 5000, 9000, 17000, 30000], size=S))
        out.append(n)
        left -= n
    return out


def _push(st, rec, R, n):
    return st.push([rec[s, :, R[s]:R[s] + n[s]].contiguous() for s in range(rec.shape[0])])


def _station_csr(csr, s):
    *vals, off = csr
    o = off.cpu().numpy()
    return [v[o[s]:o[s + 1]].cpu() for v in vals]


def _blocks(n, seed, gaps=40):
    rng = np.random.default_rng(seed)
    blocks = [rng.standard_normal((3, k)).astype(np.float32) for k in n]
    for b in blocks:
        if b.shape[1] == 0:
            continue
        for _ in range(int(rng.integers(0, gaps))):
            a = int(rng.integers(0, b.shape[1]))
            b[rng.integers(0, 3) if rng.random() < 0.3 else slice(None), a:a + int(rng.integers(1, 50))] = \
                rng.choice([np.nan, np.inf, -np.inf])
    return blocks


def _scan(blocks):
    chunk = torch.from_numpy(np.concatenate([b.reshape(-1) for b in blocks])).cuda()
    return ST.gap_stream_segments(chunk, ST._prefix([b.shape[1] for b in blocks]), 3)


@pytest.mark.parametrize("seed", range(3))
def test_scan_matches_numpy_on_packed_blocks(seed):
    n = [0, 1, 5000, 70000, 3, 4097, 4096, 2]
    blocks = _blocks(n, seed)
    blocks[4][:, 1] = np.nan                                            # [0, 0] and [2, 2]
    blocks[5][:, 0] = np.nan
    blocks[5][1, -1] = np.inf                                           # gaps at both ends
    blocks[7][:] = np.nan                                               # all gap
    for g, w in zip(_scan(blocks), _pieces(blocks)):
        assert np.array_equal(g, w)


def test_scan_reads_more_than_65536_segments():
    b = np.ones((3, 300001), np.float32)
    b[0, 1::2] = np.nan                                                 # 150 001 one-sample segments
    blocks = [np.ones((3, 7), np.float32), b]
    got = _scan(blocks)
    assert len(got[0]) == 150002
    for g, w in zip(got, _pieces(blocks)):
        assert np.array_equal(g, w)


def test_argument_errors_raise_before_any_launch():
    lib = _lib.lib()
    x = torch.ones(3 * 10, device="cuda")
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        ST.gap_stream_segments(x, [0, 5, 11], 3)                        # past the chunk
    with pytest.raises(ValueError):
        ST.gap_stream_segments(x, [0, 6, 5], 3)                         # negative length
    with pytest.raises(ValueError):
        ST.gap_stream_segments(x.double(), [0, 10], 3)
    with pytest.raises(RuntimeError):
        ST.gap_stream_segments(x.cpu(), [0, 10], 3)
    assert lib.seist_launch_count() == before
    z = ST.gap_stream_segments(x, [0, 0, 0], 3)
    assert all(len(v) == 0 for v in z) and lib.seist_launch_count() == before


@pytest.mark.parametrize("stride", [4096, 3000])
@pytest.mark.parametrize("stack", ["mean", "max"])
@pytest.mark.parametrize("kind", ["equal", "ragged"])
def test_end_to_end_equals_whole_record_with_segments(model, stride, stack, kind):
    rec = _gapped()
    S, C, T = rec.shape
    ann = _annotator(model, stride, stack)
    st = ann.open_gap_stream(S)
    outs, R = [], np.zeros(S, np.int64)
    rec_np = rec.cpu().numpy()
    for n in _schedule(S, T, kind, seed=stride) + [None]:
        f = st.forwards
        out = st.close() if n is None else _push(st, rec, R, n)
        R1 = R if n is None else R + n
        n_win = 0
        for s in range(S):                                              # clause 4: what the call makes final
            t0, m, win = GSR.call(rec_np[s, :, :R[s]], rec_np[s, :, :R1[s]], W, stride, n is None)
            assert (out.t0[s], out.probs[s].shape[1]) == (t0, m)
            n_win += len(win)
        assert st.forwards - f == -(-n_win // ann.batch)                # clause 7: replays
        outs.append(out)
        R = R1
    assert st.closed
    for s in range(S):
        one = rec[s:s + 1].contiguous()
        segs = ann.segments(one)
        want = ann.annotate(one, segments=segs)
        got = torch.cat([o.probs[s] for o in outs], 1)
        assert got.shape == want[0].shape
        nan = torch.isnan(want[0])
        assert torch.equal(torch.isnan(got), nan), s
        assert torch.equal(got[~nan], want[0][~nan]), s
        pk = ann.pick_phases(want, segments=segs)
        det = ann.detect_events(want)
        for k in ("ppk", "spk"):
            parts = [_station_csr(getattr(o, k), s) for o in outs]
            for v in range(2):
                assert torch.equal(torch.cat([p[v] for p in parts]), _station_csr(pk[k], 0)[v]), (s, k)
        parts = [_station_csr(o.det, s)[0] for o in outs]
        assert torch.equal(torch.cat(parts).reshape(-1, 2), _station_csr(det, 0)[0]), s


def test_gap_free_equals_ragged_stream_call_by_call(model):
    rec = _record(4, 3, 3 * W + 999, 7)
    S, _, T = rec.shape
    ann = _annotator(model, 3000)
    a, b = ann.open_gap_stream(S), ann.open_ragged_stream(S)
    R = np.zeros(S, np.int64)
    for n in _schedule(S, T, "ragged", 3) + [None]:
        oa = a.close() if n is None else _push(a, rec, R, n)
        ob = b.close() if n is None else _push(b, rec, R, n)
        assert oa.t0 == ob.t0 and a.forwards == b.forwards
        for s in range(S):
            assert torch.equal(oa.probs[s], ob.probs[s])
        for k in ("ppk", "spk", "det"):
            for x, y in zip(getattr(oa, k), getattr(ob, k)):
                assert torch.equal(x, y), k
        R = R if n is None else R + n


def test_sync_budgets_and_short_stations_at_close(model):
    rec = _gapped()
    S = rec.shape[0]
    ann = _annotator(model)
    st = ann.open_gap_stream(S)
    R = np.zeros(S, np.int64)
    for n in ([7000, 7000, 7000, 7000, 0], [3000, 1, 12000, 40, 9000]):
        n = np.array(n)
        _, k = _syncs(lambda: _push(st, rec, R, n))
        assert k == 2
        R += n
    out, k = _syncs(st.close)                                           # stations 1 and 3 end in short segments
    assert k == 1
    assert [p.shape[1] for p in out.probs] == (R - np.array(out.t0)).tolist()


def test_stream_argument_errors_leave_the_stream_usable(model):
    ann = _annotator(model)
    with pytest.raises(ValueError):
        ann.open_gap_stream(32768)
    with pytest.raises(ValueError):
        ST.ContinuousAnnotator(model, window=W, batch=3).open_gap_stream(2)
    st = ann.open_gap_stream(2)
    lib = _lib.lib()
    ok = torch.randn(3, 100, device="cuda")
    before = lib.seist_launch_count()
    for chunks, err in (([ok], ValueError), ([ok, ok.cpu()], RuntimeError), ([ok, ok.double()], ValueError),
                        ([ok, ok[:2]], ValueError), ([ok, ok.t().contiguous().t()], ValueError)):
        with pytest.raises(err):
            st.push(chunks)
    assert lib.seist_launch_count() == before
    st.push([ok, ok])
    st.close()
    with pytest.raises(RuntimeError):
        st.push([ok, ok])
    with pytest.raises(RuntimeError):
        st.close()


def test_memory_held_does_not_grow(model):
    ann = _annotator(model, batch=8)
    S = 3
    st = ann.open_gap_stream(S)
    g = torch.Generator().manual_seed(0)
    marks = []
    for i in range(50):
        x = torch.randn(S, 3, 3000, generator=g)
        x[:, :, (i * 37) % 2900:(i * 37) % 2900 + 40] = NAN
        st.push(list(x.cuda().unbind(0)))
        torch.cuda.synchronize()
        if i in (10, 49):
            marks.append(torch.cuda.memory_allocated())
    assert marks[1] <= marks[0] + (1 << 20)
    st.close()
