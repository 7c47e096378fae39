"""-m gpu: polyphase resampling on the device (seist_b200/resample.py, csrc/resample.cu, DESIGN §4.24).  Whole records
against the float64 oracle (oracle/resample_ref.py) within 1e-5 * max|x| of the row, an hour of four stations included;
streams against the whole record bit for bit under equal tensor pushes and ragged list pushes (empty pushes, pushes
shorter than the latency, a station silent until the close); the NaN rule exactly; 100 Hz records through a resampling
stream into the seist_s_dpk annotator's ragged and gap streams against `annotate` of the resampled record; the host
synchronisation and memory budgets of a push and the argument errors."""
import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import resample_ref as RR
from seist_b200 import _lib
from seist_b200 import resample as RS
from seist_b200.models import create_model
from test_gpu_gap_stream import _station_csr
from test_gpu_gaps import _syncs
from test_gpu_stream_ragged import _annotator, _check_station

pytestmark = pytest.mark.gpu

PAIRS = [(100, 50), (200, 100), (500, 100), (1000, 100), (250, 100), (125, 100), (80, 100), (40, 100), (50, 100), (100, 100)]
W = 8192


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g, dtype=torch.float64) * (0.5 + 10 * torch.rand(S, C, 1, generator=g, dtype=torch.float64))
    return (x + torch.randn(S, C, 1, generator=g, dtype=torch.float64)).float()


def _close_to_oracle(x, y, up, down):
    want = RR.resample(x.double().numpy(), up, down)
    got = y.cpu().double().numpy()
    assert got.shape == want.shape
    scale = np.abs(x.double().numpy()).max(axis=-1, keepdims=True)
    err = np.abs(got - want) / scale
    assert err.max() <= 1e-5, err.max()


@pytest.mark.parametrize("fin,fout", PAIRS)
def test_whole_record_matches_oracle(fin, fout):
    rs = RS.Resampler(fin, fout)
    for shape in ((2, 3, 10007), (1, 3, 1), (3, 3, 2), (1, 1, 77), (5, 3, 4096)):
        x = _record(*shape, seed=sum(shape))
        y = rs(x.cuda())
        torch.cuda.synchronize()
        _close_to_oracle(x, y, rs.up, rs.down)


def test_an_hour_of_four_stations_matches_oracle():
    rs = RS.Resampler(100, 50)
    x = _record(4, 3, 360000, 3)
    _close_to_oracle(x, rs(x.cuda()), rs.up, rs.down)


def _ragged_schedule(T, rng, silent=False):
    if silent:
        return [0, 0, 0, 0, T]
    cuts = sorted(rng.integers(0, T + 1, 5).tolist() + [1, 2, 3])
    n = np.diff([0] + cuts + [T]).tolist()
    return n[:2] + [0, 5] + n[2:]             # an empty push and one shorter than the latency


@pytest.mark.parametrize("fin,fout", PAIRS)
def test_stream_equals_whole_record_bit_for_bit(fin, fout):
    rs = RS.Resampler(fin, fout)
    rng = np.random.default_rng(fin + fout)
    totals = [12345, 9000, 1, 4444]
    recs = [_record(1, 3, T, 40 + s)[0].cuda() for s, T in enumerate(totals)]
    whole = [rs(r[None])[0] for r in recs]
    # ragged list pushes: station 3 silent until the close
    scheds = [_ragged_schedule(T, rng, silent=(s == 3)) for s, T in enumerate(totals)]
    calls = max(map(len, scheds))
    scheds = [sc + [0] * (calls - len(sc)) for sc in scheds]
    st = rs.open_stream(len(totals))
    got, pos = [[] for _ in totals], [0] * len(totals)
    for c in range(calls):
        out = st.push([recs[s][:, pos[s]:pos[s] + scheds[s][c]].contiguous() for s in range(len(totals))])
        for s in range(len(totals)):
            got[s].append(out[s])
            pos[s] += scheds[s][c]
    for s, y in enumerate(st.close()):
        got[s].append(y)
    for s in range(len(totals)):
        assert torch.equal(torch.cat(got[s], 1), whole[s]), s
    # equal tensor pushes, the chunk shorter than the filter's latency included
    x = torch.stack([r[:, :9000] for r in recs[:2]]).contiguous()
    want = rs(x)
    for n in (1000, 7, 333):
        st = rs.open_stream(2)
        parts = [st.push(x[:, :, a:a + n].contiguous()) for a in range(0, 9000, n)] + [st.close()]
        assert all(torch.is_tensor(p) and p.shape[:2] == (2, 3) for p in parts)
        assert torch.equal(torch.cat(parts, 2), want), n


@pytest.mark.parametrize("fin,fout", [(100, 50), (40, 100), (125, 100)])
def test_nan_propagates_exactly_over_the_support(fin, fout):
    rs = RS.Resampler(fin, fout)
    x = _record(2, 3, 20000, 9)
    clean = rs(x.cuda())
    gapped = x.clone()
    gapped[0, :, 5000:5300] = float("nan")
    gapped[0, 1, 9000] = float("nan")
    gapped[1, :, :40] = float("nan")
    gapped[1, 2, 19990:] = float("nan")
    y = rs(gapped.cuda())
    want = RR.resample(gapped.double().numpy(), rs.up, rs.down)
    nan = torch.from_numpy(np.isnan(want)).cuda()
    assert torch.equal(torch.isnan(y), nan)
    assert torch.equal(y[~nan], clean[~nan])
    st = rs.open_stream(2)                                             # and through a stream
    parts = [st.push(gapped[:, :, a:a + 3001].contiguous().cuda()) for a in range(0, 20000, 3001)] + [st.close()]
    assert torch.equal(torch.isnan(torch.cat(parts, 2)), nan) and torch.equal(torch.cat(parts, 2)[~nan], y[~nan])


@pytest.fixture(scope="module")
def model():
    m = create_model("seist_s_dpk", in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict("seist_s_dpk", W), strict=True)
    return m.cuda().eval()


def test_resampled_ragged_stream_equals_annotate_of_the_resampled_record(model):
    rs = RS.Resampler(100, 50)
    ann = _annotator(model, 4096, 4)
    totals = [4 * W + 3001, 2 * W + 17, 3 * W]                       # 100 Hz samples
    recs = [_record(1, 3, T, 70 + s)[0].cuda() for s, T in enumerate(totals)]
    rng = np.random.default_rng(1)
    scheds = [_ragged_schedule(T, rng) for T in totals]
    calls = max(map(len, scheds))
    scheds = [sc + [0] * (calls - len(sc)) for sc in scheds]
    st, ast = rs.open_stream(len(totals)), ann.open_ragged_stream(len(totals))
    outs, pos = [], [0] * len(totals)
    for c in range(calls):
        outs.append(ast.push(st.push([recs[s][:, pos[s]:pos[s] + scheds[s][c]].contiguous() for s in range(len(totals))])))
        pos = [p + sc[c] for p, sc in zip(pos, scheds)]
    outs.append(ast.push(st.close()))
    outs.append(ast.close())
    for s, rec in enumerate(recs):
        _check_station(ann, outs, rs(rec[None])[0], s)


def test_resampled_gap_stream_equals_annotate_with_segments(model):
    rs = RS.Resampler(100, 50)
    ann = _annotator(model, 4096, 3)
    S, T = 3, 5 * W + 999
    rec = _record(S, 3, T, 12)
    rec[0, :, 7000:9000] = float("nan")
    rec[1, 2, 30000:30050] = float("inf")
    rec[2, :, 100:130] = float("nan")
    rec = rec.cuda()
    st, gst = rs.open_stream(S), ann.open_gap_stream(S)
    outs, n = [], 6007
    for a in range(0, T, n):
        outs.append(gst.push(list(st.push(rec[:, :, a:a + n].contiguous()))))
    outs.append(gst.push(list(st.close())))
    outs.append(gst.close())
    y = rs(rec)
    for s in range(S):
        one = y[s:s + 1].contiguous()
        segs = ann.segments(one)
        want = ann.annotate(one, segments=segs)
        got = torch.cat([o.probs[s] for o in outs], 1)
        nan = torch.isnan(want[0])
        assert torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan], want[0][~nan]), s
        pk = ann.pick_phases(want, segments=segs)
        for k in ("ppk", "spk"):
            parts = [_station_csr(getattr(o, k), s) for o in outs]
            for v in range(2):
                assert torch.equal(torch.cat([p[v] for p in parts]), _station_csr(pk[k], 0)[v]), (s, k)
        det = ann.detect_events(want)
        parts = [_station_csr(o.det, s)[0] for o in outs]
        assert torch.equal(torch.cat(parts).reshape(-1, 2), _station_csr(det, 0)[0]), s


def test_push_budgets_and_argument_errors():
    rs = RS.Resampler(100, 50)
    st = rs.open_stream(2)
    held = [h.data_ptr() for h in st.held]
    x = _record(2, 3, 50000, 5).cuda()
    st.push(x[:, :, :10].contiguous())                                 # uploads the taps
    lib = _lib.lib()
    for n in (1, 20000, 0, 29989):
        a = int(st.N[0])
        before = lib.seist_launch_count()
        _, k = _syncs(lambda: st.push(x[:, :, a:a + n].contiguous()))
        assert k == 0 and lib.seist_launch_count() - before == 1
        _, k = _syncs(lambda: st.push([x[0, :, a + n:a + n], x[1, :, a + n:a + n]]))
        assert k == 0
    assert sorted(h.data_ptr() for h in st.held) == sorted(held) and all(h.shape == (2, 3, rs.held_bound) for h in st.held)
    before = lib.seist_launch_count()
    for bad in ([x[0, :, :5].contiguous()], [x[0, :, :5].contiguous(), x[1, :2, :5].contiguous()], x[:1, :, :5].contiguous(),
                x[:, :, :5].double(), x[:, :, :5].cpu(), [x[0, :, :5].contiguous(), x[1, :, :5].t().contiguous().t()]):
        with pytest.raises(ValueError):
            st.push(bad)
    st.push([x[0, :, :5].contiguous(), x[1, :, :0].contiguous()])
    with pytest.raises(ValueError):                                    # stations now stand apart: tensors no longer fit
        st.push(x[:, :, :5].contiguous())
    assert lib.seist_launch_count() - before == 1
    st.close()
    with pytest.raises(RuntimeError):
        st.push([x[0, :, :5].contiguous(), x[1, :, :5].contiguous()])
    with pytest.raises(RuntimeError):
        st.close()
    with pytest.raises(ValueError):
        rs(torch.zeros(2, 3, 0, device="cuda"))
