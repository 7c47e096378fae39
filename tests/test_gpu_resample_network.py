"""-m gpu: a network of mixed input rates in one Resampler (seist_b200/resample.py, csrc/resample.cu, DESIGN §4.24).  Whole
records of {100, 40, 200, 50, 125, 1000} Hz stations to 50 and 100 Hz, 1, 2 and 10 007 samples and an hour among them,
each row bit for bit the single-rate Resampler of its station then NaN, within 1e-5 * max|x| of the float64 oracle, in
one launch and no host synchronisation; ragged list streams (empty pushes, pushes shorter than a station's latency, a
station silent until the close) bit for bit the single-rate whole record, one launch per push; the NaN rule at two rates
in one call; and the mixed outputs through the seist_s_dpk ragged and gap streams, `annotate` with segments and the
characteriser with segments, each station equal to its own single-rate record."""
import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import resample_ref as RR
from seist_b200 import _lib
from seist_b200 import events as EV
from seist_b200 import resample as RS
from seist_b200.models import create_model
from test_gpu_gap_stream import _station_csr
from test_gpu_gaps import _syncs
from test_gpu_stream_ragged import _annotator, _check_station

pytestmark = pytest.mark.gpu

RATES = [100, 40, 200, 50, 125, 1000, 100, 40]
W = 8192


def _piece(C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(C, T, generator=g, dtype=torch.float64) * (0.5 + 10 * torch.rand(C, 1, generator=g, dtype=torch.float64))
    return (x + torch.randn(C, 1, generator=g, dtype=torch.float64)).float()


def _check_rows(rs, out, pieces):
    T_out = rs.output_lengths([p.shape[1] for p in pieces])
    assert out.shape == (len(pieces), pieces[0].shape[0], int(T_out.max()))
    for s, p in enumerate(pieces):
        alone = RS.Resampler(rs.input_rate[s], rs.output_rate)(p[None])[0]
        assert torch.equal(out[s, :, :T_out[s]], alone), s
        assert torch.isnan(out[s, :, T_out[s]:]).all(), s


@pytest.mark.parametrize("fout", [50, 100])
def test_whole_network_equals_each_station_alone(fout):
    totals = [10007, 1, 2, 360000, 4096, 10007, 77, 3]
    pieces = [_piece(3, T, 10 + s).cuda() for s, T in enumerate(totals)]
    rs = RS.Resampler(RATES, fout)
    rs(pieces)                                                          # uploads the taps and the table
    lib = _lib.lib()
    before = lib.seist_launch_count()
    out, k = _syncs(lambda: rs(pieces))
    assert k == 0 and lib.seist_launch_count() - before == 1
    _check_rows(rs, out, pieces)
    T_out = rs.output_lengths(totals)
    for s, p in enumerate(pieces):
        if totals[s] > 20000:
            continue                                                    # the hour: equal to the single-rate path above
        x = p.cpu().double().numpy()
        want = RR.resample(x, int(rs.up[s]), int(rs.down[s]))
        err = np.abs(out[s, :, :T_out[s]].cpu().double().numpy() - want) / np.abs(x).max(axis=-1, keepdims=True)
        assert err.max() <= 1e-5, (s, err.max())


def test_identity_stations_copy_bit_for_bit():
    x = _piece(3, 5000, 3)
    bits = x.view(torch.int32)
    bits[0, 10] = int(np.array(0x80000000, np.uint32).view(np.int32))          # -0.0
    bits[1, 20] = 0x7fc01234                                                    # a NaN with a payload
    bits[2, 30] = int(np.array(0xffa00001, np.uint32).view(np.int32))
    x = x.cuda()
    rs = RS.Resampler([50, 100, 50], 50)
    out = rs([x, _piece(3, 999, 4).cuda(), x[:, :17].contiguous()])
    assert torch.equal(out[0].view(torch.int32), x.view(torch.int32))
    assert torch.equal(out[2, :, :17].view(torch.int32), x[:, :17].view(torch.int32))
    st = rs.open_stream(3)
    a = st.push([x[:, :7].contiguous(), _piece(3, 10, 5).cuda(), x[:, :0].contiguous()])
    assert a[0].shape == (3, 7) and torch.equal(a[0].view(torch.int32), x[:, :7].view(torch.int32)) and a[2].shape == (3, 0)


def _ragged(T, rng, silent):
    if silent:
        return [0, 0, 0, 0, T]
    cuts = sorted(rng.integers(0, T + 1, 5).tolist() + [1, 2, 3])
    n = np.diff([0] + cuts + [T]).tolist()
    return n[:2] + [0, 5] + n[2:]                                      # an empty push and one shorter than the latency


def _stream(rs, recs, rng, silent=None):
    scheds = [_ragged(r.shape[1], rng, s == silent) for s, r in enumerate(recs)]
    calls = max(map(len, scheds))
    scheds = [sc + [0] * (calls - len(sc)) for sc in scheds]
    st = rs.open_stream(len(recs))
    outs, pos = [], [0] * len(recs)
    for c in range(calls):
        outs.append(st.push([r[:, p:p + sc[c]].contiguous() for r, p, sc in zip(recs, pos, scheds)]))
        pos = [p + sc[c] for p, sc in zip(pos, scheds)]
    outs.append(st.close())
    return st, outs


@pytest.mark.parametrize("fout", [50, 100])
def test_stream_equals_each_station_alone_bit_for_bit(fout):
    totals = [12345, 9000, 1, 4444, 20011, 2, 7000, 15000]
    recs = [_piece(3, T, 40 + s).cuda() for s, T in enumerate(totals)]
    rs = RS.Resampler(RATES, fout)
    st, outs = _stream(rs, recs, np.random.default_rng(fout), silent=3)
    for s, r in enumerate(recs):
        alone = RS.Resampler(RATES[s], fout)(r[None])[0]
        assert torch.equal(torch.cat([o[s] for o in outs], 1), alone), s
    # every push one launch, no synchronisation, the held buffers fixed
    st = rs.open_stream(len(recs))
    held = [(h.data_ptr(), tuple(h.shape)) for h in st.held]
    assert held[0][1] == (len(recs), 3, rs.held_bound)
    lib = _lib.lib()
    pos = 0
    for n in (1, 0, 3000, 17, 5000):
        before = lib.seist_launch_count()
        out, k = _syncs(lambda: st.push([r[:, pos:pos + n].contiguous() for r in recs]))
        assert k == 0 and lib.seist_launch_count() - before == 1 and isinstance(out, list)
        pos += n
    assert sorted((h.data_ptr(), tuple(h.shape)) for h in st.held) == sorted(held)
    with pytest.raises(ValueError):
        st.push(torch.stack([r[:, :1] for r in recs]).contiguous())             # a tensor push
    st.close()


def test_nan_propagates_exactly_over_the_support_at_each_rate():
    rs = RS.Resampler([100, 40, 125], 100)
    x = [_piece(3, 20000, 9), _piece(3, 8000, 10), _piece(3, 25000, 11)]
    clean = rs([p.cuda() for p in x])
    x[0][:, 5000:5300] = float("nan")
    x[0][1, 9000] = float("nan")
    x[1][:, :40] = float("nan")
    x[1][2, 7990:] = float("nan")
    x[2][0, 12345] = float("nan")
    y = rs([p.cuda() for p in x])
    T_out = rs.output_lengths([p.shape[1] for p in x])
    for s, p in enumerate(x):
        want = RR.resample(p.double().numpy(), int(rs.up[s]), int(rs.down[s]))
        nan = torch.from_numpy(np.isnan(want)).cuda()
        got = y[s, :, :T_out[s]]
        assert torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan], clean[s, :, :T_out[s]][~nan]), s


@pytest.fixture(scope="module")
def models():
    out = {}
    for h in ("dpk", "pmp", "baz"):
        name = f"seist_s_{h}"
        m = create_model(name, in_channels=3, in_samples=W)
        m.load_state_dict(G.model_state_dict(name, W), strict=True)
        out[h] = m.cuda().eval()
    return out


def test_network_stream_into_ragged_stream_equals_annotate(models):
    rates = [100, 40, 50, 200]
    rs = RS.Resampler(rates, 50)
    ann = _annotator(models["dpk"], 4096, 4)
    recs = [_piece(3, int(T * f / 50), 70 + s).cuda() for s, (T, f) in enumerate(zip([2 * W + 3001, W + 17, 3 * W, 2 * W], rates))]
    st, outs = _stream(rs, recs, np.random.default_rng(1), silent=2)
    ast = ann.open_ragged_stream(len(recs))
    got = [ast.push(o) for o in outs] + [ast.close()]
    for s, r in enumerate(recs):
        _check_station(ann, got, RS.Resampler(rates[s], 50)(r[None])[0], s)


def test_network_stream_into_gap_stream_equals_annotate_with_segments(models):
    rates = [100, 40, 50]
    rs = RS.Resampler(rates, 50)
    ann = _annotator(models["dpk"], 4096, 3)
    recs = [_piece(3, int((3 * W + 999) * f / 50), 12 + s) for s, f in enumerate(rates)]
    recs[0][:, 7000:9000] = float("nan")
    recs[2][:, 100:130] = float("nan")
    recs = [r.cuda() for r in recs]
    st, outs = _stream(rs, recs, np.random.default_rng(2))
    gst = ann.open_gap_stream(len(recs))
    got = [gst.push(o) for o in outs] + [gst.close()]
    for s, r in enumerate(recs):
        one = RS.Resampler(rates[s], 50)(r[None])
        segs = ann.segments(one)
        want = ann.annotate(one, segments=segs)
        probs = torch.cat([o.probs[s] for o in got], 1)
        nan = torch.isnan(want[0])
        assert torch.equal(torch.isnan(probs), nan) and torch.equal(probs[~nan], want[0][~nan]), s
        pk = ann.pick_phases(want, segments=segs)
        for k in ("ppk", "spk"):
            parts = [_station_csr(getattr(o, k), s) for o in got]
            for v in range(2):
                assert torch.equal(torch.cat([p[v] for p in parts]), _station_csr(pk[k], 0)[v]), (s, k)
        det = ann.detect_events(want)
        parts = [_station_csr(o.det, s)[0] for o in got]
        assert torch.equal(torch.cat(parts).reshape(-1, 2), _station_csr(det, 0)[0]), s


def test_whole_network_through_annotate_and_characterise_with_segments(models):
    rates = [100, 40, 200, 50]
    rs = RS.Resampler(rates, 50)
    ann = _annotator(models["dpk"], 4096, 4)
    pieces = [_piece(3, int(T * f / 50), 90 + s).cuda() for s, (T, f) in enumerate(zip([3 * W + 77, W + 5, 2 * W, 4 * W], rates))]
    out = rs(pieces)
    segs = ann.segments(out)
    probs = ann.annotate(out, segments=segs)
    picks = ann.pick_phases(probs, segments=segs)
    ch = EV.EventCharacterizer({"pmp": models["pmp"], "baz": models["baz"]}, window=W, p_position_ratio=0.3, batch=4)
    got = ch(out, picks["ppk"], segments=segs)
    off = picks["ppk"][2].cpu()
    for s, p in enumerate(pieces):
        one = RS.Resampler(rates[s], 50)(p[None])
        want = ann.annotate(one, segments=ann.segments(one))
        T = one.shape[2]
        assert torch.equal(probs[s, :, :T], want[0]) and torch.isnan(probs[s, :, T:]).all(), s
        pk = ann.pick_phases(want, segments=ann.segments(one))
        for v in range(2):
            assert torch.equal(_station_csr(picks["ppk"], s)[v], _station_csr(pk["ppk"], 0)[v]), s
        alone = ch(one, pk["ppk"], segments=ann.segments(one))
        for h in ("pmp", "baz"):
            assert torch.equal(got[h][int(off[s]):int(off[s + 1])], alone[h]), (s, h)
