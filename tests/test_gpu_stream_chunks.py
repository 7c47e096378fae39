"""-m gpu: continuous records streamed chunk by chunk (seist_b200/stream.py ContinuousStream / RaggedPickStream, csrc/stream.cu)
against the streaming oracle (tests/stream_chunks_ref.py) call by call, and end to end against `annotate` + whole-record
picking on the same record."""
import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import stream_ref as SR
from seist_b200 import _lib
from seist_b200 import preprocess as PP
from seist_b200 import stream as ST
from seist_b200.models import create_model
from stream_chunks_ref import PickStreamRef, StreamRef, concat
from test_gpu_stream import _long_probs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    m = create_model("seist_s_dpk", in_channels=3, in_samples=8192)
    m.load_state_dict(G.model_state_dict("seist_s_dpk", 8192), strict=True)
    return m.cuda().eval()


def _np(out):
    """A StreamOutput (or a RaggedPickStream result) as numpy."""
    return tuple(tuple(t.cpu().numpy() for t in part) if isinstance(part, tuple) else part.cpu().numpy() if torch.is_tensor(part)
                 else part for part in out)


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, tuple):
            _same(g, w)
        else:
            assert np.array_equal(np.asarray(g), np.asarray(w)), (g, w)


def _injected(W):
    """Window outputs that depend only on (station, start): what the model would return, without a model."""
    def outputs(x, ids):
        s = np.array([i[0] for i in ids], dtype=np.float64)[:, None, None]
        a = np.array([i[1] for i in ids], dtype=np.float64)[:, None, None]
        c = np.arange(3, dtype=np.float64)[None, :, None]
        t = np.arange(W, dtype=np.float64)[None, None, :]
        v = 0.5 + 0.5 * np.sin(0.013 * (a + t) * (1 + c) + 0.7 * s) * np.cos(0.0011 * (a + t) + 0.3 * (a % 7))
        return v.astype(np.float32)
    return outputs


def _drive_helpers(rec, split, W, P, B, mode, fn, mpd, thr):
    """The streaming pipeline through the low-level helpers, window outputs from fn; yields each call's output."""
    S, C, T = rec.shape
    dev = "cuda"
    tail = [torch.zeros(S, C, W, device=dev) for _ in range(2)]
    carry = [torch.zeros(S, 3, W, device=dev) for _ in range(2)]
    picker = ST.RaggedPickStream(S, dev, mpd, thr[1], thr[2], thr[0])
    R = F = k = 0
    pos = 0
    for n in list(split) + [None]:
        if n is None:
            kr = (R - W) // P + 1
            tl = R - W if (kr - 1) * P + W < R else -1
            r1, f1, nk, chunk = R, R, 0, None
        else:
            r1 = R + n
            k1 = (r1 - W) // P + 1 if r1 >= W else 0
            tl, kr, f1, nk = -1, -1, max(0, r1 - W), k1 - k
            chunk = torch.from_numpy(np.ascontiguousarray(rec[:, :, pos:pos + n])).cuda()
            pos += n
        step = ST.stream_step(S, C, W, P, F, R, f1, r1, k, nk, tl, kr, "std", mode)
        starts = [(k + q) * P for q in range(nk)] + ([tl] if tl >= 0 else [])
        ids = [(s, a) for s in range(S) for a in starts]
        acc = torch.empty(S, 3, r1 - F, device=dev)
        x = torch.empty(B, C, W, device=dev)
        full = torch.from_numpy(np.ascontiguousarray(rec[:, :, :r1])).cuda()
        for j0 in range(0, len(ids), B):
            ST.stream_window_(x, step, tail[0], chunk, j0)
            m = min(B, len(ids) - j0)
            want = torch.stack([full[s, :, a:a + W] for s, a in ids[j0:j0 + m]]).contiguous()
            PP.normalize_(want, "std")
            assert torch.equal(x[:m], want) and (x[m:] == 0).all()
            y = torch.full((B, 3, W), float("nan"), device=dev)
            y[:m] = torch.from_numpy(fn(None, ids[j0:j0 + m])).cuda()
            ST.stream_stack_(acc, y, step, j0, carry[0])
        probs = torch.empty(S, 3, f1 - F, device=dev)
        ST.stream_emit_(probs, carry[1], step, carry[0], acc)
        ST.stream_keep_(tail[1], step, tail[0], chunk)
        tail.reverse()
        carry.reverse()
        t0 = F
        R, F, k = r1, f1, k + nk
        picks = picker.close(probs) if n is None else picker.push(probs)
        yield (t0, probs) + tuple(picks)


@pytest.mark.parametrize("mode", ["mean", "max"])
@pytest.mark.parametrize("W,P,B", [(512, 256, 3), (600, 250, 5)])
def test_helpers_and_ragged_picker_equal_stream_ref_call_by_call(mode, W, P, B):
    S, C, T = 3, 3, 4 * 600 + 77
    rng = np.random.default_rng(W + P)
    rec = (rng.standard_normal((S, C, T)) * 3 + 1).astype(np.float32)
    fn, mpd, thr = _injected(W), 9, (0.6, 0.7, 0.65)
    head = [1, W - 2, 1, 0, P, 333] + [1] * 5
    rest = T - sum(head)
    split = head + np.diff(sorted(rng.integers(0, rest, 4).tolist() + [0, rest])).tolist()
    assert sum(split) == T
    ref = StreamRef(S, C, W, P, fn, mpd, thr, "std", mode)
    want = [ref.push(rec[:, :, a:a + n]) for a, n in zip(np.cumsum([0] + split[:-1]), split)] + [ref.close()]
    got = [_np(o) for o in _drive_helpers(rec, split, W, P, B, mode, fn, mpd, thr)]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g[0] == w[0]
        _same(g[1:], w[1:])
    allp = concat(want, S)
    assert np.array_equal(allp[0], SR.stack(fn(None, [(s, a) for s in range(S) for a in SR.window_starts(T, W, P)]), S, T, W, P, mode))


def _feed(probs, split, mpd, thr, t0=0):
    S = probs.shape[0]
    ref = PickStreamRef(S, mpd, thr, t0)
    dev = ST.RaggedPickStream(S, "cuda", mpd, thr[1], thr[2], thr[0], t0=t0)
    pc = torch.from_numpy(probs).cuda()
    outs, pos = [], 0
    for n in list(split) + [None]:
        last = n is None
        stretch = pc[:, :, pos:] if last else pc[:, :, pos:pos + n]
        w = ref.close(probs[:, :, pos:]) if last else ref.push(probs[:, :, pos:pos + n])
        g = _np(dev.close(stretch.contiguous()) if last else dev.push(stretch.contiguous()))
        _same(g, w)
        outs.append((pos, probs[:, :, pos:pos + (0 if last else n)] if not last else probs[:, :, pos:]) + g)
        pos += 0 if last else n
    return outs


def test_dense_probability_pushes_long_rows_match_oracle():
    probs = _long_probs()
    T = probs.shape[2]
    rng = np.random.default_rng(5)
    split = np.diff([0] + sorted(rng.integers(0, T, 60).tolist())).tolist()
    for mpd, (tp, ts), td in ((100, (0.3, 0.1), 0.5), (7, (0.05, 0.5), 0.3)):
        got = concat(_feed(probs, split, mpd, (td, tp, ts)), 4)
        for k, ch, thr in ((1, 1, tp), (2, 2, ts)):
            want = SR.pick_all(probs, ch, thr, mpd)
            assert all(np.array_equal(a, b) for a, b in zip(got[k], want)), (ch, mpd)
        pairs, off = SR.detect_all(probs, 0, td)
        assert np.array_equal(got[3][0], pairs) and np.array_equal(got[3][1], off)


def test_dense_probability_pushes_cross_2_31():
    t0 = (1 << 31) - 40_000
    probs = _long_probs()[:, :, :100_000].copy()
    got = concat(_feed(probs, [30_000, 1, 9_999, 25_000, 7], 50, (0.3, 0.3, 0.1), t0), 4)
    want = SR.pick_all(probs, 1, 0.3, 50)
    assert np.array_equal(got[1][0], want[0] + t0) and np.array_equal(got[1][2], want[2])
    assert (got[1][0] >= 1 << 31).any() and (got[1][0] < 1 << 31).any()
    pairs, off = SR.detect_all(probs, 0, 0.3)
    assert np.array_equal(got[3][0], pairs + t0) and np.array_equal(got[3][1], off)


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g) * (0.5 + 10 * torch.rand(S, C, 1, generator=g)) + torch.randn(S, C, 1, generator=g)
    return x.cuda()


@pytest.mark.parametrize("stride,batch", [(4096, 4), (3000, 7)])
def test_stream_equals_annotate_end_to_end(model, stride, batch):
    S, W = 3, 8192
    T = 5 * W + 1234
    rec = _record(S, 3, T, 11)
    for mode in ("mean", "max"):
        ann = ST.ContinuousAnnotator(model, window=W, stride=stride, batch=batch, stack=mode)
        ann.min_peak_dist = 100
        ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
        want = ann.annotate(rec)
        st = ann.open_stream(S)
        outs, pos = [], 0
        for n in [5000, 1, 8191, 0, 12000, 3000, 7]:
            outs.append(_np(st.push(rec[:, :, pos:pos + n].contiguous())))
            pos += n
        outs.append(_np(st.push(rec[:, :, pos:].contiguous())))
        outs.append(_np(st.close()))
        with pytest.raises(RuntimeError):
            st.push(rec[:, :, :10].contiguous())
        got = concat(outs, S)
        assert np.array_equal(got[0], want.cpu().numpy()), (mode, np.abs(got[0] - want.cpu().numpy()).max())
        picks = ann.pick_phases(want)
        for k, name, ch in ((1, "ppk", 1), (2, "spk", 2)):
            ora = SR.pick_all(got[0], ch, 0.2, 100)
            assert all(np.array_equal(a, b) for a, b in zip(got[k], ora))
            assert all(np.array_equal(a, b.cpu().numpy()) for a, b in zip(got[k], picks[name]))
        pairs, off = ann.detect_events(want)
        assert np.array_equal(got[3][0], pairs.cpu().numpy()) and np.array_equal(got[3][1], off.cpu().numpy())
        assert np.array_equal(got[3][0], SR.detect_all(got[0], 0, 0.3)[0])


def test_stream_and_picker_argument_errors_raise_before_launch(model):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=4096, batch=2)
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        ann.open_stream(2)                                          # min_peak_dist unset
    for mpd in (1, 0, -3):
        ann.min_peak_dist = mpd
        with pytest.raises(ValueError):
            ann.open_stream(2)
    ann.min_peak_dist = 100
    st = ann.open_stream(2)
    with pytest.raises(RuntimeError):
        st.push(torch.zeros(2, 3, 100))                             # CPU tensor
    with pytest.raises(ValueError):
        st.push(torch.zeros(3, 3, 100, device="cuda"))              # wrong S
    with pytest.raises(ValueError):
        st.push(torch.zeros(2, 2, 100, device="cuda"))              # wrong C
    with pytest.raises(ValueError):
        st.push(torch.zeros(2, 3, 100, device="cuda", dtype=torch.float64))
    with pytest.raises(ValueError):
        st.push(torch.zeros(2, 3, 200, device="cuda")[:, :, ::2])   # not contiguous
    assert lib.seist_launch_count() == before
    st.push(torch.zeros(2, 3, 100, device="cuda"))
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        st.close()                                                  # fewer than `window` samples
    with pytest.raises(ValueError):
        ST.RaggedPickStream(2, "cuda", 1)
    pk = ST.RaggedPickStream(2, "cuda", 10)
    with pytest.raises(ValueError):
        pk.push(torch.zeros(3, 3, 10, device="cuda"))
    step = ST.stream_step(2, 3, 8192, 4096, 0, 0, 0, 100, 0, 0)
    with pytest.raises(ValueError):
        ST.stream_window_(torch.zeros(2, 3, 8192, device="cuda"), step, torch.zeros(2, 3, 4096, device="cuda"), None, 0)
    with pytest.raises(ValueError):
        ST.stream_stack_(torch.zeros(2, 3, 99, device="cuda"), torch.zeros(2, 3, 8192, device="cuda"), step, 0,
                         torch.zeros(2, 3, 8192, device="cuda"))
    c = torch.zeros(2, 3, 8192, device="cuda")
    with pytest.raises(ValueError):
        ST.stream_emit_(torch.zeros(2, 3, 0, device="cuda"), c, step, c, torch.zeros(2, 3, 100, device="cuda"))   # in place
    assert lib.seist_launch_count() == before
    st2 = ann.open_stream(2)
    st2.push(torch.zeros(2, 3, 8192, device="cuda"))
    st2.close()
    with pytest.raises(RuntimeError):
        st2.push(torch.zeros(2, 3, 10, device="cuda"))
    with pytest.raises(RuntimeError):
        st2.close()


def test_stream_state_is_bounded(model):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=4096, batch=8)
    ann.min_peak_dist = 100
    S, n = 2, 3000
    st = ann.open_stream(S)
    quiet = torch.zeros(S, 3, n, device="cuda")
    held = []
    for i in range(50):
        st.push(quiet)
        torch.cuda.synchronize()
        held.append(torch.cuda.memory_allocated())
    assert max(held[25:]) <= max(held[5:25]), held                # no growth with the number of pushes
