"""-m gpu: ragged streams, stations that advance at different rates (seist_b200/stream.py RaggedStream / RaggedPickStream,
csrc/stream.cu, DESIGN §4.19), station by station against a one-station streaming oracle (tests/stream_chunks_ref.py),
against the equal-rate stream, and end to end against `annotate` + whole-record picking of each station's own record."""
import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import stream_ref as SR
from seist_b200 import _lib
from seist_b200 import preprocess as PP
from seist_b200 import stream as ST
from seist_b200.models import create_model
from stream_chunks_ref import StreamRef
from test_gpu_stream import _long_probs
from test_gpu_stream_chunks import _injected, _np, _same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    m = create_model("seist_s_dpk", in_channels=3, in_samples=8192)
    m.load_state_dict(G.model_state_dict("seist_s_dpk", 8192), strict=True)
    return m.cuda().eval()


def _station(out, s):
    """Station s of one ragged call (t0 list, probs list, ppk, spk, det) as a one-station StreamRef-style output."""
    t0, probs, *rest = out

    def row(csr):
        *vals, off = csr
        o = off.cpu().numpy()
        return tuple(v[o[s]:o[s + 1]].cpu().numpy() for v in vals) + (np.array([0, o[s + 1] - o[s]], np.int64),)
    return (t0[s], probs[s].cpu().numpy()[None]) + tuple(row(c) for c in rest)


def _schedule(totals, calls, seed, silent=()):
    """Per-call lengths of every station: random cuts, 0- and 1-sample pushes; `silent` stations push nothing until
    their whole record arrives in the last call."""
    rng = np.random.default_rng(seed)
    rows = []
    for s, T in enumerate(totals):
        if s in silent:
            rows.append([0] * (calls - 1) + [T])
            continue
        cuts = sorted(rng.integers(0, T + 1, calls - 3).tolist() + [1, 2])
        rows.append(np.diff([0] + cuts + [T]).tolist())
    return [list(c) for c in zip(*rows)]


def _drive_ragged(recs, sched, W, P, B, mode, fn, mpd, thr):
    """The ragged pipeline through the low-level helpers, window outputs from fn; yields each call's output."""
    S, C = len(recs), recs[0].shape[0]
    dev = "cuda"
    tail = [torch.zeros(S, C, W, device=dev) for _ in range(2)]
    carry = [torch.zeros(S, 3, W, device=dev) for _ in range(2)]
    picker = ST.RaggedPickStream(S, dev, mpd, thr[1], thr[2], thr[0])
    full = [torch.from_numpy(r).cuda() for r in recs]
    R = np.zeros(S, np.int64)
    for lengths in list(sched) + [None]:
        close = lengths is None
        step = ST.ragged_stream_step(C, W, P, R, lengths, close, "std", mode)
        plan = step.plan
        parts = [] if close else [full[s][:, R[s]:R[s] + lengths[s]].reshape(-1) for s in range(S)]
        chunk = torch.cat(parts) if parts and plan["chunk_off"][-1] else torch.zeros(1, device=dev)
        ids = ST.ragged_window_ids(plan, P)
        acc = torch.empty(max(1, 3 * int(plan["acc_off"][-1])), device=dev)
        x = torch.empty(B, C, W, device=dev)
        for j0 in range(0, len(ids), B):
            ST.ragged_window_(x, step, tail[0], chunk, j0)
            m = min(B, len(ids) - j0)
            want = torch.stack([full[s][:, a:a + W] for s, a in ids[j0:j0 + m]]).contiguous()
            PP.normalize_(want, "std")
            assert torch.equal(x[:m], want) and (x[m:] == 0).all()
            y = torch.full((B, 3, W), float("nan"), device=dev)
            y[:m] = torch.from_numpy(fn(None, ids[j0:j0 + m])).cuda()
            ST.ragged_stack_(acc, y, step, j0, carry[0])
        out = plan["out_off"]
        probs = torch.empty(max(1, 3 * int(out[-1])), device=dev)
        ST.ragged_emit_(probs, carry[1], step, carry[0], acc)
        ST.ragged_keep_(tail[1], step, tail[0], chunk)
        tail.reverse()
        carry.reverse()
        m = plan["f1"] - plan["f0"]
        views = [probs[3 * int(out[s]):3 * int(out[s + 1])].view(3, int(m[s])) for s in range(S)]
        picks = picker.close(views) if close else picker.push(views)
        R = plan["r1"]
        yield (plan["f0"].tolist(), views) + tuple(picks)


@pytest.mark.parametrize("mode", ["mean", "max"])
@pytest.mark.parametrize("W,P,B", [(512, 256, 3), (600, 250, 5)])
def test_helpers_equal_one_station_streams_call_by_call(mode, W, P, B):
    totals = [4 * 600 + 77, W, W + 1, 3 * W + 5, 2 * W + P]
    S, C = len(totals), 3
    rng = np.random.default_rng(W + P)
    recs = [(rng.standard_normal((C, T)) * 3 + 1).astype(np.float32) for T in totals]
    fn, mpd, thr = _injected(W), 9, (0.6, 0.7, 0.65)
    sched = _schedule(totals, 9, W, silent=(3,))
    refs = [StreamRef(1, C, W, P, (lambda s: lambda x, ids: fn(x, [(s, a) for _, a in ids]))(s), mpd, thr, "std", mode)
            for s in range(S)]
    pos = np.zeros(S, np.int64)
    calls = 0
    for lengths, got in zip(list(sched) + [None], _drive_ragged(recs, sched, W, P, B, mode, fn, mpd, thr)):
        for s in range(S):
            if lengths is None:
                want = refs[s].close()
            else:
                want = refs[s].push(recs[s][None, :, pos[s]:pos[s] + lengths[s]])
                pos[s] += lengths[s]
            g = _station(got, s)
            assert g[0] == want[0], (calls, s)
            _same(g[1:], want[1:])
        calls += 1
    assert calls == len(sched) + 1


def test_probability_stage_rows_of_different_lengths():
    probs = _long_probs()
    S, T = probs.shape[0], probs.shape[2]
    lengths = [T, T - 12_345, 1_500_000, T - 1]
    t0 = [0, 0, 0, (1 << 31) - 1_000_000]                          # the last row's indices cross 2^31
    rng = np.random.default_rng(5)
    splits = [np.diff([0] + sorted(rng.integers(0, n, 40 + 7 * s).tolist()) + [n]).tolist() for s, n in enumerate(lengths)]
    calls = max(len(p) for p in splits)
    splits = [p + [0] * (calls - len(p)) for p in splits]
    pc = torch.from_numpy(probs).cuda()
    for mpd, (tp, ts), td in ((100, (0.3, 0.1), 0.5), (7, (0.05, 0.5), 0.3)):
        pk = ST.RaggedPickStream(S, "cuda", mpd, tp, ts, td, t0=t0)
        pos = [0] * S
        outs = []
        for c in range(calls):
            outs.append(_np(pk.push([pc[s, :, pos[s]:pos[s] + splits[s][c]].contiguous() for s in range(S)])))
            pos = [p + splits[s][c] for s, p in enumerate(pos)]
        outs.append(_np(pk.close()))
        assert pos == lengths
        for s in range(S):
            rec = probs[s:s + 1, :, :lengths[s]]
            for k, ch, thr in ((0, 1, tp), (1, 2, ts)):
                want = SR.pick_all(rec, ch, thr, mpd)
                idx = np.concatenate([o[k][0][o[k][2][s]:o[k][2][s + 1]] for o in outs])
                val = np.concatenate([o[k][1][o[k][2][s]:o[k][2][s + 1]] for o in outs])
                assert np.array_equal(idx, want[0] + t0[s]) and np.array_equal(val, want[1]), (mpd, s, ch)
            pairs = np.concatenate([o[2][0][o[2][1][s]:o[2][1][s + 1]] for o in outs]).reshape(-1, 2)
            assert np.array_equal(pairs, SR.detect_all(rec, 0, td)[0] + t0[s]), (mpd, s)
        last = np.concatenate([o[k][0][o[k][2][3]:o[k][2][4]] for o in outs for k in (0, 1)] +
                              [o[2][0][o[2][1][3]:o[2][1][4]].ravel() for o in outs])
        assert (last >= 1 << 31).any() and (last < 1 << 31).any()


def _record(T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(3, T, generator=g) * (0.5 + 10 * torch.rand(3, 1, generator=g)) + torch.randn(3, 1, generator=g)
    return x.cuda()


def _annotator(model, stride, batch, mode="mean"):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=stride, batch=batch, stack=mode)
    ann.min_peak_dist = 100
    ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
    return ann


def _run(st, recs, sched):
    outs, pos = [], [0] * len(recs)
    for lengths in sched:
        outs.append(st.push([r[:, p:p + n].contiguous() for r, p, n in zip(recs, pos, lengths)]))
        pos = [p + n for p, n in zip(pos, lengths)]
    outs.append(st.close())
    return outs


def _check_station(ann, outs, rec, s):
    """Station s of a ragged stream's outputs, concatenated, against annotate + picking of its own record."""
    want = ann.annotate(rec[None])
    got = torch.cat([o.probs[s] for o in outs], 1)
    assert [o.t0[s] for o in outs] == np.cumsum([0] + [o.probs[s].shape[1] for o in outs[:-1]]).tolist()
    assert torch.equal(got, want[0]), (s, (got - want[0]).abs().max().item())
    picks = ann.pick_phases(want)
    for name in ("ppk", "spk"):
        for j in range(2):
            cat = torch.cat([getattr(o, name)[j][getattr(o, name)[2][s]:getattr(o, name)[2][s + 1]] for o in outs])
            assert torch.equal(cat, picks[name][j]), (s, name)
    pairs, _ = ann.detect_events(want)
    cat = torch.cat([o.det[0][o.det[1][s]:o.det[1][s + 1]] for o in outs])
    assert torch.equal(cat, pairs), s


@pytest.mark.parametrize("stride,batch", [(4096, 4), (3000, 7)])
def test_ragged_stream_equals_annotate_per_station(model, stride, batch):
    W = 8192
    totals = [5 * W + 1234, 3 * W + 17, W, 2 * W + stride]
    recs = [_record(T, 11 + s) for s, T in enumerate(totals)]
    sched = _schedule(totals, 7, stride)
    for mode in ("mean", "max"):
        ann = _annotator(model, stride, batch, mode)
        st = ann.open_ragged_stream(len(totals))
        outs = _run(st, recs, sched)
        with pytest.raises(RuntimeError):
            st.push([r[:, :10].contiguous() for r in recs])
        for s, rec in enumerate(recs):
            _check_station(ann, outs, rec, s)


def test_equal_lengths_equal_the_equal_rate_stream(model):
    S, W = 3, 8192
    rec = torch.stack([_record(4 * W + 999, 3 + s) for s in range(S)])
    ann = _annotator(model, 3000, 5)
    plain, ragged = ann.open_stream(S), ann.open_ragged_stream(S)
    pos = 0
    for n in [5000, 1, 8191, 0, 12000, 3000, 7, rec.shape[2] - 28199, None]:
        if n is None:
            a, b = plain.close(), ragged.close()
        else:
            a = plain.push(rec[:, :, pos:pos + n].contiguous())
            b = ragged.push([rec[s, :, pos:pos + n].contiguous() for s in range(S)])
            pos += n
        assert b.t0 == [a.t0] * S
        assert torch.equal(torch.stack(b.probs), a.probs)
        for name in ("ppk", "spk", "det"):
            for x, y in zip(getattr(a, name), getattr(b, name)):
                assert torch.equal(x, y), name
    assert plain.forwards == ragged.forwards


def test_forwards_are_shared_across_stations(model):
    W, B = 8192, 4
    totals = [3 * W + 100, 2 * W + 5000, 4 * W, W + 1, 3 * W]
    recs = [_record(T, 40 + s) for s, T in enumerate(totals)]
    sched = _schedule(totals, 6, 1)
    ann = _annotator(model, 4096, B)
    st = ann.open_ragged_stream(len(totals))
    _run(st, recs, sched)
    R = np.zeros(len(totals), np.int64)
    want = alone = 0
    for lengths in sched + [None]:
        plan = ST.ragged_plan(R, lengths, W, 4096, close=lengths is None)
        nw = np.diff(plan["win_off"])
        want += -(-int(nw.sum()) // B)
        alone += sum(-(-int(w) // B) for w in nw)
        R = plan["r1"]
    assert st.forwards == want and want < alone, (st.forwards, want, alone)


def test_a_silent_station_does_not_hold_back_the_others(model):
    W = 8192
    totals = [4 * W + 321, 3 * W, 4 * W + 11]
    recs = [_record(T, 70 + s) for s, T in enumerate(totals)]
    calls = 8
    sched = _schedule(totals, calls, 9, silent=(1,))
    ann = _annotator(model, 4096, 6)
    st = ann.open_ragged_stream(3)
    outs = _run(st, recs, sched)
    final = [o.t0[0] + o.probs[0].shape[1] for o in outs[:calls - 1]]
    assert final[-1] == max(0, sum(c[0] for c in sched[:calls - 1]) - W) > 0          # station 0 kept coming out
    assert all(o.probs[1].shape[1] == 0 for o in outs[:calls - 1])
    for s, rec in enumerate(recs):
        _check_station(ann, outs, rec, s)


def test_ragged_argument_errors_raise_before_launch(model):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=4096, batch=2)
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        ann.open_ragged_stream(2)                                   # min_peak_dist unset
    ann.min_peak_dist = 1
    with pytest.raises(ValueError):
        ann.open_ragged_stream(2)
    ann.min_peak_dist = 100
    st = ann.open_ragged_stream(2)
    ok = torch.zeros(3, 100, device="cuda")
    with pytest.raises(ValueError):
        st.push([ok])                                               # wrong number of chunks
    with pytest.raises(ValueError):
        st.push([ok, torch.zeros(2, 100, device="cuda")])           # wrong C
    with pytest.raises(RuntimeError):
        st.push([ok, torch.zeros(3, 100)])                          # CPU chunk
    with pytest.raises(ValueError):
        st.push([ok, torch.zeros(3, 100, device="cuda", dtype=torch.float64)])
    with pytest.raises(ValueError):
        st.push([ok, torch.zeros(3, 200, device="cuda")[:, ::2]])   # not contiguous
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError):
            st.push([ok, torch.zeros(3, 100, device="cuda:1")])     # another device
    assert lib.seist_launch_count() == before
    st.push([torch.zeros(3, 9000, device="cuda"), ok])
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError, match=r"\[1\]"):
        st.close()                                                  # station 1 is shorter than `window`
    assert not st.closed
    with pytest.raises(ValueError):
        ST.RaggedPickStream(2, "cuda", 1)
    pk = ST.RaggedPickStream(2, "cuda", 10)
    with pytest.raises(ValueError):
        pk.push([torch.zeros(3, 10, device="cuda")])
    step = ST.ragged_stream_step(3, 8192, 4096, [0, 0], [100, 0])
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        ST.ragged_window_(torch.zeros(2, 3, 8192, device="cuda"), step, torch.zeros(2, 3, 4096, device="cuda"),
                          torch.zeros(300, device="cuda"), 0)
    c = torch.zeros(2, 3, 8192, device="cuda")
    with pytest.raises(ValueError):
        ST.ragged_emit_(torch.zeros(1, device="cuda"), c, step, c, torch.zeros(300, device="cuda"))   # in place
    assert lib.seist_launch_count() == before
    st.push([ok, torch.zeros(3, 8100, device="cuda")])
    st.close()
    with pytest.raises(RuntimeError):
        st.push([ok, ok])
    with pytest.raises(RuntimeError):
        st.close()


def test_ragged_stream_state_is_bounded(model):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=4096, batch=8)
    ann.min_peak_dist = 100
    S = 3
    st = ann.open_ragged_stream(S)
    rng = np.random.default_rng(0)
    held = []
    for i in range(50):
        st.push([torch.zeros(3, int(n), device="cuda") for n in rng.integers(0, 4000, S)])
        torch.cuda.synchronize()
        held.append(torch.cuda.memory_allocated())
    assert max(held[25:]) <= max(held[5:25]), held                # no growth with the number of pushes
