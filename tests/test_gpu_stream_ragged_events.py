"""-m gpu: the P picks of a ragged stream characterised as they close (seist_b200/events.py RaggedCharacterizedStream,
`seist_ragged_history` and `seist_ragged_event_windows` in csrc/stream.cu, DESIGN §4.20).  The history kernel against
slices of each station's record and the packed cut bit for bit against `seist_event_windows` on each station's own record
(bases near 2^40 included); seist_s_dpk streamed with seist_s_{pmp,emg,baz,dis} bit-identical per station to the
whole-record path of its own record; equal lengths equal CharacterizedStream call by call; the launches and replays of a
call over a plain RaggedStream and the held samples of the per-station oracle; bounded memory; argument errors before any
launch."""
import copy

import numpy as np
import pytest
import torch

from oracle import golden as G
from seist_b200 import _lib
from seist_b200 import events as EV
from seist_b200.models import create_model
from stream_ragged_events_ref import RaggedCharacterizedStreamRef
from test_gpu_events import _csr, _cut_all

pytestmark = pytest.mark.gpu

HEADS = ("pmp", "emg", "baz", "dis")


def _record(C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(C, T, generator=g) * (0.5 + 10 * torch.rand(C, 1, generator=g)) + torch.randn(C, 1, generator=g)
    return x.cuda()


def _dev(host):
    return torch.from_numpy(np.ascontiguousarray(host, dtype=np.int64)).cuda()


def _history_steps(recs, sched, keeps, base):
    """Drive ragged_history_ over the stations' records pushed in `sched`, station s keeping [keeps[i][s], R_s) at step i
    (global indices from `base`) -> per step the buffer, its device h0 / offsets, and h0, R on the host."""
    S, C = len(recs), recs[0].shape[0]
    bufs = [torch.full((1,), float("nan"), device="cuda") for _ in range(2)]
    h0, R = np.full(S, base, np.int64), np.full(S, base, np.int64)
    desc = _dev(np.concatenate([h0, np.zeros(S + 1, np.int64)]))
    for lengths, keep in zip(sched, keeps):
        n = np.asarray(lengths, np.int64)
        hp = EV.ragged_history_plan(h0, R, n, keep)
        if n.any():
            chunk = torch.cat([recs[s][:, R[s] - base:R[s] - base + n[s]].reshape(-1) for s in range(S)])
            need = C * int(hp["off"][-1])
            if bufs[1].numel() < need:
                bufs[1] = torch.full((max(need, 2 * bufs[1].numel()),), float("nan"), device="cuda")
            dev = _dev(np.concatenate([hp["h0"], hp["off"], np.concatenate([[0], np.cumsum(n)])]))
            EV.ragged_history_(bufs[1], bufs[0], desc[:S], desc[S:], chunk, dev[2 * S + 1:], dev[:S], dev[S:2 * S + 1], C,
                               int(hp["len"].max()))
            bufs.reverse()
            desc, h0 = dev[:2 * S + 1], hp["h0"]
        R = hp["R"]
        yield bufs[0], desc, h0, R, hp["off"]


def _ragged_cut_all(hist, desc, S, index, offsets, W, a, mode, B):
    C = 3
    x = torch.full((B, C, W), float("nan"), device="cuda")
    got = []
    for e0 in range(0, index.numel(), B):
        EV.ragged_event_windows_([x], hist, desc[:S], desc[S:], index, offsets, e0, W, a, mode)
        got.append(x[:min(B, index.numel() - e0)].clone())
    return torch.cat(got) if got else torch.zeros(0, C, W, device="cuda"), x


@pytest.mark.parametrize("base", [0, (1 << 40) - 7000])
def test_history_and_packed_cut_equal_each_stations_record(base):
    C, W = 3, 2048
    totals = [30_000, 9_000, 21_000, 12_500]
    S = len(totals)
    recs = [_record(C, T, 31 + s) for s, T in enumerate(totals)]
    recs[2][1, :] = 3.0                                                    # a constant channel
    rng = np.random.default_rng(7)
    sched = []
    for s, T in enumerate(totals):
        cuts = sorted(rng.integers(0, T, 8).tolist() + [1])
        row = np.diff([0] + cuts + [T]).tolist()
        row = [0] * 3 + row if s == 3 else row + [0] * 3                    # station 3: an empty history at first
        sched.append(row)
    sched = [list(c) for c in zip(*sched)]
    keeps, k, R = [], np.full(S, base, np.int64), np.full(S, base, np.int64)
    for lengths in sched:                                                  # monotone, at most R + n
        R = R + np.asarray(lengths, np.int64)
        k = np.minimum(R, k + rng.integers(0, 4000, S))
        keeps.append(k.copy())
    checked = 0
    for step, (hist, desc, h0, R, off) in enumerate(_history_steps(recs, sched, keeps, base)):
        for s in range(S):
            block = hist[C * int(off[s]):C * int(off[s + 1])].view(C, -1)
            assert torch.equal(block, recs[s][:, h0[s] - base:R[s] - base]), (step, s)
        for mode in ("std", "max", ""):
            for ratio in (0.0, 0.3, 1.0):
                a = EV.anchor(W, ratio)
                picks = []
                for s in range(S):
                    lo = h0[s] - base + a if h0[s] > base else 0           # the picks the retention rule admits
                    hi = R[s] - base - max(1, W - a)                       # a pushed pick, its window pushed
                    if s == 1 or lo > hi:
                        picks.append([])                                   # stations without picks
                        continue
                    picks.append(sorted({lo, hi} | set(rng.integers(lo, hi + 1, 3).tolist())))
                want = []
                for s in range(S):
                    i, o = _csr([picks[s]])
                    (w,), _ = _cut_all(recs[s][None], i, o, W, a, mode, 2)  # each station's own record
                    want.append(w)
                index, offsets = _csr([[p + base for p in ps] for ps in picks])
                got, x = _ragged_cut_all(hist, desc, S, index, offsets, W, a, mode, 3)   # stations split across batches
                assert torch.equal(got, torch.cat(want)), (step, mode, ratio)
                m = index.numel() % 3
                assert m == 0 or (x[m:] == 0).all()                        # rows past M are zero
                checked += index.numel()
        e_idx, e_off = _csr([[]] * S)                                      # M = 0: zero rows
        x = torch.full((2, C, W), float("nan"), device="cuda")
        EV.ragged_event_windows_([x], hist, desc[:S], desc[S:], e_idx, e_off, 0, W, 0)
        assert (x == 0).all()
    assert checked > 100


@pytest.fixture(scope="module")
def models():
    out = {}
    for h in ("dpk",) + HEADS:
        name = f"seist_s_{h}"
        m = create_model(name, in_channels=3, in_samples=8192)
        m.load_state_dict(G.model_state_dict(name, 8192), strict=True)
        out[h] = m.cuda().eval()
    return out


def _annotator(models, stride, batch=4, stack="mean"):
    from seist_b200 import stream as ST
    ann = ST.ContinuousAnnotator(models["dpk"], window=8192, stride=stride, batch=batch, stack=stack)
    ann.min_peak_dist = 100
    ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
    return ann


def _schedule(totals, calls, seed, silent=()):
    """Per-call lengths: random cuts with 0- and 1-sample pushes; `silent` stations push nothing until the last call."""
    rng = np.random.default_rng(seed)
    rows = []
    for s, T in enumerate(totals):
        if s in silent:
            rows.append([0] * (calls - 1) + [T])
            continue
        cuts = sorted(rng.integers(0, T + 1, calls - 3).tolist() + [1, 2])
        rows.append(np.diff([0] + cuts + [T]).tolist())
    return [list(c) for c in zip(*rows)]


def _threshold(ann, recs):
    p = torch.cat([ann.annotate(r[None])[0, 1] for r in recs])
    return float(torch.quantile(p[::3].float(), 0.995))


def _run(cs, recs, sched):
    outs, pos = [], [0] * len(recs)
    for lengths in sched:
        outs.append(cs.push([r[:, p:p + n].contiguous() for r, p, n in zip(recs, pos, lengths)]))
        pos = [p + n for p, n in zip(pos, lengths)]
    outs.append(cs.close())
    return outs


def _station(outs, s, key):
    parts = []
    for o in outs:
        off = o.out.ppk[2].tolist()
        parts.append((o.events[key] if key != "ppk" else o.out.ppk[0])[off[s]:off[s + 1]])
    return torch.cat(parts)


@pytest.mark.parametrize("stride", [4096, 3000])
def test_ragged_events_equal_each_stations_whole_record(models, stride):
    W = 8192
    totals = [5 * W + 1234, 3 * W + 17, 2 * W + stride, 4 * W + 5]
    recs = [_record(3, T, 11 + s) for s, T in enumerate(totals)]
    ann = _annotator(models, stride)
    ann.thresholds["ppk"] = _threshold(ann, recs)
    ppks = [ann.pick_phases(ann.annotate(r[None]))["ppk"] for r in recs]
    M = sum(p[0].numel() for p in ppks)
    assert M > 0
    for ratio in (0.0, 0.3):
        ch = EV.EventCharacterizer({h: models[h] for h in HEADS}, window=W, p_position_ratio=ratio, batch=3)
        want = [ch(r[None], p) for r, p in zip(recs, ppks)]
        for seed, silent in ((stride, (1,)), (stride + 1, (0, 2))):
            cs = ch.open_ragged_stream(ann, len(recs))
            outs = _run(cs, recs, _schedule(totals, 8, seed, silent))
            assert sum(o.out.ppk[0].numel() for o in outs) == M
            for o in outs:
                for h in HEADS:
                    assert o.events[h].shape[0] == o.out.ppk[0].numel()
            for s in range(len(recs)):
                assert torch.equal(_station(outs, s, "ppk"), ppks[s][0]), (stride, ratio, seed, s)
                for h in HEADS:
                    assert torch.equal(_station(outs, s, h), want[s][h]), (stride, ratio, seed, h, s)


def test_equal_lengths_equal_the_characterized_stream(models):
    S, W = 3, 8192
    rec = torch.stack([_record(3, 4 * W + 999, 3 + s) for s in range(S)])
    ann = _annotator(models, 3000, 5)
    ann.thresholds["ppk"] = _threshold(ann, list(rec))
    ch = EV.EventCharacterizer({"emg": models["emg"], "pmp": models["pmp"]}, window=W, p_position_ratio=0.3, batch=4)
    plain, ragged = ch.open_stream(ann, S), ch.open_ragged_stream(ann, S)
    pos, total = 0, 0
    for n in [5000, 1, 8191, 0, 12000, 3000, 7, rec.shape[2] - 28199, None]:
        if n is None:
            a, b = plain.close(), ragged.close()
        else:
            a = plain.push(rec[:, :, pos:pos + n].contiguous())
            b = ragged.push([rec[s, :, pos:pos + n].contiguous() for s in range(S)])
            pos += n
        for x, y in zip(a.out.ppk, b.out.ppk):
            assert torch.equal(x, y)
        for h in ("emg", "pmp"):
            assert torch.equal(a.events[h], b.events[h]), (n, h)
        # the equal-rate stream keeps one bound for all stations, the lowest of the per-station ones
        assert (ragged.held_samples <= plain.held_samples).all(), (n, ragged.held_samples, plain.held_samples)
        total += b.out.ppk[0].numel()
    assert total > 0 and plain.forwards == ragged.forwards


def _probs_outputs(probs):
    """Window outputs that repeat each station's stacked probabilities: with stack "max" the oracle stacks them back."""
    def outputs(x, ids):
        return np.stack([probs[s][:, a:a + 8192] for s, a in ids]).astype(np.float32)
    return outputs


def test_launches_replays_and_held_samples(models):
    W, B = 8192, 2
    totals = [4 * W + 77, 3 * W + 500, 2 * W + 11]
    S = len(totals)
    recs = [_record(3, T, 12 + s) for s, T in enumerate(totals)]
    ann = _annotator(models, 4096, stack="max")
    ann.thresholds["ppk"] = _threshold(ann, recs)
    ch = EV.EventCharacterizer({"baz": models["baz"], "emg": models["emg"]}, window=W, p_position_ratio=0.3, batch=B)
    replays = []
    for name, g in ch.graphs.items():
        orig = g.replay
        g.replay = lambda orig=orig, name=name: (replays.append(name), orig())[1]
    probs = [ann.annotate(r[None])[0].cpu().numpy() for r in recs]
    ref = RaggedCharacterizedStreamRef(S, 3, W, 4096, _probs_outputs(probs), 100, (0.3, ann.thresholds["ppk"], 0.2), W, 0.3,
                                       stack="max")
    lib = _lib.lib()
    plain, cs = ann.open_ragged_stream(S), ch.open_ragged_stream(ann, S)
    sched = _schedule(totals, 7, 5, silent=(2,))
    pos, total = [0] * S, 0
    for lengths in sched + [None]:
        chunks = None if lengths is None else [r[:, p:p + n].contiguous() for r, p, n in zip(recs, pos, lengths)]
        torch.cuda.synchronize()
        c0 = lib.seist_launch_count()
        po = plain.close() if chunks is None else plain.push(chunks)
        c1 = lib.seist_launch_count()
        r0 = len(replays)
        co = cs.close() if chunks is None else cs.push(chunks)
        c2 = lib.seist_launch_count()
        rc = ref.close() if chunks is None else ref.push([c.cpu().numpy() for c in chunks])
        m = co.out.ppk[0].numel()
        assert torch.equal(po.ppk[0], co.out.ppk[0])
        grew = chunks is not None and any(lengths)
        assert (c2 - c1) - (c1 - c0) == (1 if grew else 0) + -(-m // B), (lengths, m)
        assert replays[r0:] == ["baz", "emg"] * -(-m // B)
        assert np.array_equal(co.out.ppk[0].cpu().numpy(), rc[0][0]) and np.array_equal(co.out.ppk[2].cpu().numpy(), rc[0][2])
        assert (cs.held_samples == rc[3]).all(), (cs.held_samples, rc[3])
        total += m
        if lengths is not None:
            pos = [p + n for p, n in zip(pos, lengths)]
    assert total > 0 and cs.forwards == plain.forwards


def test_memory_does_not_grow(models):
    ann = _annotator(models, 4096, batch=8)
    ch = EV.EventCharacterizer({"dis": models["dis"]}, window=8192, p_position_ratio=0.3, batch=8)
    S = 3
    recs = [_record(3, 50 * 4000, 60 + s) for s in range(S)]
    ann.thresholds["ppk"] = _threshold(ann, [r[:, :40_000] for r in recs])
    cs = ch.open_ragged_stream(ann, S)
    rng = np.random.default_rng(0)
    pos = np.zeros(S, np.int64)
    held, mem = [], []
    for i in range(50):
        n = rng.integers(0, 4000, S)
        cs.push([r[:, p:p + k].contiguous() for r, p, k in zip(recs, pos, n)])
        pos += n
        torch.cuda.synchronize()
        held.append(int(cs.held_samples.max()))
        mem.append(torch.cuda.memory_allocated())
    assert max(held[25:]) <= max(held[5:25]) + 4000, held
    assert max(mem[25:]) <= max(mem[5:25]), mem


def test_argument_errors_raise_before_launch(models):
    ann = _annotator(models, 4096, batch=2)
    ch = EV.EventCharacterizer({"pmp": models["pmp"]}, window=8192, p_position_ratio=0.3, batch=2)
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    cpu = copy.copy(ann)
    cpu.model = torch.nn.Linear(2, 2)                                      # a model on another device
    with pytest.raises(ValueError):
        ch.open_ragged_stream(cpu, 2)
    two = copy.copy(ann)
    two.in_channels = 2
    with pytest.raises(ValueError):
        ch.open_ragged_stream(two, 2)                                      # channel counts differ
    short = copy.copy(ann)
    short.window = 4096                                                    # 8192 - 2457 > 4096
    with pytest.raises(ValueError):
        ch.open_ragged_stream(short, 2)
    unset = copy.copy(ann)
    unset.min_peak_dist = None
    with pytest.raises(ValueError):
        ch.open_ragged_stream(unset, 2)
    cs = ch.open_ragged_stream(ann, 2)
    ok = torch.zeros(3, 100, device="cuda")
    with pytest.raises(ValueError):
        cs.push([ok])                                                      # wrong number of chunks
    with pytest.raises(RuntimeError):
        cs.push([ok, torch.zeros(3, 100)])                                 # CPU chunk
    with pytest.raises(ValueError):
        cs.push([ok, torch.zeros(2, 100, device="cuda")])                  # wrong C
    with pytest.raises(ValueError):
        cs.push([ok, torch.zeros(3, 100, device="cuda", dtype=torch.float64)])
    with pytest.raises(ValueError):
        cs.push([ok, torch.zeros(3, 200, device="cuda")[:, ::2]])          # not contiguous
    assert lib.seist_launch_count() == before
    assert (cs.held_samples == 0).all()
    cs.push([ok, torch.zeros(3, 9000, device="cuda")])
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError, match=r"\[0\]"):
        cs.close()                                                         # station 0 is shorter than `window`
    big = copy.copy(cs)
    big.R = cs.R + np.array([(1 << 31) - 50, 0])                            # a history reaching 2^31 samples
    with pytest.raises(ValueError):
        big.push([ok, ok])
    flat, idx = torch.zeros(100, device="cuda"), torch.zeros(5, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        EV.ragged_history_(flat, flat, idx[:2], idx[:3], ok.view(-1), idx[:3], idx[:2], idx[:3], 3, 10)   # out is held
    with pytest.raises(ValueError):
        EV.ragged_history_(flat.clone(), flat, idx[:2], idx[:2], ok.view(-1), idx[:3], idx[:2], idx[:3], 3, 10)   # offsets (S,)
    with pytest.raises(ValueError):
        EV.ragged_history_(flat.clone(), flat, idx[:2].int(), idx[:3], ok.view(-1), idx[:3], idx[:2], idx[:3], 3, 10)   # int32
    x = torch.zeros(2, 3, 8192, device="cuda")
    with pytest.raises(ValueError):
        EV.ragged_event_windows_([x], flat, idx[:2], idx[:3], idx, idx[:2], 0, 8192, 100)   # pick offsets (S,)
    with pytest.raises(ValueError):
        EV.ragged_event_windows_([x], flat, idx[:2], idx[:3], idx, idx[:3], 0, 4096, 100)   # window mismatch
    assert lib.seist_launch_count() == before
    assert not cs.closed
    cs.push([torch.zeros(3, 8192, device="cuda"), ok])
    cs.close()
    with pytest.raises(RuntimeError):
        cs.push([ok, ok])
    with pytest.raises(RuntimeError):
        cs.close()
