"""-m gpu: the P picks of a streamed record characterised as they close (seist_b200/events.py CharacterizedStream and
push_history_, `seist_ragged_history` in csrc/stream.cu).  The history kernel against slices of the whole record and the rebased cut
bit for bit against the cut of the whole record (bases near 2^40 included); seist_s_dpk streamed with
seist_s_{pmp,emg,baz,dis} bit-identical per station to `ch(record, pick_phases(annotate(record))["ppk"])`; the launches of
a call over a plain ContinuousStream; bounded state; argument errors before any launch."""
import copy

import numpy as np
import pytest
import torch

from oracle import golden as G
from seist_b200 import _lib
from seist_b200 import events as EV
from seist_b200 import stream as ST
from seist_b200.models import create_model
from test_gpu_events import _csr, _cut_all

pytestmark = pytest.mark.gpu

HEADS = ("pmp", "emg", "baz", "dis")


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g) * (0.5 + 10 * torch.rand(S, C, 1, generator=g)) + torch.randn(S, C, 1, generator=g)
    return x.cuda()


def _history_steps(rec, split, keeps, base):
    """Drive push_history_ as CharacterizedStream does over rec pushed in `split` (one dense (S, C, n) chunk per step),
    a non-empty push keeping [keep, R) (global indices from `base`) -> per step the (S, C, R - h0) history, h0 and R.
    The buffers start NaN and large enough for the whole record, so every sample the history shows was written."""
    S, C, T = rec.shape
    bufs = [torch.full((S * C * T,), float("nan"), device="cuda") for _ in range(2)]
    desc = torch.zeros(2 * S + 1, dtype=torch.int64, device="cuda")
    h0, R = base, base
    for n, keep in zip(split, keeps):
        if n:
            hp = EV.ragged_history_plan(np.full(S, h0), np.full(S, R), np.full(S, n), np.full(S, keep))
            chunk = rec[:, :, R - base:R - base + n].contiguous()
            desc = EV.push_history_(bufs, desc, hp, chunk, n * np.arange(S + 1), C)
            h0 = keep
        R += n
        yield bufs[0][:S * C * (R - h0)].view(S, C, R - h0), h0, R


@pytest.mark.parametrize("base", [0, (1 << 40) - 7000])
def test_shared_history_and_rebased_cut_equal_the_whole_record(base):
    S, C, T, W = 5, 3, 30_000, 2048
    rec = _record(S, C, T, 31)
    rec[2, 1, :] = 3.0                                                     # a constant channel
    rng = np.random.default_rng(7)
    split = [1, 2500, 0, 4000, 1, 7000, 6000, 3000, 0, 7498]
    assert sum(split) == T
    keeps, k, R = [], base, base
    for i, n in enumerate(split):                                          # monotone, at most R + n
        k = min(R + n, k + int(rng.integers(0, 4000)))
        if i == 6:
            k = max(k, R + 100)                                            # past the held samples, into the chunk
        keeps.append(k)
        R += n
    assert all(a <= b for a, b in zip(keeps, keeps[1:]))
    checked = 0
    for step, (hist, h0, R) in enumerate(_history_steps(rec, split, keeps, base)):
        assert hist.shape == (S, C, R - h0)
        assert torch.equal(hist, rec[:, :, h0 - base:R - base])
        for mode in ("std", "max", ""):
            for ratio in (0.0, 0.3, 1.0):
                a = EV.anchor(W, ratio)
                lo = h0 - base + a if h0 > base else 0                       # the picks the retention rule admits
                hi = T - 1 if R - base == T else R - base - max(1, W - a)  # a pushed pick, its window pushed
                picks = []
                for s in range(S):
                    if s == 1 or lo > hi:
                        picks.append([])                                   # stations without picks
                        continue
                    ps = {lo, hi} | set(rng.integers(lo, hi + 1, 3).tolist())
                    picks.append(sorted(ps))
                index, offsets = _csr(picks)
                (whole,), _ = _cut_all(rec, index, offsets, W, a, mode, 3)  # stations split across batches of 3
                (got,), _ = _cut_all(hist, index + base - h0, offsets, W, a, mode, 3)
                assert torch.equal(got, whole), (step, mode, ratio)
                checked += index.numel()
        empty = torch.full((2, C, W), float("nan"), device="cuda")         # M = 0: zero rows
        e_idx, e_off = _csr([[]] * S)
        EV.event_windows_([empty], hist if hist.shape[2] else rec, e_idx, e_off, 0, W, 0)
        assert (empty == 0).all()
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


def _annotator(models, stride, batch=4):
    ann = ST.ContinuousAnnotator(models["dpk"], window=8192, stride=stride, batch=batch)
    ann.min_peak_dist = 100
    ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
    return ann


def _per_station(csr, S):
    *vals, off = csr
    o = off.tolist()
    return [[v[o[s]:o[s + 1]] for v in vals] for s in range(S)]


def _splits(T, seed):
    rng = np.random.default_rng(seed)
    yield "one chunk", [T]
    yield "1000", [1000] * (T // 1000) + [T % 1000]
    yield "8191", [8191] * (T // 8191) + [T % 8191]
    yield "random", np.diff([0] + sorted(rng.integers(0, T, 9).tolist()) + [T]).tolist()


def _stream(cs, rec, split):
    outs, pos = [], 0
    for n in split:
        outs.append(cs.push(rec[:, :, pos:pos + n].contiguous()))
        pos += n
    outs.append(cs.close())
    return outs


@pytest.mark.parametrize("stride", [4096, 3000])
def test_stream_events_equal_whole_record(models, stride):
    S, W = 3, 8192
    T = 5 * W + 1234
    rec = _record(S, 3, T, 11)
    ann = _annotator(models, stride)
    probs = ann.annotate(rec)
    # a P threshold that the synthetic parameters cross a few times per station
    ann.thresholds["ppk"] = float(torch.quantile(probs[:, 1].flatten()[::3].float(), 0.995))
    ppk = ann.pick_phases(probs)["ppk"]
    M = ppk[0].numel()
    assert M > 0
    for ratio in (0.0, 0.3):
        ch = EV.EventCharacterizer({h: models[h] for h in HEADS}, window=W, p_position_ratio=ratio, batch=3)
        want = ch(rec, ppk)
        want_s = {h: _per_station((want[h], ppk[2]), S) for h in HEADS}
        for label, split in _splits(T, stride):
            cs = ch.open_stream(ann, S)
            outs = _stream(cs, rec, split)
            assert sum(o.out.ppk[0].numel() for o in outs) == M, label
            for o in outs:
                for h in HEADS:
                    assert o.events[h].shape[0] == o.out.ppk[0].numel()
            for h in HEADS:
                got = [_per_station((o.events[h], o.out.ppk[2]), S) for o in outs]
                for s in range(S):
                    cat = torch.cat([g[s][0] for g in got])
                    assert torch.equal(cat, want_s[h][s][0]), (stride, ratio, label, h, s)
            idx = [_per_station(o.out.ppk, S) for o in outs]
            for s in range(S):
                assert torch.equal(torch.cat([i[s][0] for i in idx]), _per_station(ppk, S)[s][0])


def test_launches_over_a_plain_stream(models):
    S, W, B = 3, 8192, 2
    T = 4 * W + 77
    rec = _record(S, 3, T, 12)
    ann = _annotator(models, 4096)
    probs = ann.annotate(rec)
    ann.thresholds["ppk"] = float(torch.quantile(probs[:, 1].flatten()[::3].float(), 0.995))
    ch = EV.EventCharacterizer({"baz": models["baz"], "emg": models["emg"]}, window=W, p_position_ratio=0.3, batch=B)
    replays = []
    for name, g in ch.graphs.items():
        orig = g.replay
        g.replay = lambda orig=orig, name=name: (replays.append(name), orig())[1]
    lib = _lib.lib()
    plain, cs = ann.open_stream(S), ch.open_stream(ann, S)
    split = [5000, 0, 9000, 1, 12000] + [T - 26001]
    pos, total = 0, 0
    for n in split + [None]:
        chunk = None if n is None else rec[:, :, pos:pos + n].contiguous()
        torch.cuda.synchronize()
        c0 = lib.seist_launch_count()
        po = plain.close() if n is None else plain.push(chunk)
        c1 = lib.seist_launch_count()
        r0 = len(replays)
        co = cs.close() if n is None else cs.push(chunk)
        c2 = lib.seist_launch_count()
        m = co.out.ppk[0].numel()
        assert torch.equal(po.ppk[0], co.out.ppk[0])
        assert (c2 - c1) - (c1 - c0) == (1 if n else 0) + -(-m // B), (n, m)
        assert replays[r0:] == ["baz", "emg"] * -(-m // B)
        total += m
        pos += n or 0
    assert total > 0 and cs.forwards == plain.forwards


def test_state_is_bounded(models):
    ann = _annotator(models, 4096, batch=8)
    ch = EV.EventCharacterizer({"dis": models["dis"]}, window=8192, p_position_ratio=0.3, batch=8)
    S, n = 2, 3000
    cs = ch.open_stream(ann, S)
    rec = _record(S, 3, 50 * n, 13)
    held, mem = [], []
    for i in range(50):
        cs.push(rec[:, :, i * n:(i + 1) * n].contiguous())
        torch.cuda.synchronize()
        held.append(cs.held_samples)
        mem.append(torch.cuda.memory_allocated())
    assert max(held[25:]) <= max(held[5:25]), held
    assert max(mem[25:]) <= max(mem[5:25]), mem


def test_stream_and_history_argument_errors_raise_before_launch(models):
    ann = _annotator(models, 4096, batch=2)
    ch = EV.EventCharacterizer({"pmp": models["pmp"]}, window=8192, p_position_ratio=0.3, batch=2)
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    cpu = copy.copy(ann)
    cpu.model = torch.nn.Linear(2, 2)                                      # a model on another device
    with pytest.raises(ValueError):
        ch.open_stream(cpu, 2)
    two = copy.copy(ann)
    two.in_channels = 2
    with pytest.raises(ValueError):
        ch.open_stream(two, 2)                                             # channel counts differ
    short = copy.copy(ann)
    short.window = 4096                                                    # 8192 - 2457 > 4096
    with pytest.raises(ValueError):
        ch.open_stream(short, 2)
    unset = copy.copy(ann)
    unset.min_peak_dist = None
    with pytest.raises(ValueError):
        ch.open_stream(unset, 2)
    cs = ch.open_stream(ann, 2)
    with pytest.raises(RuntimeError):
        cs.push(torch.zeros(2, 3, 100))                                    # CPU chunk
    with pytest.raises(ValueError):
        cs.push(torch.zeros(3, 3, 100, device="cuda"))                     # wrong S
    with pytest.raises(ValueError):
        cs.push(torch.zeros(2, 2, 100, device="cuda"))                     # wrong C
    with pytest.raises(ValueError):
        cs.push(torch.zeros(2, 3, 100, device="cuda", dtype=torch.float64))
    with pytest.raises(ValueError):
        cs.push(torch.zeros(2, 3, 200, device="cuda")[:, :, ::2])          # not contiguous
    assert lib.seist_launch_count() == before
    assert cs.held_samples == 0
    cs.push(torch.zeros(2, 3, 100, device="cuda"))
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        cs.close()                                                         # fewer than `window` samples
    idx = torch.zeros(3, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        EV.ragged_history_(torch.zeros(0, device="cuda"), torch.zeros(30, device="cuda"), idx[:2], idx, torch.zeros(30, device="cuda"),
                           idx, idx[:2], idx, 3, 5)                                            # an empty history buffer
    with pytest.raises(ValueError):
        EV.ragged_history_plan([10, 10], [15, 15], [5, 5], [9, 9])                          # h0_out < h0_held
    assert lib.seist_launch_count() == before
    cs.push(torch.zeros(2, 3, 8192, device="cuda"))
    cs.close()
    with pytest.raises(RuntimeError):
        cs.push(torch.zeros(2, 3, 10, device="cuda"))
    with pytest.raises(RuntimeError):
        cs.close()
