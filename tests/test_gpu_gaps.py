"""-m gpu: whole records with data gaps (seist_b200/stream.py `gap_segments`, `annotate` / `pick_phases` with segments,
`EventCharacterizer` with segments, csrc/stream.cu, DESIGN §4.21).  The finder against numpy (tests/gaps_ref.py); the
cut and the stack bit for bit against `window_batch_` / `stack_batch_` on each segment's slice; end to end with
seist_s_dpk, each annotated segment equal to `annotate` of its own slice (probabilities, picks, detections) and NaN
everywhere else; picking across a gap shorter than min_peak_dist and more than 65 535 segments with injected
probabilities; the picking memory of many short segments next to a long one against the whole-record picker; the P picks characterised as if cut from their segment alone; the launch and synchronisation budgets
and argument errors."""
import warnings

import numpy as np
import pytest
import torch

import gaps_ref as GR
from oracle import golden as G
from seist_b200 import _lib
from seist_b200 import events as EV
from seist_b200 import preprocess as PP
from seist_b200 import stream as ST
from seist_b200.models import create_model
from test_cpu_gaps import crafted

pytestmark = pytest.mark.gpu

HEADS = ("pmp", "emg", "baz", "dis")
NAN = float("nan")


@pytest.fixture(scope="module")
def models():
    out = {}
    for h in ("dpk",) + HEADS:
        name = f"seist_s_{h}"
        m = create_model(name, in_channels=3, in_samples=8192)
        m.load_state_dict(G.model_state_dict(name, 8192), strict=True)
        out[h] = m.cuda().eval()
    return out


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g) * (0.5 + 10 * torch.rand(S, C, 1, generator=g)) + torch.randn(S, C, 1, generator=g)
    return x.cuda()


def _syncs(fn):
    """fn() and the number of host synchronisations torch reports during it."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, sum("called a synchronizing CUDA operation" in str(x.message) for x in w)   # not torch's one-time notice


def _same_table(segs, rec_np, W):
    pairs, off = GR.table(rec_np)
    assert torch.equal(segs.pairs.cpu(), torch.from_numpy(pairs)) and torch.equal(segs.offsets.cpu(), torch.from_numpy(off))
    assert np.array_equal(np.stack([segs.on, segs.off], 1).reshape(-1, 2), pairs) and np.array_equal(segs.host_offsets, off)
    assert torch.equal(segs.annotated.cpu(), torch.from_numpy(pairs[:, 1] - pairs[:, 0] + 1 >= W))
    assert torch.equal(segs.station.cpu(), torch.from_numpy(np.repeat(np.arange(rec_np.shape[0]), np.diff(off))))


def test_finder_against_numpy():
    rec, _ = crafted(16)
    dev = torch.from_numpy(rec).cuda()
    segs, n = _syncs(lambda: ST.gap_segments(dev, 16))
    _same_table(segs, rec, 16)
    assert n == 1
    short = np.ones((2, 3, 10), np.float32)
    short[1, 0, 4] = np.inf
    _same_table(ST.gap_segments(torch.from_numpy(short).cuda(), 16), short, 16)
    rng = np.random.default_rng(5)
    big = rng.standard_normal((4, 3, 1 << 20)).astype(np.float32)
    for s in range(3):                                                   # random gaps, one station gap free
        for a in rng.integers(0, 1 << 20, 300):
            big[s, rng.integers(0, 3), a:a + rng.integers(1, 2000)] = [np.nan, np.inf, -np.inf][s]
    big[1, :, :5] = np.nan
    big[2, 0, -1] = np.nan
    dev = torch.from_numpy(big).cuda()
    segs, n = _syncs(lambda: ST.gap_segments(dev, 8192))
    _same_table(segs, big, 8192)
    assert n == 1 and len(segs.on) > 600


def _gapped(S, T, seed, W):
    rec = _record(S, 3, T, seed)
    rng = np.random.default_rng(seed)
    for s in range(S - 1):
        for a in rng.integers(0, T, 3):
            rec[s, rng.integers(0, 3), a:a + rng.integers(1, 700)] = NAN
    rec[0, :, W + 5] = NAN                                               # segment [0, W + 4]
    return rec


@pytest.mark.parametrize("mode", ["mean", "max"])
@pytest.mark.parametrize("P,B", [(4096, 4), (3000, 7)])
def test_cut_and_stack_equal_each_slice(mode, P, B):
    S, W, T = 4, 8192, 60000
    rec = _gapped(S, T, P + B, W)
    segs = ST.gap_segments(rec, W)
    plan = ST.segment_plan(segs.on, segs.off, W, P, B)
    n_win = int(plan["win_off"][-1])
    win_off = torch.from_numpy(plan["win_off"]).cuda()
    y_all = torch.rand(n_win, 3, W, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    x = torch.full((B, 3, W), NAN, device="cuda")
    y = torch.full((B, 3, W), NAN, device="cuda")
    probs = torch.empty(S, 3, T, device="cuda")
    _, _, _, _, ids = GR.plan(np.stack([segs.on, segs.off], 1), W, P, B)
    assert len(ids) == n_win and len(plan["first"]) > 2
    for b, j0 in enumerate(range(0, n_win, B)):
        ST.segment_window_(x, rec, segs, win_off, n_win, W, P, j0, "std")
        m = min(B, n_win - j0)
        want = torch.stack([rec[int(segs.station[g]), :, segs.on[g] + a:segs.on[g] + a + W] for g, a in ids[j0:j0 + m]]).contiguous()
        PP.normalize_(want, "std")
        assert torch.equal(x[:m], want) and (x[m:] == 0).all()
        y[:m] = y_all[j0:j0 + m]
        ST.segment_stack_(probs, y, segs, win_off, n_win, W, P, j0, int(plan["first"][b]), int(plan["last"][b]), mode)
    ST.segment_finish_(probs, segs, W, P, mode)
    ok = torch.zeros(S, T, dtype=torch.bool)
    for g in range(len(segs.on)):
        s, on, off = int(segs.station[g]), int(segs.on[g]), int(segs.off[g])
        if off - on + 1 < W:
            continue
        ok[s, on:off + 1] = True
        sl = rec[s:s + 1, :, on:off + 1].contiguous()
        want = torch.empty(1, 3, off - on + 1, device="cuda")
        yg = y_all[plan["win_off"][g]:plan["win_off"][g + 1]]
        xs = torch.empty(B, 3, W, device="cuda")
        for w0 in range(0, yg.shape[0], B):                              # the slice's own windows and batches
            ST.window_batch_(xs, sl, W, P, w0, "std")
            yb = torch.zeros(B, 3, W, device="cuda")
            yb[:min(B, yg.shape[0] - w0)] = yg[w0:w0 + B]
            ST.stack_batch_(want, yb, W, P, w0, mode)
        ST.stack_finish_(want, W, P, mode)
        assert torch.equal(probs[s:s + 1, :, on:off + 1], want), (g, s, on, off)
    assert torch.isnan(probs).cpu().equal(~ok[:, None].expand(S, 3, T))


def _annotator(model, stride=4096, batch=3):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=stride, batch=batch)
    ann.min_peak_dist = 100
    ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
    return ann


def _e2e_record(W):
    """Four stations: gap free; gaps at 0 and T - 1 with segments of W - 1 and W; all NaN; one 50-sample gap."""
    T = 5 * W + 1234
    rec = _record(4, 3, T, 31)
    rec[1, :, 0] = NAN
    rec[1, 2, T - 1] = NAN
    rec[1, 0, W] = NAN                                                   # [1, W - 1]: W - 1 samples
    rec[1, 1, 2 * W + 1] = NAN                                           # [W + 1, 2W]: W samples
    rec[2] = NAN
    rec[3, :, 20000:20050] = NAN
    return rec


def _counting(ann):
    n = [0]
    replay = ann.graph.replay

    def counted():
        n[0] += 1
        return replay()
    ann.graph.replay = counted
    return n


def _slices(segs, W):
    return [(int(segs.station[g]), int(segs.on[g]), int(segs.off[g])) for g in range(len(segs.on)) if segs.off[g] - segs.on[g] + 1 >= W]


def test_end_to_end_equals_annotate_of_each_segment(models):
    W = 8192
    rec = _e2e_record(W)
    S, _, T = rec.shape
    ann = _annotator(models["dpk"])
    segs = ann.segments(rec)
    assert [(int(a), int(b)) for a, b in zip(segs.on[segs.host_offsets[1]:segs.host_offsets[2]], segs.off[segs.host_offsets[1]:
                                                                                                        segs.host_offsets[2]])] == \
        [(1, W - 1), (W + 1, 2 * W), (2 * W + 2, T - 2)]
    assert segs.host_offsets[3] == segs.host_offsets[2]
    n = _counting(ann)
    probs = ann.annotate(rec, segments=segs)
    plan = ST.segment_plan(segs.on, segs.off, W, ann.stride, ann.batch)
    assert n[0] == -(-int(plan["win_off"][-1]) // ann.batch)
    ann.thresholds["ppk"] = float(torch.quantile(probs[:, 1][~torch.isnan(probs[:, 1])][::3].float(), 0.995))
    picks = ann.pick_phases(probs, segments=segs)
    det = ann.detect_events(probs)
    ok = torch.zeros(S, T, dtype=torch.bool, device="cuda")
    want_pk = {k: [[] for _ in range(S)] for k in ("ppk", "spk")}
    want_det = [[] for _ in range(S)]
    for s, on, off in _slices(segs, W):
        ok[s, on:off + 1] = True
        alone = ann.annotate(rec[s:s + 1, :, on:off + 1].contiguous())
        assert torch.equal(probs[s:s + 1, :, on:off + 1], alone), (s, on, off)
        pk = ann.pick_phases(alone)
        for k in want_pk:
            want_pk[k][s].append((pk[k][0] + on, pk[k][1]))
        want_det[s].append(ann.detect_events(alone)[0] + on)
    assert torch.equal(torch.isnan(probs), ~ok[:, None].expand(S, 3, T))
    M = 0
    for k in want_pk:
        idx, val, off = picks[k]
        o = off.tolist()
        for s in range(S):
            wi = torch.cat([p[0] for p in want_pk[k][s]]) if want_pk[k][s] else idx[:0]
            wv = torch.cat([p[1] for p in want_pk[k][s]]) if want_pk[k][s] else val[:0]
            assert torch.equal(idx[o[s]:o[s + 1]], wi) and torch.equal(val[o[s]:o[s + 1]], wv), (k, s)
        M += idx.numel() if k == "ppk" else 0
    assert M > 0
    pairs, doff = det
    d = doff.tolist()
    for s in range(S):
        want = torch.cat(want_det[s]) if want_det[s] else pairs[:0]
        assert torch.equal(pairs[d[s]:d[s + 1]], want), s
    # clause 5: a gap-free record gives one segment per station and the whole-record annotation, replay for replay
    clean = _record(2, 3, T, 32)
    cs = ann.segments(clean)
    assert cs.on.tolist() == [0, 0] and cs.off.tolist() == [T - 1, T - 1]
    n[0] = 0
    a = ann.annotate(clean, segments=cs)
    r1 = n[0]
    b = ann.annotate(clean)
    assert torch.equal(a, b) and r1 == n[0] - r1
    for k in ("ppk", "spk"):
        assert all(torch.equal(u, v) for u, v in zip(ann.pick_phases(a, segments=cs)[k], ann.pick_phases(b)[k]))


def test_short_records_and_all_short_segments(models):
    ann = _annotator(models["dpk"])
    rec = _record(2, 3, 5000, 3)                                         # T < W
    rec[0, :, 100] = NAN
    segs = ann.segments(rec)
    n = _counting(ann)
    probs = ann.annotate(rec, segments=segs)
    assert n[0] == 0 and torch.isnan(probs).all()
    picks = ann.pick_phases(probs, segments=segs)
    assert picks["ppk"][0].numel() == 0 and picks["ppk"][2].tolist() == [0, 0, 0]


def test_picks_across_a_short_gap_and_many_segments():
    """Injected probabilities: candidates on both sides of a gap shorter than min_peak_dist are both kept; more than
    65 535 annotated segments (five samples each, windows of 3) are picked in groups."""
    T, mpd = 400, 30
    p = np.full(T, 0.1, np.float32)
    p[95], p[110] = 0.9, 0.8
    rec = np.ones((1, 3, T), np.float32)
    rec[0, :, 100:103] = np.nan
    probs = np.stack([p, p, p])[None].copy()
    probs[0, :, 100:103] = np.nan
    segs = ST.gap_segments(torch.from_numpy(rec).cuda(), 3)
    got = ST.pick_segments(torch.from_numpy(probs).cuda(), segs, (0.3, 0.3), mpd)
    want = GR.pick(probs, rec, 3, 1, 0.3, mpd)
    assert got[0][0].tolist() == [95, 110] == want[0].tolist()
    n = 70_000
    T = 6 * n
    rec = np.ones((2, 3, T), np.float32)
    rec[0, :, 5::6] = np.nan
    rec[1, :, 5::6] = np.nan
    rec[1, :, T // 2:] = np.nan
    rng = np.random.default_rng(8)
    probs = rng.uniform(0, 1, (2, 3, T)).astype(np.float32)
    probs[np.broadcast_to(~np.isfinite(rec).all(1, keepdims=True), probs.shape)] = np.nan
    segs = ST.gap_segments(torch.from_numpy(rec).cuda(), 3)
    assert int(segs.annotated.sum()) > 65535
    got = ST.pick_segments(torch.from_numpy(probs).cuda(), segs, (0.3, 0.4), 3)
    for k, ch, thr in ((0, 1, 0.3), (1, 2, 0.4)):
        want = GR.pick(probs, rec, 3, ch, thr, 3)
        for g, w in zip(got[k], want):
            assert np.array_equal(g.cpu().numpy(), w)
        assert want[0].size > 1000


def test_characterisation_equals_each_segment_alone(models):
    W = 8192
    rec = _e2e_record(W)
    S, _, T = rec.shape
    ann = _annotator(models["dpk"])
    segs = ann.segments(rec)
    a = EV.anchor(W, 0.3)
    spans = _slices(segs, W)
    per = [[] for _ in range(S)]
    for s, on, off in spans:                                             # picks within a of both segment edges
        per[s] += [on, on + 3, on + a // 2, (on + off) // 2, off - a // 2, off - 1, off]
    per[1] += [0, W]                                                     # in a gap
    per[3] += [20010]
    per = [sorted(p) for p in per]
    index = torch.tensor([p for ps in per for p in ps], dtype=torch.int64, device="cuda")
    offsets = torch.tensor(np.concatenate([[0], np.cumsum([len(p) for p in per])]), dtype=torch.int64, device="cuda")
    ch = EV.EventCharacterizer({h: models[h] for h in HEADS}, window=W, p_position_ratio=0.3, batch=5)
    got = ch(rec, (index, offsets), segments=segs)
    zero = ch(torch.zeros(1, 3, T, device="cuda"), (torch.tensor([5], device="cuda"), torch.tensor([0, 1], device="cuda")))
    for s in range(S):
        for e in range(int(offsets[s]), int(offsets[s + 1])):
            p = int(index[e])
            span = [(on, off) for t, on, off in spans if t == s and on <= p <= off]
            if span:
                on, off = span[0]
                alone = ch(rec[s:s + 1, :, on:off + 1].contiguous(), (torch.tensor([p - on], device="cuda"),
                                                                     torch.tensor([0, 1], device="cuda")))
            else:
                alone = zero                                             # a zero window
            for h in HEADS:
                assert torch.equal(got[h][e:e + 1], alone[h]), (s, p, h)
    empty = ch(rec, (index[:0], torch.zeros(S + 1, dtype=torch.int64, device="cuda")), segments=segs)
    assert all(empty[h].shape[0] == 0 for h in HEADS)


def test_budgets_and_argument_errors(models):
    W = 8192
    rec = _e2e_record(W)
    S, _, T = rec.shape
    ann = _annotator(models["dpk"])
    segs = ann.segments(rec)
    plan = ST.segment_plan(segs.on, segs.off, W, ann.stride, ann.batch)
    lib = _lib.lib()
    n = _counting(ann)
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        probs = ann.annotate(rec, segments=segs)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    # per batch a cut, a replay (a graph launch, not a library kernel) and a stack; one finish
    assert lib.seist_launch_count() - before == 2 * len(plan["first"]) + 1 and n[0] == len(plan["first"])
    ppk, n = _syncs(lambda: ann.pick_phases(probs, segments=segs)["ppk"])
    assert n == 1
    ch = EV.EventCharacterizer({"baz": models["baz"]}, window=W, p_position_ratio=0.3, batch=4)
    torch.cuda.set_sync_debug_mode("error")
    try:
        ch(rec, ppk, segments=segs)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    other = ann.segments(rec[:, :, :T - 1].contiguous())
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    bad = [other,                                                         # another (S, T)
           segs._replace(device=torch.device("cpu")),                     # another device
           segs._replace(pairs=segs.pairs.cpu()),                         # CPU tensors
           segs._replace(offsets=segs.offsets.int()),                     # wrong dtype
           segs._replace(pairs=segs.pairs.reshape(-1)),                   # wrong rank
           segs._replace(annotated=segs.annotated.long()),
           (segs.pairs, segs.offsets)]
    for b in bad:
        with pytest.raises(ValueError):
            ann.annotate(rec, segments=b)
        with pytest.raises(ValueError):
            ann.pick_phases(probs, segments=b)
        with pytest.raises(ValueError):
            ch(rec, ppk, segments=b)
    small = ST.ContinuousAnnotator.__new__(ST.ContinuousAnnotator)
    small.__dict__.update(ann.__dict__, window=4096)
    with pytest.raises(ValueError):
        small.annotate(rec, segments=segs)                                 # made for another window
    with pytest.raises(ValueError):
        small.pick_phases(probs, segments=segs)
    with pytest.raises(RuntimeError):
        ST.gap_segments(rec.cpu(), W)
    with pytest.raises(ValueError):
        ST.gap_segments(rec.double(), W)
    assert lib.seist_launch_count() == before


def test_picking_memory_follows_the_samples_not_rows_times_the_longest_row():
    """One gap-free station of 2^21 samples next to a station cut into 4 000 segments of 200-300 samples: picking
    pads each segment only to the longest of its power-of-two length class, so its peak allocation stays within a small
    multiple of the whole-record picker's on the same probabilities (rows x the longest row would be about 36 GB)."""
    T = 1 << 21
    rng = np.random.default_rng(11)
    rec = np.ones((2, 3, T), np.float32)
    cuts = np.cumsum(rng.integers(201, 302, 4000))
    rec[1, :, cuts[cuts < T]] = np.nan
    rec[1, :, cuts[-1]:] = np.nan
    probs = torch.from_numpy(rng.uniform(0, 1, (2, 3, T)).astype(np.float32)).cuda()
    dev_rec = torch.from_numpy(rec).cuda()
    segs = ST.gap_segments(dev_rec, 64)
    probs[torch.from_numpy(~np.isfinite(rec).all(1, keepdims=True)).expand(2, 3, T).cuda()] = NAN
    assert int(segs.annotated.sum()) > 3900 and segs.off.max() - segs.on.min() == T - 1

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated() - base

    got, seg_peak = peak(lambda: ST.pick_segments(probs, segs, (0.9, 0.95), 20))
    _, whole_peak = peak(lambda: ST.pick_peaks(probs, (1, 2), (0.9, 0.95), 20))
    assert seg_peak <= 6 * whole_peak, (seg_peak, whole_peak)
    want = GR.pick(probs.cpu().numpy(), rec, 64, 1, 0.9, 20)
    assert all(np.array_equal(g.cpu().numpy(), w) for g, w in zip(got[0], want)) and want[0].size > 1000
