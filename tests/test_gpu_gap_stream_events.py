"""-m gpu: streams with data gaps with their P picks characterised as they close (seist_b200/events.py
GapCharacterizedStream, `gap_event_windows_`, csrc/stream.cu seist_gap_event_windows, DESIGN §4.23).  The cut from packed
histories over a position table equals `segment_event_windows_` on the whole record bit for bit (every norm mode, ratios
0 / 0.3 / 1, picks within `a` samples of both segment edges, stations split across batches, positions without picks,
M = 0); end to end with seist_s_dpk and seist_s_{pmp,emg,baz,dis}, each station's events equal the whole-record path with
segments bit for bit, each in the call that emits its pick and all finite, with windows cut by segment edges; gap-free
input equals RaggedCharacterizedStream call by call; the synchronisation, launch and replay budgets, held memory over 50
gapped pushes and argument errors."""
import copy

import numpy as np
import pytest
import torch

from oracle import golden as G
from seist_b200 import _lib
from seist_b200 import events as EV
from seist_b200 import stream as ST
from seist_b200.models import create_model
from test_gpu_gaps import _syncs

pytestmark = pytest.mark.gpu

HEADS = ("pmp", "emg", "baz", "dis")
W = 8192
NAN = float("nan")


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g) * (0.5 + 10 * torch.rand(S, C, 1, generator=g)) + torch.randn(S, C, 1, generator=g)
    return x.cuda()


def _dev(host):
    return torch.as_tensor(np.asarray(host, np.int64)).cuda()


# ---- the cut ------------------------------------------------------------------------------------------------------------
def _kernel_case(seed, window, a):
    """A gapped (4, 3, T) record, per station picks at and within `a` of both edges of its segments, and for each station
    a history [h0_s, R_s) that holds its picks and what they read of their segments (gap samples included)."""
    T = 3 * window + 500
    rec = _record(4, 3, T, seed)
    rng = np.random.default_rng(seed)
    rec[0, :, 1000:1010] = NAN
    rec[0, 1, 2 * window:2 * window + 3] = float("inf")
    rec[1, :, :window // 2] = NAN
    rec[3, :, 5:T - 7:window // 3] = NAN                           # many short segments
    segs = ST.gap_segments(rec, 1)
    picks, table = [[] for _ in range(4)], []
    for s in range(4):
        for on, off in zip(segs.on[segs.host_offsets[s]:segs.host_offsets[s + 1]], segs.off[segs.host_offsets[s]:segs.host_offsets[s + 1]]):
            on, off = int(on), int(off)
            cand = {on, on + 1, on + a - 1, on + a, off, off - 1, off - (window - a) + 1, off - (window - a)}
            cand |= set(rng.integers(on, off + 1, 3).tolist())
            p = sorted(c for c in cand if on <= c <= off)
            if rng.random() < 0.2:
                table.append((s, 0, -1, 0))                       # a position without picks
            table.append((s, on, off, len(p)))
            picks[s] += p
        table.append((s, 0, -1, 0))
    h0 = [max(0, min(max(t[1], p - a) for t in table if t[0] == s for p in picks[s] if t[1] <= p <= t[2]) - int(rng.integers(0, 9)))
          if picks[s] else 0 for s in range(4)]
    R = [min(T, max(min(t[2] + 1, max(p + 1, p - a + window)) for t in table if t[0] == s for p in picks[s] if t[1] <= p <= t[2])
             + int(rng.integers(0, 9))) if picks[s] else 0 for s in range(4)]
    return rec, segs, picks, table, h0, R


def _packed(rec, h0, R):
    rows = [rec[s, :, h0[s]:R[s]].reshape(-1) for s in range(rec.shape[0])]
    off = np.concatenate([[0], np.cumsum([R[s] - h0[s] for s in range(rec.shape[0])])])
    return torch.cat(rows + [torch.zeros(1, device="cuda")]), _dev(h0), _dev(off)


@pytest.mark.parametrize("mode", list(ST._MODES))
@pytest.mark.parametrize("ratio", [0.0, 0.3, 1.0])
def test_cut_equals_segment_cut_on_the_whole_record(mode, ratio):
    window = 4096
    a = EV.anchor(window, ratio)
    rec, segs, picks, table, h0, R = _kernel_case(int(ratio * 10) + len(mode), window, a)
    hist, d_h0, d_off = _packed(rec, h0, R)
    st, on, end, cnt = (np.array(v, np.int64) for v in zip(*table))
    pos_off = np.concatenate([[0], np.cumsum(cnt)])
    index = _dev([p for ps in picks for p in ps])
    offsets = _dev(np.concatenate([[0], np.cumsum([len(p) for p in picks])]))
    M, B = index.numel(), 5                                        # stations split across batches
    assert M > 20
    for e0 in range(0, M + B, B):
        got = [torch.full((B, 3, window), NAN, device="cuda") for _ in range(2)]
        want = [torch.full((B, 3, window), NAN, device="cuda")]
        EV.gap_event_windows_(got, hist, d_h0, d_off, _dev(st), _dev(on), _dev(end), _dev(pos_off), index, e0, window, a, mode)
        EV.segment_event_windows_(want, rec, segs, index, offsets, e0, window, a, mode)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[0]), e0
        assert torch.isfinite(got[0]).all()
    # M = 0: zero rows
    z = [torch.full((2, 3, window), NAN, device="cuda")]
    EV.gap_event_windows_(z, hist, d_h0, d_off, _dev(st), _dev(on), _dev(end), _dev(np.zeros(len(st) + 1)),
                          torch.zeros(0, dtype=torch.int64, device="cuda"), 0, window, a, mode)
    assert (z[0] == 0).all()


def test_malformed_table_gives_zero_rows():
    window, a = 1024, 300
    rec = _record(2, 3, 5000, 3)
    hist, d_h0, d_off = _packed(rec, [0, 100], [5000, 4000])
    x = [torch.full((4, 3, window), NAN, device="cuda")]
    # stations outside [0, S), a segment that does not hold its pick, and a pick outside the station's history
    EV.gap_event_windows_(x, hist, d_h0, d_off, _dev([7, -1, 0, 1]), _dev([0, 0, 900, 0]), _dev([4999] * 4), _dev([0, 1, 2, 3, 4]),
                          _dev([500, 600, 700, 50]), 0, window, a)
    assert (x[0] == 0).all()


# ---- end to end -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models():
    out = {}
    for h in ("dpk",) + HEADS:
        name = f"seist_s_{h}"
        m = create_model(name, in_channels=3, in_samples=W)
        m.load_state_dict(G.model_state_dict(name, W), strict=True)
        out[h] = m.cuda().eval()
    return out


def _annotator(models, stride, batch=4):
    ann = ST.ContinuousAnnotator(models["dpk"], window=W, stride=stride, batch=batch)
    ann.min_peak_dist = 100
    ann.thresholds = {"ppk": 0.2, "spk": 0.2, "det": 0.3}
    return ann


def _threshold(ann, rec):
    p = torch.cat([ann.annotate(rec[s:s + 1])[0, 1] for s in range(rec.shape[0])])
    return float(torch.quantile(p[::3].float(), 0.995))


def _gapped(ann, a):
    """Six stations of one length: random gaps; gap free; all NaN; gaps at both ends; a feed that goes down for about
    three windows; and gaps placed 200 samples after (station 5) and before (station 0) picks of the record without gaps,
    so that segment edges cut windows -> the gapped record and the gap-free one."""
    T = 6 * W + 777
    clean = _record(6, 3, T, 23)
    ann.thresholds["ppk"] = _threshold(ann, clean)
    pk = ann.pick_phases(ann.annotate(clean))["ppk"]
    idx, off = pk[0].cpu().numpy(), pk[2].cpu().numpy()
    rec = clean.clone()
    rng = np.random.default_rng(4)
    for _ in range(5):
        s0 = int(rng.integers(0, T))
        rec[0, :, s0:s0 + int(rng.integers(1, 2000))] = NAN
    rec[2] = NAN
    rec[3, :, 0] = NAN
    rec[3, 1, T - 1] = NAN
    rec[4, :, 2 * W:5 * W + 100] = NAN
    for s, sign in ((5, 1), (0, -1)):
        last = -W
        for p in idx[off[s]:off[s + 1]].tolist():
            g = p + sign * 200
            if g - last > W + 300 and W < g < T - W:
                rec[s, :, g:g + 30] = NAN
                last = g
    return rec, clean


def _schedule(S, T, kind, seed):
    if kind == "equal":
        return [np.full(S, min(6000, T - r)) for r in range(0, T, 6000)]
    rng = np.random.default_rng(seed)
    out, left = [], np.full(S, T)
    while left.any():
        n = np.minimum(left, rng.choice([0, 1, 777, 5000, 9000, 17000], size=S))
        out.append(n)
        left -= n
    return out


def _push(cs, rec, R, n):
    return cs.push([rec[s, :, R[s]:R[s] + n[s]].contiguous() for s in range(rec.shape[0])])


def _station(outs, s, key):
    parts = []
    for o in outs:
        off = o.out.ppk[2].tolist()
        parts.append((o.events[key] if key != "ppk" else o.out.ppk[0])[off[s]:off[s + 1]])
    return torch.cat(parts)


def _whole(ann, ch, rec):
    """Per station: the whole-record path with segments -> (ppk, events), and how many windows a segment edge cuts."""
    want, edged, T = [], 0, rec.shape[2]
    for s in range(rec.shape[0]):
        one = rec[s:s + 1].contiguous()
        segs = ann.segments(one)
        ppk = ann.pick_phases(ann.annotate(one, segments=segs), segments=segs)["ppk"]
        want.append((ppk, ch(one, ppk, segments=segs)))
        for p in ppk[0].tolist():
            k = int(np.searchsorted(segs.on, p, "right") - 1)
            on, off = int(segs.on[k]), int(segs.off[k])
            edged += (p - ch.anchor < on and on > 0) or (p - ch.anchor + ch.window > off + 1 and off < T - 1)
    return want, edged


@pytest.mark.parametrize("stride", [4096, 3000])
@pytest.mark.parametrize("kind", ["equal", "ragged"])
def test_events_equal_each_stations_whole_record_with_segments(models, stride, kind):
    ann = _annotator(models, stride)
    ch = EV.EventCharacterizer({h: models[h] for h in HEADS}, window=W, p_position_ratio=0.3, batch=3)
    rec, _ = _gapped(ann, ch.anchor)
    S, _, T = rec.shape
    want, edged = _whole(ann, ch, rec)
    M = sum(p[0][0].numel() for p in want)
    assert M > 0 and edged > 0, (M, edged)
    cs = ch.open_gap_stream(ann, S)
    plain = ann.open_gap_stream(S)
    outs, R = [], np.zeros(S, np.int64)
    for n in _schedule(S, T, kind, stride) + [None]:
        o = cs.close() if n is None else _push(cs, rec, R, n)
        po = plain.close() if n is None else _push(plain, rec, R, n)
        for x, y in zip(o.out.ppk, po.ppk):                           # clause 2: each event in the call of its pick
            assert torch.equal(x, y)
        for h in HEADS:
            assert o.events[h].shape[0] == o.out.ppk[0].numel()
            assert torch.isfinite(o.events[h]).all(), h                # clause 4
        outs.append(o)
        R = R if n is None else R + n
    assert cs.closed
    for s in range(S):                                                 # clause 1
        assert torch.equal(_station(outs, s, "ppk"), want[s][0][0]), s
        for h in HEADS:
            assert torch.equal(_station(outs, s, h), want[s][1][h]), (s, h)


def test_gap_free_equals_the_ragged_characterized_stream(models):
    ann = _annotator(models, 3000)
    rec = _record(4, 3, 4 * W + 999, 8)
    ann.thresholds["ppk"] = _threshold(ann, rec)
    ch = EV.EventCharacterizer({"emg": models["emg"], "baz": models["baz"]}, window=W, p_position_ratio=0.3, batch=4)
    S, _, T = rec.shape
    a, b = ch.open_gap_stream(ann, S), ch.open_ragged_stream(ann, S)
    R, total = np.zeros(S, np.int64), 0
    for n in _schedule(S, T, "ragged", 9) + [None]:
        oa = a.close() if n is None else _push(a, rec, R, n)
        ob = b.close() if n is None else _push(b, rec, R, n)
        for x, y in zip(oa.out.ppk, ob.out.ppk):
            assert torch.equal(x, y)
        for h in ("emg", "baz"):
            assert torch.equal(oa.events[h], ob.events[h]), h
        assert np.array_equal(a.held_samples, b.held_samples), (a.held_samples, b.held_samples)
        assert a.forwards == b.forwards
        total += oa.out.ppk[0].numel()
        R = R if n is None else R + n
    assert total > 0


def test_syncs_launches_and_replays(models):
    B = 2
    ann = _annotator(models, 4096)
    ch = EV.EventCharacterizer({"baz": models["baz"], "emg": models["emg"]}, window=W, p_position_ratio=0.3, batch=B)
    rec, _ = _gapped(ann, ch.anchor)
    S, _, T = rec.shape
    replays = []
    for name, g in ch.graphs.items():
        orig = g.replay
        g.replay = lambda orig=orig, name=name: (replays.append(name), orig())[1]
    lib = _lib.lib()
    plain, cs = ann.open_gap_stream(S), ch.open_gap_stream(ann, S)
    R, total = np.zeros(S, np.int64), 0
    for n in _schedule(S, T, "ragged", 11) + [None]:
        torch.cuda.synchronize()
        c0 = lib.seist_launch_count()
        po, k0 = _syncs(lambda: plain.close() if n is None else _push(plain, rec, R, n))
        c1 = lib.seist_launch_count()
        r0 = len(replays)
        co, k = _syncs(lambda: cs.close() if n is None else _push(cs, rec, R, n))
        c2 = lib.seist_launch_count()
        # the gapped stream's own: 2 per push, 1 per close and per push without samples (nothing to scan)
        assert k == k0 == (1 if n is None or not n.any() else 2), (n, k, k0)
        m = co.out.ppk[0].numel()
        assert torch.equal(po.ppk[0], co.out.ppk[0])
        grew = n is not None and n.any()
        assert (c2 - c1) - (c1 - c0) == (1 if grew else 0) + -(-m // B), (n, m)
        assert replays[r0:] == ["baz", "emg"] * -(-m // B)
        total += m
        R = R if n is None else R + n
    assert total > 0 and cs.forwards == plain.forwards


def test_memory_does_not_grow_over_gapped_pushes(models):
    ann = _annotator(models, 4096, batch=8)
    ch = EV.EventCharacterizer({"dis": models["dis"]}, window=W, p_position_ratio=0.3, batch=8)
    S = 3
    rec = _record(S, 3, 50 * 4000, 61)
    ann.thresholds["ppk"] = _threshold(ann, rec[:, :, :40_000])
    rng = np.random.default_rng(1)
    for s in range(S):
        for _ in range(40):
            g = int(rng.integers(0, rec.shape[2]))
            rec[s, :, g:g + int(rng.integers(1, 300))] = NAN
    rec[1, :, 60_000:120_000] = NAN                                    # a feed that goes down
    cs = ch.open_gap_stream(ann, S)
    pos = np.zeros(S, np.int64)
    held, mem = [], []
    for i in range(50):
        n = rng.integers(0, 4000, S)
        _push(cs, rec, pos, n)
        pos += n
        torch.cuda.synchronize()
        held.append(int(cs.held_samples.max()))
        mem.append(torch.cuda.memory_allocated())
    assert max(held[25:]) <= max(held[5:25]) + 4000, held
    assert max(mem[25:]) <= max(mem[5:25]) + (1 << 20), mem         # the picker's work buffers follow each push's length
    cs.close()


def test_argument_errors_raise_before_launch(models):
    ann = _annotator(models, 4096, batch=2)
    ch = EV.EventCharacterizer({"pmp": models["pmp"]}, window=W, p_position_ratio=0.3, batch=2)
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    cpu = copy.copy(ann)
    cpu.model = torch.nn.Linear(2, 2)
    two = copy.copy(ann)
    two.in_channels = 2
    short = copy.copy(ann)
    short.window = 4096                                                # 8192 - 2457 > 4096
    unset = copy.copy(ann)
    unset.min_peak_dist = None
    for bad in (cpu, two, short, unset):
        with pytest.raises(ValueError):
            ch.open_gap_stream(bad, 2)
    with pytest.raises(ValueError, match="65535"):
        ch.open_gap_stream(ann, 21846)                                 # S * C = 65 538 history rows
    cs = ch.open_gap_stream(ann, 2)
    ok = torch.zeros(3, 100, device="cuda")
    for chunks, err in (([ok], ValueError), ([ok, torch.zeros(3, 100)], RuntimeError),
                        ([ok, torch.zeros(2, 100, device="cuda")], ValueError),
                        ([ok, torch.zeros(3, 100, device="cuda", dtype=torch.float64)], ValueError),
                        ([ok, torch.zeros(3, 200, device="cuda")[:, ::2]], ValueError)):
        with pytest.raises(err):
            cs.push(chunks)
    assert lib.seist_launch_count() == before
    assert (cs.held_samples == 0).all()
    cs.push([ok, torch.zeros(3, 9000, device="cuda")])
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    big = copy.copy(cs)
    big.R = cs.R + np.array([(1 << 31) - 50, 0])                        # a history reaching 2^31 samples
    with pytest.raises(ValueError):
        big.push([ok, ok])
    flat, idx = torch.zeros(100, device="cuda"), torch.zeros(5, dtype=torch.int64, device="cuda")
    x = torch.zeros(2, 3, W, device="cuda")
    with pytest.raises(ValueError):
        EV.gap_event_windows_([x], flat, idx[:2], idx[:3], idx[:2], idx[:2], idx[:2], idx[:2], idx, 0, W, 100)   # pos_off (n_pos,)
    with pytest.raises(ValueError):
        EV.gap_event_windows_([x], flat, idx[:2], idx[:3], idx[:2], idx[:3], idx[:2], idx[:3], idx, 0, W, 100)   # on (n_pos + 1,)
    with pytest.raises(ValueError):
        EV.gap_event_windows_([x], flat, idx[:2], idx[:3], idx[:2].int(), idx[:2], idx[:2], idx[:3], idx, 0, W, 100)   # int32
    with pytest.raises(ValueError):
        EV.gap_event_windows_([x], flat, idx[:2], idx[:3], idx[:2], idx[:2], idx[:2], idx[:3], idx, 0, 4096, 100)   # window
    assert lib.seist_launch_count() == before
    assert not cs.closed
    cs.push([torch.zeros(3, 8192, device="cuda"), ok])
    cs.close()
    with pytest.raises(RuntimeError):
        cs.push([ok, ok])
    with pytest.raises(RuntimeError):
        cs.close()
