"""-m gpu: characterising picked events (seist_b200/events.py, `seist_event_windows` in csrc/stream.cu).  The window cut
bit for bit against a torch restatement (zero-padded slice + `preprocess.normalize_`, the same `pr_normalize_row`) and
within 2e-6 * max|x| of the reference fixture; several destinations bit-identical to one; `EventCharacterizer` end to end
with seist_s_{pmp,emg,baz,dis} bit-identical to the module-path eval forward of the same window batches, and four models
together bit-identical to each alone; argument errors before any launch; one cut and one replay per model per batch,
without a host synchronisation."""
import os
from types import SimpleNamespace

import pytest
import torch

from oracle import event_ref as ER
from oracle import golden as G
from seist_b200 import _lib
from seist_b200 import events as EV
from seist_b200 import preprocess as PP
from seist_b200.models import create_model
import test_cpu_events as TE

pytestmark = pytest.mark.gpu

HEADS = ("pmp", "emg", "baz", "dis")


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g) * (0.5 + 10 * torch.rand(S, C, 1, generator=g)) + torch.randn(S, C, 1, generator=g)
    return x.cuda()


def _csr(per_station):
    """[[p, ...] per station] -> (index (M,) int64, offsets (S + 1,) int64) on the GPU."""
    index = torch.tensor([p for ps in per_station for p in ps], dtype=torch.int64)
    offsets = torch.zeros(len(per_station) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor([len(ps) for ps in per_station], dtype=torch.int64), 0)
    return index.cuda(), offsets.cuda()


def restate(rec, index, offsets, W, a, mode):
    """(M, C, W): torch slicing into zeros, then preprocess.normalize_."""
    S, C, T = rec.shape
    idx, off = index.tolist(), offsets.tolist()
    x = torch.zeros(len(idx), C, W, device=rec.device)
    for s in range(S):
        for e in range(off[s], off[s + 1]):
            p = idx[e]
            lo, hi = max(p - a, 0), min(p - a + W, T)
            if 0 <= p < T and lo < hi:
                x[e, :, lo - (p - a):hi - (p - a)] = rec[s, :, lo:hi]
    if len(idx):
        PP.normalize_(x, mode)
    return x


def _cut_all(rec, index, offsets, W, a, mode, B, n_dst=1):
    """Every batch of the cut, concatenated, plus the rows past M of the last batch."""
    xs = [torch.full((B, rec.shape[1], W), float("nan"), device="cuda") for _ in range(n_dst)]
    M = index.numel()
    got = [[] for _ in range(n_dst)]
    tail = None
    for e0 in range(0, M, B):
        EV.event_windows_(xs, rec, index, offsets, e0, W, a, mode)
        n = min(B, M - e0)
        for d in range(n_dst):
            got[d].append(xs[d][:n].clone())
        tail = [x[n:].clone() for x in xs]
    return [torch.cat(g) if g else torch.zeros(0, rec.shape[1], W, device="cuda") for g in got], tail


@pytest.mark.parametrize("mode", ["std", "max", ""])
@pytest.mark.parametrize("ratio", [0.0, 0.3, 1.0])
def test_event_windows_equal_torch_restatement(mode, ratio):
    S, C, W, T = 5, 3, 2048, 7000
    a = EV.anchor(W, ratio)
    rec = _record(S, C, T, 21)
    rec[3, 1, :] = -4.0                                          # constant channel: zero scale -> 1
    picks = [[0, 1, max(a - 1, 0), 3500], [], [T - 1, T - 2, 4000, 10, min(T - W + a, T - 1)], [3000, 3001], []]
    index, offsets = _csr(picks)
    want = restate(rec, index, offsets, W, a, mode)
    for B in (3, 4, 16):                                         # stations split across batches, partial last batches
        (got,), tail = _cut_all(rec, index, offsets, W, a, mode, B)
        assert torch.equal(got, want), (B, mode, ratio)
        assert (tail[0] == 0).all(), B                           # rows past M are zero
    short = _record(2, C, 1500, 22)                              # T < W: zero fill on both sides
    index, offsets = _csr([[0, 700, 1499], [a - 1 if a else 0, 20]])
    (got,), _ = _cut_all(short, index, offsets, W, a, mode, 2)
    assert torch.equal(got, restate(short, index, offsets, W, a, mode))


def test_empty_pick_lists_and_out_of_range_picks():
    rec = _record(3, 3, 5000, 23)
    index, offsets = _csr([[], [], []])
    x = torch.full((4, 3, 1024), float("nan"), device="cuda")
    EV.event_windows_([x], rec, index, offsets, 0, 1024, 300)   # M = 0: every row past M
    assert (x == 0).all()
    index, offsets = _csr([[-5, 5000], [], [123]])               # picks outside [0, T): zero rows (a divergence)
    x.fill_(float("nan"))
    EV.event_windows_([x], rec, index, offsets, 0, 1024, 300)
    assert (x[:2] == 0).all() and (x[3] == 0).all()
    assert torch.equal(x[2:3], restate(rec[2:3], index[2:], torch.tensor([0, 1], device="cuda"), 1024, 300, "std"))


def test_event_windows_match_reference_fixture():
    recs = {k: torch.from_numpy(v).cuda() for k, v in TE.records().items()}
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_event_windows.pt"))
    assert g["cases"] == TE.cases()
    samples = G.unpack(g["x"], [(TE.EW_C, TE.EW_W)] * len(TE.cases()))
    x = torch.empty(1, TE.EW_C, TE.EW_W, device="cuda")
    for case, smp in zip(TE.cases(), samples):
        rec, s, r, p, mode = case
        S = recs[rec].shape[0]
        index = torch.tensor([p], dtype=torch.int64, device="cuda")
        offsets = torch.tensor([0] * (s + 1) + [1] * (S - s), dtype=torch.int64, device="cuda")
        EV.event_windows_([x], recs[rec], index, offsets, 0, TE.EW_W, ER.anchor(TE.EW_W, r), mode)
        assert smp.err(x[0]) <= 2e-6 * smp.absmax, case


@pytest.mark.parametrize("n_dst", [2, 3, 4])
def test_every_destination_equals_the_single_one(n_dst):
    rec = _record(3, 3, 9000, 24)
    index, offsets = _csr([[0, 4000, 8999], [50], [8000, 8500, 2]])
    (one,), _ = _cut_all(rec, index, offsets, 4096, 1228, "std", 4)
    many, tail = _cut_all(rec, index, offsets, 4096, 1228, "std", 4, n_dst)
    for d in range(n_dst):
        assert torch.equal(many[d], one), d
        assert (tail[d] == 0).all(), d


@pytest.fixture(scope="module")
def models():
    out = {}
    for h in HEADS:
        name = f"seist_s_{h}"
        m = create_model(name, in_channels=3, in_samples=8192)
        m.load_state_dict(G.model_state_dict(name, 8192), strict=True)
        out[h] = m.cuda().eval()
    return out


def _picks_e2e():
    S, T, W = 3, 20000, 8192
    rec = _record(S, 3, T, 25)
    index, offsets = _csr([[0, 5000, 12000, T - 1], [], [17, 2457, 9000, 15000, T - 2, 19000]])
    return rec, index, offsets


@pytest.mark.parametrize("mode,ratio", [("std", 0.3), ("max", 0.25)])
def test_characterizer_equals_module_forward(models, mode, ratio):
    rec, index, offsets = _picks_e2e()
    W, B = 8192, 4
    M = index.numel()
    assert M % B != 0
    ch = EV.EventCharacterizer(models, window=W, p_position_ratio=ratio, batch=B, norm_mode=mode)
    out = ch(rec, (index, torch.zeros(M, device="cuda"), offsets))
    x = restate(rec, index, offsets, W, EV.anchor(W, ratio), mode)
    for h, m in models.items():
        want = []
        for e0 in range(0, M, B):
            xb = torch.zeros(B, 3, W, device="cuda")
            n = min(B, M - e0)
            xb[:n] = x[e0:e0 + n]
            with torch.no_grad():
                y = m.eval()(xb)
            want.append(y[:n, 0] if h != "pmp" else y[:n])
        want = torch.cat(want)
        assert out[h].shape == ((M, 2) if h == "pmp" else (M,)), h
        assert torch.equal(out[h], want), (h, (out[h] - want).abs().max().item())
    assert torch.allclose(out["pmp"].sum(1), torch.ones(M, device="cuda"), atol=1e-6)
    for h in HEADS:                                               # each model alone: the same bits
        alone = EV.EventCharacterizer({h: models[h]}, window=W, p_position_ratio=ratio, batch=B, norm_mode=mode)(rec, (index, offsets))
        assert list(alone) == [h] and torch.equal(alone[h], out[h]), h


def test_one_cut_and_one_replay_per_model_per_batch_without_host_sync(models):
    rec, index, offsets = _picks_e2e()
    ch = EV.EventCharacterizer({"baz": models["baz"], "dis": models["dis"]}, window=8192, p_position_ratio=0.3, batch=4)
    replays = []
    for name, g in ch.graphs.items():
        orig = g.replay
        g.replay = lambda orig=orig, name=name: (replays.append(name), orig())[1]
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ch(rec, (index, offsets))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    batches = -(-index.numel() // 4)
    assert lib.seist_launch_count() - before == batches
    assert replays == ["baz", "dis"] * batches
    empty = ch(rec, _csr([[], [], []]))
    assert lib.seist_launch_count() - before == batches and replays == ["baz", "dis"] * batches    # M = 0: nothing runs
    assert empty["baz"].shape == (0,) and empty["dis"].shape == (0,)
    assert out["baz"].shape == (index.numel(),)


def test_argument_errors_raise_before_launch(models):
    ch = EV.EventCharacterizer({"pmp": models["pmp"]}, window=8192, p_position_ratio=0.3, batch=2)
    rec, index, offsets = _picks_e2e()
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(RuntimeError):
        ch(rec.cpu(), (index, offsets))                                   # CPU record
    with pytest.raises(RuntimeError):
        ch(rec, (index.cpu(), offsets))                                   # CPU picks
    with pytest.raises(ValueError):
        ch(rec.double(), (index, offsets))                                # wrong dtype
    with pytest.raises(ValueError):
        ch(rec[0], (index, offsets))                                      # wrong shape
    with pytest.raises(ValueError):
        ch(rec[:, :2].contiguous(), (index, offsets))                     # wrong channel count
    with pytest.raises(ValueError):
        ch(rec, (index.int(), offsets))                                   # int32 picks
    with pytest.raises(ValueError):
        ch(rec, (index, offsets[:-1]))                                    # offsets not (S + 1,)
    with pytest.raises(ValueError):
        EV.event_windows_([torch.zeros(2, 3, 4096, device="cuda")], rec, index, offsets, 0, 8192, 2457)   # short rows
    with pytest.raises(ValueError):
        EV.event_windows_([torch.zeros(2, 3, 8192, device="cuda")] * 5, rec, index, offsets, 0, 8192, 2457)
    with pytest.raises(ValueError):
        EV.event_windows_([torch.zeros(2, 3, 8192, device="cuda")], rec, index, offsets, 0, 8192, 8193)  # anchor > W
    m = models["pmp"]
    for kw in (dict(p_position_ratio=-1), dict(p_position_ratio=1.5), dict(p_position_ratio=0.3, window=49153),
               dict(p_position_ratio=0.3, norm_mode="abs"), dict(p_position_ratio=0.3, batch=0)):
        with pytest.raises(ValueError):
            EV.EventCharacterizer({"pmp": m}, **kw)
    with pytest.raises(ValueError):
        EV.EventCharacterizer({f"m{i}": m for i in range(5)}, p_position_ratio=0.3)              # more than 4 models
    with pytest.raises(ValueError):
        EV.EventCharacterizer({}, p_position_ratio=0.3)
    two = create_model("seist_s_emg", in_channels=2, in_samples=8192).cuda()
    with pytest.raises(ValueError):
        EV.EventCharacterizer({"pmp": m, "emg": two}, p_position_ratio=0.3)                      # channel counts differ
    with pytest.raises(NotImplementedError):
        EV.EventCharacterizer({"dpk": create_model("seist_s_dpk", in_channels=3, in_samples=8192).cuda()}, p_position_ratio=0.3)
    with pytest.raises(TypeError):
        EV.EventCharacterizer({"pmp": m})                                                        # no default ratio
    assert lib.seist_launch_count() == before


def test_from_args_reads_the_reference_names(models):
    args = SimpleNamespace(in_samples=4096, norm_mode="max", p_position_ratio=0.3)
    ch = EV.EventCharacterizer.from_args({"emg": models["emg"]}, args, batch=2)
    assert (ch.window, ch.norm_mode, ch.anchor, ch.batch) == (4096, "max", int(4096 * 0.3), 2)
