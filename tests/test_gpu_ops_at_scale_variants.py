"""The op-by-op float64 check of test_gpu_ops_at_scale.py on the production configurations other than the benchmark's,
and the loss kernels at the benchmark's shape against float64 restatements of models/loss.py.

  * seist_m_dpk on (500, 3, 6000): the reference's default batch (main.py) at 60 s of 100 Hz data.  Its conv lengths
    (6000, 3001, 3000, 1501, 1500, 750, 375, 188, 187, 94) are not multiples of 4 * 2^k, so the plan reaches the generic
    conv.cu kernels (conv_fwd / conv_bwd_data), res_bwd (L % 4 != 0), ceil-mode max-pool windows with a partial tail,
    rows whose last tcconv tile / bww / bwwk chunk is partial, an uneven tile count per tcconv CTA, and a batch that is
    not a power of two.  Once with the default dispatch, once with SEIST_TCC=1.
  * seist_l_dpk and seist_s_dpk on (512, 3, 8192): pw_fwd with G = 8 and the widest channel tiles; the narrow ones.
  * seist_m_baz on (512, 3, 8192), training: headvec_fwd / headvec_bwd with the scaled sigmoid (x 360) at scale.
  * seist_m_pmp on (256, 3, 8192), eval with calibrated running statistics: the softmax headvec_fwd at the batch of
    seist_b200.events.EventCharacterizer.

The CPU tests pin what these configurations reach: together with the benchmark's they cover every kernel family of
api.cu::choose but conv_bwd_w, which no registered model uses; each runs more than one iteration of every persistent
loop it has; and the host mirror of the launch rules (test_gpu_ops_at_scale.loop_counts) assigns exactly the ops that
the library assigns to each persistent family.

seist_l_dpk at 512 holds two 13.5 GB arenas plus the float64 temporaries of its widest layer; it fits on an 80 GB
H100.  The six GPU op-by-op tests take about 90 s together there, the loss tests a few seconds.
"""
import collections
import os
import re

import pytest
import torch

import test_gpu_ops_at_scale as S
from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.models import create_model, get_model_list

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

BENCH = (S.NAME, S.N, S.L, True)
RAGGED = ("seist_m_dpk", 500, 6000, True)
LARGE = ("seist_l_dpk", 512, 8192, True)
SMALL = ("seist_s_dpk", 512, 8192, True)
BAZ = ("seist_m_baz", 512, 8192, True)
PMP_EVAL = ("seist_m_pmp", 256, 8192, False)
VARIANTS = [RAGGED, LARGE, SMALL, BAZ, PMP_EVAL]


# ---- what the configurations reach (CPU: the plan and the library's dispatch, no device) ----------------------------
def plan_families(name, length, training):
    """seist_op_family of every forward and backward op of a one-waveform plan on the CPU (the dispatch depends on the
    op's shape and channels, not on the batch)."""
    m = create_model(name, in_channels=3, in_samples=length)
    m.set_drop_rates(**S.ZERO_DROPS)
    pl = P.finalize(P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), 1, length, training).build(), training)
    return {"fwd": S._families(pl.c_fwd), "bwd": S._families(pl.c_bwd) if training else []}


def _family_names():
    src = open(os.path.join(ROOT, "seist_b200", "csrc", "api.cu")).read()
    body = src[src.index("kFamilyName[] = {"):]
    return re.findall(r'"([^"]+)"', body[:body.index("};")])


def test_every_kernel_family_is_checked_at_scale():
    """The benchmark's configuration and the variants below run every kernel family but conv_bwd_w at scale; a new
    family fails this until a configuration that reaches it is added."""
    seen = collections.Counter()
    for name, _, length, training in [BENCH] + VARIANTS:
        fams = plan_families(name, length, training)
        seen.update(fams["fwd"] + fams["bwd"])
    want = set(_family_names()) - {"none", "zero", "conv_bwd_w(simt)"}
    assert want <= set(seen), sorted(want - set(seen))
    assert "conv_bwd_w(simt)" not in seen


@pytest.mark.parametrize("length", [8192, 6000])
def test_no_registered_model_uses_conv_bwd_w(length):
    """conv_bwd_w (conv.cu) serves the weight gradients that neither bwwk nor bww has a kernel for.  No registered
    model produces such an op, so no at-scale test covers that kernel; a plan that starts using it fails here."""
    names = [n for n in get_model_list() if n.startswith("seist_")]
    assert len(names) == 15, names
    for name in names:
        fams = plan_families(name, length, True)
        assert "conv_bwd_w(simt)" not in fams["bwd"], name


@pytest.mark.parametrize("cfg,tcc_all", [(BENCH, False), (RAGGED, False), (RAGGED, True), (LARGE, False),
                                         (SMALL, False), (BAZ, False), (PMP_EVAL, False)],
                         ids=["bench", "ragged", "ragged-tcc", "large", "small", "baz", "pmp-eval"])
def test_loop_counts_of_the_variants(cfg, tcc_all):
    """Each configuration runs more than one iteration of every persistent loop it has (G > 1 for pw_fwd), and the
    host mirror of the launch rules puts exactly the ops in each persistent family that the library does."""
    name, n, length, training = cfg
    lc = S.loop_counts(name, n, length, training, tcc_all)
    fams = plan_families(name, length, training)
    # with SEIST_TCC=1 the tensor-core engine takes every 1x1 forward of the ragged plan that pw_fwd could run
    present = {"tcconv tiles/CTA"} | ({"pw_fwd G"} if not tcc_all else set()) | \
        ({"bwwk chunks/CTA", "bww chunks/CTA"} if training else set())
    assert present <= {what for what in lc if lc[what]}, {what: len(lc[what]) for what in lc}
    for what, by_phase in S.LOOP_FAMILY.items():
        assert not lc[what] or max(S.counts(lc, what)) > 1, (what, lc[what])
        if tcc_all:       # the library reads SEIST_TCC once per process: its default rule is what it reports here
            continue
        mirror = {(ph, i) for ph, i, _, _ in lc[what]}
        lib = {(ph, i) for ph, fam in by_phase.items() for i, f in enumerate(fams[ph]) if f == fam}
        assert mirror == lib, (what, "mirror only", sorted(mirror - lib), "library only", sorted(lib - mirror))
    if length % 128:
        # rows that end in a partial tile / chunk, several per CTA; tcconv CTAs that run different tile counts
        for what in ("tcconv tiles/CTA", "bwwk chunks/CTA", "bww chunks/CTA"):
            assert any(row % 128 and c > 1 for _, _, row, c in lc[what]), (what, lc[what])
        assert any(row % 128 and c != int(c) for _, _, row, c in lc["tcconv tiles/CTA"]), lc["tcconv tiles/CTA"]
    if name == "seist_l_dpk":
        assert 8 in S.counts(lc, "pw_fwd G")


# ---- the op-by-op runs ------------------------------------------------------------------------------------------------
def _ran(rep, *families):
    missing = [f for f in families if not any(fam == f for fam, _ in rep.worst)]
    assert not missing, ("no op of these families was checked", missing)


@pytest.mark.gpu
def test_training_ops_at_ragged_length():
    rep = S.check_at_scale(*RAGGED)
    _ran(rep, "conv_fwd(simt)", "conv_bwd_data(simt)", "res_bwd", "tcconv_fwd(wgmma+TMA) partial tile")


@pytest.mark.gpu
def test_training_ops_at_ragged_length_on_tensor_cores():
    S.check_on_tensor_cores(*RAGGED[:3], families=("tcconv_fwd(wgmma+TMA) partial tile",
                                                   "tcconv_bwd_data(wgmma+TMA) partial tile"))


@pytest.mark.gpu
def test_training_ops_of_the_large_model():
    S.check_at_scale(*LARGE)


@pytest.mark.gpu
def test_training_ops_of_the_small_model():
    S.check_at_scale(*SMALL)


@pytest.mark.gpu
def test_training_ops_of_the_back_azimuth_model():
    _ran(S.check_at_scale(*BAZ), "headvec_fwd", "headvec_bwd")


@pytest.mark.gpu
def test_eval_forward_of_the_polarity_model():
    _ran(S.check_at_scale(*PMP_EVAL), "headvec_fwd")


# ---- the loss kernels against float64 restatements of models/loss.py ------------------------------------------------
U = 2.0 ** -24          # fp32 unit roundoff
EPS = 1e-6              # BCELoss / CELoss._epsilon
GOUT = 0.37             # the gradient flowing into the loss scalar


def _plant(x, values, gen, frac=0.01):
    """Overwrites about `frac` of x (flattened) with each of `values`, at random positions."""
    flat = x.view(-1)
    for v in values:
        idx = torch.randint(0, flat.numel(), (max(1, int(frac * flat.numel())),), generator=gen)
        flat[idx] = v
    return x


def _run_loss(loss_fn, p, t):
    """(loss, dL/dp) of the module on the device for GOUT flowing into the loss, checking the kernels ran."""
    lib = _lib.lib()
    p = p.cuda().requires_grad_(True)
    before = lib.seist_launch_count()
    loss = loss_fn(p, t.cuda())
    (loss * GOUT).backward()
    torch.cuda.synchronize()
    assert lib.seist_launch_count() - before >= 3      # forward, mean finalize, backward
    return loss.item(), p.grad.double().cpu()


def _check(name, loss, ref, mag, grad, gref, gmag, k_loss=8, k_grad=16):
    """The loss within k_loss * u of its rounding magnitude (the mean of |term| plus the unit the logs' argument
    rounding adds), a few fp32 ulps of the loss; the gradient elementwise within k_grad * u of its magnitude (each
    element is a handful of roundings over sums and quotients of non-negative parts)."""
    assert abs(loss - ref) <= k_loss * U * mag, (name, loss, ref, (loss - ref) / (U * mag))
    r = ((grad - gref).abs() / (U * gmag).clamp_min(1e-300)).where(grad != gref, torch.zeros_like(gref))
    i = int(r.argmax())
    assert r.view(-1)[i] <= k_grad, (name, i, grad.view(-1)[i].item(), gref.view(-1)[i].item(), r.view(-1)[i].item())


def _probabilities(shape, gen):
    """Uniform (0, 1) values with exact 0 and 1 and values within eps of them planted."""
    p = torch.rand(shape, generator=gen)
    edges = [0.0, 1.0, 1e-7, 5e-7, 1e-6, 2e-6, 1.0 - 2.0 ** -24, 1.0 - 5e-7, 1.0 - 1e-6]
    return _plant(p, [torch.tensor(v, dtype=torch.float32).item() for v in edges], gen)


LOSS_SHAPES = [(512, 3, 8192), (1, 3, 1001)]    # the bench shape; one waveform with a total not a multiple of 256


@pytest.mark.gpu
@pytest.mark.parametrize("shape", LOSS_SHAPES, ids=["bench", "one-ragged"])
def test_bce_loss_kernels(shape):
    from seist_b200.models import BCELoss
    gen = torch.Generator().manual_seed(5)
    p = _probabilities(shape, gen)
    t = _plant(torch.rand(shape, generator=gen), [0.0, 1.0], gen, frac=0.2)
    loss, grad = _run_loss(BCELoss(weight=[[0.5], [1], [1]]), p, t)

    pd, td = p.double(), t.double()
    w = torch.tensor([0.5, 1.0, 1.0], dtype=torch.float64)[None, :, None]
    l1, l2 = (pd + EPS).log(), (1 - pd + EPS).log()
    ref = (-w * (td * l1 + (1 - td) * l2)).mean().item()
    mag = (w * (td * (l1.abs() + 1) + (1 - td) * (l2.abs() + 1))).mean().item()
    a, b = td / (pd + EPS), (1 - td) / (1 - pd + EPS)
    gref = -GOUT / pd.numel() * w * (a - b)
    gmag = GOUT / pd.numel() * w * (a + b)
    _check("bce", loss, ref, mag, grad, gref, gmag)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", LOSS_SHAPES, ids=["bench", "one-ragged"])
def test_huber_loss_kernels(shape):
    """delta = 1; residuals exactly +-delta and just either side of it (exact in fp32: targets on a 2^-10 grid)."""
    from seist_b200.models import HuberLoss
    gen = torch.Generator().manual_seed(6)
    t = torch.randint(-2048, 2049, shape, generator=gen).float() / 1024
    r = 3 * torch.randn(shape, generator=gen)
    offs = [s * (1 + d) for s in (1.0, -1.0) for d in (0.0, 2.0 ** -12, -2.0 ** -12, 2.0 ** -20, -2.0 ** -20)]
    r = _plant(r, offs + [0.0], gen, frac=0.02)
    p = t + r
    assert ((p - t).abs() == 1).sum() > 0
    loss, grad = _run_loss(HuberLoss(delta=1.0), p, t)

    z = (p.double() - t.double())
    az = z.abs()
    ref = torch.where(az < 1, 0.5 * az * az, az - 0.5).mean().item()
    mag = torch.where(az < 1, 0.5 * az * az, az + 0.5).mean().item()
    gref = GOUT / z.numel() * z.clamp(-1, 1)
    _check("huber", loss, ref, mag, grad, gref, gref.abs(), k_grad=8)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [512 * 8192, 1, 1001], ids=["bench", "one", "ragged"])
def test_ce_loss_kernels(rows):
    """Softmax-like rows of 3 class probabilities with soft targets; some classes have probability exactly 0 where the
    target is 0, others probability 0 or within eps of 0 and 1 under a non-zero target."""
    from seist_b200.models import CELoss
    gen = torch.Generator().manual_seed(7)
    p = torch.rand(rows, 3, generator=gen)
    t = torch.rand(rows, 3, generator=gen)
    zero = torch.rand(rows, 3, generator=gen) < 0.1
    zero[:, 0] &= ~(zero[:, 1] & zero[:, 2])
    p[zero], t[zero] = 0, 0
    p = _plant(p / p.sum(1, keepdim=True), [0.0, 1e-7, 1.0, 1.0 - 2.0 ** -24], gen, frac=0.005)
    t = t / t.sum(1, keepdim=True).clamp_min(1e-3)
    if rows == 1:
        p = torch.tensor([[0.0, 1e-7, 1.0 - 1e-7]])
        t = torch.tensor([[0.0, 0.25, 0.75]])
    w = [0.7, 1.0, 1.3]
    loss, grad = _run_loss(CELoss(weight=w), p, t)

    pd, td, wd = p.double(), t.double(), torch.tensor(w, dtype=torch.float64)[None, :]
    lg = (pd + EPS).log()
    ref = (-wd * td * lg).sum(1).mean().item()
    mag = (wd * td * (lg.abs() + 1)).sum(1).mean().item()
    gref = -GOUT / rows * wd * td / (pd + EPS)
    _check("ce", loss, ref, mag, grad, gref, gref.abs())
