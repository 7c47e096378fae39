"""The three attention kernels (csrc/attention.cu) against a float64 attention written here, at shapes chosen for the
kernels rather than the ones a model happens to make.

att_fwd and att_bwd_q stage keys and values in chunks of 128 (KV_CHUNK) and att_fwd carries an online softmax across
them; att_bwd_kv stages queries 64 at a time and runs one 128-key block per CTA.  Every model window up to 8192 samples
has at most 128 keys per attention op (Lk = L / 64), so the op-by-op tests of the models never reach a second chunk.
Here one attention op is built by hand (`att_ops`, pinned field by field to the plan's own ops on the CPU) and run with
`seist_plan_run` as training runs it: att_fwd, then att_bwd_q on the kernel's own output and log-sum-exp, then att_bwd_kv
on the `delta` that att_bwd_q wrote.

The logits of each (waveform, head) follow one pattern (`PATTERNS`): s_lj = c_l * t_j with k_j = t_j * u and q_l
proportional to the unit feature vector u - the maximum moving at every key, sitting in the last key or in key 0 with
the second chunk 100 below (its weights underflow), exact ties on both sides of the chunk boundary, |s| up to 200 - or
q = 0 (uniform weights), or random q and k at logit scales 0.1, 3 and 30.  Views start at channel c0 > 0 of buffers
wider than the op (Ct > C); the bytes around them must stay untouched.

Criterion, per (waveform, channel): the largest error over the row <= tol x the row's largest float64 magnitude, the
same expression on absolute values (as test_gpu_ops_at_scale.CHAN_TOL).  A logit computed in fp32 carries an absolute
rounding error of a few units of S_lj = |q_l|/sqrt(E) . |k_j| (a few 1e-5 at |s| = 200), which is the same relative
error in its weight, so every weight a_lj in these magnitudes carries the factor (1 + S_lj):
  out   sum_j a_j keep_j (1 + S_j) |v_j| + |o| sum_j a_j S_j
  dq    sum_j a_j (1 + S_j) (DP_j keep_j + Delta) |k_j| / sqrt(E)      DP_j = |dO| . |v_j|, Delta = |dO| . |O|
  dk    sum_l a_l (1 + S_l) (DP_l keep_l + Delta_l) |q_l| / sqrt(E)
  dv    sum_l a_l keep_l (1 + S_l) |dO_l|
  lse   max_j S_j + 1 (absolute error)            delta   Delta (the kernel's own O, contracted in float64)
"""
import ctypes
import math
import zlib
from dataclasses import dataclass
from typing import Optional

import pytest
import torch

from harness import model_drops
from oracle.plan_interp import keep_mask_range
from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.models import create_model

D = torch.float64

# About 5x the worst ratio over every case below (the comment of each entry), measured on an NVIDIA H100 80GB HBM3 at a
# 700 W power limit; the inputs are seeded and the kernels sum in a fixed order, so a rerun measures the same.  Every one
# is a few fp32 roundings of its magnitude: a case that needs a looser bound is a bug, not a tolerance.
TOL = {
    "out": 1.2e-6,       # 2.42e-7 (E16-Lq129-Lk188)
    "lse": 6e-6,         # 1.24e-6 (E16-Lq129-Lk1000)
    "delta": 1.3e-6,     # 2.58e-7 (E32-Lq2048-Lk129)
    "dq": 7e-7,          # 1.32e-7 (E8-Lq2048-Lk129)
    "dk": 3e-6,          # 5.57e-7 (E16-Lq1-Lk257)
    "dv": 3.5e-6,        # 7.20e-7 (E16-Lq1-Lk257)
}


# ---- one attention op, laid out as plan.to_c lays out the plan's -----------------------------------------------------
@dataclass
class Slot:
    """One operand view: channels c0 .. c0+C of an (N, Ct, L) buffer `x`, its gradient buffer `g` (same layout; None:
    no gradient wanted) and whether the gradient is added into `g` (`accum`)."""
    Ct: int
    c0: int
    C: int
    L: int
    x: Optional[torch.Tensor] = None
    g: Optional[torch.Tensor] = None
    accum: int = 0


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _view(s: Slot, grad: bool) -> _lib.SeistView:
    v = _lib.SeistView()
    v.x, v.g = _ptr(s.x), (_ptr(s.g) if grad else 0)
    v.Ct, v.c0, v.C, v.L = s.Ct, s.c0, s.C, s.L
    v.bn, v.bn_c0, v.act, v.accum = -1, 0, 0, (s.accum if grad else 0)
    return v


def att_ops(N, heads, q: Slot, k: Slot, v: Slot, o: Slot, p_attn=0.0, seed_attn=0, lse=None, delta=None,
            step_seed=None, dO=None):
    """(att_fwd, att_bwd_q, att_bwd_kv) as a ctypes array of three SeistOps: q (N, C, Lq), k / v (N, C, Lk), output o
    (N, C, Lq) with its gradient `dO` (same layout as o.x), scratch lse / delta (N, heads, Lq), `step_seed` a device
    int64 scalar.  The backward ops take q / k / v with their gradient buffers and `accum` flags."""
    ops = (_lib.SeistOp * 3)()
    for i, kind in enumerate((_lib.ATT_FWD, _lib.ATT_BWD_Q, _lib.ATT_BWD_KV)):
        c, bw = ops[i], kind != _lib.ATT_FWD
        c.kind, c.N = kind, N
        c.step_seed = _ptr(step_seed)
        for j, s in enumerate((q, k, v)):
            c.inp[j] = _view(s, bw)
        c.out = _view(o, False)
        if bw:
            c.out_dxd = _ptr(dO)
        c.n_in, c.Cin, c.Cout, c.k, c.stride, c.groups, c.pool = 3, q.C, q.C, 1, 1, 1, 1
        c.L_in, c.L_out, c.out_scale = k.L, q.L, 1.0
        c.heads, c.p_attn, c.seed_attn = heads, p_attn, seed_attn
        c.lse, c.delta = _ptr(lse), _ptr(delta)
    return ops


def _run(ops, i):
    base = ctypes.addressof(ops) + i * ctypes.sizeof(_lib.SeistOp)
    _lib.check(_lib.lib().seist_plan_run(base, 1, torch.cuda.current_stream().cuda_stream), f"attention op {i}")
    torch.cuda.synchronize()


# ---- the helper against the plan (CPU) -----------------------------------------------------------------------------
_OP_FIELDS = ("kind", "N", "n_in", "Cin", "Cout", "k", "stride", "pad_left", "groups", "pool", "up_src_L", "L_in",
              "L_out", "out_act", "out_scale", "p_elem", "p_path", "p_alpha", "heads", "p_attn", "seed_attn")
_VIEW_FIELDS = ("Ct", "c0", "C", "L", "bn", "bn_c0", "act", "accum")


def _fields(c):
    views = {name: getattr(c, name) for name in ("res_a", "res_b", "out")}
    views.update({f"in{j}": c.inp[j] for j in range(3)})
    return {f: getattr(c, f) for f in _OP_FIELDS} | \
        {(name, f): getattr(v, f) for name, v in views.items() for f in _VIEW_FIELDS}


def _slot(view, grad_view=None):
    t = grad_view if grad_view is not None and grad_view.buf is not None else view
    return Slot(view.buf.C, view.c0, view.C, view.buf.L, accum=t.accum if t is not view else 0)


@pytest.mark.parametrize("length", [8192, 10000])
def test_att_ops_equal_the_plans(length):
    """For every attention op of seist_m_dpk training with its default drop rates, att_ops of the same geometry equals
    the plan's att_fwd / att_bwd_q / att_bwd_kv entries in every field but the pointers."""
    m = create_model("seist_m_dpk", in_channels=3, in_samples=length)
    drops = model_drops("seist_m_dpk")
    assert drops["attn_drop_rate"] > 0
    m.set_drop_rates(**drops)
    pl = P.finalize(P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), 2, length, True).build(), True)
    fwd = [(i, f) for i, f in enumerate(pl.fwd_ops) if f.kind == _lib.ATT_FWD]
    assert len(fwd) == 4
    for i, f in fwd:
        assert f.p_attn > 0 and f.seed_attn != 0
        bq = next(j for j, b in enumerate(pl.bwd_ops) if b.fwd is f and b.kind == _lib.ATT_BWD_Q)
        assert pl.bwd_ops[bq + 1].kind == _lib.ATT_BWD_KV and pl.bwd_ops[bq + 1].fwd is f
        tq, tk, tv = pl.bwd_ops[bq].ins
        mine = att_ops(f.N, f.heads, _slot(f.ins[0], tq), _slot(f.ins[1], tk), _slot(f.ins[2], tv), _slot(f.out),
                       f.p_attn, f.seed_attn)
        for c_mine, c_plan in zip(mine, (pl.c_fwd[i], pl.c_bwd[bq], pl.c_bwd[bq + 1])):
            a, b = _fields(c_mine), _fields(c_plan)
            assert a == b, (f.name, {k: (a[k], b[k]) for k in a if a[k] != b[k]})


# ---- inputs ------------------------------------------------------------------------------------------------------------
PATTERNS = ("increasing", "last_key", "first_key", "ties", "zero_q", "large", "random0.1", "random3", "random30")


def _head_inputs(pattern, E, Lq, Lk, g):
    """(q (E, Lq), k (E, Lk)) of one (waveform, head) in float64, exactly representable in fp32."""
    u = torch.randn(E, generator=g, dtype=D)
    u /= u.norm()
    c = 1 + torch.rand(Lq, generator=g, dtype=D)                    # s_lj = c_l * t_j, c in [1, 2)
    j = torch.arange(Lk, dtype=D)
    if pattern == "increasing":                                     # the max moves at every key
        t = 12.0 * j / max(Lk - 1, 1)
    elif pattern == "last_key":
        t = torch.randn(Lk, generator=g, dtype=D)
        t[-1] = t.max() + 2.0
    elif pattern == "first_key":                                    # keys past the first chunk 100 below key 0
        t = -3 * torch.rand(Lk, generator=g, dtype=D)
        t[0] = 1.0
        t[128:] -= 100.0
    elif pattern == "ties":                                         # equal keys: bit-identical fp32 scores
        t = torch.randn(Lk, generator=g, dtype=D)
        t[[i for i in (0, 126, 127, 128, 129, 255, 256, Lk - 1) if i < Lk]] = t.max() + 1.0
    elif pattern == "large":                                        # |s| up to 200: a plain exp(s) overflows
        t = 200 * torch.rand(Lk, generator=g, dtype=D) - 100
        top = [i for i in (1, 127, 128, Lk - 2, Lk - 1) if 0 <= i < Lk]
        t[top] = 100.0 - torch.rand(len(top), generator=g, dtype=D)
    else:
        q = torch.randn(E, Lq, generator=g, dtype=D)
        k = torch.randn(E, Lk, generator=g, dtype=D)
        if pattern == "zero_q":
            q.zero_()
        else:
            q *= float(pattern[len("random"):])
        return q.float().double(), k.float().double()
    k = t[None, :] * u[:, None]
    q = (c * math.sqrt(E))[None, :] * u[:, None]
    return q.float().double(), k.float().double()


# ---- float64 reference and magnitudes -------------------------------------------------------------------------------
def _reference(q, k, v, dO, keep, E):
    """q (N, H, E, Lq), k / v (N, H, E, Lk), dO (N, H, E, Lq), keep (N, H, Lq, Lk) or None: out, lse, dq, dk, dv and the
    magnitude tensors, float64."""
    q, k, v = (t.detach().requires_grad_(True) for t in (q, k, v))
    s = q.transpose(-1, -2) @ k / math.sqrt(E)
    a = s.softmax(-1)
    lse = torch.logsumexp(s, -1)
    ak = a * keep if keep is not None else a
    o = (ak @ v.transpose(-1, -2)).transpose(-1, -2)
    dq, dk, dv = torch.autograd.grad(o, (q, k, v), dO)
    with torch.no_grad():
        a = a.detach()
        kp = keep if keep is not None else torch.ones_like(a)
        qa, ka, va, da, oa = q.abs(), k.abs(), v.abs(), dO.abs(), o.detach().abs()
        S = qa.transpose(-1, -2) @ ka / math.sqrt(E)
        aS = a * (1 + S)
        m_out = ((aS * kp) @ va.transpose(-1, -2)).transpose(-1, -2) + oa * (a * S).sum(-1)[:, :, None, :]
        DP = da.transpose(-1, -2) @ va                                       # (N, H, Lq, Lk)
        Delta = (da * oa).sum(2)                                             # (N, H, Lq)
        W = aS * (DP * kp + Delta[..., None])
        m_dq = (W @ ka.transpose(-1, -2)).transpose(-1, -2) / math.sqrt(E)
        m_dk = (qa @ W) / math.sqrt(E)
        m_dv = da @ (aS * kp)
        m_lse = S.amax(-1) + 1
    return dict(out=o.detach(), lse=lse.detach(), dq=dq, dk=dk, dv=dv, m_out=m_out, m_dq=m_dq, m_dk=m_dk, m_dv=m_dv,
                m_lse=m_lse)


def _ratio(got, ref, mag):
    """Worst over rows (all but the last index) of max |got - ref| / max mag; a row whose magnitude is 0 must match."""
    err = (got.double() - ref).abs().reshape(-1, got.shape[-1]).amax(-1)
    m = mag.reshape(-1, mag.shape[-1]).amax(-1)
    r = torch.where(err == 0, torch.zeros_like(err), err / m.clamp_min(1e-300))
    return r.max().item()


# ---- the cases -------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    E: int
    Lq: int
    Lk: int
    p_attn: float = 0.0
    step_seed: int = 0

    def __str__(self):
        return f"E{self.E}-Lq{self.Lq}-Lk{self.Lk}" + (f"-p{self.p_attn}-seed{self.step_seed:#x}" if self.p_attn else "")


LK_SWEEP = (1, 3, 4, 127, 128, 129, 131, 157, 188, 255, 256, 257, 1000)
CASES = [Case(16, 129, lk) for lk in LK_SWEEP] + \
    [Case(e, lq, lk) for lk in (128, 129, 257) for e in (8, 16, 32) for lq in (1, 63, 64, 65, 129, 2048)
     if not (e == 16 and lq == 129)] + \
    [Case(e, 129, lk, 0.2, seed) for e in (8, 32) for lk, seed in ((256, (1 << 32) + 12345), (157, (1 << 63) + 977))]
N, H = 2, 5                  # ten (waveform, head) pairs: every pattern in each case
SEED_ATTN = 0x5EED0A77


def _buffers(case, g):
    """Inputs in views of wider buffers: q at channels 2.., k and v in one buffer (v after k), out at channel 1."""
    E, Lq, Lk = case.E, case.Lq, case.Lk
    C = H * E
    qs, ks = zip(*[_head_inputs(PATTERNS[i % len(PATTERNS)], E, Lq, Lk, g) for i in range(N * H)])
    q = torch.stack(qs).view(N, C, Lq)
    k = torch.stack(ks).view(N, C, Lk)
    v = torch.randn(N, C, Lk, generator=g, dtype=D).float().double()
    dO = (torch.randn(N, C, Lq, generator=g, dtype=D) / math.sqrt(Lq)).float().double()
    qb = torch.randn(N, C + 5, Lq, generator=g)
    qb[:, 2:2 + C] = q.float()
    kvb = torch.randn(N, 2 * C + 3, Lk, generator=g)
    kvb[:, 1:1 + C] = k.float()
    kvb[:, 2 + C:2 + 2 * C] = v.float()
    return q, k, v, dO, qb.cuda(), kvb.cuda()


def _run_case(case, accum, q_grad=True):
    """Runs the three kernels on one case; returns {quantity: worst ratio}."""
    g = torch.Generator().manual_seed(zlib.crc32(str(case).encode()) + accum)
    E, Lq, Lk = case.E, case.Lq, case.Lk
    C = H * E
    q, k, v, dO, qb, kvb = _buffers(case, g)
    dev = torch.device("cuda")
    ob = torch.full((N, C + 4, Lq), float("nan"), device=dev)
    dOb = torch.randn(N, C + 4, Lq, generator=g).cuda()
    dOb[:, 1:1 + C] = dO.float().cuda()
    pre_q = torch.randn(qb.shape, generator=g).cuda()
    pre_kv = torch.randn(kvb.shape, generator=g).cuda()
    gq, gkv = pre_q.clone(), pre_kv.clone()
    lse = torch.full((N, H, Lq), float("nan"), device=dev)
    delta = torch.full((N, H, Lq), float("nan"), device=dev)
    seed_t = torch.tensor([case.step_seed - (1 << 64) if case.step_seed >> 63 else case.step_seed],
                          dtype=torch.int64, device=dev)
    qs = Slot(C + 5, 2, C, Lq, qb, gq if q_grad else None, accum)
    ks = Slot(2 * C + 3, 1, C, Lk, kvb, gkv, accum)
    vs = Slot(2 * C + 3, 2 + C, C, Lk, kvb, gkv, accum)
    os_ = Slot(C + 4, 1, C, Lq, ob)
    ops = att_ops(N, H, qs, ks, vs, os_, case.p_attn, SEED_ATTN if case.p_attn else 0, lse, delta, seed_t, dOb)
    qb0, kvb0, dOb0 = qb.clone(), kvb.clone(), dOb.clone()
    for i in range(3):
        _run(ops, i)
    assert torch.equal(qb, qb0) and torch.equal(kvb, kvb0) and torch.equal(dOb, dOb0)

    keep = None
    if case.p_attn > 0:
        keep = keep_mask_range(case.p_attn, case.step_seed, SEED_ATTN, N * H * Lq * Lk, dev).to(D).view(N, H, Lq, Lk)
    sh = lambda t, L: t.to(dev).view(N, H, E, L)                         # noqa: E731
    ref = _reference(sh(q, Lq), sh(k, Lk), sh(v, Lk), sh(dO, Lq), keep, E)
    out = ob[:, 1:1 + C].view(N, H, E, Lq)
    Delta_ref = (dO.to(dev).view(N, H, E, Lq) * out.double()).sum(2)
    Delta_mag = (dO.to(dev).view(N, H, E, Lq).abs() * out.double().abs()).sum(2)
    r = {"out": _ratio(out, ref["out"], ref["m_out"]),
         "lse": _ratio(lse[..., None], ref["lse"][..., None], ref["m_lse"][..., None]),
         "delta": _ratio(delta[..., None], Delta_ref[..., None], Delta_mag[..., None])}
    # bytes outside the views are untouched
    assert torch.isnan(ob[:, :1]).all() and torch.isnan(ob[:, 1 + C:]).all()
    outside_q = torch.ones(qb.shape[1], dtype=torch.bool)
    outside_q[2:2 + C] = False
    outside_kv = torch.ones(kvb.shape[1], dtype=torch.bool)
    outside_kv[1:1 + C] = outside_kv[2 + C:2 + 2 * C] = False
    assert torch.equal(gq[:, outside_q], pre_q[:, outside_q]) and torch.equal(gkv[:, outside_kv], pre_kv[:, outside_kv])
    base_q, base_kv = (pre_q, pre_kv) if accum else (torch.zeros_like(pre_q), torch.zeros_like(pre_kv))
    dq = (gq[:, 2:2 + C].double() - base_q[:, 2:2 + C].double()).view(N, H, E, Lq)
    dk = (gkv[:, 1:1 + C].double() - base_kv[:, 1:1 + C].double()).view(N, H, E, Lk)
    dv = (gkv[:, 2 + C:2 + 2 * C].double() - base_kv[:, 2 + C:2 + 2 * C].double()).view(N, H, E, Lk)
    # added into a pre-filled gradient: its rounding scales with the pre-filled values too
    pq = base_q[:, 2:2 + C].double().abs().view(N, H, E, Lq)
    pk = base_kv[:, 1:1 + C].double().abs().view(N, H, E, Lk)
    pv = base_kv[:, 2 + C:2 + 2 * C].double().abs().view(N, H, E, Lk)
    if q_grad:
        r["dq"] = _ratio(dq, ref["dq"], ref["m_dq"] + pq)
    else:
        assert torch.equal(gq, pre_q)
    r["dk"] = _ratio(dk, ref["dk"], ref["m_dk"] + pk)
    r["dv"] = _ratio(dv, ref["dv"], ref["m_dv"] + pv)
    return r


@pytest.mark.gpu
def test_attention_kernels_against_float64():
    """Every case, with the gradients written (accum = 0), added into pre-filled buffers (accum = 1) and, for q, not
    wanted (a null gradient pointer: nothing written)."""
    _lib.lib()
    worst = {}
    fails = []
    for case in CASES:
        for accum, q_grad in ((0, True), (1, True), (0, False)):
            for what, r in _run_case(case, accum, q_grad).items():
                if what not in worst or r > worst[what][0]:
                    worst[what] = (r, f"{case} accum={accum}")
                if not r <= TOL[what]:
                    fails.append(f"{case} accum={accum} q_grad={q_grad} {what}: {r:.3e} (tol {TOL[what]})")
    print(f"\n{len(CASES)} attention cases, worst error / magnitude per (waveform, channel):")
    for what, (r, where) in sorted(worst.items()):
        print(f"  {what:6s} {r:.3e}  ({where})")
    assert not fails, f"{len(fails)} failures:\n" + "\n".join(fails[:30])


def test_cases_cross_the_chunk_boundaries():
    """The cases run a second key chunk, a partial last chunk, both dropout keep paths across a chunk, more than one
    att_bwd_kv key block and query stage, and a step seed above 2^32."""
    assert {1, 127, 128, 129, 157, 256, 257, 1000} <= {c.Lk for c in CASES}
    assert {(c.E, c.Lq) for c in CASES if c.Lk == 129} == {(e, lq) for e in (8, 16, 32) for lq in (1, 63, 64, 65, 129, 2048)}
    drop = [c for c in CASES if c.p_attn > 0]
    assert any(c.Lk % 4 == 0 and c.Lk > 128 for c in drop) and any(c.Lk % 4 and c.Lk > 128 for c in drop)
    assert all(c.step_seed >= 1 << 32 for c in drop)
    assert N * H >= len(PATTERNS)
