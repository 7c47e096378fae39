"""Every training kernel op by op at the benchmark's batch shape — seist_m_dpk on (512, 3, 8192) — against the plan
interpreter in float64 on the device, with teacher forcing (the kernel plan starts each op from the interpreter's state).

At the small shapes of test_gpu_ops.py the kernels whose launch geometry follows N·L and the SM count run only their
first iteration: one sample quad per pw_fwd / pw_bwd_data / res_bwd4 thread (pw.cu::pick_G), one tile per persistent
tcconv CTA (so its mbarrier ring never changes phase between tiles), one strided chunk per bwwk / bww / conv_bwd_w CTA.
The bench shape runs all of them; `test_loop_counts_of_the_bench_shape` mirrors those rules on the host and pins that.

Two criteria per checked quantity:
  * the whole tensor: max error <= 2e-4 of the tensor's max-abs (the criterion of test_gpu_ops.py);
  * per channel: the largest error in each channel <= tol x that channel's float64 magnitude, the interpreter's
    expression evaluated on |operands| (|inputs after BN-apply / GELU|, |weights|, |gradient into the op|): sum |a||b|
    bounds the rounding of a sum of products whatever cancels in it, and a wrong channel of small magnitude (a ragged
    last channel tile, a dropped chunk) is not hidden behind the largest channel.  stat / gstat / bias entries use the
    same sums over absolute values; attention and head-vector ops use the channel's float64 max-abs.  The BatchNorm
    finalize ops and the stem composition backward (O(C) work, no batch-dependent loops) are held to the whole-tensor
    criterion only.

The three GPU tests take about 90 s together on an H100 (two ~11 GB arenas, float64 reference on the device).
test_gpu_ops_at_scale_variants.py runs the same check (`check_at_scale(name, n, length, training)`) on the other
production configurations: a ragged input length, the s and l model sizes and the vector heads;
test_gpu_ops_at_scale_dropout.py runs it with the model's default drop rates, as the benchmark trains.
"""
import ctypes
import gc
import os
import subprocess
import sys
import time

import pytest
import torch
import torch.nn.functional as F

from harness import ZERO_DROPS, build_pair, chan_err, chan_max, push_state, randomize, rel_err, run_gpu_op
from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.models import create_model
from seist_b200.plan import ACT_GELU, OUT_SIGMOID

NAME, N, L = "seist_m_dpk", 512, 8192       # bench.py's flagship workload
SM_COUNT = 132                              # H100 SXM
TOL = 2e-4
D = torch.float64

# Per-channel tolerance by (kernel family, quantity): about 5x the worst ratio measured on an NVIDIA H100 80GB HBM3 at a
# 700 W power limit over two runs of the three GPU tests below and of those of test_gpu_ops_at_scale_variants.py (the
# comment of each entry: the worst over every configuration, with the configuration where it is not the bench's).  fp32
# rounding of an n-term sum is ~sqrt(n) * 2^-24 of its magnitude (3xTF32 is about the same): up to ~1e-4 for the 4.2 M-term
# weight-gradient and BatchNorm sums of the full-length layers, ~1e-6 for the contractions over channels and taps.
# Every family sits at or below that; one that needs a looser bound than its rounding explains is a bug, not a tolerance.
CHAN_TOL = {
    ("att_bwd_kv", "grad"): 3e-5,                         # 8.89e-6 (ragged)
    ("att_bwd_q", "grad"): 3e-5,                          # 1.72e-5 (baz)
    ("att_fwd", "out"): 1e-5,                             # 2.75e-6 (l)
    ("bww(simt)", "dW"): 3e-7,                            # 7.80e-8 (baz)
    ("bww(simt)", "dbias"): 1e-7,                         # 8.46e-8 (baz; 2.45e-8 at the bench shape)
    ("bwwk(simt)", "dW"): 1e-7,                           # 5.05e-8 (baz)
    ("bwwk(simt)", "dbias"): 3e-8,                        # 6.65e-9 (l)
    ("conv_bwd_data(simt)", "grad"): 1.5e-6,              # 2.89e-7 (ragged)
    ("conv_bwd_data(simt)", "gstat"): 5e-8,               # 1.07e-8 (ragged)
    ("conv_fwd(simt)", "out"): 1.5e-6,                    # 2.89e-7 (ragged)
    ("conv_fwd(simt)", "stat"): 2e-7,                     # 3.74e-8 (ragged)
    ("convk_bwd_data(simt)", "grad"): 2e-6,               # 4.08e-7
    ("convk_bwd_data(simt)", "gstat"): 3e-9,              # 5.88e-10
    ("convk_fwd(simt)", "out"): 2e-6,                     # 3.63e-7
    ("convk_fwd(simt)", "stat"): 7e-8,                    # 1.41e-8
    ("headvec_bwd", "dW"): 3.5e-6,                        # 6.86e-7 (baz)
    ("headvec_bwd", "dbias"): 2e-5,                       # 3.80e-6 (baz; a 512-term sum against its own |value|)
    ("headvec_bwd", "grad"): 8e-7,                        # 1.56e-7 (baz)
    ("headvec_fwd", "out"): 1.5e-6,                       # 2.81e-7 (pmp eval)
    ("pw_bwd_data(simt)", "grad"): 1.5e-6,                # 3.42e-7 (l)
    ("pw_bwd_data(simt)", "gstat"): 1.5e-8,               # 4.23e-9 (baz)
    ("pw_bwd_data_staged(simt)", "grad"): 1.5e-6,         # 2.71e-7
    ("pw_bwd_data_staged(simt)", "gstat"): 1e-8,          # 3.82e-9 (baz)
    ("pw_fwd(simt)", "out"): 2e-6,                        # 4.16e-7
    ("pw_fwd(simt)", "stat"): 2e-7,                       # 5.25e-8 (s)
    ("res_bwd", "grad"): 1e-6,                            # 2.10e-7 (ragged)
    ("res_bwd", "gstat"): 1e-7,                           # 2.09e-8 (ragged)
    ("res_bwd4", "grad"): 7e-7,                           # 1.75e-7 (l)
    ("res_bwd4", "gstat"): 1.5e-8,                        # 1.17e-8 (baz; 2.85e-9 at the bench shape)
    ("stem_compose_fwd", "W_eff"): 7e-7,                  # 1.66e-7
    ("tcconv_bwd_data(wgmma+TMA)", "grad"): 5e-6,         # 1.04e-6 (baz)
    ("tcconv_bwd_data(wgmma+TMA)", "gstat"): 5e-8,        # 1.34e-8 (baz)
    ("tcconv_fwd(wgmma+TMA)", "out"): 7e-6,               # 1.42e-6 (l)
    ("tcconv_fwd(wgmma+TMA)", "stat"): 2e-6,              # 4.88e-7
}


# ---- host mirror of the launch rules (csrc/pw.cu, tcconv.cu, bwwk.cu, api.cu) ---------------------------------------
def _pick_G(nq, tiles_y, sm=SM_COUNT):
    ctas, G = -(-nq // 128), 1
    while G < 8 and (ctas // (2 * G)) * tiles_y >= 4 * sm:
        G *= 2
    return G


def _pw_eligible(f):
    if f.k != 1 or f.stride != 1 or f.groups != 1 or f.up_src_L > 0 or f.L_out % 4:
        return False
    if f.pool > 1:
        return (f.pool in (2, 4, 8) and len(f.ins) == 1 and f.ins[0].act == 0 and f.ins[0].L == f.L_out * f.pool
                and f.p_elem <= 0 and f.res_a is None and f.res_b is None)
    return True


def _tcc_eligible(f, mode, targets=()):
    if f.stride != 1 or f.pool > 1 or f.k > 32 or (f.Cout if mode == 0 else f.Cin) > 128:
        return False
    if f.L_in != f.L_out or f.L_out % 4:
        return False
    if f.up_src_L > 0:
        return (mode == 0 and len(f.ins) == 1 and f.L_in == 2 * f.up_src_L and f.up_src_L % 4 == 0
                and f.ins[0].L == f.up_src_L)
    if f.Cout > 256 or f.Cin > 256 or (f.k > 1 and f.p_elem > 0):
        return False
    if any(v.L != f.L_in or (len(f.ins) > 1 and v.C % 8) for v in f.ins):
        return False
    return mode == 0 or any(t.buf is not None for t in targets)


def _tcc_auto(f, mode):
    Kd = f.Cin if mode == 0 else f.Cout
    if f.up_src_L > 0:
        return mode == 0 and Kd >= 32
    if f.k > 1:
        return (f.L_out <= 512 and Kd >= 16) if mode == 0 else (f.L_out <= 256 and Kd >= 32)
    return mode == 0 and Kd >= 64 and f.L_out <= 256


def _per_cta(tiles, waves, gy_gz, sm=SM_COUNT):
    """Work items per CTA of a grid of min(waves*sm/(gy*gz), tiles) CTAs in x striding over `tiles`."""
    gx = max(1, min(tiles, -(-waves * sm // gy_gz)))
    return tiles / gx


def loop_counts(name, n, length, training=True, tcc_all=False, drops=None):
    """Per persistent family, one (phase, op index, row length, count) per op: quads per pw_fwd thread, tiles per
    tcconv CTA (the default dispatch rule, or every eligible op with `tcc_all`, as SEIST_TCC=1), strided chunks per
    bwwk CTA and per bww CTA (1x1 and the k-tap convs that bwwk has no kernel for) - from the plan's op fields only
    (no CUDA library).  `drops`: the drop rates of the plan (None: no dropout)."""
    m = create_model(name, in_channels=3, in_samples=length)
    m.set_drop_rates(**(ZERO_DROPS if drops is None else drops))
    pl = P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), n, length, training).build()
    out = {what: [] for what in LOOP_FAMILY}
    for i, f in enumerate(pl.fwd_ops):
        if f.kind != _lib.CONV_FWD:
            continue
        if _tcc_eligible(f, 0) and (tcc_all or _tcc_auto(f, 0)):
            out["tcconv tiles/CTA"].append(("fwd", i, f.L_out, _per_cta(n * -(-f.L_out // 128), 1, 1)))
        elif _pw_eligible(f):
            cot = 16 if f.Cout > 8 else 8
            out["pw_fwd G"].append(("fwd", i, f.L_out, _pick_G(n * (f.L_out >> 2), -(-f.Cout // cot))))
    if not training:
        return out
    for i, op in enumerate(pl.bwd_ops):
        f = op.fwd
        if op.kind == _lib.CONV_BWD_DATA and _tcc_eligible(f, 1, op.ins) and (tcc_all or _tcc_auto(f, 1)):
            out["tcconv tiles/CTA"].append(("bwd", i, f.L_in, _per_cta(n * -(-f.L_in // 128), 1, 1)))
        if op.kind != _lib.CONV_BWD_W:
            continue
        gs_in, gs_out = f.Cin // f.groups, f.Cout // f.groups
        bwwk_ks = {1: (3, 5, 7, 9, 11, 13), 2: (7, 11, 15, 19)}
        if len(f.ins) == 1 and f.pool <= 1 and f.L_out % 4 == 0 and f.k in bwwk_ks.get(f.stride, ()):
            co_b = 8 if gs_out <= 8 else (32 if f.k <= 7 and f.stride == 1 and gs_out >= 32 else 16)
            ntile = -(-gs_in // 16)
            ci_b = -(-gs_in // ntile)
            pc = 512 if f.L_out >= 2048 and co_b + ci_b <= 24 else (256 if f.L_out >= 256 else 128)
            pc = min(pc, (f.L_out + 3) & ~3)
            gy = f.groups * -(-gs_out // co_b)
            out["bwwk chunks/CTA"].append(("bwd", i, f.L_out, _per_cta(n * -(-f.L_out // pc), 2, gy * ntile)))
        elif not (f.groups > 1 and (gs_in < 8 or gs_out < 8)) and not ((f.k > 1 or f.pool > 1) and len(f.ins) != 1):
            # pw.cu::launch_bww_sel / launch_bww: the reduction runs over R = gs_in * k (input channel, tap) rows
            R = gs_in * f.k
            co_b = 8 if gs_out <= 8 else (16 if gs_out <= 16 else 32)
            r_b = 8 if R <= 8 else (16 if R <= 16 else (32 if R <= 32 else 64))
            rows = co_b + min((r_b + f.k - 1) // f.k + 1, gs_in)
            pc = 512 if rows <= 32 and f.L_out >= 2048 else (256 if rows <= 96 and f.L_out >= 512 else 128)
            gy, gz = f.groups * -(-gs_out // co_b), -(-R // r_b)
            out["bww chunks/CTA"].append(("bwd", i, f.L_out, _per_cta(n * -(-f.L_out // pc), 2, gy * gz)))
    return out


# the kernel family (api.cu::choose) of every op that loop_counts puts under a key, by phase
LOOP_FAMILY = {
    "pw_fwd G": {"fwd": "pw_fwd(simt)"},
    "tcconv tiles/CTA": {"fwd": "tcconv_fwd(wgmma+TMA)", "bwd": "tcconv_bwd_data(wgmma+TMA)"},
    "bwwk chunks/CTA": {"bwd": "bwwk(simt)"},
    "bww chunks/CTA": {"bwd": "bww(simt)"},
}


def counts(lc, what):
    return [c for _, _, _, c in lc[what]]


def test_loop_counts_of_the_bench_shape():
    """The at-scale GPU tests below run the multi-iteration paths that the small op-by-op shapes never reach."""
    big = loop_counts(NAME, N, L)
    assert {2, 4} <= set(counts(big, "pw_fwd G")), counts(big, "pw_fwd G")
    for what in ("tcconv tiles/CTA", "bwwk chunks/CTA", "bww chunks/CTA"):
        assert big[what] and max(counts(big, what)) > 1, (what, big[what])
    from test_gpu_ops import CASES
    for name, n, length, training, _ in CASES:
        small = loop_counts(name, n, length, training)
        for what in small:
            assert all(c == 1 for c in counts(small, what)), (name, n, length, what, small[what])


# ---- float64 magnitudes of the interpreter's expressions -------------------------------------------------------------
def _conv_lin(f, X, W):
    """Interp._conv_expr on input channels that are already activated."""
    if f.pool > 1:
        X = F.avg_pool1d(X, f.pool, ceil_mode=True) + F.max_pool1d(X, f.pool, ceil_mode=True)
    elif f.up_src_L > 0:
        X = F.interpolate(X, size=f.L_in, mode="linear")
    pr = (f.L_out - 1) * f.stride + f.k - f.L_in - f.pad_left
    return F.conv1d(F.pad(X, (f.pad_left, pr)), W, None, stride=f.stride, groups=f.groups)


def _fwd_mag(it, f):
    Y = _conv_lin(f, torch.cat([it.value(v).abs() for v in f.ins], 1), it._W(f).abs())
    b = it._bias(f)
    if b is not None:
        Y = Y + b.abs()[None, :, None]
    fac, alpha = it._drop_factor(f)
    Y = Y * fac
    if f.res_a is not None:
        Y = Y + it.value(f.res_a).abs()
    Y = Y * alpha
    if f.res_b is not None:
        Y = Y + it.value(f.res_b).abs()
    if f.out_act == OUT_SIGMOID:
        Y = 0.25 * Y                          # |sigmoid'| <= 1/4
    return Y


def _grad_in_mag(it, f):
    """Interp.out_grad on absolute values: the magnitude of the gradient flowing into the op's output."""
    o = f.out
    sl = slice(o.c0, o.c0 + o.C)
    g = torch.zeros(f.N, o.C, o.buf.L, dtype=D, device=it.dev)
    if o.buf.dxd is not None:
        g = g + o.buf.dxd[:, sl].to(D).abs()
    if o.bn >= 0 and o.buf.du is not None:
        A, Bx, Cc = it.bn_bwd(o.bn, o.bn_c0, o.C)
        g = g + A.abs()[None, :, None] * o.buf.du[:, sl].to(D).abs() + Bx.abs()[None, :, None] * o.buf.x[:, sl].to(D).abs() \
            + Cc.abs()[None, :, None]
    if f.out_act == OUT_SIGMOID and f.kind == _lib.CONV_FWD:
        pr = o.buf.x[:, sl].to(D)
        g = g * (pr * (1 - pr)).abs()
    return g


def _data_grad_mags(it, op, gmag):
    """|J|^T gmag for every input that receives a gradient: the transposed conv with |W| (pooling / up-sampling /
    padding have non-negative coefficients; max-pool keeps the interpreter's selection), times |GELU'|."""
    f = op.fwd
    bases = [it.base(v) for v in f.ins]
    Xs = [it.act(b, v.act).detach().requires_grad_(True) for b, v in zip(bases, f.ins)]
    Y = _conv_lin(f, torch.cat(Xs, 1), it._W(f).abs())
    need = [i for i, t in enumerate(op.ins) if t.buf is not None]
    grads = torch.autograd.grad(Y, [Xs[i] for i in need], gmag)
    mags = {}
    for i, g in zip(need, grads):
        if f.ins[i].act == ACT_GELU:
            b = bases[i].detach().requires_grad_(True)
            (d,) = torch.autograd.grad(F.gelu(b), b, torch.ones_like(b))
            g = g * d.abs()
        mags[i] = g
    return mags


def _dw_mag(it, f, gmag):
    W = torch.zeros_like(it._W(f)).requires_grad_(True)
    Y = _conv_lin(f, torch.cat([it.value(v).abs() for v in f.ins], 1), W)
    (dW,) = torch.autograd.grad(Y, W, gmag)
    return dW


def _pool_ties(it, f, i):
    """Source samples of input i whose max-pool window has its two largest BN-applied values within fp32 rounding of
    each other.  The max's gradient goes to the first arg max, a discrete choice the kernels make on their fp32 values
    and the interpreter on float64 ones; at such a near tie either routing is right, so these samples are left out of
    the data-gradient comparison (a handful among the ~10^7 windows of a full-length pooled op).  With ceil_mode the
    last window of a row holds the remaining v.L - pool * (L_out - 1) samples only; a window of one sample has no tie."""
    v, P_ = f.ins[i], f.pool
    pad = P_ * f.L_out - v.L
    assert 0 <= pad < P_ and v.act == 0
    x = v.buf.x[:, v.c0:v.c0 + v.C].to(D)
    if v.bn >= 0:
        s_, t_ = it.bn_fwd(v.bn, v.bn_c0, v.C)
        xs, t_ = x * s_[None, :, None], t_[None, :, None]
    else:
        xs, t_ = x, torch.zeros(1, 1, 1, dtype=D, device=x.device)
    u = F.pad(xs + t_, (0, pad), value=-float("inf")).view(f.N, v.C, f.L_out, P_)
    top2 = u.topk(2, -1).values
    slack = 2.0 ** -19 * F.pad(xs.abs() + t_.abs(), (0, pad)).view(f.N, v.C, f.L_out, P_).amax(-1)   # 16 fp32 ulps
    return (top2[..., 0] - top2[..., 1] <= slack).repeat_interleave(P_, -1)[..., :v.L]


def _grad_buf(t):
    return (t.buf.du if t.bn >= 0 else t.buf.dxd)[:, t.c0:t.c0 + t.C]


# ---- the op-by-op run ------------------------------------------------------------------------------------------------
class _Report:
    def __init__(self):
        self.failures = []          # whole-tensor criterion
        self.chan_failures = []     # per-channel criterion
        self.worst = {}             # (family, quantity) -> (ratio, where)
        self.pool_ties = 0          # max-pool windows left out of the data-gradient comparison
        self.op = None              # (phase, op index) being checked
        self.drop = ""              # its dropout variant (drop_label)
        self.checked = set()        # (phase, op index) of every op held to the per-channel criterion
        self.sites = set()          # dropout_sites of the plan

    def whole(self, where, what, got, ref):
        err, mx = rel_err(got, ref)
        if not err < TOL:
            self.failures.append(f"{where} {what}: rel {err:.3e} (max {mx:.3e})")

    def chan(self, family, where, what, got, ref, scale, dim=1, mask=None, partial_tile=False):
        """`partial_tile`: a tcconv op whose rows end in a partial 128-sample tile, also reported on its own line; an op
        that applies a dropout mask or factor is also reported under its family with the variant appended."""
        if mask is not None:
            got, ref, scale, dim = got[mask], ref[mask], scale[mask], 0
        r, c = chan_err(got, ref, scale, dim)
        self.checked.add(self.op)
        key = (family, what)
        keys = [key] + ([(family + " partial tile", what)] if partial_tile else []) + \
            ([(f"{family} {self.drop}", what)] if self.drop else [])
        for k in keys:
            if k not in self.worst or r > self.worst[k][0]:
                self.worst[k] = (r, f"{where} channel {c}")
        tol = CHAN_TOL.get(key)
        if tol is None or not r <= tol:
            self.chan_failures.append(f"{where} [{family}] {what}: channel {c} error {r:.3e} x magnitude (tol {tol})")


def _families(c_ops):
    lib = _lib.lib()
    base, size = ctypes.addressof(c_ops), ctypes.sizeof(_lib.SeistOp)
    return [lib.seist_op_family(base + i * size).decode() for i in range(len(c_ops))]


def drop_label(kind, f):
    """The dropout an op of `kind` applies, its forward op `f` holding the rates: "p_elem" (element mask of a conv
    output, with its per-sample factors), "p_path" (per-sample stochastic-depth factors only), "p_alpha" (the
    residual's factor that RES_BWD applies), "p_attn" (attention-weight mask), or ""."""
    if kind in (_lib.CONV_FWD, _lib.CONV_BWD_DATA, _lib.CONV_BWD_W):
        return "p_elem" if f.p_elem > 0 else ("p_path" if f.p_path > 0 or f.p_alpha > 0 else "")
    if kind == _lib.RES_BWD:
        return "p_alpha" if f.p_alpha > 0 else ""
    if kind in (_lib.ATT_FWD, _lib.ATT_BWD_Q, _lib.ATT_BWD_KV):
        return "p_attn" if f.p_attn > 0 else ""
    return ""


def dropout_sites(pl):
    """{(phase, op index)} of every op whose kernel applies a dropout mask or factor."""
    return {("fwd", i) for i, f in enumerate(pl.fwd_ops) if drop_label(f.kind, f)} | \
        {("bwd", i) for i, op in enumerate(pl.bwd_ops) if op.fwd is not None and drop_label(op.kind, op.fwd)}


def _stat_slices(p, v):
    e = p.bns[v.bn]
    a = e.st_off + v.bn_c0
    return a, a + e.C


def _calibrated_state(name, length, steps=40):
    """harness.randomize parameters with running statistics that match them: training forwards of small batches at
    momentum 0.1 (40 steps leave 1.5 % of the random start).  Random running statistics blow the eval activations of
    the deep model up to ~1e6 and its attention softmax to a near-arg-max, where fp32 rounding of the scores decides
    the output and no kernel could be held to a tolerance."""
    m = create_model(name, in_channels=3, in_samples=length)
    randomize(m)
    m.set_drop_rates(**ZERO_DROPS)
    m.cuda().train()
    g = torch.Generator(device="cuda").manual_seed(3)
    with torch.no_grad():
        for _ in range(steps):
            m(torch.randn(8, 3, length, device="cuda", generator=g))
    torch.cuda.synchronize()
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


def run_at_scale(name, n, length, training, drops=None, step_seed=12345):
    """Runs every op of the plan on the kernels and on the float64 interpreter; returns the _Report.  `drops`: the
    drop rates (None: no dropout); `step_seed`: the dropout step counter, an unsigned 64-bit value."""
    sd = None if training else _calibrated_state(name, length)
    p_ref, p_gpu, it, _, _ = build_pair(name, n, length, training, drops=drops, ref_device="cuda", ref_dtype=D,
                                        state_dict=sd)
    rep = _Report()
    rep.sites = dropout_sites(p_ref)
    g = torch.Generator().manual_seed(1)
    p_ref.step_seed.fill_(step_seed - (1 << 64) if step_seed >> 63 else step_seed)     # int64 holds the same bits
    p_ref.x_in.x.copy_(torch.randn(n, 3, length, generator=g))
    p_ref.stat.zero_()

    for i, (fr, fg, fam) in enumerate(zip(p_ref.fwd_ops, p_gpu.fwd_ops, _families(p_gpu.c_fwd))):
        push_state(p_ref, p_gpu)
        where = f"fwd[{i}] {fr.name}"
        rep.op, rep.drop = ("fwd", i), drop_label(fr.kind, fr)
        mag = None
        pt = fam.startswith("tcconv") and fr.L_out % 128 != 0
        if fr.kind == _lib.CONV_FWD:
            mag = _fwd_mag(it, fr)
        stat0 = p_ref.stat.clone()
        it.run_fwd_op(fr)
        run_gpu_op(p_gpu, p_gpu.c_fwd, i)
        if fr.out is not None:
            sl = slice(fr.out.c0, fr.out.c0 + fr.out.C)
            got, ref = fg.out.buf.x[:, sl], fr.out.buf.x[:, sl]
            rep.whole(where, "out", got, ref)
            rep.chan(fam, where, "out", got, ref, chan_max(mag if mag is not None else ref.to(D).abs()), partial_tile=pt)
            if training and fr.out.bn >= 0:
                e = p_ref.bns[fr.out.bn]
                rep.whole(where, "stat", p_gpu.stat[e.st_off:e.st_off + 2 * e.C], p_ref.stat[e.st_off:e.st_off + 2 * e.C])
            if training and fr.out.bn >= 0 and mag is not None:
                a, a2 = _stat_slices(p_ref, fr.out)
                scale = stat0.abs()
                scale[a:a + fr.out.C] += mag.sum((0, 2))
                scale[a2:a2 + fr.out.C] += (mag * mag).sum((0, 2))
                touched = torch.zeros_like(scale, dtype=torch.bool)
                touched[a:a + fr.out.C] = touched[a2:a2 + fr.out.C] = True
                rep.chan(fam, where, "stat", p_gpu.stat, p_ref.stat, scale, mask=touched, partial_tile=pt)
        if fr.lse is not None:
            rep.whole(where, "lse", fg.lse, fr.lse)
        if fr.kind == _lib.BN_FINALIZE_FWD:
            rep.whole(where, "running", p_gpu.flat.RB, p_ref.flat.RB)
        if fr.kind == _lib.STEM_COMPOSE_FWD:
            rep.whole(where, "W_eff", p_gpu.Wx, p_ref.Wx)
            i_, d_, pc = it._parts(fr)
            wmag = torch.einsum("oc,ct,ci->oit", pc.abs(), d_.abs(), i_.abs()).reshape(fr.Cout, -1)
            sl = slice(fr.Wx.off, fr.Wx.off + fr.Wx.numel)
            rep.chan(fam, where, "W_eff", p_gpu.Wx[sl].view(fr.Cout, -1), p_ref.Wx[sl].view(fr.Cout, -1),
                     chan_max(wmag, 0), dim=0)
        del mag
    if not training:
        return rep

    p_ref.gstat.zero_()
    p_ref.flat.G.zero_()
    p_ref.dWx.zero_()
    p_ref.y_out.dxd.copy_(torch.randn(p_ref.y_out.dxd.shape, generator=g) / p_ref.y_out.dxd[0].numel() ** 0.5)
    for i, (br, bg, fam) in enumerate(zip(p_ref.bwd_ops, p_gpu.bwd_ops, _families(p_gpu.c_bwd))):
        push_state(p_ref, p_gpu)
        if br.kind == _lib.ATT_BWD_KV:      # reads the `delta` scratch its sibling kernel produces
            run_gpu_op(p_gpu, p_gpu.c_bwd, i - 1)
        where = f"bwd[{i}] {br.name}"
        f = br.fwd
        rep.op, rep.drop = ("bwd", i), (drop_label(br.kind, f) if f is not None else "")
        pt = fam.startswith("tcconv") and f.L_in % 128 != 0
        # deposits checked against a magnitude: (ref target, gpu target, elementwise magnitude or None = max-abs)
        deposits = []
        if br.kind in (_lib.CONV_BWD_DATA, _lib.RES_BWD, _lib.CONV_BWD_W):
            gmag = _grad_in_mag(it, f)
            fac, alpha = it._drop_factor(f)
        ties = {}
        if br.kind == _lib.CONV_BWD_DATA:
            mags = _data_grad_mags(it, br, gmag * alpha * fac)
            deposits = [(br.ins[j], bg.ins[j], mags[j]) for j in sorted(mags)]
            if f.pool > 1:
                ties = {id(br.ins[j]): _pool_ties(it, f, j) for j in mags}
        elif br.kind == _lib.RES_BWD:
            deposits = [(t, u, m) for t, u, m in ((br.res_a, bg.res_a, gmag * alpha), (br.res_b, bg.res_b, gmag))
                        if t is not None and t.buf is not None]
        elif br.kind in (_lib.ATT_BWD_Q, _lib.ATT_BWD_KV, _lib.HEADVEC_BWD):
            ts = [(t, u, None) for t, u in zip(br.ins, bg.ins) if t is not None and t.buf is not None]
            deposits = ts[:1] if br.kind == _lib.ATT_BWD_Q else (ts[1:] if br.kind == _lib.ATT_BWD_KV else ts)
        before = [_grad_buf(t).abs().clone() if t.accum else None for t, _, _ in deposits]
        gstat0, G0, dWx0 = p_ref.gstat.clone(), p_ref.flat.G.clone(), p_ref.dWx.clone()
        dwmag = _dw_mag(it, f, gmag * alpha * fac) if br.kind == _lib.CONV_BWD_W else None

        it.run_bwd_op(br)
        run_gpu_op(p_gpu, p_gpu.c_bwd, i)

        if br.kind in (_lib.CONV_BWD_DATA, _lib.RES_BWD, _lib.ATT_BWD_Q, _lib.ATT_BWD_KV, _lib.HEADVEC_BWD):
            gscale = gstat0.abs()
            touched = torch.zeros_like(gscale, dtype=torch.bool)
            for (tr, tg, m), b0 in zip(deposits, before):
                got, ref = _grad_buf(tg), _grad_buf(tr)
                if id(tr) in ties:
                    got = torch.where(ties[id(tr)], ref, got)
                    rep.pool_ties += int(ties[id(tr)].sum()) // f.pool
                what = f"grad({tr.buf.name})"
                rep.whole(where, what, got, ref)
                scale = chan_max(m if m is not None else ref.to(D).abs())
                if b0 is not None:
                    scale = scale + chan_max(b0)
                rep.chan(fam, where, "grad", got, ref, scale, partial_tile=pt)
                if tr.bn >= 0 and m is not None:
                    mu, istd = it.bn_khat(tr.bn, tr.bn_c0, tr.C)
                    kh = ((tr.buf.x[:, tr.c0:tr.c0 + tr.C].to(D) - mu[None, :, None]) * istd[None, :, None]).abs()
                    a, a2 = _stat_slices(p_ref, tr)
                    gscale[a:a + tr.C] += m.sum((0, 2))
                    gscale[a2:a2 + tr.C] += (m * kh).sum((0, 2))
                    touched[a:a + tr.C] = touched[a2:a2 + tr.C] = True
            rep.whole(where, "gstat", p_gpu.gstat, p_ref.gstat)
            if touched.any():
                rep.chan(fam, where, "gstat", p_gpu.gstat, p_ref.gstat, gscale, mask=touched, partial_tile=pt)
        if br.kind in (_lib.CONV_BWD_W, _lib.HEADVEC_BWD, _lib.BN_FINALIZE_BWD, _lib.STEM_COMPOSE_BWD):
            rep.whole(where, "G", p_gpu.flat.G, p_ref.flat.G)
            rep.whole(where, "dWx", p_gpu.dWx, p_ref.dWx)
        if br.kind in (_lib.CONV_BWD_W, _lib.HEADVEC_BWD):
            wr = f.Wx if f.Wx is not None else f.W
            gbuf_g, gbuf_r, gbuf_0 = (p_gpu.dWx, p_ref.dWx, dWx0) if f.Wx is not None else (p_gpu.flat.G, p_ref.flat.G, G0)
            sl = slice(wr.off, wr.off + wr.numel)
            got, ref = gbuf_g[sl].view(f.Cout, -1), gbuf_r[sl].view(f.Cout, -1)
            m = dwmag.reshape(f.Cout, -1) if dwmag is not None else ref.to(D).abs()
            rep.chan(fam, where, "dW", got, ref, chan_max(m, 0) + chan_max(gbuf_0[sl].view(f.Cout, -1).abs(), 0), dim=0)
            if f.bias is not None:
                sl = slice(f.bias.off, f.bias.off + f.bias.numel)
                m = (gmag * alpha * fac).sum((0, 2)) if dwmag is not None else p_ref.flat.G[sl].to(D).abs()
                rep.chan(fam, where, "dbias", p_gpu.flat.G[sl], p_ref.flat.G[sl], m + G0[sl].abs(), dim=0)
        deposits = before = dwmag = gmag = ties = None
    assert _lib.lib().seist_tc_error_flag() == 0, "a tensor-core kernel timed out on an mbarrier"
    return rep


def _release():
    gc.collect()
    torch.cuda.empty_cache()


def check_at_scale(name, n, length, training, drops=None, step_seed=12345):
    """run_at_scale on one configuration; prints the worst per-channel ratio of every (family, quantity) it reached and
    fails on any whole-tensor or per-channel failure, or on a dropout site that was not held to the per-channel
    criterion."""
    t0 = time.time()
    try:
        rep = run_at_scale(name, n, length, training, drops, step_seed)
    finally:
        _release()
    print(f"\n{name} N={n} L={length} training={training} SEIST_TCC={os.environ.get('SEIST_TCC', '')}"
          + (f" drops={drops} step_seed={step_seed}" if drops is not None else "") +
          f": {time.time() - t0:.0f} s; {rep.pool_ties} max-pool near ties left out; "
          + (f"{len(rep.sites)} dropout sites; " if rep.sites else "") + "worst per-channel error / magnitude by family:")
    for (fam, what), (r, where) in sorted(rep.worst.items()):
        print(f"  {fam:40s} {what:6s} {r:.3e}  ({where})")
    unchecked = [f"{ph}[{i}]: dropout site not checked" for ph, i in sorted(rep.sites - rep.checked)]
    failures = rep.failures[:20] + rep.chan_failures[:20] + unchecked[:20]
    assert not failures, f"{len(rep.failures)} + {len(rep.chan_failures)} + {len(unchecked)} failures:\n" + \
        "\n".join(failures)
    return rep


def check_on_tensor_cores(name, n, length, families=("tcconv_bwd",), drops=None, step_seed=12345):
    """check_at_scale in a child process with SEIST_TCC=1 (read once per process): every eligible forward /
    data-gradient conv runs on the persistent wgmma engine.  Each of `families` must prefix a family that ran."""
    _release()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path.insert(0, 'tests'); import test_gpu_ops_at_scale as T;"
            f"rep = T.check_at_scale({name!r}, {n}, {length}, True, {drops!r}, {step_seed});"
            f"missing = [p for p in {tuple(families)!r} if not any(f.startswith(p) for f, _ in rep.worst)];"
            "assert not missing, ('no op of these families ran', missing);"
            "print('TC-OK')")
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=dict(os.environ, SEIST_TCC="1"),
                       capture_output=True, text=True, timeout=1800)
    print(r.stdout[-6000:])
    assert r.returncode == 0 and "TC-OK" in r.stdout, (r.stdout[-4000:], r.stderr[-4000:])


@pytest.mark.gpu
def test_training_ops_at_bench_shape():
    check_at_scale(NAME, N, L, True)


@pytest.mark.gpu
def test_eval_forward_at_bench_shape():
    """Eval-mode template variants (no statistic epilogues, BN from the running buffers)."""
    check_at_scale(NAME, N, L, False)


@pytest.mark.gpu
def test_training_ops_at_bench_shape_on_tensor_cores():
    """SEIST_TCC=1: every eligible forward / data-gradient conv runs on the persistent wgmma engine, many tiles per
    CTA."""
    check_on_tensor_cores(NAME, N, L)
