"""Plan compiler: turns a `SeismogramTransformer` parameter tree + (N, L, mode) into the flat list
of fused-kernel descriptors (`SeistOp`, include/seist_b200.h) that the C runtime executes.

Design (DESIGN.md §3): the only tensors that ever reach HBM are the inputs of BatchNorm layers
(unavoidable in training: batch statistics need the whole tensor) and a handful of plain tensors
(q/k/v, MLP hidden, stage outputs).  Everything else — padding, BN-apply, GELU, residual adds,
channel concat, pooling, linear up-sampling, dropout/droppath — is expressed as a *view* that the
consuming kernel evaluates while loading, or as an epilogue of the producing kernel.  The backward
plan is derived here from the forward tape: each forward op emits up to three backward ops, and the
compiler tracks which gradient buffers have been written to choose overwrite vs accumulate.

Reference semantics cited per emitter (paths relative to the reference's models/seist.py).
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .models.seist import (HParams, dpk_head_layers, dpk_up_sizes, same_pad, split_mptl, split_msmc)

ACT_NONE, ACT_GELU = 0, 1
OUT_NONE, OUT_SIGMOID, OUT_SOFTMAX = 0, 1, 2


@dataclass(eq=False)
class Buf:
    """A materialised (N, C, L) fp32 tensor of the plan."""
    name: str
    C: int
    L: int
    x: Optional[torch.Tensor] = None
    du: Optional[torch.Tensor] = None    # gradient w.r.t. BN(x)
    dxd: Optional[torch.Tensor] = None   # gradient w.r.t. x directly
    need_du: bool = False
    need_dxd: bool = False
    no_grad: bool = False                # network input


@dataclass(eq=False)
class View:
    buf: Optional[Buf]
    c0: int = 0
    C: int = 0
    bn: int = -1
    bn_c0: int = 0
    act: int = ACT_NONE
    accum: int = 0          # backward only

    @property
    def L(self):
        return self.buf.L


@dataclass(eq=False)
class PRef:
    """Slice of the flat parameter / gradient buffers."""
    off: int
    numel: int
    shape: Tuple[int, ...]


@dataclass(eq=False)
class BNEntry:
    idx: int
    path: str
    C: int
    gamma: PRef
    beta: PRef
    rb_off: int                 # offset of running_mean in the flat running-stat buffer (var follows at +C)
    st_off: int                 # offset (in doubles) into the flat stat / gstat buffers
    count: float = 0.0
    chain: int = -1
    is_chained: bool = False
    sync: bool = False          # module is a SyncBatchNorm


@dataclass(eq=False)
class Op:
    kind: int
    N: int
    ins: List[View] = field(default_factory=list)
    res_a: Optional[View] = None
    res_b: Optional[View] = None
    out: Optional[View] = None
    W: Optional[PRef] = None
    bias: Optional[PRef] = None
    Wx: Optional[PRef] = None             # weights in the plan's scratch buffer (composed stem weights)
    wparts: Optional[List[PRef]] = None   # STEM_COMPOSE: in_proj, dconv, pconv
    Cin: int = 0
    Cout: int = 0
    k: int = 1
    stride: int = 1
    pad_left: int = 0
    groups: int = 1
    pool: int = 1
    up_src_L: int = 0
    L_in: int = 0
    L_out: int = 0
    out_act: int = OUT_NONE
    out_scale: float = 1.0
    p_elem: float = 0.0
    p_path: float = 0.0
    p_alpha: float = 0.0
    seed_elem: int = 0
    seed_path: int = 0
    seed_alpha: int = 0
    heads: int = 0
    p_attn: float = 0.0
    seed_attn: int = 0
    lse: Optional[torch.Tensor] = None
    delta: Optional[torch.Tensor] = None
    zero: Optional[torch.Tensor] = None   # ZERO target
    bn_lo: int = 0                        # BN_PREPARE: first entry / count
    n_bn: int = 0
    name: str = ""
    fwd: Optional["Op"] = None            # backward ops point at their forward op
    sync_bn: List[int] = field(default_factory=list)  # BN indices whose (g)stat must be all-reduced BEFORE this op


class Plan:
    """Compiled forward (+ backward) program for one (N, L, training) configuration."""

    def __init__(self):
        self.N = 0
        self.L = 0
        self.training = False
        self.world = 1
        self.device = None
        self.bufs: List[Buf] = []
        self.bns: List[BNEntry] = []
        self.fwd_ops: List[Op] = []
        self.bwd_ops: List[Op] = []
        self.x_in: Optional[Buf] = None
        self.y_out: Optional[Buf] = None
        self.flat = None                 # FlatState
        self.stat = None                 # double [2*sumC]
        self.gstat = None
        self.bn_table_dev = None
        self.step_seed = None
        self.arena_bytes = 0
        self.c_fwd = None
        self.c_bwd = None
        self.fwd_segments: List[Tuple[int, int, List[int]]] = []
        self.bwd_segments: List[Tuple[int, int, List[int]]] = []

    @property
    def n_main(self) -> int:
        """Main lanes of the lane schedule (schedule.py), besides the weight-gradient lane.  Data-parallel plans use
        one: their BN_PREPARE kernels pair up across ranks by an epoch counter, so every rank must issue them in the
        same order, which one stream guarantees."""
        return 2 if self.world == 1 else 1


class FlatState:
    """One contiguous fp32 buffer for all parameters (+ one for grads, one for BN running stats,
    one int64 for num_batches_tracked).  Module parameters are re-pointed to views of it, so
    optimizer / state_dict / DDP keep working while kernels and the fused Adam see a single array."""

    def __init__(self, model: nn.Module, device):
        self.device = device
        self.params: List[nn.Parameter] = []
        self.pref: Dict[str, PRef] = {}
        off = 0
        named = list(model.named_parameters())
        for name, p in named:
            n = p.numel()
            self.pref[name] = PRef(off, n, tuple(p.shape))
            off += (n + 3) // 4 * 4       # keep every tensor 16-byte aligned
        self.numel = off
        self.P = torch.zeros(off, dtype=torch.float32, device=device)
        self.G = torch.zeros(off, dtype=torch.float32, device=device)
        with torch.no_grad():
            for name, p in named:
                r = self.pref[name]
                v = self.P[r.off:r.off + r.numel].view(r.shape)
                v.copy_(p.detach().to(device=device, dtype=torch.float32))
                p.data = v
                self.params.append(p)
        # BN running statistics
        self.rb_off: Dict[str, int] = {}
        bns = [(n, m) for n, m in model.named_modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]
        tot = sum(2 * m.num_features for _, m in bns)
        self.RB = torch.zeros(max(tot, 1), dtype=torch.float32, device=device)
        self.NBT = torch.zeros(max(len(bns), 1), dtype=torch.int64, device=device)
        off = 0
        with torch.no_grad():
            for i, (n, m) in enumerate(bns):
                c = m.num_features
                rm = self.RB[off:off + c]
                rv = self.RB[off + c:off + 2 * c]
                rm.copy_(m.running_mean.to(device))
                rv.copy_(m.running_var.to(device))
                m.running_mean = rm
                m.running_var = rv
                nb = self.NBT[i:i + 1].view(())
                nb.copy_(m.num_batches_tracked.to(device))
                m.num_batches_tracked = nb
                self.rb_off[n] = off
                off += 2 * c
        self.param_ptrs = [p.data_ptr() for p in self.params]

    def valid(self) -> bool:
        return all(p.data_ptr() == q for p, q in zip(self.params, self.param_ptrs))

    def grad_view(self, name: str) -> torch.Tensor:
        r = self.pref[name]
        return self.G[r.off:r.off + r.numel].view(r.shape)


# =================================================================================================
class PlanBuilder:
    def __init__(self, model, flat: FlatState, N: int, L: int, training: bool, world: int = 1,
                 device=None, need_backward: Optional[bool] = None):
        self.m = model
        self.hp: HParams = model.hp
        self.flat = flat
        self.N, self.Lx = N, L
        self.training = training
        self.world = world
        self.device = device if device is not None else flat.device
        self.need_backward = training if need_backward is None else need_backward
        self.plan = Plan()
        self.mods = dict(model.named_modules())
        self.seed_ctr = 1
        self._bn_idx: Dict[str, int] = {}
        self._st_off = 0
        self._wx_off = 0

    # ---- small helpers --------------------------------------------------------------------------
    def buf(self, name, C, L, no_grad=False) -> Buf:
        b = Buf(name, C, L, no_grad=no_grad)
        self.plan.bufs.append(b)
        return b

    def seed(self) -> int:
        self.seed_ctr += 1
        return self.seed_ctr

    def pref(self, path: str) -> Optional[PRef]:
        return self.flat.pref.get(path)

    def bn(self, path: str, L: int, chain_path: Optional[str] = None) -> int:
        """Register the BN at `path` (and optionally the BN chained on top of it)."""
        if path in self._bn_idx:
            return self._bn_idx[path]
        mod = self.mods[path]
        C = mod.num_features
        e = BNEntry(len(self.plan.bns), path, C, self.pref(path + ".weight"), self.pref(path + ".bias"),
                    self.flat.rb_off[path], self._st_off, count=float(self.N * self.world * L),
                    sync=isinstance(mod, nn.SyncBatchNorm))
        self._st_off += 2 * C
        self.plan.bns.append(e)
        self._bn_idx[path] = e.idx
        if chain_path is not None:
            e.chain = self.bn(chain_path, L)
            self.plan.bns[e.chain].is_chained = True
        return e.idx

    def drop(self, p: float) -> float:
        return float(p) if self.training else 0.0

    def conv(self, name, ins: List[View], wpath: str, out: View, *, k=1, stride=1, groups=1, pool=1,
             up_to: int = 0, pad: Optional[Tuple[int, int]] = None, res_a=None, res_b=None,
             p_elem=0.0, p_path=0.0, p_alpha=0.0, out_act=OUT_NONE, wx: Optional[PRef] = None) -> Op:
        src_L = ins[0].L
        for v in ins:
            assert v.L == src_L
        if pool > 1:
            L_in = -(-src_L // pool)
        elif up_to > 0:
            L_in = up_to
        else:
            L_in = src_L
        if pad is None:
            pad = same_pad(L_in, k, stride) if k > 1 else (0, 0)
        L_out = (L_in + pad[0] + pad[1] - k) // stride + 1
        assert L_out == out.L, (name, L_out, out.L)
        Cin = sum(v.C for v in ins)
        W = self.pref(wpath + ".weight") if wx is None else None
        assert (wx or W).shape == (out.C, Cin // groups, k), (name, (wx or W).shape, out.C, Cin, groups, k)
        op = Op(_lib.CONV_FWD, self.N, ins=ins, res_a=res_a, res_b=res_b, out=out, W=W, Wx=wx,
                bias=self.pref(wpath + ".bias") if wx is None else None, Cin=Cin, Cout=out.C, k=k, stride=stride, pad_left=pad[0],
                groups=groups, pool=pool, up_src_L=(src_L if up_to > 0 else 0), L_in=L_in, L_out=L_out,
                out_act=out_act, p_elem=self.drop(p_elem), p_path=self.drop(p_path),
                p_alpha=self.drop(p_alpha), name=name)
        if op.p_elem > 0:
            op.seed_elem = self.seed()
        if op.p_path > 0:
            op.seed_path = self.seed()
        if op.p_alpha > 0:
            op.seed_alpha = self.seed()
        for v in ins + [r for r in (res_a, res_b) if r is not None]:
            if v.buf.no_grad:
                continue
            if v.bn >= 0:
                v.buf.need_du = True
            else:
                v.buf.need_dxd = True
        for r in (res_a, res_b):
            if r is not None:
                assert r.C == out.C and r.L == out.L and r.act == ACT_NONE
        self.plan.fwd_ops.append(op)
        return op

    # ---- network emitters -----------------------------------------------------------------------
    def stem_block(self, i: int, vin: View) -> View:
        """StemBlock (:158-195) = 3 x DSConvNormAct (:124-155) + concat + 1x1 + BN."""
        hp = self.hp
        p = f"stem.{i}"
        cin, cout, k0, s = vin.C, hp.stem_channels[i], hp.stem_kernel_sizes[i], hp.stem_strides[i]
        L_in = vin.L
        L_out = -(-L_in // s)
        cat = self.buf(f"{p}.cat", 3 * cout, L_out)
        views = []
        for j in range(3):
            k = k0 + 4 * j
            pj = f"{p}.convs.{j}"
            # in_proj -> pad -> depthwise -> pconv is linear: run it as ONE dense k-tap conv whose weights
            # are composed on the device each step (SEIST_OP_STEM_COMPOSE_*); no intermediate tensors.
            parts = [self.pref(f"{pj}.in_proj.weight"), self.pref(f"{pj}.dconv.weight"), self.pref(f"{pj}.pconv.weight")]
            wx = PRef(self._wx_off, cout * cin * k, (cout, cin, k))
            self._wx_off += (wx.numel + 3) // 4 * 4
            self.plan.fwd_ops.append(Op(_lib.STEM_COMPOSE_FWD, self.N, Wx=wx, wparts=parts, Cin=cin, Cout=cout, k=k,
                                        name=f"{pj}.compose"))
            b = self.bn(f"{pj}.norm", L_out)
            self.conv(f"{pj}.conv", [View(vin.buf, vin.c0, vin.C, vin.bn, vin.bn_c0, vin.act)], pj, View(cat, j * cout, cout, bn=b),
                      k=k, stride=s, wx=wx)
            views.append(View(cat, j * cout, cout, bn=b, act=ACT_GELU))
        w = self.buf(f"{p}.out", cout, L_out)
        b = self.bn(f"{p}.norm", L_out)
        self.conv(f"{p}.out_proj", views, f"{p}.out_proj", View(w, 0, cout, bn=b))
        return View(w, 0, cout, bn=b)

    def mlp(self, p: str, vin: View, out: View, *, res_a=None, res_b=None, p_path=0.0, p_alpha=0.0):
        """MLP (:99-121): lin0 -> GELU -> lin1 -> Dropout; residual/droppath folded in the epilogue."""
        hid = self.mods[p + ".lin0"].out_channels
        h = self.buf(f"{p}.hidden", hid, vin.L)
        self.conv(f"{p}.lin0", [vin], f"{p}.lin0", View(h, 0, hid))
        self.conv(f"{p}.lin1", [View(h, 0, hid, act=ACT_GELU)], f"{p}.lin1", out, res_a=res_a, res_b=res_b,
                  p_elem=self.hp.mlp_drop_rate, p_path=p_path, p_alpha=p_alpha)

    def gconv_block(self, p: str, xin: View, k: int, groups: int, pdpr: float, out: View, *,
                    outer_res: View, p_alpha=0.0):
        """GroupConvBlock (:198-256) followed by the caller's residual:
             r1  = xin + dp0(proj(GELU(BN0(gconv_k(xin)))))
             out = alpha * [ r1 + dp1(mlp(BN1(r1))) ] + outer_res"""
        C, L = xin.C, xin.L
        c = self.buf(f"{p}.c", C, L)
        b0 = self.bn(f"{p}.norm0", L)
        self.conv(f"{p}.conv", [xin], f"{p}.conv", View(c, 0, C, bn=b0), k=k, groups=groups)
        r1 = self.buf(f"{p}.r1", C, L)
        b1 = self.bn(f"{p}.norm1", L)
        self.conv(f"{p}.proj", [View(c, 0, C, bn=b0, act=ACT_GELU)], f"{p}.proj", View(r1, 0, C, bn=b1),
                  res_b=xin, p_path=pdpr)
        self.mlp(f"{p}.mlp", View(r1, 0, C, bn=b1), out, res_a=View(r1, 0, C), res_b=outer_res,
                 p_path=pdpr, p_alpha=p_alpha)

    def msmc(self, p: str, cur: View, head_dim: int, pdpr: float) -> View:
        """MultiScaleMixedConv (:259-318)."""
        C, L = cur.C, cur.L
        ks = self.hp.msmc_kernel_sizes
        dims = split_msmc(C, C // head_dim, len(ks))
        a = self.buf(f"{p}.a", C, L)
        o = self.buf(f"{p}.out", C, L)
        bo = self.bn(f"{p}.out_norm", L)
        off = 0
        for j, (d, k) in enumerate(zip(dims, ks)):
            bj = self.bn(f"{p}.norms.{j}", L)
            self.conv(f"{p}.projs.{j}", [cur], f"{p}.projs.{j}", View(a, off, d, bn=bj))
            xi = View(a, off, d, bn=bj)
            self.gconv_block(f"{p}.convs.{j}", xi, k, d // head_dim, pdpr,
                             View(o, off, d, bn=bo, bn_c0=off), outer_res=View(a, off, d, bn=bj))
            off += d
        return View(o, 0, C, bn=bo)

    def attention(self, p: str, x1: View, head_dim: int, r: int, out: View, p_path: float):
        """AttentionBlock (:321-393) + the caller's `x1 + droppath(...)` (:492)."""
        hp = self.hp
        C, L = x1.C, x1.L
        q = self.buf(f"{p}.q", C, L)
        self.conv(f"{p}.q_proj", [x1], f"{p}.q_proj", View(q, 0, C))
        if r > 1:
            Lk = -(-L // r)
            kv = self.buf(f"{p}.kv", C, Lk)
            b = self.bn(f"{p}.aggr.norm", Lk, chain_path=f"{p}.norm")
            self.conv(f"{p}.aggr.proj", [x1], f"{p}.aggr.proj", View(kv, 0, C, bn=b), pool=r)
            kvv = View(kv, 0, C, bn=b)
        else:
            Lk = L
            kvv = View(x1.buf, x1.c0, C, bn=x1.bn, bn_c0=x1.bn_c0)
        kb = self.buf(f"{p}.k", C, Lk)
        vb = self.buf(f"{p}.v", C, Lk)
        self.conv(f"{p}.k_proj", [kvv], f"{p}.k_proj", View(kb, 0, C), p_elem=hp.key_drop_rate)
        self.conv(f"{p}.v_proj", [View(kvv.buf, kvv.c0, C, bn=kvv.bn, bn_c0=kvv.bn_c0)], f"{p}.v_proj",
                  View(vb, 0, C))
        o = self.buf(f"{p}.o", C, L)
        heads = C // head_dim
        op = Op(_lib.ATT_FWD, self.N, ins=[View(q, 0, C), View(kb, 0, C), View(vb, 0, C)], out=View(o, 0, C),
                Cin=C, Cout=C, L_in=Lk, L_out=L, heads=heads, p_attn=self.drop(hp.attn_drop_rate),
                name=f"{p}.core")
        if op.p_attn > 0:
            op.seed_attn = self.seed()
        for b_ in (q, kb, vb):
            b_.need_dxd = True
        self.plan.fwd_ops.append(op)
        self.conv(f"{p}.out_proj", [View(o, 0, C)], f"{p}.out_proj", out,
                  res_b=View(x1.buf, x1.c0, C, bn=x1.bn, bn_c0=x1.bn_c0),
                  p_elem=hp.other_drop_rate, p_path=p_path)

    def mptl(self, p: str, cur: View, head_dim: int, r: int, pdpr: float) -> View:
        """MultiPathTransformerLayer (:396-504)."""
        hp = self.hp
        C, L = cur.C, cur.L
        a_dim, c_dim = split_mptl(C, hp.attn_ratio, head_dim)
        pr = self.buf(f"{p}.proj", C, L)
        cat = self.buf(f"{p}.cat", C, L)
        b2 = self.bn(f"{p}.norm2", L)
        if a_dim > 0:
            b0 = self.bn(f"{p}.norm0", L)
            self.conv(f"{p}.attn_proj", [cur], f"{p}.attn_proj", View(pr, 0, a_dim, bn=b0))
            self.attention(f"{p}.attention", View(pr, 0, a_dim, bn=b0), head_dim, r,
                           View(cat, 0, a_dim, bn=b2, bn_c0=0), p_path=pdpr * hp.attn_ratio)
        if c_dim > 0:
            b1 = self.bn(f"{p}.norm1", L)
            self.conv(f"{p}.conv_proj", [View(cur.buf, cur.c0, C, bn=cur.bn, bn_c0=cur.bn_c0, act=cur.act)],
                      f"{p}.conv_proj", View(pr, a_dim, c_dim, bn=b1))
            x2 = View(pr, a_dim, c_dim, bn=b1)
            self.gconv_block(f"{p}.gconv", x2, 3, c_dim // head_dim, pdpr,
                             View(cat, a_dim, c_dim, bn=b2, bn_c0=a_dim),
                             outer_res=View(pr, a_dim, c_dim, bn=b1), p_alpha=pdpr * (1 - hp.attn_ratio))
        y = self.buf(f"{p}.y", C, L)
        x = View(cat, 0, C, bn=b2)
        self.mlp(f"{p}.mlp", x, View(y, 0, C), res_b=View(cat, 0, C, bn=b2), p_path=pdpr)
        return View(y, 0, C)

    def head_dpk(self, vin: View, L_full: int) -> Buf:
        """HeadDetectionPicking (:507-572)."""
        hp = self.hp
        layers = dpk_head_layers(hp)
        sizes = dpk_up_sizes(vin.L, L_full, len(layers))
        for i, (cin, cout, k) in enumerate(layers):
            p = f"out_head.up_layers.{i}"
            u = self.buf(f"{p}.u", cout, sizes[i])
            b = self.bn(f"{p}.norm", sizes[i])
            self.conv(f"{p}.conv", [vin], f"{p}.conv", View(u, 0, cout, bn=b), k=k, up_to=sizes[i])
            vin = View(u, 0, cout, bn=b, act=ACT_GELU)
        y = self.buf("out_head.y", hp.head_out_channels, L_full)
        self.conv("out_head.out_conv", [vin], "out_head.out_conv", View(y, 0, hp.head_out_channels), k=7,
                  pad=(3, 3), out_act=OUT_SIGMOID if hp.head_sigmoid else OUT_NONE)
        return y

    def head_vec(self, vin: View) -> Buf:
        """HeadRegression / HeadClassification (:575-610)."""
        hp = self.hp
        nout = self.mods["out_head.lin"].out_features
        y = self.buf("out_head.y", nout, 1)
        op = Op(_lib.HEADVEC_FWD, self.N, ins=[vin], out=View(y, 0, nout), W=self.pref("out_head.lin.weight"),
                bias=self.pref("out_head.lin.bias"), Cin=vin.C, Cout=nout, L_in=vin.L, L_out=1,
                out_act=OUT_SIGMOID if hp.head == "reg" else OUT_SOFTMAX,
                out_scale=hp.head_scale if hp.head == "reg" else 1.0, name="out_head.lin")
        vin.buf.need_dxd = True
        self.plan.fwd_ops.append(op)
        return y

    # ---- whole network ---------------------------------------------------------------------------
    def build(self) -> Plan:
        hp, pl = self.hp, self.plan
        pl.N, pl.L, pl.training, pl.world, pl.device, pl.flat = self.N, self.Lx, self.training, self.world, self.device, self.flat
        xin = self.buf("x", hp.in_channels, self.Lx, no_grad=True)
        pl.x_in = xin
        cur = View(xin, 0, hp.in_channels)
        for i in range(len(hp.stem_channels)):
            cur = self.stem_block(i, cur)
        pdprs = self.m.block_drop_path_rates()
        blk = 0
        for i, lc in enumerate(hp.layer_channels):
            p = f"encoder_layers.{i}"
            r = hp.stage_aggr_ratios[i]
            L = -(-cur.L // r) if r > 1 else cur.L
            a = self.buf(f"{p}.0.a", lc, L)
            b = self.bn(f"{p}.0.norm", L)
            self.conv(f"{p}.0.proj", [cur], f"{p}.0.proj", View(a, 0, lc, bn=b), pool=r)   # LAAB :73-96
            cur = View(a, 0, lc, bn=b)
            n_conv = hp.layer_blocks[i] - hp.attn_blocks[i]
            for j in range(hp.layer_blocks[i]):
                if j >= n_conv:
                    cur = self.mptl(f"{p}.{j + 1}", cur, hp.head_dims[i], hp.attn_aggr_ratios[i], pdprs[blk])
                else:
                    cur = self.msmc(f"{p}.{j + 1}", cur, hp.head_dims[i], pdprs[blk])
                blk += 1
        pl.y_out = self.head_dpk(cur, self.Lx) if hp.head == "dpk" else self.head_vec(cur)
        pl.y_out.need_dxd = True
        pl.wx_numel = self._wx_off
        if self.training:
            pl.fwd_ops.append(Op(_lib.BN_FINALIZE_FWD, self.N, name="bn_finalize_fwd"))
        pl.fwd_ops = self._insert_prepares(pl.fwd_ops, forward=True)
        if self.need_backward:
            self._emit_backward()
            pl.bwd_ops = self._insert_prepares(pl.bwd_ops, forward=False)
        return pl

    # ---- backward --------------------------------------------------------------------------------
    def _emit_backward(self):
        pl = self.plan
        written: Dict[Tuple[int, str, int], int] = {}

        def grad_target(v: View) -> Optional[View]:
            if v is None or v.buf.no_grad:
                return None
            kind = "du" if v.bn >= 0 else "dxd"
            key = (id(v.buf), kind, v.c0)
            for (bid, kd, c0), C in written.items():     # slices of one buffer are identical or disjoint
                if bid == id(v.buf) and kd == kind and c0 != v.c0:
                    assert v.c0 + v.C <= c0 or c0 + C <= v.c0, f"overlapping gradient slices on {v.buf.name}"
            acc = 1 if key in written else 0
            written[key] = v.C
            return View(v.buf, v.c0, v.C, v.bn, v.bn_c0, v.act, accum=acc)

        ops = pl.bwd_ops
        for f in reversed(pl.fwd_ops):
            if f.kind == _lib.CONV_FWD:
                up_atomic = f.up_src_L > 0
                if f.res_a is not None or f.res_b is not None:
                    ra, rb = grad_target(f.res_a), grad_target(f.res_b)
                    if ra is not None or rb is not None:
                        ops.append(Op(_lib.RES_BWD, f.N, res_a=ra, res_b=rb, out=f.out, fwd=f, name=f.name + ":res_bwd"))
                ops.append(Op(_lib.CONV_BWD_W, f.N, ins=f.ins, out=f.out, fwd=f, name=f.name + ":bwd_w"))
                tg = [grad_target(v) for v in f.ins]
                if any(t is not None for t in tg):
                    if up_atomic:
                        # the up-sampling transpose scatters with atomics: target must start from zero
                        for t in tg:
                            if t is not None and t.accum == 0:
                                ops.append(Op(_lib.ZERO, f.N, out=t, name=f.name + ":zero_g"))
                                t.accum = 1
                    ops.append(Op(_lib.CONV_BWD_DATA, f.N, ins=[t if t is not None else View(None) for t in tg],
                                  out=f.out, fwd=f, name=f.name + ":bwd_data"))
            elif f.kind == _lib.ATT_FWD:
                tq, tk, tv = (grad_target(v) for v in f.ins)
                ops.append(Op(_lib.ATT_BWD_Q, f.N, ins=[tq, tk, tv], out=f.out, fwd=f, name=f.name + ":bwd_q"))
                ops.append(Op(_lib.ATT_BWD_KV, f.N, ins=[tq, tk, tv], out=f.out, fwd=f, name=f.name + ":bwd_kv"))
            elif f.kind == _lib.HEADVEC_FWD:
                t = grad_target(f.ins[0])
                ops.append(Op(_lib.HEADVEC_BWD, f.N, ins=[t], out=f.out, fwd=f, name=f.name + ":bwd"))
            elif f.kind == _lib.STEM_COMPOSE_FWD:
                ops.append(Op(_lib.STEM_COMPOSE_BWD, f.N, fwd=f, name=f.name + ":bwd"))
            elif f.kind == _lib.BN_FINALIZE_FWD:
                pass
        ops.append(Op(_lib.BN_FINALIZE_BWD, self.N, name="bn_finalize_bwd"))

    def _insert_prepares(self, ops: List[Op], forward: bool) -> List[Op]:
        """Insert the BN_PREPARE ops: the per-channel coefficient table of a BN is computed once, after its
        last producer and before its first consumer (forward: scale/shift/khat from the batch statistics;
        backward: A/Bx/Cc from gstat).  Under data parallelism that is also the point where the (g)stat
        slots are summed over ranks (reference training/train.py:374, SyncBatchNorm)."""
        kind = _lib.BN_PREPARE_FWD if forward else _lib.BN_PREPARE_BWD
        nb = len(self.plan.bns)
        if forward and not self.training:
            return [Op(kind, self.N, bn_lo=0, n_bn=nb, name="bn_prepare_all")] + ops
        out: List[Op] = []
        ready = set()
        for op in ops:
            needs = set()
            if forward:
                for v in list(op.ins) + [op.res_a, op.res_b]:
                    if v is not None and v.buf is not None and v.bn >= 0:
                        needs.add(v.bn)
            elif op.kind in (_lib.CONV_BWD_DATA, _lib.CONV_BWD_W, _lib.RES_BWD) and op.out.bn >= 0 \
                    and op.out.buf.need_du:
                needs.add(op.out.bn)
            todo = sorted(b for b in needs if b not in ready)
            run: List[int] = []
            for b in todo + [None]:
                if run and (b is None or b != run[-1] + 1):
                    out.append(Op(kind, self.N, bn_lo=run[0], n_bn=len(run), name=f"bn_prepare[{run[0]}:{run[-1] + 1}]",
                                  sync_bn=list(run) if self.world > 1 else []))
                    run = []
                if b is not None:
                    run.append(b)
            ready.update(todo)
            out.append(op)
        return out


# =================================================================================================
# materialisation: allocate buffers, build ctypes descriptors
# =================================================================================================
def allocate(plan: Plan, with_backward: bool, step_seed: Optional[torch.Tensor] = None, comm=None):
    dev = plan.device
    N = plan.N
    total = 0
    layout = []

    def take(n):
        nonlocal total
        off = total
        total += (n + 63) // 64 * 64
        return off

    for b in plan.bufs:
        n = N * b.C * b.L
        layout.append((b, "x", take(n), n))
        if with_backward and not b.no_grad:
            if b.need_du:
                layout.append((b, "du", take(n), n))
            if b.need_dxd:
                layout.append((b, "dxd", take(n), n))
    extra = []
    for op in plan.fwd_ops:
        if op.kind == _lib.ATT_FWD:
            n = N * op.heads * op.L_out
            extra.append((op, "lse", take(n), n))
            if with_backward:
                extra.append((op, "delta", take(n), n))
    arena = torch.empty(total, dtype=torch.float32, device=dev)
    plan.arena = arena
    plan.arena_bytes = total * 4
    for b, what, off, n in layout:
        setattr(b, what, arena[off:off + n].view(N, b.C, b.L))
    for op, what, off, n in extra:
        setattr(op, what, arena[off:off + n].view(N, op.heads, op.L_out))
    nst = max(sum(2 * e.C for e in plan.bns), 2)
    plan.stat = torch.zeros(nst, dtype=torch.float64, device=dev)
    plan.gstat = torch.zeros(nst, dtype=torch.float64, device=dev)
    # where the producers' epilogues accumulate: the same buffers on one GPU; with a peer-memory exchange (comm.py) this
    # rank's partial sums live in symmetric memory and the BN_PREPARE kernels sum all ranks' parts into stat / gstat
    plan.comm = comm
    if comm is not None:
        assert comm.n_stat >= nst, (comm.n_stat, nst)
        plan.stat_acc, plan.gstat_acc = comm.stat_acc[:nst], comm.gstat_acc[:nst]
    else:
        plan.stat_acc, plan.gstat_acc = plan.stat, plan.gstat
    plan.Wx = torch.zeros(max(getattr(plan, "wx_numel", 0), 4), dtype=torch.float32, device=dev)
    plan.dWx = torch.zeros_like(plan.Wx)
    plan.coef = torch.zeros(4 * nst, dtype=torch.float32, device=dev)   # [C][8] per BN entry
    # dropout step counter: the engine passes ONE device scalar shared by all its plans (a per-plan counter would
    # restart whenever the batch shape changes)
    plan.step_seed = step_seed if step_seed is not None else torch.zeros(1, dtype=torch.int64, device=dev)


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def bn_table_struct(plan: Plan):
    flat = plan.flat
    arr = (_lib.SeistBN * max(len(plan.bns), 1))()
    for e in plan.bns:
        s = arr[e.idx]
        s.gamma = flat.P.data_ptr() + 4 * e.gamma.off
        s.beta = flat.P.data_ptr() + 4 * e.beta.off
        s.running_mean = flat.RB.data_ptr() + 4 * e.rb_off
        s.running_var = flat.RB.data_ptr() + 4 * (e.rb_off + e.C)
        s.stat = plan.stat.data_ptr() + 8 * e.st_off
        s.gstat = plan.gstat.data_ptr() + 8 * e.st_off
        s.stat_acc = plan.stat_acc.data_ptr() + 8 * e.st_off
        s.gstat_acc = plan.gstat_acc.data_ptr() + 8 * e.st_off
        s.dgamma = flat.G.data_ptr() + 4 * e.gamma.off
        s.dbeta = flat.G.data_ptr() + 4 * e.beta.off
        s.coef = plan.coef.data_ptr() + 4 * (4 * e.st_off)
        s.count = e.count
        s.C = e.C
        s.chain = e.chain
        s.use_batch = 1 if plan.training else 0
        s.is_chained = 1 if e.is_chained else 0
        s.eps = 1e-5
        s.momentum = 0.1
        s.grad_scale = 1.0 / plan.world
    return arr


def _cview(v: Optional[View], use_grad: bool) -> _lib.SeistView:
    s = _lib.SeistView()
    if v is None or v.buf is None:
        return s
    s.x = _ptr(v.buf.x)
    if use_grad:
        s.g = _ptr(v.buf.du if v.bn >= 0 else v.buf.dxd)
    s.Ct, s.c0, s.C, s.L = v.buf.C, v.c0, v.C, v.buf.L
    s.bn, s.bn_c0, s.act, s.accum = v.bn, v.bn_c0, v.act, v.accum
    return s


def to_c(plan: Plan, ops: List[Op], segs: List[Tuple[int, int, List[int]]]):
    flat = plan.flat
    arr = (_lib.SeistOp * max(len(ops), 1))()
    for i, op in enumerate(ops):
        f = op.fwd if op.fwd is not None else op
        c = arr[i]
        c.kind, c.N = op.kind, op.N
        c.bn_table = plan.bn_table_dev.data_ptr()
        c.step_seed = plan.step_seed.data_ptr()
        bw = op.fwd is not None
        for j, v in enumerate(op.ins[:_lib.MAX_IN]):
            c.inp[j] = _cview(v, bw)
            if bw and (v is None or v.buf is None):      # no gradient wanted: keep geometry of the forward view
                c.inp[j] = _cview(f.ins[j], False)
        c.res_a = _cview(op.res_a if bw else f.res_a, bw)
        c.res_b = _cview(op.res_b if bw else f.res_b, bw)
        if bw and op.kind != _lib.RES_BWD:
            c.res_a = _cview(f.res_a, False)
            c.res_b = _cview(f.res_b, False)
        if bw and op.kind == _lib.RES_BWD:
            # absent targets keep C = 0 so the kernel skips them
            if op.res_a is None:
                c.res_a = _lib.SeistView()
            if op.res_b is None:
                c.res_b = _lib.SeistView()
        if op.out is not None:
            c.out = _cview(op.out, False)
            ob = op.out.buf
            if bw and ob is not None:
                c.out.g = _ptr(ob.du) if op.out.bn >= 0 else 0
                c.out_dxd = _ptr(ob.dxd)
        if op.kind == _lib.ZERO:
            t = op.out.buf.du if op.out.bn >= 0 else op.out.buf.dxd
            assert op.out.c0 == 0 and op.out.C == op.out.buf.C, "ZERO clears whole buffers only"
            c.out.x = t.data_ptr()
            c.zero_bytes = t.numel() * 4
        if f.W is not None:
            c.W = flat.P.data_ptr() + 4 * f.W.off
            c.dW = flat.G.data_ptr() + 4 * f.W.off
        if f.Wx is not None:
            c.W = plan.Wx.data_ptr() + 4 * f.Wx.off
            c.dW = plan.dWx.data_ptr() + 4 * f.Wx.off
        if f.kind == _lib.STEM_COMPOSE_FWD:
            for j, r in enumerate(f.wparts):
                c.inp[j].x = flat.P.data_ptr() + 4 * r.off
                c.inp[j].g = flat.G.data_ptr() + 4 * r.off
            c.out.x = plan.Wx.data_ptr() + 4 * f.Wx.off
            c.out.g = plan.dWx.data_ptr() + 4 * f.Wx.off
        if f.bias is not None:
            c.bias = flat.P.data_ptr() + 4 * f.bias.off
            c.dbias = flat.G.data_ptr() + 4 * f.bias.off
        c.n_in = len(f.ins)
        for name in ("Cin", "Cout", "k", "stride", "pad_left", "groups", "pool", "up_src_L", "L_in", "L_out",
                     "out_act", "out_scale", "p_elem", "p_path", "p_alpha", "seed_elem", "seed_path",
                     "seed_alpha", "heads", "p_attn", "seed_attn"):
            setattr(c, name, getattr(f, name))
        c.lse = _ptr(f.lse)
        c.delta = _ptr(f.delta)
        c.n_bn = len(plan.bns)
        if op.kind in (_lib.BN_PREPARE_FWD, _lib.BN_PREPARE_BWD):
            c.n_bn, c.bn_lo = op.n_bn, op.bn_lo
            if plan.comm is not None and op.sync_bn:
                c.comm = plan.comm.dev_ptr          # statistic sum over NVLink peer memory fused into this kernel
    # lane / event fields, one schedule per segment: seist_plan_run_lanes issues a segment per call and joins all lanes at
    # its end, so event ids are local to the segment
    from .schedule import schedule_lanes
    size = ctypes.sizeof(_lib.SeistOp)
    for start, end, _ in segs:
        view = (_lib.SeistOp * (end - start)).from_address(ctypes.addressof(arr) + start * size)
        schedule_lanes(plan, ops[start:end], view, plan.n_main)
    return arr


def segments(ops: List[Op], fused: bool = False) -> List[Tuple[int, int, List[int]]]:
    """[(start, end, bn indices to all-reduce before running ops[start:end])].  `fused`: the statistic exchange is
    inside the BN_PREPARE kernels (peer memory) - one segment, no host-issued collectives."""
    if fused:
        return [(0, len(ops), [])]
    segs, start, pend = [], 0, []
    for i, op in enumerate(ops):
        if op.sync_bn:
            if i > start:
                segs.append((start, i, pend))
            start, pend = i, list(op.sync_bn)
    segs.append((start, len(ops), pend))
    return segs


def finalize(plan: Plan, with_backward: bool, step_seed: Optional[torch.Tensor] = None, comm=None):
    """Allocate device memory and freeze the descriptors (device must be CUDA for execution)."""
    allocate(plan, with_backward, step_seed, comm)
    tab = bn_table_struct(plan)
    raw = np.frombuffer(bytes(tab), dtype=np.uint8).copy()
    plan.bn_table_host = tab
    plan.bn_table_dev = torch.from_numpy(raw).to(plan.device)
    plan.fwd_segments = segments(plan.fwd_ops, fused=comm is not None)
    plan.c_fwd = to_c(plan, plan.fwd_ops, plan.fwd_segments)
    if with_backward:
        plan.bwd_segments = segments(plan.bwd_ops, fused=comm is not None)
        plan.c_bwd = to_c(plan, plan.bwd_ops, plan.bwd_segments)
    return plan
