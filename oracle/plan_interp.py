"""Interpreter of seist_b200 plans.  TEST INFRASTRUCTURE ONLY (never imported by the product).

Executes the *semantics* of every SeistOp kind (include/seist_b200.h) with plain torch ops on the plan's own
buffers, on the plan's device (a CPU plan on the CPU, a CUDA plan on the GPU) in the arithmetic `dtype` names,
so that
  (1) the plan compiler (seist_b200/plan.py: forward tape, derived backward, accumulate flags,
      BatchNorm-backward coefficient algebra, chained-BN folding) is checked end-to-end against the
      pinned oracle (oracle/seist_ref.py) without a GPU, and
  (2) each CUDA kernel is checked op-by-op on the GPU box against exactly the contract the compiler
      assumes.
Local gradients are obtained with torch.autograd on the forward expression of the op; BatchNorm is
deliberately NOT differentiated by autograd here — its backward goes through the same closed-form
coefficients (A, Bx, Cc) the kernels use, which is what makes the end-to-end comparison meaningful.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from seist_b200 import _lib
from seist_b200.plan import ACT_GELU, OUT_SIGMOID, OUT_SOFTMAX, Op, Plan, View

M64 = (1 << 64) - 1


def rng_u64(step_seed: int, stream: int, qidx: np.ndarray) -> np.ndarray:
    """Counter-based generator shared with csrc/common.cuh::rng_u64 (splitmix64 finaliser of the QUAD index)."""
    with np.errstate(over="ignore"):
        z = np.uint64((step_seed * 0xD1342543DE82EF95 + ((stream << 32) | 0x9E3779B9)) & M64)
        z = z + qidx.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z


def rng_u16(step_seed: int, stream: int, idx: np.ndarray) -> np.ndarray:
    """16-bit lane (idx & 3) of the hash of quad (idx >> 2) - csrc/common.cuh::keep_scale."""
    idx = idx.astype(np.uint64)
    h = rng_u64(step_seed, stream, idx >> np.uint64(2))
    return ((h >> (np.uint64(16) * (idx & np.uint64(3)))) & np.uint64(0xFFFF)).astype(np.uint32)


def _drop_threshold(p: float) -> int:
    """csrc/common.cuh::drop_threshold: round(p * 65536) in fp32, at most 65535."""
    return int(min(np.rint(np.float32(p) * np.float32(65536.0)), np.float32(65535.0)))


def keep_mask(p: float, step_seed: int, stream: int, idx: np.ndarray) -> torch.Tensor:
    """1/(1-p) where kept, 0 where dropped (drop probability quantised to 2^-16 like the CUDA side)."""
    keep = rng_u16(step_seed, stream, idx) >= np.uint32(_drop_threshold(p))
    return torch.from_numpy(keep.astype(np.float32)) / np.float32(1.0 - np.float32(p))


# ---- the same generator on torch int64 tensors, for masks built on the interpreter's device ------------------------
# torch has no uint64 arithmetic: the hash runs on int64 with the same bits.  Multiplies wrap modulo 2^64 like the
# unsigned ones, the right shifts are arithmetic and are made logical by masking the sign-extended high bits, and the
# Python-int constants are reduced to their two's complement int64 value.
def _i64(v: int) -> int:
    v &= M64
    return v - (1 << 64) if v >> 63 else v


def _srl(z: torch.Tensor, s: int) -> torch.Tensor:
    return (z >> s) & ((1 << (64 - s)) - 1)


def rng_u64_t(step_seed: int, stream: int, qidx: torch.Tensor) -> torch.Tensor:
    """rng_u64 on an int64 tensor of quad indices; the uint64 result as int64 bits."""
    z = qidx.to(torch.int64) * _i64(0x9E3779B97F4A7C15)
    z += _i64(step_seed * 0xD1342543DE82EF95 + ((stream << 32) | 0x9E3779B9))
    z ^= _srl(z, 30)
    z *= _i64(0xBF58476D1CE4E5B9)
    z ^= _srl(z, 27)
    z *= _i64(0x94D049BB133111EB)
    z ^= _srl(z, 31)
    return z


def rng_u16_t(step_seed: int, stream: int, idx: torch.Tensor) -> torch.Tensor:
    """rng_u16 on an int64 tensor of element indices."""
    idx = idx.to(torch.int64)
    return (rng_u64_t(step_seed, stream, _srl(idx, 2)) >> ((idx & 3) * 16)) & 0xFFFF


def keep_mask_t(p: float, step_seed: int, stream: int, idx: torch.Tensor) -> torch.Tensor:
    """keep_mask on an int64 tensor of element indices, on that tensor's device."""
    keep = rng_u16_t(step_seed, stream, idx) >= _drop_threshold(p)
    return keep.to(torch.float32) / np.float32(1.0 - np.float32(p))


def keep_mask_range(p: float, step_seed: int, stream: int, n: int, device) -> torch.Tensor:
    """keep_mask of the element indices 0 .. n-1, built on `device`: one hash per quad, its four 16-bit lanes in
    order, so a mask of N*C*L elements costs N*C*L/4 hashes and no index array of its own size."""
    h = rng_u64_t(step_seed, stream, torch.arange((n + 3) // 4, dtype=torch.int64, device=device))
    thr = _drop_threshold(p)
    keep = torch.stack([(_srl(h, 16 * j) & 0xFFFF) >= thr for j in range(4)], 1).view(-1)[:n]
    del h
    return keep.to(torch.float32) / np.float32(1.0 - np.float32(p))


def upsample_linear(X: torch.Tensor, size: int) -> torch.Tensor:
    """F.interpolate(X, size=size, mode="linear") (align_corners=False) with the source coordinates the fp32 model
    computes, whatever the dtype of X: ratio = fp32(L_src) / fp32(size) and src = ratio * (p + 0.5) - 0.5 rounded to fp32
    once (the fused multiply-add of csrc/conv_common.cuh::upsample_coords).  Where size / L_src is not a power of two,
    the fp32 coordinate of a sample near the end of a row is ~L_src * 2^-24 off the exact one (1e-4 at L_src = 1501),
    which shifts its interpolation weights by as much; the coordinates are part of what the op computes, so the
    interpreter takes them from the fp32 model and only the blend runs in X's dtype."""
    Ls = X.shape[-1]
    ratio = (torch.tensor(Ls, dtype=torch.float32) / torch.tensor(size, dtype=torch.float32)).item()
    p = torch.arange(size, dtype=torch.float64, device=X.device)
    src = (ratio * (p + 0.5) - 0.5).float().double().clamp_min(0)     # exact in float64, then one fp32 rounding
    i0 = src.long().clamp_max(Ls - 1)
    i1 = (i0 + 1).clamp_max(Ls - 1)
    lam = (src - i0).clamp(0, 1).to(X.dtype)
    return X[..., i0] * (1 - lam) + X[..., i1] * lam


class Interp:
    def __init__(self, plan: Plan, dtype=torch.float32):
        self.p = plan
        self.dt = dtype
        self.dev = plan.flat.P.device       # the plan's own device: a CUDA plan is interpreted there

    # ---- BatchNorm coefficient algebra (mirrors csrc/common.cuh) ---------------------------------
    def _stats(self, e):
        st = self.p.stat
        s1 = st[e.st_off:e.st_off + e.C]
        s2 = st[e.st_off + e.C:e.st_off + 2 * e.C]
        mean = s1 / e.count
        var = (s2 / e.count - mean * mean).clamp_min(0.0)
        return mean, var

    def _pv(self, ref):
        return self.p.flat.P[ref.off:ref.off + ref.numel].double()

    def _rb(self, e):
        rb = self.p.flat.RB
        return rb[e.rb_off:e.rb_off + e.C].double(), rb[e.rb_off + e.C:e.rb_off + 2 * e.C].double()

    def bn_fwd(self, bn: int, c0: int, C: int):
        """(scale, shift) with BN(x) = scale*x + shift, chained BN folded in."""
        e = self.p.bns[bn]
        eps = 1e-5
        g1, b1 = self._pv(e.gamma), self._pv(e.beta)
        if self.p.training:
            mean, var = self._stats(e)
        else:
            mean, var = self._rb(e)
        s1 = g1 / torch.sqrt(var + eps)
        t1 = b1 - mean * s1
        if e.chain >= 0:
            e2 = self.p.bns[e.chain]
            g2, b2 = self._pv(e2.gamma), self._pv(e2.beta)
            if self.p.training:
                mean2, var2 = b1, s1 * s1 * var
            else:
                mean2, var2 = self._rb(e2)
            s2 = g2 / torch.sqrt(var2 + eps)
            scale, shift = s2 * s1, s2 * (t1 - mean2) + b2
        else:
            scale, shift = s1, t1
        sl = slice(c0, c0 + C)
        return scale[sl].to(self.dt), shift[sl].to(self.dt)

    def bn_khat(self, bn: int, c0: int, C: int):
        """(mu, istd) of the FIRST bn: khat = (x - mu) * istd is the basis of gstat's second sum."""
        e = self.p.bns[bn]
        mean, var = self._stats(e)
        sl = slice(c0, c0 + C)
        return mean[sl].to(self.dt), (1.0 / torch.sqrt(var + 1e-5))[sl].to(self.dt)

    def bn_bwd(self, bn: int, c0: int, C: int):
        """(A, Bx, Cc): d/dx = A*du + Bx*x + Cc."""
        e = self.p.bns[bn]
        eps = 1e-5
        cnt = e.count
        mean, var = self._stats(e)
        istd = 1.0 / torch.sqrt(var + eps)
        g1 = self._pv(e.gamma)
        gs = self.p.gstat
        S1 = gs[e.st_off:e.st_off + e.C]
        S2 = gs[e.st_off + e.C:e.st_off + 2 * e.C]
        if e.chain < 0:
            A = g1 * istd
            kc = -A * S2 / cnt                       # coefficient of khat
            c0_ = -A * S1 / cnt
        else:
            e2 = self.p.bns[e.chain]
            g2 = self._pv(e2.gamma)
            vk = var * istd * istd                  # var of khat
            istd2 = 1.0 / torch.sqrt(g1 * g1 * vk + eps)
            dg1 = g2 * istd2 * S2 * (1.0 - g1 * g1 * istd2 * istd2 * vk)
            A = g1 * istd * g2 * istd2
            kc = -g1 * istd * (g2 * istd2 * g1 * g1 * istd2 * istd2 * S2 / cnt + dg1 / cnt)
            c0_ = -A * S1 / cnt
        Bx = kc * istd
        Cc = c0_ - kc * istd * mean
        sl = slice(c0, c0 + C)
        return A[sl].to(self.dt), Bx[sl].to(self.dt), Cc[sl].to(self.dt)

    # ---- views ------------------------------------------------------------------------------------
    def base(self, v: View) -> torch.Tensor:
        x = v.buf.x[:, v.c0:v.c0 + v.C].to(self.dt)
        if v.bn >= 0:
            s, t = self.bn_fwd(v.bn, v.bn_c0, v.C)
            x = x * s[None, :, None] + t[None, :, None]
        return x

    @staticmethod
    def act(u, a):
        return F.gelu(u) if a == ACT_GELU else u

    def value(self, v: View) -> torch.Tensor:
        return self.act(self.base(v), v.act)

    # ---- forward ----------------------------------------------------------------------------------
    def _conv_expr(self, f: Op, bases, W):
        X = torch.cat([self.act(b, v.act) for b, v in zip(bases, f.ins)], 1)
        if f.pool > 1:
            X = F.avg_pool1d(X, f.pool, ceil_mode=True) + F.max_pool1d(X, f.pool, ceil_mode=True)
        elif f.up_src_L > 0:
            X = upsample_linear(X, f.L_in)
        pr = (f.L_out - 1) * f.stride + f.k - f.L_in - f.pad_left
        X = F.pad(X, (f.pad_left, pr))
        return F.conv1d(X, W, None, stride=f.stride, groups=f.groups)

    def _mask(self, p: float, stream: int, n: int) -> torch.Tensor:
        """keep_mask of the element indices 0 .. n-1 in the interpreter's dtype, on its device: built there for a CUDA
        plan (a mask of a full-length layer at a production batch is 10^8 elements), with numpy for a CPU plan."""
        seed = int(self.p.step_seed.item())
        if self.dev.type == "cuda":
            return keep_mask_range(p, seed, stream, n, self.dev).to(self.dt)
        return keep_mask(p, seed, stream, np.arange(n, dtype=np.uint64)).to(self.dev, self.dt)

    def _drop_factor(self, f: Op):
        """delta(n) * D(n,c,l) multiplying conv+bias, and alpha(n)."""
        N, C, L = f.N, f.Cout, f.L_out
        fac = torch.ones(N, C, L, dtype=self.dt, device=self.dev)
        if f.p_elem > 0:
            fac = fac * self._mask(f.p_elem, f.seed_elem, N * C * L).view(N, C, L)
        if f.p_path > 0:
            fac = fac * self._mask(f.p_path, f.seed_path, N).view(N, 1, 1)
        alpha = torch.ones(N, 1, 1, dtype=self.dt, device=self.dev)
        if f.p_alpha > 0:
            alpha = self._mask(f.p_alpha, f.seed_alpha, N).view(N, 1, 1)
        return fac, alpha

    def _W(self, f: Op):
        if f.Wx is not None:
            return self.p.Wx[f.Wx.off:f.Wx.off + f.Wx.numel].view(f.Wx.shape).to(self.dt)
        return self.p.flat.P[f.W.off:f.W.off + f.W.numel].view(f.W.shape).to(self.dt)

    def _parts(self, f: Op):
        P = self.p.flat.P
        i, d, pc = (P[r.off:r.off + r.numel].view(r.shape).double() for r in f.wparts)
        return i[:, :, 0], d[:, 0, :], pc[:, :, 0]          # [C,C], [C,k], [Cout,C]

    def _bias(self, f: Op):
        return None if f.bias is None else self.p.flat.P[f.bias.off:f.bias.off + f.bias.numel].to(self.dt)

    def conv_fwd(self, f: Op):
        Y = self._conv_expr(f, [self.base(v) for v in f.ins], self._W(f))
        b = self._bias(f)
        if b is not None:
            Y = Y + b[None, :, None]
        fac, alpha = self._drop_factor(f)
        Y = Y * fac
        if f.res_a is not None:
            Y = Y + self.value(f.res_a)
        Y = Y * alpha
        if f.res_b is not None:
            Y = Y + self.value(f.res_b)
        if f.out_act == OUT_SIGMOID:
            Y = torch.sigmoid(Y)
        o = f.out
        o.buf.x[:, o.c0:o.c0 + o.C] = Y.float()
        if o.bn >= 0 and self.p.training:
            e = self.p.bns[o.bn]
            Yd = o.buf.x[:, o.c0:o.c0 + o.C].double()
            self.p.stat[e.st_off + o.bn_c0:e.st_off + o.bn_c0 + o.C] += Yd.sum((0, 2))
            self.p.stat[e.st_off + e.C + o.bn_c0:e.st_off + e.C + o.bn_c0 + o.C] += (Yd * Yd).sum((0, 2))

    def _att_expr(self, f: Op, q, k, v):
        N, C, Lq = q.shape
        H = f.heads
        E = C // H
        qh = q.view(N, H, E, Lq) / math.sqrt(E)
        kh = k.view(N, H, E, -1)
        vh = v.view(N, H, E, -1)
        s = qh.transpose(-1, -2) @ kh
        a = s.softmax(-1)
        lse = torch.logsumexp(s, -1)
        if f.p_attn > 0:
            Lk = kh.shape[-1]
            a = a * self._mask(f.p_attn, f.seed_attn, N * H * Lq * Lk).view(N, H, Lq, Lk)
        o = (a @ vh.transpose(-1, -2)).transpose(-1, -2).reshape(N, C, Lq)
        return o, lse

    def att_fwd(self, f: Op):
        q, k, v = (self.value(x) for x in f.ins)
        o, lse = self._att_expr(f, q, k, v)
        f.out.buf.x[:, f.out.c0:f.out.c0 + f.out.C] = o.float()
        if f.lse is not None:
            f.lse.copy_(lse.float())

    def _headvec_expr(self, f: Op, xin):
        z = F.linear(xin.mean(-1), self._W(f).view(f.Cout, f.Cin), self._bias(f))
        if f.out_act == OUT_SIGMOID:
            return torch.sigmoid(z) * f.out_scale
        if f.out_act == OUT_SOFTMAX:
            return torch.softmax(z, -1)
        return z

    def run_fwd(self, x: torch.Tensor, upto: int | None = None):
        p = self.p
        p.x_in.x.copy_(x)
        p.stat.zero_()
        for i, f in enumerate(p.fwd_ops):
            if upto is not None and i >= upto:
                break
            self.run_fwd_op(f)
        return p.y_out.x

    def run_fwd_op(self, f: Op):
        p = self.p
        if f.kind == _lib.CONV_FWD:
            self.conv_fwd(f)
        elif f.kind == _lib.ATT_FWD:
            self.att_fwd(f)
        elif f.kind == _lib.HEADVEC_FWD:
            f.out.buf.x[:, :, 0] = self._headvec_expr(f, self.value(f.ins[0])).float()
        elif f.kind == _lib.BN_FINALIZE_FWD:
            self.bn_finalize_fwd()
        elif f.kind == _lib.STEM_COMPOSE_FWD:
            i, d, pc = self._parts(f)
            we = torch.einsum("oc,ct,ci->oit", pc, d, i)
            self.p.Wx[f.Wx.off:f.Wx.off + f.Wx.numel] = we.reshape(-1).float()
        elif f.kind == _lib.BN_PREPARE_FWD:
            pass        # coefficients are evaluated on the fly here (bn_fwd / bn_khat)
        else:
            raise ValueError(f.kind)

    def bn_finalize_fwd(self):
        p = self.p
        rb = p.flat.RB
        for e in p.bns:
            if e.is_chained:
                continue
            mean, var = self._stats(e)
            unb = e.count / max(e.count - 1.0, 1.0)

            def upd(ent, m, v):
                rb[ent.rb_off:ent.rb_off + ent.C] = (0.9 * rb[ent.rb_off:ent.rb_off + ent.C].double() + 0.1 * m).float()
                rb[ent.rb_off + ent.C:ent.rb_off + 2 * ent.C] = (
                    0.9 * rb[ent.rb_off + ent.C:ent.rb_off + 2 * ent.C].double() + 0.1 * v * unb).float()

            upd(e, mean, var)
            if e.chain >= 0:
                g1, b1 = self._pv(e.gamma), self._pv(e.beta)
                upd(p.bns[e.chain], b1, g1 * g1 * var / (var + 1e-5))
        p.flat.NBT[:len(p.bns)] += 1

    # ---- backward ---------------------------------------------------------------------------------
    def out_grad(self, f: Op) -> torch.Tensor:
        o = f.out
        sl = slice(o.c0, o.c0 + o.C)
        g = torch.zeros(f.N, o.C, o.buf.L, dtype=self.dt, device=self.dev)
        if o.buf.dxd is not None:
            g = g + o.buf.dxd[:, sl].to(self.dt)
        if o.bn >= 0 and o.buf.du is not None:
            A, Bx, Cc = self.bn_bwd(o.bn, o.bn_c0, o.C)
            g = g + A[None, :, None] * o.buf.du[:, sl].to(self.dt) + Bx[None, :, None] * o.buf.x[:, sl].to(self.dt) \
                + Cc[None, :, None]
        if f.out_act == OUT_SIGMOID and f.kind == _lib.CONV_FWD:
            pr = o.buf.x[:, sl].to(self.dt)
            g = g * pr * (1 - pr)
        return g

    def _deposit(self, t: View, g: torch.Tensor):
        """Write / accumulate `g` into the view's gradient buffer and its BN's gstat."""
        buf = t.buf.du if t.bn >= 0 else t.buf.dxd
        sl = slice(t.c0, t.c0 + t.C)
        if t.accum:
            buf[:, sl] += g.float()
        else:
            buf[:, sl] = g.float()
        if t.bn >= 0:
            e = self.p.bns[t.bn]
            mu, istd = self.bn_khat(t.bn, t.bn_c0, t.C)
            kh = (t.buf.x[:, sl].to(self.dt) - mu[None, :, None]) * istd[None, :, None]
            gd = g.double()
            a = e.st_off + t.bn_c0
            self.p.gstat[a:a + t.C] += gd.sum((0, 2))
            self.p.gstat[a + e.C:a + e.C + t.C] += (gd * kh.double()).sum((0, 2))

    def run_bwd_op(self, op: Op):
        p = self.p
        f = op.fwd
        G = p.flat.G
        if op.kind == _lib.BN_PREPARE_BWD:
            return      # coefficients are evaluated on the fly here (bn_bwd)
        if op.kind == _lib.STEM_COMPOSE_BWD:
            i, d, pc = (t.detach().requires_grad_(True) for t in self._parts(f))
            we = torch.einsum("oc,ct,ci->oit", pc, d, i)
            dwe = p.dWx[f.Wx.off:f.Wx.off + f.Wx.numel].view(f.Wx.shape).double()
            gi, gd, gp = torch.autograd.grad(we, [i, d, pc], dwe)
            for r, gq in zip(f.wparts, (gi, gd, gp)):
                G[r.off:r.off + r.numel] += gq.reshape(-1).float()
            return
        if op.kind == _lib.ZERO:
            (op.out.buf.du if op.out.bn >= 0 else op.out.buf.dxd).zero_()
        elif op.kind == _lib.RES_BWD:
            g = self.out_grad(f)
            _, alpha = self._drop_factor(f)
            if op.res_a is not None:
                self._deposit(op.res_a, g * alpha)
            if op.res_b is not None:
                self._deposit(op.res_b, g)
        elif op.kind in (_lib.CONV_BWD_W, _lib.CONV_BWD_DATA):
            fac, alpha = self._drop_factor(f)
            gacc = self.out_grad(f) * alpha * fac
            bases = [self.base(v).detach().requires_grad_(True) for v in f.ins]
            W = self._W(f).detach().requires_grad_(True)
            Y = self._conv_expr(f, bases, W)
            if op.kind == _lib.CONV_BWD_W:
                (dW,) = torch.autograd.grad(Y, W, gacc)
                if f.Wx is not None:
                    p.dWx[f.Wx.off:f.Wx.off + f.Wx.numel] += dW.reshape(-1).float()
                else:
                    G[f.W.off:f.W.off + f.W.numel] += dW.reshape(-1).float()
                if f.bias is not None:
                    G[f.bias.off:f.bias.off + f.bias.numel] += gacc.sum((0, 2)).float()
            else:
                need = [i for i, t in enumerate(op.ins) if t.buf is not None]
                grads = torch.autograd.grad(Y, [bases[i] for i in need], gacc)
                for i, g in zip(need, grads):
                    self._deposit(op.ins[i], g)
        elif op.kind == _lib.ATT_BWD_Q or op.kind == _lib.ATT_BWD_KV:
            q, k, v = (self.value(x).detach().requires_grad_(True) for x in f.ins)
            o, _ = self._att_expr(f, q, k, v)
            do = f.out.buf.dxd[:, f.out.c0:f.out.c0 + f.out.C].to(self.dt)
            dq, dk, dv = torch.autograd.grad(o, [q, k, v], do)
            if op.kind == _lib.ATT_BWD_Q:
                self._deposit(op.ins[0], dq)
            else:
                self._deposit(op.ins[1], dk)
                self._deposit(op.ins[2], dv)
        elif op.kind == _lib.HEADVEC_BWD:
            xin = self.value(f.ins[0]).detach().requires_grad_(True)
            W = self._W(f).detach().requires_grad_(True)
            b = self._bias(f).detach().requires_grad_(True)
            z = F.linear(xin.mean(-1), W.view(f.Cout, f.Cin), b)
            y = torch.sigmoid(z) * f.out_scale if f.out_act == OUT_SIGMOID else (
                torch.softmax(z, -1) if f.out_act == OUT_SOFTMAX else z)
            dy = f.out.buf.dxd[:, :, 0].to(self.dt)
            dx, dW, db = torch.autograd.grad(y, [xin, W, b], dy)
            G[f.W.off:f.W.off + f.W.numel] += dW.reshape(-1).float()
            G[f.bias.off:f.bias.off + f.bias.numel] += db.float()
            self._deposit(op.ins[0], dx)
        elif op.kind == _lib.BN_FINALIZE_BWD:
            self.bn_finalize_bwd()
        else:
            raise ValueError(op.kind)

    def bn_finalize_bwd(self):
        p = self.p
        G = p.flat.G
        gs = p.gstat
        for e in p.bns:
            if e.is_chained:
                continue
            S1 = gs[e.st_off:e.st_off + e.C]
            S2 = gs[e.st_off + e.C:e.st_off + 2 * e.C]
            sc = 1.0 / p.world
            if e.chain < 0:
                G[e.gamma.off:e.gamma.off + e.C] += (S2 * sc).float()
                G[e.beta.off:e.beta.off + e.C] += (S1 * sc).float()
            else:
                e2 = p.bns[e.chain]
                mean, var = self._stats(e)
                istd = 1.0 / torch.sqrt(var + 1e-5)
                g1, g2 = self._pv(e.gamma), self._pv(e2.gamma)
                vk = var * istd * istd
                istd2 = 1.0 / torch.sqrt(g1 * g1 * vk + 1e-5)
                G[e2.beta.off:e2.beta.off + e.C] += (S1 * sc).float()
                G[e2.gamma.off:e2.gamma.off + e.C] += (g1 * istd2 * S2 * sc).float()
                G[e.gamma.off:e.gamma.off + e.C] += (g2 * istd2 * S2 * (1.0 - g1 * g1 * istd2 * istd2 * vk) * sc).float()
                # dbeta of the first BN is analytically zero

    def run_bwd(self, dy: torch.Tensor):
        p = self.p
        p.gstat.zero_()
        p.flat.G.zero_()
        p.dWx.zero_()
        p.y_out.dxd.copy_(dy.view_as(p.y_out.dxd))
        for op in p.bwd_ops:
            self.run_bwd_op(op)
