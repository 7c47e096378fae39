"""Lane scheduler: spreads the ops of a plan over a few CUDA streams ("lanes") by data dependence.

The plan is emitted as one linear list, but the network has branches that do not depend on each other — the two to four
kernel-size paths of every `MultiScaleMixedConv` (reference models/seist.py:259-318), the attention and convolution paths
of `MultiPathTransformerLayer` (:396-504), q / k / v projections, the three `DSConvNormAct` paths of a stem block
(:158-195) — and at the encoder's lengths (128-1024 samples) one kernel neither fills the GPU nor hides its own latency.
`schedule_lanes` derives the dependences from the operands' buffers (x / du / dxd slices, BatchNorm statistic slots and
coefficient tables, composed-weight scratch) and assigns every op a lane; the C executor (`seist_plan_run_lanes`)
issues each op on its lane's stream and connects the lanes with events, which a CUDA-graph capture turns into graph edges.
Lane 0 = critical chain (high priority), lane 1 = independent branches, last lane = weight gradients (never on the
critical path; what `seist_plan_run2` did before).
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Set, Tuple

from . import _lib

MAX_WAIT = 4


class _Tracker:
    """last writers / readers-since-write of (key, channel slice) resources"""

    def __init__(self):
        self.writers: Dict[tuple, List[Tuple[int, int, int]]] = {}
        self.readers: Dict[tuple, List[Tuple[int, int, int]]] = {}

    @staticmethod
    def _ov(a0, a1, b0, b1):
        return a0 < b1 and b0 < a1

    def read(self, key, c0, c1, op, deps: Set[int]):
        for (a, b, w) in self.writers.get(key, ()):
            if self._ov(a, b, c0, c1):
                deps.add(w)
        self.readers.setdefault(key, []).append((c0, c1, op))

    def write(self, key, c0, c1, op, deps: Set[int]):
        ws = self.writers.setdefault(key, [])
        for (a, b, w) in ws:
            if self._ov(a, b, c0, c1):
                deps.add(w)
        rs = self.readers.get(key, [])
        for (a, b, r) in rs:
            if self._ov(a, b, c0, c1) and r != op:
                deps.add(r)
        self.readers[key] = [(a, b, r) for (a, b, r) in rs if not self._ov(a, b, c0, c1)]
        ws[:] = [(a, b, w) for (a, b, w) in ws if not (c0 <= a and b <= c1)]
        ws.append((c0, c1, op))


BIG = 1 << 30


def _deps(plan, ops) -> List[Set[int]]:
    L = _lib
    tr = _Tracker()
    out: List[Set[int]] = []
    barrier_prev: Optional[int] = None

    def rd_view(v, i, d, want_x=True):
        if v is None or v.buf is None or v.C == 0:
            return
        if want_x:
            tr.read(("x", id(v.buf)), v.c0, v.c0 + v.C, i, d)
        if v.bn >= 0:
            tr.read(("coef_f", v.bn), 0, BIG, i, d)

    def gkey(v):
        return ("du" if v.bn >= 0 else "dxd", id(v.buf))

    def rd_outgrad(f, i, d):
        o = f.out
        sl = (o.c0, o.c0 + o.C)
        tr.read(("du", id(o.buf)), *sl, i, d)
        tr.read(("dxd", id(o.buf)), *sl, i, d)
        tr.read(("x", id(o.buf)), *sl, i, d)
        if o.bn >= 0:
            tr.read(("coef_b", o.bn), 0, BIG, i, d)

    def wr_target(t, i, d):
        if t is None or t.buf is None or t.C == 0:
            return
        tr.write(gkey(t), t.c0, t.c0 + t.C, i, d)
        tr.read(("x", id(t.buf)), t.c0, t.c0 + t.C, i, d)
        if t.bn >= 0:
            tr.read(("coef_f", t.bn), 0, BIG, i, d)
            tr.write(("gstat", t.bn), t.bn_c0, t.bn_c0 + t.C, i, d)

    for i, op in enumerate(ops):
        d: Set[int] = set()
        f = op.fwd if op.fwd is not None else op
        k = op.kind
        if barrier_prev is not None:
            d.add(barrier_prev)
        if k == L.CONV_FWD:
            for v in op.ins:
                rd_view(v, i, d)
            rd_view(op.res_a, i, d)
            rd_view(op.res_b, i, d)
            if op.Wx is not None:
                tr.read(("Wx", op.Wx.off), 0, BIG, i, d)
            o = op.out
            tr.write(("x", id(o.buf)), o.c0, o.c0 + o.C, i, d)
            if o.bn >= 0 and plan.training:
                tr.write(("stat", o.bn), o.bn_c0, o.bn_c0 + o.C, i, d)
        elif k == L.ATT_FWD:
            for v in op.ins:
                rd_view(v, i, d)
            tr.write(("x", id(op.out.buf)), op.out.c0, op.out.c0 + op.out.C, i, d)
            tr.write(("lse", id(op)), 0, BIG, i, d)
        elif k == L.HEADVEC_FWD:
            rd_view(op.ins[0], i, d)
            tr.write(("x", id(op.out.buf)), 0, BIG, i, d)
        elif k == L.STEM_COMPOSE_FWD:
            tr.write(("Wx", op.Wx.off), 0, BIG, i, d)
        elif k == L.BN_PREPARE_FWD:
            for b in range(op.bn_lo, op.bn_lo + op.n_bn):
                tr.read(("stat", b), 0, BIG, i, d)
                tr.write(("coef_f", b), 0, BIG, i, d)
        elif k == L.BN_PREPARE_BWD:
            for b in range(op.bn_lo, op.bn_lo + op.n_bn):
                tr.read(("gstat", b), 0, BIG, i, d)
                tr.write(("coef_b", b), 0, BIG, i, d)
        elif k == L.RES_BWD:
            rd_outgrad(f, i, d)
            wr_target(op.res_a, i, d)
            wr_target(op.res_b, i, d)
        elif k == L.CONV_BWD_W:
            rd_outgrad(f, i, d)
            for v in f.ins:
                rd_view(v, i, d)
            if f.Wx is not None:
                tr.write(("dWx", f.Wx.off), 0, BIG, i, d)
        elif k == L.CONV_BWD_DATA:
            rd_outgrad(f, i, d)
            for t in op.ins:
                wr_target(t, i, d)
        elif k == L.ZERO:
            t = op.out
            tr.write(gkey(t), 0, BIG, i, d)
        elif k in (L.ATT_BWD_Q, L.ATT_BWD_KV):
            for v in f.ins:
                rd_view(v, i, d)
            tr.read(("dxd", id(f.out.buf)), f.out.c0, f.out.c0 + f.out.C, i, d)
            tr.read(("x", id(f.out.buf)), f.out.c0, f.out.c0 + f.out.C, i, d)
            tr.read(("lse", id(f)), 0, BIG, i, d)
            tgt = op.ins[:1] if k == L.ATT_BWD_Q else op.ins[1:]
            if k == L.ATT_BWD_Q:
                tr.write(("delta", id(f)), 0, BIG, i, d)
            else:
                tr.read(("delta", id(f)), 0, BIG, i, d)
            for t in tgt:
                if t is not None and t.buf is not None:
                    tr.write(("dxd", id(t.buf)), t.c0, t.c0 + t.C, i, d)
        elif k == L.HEADVEC_BWD:
            tr.read(("dxd", id(f.out.buf)), 0, BIG, i, d)
            tr.read(("x", id(f.out.buf)), 0, BIG, i, d)
            for t in op.ins:
                wr_target(t, i, d)
        elif k == L.STEM_COMPOSE_BWD:
            tr.read(("dWx", f.Wx.off), 0, BIG, i, d)
        else:
            # BN_FINALIZE_*, GRAD_COMBINE, anything unknown: a full barrier
            d.update(range(i))
            barrier_prev = i
        d.discard(i)
        out.append(d)
    return out


def _cost(op) -> float:
    """rough relative duration of an op: elements it touches"""
    f = op.fwd if op.fwd is not None else op
    n = 0
    for v in list(f.ins) + [f.res_a, f.res_b, f.out]:
        if v is not None and getattr(v, "buf", None) is not None:
            n += v.C * v.buf.L
    return float(n) * max(1, f.k) ** 0.5 + 2000.0


def n_main_lanes() -> int:
    """main lanes (critical chain + independent branches); SEIST_NMAIN=1..3, default 2"""
    return min(3, max(1, int(os.environ.get("SEIST_NMAIN", "2"))))


def schedule_lanes(plan, ops, c_ops, n_main: Optional[int] = None, cost=_cost) -> dict:
    """Fill `lane`, `n_wait`, `wait_ev`, `rec_event` of the ctypes descriptors `c_ops`.  Returns a small summary."""
    L = _lib
    if n_main is None:
        n_main = n_main_lanes()
    deps = _deps(plan, ops)
    w_lane = n_main                                     # weight-gradient lane
    lane_of: List[int] = []
    tail = [-1] * (n_main + 1)
    load = [0.0] * (n_main + 1)
    synced = [[-1] * (n_main + 1) for _ in range(n_main + 1)]     # synced[l][m]: latest op of lane m that lane l has waited for
    rec: Dict[int, int] = {}
    n_ev = 0
    cross = 0
    # the weight gradients behind the last data-gradient op (the first stem block: its input needs no gradient) are the
    # tail of the step: nothing else is left to overlap with, so they are spread over all lanes instead of queueing on one
    main_kinds = (L.CONV_BWD_DATA, L.RES_BWD, L.ATT_BWD_Q, L.ATT_BWD_KV, L.HEADVEC_BWD, L.CONV_FWD, L.ATT_FWD, L.HEADVEC_FWD)
    last_main = max((i for i, op in enumerate(ops) if op.kind in main_kinds), default=len(ops))
    spread_tail = os.environ.get("SEIST_TAIL_SPREAD", "1") != "0"
    rr = 0
    for i, op in enumerate(ops):
        d = deps[i]
        if op.kind == L.CONV_BWD_W and spread_tail and i > last_main:
            lane = (w_lane + rr) % (n_main + 1)
            rr += 1
        elif op.kind in (L.CONV_BWD_W, L.STEM_COMPOSE_BWD):
            lane = w_lane
        else:
            mains = [l for l in range(n_main) if tail[l] in d]
            if len(mains) == 1:
                lane = mains[0]
            elif len(mains) > 1:
                lane = 0
            else:
                lane = min(range(n_main), key=lambda l: (load[l], l))
        waits: List[int] = []
        for m in range(n_main + 1):
            if m == lane:
                continue
            dm = [j for j in d if lane_of[j] == m]
            if not dm:
                continue
            j = max(dm)
            if j <= synced[lane][m]:
                continue
            if j not in rec:
                rec[j] = n_ev
                n_ev += 1
            waits.append(rec[j])
            synced[lane][m] = j
        assert len(waits) <= MAX_WAIT
        c = c_ops[i]
        c.lane = lane
        c.n_wait = len(waits)
        for q in range(MAX_WAIT):
            c.wait_ev[q] = waits[q] if q < len(waits) else -1
        c.rec_event = -1
        cross += len(waits)
        lane_of.append(lane)
        tail[lane] = i
        load[lane] += (cost(op) if cost else 1.0)
    for j, e in rec.items():
        c_ops[j].rec_event = e
    return {"events": n_ev, "cross_lane_waits": cross,
            "ops_per_lane": [sum(1 for x in lane_of if x == l) for l in range(n_main + 1)]}
