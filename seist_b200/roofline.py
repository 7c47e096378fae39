"""Algorithmic-byte model of plan ops (DESIGN.md §5) and per-op device timing.

Algorithmic bytes of an op = the tensors it must read and write once (fp32, N waveforms); weights are
negligible.  The whole-step figure is SURVEY §8d's BN-barrier model: 6 accesses per BatchNorm-input
element + I/O."""
from __future__ import annotations

import ctypes
from typing import Dict, List

import torch

from . import _lib
from . import plan as P

# SURVEY §8d / BASELINE.md §3: bytes per waveform of one training step (fwd+bwd), fp32 storage, L = 8192
STEP_BYTES_PER_WAVEFORM = {"seist_s_dpk": 32.7e6, "seist_m_dpk": 45.2e6, "seist_l_dpk": 48.8e6, "seist_m_emg": 40.1e6}


def _vbytes(v, N, with_x=True):
    if v is None or v.buf is None or v.C == 0:
        return 0
    return 4 * N * v.C * v.buf.L


def op_bytes(op: P.Op) -> int:
    f = op.fwd if op.fwd is not None else op
    N = f.N
    k = op.kind
    out_b = _vbytes(f.out, N)
    if k == _lib.CONV_FWD:
        return sum(_vbytes(v, N) for v in f.ins) + _vbytes(f.res_a, N) + _vbytes(f.res_b, N) + out_b
    # gradient of the output: du and/or dxd, plus x when the BN-backward prologue or sigmoid' needs it
    og = 0
    if f.out is not None and f.out.buf is not None:
        if f.out.buf.dxd is not None:
            og += out_b
        if f.out.bn >= 0 and f.out.buf.du is not None:
            og += 2 * out_b
        elif f.out_act:
            og += out_b
    if k == _lib.CONV_BWD_W:
        return og + sum(_vbytes(v, N) for v in f.ins)
    if k == _lib.CONV_BWD_DATA:
        b = og
        for t, v in zip(op.ins, f.ins):
            if t is None or t.buf is None:
                continue
            b += _vbytes(v, N) * (1 + 1 + (1 if t.accum else 0))     # x (act'/khat) + g write (+ g read)
        return b
    if k == _lib.RES_BWD:
        b = og
        for t in (op.res_a, op.res_b):
            if t is not None and t.buf is not None:
                b += _vbytes(t, N) * (1 + (1 if t.accum else 0) + (1 if t.bn >= 0 else 0))
        return b
    if k == _lib.ATT_FWD:
        return sum(_vbytes(v, N) for v in f.ins) + out_b
    if k in (_lib.ATT_BWD_Q, _lib.ATT_BWD_KV):
        return sum(_vbytes(v, N) for v in f.ins) + 2 * out_b + (_vbytes(f.ins[0], N) if k == _lib.ATT_BWD_Q
                                                               else 2 * _vbytes(f.ins[1], N))
    if k == _lib.HEADVEC_FWD:
        return _vbytes(f.ins[0], N)
    if k == _lib.HEADVEC_BWD:
        return 2 * _vbytes(f.ins[0], N)
    if k == _lib.ZERO:
        t = op.out.buf.du if op.out.bn >= 0 else op.out.buf.dxd
        return t.numel() * 4
    return 0


def op_flops(op: P.Op) -> float:
    f = op.fwd if op.fwd is not None else op
    if op.kind in (_lib.CONV_FWD, _lib.CONV_BWD_DATA, _lib.CONV_BWD_W):
        return 2.0 * f.N * f.L_out * f.Cout * (f.Cin // f.groups) * f.k
    if op.kind in (_lib.ATT_FWD,):
        return 4.0 * f.N * f.L_out * f.L_in * f.Cout
    if op.kind in (_lib.ATT_BWD_Q, _lib.ATT_BWD_KV):
        return 6.0 * f.N * f.L_out * f.L_in * f.Cout
    return 0.0


def time_ops(plan: P.Plan, reps: int = 3, skip_kinds=(_lib.BN_FINALIZE_FWD,)) -> List[Dict]:
    """Device time of every op of the plan, each launched alone `reps` times (CUDA events on the launching
    stream).  The working set of one op at bench batch sizes exceeds L2, and a 256 MB scratch write between
    launches evicts whatever is left."""
    lib = _lib.lib()
    stream = torch.cuda.current_stream()
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=plan.device)
    size = ctypes.sizeof(_lib.SeistOp)
    rows = []
    for tag, ops, c_ops in (("fwd", plan.fwd_ops, plan.c_fwd), ("bwd", plan.bwd_ops, plan.c_bwd)):
        if c_ops is None:
            continue
        base = ctypes.addressof(c_ops)
        for i, op in enumerate(ops):
            if op.kind in skip_kinds:
                continue
            # an op timed alone must not wait for peers: run BN_PREPARE without its cross-rank exchange
            saved_comm = c_ops[i].comm
            c_ops[i].comm = None
            best = []
            for _ in range(reps):
                flush.fill_(0.0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                _lib.check(lib.seist_plan_run(base + i * size, 1, stream.cuda_stream))
                e1.record(stream)
                e1.synchronize()
                best.append(e0.elapsed_time(e1))
            c_ops[i].comm = saved_comm
            ms = sorted(best)[len(best) // 2]
            fam = lib.seist_op_family(base + i * size)
            rows.append(dict(phase=tag, index=i, name=op.name, kind=op.kind, ms=ms, bytes=op_bytes(op),
                             flops=op_flops(op), family=fam.decode() if fam else str(op.kind)))
    return rows
