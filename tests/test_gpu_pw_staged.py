"""The staged 1x1 data-gradient kernel (pw.cu: pw_bwd_data_staged_kernel): which ops it serves, and its results op by
op against the plan interpreter."""
import ctypes

import pytest
import torch

from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.models import create_model

STAGED = "pw_bwd_data_staged(simt)"
_DROPS = dict(path_drop_rate=0.3, attn_drop_rate=0.2, key_drop_rate=0.2, mlp_drop_rate=0.25, other_drop_rate=0.15)


def _staged_rule(op):
    """Non-pooled 1x1 data gradients with more than one 16-target tile whose weights and operand ring fit one CTA;
    two-tile ops with a GELU target excepted."""
    if op.kind != _lib.CONV_BWD_DATA or op.k != 1 or op.stride != 1 or op.groups != 1 or op.up_src_L > 0:
        return False
    if op.L_out % 4 or op.pool > 1 or not 16 < op.Cin <= 192:
        return False
    if op.Cin <= 32 and any(op.inp[j].act == 1 for j in range(op.n_in)):
        return False
    cin16, coutc = -(-op.Cin // 16) * 16, -(-op.Cout // 8) * 8
    smem = 56 * cin16 + 12 * coutc + 4 * coutc * cin16 + 3 * 8 * 3 * 32 * 16   # PwChan, PwOut, weights, ring
    return smem <= 227 * 1024


def _families(pl, c_ops):
    lib = _lib.lib()
    base, size = ctypes.addressof(c_ops), ctypes.sizeof(_lib.SeistOp)
    return [lib.seist_op_family(base + i * size).decode() for i in range(len(c_ops))]


@pytest.mark.parametrize("name,N,L", [("seist_m_dpk", 2, 8192), ("seist_s_dpk", 3, 1000)])
def test_staged_family_follows_the_shape_rule(name, N, L):
    m = create_model(name, in_channels=3, in_samples=L)
    pl = P.finalize(P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), N, L, training=True).build(), True)
    n_staged = 0
    for c_ops in (pl.c_fwd, pl.c_bwd):
        for op, fam in zip(c_ops, _families(pl, c_ops)):
            assert (fam == STAGED) == _staged_rule(op), (fam, op.Cin, op.Cout, op.L_out, op.pool)
            n_staged += fam == STAGED
    assert n_staged > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,L,drops", [
    ("seist_m_dpk", 3, 2048, None),     # deepest layers: fewer than 128 samples per waveform, ragged last tile
    ("seist_m_dpk", 3, 2048, _DROPS),
    ("seist_s_dpk", 2, 1024, _DROPS),
])
def test_staged_ops_match_interpreter(name, N, L, drops):
    from test_gpu_ops import test_ops_match_interpreter
    staged = _staged_ops(name, N, L, drops)
    # the cases cover targets that accumulate, targets behind GELU and BatchNorm, and dropout when drops are on
    targets = [op.inp[j] for op in staged for j in range(op.n_in)]
    assert any(t.accum for t in targets) and any(t.act == 1 for t in targets) and any(t.bn >= 0 for t in targets)
    assert any(op.p_elem > 0 for op in staged) == (drops is not None)
    assert any(op.N * op.L_out % 128 for op in staged)      # a partial last tile of 128 samples
    test_ops_match_interpreter(name, N, L, True, drops)


def _staged_ops(name, N, L, drops):
    from harness import ZERO_DROPS
    m = create_model(name, in_channels=3, in_samples=L)
    m.set_drop_rates(**(ZERO_DROPS if drops is None else drops))
    pl = P.finalize(P.PlanBuilder(m, P.FlatState(m, torch.device("cpu")), N, L, training=True).build(), True)
    return [op for op, fam in zip(pl.c_bwd, _families(pl, pl.c_bwd)) if fam == STAGED]
