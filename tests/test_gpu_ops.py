"""-m gpu: every CUDA kernel against the plan interpreter, op by op with teacher forcing, through the
C-ABI (seist_plan_run).  Tolerance: 2e-4 of the tensor's max-abs per op (fp32 arithmetic, different
summation order); end-to-end parity with the reference has its own test (test_gpu_model.py)."""
import pytest
import torch

from harness import build_pair, push_state, rel_err, run_gpu_op
from seist_b200 import _lib

TOL = 2e-4

CASES = [
    # name, N, L, training, drops
    ("seist_s_dpk", 2, 1024, False, None),
    ("seist_s_dpk", 3, 1000, True, None),          # ragged length: pool tails, irregular up-sampling sizes
    ("seist_m_dpk", 2, 2048, True, None),
    ("seist_l_dpk", 2, 1024, True, None),
    ("seist_m_emg", 2, 1024, True, None),
    ("seist_s_pmp", 2, 1024, True, None),
    ("seist_s_dpk", 2, 1024, True, dict(path_drop_rate=0.3, attn_drop_rate=0.2, key_drop_rate=0.2,
                                        mlp_drop_rate=0.25, other_drop_rate=0.15)),
]


def _slices_of(view):
    return slice(view.c0, view.c0 + view.C)


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,L,training,drops", CASES)
def test_ops_match_interpreter(name, N, L, training, drops):
    p_cpu, p_gpu, it, _, _ = build_pair(name, N, L, training, drops)
    torch.manual_seed(1)
    x = torch.randn(N, 3, L)
    p_cpu.step_seed.fill_(12345)
    p_cpu.x_in.x.copy_(x)
    p_cpu.stat.zero_()
    failures = []
    bufs_c = {b.name: b for b in p_cpu.bufs}
    bufs_g = {b.name: b for b in p_gpu.bufs}

    for i, (fc, fg) in enumerate(zip(p_cpu.fwd_ops, p_gpu.fwd_ops)):
        push_state(p_cpu, p_gpu)
        it.run_fwd_op(fc)
        run_gpu_op(p_gpu, p_gpu.c_fwd, i)
        errs = []
        if fc.out is not None:
            sl = _slices_of(fc.out)
            errs.append(("out",) + rel_err(fg.out.buf.x[:, sl], fc.out.buf.x[:, sl]))
            if training and fc.out.bn >= 0:
                e = p_cpu.bns[fc.out.bn]
                errs.append(("stat",) + rel_err(p_gpu.stat[e.st_off:e.st_off + 2 * e.C], p_cpu.stat[e.st_off:e.st_off + 2 * e.C]))
        if fc.lse is not None:
            errs.append(("lse",) + rel_err(fg.lse, fc.lse))
        if fc.kind == _lib.BN_FINALIZE_FWD:
            errs.append(("running",) + rel_err(p_gpu.flat.RB, p_cpu.flat.RB))
        if fc.kind == _lib.STEM_COMPOSE_FWD:
            errs.append(("W_eff",) + rel_err(p_gpu.Wx, p_cpu.Wx))
        for what, err, ref in errs:
            if not err < TOL:
                failures.append(f"fwd[{i}] {fc.name} {what}: rel {err:.3e} (max {ref:.3e})")
    assert not failures, "\n".join(failures[:20])
    if not training:
        return

    # backward, seeded with a smooth gradient
    p_cpu.gstat.zero_()
    p_cpu.flat.G.zero_()
    p_cpu.dWx.zero_()
    g = torch.Generator().manual_seed(2)
    p_cpu.y_out.dxd.copy_(torch.randn(p_cpu.y_out.dxd.shape, generator=g) / p_cpu.y_out.dxd[0].numel() ** 0.5)
    for i, (bc, bg) in enumerate(zip(p_cpu.bwd_ops, p_gpu.bwd_ops)):
        push_state(p_cpu, p_gpu)
        if bc.kind == _lib.ATT_BWD_KV:      # reads the `delta` scratch its sibling kernel produces
            run_gpu_op(p_gpu, p_gpu.c_bwd, i - 1)
        it.run_bwd_op(bc)
        run_gpu_op(p_gpu, p_gpu.c_bwd, i)
        errs = []
        targets = [t for t in list(bc.ins) + [bc.res_a, bc.res_b] if t is not None and t.buf is not None]
        if bc.kind in (_lib.CONV_BWD_DATA, _lib.RES_BWD, _lib.ATT_BWD_Q, _lib.ATT_BWD_KV, _lib.HEADVEC_BWD):
            gtargets = [t for t in list(bg.ins) + [bg.res_a, bg.res_b] if t is not None and t.buf is not None]
            if bc.kind == _lib.ATT_BWD_Q:
                targets, gtargets = targets[:1], gtargets[:1]
            if bc.kind == _lib.ATT_BWD_KV:
                targets, gtargets = targets[1:], gtargets[1:]
            for tc, tg in zip(targets, gtargets):
                sl = _slices_of(tc)
                a = (tg.buf.du if tg.bn >= 0 else tg.buf.dxd)[:, sl]
                b = (tc.buf.du if tc.bn >= 0 else tc.buf.dxd)[:, sl]
                errs.append((f"grad({tc.buf.name})",) + rel_err(a, b))
            errs.append(("gstat",) + rel_err(p_gpu.gstat, p_cpu.gstat))
        if bc.kind in (_lib.CONV_BWD_W, _lib.HEADVEC_BWD, _lib.BN_FINALIZE_BWD, _lib.STEM_COMPOSE_BWD):
            errs.append(("G",) + rel_err(p_gpu.flat.G, p_cpu.flat.G))
            errs.append(("dWx",) + rel_err(p_gpu.dWx, p_cpu.dWx))
        for what, err, ref in errs:
            if not err < TOL:
                failures.append(f"bwd[{i}] {bc.name} {what}: rel {err:.3e} (max {ref:.3e})")
    assert not failures, "\n".join(failures[:30])
    assert _lib.lib().seist_tc_error_flag() == 0, "a tensor-core kernel timed out on an mbarrier"


@pytest.mark.gpu
def test_grad_combine_ops_match_interpreter(monkeypatch):
    """GRAD_COMBINE (BN backward of the output gradient evaluated once, in place) is opt-in: compile the plans with
    it enabled for every 1x1 conv of width >= 16 and run the same op-by-op comparison."""
    monkeypatch.setenv("SEIST_COMBINE_CIN", "16")
    test_ops_match_interpreter("seist_m_dpk", 2, 2048, True, None)
    test_ops_match_interpreter("seist_s_dpk", 3, 1000, True, None)      # ragged length: scalar combine path


def _run_cases_in_child(env_extra, cases):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, **env_extra)
    calls = "".join(f"T.test_ops_match_interpreter({c});" for c in cases)
    code = ("import sys; sys.path.insert(0, 'tests'); import test_gpu_ops as T; from seist_b200 import _lib;" + calls +
            "assert _lib.lib().seist_tc_error_flag() == 0, 'tensor-core mbarrier wait timed out'; print('TC-OK')")
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "TC-OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


_DROPS = "dict(path_drop_rate=0.3, attn_drop_rate=0.2, key_drop_rate=0.2, mlp_drop_rate=0.25, other_drop_rate=0.15)"


@pytest.mark.gpu
def test_tcconv_engine_on_every_eligible_op():
    """The warp-specialised wgmma + TMA engine (tcconv.cu) is dispatched by a measured rule (api.cu::tcc_auto); here
    it is FORCED onto every eligible forward / data-gradient conv (SEIST_TCC=1, read once per process -> child process):
    stride-1 k-tap and 1x1 convs of every width, grouped convs, multi-view inputs, residuals, dropout, sigmoid head."""
    _run_cases_in_child({"SEIST_TCC": "1"}, [
        "'seist_m_dpk', 2, 2048, True, None",
        "'seist_l_dpk', 2, 1024, True, None",
        f"'seist_s_dpk', 2, 1024, True, {_DROPS}",
        "'seist_s_dpk', 2, 1024, False, None",
    ])
