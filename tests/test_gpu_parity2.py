"""-m gpu: the parity items the round-1 review found unpinned.

* fused Adam (`seist_adam_step`) against `torch.optim.Adam` / `AdamW` (reference training/train.py:304-316);
* dropout / DropPath ON: the kernels' masks against the reference semantics (nn.Dropout: Bernoulli(1-p) keep, survivors
  scaled 1/(1-p); timm DropPath: one Bernoulli per sample, constant over (C, L), models/seist.py:114,228-253,360-391,
  446-502) — statistical (keep rate within 3 sigma), structural (mask values, per-sample constancy) and per step seed;
* the SyncBatchNorm data-parallel path on ONE GPU: two "virtual ranks" (half batches, world = 2 plans) run the real CUDA
  segments with the statistic all-reduce injected as a plain sum and must equal one rank on the whole batch;
* train-mode parity at the benchmark length (seist_m_dpk B = 16, L = 8192; seist_l_dpk L = 8192) against the oracle;
* the reference's own step order (train.py:87-116) with `torch.optim.Adam`, `torch.compile(model)` and a world-size-1
  `DistributedDataParallel` + `SyncBatchNorm.convert_sync_batchnorm` wrapper — the defaults of training/train.py.
"""
import ctypes
import math
import os
import socket

import pytest
import torch

from harness import ZERO_DROPS, randomize
from oracle import seist_ref as R
from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.engine import run_segment
from seist_b200.models import create_model
from seist_b200.models.loss import BCELoss

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# Adam
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd,decoupled,gscale", [(0.0, False, 1.0), (0.01, False, 1.0), (0.01, True, 1.0), (0.0, False, 0.5)])
def test_fused_adam_matches_torch(wd, decoupled, gscale):
    torch.manual_seed(0)
    n = 100003
    p0 = torch.randn(n, device="cuda")
    grads = [torch.randn(n, device="cuda") * (0.1 + i) for i in range(3)]
    lr, betas, eps = 1e-3, (0.9, 0.999), 1e-8
    ref = torch.nn.Parameter(p0.clone())
    opt = (torch.optim.AdamW if decoupled else torch.optim.Adam)([ref], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    p = p0.clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    lr_t, step_t = torch.full((1,), lr, device="cuda"), torch.zeros(1, device="cuda")
    lib = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    for i, g in enumerate(grads):
        ref.grad = (g * gscale).clone()          # grad_scale = 1/world: the kernel scales the all-reduced sum itself
        opt.step()
        step_t += 1
        _lib.check(lib.seist_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, lr_t.data_ptr(),
                                       step_t.data_ptr(), betas[0], betas[1], eps, wd, 1 if decoupled else 0, gscale, s))
        torch.cuda.synchronize()
        upd_ref = (ref.detach() - p0).abs().max().item()
        err = (p - ref.detach()).abs().max().item()
        # the parameters are O(1): one fp32 ulp of a value in [2, 8) is 2.4e-7 .. 4.8e-7
        assert err <= 1e-6, (i, err, upd_ref)
        assert upd_ref > 0.5 * lr
    st = opt.state[ref]
    assert (m - st["exp_avg"]).abs().max().item() <= 1e-6 * st["exp_avg"].abs().max().item()
    assert (v - st["exp_avg_sq"]).abs().max().item() <= 1e-6 * st["exp_avg_sq"].abs().max().item()


# ------------------------------------------------------------------------------------------------
# dropout / DropPath semantics
# ------------------------------------------------------------------------------------------------
RATES = dict(path_drop_rate=0.3, attn_drop_rate=0.2, key_drop_rate=0.25, mlp_drop_rate=0.2, other_drop_rate=0.15)


def _gpu_plan(name, N, L, drops, seed=1):
    m = randomize(create_model(name, in_channels=3, in_samples=L), seed)
    m.set_drop_rates(**drops)
    m.train().cuda()
    flat = P.FlatState(m, torch.device("cuda"))
    return m, P.finalize(P.PlanBuilder(m, flat, N, L, True).build(), True)


def _run(c_op_or_array, index=None):
    base = ctypes.addressof(c_op_or_array) + (0 if index is None else index * ctypes.sizeof(_lib.SeistOp))
    _lib.check(_lib.lib().seist_plan_run(base, 1, torch.cuda.current_stream().cuda_stream), "op")
    torch.cuda.synchronize()


def _variant(c_ops, i, **changes):
    op = _lib.SeistOp.from_buffer_copy(c_ops[i])
    for k, v in changes.items():
        if k in ("res_a_off", "res_b_off"):
            view = op.res_a if k == "res_a_off" else op.res_b
            view.C = 0
        else:
            setattr(op, k, v)
    return op


def test_dropout_masks_follow_reference_semantics():
    """Every conv op that carries a dropout / DropPath factor, with teacher-forced inputs: out = alpha_n * (F * c + res_a)
    + res_b must decompose with alpha_n in {0, 1/(1-p_alpha)} per sample, F = pf_n * E, pf_n in {0, 1/(1-p_path)} per
    sample and E in {0, 1/(1-p_elem)} per element; keep rates within 3 sigma of 1-p (plus the 2^-16 quantisation)."""
    N, L = 48, 1024
    mA, pa = _gpu_plan("seist_s_dpk", N, L, RATES)
    mB, pb = _gpu_plan("seist_s_dpk", N, L, ZERO_DROPS)
    x, _ = R.synth_waveforms(N, L, seed=4)
    with torch.no_grad():
        pb.x_in.x.copy_(x.cuda())
        pb.stat.zero_()
        _lib.check(_lib.lib().seist_plan_run(ctypes.addressof(pb.c_fwd), len(pb.fwd_ops), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
    state = pb.arena.clone()
    pa.coef.copy_(pb.coef)          # teacher forcing includes the BatchNorm coefficient tables of the consumer views
    pa.stat.copy_(pb.stat)
    pa.step_seed.fill_(777)
    keeps = {"elem": [], "path": [], "alpha": []}
    checked = 0
    for i, (oa, ob) in enumerate(zip(pa.fwd_ops, pb.fwd_ops)):
        if oa.kind != _lib.CONV_FWD or (oa.p_elem == 0 and oa.p_path == 0 and oa.p_alpha == 0):
            continue
        assert oa.name == ob.name
        sl = slice(ob.out.c0, ob.out.c0 + ob.out.C)

        def out_of(plan, op_struct_or_idx, c_ops=None):
            plan.arena.copy_(state)
            if c_ops is None:
                _run(op_struct_or_idx)
            else:
                _run(c_ops, op_struct_or_idx)
            return plan.fwd_ops[i].out.buf.x[:, sl].clone()

        c = out_of(pb, _variant(pb.c_fwd, i, res_a_off=1, res_b_off=1))
        ra = out_of(pb, _variant(pb.c_fwd, i, res_b_off=1)) - c if oa.res_a is not None else torch.zeros_like(c)
        rb = out_of(pb, _variant(pb.c_fwd, i, res_a_off=1)) - c if oa.res_b is not None else torch.zeros_like(c)
        y = out_of(pa, i, pa.c_fwd)
        scale = c.abs().max().item() + 1e-12
        tol = 2e-5 * (scale + ra.abs().max().item() + rb.abs().max().item())
        # alpha (outer DropPath): per sample
        inner = y - rb
        if oa.p_alpha > 0:
            ka = 1.0 - oa.p_alpha
            dropped = inner.abs().amax(dim=(1, 2)) <= tol
            keeps["alpha"].append((float((~dropped).float().mean()), ka, N))
            inner = torch.where(dropped[:, None, None], torch.zeros_like(inner), inner * ka)
            inner = inner - torch.where(dropped[:, None, None], torch.zeros_like(ra), ra)
            alive = ~dropped
        else:
            inner = inner - ra
            alive = torch.ones(N, dtype=torch.bool, device="cuda")
        fc = inner                                 # = pf_n * E * c on the samples alpha kept
        if oa.p_path > 0:
            kp = 1.0 - oa.p_path
            pd = fc.abs().amax(dim=(1, 2)) <= tol
            n_alive = int(alive.sum())
            keeps["path"].append((float((~pd & alive).float().sum() / max(n_alive, 1)), kp, n_alive))
            fc = fc * kp
            alive = alive & ~pd
        big = (c.abs() > 1e-2 * scale) & alive[:, None, None]
        ratio = (fc / torch.where(big, c, torch.ones_like(c)))[big]
        if oa.p_elem > 0:
            ke = 1.0 - oa.p_elem
            is0 = ratio.abs() <= 1e-3
            is1 = (ratio - 1.0 / ke).abs() <= 2e-3 / ke
            assert bool((is0 | is1).all()), (oa.name, "element mask values", ratio[~(is0 | is1)][:5])
            keeps["elem"].append((float(is1.float().mean()), ke, int(ratio.numel())))
        else:
            assert bool(((ratio - 1.0).abs() <= 2e-3).all()), (oa.name, "unit factor", ratio[(ratio - 1).abs() > 2e-3][:5])
        checked += 1
    assert checked >= 15, checked
    for kind, rows in keeps.items():
        assert rows, kind
        for rate, keep, n in rows:
            sigma = math.sqrt(keep * (1 - keep) / max(n, 1))
            assert abs(rate - keep) <= 4.0 * sigma + 2e-4, (kind, rate, keep, n)
        # pooled over all sites of the same nominal rate: tighter
        by = {}
        for rate, keep, n in rows:
            a = by.setdefault(round(keep, 6), [0.0, 0])
            a[0] += rate * n
            a[1] += n
        for keep, (s, n) in by.items():
            assert abs(s / n - keep) <= 4.0 * math.sqrt(keep * (1 - keep) / n) + 2e-4, (kind, keep, s / n, n)


def test_dropout_advances_per_forward_and_follows_manual_seed():
    """ADVICE r1 (high): the autograd/module path must draw NEW masks every training forward; the counter starts from
    torch.manual_seed, is shared by all plans and can be checkpointed / restored."""
    torch.manual_seed(123)
    m = randomize(create_model("seist_s_dpk", in_channels=3, in_samples=1024), 2).cuda().train()
    x = torch.randn(4, 3, 1024, device="cuda")
    with torch.no_grad():
        y0 = m(x)
        s_after_first = m.engine().dropout_seed()
        y1 = m(x)
        assert not torch.equal(y0, y1)                       # new masks each forward
        m.engine().set_dropout_seed(s_after_first - 1)
        y0b = m(x)
        assert torch.equal(y0, y0b)                          # restoring the counter reproduces the step
        y_other_shape = m(x[:2].contiguous())                # a second plan continues the same counter
        assert m.engine().dropout_seed() == s_after_first + 1
    torch.manual_seed(123)
    m2 = randomize(create_model("seist_s_dpk", in_channels=3, in_samples=1024), 2).cuda().train()
    with torch.no_grad():
        assert torch.equal(m2(x), y0)                        # same torch seed -> same first masks
    torch.manual_seed(124)
    m3 = randomize(create_model("seist_s_dpk", in_channels=3, in_samples=1024), 2).cuda().train()
    with torch.no_grad():
        assert not torch.equal(m3(x), y0)
    assert torch.isfinite(y_other_shape).all()


# ------------------------------------------------------------------------------------------------
# SyncBatchNorm data parallelism on one GPU ("virtual world 2")
# ------------------------------------------------------------------------------------------------
def _extra_lanes(plan):
    """one stream for every lane of the plan's schedule after the first (the caller supplies lane 0)"""
    return [torch.cuda.Stream() for _ in range(plan.n_main)]


def _run_segments_lockstep(plans, which, reduce_slices):
    """Issue segment j of every rank's plan, then segment j + 1, ...  Every rank runs its lane schedule from the current
    stream on lanes of its own; `reduce_slices` sums the statistics on the current stream before a segment needs them."""
    s = torch.cuda.current_stream().cuda_stream
    extra = [_extra_lanes(p) for p in plans]
    segs = [getattr(p, which + "_segments") for p in plans]
    assert all(len(sg) == len(segs[0]) for sg in segs)
    for j in range(len(segs[0])):
        start, end, sync = segs[0][j]
        if sync:
            reduce_slices(sync)
        for p, ex in zip(plans, extra):
            c_ops = p.c_fwd if which == "fwd" else p.c_bwd
            run_segment(c_ops, start, end, [s] + [e.cuda_stream for e in ex])
    torch.cuda.synchronize()


def test_virtual_world2_syncbn_equals_single_rank():
    name, L, NB = "seist_s_dpk", 2048, 8
    base = randomize(create_model(name, in_channels=3, in_samples=L), seed=5)
    base.set_drop_rates(**ZERO_DROPS)
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    x, t = R.synth_waveforms(NB, L, seed=3)
    x, t = x.cuda(), t.cuda()
    w = torch.tensor([0.5, 1.0, 1.0], device="cuda")
    lib = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream

    def make(N, world):
        m = create_model(name, in_channels=3, in_samples=L)
        m.load_state_dict(sd)
        m.set_drop_rates(**ZERO_DROPS)
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m).cuda().train()
        flat = P.FlatState(m, torch.device("cuda"))
        return m, P.finalize(P.PlanBuilder(m, flat, N, L, True, world=world).build(), True)

    def loss_bwd(plan, tgt, total_elems):
        """BCE over the GLOBAL batch: d loss / d y of the mean over all ranks' elements."""
        y = plan.y_out.x
        N, C, Ls = y.shape
        gout = torch.full((1,), float(N * C * Ls) / total_elems, device="cuda")
        _lib.check(lib.seist_bce_bwd(y.data_ptr(), tgt.data_ptr(), w.data_ptr(), gout.data_ptr(), N, C, Ls, 1e-6,
                                     plan.y_out.dxd.data_ptr(), s))

    # one rank, whole batch
    m1, p1 = make(NB, 1)
    p1.x_in.x.copy_(x)
    p1.stat.zero_()
    _run_segments_lockstep([p1], "fwd", lambda sync: None)
    loss_bwd(p1, t, NB * 3 * L)
    p1.flat.G.zero_(); p1.gstat.zero_(); p1.dWx.zero_()
    _run_segments_lockstep([p1], "bwd", lambda sync: None)

    # two virtual ranks, half batches, statistics summed at the plan's sync points
    ranks = [make(NB // 2, 2) for _ in range(2)]
    plans = [p for _, p in ranks]
    assert any(seg[2] for seg in plans[0].fwd_segments), "world-2 plan has no sync points"
    for r, p in enumerate(plans):
        p.x_in.x.copy_(x[r * NB // 2:(r + 1) * NB // 2])
        p.stat.zero_()

    def reducer(attr):
        def red(sync):
            for b in sync:
                e = plans[0].bns[b]
                sl = slice(e.st_off, e.st_off + 2 * e.C)
                tot = getattr(plans[0], attr)[sl] + getattr(plans[1], attr)[sl]
                for p in plans:
                    getattr(p, attr)[sl] = tot
        return red

    _run_segments_lockstep(plans, "fwd", reducer("stat"))
    for r, p in enumerate(plans):
        loss_bwd(p, t[r * NB // 2:(r + 1) * NB // 2].contiguous(), NB * 3 * L)
        p.flat.G.zero_(); p.gstat.zero_(); p.dWx.zero_()
    _run_segments_lockstep(plans, "bwd", reducer("gstat"))

    y2 = torch.cat([p.y_out.x for p in plans])
    assert (y2 - p1.y_out.x).abs().max().item() <= 2e-5 * p1.y_out.x.abs().max().item()
    # weight gradients: each rank holds the gradient of ITS samples of the global-mean loss; BN affine gradients carry
    # grad_scale = 1/world (they are computed from the already-reduced sums on every rank) -> the rank SUM is the gradient
    G2 = plans[0].flat.G + plans[1].flat.G
    G1 = p1.flat.G
    assert (G2 - G1).abs().max().item() <= 3e-4 * G1.abs().max().item(), (G2 - G1).abs().max().item()
    for p in plans:
        assert (p.flat.RB - p1.flat.RB).abs().max().item() <= 1e-5 * (p1.flat.RB.abs().max().item() + 1e-3)


# ------------------------------------------------------------------------------------------------
# train-mode parity at the benchmark length
# ------------------------------------------------------------------------------------------------
def _train_parity(name, N, L, seed, out_tol=1e-3):
    m = randomize(create_model(name, in_channels=3, in_samples=L), seed=seed)
    m.set_drop_rates(**ZERO_DROPS)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    x, tgt = R.synth_waveforms(N, L, seed=seed + 10)
    sd_g = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point and "running" not in k else v.clone())
            for k, v in sd.items()}
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, 32)))
    y_ref, _ = R.forward(sd_g, x, R.spec_for(name), training=True)
    loss_ref = R.bce_loss(y_ref, tgt)
    loss_ref.backward()
    m = m.cuda().train()
    y = m(x.cuda())
    err = (y.detach().cpu() - y_ref.detach()).abs().max().item()
    assert err <= out_tol * y_ref.abs().max().item(), err
    loss = BCELoss(weight=[[0.5], [1], [1]])(y, tgt.cuda())
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= 1e-4 * abs(loss_ref.item())
    gmax = max(sd_g[k].grad.abs().max().item() for k, _ in m.named_parameters())
    bad = []
    for k, p in m.named_parameters():
        ref = sd_g[k].grad
        e = (p.grad.cpu() - ref).abs().max().item()
        if e > 2e-3 * ref.abs().max().item() + 1e-5 * gmax:
            bad.append((k, e, ref.abs().max().item()))
    assert not bad, bad[:8]


def test_m_dpk_train_parity_b16_l8192():
    _train_parity("seist_m_dpk", 16, 8192, seed=7)


def test_l_dpk_train_parity_l8192():
    _train_parity("seist_l_dpk", 4, 8192, seed=9)


# ------------------------------------------------------------------------------------------------
# the reference's own step under its defaults: torch.optim.Adam + torch.compile + DDP(world 1) + SyncBN
# ------------------------------------------------------------------------------------------------
def test_reference_step_order_with_torch_adam_compile_and_ddp():
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel
    name, N, L = "seist_s_dpk", 4, 2048
    base = randomize(create_model(name, in_channels=3, in_samples=L), seed=11)
    base.set_drop_rates(**ZERO_DROPS)
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    x, tgt = R.synth_waveforms(N, L, seed=21)
    # oracle: forward, loss, backward, one torch Adam step on the reference restatement
    sd_g = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point and "running" not in k else v.clone())
            for k, v in sd.items()}
    y_ref, _ = R.forward(sd_g, x, R.spec_for(name), training=True)
    loss_ref = R.bce_loss(y_ref, tgt)
    loss_ref.backward()
    names = [k for k, _ in base.named_parameters()]
    own_pg = not dist.is_initialized()
    if own_pg:
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1,
                                device_id=torch.device("cuda", 0))
    try:
        model = create_model(name, in_channels=3, in_samples=L)
        model.load_state_dict(sd)
        model.set_drop_rates(**ZERO_DROPS)
        model = torch.compile(model)                                   # train.py:296-297 (default True)
        model = model.cuda()
        optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)      # train.py:304-308
        model = DistributedDataParallel(model, device_ids=[0])         # train.py:369-373
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)   # train.py:374
        loss_fn = BCELoss(weight=[[0.5], [1], [1]]).cuda()
        model.train()
        outputs = model(x.cuda())                                      # train.py:87
        loss = loss_fn(outputs, tgt.cuda())                            # train.py:98
        optimizer.zero_grad()                                          # train.py:109
        loss.backward()                                                # train.py:110
        optimizer.step()                                               # train.py:111
        torch.cuda.synchronize()
        assert (outputs.detach().cpu() - y_ref.detach()).abs().max().item() <= 1e-3 * y_ref.abs().max().item()
        assert abs(loss.item() - loss_ref.item()) <= 1e-4 * abs(loss_ref.item())
        inner = model.module
        inner = getattr(inner, "_orig_mod", inner)
        got = dict(inner.named_parameters())
        gmax = max(sd_g[k].grad.abs().max().item() for k in names)
        for k in names:                      # DDP's reducer saw autograd-produced gradients for every parameter
            assert got[k].grad is not None, k
            ref = sd_g[k].grad
            e = (got[k].grad.cpu() - ref).abs().max().item()
            assert e <= 2e-3 * ref.abs().max().item() + 1e-5 * gmax, (k, e)
        moved = max((got[k].detach().cpu() - sd[k]).abs().max().item() for k in names)
        assert 0.5e-3 <= moved <= 1.5e-3, moved          # torch Adam's first step is ~lr per element
        # the in-place optimizer update is what the next forward runs on
        sd2 = {k: v.detach().cpu().clone() for k, v in inner.state_dict().items()}
        y2_ref, _ = R.forward(sd2, x, R.spec_for(name), training=True)
        with torch.no_grad():
            y2 = model(x.cuda())
        assert (y2.cpu() - y2_ref).abs().max().item() <= 1e-3 * y2_ref.abs().max().item()
    finally:
        if own_pg:
            dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------
# Trainer: optimizer-state checkpoint round trip, torch.optim.Adam-compatible layout
# ------------------------------------------------------------------------------------------------
def test_trainer_state_dict_roundtrip_and_torch_layout():
    import copy
    from seist_b200.train import Trainer, make_cyclic_lr
    name, N, L = "seist_s_dpk", 4, 1024
    m = randomize(create_model(name, in_channels=3, in_samples=L), seed=3)
    m2 = copy.deepcopy(m)
    x, tgt = R.synth_waveforms(N, L, seed=2)
    x, tgt = x.cuda(), tgt.cuda()
    sched = make_cyclic_lr(1000)
    ta = Trainer(m, lr_schedule=sched)
    for _ in range(2):
        ta.step(x, tgt)
    sd_opt = ta.state_dict()
    sd_model = {k: v.clone() for k, v in m.state_dict().items()}
    la = [float(ta.step(x, tgt)) for _ in range(2)]
    # resume in a fresh trainer / model
    m2.load_state_dict(sd_model)
    tb = Trainer(m2, lr_schedule=sched)
    tb._setup(x, tgt)
    tb.load_state_dict(sd_opt)
    lb = [float(tb.step(x, tgt)) for _ in range(2)]
    assert all(abs(a - b) <= 2e-4 * abs(a) for a, b in zip(la, lb)), (la, lb)
    # the dict loads into a real torch.optim.Adam over the same parameters
    opt = torch.optim.Adam(m2.parameters(), lr=1e-3)
    plain = {"state": sd_opt["state"], "param_groups": sd_opt["param_groups"]}
    opt.load_state_dict(plain)
    assert len(opt.state) == len(list(m2.parameters()))
    # reference schedule: gamma = base_lr ** (1 / (2 * steps)) (training/train.py:343-354) against torch's CyclicLR
    dummy = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=8e-5)
    ref = torch.optim.lr_scheduler.CyclicLR(dummy, base_lr=8e-5, max_lr=1e-3, step_size_up=2000, step_size_down=3000,
                                            mode="exp_range", gamma=8e-5 ** (1 / 2000), cycle_momentum=False)
    for it in range(0, 40):
        assert abs(sched(it) - ref.get_last_lr()[0]) <= 1e-12 + 1e-9 * ref.get_last_lr()[0], it
        dummy.step()
        ref.step()


# ------------------------------------------------------------------------------------------------
# the fused peer-memory exchange (csrc/comm.cu) with two virtual ranks in ONE process on ONE GPU: each rank's blob is an
# ordinary device buffer and the "peer pointers" are the other rank's buffer; the two ranks run on two streams fed by two
# host threads (the exchange kernels spin until the peer arrives), exactly the kernels a multi-GPU run executes
# ------------------------------------------------------------------------------------------------
def test_fused_peer_exchange_two_virtual_ranks_equal_single_rank():
    from seist_b200.comm import PeerComm
    name, L, NB, W = "seist_s_dpk", 2048, 8, 2
    base = randomize(create_model(name, in_channels=3, in_samples=L), seed=5)
    base.set_drop_rates(**ZERO_DROPS)
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    x, t = R.synth_waveforms(NB, L, seed=3)
    x, t = x.cuda(), t.cuda()
    w = torch.tensor([0.5, 1.0, 1.0], device="cuda")
    lib = _lib.lib()
    dev = torch.device("cuda", 0)

    def model_and_flat():
        m = create_model(name, in_channels=3, in_samples=L)
        m.load_state_dict(sd)
        m.set_drop_rates(**ZERO_DROPS)
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m).cuda().train()
        return m, P.FlatState(m, dev)

    # reference: one rank, whole batch
    m1, f1 = model_and_flat()
    p1 = P.finalize(P.PlanBuilder(m1, f1, NB, L, True, world=1).build(), True)
    s0 = torch.cuda.current_stream().cuda_stream
    p1.x_in.x.copy_(x)
    p1.stat_acc.zero_()
    _run_segments_lockstep([p1], "fwd", lambda sync: None)
    y = p1.y_out.x
    gout = torch.ones(1, device="cuda")
    _lib.check(lib.seist_bce_bwd(y.data_ptr(), t.data_ptr(), w.data_ptr(), gout.data_ptr(), NB, 3, L, 1e-6, p1.y_out.dxd.data_ptr(), s0))
    f1.G.zero_(); p1.gstat_acc.zero_(); p1.dWx.zero_()
    _run_segments_lockstep([p1], "bwd", lambda sync: None)

    # two virtual ranks
    ranks = [model_and_flat() for _ in range(W)]
    n_stat = sum(2 * mod.num_features for mod in ranks[0][0].modules() if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm))
    blobs, comms = [], []
    # size of the blob: ask a throw-away layout computation
    from seist_b200.comm import _align
    nbytes = _align(8 * n_stat) * 2 + _align(4 * ranks[0][1].numel) + _align(4 * _lib.SIG_LANES * _lib.MAX_WORLD)
    for r in range(W):
        blobs.append(torch.zeros(nbytes, dtype=torch.uint8, device=dev))
    bases = [b.data_ptr() for b in blobs]
    for r in range(W):
        comms.append(PeerComm(dev, W, r, n_stat, ranks[r][1].numel, blob=blobs[r], peer_bases=bases))
        ranks[r][1].G = comms[r].grad
    plans = [P.finalize(P.PlanBuilder(m, f, NB // W, L, True, world=W).build(), True, comm=comms[r])
             for r, (m, f) in enumerate(ranks)]
    assert any(op.kind == _lib.BN_PREPARE_FWD and op.sync_bn for op in plans[0].fwd_ops)
    streams = [torch.cuda.Stream() for _ in range(W)]
    extra = [_extra_lanes(p) for p in plans]
    n = NB // W
    gos = [torch.ones(1, device="cuda") for _ in range(W)]
    tts = [t[r * n:(r + 1) * n].contiguous() for r in range(W)]
    torch.cuda.synchronize()

    # one host thread feeds both ranks' streams, phase by phase (a phase is a few hundred asynchronous launches per rank;
    # rank 0's stream waits inside its first exchange kernel until rank 1's stream gets there a few milliseconds later)
    def phase(fn):
        for r in range(W):
            with torch.cuda.stream(streams[r]):
                fn(r, plans[r], comms[r], ranks[r][1], streams[r].cuda_stream)
        for st in streams:
            st.synchronize()

    def issue(r, pl, which, s):
        """rank r's plan by its lane schedule: lane 0 on the rank's stream, the other lanes on streams of its own"""
        c_ops = pl.c_fwd if which == "fwd" else pl.c_bwd
        for start, end, sync in getattr(pl, which + "_segments"):
            assert not sync          # the statistic exchange is inside the BN_PREPARE kernels
            run_segment(c_ops, start, end, [s] + [e.cuda_stream for e in extra[r]])

    def p_fwd(r, pl, cm, fl, s):
        pl.x_in.x.copy_(x[r * n:(r + 1) * n])
        cm.barrier(stream=s)
        pl.stat_acc.zero_()
        issue(r, pl, "fwd", s)

    def p_bwd(r, pl, cm, fl, s):
        yy = pl.y_out.x        # local-mean loss, like every rank of the real job (1/world is applied to the reduced sum)
        _lib.check(lib.seist_bce_bwd(yy.data_ptr(), tts[r].data_ptr(), w.data_ptr(), gos[r].data_ptr(), n, 3, L, 1e-6,
                                     pl.y_out.dxd.data_ptr(), s))
        fl.G.zero_(); pl.gstat_acc.zero_(); pl.dWx.zero_()
        issue(r, pl, "bwd", s)

    def p_red(r, pl, cm, fl, s):
        cm.allreduce_grads(stream=s)

    phase(p_fwd)
    phase(p_bwd)
    phase(p_red)
    torch.cuda.synchronize()
    assert not any(c.timed_out() for c in comms), "a peer wait timed out"
    y2 = torch.cat([p.y_out.x for p in plans])
    assert (y2 - p1.y_out.x).abs().max().item() <= 2e-5 * p1.y_out.x.abs().max().item()
    # every rank holds the same all-reduced gradient sum; / world = gradient of the global-mean loss
    G1 = f1.G
    for c in comms:
        assert torch.equal(c.grad_red, comms[0].grad_red)           # fixed summation order: bit-identical on all ranks
    G2 = comms[0].grad_red / W
    assert (G2 - G1).abs().max().item() <= 3e-4 * G1.abs().max().item(), (G2 - G1).abs().max().item()
    for p in plans:
        assert (p.flat.RB - p1.flat.RB).abs().max().item() <= 1e-5 * (p1.flat.RB.abs().max().item() + 1e-3)
        assert torch.equal(p.stat, plans[0].stat) and torch.equal(p.gstat, plans[0].gstat)


# ------------------------------------------------------------------------------------------------
# several consecutive steps: the fused step (graph replay: seed advance, forward, BCE, backward, Adam, CyclicLR) against
# the oracle restatement driven by torch.optim.Adam + torch's CyclicLR in the reference's step order (train.py:87-116)
# ------------------------------------------------------------------------------------------------
def test_five_step_trajectory_matches_oracle():
    from seist_b200.train import Trainer, make_cyclic_lr
    name, N, L, steps = "seist_s_dpk", 4, 2048, 5
    base = randomize(create_model(name, in_channels=3, in_samples=L), seed=13)
    base.set_drop_rates(**ZERO_DROPS)
    sd0 = {k: v.clone() for k, v in base.state_dict().items()}
    x, tgt = R.synth_waveforms(N, L, seed=31)
    # oracle trajectory
    sd = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point and "running" not in k else v.clone())
          for k, v in sd0.items()}
    params = [v for v in sd.values() if v.requires_grad]
    opt = torch.optim.Adam(params, lr=8e-5)
    sched = torch.optim.lr_scheduler.CyclicLR(opt, base_lr=8e-5, max_lr=1e-3, step_size_up=2000, step_size_down=3000,
                                              mode="exp_range", gamma=8e-5 ** (1 / 2000), cycle_momentum=False)
    ref_losses = []
    for _ in range(steps):
        y, bufs = R.forward(sd, x, R.spec_for(name), training=True)
        loss = R.bce_loss(y, tgt)
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
        for k, b in bufs.items():
            sd[k] = b
        ref_losses.append(loss.item())
    # fused trajectory
    m = create_model(name, in_channels=3, in_samples=L)
    m.load_state_dict(sd0)
    m.set_drop_rates(**ZERO_DROPS)
    m.cuda()
    tr = Trainer(m, lr_schedule=make_cyclic_lr(1000))
    got = [float(tr.step(x.cuda(), tgt.cuda())) for _ in range(steps)]
    for a, b in zip(got, ref_losses):
        assert abs(a - b) <= 2e-3 * abs(b), (got, ref_losses)
    assert got[-1] != got[0]
    # BatchNorm running statistics after 5 steps (momentum accumulation) and the parameters themselves
    sdm = m.state_dict()
    for k, v in sd.items():
        if "running_" in k:
            assert (sdm[k].cpu() - v).abs().max().item() <= 2e-3 * (v.abs().max().item() + 1e-3), k
        if k.endswith("num_batches_tracked"):
            assert int(sdm[k]) == int(v) == steps
