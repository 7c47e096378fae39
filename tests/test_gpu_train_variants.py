"""-m gpu: the fused training step beyond dpk + Adam: the polarity models' cross-entropy, the fused SGD
(`seist_sgd_step`) and the triangular CyclicLR modes, against `torch.optim` and the oracle restatement driven in the
reference's step order (training/train.py:87-116), plus SGD checkpoints and the step's host-sync budget."""
import copy

import pytest
import torch

from harness import ZERO_DROPS, randomize
from oracle import golden as G
from oracle import seist_ref as R
from seist_b200 import _lib
from seist_b200.models import CELoss, create_model
from seist_b200.train import Trainer, make_cyclic_lr
from test_gpu_gaps import _syncs

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# the SGD kernel against torch.optim.SGD
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("momentum,wd,dampening,nesterov,gscale", [
    (0.0, 0.0, 0.0, False, 1.0), (0.0, 1e-2, 0.0, False, 0.5), (0.9, 0.0, 0.0, False, 1.0), (0.9, 1e-2, 0.0, False, 0.5),
    (0.9, 0.0, 0.0, True, 0.5), (0.9, 1e-2, 0.0, True, 1.0), (0.9, 1e-2, 0.1, False, 1.0), (0.9, 0.0, 0.1, False, 0.5)])
def test_fused_sgd_matches_torch(momentum, wd, dampening, nesterov, gscale):
    torch.manual_seed(0)
    n = 100003
    p0 = torch.randn(n, device="cuda")
    grads = [torch.randn(n, device="cuda") * (0.1 + i) for i in range(3)]
    lr = 1e-2
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([ref], lr=lr, momentum=momentum, dampening=dampening, weight_decay=wd, nesterov=nesterov)
    p = p0.clone()
    buf = torch.full_like(p, float("nan")) if momentum != 0 else None     # the first step must not read it
    lr_t, step_t = torch.full((1,), lr, device="cuda"), torch.zeros(1, device="cuda")
    lib = _lib.lib()
    s = torch.cuda.current_stream().cuda_stream
    for i, g in enumerate(grads):
        ref.grad = (g * gscale).clone()          # grad_scale = 1/world: the kernel scales the all-reduced sum itself
        opt.step()
        step_t += 1
        _lib.check(lib.seist_sgd_step(p.data_ptr(), g.data_ptr(), None if buf is None else buf.data_ptr(), n,
                                      lr_t.data_ptr(), step_t.data_ptr(), momentum, dampening, wd,
                                      1 if nesterov else 0, gscale, s))
        torch.cuda.synchronize()
        upd_ref = (ref.detach() - p0).abs().max().item()
        err = (p - ref.detach()).abs().max().item()
        assert err <= 1e-6, (i, err, upd_ref)
        assert upd_ref > 0.1 * lr * gscale
    if momentum != 0:
        b = opt.state[ref]["momentum_buffer"]
        assert (buf - b).abs().max().item() <= 1e-6 * b.abs().max().item()
    else:
        assert "momentum_buffer" not in opt.state[ref]


def test_fused_sgd_rejects_bad_arguments():
    lib = _lib.lib()
    p = torch.zeros(8, device="cuda")
    one = torch.ones(1, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert lib.seist_sgd_step(p.data_ptr(), p.data_ptr(), None, 8, one.data_ptr(), one.data_ptr(), 0.9, 0.0, 0.0, 0, 1.0, s) != 0
    assert lib.seist_sgd_step(p.data_ptr(), p.data_ptr(), p.data_ptr(), 8, one.data_ptr(), one.data_ptr(), 0.9, 0.1, 0.0, 1,
                              1.0, s) != 0
    assert lib.seist_sgd_step(p.data_ptr(), p.data_ptr(), None, 0, one.data_ptr(), one.data_ptr(), 0.0, 0.0, 0.0, 0, 1.0, s) != 0


# ------------------------------------------------------------------------------------------------
# the polarity model's fused step against the golden fixture of the unmodified reference
# ------------------------------------------------------------------------------------------------
def test_pmp_trainer_step_matches_reference_golden():
    g = G.load("seist_s_pmp")
    m = create_model("seist_s_pmp", in_channels=3, in_samples=g["length"])
    m.load_state_dict(g["state_dict"], strict=True)
    m.set_drop_rates(**ZERO_DROPS)
    m.cuda()
    tr = Trainer(m)
    onehot = g["target"].long()                         # the reference's labels: int64 rows of np.eye(2)
    loss = float(tr.step(g["x"].cuda(), onehot.cuda()))
    assert isinstance(tr.loss_fn, CELoss)
    assert torch.equal(tr.loss_fn.weight, torch.tensor([1.0, 1.0]))
    assert abs(loss - g["loss"].item()) <= 1e-4 * abs(g["loss"].item())
    flat = tr.flat
    got = {name: tr.last_grads[flat.pref[name].off:flat.pref[name].off + flat.pref[name].numel].view(flat.pref[name].shape)
           for name, _ in tr.eng._named}
    gmax = max(v.absmax for v in g["grads"].values())
    bad = [(k, ref.err(got[k]), ref.absmax) for k, ref in g["grads"].items()
           if ref.err(got[k]) > 2e-3 * ref.absmax + 1e-5 * gmax]
    assert not bad, bad[:10]
    sd = m.state_dict()
    for k, b in g["buffers_after"].items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(b.val[0]), k
        else:
            assert b.err(sd[k]) <= 1e-3 * (b.absmax + 1e-3), k


# ------------------------------------------------------------------------------------------------
# five-step trajectories against the oracle stepped by torch.optim and torch's CyclicLR
# ------------------------------------------------------------------------------------------------
def _ce_ref(preds, targets, eps=1e-6):
    """CELoss(weight=[1, 1]) of the reference (models/loss.py:8-29, config.py:147-155)."""
    return (-targets * torch.log(preds + eps) * torch.tensor([1.0, 1.0])).sum(1).mean()


def _trajectory(name, N, L, seed, make_opt, mode, up, down, max_lr, steps=5, **trainer_kw):
    base = randomize(create_model(name, in_channels=3, in_samples=L), seed=seed)
    base.set_drop_rates(**ZERO_DROPS)
    sd0 = {k: v.clone() for k, v in base.state_dict().items()}
    x, tgt = R.synth_waveforms(N, L, seed=seed + 18)
    if name.endswith("pmp"):
        cls = torch.randint(0, 2, (N,), generator=torch.Generator().manual_seed(seed))
        tgt = torch.eye(2, dtype=torch.int64)[cls]
        loss_ref_fn = _ce_ref
    else:
        loss_ref_fn = R.bce_loss
    base_lr, total = 8e-5, 1000
    sd = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point and "running" not in k else v.clone())
          for k, v in sd0.items()}
    params = [v for v in sd.values() if v.requires_grad]
    opt = make_opt([{"params": params, "initial_lr": base_lr}], base_lr)
    sched = torch.optim.lr_scheduler.CyclicLR(opt, base_lr=base_lr, max_lr=max_lr, step_size_up=up, step_size_down=down,
                                              mode=mode, gamma=base_lr ** (1 / (2 * total)), cycle_momentum=False)
    ref_losses = []
    for _ in range(steps):
        y, bufs = R.forward(sd, x, R.spec_for(name), training=True)
        loss = loss_ref_fn(y, tgt.float())
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
        for k, b in bufs.items():
            sd[k] = b
        ref_losses.append(loss.item())
    m = create_model(name, in_channels=3, in_samples=L)
    m.load_state_dict(sd0)
    m.set_drop_rates(**ZERO_DROPS)
    m.cuda()
    tr = Trainer(m, lr=base_lr, lr_schedule=make_cyclic_lr(total, base_lr, max_lr, up, down, mode), **trainer_kw)
    got = [float(tr.step(x.cuda(), tgt.cuda())) for _ in range(steps)]
    for a, b in zip(got, ref_losses):
        assert abs(a - b) <= 2e-3 * abs(b), (got, ref_losses)
    assert got[-1] != got[0]
    sdm = m.state_dict()
    diff = upd = 0.0
    for k, v in sd.items():
        if "running_" in k:
            assert (sdm[k].cpu() - v).abs().max().item() <= 2e-3 * (v.abs().max().item() + 1e-3), k
        if k.endswith("num_batches_tracked"):
            assert int(sdm[k]) == int(v) == steps
        if v.requires_grad:
            diff += (sdm[k].cpu() - v.detach()).double().square().sum().item()
            upd += (v.detach() - sd0[k]).double().square().sum().item()
    return (diff / upd) ** 0.5


def test_five_step_pmp_adam_exp_range_matches_oracle():
    # Adam moves every element by about lr whatever its gradient's size, so the sign of a gradient that is small next to
    # its tensor's rounding error decides a +-lr step: the peak lr is kept near the reference's first steps (8e-5 there)
    # and the parameters are held to an L2 bound on their difference over their update (3.5e-2 measured on an H100)
    rel = _trajectory("seist_s_pmp", 8, 2048, 41, lambda g, lr: torch.optim.Adam(g, lr=lr), "exp_range", 2, 2, 2e-4)
    assert rel <= 1e-1, rel


def test_five_step_dpk_sgd_triangular2_matches_oracle():
    rel = _trajectory("seist_s_dpk", 4, 2048, 43,
                      lambda g, lr: torch.optim.SGD(g, lr=lr, momentum=0.9, weight_decay=1e-4), "triangular2", 1, 2, 1e-3,
                      optimizer="sgd", momentum=0.9, weight_decay=1e-4)
    assert rel <= 1e-3, rel                  # SGD's update is linear in the gradient: 5e-5 measured on an H100


# ------------------------------------------------------------------------------------------------
# SGD checkpoints, graph replay and the host-sync budget
# ------------------------------------------------------------------------------------------------
def _sgd_setup(seed=3):
    name, N, L = "seist_s_dpk", 4, 1024
    m = randomize(create_model(name, in_channels=3, in_samples=L), seed=seed)
    m.set_drop_rates(**ZERO_DROPS)
    x, tgt = R.synth_waveforms(N, L, seed=2)
    return m, x.cuda(), tgt.cuda()


SGD_KW = dict(optimizer="sgd", lr=2e-3, momentum=0.9, weight_decay=1e-4,
              lr_schedule=make_cyclic_lr(1000, 2e-3, 1e-2, 2, 3, "triangular"))


def _close(a, b):
    return all(abs(u - v) <= 2e-4 * abs(u) for u, v in zip(a, b))


def test_sgd_checkpoint_resume_and_torch_layout():
    m, x, tgt = _sgd_setup()
    m_fresh = copy.deepcopy(m)
    ta = Trainer(m, **SGD_KW)
    for _ in range(2):
        ta.step(x, tgt)
    sd_opt = ta.state_dict()
    sd_model = {k: v.clone() for k, v in m.state_dict().items()}
    la = [float(ta.step(x, tgt)) for _ in range(3)]
    assert la[2] != la[0]
    g0 = sd_opt["param_groups"][0]
    assert (g0["momentum"], g0["dampening"], g0["weight_decay"], g0["nesterov"]) == (0.9, 0.0, 1e-4, False)
    assert sd_opt["seist_b200"]["it"] == 2 and len(sd_opt["state"]) == len(list(m.parameters()))

    # the dict loads into a real torch.optim.SGD over the same parameters, and torch's own dict loads back
    mb = copy.deepcopy(m_fresh)
    mb.load_state_dict(sd_model)
    opt = torch.optim.SGD(mb.parameters(), lr=1e-3)
    opt.load_state_dict({"state": sd_opt["state"], "param_groups": sd_opt["param_groups"]})
    assert len(opt.state) == len(list(mb.parameters()))
    assert opt.param_groups[0]["momentum"] == 0.9
    plain = opt.state_dict()
    for i, (k, _) in enumerate(m.named_parameters()):
        assert torch.equal(plain["state"][i]["momentum_buffer"].cpu(), sd_opt["state"][i]["momentum_buffer"].cpu()), k

    # resumed from the trainer's own dict, and from torch's (the schedule position comes from the caller there)
    lb = []
    for src in (sd_opt, plain):
        mr = copy.deepcopy(m_fresh)
        mr.load_state_dict(sd_model)
        tb = Trainer(mr, optimizer="sgd", lr_schedule=SGD_KW["lr_schedule"])       # momentum / decay come from the dict
        tb._setup(x, tgt)
        tb.load_state_dict(src)
        if src is plain:
            tb.it = 2
        assert tb.momentum == 0.9 and tb.weight_decay == 1e-4
        lb.append([float(tb.step(x, tgt)) for _ in range(3)])
    assert _close(la, lb[0]) and _close(la, lb[1]), (la, lb)

    # a dict without momentum buffers is a fresh optimizer: the next step initialises them
    mc, md = copy.deepcopy(m_fresh), copy.deepcopy(m_fresh)
    tc = Trainer(mc, **SGD_KW)
    for _ in range(2):
        tc.step(x, tgt)
    mc.load_state_dict(md.state_dict())
    tc.load_state_dict(torch.optim.SGD(mc.parameters(), lr=2e-3, momentum=0.9, weight_decay=1e-4).state_dict())
    tc.it = 0
    assert tc.state_dict()["state"] == {}
    td = Trainer(md, **SGD_KW)
    lc = [float(tc.step(x, tgt)) for _ in range(3)]
    ld = [float(td.step(x, tgt)) for _ in range(3)]
    assert _close(ld, lc), (ld, lc)


def test_sgd_graph_equals_eager():
    m, x, tgt = _sgd_setup(seed=5)
    m2 = copy.deepcopy(m)
    kw = dict(SGD_KW, nesterov=True)
    ta, tb = Trainer(m, **kw), Trainer(m2, use_graph=False, **kw)
    la = [float(ta.step(x, tgt)) for _ in range(4)]
    lb = [float(tb.step(x, tgt)) for _ in range(4)]
    assert ta.graph is not None and tb.graph is None
    assert _close(la, lb) and la[3] != la[0], (la, lb)


@pytest.mark.parametrize("name,kw", [("seist_s_pmp", {}), ("seist_s_dpk", SGD_KW)])
def test_graph_replay_does_not_synchronise(name, kw):
    L, N = 1024, 4
    m = randomize(create_model(name, in_channels=3, in_samples=L), seed=7).cuda()
    x, tgt = R.synth_waveforms(N, L, seed=9)
    if name.endswith("pmp"):
        tgt = torch.eye(2, dtype=torch.int64)[torch.arange(N) % 2]
    x, tgt = x.cuda(), tgt.cuda()
    tr = Trainer(m, **kw)
    tr.step(x, tgt)
    tr.step(x, tgt)                        # warm-up and capture
    assert tr.graph is not None
    losses = []
    for _ in range(3):
        loss, n = _syncs(lambda: tr.step(x, tgt))
        assert n == 0
        losses.append(loss)
    assert all(torch.isfinite(v) for v in losses)
