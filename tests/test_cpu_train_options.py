"""The host side of the fused training step's options: the CyclicLR modes, the --warmup-steps / --down-steps rules,
`Trainer.from_args` against what the reference's `train_worker` builds (training/train.py:250-354) from the defaults of
its `main.py`, and the default loss of every registered variant against `Config.get_loss`.  No GPU is needed."""
import argparse
import math

import pytest
import torch

from seist_b200.config import Config
from seist_b200.models import BCELoss, CELoss, HuberLoss, create_model, get_model_list
from seist_b200.train import Trainer, cyclic_lr, cyclic_steps, default_loss, make_cyclic_lr, trainer_args


def _reference_args(**changes):
    """The training arguments of the reference's main.py with their defaults."""
    a = argparse.Namespace(model_name="seist_m_dpk", epochs=200, steps=0, start_epoch=0, optim="Adam", momentum=0.9,
                           weight_decay=0.0, use_lr_scheduler=True, lr_scheduler_mode="exp_range", base_lr=8e-5,
                           max_lr=1e-3, warmup_steps=2000, down_steps=3000)
    for k, v in changes.items():
        setattr(a, k, v)
    return a


def _reference_build(args, steps_per_epoch):
    """train_worker's optimizer and scheduler over one dummy parameter (training/train.py:250-354), restated."""
    if args.steps > 0:
        args.epochs = math.ceil(args.steps / steps_per_epoch)
    args.steps = args.epochs * steps_per_epoch
    p = torch.nn.Parameter(torch.zeros(1))
    groups = [{"params": [p], "initial_lr": args.base_lr}]
    name = args.optim.lower()
    if name == "adam":
        opt = torch.optim.Adam(groups, lr=args.base_lr, weight_decay=args.weight_decay)
    elif name == "adamw":
        opt = torch.optim.AdamW(groups, lr=args.base_lr, weight_decay=args.weight_decay)
    elif name == "sgd":
        opt = torch.optim.SGD(groups, lr=args.base_lr, momentum=args.momentum, weight_decay=args.weight_decay)
    else:
        raise ValueError(f"Unsupported optimizer:'{args.optim}'")
    sched = None
    if args.use_lr_scheduler:
        if args.warmup_steps < 1:
            args.warmup_steps = int(args.steps * args.warmup_steps) if args.warmup_steps > 0 else 1
        if args.down_steps < 1:
            args.down_steps = int(args.steps * args.down_steps) if args.down_steps > 0 else args.steps - args.warmup_steps
        sched = torch.optim.lr_scheduler.CyclicLR(
            optimizer=opt, base_lr=args.base_lr, max_lr=args.max_lr, step_size_up=args.warmup_steps,
            step_size_down=args.down_steps, mode=args.lr_scheduler_mode, gamma=args.base_lr ** ((args.steps * 2) ** -1),
            cycle_momentum=False, last_epoch=args.start_epoch * steps_per_epoch - 1)
    return opt, sched


def _same_schedule(fn, start, sched, n):
    """fn(it) for it = start, start + 1, ... against the lr torch's scheduler gives each of the next n steps."""
    for k in range(n):
        want = sched.get_last_lr()[0]
        got = fn(start + k)
        assert abs(got - want) <= 1e-15 + 1e-12 * abs(want), (start + k, got, want)
        sched.optimizer.step()
        sched.step()


@pytest.mark.parametrize("mode", ["triangular", "triangular2", "exp_range"])
@pytest.mark.parametrize("start", [0, 1, 23])
def test_cyclic_lr_modes_equal_torch(mode, start):
    """Several full cycles of small, uneven up / down phases over an odd step count, fresh and resumed."""
    steps, up, down, base, top = 101, 3, 7, 2e-4, 5e-3
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([{"params": [p], "initial_lr": base}], lr=base)
    sched = torch.optim.lr_scheduler.CyclicLR(opt, base_lr=base, max_lr=top, step_size_up=up, step_size_down=down,
                                              mode=mode, gamma=base ** ((steps * 2) ** -1), cycle_momentum=False,
                                              last_epoch=start - 1)
    _same_schedule(make_cyclic_lr(steps, base, top, up, down, mode), start, sched, 60)


def test_cyclic_lr_modes_differ_and_reject_unknown():
    lrs = {m: [cyclic_lr(it, 1e-4, 1e-3, 2, 3, 0.9, m) for it in range(16)] for m in ("triangular", "triangular2", "exp_range")}
    assert lrs["triangular"][:5] == lrs["triangular2"][:5]          # the first cycle is unscaled in both
    assert lrs["triangular"][7] > lrs["triangular2"][7] > lrs["exp_range"][7]
    assert cyclic_lr(5, 1e-4, 1e-3, 2, 3) == cyclic_lr(5, 1e-4, 1e-3, 2, 3, None, "exp_range")
    with pytest.raises(ValueError):
        cyclic_lr(0, mode="cosine")
    with pytest.raises(ValueError):
        make_cyclic_lr(10, mode="Triangular")


def test_cyclic_steps_ratio_rules():
    assert cyclic_steps(1000, 2000, 3000) == (2000, 3000)
    assert cyclic_steps(1000, 0.25, 0.5) == (250, 500)
    assert cyclic_steps(999, 0.1, 0.3) == (99, 299)
    assert cyclic_steps(1000, 0, 0) == (1, 999)
    assert cyclic_steps(1000, -1, -2) == (1, 999)
    assert cyclic_steps(1000, 0.2, 0) == (200, 800)
    assert cyclic_steps(1000, 50, 0.0) == (50, 950)
    assert cyclic_steps(1000, 1, 1) == (1, 1)


def _check_from_args(args, steps_per_epoch, kind, n=40):
    kw, start = trainer_args(argparse.Namespace(**vars(args)), steps_per_epoch)
    opt, sched = _reference_build(argparse.Namespace(**vars(args)), steps_per_epoch)
    assert kw["optimizer"] == kind
    g = opt.param_groups[0]
    assert kw["lr"] == args.base_lr == g["initial_lr"]
    assert kw["weight_decay"] == g["weight_decay"]
    if kind == "sgd":
        assert kw["momentum"] == g["momentum"] and g["dampening"] == 0 and not g["nesterov"]
    else:
        assert "momentum" not in kw
        tr = Trainer(create_model(args.model_name), **kw)
        assert tr.betas == g["betas"] and tr.eps == g["eps"] and tr.decoupled == (kind == "adamw")
    want = Config.get_loss(args.model_name)
    assert type(kw["loss_fn"]) is type(want)
    assert start == args.start_epoch * steps_per_epoch
    if sched is None:
        assert "lr_schedule" not in kw
    else:
        _same_schedule(kw["lr_schedule"], start, sched, n)
    return kw


def test_from_args_reference_defaults():
    kw = _check_from_args(_reference_args(), 50, "adam", n=12000)        # 200 epochs x 50: two full 5000-step cycles
    assert isinstance(kw["loss_fn"], BCELoss)


@pytest.mark.parametrize("changes,kind", [
    (dict(optim="SGD"), "sgd"),
    (dict(optim="sgd", momentum=0.0, weight_decay=1e-4, lr_scheduler_mode="triangular2"), "sgd"),
    (dict(optim="adamw", weight_decay=1e-2, lr_scheduler_mode="triangular"), "adamw"),
    (dict(optim="AdamW", model_name="seist_s_pmp", warmup_steps=0.1, down_steps=0, epochs=3), "adamw"),
    (dict(model_name="seist_l_baz", steps=1001, warmup_steps=0.25, down_steps=0.5), "adam"),
    (dict(start_epoch=7, epochs=11, warmup_steps=0, down_steps=0.3, lr_scheduler_mode="triangular2"), "adam"),
    (dict(optim="Sgd", use_lr_scheduler=False, model_name="seist_m_dis"), "sgd"),
])
def test_from_args_variants(changes, kind):
    _check_from_args(_reference_args(**changes), 37, kind, n=400)


def test_from_args_unknown_optimizer_raises_like_the_reference():
    with pytest.raises(ValueError, match="Unsupported optimizer:'bogus'"):
        trainer_args(_reference_args(optim="bogus"), 10)
    with pytest.raises(ValueError, match="Unsupported optimizer:'bogus'"):
        _reference_build(_reference_args(optim="bogus"), 10)
    with pytest.raises(ValueError, match="Unsupported optimizer:'RMSprop'"):
        Trainer.from_args(create_model("seist_s_dpk"), _reference_args(optim="RMSprop"), 10)


def test_from_args_positions_the_trainer():
    tr = Trainer.from_args(create_model("seist_s_pmp"), _reference_args(optim="SGD", start_epoch=3, model_name="seist_s_pmp"), 25)
    assert tr.it == 75 and tr.optimizer == "sgd" and tr.momentum == 0.9 and isinstance(tr.loss_fn, CELoss)
    assert tr.lr_schedule(75) == make_cyclic_lr(200 * 25, 8e-5, 1e-3, 2000, 3000)(75)


def test_trainer_optimizer_names():
    m = create_model("seist_s_dpk")
    assert Trainer(m).optimizer == "adam" and not Trainer(m).decoupled
    assert Trainer(m, decoupled_wd=True).optimizer == "adamw"
    assert Trainer(m, optimizer="ADAMW").decoupled
    assert Trainer(m, optimizer="Sgd", momentum=0.9, nesterov=True).nesterov
    with pytest.raises(ValueError, match="Unsupported optimizer:'lbfgs'"):
        Trainer(m, optimizer="lbfgs")
    with pytest.raises(ValueError):
        Trainer(m, optimizer="sgd", nesterov=True)                 # torch: nesterov needs momentum, no dampening
    with pytest.raises(ValueError):
        Trainer(m, optimizer="sgd", momentum=0.9, dampening=0.1, nesterov=True)
    with pytest.raises(ValueError):
        Trainer(m, optimizer="sgd", decoupled_wd=True)


def test_default_loss_of_every_variant_matches_config():
    names = get_model_list()
    assert len(names) == 15
    for name in names:
        got, want = default_loss(create_model(name).hp), Config.get_loss(name)
        assert type(got) is type(want), name
        if isinstance(want, HuberLoss):
            assert got.delta == want.delta
        else:
            assert torch.equal(got.weight, want.weight), name
