"""The training step of the reference (training/train.py:75-121) as one device-side program.

Reference order (SURVEY §3.2): x.to(device) -> model(x) -> loss -> optimizer.zero_grad() -> loss.backward()
-> optimizer.step() -> scheduler.step().  Here the whole step — dropout-seed advance, forward plan,
fused loss forward+backward, backward plan, one flat gradient all-reduce, one fused Adam over the flat
parameter buffer (or one fused SGD) — is issued through the C-ABI on one stream and, on a single GPU, captured once into
a CUDA graph and replayed (812 kernel launches per step for seist_m_dpk would otherwise be CPU-launch bound).
The per-step host syncs of the reference (`.item()`, barrier; train.py:124-135) are not on this path:
`step()` returns the loss as a device scalar.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.distributed as dist

from . import _lib
from .config import Config
from .models.loss import BCELoss, CELoss, HuberLoss

OPTIMIZERS = ("adam", "adamw", "sgd")
CYCLIC_MODES = ("triangular", "triangular2", "exp_range")


def cyclic_lr(it: int, base_lr=8e-5, max_lr=1e-3, up=2000, down=3000, gamma: Optional[float] = None,
              mode: str = "exp_range") -> float:
    """Learning rate of torch CyclicLR(mode=mode, cycle_momentum=False) after `it` scheduler steps.  The amplitude is
    scaled per cycle by 1 ('triangular') or 1 / 2**(cycle - 1) ('triangular2'), or per iteration by gamma**it
    ('exp_range'; `gamma=None` means no decay).  The reference always decays — build its schedule with `make_cyclic_lr`."""
    total = up + down
    ratio = up / total
    cycle = math.floor(1 + it / total)
    x = 1.0 + it / total - cycle
    sf = x / ratio if x <= ratio else (x - 1) / (ratio - 1)
    if mode == "triangular":
        g = 1.0
    elif mode == "triangular2":
        g = 1 / (2.0 ** (cycle - 1))
    elif mode == "exp_range":
        g = 1.0 if gamma is None else gamma ** it
    else:
        raise ValueError(f"cyclic_lr: mode must be one of {CYCLIC_MODES}, got {mode!r}")
    return base_lr + (max_lr - base_lr) * sf * g


def make_cyclic_lr(steps: int, base_lr=8e-5, max_lr=1e-3, up=2000, down=3000, mode: str = "exp_range"):
    """The reference's schedule (training/train.py:343-354): CyclicLR(base_lr, max_lr, step_size_up=up,
    step_size_down=down, mode=mode, gamma=base_lr ** (1 / (2 * steps)), cycle_momentum=False), where
    `steps` = epochs * len(train_loader).  Returns `it -> lr` for `Trainer(lr_schedule=...)`."""
    if steps <= 0:
        raise ValueError("make_cyclic_lr: steps must be positive")
    if mode not in CYCLIC_MODES:
        raise ValueError(f"make_cyclic_lr: mode must be one of {CYCLIC_MODES}, got {mode!r}")
    gamma = float(base_lr) ** (1.0 / (2 * steps))
    return lambda it: cyclic_lr(it, base_lr, max_lr, up, down, gamma, mode)


def cyclic_steps(steps: int, warmup_steps: float, down_steps: float):
    """(step_size_up, step_size_down) from the reference's --warmup-steps / --down-steps (training/train.py:329-341):
    a value in (0, 1) is a fraction of `steps`; warmup <= 0 becomes 1 and down <= 0 becomes `steps - warmup`."""
    if warmup_steps < 1:
        warmup_steps = int(steps * warmup_steps) if warmup_steps > 0 else 1
    if down_steps < 1:
        down_steps = int(steps * down_steps) if down_steps > 0 else steps - warmup_steps
    return warmup_steps, down_steps


def default_loss(hp):
    """The loss `Config.get_loss` gives a model with hyper-parameters `hp` (config.py:137-185): BCELoss for the
    detection / picking head, CELoss for the classification head and HuberLoss for the regression heads."""
    if hp.head == "dpk":
        return BCELoss(weight=[[0.5], [1], [1]])
    if hp.head == "cls":
        return CELoss(weight=[1] * hp.head_num_classes)
    return HuberLoss()


def trainer_args(args, steps_per_epoch: int):
    """What the reference's `train_worker` builds from its `main.py` arguments (training/train.py:250-354), as
    `(Trainer keyword arguments, starting iteration)`: the optimizer from `optim`, `base_lr`, `momentum` and
    `weight_decay`; the loss from `Config.get_loss(model_name)`; the CyclicLR schedule from `use_lr_scheduler`,
    `warmup_steps`, `down_steps`, `lr_scheduler_mode` and `max_lr` over `steps = epochs * steps_per_epoch` (`steps > 0`
    rounds the epochs up); and the iteration `start_epoch * steps_per_epoch` the schedule resumes at."""
    spe = int(steps_per_epoch)
    if spe <= 0:
        raise ValueError("trainer_args: steps_per_epoch must be positive")
    name = args.optim.lower()
    if name not in OPTIMIZERS:
        raise ValueError(f"Unsupported optimizer:'{args.optim}'")
    epochs = math.ceil(args.steps / spe) if args.steps > 0 else args.epochs
    steps = epochs * spe
    kw = dict(loss_fn=Config.get_loss(args.model_name), optimizer=name, lr=args.base_lr,
              weight_decay=args.weight_decay)
    if name == "sgd":
        kw["momentum"] = args.momentum
    if args.use_lr_scheduler:
        up, down = cyclic_steps(steps, args.warmup_steps, args.down_steps)
        kw["lr_schedule"] = make_cyclic_lr(steps, args.base_lr, args.max_lr, up, down, args.lr_scheduler_mode)
    return kw, args.start_epoch * spe


class Trainer:
    """Fused train step for a `SeismogramTransformer`.  The loss defaults to `default_loss(model.hp)` (dpk -> BCELoss,
    cls -> CELoss, reg -> HuberLoss).  `optimizer` is "adam", "adamw" (also `decoupled_wd=True`) or "sgd", which is
    torch.optim.SGD with `momentum`, `dampening`, `nesterov` and `weight_decay`."""

    def __init__(self, model, loss_fn=None, lr=8e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                 decoupled_wd=False, lr_schedule=None, use_graph=True, optimizer="adam", momentum=0.0,
                 dampening=0.0, nesterov=False):
        name = str(optimizer).lower()
        if name not in OPTIMIZERS:
            raise ValueError(f"Unsupported optimizer:'{optimizer}'")
        if decoupled_wd and name == "sgd":
            raise ValueError("Trainer: decoupled_wd applies to Adam only")
        if name == "sgd" and nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        self.model = model
        self.loss_fn = loss_fn
        self.optimizer = "adamw" if decoupled_wd else name
        self.lr, self.betas, self.eps = lr, betas, eps
        self.weight_decay, self.decoupled = weight_decay, self.optimizer == "adamw"
        self.momentum, self.dampening, self.nesterov = float(momentum), float(dampening), bool(nesterov)
        self.exp_avg = self.exp_avg_sq = self.momentum_buffer = None
        self.lr_schedule = lr_schedule
        self.use_graph = use_graph
        self.it = 0
        self.graph = None
        self._shape = None
        self.launches_per_step = 0
        self.world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1

    # ---- setup -----------------------------------------------------------------------------------
    def _setup(self, x: torch.Tensor, target: torch.Tensor):
        m = self.model
        eng = m.engine()
        dev = x.device
        eng._ensure_flat(dev)
        m.train()
        N, _, L = x.shape
        self.plan = eng.get_plan(N, L, True, True)
        self.eng, self.flat = eng, eng.flat
        n = self.flat.numel
        if getattr(self, "_state_numel", None) != n:
            self.exp_avg = self.exp_avg_sq = self.momentum_buffer = None
            self.step_t = torch.zeros(1, device=dev)
            self._state_numel = n
        self._alloc_state()
        self.lr_t = torch.full((1,), float(self.lr), device=dev)
        self.x_static = self.plan.x_in.x
        if tuple(target.shape) != tuple(self.plan.y_out.x.shape if self.plan.y_out.L > 1 else self.plan.y_out.x[:, :, 0].shape):
            raise ValueError(f"Trainer: target shape {tuple(target.shape)} does not match the model output "
                             f"{tuple(self.plan.y_out.x.shape)}")
        self.t_static = torch.empty(target.shape, dtype=torch.float32, device=dev)   # kernels read raw fp32
        for a in ("_copy_stream", "_x_stage", "_t_stage", "_staged", "_consumed"):   # staging is per batch shape
            if hasattr(self, a):
                delattr(self, a)
        self._has_staged = False
        self.loss_acc = torch.zeros(1, dtype=torch.float64, device=dev)
        self.loss_out = torch.zeros((), device=dev)
        self.gout = torch.ones(1, device=dev)
        hp = m.hp
        if self.loss_fn is None:
            self.loss_fn = default_loss(hp)
        if isinstance(self.loss_fn, CELoss) and hp.head != "cls":
            raise ValueError(f"Trainer: CELoss needs the classification head, the model's head is '{hp.head}'")
        if isinstance(self.loss_fn, (BCELoss, CELoss)):
            C = hp.head_out_channels if isinstance(self.loss_fn, BCELoss) else hp.head_num_classes
            w = self.loss_fn.weight.to(dev, torch.float32)
            self.wvec = (w.reshape(1).expand(C) if w.numel() == 1 else w.reshape(C)).contiguous()
        elif not isinstance(self.loss_fn, HuberLoss):
            raise NotImplementedError("Trainer fuses BCELoss (dpk), CELoss (cls) and HuberLoss (regression) only")
        self._shape = (tuple(x.shape), tuple(target.shape))
        self.graph = None
        for _, p in eng._named:            # .grad are views of the flat gradient buffer
            p.grad = None
        for name, p in eng._named:
            p.grad = self.flat.grad_view(name)

    def _alloc_state(self):
        """The optimizer's flat state: Adam's two moments, or SGD's momentum buffer when momentum != 0."""
        n, dev = self.flat.numel, self.step_t.device
        if self.optimizer == "sgd":
            if self.momentum != 0 and self.momentum_buffer is None:
                self.momentum_buffer = torch.zeros(n, device=dev)
        elif self.exp_avg is None:
            self.exp_avg = torch.zeros(n, device=dev)
            self.exp_avg_sq = torch.zeros(n, device=dev)

    @classmethod
    def from_args(cls, model, args, steps_per_epoch: int) -> "Trainer":
        """The trainer the reference's `train_worker` builds from its `main.py` namespace `args` for a loader of
        `steps_per_epoch` batches (see `trainer_args`), positioned at iteration `start_epoch * steps_per_epoch`."""
        kw, start = trainer_args(args, steps_per_epoch)
        tr = cls(model, **kw)
        tr.it = start
        return tr

    # ---- one step on the current stream ----------------------------------------------------------
    def _issue(self):
        lib = _lib.lib()
        plan, eng, flat = self.plan, self.eng, self.flat
        s = torch.cuda.current_stream().cuda_stream
        eng._issue_forward(plan)         # its barrier: every peer has finished reading last step's statistics / gradients
        y, dy, t = plan.y_out.x, plan.y_out.dxd, self.t_static
        if isinstance(self.loss_fn, BCELoss):
            N, C, L = y.shape
            _lib.check(lib.seist_bce_fwd(y.data_ptr(), t.data_ptr(), self.wvec.data_ptr(), N, C, L,
                                         float(self.loss_fn._epsilon), self.loss_acc.data_ptr(),
                                         self.loss_out.data_ptr(), s))
            _lib.check(lib.seist_bce_bwd(y.data_ptr(), t.data_ptr(), self.wvec.data_ptr(), self.gout.data_ptr(),
                                         N, C, L, float(self.loss_fn._epsilon), dy.data_ptr(), s))
        elif isinstance(self.loss_fn, CELoss):
            N, C = y.shape[0], y.shape[1]
            eps = float(self.loss_fn._epsilon)
            _lib.check(lib.seist_ce_fwd(y.data_ptr(), t.data_ptr(), self.wvec.data_ptr(), N, C, eps,
                                        self.loss_acc.data_ptr(), self.loss_out.data_ptr(), s))
            _lib.check(lib.seist_ce_bwd(y.data_ptr(), t.data_ptr(), self.wvec.data_ptr(), self.gout.data_ptr(), N, C, eps,
                                        dy.data_ptr(), s))
        else:
            _lib.check(lib.seist_huber_fwd(y.data_ptr(), t.data_ptr(), y.numel(), self.loss_fn.delta,
                                           self.loss_acc.data_ptr(), self.loss_out.data_ptr(), s))
            _lib.check(lib.seist_huber_bwd(y.data_ptr(), t.data_ptr(), self.gout.data_ptr(), y.numel(),
                                           self.loss_fn.delta, dy.data_ptr(), s))
        flat.G.zero_()
        eng._issue_backward(plan)
        gscale = 1.0
        grads = flat.G
        if self.world > 1:
            if plan.comm is not None:
                grads = plan.comm.allreduce_grads()   # one kernel reading every peer's 1.5 MB over NVLink (C1), no NCCL
            else:
                dist.all_reduce(flat.G)          # NCCL fallback (SEIST_SYMM=0 / plain BatchNorm)
            gscale = 1.0 / self.world
        self.last_grads = grads            # what the optimizer consumed: the rank-summed gradients (x gscale = mean)
        self.step_t += 1
        if self.optimizer == "sgd":
            buf = self.momentum_buffer.data_ptr() if self.momentum_buffer is not None else None
            _lib.check(lib.seist_sgd_step(flat.P.data_ptr(), grads.data_ptr(), buf, flat.numel, self.lr_t.data_ptr(),
                                          self.step_t.data_ptr(), self.momentum, self.dampening, self.weight_decay,
                                          1 if self.nesterov else 0, gscale, s))
        else:
            _lib.check(lib.seist_adam_step(flat.P.data_ptr(), grads.data_ptr(), self.exp_avg.data_ptr(),
                                           self.exp_avg_sq.data_ptr(), flat.numel, self.lr_t.data_ptr(),
                                           self.step_t.data_ptr(), self.betas[0], self.betas[1], self.eps,
                                           self.weight_decay, 1 if self.decoupled else 0, gscale, s))

    # ---- input prefetch (the data-loader side of reference training/train.py:76-80) -------------------
    def prefetch(self, x: torch.Tensor, target: torch.Tensor):
        """Start the host -> device copy of the NEXT step's batch on a copy stream; it overlaps the step that is
        running.  The following `step()` (called without arguments) consumes it.  Pinned host tensors make the
        copy asynchronous (the reference moves batches with `.to(device)` inside the step instead)."""
        if self._shape is None:
            raise RuntimeError("prefetch() needs one step(x, target) first (it sizes the static buffers)")
        if self._shape != (tuple(x.shape), tuple(target.shape)):
            raise ValueError(f"prefetch(): batch of shape {tuple(x.shape)} / {tuple(target.shape)} does not match the "
                             f"shapes the trainer was set up for {self._shape}; call step(x, target) to re-plan")
        if not hasattr(self, "_copy_stream"):
            dev = self.x_static.device
            self._copy_stream = torch.cuda.Stream(device=dev)
            self._x_stage = torch.empty_like(self.x_static)
            self._t_stage = torch.empty_like(self.t_static)
            self._staged = torch.cuda.Event()
            self._consumed = torch.cuda.Event()
            self._consumed.record(torch.cuda.current_stream())
        cs = self._copy_stream
        cs.wait_event(self._consumed)              # the previous staged batch has been moved into the plan's input
        with torch.cuda.stream(cs):
            self._x_stage.copy_(x, non_blocking=True)
            self._t_stage.copy_(target.reshape(self._t_stage.shape), non_blocking=True)
            self._staged.record(cs)
        self._has_staged = True

    def step(self, x: Optional[torch.Tensor] = None, target: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x (N,3,L), target on the device (or pinned host tensors: copied with non_blocking=True); without
        arguments: the batch staged by `prefetch()`.  Returns the (device) loss of this step."""
        if x is None:
            if not getattr(self, "_has_staged", False):
                raise RuntimeError("step() without arguments needs a prefetch()ed batch")
            if not self.flat.valid():
                raise RuntimeError("step(): the model's parameters were re-allocated (.to()/.cuda()); call step(x, target)")
            cur = torch.cuda.current_stream()
            cur.wait_event(self._staged)
            self.x_static.copy_(self._x_stage, non_blocking=True)      # device -> device, ~0.1 ms
            self.t_static.copy_(self._t_stage, non_blocking=True)
            self._consumed.record(cur)
            self._has_staged = False
        else:
            if self._shape != (tuple(x.shape), tuple(target.shape)) or not self.flat.valid():
                self._setup(x if x.is_cuda else x.cuda(non_blocking=True), target)
            self.x_static.copy_(x, non_blocking=True)
            self.t_static.copy_(target.reshape(self.t_static.shape), non_blocking=True)
        if self.lr_schedule is not None:
            self.lr_t.fill_(float(self.lr_schedule(self.it)))
        # world > 1: with the peer-memory exchange (comm.py) a step contains no NCCL call and is captured like on one
        # GPU; the NCCL fallback is issued eagerly (a graph holding NCCL work hung at teardown)
        if self.use_graph and (self.world == 1 or self.plan.comm is not None):
            if self.graph is None:
                before = _lib.lib().seist_launch_count()
                self._issue()                    # warm-up (also sets kernel attributes)
                torch.cuda.synchronize()
                self.launches_per_step = int(_lib.lib().seist_launch_count() - before)
                g = torch.cuda.CUDAGraph()
                # capture on a HIGH-priority stream: the forward/data-gradient chain is the critical path, the
                # weight-gradient kernels forked onto the engine's default-priority side stream only fill the gaps
                # (kernel nodes inherit the priority of the stream they were captured from)
                cap = torch.cuda.Stream(device=self.x_static.device, priority=-1)
                with torch.cuda.graph(g, stream=cap):
                    self._issue()
                self.graph = g
            else:
                self.graph.replay()
        else:
            before = _lib.lib().seist_launch_count()
            # same priority split as the captured graph: the step runs on a high-priority stream, the
            # weight-gradient side stream (default priority) only fills what the main chain leaves idle
            cur = torch.cuda.current_stream()
            if getattr(self, "_hp_stream", None) is None:
                self._hp_stream = torch.cuda.Stream(device=self.x_static.device, priority=-1)
            self._hp_stream.wait_stream(cur)
            with torch.cuda.stream(self._hp_stream):
                self._issue()
            cur.wait_stream(self._hp_stream)
            self.launches_per_step = int(_lib.lib().seist_launch_count() - before)
        self.it += 1
        return self.loss_out.clone()      # a fresh scalar per step (loss_out itself is overwritten by the next step)

    # ---- checkpointing (reference models/_factory.py:59-87 stores optimizer.state_dict()) ----------------------
    def state_dict(self) -> dict:
        """A `torch.optim.Adam.state_dict()`-compatible dict (per-parameter `step`, `exp_avg`, `exp_avg_sq` in
        `model.parameters()` order, one param group) — or, with SGD, a `torch.optim.SGD.state_dict()`-compatible one
        (per-parameter `momentum_buffer` once the buffers exist) — plus the trainer's own counters (`seist_b200`:
        LR-schedule position and dropout step counter), so `save_checkpoint(..., optimizer=trainer, ...)` round-trips."""
        if self._shape is None:
            raise RuntimeError("Trainer.state_dict(): run one step first (the optimizer state lives on the device)")
        extra = {"it": self.it, "dropout_seed": self.eng.dropout_seed()}
        if self.optimizer == "sgd":
            return {"state": self._sgd_state(), "param_groups": [self._sgd_group()], "seist_b200": extra}
        state = {}
        for i, (name, _) in enumerate(self.eng._named):
            r = self.flat.pref[name]
            state[i] = {"step": self.step_t[0].detach().clone().cpu(),
                        "exp_avg": self.exp_avg[r.off:r.off + r.numel].view(r.shape).clone(),
                        "exp_avg_sq": self.exp_avg_sq[r.off:r.off + r.numel].view(r.shape).clone()}
        group = {"lr": float(self.lr_t.item()), "betas": tuple(self.betas), "eps": self.eps,
                 "weight_decay": self.weight_decay, "amsgrad": False, "maximize": False, "foreach": None,
                 "capturable": False, "differentiable": False, "fused": None, "decoupled_weight_decay": bool(self.decoupled),
                 "params": list(range(len(self.eng._named)))}
        return {"state": state, "param_groups": [group], "seist_b200": extra}

    def _sgd_state(self) -> dict:
        # torch.optim.SGD has no state before its first step, and none at all without momentum
        if self.momentum == 0 or float(self.step_t.item()) < 1:
            return {}
        state = {}
        for i, (name, _) in enumerate(self.eng._named):
            r = self.flat.pref[name]
            state[i] = {"momentum_buffer": self.momentum_buffer[r.off:r.off + r.numel].view(r.shape).clone()}
        return state

    def _sgd_group(self) -> dict:
        return {"lr": float(self.lr_t.item()), "momentum": self.momentum, "dampening": self.dampening,
                "weight_decay": self.weight_decay, "nesterov": self.nesterov, "maximize": False, "foreach": None,
                "differentiable": False, "fused": None, "params": list(range(len(self.eng._named)))}

    def load_state_dict(self, sd: dict):
        """Accepts `Trainer.state_dict()` or a plain `torch.optim.Adam.state_dict()` (with SGD:
        `torch.optim.SGD.state_dict()`) of the same model."""
        if self._shape is None:
            raise RuntimeError("Trainer.load_state_dict(): run (or set up) one step first")
        named = self.eng._named
        st = sd.get("state", {})
        if len(st) not in (0, len(named)):
            raise ValueError(f"optimizer state has {len(st)} entries, the model has {len(named)} parameters")
        groups = sd.get("param_groups") or []
        if self.optimizer == "sgd":
            self._load_sgd(st, groups[0] if groups else {})
        else:
            self._load_adam(st)
        if groups:
            g0 = groups[0]
            self.lr = float(g0.get("lr", self.lr))
            if self.optimizer != "sgd":
                self.betas = tuple(g0.get("betas", self.betas))
                self.eps = float(g0.get("eps", self.eps))
            self.weight_decay = float(g0.get("weight_decay", self.weight_decay))
            self.lr_t.fill_(self.lr)
            self.graph = None                       # the hyper-parameters are baked into the captured launch
        extra = sd.get("seist_b200")
        if extra:
            self.it = int(extra.get("it", self.it))
            if "dropout_seed" in extra:
                self.eng.set_dropout_seed(int(extra["dropout_seed"]))

    def _load_sgd(self, st: dict, g0: dict):
        """Momentum buffers and SGD hyper-parameters.  A state without buffers is a fresh optimizer: the next step
        initialises them; with buffers, the device step counter is set so the next step is not the first."""
        if g0.get("maximize", False):
            raise ValueError("Trainer: SGD with maximize=True is not supported")
        momentum = float(g0.get("momentum", self.momentum))
        dampening = float(g0.get("dampening", self.dampening))
        nesterov = bool(g0.get("nesterov", self.nesterov))
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        self.momentum, self.dampening, self.nesterov = momentum, dampening, nesterov
        self._alloc_state()
        bufs = []
        for i, (name, _) in enumerate(self.eng._named):
            e = st.get(i, st.get(str(i)))
            if e is None:
                continue
            if "momentum_buffer" not in e:
                raise ValueError(f"optimizer state of {name} has no momentum_buffer: not a torch.optim.SGD state")
            if e["momentum_buffer"] is not None:
                bufs.append((name, e["momentum_buffer"]))
        if not bufs:
            self.step_t.fill_(0)
            return
        if len(bufs) != len(self.eng._named) or self.momentum == 0:
            raise ValueError("momentum buffers must be given for every parameter, with a non-zero momentum")
        for name, b in bufs:
            r = self.flat.pref[name]
            if tuple(b.shape) != tuple(r.shape):
                raise ValueError(f"optimizer state of {name}: shape {tuple(b.shape)} != {tuple(r.shape)}")
            self.momentum_buffer[r.off:r.off + r.numel].copy_(b.reshape(-1))
        self.step_t.fill_(1)

    def _load_adam(self, st: dict):
        step = None
        named = self.eng._named
        for i, (name, p) in enumerate(named):
            e = st.get(i, st.get(str(i)))
            if e is None:
                continue
            r = self.flat.pref[name]
            if tuple(e["exp_avg"].shape) != tuple(r.shape):
                raise ValueError(f"optimizer state of {name}: shape {tuple(e['exp_avg'].shape)} != {tuple(r.shape)}")
            self.exp_avg[r.off:r.off + r.numel].copy_(e["exp_avg"].reshape(-1))
            self.exp_avg_sq[r.off:r.off + r.numel].copy_(e["exp_avg_sq"].reshape(-1))
            s_i = float(e["step"])
            if step is not None and s_i != step:
                raise ValueError("per-parameter Adam step counts differ; the fused update keeps one")
            step = s_i
        if step is not None:
            self.step_t.fill_(step)
