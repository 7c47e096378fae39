"""Execution engine: owns the flat parameter state and the compiled plans of one model and runs
them through the C-ABI (`seist_plan_run_lanes`) from the current CUDA stream.

`Engine.forward` is what `SeismogramTransformer.forward` calls: it is autograd-compatible (the
returned tensor carries a grad_fn whose backward runs the backward plan and deposits parameter
gradients into views of one flat gradient buffer), works under `torch.no_grad()` / `.eval()`, and
under data parallelism reduces SyncBatchNorm statistics across ranks between the producing and the
consuming kernels (reference training/train.py:374 converts every BN to SyncBatchNorm).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib
from . import plan as P


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def run_segment(c_ops, start: int, end: int, streams: Sequence[int]):
    """Issue the descriptors c_ops[start:end] (one segment of a compiled plan) by their lane schedule on `streams`: the
    plan's main lanes, then its weight-gradient lane.  Every lane is forked from streams[0] and joined back into it."""
    arr = (ctypes.c_void_p * len(streams))(*streams)
    base = ctypes.addressof(c_ops) + start * ctypes.sizeof(_lib.SeistOp)
    _lib.check(_lib.lib().seist_plan_run_lanes(base, end - start, arr, len(streams)), "seist_plan_run_lanes")


class _PlanFn(torch.autograd.Function):
    """(x, *parameters) -> y through the forward plan; backward runs the backward plan and returns the parameter
    gradients as ordinary autograd outputs (views of the engine's flat gradient buffer), so that
    `loss.backward()` accumulates into `.grad`, `DistributedDataParallel`'s reducer hooks fire
    (reference training/train.py:367-374) and `torch.optim` optimizers work unchanged."""

    @staticmethod
    def forward(ctx, x, engine, plan, *params):
        ctx.engine, ctx.plan = engine, plan
        ctx.n_params = len(params)
        y = engine.run_forward(plan, x)
        return y.clone()

    @staticmethod
    def backward(ctx, dy):
        grads = ctx.engine.run_backward(ctx.plan, dy)
        return (None, None, None) + tuple(grads)


class Engine:
    def __init__(self, model: nn.Module):
        self.model = model
        self.flat: Optional[P.FlatState] = None
        self.plans: Dict[Tuple, P.Plan] = {}
        self.last_plan: Optional[P.Plan] = None
        self._side = {}
        self._aux = {}
        self.seed_dev: Optional[torch.Tensor] = None     # ONE dropout step counter (device int64) shared by every plan
        self.comm = None                                  # PeerComm (NVLink peer-memory exchange) under data parallelism

    # ---- lifecycle -------------------------------------------------------------------------------
    def invalidate(self, release_flat: bool = False):
        self.plans.clear()
        self.last_plan = None
        if release_flat:
            self.flat = None

    def _ensure_flat(self, device):
        if self.flat is None or self.flat.device != device or not self.flat.valid():
            self.plans.clear()
            self.flat = P.FlatState(self.model, device)
            self._named = list(self.model.named_parameters())
            if self.comm is not None:                 # the flat gradient buffer lives in symmetric memory
                if self.comm.n_grad != self.flat.numel or self.comm.device != device:
                    self.comm = None
                else:
                    self.flat.G = self.comm.grad
                    self.flat.G.zero_()
        if self.seed_dev is None or self.seed_dev.device != device:
            old = None if self.seed_dev is None else int(self.seed_dev.item())
            self.seed_dev = torch.zeros(1, dtype=torch.int64, device=device)
            self.seed_dev.fill_(self._initial_seed() if old is None else old)
        return self.flat

    @staticmethod
    def _initial_seed() -> int:
        """Start of the dropout/DropPath step counter: follows torch.manual_seed() and differs per rank (the
        reference's torch RNG streams do, training/train.py sets the seed per process); 62 bits, non-negative."""
        rank = dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0
        z = (torch.initial_seed() * 0x9E3779B97F4A7C15 + (rank + 1) * 0xD1B54A32D192ED03) & ((1 << 64) - 1)
        z ^= z >> 29
        return z & ((1 << 62) - 1)

    def dropout_seed(self) -> int:
        """Current value of the dropout step counter (checkpoint it next to the optimizer state)."""
        return 0 if self.seed_dev is None else int(self.seed_dev.item())

    def set_dropout_seed(self, value: int):
        if self.seed_dev is None:
            raise RuntimeError("set_dropout_seed: the model has not been moved to a CUDA device yet")
        self.seed_dev.fill_(int(value) & ((1 << 62) - 1))

    def sync_world(self) -> int:
        """World size over which BatchNorm statistics are shared (1 unless the BNs are SyncBatchNorm)."""
        if not (dist.is_available() and dist.is_initialized()):
            return 1
        if any(isinstance(m, nn.SyncBatchNorm) for m in self.model.modules()):
            return dist.get_world_size()
        return 1

    def _ensure_comm(self, world: int):
        """Peer-memory exchange for SyncBatchNorm statistics and gradients (comm.py); None on one GPU or with
        SEIST_SYMM=0 (then the statistics are all-reduced with NCCL at the plan's sync points)."""
        from .comm import PeerComm, symmetric_memory_enabled
        if world <= 1 or not symmetric_memory_enabled():
            return None
        if self.comm is None and not getattr(self, "_comm_failed", False):
            n_stat = sum(2 * m.num_features for m in self.model.modules()
                         if isinstance(m, nn.modules.batchnorm._BatchNorm))
            ok = torch.ones(1, device=self.flat.device)
            try:
                if world > _lib.MAX_WORLD:
                    raise RuntimeError(f"more than {_lib.MAX_WORLD} ranks")
                comm = PeerComm(self.flat.device, world, dist.get_rank(), max(n_stat, 2), self.flat.numel)
            except Exception as e:      # noqa: BLE001 - e.g. no peer access / symmetric memory unsupported on this box
                comm = None
                ok.zero_()
                import warnings
                warnings.warn(f"seist_b200: NVLink peer-memory exchange unavailable ({e!r}); using NCCL collectives")
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)      # all ranks take the same path
            if ok.item() < 1:
                self._comm_failed = True
                return None
            self.comm = comm
            self.flat.G = self.comm.grad
            self.flat.G.zero_()
        return self.comm

    def get_plan(self, N: int, L: int, training: bool, need_backward: bool) -> P.Plan:
        _lib.lib()   # fail loudly if the CUDA extension is missing
        world = self.sync_world() if training else 1
        key = (N, L, training, need_backward, world)
        pl = self.plans.get(key)
        if pl is None:
            if len(self.plans) >= 4:      # plans own large arenas; keep the cache small
                self.plans.pop(next(iter(self.plans)))
            b = P.PlanBuilder(self.model, self.flat, N, L, training, world=world, need_backward=need_backward)
            comm = self._ensure_comm(world) if training else None
            pl = P.finalize(b.build(), need_backward, step_seed=self.seed_dev, comm=comm)
            self.plans[key] = pl
        return pl

    # ---- execution -------------------------------------------------------------------------------
    def _lane_streams(self, device, n_main: int):
        """[current stream, aux lanes (independent branches, high priority), weight-gradient lane (default priority)]"""
        aux = self._aux.setdefault(device, [])
        while len(aux) < n_main - 1:
            aux.append(torch.cuda.Stream(device=device, priority=-1))
        side = self._side.get(device)
        if side is None:
            side = self._side[device] = torch.cuda.Stream(device=device)
        return [_stream_ptr()] + [a.cuda_stream for a in aux[:n_main - 1]] + [side.cuda_stream]

    def _run_segments(self, plan: P.Plan, c_ops, segs, stat: torch.Tensor):
        streams = self._lane_streams(plan.device, plan.n_main)
        for start, end, sync in segs:
            i = 0
            while i < len(sync):          # BN entries registered consecutively own contiguous slots: one call
                j = i
                while j + 1 < len(sync) and sync[j + 1] == sync[j] + 1:
                    j += 1
                lo, hi = plan.bns[sync[i]], plan.bns[sync[j]]
                dist.all_reduce(stat[lo.st_off:hi.st_off + 2 * hi.C])
                i = j + 1
            run_segment(c_ops, start, end, streams)

    def _issue_forward(self, plan: P.Plan):
        """The forward plan on the current stream; its input is already in `plan.x_in`."""
        if plan.training:
            # a new set of dropout / DropPath masks for every training forward (the backward of this forward
            # regenerates the same masks from the same counter value)
            _lib.check(_lib.lib().seist_advance_seed(plan.step_seed.data_ptr(), _stream_ptr()), "seist_advance_seed")
            if plan.comm is not None:
                plan.comm.barrier()      # no peer is still reading last step's partial sums when they are cleared
            plan.stat_acc.zero_()
        self._run_segments(plan, plan.c_fwd, plan.fwd_segments, plan.stat_acc)
        if plan.training:
            self.flat.NBT[:len(plan.bns)] += 1

    def _issue_backward(self, plan: P.Plan):
        """The backward plan on the current stream; the output gradient is already in `plan.y_out.dxd`.  It accumulates
        into the flat gradient buffer, which the caller clears."""
        plan.gstat_acc.zero_()
        plan.dWx.zero_()
        self._run_segments(plan, plan.c_bwd, plan.bwd_segments, plan.gstat_acc)

    def run_forward(self, plan: P.Plan, x: torch.Tensor) -> torch.Tensor:
        plan.x_in.x.copy_(x)
        self._issue_forward(plan)
        self.last_plan = plan
        y = plan.y_out.x
        return y if plan.y_out.L > 1 else y[:, :, 0]

    def run_backward(self, plan: P.Plan, dy: torch.Tensor):
        """Run the backward plan for the output gradient `dy`; returns one gradient per parameter, in
        `model.named_parameters()` order, as views of the flat gradient buffer (None for frozen parameters)."""
        flat = self.flat
        flat.G.zero_()
        if plan.comm is not None:
            # no peer is still reading the last backward's partial sums when they are cleared (two backward calls need
            # not have a forward, and its barrier, in between)
            plan.comm.barrier()
        plan.y_out.dxd.copy_(dy.reshape(plan.y_out.dxd.shape))
        self._issue_backward(plan)
        # one copy of the 1.5 MB buffer: autograd may keep ("steal") the returned tensors as `.grad`, and the flat
        # buffer is zeroed again by the next backward (gradient accumulation over several backward calls must add up)
        out = flat.G.clone()
        return [out[flat.pref[name].off:flat.pref[name].off + flat.pref[name].numel].view(flat.pref[name].shape)
                if p.requires_grad else None for name, p in self._named]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        model = self.model
        if x.dtype != torch.float32:
            x = x.float()
        x = x.contiguous()
        if x.dim() != 3 or x.shape[1] != model.hp.in_channels:
            raise ValueError(f"expected input of shape (N, {model.hp.in_channels}, L), got {tuple(x.shape)}")
        self._ensure_flat(x.device)
        N, _, L = x.shape
        training = model.training
        need_bwd = training and torch.is_grad_enabled()
        plan = self.get_plan(N, L, training, need_bwd)
        with torch.cuda.device(x.device):
            if need_bwd:
                return _PlanFn.apply(x, self, plan, *[p for _, p in self._named])
            return self.run_forward(plan, x).clone()

    # ---- data-parallel helpers -------------------------------------------------------------------
    def allreduce_grads(self, average: bool = True):
        """One collective over all parameter gradients (an alternative to wrapping the model in
        DistributedDataParallel, whose bucket reducer also works: the gradients are autograd outputs)."""
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        grads = [p.grad for _, p in self._named if p.grad is not None]
        if not grads:
            return
        flat = torch.cat([g.reshape(-1) for g in grads])
        dist.all_reduce(flat)
        if average:
            flat.div_(dist.get_world_size())
        off = 0
        for g in grads:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()
