"""Forward-only fast path (SURVEY §8f-4): the eval-mode plan of one (N, L) captured into a CUDA graph.

The reference's inference callers (`training/validate.py:53-66`, `demo_predict.py:77-82`) call `model(x)` under
`torch.no_grad()` in eval mode: BatchNorm is a per-channel affine from the running statistics there, which the plan applies
in the consumers' load prologue (the coefficient table is written once per replay by one `BN_PREPARE` launch over all 115
layers) — no BatchNorm kernel, no statistics pass.  At deployment batch sizes (a few waveforms) the forward is bound by
issuing its ~290 kernel launches, so the whole plan is captured once and replayed: one `cudaGraphLaunch` per batch.
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib


class InferenceGraph:
    """`g = InferenceGraph(model, N, L); y = g(x)` — x (N, C, L) float32 on the model's device (or pinned host memory:
    copied asynchronously); returns the static output tensor (valid until the next call; `.clone()` to keep it)."""

    def __init__(self, model, N: int, L: int):
        if next(model.parameters()).device.type != "cuda":
            raise RuntimeError("InferenceGraph needs the model on a CUDA device (no CPU path)")
        model.eval()
        eng = model.engine()
        dev = next(model.parameters()).device
        eng._ensure_flat(dev)
        self.model, self.eng = model, eng
        self.plan = eng.get_plan(N, L, False, False)
        self.x = self.plan.x_in.x
        y = self.plan.y_out.x
        self.y = y if self.plan.y_out.L > 1 else y[:, :, 0]
        self._stream = torch.cuda.Stream(device=dev)
        lib = _lib.lib()
        base = ctypes.addressof(self.plan.c_fwd)
        n_ops = len(self.plan.fwd_ops)
        with torch.cuda.device(dev):
            with torch.cuda.stream(self._stream):        # warm-up: loads the kernels, sets their attributes
                _lib.check(lib.seist_plan_run(base, n_ops, self._stream.cuda_stream), "seist_plan_run")
            self._stream.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self._stream):
                _lib.check(lib.seist_plan_run(base, n_ops, torch.cuda.current_stream().cuda_stream), "seist_plan_run")
        self.launches = n_ops

    @torch.no_grad()
    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if tuple(x.shape) != tuple(self.x.shape):
            raise ValueError(f"InferenceGraph was built for {tuple(self.x.shape)}, got {tuple(x.shape)}")
        if not self.eng.flat.valid():
            raise RuntimeError("the model's parameters were re-allocated (.to()/.cuda()); build a new InferenceGraph")
        self.x.copy_(x, non_blocking=True)
        return self.replay()

    def replay(self) -> torch.Tensor:
        """Run the captured plan on the current stream on whatever the static input `self.x` holds (filled in place by
        the caller's own kernels); returns the static output tensor."""
        if not self.eng.flat.valid():
            raise RuntimeError("the model's parameters were re-allocated (.to()/.cuda()); build a new InferenceGraph")
        self.graph.replay()
        return self.y
