"""Shared test helpers: build interpreter (CPU, or float64 on the device) and CUDA plans of the same model and compare
them op by op with teacher forcing (the GPU op always starts from the interpreter's state)."""
import copy
import ctypes

import torch

from oracle.plan_interp import Interp
from seist_b200 import _lib
from seist_b200 import plan as P
from seist_b200.models import create_model

ZERO_DROPS = dict(path_drop_rate=0, attn_drop_rate=0, key_drop_rate=0, mlp_drop_rate=0, other_drop_rate=0)


def model_drops(name):
    """The drop rates model `name` trains with when nobody sets them (its registered preset), as a `drops` dict."""
    hp = create_model(name, in_channels=3, in_samples=8192).hp
    return {k: getattr(hp, k) for k in ZERO_DROPS}


def randomize(model, seed=0, wstd=0.25):
    """Non-degenerate parameters / running statistics (random-init eval output is a flat 0.5, SURVEY §0.6)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() > 1:
                fan = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) * (1.0 / fan ** 0.5))
            elif name.endswith("norm.weight") or ".norm" in name and name.endswith("weight") or "norms." in name and name.endswith("weight"):
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
        for name, b in model.named_buffers():
            if name.endswith("running_mean"):
                b.copy_(0.1 * torch.randn(b.shape, generator=g))
            elif name.endswith("running_var"):
                b.copy_(0.5 + torch.rand(b.shape, generator=g))
    return model


def build_pair(name, N, L, training, drops=None, seed=0, hp_overrides=None, state_dict=None, ref_device=None,
               ref_dtype=torch.float32):
    """(ref_plan, gpu_plan, interp, ref_model, gpu_model) for two identical copies of model `name`.  The interpreter's
    plan lives on the CPU unless `ref_device` names another device ("cuda": both plans on cuda:0, so the teacher-forcing
    copies stay on the device); `ref_dtype` is the interpreter's arithmetic."""
    m_ref = create_model(name, in_channels=3, in_samples=L, **(hp_overrides or {}))
    if state_dict is not None:
        m_ref.load_state_dict(state_dict, strict=True)
    else:
        randomize(m_ref, seed)
    m_ref.set_drop_rates(**(ZERO_DROPS if drops is None else drops))
    m_ref.train(training)
    m_gpu = copy.deepcopy(m_ref)
    dev = torch.device("cuda:0")
    rdev = torch.device("cpu") if ref_device is None else torch.device(ref_device)
    if rdev.type == "cuda" and rdev.index is None:
        rdev = dev
    m_ref.to(rdev)
    f_ref = P.FlatState(m_ref, rdev)
    p_ref = P.PlanBuilder(m_ref, f_ref, N, L, training).build()
    P.allocate(p_ref, training)
    m_gpu.to(dev)
    f_gpu = P.FlatState(m_gpu, dev)
    p_gpu = P.finalize(P.PlanBuilder(m_gpu, f_gpu, N, L, training).build(), training)
    assert p_ref.arena.numel() == p_gpu.arena.numel()
    return p_ref, p_gpu, Interp(p_ref, ref_dtype), m_ref, m_gpu


def push_state(p_cpu, p_gpu):
    p_gpu.arena.copy_(p_cpu.arena)
    p_gpu.stat.copy_(p_cpu.stat)
    p_gpu.gstat.copy_(p_cpu.gstat)
    p_gpu.flat.G.copy_(p_cpu.flat.G)
    p_gpu.flat.RB.copy_(p_cpu.flat.RB)
    p_gpu.step_seed.copy_(p_cpu.step_seed)
    p_gpu.Wx.copy_(p_cpu.Wx)
    p_gpu.dWx.copy_(p_cpu.dWx)


def run_gpu_op(p_gpu, c_ops, i):
    base = ctypes.addressof(c_ops) + i * ctypes.sizeof(_lib.SeistOp)
    _lib.check(_lib.lib().seist_plan_run(base, 1, torch.cuda.current_stream().cuda_stream), f"op {i}")
    torch.cuda.synchronize()


def rel_err(a, b):
    """max |a - b| over max |b| of the whole tensor (and max |b|), in float64 on a's device."""
    a, b = a.double(), b.to(a.device).double()
    return ((a - b).abs().max() / (b.abs().max() + 1e-20)).item(), b.abs().max().item()


def chan_err(got, ref, scale, dim=1):
    """Per-channel error: the largest |got - ref| in each channel (index `dim`: 1 for activations and data gradients,
    0 for weight-gradient rows and for per-entry vectors such as stat / gstat / bias) divided by that channel's
    scale[c].  Returns (worst ratio, its channel).  A channel whose scale is 0 must match exactly."""
    d = (got.double() - ref.to(got.device).double()).abs().movedim(dim, 0).reshape(got.shape[dim], -1).amax(1)
    r = d / scale.to(d.device).double().clamp_min(1e-300)
    r = torch.where(d == 0, torch.zeros_like(r), r)
    c = int(r.argmax())
    return r[c].item(), c


def chan_max(t, dim=1):
    """Per-channel max of t along every index but `dim` (the scale of `chan_err` from an elementwise magnitude)."""
    return t.movedim(dim, 0).reshape(t.shape[dim], -1).amax(1)
