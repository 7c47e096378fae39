"""Model registry and checkpoint I/O with the reference's contract.

Mirrors the reference's models/_factory.py: `register_model` (:24-38) keys the registry by the
creator's ``__name__`` and rejects duplicates; `create_model` (:41-56) raises ValueError listing
what is available; `save_checkpoint` (:59-87) / `load_checkpoint` (:90-126) keep the reference's
checkpoint dictionary layout so files are interchangeable in both directions.
"""
import sys
import warnings
from typing import Callable, Dict, List

import torch

__all__ = ["get_model_list", "register_model", "create_model", "save_checkpoint", "load_checkpoint"]

_REGISTRY: Dict[str, Callable] = {}


def get_model_list() -> List[str]:
    return list(_REGISTRY)


def register_model(func: Callable) -> Callable:
    name = func.__name__
    if name in _REGISTRY:
        raise Exception(f"Model '{name}' already exists.")
    mod = sys.modules.get(func.__module__)
    if mod is not None and hasattr(mod, "__all__") and name not in mod.__all__:
        mod.__all__.append(name)
    _REGISTRY[name] = func
    return func


def create_model(model_name: str, **kwargs):
    if model_name not in _REGISTRY:
        raise ValueError(f"Model '{model_name}' does not exist. \nAvailable: {get_model_list()}")
    return _REGISTRY[model_name](**kwargs)


def _unwrap(model):
    use_ddp = hasattr(model, "module")
    inner = model.module if use_ddp else model
    # the reference probes `_orig_mod` on the OUTER object (models/_factory.py:70)
    use_compile = hasattr(model, "_orig_mod")
    if use_compile:
        inner = inner._orig_mod
    return inner, use_ddp, use_compile


def save_checkpoint(save_path: str, epoch: int, model, optimizer, best_loss: float) -> None:
    inner, use_ddp, use_compile = _unwrap(model)
    torch.save(
        {
            "epoch": epoch,
            "optimizer_dict": optimizer.state_dict(),
            "model_dict": inner.state_dict(),
            "loss": best_loss,
            "use_compile": use_compile,
            "use_ddp": use_ddp,
        },
        save_path,
    )


def load_checkpoint(save_path: str, device, dist_mode=False, compile_mode=False, resume=False):
    ckpt = torch.load(save_path, map_location=device)
    if "model_dict" not in ckpt:
        ckpt = {"model_dict": ckpt}
    ckpt["model_dict"] = {
        k.replace("module.", "").replace("_orig_mod.", ""): v for k, v in ckpt["model_dict"].items()
    }
    if resume:
        used_ddp = ckpt.get("use_ddp", False)
        used_compile = ckpt.get("use_compile", False)
        if used_ddp != dist_mode:
            warnings.warn(
                f"The model was trained {'with' if used_ddp else 'without'} using distributed mode, "
                f"but distributed mode is {'enabled' if dist_mode else 'disabled'} now, "
                "which may lead to unreproducible results.")
        if used_compile != compile_mode:
            warnings.warn(
                f"The model was trained {'with' if used_compile else 'without'} using `torch.compile`, "
                f"but the argument `use_torch_compile` is `{compile_mode}`, "
                "which may lead to unreproducible results.")
    return ckpt
