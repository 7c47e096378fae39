"""Import the UNMODIFIED reference from a SeisT checkout (SEIST_REFERENCE_ROOT, default /root/reference).

Used only to generate the tests/golden fixtures (tests/golden/make_golden.py); nothing in the tests, the
benchmark or the package needs a reference checkout.
"""
import os
import sys

REF_ROOT = os.environ.get("SEIST_REFERENCE_ROOT", "/root/reference")
_SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "timm_shim")


def available() -> bool:
    return bool(REF_ROOT) and os.path.isfile(os.path.join(REF_ROOT, "models", "seist.py"))


def import_reference_models():
    """Returns the reference's `models` package (create_model, BCELoss, ...)."""
    if not available():
        raise RuntimeError(f"reference not present at {REF_ROOT}")
    for p in (_SHIM, REF_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    # The product package also ships a `models`-like surface under seist_b200.models; the bare
    # top-level name `models` is the reference's.
    import models as ref_models  # noqa: E402

    assert os.path.abspath(ref_models.__file__).startswith(os.path.abspath(REF_ROOT))
    return ref_models


def zero_drop_rates(model):
    """Set every Dropout.p / DropPath.drop_prob to 0 after construction (SURVEY §7.1)."""
    import torch.nn as nn

    for m in model.modules():
        if isinstance(m, nn.Dropout):
            m.p = 0.0
        if m.__class__.__name__ == "DropPath":
            m.drop_prob = 0.0
    return model
