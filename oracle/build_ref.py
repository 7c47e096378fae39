"""Recipe for `oracle/_ref/`: the UNMODIFIED reference model code, staged beside the package.

MEASUREMENT INFRASTRUCTURE, not product: only `bench.py` (the `--impl reference` arm, `cpu_baseline`, and the
informational same-GPU line) imports what this script stages.  `oracle/_ref/` is git-ignored (never committed); with it
the reference's own `models/seist.py` + `models/loss.py` — default drop rates, torch's own kernels — are timed instead
of the oracle port.  Run by `__graft_entry__.build()`; the checkout is SEIST_REFERENCE_ROOT (default /root/reference),
and nothing is staged where it does not exist:

    python oracle/build_ref.py            # <checkout>/models/*.py -> oracle/_ref/models/, timm shim beside it

Nothing is edited: files are copied byte for byte and their SHA-256 recorded in oracle/_ref/MANIFEST.json.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("SEIST_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref")


def available() -> bool:
    return os.path.isfile(os.path.join(OUT, "models", "seist.py"))


def build() -> bool:
    src = os.path.join(REF_ROOT, "models")
    if not os.path.isfile(os.path.join(src, "seist.py")):
        return available()
    dst = os.path.join(OUT, "models")
    os.makedirs(dst, exist_ok=True)
    manifest = {}
    for fn in sorted(os.listdir(src)):
        if fn.endswith(".py"):
            shutil.copyfile(os.path.join(src, fn), os.path.join(dst, fn))
            manifest["models/" + fn] = hashlib.sha256(open(os.path.join(dst, fn), "rb").read()).hexdigest()
    shim_dst = os.path.join(OUT, "timm")
    if os.path.isdir(shim_dst):
        shutil.rmtree(shim_dst)
    shutil.copytree(os.path.join(HERE, "timm_shim", "timm"), shim_dst)     # DropPath only (models/seist.py:7)
    json.dump({"source": REF_ROOT, "files": manifest}, open(os.path.join(OUT, "MANIFEST.json"), "w"), indent=1)
    return True


def import_models():
    """The staged reference `models` package (create_model, BCELoss, ...)."""
    if not available():
        raise RuntimeError("oracle/_ref is not staged (run oracle/build_ref.py where a reference checkout exists)")
    if OUT not in sys.path:
        sys.path.insert(0, OUT)
    import models as ref_models
    assert os.path.abspath(ref_models.__file__).startswith(os.path.abspath(OUT)), ref_models.__file__
    return ref_models


if __name__ == "__main__":
    print("staged" if build() else "reference not present; nothing staged")
