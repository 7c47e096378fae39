"""Recipe for `oracle/_ref/`: the UNMODIFIED reference model code and its trained checkpoints, staged beside the package.

MEASUREMENT AND TEST INFRASTRUCTURE, not product.  `oracle/_ref/` is git-ignored (never committed).  Two things use it:
  * `bench.py` (the `--impl reference` arm, `cpu_baseline`, and the informational same-GPU line) imports the staged
    `models/seist.py` + `models/loss.py` — default drop rates, torch's own kernels — and times them instead of the
    oracle port;
  * the pretrained-regime tests (tests/test_cpu_pretrained.py, tests/test_gpu_pretrained.py) load the 18 shipped
    checkpoints from `pretrained/` through `oracle/pretrained.py`, which checks each file's SHA-256 against
    tests/golden/reference_pretrained.pt and raises where a file is missing or differs.
Run by `__graft_entry__.build()`; the checkout is SEIST_REFERENCE_ROOT (default /root/reference), and nothing is staged
where it does not exist:

    python oracle/build_ref.py            # <checkout>/models/*.py -> oracle/_ref/models/, timm shim beside it,
                                          # <checkout>/pretrained/*.pth -> oracle/_ref/pretrained/

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


def sha256(path) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


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
            manifest["models/" + fn] = sha256(os.path.join(dst, fn))
    ckpt_src, ckpt_dst = os.path.join(REF_ROOT, "pretrained"), os.path.join(OUT, "pretrained")
    if os.path.isdir(ckpt_src):
        os.makedirs(ckpt_dst, exist_ok=True)
        for fn in sorted(os.listdir(ckpt_src)):
            if fn.endswith(".pth"):
                shutil.copyfile(os.path.join(ckpt_src, fn), os.path.join(ckpt_dst, fn))
                manifest["pretrained/" + fn] = sha256(os.path.join(ckpt_dst, fn))
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
