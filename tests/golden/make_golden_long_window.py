"""Generate tests/golden/reference_long_window.pt by executing the UNMODIFIED reference (a SeisT checkout,
SEIST_REFERENCE_ROOT) on its shipped seist_m_dpk and seist_s_dpk checkpoints at a window of 16384 samples, twice the
8192 of reference_pretrained.pt: every attention op then has 256 keys (two 128-key chunks of csrc/attention.cu).

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_long_window.py

The inputs are oracle/pretrained.dpk_records (the 8 event records of the picker fixture, whole, normalised "std"); they
are regenerated from seeds and only their SHA-256 is stored.  Per model: the checkpoint's SHA-256, the reference's
float64 eval output (`model.double()`) as a float64 sample, `dev` = max |fp32 output - float64 output| of the reference
itself, the arg max of the P and S rows and whether it is well posed (the top value beats every other value of its row
by >= 1e-5, as make_golden_pretrained.py).
"""
import hashlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import golden as G  # noqa: E402
from oracle import pretrained as PT  # noqa: E402
from oracle import reference_import as ri  # noqa: E402
from make_golden_pretrained import well_posed  # noqa: E402

LENGTH = 16384
MODELS = ("seist_m_dpk", "seist_s_dpk")
FIXTURE = os.path.join(G.GOLD, "reference_long_window.pt")


def inputs_sha(x):
    return hashlib.sha256(x.contiguous().numpy().tobytes()).hexdigest()


def eval_entry(M, name, x):
    path = os.path.join(ri.REF_ROOT, "pretrained", f"{name}_diting.pth")
    model = M.create_model(name, in_channels=3, in_samples=LENGTH)
    model.load_state_dict(PT.read_checkpoint(path), strict=True)
    model.eval()
    with torch.no_grad():
        y32 = model(x)
        y64 = model.double()(x.double())
    return {"sha256": PT.sha256(path), "y": PT.sample64(y64, 8192, seed=7), "dev": (y32.double() - y64).abs().max().item(),
            "pick": y64[:, 1:].argmax(-1),
            "well_posed": torch.tensor([[well_posed(y64[n, c]) for c in (1, 2)] for n in range(x.shape[0])])}


def main():
    M = ri.import_reference_models()
    torch.set_num_threads(8)
    x = PT.dpk_records(PT.DPK_N, PT.DPK_SEED, LENGTH)
    res = {"length": LENGTH, "n": PT.DPK_N, "seed": PT.DPK_SEED, "x_sha256": inputs_sha(x), "eval": {}}
    for name in MODELS:
        e = res["eval"][name] = eval_entry(M, name, x)
        print(f"{name} L={LENGTH}: max |y| {e['y']['absmax']:.4g}, fp32 - float64 {e['dev']:.3g}, "
              f"well-posed picks {int(e['well_posed'].sum())}/{2 * PT.DPK_N}", flush=True)
    torch.save(res, FIXTURE)
    print("->", FIXTURE, os.path.getsize(FIXTURE) // 1024, "KiB")


if __name__ == "__main__":
    main()
