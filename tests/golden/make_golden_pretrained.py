"""Generate tests/golden/reference_pretrained.pt by executing the UNMODIFIED reference (a SeisT checkout,
SEIST_REFERENCE_ROOT) on its own trained checkpoints (`pretrained/*.pth`).

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_pretrained.py

The inputs are regenerated from seeds by oracle/pretrained.py (event windows, not white noise) and not stored.

"eval", for each of the 18 checkpoints (`<name>_<dataset>`): the file's SHA-256 and state-dict layout digest, the
reference's float64 eval output (`model.double()`) as a float64 sample, `dev` = max |fp32 output - float64 output| of
the reference itself (its own rounding scale), and for the pickers
  * pick: the arg max of the P and S rows; well_posed: the top value beats every other value of its row by >= 1e-5;
  * det_above / det_amb: detection row > 0.5, and within 2e-3 of 0.5 (as make_golden.py);
  * peaks[topk]: `_detect_peaks` of the P and S rows (oracle/postprocess_ref.py, pinned to the reference's own function)
    at ContinuousAnnotator's threshold and min_peak_dist; peaks_amb: a (trace, phase) where a peak candidate lies
    within 1e-5 of the threshold, of a neighbouring sample or of another candidate's height, where float rounding
    may change the picks.
"step", for oracle/pretrained.STEP_MODELS: one fine-tuning step from the checkpoint (make_golden.fixture: train mode,
drop rates zeroed, the head's default loss): loss, train output, parameter gradients and post-step BN buffers.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import golden as G  # noqa: E402
from oracle import postprocess_ref as PP  # noqa: E402
from oracle import pretrained as PT  # noqa: E402
from oracle import reference_import as ri  # noqa: E402
import make_golden  # noqa: E402

AMB = 1e-5


def peaks_ambiguous(x, thr=PT.THRESHOLD, tol=AMB):
    """Whether rounding at the scale `tol` may change `_detect_peaks` of row x (float64)."""
    x = np.asarray(x, dtype=np.float64)
    mid, lo, hi = x[1:-1], x[:-2], x[2:]
    near = (mid >= lo - tol) & (mid >= hi - tol) & (mid >= thr - tol)
    close = (np.abs(mid - lo) < tol) | (np.abs(mid - hi) < tol) | (np.abs(mid - thr) < tol)
    if (near & close).any():
        return True
    h = np.sort(mid[near & (mid > lo) & (mid >= hi)])
    return bool(h.size > 1 and (np.diff(h) < tol).any())


def well_posed(row, tol=AMB):
    top2 = torch.topk(row, 2).values
    return bool(top2[0] - top2[1] >= tol)


def eval_entry(M, name, dataset):
    path = os.path.join(ri.REF_ROOT, "pretrained", f"{name}_{dataset}.pth")
    sd = PT.read_checkpoint(path)
    model = M.create_model(name, in_channels=3, in_samples=PT.WINDOW)
    model.load_state_dict(sd, strict=True)
    model.eval()
    x = PT.inputs(name)
    with torch.no_grad():
        y32 = model(x)
        y64 = model.double()(x.double())
    out = {"sha256": PT.sha256(path), "layout_sha": G.digest(G.layout(sd)), "y": PT.sample64(y64, 8192, seed=7),
           "dev": (y32.double() - y64).abs().max().item()}
    if name.endswith("dpk"):
        det = y64[:, 0]
        out["pick"] = y64[:, 1:].argmax(-1)
        out["well_posed"] = torch.tensor([[well_posed(y64[n, c]) for c in (1, 2)] for n in range(x.shape[0])])
        out["det_above"] = torch.from_numpy(np.packbits((det > 0.5).numpy(), axis=-1))
        out["det_amb"] = torch.from_numpy(np.packbits(((det - 0.5).abs() < 2e-3).numpy(), axis=-1))
        out["peaks"] = {topk: [[PP.detect_peaks_topk(y64[n, c].numpy(), PT.THRESHOLD, PT.MIN_PEAK_DIST, topk).tolist()
                                for c in (1, 2)] for n in range(x.shape[0])] for topk in PT.TOPKS}
        out["peaks_amb"] = torch.tensor([[peaks_ambiguous(y64[n, c].numpy()) for c in (1, 2)] for n in range(x.shape[0])])
    return out


def step_entry(M, name):
    sd = PT.read_checkpoint(os.path.join(ri.REF_ROOT, "pretrained", f"{name}_diting.pth"))
    x = PT.inputs(name)
    out = make_golden.fixture(M, name, x.shape[0], PT.WINDOW, sd=sd, x=x, tgt=PT.step_target(name, x), ks=(4096, 64, 64))
    return {k: out[k] for k in ("batch", "length", "layout_sha", "param_sha", "y_shape", "y_train", "loss", "grads",
                                "buffers_after")}


def main():
    M = ri.import_reference_models()
    torch.set_num_threads(8)
    res = {"eval": {}, "step": {}}
    for name, dataset in PT.CHECKPOINTS:
        e = res["eval"][f"{name}_{dataset}"] = eval_entry(M, name, dataset)
        print(f"{name}_{dataset}: max |y| {e['y'].get('absmax'):.4g}, fp32 - float64 {e['dev']:.3g}"
              + (f", well-posed picks {int(e['well_posed'].sum())}/16, unambiguous peak rows "
                 f"{int((~e['peaks_amb']).sum())}/16" if name.endswith("dpk") else ""), flush=True)
    for name in PT.STEP_MODELS:
        res["step"][name] = step_entry(M, name)
        print(f"{name} step: loss {res['step'][name]['loss'].item():.6g}", flush=True)
    torch.save(res, PT.FIXTURE)
    print("->", PT.FIXTURE, os.path.getsize(PT.FIXTURE) // 1024, "KiB")


if __name__ == "__main__":
    main()
