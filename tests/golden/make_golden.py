"""Generate the tests/golden fixtures by executing the UNMODIFIED reference (a SeisT checkout, SEIST_REFERENCE_ROOT).

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden.py [model ...]

<model>.pt (oracle/golden.py reads them): the reference model with seeded parameters (oracle.golden.synth_state_dict)
on seeded synthetic inputs, all drop rates zeroed: eval output, train-mode output, loss, every parameter gradient and the
post-step BN running buffers, large tensors as seeded samples.

reference_functions.pt: what the reference's own code returns where the tests compare a restatement with it -
train-mode outputs of three more variants (test_cpu_oracle.py), the dropout sites and rates of the reference modules
(test_cpu_oracle.py), `_normalize` / `_generate_soft_label` of training/preprocess.py (test_cpu_preprocess.py) and
`_detect_peaks` of training/postprocess.py (test_cpu_postprocess.py).
"""
import ast
import os
import sys
import zlib
from types import SimpleNamespace
from typing import Any, List, Tuple, Union

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import golden as G  # noqa: E402
from oracle import reference_import as ri  # noqa: E402

ONLY = set(sys.argv[1:])      # model names and / or "functions": regenerate only these files


def fixture(M, name, n, length, sd=None, x=None, tgt=None, ks=(16384, 512, 512)):
    """The reference's results for model `name`: seeded parameters and inputs (G.synth_state_dict / G.synth_inputs)
    unless a state dict `sd` and inputs `x`, `tgt` are given.  `ks`: the sample sizes of the outputs, the parameter
    gradients and the buffers."""
    model = M.create_model(name, in_channels=3, in_samples=length)
    lay = G.layout(model.state_dict())
    blob = torch.load(os.path.join(ri.REF_ROOT, "pretrained", f"{name}_diting.pth"), map_location="cpu")
    assert G.layout(blob.get("model_dict", blob)) == lay              # the shipped checkpoint has this layout
    if sd is None:
        sd = G.synth_state_dict(lay)
        assert G.layout(G.model_state_dict(name, length)) == lay      # load() rebuilds exactly these parameters
    model.load_state_dict(sd, strict=True)
    ri.zero_drop_rates(model)
    if x is None:
        x, tgt = G.synth_inputs(name, n, length)
    model.eval()
    with torch.no_grad():
        y_eval = model(x)
    model.train()
    y_train = model(x)
    if name.endswith("dpk"):
        loss = M.BCELoss(weight=[[0.5], [1], [1]])(y_train, tgt)
    elif name.endswith("pmp"):
        loss = M.CELoss(weight=[1, 1])(y_train, tgt)
    else:
        loss = M.HuberLoss()(y_train, tgt)
    loss.backward()
    out = {
        "model": name, "batch": n, "length": length, "layout_sha": G.digest(lay),
        "param_sha": G.digest([k for k, _ in model.named_parameters()]),
        "y_shape": tuple(y_eval.shape), "y_eval": G.pack([y_eval], ks[0], seed=1), "y_train": G.pack([y_train], ks[0], seed=2),
        "loss": loss.detach(),
        "grads": G.pack([p.grad for _, p in model.named_parameters()], ks[1], seed=1000),
        "buffers_after": G.pack([b for _, b in model.named_buffers()], ks[2], seed=3000),
    }
    if name.endswith("dpk"):
        det = y_eval[:, 0]
        out["pick"] = y_eval[:, 1:].argmax(-1)
        out["det_above"] = torch.from_numpy(np.packbits((det > 0.5).numpy(), axis=-1))
        out["det_amb"] = torch.from_numpy(np.packbits(((det - 0.5).abs() < 2e-3).numpy(), axis=-1))
    return out


def reference_sources(rel, fn_names, cls_name=None, cls_fns=()):
    path = os.path.join(ri.REF_ROOT, rel)
    tree = ast.parse(open(path).read())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in fn_names]
    if cls_name:
        cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name)
        body += [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in cls_fns]
    ns = {"np": np, "Tuple": Tuple, "Union": Union, "List": List, "Any": Any}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)      # noqa: S102 - the reference's own code
    return ns


def reference_functions(M):
    import test_cpu_oracle as TO
    import test_cpu_postprocess as TP
    import test_cpu_preprocess as TR
    out = {"modules": {}, "dropout_sites": {}}
    for name in TO.MODULE_MODELS:
        ref = ri.zero_drop_rates(M.create_model(name, in_channels=3, in_samples=TO.MODULE_L))
        lay = G.layout(ref.state_dict())
        assert G.layout(G.model_state_dict(name, TO.MODULE_L, seed=TO.MODULE_SEED)) == lay
        ref.load_state_dict(G.synth_state_dict(lay, seed=TO.MODULE_SEED), strict=True)
        ref.train()
        out["modules"][name] = G.pack([ref(TO.module_input())], 1024, seed=4)
    for name in TO.SITE_MODELS:
        ref = M.create_model(name, in_channels=3, in_samples=1024)
        sites = []
        for path, mod in ref.named_modules():
            cls = mod.__class__.__name__
            if cls == "Dropout":
                sites.append((path, float(mod.p)))
            elif cls == "DropPath":
                sites.append((path, float(mod.drop_prob or 0.0)))
        out["dropout_sites"][name] = sites
    ns = reference_sources("training/preprocess.py", ("_pad_phases",), "DataPreprocessor", ("_normalize", "_generate_soft_label"))
    x = TR.normalize_input()
    out["normalize"] = {mode: torch.from_numpy(ns["_normalize"](None, x.copy(), mode)) for mode in TR.MODES}
    for want in out["normalize"].values():
        assert want.dtype == torch.float32
    me = SimpleNamespace(coda_ratio=1.4, dtype=np.float32, data_channels=["z", "n", "e"])
    rows = []
    for shape, width, ppks, spks in TR.label_cases():
        ev = {"data": np.zeros((3, TR.LABEL_L), np.float32), "ppks": list(ppks), "spks": list(spks)}
        rows += [ns["_generate_soft_label"](me, row, ev, width, shape) for row in ("det", "ppk", "spk")]
    lab = np.stack(rows).astype(np.float32)          # mostly zeros and ones: stored deflated
    out["labels"] = {"shape": lab.shape, "deflated": torch.frombuffer(bytearray(zlib.compress(lab.tobytes(), 9)), dtype=torch.uint8)}
    detect_peaks = reference_sources("training/postprocess.py", ("_detect_peaks",))["_detect_peaks"]
    peaks = {}
    for topk, mpd in TP.CASES:
        x = TP.peak_traces(topk, mpd)
        for thr in TP.THRESHOLDS:      # one list of peak indices per trace
            peaks[(topk, mpd, thr)] = [[int(v) for v in detect_peaks(row, mph=thr, mpd=mpd, topk=topk)] for row in x]
    out["detect_peaks"] = peaks
    return out


def main():
    M = ri.import_reference_models()
    torch.manual_seed(0)
    torch.set_num_threads(8)
    for name, (n, length) in G.FIXTURES.items():
        if ONLY and name not in ONLY:
            continue
        path = os.path.join(HERE, f"{name}.pt")
        torch.save(fixture(M, name, n, length), path)
        print(name, "->", path, os.path.getsize(path) // 1024, "KiB")
    if not ONLY or "functions" in ONLY:
        path = os.path.join(HERE, "reference_functions.pt")
        torch.save(reference_functions(M), path)
        print("functions ->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
