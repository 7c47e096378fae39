"""Generate tests/golden/reference_augmentation.pt by executing the UNMODIFIED reference's `DataPreprocessor` class
(training/preprocess.py, extracted with `ast` with `_pad_phases` / `_pad_array`; a SeisT checkout at SEIST_REFERENCE_ROOT).

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_augmentation.py

For every case of tests/test_cpu_augment.py::cases() - configurations (main.py defaults, every rate at 1.0, generate-noise,
add-event with max_event_num 2 and 3, p_position_ratio 0.3, mask and noise windows, each norm mode, raw length below,
equal to and above in_samples) x events (one, two, P near either edge, two noise events) x (augmentation False, three
seeds with augmentation True) - it stores what `process(event, augmentation)` returned under `np.random.seed(seed)`:
`x` as oracle.golden.pack samples plus the maximum, the output phase lists whole, whether the event dict was cleared, and
`get_targets_for_metrics` for det / ppk / spk (None where the reference raises).  It also stores `_generate_soft_label`
with the sigmoid shape for tests/test_cpu_augment.py::sigmoid_cases().
"""
import ast
import copy
import os
import sys
import zlib
from operator import itemgetter
from typing import Any, List, Tuple, Union

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import golden as G  # noqa: E402
from oracle import reference_import as ri  # noqa: E402
import test_cpu_augment as TA  # noqa: E402


class _Logger:
    def warning(self, *a, **k):
        pass


def reference_preprocessor():
    ri.import_reference_models()            # puts the checkout on sys.path: its config.py imports models
    import config as ref_config
    path = os.path.join(ri.REF_ROOT, "training", "preprocess.py")
    tree = ast.parse(open(path).read())
    body = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef))
            and n.name in ("_pad_phases", "_pad_array", "DataPreprocessor")]
    ns = {"np": np, "Tuple": Tuple, "Union": Union, "List": List, "Any": Any, "itemgetter": itemgetter, "copy": copy,
          "logger": _Logger(), "Config": ref_config.Config}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)      # noqa: S102 - the reference's own code
    return ns["DataPreprocessor"]


def main():
    DP = reference_preprocessor()
    out = {"cases": TA.cases(), "ppks": [], "spks": [], "cleared": [], "metrics": []}
    xs = []
    for name, ei, seed in out["cases"]:
        cfg, _ = TA.config(name)
        pre = DP(**cfg)
        data, ppks, spks, snr = TA.case_input(name, ei)
        ev = {"data": data.copy(), "ppks": list(ppks), "spks": list(spks), "snr": snr.copy()}
        np.random.seed(0 if seed is None else seed)
        ev = pre.process(ev, augmentation=seed is not None)
        xs.append(torch.from_numpy(np.asarray(ev["data"]).astype(np.float32)))
        out["ppks"].append([int(v) for v in ev["ppks"]])
        out["spks"].append([int(v) for v in ev["spks"]])
        out["cleared"].append(len(ev["snr"]) == 0)
        try:
            tg = pre.get_targets_for_metrics(ev, max_event_num=cfg["max_event_num"], task_names=["det", "ppk", "spk"])
            out["metrics"].append({k: torch.from_numpy(np.asarray(v)) for k, v in tg.items()})
        except Exception:               # _pad_array: a phase list longer than max_event_num
            out["metrics"].append(None)
    out["x"] = G.pack(xs, 256, seed=7)
    pre = DP(**dict(TA.BASE, coda_ratio=2.0))
    rows = []
    for width, p, s in TA.sigmoid_cases():
        ev = {"data": np.zeros((3, TA.SIGMOID_L), np.float32), "ppks": list(p), "spks": list(s)}
        rows += [pre._generate_soft_label(row, ev, width, "sigmoid") for row in ("det", "ppk", "spk")]
    lab = np.stack(rows).astype(np.float32)
    out["sigmoid"] = {"shape": lab.shape, "deflated": torch.frombuffer(bytearray(zlib.compress(lab.tobytes(), 9)), dtype=torch.uint8)}
    path = os.path.join(HERE, "reference_augmentation.pt")
    torch.save(out, path)
    print("augmentation ->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
