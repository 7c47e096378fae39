"""Generate tests/golden/reference_peak_ties.pt by executing the UNMODIFIED reference's `_detect_peaks`
(training/postprocess.py, extracted with `ast` as make_golden.py::reference_sources does; a SeisT checkout at
SEIST_REFERENCE_ROOT) on the tie-rich and NaN traces of tests/peak_ties.py, with `np.argsort` made stable.

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_peak_ties.py

The reference orders equal heights by numpy's default (unstable) sort; with a stable one, equal heights keep their
ascending index order before the reversal, so the larger index ranks first: the rule the oracle and the device pickers
implement.  Everything but `argsort` passes through to numpy (`in1d` is aliased to `isin` where numpy has dropped it).
Only the seeds, parameters and peak indices are stored; the traces are regenerated from their seed.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
from make_golden import reference_sources  # noqa: E402
import peak_ties as PT  # noqa: E402


class _StableNumpy(types.ModuleType):
    def __init__(self, stable: bool):
        super().__init__("numpy")
        self.stable = stable

    def __getattr__(self, name):
        if name == "in1d" and not hasattr(np, "in1d"):
            return np.isin
        return getattr(np, name)

    def argsort(self, a, *args, **kwargs):
        if self.stable:
            kwargs["kind"] = "stable"
        return np.argsort(a, *args, **kwargs)


def detect_peaks(stable: bool):
    ns = reference_sources("training/postprocess.py", ("_detect_peaks",))
    ns["np"] = _StableNumpy(stable)          # the function's globals: its `np.` lookups go through the shim
    return ns["_detect_peaks"]


def main():
    stable, default = detect_peaks(True), detect_peaks(False)
    cases, differ = [], 0
    for mph, mpd, topk in PT.FIXTURE_PARAMS:
        for seed, L, nan, x in PT.fixture_traces(mpd):
            with np.errstate(invalid="ignore"):
                got = [int(v) for v in stable(x.copy(), mph=mph, mpd=mpd, topk=topk)]
                differ += got != [int(v) for v in default(x.copy(), mph=mph, mpd=mpd, topk=topk)]
            cases.append({"seed": seed, "L": L, "nan": nan, "mph": mph, "mpd": mpd, "topk": topk, "peaks": got})
    path = os.path.join(HERE, "reference_peak_ties.pt")
    torch.save({"cases": cases}, path)
    print(f"peak ties -> {path} {os.path.getsize(path) // 1024} KiB: {len(cases)} cases, {differ} differ under numpy's default sort")


if __name__ == "__main__":
    main()
