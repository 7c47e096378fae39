"""Generate tests/golden/reference_continuous.pt by executing the UNMODIFIED reference's `_detect_peaks`
(training/postprocess.py, extracted with `ast` as make_golden.py::reference_sources does; a SeisT checkout at
SEIST_REFERENCE_ROOT) with topk=None on the long traces of tests/test_cpu_stream.py::long_traces().

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_continuous.py

Only the peak indices are stored (per (mph, mpd) case of test_cpu_stream.CONT_CASES, one list per row); the traces are
regenerated from their seed.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
from make_golden import reference_sources  # noqa: E402
import test_cpu_stream as TS  # noqa: E402


def main():
    detect_peaks = reference_sources("training/postprocess.py", ("_detect_peaks",))["_detect_peaks"]
    x = TS.long_traces()
    peaks = {}
    for mph, mpd in TS.CONT_CASES:
        peaks[(mph, mpd)] = [[int(v) for v in detect_peaks(row, mph=mph, mpd=mpd, topk=None)] for row in x]
    path = os.path.join(HERE, "reference_continuous.pt")
    torch.save({"length": TS.CONT_L, "seed": TS.SEED, "detect_peaks": peaks}, path)
    print("continuous ->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
