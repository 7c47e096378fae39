"""Generate tests/golden/reference_event_windows.pt by executing the UNMODIFIED reference's `DataPreprocessor._cut_window`
(with 0 <= p_position_ratio <= 1) and `_normalize` (training/preprocess.py, extracted with `ast` as
make_golden_augmentation.py does; a SeisT checkout at SEIST_REFERENCE_ROOT) on the seeded records of
tests/test_cpu_events.py, one event (ppks=[p], spks=[]) per case of test_cpu_events.cases().

    SEIST_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_event_windows.py

Only data is stored: the windows as oracle.golden.pack samples plus their maxima; the records are regenerated from their
seed.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
from make_golden_augmentation import reference_preprocessor  # noqa: E402
from oracle import golden as G  # noqa: E402
import test_cpu_augment as TA  # noqa: E402
import test_cpu_events as TE  # noqa: E402


def main():
    DP = reference_preprocessor()
    recs = TE.records()
    xs = []
    for rec, s, r, p, mode in TE.cases():
        pre = DP(**dict(TA.BASE, in_samples=TE.EW_W, p_position_ratio=r, norm_mode=mode))
        data, _, _ = pre._cut_window(recs[rec][s].copy(), [p], [], TE.EW_W)
        data = pre._normalize(data, mode)
        xs.append(torch.from_numpy(data.copy()))
    out = {"window": TE.EW_W, "cases": TE.cases(), "x": G.pack(xs, 64, seed=11)}
    path = os.path.join(HERE, "reference_event_windows.pt")
    torch.save(out, path)
    print("event windows ->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
