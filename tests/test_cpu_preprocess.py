"""not-gpu: the input-side oracle (oracle/preprocess_ref.py) against what the reference's own `_normalize` and
`_generate_soft_label` (training/preprocess.py) returned for the same inputs (tests/golden/reference_functions.pt,
written by tests/golden/make_golden.py)."""
import os
import zlib

import numpy as np
import torch

from oracle import preprocess_ref as PR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_functions.pt")
MODES = ("std", "max", "")
LABEL_L = 2048


def normalize_input():
    x = np.random.default_rng(0).standard_normal((3, 1024)).astype(np.float32) * 3 + 1
    x[1] = 2.5                                                   # constant channel: scale 0 -> 1
    return x


def label_cases():
    cases = [([300], [700]), ([5], [60]), ([1900], [2040]), ([], []), ([100, 900], [400, 1300]), ([800], []), ([], [500]),
             ([2047], [2047 + 30]), ([0], [3])]
    return [(shape, width, ppks, spks) for shape in ("gaussian", "triangle", "box") for width in (25, 50, 11)
            for ppks, spks in cases]


def test_input_side_oracle_matches_reference_sources():
    ref = torch.load(GOLD)
    x = normalize_input()
    for mode in MODES:
        assert np.array_equal(PR.normalize(x, mode), ref["normalize"][mode].numpy()), mode
    lab = ref["labels"]
    want = np.frombuffer(zlib.decompress(lab["deflated"].numpy().tobytes()), np.float32).reshape(lab["shape"])
    for i, (shape, width, ppks, spks) in enumerate(label_cases()):
        got = PR.dpk_labels(ppks, spks, LABEL_L, width, shape, 1.4)
        for row, name in enumerate(("det", "ppk", "spk")):
            assert np.array_equal(got[row], want[3 * i + row]), (shape, width, ppks, spks, name)
