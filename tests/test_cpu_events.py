"""P-anchored event windows (DESIGN §4.17): oracle/event_ref.py against what the unmodified reference's
`DataPreprocessor._cut_window` (0 <= p_position_ratio <= 1) and `_normalize` computed (tests/golden/
reference_event_windows.pt, written by make_golden_event_windows.py), bit for bit; the anchor arithmetic; the CSR walk."""
import os

import numpy as np
import pytest
import torch

from oracle import event_ref as ER
from oracle import golden as G

EW_W = 2048                       # window of the fixture
EW_T, EW_TS = 6000, 1500          # a record longer and one shorter than the window
EW_C = 3
RATIOS = (0.0, 0.25, 0.3, 1.0)
MODES = ("std", "max", "")
SEED = 20261016
CONST = 2.5                       # station 1, channel 2 of the long record: zero scale -> 1


def records():
    """{"long": (2, C, EW_T), "short": (1, C, EW_TS)} float32 numpy, seeded; offsets and gains differ per channel."""
    g = torch.Generator().manual_seed(SEED)
    out = {}
    for name, S, T in (("long", 2, EW_T), ("short", 1, EW_TS)):
        x = torch.randn(S, EW_C, T, generator=g) * (0.5 + 10 * torch.rand(S, EW_C, 1, generator=g)) + torch.randn(S, EW_C, 1, generator=g)
        out[name] = x.numpy().astype(np.float32)
    out["long"][1, 2, :] = CONST
    return out


def positions(T, W, a):
    """P picks at 0, 1, a - 1, a, mid-record, T - W + a, T - 2 and T - 1 (those inside [0, T), each once)."""
    return list(dict.fromkeys(p for p in (0, 1, a - 1, a, T // 2, T - W + a, T - 2, T - 1) if 0 <= p < T))


def cases():
    """[(record, station, p_position_ratio, p, norm mode)] in the order of the fixture."""
    out = []
    for rec, S, T in (("long", 2, EW_T), ("short", 1, EW_TS)):
        i = 0
        for r in RATIOS:
            for p in positions(T, EW_W, ER.anchor(EW_W, r)):
                for mode in MODES:
                    out.append((rec, i % S, r, p, mode))
                    i += 1
    out += [("long", 1, 0.3, EW_T // 2, mode) for mode in MODES]       # the constant channel wholly inside the window
    return out


@pytest.fixture(scope="module")
def golden():
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_event_windows.pt"))
    assert g["cases"] == cases() and g["window"] == EW_W
    return g


def test_anchor_is_the_references_int_of_the_product():
    assert ER.anchor(8192, 0.3) == 2457                 # 8192 * 0.3 = 2457.6
    assert ER.anchor(EW_W, 0.3) == 614 and ER.anchor(EW_W, 0.25) == 512
    assert ER.anchor(EW_W, 0.0) == 0 and ER.anchor(EW_W, 1.0) == EW_W
    from seist_b200 import events
    assert events.anchor(8192, 0.3) == 2457 and events.anchor(3000, 0.7) == int(3000 * 0.7)


def test_oracle_equals_reference_fixture_bit_for_bit(golden):
    recs = records()
    samples = G.unpack(golden["x"], [(EW_C, EW_W)] * len(cases()))
    for case, smp in zip(cases(), samples):
        rec, s, r, p, mode = case
        got = torch.from_numpy(ER.window(recs[rec][s], p, EW_W, r, mode))
        assert smp.err(got) == 0.0, case
        assert got.abs().max().item() == smp.absmax, case


def test_fixture_covers_zero_fill_and_the_constant_channel():
    recs = records()
    a = ER.anchor(EW_W, 0.3)
    both = ER.cut(recs["short"][0], a - 1, EW_W, a)                      # T < W: zeros on both sides
    assert (both[:, 0] == 0).all() and (both[:, -1] == 0).all() and (both[:, 1:EW_TS] != 0).all()
    flat = ER.window(recs["long"][1], EW_T // 2, EW_W, 0.3, "std")
    assert (flat[2] == 0).all()                                          # constant channel: centred, scale 1
    first = ER.cut(recs["long"][0], 0, EW_W, EW_W)                       # ratio 1.0, p = 0: the pick falls at sample W
    assert (first == 0).all()


def test_windows_walk_the_csr_and_zero_out_of_range_picks():
    rec = records()["long"]
    index = np.array([5, 3000, 4000, -1, EW_T])                         # station 0: 2 picks, station 1: 3 (two invalid)
    offsets = np.array([0, 2, 5])
    x = ER.windows(rec, index, offsets, EW_W, 0.25, "max")
    assert np.array_equal(x[1], ER.window(rec[0], 3000, EW_W, 0.25, "max"))
    assert np.array_equal(x[2], ER.window(rec[1], 4000, EW_W, 0.25, "max"))
    assert (x[3] == 0).all() and (x[4] == 0).all()
    assert ER.windows(rec, index[:0], np.zeros(3, np.int64), EW_W, 0.25, "max").shape == (0, EW_C, EW_W)
