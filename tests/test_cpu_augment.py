"""not-gpu: the augmentation oracle (tests/augment_ref.py) against what the reference's own `DataPreprocessor.process`,
`_generate_soft_label` (sigmoid) and `get_targets_for_metrics` returned (tests/golden/reference_augmentation.pt, written
by tests/golden/make_golden_augmentation.py); the device's counter draws at the reference's rates and ranges; the torch
metric-target helper against the oracle."""
import math
import os
import zlib

import numpy as np
import pytest
import torch

import augment_ref as AR
from oracle import golden as G
from seist_b200 import preprocess as PP

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_augmentation.pt")

BASE = dict(data_channels=["z", "n", "e"], sampling_rate=50, in_samples=8192, min_snr=-float("inf"), p_position_ratio=-1,
            coda_ratio=2.0, norm_mode="std", add_event_rate=0.0, add_noise_rate=0.4, add_gap_rate=0.4,
            drop_channel_rate=0.4, scale_amplitude_rate=0.4, pre_emphasis_rate=0.4, pre_emphasis_ratio=0.97,
            max_event_num=1, generate_noise_rate=0.05, shift_event_rate=0.2, mask_percent=0, noise_percent=0,
            min_event_gap_sec=0.5, soft_label_shape="gaussian", soft_label_width=25)        # main.py defaults, 50 Hz
ALL_ON = dict(add_event_rate=1.0, shift_event_rate=1.0, drop_channel_rate=1.0, scale_amplitude_rate=1.0,
              pre_emphasis_rate=1.0, add_noise_rate=1.0, add_gap_rate=1.0, generate_noise_rate=0.0, max_event_num=2,
              in_samples=4096)
CONFIGS = {  # name: (overrides of BASE, raw length)
    "default": ({}, 9000),
    "all_on": (ALL_ON, 4600),
    "generate_noise": (dict(generate_noise_rate=1.0, drop_channel_rate=1.0, scale_amplitude_rate=1.0, in_samples=4096), 4600),
    "add3": (dict(add_event_rate=1.0, max_event_num=3, in_samples=4096, min_event_gap_sec=0.2), 4600),
    "p_position": (dict(ALL_ON, p_position_ratio=0.3), 4600),
    "windows": (dict(mask_percent=10, noise_percent=10, in_samples=4096), 4600),
    "norm_max": (dict(ALL_ON, norm_mode="max"), 4600),
    "norm_none": (dict(norm_mode=""), 9000),
    "lin_below": (ALL_ON, 3000),
    "lin_equal": (ALL_ON, 4096),
}
SEEDS = (None, 1, 2, 3)         # None: augmentation=False (under seed 0)


def config(name):
    over, lin = CONFIGS[name]
    return dict(BASE, **over), lin


def events(lin):
    """(ppks, spks) of the golden events for a raw length."""
    p = int(lin * 0.3)
    return [([p], [p + 400]), ([500, int(lin * 0.6)], [900, int(lin * 0.6) + 300]), ([3], [200]), ([lin - 300], [lin - 20]),
            ([], []), ([800], [700])]


def raw(ci, ei, lin, ppks):
    rng = np.random.default_rng(1000 + 10 * ci + ei)
    x = rng.standard_normal((3, lin)) * rng.uniform(0.5, 20, (3, 1)) + rng.uniform(-3, 3, (3, 1))
    for p in ppks:
        x[:, p:p + 300] *= 6.0
    return x.astype(np.float32)


def cases():
    """[(config name, event index, seed)] in the order of the fixture.  Under p_position_ratio the reference raises for
    the noise events (no P pick to place), so they are not cases there."""
    return [(name, ei, seed) for name in CONFIGS for ei in range(len(events(CONFIGS[name][1]))) for seed in SEEDS
            if not (name == "p_position" and ei >= 4)]


def case_input(name, ei):
    ci = list(CONFIGS).index(name)
    lin = CONFIGS[name][1]
    ppks, spks = events(lin)[ei]
    return raw(ci, ei, lin, ppks), ppks, spks, np.array([10.0, 10.0, 10.0])


SIGMOID_L = 2048


def sigmoid_cases():
    cases_ = [([300], [700]), ([5], [60]), ([1900], [2040]), ([], []), ([100, 900], [400, 1300]), ([2047], [2047 + 30]),
              ([0], [3])]
    return [(width, p, s) for width in (25, 50, 11, 2, 3) for p, s in cases_]


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def test_oracle_reproduces_reference_process(gold):
    cs = cases()
    assert gold["cases"] == cs
    shapes = [(3, config(name)[0]["in_samples"]) for name, _, _ in cs]
    xs = G.unpack(gold["x"], shapes)
    for i, (name, ei, seed) in enumerate(cs):
        cfg, _ = config(name)
        pre = AR.Preprocessor(**cfg)
        data, ppks, spks, snr = case_input(name, ei)
        np.random.seed(0 if seed is None else seed)
        x, po, so, cleared = pre.process(data, ppks, spks, snr, seed is not None, AR.NumpyDraws())
        assert xs[i].err(torch.from_numpy(x)) == 0.0 and np.abs(x).max() == np.float32(xs[i].absmax), (name, ei, seed)
        assert po == gold["ppks"][i] and so == gold["spks"][i] and cleared == gold["cleared"][i], (name, ei, seed)
        want = gold["metrics"][i]
        if want is None:
            with pytest.raises(ValueError):
                pre.metric_targets(po, so)
        else:
            got = pre.metric_targets(po, so)
            for k in ("det", "ppk", "spk"):
                assert np.array_equal(got[k], want[k].numpy()), (name, ei, seed, k)


def test_sigmoid_labels_match_reference(gold):
    lab = gold["sigmoid"]
    want = np.frombuffer(zlib.decompress(lab["deflated"].numpy().tobytes()), np.float32).reshape(lab["shape"])
    for i, (width, p, s) in enumerate(sigmoid_cases()):
        got = AR.dpk_labels(p, s, SIGMOID_L, width, "sigmoid", 2.0)
        for row in range(3):
            assert np.array_equal(got[row], want[3 * i + row]), (width, p, s, row)


def _within(count, n, p):
    return abs(count - n * p) <= 4 * math.sqrt(n * p * (1 - p)) + 1e-9


def test_counter_draws_rates_and_ranges():
    """>= 20000 traces at the default rates (small traces: the draws do not depend on the sample values)."""
    cfg = dict(BASE, in_samples=1024)
    pre = AR.Preprocessor(**cfg)
    pre.log = {}
    n, lin, seed = 20000, 1200, 987654321
    data = np.ones((3, lin), np.float32)
    for t in range(n):
        p = 100 + (t * 37) % 800
        pre.process(data, [p], [p + 150], None, True, AR.CounterDraws(seed, t, 3))
    log = pre.log
    g = len(log.get("generate_noise", []))
    assert _within(g, n, 0.05)
    assert _within(len(log["drop_channel"]), n, 0.4)
    assert _within(len(log["scale"]), n, 0.4)
    assert _within(len(log["shift"]), n, 0.95 * 0.2)
    assert _within(len(log["pre_emphasis"]), n, 0.95 * 0.4)
    assert _within(len(log["snr"]) // 3, n, 0.95 * 0.4)
    assert _within(len(log["gap"]), n, 0.95 * 0.4)
    assert all(0 <= v < lin for v in log["shift"])
    assert all(1.0 <= v < 3.0 for v in log["scale"])
    snr = np.array(log["snr"])
    assert snr.min() == 10 and snr.max() == 49
    assert all(lo <= a <= b <= hi and a < hi for a, b, lo, hi in log["gap"])
    assert all(0 <= c < hi for c, hi in log["cut"]) and len(log["cut"]) == n
    assert max(c for c, _ in log["cut"]) > 0.9 * max(hi for _, hi in log["cut"])


def test_counter_draws_add_event_and_windows():
    cfg = dict(BASE, in_samples=1024, add_event_rate=0.5, max_event_num=3, mask_percent=20, noise_percent=10)
    pre = AR.Preprocessor(**cfg)
    pre.log = {}
    n, lin = 4000, 4000
    data = np.ones((3, lin), np.float32)
    grown = 0
    for t in range(n):
        d = AR.CounterDraws(5, t, 3)
        _, po, _, cleared = pre.process(data, [300], [400], None, True, d)
        grown += len(pre.log.get("add_event", [])) > 0
        pre.log.pop("add_event", None)
    assert grown > 0.5 * n                      # two chances at rate 0.5 (the window can be too short for a second)
    d = AR.CounterDraws(5, 0, 3)
    sel = d.windows(80, 16)
    assert len(sel) == 16 and sel == sorted(set(sel)) and 0 <= sel[0] and sel[-1] < 80


def test_counter_normals_mean_and_variance():
    z = AR.counter_normal(42, AR.STREAM_NORMAL + AR.NOISE_ADD, np.arange(1 << 20, dtype=np.uint64))
    n = z.size
    assert abs(z.mean()) <= 4 / math.sqrt(n)
    assert abs(z.var() - 1.0) <= 4 * math.sqrt(2.0 / n)


def test_metric_target_helper_matches_oracle(gold):
    """seist_b200.preprocess.metric_targets (torch, here on CPU tensors) against the oracle on the fixture's outputs."""
    for i, (name, ei, seed) in enumerate(cases()):
        cfg, _ = config(name)
        pre = AR.Preprocessor(**cfg)
        po, so = gold["ppks"][i], gold["spks"][i]
        k = max(1, len(po), len(so))
        pt = torch.tensor([po + [PP.ABSENT] * (k - len(po))])
        st = torch.tensor([so + [PP.ABSENT] * (k - len(so))])
        got = PP.metric_targets(pt, st, cfg["max_event_num"], cfg["soft_label_width"], cfg["in_samples"], cfg["coda_ratio"],
                                pre.expected_det_num())
        if gold["metrics"][i] is None:
            continue
        want = pre.metric_targets(po, so)
        w = len(want["ppk"])
        assert np.array_equal(got["ppk"][0, :w].numpy(), want["ppk"]) and (got["ppk"][0, w:] == PP.ABSENT).all()
        assert np.array_equal(got["spk"][0, :w].numpy(), want["spk"])
        wd = len(want["det"])
        assert np.array_equal(got["det"][0, :wd].numpy(), want["det"]), (name, ei, seed)
        assert (got["det"][0, wd:].view(-1, 2) == torch.tensor([1, 0])).all()


def test_device_preprocessor_config_from_reference_arguments():
    from types import SimpleNamespace
    args = SimpleNamespace(in_samples=8192, min_snr=-float("inf"), coda_ratio=2.0, norm_mode="std", p_position_ratio=0.25,
                           add_event_rate=0.3, add_noise_rate=0.4, add_gap_rate=0.4, drop_channel_rate=0.4,
                           scale_amplitude_rate=0.4, pre_emphasis_rate=0.4, pre_emphasis_ratio=0.97, max_event_num=2,
                           generate_noise_rate=0.05, shift_event_rate=0.2, mask_percent=0, noise_percent=0,
                           min_event_gap=0.5, label_shape="sigmoid", label_width=0.5)
    dp = PP.DevicePreprocessor.from_args(args, 100, ["z", "n", "e"])
    assert dp.min_event_gap == 50 and dp.soft_label_width == 50 and dp.soft_label_shape == "sigmoid"
    assert dp.add_event_rate == dp.shift_event_rate == dp.generate_noise_rate == 0.0       # p_position_ratio in [0, 1]
    assert dp.expected_det_num() == 3
    with pytest.raises(ValueError):
        PP.DevicePreprocessor(["z"], 50, 1024, max_event_num=9)
