"""-m gpu: the device augmentation pipeline (seist_augment through DevicePreprocessor) against the oracle with the device's
counter draws (tests/augment_ref.py::CounterDraws, pinned to the reference's own process in test_cpu_augment.py), the
sigmoid soft labels, the metric targets and CUDA-graph replay.  Floating point: 2e-6 x max |x|, labels 2e-6."""
import math

import numpy as np
import pytest
import torch

import augment_ref as AR
import test_cpu_augment as TA
from seist_b200 import preprocess as PP

pytestmark = pytest.mark.gpu
A = PP.ABSENT


def _pad(lists, k):
    return torch.tensor([list(v) + [A] * (k - len(v)) for v in lists], dtype=torch.int64)


def _device(cfg):
    return PP.DevicePreprocessor(**{k: v for k, v in cfg.items()})


def _check_batch(cfg, data, ppks, spks, snr, augment, label_shapes=("gaussian",)):
    dp = _device(cfg)
    k = max(1, max(len(p) for p in ppks), max(len(s) for s in spks))
    dp._seed_on(torch.device("cuda"))
    seed = int(dp.seed.item())
    x, po, so, cl = dp.process_batch(torch.from_numpy(np.stack(data)).cuda(), _pad(ppks, k).cuda(), _pad(spks, k).cuda(),
                                     torch.from_numpy(np.stack(snr)).cuda(), torch.tensor(augment).cuda())
    assert int(dp.seed.item()) == seed + 1
    x, po, so, cl = x.cpu().numpy(), po.cpu(), so.cpu(), cl.cpu().numpy()
    pre = AR.Preprocessor(**cfg)
    for n in range(len(data)):
        want, wp, ws, wc = pre.process(data[n], ppks[n], spks[n], snr[n], augment[n], AR.CounterDraws(seed, n, data[n].shape[0]))
        gp = [int(v) for v in po[n] if v > A]
        gs = [int(v) for v in so[n] if v > A]
        assert (gp, gs, bool(cl[n])) == (wp, ws, wc), (n, gp, wp, gs, ws)
        err = np.abs(x[n] - want).max()
        assert err <= 2e-6 * max(1.0, np.abs(want).max()), (n, err, np.abs(want).max())
        for shape in label_shapes:
            lab = PP.dpk_soft_labels(po[n:n + 1].cuda(), so[n:n + 1].cuda(), cfg["in_samples"], cfg["soft_label_width"], shape,
                                     cfg["coda_ratio"]).cpu().numpy()[0]
            wl = AR.dpk_labels(wp, ws, cfg["in_samples"], cfg["soft_label_width"], shape, cfg["coda_ratio"])
            assert np.abs(lab - wl).max() <= 2e-6, (n, shape)
    return po, so


@pytest.mark.parametrize("name", list(TA.CONFIGS))
def test_golden_configurations_match_oracle(name):
    cfg, lin = TA.config(name)
    data, ppks, spks, snr, aug = [], [], [], [], []
    for ei in range(len(TA.events(lin))):
        d, p, s, r = TA.case_input(name, ei)
        for flag in (False, True, True):
            data.append(d)
            ppks.append(p)
            spks.append(s)
            snr.append(r)
            aug.append(flag)
    _check_batch(cfg, data, ppks, spks, snr, aug, ("gaussian", "sigmoid"))


def test_default_rates_batch_512():
    cfg = dict(TA.BASE)
    rng = np.random.default_rng(3)
    data = list((rng.standard_normal((512, 3, 9000)) * rng.uniform(0.5, 20, (512, 3, 1))).astype(np.float32))
    p = rng.integers(300, 7000, 512)
    ppks = [[int(v)] for v in p]
    spks = [[int(v + rng.integers(50, 1500))] for v in p]
    ppks[7], spks[7] = [], []                                   # a noise trace
    snr = [np.array([10.0, 10.0, 10.0])] * 512
    aug = [i >= 256 for i in range(512)]                          # the reference augments the second half
    po, so = _check_batch(cfg, data, ppks, spks, snr, aug)
    dp = _device(cfg)
    tg = dp.metric_targets(po.cuda(), so.cuda())
    ref = PP.metric_targets(po, so, 1, 25, 8192, 2.0, dp.expected_det_num())
    for k in ("det", "ppk", "spk"):
        assert torch.equal(tg[k].cpu(), ref[k]), k


def test_counter_normals_on_device():
    """Noise windows over every sample, no other branch, no normalisation: x is the counter normals less their mean."""
    cfg = dict(TA.BASE, noise_percent=100, drop_channel_rate=0.0, scale_amplitude_rate=0.0, pre_emphasis_rate=0.0,
               add_noise_rate=0.0, add_gap_rate=0.0, generate_noise_rate=0.0, shift_event_rate=0.0, norm_mode="",
               in_samples=16000)
    dp = _device(cfg)
    n = 24
    data = torch.zeros(n, 3, 16000, device="cuda")
    p = torch.full((n, 1), 100, dtype=torch.int64, device="cuda")
    dp._seed_on(torch.device("cuda"))
    seed = int(dp.seed.item())
    x, *_ = dp.process_batch(data, p, p + 50)
    z = x.double().cpu().numpy().reshape(-1)
    assert z.size >= 10 ** 6
    assert abs(z.var() - 1.0) <= 4 * math.sqrt(2.0 / z.size)
    want = AR.counter_normal(seed, AR.STREAM_NORMAL + AR.NOISE_WINDOW, AR.normal_index(0, 3, np.arange(3)[:, None],
                                                                                           np.arange(16000)[None, :]))
    want = (want.astype(np.float32) - want.astype(np.float32).mean(1, keepdims=True))
    assert np.abs(x[0].cpu().numpy() - want).max() < 1e-5
    raw = AR.counter_normal(seed, AR.STREAM_NORMAL + AR.NOISE_WINDOW, np.arange(1 << 20, dtype=np.uint64))
    assert abs(raw.mean()) <= 4 / math.sqrt(raw.size)


def test_graph_replay_draws_new_augmentations():
    cfg = dict(TA.BASE, **TA.ALL_ON)
    dp = _device(cfg)
    rng = np.random.default_rng(9)
    data = torch.from_numpy(rng.standard_normal((16, 3, 4600)).astype(np.float32)).cuda()
    p = torch.from_numpy(rng.integers(300, 3000, (16, 1))).cuda()
    s = p + 200
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                                 # warm-up outside the capture
        dp.process_batch(data, p, s)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        x, po, so, cl = dp.process_batch(data, p, s)
        lab = dp.labels(po, so)
    outs, seeds = [], []
    for _ in range(2):
        seeds.append(int(dp.seed.item()))
        g.replay()
        torch.cuda.synchronize()
        outs.append([t.clone() for t in (x, po, so, cl, lab)])
    assert seeds[1] == seeds[0] + 1
    assert not torch.equal(outs[0][0], outs[1][0])
    for seed, got in zip(seeds, outs):
        dp.load_state_dict({"seed": seed})
        ex = dp.process_batch(data, p, s)
        want = list(ex) + [dp.labels(ex[1], ex[2])]
        for a, b in zip(got, want):
            assert torch.equal(a, b)


def test_bad_inputs_raise():
    dp = _device(dict(TA.BASE))
    p = torch.full((2, 1), 100, dtype=torch.int64)
    with pytest.raises(RuntimeError):
        dp.process_batch(torch.zeros(2, 3, 9000), p, p + 10)
    with pytest.raises(ValueError):
        dp.process_batch(torch.zeros(2, 3, 16385, device="cuda"), p.cuda(), p.cuda() + 10)
    k9 = torch.full((2, 9), A, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        dp.process_batch(torch.zeros(2, 3, 9000, device="cuda"), k9, k9)
    with pytest.raises(ValueError):
        PP.dpk_soft_labels(p.cuda(), p.cuda() + 10, 1024, 1, "sigmoid")
    st = dp.state_dict()
    assert st["seed"] is None or isinstance(st["seed"], int)
