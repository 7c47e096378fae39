"""-m gpu: phase picking on continuous records (seist_b200/stream.py, csrc/stream.cu) against the numpy oracle
(oracle/stream_ref.py): the window cut bit for bit against torch slicing + `preprocess.normalize_`, stacking bit for bit,
whole-record picks and detection runs index for index, and `annotate` end to end against the module-path eval forward of
every window (2e-6, the per-waveform independence bound of the eval plan across batch layouts)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import stream_ref as SR
from seist_b200 import _lib
from seist_b200 import preprocess as PP
from seist_b200 import stream as ST
from seist_b200.models import create_model
from test_cpu_stream import long_traces

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    m = create_model("seist_s_dpk", in_channels=3, in_samples=8192)
    m.load_state_dict(G.model_state_dict("seist_s_dpk", 8192), strict=True)
    return m.cuda().eval()


def _record(S, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, C, T, generator=g) * (0.5 + 10 * torch.rand(S, C, 1, generator=g)) + torch.randn(S, C, 1, generator=g)
    return x.cuda()


@pytest.mark.parametrize("mode", ["std", "max", ""])
def test_window_batch_equals_sliced_normalize(mode):
    S, C, W, P = 2, 3, 2048, 1500
    T = 3 * W + 311
    rec = _record(S, C, T, 3)
    rec[1, 2, :] = 2.5                               # constant channel: zero scale -> 1
    starts = ST.window_starts(T, W, P)
    assert starts[-1] == T - W and (T - W) % P != 0
    K = len(starts)
    want = torch.stack([rec[s, :, a:a + W] for s in range(S) for a in starts]).contiguous()
    PP.normalize_(want, mode)
    B = 5
    x = torch.full((B, C, W), float("nan"), device="cuda")
    for w0 in range(0, S * K, B):
        ST.window_batch_(x, rec, W, P, w0, mode)
        n = min(B, S * K - w0)
        assert torch.equal(x[:n], want[w0:w0 + n]), w0
        assert (x[n:] == 0).all()                    # past the last window: zero rows


@pytest.mark.parametrize("stride,batch", [(4096, 4), (3000, 7)])
def test_annotate_equals_module_forward(model, stride, batch):
    S, W = 3, 8192
    T = 5 * W + 1234
    rec = _record(S, 3, T, 11)
    ann = ST.ContinuousAnnotator(model, window=W, stride=stride, batch=batch)
    K = ann.window_count(T)
    assert (S * K) % batch != 0 and K % batch != 0   # a station split across batches, a partial last batch
    probs = ann.annotate(rec)
    starts = ST.window_starts(T, W, stride)
    x = torch.stack([rec[s, :, a:a + W] for s in range(S) for a in starts]).contiguous()
    PP.normalize_(x, "std")
    with torch.no_grad():
        y = model(x).cpu().numpy()
    for mode in ("mean", "max"):
        if mode == "max":
            probs = ST.ContinuousAnnotator(model, window=W, stride=stride, batch=batch, stack="max").annotate(rec)
        want = SR.stack(y, S, T, W, stride, mode)
        err = np.abs(probs.cpu().numpy() - want).max()
        assert err <= 2e-6, (mode, err)


@pytest.mark.parametrize("P,B", [(200, 3), (512, 5), (37, 64)])
def test_stack_bit_identical(P, B):
    S, W = 2, 512
    T = 3 * W + 100
    K = len(ST.window_starts(T, W, P))
    g = torch.Generator().manual_seed(P)
    outs = torch.rand(S * K, 3, W, generator=g)
    for mode in ("mean", "max"):
        probs = torch.full((S, 3, T), float("nan"), device="cuda")
        y = torch.empty(B, 3, W, device="cuda")
        for w0 in range(0, S * K, B):
            n = min(B, S * K - w0)
            y.fill_(float("nan"))                    # the rows past S * K are never read
            y[:n] = outs[w0:w0 + n].cuda()
            ST.stack_batch_(probs, y, W, P, w0, mode)
        ST.stack_finish_(probs, W, P, mode)
        want = SR.stack(outs.numpy(), S, T, W, P, mode)
        assert np.array_equal(probs.cpu().numpy(), want), mode


def _long_probs():
    T = 1 << 21
    p = long_traces(T, seed=1, n_bumps=3000, teeth=6000)           # one cluster of ~6000 candidates (global memory)
    s = long_traces(T, seed=2, n_bumps=3000, teeth=1000)           # one of ~1000 (shared memory)
    det = long_traces(T, seed=3, n_bumps=2000, teeth=10)
    det[2, :5], det[2, -7:] = 0.9, 0.9                             # runs touching both ends
    det[3] = 0.9                                                   # one run over the whole trace
    return np.stack([det, p, s], axis=1).astype(np.float32)


def test_pick_and_detect_long_traces_match_oracle(model):
    probs = _long_probs()
    pc = torch.from_numpy(probs).cuda()
    ann = ST.ContinuousAnnotator(model, window=8192, batch=1)
    for mpd, (tp, ts) in ((100, (0.3, 0.1)), (7, (0.05, 0.5))):
        picks = ann.pick_phases(pc, ppk_threshold=tp, spk_threshold=ts, min_peak_dist=mpd)
        for name, ch, thr in (("ppk", 1, tp), ("spk", 2, ts)):
            index, prob, off = SR.pick_all(probs, ch, thr, mpd)
            gi, gp, go = (t.cpu().numpy() for t in picks[name])
            assert np.array_equal(go, off), (name, mpd, go, off)
            assert np.array_equal(gi, index), (name, mpd)
            assert np.array_equal(gp, prob), (name, mpd)
        per = ann.split(picks["ppk"])
        o = picks["ppk"][2].tolist()
        assert len(per) == 4 and all(torch.equal(per[i][0], picks["ppk"][0][o[i]:o[i + 1]]) for i in range(4))
        if tp > 0.09:
            assert per[3][0].numel() == 0                          # the row without a peak above 0.09
    for thr in (0.5, 0.3):
        pairs, off = SR.detect_all(probs, 0, thr)
        gpairs, goff = ann.detect_events(pc, det_threshold=thr)
        assert np.array_equal(goff.cpu().numpy(), off) and np.array_equal(gpairs.cpu().numpy(), pairs), thr
    assert gpairs[goff[3]].tolist() == [0, (1 << 21) - 1]


def test_argument_errors_raise_before_launch(model):
    ann = ST.ContinuousAnnotator(model, window=8192, stride=4096, batch=2)
    lib = _lib.lib()
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    rec = torch.zeros(1, 3, 9000)
    with pytest.raises(RuntimeError):
        ann.annotate(rec)                                          # CPU tensor
    with pytest.raises(ValueError):
        ann.annotate(torch.zeros(1, 2, 9000, device="cuda"))       # wrong C
    with pytest.raises(ValueError):
        ann.annotate(torch.zeros(1, 3, 8191, device="cuda"))       # T < W
    probs = torch.zeros(1, 3, 9000, device="cuda")
    for mpd in (1, 0, -3):
        with pytest.raises(ValueError):
            ann.pick_phases(probs, 0.3, 0.3, min_peak_dist=mpd)
    with pytest.raises(ValueError):
        ann.pick_phases(probs, 0.3, 0.3)                           # no min_peak_dist given or configured
    assert lib.seist_launch_count() == before
    for stride in (0, 8193):
        with pytest.raises(ValueError):
            ST.ContinuousAnnotator(model, window=8192, stride=stride)
    with pytest.raises(NotImplementedError):
        ST.ContinuousAnnotator(create_model("seist_s_pmp", in_channels=3, in_samples=8192))
    assert lib.seist_launch_count() == before


def test_from_args_reads_the_reference_names(model):
    args = SimpleNamespace(in_samples=8192, norm_mode="max", ppk_threshold=0.4, spk_threshold=0.35, det_threshold=0.6,
                           min_peak_dist=1.0)
    ann = ST.ContinuousAnnotator.from_args(model, args, sampling_rate=50, batch=2)
    assert (ann.window, ann.stride, ann.norm_mode, ann.min_peak_dist) == (8192, 4096, "max", 50)
    assert ann.thresholds == {"ppk": 0.4, "spk": 0.35, "det": 0.6}


def test_in_place_helpers_reject_wrong_buffers():
    lib = _lib.lib()
    rec = torch.zeros(2, 3, 9000, device="cuda")
    probs = torch.zeros(2, 3, 9000, device="cuda")
    torch.cuda.synchronize()
    before = lib.seist_launch_count()
    with pytest.raises(ValueError):
        ST.window_batch_(torch.zeros(4, 3, 4096, device="cuda"), rec, 8192, 4096, 0)     # rows shorter than the window
    with pytest.raises(ValueError):
        ST.window_batch_(torch.zeros(4, 2, 8192, device="cuda"), rec, 8192, 4096, 0)     # wrong channel count
    with pytest.raises(ValueError):
        ST.window_batch_(torch.zeros(4, 3, 8192, device="cuda"), rec[:, :, ::2], 4096, 2048, 0)   # strided record
    with pytest.raises(ValueError):
        ST.stack_batch_(probs, torch.zeros(4, 3, 4096, device="cuda"), 8192, 4096, 0)    # outputs shorter than the window
    with pytest.raises(ValueError):
        ST.stack_batch_(probs.transpose(0, 1), torch.zeros(4, 3, 8192, device="cuda"), 8192, 4096, 0)
    with pytest.raises(ValueError):
        ST.stack_finish_(probs.double(), 8192, 4096)
    assert lib.seist_launch_count() == before
