"""not-gpu: the streaming oracle (tests/stream_chunks_ref.py) against the whole-record oracle (oracle/stream_ref.py): for
any split of a record into chunks the concatenated probabilities equal `stack` bit for bit and the picks / runs equal
`pick_all` / `detect_all` index for index; the finality rules hold call by call."""
import numpy as np
import pytest

from oracle import stream_ref as SR
from stream_chunks_ref import PickStreamRef, StreamRef, concat
from test_cpu_stream import long_traces


def _standin(C: int, seed: int = 7):
    """A fixed model stand-in: sigmoid of a 9-tap convolution of the normalised window, 3 output channels."""
    k = np.random.default_rng(seed).standard_normal((3, C, 9)).astype(np.float32) * np.float32(0.4)

    def outputs(x, ids=None):
        n, _, W = x.shape
        y = np.zeros((n, 3, W), np.float32)
        xp = np.pad(x, ((0, 0), (0, 0), (4, 4)))
        for o in range(3):
            for c in range(C):
                for j in range(9):
                    y[:, o] += k[o, c, j] * xp[:, c, j:j + W]
        return (np.float32(1) / (np.float32(1) + np.exp(np.minimum(-y * np.float32(3), np.float32(80))))).astype(np.float32)
    return outputs


def _record(S, C, T, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((S, C, T)) * rng.uniform(0.5, 10, (S, C, 1)) + rng.standard_normal((S, C, 1))).astype(np.float32)


def _whole(rec, W, P, mode, norm, fn, mpd, thr):
    S, _, T = rec.shape
    y = fn(SR.windows(rec, W, P, norm))
    probs = SR.stack(y, S, T, W, P, mode)
    return probs, SR.pick_all(probs, 1, thr[1], mpd), SR.pick_all(probs, 2, thr[2], mpd), SR.detect_all(probs, 0, thr[0])


def _assert_equal(got, want):
    assert np.array_equal(got[0], want[0])
    for g, w in zip(got[1:3], want[1:3]):
        for a, b in zip(g, w):
            assert np.array_equal(a, b)
    assert np.array_equal(got[3][0], want[3][0]) and np.array_equal(got[3][1], want[3][1])


def _splits(T, W, P, seed):
    rng = np.random.default_rng(seed)
    yield [T]                                                     # a single chunk
    yield [1] * T                                                 # 1-sample chunks
    yield [W] + [P] * ((T - W) // P) + ([(T - W) % P] if (T - W) % P else [])  # every push ends on a window end
    cuts = sorted(c for c in set(rng.integers(0, T, 6).tolist()) | {W - 1, W + P, T - W} if 0 <= c <= T)   # R - W boundaries
    yield np.diff([0] + cuts + [T]).tolist()
    yield np.diff([0] + sorted(rng.integers(0, T, 12).tolist()) + [T]).tolist()


def _stream(rec, W, P, mode, norm, fn, mpd, thr, split):
    S = rec.shape[0]
    ref = StreamRef(S, rec.shape[1], W, P, fn, mpd, thr, norm, mode)
    outs, pos = [], 0
    for n in split:
        o = ref.push(rec[:, :, pos:pos + n])
        pos += n
        assert o[0] + o[1].shape[2] == max(0, pos - W)            # nothing at t >= R - W before the close
        outs.append(o)
    outs.append(ref.close())
    assert pos == rec.shape[2] and outs[-1][0] + outs[-1][1].shape[2] == pos
    return outs


@pytest.mark.parametrize("T,W,P", [
    (64, 64, 32),          # T = W
    (65, 64, 32),          # T = W + 1: a tail window
    (64 * 4, 64, 32),      # no tail window
    (64 * 4 + 17, 64, 64),  # P = W
    (64 * 5 + 9, 64, 24),  # P does not divide W
])
@pytest.mark.parametrize("mode", ["mean", "max"])
def test_stream_equals_whole_record(T, W, P, mode):
    S, C = 2, 3
    rec = _record(S, C, T, T + W + P)
    fn = _standin(C)
    thr, mpd = (0.5, 0.3, 0.3), 5
    want = _whole(rec, W, P, mode, "std", fn, mpd, thr)
    for i, split in enumerate(_splits(T, W, P, T)):
        outs = _stream(rec, W, P, mode, "std", fn, mpd, thr, split)
        _assert_equal(concat(outs, S), want)


@pytest.mark.parametrize("norm", ["max", ""])
def test_stream_norm_modes(norm):
    S, C, T, W, P = 2, 3, 400, 64, 40
    rec = _record(S, C, T, 5)
    fn = _standin(C, 3)
    want = _whole(rec, W, P, "mean", norm, fn, 3, (0.4, 0.2, 0.2))
    for split in list(_splits(T, W, P, 9))[2:]:
        _assert_equal(concat(_stream(rec, W, P, "mean", norm, fn, 3, (0.4, 0.2, 0.2), split), S), want)


def _feed_probs(probs, split, mpd, thr, t0=0):
    S = probs.shape[0]
    ref = PickStreamRef(S, mpd, thr, t0)
    outs, pos = [], 0
    for n in split:
        outs.append((pos, probs[:, :, pos:pos + n]) + ref.push(probs[:, :, pos:pos + n]))
        pos += n
    outs.append((pos, probs[:, :, pos:]) + ref.close(probs[:, :, pos:]))
    return outs


def _uneven(T, seed, n=40):
    rng = np.random.default_rng(seed)
    return np.diff([0] + sorted(rng.integers(0, T, n).tolist())).tolist()


@pytest.mark.parametrize("mpd,tp,ts", [(100, 0.3, 0.1), (7, 0.05, 0.5)])
def test_probability_stage_long_traces(mpd, tp, ts):
    T = 200_000
    p = long_traces(T, seed=1)                                      # the 6000-candidate sawtooth cluster
    s = long_traces(T, seed=2, teeth=1000)
    det = long_traces(T, seed=3, n_bumps=200, teeth=10)
    det[2, :5], det[2, -7:] = 0.9, 0.9                               # runs touching both ends
    det[3] = 0.9                                                     # one run over the whole row
    probs = np.stack([det, p, s], axis=1).astype(np.float32)
    for thr_det in (0.5, 0.3):
        thr = (thr_det, tp, ts)
        outs = _feed_probs(probs, _uneven(T, mpd), mpd, thr)
        got = concat(outs, 4)
        assert np.array_equal(got[0], probs)
        for k, ch in ((1, 1), (2, 2)):
            want = SR.pick_all(probs, ch, thr[ch], mpd)
            assert all(np.array_equal(a, b) for a, b in zip(got[k], want)), (ch, mpd)
        pairs, off = SR.detect_all(probs, 0, thr_det)
        assert np.array_equal(got[3][0], pairs) and np.array_equal(got[3][1], off)
    assert got[3][0][got[3][1][3]].tolist() == [0, T - 1]
    idx2 = SR.pick_all(probs, 2, ts, mpd)[0]
    if ts <= 0.3:
        assert 1 in idx2.tolist() and T - 2 in idx2.tolist() and 1000 in idx2.tolist()   # both ends, the flat top


def test_picks_wait_for_their_cluster():
    """No pick is emitted while a candidate within mpd of it is undecided; the sawtooth cluster arrives in one call."""
    T, mpd = 200_000, 100
    p = long_traces(T, seed=1)
    probs = np.stack([p, p, p], axis=1).astype(np.float32)
    split = [5000] * (T // 5000)
    outs = _feed_probs(probs, split, mpd, (0.5, 0.3, 0.3))
    a = T // 4
    for pos, stretch, ppk, _, _ in outs:
        f1 = pos + stretch.shape[2]
        idx, _, off = ppk
        for s in range(4):
            for i in idx[off[s]:off[s + 1]]:
                assert i + 1 < f1                                       # decided
        # every emitted pick's cluster is closed: no undecided candidate within mpd (the undecided ones start at f1 - 1)
        if idx.size:
            assert idx.max() + mpd <= f1 - 2 or f1 == T
    saw_calls = [k for k, o in enumerate(outs) if any(a <= i < a + 30_000 for i in o[2][0][o[2][2][1]:o[2][2][2]])]
    assert len(saw_calls) == 1 and outs[saw_calls[0]][0] >= a + 30_000 - 5000


def test_probability_stage_at_a_large_offset():
    t0 = (1 << 31) - 3000
    p = long_traces(20_000, seed=4, n_bumps=60, teeth=50)
    probs = np.stack([p, p, p], axis=1).astype(np.float32)
    outs = _feed_probs(probs, _uneven(20_000, 1), 20, (0.3, 0.3, 0.3), t0)
    got = concat(outs, 4)
    want = SR.pick_all(probs, 1, 0.3, 20)
    assert np.array_equal(got[1][0], want[0] + t0) and np.array_equal(got[1][2], want[2])
    pairs, off = SR.detect_all(probs, 0, 0.3)
    assert np.array_equal(got[3][0], pairs + t0) and (got[3][0] >= 1 << 31).any() and (got[3][0] < 1 << 31).any()
