"""not-gpu: the characterised-stream oracle (tests/stream_events_ref.py) against the whole-record cut
(oracle/event_ref.py on the whole-record picks of oracle/stream_ref.py): for any split of a record the windows of the
streamed P picks, concatenated per station, equal `event_ref.windows` bit for bit; no cut reads a sample that is >= 0 but
below the history's first sample h0, or at or past R before the close; the history stays within its bound."""
import numpy as np
import pytest

from oracle import event_ref as ER
from oracle import stream_ref as SR
from stream_events_ref import CharacterizedStreamRef, concat_windows
from test_cpu_stream import long_traces
from test_cpu_stream_chunks import _record, _splits, _standin, _whole


def _run(rec, W, P, fn, mpd, thr, window, ratio, split, stack="mean"):
    S, C, T = rec.shape
    ref = CharacterizedStreamRef(S, C, W, P, fn, mpd, thr, window, ratio, stack=stack)
    a = ref.a
    calls, pos, held = [], 0, []
    for n in split:
        bound = ref.held_samples if n == 0 else n + W + a + 1 + ref.span
        calls.append(ref.push(rec[:, :, pos:pos + n]))
        pos += n
        held.append(ref.held_samples)
        assert held[-1] <= bound, (held[-1], bound)
    assert pos == T
    calls.append(ref.close())
    for _, _, reads in calls:
        for s, lo, hi, h0, R, closed in reads:
            assert max(lo, 0) >= h0, (lo, h0)                    # nothing below the history that exists in the record
            assert closed or hi <= R, (hi, R)                    # nothing not pushed yet, except past T at the close
    return calls, held


def _check(rec, W, P, fn, mpd, thr, window, ratio, split, want_ppk):
    S = rec.shape[0]
    calls, _ = _run(rec, W, P, fn, mpd, thr, window, ratio, split)
    index, _, off = want_ppk
    got = concat_windows(calls, S)
    want = ER.windows(rec, index, off, window, ratio, "std")
    assert got.shape == want.shape and np.array_equal(got, want)
    return len(index)


@pytest.mark.parametrize("T,W,P", [
    (64, 64, 32),          # T = W
    (65, 64, 32),          # T = W + 1: a tail window
    (64 * 4, 64, 32),      # stride W / 2
    (64 * 4 + 17, 64, 64),  # stride W
    (64 * 5 + 9, 64, 24),  # P does not divide W
])
@pytest.mark.parametrize("window,ratio", [(40, 0.0), (40, 0.3), (40, 1.0), (64, 0.0), (64, 0.3), (64, 1.0),
                                          (96, 0.5), (96, 1.0)])     # W_ch < W_ann, = W_ann, > W_ann with W_ch - a <= W_ann
def test_stream_windows_equal_whole_record(T, W, P, window, ratio):
    assert window - ER.anchor(window, ratio) <= W
    S, C = 2, 3
    rec = _record(S, C, T, T + W + P)
    fn = _standin(C)
    thr, mpd = (0.5, 0.3, 0.3), 5
    _, ppk, _, _ = _whole(rec, W, P, "mean", "std", fn, mpd, thr)
    assert len(ppk[0]) > 0
    for split in list(_splits(T, W, P, T)) + [[0, T // 2, 0, T - T // 2, 0]]:    # empty pushes keep the history
        _check(rec, W, P, fn, mpd, thr, window, ratio, split, ppk)


def _injected(traces, W):
    """Window outputs that repeat the given (S, T) rows at the window's samples on every channel: the stacked P trace
    is the row itself (the mean of equal values)."""
    def outputs(x, ids):
        return np.stack([np.repeat(traces[s, None, a:a + W], 3, axis=0) for s, a in ids]).astype(np.float32)
    return outputs


@pytest.mark.parametrize("mpd,tp", [(100, 0.3), (7, 0.05)])
def test_sawtooth_cluster_and_picks_at_the_ends(mpd, tp):
    """long_traces: a 6000-candidate sawtooth cluster (one pick cluster spanning 30 000 samples), peaks at 1 and T - 2;
    the history grows with the open cluster and shrinks once it closes."""
    T, W, P = 60_000, 256, 128
    tr = long_traces(T, seed=1, n_bumps=80)
    assert tr[2, 1] > tr[2, 0] and tr[2, T - 2] > tr[2, T - 1]
    S, C = 4, 3
    rec = _record(S, C, T, 3)
    fn = _injected(tr, W)
    thr = (0.5, tp, 0.3)
    probs = SR.stack(fn(None, [(s, a) for s in range(S) for a in SR.window_starts(T, W, P)]), S, T, W, P, "mean")
    ppk = SR.pick_all(probs, 1, tp, mpd)
    assert {1, T - 2} <= set(ppk[0][ppk[2][2]:ppk[2][3]].tolist())
    rng = np.random.default_rng(mpd)
    split = np.diff([0] + sorted(rng.integers(0, T, 50).tolist()) + [T]).tolist()
    for ratio, window in ((0.3, 256), (1.0, 200), (0.0, 256)):
        calls, held = _run(rec, W, P, fn, mpd, thr, window, ratio, split)
        got = concat_windows(calls, S)
        assert np.array_equal(got, ER.windows(rec, ppk[0], ppk[2], window, ratio, "std"))
        if mpd == 100:                                           # the cluster is held, then released
            assert max(held) > 30_000 - W and held[-1] < max(split) + W + window + 1, (max(held), held[-1])
