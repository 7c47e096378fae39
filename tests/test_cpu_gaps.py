"""not-gpu: whole records with data gaps (DESIGN §4.21) on the CPU.  Library code: `segment_plan` against
`window_starts` segment by segment and `segment_groups`.  Oracle only (tests/gaps_ref.py; the kernels are checked against
it on the GPU): the segment finder on crafted records, the packed algorithm the kernels implement against per-slice
annotation with a model stand-in, and per-segment picking across a gap shorter than min_peak_dist."""
import numpy as np
import pytest

import gaps_ref as GR
from oracle import stream_ref as SR
from seist_b200 import stream as ST
from test_cpu_stream_chunks import _standin

NAN, INF = np.float32(np.nan), np.float32(np.inf)


def crafted(W: int = 16):
    """(S, 3, T) records with their expected segments: gaps at 0 and T - 1, one-sample and adjacent gaps, NaN in one
    channel, +-Inf, an all-gap and a gap-free station, segments of W - 1, W and W + 1 samples."""
    T = 6 * W + 10
    rec = np.random.default_rng(3).standard_normal((6, 3, T)).astype(np.float32)
    rec[0, :, 0] = NAN
    rec[0, 1, T - 1] = NAN                                              # one channel only
    rec[1, 2, 5] = INF
    rec[1, 0, 6] = -INF                                                 # adjacent gaps of different kinds
    rec[1, :, 20] = NAN                                                 # a one-sample gap
    rec[2] = NAN                                                        # all gap
    # station 3: gap free
    a = W - 1
    rec[4, 0, a] = NAN                                                  # [0, W - 2]: W - 1 samples
    rec[4, 0, 2 * W + 1] = NAN                                          # [W, 2W]: W + 1 samples
    rec[4, 0, 3 * W + 1] = NAN                                          # [2W + 2, 3W]: W - 1 samples
    rec[4, 0, 4 * W + 2] = NAN                                          # [3W + 2, 4W + 1]: W samples
    rec[5, :, 1:T - 1] = NAN                                            # two one-sample segments at the ends
    want = [[(1, T - 2)], [(0, 4), (7, 19), (21, T - 1)], [], [(0, T - 1)],
            [(0, W - 2), (W, 2 * W), (2 * W + 2, 3 * W), (3 * W + 2, 4 * W + 1), (4 * W + 3, T - 1)], [(0, 0), (T - 1, T - 1)]]
    return rec, want


def test_finder_on_crafted_records():
    rec, want = crafted()
    got = GR.segments(rec)
    assert [[tuple(map(int, p)) for p in g] for g in got] == want
    pairs, off = GR.table(rec)
    assert off.tolist() == np.cumsum([0] + [len(w) for w in want]).tolist() and pairs.shape == (off[-1], 2)
    short = np.full((2, 3, 10), 1.0, np.float32)                        # T < W: reported, not annotated
    short[1, :, 4] = NAN
    assert [g.tolist() for g in GR.segments(short)] == [[[0, 9]], [[0, 3], [5, 9]]]
    K, win_off, first, last, ids = GR.plan(GR.table(short)[0], 16, 8, 4)
    assert K.tolist() == [0, 0, 0] and ids == [] and first == [] and last == []


@pytest.mark.parametrize("W,P,B", [(16, 16, 3), (16, 8, 4), (16, 5, 7), (16, 5, 1)])
def test_segment_plan_against_window_starts(W, P, B):
    rec, _ = crafted(W)
    pairs, _ = GR.table(rec)
    rng = np.random.default_rng(W * P + B)
    extra = np.sort(rng.integers(0, 400, (40, 2)), axis=1)             # random segments, some long
    pairs = np.concatenate([pairs, extra])
    plan = ST.segment_plan(pairs[:, 0], pairs[:, 1], W, P, B)
    K, win_off, first, last, ids = GR.plan(pairs, W, P, B)
    for g, (on, off) in enumerate(pairs):
        n = int(off - on + 1)
        assert plan["K"][g] == (len(ST.window_starts(n, W, P)) if n >= W else 0)
    assert np.array_equal(plan["K"], K) and np.array_equal(plan["win_off"], win_off)
    assert plan["first"].tolist() == first and plan["last"].tolist() == last
    assert len(first) == -(-int(win_off[-1]) // B)


@pytest.mark.parametrize("P", [16, 8, 5])                              # stride W, W / 2 and one that does not divide W
@pytest.mark.parametrize("mode", ["mean", "max"])
def test_packed_pipeline_equals_per_slice_annotation(P, mode):
    W, B = 16, 5
    rec, _ = crafted(W)
    rng = np.random.default_rng(P)
    rec = np.concatenate([rec, rng.standard_normal((2, 3, rec.shape[2])).astype(np.float32)])
    rec[6, :, 30:33] = NAN
    fn = _standin(3)
    want = GR.annotate(rec, W, P, mode, "std", fn)
    got = GR.packed(rec, W, P, B, mode, "std", fn)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])
    for s, segs in enumerate(GR.segments(rec)):                         # NaN at every gap and short segment
        ok = np.zeros(rec.shape[2], bool)
        for a, b in segs:
            ok[a:b + 1] = b - a + 1 >= W
        assert np.isnan(want[s, :, ~ok]).all() and not np.isnan(want[s, :, ok]).any()
    if P == 16:                                                         # gap-free: the whole-record annotation
        clean = rec[3:4]
        assert np.array_equal(want[3:4], SR.stack(fn(SR.windows(clean, W, P, "std")), 1, clean.shape[2], W, P, mode))
    for ch in (1, 2):
        idx, val, off = GR.pick(want, rec, W, ch, 0.3, 3)
        for s, segs in enumerate(GR.segments(rec)):
            for a, b in segs:
                if b - a + 1 >= W:
                    sl = idx[off[s]:off[s + 1]]
                    assert np.array_equal(sl[(sl >= a) & (sl <= b)] - a, SR.detect_peaks_all(want[s, ch, a:b + 1], 0.3, 3))
    pairs, off = SR.detect_all(want, 0, 0.5)                          # detections of the NaN-filled trace are per segment
    wp, wo = GR.detect(want, rec, W, 0, 0.5)
    assert np.array_equal(pairs, wp) and np.array_equal(off, wo)


def test_picking_does_not_suppress_across_a_gap():
    """Two candidates 12 samples apart on both sides of a 2-sample gap, mpd 20: whole-row picking of the NaN-filled trace
    keeps only the higher one, per-segment picking keeps both."""
    W, T = 16, 200
    rec = np.ones((1, 3, T), np.float32)
    rec[0, :, 100:102] = NAN
    p = np.full(T, 0.1, np.float32)
    p[95], p[107] = 0.9, 0.8
    p[100:102] = NAN
    probs = np.stack([p, p, p])[None]
    whole = SR.detect_peaks_all(p, 0.3, 20)
    idx, val, off = GR.pick(probs, rec, W, 1, 0.3, 20)
    assert whole.tolist() == [95]
    assert idx.tolist() == [95, 107] and off.tolist() == [0, 2] and val.tolist() == [p[95], p[107]]
    assert idx.tolist() == [SR.detect_peaks_all(p[:100], 0.3, 20)[0], 102 + SR.detect_peaks_all(p[102:], 0.3, 20)[0]]


def test_segment_groups_pad_each_row_at_most_twofold():
    rng = np.random.default_rng(4)
    lengths = np.concatenate([rng.integers(16, 300, 5000), [1 << 21, 3, 1 << 20, 70000]])
    rng.shuffle(lengths)
    groups = ST.segment_groups(lengths, max_rows=1000)
    rows = np.concatenate(groups)
    assert np.array_equal(np.sort(rows), np.arange(lengths.size))          # every row exactly once
    padded = sum(g.size * lengths[g].max() for g in groups)
    assert padded < 2 * lengths.sum()
    for g in groups:
        assert g.size <= 1000 and np.all(np.diff(g) > 0)                   # row order kept within a group
        assert lengths[g].max() < 2 * lengths[g].min()
    assert [g.size for g in ST.segment_groups([5] * 70000)] == [65535, 4465]
