"""CPU oracle (TEST INFRASTRUCTURE) for streams with data gaps (seist_b200/stream.py `gap_stream_plan`, GapStream, DESIGN
§4.22), station by station from the whole record pushed so far: its segments (gaps_ref.segments), each a one-station
record of its own that stays open while it reaches the last pushed sample and closes once a gap sample (or the close)
follows it.  `call` gives what one call makes final: the first final sample t0, the number of samples made final, and
the windows run, as (first sample in the station's index) per window."""
import numpy as np

import gaps_ref as GR
from oracle import stream_ref as SR


def segments(rec: np.ndarray):
    """rec (C, T) -> inclusive [on, off] pairs (n, 2)."""
    return GR.segments(rec[None])[0]


def windows(rec: np.ndarray, W: int, P: int, closed: bool) -> set:
    """Every window run by the time rec (C, T) is pushed (`closed`: and the stream closed), as first samples."""
    T = rec.shape[1]
    out = set()
    for on, off in segments(rec):
        n = int(off - on + 1)
        if off == T - 1 and not closed:             # open: the regular windows that end by its last sample
            out |= {int(on) + k * P for k in range((n - W) // P + 1)} if n >= W else set()
        elif n >= W:
            out |= {int(on) + int(a) for a in SR.window_starts(n, W, P)}
    return out


def final(rec: np.ndarray, W: int, closed: bool) -> int:
    """Samples of rec (C, T) final: all before the open segment and that segment's own §4.16 prefix."""
    T = rec.shape[1]
    segs = segments(rec)
    if closed or not len(segs) or segs[-1][1] != T - 1:
        return T
    on, off = (int(v) for v in segs[-1])
    return on + max(0, off - on + 1 - W)


def call(before: np.ndarray, after: np.ndarray, W: int, P: int, closed: bool):
    """(t0, m, sorted windows) of the call that takes a station from record `before` to `after` (C, T)."""
    t0 = final(before, W, False)
    return t0, final(after, W, closed) - t0, sorted(windows(after, W, P, closed) - windows(before, W, P, False))


def window_ids(plan: dict, stride: int) -> list:
    """The windows of a `gap_stream_plan` call in packed order as (station, first sample in the station's index)."""
    ids = []
    for r in range(len(plan["station"])):
        s, on = int(plan["station"][r]), int(plan["on"][r])
        ids += [(s, on + (int(plan["k0"][r]) + q) * int(stride)) for q in range(int(plan["nk"][r]))]
        if plan["tail"][r] >= 0:
            ids.append((s, on + int(plan["tail"][r])))
    return ids
