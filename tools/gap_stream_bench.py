"""Time streams with data gaps on the device (DESIGN §4.22).

    python tools/gap_stream_bench.py [--stations 256] [--hours 1] [--fs 100] [--window 8192] [--stride 4096]
                                     [--batch 256] [--model seist_m_dpk] [--iters 2] [--warmup 1]

The record and gaps of tools/gap_annotate_bench.py (about one gap per 10 min per station, station 0 down for 30 min,
the last station gap free).  Four modes alternate in one process, each a warm-up and then timed passes (host clock
around work that ends in a synchronise):
  (a) GapStream of the gapped record in 60 s chunks, then close;
  (b) GapStream of the gapped record on §4.19's ragged schedule (every station pushes a random 0-120 s piece per call);
  (c) RaggedStream of the record before the gaps were added, in 60 s chunks;
  (d) segments -> annotate(record, segments) -> pick_phases(probs, segments=...) of the whole gapped record.
Every station's concatenated probabilities and P / S picks of (a) and (b) are checked against (d), and (c) against
annotate of the clean record.  Prints the card and its power limit, station-hours per second, forward replays, the wall
time spent in the scan of the pushes (its host read included), the rest of the host-side time per call outside the
forwards, and the peak of torch.cuda.max_memory_allocated.  The last line is one JSON record.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden as G  # noqa: E402
from seist_b200 import stream as ST  # noqa: E402
from seist_b200.models import create_model  # noqa: E402
from tools.annotate_bench import card  # noqa: E402
from tools.gap_annotate_bench import add_gaps  # noqa: E402


def schedules(S, T, fs, seed):
    equal = [np.full(S, min(60 * fs, T - r), np.int64) for r in range(0, T, 60 * fs)]
    rng = np.random.default_rng(seed)
    ragged, left = [], np.full(S, T, np.int64)
    while left.any():
        n = np.minimum(left, rng.integers(0, 120 * fs + 1, size=S))
        ragged.append(n)
        left -= n
    return equal, ragged


def run_stream(st, rec, sched):
    S = rec.shape[0]
    R = np.zeros(S, np.int64)
    outs = []
    for n in sched:
        outs.append(st.push([rec[s, :, R[s]:R[s] + n[s]].contiguous() for s in range(S)]))
        R += n
    outs.append(st.close())
    torch.cuda.synchronize()
    return outs


def assemble(outs, S, T):
    """The calls' outputs as one (S, 3, T) record and per-pick-channel (station, index, prob) in station, index order."""
    probs = torch.full((S, 3, T), float("nan"), device="cuda")
    for o in outs:
        for s in range(S):
            probs[s, :, o.t0[s]:o.t0[s] + o.probs[s].shape[1]] = o.probs[s]
    picks = {}
    for k in ("ppk", "spk"):
        st = torch.cat([torch.repeat_interleave(torch.arange(S, device="cuda"), getattr(o, k)[2].diff()) for o in outs])
        idx = torch.cat([getattr(o, k)[0] for o in outs])
        val = torch.cat([getattr(o, k)[1] for o in outs])
        order = torch.sort(st, stable=True).indices
        picks[k] = (st[order], idx[order], val[order])
    return probs, picks


def csr_picks(picks):
    out = {}
    for k in ("ppk", "spk"):
        idx, val, off = picks[k]
        st = torch.repeat_interleave(torch.arange(off.numel() - 1, device="cuda"), off.diff())
        out[k] = (st, idx, val)
    return out


def same(p, q):
    pp, qp = p[0], q[0]
    ok = torch.equal(torch.isnan(pp), torch.isnan(qp)) and torch.equal(pp.nan_to_num(), qp.nan_to_num())
    return ok and all(torch.equal(u, v) for k in ("ppk", "spk") for u, v in zip(p[1][k], q[1][k]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=256)
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--fs", type=int, default=100)
    ap.add_argument("--window", type=int, default=8192)
    ap.add_argument("--stride", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--model", default="seist_m_dpk")
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gap_stream_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    m = create_model(a.model, in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict(a.model, W), strict=True)
    m = m.cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    clean = torch.randn(S, 3, T, device="cuda", generator=g) * 5.0
    gapped = add_gaps(clean, a.fs, 1)
    ann = ST.ContinuousAnnotator(m, window=W, stride=P, batch=B)
    ann.min_peak_dist = int(1.0 * a.fs)
    equal, ragged = schedules(S, T, a.fs, 2)
    replays, fwd_ms = [0], [0.0]
    replay = ann.graph.replay

    def counted():
        replays[0] += 1
        return replay()
    ann.graph.replay = counted
    scan_s = [0.0]
    scan = ST.gap_stream_segments

    def timed_scan(*args):
        t = time.perf_counter()
        out = scan(*args)                                               # ends in its host read
        scan_s[0] += time.perf_counter() - t
        return out
    ST.gap_stream_segments = timed_scan

    def whole(rec):
        segs = ann.segments(rec)
        probs = ann.annotate(rec, segments=segs)
        picks = ann.pick_phases(probs, segments=segs)
        torch.cuda.synchronize()
        return probs, picks

    modes = {"a_gap_stream_60s": lambda: run_stream(ann.open_gap_stream(S), gapped, equal),
             "b_gap_stream_ragged": lambda: run_stream(ann.open_gap_stream(S), gapped, ragged),
             "c_ragged_stream_clean_60s": lambda: run_stream(ann.open_ragged_stream(S), clean, equal),
             "d_annotate_segments": lambda: whole(gapped)}
    times = {k: [] for k in modes}
    peak, fwd, scans, out = {k: 0 for k in modes}, {}, {}, {}
    for it in range(a.warmup + a.iters):
        for k, fn in modes.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            replays[0], scan_s[0] = 0, 0.0
            t0 = time.perf_counter()
            out[k] = fn()
            dt = time.perf_counter() - t0
            peak[k] = max(peak[k], torch.cuda.max_memory_allocated())
            fwd[k], scans[k] = replays[0], scan_s[0]
            if it >= a.warmup:
                times[k].append(dt)
            if k != "d_annotate_segments":
                out[k] = (out[k], len(out[k]))

    # the forwards alone: the same number of replays of the captured graph, timed with CUDA events
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        replay()
    e1.record()
    torch.cuda.synchronize()
    per_replay = e0.elapsed_time(e1) / 20 / 1e3

    ref = out["d_annotate_segments"]
    ref = (ref[0], csr_picks(ref[1]))
    clean_probs = ann.annotate(clean)
    clean_ref = (clean_probs, csr_picks(ann.pick_phases(clean_probs)))
    checks = {"a_gap_stream_60s": same(assemble(out["a_gap_stream_60s"][0], S, T), ref),
              "b_gap_stream_ragged": same(assemble(out["b_gap_stream_ragged"][0], S, T), ref),
              "c_ragged_stream_clean_60s": same(assemble(out["c_ragged_stream_clean_60s"][0], S, T), clean_ref)}
    name = card()
    print(f"card: {name}")
    print(f"{a.model}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), W = {W}, P = {P}, batch {B}; "
          f"one replay {per_replay * 1e3:.2f} ms")
    res = {}
    for k in modes:
        t = float(np.mean(times[k]))
        calls = out[k][1] if k != "d_annotate_segments" else 1
        host = (t - fwd[k] * per_replay - scans[k]) / calls
        res[k] = {"ms": t * 1e3, "station_hours_per_s": S * a.hours / t, "replays": fwd[k], "calls": calls,
                  "scan_ms": scans[k] * 1e3, "rest_outside_forwards_ms_per_call": host * 1e3, "peak_gb": peak[k] / 1e9,
                  "equal_to_whole_record": checks.get(k)}
        print(f"{k}: {t * 1e3:.1f} ms, {S * a.hours / t:.1f} station-hours/s, {fwd[k]} replays, {calls} calls, scan "
              f"{scans[k] * 1e3:.1f} ms, rest outside the forwards {host * 1e3:.2f} ms per call, peak {peak[k] / 1e9:.2f} GB"
              + (f", equal to the whole-record path: {checks[k]}" if k in checks else ""))
    print(json.dumps({"card": name, "model": a.model, "stations": S, "T": T, "window": W, "stride": P, "batch": B,
                      "replay_ms": per_replay * 1e3, "modes": res}))
    if not all(checks.values()):
        raise SystemExit("a streamed mode differs from the whole-record path")


if __name__ == "__main__":
    main()
