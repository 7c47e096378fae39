"""Stream a continuous record whose stations advance at different rates and compare it with the equal-length stream.

    python tools/ragged_stream_bench.py [--stations 256] [--hours 1] [--fs 100] [--max-push-s 120] [--chunk-s 60]
                                        [--window 8192] [--stride 4096] [--batch 256] [--model seist_m_dpk] [--iters 2]
                                        [--warmup 1] [--seed 0]

A seeded synthetic 3-component record (as tools/stream_bench.py builds it) already on the device, the golden synthetic
parameters of the model, the main.py thresholds (P / S 0.3, det 0.5, min_peak_dist 1 s).  The two modes alternate in one
process: "ragged" pushes each station a seeded random length in [0, max-push-s] per call through
`ContinuousAnnotator.open_ragged_stream` (station 0 pushes nothing for the first half of the record's duration in calls,
a last push tops every station up to T) and closes it; "equal" pushes chunks of `chunk-s` seconds through `open_stream`
and closes it.  Both copy each pushed piece to a contiguous tensor inside the timed region.  For each mode:
station-hours per second (host clock around work that ends in a synchronise), the peak `torch.cuda.max_memory_allocated`
(the record included) and the number of forward replays.  Asserts that each station's concatenated ragged output equals
`annotate(rec)[s]` and its picks and runs.  Prints the card and its power limit read in the same run; the last line is one
JSON record.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from annotate_bench import card  # noqa: E402
from oracle import golden as G  # noqa: E402
from seist_b200 import stream as ST  # noqa: E402
from seist_b200.models import create_model  # noqa: E402
from stream_bench import per_station  # noqa: E402


def ragged_schedule(S, T, max_push, calls_silent, seed):
    """Per-call lengths (S,) until every station holds T samples: seeded uniform lengths in [0, max_push], station 0
    silent for the first calls_silent calls, the last call tops every station up to T."""
    rng = np.random.default_rng(seed)
    R = np.zeros(S, np.int64)
    sched = []
    while True:
        n = rng.integers(0, max_push + 1, S)
        if len(sched) < calls_silent:
            n[0] = 0
        n = np.minimum(n, T - R)
        if (R + n >= T).all() or len(sched) > 100_000:
            break
        sched.append(n)
        R += n
    sched.append(T - R)
    return sched


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=256)
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--fs", type=int, default=100)
    ap.add_argument("--max-push-s", type=float, default=120.0)
    ap.add_argument("--chunk-s", type=float, default=60.0)
    ap.add_argument("--window", type=int, default=8192)
    ap.add_argument("--stride", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--model", default="seist_m_dpk")
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_stream_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    n = int(round(a.chunk_s * a.fs))
    max_push = int(round(a.max_push_s * a.fs))
    mean_push = max_push / 2
    sched = ragged_schedule(S, T, max_push, int(round(T / 2 / mean_push)), a.seed)
    m = create_model(a.model, in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict(a.model, W), strict=True)
    m = m.cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    rec = torch.randn(S, 3, T, device="cuda", generator=g) * 5.0
    ann = ST.ContinuousAnnotator(m, window=W, stride=P, batch=B)
    ann.min_peak_dist = int(1.0 * a.fs)

    def ragged():
        st = ann.open_ragged_stream(S)
        pos = np.zeros(S, np.int64)
        outs = []
        for lengths in sched:
            outs.append(st.push([rec[s, :, pos[s]:pos[s] + lengths[s]].contiguous() for s in range(S)]))
            pos += lengths
        outs.append(st.close())
        torch.cuda.synchronize()
        return outs, st.forwards

    def equal():
        st = ann.open_stream(S)
        outs = [st.push(rec[:, :, i:i + n].contiguous()) for i in range(0, T, n)] + [st.close()]
        torch.cuda.synchronize()
        return outs, st.forwards

    res = {"ragged": [], "equal": []}
    peak, fw, last = {}, {}, {}
    for it in range(a.warmup + a.iters):
        for mode in ("ragged", "equal"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            out, fw[mode] = ragged() if mode == "ragged" else equal()
            dt = time.perf_counter() - t0
            peak[mode] = torch.cuda.max_memory_allocated()
            if it >= a.warmup:
                res[mode].append(dt)
            last[mode] = out
            del out
    r_out = last["ragged"]
    last.clear()
    probs = ann.annotate(rec)
    picks = ann.pick_phases(probs)
    want = {"ppk": per_station(picks["ppk"], S), "spk": per_station(picks["spk"], S), "det": per_station(ann.detect_events(probs), S)}
    for s in range(S):
        assert torch.equal(torch.cat([o.probs[s] for o in r_out], 1), probs[s]), ("probs", s)
    for name in ("ppk", "spk", "det"):
        got = [per_station(getattr(o, name), S) for o in r_out]
        for s in range(S):
            for j in range(len(want[name][s])):
                assert torch.equal(torch.cat([gg[s][j] for gg in got]), want[name][s][j]), (name, s)
    name = card()
    sh = S * a.hours
    rate = {k: sh / (sum(v) / len(v)) for k, v in res.items()}
    print(f"card: {name}")
    print(f"{a.model}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), W = {W}, P = {P}, batch {B}")
    print(f"ragged: {len(sched)} pushes of [0, {max_push}] samples per station (station 0 silent for the first "
          f"{int(round(T / 2 / mean_push))}), equal: chunks of {n} samples")
    for k in ("ragged", "equal"):
        print(f"{k:>6}: {rate[k]:.1f} station-hours/s ({', '.join(f'{sh / t:.1f}' for t in res[k])}), peak memory "
              f"{peak[k] / 2**20:.0f} MiB (record {rec.numel() * 4 / 2**20:.0f} MiB), {fw[k]} forward replays")
    print("ragged outputs identical to annotate per station: probabilities, picks and detections")
    print(json.dumps({"card": name, "model": a.model, "stations": S, "T": T, "pushes": len(sched), "max_push": max_push, "chunk": n,
                      "window": W, "stride": P, "batch": B, "station_hours_per_s": rate, "peak_bytes": peak, "forwards": fw,
                      "identical": True}))


if __name__ == "__main__":
    main()
