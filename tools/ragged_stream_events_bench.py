"""Stream a continuous record whose stations advance at different rates with every P pick characterised as it closes,
against the equal-rate characterised stream of the same record in the same run.

    python tools/ragged_stream_events_bench.py [--stations 256] [--hours 1] [--fs 100] [--max-push-s 120] [--chunk-s 60]
                                               [--window 8192] [--stride 4096] [--batch 256] [--ratio 0.3] [--size m]
                                               [--per-min 3] [--iters 2] [--warmup 1] [--seed 0]

A seeded synthetic 3-component record already on the device (as tools/stream_bench.py builds it), the golden synthetic
parameters of seist_<size>_dpk and seist_<size>_{pmp, emg, baz, dis}, min_peak_dist 1 s.  The P threshold is bisected on
the whole record's probabilities so that the picker yields about `per-min` P picks per station-minute (as
tools/stream_events_bench.py does).  Two modes alternate in one process: "ragged" pushes each station a seeded random
length in [0, max-push-s] per call (the schedule of tools/ragged_stream_bench.py: station 0 silent for the first half of
the record's duration in calls, a last push tops every station up to T) through `EventCharacterizer.open_ragged_stream`
and closes it; "equal" pushes chunks of `chunk-s` seconds through `EventCharacterizer.open_stream` and closes it.  Both
copy each pushed piece to a contiguous tensor inside the timed region.  For each: station-hours per second and events per
second (host clock around work that ends in a synchronise), the forward replays of the annotator and of each head, the
peak `torch.cuda.max_memory_allocated` (the record included) and the largest held_samples of any station.  Asserts that
both modes' events equal `EventCharacterizer` on the whole record's picks bit for bit.  Prints the card and its power
limit read in the same run; the last line is one JSON record.
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
from ragged_stream_bench import ragged_schedule  # noqa: E402
from stream_events_bench import HEADS, load  # noqa: E402
from seist_b200 import events as EV  # noqa: E402
from seist_b200 import stream as ST  # noqa: E402


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
    ap.add_argument("--ratio", type=float, default=0.3)
    ap.add_argument("--size", default="m")
    ap.add_argument("--per-min", type=float, default=3.0)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_stream_events_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    n = int(round(a.chunk_s * a.fs))
    max_push = int(round(a.max_push_s * a.fs))
    silent = int(round(T / 2 / (max_push / 2)))
    sched = ragged_schedule(S, T, max_push, silent, a.seed)
    ann = ST.ContinuousAnnotator(load(f"seist_{a.size}_dpk", W), window=W, stride=P, batch=B)
    ann.min_peak_dist = int(1.0 * a.fs)
    ch = EV.EventCharacterizer({h: load(f"seist_{a.size}_{h}", W) for h in HEADS}, window=W, p_position_ratio=a.ratio, batch=B)
    g = torch.Generator(device="cuda").manual_seed(0)
    rec = torch.randn(S, 3, T, device="cuda", generator=g) * 5.0

    probs = ann.annotate(rec)
    target = a.per_min * S * a.hours * 60
    lo, hi = 0.0, 1.0
    for _ in range(20):                                    # more picks below the threshold, fewer above
        mid = (lo + hi) / 2
        m = ann.pick_phases(probs, ppk_threshold=mid)["ppk"][0].numel()
        lo, hi = (mid, hi) if m > target else (lo, mid)
    ann.thresholds["ppk"] = hi
    ppk = ann.pick_phases(probs)["ppk"]
    M = ppk[0].numel()
    want = ch(rec, ppk)
    del probs
    torch.cuda.synchronize()

    replays = {h: 0 for h in HEADS}
    for h, gr in ch.graphs.items():
        orig = gr.replay

        def counted(orig=orig, h=h):
            replays[h] += 1
            return orig()
        gr.replay = counted

    def ragged():
        cs = ch.open_ragged_stream(ann, S)
        pos = np.zeros(S, np.int64)
        outs, held = [], 0
        for lengths in sched:
            c = cs.push([rec[s, :, pos[s]:pos[s] + lengths[s]].contiguous() for s in range(S)])
            pos += lengths
            outs.append((c.out.ppk[2], c.events))          # not the probabilities: memory held is the stream's
            held = max(held, int(cs.held_samples.max()))
        c = cs.close()
        outs.append((c.out.ppk[2], c.events))
        torch.cuda.synchronize()
        return outs, held, cs.forwards

    def equal():
        cs = ch.open_stream(ann, S)
        outs, held = [], 0
        for i in range(0, T, n):
            c = cs.push(rec[:, :, i:i + n].contiguous())
            outs.append((c.out.ppk[2], c.events))
            held = max(held, cs.held_samples)
        c = cs.close()
        outs.append((c.out.ppk[2], c.events))
        torch.cuda.synchronize()
        return outs, held, cs.forwards

    res = {"ragged": [], "equal": []}
    peak, held, fw, heads, last = {}, {}, {}, {}, {}
    for it in range(a.warmup + a.iters):
        for mode in ("ragged", "equal"):
            for h in HEADS:
                replays[h] = 0
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            outs, held[mode], fw[mode] = ragged() if mode == "ragged" else equal()
            dt = time.perf_counter() - t0
            peak[mode] = torch.cuda.max_memory_allocated()
            heads[mode] = dict(replays)
            if it >= a.warmup:
                res[mode].append(dt)
            last[mode] = outs
            del outs

    # both modes' events, per station in call order, against the whole record
    for mode, outs in last.items():
        for h in HEADS:
            parts = []
            for s in range(S):
                for off, ev in outs:
                    off = off.tolist()
                    parts.append(ev[h][off[s]:off[s + 1]])
            assert torch.equal(torch.cat(parts), want[h]), (mode, h)
        assert sum(int(off[-1]) for off, _ in outs) == M

    name = card()
    sh = S * a.hours
    t = {k: sum(v) / len(v) for k, v in res.items()}
    print(f"card: {name}")
    print(f"seist_{a.size}_dpk + seist_{a.size}_{{{','.join(HEADS)}}}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), "
          f"W = {W}, P = {P}, batch {B}, p_position_ratio {a.ratio}")
    print(f"ragged: {len(sched)} pushes of [0, {max_push}] samples per station (station 0 silent for the first {silent}), "
          f"equal: chunks of {n} samples")
    print(f"P threshold {ann.thresholds['ppk']:.6f}: M = {M} P picks ({M / (S * a.hours * 60):.2f} per station-minute)")
    for k in ("ragged", "equal"):
        print(f"{k:>6}: {sh / t[k]:.1f} station-hours/s ({', '.join(f'{sh / x:.1f}' for x in res[k])}), {M / t[k]:.0f} events/s, "
              f"{fw[k]} annotator replays, head replays {heads[k]}, peak memory {peak[k] / 2**20:.0f} MiB "
              f"(record {rec.numel() * 4 / 2**20:.0f} MiB), largest held_samples {held[k]}")
    print("ragged and equal-rate events identical to the whole-record characterisation")
    print(json.dumps({"card": name, "size": a.size, "stations": S, "T": T, "pushes": len(sched), "max_push": max_push, "chunk": n,
                      "window": W, "stride": P, "batch": B, "ratio": a.ratio, "ppk_threshold": ann.thresholds["ppk"], "events": M,
                      "station_hours_per_s": {k: sh / v for k, v in t.items()}, "events_per_s": {k: M / v for k, v in t.items()},
                      "seconds": t, "annotator_replays": fw, "head_replays": heads, "peak_bytes": peak, "max_held_samples": held,
                      "identical": True}))


if __name__ == "__main__":
    main()
