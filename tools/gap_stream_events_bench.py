"""Stream a continuous record with data gaps with every P pick characterised as it closes (DESIGN §4.23), against the
gap-free characterised stream and the whole-record path in the same run.

    python tools/gap_stream_events_bench.py [--stations 256] [--hours 1] [--fs 100] [--max-push-s 120] [--chunk-s 60]
                                            [--window 8192] [--stride 4096] [--batch 256] [--ratio 0.3] [--size m]
                                            [--per-min 3] [--iters 2] [--warmup 1] [--seed 0]

A seeded synthetic 3-component record already on the device, the golden synthetic parameters of seist_<size>_dpk and
seist_<size>_{pmp, emg, baz, dis}, min_peak_dist 1 s, and the gaps of tools/gap_annotate_bench.py (about one gap per
10 min per station, station 0 down for 30 min, the last station gap free).  The P threshold is bisected on the whole
gap-free record to about `per-min` P picks per station-minute, as tools/ragged_stream_events_bench.py does.  Five modes
alternate in one process, each a warm-up and then timed passes (host clock around work that ends in a synchronise):
  (a) GapCharacterizedStream of the gapped record in `chunk-s` chunks, then close;
  (b) GapCharacterizedStream of the gapped record on the ragged schedule of tools/ragged_stream_bench.py ([0, max-push-s]
      per station and call, station 0 silent for the first calls);
  (c) RaggedCharacterizedStream of the gap-free record in `chunk-s` chunks;
  (c') RaggedCharacterizedStream of the gap-free record on the ragged schedule;
  (d) segments -> annotate(segments=) -> pick_phases(segments=) -> ch(segments=) of the whole gapped record.
The streamed modes copy each pushed piece to a contiguous tensor inside the timed region.  For each: station-hours and
events per second, the calls, the annotator and head replays, the wall time of the push scans (their host read
included, the queued work before it not), the host time per call outside the forwards and the scans (forwards =
replays x the per-replay time of each captured graph, timed with CUDA events), the peak torch.cuda.max_memory_allocated
(both records included) and the largest held_samples.  Asserts that (a) and (b) equal (d) per station bit for bit, and (c), (c') the whole-record
characterisation of the gap-free record.  Prints the card and its power limit read in the same run; the last line is
one JSON record.
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
from gap_annotate_bench import add_gaps  # noqa: E402
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
        raise SystemExit("gap_stream_events_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    n = int(round(a.chunk_s * a.fs))
    max_push = int(round(a.max_push_s * a.fs))
    silent = int(round(T / 2 / (max_push / 2)))
    ragged = ragged_schedule(S, T, max_push, silent, a.seed)
    equal = [np.full(S, min(n, T - r), np.int64) for r in range(0, T, n)]
    ann = ST.ContinuousAnnotator(load(f"seist_{a.size}_dpk", W), window=W, stride=P, batch=B)
    ann.min_peak_dist = int(1.0 * a.fs)
    ch = EV.EventCharacterizer({h: load(f"seist_{a.size}_{h}", W) for h in HEADS}, window=W, p_position_ratio=a.ratio, batch=B)
    g = torch.Generator(device="cuda").manual_seed(0)
    clean = torch.randn(S, 3, T, device="cuda", generator=g) * 5.0
    gapped = add_gaps(clean, a.fs, 1)

    probs = ann.annotate(clean)
    target = a.per_min * S * a.hours * 60
    lo, hi = 0.0, 1.0
    for _ in range(20):                                    # more picks below the threshold, fewer above
        mid = (lo + hi) / 2
        m = ann.pick_phases(probs, ppk_threshold=mid)["ppk"][0].numel()
        lo, hi = (mid, hi) if m > target else (lo, mid)
    ann.thresholds["ppk"] = hi
    ppk_clean = ann.pick_phases(probs)["ppk"]
    want_clean = ch(clean, ppk_clean)
    del probs
    torch.cuda.synchronize()

    graphs = {"annotator": ann.graph, **ch.graphs}
    replays = {k: 0 for k in graphs}
    per_replay = {}
    for k, gr in graphs.items():                           # the forwards alone, timed with CUDA events
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        gr.replay()
        e0.record()
        for _ in range(20):
            gr.replay()
        e1.record()
        torch.cuda.synchronize()
        per_replay[k] = e0.elapsed_time(e1) / 20 / 1e3
        orig = gr.replay

        def counted(orig=orig, k=k):
            replays[k] += 1
            return orig()
        gr.replay = counted
    scan_s = [0.0]
    scan = ST.gap_stream_segments

    def timed_scan(*args):
        torch.cuda.synchronize()                           # the scan's host read would wait for the queued forwards here
        t = time.perf_counter()
        out = scan(*args)                                  # ends in its host read
        scan_s[0] += time.perf_counter() - t
        return out
    ST.gap_stream_segments = timed_scan

    def stream(cs, rec, sched):
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
        return outs, held, len(sched) + 1

    def whole():
        segs = ann.segments(gapped)
        pk = ann.pick_phases(ann.annotate(gapped, segments=segs), segments=segs)["ppk"]
        ev = ch(gapped, pk, segments=segs)
        torch.cuda.synchronize()
        return [(pk[2], ev)], 0, 1

    modes = {"a_gap_60s": lambda: stream(ch.open_gap_stream(ann, S), gapped, equal),
             "b_gap_ragged": lambda: stream(ch.open_gap_stream(ann, S), gapped, ragged),
             "c_ragged_clean_60s": lambda: stream(ch.open_ragged_stream(ann, S), clean, equal),
             "c2_ragged_clean_ragged": lambda: stream(ch.open_ragged_stream(ann, S), clean, ragged),
             "d_whole_segments": whole}
    times = {k: [] for k in modes}
    peak, held, counts, calls, scans, last = {}, {}, {}, {}, {}, {}
    for it in range(a.warmup + a.iters):
        for k, fn in modes.items():
            for r in replays:
                replays[r] = 0
            scan_s[0] = 0.0
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            outs, held[k], calls[k] = fn()
            dt = time.perf_counter() - t0
            peak[k] = torch.cuda.max_memory_allocated()
            counts[k], scans[k] = dict(replays), scan_s[0]
            if it >= a.warmup:
                times[k].append(dt)
            last[k] = outs
            del outs

    def per_station(outs, h):
        parts = []
        for s in range(S):
            for off, ev in outs:
                off = off.tolist()
                parts.append(ev[h][off[s]:off[s + 1]])
        return torch.cat(parts)

    want_gap = {h: per_station(last["d_whole_segments"], h) for h in HEADS}
    M = {k: sum(int(off[-1]) for off, _ in outs) for k, outs in last.items()}
    for k, outs in last.items():
        if k == "d_whole_segments":
            continue
        want = want_clean if k.startswith("c") else want_gap
        for h in HEADS:
            assert torch.equal(per_station(outs, h), want[h]), (k, h)

    name = card()
    sh = S * a.hours
    t = {k: sum(v) / len(v) for k, v in times.items()}
    fwd = {k: sum(counts[k][r] * per_replay[r] for r in graphs) for k in modes}
    host = {k: (t[k] - fwd[k] - scans[k]) / calls[k] for k in modes}
    print(f"card: {name}")
    print(f"seist_{a.size}_dpk + seist_{a.size}_{{{','.join(HEADS)}}}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), "
          f"W = {W}, P = {P}, batch {B}, p_position_ratio {a.ratio}")
    print(f"gaps: {int(torch.isnan(gapped[:, 0]).sum())} gap samples of {S * T}; chunks of {n} samples; ragged: {len(ragged)} "
          f"pushes of [0, {max_push}] samples per station (station 0 silent for the first {silent})")
    print(f"P threshold {ann.thresholds['ppk']:.6f}: {M['c_ragged_clean_60s']} P picks on the gap-free record, "
          f"{M['d_whole_segments']} on the gapped one")
    print("per replay (ms): " + ", ".join(f"{r} {v * 1e3:.2f}" for r, v in per_replay.items()))
    for k in modes:
        print(f"{k:>22}: {sh / t[k]:.1f} station-hours/s ({', '.join(f'{sh / x:.1f}' for x in times[k])}), {M[k] / t[k]:.0f} "
              f"events/s, {calls[k]} calls, replays {counts[k]}, forwards {fwd[k] * 1e3:.0f} ms, scans {scans[k] * 1e3:.1f} ms, "
              f"other host time {host[k] * 1e3:.2f} ms/call, peak memory {peak[k] / 2**30:.2f} GiB, largest held_samples "
              f"{held[k]}")
    print("streamed events identical to the whole-record path (gapped modes: with segments)")
    print(json.dumps({"card": name, "size": a.size, "stations": S, "T": T, "chunk": n, "ragged_pushes": len(ragged),
                      "max_push": max_push, "window": W, "stride": P, "batch": B, "ratio": a.ratio,
                      "ppk_threshold": ann.thresholds["ppk"], "events": M, "per_replay_s": per_replay,
                      "station_hours_per_s": {k: sh / v for k, v in t.items()}, "events_per_s": {k: M[k] / v for k, v in t.items()},
                      "seconds": t, "calls": calls, "replays": counts, "forward_s": fwd, "scan_s": scans, "host_s_per_call": host,
                      "peak_bytes": peak, "max_held_samples": held, "identical": True}))


if __name__ == "__main__":
    main()
