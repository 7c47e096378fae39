"""Time the annotation of whole records with data gaps on the device (DESIGN §4.21).

    python tools/gap_annotate_bench.py [--stations 256] [--hours 1] [--fs 100] [--window 8192] [--stride 4096]
                                       [--batch 256] [--model seist_m_dpk] [--iters 2] [--warmup 1]

A seeded synthetic 3-component record already on the device, the golden synthetic parameters of the model
(oracle.golden.model_state_dict), main.py thresholds (P / S 0.3, min_peak_dist 1 s).  Gaps (NaN in every channel) are
added at about one per 10 min per station with lengths uniform in 0.01-60 s; station 0 is also down for 30 min and the
last station has no gap.  Three paths run in one process, alternating, each timed from record to CSR picks (host clock
around work that ends in a synchronise):
  (a) the gapped record:      segments -> annotate(record, segments) -> pick_phases(probs, segments=...)
  (b) the record before the gaps were added: annotate -> pick_phases
  (c) that gap-free record through the segments path, as (a).
Prints the card and its power limit read in the same run, station-hours per second and forward replays of each path,
the CUDA-event time of each phase (scan, cut, forwards, stack, finish, picks) from a separate instrumented pass, the
scan's GB/s over the bytes it must read (the record once), and the peak of torch.cuda.max_memory_allocated during
each path.  The last line is one JSON record.
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


def add_gaps(rec: torch.Tensor, fs: int, seed: int) -> torch.Tensor:
    S, _, T = rec.shape
    rng = np.random.default_rng(seed)
    out = rec.clone()
    minutes = T / fs / 60
    for s in range(S - 1):                                              # the last station stays gap free
        for _ in range(rng.poisson(minutes / 10)):
            a = int(rng.integers(0, T))
            out[s, :, a:a + int(round(rng.uniform(0.01, 60) * fs))] = float("nan")
    down = min(T, 30 * 60 * fs)
    out[0, :, (T - down) // 2:(T - down) // 2 + down] = float("nan")
    return out


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
        raise SystemExit("gap_annotate_bench needs a CUDA device")
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
    replays = [0]
    replay = ann.graph.replay

    def counted():
        replays[0] += 1
        return replay()
    ann.graph.replay = counted

    def seg_path(rec):
        segs = ann.segments(rec)
        probs = ann.annotate(rec, segments=segs)
        picks = ann.pick_phases(probs, segments=segs)
        torch.cuda.synchronize()
        return probs, picks, segs

    def whole_path(rec):
        probs = ann.annotate(rec)
        picks = ann.pick_phases(probs)
        torch.cuda.synchronize()
        return probs, picks, None

    paths = {"a_gapped_segments": (seg_path, gapped), "b_clean_annotate": (whole_path, clean), "c_clean_segments": (seg_path, clean)}
    times = {k: [] for k in paths}
    peak = {k: 0 for k in paths}
    fwd = {}
    out = {}
    for it in range(a.warmup + a.iters):
        for k, (fn, rec) in paths.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            replays[0] = 0
            t0 = time.perf_counter()
            out[k] = fn(rec)
            dt = time.perf_counter() - t0
            peak[k] = max(peak[k], torch.cuda.max_memory_allocated())
            fwd[k] = replays[0]
            if it >= a.warmup:
                times[k].append(dt)
    same = torch.equal(out["b_clean_annotate"][0], out["c_clean_segments"][0]) and all(
        torch.equal(u, v) for key in ("ppk", "spk") for u, v in zip(out["b_clean_annotate"][1][key], out["c_clean_segments"][1][key]))

    # instrumented pass: CUDA events between the phases
    def phases(rec, segmented):
        ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
        ph = {"scan": 0.0, "cut": 0.0, "forwards": 0.0, "stack": 0.0, "finish": 0.0, "picks": 0.0}
        marks = []
        with torch.no_grad():
            e0 = ev()
            e0.record()
            segs = ann.segments(rec) if segmented else None
            e1 = ev()
            e1.record()
            probs = torch.empty(S, 3, T, device="cuda")
            if segmented:
                plan = ST.segment_plan(segs.on, segs.off, W, P, B)
                n_win = int(plan["win_off"][-1])
                win_off = torch.from_numpy(plan["win_off"]).cuda()
                starts = range(0, n_win, B)
            else:
                n_win = S * ann.window_count(T)
                starts = range(0, n_win, B)
            for b, j0 in enumerate(starts):
                es = [ev() for _ in range(4)]
                es[0].record()
                if segmented:
                    ST.segment_window_(ann.graph.x, rec, segs, win_off, n_win, W, P, j0, ann.norm_mode)
                else:
                    ST.window_batch_(ann.graph.x, rec, W, P, j0, ann.norm_mode)
                es[1].record()
                y = replay()
                es[2].record()
                if segmented:
                    ST.segment_stack_(probs, y, segs, win_off, n_win, W, P, j0, int(plan["first"][b]), int(plan["last"][b]), ann.stack)
                else:
                    ST.stack_batch_(probs, y, W, P, j0, ann.stack)
                es[3].record()
                marks.append(es)
            f0, f1, f2 = ev(), ev(), ev()
            f0.record()
            if segmented:
                ST.segment_finish_(probs, segs, W, P, ann.stack)
            else:
                ST.stack_finish_(probs, W, P, ann.stack)
            f1.record()
            ann.pick_phases(probs, segments=segs)
            f2.record()
        torch.cuda.synchronize()
        ph["scan"] = e0.elapsed_time(e1)
        for es in marks:
            ph["cut"] += es[0].elapsed_time(es[1])
            ph["forwards"] += es[1].elapsed_time(es[2])
            ph["stack"] += es[2].elapsed_time(es[3])
        ph["finish"] = f0.elapsed_time(f1)
        ph["picks"] = f1.elapsed_time(f2)
        return ph, probs

    ph = {}
    for k, (fn, rec) in paths.items():
        ph[k], probs = phases(rec, fn is seg_path)
        assert torch.equal(torch.isnan(probs), torch.isnan(out[k][0])) and torch.equal(probs.nan_to_num(), out[k][0].nan_to_num())
    segs = out["a_gapped_segments"][2]
    n_seg = len(segs.on)
    n_ann = int((segs.off - segs.on + 1 >= W).sum())
    lost = float(torch.isnan(out["a_gapped_segments"][0][:, 0]).float().mean())
    scan_bytes = S * 3 * T * 4
    name = card()
    print(f"card: {name}")
    print(f"{a.model}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), W = {W}, P = {P}, batch {B}")
    print(f"gapped record: {n_seg} segments, {n_ann} annotated, {lost * 100:.2f} % of the samples not annotated")
    res = {}
    for k in paths:
        t = float(np.mean(times[k]))
        res[k] = {"ms": t * 1e3, "station_hours_per_s": S * a.hours / t, "replays": fwd[k], "phase_ms": ph[k],
                  "peak_gb": peak[k] / 1e9, "picks_p": out[k][1]["ppk"][0].numel()}
        if k != "b_clean_annotate":
            res[k]["scan_gb_per_s"] = scan_bytes / ph[k]["scan"] / 1e6
        print(f"{k}: {t * 1e3:.1f} ms, {S * a.hours / t:.1f} station-hours/s, {fwd[k]} replays, peak {peak[k] / 1e9:.2f} GB, "
              f"{res[k]['picks_p']} P picks")
        print("  phases (CUDA events, ms): " + ", ".join(f"{p} {v:.2f}" for p, v in ph[k].items())
              + (f"; scan {res[k]['scan_gb_per_s']:.0f} GB/s over the record's bytes" if "scan_gb_per_s" in res[k] else ""))
    print(f"(c) equals (b) bit for bit: {same}")
    print(json.dumps({"card": name, "model": a.model, "stations": S, "T": T, "window": W, "stride": P, "batch": B, "segments": n_seg,
                      "annotated_segments": n_ann, "not_annotated_fraction": lost, "c_equals_b": same, "paths": res}))


if __name__ == "__main__":
    main()
