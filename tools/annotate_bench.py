"""Time continuous annotation on the device: record -> stacked probabilities -> CSR picks and detections.

    python tools/annotate_bench.py [--stations 4] [--hours 24] [--fs 100] [--window 8192] [--stride 4096] [--batch 256]
                                   [--model seist_m_dpk] [--iters 3] [--warmup 1]

A seeded synthetic 3-component record of `stations` x `hours` at `fs` Hz already on the device, the golden synthetic
parameters of the model (oracle.golden.model_state_dict), `ContinuousAnnotator` with the main.py thresholds (P / S 0.3,
det 0.5, min_peak_dist 1 s).  Prints the card and its power limit read in the same run, station-hours annotated per second
from record to CSR picks (host clock around work that ends in a synchronise), the CUDA-event time of each phase (window
cut, forward, stack, pick + detect) from a separate instrumented pass, and the achieved GB/s of the window and stack
kernels over the bytes they must move.  The last line is one JSON record.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden as G  # noqa: E402
from seist_b200 import stream as ST  # noqa: E402
from seist_b200.models import create_model  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def stack_bytes(S, T, W, P, B):
    """Window outputs read once; every probability sample a batch covers read and written once by that batch."""
    starts = ST.window_starts(T, W, P)
    K = len(starts)
    total = S * K * 3 * W * 4
    for w0 in range(0, S * K, B):
        w1 = min(w0 + B, S * K) - 1
        for s in range(w0 // K, w1 // K + 1):
            ka, kb = max(w0 - s * K, 0), min(w1 - s * K, K - 1)
            total += 2 * 3 * 4 * (starts[kb] + W - starts[ka])
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=4)
    ap.add_argument("--hours", type=float, default=24.0)
    ap.add_argument("--fs", type=int, default=100)
    ap.add_argument("--window", type=int, default=8192)
    ap.add_argument("--stride", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--model", default="seist_m_dpk")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("annotate_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    m = create_model(a.model, in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict(a.model, W), strict=True)
    m = m.cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    rec = torch.randn(S, 3, T, device="cuda", generator=g) * 5.0
    ann = ST.ContinuousAnnotator(m, window=W, stride=P, batch=B)
    mpd = int(1.0 * a.fs)

    def run():
        probs = ann.annotate(rec)
        picks = ann.pick_phases(probs, 0.3, 0.3, mpd)
        dets = ann.detect_events(probs, 0.5)
        torch.cuda.synchronize()
        return probs, picks, dets

    for _ in range(a.warmup):
        run()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        probs, picks, dets = run()
    e2e = (time.perf_counter() - t0) / a.iters

    # instrumented pass: events between the phases of every batch
    K = ann.window_count(T)
    n = S * K
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4 * ((n + B - 1) // B) + 2)]
    ph = {"window": 0.0, "forward": 0.0, "stack": 0.0}
    probs2 = torch.empty(S, 3, T, device="cuda")
    i = 0
    with torch.no_grad():
        for w0 in range(0, n, B):
            ev[i].record()
            ST.window_batch_(ann.graph.x, rec, W, P, w0, ann.norm_mode)
            ev[i + 1].record()
            y = ann.graph.replay()
            ev[i + 2].record()
            ST.stack_batch_(probs2, y, W, P, w0, ann.stack)
            ev[i + 3].record()
            i += 4
        f0 = torch.cuda.Event(enable_timing=True)
        f0.record()
        ST.stack_finish_(probs2, W, P, ann.stack)
        ev[i].record()
        ann.pick_phases(probs2, 0.3, 0.3, mpd)
        ann.detect_events(probs2, 0.5)
        ev[i + 1].record()
    torch.cuda.synchronize()
    for j in range(0, i, 4):
        ph["window"] += ev[j].elapsed_time(ev[j + 1])
        ph["forward"] += ev[j + 1].elapsed_time(ev[j + 2])
        ph["stack"] += ev[j + 2].elapsed_time(ev[j + 3])
    ph["stack_finish"] = f0.elapsed_time(ev[i])
    ph["pick_detect"] = ev[i].elapsed_time(ev[i + 1])
    assert torch.equal(probs, probs2)

    win_bytes = n * 3 * W * 4 * 2                  # record slice read once, normalised row written once
    stk_bytes = stack_bytes(S, T, W, P, B)
    name = card()
    n_p, n_s, n_d = picks["ppk"][0].numel(), picks["spk"][0].numel(), dets[0].shape[0]
    print(f"card: {name}")
    print(f"{a.model}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), W = {W}, P = {P}, batch {B}: {n} windows")
    print(f"end to end (record -> CSR picks + detections): {e2e * 1e3:.1f} ms, {S * a.hours / e2e:.1f} station-hours/s")
    print("phases (CUDA events, ms): " + ", ".join(f"{k} {v:.2f}" for k, v in ph.items()))
    print(f"window kernel {win_bytes / ph['window'] / 1e6:.0f} GB/s, stack kernel {stk_bytes / ph['stack'] / 1e6:.0f} GB/s")
    print(f"picks: {n_p} P, {n_s} S, {n_d} detections")
    print(json.dumps({"card": name, "model": a.model, "stations": S, "T": T, "window": W, "stride": P, "batch": B, "windows": n,
                      "e2e_ms": e2e * 1e3, "station_hours_per_s": S * a.hours / e2e, "phase_ms": ph,
                      "window_gb_per_s": win_bytes / ph["window"] / 1e6, "stack_gb_per_s": stk_bytes / ph["stack"] / 1e6,
                      "picks_p": n_p, "picks_s": n_s, "detections": n_d}))


if __name__ == "__main__":
    main()
