"""Time the device input pipeline: DevicePreprocessor.process_batch (augmentation, cut, normalisation) + dpk_soft_labels.

    python tools/augbench.py [--batch 512] [--raw 9000] [--in-samples 8192] [--iters 50] [--warmup 5]

main.py's default rates at 50 Hz, every trace augmented (the reference's augmented half of an epoch), one event per
trace.  Prints the card and its power limit read in the same run, the device time per batch from CUDA events, the
algorithmic bytes (raw traces read, model input and labels written) with the achieved rate, and the CPU time per event of
the numpy oracle (tests/augment_ref.py with the device's draws) for the same configuration - the oracle, not the
reference.  The last line is one JSON record.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from seist_b200 import preprocess as PP  # noqa: E402

DEFAULTS = dict(data_channels=["z", "n", "e"], sampling_rate=50, min_snr=-float("inf"), p_position_ratio=-1, coda_ratio=2.0,
                norm_mode="std", add_event_rate=0.0, add_noise_rate=0.4, add_gap_rate=0.4, drop_channel_rate=0.4,
                scale_amplitude_rate=0.4, pre_emphasis_rate=0.4, pre_emphasis_ratio=0.97, max_event_num=1,
                generate_noise_rate=0.05, shift_event_rate=0.2, mask_percent=0, noise_percent=0, min_event_gap_sec=0.5,
                soft_label_shape="gaussian", soft_label_width=25)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--raw", type=int, default=9000)
    ap.add_argument("--in-samples", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--oracle-events", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augbench needs a CUDA device")
    n, lin, w = a.batch, a.raw, a.in_samples
    cfg = dict(DEFAULTS, in_samples=w)
    rng = np.random.default_rng(0)
    data = (rng.standard_normal((n, 3, lin)) * rng.uniform(0.5, 20, (n, 3, 1))).astype(np.float32)
    p = rng.integers(300, lin - 2000, (n, 1))
    s = p + rng.integers(50, 1500, (n, 1))
    dp = PP.DevicePreprocessor(**cfg)
    xd, pd, sd = torch.from_numpy(data).cuda(), torch.from_numpy(p).cuda(), torch.from_numpy(s).cuda()

    def run():
        x, po, so, _ = dp.process_batch(xd, pd, sd)
        return x, dp.labels(po, so)

    for _ in range(a.warmup):
        run()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(a.iters):
        run()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / a.iters
    nbytes = n * 3 * lin * 4 + n * 3 * w * 4 + n * 3 * w * 4 + 2 * 2 * n * 8

    import augment_ref as AR
    pre = AR.Preprocessor(**cfg)
    m = min(a.oracle_events, n)
    c0 = time.perf_counter()
    for i in range(m):
        _, wp, ws, _ = pre.process(data[i], [int(p[i, 0])], [int(s[i, 0])], None, True, AR.CounterDraws(1, i, 3))
        AR.dpk_labels(wp, ws, w, cfg["soft_label_width"], cfg["soft_label_shape"], cfg["coda_ratio"])
    oracle_ms = (time.perf_counter() - c0) * 1e3 / m

    name = card()
    print(f"card: {name}")
    print(f"device: process_batch + dpk_soft_labels, B = {n}, {lin} -> {w} samples: {ms:.3f} ms per batch, "
          f"{nbytes / 1e6:.1f} MB algorithmic, {nbytes / ms / 1e6:.0f} GB/s")
    print(f"numpy oracle (not the reference), one CPU core: {oracle_ms:.3f} ms per event")
    print(json.dumps({"card": name, "batch": n, "raw": lin, "in_samples": w, "device_ms_per_batch": ms, "bytes": nbytes,
                      "gb_per_s": nbytes / ms / 1e6, "oracle_cpu_ms_per_event": oracle_ms}))


if __name__ == "__main__":
    main()
