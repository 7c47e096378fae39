"""Time the characterisation of picked events on the device: P pick CSR -> P-anchored windows -> polarity, magnitude,
back-azimuth and distance for every pick.

    python tools/characterize_bench.py [--stations 256] [--hours 1] [--fs 100] [--every 30] [--window 8192]
                                       [--ratio 0.3] [--batch 256] [--size m] [--iters 3] [--warmup 1]

A seeded synthetic 3-component record of `stations` x `hours` at `fs` Hz already on the device, seeded P picks about every
`every` seconds per station, the golden synthetic parameters (oracle.golden.model_state_dict) of seist_<size>_{pmp, emg,
baz, dis}, `EventCharacterizer` with norm_mode "std".  Prints the card and its power limit read in the same run, events
characterised per second with 1 model (pmp) and with all 4 (host clock around work that ends in a synchronise), the
CUDA-event time of the window cut versus the forwards from a separate instrumented pass of the 4 models, the cut kernel's
achieved GB/s over its compulsory bytes (C * W * 4 read and n_dst * C * W * 4 written per event) and the peak
`torch.cuda.max_memory_allocated`.  The last line is one JSON record.
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
from seist_b200 import events as EV  # noqa: E402
from seist_b200.models import create_model  # noqa: E402

HEADS = ("pmp", "emg", "baz", "dis")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def seeded_picks(S, T, step, seed=0):
    """P picks at k * step + a seeded jitter in [0, step / 2) per station, k = 0, 1, ... while inside [0, T): CSR."""
    g = torch.Generator().manual_seed(seed)
    per = (T + step - 1) // step
    p = torch.arange(per, dtype=torch.int64) * step + torch.randint(0, max(step // 2, 1), (S, per), generator=g)
    counts = (p < T).sum(1)
    index = p[p < T]                                       # row-major: station by station, ascending
    offsets = torch.zeros(S + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(counts, 0)
    return index.cuda(), offsets.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=256)
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--fs", type=int, default=100)
    ap.add_argument("--every", type=float, default=30.0)
    ap.add_argument("--window", type=int, default=8192)
    ap.add_argument("--ratio", type=float, default=0.3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", default="m")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("characterize_bench needs a CUDA device")
    S, W, B = a.stations, a.window, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    models = {}
    for h in HEADS:
        name = f"seist_{a.size}_{h}"
        m = create_model(name, in_channels=3, in_samples=W)
        m.load_state_dict(G.model_state_dict(name, W), strict=True)
        models[h] = m.cuda().eval()
    gen = torch.Generator(device="cuda").manual_seed(0)
    rec = torch.randn(S, 3, T, device="cuda", generator=gen) * 5.0
    index, offsets = seeded_picks(S, T, int(a.every * a.fs))
    M = index.numel()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    rate, outs = {}, {}
    for label, sel in (("1", ("pmp",)), ("4", HEADS)):
        ch = EV.EventCharacterizer({h: models[h] for h in sel}, window=W, p_position_ratio=a.ratio, batch=B)
        for _ in range(a.warmup):
            ch(rec, (index, offsets))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            out = ch(rec, (index, offsets))
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / a.iters
        rate[label] = {"ms": dt * 1e3, "events_per_s": M / dt}
        outs[label] = out

    # instrumented pass of the 4 models: events around the cut and the forwards of every batch
    nb = (M + B - 1) // B
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3 * nb)]
    xs = [g.x for g in ch.graphs.values()]
    ph = {"cut": 0.0, "forwards": 0.0}
    with torch.no_grad():
        for j, e0 in enumerate(range(0, M, B)):
            ev[3 * j].record()
            EV.event_windows_(xs, rec, index, offsets, e0, W, ch.anchor, ch.norm_mode)
            ev[3 * j + 1].record()
            for g in ch.graphs.values():
                g.replay()
            ev[3 * j + 2].record()
    torch.cuda.synchronize()
    for j in range(nb):
        ph["cut"] += ev[3 * j].elapsed_time(ev[3 * j + 1])
        ph["forwards"] += ev[3 * j + 1].elapsed_time(ev[3 * j + 2])
    share = ph["cut"] / (ph["cut"] + ph["forwards"])
    assert torch.equal(outs["1"]["pmp"], outs["4"]["pmp"])
    cut_bytes = M * 3 * W * 4 * (1 + len(HEADS))
    peak = torch.cuda.max_memory_allocated()
    name = card()
    print(f"card: {name}")
    print(f"seist_{a.size}_{{{','.join(HEADS)}}}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), W = {W}, "
          f"p_position_ratio {a.ratio}, batch {B}: {M} P picks")
    print(f"1 model: {rate['1']['ms']:.1f} ms, {rate['1']['events_per_s']:.0f} events/s; "
          f"4 models: {rate['4']['ms']:.1f} ms, {rate['4']['events_per_s']:.0f} events/s")
    print(f"4 models, CUDA events: cut {ph['cut']:.2f} ms ({100 * share:.2f} %), forwards {ph['forwards']:.1f} ms")
    print(f"cut kernel {cut_bytes / ph['cut'] / 1e6:.0f} GB/s over {cut_bytes / 1e9:.2f} GB compulsory")
    print(f"peak max_memory_allocated {peak / 2 ** 30:.2f} GiB (record {rec.numel() * 4 / 2 ** 30:.2f} GiB)")
    print(json.dumps({"card": name, "size": a.size, "stations": S, "T": T, "window": W, "ratio": a.ratio, "batch": B,
                      "events": M, "models_1": rate["1"], "models_4": rate["4"], "phase_ms_4": ph, "cut_share": share,
                      "cut_gb_per_s": cut_bytes / ph["cut"] / 1e6, "peak_bytes": peak}))


if __name__ == "__main__":
    main()
