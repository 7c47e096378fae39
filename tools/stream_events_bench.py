"""Stream a continuous record chunk by chunk with every P pick characterised as it closes, against a plain stream of the
same record in the same run.

    python tools/stream_events_bench.py [--stations 256] [--hours 1] [--fs 100] [--chunk-s 60] [--window 8192]
                                        [--stride 4096] [--batch 256] [--ratio 0.3] [--size m] [--per-min 3]
                                        [--iters 2] [--warmup 1]

A seeded synthetic 3-component record already on the device (as tools/stream_bench.py builds it), the golden synthetic
parameters of seist_<size>_dpk and seist_<size>_{pmp, emg, baz, dis}, min_peak_dist 1 s.  The P threshold is bisected on
the whole record's probabilities so that the picker yields about `per-min` P picks per station-minute (the synthetic
parameters have no calibrated threshold).  Two modes alternate: "events" pushes the record in (contiguous copies of)
chunks of `chunk-s` seconds through `EventCharacterizer.open_stream` and closes it; "plain" does the same through
`ContinuousAnnotator.open_stream`.  For each: station-hours per second (host clock around work that ends in a
synchronise); for "events" also events per second, the peak `torch.cuda.max_memory_allocated` (the record included) and
the largest `held_samples`.  A separate instrumented pass times the history kernel and the window cuts with CUDA events.
Asserts that the streamed events equal `EventCharacterizer` on the whole record's picks bit for bit.  Prints the card and
its power limit read in the same run; the last line is one JSON record.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from annotate_bench import card  # noqa: E402
from oracle import golden as G  # noqa: E402
from seist_b200 import events as EV  # noqa: E402
from seist_b200 import stream as ST  # noqa: E402
from seist_b200.models import create_model  # noqa: E402

HEADS = ("pmp", "emg", "baz", "dis")


def load(name, W):
    m = create_model(name, in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict(name, W), strict=True)
    return m.cuda().eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=256)
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--fs", type=int, default=100)
    ap.add_argument("--chunk-s", type=float, default=60.0)
    ap.add_argument("--window", type=int, default=8192)
    ap.add_argument("--stride", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--ratio", type=float, default=0.3)
    ap.add_argument("--size", default="m")
    ap.add_argument("--per-min", type=float, default=3.0)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_events_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    n = int(round(a.chunk_s * a.fs))
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

    chunks = [(i, min(n, T - i)) for i in range(0, T, n)]

    def events():
        cs = ch.open_stream(ann, S)
        outs, held = [], 0
        for i, k in chunks:
            c = cs.push(rec[:, :, i:i + k].contiguous())
            outs.append((c.out.ppk[2], c.events))          # not the probabilities: memory held is the stream's
            held = max(held, cs.held_samples)
        c = cs.close()
        outs.append((c.out.ppk[2], c.events))
        torch.cuda.synchronize()
        return outs, held

    def plain():
        st = ann.open_stream(S)
        for i, k in chunks:
            st.push(rec[:, :, i:i + k].contiguous())
        st.close()
        torch.cuda.synchronize()

    res = {"events": [], "plain": []}
    for it in range(a.warmup + a.iters):
        for mode in ("events", "plain"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            out = events() if mode == "events" else plain()
            dt = time.perf_counter() - t0
            if mode == "events":
                peak = torch.cuda.max_memory_allocated()
                outs, held = out
            if it >= a.warmup:
                res[mode].append(dt)

    # the streamed events, per station in call order, against the whole record
    o = ppk[2].tolist()
    for h in HEADS:
        parts = []
        for s in range(S):
            for off, ev in outs:
                off = off.tolist()
                parts.append(ev[h][off[s]:off[s + 1]])
        assert torch.equal(torch.cat(parts), want[h]), h
    assert sum(int(off[-1]) for off, _ in outs) == M == o[-1]

    # instrumented pass: CUDA events around every history launch and every cut
    spans = {"history": [], "cut": []}
    orig = {"history": EV.ragged_history_, "cut": EV.event_windows_}

    def timed(kind):
        def f(*args, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = orig[kind](*args, **kw)
            e1.record()
            spans[kind].append((e0, e1))
            return r
        return f

    EV.ragged_history_, EV.event_windows_ = timed("history"), timed("cut")
    try:
        events()
    finally:
        EV.ragged_history_, EV.event_windows_ = orig["history"], orig["cut"]
    ms = {k: sum(e0.elapsed_time(e1) for e0, e1 in v) for k, v in spans.items()}

    name = card()
    sh = S * a.hours
    t = {k: sum(v) / len(v) for k, v in res.items()}
    rate = {k: sh / v for k, v in t.items()}
    print(f"card: {name}")
    print(f"seist_{a.size}_dpk + seist_{a.size}_{{{','.join(HEADS)}}}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), "
          f"chunks of {n} samples, W = {W}, P = {P}, batch {B}, p_position_ratio {a.ratio}")
    print(f"P threshold {ann.thresholds['ppk']:.6f}: M = {M} P picks ({M / (S * a.hours * 60):.2f} per station-minute)")
    print(f"events: {rate['events']:.1f} station-hours/s, {M / t['events']:.0f} events/s, peak memory {peak / 2**20:.0f} MiB "
          f"(record {rec.numel() * 4 / 2**20:.0f} MiB), largest held_samples {held}")
    print(f" plain: {rate['plain']:.1f} station-hours/s")
    print(f"CUDA events: history {ms['history']:.2f} ms over {len(spans['history'])} launches, "
          f"cuts {ms['cut']:.2f} ms over {len(spans['cut'])} launches")
    print("streamed events identical to the whole-record characterisation")
    print(json.dumps({"card": name, "size": a.size, "stations": S, "T": T, "chunk": n, "window": W, "stride": P, "batch": B,
                      "ratio": a.ratio, "ppk_threshold": ann.thresholds["ppk"], "events": M,
                      "station_hours_per_s": rate, "events_per_s": M / t["events"], "seconds": t, "history_ms": ms["history"],
                      "cut_ms": ms["cut"], "peak_bytes": peak, "max_held_samples": held, "identical": True}))


if __name__ == "__main__":
    main()
