"""Stream a continuous record chunk by chunk and compare it with whole-record annotation in the same run.

    python tools/stream_bench.py [--stations 256] [--hours 1] [--fs 100] [--chunk-s 60] [--window 8192] [--stride 4096]
                                 [--batch 256] [--model seist_m_dpk] [--iters 2] [--warmup 1]

A seeded synthetic 3-component record (as tools/annotate_bench.py builds it) already on the device, the golden synthetic
parameters of the model, the main.py thresholds (P / S 0.3, det 0.5, min_peak_dist 1 s).  The two modes alternate:
"stream" pushes the record in (contiguous copies of) chunks of `chunk-s` seconds through `ContinuousAnnotator.open_stream` and closes it;
"whole" runs `annotate` + `pick_phases` + `detect_events` on the whole record.  For each mode: station-hours per second
(host clock around work that ends in a synchronise), the peak `torch.cuda.max_memory_allocated` (the record itself
included) and the number of forward replays.  Asserts that both modes give identical probabilities, picks and
detections.  Prints the card and its power limit read in the same run; the last line is one JSON record.
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
from seist_b200 import stream as ST  # noqa: E402
from seist_b200.models import create_model  # noqa: E402


def per_station(csr, S):
    *vals, off = csr
    o = off.tolist()
    return [[v[o[s]:o[s + 1]] for v in vals] for s in range(S)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=256)
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--fs", type=int, default=100)
    ap.add_argument("--chunk-s", type=float, default=60.0)
    ap.add_argument("--window", type=int, default=8192)
    ap.add_argument("--stride", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--model", default="seist_m_dpk")
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_bench needs a CUDA device")
    S, W, P, B = a.stations, a.window, a.stride, a.batch
    T = int(round(a.hours * 3600 * a.fs))
    n = int(round(a.chunk_s * a.fs))
    m = create_model(a.model, in_channels=3, in_samples=W)
    m.load_state_dict(G.model_state_dict(a.model, W), strict=True)
    m = m.cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    rec = torch.randn(S, 3, T, device="cuda", generator=g) * 5.0
    ann = ST.ContinuousAnnotator(m, window=W, stride=P, batch=B)
    ann.min_peak_dist = int(1.0 * a.fs)

    def whole():
        probs = ann.annotate(rec)
        picks = ann.pick_phases(probs)
        dets = ann.detect_events(probs)
        torch.cuda.synchronize()
        return probs, picks["ppk"], picks["spk"], dets, (S * ann.window_count(T) + B - 1) // B

    def stream():
        st = ann.open_stream(S)
        outs = [st.push(rec[:, :, i:i + n].contiguous()) for i in range(0, T, n)] + [st.close()]
        torch.cuda.synchronize()
        return outs, st.forwards

    res = {"whole": [], "stream": []}
    peak = {}
    for it in range(a.warmup + a.iters):
        for mode in ("stream", "whole"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            out = stream() if mode == "stream" else whole()
            dt = time.perf_counter() - t0
            peak[mode] = torch.cuda.max_memory_allocated()
            if it >= a.warmup:
                res[mode].append(dt)
            if mode == "stream":
                s_out, s_fw = out
            else:
                w_out = out
    probs = torch.cat([o.probs for o in s_out], 2)
    assert torch.equal(probs, w_out[0]), "stream probabilities differ from annotate"
    for k, name in ((2, "ppk"), (3, "spk"), (4, "det")):
        want = per_station(w_out[k - 1], S)
        got = [per_station(getattr(o, name), S) for o in s_out]
        for s in range(S):
            for j in range(len(want[s])):
                assert torch.equal(torch.cat([gg[s][j] for gg in got]), want[s][j]), (name, s)
    name = card()
    sh = S * a.hours
    rate = {k: sh / (sum(v) / len(v)) for k, v in res.items()}
    fw = {"stream": s_fw, "whole": w_out[4]}
    print(f"card: {name}")
    print(f"{a.model}, {S} stations x {a.hours:g} h at {a.fs} Hz (T = {T}), chunks of {n} samples, W = {W}, P = {P}, batch {B}")
    for k in ("stream", "whole"):
        print(f"{k:>6}: {rate[k]:.1f} station-hours/s, peak memory {peak[k] / 2**20:.0f} MiB (record {rec.numel() * 4 / 2**20:.0f} MiB), "
              f"{fw[k]} forward replays")
    print("outputs identical: probabilities, picks and detections")
    print(json.dumps({"card": name, "model": a.model, "stations": S, "T": T, "chunk": n, "window": W, "stride": P, "batch": B,
                      "station_hours_per_s": rate, "peak_bytes": peak, "forwards": fw, "identical": True}))


if __name__ == "__main__":
    main()
