"""Time polyphase resampling on the device (seist_b200/resample.py, DESIGN §4.24) and, for context, annotation of the
resampled record.

    python tools/resample_bench.py [--stations 256] [--hours 1] [--chunk-s 60] [--model seist_m_dpk] [--iters 5] [--warmup 2]

Seeded synthetic 3-component records of `stations` x `hours` already on the device, resampled 100 -> 50 Hz and 40 -> 100 Hz,
each as a whole record and as a stream of tensor pushes of `chunk-s` seconds (the chunks cut before timing).  Times are
CUDA events over `iters` calls after `warmup`.  Prints the card and its power limit read in the same run; per case the
time, station-hours/s and the compulsory bytes 4 * S * C * (T_in + T_out) over the time as GB/s and as a share of the
H100 SXM's 3.35 TB/s; then the time of `annotate` of the 100 -> 50 Hz record with `model` (golden synthetic parameters)
and the share resampling adds to it.  The last line is one JSON record.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from annotate_bench import card  # noqa: E402
from oracle import golden as G  # noqa: E402
from seist_b200 import stream as ST  # noqa: E402
from seist_b200.models import create_model  # noqa: E402
from seist_b200.resample import Resampler  # noqa: E402

HBM = 3.35e12


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters / 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stations", type=int, default=256)
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--chunk-s", type=int, default=60)
    ap.add_argument("--model", default="seist_m_dpk")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resample_bench needs a CUDA device")
    S, C = a.stations, 3
    g = torch.Generator(device="cuda").manual_seed(0)
    name = card()
    print(f"card: {name}")
    res, resampled = {}, None
    for fin, fout in ((100, 50), (40, 100)):
        rs = Resampler(fin, fout)
        T = int(round(a.hours * 3600 * fin))
        x = torch.randn(S, C, T, device="cuda", generator=g) * 5.0
        t_whole, y = timed(lambda: rs(x), a.iters, a.warmup)
        n = a.chunk_s * fin
        chunks = [x[:, :, i:i + n].contiguous() for i in range(0, T, n)]

        def stream():
            st = rs.open_stream(S, C)
            parts = [st.push(c) for c in chunks] + [st.close()]
            return parts
        t_stream, parts = timed(stream, max(1, a.iters // 2), 1)
        assert torch.equal(torch.cat(parts, 2), y)
        nbytes = 4 * S * C * (T + y.shape[2])
        for kind, t in (("whole", t_whole), ("stream", t_stream)):
            key = f"{fin}->{fout} {kind}"
            res[key] = {"ms": t * 1e3, "station_hours_per_s": S * a.hours / t, "gb_per_s": nbytes / t / 1e9,
                        "hbm_share": nbytes / t / HBM, "pushes": len(chunks) + 1 if kind == "stream" else 1}
            r = res[key]
            print(f"{key}: {S} stations x {a.hours:g} h, T {T} -> {y.shape[2]}: {r['ms']:.3f} ms, "
                  f"{r['station_hours_per_s']:.0f} station-hours/s, {r['gb_per_s']:.0f} GB/s = {100 * r['hbm_share']:.1f}% of 3.35 TB/s")
        if (fin, fout) == (100, 50):
            resampled = y
        del x, chunks, parts, y
    m = create_model(a.model, in_channels=3, in_samples=8192)
    m.load_state_dict(G.model_state_dict(a.model, 8192), strict=True)
    ann = ST.ContinuousAnnotator(m.cuda().eval(), window=8192, stride=4096, batch=256)
    t_ann, _ = timed(lambda: ann.annotate(resampled), 2, 1)
    share = res["100->50 whole"]["ms"] / (t_ann * 1e3)
    print(f"annotate of the 50 Hz record with {a.model}: {t_ann * 1e3:.1f} ms; resampling 100 -> 50 Hz adds {100 * share:.1f}%")
    print(json.dumps({"card": name, "stations": S, "hours": a.hours, "chunk_s": a.chunk_s, "cases": res,
                      "annotate_ms": t_ann * 1e3, "resample_share_of_annotate": share}))


if __name__ == "__main__":
    main()
