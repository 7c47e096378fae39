"""Time a network of mixed input rates in one Resampler (seist_b200/resample.py, DESIGN §4.24) against one single-rate
Resampler per rate group.

    python tools/network_resample_bench.py [--hours 1] [--chunk-s 60] [--out 50] [--iters 5] [--warmup 2]

Seeded synthetic 3-component records already on the device: 256 stations, 128 at 100 Hz, 64 at 40 Hz, 32 at 200 Hz and
32 at 50 Hz, `hours` long each, resampled to `out` Hz.  Whole records: the mixed Resampler's one call against four
single-rate Resamplers plus assembling their outputs into the same padded (S, C, T_max) record.  Streams of `chunk-s`
second list pushes (cut before timing): the mixed stream against four single-rate streams with each push split into rate
groups and the outputs merged back into station order.  Both sides are checked equal.  Times are CUDA events over `iters`
calls after `warmup`; GB/s is the compulsory bytes 4 * C * (sum T_in + sum T_out) over the time, also as a share of the
H100 SXM's 3.35 TB/s.  Prints the card and its power limit read in the same run; the last line is one JSON record.
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
from resample_bench import HBM, timed  # noqa: E402
from seist_b200.resample import Resampler  # noqa: E402

GROUPS = ((100, 128), (40, 64), (200, 32), (50, 32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--chunk-s", type=int, default=60)
    ap.add_argument("--out", type=int, default=50)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("network_resample_bench needs a CUDA device")
    C = 3
    name = card()
    print(f"card: {name}")
    rates = [f for f, n in GROUPS for _ in range(n)]
    S = len(rates)
    g = torch.Generator(device="cuda").manual_seed(0)
    pieces = [torch.randn(C, int(round(a.hours * 3600 * f)), device="cuda", generator=g) * 5.0 for f in rates]
    members = {f: [s for s in range(S) if rates[s] == f] for f, _ in GROUPS}
    mixed = Resampler(rates, a.out)
    single = {f: Resampler(f, a.out) for f, _ in GROUPS}
    T_out = mixed.output_lengths([p.shape[1] for p in pieces])
    T_max = int(T_out.max())
    nbytes = 4 * C * (sum(p.shape[1] for p in pieces) + int(T_out.sum()))
    grouped = {f: torch.stack([pieces[s] for s in members[f]]) for f in members}

    def per_group():
        out = torch.full((S, C, T_max), float("nan"), device="cuda")
        for f, idx in members.items():
            y = single[f](grouped[f])
            out[torch.tensor(idx, device="cuda"), :, :y.shape[2]] = y
        return out
    res = {}
    t_mixed, y_mixed = timed(lambda: mixed(pieces), a.iters, a.warmup)
    t_group, y_group = timed(per_group, a.iters, a.warmup)
    assert torch.equal(torch.isnan(y_mixed), torch.isnan(y_group)) and torch.equal(y_mixed.nan_to_num(), y_group.nan_to_num())
    res["whole mixed"], res["whole per group"] = t_mixed, t_group
    del y_group, grouped

    n_push = -(-int(round(a.hours * 3600)) // a.chunk_s)
    pushes = [[p[:, i * a.chunk_s * f:(i + 1) * a.chunk_s * f].contiguous() for p, f in zip(pieces, rates)] for i in range(n_push)]

    def stream_mixed():
        st = mixed.open_stream(S, C)
        return [st.push(c) for c in pushes] + [st.close()]

    def stream_group():
        sts = {f: single[f].open_stream(len(idx), C) for f, idx in members.items()}
        outs = []
        for c in pushes + [None]:
            merged = [None] * S
            for f, idx in members.items():
                y = sts[f].push([c[s] for s in idx]) if c is not None else sts[f].close()
                for s, ys in zip(idx, y):
                    merged[s] = ys
            outs.append(merged)
        return outs
    it = max(1, a.iters // 2)
    t_smixed, o_mixed = timed(stream_mixed, it, 1)
    t_sgroup, o_group = timed(stream_group, it, 1)
    for s in range(S):
        whole = torch.cat([o[s] for o in o_mixed], 1)
        assert torch.equal(whole, torch.cat([o[s] for o in o_group], 1)) and torch.equal(whole, y_mixed[s, :, :T_out[s]]), s
    res["stream mixed"], res["stream per group"] = t_smixed, t_sgroup
    cases = {}
    for key, t in res.items():
        cases[key] = {"ms": t * 1e3, "station_hours_per_s": S * a.hours / t, "gb_per_s": nbytes / t / 1e9, "hbm_share": nbytes / t / HBM}
        r = cases[key]
        print(f"{key}: {S} stations x {a.hours:g} h to {a.out} Hz: {r['ms']:.3f} ms, {r['station_hours_per_s']:.0f} station-hours/s, "
              f"{r['gb_per_s']:.0f} GB/s = {100 * r['hbm_share']:.1f}% of 3.35 TB/s")
    print(json.dumps({"card": name, "stations": S, "groups": GROUPS, "hours": a.hours, "chunk_s": a.chunk_s, "out": a.out,
                      "pushes": len(pushes) + 1, "table_rows": len(mixed.table), "cases": cases}))


if __name__ == "__main__":
    main()
