"""Time the fused training step (seist_b200/train.py) for the losses and optimizers beyond dpk + Adam.

    python tools/train_variants_bench.py [--batch 512] [--length 8192] [--steps 20] [--warmup 3] [--rounds 3]

Cases: `seist_m_pmp` with Adam (the CELoss branch), and `seist_m_dpk` with Adam and with SGD(momentum=0.9), the two
dpk cases timed in alternating rounds in the same run.  Every case is a `Trainer` with the reference's CyclicLR schedule
and the registered drop rates, on seeded synthetic batches already on the device; the first steps warm up and capture
the step's CUDA graph.  A round is CUDA events around `steps` graph replays; the reported ms/step is the median round.
The fused Adam and SGD updates alone are also timed over seist_m_dpk's flat parameter buffer (CUDA events over 200
launches).  Prints the card and its power limit, read in the same run; the last line is one JSON record.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from annotate_bench import card  # noqa: E402
from seist_b200 import _lib  # noqa: E402
from seist_b200.models import create_model  # noqa: E402
from seist_b200.train import Trainer, make_cyclic_lr  # noqa: E402


def batch(head, n, length, seed):
    """N(0,1) standardised waveforms; one-hot int64 class rows (cls) or Gaussian-bump P/S labels and a box (dpk)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, length, generator=g)
    x = (x - x.mean(-1, keepdim=True)) / x.std(-1, keepdim=True)
    if head == "cls":
        return x, torch.eye(2, dtype=torch.int64)[torch.randint(0, 2, (n,), generator=g)]
    t = torch.arange(length, dtype=torch.float32)[None, :]
    p = torch.randint(length // 8, length // 2, (n, 1), generator=g).float()
    s = p + torch.randint(length // 32, length // 4, (n, 1), generator=g).float()
    tgt = torch.zeros(n, 3, length)
    tgt[:, 1] = torch.exp(-((t - p) ** 2) / 200.0)
    tgt[:, 2] = torch.exp(-((t - s) ** 2) / 200.0)
    tgt[:, 0] = ((t >= p) & (t <= s + 2 * (s - p))).float()
    return x, tgt


def rounds_ms(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--length", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "train_variants_bench needs a CUDA device"
    dev = torch.device("cuda")
    gpu = card()
    print(f"card: {gpu}")
    sched = make_cyclic_lr(1000)
    cases = {"seist_m_pmp adam": ("seist_m_pmp", {}),
             "seist_m_dpk adam": ("seist_m_dpk", {}),
             "seist_m_dpk sgd": ("seist_m_dpk", dict(optimizer="sgd", momentum=0.9))}
    runs = {}
    for label, (name, kw) in cases.items():
        torch.manual_seed(0)
        model = create_model(name, in_channels=3, in_samples=args.length).to(dev)
        x, t = batch(model.hp.head, args.batch, args.length, 1234)
        x, t = x.to(dev), t.to(dev)
        tr = Trainer(model, lr_schedule=sched, **kw)
        for _ in range(args.warmup):
            tr.step(x, t)
        assert tr.graph is not None
        runs[label] = (tr, x, t)
    times = {label: [] for label in cases}
    for _ in range(args.rounds):               # alternate the cases so drift in clocks or neighbours hits all of them
        for label, (tr, x, t) in runs.items():
            times[label].append(rounds_ms(lambda: tr.step(x, t), args.steps))
    result = {}
    for label, ts in times.items():
        tr = runs[label][0]
        ms = statistics.median(ts)
        loss = float(tr.loss_out.item())
        result[label] = {"ms_per_step": round(ms, 3), "rounds_ms": [round(v, 3) for v in ts],
                         "waveforms_per_s": round(args.batch / (ms / 1e3), 1), "loss": loss,
                         "launches_per_step": tr.launches_per_step}
        print(f"{label:18s} {ms:8.3f} ms/step  ({', '.join(f'{v:.3f}' for v in ts)})  "
              f"{args.batch / (ms / 1e3):9.1f} waveforms/s  loss {loss:.5f}  {tr.launches_per_step} launches")

    # the two optimizer updates alone, over seist_m_dpk's flat buffer
    tr = runs["seist_m_dpk sgd"][0]
    n = tr.flat.numel
    p, g = torch.randn(n, device=dev) * 1e-2, torch.randn(n, device=dev) * 1e-3
    m, v, buf = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    lr, step = torch.full((1,), 1e-4, device=dev), torch.full((1,), 2.0, device=dev)
    lib, s = _lib.lib(), torch.cuda.current_stream().cuda_stream
    adam = lambda: _lib.check(lib.seist_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, lr.data_ptr(),  # noqa: E731
                                                  step.data_ptr(), 0.9, 0.999, 1e-8, 0.0, 0, 1.0, s))
    sgd = lambda: _lib.check(lib.seist_sgd_step(p.data_ptr(), g.data_ptr(), buf.data_ptr(), n, lr.data_ptr(),  # noqa: E731
                                                step.data_ptr(), 0.9, 0.0, 0.0, 0, 1.0, s))
    for f in (adam, sgd):
        for _ in range(10):
            f()
    upd = {"numel": n, "adam_us": round(1e3 * rounds_ms(adam, 200), 2), "sgd_us": round(1e3 * rounds_ms(sgd, 200), 2)}
    print(f"flat update over {n} parameters: adam {upd['adam_us']:.2f} us, sgd {upd['sgd_us']:.2f} us")
    print(json.dumps({"card": gpu, "batch": args.batch, "length": args.length, "steps": args.steps,
                      "rounds": args.rounds, "cases": result, "update_alone": upd}))


if __name__ == "__main__":
    main()
