#!/usr/bin/env python
"""MonoRecModel.forward eager, by CUDA-graph replay (GraphedMonoRec) and under torch.compile, on one GPU: B 8, 256x512,
2 source frames, D 32, f16 mode, the random-init reference architecture.

  eager_host_ms      host time of one eager forward call (the call returns before the device finishes)
  eager_ms           eager forward, host clock around calls that end in a synchronise
  eager_device_ms    CUDA events around one eager forward
  graphed_ms         GraphedMonoRec replay (inputs copied into the static buffers)
  compile_ms         torch.compile(model, fullgraph=True) (Inductor)
  reduce_overhead_ms torch.compile(model, fullgraph=True, mode="reduce-overhead")
  *_first_s          first call of each compiled variant (tracing + compilation + the run)

Every timed variant runs once per round, in turn, and the median over the rounds is reported; each round times `--steps`
calls after the warm-up.  The outputs of every variant are checked against eager (bit for bit).  Prints one JSON line with
the card's name, power limit and maximum SM clock.

`--eager-only --root DIR` times only the eager forward of the package in DIR (another checkout), so that two builds can be
compared by alternating processes.

    python tools/time_compile.py [--rounds 7] [--steps 10] [--warmup 3] [--eager-only --root DIR]
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=7)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--eager-only", action="store_true")
ap.add_argument("--root", default=str(Path(__file__).resolve().parent.parent))
args = ap.parse_args()
sys.path.insert(0, args.root)

import torch  # noqa: E402

from monorec_b200 import conv as C  # noqa: E402
from monorec_b200.model import GraphedMonoRec, MonoRecModel  # noqa: E402
from monorec_b200.synthetic import make_inputs, to_device  # noqa: E402

B, F, H, W = 8, 2, 256, 512


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def wall(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def host(fn, steps):
    """Mean host time of a call; the device is drained after each so the host never waits on a full queue."""
    total = 0.0
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        total += time.perf_counter() - t0
    torch.cuda.synchronize()
    return total / steps * 1e3


def device(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(steps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        total += a.elapsed_time(b)
    return total / steps


def main():
    if not torch.cuda.is_available():
        raise SystemExit("time_compile.py needs a GPU")
    C.set_mode("f16")
    torch.manual_seed(0)
    model = MonoRecModel().to("cuda:0").eval()
    data = to_device(make_inputs(B, F, H, W, seed=1), "cuda:0")
    res = {"card": card(), "mode": "f16", "batch": B, "shape": [F, H, W], "rounds": args.rounds, "steps": args.steps,
           "root": args.root}
    with torch.no_grad():
        eager = lambda: model(dict(data))    # noqa: E731
        for _ in range(args.warmup):
            ref = eager()
        variants = {"eager_host_ms": lambda: host(eager, args.steps), "eager_ms": lambda: wall(eager, args.steps),
                    "eager_device_ms": lambda: device(eager, args.steps)}
        outs = {}
        if not args.eager_only:
            graphed = GraphedMonoRec(model, data)
            variants["graphed_ms"] = lambda: wall(lambda: graphed(data), args.steps)
            outs["graphed"] = graphed(data)["result"].clone()
            for name, kw in (("compile", {}), ("reduce_overhead", {"mode": "reduce-overhead"})):
                fn = torch.compile(model, fullgraph=True, **kw)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(dict(data))
                torch.cuda.synchronize()
                res[f"{name}_first_s"] = round(time.perf_counter() - t0, 2)
                for _ in range(args.warmup):
                    out = fn(dict(data))
                outs[name] = out["result"].clone()
                variants[f"{name}_ms"] = (lambda f: lambda: wall(lambda: f(dict(data)), args.steps))(fn)
        samples = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, v in variants.items():
                samples[k].append(v())
    for k, s in samples.items():
        res[k] = round(statistics.median(s), 3)
    res["bitwise_equal_to_eager"] = {k: bool(torch.equal(v, ref["result"])) for k, v in outs.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
