#!/usr/bin/env python
"""Keyframes/s of the eager MonoRecModel.forward under torch.nn.DataParallel -- the way the reference's evaluate.py
(base/base_trainer.py:26-29) and create_pointcloud.py (:38-39) run it -- next to the plain single-GPU forward.  B 8 keyframes
per GPU, 256x512, 2 source frames, D 32, the batch resident on cuda:0 as the evaluater leaves it.

  single      model(batch) on cuda:0, B 8
  dp<N>       torch.nn.DataParallel(model, device_ids=[0 .. N-1])(batch), B 8 N, for N = 1, 2, 4, 8 up to the visible GPUs
              (with one device id DataParallel calls the module directly)
  dp<N>_first the first DataParallel forward of a freshly constructed model, whose replicas build the kernel-layout copies
              of the weights on every device, against the steady-state forward

Host clock around forwards that end in a synchronise of every device used; shapes, cuDNN and the library are warmed up on
another model first, so the first-forward number is packing + replication.  Prints one JSON line with the card's name and
power limit.

    python tools/time_data_parallel.py [--mode f16|tf32] [--steps 10] [--warmup 3]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200.model import MonoRecModel  # noqa: E402
from monorec_b200.synthetic import make_inputs, to_device  # noqa: E402

B_PER_GPU, F, H, W = 8, 2, 256, 512


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def sync(n):
    for i in range(n):
        torch.cuda.synchronize(i)


def timed(fn, n_dev, steps):
    sync(n_dev)
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    sync(n_dev)
    return (time.perf_counter() - t0) / steps


def fresh_model():
    torch.manual_seed(0)
    return MonoRecModel().to("cuda:0").eval()      # random-init weights of the reference architecture


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16", choices=("f16", "tf32"))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_data_parallel.py needs a GPU")
    C.set_mode(args.mode)
    n_vis = torch.cuda.device_count()
    counts = [n for n in (1, 2, 4, 8) if n <= n_vis]
    batches = {n: to_device(make_inputs(B_PER_GPU * n, F, H, W, seed=n), "cuda:0") for n in counts}
    res = {"card": card(), "gpus_visible": n_vis, "mode": args.mode, "per_gpu_batch": B_PER_GPU, "shape": [F, H, W],
           "steps": args.steps}
    with torch.no_grad():
        model = fresh_model()
        for _ in range(args.warmup):
            model(dict(batches[1]))
        t = timed(lambda: model(dict(batches[1])), 1, args.steps)
        res["single_ms"], res["single_kf_s"] = round(t * 1e3, 2), round(B_PER_GPU / t, 1)
        for n in counts:
            dp = torch.nn.DataParallel(model, device_ids=list(range(n)))
            for _ in range(args.warmup):
                dp(dict(batches[n]))
            t = timed(lambda: dp(dict(batches[n])), n, args.steps)
            res[f"dp{n}_ms"], res[f"dp{n}_kf_s"] = round(t * 1e3, 2), round(B_PER_GPU * n / t, 1)
            # a new model: the first forward packs its weights on every device (the library, cuDNN and the shapes are warm)
            dp_new = torch.nn.DataParallel(fresh_model(), device_ids=list(range(n)))
            first = timed(lambda: dp_new(dict(batches[n])), n, 1)
            steady = timed(lambda: dp_new(dict(batches[n])), n, args.steps)
            res[f"dp{n}_first_ms"], res[f"dp{n}_steady_ms"] = round(first * 1e3, 2), round(steady * 1e3, 2)
            del dp_new
    print(json.dumps(res))


if __name__ == "__main__":
    main()
