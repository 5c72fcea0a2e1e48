#!/usr/bin/env python
"""Timing of the dense / completeness metrics and the evaluater's median scaling on the device (monorec_b200.metrics), next to
the same functions written like the reference with stock PyTorch CUDA ops (model/metric_functions/, utils/util.py:135-142),
on the same GPU: B 8, 256x512, a LiDAR-like target (~5 % of the pixels), max_distance 80 as in the KITTI evaluation config.

Three numbers per side, host clock around work that ends in a device synchronise (the evaluater converts every metric to a
Python float, evaluater/evaluater.py:41-43):
  metrics        the twelve reference-named functions of one call set, each converted to float
  median         one median_scaling call
  evaluater      evaluater._eval_metrics with median_scaling on: scaling, then metric and float, for each of the twelve
Prints one JSON line with the card's name and power limit.

    python tools/time_metrics.py [--reps 30]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from monorec_b200 import metrics as M  # noqa: E402

DENSE = ("a1", "a2", "a3", "rmse", "rmse_log", "abs_rel", "sq_rel")
TENSOR = ("sc_inv", "l1_rel", "l1_inv", "completeness", "covered_gt")


# ---- the reference's functions restated with the same torch calls ----------------------------------------------------------
def _prep(p, g, roi, md, clamp=True):
    if roi is not None:
        p, g = p[:, :, roi[0]:roi[1], roi[2]:roi[3]], g[:, :, roi[0]:roi[1], roi[2]:roi[3]]
    p, g = torch.nn.functional.relu(p), torch.nn.functional.relu(g)
    if not clamp:
        return p, g
    if md is not None:
        p, g = torch.clamp_min(p, 1 / md), torch.clamp_min(g, 1 / md)
    return 1 / p, 1 / g


def _thresh(p, g):
    return torch.max(g / p, p / g)


def _mask_mean(t, m):
    t = t.clone()
    t[m] = 0
    return torch.sum(t) / (t.numel() - torch.sum(m.to(torch.float)))


def _sc_inv(p, g):
    n = g.shape[2] * g.shape[3]
    E = torch.log(p) - torch.log(g)
    E[torch.isnan(E)] = 0
    bm = torch.sqrt(1 / n * torch.sum(E ** 2, dim=[2, 3]) - 1 / (n ** 2) * (torch.sum(E, dim=[2, 3]) ** 2))
    bm[torch.isnan(bm)] = 0
    return torch.mean(bm)


TORCH = {
    "a1": lambda p, g: torch.mean((_thresh(p, g) < 1.25).float()),
    "a2": lambda p, g: torch.mean((_thresh(p, g) < 1.25 ** 2).float()),
    "a3": lambda p, g: torch.mean((_thresh(p, g) < 1.25 ** 3).float()),
    "rmse": lambda p, g: torch.mean(torch.sqrt(torch.mean((p - g) ** 2, dim=[1, 2, 3]))),
    "rmse_log": lambda p, g: torch.mean(torch.sqrt(torch.mean((torch.log(p) - torch.log(g)) ** 2, dim=[1, 2, 3]))),
    "abs_rel": lambda p, g: torch.mean(torch.abs(p - g) / g),
    "sq_rel": lambda p, g: torch.mean(((p - g) ** 2) / g),
    "sc_inv": _sc_inv,
    "l1_rel": lambda p, g: torch.mean(torch.abs(p - g) / g),
}


def torch_metric(name, pred, gt, roi, md):
    if name == "completeness":
        return torch.mean((pred != 0).float())
    if name == "covered_gt":
        return _mask_mean((pred != 0).float(), gt != 0)
    if name == "l1_inv":
        p, g = _prep(pred, gt, roi, md, clamp=False)
        return torch.mean(torch.abs(p - g))
    return TORCH[name](*_prep(pred, gt, roi, md))


def torch_median_scaling(d):
    target, prediction = d["target"], d["result"]
    mask = target > 0
    ratios = mask.new_tensor([torch.median(target[i, mask[i]]) / torch.median(prediction[i, mask[i]])
                              for i in range(target.shape[0])], dtype=torch.float32)
    d = dict(d)
    d["result"] = prediction * ratios.view(-1, 1, 1, 1)
    return d


# ---- the call sets ------------------------------------------------------------------------------------------------------
def device_metric(name, d, roi, md):
    f = getattr(M, f"{name}_metric")
    return f(d["result"], d["target"], roi, md) if name in TENSOR else f(d, roi, md)


def call_set(metric, d, roi, md):
    return [float(metric(n, d, roi, md)) for n in DENSE + TENSOR]


def evaluater(metric, scale, d, roi, md):
    acc = []
    for n in DENSE + TENSOR:
        d = scale(d)
        acc.append(float(metric(n, d, roi, md)))
    return acc


def wall_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_metrics.py needs a GPU")
    B, H, W, roi, md = 8, 256, 512, None, 80.0
    gen = torch.Generator().manual_seed(0)
    pred = torch.rand(B, 1, H, W, generator=gen) * 0.3 + 0.002
    gt = (pred * (1 + 0.2 * torch.randn(B, 1, H, W, generator=gen))).clamp_min(1e-3)
    gt[torch.rand(B, 1, H, W, generator=gen) > 0.05] = 0.0
    d = {"result": pred.cuda(), "target": gt.cuda()}

    def fresh():           # a new data_dict with a new result tensor, so no cached pass is reused across repetitions
        return {"result": d["result"].clone(), "target": d["target"]}

    ours = lambda n, dd, r, m: device_metric(n, dd, r, m)           # noqa: E731
    ref = lambda n, dd, r, m: torch_metric(n, dd["result"], dd["target"], r, m)  # noqa: E731
    # same values first (tolerance of the fp32 reference sums)
    a, b = call_set(ours, fresh(), roi, md), call_set(ref, fresh(), roi, md)
    worst = max(abs(x - y) / max(abs(y), 1e-12) for x, y in zip(a, b))
    ms_same = torch.equal(M.median_scaling(d)["result"], torch_median_scaling(d)["result"])
    res = {"card": card(), "shape": [B, 1, H, W], "target_density": float((gt > 0).float().mean()), "max_distance": md,
           "max_rel_diff_metrics": worst, "median_scaling_bitwise_equal": ms_same}
    for tag, fn_dev, fn_ref in (
            ("metrics", lambda: call_set(ours, fresh(), roi, md), lambda: call_set(ref, fresh(), roi, md)),
            ("median", lambda: M.median_scaling(d)["result"], lambda: torch_median_scaling(d)["result"]),
            ("evaluater", lambda: evaluater(ours, M.median_scaling, fresh(), roi, md),
             lambda: evaluater(ref, torch_median_scaling, fresh(), roi, md))):
        t_dev, t_ref = wall_ms(fn_dev, args.reps), wall_ms(fn_ref, args.reps)
        res[f"{tag}_device_ms"], res[f"{tag}_torch_ms"] = round(t_dev, 4), round(t_ref, 4)
        res[f"{tag}_speedup"] = round(t_ref / t_dev, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
