"""Key frames per second of evaluate.py's list of models over several lanes: one MultiDeviceModelsEvaluater against one
MultiDeviceEvaluater per model, on the same lanes and the same stream.

    python tools/time_eval_models_devices.py [--frames=N] [--rounds=R] [--mode=f16|tf32|fp32] [--models=4] [--shared=2]

The stream and models of time_eval_models.py: a synthetic 256x512 (KITTI) sequence of N host frames with LiDAR-like
targets, frame_count 2, evaluater batch 2, the seven sparse metrics, max_distance 80, 8 key frames per forward; the list
is two checkpoints on one trunk, a third such checkpoint and a use_ssim=2 model on that trunk (--models takes the first M).
Lane layouts: --shared lanes taking turns on cuda:0 and, with several GPUs visible, one lane per GPU.  For each layout two
variants, alternated round by round in one process:
  separate  one MultiDeviceEvaluater per model over the lanes (each reads and copies every frame, and runs every stage)
  shared    one MultiDeviceModelsEvaluater over the list (one pass; shared cost-volume and trunk stages on every lane)
A round's number is models x key frames over the host time from the first push to the last log, fresh runs (graph
captures included); the report is the median over R rounds after one warm-up round, with the card name and power limit,
and whether the logs of the two variants are equal bit for bit.
"""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200.lanes import MultiDeviceEvaluater, MultiDeviceModelsEvaluater  # noqa: E402
from monorec_b200.synthetic import make_sequence  # noqa: E402
from tools.time_eval_models import BATCH, H, MAX_D, NAMES, SEQ_BATCH, W, models  # noqa: E402
from tools.time_sequence import power_limit  # noqa: E402


def _feed(run, data):
    images, poses, Ks, targets = data
    for s, n in run.order:
        run.push(s, n, images[n], poses[n], Ks[n], targets[n])
    run.flush()


def run_separate(ms, devices, data):
    logs = []
    for m in ms:
        run = MultiDeviceEvaluater(m, devices, [data[0].shape[0]], NAMES, BATCH, seq_batch=SEQ_BATCH, max_distance=MAX_D)
        _feed(run, data)
        logs.append(run.log())
    return logs


def run_shared(ms, devices, data):
    run = MultiDeviceModelsEvaluater(ms, devices, [data[0].shape[0]], NAMES, BATCH, seq_batch=SEQ_BATCH,
                                     max_distance=MAX_D)
    _feed(run, data)
    return run.logs()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    ap.add_argument("--models", type=int, default=4)
    ap.add_argument("--shared", default="2", help="lane counts to run on cuda:0 alone")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_eval_models_devices.py needs a GPU")
    C.set_mode(args.mode)
    gpus = torch.cuda.device_count()
    ms = models()[:args.models]
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "gpus": gpus, "mode": args.mode,
            "size": [H, W], "frames": args.frames, "frame_count": 2, "eval_batch": BATCH, "seq_batch": SEQ_BATCH,
            "models": len(ms)}
    gen = torch.Generator().manual_seed(2)
    targets = torch.rand(args.frames, 1, H, W, generator=gen) * 0.3 + 0.0125
    targets[torch.rand(args.frames, 1, H, W, generator=gen) > 0.05] = 0.0
    data = make_sequence(args.frames, H, W, seed=1) + (targets,)
    keyframes = args.frames - 2
    layouts = [("shared", [0] * int(n)) for n in args.shared.split(",") if n]
    layouts += [("gpus", list(range(gpus)))] if gpus >= 2 else []
    variants = {"separate": run_separate, "shared": run_shared}
    with torch.no_grad():
        for kind, devices in layouts:
            rates, logs = {k: [] for k in variants}, {}
            for r in range(args.rounds + 1):               # round 0: warm-up (packing on every device, algorithms)
                for name, fn in variants.items():
                    for d in set(devices):
                        torch.cuda.synchronize(d)
                    t0 = time.perf_counter()
                    logs[name] = fn(ms, devices, data)     # (the logs read the totals back: the run has ended)
                    if r:
                        rates[name].append(len(ms) * keyframes / (time.perf_counter() - t0))
            same = all(np.array_equal(np.asarray(a[k]).view(np.uint64), np.asarray(b[k]).view(np.uint64))
                       for a, b in zip(logs["separate"], logs["shared"]) for k in ("metrics", "metrics_correct"))
            med = {k: statistics.median(v) for k, v in rates.items()}
            print(json.dumps(dict(card, layout=kind, devices=devices, keyframes=keyframes, model_keyframes_per_s=med,
                                  rounds=rates, speedup=med["shared"] / med["separate"], logs_bit_identical=same)),
                  flush=True)


if __name__ == "__main__":
    main()
