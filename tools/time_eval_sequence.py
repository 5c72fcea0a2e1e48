"""Key frames per second of evaluate.py's evaluation: the Evaluater.eval loop against SequenceEvaluater.

    python tools/time_eval_sequence.py [--frames=N] [--rounds=R] [--mode=f16|tf32|fp32]

configs/evaluate/eval_monorec.json's settings: frame_count 2, evaluater batch 2, the seven sparse metrics, max_distance 80,
no median scaling.  A synthetic KITTI-shaped sequence (256x512, host tensors as a loader yields them, a LiDAR-like target
covering ~5 % of the pixels), random-init weights.  Two variants, alternated round by round in one process:
  loop_b2       evaluater.py:78-119 on the device path: one dict per key frame with its own copies of the source frames,
                collated in pairs and copied to the device, an eager forward at B 2, every metric (this package's
                functions) turned into a Python float, the totals kept in numpy
  sequence_b8   SequenceEvaluater over a MonoRecSequence at B 8 with CUDA-graph replay (the same evaluater batches of 2),
                frames and targets pushed from the host, one log() at the end
A round's number is the key frames evaluated over the host time from the first frame to the log dict, for a fresh sequence
(its graph capture included); the report is the median over R rounds.  The card name and power limit are printed with the
numbers, and the largest relative difference between the two logs.
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
import monorec_b200.model as MM  # noqa: E402
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200 import metrics as M  # noqa: E402
from monorec_b200.evaluation import SequenceEvaluater  # noqa: E402
from monorec_b200.sequence import MonoRecSequence, neighbour_offsets  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402
from tools.time_sequence import power_limit  # noqa: E402

DEV = "cuda:0"
H, W = 256, 512
NAMES = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
         "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]
BATCH, MAX_D = 2, 80


def run_loop(model, seqdata, targets):
    """Evaluater.eval at batch 2; returns (key frames, log)."""
    images, poses, Ks = seqdata
    offs = neighbour_offsets(2)
    keys = list(range(-min(offs), images.shape[0] - max(offs)))
    metrics = [getattr(M, n) for n in NAMES]
    total, valid, avg, n_samples = np.zeros(len(NAMES)), np.zeros(len(NAMES)), np.zeros(len(NAMES)), 0
    for b in range(0, len(keys), BATCH):
        rows = keys[b:b + BATCH]
        cat = lambda t, d: torch.cat([t[i + d:i + d + 1] for i in rows])      # noqa: E731  (the loader's collation)
        data = {"keyframe": cat(images, 0), "keyframe_pose": cat(poses, 0), "keyframe_intrinsics": cat(Ks, 0),
                "frames": [cat(images, d) for d in offs], "poses": [cat(poses, d) for d in offs],
                "intrinsics": [cat(Ks, d) for d in offs], "target": cat(targets, 0)}
        data = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in data.items()}
        data = model(data)
        acc = np.zeros(len(NAMES))
        for i, metric in enumerate(metrics):
            acc[i] += float(metric(data, None, MAX_D))
        ok = np.zeros(len(NAMES)) if np.any(np.isnan(acc)) else np.ones(len(NAMES))
        acc = acc * ok
        total, valid = total + acc, valid + ok
        bs = len(rows)
        avg = avg + acc if n_samples == 0 else avg * (n_samples / (n_samples + bs)) + acc * (bs / (n_samples + bs))
        n_samples += bs
    return len(keys), {"metrics": (total / valid).tolist(), "metrics_correct": avg.tolist()}


def run_sequence(model, seqdata, targets):
    images, poses, Ks = seqdata
    ev = SequenceEvaluater(MonoRecSequence(model, batch_size=8, graphed=True), NAMES, BATCH, max_distance=MAX_D)
    n = 0
    for f in range(images.shape[0]):
        n += len(ev.push(images[f], poses[f], Ks[f], targets[f]))
    n += len(ev.flush())
    return n, ev.log()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    args = ap.parse_args()
    C.set_mode(args.mode)
    model = MM.MonoRecModel()
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(DEV).eval()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "mode": args.mode, "size": [H, W],
            "frames": args.frames, "frame_count": 2, "eval_batch": BATCH, "metrics": len(NAMES)}
    seqdata = make_sequence(args.frames, H, W, seed=1)
    gen = torch.Generator().manual_seed(2)
    targets = torch.rand(args.frames, 1, H, W, generator=gen) * 0.3 + 0.0125
    targets[torch.rand(args.frames, 1, H, W, generator=gen) > 0.05] = 0.0
    variants = {"loop_b2": run_loop, "sequence_b8": run_sequence}
    with torch.no_grad():
        logs = {k: fn(model, seqdata, targets)[1] for k, fn in variants.items()}   # warm-up: packing, graph capture
        rates = {k: [] for k in variants}
        for _ in range(args.rounds):
            for name, fn in variants.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                n, _ = fn(model, seqdata, targets)
                rates[name].append(n / (time.perf_counter() - t0))
    a, b = (np.array(logs[k]["metrics"] + logs[k]["metrics_correct"]) for k in variants)
    med = {k: statistics.median(v) for k, v in rates.items()}
    print(json.dumps(dict(card, keyframes_per_s=med, rounds=rates, speedup=med["sequence_b8"] / med["loop_b2"],
                          max_rel_diff_of_logs=float(np.max(np.abs(a - b) / np.abs(b))))), flush=True)


if __name__ == "__main__":
    main()
