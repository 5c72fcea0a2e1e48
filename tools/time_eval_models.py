"""Key frames per second of evaluate.py's list of models: MultiModelEvaluater against one SequenceEvaluater per model.

    python tools/time_eval_models.py [--frames=N] [--rounds=R] [--mode=f16|tf32|fp32]

The stream and settings of time_eval_sequence.py: a synthetic 256x512 sequence of N host frames with LiDAR-like targets,
frame_count 2, evaluater batch 2, the seven sparse metrics, max_distance 80, 8 key frames per forward.  The model lists:
  1  one checkpoint
  2  two checkpoints with the same trunk (other Mask / Depth weights): they share the cost volume and the trunk
  4  those two, a third such checkpoint and one use_ssim=2 model on the same trunk, which shares only the trunk
For each list two variants, alternated round by round in one process:
  separate  one SequenceEvaluater(MonoRecSequence(model, batch_size=8)) per model, each over the whole stream
  shared    one MultiModelEvaluater over the list (one pass over the stream)
A round's number is models x key frames over the host time from the first frame to the last log, fresh sequences (graph
capture included); the report is the median over R rounds, with the card name and power limit, and whether the logs of
the two variants are equal bit for bit.
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
from monorec_b200.evaluation import SequenceEvaluater  # noqa: E402
from monorec_b200.models_eval import MultiModelEvaluater  # noqa: E402
from monorec_b200.sequence import MonoRecSequence  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402
from tools.time_sequence import power_limit  # noqa: E402

DEV = "cuda:0"
H, W = 256, 512
NAMES = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
         "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]
BATCH, SEQ_BATCH, MAX_D = 2, 8, 80


def models():
    """Four models on one trunk: checkpoints of seeds 7, 8, 9 and a use_ssim=2 model."""
    out = []
    for seed, kw in ((7, {}), (8, {}), (9, dict(use_ssim=2)), (10, {})):
        m = MM.MonoRecModel(**kw)
        m.load_state_dict(seeded_state_dict(m, seed=seed, gain=0.7))
        if out:
            m._feature_extractor.load_state_dict(out[0]._feature_extractor.state_dict())
        out.append(m.to(DEV).eval())
    return [out[0], out[1], out[3], out[2]]          # the list of 4 ends with the use_ssim=2 model


def run_separate(ms, seqdata, targets):
    images, poses, Ks = seqdata
    n, logs = 0, []
    for m in ms:
        ev = SequenceEvaluater(MonoRecSequence(m, batch_size=SEQ_BATCH), NAMES, BATCH, max_distance=MAX_D)
        for f in range(images.shape[0]):
            n += len(ev.push(images[f], poses[f], Ks[f], targets[f]))
        n += len(ev.flush())
        logs.append(ev.log())
    return n, logs


def run_shared(ms, seqdata, targets):
    images, poses, Ks = seqdata
    ev = MultiModelEvaluater(ms, NAMES, BATCH, max_distance=MAX_D, seq_batch=SEQ_BATCH)
    n = 0
    for f in range(images.shape[0]):
        n += len(ev.push(images[f], poses[f], Ks[f], targets[f]))
    n += len(ev.flush())
    return n * len(ms), ev.logs()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    args = ap.parse_args()
    C.set_mode(args.mode)
    all_models = models()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "mode": args.mode, "size": [H, W],
            "frames": args.frames, "frame_count": 2, "eval_batch": BATCH, "seq_batch": SEQ_BATCH}
    seqdata = make_sequence(args.frames, H, W, seed=1)
    gen = torch.Generator().manual_seed(2)
    targets = torch.rand(args.frames, 1, H, W, generator=gen) * 0.3 + 0.0125
    targets[torch.rand(args.frames, 1, H, W, generator=gen) > 0.05] = 0.0
    variants = {"separate": run_separate, "shared": run_shared}
    report = {}
    with torch.no_grad():
        for count in (1, 2, 4):
            ms = all_models[:count]
            logs = {k: fn(ms, seqdata, targets)[1] for k, fn in variants.items()}     # warm-up: packing, capture
            rates = {k: [] for k in variants}
            for _ in range(args.rounds):
                for name, fn in variants.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    n, _ = fn(ms, seqdata, targets)
                    rates[name].append(n / (time.perf_counter() - t0))
            same = all(np.array_equal(np.asarray(a[k]), np.asarray(b[k]), equal_nan=True)
                       for a, b in zip(logs["separate"], logs["shared"]) for k in ("metrics", "metrics_correct"))
            med = {k: statistics.median(v) for k, v in rates.items()}
            report[count] = dict(model_keyframes_per_s=med, rounds=rates, speedup=med["shared"] / med["separate"],
                                 logs_bit_identical=same)
            print(json.dumps(dict(card, models=count, **report[count])), flush=True)


if __name__ == "__main__":
    main()
