"""Key frames per second of the stereo and index-masked configurations over a sequence: the loader's per-key-frame dicts
against MonoRecSequence.

    python tools/time_sequence_keys.py [--frames=N] [--rounds=R] [--mode=f16|tf32|fp32]

A synthetic KITTI-shaped sequence (256x512, host tensors as a loader yields them), frame_count 2, random-init weights.
Two configurations:
  stereo        MonoRecModel(use_stereo=True), every key frame, each with its right-camera frame (return_stereo)
  index_masked  MonoRecModel(), the key frames of loader_keys with annotated lidar (offset 5 / extra 10) and an index
                mask that drops a third of them (use_index_mask)
and two variants of each, alternated round by round in one process:
  loop          evaluate.py's loader path: one dict per key frame with its own copies of the source (and stereo) frames,
                collated at the loader's batch size 2, copied to the device, an eager forward per batch
  sequence      MonoRecSequence at B 8 with CUDA-graph replay (keys= / stereo=True); frames no listed key frame needs
                are skipped unread
A round's number is key frames run over the host time from the first batch to a device synchronise after the last, for a
fresh sequence (its graph capture included); the report is the median over R rounds.  The card name and power limit are
printed with the numbers (one JSON line per configuration).
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import monorec_b200.model as M  # noqa: E402
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200.sequence import MonoRecSequence, loader_keys, neighbour_offsets  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402

DEV = "cuda:0"
H, W = 256, 512


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # (no nvidia-smi: report why)
        return f"unknown ({e})"


def run_loop(model, st, keys, stereo):
    """The loader's collated dicts at batch 2, an eager forward each; returns the number of key frames run."""
    images, poses, Ks = st["images"], st["poses"], st["Ks"]
    offs = neighbour_offsets(2)
    for b in range(0, len(keys), 2):
        ks = keys[b:b + 2]
        rows = lambda t, d: torch.stack([t[i + d] for i in ks])                  # noqa: E731
        data = {"keyframe": rows(images, 0), "keyframe_pose": rows(poses, 0), "keyframe_intrinsics": rows(Ks, 0),
                "frames": [rows(images, d) for d in offs], "poses": [rows(poses, d) for d in offs],
                "intrinsics": [rows(Ks, d) for d in offs]}
        if stereo:
            data.update(stereoframe=rows(st["right"], 0), stereoframe_pose=rows(st["right_poses"], 0),
                        stereoframe_intrinsics=rows(Ks, 0))
        data = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in data.items()}
        model(data)
    torch.cuda.synchronize()
    return len(keys)


def run_sequence(model, st, keys, stereo):
    seq = MonoRecSequence(model, frame_count=2, batch_size=8, graphed=True, keys=keys, stereo=stereo)
    n = 0
    for f in range(st["images"].shape[0]):
        if not seq.needs(f):
            seq.skip()
            continue
        kw = dict(stereo=(st["right"][f], st["right_poses"][f], st["Ks"][f])) if stereo else {}
        n += len(seq.push(st["images"][f], st["poses"][f], st["Ks"][f], **kw))
    n += len(seq.flush())
    torch.cuda.synchronize()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    args = ap.parse_args()
    C.set_mode(args.mode)
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "mode": args.mode, "size": [H, W],
            "frames": args.frames}
    images, poses, Ks = make_sequence(args.frames, H, W, seed=1)
    base = torch.eye(4)
    base[0, 3] = 0.54
    st = dict(images=images, poses=poses, Ks=Ks, right=make_sequence(args.frames, H, W, seed=2)[0],
              right_poses=poses @ base)
    g = np.random.default_rng(3)
    mask = {str(i): bool(g.random() < 2 / 3) for i in range(args.frames)}
    configs = {"stereo": (True, loader_keys(args.frames, 2, 1)),
               "index_masked": (False, loader_keys(args.frames, 2, 1, lidar_depth=True, index_masks=[mask]))}
    variants = {"loop_b2": run_loop, "sequence_b8": run_sequence}
    with torch.no_grad():
        for name, (stereo, keys) in configs.items():
            model = M.MonoRecModel(use_stereo=stereo)
            model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
            model = model.to(DEV).eval()
            for fn in variants.values():                 # warm-up: packing, cuDNN algorithms, graph capture
                fn(model, st, keys, stereo)
            rates = {k: [] for k in variants}
            for _ in range(args.rounds):
                for v, fn in variants.items():
                    t0 = time.perf_counter()
                    n = fn(model, st, keys, stereo)
                    rates[v].append(n / (time.perf_counter() - t0))
            med = {k: statistics.median(v) for k, v in rates.items()}
            print(json.dumps(dict(card, config=name, frame_count=2, key_frames=len(keys), keyframes_per_s=med,
                                  rounds=rates, speedup=med["sequence_b8"] / med["loop_b2"])), flush=True)


if __name__ == "__main__":
    main()
