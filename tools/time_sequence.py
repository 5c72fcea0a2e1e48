"""Key frames per second of the point-cloud export over a sequence: the create_pointcloud.py loop against MonoRecSequence.

    python tools/time_sequence.py [--frames=N] [--rounds=R] [--mode=f16|tf32|fp32]

A synthetic KITTI-shaped sequence (256x512, z-forward poses, host tensors as a loader yields them), F = 2 and F = 4 at
dilation 1, random-init weights.  Two variants, alternated round by round in one process:
  loop      create_pointcloud.py:65-105 on the device path: one dict per key frame with its own copies of the F source
            frames, copied to the device, an eager forward at B 1, MaskVoter + PLYSaver.add_depthmap
  sequence  MonoRecSequence at B 8 with CUDA-graph replay + sequence_pointcloud
Both use the config's roi, max_d 20 and dropout 0.75, and the model's inverse-depth range keeps every depth inside
[3, 20] m; the random-init MaskModule's cv_mask can still veto every pixel, so the vertex counts are printed too.  A round's number is key frames run over the host time from
the first push to a device synchronise after the last, for a fresh sequence (its graph capture included); the report is the
median over R rounds.  The card name and power limit are printed with the numbers (one JSON line per frame count).
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import monorec_b200.model as M  # noqa: E402
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200 import pointcloud as PC  # noqa: E402
from monorec_b200.sequence import MonoRecSequence, neighbour_offsets  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402

DEV = "cuda:0"
H, W = 256, 512
ROI, MAX_D, DROPOUT = [40, 256, 48, 464], 20, 0.75


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # (no nvidia-smi: report why)
        return f"unknown ({e})"


def run_loop(model, seqdata, frame_count):
    """create_pointcloud.py's loop, B 1; returns the number of key frames run."""
    images, poses, Ks = seqdata
    offs = neighbour_offsets(frame_count)
    saver = PC.PLYSaver(H, W, max_d=MAX_D, roi=ROI, dropout=DROPOUT)
    voter = PC.MaskVoter()
    keys = range(-min(offs), images.shape[0] - max(offs))
    for i in keys:
        data = {"keyframe": images[i:i + 1], "keyframe_pose": poses[i:i + 1], "keyframe_intrinsics": Ks[i:i + 1],
                "frames": [images[i + d:i + d + 1] for d in offs], "poses": [poses[i + d:i + d + 1] for d in offs],
                "intrinsics": [Ks[i + d:i + d + 1] for d in offs]}
        data = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in data.items()}
        key = voter.push(model(data), data)
        if key is not None:
            saver.add_depthmap(key["depth"], key["keyframe"], key["intrinsics"], key["pose"], keep_masks=key["keep_masks"],
                               min_hits=key["min_hits"])
    torch.cuda.synchronize()
    return len(keys), len(saver)


def run_sequence(model, seqdata, frame_count):
    images, poses, Ks = seqdata
    seq = MonoRecSequence(model, frame_count=frame_count, batch_size=8, graphed=True)
    saver = PC.PLYSaver(H, W, max_d=MAX_D, roi=ROI, dropout=DROPOUT)
    pc = PC.sequence_pointcloud(seq, saver)
    n = 0
    for f in range(images.shape[0]):
        n += len(pc.push(images[f], poses[f], Ks[f]))
    n += len(pc.flush())
    torch.cuda.synchronize()
    return n, len(saver)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    args = ap.parse_args()
    C.set_mode(args.mode)
    model = M.MonoRecModel(inv_depth_min_max=(0.33, 0.06))     # every depth inside [3, 20] m
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(DEV).eval()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "mode": args.mode, "size": [H, W],
            "frames": args.frames}
    seqdata = make_sequence(args.frames, H, W, seed=1)
    variants = {"loop_b1": run_loop, "sequence_b8": run_sequence}
    with torch.no_grad():
        for frame_count in (2, 4):
            for fn in variants.values():                 # warm-up: packing, cuDNN algorithms, graph capture
                fn(model, seqdata, frame_count)
            rates = {k: [] for k in variants}
            counts = {}
            for _ in range(args.rounds):
                for name, fn in variants.items():
                    t0 = time.perf_counter()
                    n, verts = fn(model, seqdata, frame_count)
                    rates[name].append(n / (time.perf_counter() - t0))
                    counts[name] = verts
            med = {k: statistics.median(v) for k, v in rates.items()}
            print(json.dumps(dict(card, frame_count=frame_count, dilation=1, keyframes_per_s=med, rounds=rates,
                                  vertices=counts, speedup=med["sequence_b8"] / med["loop_b1"])), flush=True)


if __name__ == "__main__":
    main()
