"""Per-key-frame latency of a live stream, from the push of the frame that completes a key frame to its emitted result on
the device, for the causal and the centred KITTI layouts.

    python tools/time_sequence_layouts.py [--frames=N] [--rounds=R] [--mode=f16|tf32|fp32]

A synthetic KITTI-shaped sequence (256x512, frames already on the device, as a camera pipeline would hand them over),
frame_count 2, random-init weights, MonoRecSequence with CUDA-graph replay.  Two layouts:
  centred  kitti_layout(n, 2, 1): sources k-1, k+1; key frame k is emitted at the push of frame k+1
  causal   kitti_layout(n, 2, 1, offset_d=-1): sources k-2, k; key frame k is emitted at the push of frame k itself
at sequence batch 1 (one key frame per push: the latency of a live stream) and 4 (a batch per four pushes; its first key
frame also waits for the next three frames).  A push's number is the host time from the call to a device synchronise after
it returns, for every push that emits a batch after the graph's capture; the report is the median and the 90th percentile
over R rounds of a fresh sequence, with the frames a key frame waits for after its own (`frames_after_key`: the layout's
largest offset, plus batch - 1 for the first key frame of a batch).  The card name and power limit are printed with the
numbers (one JSON line per layout and batch).
"""
import argparse
import json
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
from monorec_b200.sequence import MonoRecSequence, kitti_layout  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402

DEV = "cuda:0"
H, W = 256, 512


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # (no nvidia-smi: report why)
        return f"unknown ({e})"


def run(model, st, layout, batch):
    """One fresh sequence over the stream; returns the push-to-result latencies (s) of the pushes that emit, after the
    capture."""
    seq = MonoRecSequence(model, batch_size=batch, graphed=True, layout=layout)
    out = []
    for f in range(st["images"].shape[0]):
        captured = seq._graph is not None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        emitted = seq.push(st["images"][f], st["poses"][f], st["Ks"][f])
        torch.cuda.synchronize()
        if emitted and captured and len(emitted) == batch:
            out.append(time.perf_counter() - t0)
    seq.flush()
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    args = ap.parse_args()
    C.set_mode(args.mode)
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "mode": args.mode, "size": [H, W],
            "frames": args.frames}
    images, poses, Ks = make_sequence(args.frames, H, W, seed=1)
    st = dict(images=images.to(DEV), poses=poses.to(DEV), Ks=Ks.to(DEV))
    layouts = {"centred": kitti_layout(args.frames, 2, 1),
               "causal": kitti_layout(args.frames, 2, 1, offset_d=-1, drop_outside=True)}
    model = M.MonoRecModel()
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(DEV).eval()
    with torch.no_grad():
        for batch in (1, 4):
            for lay in layouts.values():                 # warm-up: packing, cuDNN algorithms, graph capture
                run(model, st, lay, batch)
            lat = {k: [] for k in layouts}
            for _ in range(args.rounds):                 # the layouts alternated round by round
                for name, lay in layouts.items():
                    lat[name] += run(model, st, lay, batch)
            for name, lay in layouts.items():
                v = np.array(lat[name]) * 1e3
                hi = max(0, max(lay.offsets))
                print(json.dumps(dict(card, layout=name, offsets=list(lay.offsets), batch=batch, pushes=int(v.size),
                                      push_to_result_ms={"median": float(np.median(v)),
                                                         "p90": float(np.percentile(v, 90))},
                                      per_key_ms=float(np.median(v)) / batch,
                                      frames_after_key={"last_of_batch": hi, "first_of_batch": hi + batch - 1})),
                      flush=True)


if __name__ == "__main__":
    main()
