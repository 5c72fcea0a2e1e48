#!/usr/bin/env python
"""CUDA-event timing of the residual image (csrc/residual_image.cu) at B 8, F 4, 256x512, next to the reference's torch
arithmetic on the same device (oracle.residual_image_torch: torch.inverse, two matmuls, grid_sample and the five pooled
maps of the SSIM per frame), and the cost of MonoRecSequence(residual_image=True) per key frame.

    python tools/time_residual_image.py [--out results/time_residual_image.json]

Prints the card and its power limit with the numbers, and one JSON line."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from monorec_b200 import _lib  # noqa: E402
from monorec_b200 import layers as LY  # noqa: E402
from monorec_b200 import losses as L  # noqa: E402
from monorec_b200.synthetic import make_inputs, make_sequence, seeded_state_dict, to_device  # noqa: E402
from oracle.residual_image_oracle import residual_image_torch  # noqa: E402
from tests.residual_cases import smooth_inverse_depth  # noqa: E402


def timeit(fn, n=50, warm=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:   # noqa: BLE001
        q = torch.cuda.get_device_name()
    return q


def sequence_ms_per_key(model, images, poses, intr, flag, reps=3):
    """Host wall time of pushing the stream (graphed batches of 8, the capture included) per key frame run, ending in a
    device synchronise; the best of `reps` fresh sequences."""
    from monorec_b200.sequence import MonoRecSequence
    best = None
    for _ in range(reps):
        seq = MonoRecSequence(model, frame_count=2, batch_size=8, graphed=True, residual_image=flag)
        torch.cuda.synchronize()
        t0, n = time.perf_counter(), 0
        for i in range(len(images)):
            n += len(seq.push(images[i], poses[i], intr[i]))
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) * 1e3 / n
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_residual_image: needs a GPU")
    B, Fn, H, W = 8, 4, 256, 512
    dev = "cuda:0"
    d = to_device(make_inputs(B, Fn, H, W, seed=0), dev)
    invd = smooth_inverse_depth(B, H, W, 1).to(dev)
    args_k = (d["keyframe"], d["frames"], d["keyframe_pose"], d["keyframe_intrinsics"], d["poses"], d["intrinsics"], invd, None)
    lib = _lib.load()
    proj = L.projection(d["keyframe"], d["keyframe_pose"], d["keyframe_intrinsics"], d["poses"], d["intrinsics"])
    out = torch.empty(B, 1, H, W, device=dev)
    fr = _lib.ptr_array(d["frames"])
    stream = torch.cuda.current_stream().cuda_stream

    def kernel():
        lib.mr_residual_image(d["keyframe"].data_ptr(), fr, proj.data_ptr(), invd.data_ptr(), None, B, Fn, 3, H, W,
                              out.data_ptr(), stream)

    gray = d["keyframe"][:, :1].contiguous()
    gframes = [f[:, :1].contiguous() for f in d["frames"]]
    gfr = _lib.ptr_array(gframes)

    def kernel_gray():
        lib.mr_residual_image(gray.data_ptr(), gfr, proj.data_ptr(), invd.data_ptr(), None, B, Fn, 1, H, W, out.data_ptr(),
                              stream)

    def module():
        LY.residual_image_impl(*args_k)

    def reference():
        residual_image_torch(d["keyframe"], d["keyframe_pose"], d["keyframe_intrinsics"], invd, d["frames"], d["poses"],
                             d["intrinsics"])

    # the kernel and the reference arithmetic agree on these inputs (the tests gate it; printed here as a sanity figure)
    ref = residual_image_torch(d["keyframe"], d["keyframe_pose"], d["keyframe_intrinsics"], invd, d["frames"], d["poses"],
                               d["intrinsics"])
    diff = (LY.residual_image_impl(*args_k) - ref).abs().nan_to_num().max().item()
    t_k, t_g, t_m, t_r = [], [], [], []
    for _ in range(3):                    # alternated, so that a shared machine's drift hits all alike
        t_k.append(timeit(kernel, 200))
        t_g.append(timeit(kernel_gray, 200))
        t_m.append(timeit(module, 100))
        t_r.append(timeit(reference, 20, 3))
    nbytes = 4 * B * H * W * (3 * (1 + Fn) + 1 + 1)     # one read of the keyframe, the frames, the inverse depth; one write

    from monorec_b200.model import MonoRecModel
    model = MonoRecModel()
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(dev).eval()
    images, sposes, sintr = make_sequence(8 * 6 + 2, H, W, seed=3)
    s_off, s_on = [], []
    with torch.no_grad():
        from monorec_b200.sequence import MonoRecSequence
        for flag in (False, True):               # warm-up: packing, cuDNN algorithms (eager)
            seq = MonoRecSequence(model, frame_count=2, batch_size=8, graphed=False, residual_image=flag)
            for i in range(10):
                seq.push(images[i], sposes[i], sintr[i])
        for _ in range(2):
            s_off.append(sequence_ms_per_key(model, images, sposes, sintr, False))
            s_on.append(sequence_ms_per_key(model, images, sposes, sintr, True))

    res = {"card": card(), "B": B, "F": Fn, "H": H, "W": W,
           "kernel_ms": min(t_k), "kernel_gray_ms": min(t_g), "entry_ms": min(t_m), "reference_torch_ms": min(t_r),
           "kernel_ms_runs": t_k, "reference_torch_ms_runs": t_r, "kernel_dram_bytes": nbytes,
           "kernel_GBps": nbytes / min(t_k) / 1e6, "max_abs_diff_vs_reference": diff,
           "sequence_ms_per_key_off": min(s_off), "sequence_ms_per_key_on": min(s_on),
           "sequence_overhead_ms_per_key": min(s_on) - min(s_off)}
    print(f"{res['card']}")
    print(f"residual image B={B} F={Fn} {H}x{W}: kernel {res['kernel_ms']:.3f} ms (gray {res['kernel_gray_ms']:.3f} ms, "
          f"with projection tables {res['entry_ms']:.3f} ms), reference torch arithmetic {res['reference_torch_ms']:.3f} ms; "
          f"{nbytes / 1e6:.1f} MB -> {res['kernel_GBps']:.0f} GB/s; max |d| vs reference {diff:.2e}")
    print(f"MonoRecSequence graphed B=8: {res['sequence_ms_per_key_off']:.3f} ms per key frame, "
          f"{res['sequence_ms_per_key_on']:.3f} ms with residual_image=True")
    print(json.dumps(res))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
