"""Interleaved A/B timing of the cost-volume kernel across library builds, in one process.

    python tools/ab_cv.py B F D H W [--iters=N] [--rounds=R] tag=path/to/libmonorec_b200_x.so ...

Every round times each library in turn (N launches of mr_cost_volume_fwd, CUDA events around each launch, outputs
preallocated, the projection tables computed once), so that clock drift and neighbours on the GPU fall on all variants
alike.  Prints one JSON line per library: the mean launch time of every round, their median and spread.
"""
import ctypes
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from monorec_b200 import _lib  # noqa: E402
from monorec_b200.synthetic import make_inputs, to_device  # noqa: E402


def load(path):
    lib = ctypes.CDLL(str(path))
    for name in ("mr_last_error", "mr_projection_tables", "mr_cost_volume_fwd"):
        res, args = _lib.SIGNATURES[name]
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    return lib


def check(lib, rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed (code {rc}): {lib.mr_last_error().decode(errors='replace')}")


def main():
    pos = [a for a in sys.argv[1:] if not a.startswith("--") and "=" not in a]
    opts = dict(a[2:].split("=", 1) for a in sys.argv[1:] if a.startswith("--"))
    libs = [(a.split("=", 1)[0], load(a.split("=", 1)[1])) for a in sys.argv[1:] if "=" in a and not a.startswith("--")]
    B, F, D, H, W = [int(x) for x in pos[:5]]
    iters, rounds = int(opts.get("iters", 20)), int(opts.get("rounds", 3))
    dev = "cuda:0"
    d = to_device(make_inputs(B, F, H, W, seed=0), dev)
    proj = torch.empty(B, F, 3, 4, device=dev)
    depths = torch.empty(D, device=dev)
    cv = torch.empty(B, D, H, W, device=dev)
    sfcv = torch.empty(F, B, D, H, W, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    frames = _lib.ptr_array(d["frames"])
    lib0 = libs[0][1]
    check(lib0, lib0.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                          _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H, W,
                                          proj.data_ptr(), depths.data_ptr(), D, 0.0025, 0.33, stream), "tables")

    def launch(lib):
        check(lib, lib.mr_cost_volume_fwd(d["keyframe"].data_ptr(), frames, proj.data_ptr(), depths.data_ptr(), cv.data_ptr(),
                                          sfcv.data_ptr(), B, F, D, H, W, 10.0, None, stream), "mr_cost_volume_fwd")

    means = {tag: [] for tag, _ in libs}
    for _ in range(rounds):
        for tag, lib in libs:
            for _ in range(3):
                launch(lib)
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for e0, e1 in ev:
                e0.record()
                launch(lib)
                e1.record()
            torch.cuda.synchronize()
            means[tag].append(sum(e0.elapsed_time(e1) for e0, e1 in ev) / iters)
    for tag, _ in libs:
        m = means[tag]
        print(json.dumps({"shape": [B, F, D, H, W], "lib": tag, "ms_median": round(statistics.median(m), 4),
                          "ms_min": round(min(m), 4), "ms_max": round(max(m), 4), "rounds": [round(x, 4) for x in m]}))


if __name__ == "__main__":
    main()
