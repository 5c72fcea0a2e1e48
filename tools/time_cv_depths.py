"""Kernel time of the cost volume on plane depths vs per-pixel depths (cv_depths), interleaved, in one process.

    python tools/time_cv_depths.py [--iters=N] [--rounds=R]

For config 2 (B 8, F 4, D 32, 256x512) and hires (B 4, F 6, D 64, 512x1024) it times four cases in turn, every round:
  plane      mr_cost_volume_fwd on the default inverse-depth planes
  broadcast  mr_cost_volume_fwd_depthmap on those planes repeated at every pixel (same results, bit for bit)
  band       a +-10 % band (geometric, 0.9x - 1.1x) around a smooth seeded 4-60 m surface
  step       a +-10 % band around 2 m left of a vertical edge and 300 m right of it
CUDA events bracket each launch; a round's number is the mean over N launches, the report the median over the rounds.
The card name and its power limit are printed with the numbers.
"""
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from monorec_b200 import _lib  # noqa: E402
from monorec_b200.synthetic import make_inputs, to_device  # noqa: E402
from tests.cv_cases import band_depths  # noqa: E402


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # (no nvidia-smi: report why)
        return f"unknown ({e})"


def main():
    opts = dict(a[2:].split("=", 1) for a in sys.argv[1:] if a.startswith("--"))
    iters, rounds = int(opts.get("iters", 20)), int(opts.get("rounds", 5))
    lib = _lib.load()
    dev = "cuda:0"
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}))
    for name, (B, F, D, H, W) in (("config2", (8, 4, 32, 256, 512)), ("hires", (4, 6, 64, 512, 1024))):
        d = to_device(make_inputs(B, F, H, W, seed=0), dev)
        proj = torch.empty(B, F, 3, 4, device=dev)
        planes = torch.empty(D, device=dev)
        cv = torch.empty(B, D, H, W, device=dev)
        sfcv = torch.empty(F, B, D, H, W, device=dev)
        stream = torch.cuda.current_stream().cuda_stream
        frames = _lib.ptr_array(d["frames"])
        _lib.check(lib.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                            _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H, W,
                                            proj.data_ptr(), planes.data_ptr(), D, 0.0025, 0.33, stream), "tables")
        step = torch.full((B, 1, H, W), 300.0)
        step[..., : int(0.43 * W)] = 2.0
        f = torch.exp(torch.linspace(-0.0953102, 0.0953102, D, dtype=torch.float64)).float().view(1, D, 1, 1)
        maps = {"broadcast": planes.view(1, D, 1, 1).expand(B, D, H, W).contiguous(),
                "band": band_depths(B, D, H, W, seed=1, rel=1.1).to(dev),
                "step": (step * f).contiguous().to(dev)}

        def launch(case):
            if case == "plane":
                rc = lib.mr_cost_volume_fwd(d["keyframe"].data_ptr(), frames, proj.data_ptr(), planes.data_ptr(), cv.data_ptr(),
                                            sfcv.data_ptr(), B, F, D, H, W, 10.0, None, stream)
            else:
                rc = lib.mr_cost_volume_fwd_depthmap(d["keyframe"].data_ptr(), frames, proj.data_ptr(), maps[case].data_ptr(),
                                                     cv.data_ptr(), sfcv.data_ptr(), None, 0, B, F, D, H, W, 10.0, None, stream)
            _lib.check(rc, case)

        cases = ["plane", "broadcast", "band", "step"]
        means = {c: [] for c in cases}
        for _ in range(rounds):
            for c in cases:
                for _ in range(3):
                    launch(c)
                ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
                for e0, e1 in ev:
                    e0.record()
                    launch(c)
                    e1.record()
                torch.cuda.synchronize()
                means[c].append(sum(e0.elapsed_time(e1) for e0, e1 in ev) / iters)
        base = statistics.median(means["plane"])
        for c in cases:
            m = means[c]
            print(json.dumps({"config": name, "shape": [B, F, D, H, W], "case": c, "ms_median": round(statistics.median(m), 4),
                              "ms_min": round(min(m), 4), "ms_max": round(max(m), 4),
                              "vs_plane": round(statistics.median(m) / base, 3)}))


if __name__ == "__main__":
    main()
