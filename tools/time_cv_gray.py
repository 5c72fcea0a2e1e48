"""Grayscale against replicated three-channel frames (mr_cost_volume_fwd_channels, MonoRecSequence(use_color=False)),
interleaved, in one process.

    python tools/time_cv_gray.py [--iters=N] [--rounds=R]

Two measurements, each alternating the one-channel frames ("gray") and the same frames replicated to three channels ("rgb")
every round; a round's number is the mean over N calls, the report the median over R rounds, and the outputs of both are
checked equal (torch.equal) before timing:
  kernel   one launch of the cost-volume kernel (CUDA events), plane depths, SSIM, centred, fp32 volumes, at config 2
           (B 8, F 4, D 32, 256x512), hires (B 4, F 6, D 64, 512x1024) and TUM Mono-VO's shape (B 8, F 4, D 32, 480x640)
  model    MonoRecModel.forward in f16 engine mode, replayed from a CUDA graph (random-init weights), B 8, F 4, D 32,
           256x512
The card name and its power limit are printed with the numbers (one JSON line per measurement).
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

DEV = "cuda:0"


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # (no nvidia-smi: report why)
        return f"unknown ({e})"


def event_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def report(what, shape, times):
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({"what": what, "shape": shape, "median_ms": med, "rounds": times,
                      "gray_over_rgb": med["gray"] / med["rgb"]}), flush=True)


def gray_and_rgb(d):
    """(gray dict, replicated dict): the first plane of every image, and that plane three times."""
    g, r = dict(d), dict(d)
    g["keyframe"] = d["keyframe"][:, :1].contiguous()
    g["frames"] = [f[:, :1].contiguous() for f in d["frames"]]
    r["keyframe"] = g["keyframe"].expand(-1, 3, -1, -1).contiguous()
    r["frames"] = [f.expand(-1, 3, -1, -1).contiguous() for f in g["frames"]]
    return g, r


def kernel(lib, iters, rounds):
    for name, (B, F, D, H, W) in (("config2", (8, 4, 32, 256, 512)), ("hires", (4, 6, 64, 512, 1024)),
                                  ("tum", (8, 4, 32, 480, 640))):
        sets = dict(zip(("gray", "rgb"), gray_and_rgb(to_device(make_inputs(B, F, H, W, seed=0), DEV))))
        d = sets["gray"]
        proj = torch.empty(B, F, 3, 4, device=DEV)
        planes = torch.empty(D, device=DEV)
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                            _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H, W,
                                            proj.data_ptr(), planes.data_ptr(), D, 0.0025, 0.33, stream), "tables")
        cw = (_lib.c_float * 3)(5 / 32, 16 / 32, 11 / 32)
        outs = {k: (torch.empty(B, D, H, W, device=DEV), torch.empty(F, B, D, H, W, device=DEV)) for k in sets}
        frames = {k: _lib.ptr_array(s["frames"]) for k, s in sets.items()}

        def launch(k):
            cv, sf = outs[k]
            _lib.check(lib.mr_cost_volume_fwd_channels(sets[k]["keyframe"].data_ptr(), frames[k], proj.data_ptr(),
                                                       planes.data_ptr(), None, cv.data_ptr(), sf.data_ptr(), None, 0, B, F,
                                                       D, H, W, 10.0, cw, 1, 1, 0, 1 if k == "gray" else 3, stream),
                       "mr_cost_volume_fwd_channels")
        for k in outs:
            for _ in range(3):
                launch(k)
        torch.cuda.synchronize()
        assert torch.equal(outs["gray"][0], outs["rgb"][0]) and torch.equal(outs["gray"][1], outs["rgb"][1]), name
        times = {k: [] for k in outs}
        for _ in range(rounds):
            for k in outs:
                times[k].append(event_ms(lambda: launch(k), iters))
        report(f"kernel {name}", [B, F, D, H, W], times)
        del outs, sets, d
        torch.cuda.empty_cache()


def model(iters, rounds):
    from monorec_b200 import conv as C
    from monorec_b200.model import GraphedMonoRec, MonoRecModel
    C.set_mode("f16")
    B, F, H, W = 8, 4, 256, 512
    pairs = [gray_and_rgb(to_device(make_inputs(B, F, H, W, seed=500 + i), DEV)) for i in range(2)]
    torch.manual_seed(0)
    m = MonoRecModel().to(DEV).eval()
    graphs = {k: GraphedMonoRec(m, pairs[0][j]) for j, k in enumerate(("gray", "rgb"))}
    sets = {k: [p[j] for p in pairs] for j, k in enumerate(("gray", "rgb"))}
    res = {k: g(sets[k][0])["result"].clone() for k, g in graphs.items()}
    assert torch.equal(res["gray"], res["rgb"])
    for k, g in graphs.items():
        for i in range(3):
            g(sets[k][i % 2])
    torch.cuda.synchronize()
    times = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            c = [0]

            def step():
                g(sets[k][c[0] % 2])
                c[0] += 1
            times[k].append(event_ms(step, iters))
    report("model f16 graph replay", [B, F, 32, H, W], times)


def main():
    opts = dict(a[2:].split("=", 1) for a in sys.argv[1:] if a.startswith("--"))
    iters, rounds = int(opts.get("iters", 20)), int(opts.get("rounds", 7))
    if not torch.cuda.is_available():
        raise SystemExit("time_cv_gray.py needs a CUDA device")
    lib = _lib.load()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}), flush=True)
    kernel(lib, iters, rounds)
    model(iters, rounds)


if __name__ == "__main__":
    main()
