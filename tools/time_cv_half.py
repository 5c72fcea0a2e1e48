"""fp32 vs half cost volumes (mr_cost_volume_fwd_typed / volume_dtype=torch.float16), interleaved, in one process.

    python tools/time_cv_half.py [--iters=N] [--rounds=R]

Three measurements, each alternating fp32 and half volumes every round; a round's number is the mean over N calls, the
report the median over R rounds:
  kernel   one launch of the cost-volume kernel (CUDA events) at config 2 (B 8, F 4, D 32, 256x512) and hires (B 4, F 6,
           D 64, 512x1024), plane depths, SSIM, centred
  model    MonoRecModel.forward in f16 engine mode, replayed from a CUDA graph (random-init weights), B 8 and B 16 at
           F 4, D 32, 256x512
  host     mr_cost_volume_host vs mr_cost_volume_host_f16 at config 2 (pinned host buffers, fused volume downloaded,
           single-frame volumes left on the device as bench.py's e2e does), host clock around the synchronous call
The card name and its power limit are printed with the numbers (one JSON line per measurement).
"""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from monorec_b200 import _lib  # noqa: E402
from monorec_b200.synthetic import make_inputs, to_device  # noqa: E402

DEV = "cuda:0"
DTYPES = (("fp32", torch.float32, 0), ("half", torch.float16, 1))


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
    print(json.dumps({"what": what, "shape": shape, "median_ms": med, "rounds": {k: v for k, v in times.items()},
                      "half_over_fp32": med["half"] / med["fp32"]}), flush=True)


def kernel(lib, iters, rounds):
    for name, (B, F, D, H, W) in (("config2", (8, 4, 32, 256, 512)), ("hires", (4, 6, 64, 512, 1024))):
        d = to_device(make_inputs(B, F, H, W, seed=0), DEV)
        proj = torch.empty(B, F, 3, 4, device=DEV)
        planes = torch.empty(D, device=DEV)
        stream = torch.cuda.current_stream().cuda_stream
        frames = _lib.ptr_array(d["frames"])
        _lib.check(lib.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                            _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H, W,
                                            proj.data_ptr(), planes.data_ptr(), D, 0.0025, 0.33, stream), "tables")
        cw = (_lib.c_float * 3)(5 / 32, 16 / 32, 11 / 32)
        outs = {k: (torch.empty(B, D, H, W, device=DEV, dtype=dt), torch.empty(F, B, D, H, W, device=DEV, dtype=dt), code)
                for k, dt, code in DTYPES}

        def launch(k):
            cv, sf, code = outs[k]
            _lib.check(lib.mr_cost_volume_fwd_typed(d["keyframe"].data_ptr(), frames, proj.data_ptr(), planes.data_ptr(), None,
                                                    cv.data_ptr(), sf.data_ptr(), None, 0, B, F, D, H, W, 10.0, cw, 1, 1, code,
                                                    stream), "mr_cost_volume_fwd_typed")
        for k in outs:
            for _ in range(3):
                launch(k)
        torch.cuda.synchronize()
        times = {k: [] for k in outs}
        for _ in range(rounds):
            for k in outs:
                times[k].append(event_ms(lambda: launch(k), iters))
        report(f"kernel {name}", [B, F, D, H, W], times)
        del outs, d
        torch.cuda.empty_cache()


def model(iters, rounds):
    from monorec_b200 import conv as C
    from monorec_b200.model import GraphedMonoRec, MonoRecModel
    C.set_mode("f16")
    F, H, W = 4, 256, 512
    for B in (8, 16):
        sets = [to_device(make_inputs(B, F, H, W, seed=500 + i), DEV) for i in range(2)]
        graphs = {}
        for k, dt, _ in DTYPES:
            torch.manual_seed(0)
            m = MonoRecModel(volume_dtype=dt).to(DEV).eval()
            graphs[k] = GraphedMonoRec(m, sets[0])
        for g in graphs.values():
            for i in range(3):
                g(sets[i % 2])
        torch.cuda.synchronize()
        times = {k: [] for k in graphs}
        for _ in range(rounds):
            for k, g in graphs.items():
                c = [0]

                def step():
                    g(sets[c[0] % 2])
                    c[0] += 1
                times[k].append(event_ms(step, iters))
        report("model f16 graph replay", [B, F, 32, H, W], times)
        del graphs, sets
        torch.cuda.empty_cache()


def host(lib, iters, rounds):
    B, F, D, H, W = 8, 4, 32, 256, 512
    h = make_inputs(B, F, H, W, seed=7)
    h_key = h["keyframe"].contiguous().pin_memory()
    h_frames = torch.stack(h["frames"]).contiguous().pin_memory()
    h_kp = h["keyframe_pose"].contiguous().pin_memory()
    h_kk = h["keyframe_intrinsics"].contiguous().pin_memory()
    h_poses = torch.stack(h["poses"]).contiguous().pin_memory()
    h_intr = torch.stack(h["intrinsics"]).contiguous().pin_memory()
    cfg = {"fp32": (lib.mr_cost_volume_host, lib.mr_cost_volume_host_workspace(B, F, D, H, W), torch.float32),
           "half": (lib.mr_cost_volume_host_f16, lib.mr_cost_volume_host_f16_workspace(B, F, D, H, W), torch.float16)}
    bufs = {k: (torch.empty(ws, dtype=torch.uint8, device=DEV), torch.empty(B, D, H, W, dtype=dt).pin_memory())
            for k, (_, ws, dt) in cfg.items()}

    def call(k):
        fn, ws_bytes, _ = cfg[k]
        ws, h_cv = bufs[k]
        _lib.check(fn(h_key.data_ptr(), h_frames.data_ptr(), h_kp.data_ptr(), h_kk.data_ptr(), h_poses.data_ptr(),
                      h_intr.data_ptr(), h_cv.data_ptr(), None, B, F, D, H, W, 0.0025, 0.33, 10.0, ws.data_ptr(), ws_bytes), k)
    for k in cfg:
        for _ in range(3):
            call(k)
    times = {k: [] for k in cfg}
    for _ in range(rounds):
        for k in cfg:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(iters):
                call(k)       # synchronous: returns after the last device-to-host copy has landed
            times[k].append((time.perf_counter() - t0) * 1e3 / iters)
    report("mr_cost_volume_host (fused volume downloaded)", [B, F, D, H, W], times)


def main():
    opts = dict(a[2:].split("=", 1) for a in sys.argv[1:] if a.startswith("--"))
    iters, rounds = int(opts.get("iters", 20)), int(opts.get("rounds", 7))
    if not torch.cuda.is_available():
        raise SystemExit("time_cv_half.py needs a CUDA device")
    lib = _lib.load()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}), flush=True)
    kernel(lib, iters, rounds)
    host(lib, max(3, iters // 2), rounds)
    model(iters, rounds)


if __name__ == "__main__":
    main()
