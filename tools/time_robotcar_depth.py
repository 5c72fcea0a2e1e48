"""Per-key-frame cost of Oxford RobotCar's lidar depth targets against the model, at the loader's default settings.

    python tools/time_robotcar_depth.py [--points=N] [--keys=K] [--batch=B] [--rounds=R] [--scale=S]

A synthetic RobotCar sequence: 1280x960 stereo images at 16 Hz, LD-MRS scans of `--points` points at 12.5 Hz (real scan
sizes are not known here: pass them), lidar_timestamp_range 0.5 s, the default cutout (1/6, 1/6, 0, 0).  Three numbers per
key frame, each the median over R rounds:
  device_ms   RobotCarLidar over the stream: every scan uploaded and transformed once, targets in batches of B key frames,
              check() at the end; host time from the first add_scan to a device synchronise after the last call, over K;
  loader_ms   the loader's get_depth arithmetic (oxford_robotcar_dataset.py:121-144, restated below with its numpy calls)
              with the scans already read from their files, on one CPU thread;
  model_ms    MonoRecModel (random-init weights, f16 mode) over MonoRecSequence with robotcar_layout at sequence batch B, at
              the key-frame size the loader produces for the same scale and cutout, frames already on the device.
The card name and power limit are printed with the numbers (one JSON line).
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
from monorec_b200.robotcar import SWAPAXES, SWAPAXES_, RobotCarLidar, target_geometry  # noqa: E402
from monorec_b200.sequence import MonoRecSequence, robotcar_layout  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402

DEV = "cuda:0"
FULL = (960, 1280)
CUTOUT = (1 / 6, 1 / 6, 0, 0)
RANGE = 0.5


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # (no nvidia-smi: report why)
        return f"unknown ({e})"


def se3(x, yaw):
    m = np.eye(4)
    m[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    m[0, 3] = x
    return m


class Camera:
    G_camera_image = np.array([[0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 1.0]])
    focal_length = (983.0, 983.0)
    principal_point = (643.0, 484.0)


def scene(n_keys, points, seed=0):
    """Image and scan timestamps (microseconds), poses at 5 m/s and the scans (points ahead of the vehicle)."""
    g = np.random.default_rng(seed)
    t0 = 1_400_000_000_000_000
    image_t = [t0 + 62_500 * k for k in range(n_keys)]
    scan_t = list(range(t0 - 600_000, image_t[-1] + 600_000, 80_000))
    pose = lambda t: se3(5.0 * (t - t0) / 1e6, 0.02 * (t - t0) / 1e6)               # noqa: E731
    scans = [g.normal([20.0, 0.0, 0.0], [12.0, 10.0, 2.0], (points, 3)) for _ in scan_t]
    # the loader's _sequence_poses are the VO poses @ swapaxes (:73)
    return image_t, [pose(t) @ SWAPAXES for t in image_t], scan_t, scans, [pose(t) for t in scan_t]


def loader_get_depth(T, pose, scan_t, scans, lidar_poses, lidar_transform, camera_transform, shape, scale):
    """get_depth's arithmetic, numpy call by numpy call, with the scans already read (the SDK's pinhole project inline)."""
    idx = [i for i, t in enumerate(scan_t) if T - RANGE * 1e6 <= t <= T + RANGE * 1e6]
    pointcloud = np.array([[0], [0], [0], [0]])
    for i in idx:
        scan = scans[i].T
        scan = lidar_poses[i] @ lidar_transform @ np.vstack([scan, np.ones((1, scan.shape[1]))])
        pointcloud = np.hstack([pointcloud, scan])
    pointcloud = camera_transform @ (np.linalg.inv(pose @ SWAPAXES_)) @ pointcloud
    size = (shape[0] / scale / (1 - CUTOUT[0] - CUTOUT[1]), shape[1] / scale / (1 - CUTOUT[2] - CUTOUT[3]))
    xyzw = Camera.G_camera_image @ pointcloud
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = np.vstack((Camera.focal_length[0] * xyzw[0] / xyzw[2] + Camera.principal_point[0],
                        Camera.focal_length[1] * xyzw[1] / xyzw[2] + Camera.principal_point[1]))
        keep = (xyzw[2] > 0) & (0.5 <= uv[0]) & (uv[0] <= size[1]) & (0.5 <= uv[1]) & (uv[1] <= size[0])
    uv, d = uv[:, keep], xyzw[2, keep]
    uv *= scale
    uv = uv.astype(int)
    d = 1 / d
    order = np.argsort(d)
    uv, d = uv[:, order], d[order]
    depth = np.zeros((round(shape[0] / (1 - CUTOUT[0] - CUTOUT[1])), round(shape[1] / (1 - CUTOUT[2] - CUTOUT[3]))))
    depth[uv[1, :], uv[0, :]] = d
    depth = depth[int(CUTOUT[0] * depth.shape[0]):int(depth.shape[0] - CUTOUT[1] * depth.shape[0]),
                  int(CUTOUT[2] * depth.shape[1]):int(depth.shape[1] - CUTOUT[3] * depth.shape[1])]
    return np.expand_dims(depth, 0)


def time_device(st, shape, scale, batch, lt, ct):
    image_t, poses, scan_t, scans, lidar_poses = st
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ring = RobotCarLidar(Camera, ct, lt, shape, scale, CUTOUT, RANGE, device=DEV)
    i, out = 0, []
    for j in range(0, len(image_t), batch):
        hi = image_t[min(j + batch, len(image_t)) - 1] + RANGE * 1e6
        while i < len(scan_t) and scan_t[i] <= hi:
            ring.add_scan(scan_t[i], scans[i], lidar_poses[i])
            i += 1
        out.append(ring.targets(image_t[j:j + batch], poses[j:j + batch]))
    ring.check()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / len(image_t), torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=4000, help="points per LD-MRS scan")
    ap.add_argument("--keys", type=int, default=128)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--scale", type=float, default=0.25)
    args = ap.parse_args()
    C.set_mode("f16")
    # the key-frame shape the loader's crop gives at this scale (get_timestamp, :111-117)
    sh = int(FULL[0] * args.scale)
    shape = (int(sh - CUTOUT[1] * sh) - int(CUTOUT[0] * sh), int(FULL[1] * args.scale))
    _, _, crop = target_geometry(shape, args.scale, CUTOUT)
    lt, ct = se3(1.7, 0.01), se3(1.9, -0.01)
    st = scene(args.keys, args.points)
    dev, ref = [], []
    time_device(st, shape, args.scale, args.batch, lt, ct)                            # warm-up
    for _ in range(args.rounds):
        dt, out = time_device(st, shape, args.scale, args.batch, lt, ct)
        dev.append(dt)
        t0 = time.perf_counter()
        n_ref = 8
        for k in range(n_ref):
            ref_k = loader_get_depth(st[0][k], st[1][k], st[2], st[3], st[4], lt, ct, shape, args.scale)
        ref.append((time.perf_counter() - t0) / n_ref)
    got = out[n_ref - 1].cpu().numpy()
    differing = int((got != ref_k.astype(np.float32)).sum())
    # the model at the key-frame size
    n = args.keys + 2
    images, vo, Ks = make_sequence(n, shape[0], shape[1], seed=1)
    images, vo, Ks = images.to(DEV), vo.to(DEV), Ks.to(DEV)
    model = M.MonoRecModel()
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(DEV).eval()
    lay = robotcar_layout(n, 2)
    mod = []
    with torch.no_grad():
        for r in range(args.rounds + 1):
            seq = MonoRecSequence(model, batch_size=args.batch, graphed=True, layout=lay)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for f in range(n):
                seq.push(images[f], vo[f], Ks[f])
            seq.flush()
            torch.cuda.synchronize()
            if r:
                mod.append((time.perf_counter() - t0) / len(lay.keys))
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scale": args.scale,
                      "cutout": list(CUTOUT), "key_frame_shape": list(shape), "target_shape": [crop[1] - crop[0],
                                                                                                crop[3] - crop[2]],
                      "points_per_scan": args.points, "scans_per_window": int(round(2 * RANGE * 12.5)),
                      "keys": args.keys, "batch": args.batch, "rounds": args.rounds,
                      "per_key_ms": {"device": statistics.median(dev) * 1e3, "loader": statistics.median(ref) * 1e3,
                                     "model": statistics.median(mod) * 1e3},
                      "pixels_differing_from_loader_arithmetic": differing}), flush=True)


if __name__ == "__main__":
    main()
