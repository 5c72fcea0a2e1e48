#!/usr/bin/env python
"""Writes tests/golden/robotcar_depth.npz by running the UNMODIFIED reference `OxfordRobotCarDataset.get_depth`
(data_loader/oxford_robotcar_dataset.py:121-144) on CPU:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_robotcar_depth.py

The loader's RobotCar SDK package (`oxford_robotcar`: CameraModel, VO pose interpolation, SE(3) from extrinsics) is not part
of the reference; stubs are put into the loaded module's namespace (`PinholeCameraModel` below restates the SDK's pinhole
projection), with the stub `skimage` and numpy aliases of make_golden_loader_streams.py.  Each case is a stub tree in a
temporary directory: empty image files named by their timestamps, synthetic LD-MRS scans as `.bin` files of float64 triples,
and the extrinsics files.  The scans' points are drawn in the image of a nearby key frame (pixel and depth, some behind the
camera, some outside the image, several at one pixel with different depths) and mapped back through the chain to the lidar
frame, so most of them land in the target.

Cases: overlapping windows of consecutive key frames with scans exactly on and one microsecond outside each bound of one key
frame and an empty scan (scale 0.25, the default cutout); scale 0.5 with a zero cutout; a size whose target is larger than
the image (h' != h); an image timestamp whose window holds no scan; a size whose depth array is rounded down, where the loader
raises IndexError.

Every point's float64 u * scale and v * scale is checked to lie more than 1e-6 from an integer, and u, v more than 1e-6 from
the projection's bounds, so that no last-bit difference between numpy's matrix products and the device's op-by-op
arithmetic can move a point across a pixel or a bound unnoticed.

Stored per case `<name>/...`: the loader's arguments and matrices (`shape`, `scale`, `cutout`, `range`, `G`, `focal`,
`principal`, `camera_transform`, `lidar_transform`), the image timestamps and `_sequence_poses` (`image_t`, `poses`), the
scans (`scan_t`, `scan_offsets`, `scan_points` concatenated, `lidar_poses`), and per evaluated key frame (`keys`) the
loader's output `depth` [K,1,h',w'] float32 (zeros where it raised) and `error` (1: IndexError).
"""
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)
from make_golden_loader_streams import _stubs  # noqa: E402
from oracle import robotcar_depth_oracle as O  # noqa: E402


class PinholeCameraModel:
    """The RobotCar SDK's CameraModel.project (camera_model.py), restated from the published SDK; it could not be checked
    against the SDK here, which is not part of the reference.  The points go through G_camera_image, uv = f xy / z +
    principal_point, and a point is kept iff z > 0, 0.5 <= u <= W and 0.5 <= v <= H (image_size = (H, W)).  NaN compares
    false, so the loader's dummy column [0, 0, 0, 0] (0 / 0) drops out."""
    camera = "stereo"

    def __init__(self, model_folder, sequence_folder):
        pass

    def project(self, xyz, image_size):
        xyzw = self.G_camera_image @ xyz
        with np.errstate(divide="ignore", invalid="ignore"):
            uv = np.vstack((self.focal_length[0] * xyzw[0, :] / xyzw[2, :] + self.principal_point[0],
                            self.focal_length[1] * xyzw[1, :] / xyzw[2, :] + self.principal_point[1]))
            keep = (xyzw[2, :] > 0) & (0.5 <= uv[0]) & (uv[0] <= image_size[1]) & (0.5 <= uv[1]) & (uv[1] <= image_size[0])
        return uv[:, keep], np.ravel(xyzw[2, keep])


def se3(x, y, z, roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    m = np.eye(4)
    m[:3, :3] = np.array([[cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr],
                          [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr],
                          [-sp, cp * sr, cp * cr]])
    m[:3, 3] = (x, y, z)
    return m


def vehicle_pose(t):
    """The stub VO pose at timestamp t (microseconds): forward at 5 m/s, slowly turning."""
    s = (t - T0) / 1e6
    return se3(5.0 * s, 0.3 * np.sin(s), 0.02 * s, 0.01 * np.sin(2 * s), 0.005 * s, 0.04 * s)


LIDAR_EXT = (1.7, 0.05, -1.2, 0.01, -0.02, 0.015)
CAMERA_EXT = (1.9, 0.1, -1.3, -0.01, 0.01, 0.02)
G = se3(0, 0, 0, 0.003, -0.002, 0.001) @ np.array([[0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 1.0]])
FOCAL, PRINCIPAL = (160.3, 158.9), (127.3, 95.6)          # a 256 x 192 full-size image

T0 = 1_400_000_000_000_000                 # microseconds: every timestamp has 16 digits, so the files sort by time
CASES = [
    # name, shape, scale, cutout, lidar_timestamp_range, image timestamps, key indices, extra scan timestamps
    ("overlap", (32, 64), 0.25, (1 / 6, 1 / 6, 0, 0), 0.5, [T0 + 250_000 * k for k in range(6)], [1, 2, 3, 4],
     [T0 + 500_000 - 500_000, T0 + 500_000 + 500_000, T0 + 500_000 - 500_001, T0 + 500_000 + 500_001]),
    ("half_nocut", (96, 128), 0.5, (0, 0, 0, 0), 0.3, [T0 + 200_000 * k for k in range(5)], [1, 2, 3], []),
    ("rounded", None, 0.25, (0.1, 0.15, 0.05, 0.05), 0.5, [T0 + 300_000 * k for k in range(4)], [1, 2], []),
    ("empty", (32, 64), 0.25, (1 / 6, 1 / 6, 0, 0), 0.5, [T0, T0 + 3_000_000], [1], []),
    ("index_error", None, 0.25, (0.2, 0.1, 0, 0), 0.5, [T0 + 300_000 * k for k in range(4)], [1, 2], []),
]


def rounded_shape(cutout, up):
    """A key-frame shape near 32 x 64 whose target shape differs from it (up: the depth array is rounded up, so no point
    falls outside it; not up: rounded down in rows)."""
    for h in range(30, 40):
        for w in range(60, 70):
            _, (Hd, Wd), (r0, r1, c0, c1) = O.geometry((h, w), 0.25, cutout)
            exact_h, exact_w = h / (1 - cutout[0] - cutout[1]), w / (1 - cutout[2] - cutout[3])
            if up and Hd >= exact_h and Wd >= exact_w and (r1 - r0, c1 - c0) != (h, w):
                return h, w
            if not up and Hd < exact_h - 0.2 and Wd >= exact_w:
                return h, w
    raise RuntimeError("no shape found")


def scans_for(g, image_t, scan_t, chain, size):
    """Points of each scan, drawn in the image of the key frame nearest in time and mapped back to the lidar frame."""
    H0, W0 = size
    out = []
    for i, t in enumerate(scan_t):
        n = 0 if i == 3 else int(g.integers(100, 260))
        k = int(np.argmin(np.abs(np.asarray(image_t) - t)))
        u = g.uniform(-0.1 * W0, 1.1 * W0, n)
        v = g.uniform(-0.1 * H0, 1.1 * H0, n)
        z = g.uniform(2.0, 60.0, n)
        z[g.random(n) < 0.07] *= -1.0                                     # behind the camera
        dup = g.random(n) < 0.15                                          # a second point on the pixel of the previous one
        dup[:1] = False
        u[dup], v[dup] = u[np.flatnonzero(dup) - 1], v[np.flatnonzero(dup) - 1]
        img = np.stack([(u - PRINCIPAL[0]) * z / FOCAL[0], (v - PRINCIPAL[1]) * z / FOCAL[1], z, np.ones(n)])
        world_from_image, lidar_to_world = chain(k, t)
        p = np.linalg.inv(lidar_to_world) @ world_from_image @ img
        out.append(np.ascontiguousarray(p[:3].T))
    return out


class MarginError(Exception):
    pass


def check_margins(name, world, ds, keys, shape, scale, cutout):
    """No kept point within 1e-6 of a pixel edge after scaling, nor of the projection's bounds."""
    size, _, _ = O.geometry(shape, scale, cutout)
    for k in keys:
        q = O._apply(ds._camera_transform[0] @ np.linalg.inv(ds._sequence_poses[0][k] @ O.SWAPAXES_), world)
        x, y, z, _ = O._apply(G, q)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = FOCAL[0] * x / z + PRINCIPAL[0]
            v = FOCAL[1] * y / z + PRINCIPAL[1]
        front = z > 0
        for a, hi in ((u[front], size[1]), (v[front], size[0])):
            near_bound = np.minimum(np.abs(a - 0.5), np.abs(a - hi)).min() if a.size else 1.0
            if not near_bound > 1e-6:
                raise MarginError(f"{name}, key {k}: a point {near_bound:.2e} from a bound")
            inside = (0.5 <= a) & (a <= hi)
            s = a[inside] * scale
            frac = np.abs(s - np.round(s)).min() if s.size else 1.0
            if not frac > 1e-6:
                raise MarginError(f"{name}, key {k}: a scaled pixel coordinate {frac:.2e} from an integer")


def run_case(R, root, g, case):
    name, shape, scale, cutout, rng, image_t, keys, extra = case
    if shape is None:
        shape = rounded_shape(cutout, up=name != "index_error")
    size, _, _ = O.geometry(shape, scale, cutout)
    scan_t = sorted(set([image_t[0] - 400_000 + 100_000 * j for j in range((image_t[-1] - image_t[0]) // 100_000 + 9)]
                        + extra))
    if name == "empty":
        scan_t = [t for t in scan_t if abs(t - image_t[1]) > 2_000_000]
    d = root / name
    (d / "stereo").mkdir(parents=True)
    (d / "ldmrs").mkdir()
    (d / "extrinsics").mkdir()
    (d / "extrinsics" / "ldmrs.txt").write_text(" ".join(map(str, LIDAR_EXT)) + "\n")
    (d / "extrinsics" / "stereo.txt").write_text(" ".join(map(str, CAMERA_EXT)) + "\n")
    for t in image_t:
        (d / "stereo" / f"{t}.png").write_bytes(b"")
    # the points come from the loader's own matrices: build the dataset on the image tree first
    for t in scan_t:
        (d / "ldmrs" / f"{t}.bin").write_bytes(b"")
    ds = R.OxfordRobotCarDataset([str(d / "stereo")], [""], [str(d / "ldmrs")], str(d), str(d / "extrinsics"),
                                 frame_count=2, dilation=1, scale=scale, cutout=cutout, lidar_timestamp_range=rng)
    cam = ds._sequence_camera_models[0]
    assert ds._lidar_timestamps[0] == scan_t

    def chain(k, t):
        C = ds._camera_transform[0] @ np.linalg.inv(ds._sequence_poses[0][k] @ O.SWAPAXES_)
        return np.linalg.inv(G @ C), ds._lidar_poses[0][scan_t.index(t)] @ ds._lidar_transform[0]
    scans = scans_for(g, image_t, scan_t, chain, (size[0], size[1]))
    for t, s in zip(scan_t, scans):
        s.astype(np.float64).tofile(d / "ldmrs" / f"{t}.bin")
    world = np.hstack([O.world_points(s, ds._lidar_poses[0][i], ds._lidar_transform[0]) for i, s in enumerate(scans)])
    check_margins(name, world, ds, keys, shape, scale, cutout)
    depth, error = [], []
    _, _, (r0, r1, c0, c1) = O.geometry(shape, scale, cutout)
    for k in keys:
        try:
            out = np.asarray(ds.get_depth(0, k, shape))
            assert out.shape == (1, r1 - r0, c1 - c0), (name, out.shape)
            depth.append(np.asarray(out, np.float64).astype(np.float32))
            error.append(0)
        except IndexError:
            depth.append(np.zeros((1, r1 - r0, c1 - c0), np.float32))
            error.append(1)
    offsets = np.cumsum([0] + [len(s) for s in scans])
    rec = dict(shape=np.array(shape), scale=np.float64(scale), cutout=np.array(cutout, np.float64), range=np.float64(rng),
               G=cam.G_camera_image, focal=np.array(FOCAL), principal=np.array(PRINCIPAL),
               camera_transform=ds._camera_transform[0], lidar_transform=ds._lidar_transform[0],
               image_t=np.array(image_t, np.int64), poses=np.stack(ds._sequence_poses[0]),
               scan_t=np.array(scan_t, np.int64), scan_offsets=offsets, scan_points=np.concatenate(scans),
               lidar_poses=np.stack(ds._lidar_poses[0]), keys=np.array(keys), depth=np.stack(depth),
               error=np.array(error))
    hits = [int((x > 0).sum()) for x in depth]
    print(name, "shape", shape, "target", depth[0].shape, "points", offsets[-1], "errors", error, "filled", hits)
    return rec


def main():
    import_reference()
    _stubs()
    import data_loader.oxford_robotcar_dataset as R  # noqa
    PinholeCameraModel.G_camera_image, PinholeCameraModel.focal_length = G, FOCAL
    PinholeCameraModel.principal_point = PRINCIPAL
    R.CameraModel = PinholeCameraModel
    R.interpolate_vo_poses = lambda pose_file, timestamps, origin: [vehicle_pose(int(t)) for t in timestamps]
    R.build_se3_transform = lambda xyzrpy: se3(*xyzrpy)
    for seed in range(2024, 2124):          # the first seed whose points all keep the margins
        g = np.random.default_rng(seed)
        out = {}
        try:
            with tempfile.TemporaryDirectory() as tmp:
                for case in CASES:
                    for key, value in run_case(R, Path(tmp), g, case).items():
                        out[f"{case[0]}/{key}"] = value
            break
        except MarginError as e:
            print("seed", seed, "rejected:", e)
    assert out["index_error/error"].any() and not any(out[f"{c[0]}/error"].any() for c in CASES if c[0] != "index_error")
    assert not out["empty/depth"].any()
    path = HERE / "robotcar_depth.npz"
    np.savez_compressed(path, cases=np.array([c[0] for c in CASES]), **out)
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
