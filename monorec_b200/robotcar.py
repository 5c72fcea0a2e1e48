"""Oxford RobotCar's lidar depth targets on the device (the loader's `get_depth`, data_loader/oxford_robotcar_dataset.py
:121-144, with the RobotCar SDK's pinhole `CameraModel.project`).

For a key frame with image timestamp T (integer microseconds) the loader takes every LD-MRS scan whose timestamp t satisfies
`T - r * 1e6 <= t <= T + r * 1e6` (r = `lidar_timestamp_range`), moves its points to the world with
`lidar_pose @ lidar_transform`, into the camera with `camera_transform @ inv(pose @ swapaxes_)`, projects them with the
camera model at the full image size, scales and truncates the pixel coordinates, and keeps per pixel the largest inverse
depth 1 / z of an array of `round(h / (1 - top - bottom))` x `round(w / (1 - left - right))` pixels, cropped by the cutout:
[1, h', w'] float32, 0 where no point lands.  A point whose pixel lies outside that array makes the loader raise IndexError.

* `lidar_depth(...)` is one key frame with the loader's arguments; it raises IndexError as the loader does.
* `RobotCarLidar` is the stream form over one sequence: `add_scan` uploads and transforms each scan once into a device ring
  of world points, `targets` builds a batch of key frames' targets in one call without a host synchronisation, and the
  out-of-array counts are read once the device has finished them (at a later `targets` call, or at `check()`).

The 4x4 matrices are computed on the host in float64 numpy exactly as the loader computes them; the per-point arithmetic runs
on the device in float64, op by op (`csrc/lidar_depth.cu`).  The camera is anything with the SDK CameraModel's
`G_camera_image`, `focal_length` and `principal_point`.
"""
import bisect
from collections import deque

import numpy as np
import torch

from . import _lib

# oxford_robotcar_dataset.py:18-23
SWAPAXES = np.asarray([[0, 0, 1, 0], [1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1]])
SWAPAXES_ = np.linalg.inv(SWAPAXES)


def target_geometry(shape, scale, cutout):
    """The loader's sizes for a key-frame image of `shape` (h, w): the image size handed to `CameraModel.project` (H, W),
    the depth array's size (Hd, Wd) and its crop window (r0, r1, c0, c1)."""
    h, w = (int(v) for v in shape)
    top, bottom, left, right = (float(c) for c in cutout)
    if not (h >= 1 and w >= 1):
        raise ValueError(f"shape {tuple(shape)} must be two positive integers (h, w)")
    if not (scale > 0 and np.isfinite(scale)):
        raise ValueError(f"scale ({scale!r}) must be finite and > 0")
    if min(top, bottom, left, right) < 0 or top + bottom >= 1 or left + right >= 1:
        raise ValueError(f"cutout {tuple(cutout)} must be (top, bottom, left, right) >= 0 with top + bottom < 1 and "
                         "left + right < 1")
    size = (h / scale / (1 - top - bottom), w / scale / (1 - left - right))                      # :133
    Hd, Wd = round(h / (1 - top - bottom)), round(w / (1 - left - right))                        # :142
    crop = (int(top * Hd), int(Hd - bottom * Hd), int(left * Wd), int(Wd - right * Wd))          # :144
    if not (0 <= crop[0] < crop[1] <= Hd and 0 <= crop[2] < crop[3] <= Wd):
        raise ValueError(f"shape {tuple(shape)} with cutout {tuple(cutout)} leaves an empty target")
    return size, (Hd, Wd), crop


def _matrix(m, what):
    m = np.asarray(m.cpu() if isinstance(m, torch.Tensor) else m, dtype=np.float64)
    if m.shape != (4, 4):
        raise ValueError(f"{what} must be a 4x4 matrix, got shape {m.shape}")
    if not np.isfinite(m).all():
        raise ValueError(f"{what} has entries that are not finite")
    return m


def _host_matrix(m, what):
    if isinstance(m, torch.Tensor) and m.device.type != "cpu":
        raise ValueError(f"{what} must be on the host (numpy or a CPU tensor): the matrices are computed there in float64")
    return _matrix(m, what)


class RobotCarLidar:
    """The lidar depth targets of one RobotCar sequence, from scans added once each.

    `camera`: the sequence's SDK CameraModel (or anything with `G_camera_image` [4,4], `focal_length` (fx, fy) and
    `principal_point` (cx, cy)); `camera_transform` and `lidar_transform`: the loader's `_camera_transform` and
    `_lidar_transform` of the sequence (build_se3_transform of the extrinsics); `shape` (h, w): the key-frame image's shape
    after the loader's scale and cutout; `scale`, `cutout`, `lidar_timestamp_range`: the loader's arguments.

    `add_scan(timestamp, points, lidar_pose)`: one scan, `points` [n,3] float64 in the lidar frame (the `.bin` file's
    triples; host array or float64 tensor on the device) and `lidar_pose` its interpolated VO pose; it is uploaded and
    transformed into the ring at once.  Scan timestamps must increase.  Every scan a key frame's window reaches must have
    been added before that key frame's `targets` call.

    `targets(image_timestamps, poses)`: [K,1,h',w'] float32 on the device, the key frames' targets (`poses`: the loader's
    `_sequence_poses` entries, host 4x4 each); image timestamps must increase, across calls too.  The call launches the
    kernel once per 16 key frames and makes no host synchronisation.  Afterwards, the scans no later key frame can reach
    leave the ring.  The out-of-array counts of a call are read at a later `targets` call once the device has finished
    them, or at `check()`, which waits for all; a key frame with such a point raises IndexError naming its timestamp.

    Every call runs on the device's current stream; use one stream for one RobotCarLidar.
    """

    def __init__(self, camera, camera_transform, lidar_transform, shape, scale=0.25, cutout=(1 / 6, 1 / 6, 0, 0),
                 lidar_timestamp_range=0.5, device=None, capacity=1 << 18):
        self.size, (self.Hd, self.Wd), self.crop = target_geometry(shape, scale, cutout)
        self.scale, self.cutout = float(scale), tuple(cutout)
        if not (lidar_timestamp_range >= 0 and np.isfinite(lidar_timestamp_range)):
            raise ValueError(f"lidar_timestamp_range ({lidar_timestamp_range!r}) must be finite and >= 0")
        self.range = lidar_timestamp_range
        self.camera_transform = _host_matrix(camera_transform, "camera_transform")
        self.lidar_transform = _host_matrix(lidar_transform, "lidar_transform")
        self._G = np.ascontiguousarray(_host_matrix(camera.G_camera_image, "G_camera_image"))
        f, pp = camera.focal_length, camera.principal_point
        # CameraModel.project's filter: 0.5 <= u <= W, 0.5 <= v <= H (W, H: the image size of :133)
        self._proj = np.array([f[0], f[1], pp[0], pp[1], 0.5, self.size[1], self.size[0], self.scale], np.float64)
        if not np.isfinite(self._proj).all():
            raise ValueError("focal_length and principal_point must be finite")
        self._crop = np.array(self.crop, np.int32)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if int(capacity) < 1:
            raise ValueError(f"capacity ({capacity!r}) must be >= 1")
        self._ring = torch.empty(int(capacity), 4, dtype=torch.float64, device=self.device)
        self._times, self._rows = [], []         # resident scans: timestamp, (first absolute row, point count)
        self._end = 0                            # absolute rows written
        self._last_scan = None
        self._last_image = None
        self._pending = deque()                  # (image timestamps, host counts, event) of calls not yet checked

    @property
    def capacity(self):
        return self._ring.shape[0]

    def _stream(self):
        return torch.cuda.current_stream(self.device)

    def add_scan(self, timestamp, points, lidar_pose):
        t = int(timestamp)
        if t != timestamp:
            raise ValueError(f"scan timestamp {timestamp!r} must be an integer (microseconds)")
        if self._last_scan is not None and t <= self._last_scan:
            raise ValueError(f"scan timestamps must increase: {t} after {self._last_scan}")
        M = _host_matrix(lidar_pose, "lidar_pose") @ self.lidar_transform                        # :129
        if isinstance(points, torch.Tensor) and points.device.type != "cpu":
            if points.device != self.device or points.dtype != torch.float64:
                raise ValueError(f"device points must be float64 on {self.device}, got {points.dtype} on {points.device}")
            scan = points.contiguous()
        else:
            host = torch.as_tensor(np.ascontiguousarray(points.numpy() if isinstance(points, torch.Tensor) else points,
                                                        np.float64))
            scan = None
        shape = tuple(scan.shape if scan is not None else host.shape)
        if len(shape) != 2 or shape[1] != 3:
            raise ValueError(f"points must be [n,3] (x, y, z per point), got shape {shape}")
        n = shape[0]
        if scan is None:
            scan = host.pin_memory().to(self.device, non_blocking=True) if n else host.to(self.device)
        self._reserve(n)
        M = np.ascontiguousarray(M)
        lib = _lib.load()
        with torch.cuda.device(self.device):
            _lib.check(lib.mr_lidar_to_world(scan.data_ptr() if n else None, n, M.ctypes.data, self._ring.data_ptr(),
                                             self.capacity, self._end % self.capacity, self._stream().cuda_stream),
                       "mr_lidar_to_world")
        self._times.append(t)
        self._rows.append((self._end, n))
        self._end += n
        self._last_scan = t

    def _reserve(self, n):
        """Grows the ring (twice the capacity, or what the resident scans and n need) when n more rows do not fit."""
        lo = self._rows[0][0] if self._rows else self._end
        live = self._end - lo
        if live + n <= self.capacity:
            return
        cap = max(2 * self.capacity, live + n)
        ring = torch.empty(cap, 4, dtype=torch.float64, device=self.device)
        if live:
            rows = torch.arange(lo, self._end, device=self.device)
            ring[rows % cap] = self._ring[rows % self.capacity]
        self._ring = ring

    def _window(self, T):
        """The resident scans of image timestamp T's window (:124): first ring row and point count."""
        lo_t, hi_t = T - self.range * 1e6, T + self.range * 1e6
        i = bisect.bisect_left(self._times, lo_t)
        j = bisect.bisect_right(self._times, hi_t)
        if i >= j:
            return 0, 0
        first = self._rows[i][0]
        return first % self.capacity, self._rows[j - 1][0] + self._rows[j - 1][1] - first

    def targets(self, image_timestamps, poses):
        ts = []
        for t in image_timestamps:
            if int(t) != t:
                raise ValueError(f"image timestamp {t!r} must be an integer (microseconds)")
            ts.append(int(t))
        poses = [_host_matrix(p, "pose") for p in poses]
        K = len(ts)
        if K < 1 or len(poses) != K:
            raise ValueError(f"targets: one pose per image timestamp and at least one of each, got {K} and {len(poses)}")
        prev = self._last_image
        for t in ts:
            if prev is not None and t <= prev:
                raise ValueError(f"image timestamps must increase: {t} after {prev}")
            prev = t
        self._check_done(wait=False)
        cam = np.ascontiguousarray(np.stack([self.camera_transform @ np.linalg.inv(p @ SWAPAXES_) for p in poses]))  # :131
        windows = [self._window(t) for t in ts]
        first = np.array([w[0] for w in windows], np.int64)
        count = np.array([w[1] for w in windows], np.int64)
        r0, r1, c0, c1 = self.crop
        out = torch.empty(K, 1, r1 - r0, c1 - c0, dtype=torch.float32, device=self.device)
        oob = torch.empty(K, dtype=torch.int32, device=self.device)
        lib = _lib.load()
        stream = self._stream()
        with torch.cuda.device(self.device):
            _lib.check(lib.mr_lidar_depth(self._ring.data_ptr(), self.capacity, K, first.ctypes.data, count.ctypes.data,
                                          cam.ctypes.data, self._G.ctypes.data, self._proj.ctypes.data, self.Hd, self.Wd,
                                          self._crop.ctypes.data, out.data_ptr(), oob.data_ptr(), stream.cuda_stream),
                       "mr_lidar_depth")
            host = torch.empty(K, dtype=torch.int32, pin_memory=True)
            host.copy_(oob, non_blocking=True)
            done = torch.cuda.Event()
            done.record(stream)
        self._pending.append((ts, host, done))
        self._last_image = ts[-1]
        # no later image timestamp's window reaches a scan below this bound (timestamps increase)
        keep = bisect.bisect_left(self._times, ts[-1] - self.range * 1e6)
        del self._times[:keep], self._rows[:keep]
        return out

    def check(self):
        """Waits for every targets call so far and raises IndexError for a key frame with a point outside the depth array."""
        self._check_done(wait=True)

    def _check_done(self, wait):
        while self._pending:
            ts, host, done = self._pending[0]
            if wait:
                done.synchronize()
            elif not done.query():
                return
            self._pending.popleft()
            for t, n in zip(ts, host.tolist()):
                if n:
                    raise IndexError(f"lidar depth of the key frame at image timestamp {t}: {n} projected point(s) fall "
                                     f"outside the {self.Hd}x{self.Wd} depth array (the loader raises IndexError)")


def lidar_depth(image_timestamp, pose, scan_timestamps, scans, lidar_poses, camera, camera_transform, lidar_transform,
                shape, scale=0.25, cutout=(1 / 6, 1 / 6, 0, 0), lidar_timestamp_range=0.5, device=None):
    """`OxfordRobotCarDataset.get_depth` of one key frame on the device: [1, h', w'] float32.

    `image_timestamp`, `pose`: the key frame's timestamp and `_sequence_poses` entry; `scan_timestamps`, `scans` ([n,3]
    each) and `lidar_poses`: the sequence's scans and their interpolated poses (those outside the key frame's window are not
    read); the other arguments as for `RobotCarLidar`.  Raises IndexError where the loader does (waits for the device)."""
    T = int(image_timestamp)
    lo, hi = T - lidar_timestamp_range * 1e6, T + lidar_timestamp_range * 1e6
    sel = sorted((int(t), i) for i, t in enumerate(scan_timestamps) if lo <= t <= hi)                      # :124
    n = sum(len(scans[i]) for _, i in sel)
    ring = RobotCarLidar(camera, camera_transform, lidar_transform, shape, scale, cutout, lidar_timestamp_range, device,
                         capacity=max(1, n))
    for t, i in sel:
        ring.add_scan(t, scans[i], lidar_poses[i])
    out = ring.targets([T], [pose])
    ring.check()
    return out[0]
