"""numpy float64 restatement of Oxford RobotCar's lidar depth target (OxfordRobotCarDataset.get_depth, reference:
data_loader/oxford_robotcar_dataset.py:121-144) with the RobotCar SDK's pinhole projection, in the eight steps the device
path takes:

  1. the scans with T - r 1e6 <= t <= T + r 1e6 (Python floats, both bounds inclusive);
  2. world points (lidar_pose @ lidar_transform) @ [x y z 1]^T per scan (the loader's dummy column never makes a point);
  3. camera points (camera_transform @ inv(pose @ swapaxes_)) @ world;
  4. G_camera_image @ camera, uv = f xy / z + principal_point, kept iff z > 0, 0.5 <= u <= W and 0.5 <= v <= H at the image
     size (h / scale / (1 - top - bottom), w / scale / (1 - left - right));
  5. uv * scale truncated toward zero, d = 1 / z;
  6. per pixel of the round(h / (1 - top - bottom)) x round(w / (1 - left - right)) array the largest d (the loader's last
     write after its ascending sort);
  7. the cutout's crop, [1, h', w'] float32;
  8. IndexError if a kept point's pixel lies outside the array.

The 4x4 matrices are products of numpy `@` as in the loader; the per-point products are written out element by element in
the naive left-to-right order (each product and sum rounded on its own), the order of csrc/lidar_depth.cu, so the device
output equals this one bit for bit.
"""
import numpy as np

SWAPAXES_ = np.linalg.inv(np.asarray([[0, 0, 1, 0], [1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1]]))


def _apply(m, p):
    """Rows of m @ p for p [4,n], each as ((m0 p0 + m1 p1) + m2 p2) + m3 p3."""
    return np.stack([((m[r, 0] * p[0] + m[r, 1] * p[1]) + m[r, 2] * p[2]) + m[r, 3] * p[3] for r in range(4)])


def geometry(shape, scale, cutout):
    h, w = shape
    size = (h / scale / (1 - cutout[0] - cutout[1]), w / scale / (1 - cutout[2] - cutout[3]))
    Hd, Wd = round(h / (1 - cutout[0] - cutout[1])), round(w / (1 - cutout[2] - cutout[3]))
    crop = (int(cutout[0] * Hd), int(Hd - cutout[1] * Hd), int(cutout[2] * Wd), int(Wd - cutout[3] * Wd))
    return size, (Hd, Wd), crop


def world_points(scan, lidar_pose, lidar_transform):
    """Step 2: [4,n] world points of one [n,3] scan."""
    scan = np.asarray(scan, np.float64).reshape(-1, 3).T
    return _apply(lidar_pose @ lidar_transform, np.vstack([scan, np.ones((1, scan.shape[1]))]))


def project(world, pose, camera_transform, G, focal_length, principal_point, shape, scale, cutout):
    """Steps 3-5 for world points [4,n]: kept points' (u_int, v_int, d, u * scale, v * scale)."""
    size, _, _ = geometry(shape, scale, cutout)
    q = _apply(camera_transform @ np.linalg.inv(pose @ SWAPAXES_), world)
    x, y, z, _ = _apply(np.asarray(G, np.float64), q)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = focal_length[0] * x / z + principal_point[0]
        v = focal_length[1] * y / z + principal_point[1]
        keep = (z > 0) & (0.5 <= u) & (u <= size[1]) & (0.5 <= v) & (v <= size[0])
    us, vs = u[keep] * scale, v[keep] * scale
    return us.astype(np.int64), vs.astype(np.int64), 1 / z[keep], us, vs


def lidar_depth(image_timestamp, pose, scan_timestamps, scans, lidar_poses, lidar_transform, camera_transform, G,
                focal_length, principal_point, shape, scale=0.25, cutout=(1 / 6, 1 / 6, 0, 0), lidar_timestamp_range=0.5):
    """[1, h', w'] float32 inverse depth of one key frame; IndexError as the loader raises it."""
    T = image_timestamp
    sel = [i for i, t in enumerate(scan_timestamps)
           if T - lidar_timestamp_range * 1e6 <= t <= T + lidar_timestamp_range * 1e6]
    world = np.zeros((4, 0))
    for i in sel:
        world = np.hstack([world, world_points(scans[i], lidar_poses[i], lidar_transform)])
    iu, iv, d, _, _ = project(world, pose, camera_transform, G, focal_length, principal_point, shape, scale, cutout)
    _, (Hd, Wd), (r0, r1, c0, c1) = geometry(shape, scale, cutout)
    if ((iu < 0) | (iu >= Wd) | (iv < 0) | (iv >= Hd)).any():
        raise IndexError(f"a projected point falls outside the {Hd}x{Wd} depth array")
    depth = np.zeros((Hd, Wd))
    np.maximum.at(depth, (iv, iu), d)
    return depth[None, r0:r1, c0:c1].astype(np.float32)
