#!/usr/bin/env python
"""Writes tests/golden/eval_edges.npz by calling the UNMODIFIED reference on CPU fp32:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_eval_edges.py

The IEEE and slicing edges of what evaluate.py logs and create_pointcloud.py writes.  Stored (inputs in fp32, the reference's
outputs as it returns them):
  pred, gt, mvobj          [5,1,24,40] inputs of the seven sparse metrics (model/metric_functions/sparse_metrics.py:81-251).
                           Image 0: NaN, +inf, negative, +0.0 and -0.0 predictions; image 1: NaN, +inf and negative targets;
                           image 2: NaN predictions only where target == 0 (masked: they must not show); image 3: NaN in
                           mvobj; image 4: a NaN prediction in row 0 (outside the negative roi) where mvobj is NaN
  sparse_<tag>             float64 [4,7]: a1 ... sq_rel of images [0:5], [0:2], [2:4], [4:5] (the whole batch, then the rows of
                           group = 2 with a ragged last group) for the parameter set SPARSE_CASES[tag] (tests/eval_edges_cases.py), called as the evaluater
                           calls them: metric(data_dict, roi, max_distance) under the plain / _onlyvalid / _onlydynamic names
  pc_inv_depth, pc_image, pc_K, pc_pose
                           [2,1,32,48], [2,3,32,48], [2,4,4], [2,4,4] inputs of utils/ply_utils.py PLYSaver.add_depthmap
                           (min_d PC_MIN_D, max_d PC_MAX_D): inverse depths whose depth is exactly min_d or max_d and their fp32
                           neighbours on either side, 0, -0.0, negative, NaN and +-inf
  pc_vertices_<tag>        [N,6] the vertices add_depthmap collects for roi PC_ROIS[tag] (python slices: negative bounds count
                           from the end, bounds past the edge are clipped, `empty` keeps nothing)
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)
from tests.eval_edges_cases import NAMES, PC_MAX_D, PC_MIN_D, PC_ROIS, SLICES, SPARSE_CASES  # noqa: E402


def sparse_inputs():
    g = torch.Generator().manual_seed(41)
    B, H, W = 5, 24, 40
    pred = torch.rand(B, 1, H, W, generator=g) * 0.3 + 0.01
    gt = (pred * (1 + 0.25 * torch.randn(B, 1, H, W, generator=g))).clamp_min(1e-3)   # some below 1 / 80: masked at 80 m
    gt[torch.rand(B, 1, H, W, generator=g) > 0.4] = 0.0                              # sparse ground truth
    mvobj = (torch.rand(B, 1, H, W, generator=g) > 0.2).to(torch.float32)
    # the special values sit at unmasked pixels (gt > 1 / 50, mvobj 1) inside every roi, except where stated
    p, t, m = pred[:, 0], gt[:, 0], mvobj[:, 0]
    spots = [(8, 10), (9, 20), (12, 15), (15, 30), (18, 6), (6, 25)]
    for b in (0, 1):
        for y, x in spots:
            t[b, y, x], m[b, y, x] = 0.1, 1.0
    p[0, 8, 10] = float("nan")
    p[0, 9, 20] = float("inf")
    p[0, 12, 15] = -0.05
    p[0, 15, 30] = -0.0
    p[0, 18, 6] = 0.0
    t[1, 8, 10] = float("nan")
    t[1, 9, 20] = float("inf")
    t[1, 12, 15] = -0.05                                                             # masked at 80 m, not without
    hole = (t[2] == 0).nonzero()
    for y, x in hole[torch.randperm(hole.shape[0], generator=g)[:6]].tolist():
        p[2, y, x] = float("nan")
    m[3, 5:9, 5:9] = float("nan")
    p[4, 0, 20], t[4, 0, 20], m[4, 0, 20] = float("nan"), 0.1, float("nan")
    return pred, gt, mvobj


def exact_inverse(d):
    """fp32 x with fp32(1 / x) == d."""
    x = torch.tensor(1.0 / d, dtype=torch.float32)
    for _ in range(4):
        if float(1 / x) == d:
            return x
        x = torch.nextafter(x, torch.tensor(0.0 if float(1 / x) < d else 1.0))
    raise AssertionError(f"no fp32 inverse depth of {d}")


def pc_inputs():
    g = torch.Generator().manual_seed(42)
    B, H, W = 2, 32, 48
    inv = torch.rand(B, 1, H, W, generator=g) * 0.3 + 0.03                           # depths 3 .. 30 m
    edges = []
    for d in (PC_MIN_D, PC_MAX_D):
        x = exact_inverse(d)
        edges += [x, torch.nextafter(x, torch.tensor(0.0)), torch.nextafter(x, torch.tensor(1.0))]
    edges += [torch.tensor(v) for v in (0.0, -0.0, -0.1, float("nan"), float("inf"), float("-inf"))]
    idx = torch.randperm(B * H * W, generator=g)[:4 * len(edges)]
    flat = inv.view(-1)
    for k, i in enumerate(idx.tolist()):
        flat[i] = edges[k % len(edges)]
    image = torch.rand(B, 3, H, W, generator=g) - 0.5
    K = torch.eye(4).repeat(B, 1, 1)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] = 41.0, 40.5, 23.5, 15.5
    pose = torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        a = 0.3 * (b + 1)
        c, s = float(np.cos(a)), float(np.sin(a))
        pose[b, :3, :3] = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
        pose[b, :3, 3] = torch.rand(3, generator=g) * 4 - 2
    return inv, image, K, pose


def main():
    torch.manual_seed(0)
    import_reference()
    import model.metric_functions.sparse_metrics as SM  # noqa
    from utils.ply_utils import PLYSaver  # noqa
    pred, gt, mvobj = sparse_inputs()
    out = {"pred": pred.numpy(), "gt": gt.numpy(), "mvobj": mvobj.numpy()}
    for tag, (suffix, roi, md) in SPARSE_CASES.items():
        rows = []
        for lo, hi in SLICES:
            d = {"result": pred[lo:hi].clone(), "target": gt[lo:hi].clone(), "mvobj_mask": mvobj[lo:hi].clone()}
            rows.append([float(getattr(SM, f"{n}_sparse{suffix}_metric")(d, roi, md)) for n in NAMES])
        out[f"sparse_{tag}"] = np.array(rows, dtype=np.float64)
        print(tag, np.array2string(out[f"sparse_{tag}"], precision=4))
    inv, image, K, pose = pc_inputs()
    B, _, H, W = inv.shape
    out.update(pc_inv_depth=inv.numpy(), pc_image=image.numpy(), pc_K=K.numpy(), pc_pose=pose.numpy())
    for tag, roi in PC_ROIS.items():
        saver = PLYSaver(H, W, min_d=PC_MIN_D, max_d=PC_MAX_D, batch_size=B, roi=roi, dropout=0)
        saver.add_depthmap(inv.clone(), image.clone(), K.clone(), pose.clone())
        out[f"pc_vertices_{tag}"] = np.array(saver.data, dtype=np.float32).reshape(-1, 6)
        print("point cloud", tag, out[f"pc_vertices_{tag}"].shape[0], "vertices")
    path = HERE / "eval_edges.npz"
    np.savez_compressed(path, **out)
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
