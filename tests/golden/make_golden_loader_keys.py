#!/usr/bin/env python
"""Writes tests/golden/loader_keys.json by running the UNMODIFIED reference KITTI loader on CPU:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_loader_keys.py

`KittiOdometryDataset` (data_loader/kitti_odometry_dataset.py) is built on a small synthetic KITTI tree in a temporary
directory: a stub `pykitti` module serves the frames, poses and calibration of each sequence, a stub `skimage` the
nearest-neighbour resize of the dense depth maps, and the annotated-lidar depth maps and dense `.npy` depth maps are written
as tiny files.  numpy 2 dropped the `np.float` / `np.int` aliases the loader's depth code uses; they are restored as the
builtins.  Every item of the dataset is read (`__getitem__`), and its `image_id` and `sequence` recorded.

Cases: frame_count 2 and 4, dilation 1 and 2, lidar on (annotated, so offset 5 / extra_frames 10) and off (dense depth
maps), and use_index_mask None, (), one mask and two masks, over two sequences of unequal length.  The masks are JSON files
in the sequence folders, as the loader reads them; their contents are stored with the results.

Stored (JSON): lengths, masks (name -> per-sequence dict), and cases: a list of the loader arguments with `image_id` and
`sequence`, one entry per item in the dataset's order.
"""
import json
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
from PIL import Image

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)

LENGTHS = {"00": 23, "04": 17}
FRAME = (16, 32)                      # raw frame height, width
TARGET = (8, 16)                      # the loader's target_image_size


def _masks():
    """Two index masks per sequence: listed frames true or false, some frames not listed at all."""
    g = np.random.default_rng(17)
    out = {}
    for name, p_list, p_true in (("mask_a", 0.9, 0.7), ("mask_b", 0.8, 0.8)):
        out[name] = {s: {str(i): bool(g.random() < p_true) for i in range(n) if g.random() < p_list}
                     for s, n in LENGTHS.items()}
    return out


class _Calib:
    def __init__(self):
        self.P_rect_00 = self.P_rect_20 = np.array([[20.0, 0, 16, 0], [0, 20.0, 8, 0], [0, 0, 1, 0]])
        self.b_gray = self.b_rgb = 0.54


class _Odometry:
    """The part of pykitti.odometry the loader uses."""

    def __init__(self, base, sequence):
        n = LENGTHS[sequence]
        self.cam0_files = self.cam2_files = [f"{i:06d}.png" for i in range(n)]
        self.calib = _Calib()
        self.poses = [np.eye(4) for _ in range(n)]
        for i, p in enumerate(self.poses):
            p[2, 3] = 0.8 * i

    def _image(self, i):
        return Image.fromarray(np.full(FRAME + (3,), i % 255, np.uint8))

    @property
    def cam2(self):
        return iter([self._image(0)])

    cam0 = cam2

    def get_cam2(self, i):
        return self._image(i)

    get_cam0 = get_cam1 = get_cam3 = get_cam2


def _stubs():
    pykitti = types.ModuleType("pykitti")
    pykitti.odometry = _Odometry
    sys.modules["pykitti"] = pykitti
    skimage = types.ModuleType("skimage")
    transform = types.ModuleType("skimage.transform")

    def resize(a, size, order=0):
        rows = (np.arange(size[0]) * a.shape[0]) // size[0]
        cols = (np.arange(size[1]) * a.shape[1]) // size[1]
        return a[rows][:, cols]
    transform.resize = resize
    skimage.transform = transform
    sys.modules["skimage"], sys.modules["skimage.transform"] = skimage, transform
    np.float, np.int = float, int


def _tree(root, masks):
    for s, n in LENGTHS.items():
        d = root / "sequences" / s
        (d / "lidar").mkdir(parents=True)
        (d / "dense").mkdir()
        for i in range(n):
            depth = np.zeros(FRAME, np.uint16)
            depth[::3, ::4] = 256 * (5 + i)
            Image.fromarray(depth).save(d / "lidar" / f"{i:06d}.png")
            np.save(d / "dense" / f"{i:06d}.npy", np.full(FRAME, 5.0 + i))
        for name, m in masks.items():
            (d / f"{name}.json").write_text(json.dumps(m[s]))


def main():
    import_reference()
    _stubs()
    from data_loader.kitti_odometry_dataset import KittiOdometryDataset  # noqa
    masks = _masks()
    cases = []
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        _tree(root, masks)
        for fc in (2, 4):
            for dil in (1, 2):
                for lidar in (True, False):
                    for index_mask in (None, [], ["mask_a"], ["mask_a", "mask_b"]):
                        args = dict(frame_count=fc, dilation=dil, lidar_depth=lidar, annotated_lidar=True,
                                    use_index_mask=index_mask)
                        ds = KittiOdometryDataset(str(root), sequences=list(LENGTHS), target_image_size=TARGET,
                                                  depth_folder="lidar" if lidar else "dense", dso_depth=False,
                                                  **{k: (tuple(v) if k == "use_index_mask" and v is not None else v)
                                                     for k, v in args.items()})
                        items = [ds[i][0] for i in range(len(ds))]
                        args.update(image_id=[int(d["image_id"]) for d in items],
                                    sequence=[f"{int(d['sequence']):02d}" for d in items])
                        cases.append(args)
                        print(fc, dil, lidar, index_mask, len(items))
    path = HERE / "loader_keys.json"
    path.write_text(json.dumps({"lengths": LENGTHS, "masks": masks, "cases": cases}, separators=(",", ":")) + "\n")
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
