#!/usr/bin/env python
"""Writes tests/golden/loader_streams.json by running the UNMODIFIED reference KITTI, TUM Mono-VO and Oxford RobotCar
loaders on CPU:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_loader_streams.py

Each loader is built on a tiny synthetic tree in a temporary directory, and every item of the dataset is read
(`__getitem__`).  Every frame's pose holds the frame's own sequence index as its x translation, so an item records its key
frame (`keyframe_pose`) and its source frames (`poses`, in the loader's list order) exactly, including the frames a
negative index wraps to; the pose lists note a negative index, and such an item is marked `wrapped`.  An item whose read
raises IndexError (a source frame past the end of the sequence) is recorded as such.

  * KITTI (`KittiOdometryDataset`): the stubs of make_golden_loader_keys.py (`pykitti`, `skimage`, the numpy 2 aliases),
    with dense `.npy` depth maps.  offset_d -2, -1 and 1, frame_count 2 and 3, dilation 1 and 2, max_length None and 6,
    use_index_mask None and one mask, over two sequences.
  * TUM Mono-VO (`TUMMonoVODataset`): a tree with images/, result.txt, times.txt, pcalib.txt and camera.txt; a stub `cv2`
    reads the images_depth/*.exr files (their names are what `only_keyframes` reads).  only_keyframes on and off,
    frame_count 2 and 3, dilation 1 and 2, max_length None and 5.
  * Oxford RobotCar (`OxfordRobotCarDataset`): the loader's own helpers (camera model, image loading, VO pose
    interpolation, SE(3) from extrinsics) come from its `oxford_robotcar` SDK package, which is not part of the reference;
    stubs of them are put into the loaded module's namespace, and a stub `skimage` resizes.  frame_count 2, 3 and 4,
    dilation 1 and 2, over two sequences, without lidar scans.

Stored (JSON): per loader its sequence lengths (and KITTI's masks, TUM's depth-map frames) and `cases`: the loader
arguments and `items`, one per dataset item in order: {"sequence", "key", "sources", "wrapped"} or
{"error": "IndexError"}.
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

KITTI_LENGTHS = {"00": 19, "04": 13}
TUM_LENGTH = 15
TUM_DEPTH = [0, 1, 3, 5, 6, 9, 11, 12, 13, 14]      # the frames with an images_depth/*.exr
ROBOTCAR_LENGTHS = [12, 9]


class _Poses(list):
    """A pose list that notes a read at a negative index (which Python wraps to the end)."""
    wrapped = False

    def __getitem__(self, i):
        if isinstance(i, int) and i < 0:
            _Poses.wrapped = True
        return super().__getitem__(i)


def _index(pose):
    return int(round(float(np.asarray(pose)[0, 3])))


def _read(ds, sequence_of):
    items = []
    for i in range(len(ds)):
        _Poses.wrapped = False
        try:
            d = ds[i][0]
        except IndexError:
            items.append({"error": "IndexError"})
            continue
        items.append({"sequence": sequence_of(d), "key": _index(d["keyframe_pose"]),
                      "sources": [_index(p) for p in d["poses"]], "wrapped": _Poses.wrapped})
    return items


# ---- KITTI ---------------------------------------------------------------------------------------------------------------
class _Calib:
    def __init__(self):
        self.P_rect_00 = self.P_rect_20 = np.array([[20.0, 0, 16, 0], [0, 20.0, 8, 0], [0, 0, 1, 0]])
        self.b_gray = self.b_rgb = 0.54


class _Odometry:
    """The part of pykitti.odometry the loader uses; frame i's pose has x translation i."""

    def __init__(self, base, sequence):
        n = KITTI_LENGTHS[sequence]
        self.cam0_files = self.cam2_files = [f"{i:06d}.png" for i in range(n)]
        self.calib = _Calib()
        self.poses = _Poses(np.eye(4) for _ in range(n))
        for i, p in enumerate(self.poses):
            p[0, 3] = i

    def _image(self, i):
        self.cam2_files[i]                             # pykitti reads the i-th file: IndexError past the end
        return Image.fromarray(np.full((16, 32, 3), i % 255, np.uint8))

    @property
    def cam2(self):
        return iter([self._image(0)])

    cam0 = cam2

    def get_cam2(self, i):
        return self._image(i)

    get_cam0 = get_cam1 = get_cam3 = get_cam2


def _kitti_masks():
    g = np.random.default_rng(23)
    return {"mask_a": {s: {str(i): bool(g.random() < 0.75) for i in range(n) if g.random() < 0.9}
                       for s, n in KITTI_LENGTHS.items()}}


def _kitti(root):
    from data_loader.kitti_odometry_dataset import KittiOdometryDataset  # noqa
    masks = _kitti_masks()
    for s, n in KITTI_LENGTHS.items():
        d = root / "kitti" / "sequences" / s
        (d / "dense").mkdir(parents=True)
        for i in range(n):
            np.save(d / "dense" / f"{i:06d}.npy", np.full((16, 32), 5.0 + i))
        for name, m in masks.items():
            (d / f"{name}.json").write_text(json.dumps(m[s]))
    cases = []
    for offset_d in (-2, -1, 1):
        for fc in (2, 3):
            for dil in (1, 2):
                for max_length in (None, 6):
                    for index_mask in (None, ["mask_a"]):
                        args = dict(offset_d=offset_d, frame_count=fc, dilation=dil, max_length=max_length,
                                    use_index_mask=index_mask)
                        ds = KittiOdometryDataset(str(root / "kitti"), sequences=list(KITTI_LENGTHS), target_image_size=(8, 16),
                                                  depth_folder="dense", lidar_depth=False, dso_depth=False,
                                                  **dict(args, use_index_mask=None if index_mask is None else tuple(index_mask)))
                        args["items"] = _read(ds, lambda d: f"{int(d['sequence']):02d}")
                        cases.append(args)
    return {"lengths": KITTI_LENGTHS, "masks": masks, "cases": cases}


# ---- TUM Mono-VO -----------------------------------------------------------------------------------------------------------
def _tum(root):
    cv2 = types.ModuleType("cv2")
    cv2.IMREAD_ANYCOLOR, cv2.IMREAD_ANYDEPTH = 4, 2
    cv2.imread = lambda path, flags=0: np.full((16, 20), 3.0, np.float32)
    sys.modules["cv2"] = cv2
    from data_loader.tum_mono_vo_dataset import TUMMonoVODataset  # noqa
    d = root / "tum"
    (d / "images").mkdir(parents=True)
    (d / "images_depth").mkdir()
    for i in range(TUM_LENGTH):
        Image.fromarray(np.full((16, 20), 10 * i % 255, np.uint8)).save(d / "images" / f"{i:05d}.jpg")
    for i in TUM_DEPTH:
        (d / "images_depth" / f"{i:05d}_d.exr").write_bytes(b"")
    # result.txt: timestamp, translation (x = the frame's index), quaternion (x, y, z, w); times.txt: id, timestamp, exposure
    np.savetxt(d / "result.txt", [[0.1 * i, i, 0, 0, 0, 0, 0, 1] for i in range(TUM_LENGTH)])
    np.savetxt(d / "times.txt", [[i, 0.1 * i, 1.0] for i in range(TUM_LENGTH)])
    np.savetxt(d / "pcalib.txt", np.arange(256.0)[None])
    (d / "camera.txt").write_text("0.5 0.6 0.5 0.5 0\n20 16\ncrop\n20 16\n")
    cases = []
    for only_keyframes in (False, True):
        for fc in (2, 3):
            for dil in (1, 2):
                for max_length in (None, 5):
                    args = dict(only_keyframes=only_keyframes, frame_count=fc, dilation=dil, max_length=max_length)
                    ds = TUMMonoVODataset(str(d), target_image_size=(8, 16), color_augmentation=False, **args)
                    args["items"] = _read(ds, lambda _: 0)
                    cases.append(args)
    return {"length": TUM_LENGTH, "depth_frames": TUM_DEPTH, "cases": cases}


# ---- Oxford RobotCar -------------------------------------------------------------------------------------------------------
class _CameraModel:
    camera = "stereo"
    focal_length = (20.0, 20.0)
    principal_point = (16.0, 12.0)

    def __init__(self, model_folder, sequence_folder):
        pass

    def project(self, points, size):
        return np.zeros((2, 1)), np.ones(1)


def _robotcar(root):
    import data_loader.oxford_robotcar_dataset as R  # noqa
    R.CameraModel = _CameraModel
    R.load_image = lambda path, model: np.full((24, 32, 3), 2.0 * int(Path(path).stem) % 256)
    # the pose of every listed timestamp (frame i: x translation i); the lidar folders hold no scans

    def interpolate_vo_poses(pose_file, timestamps, origin):
        poses = []
        for t in timestamps:
            p = np.eye(4)
            p[0, 3] = int(t) - 1000
            poses.append(p)
        return poses
    R.interpolate_vo_poses = interpolate_vo_poses
    R.build_se3_transform = lambda xyzrpy: np.eye(4)
    ext = root / "robotcar" / "extrinsics"
    ext.mkdir(parents=True)
    for name in ("ldmrs", _CameraModel.camera):
        (ext / f"{name}.txt").write_text("0 0 0 0 0 0\n")
    seqs, lidar = [], []
    for s, n in enumerate(ROBOTCAR_LENGTHS):
        f = root / "robotcar" / f"seq{s}"
        (f / "stereo").mkdir(parents=True)
        (f / "ldmrs").mkdir()
        for i in range(n):
            (f / "stereo" / f"{1000 + i}.png").write_bytes(b"")
        seqs.append(str(f / "stereo"))
        lidar.append(str(f / "ldmrs"))
    cases = []
    for fc in (2, 3, 4):
        for dil in (1, 2):
            ds = R.OxfordRobotCarDataset(seqs, [""] * len(seqs), lidar, str(root), str(ext), frame_count=fc, dilation=dil)
            ds._sequence_poses = [_Poses(p) for p in ds._sequence_poses]
            cases.append(dict(frame_count=fc, dilation=dil, items=_read(ds, lambda d: int(d["sequence"]))))
    return {"lengths": ROBOTCAR_LENGTHS, "cases": cases}


def _stubs():
    pykitti = types.ModuleType("pykitti")
    pykitti.odometry = _Odometry
    sys.modules["pykitti"] = pykitti
    skimage = types.ModuleType("skimage")
    transform = types.ModuleType("skimage.transform")

    def resize(a, output_shape, order=0):
        size = [int(v) for v in output_shape]
        rows = (np.arange(size[0]) * a.shape[0]) // size[0]
        cols = (np.arange(size[1]) * a.shape[1]) // size[1]
        return a[rows][:, cols]
    transform.resize = resize
    skimage.transform = transform
    sys.modules["skimage"], sys.modules["skimage.transform"] = skimage, transform
    np.float, np.int = float, int


def main():
    import_reference()
    _stubs()
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        out = {"kitti": _kitti(root), "tum_mono_vo": _tum(root), "robotcar": _robotcar(root)}
    for name, v in out.items():
        print(name, len(v["cases"]), "cases", sum(len(c["items"]) for c in v["cases"]), "items")
    path = HERE / "loader_streams.json"
    path.write_text(json.dumps(out, separators=(",", ":")) + "\n")
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
