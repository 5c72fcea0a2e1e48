"""Oxford RobotCar's lidar depth targets on the CPU: the float64 oracle (oracle/robotcar_depth_oracle.py) against the
unmodified loader's `get_depth` (tests/golden/robotcar_depth.npz), the loader's sizes, and the C entries' argument checks,
which run before any CUDA call."""
import ctypes
from pathlib import Path

import numpy as np
import pytest

from oracle import robotcar_depth_oracle as O

GOLDEN = Path(__file__).resolve().parent / "golden" / "robotcar_depth.npz"


def load_cases():
    """{name: case dict} of the golden file, scans split into a list of [n,3] arrays."""
    z = np.load(GOLDEN)
    cases = {}
    for name in z["cases"].tolist():
        c = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
        off = c["scan_offsets"]
        c["scans"] = [c["scan_points"][off[i]:off[i + 1]] for i in range(len(off) - 1)]
        c["shape"] = tuple(int(v) for v in c["shape"])
        c["cutout"] = tuple(float(v) for v in c["cutout"])
        c["scale"], c["range"] = float(c["scale"]), float(c["range"])
        cases[name] = c
    return cases


CASES = load_cases()


def oracle_depth(c, k):
    return O.lidar_depth(int(c["image_t"][k]), c["poses"][k], c["scan_t"].tolist(), c["scans"], c["lidar_poses"],
                         c["lidar_transform"], c["camera_transform"], c["G"], c["focal"], c["principal"], c["shape"],
                         c["scale"], c["cutout"], c["range"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_the_loader_bit_for_bit(name):
    c = CASES[name]
    for j, k in enumerate(c["keys"].tolist()):
        if c["error"][j]:
            with pytest.raises(IndexError):
                oracle_depth(c, k)
            continue
        out = oracle_depth(c, k)
        assert out.dtype == np.float32 and out.shape == c["depth"][j].shape
        assert np.array_equal(out.view(np.uint32), c["depth"][j].view(np.uint32)), (name, k)


def test_golden_covers_the_cases_the_loader_distinguishes():
    over = CASES["overlap"]
    T, r = int(over["image_t"][2]), int(over["range"] * 1e6)
    st = set(over["scan_t"].tolist())
    assert {T - r, T + r, T - r - 1, T + r + 1} <= st                        # on each bound and just outside
    assert 0 in np.diff(over["scan_offsets"])                                # an empty scan
    keys = over["keys"].tolist()
    assert all(b - a == 1 for a, b in zip(keys, keys[1:]))                   # consecutive key frames, overlapping windows
    assert CASES["half_nocut"]["scale"] == 0.5 and CASES["half_nocut"]["cutout"] == (0, 0, 0, 0)
    assert CASES["rounded"]["depth"].shape[-2:] != CASES["rounded"]["shape"]
    assert not CASES["empty"]["depth"].any() and CASES["index_error"]["error"].all()
    for name, c in CASES.items():
        if not c["error"].any() and name != "empty":
            assert (c["depth"] > 0).sum() > 300, name


def test_several_points_on_one_pixel_keep_the_nearest():
    """The golden's pixels that receive several points hold the largest inverse depth among them."""
    c, k = CASES["overlap"], 2
    world = np.hstack([O.world_points(s, c["lidar_poses"][i], c["lidar_transform"]) for i, s in enumerate(c["scans"])
                       if abs(int(c["scan_t"][i]) - int(c["image_t"][k])) <= c["range"] * 1e6])
    iu, iv, d, _, _ = O.project(world, c["poses"][k], c["camera_transform"], c["G"], c["focal"], c["principal"],
                                c["shape"], c["scale"], c["cutout"])
    _, _, (r0, r1, c0, c1) = O.geometry(c["shape"], c["scale"], c["cutout"])
    inside = (iv >= r0) & (iv < r1) & (iu >= c0) & (iu < c1)
    pix = (iv[inside] - r0) * (c1 - c0) + (iu[inside] - c0)
    vals, counts = np.unique(pix, return_counts=True)
    shared = vals[counts > 2]
    assert shared.size > 10
    depth = c["depth"][list(c["keys"]).index(k), 0].ravel()
    for p in shared[:50]:
        assert depth[p] == np.float32(d[inside][pix == p].max())


def test_target_geometry_is_the_loaders():
    from monorec_b200.robotcar import target_geometry
    for name, c in CASES.items():
        size, hw, crop = target_geometry(c["shape"], c["scale"], c["cutout"])
        assert (size, hw, crop) == O.geometry(c["shape"], c["scale"], c["cutout"])
        if not c["error"].any():
            assert c["depth"].shape[-2:] == (crop[1] - crop[0], crop[3] - crop[2])
    for bad in (dict(shape=(0, 4)), dict(scale=0.0), dict(scale=float("nan")), dict(cutout=(0.5, 0.5, 0, 0)),
                dict(cutout=(-0.1, 0, 0, 0))):
        kw = {**dict(shape=(32, 64), scale=0.25, cutout=(1 / 6, 1 / 6, 0, 0)), **bad}
        with pytest.raises(ValueError):
            target_geometry(kw["shape"], kw["scale"], kw["cutout"])


def test_entries_check_their_arguments_before_any_cuda_call():
    from monorec_b200 import _lib
    lib = _lib.load()
    d = lambda *v: (ctypes.c_double * len(v))(*v)                                     # noqa: E731
    ll = lambda *v: (ctypes.c_longlong * len(v))(*v)                                  # noqa: E731
    eye = d(*np.eye(4).ravel())
    fake = ctypes.c_void_p(1 << 20)                                                   # never dereferenced
    proj = d(20.0, 20.0, 16.0, 12.0, 0.5, 32.0, 24.0, 0.25)
    crop = (ctypes.c_int * 4)(0, 6, 0, 8)

    def depth(**kw):
        a = dict(ring=fake, capacity=100, K=1, first=ll(0), count=ll(10), cam=eye, G=eye, proj=proj, Hd=6, Wd=8, crop=crop,
                 out=fake, oob=fake)
        a.update(kw)
        return lib.mr_lidar_depth(*a.values(), None)

    for kw, text in ((dict(ring=None), b"null pointer"), (dict(capacity=0), b"capacity"), (dict(K=0), b"key-frame count"),
                     (dict(count=ll(101)), b"count"), (dict(first=ll(100)), b"first row"),
                     (dict(crop=(ctypes.c_int * 4)(0, 7, 0, 8)), b"crop"), (dict(crop=(ctypes.c_int * 4)(3, 3, 0, 8)), b"crop"),
                     (dict(proj=d(20.0, 20.0, 16.0, 12.0, 0.5, 32.0, 24.0, 0.0)), b"scale"),
                     (dict(G=d(*([float("nan")] + [0.0] * 15))), b"G[0]"),
                     (dict(cam=d(*([0.0] * 15 + [float("inf")]))), b"camera matrix"),
                     (dict(ring=ctypes.c_void_p((1 << 20) + 8)), b"aligned")):
        assert depth(**kw) == -1, kw
        assert text in lib.mr_last_error(), (kw, lib.mr_last_error())
    for args, text in (((fake, 5, None, fake, 10, 0), b"null pointer"), ((fake, 11, eye, fake, 10, 0), b"point count"),
                       ((fake, 5, eye, fake, 10, 10), b"first row"), ((fake, 5, eye, fake, 0, 0), b"capacity"),
                       ((fake, 5, d(*([float("nan")] * 16)), fake, 10, 0), b"not finite")):
        assert lib.mr_lidar_to_world(*args, None) == -1, args
        assert text in lib.mr_last_error()
