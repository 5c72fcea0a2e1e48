"""Oxford RobotCar's lidar depth targets on the GPU (monorec_b200.robotcar, csrc/lidar_depth.cu): bit for bit the unmodified
loader's `get_depth` (tests/golden/robotcar_depth.npz) and the float64 oracle, independent of the order of the points and
scans, a batch equal to single calls, the stream form (`RobotCarLidar`, with ring growth and eviction) equal to `lidar_depth`
without host synchronisation in `targets`, and a RobotCar stream evaluated with `SequenceEvaluater` on device targets equal
to the same evaluation on the loader's targets."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import robotcar_depth_oracle as O
from tests.test_robotcar_depth import CASES, oracle_depth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _camera(c):
    return SimpleNamespace(G_camera_image=c["G"], focal_length=tuple(c["focal"]), principal_point=tuple(c["principal"]))


def _kw(c):
    return dict(camera=_camera(c), camera_transform=c["camera_transform"], lidar_transform=c["lidar_transform"],
                shape=c["shape"], scale=c["scale"], cutout=c["cutout"], lidar_timestamp_range=c["range"], device=DEV)


def _device_depth(c, k, scan_t=None, scans=None, lidar_poses=None):
    from monorec_b200.robotcar import lidar_depth
    return lidar_depth(int(c["image_t"][k]), c["poses"][k], c["scan_t"].tolist() if scan_t is None else scan_t,
                       c["scans"] if scans is None else scans, c["lidar_poses"] if lidar_poses is None else lidar_poses,
                       **_kw(c))


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("name", sorted(CASES))
def test_equals_the_loader_bit_for_bit(name):
    c = CASES[name]
    for j, k in enumerate(c["keys"].tolist()):
        if c["error"][j]:
            with pytest.raises(IndexError):
                _device_depth(c, k)
            continue
        out = _device_depth(c, k)
        assert out.dtype == torch.float32 and out.device == torch.device(DEV) and tuple(out.shape) == c["depth"][j].shape
        assert np.array_equal(_bits(out), c["depth"][j].view(np.uint32)), (name, k)


def _random_scene(c, seed, n_scans=12):
    """Random scans around the case's key frame 2 (points anywhere in a box ahead of the vehicle, some behind it)."""
    g = np.random.default_rng(seed)
    T = int(c["image_t"][2])
    scan_t = sorted(set((T + g.integers(-700_000, 700_000, n_scans)).tolist()))
    scans = [g.normal([15.0, 0.0, 0.0], [12.0, 8.0, 3.0], (int(g.integers(0, 3000)), 3)) for _ in scan_t]
    poses = [c["lidar_poses"][i % len(c["lidar_poses"])] for i in range(len(scan_t))]
    return scan_t, scans, poses


@pytest.mark.parametrize("name", ["overlap", "half_nocut", "rounded"])
def test_equals_the_oracle_on_random_scenes_and_ignores_point_and_scan_order(name):
    c = CASES[name]
    g = np.random.default_rng(5)
    for seed in range(3):
        scan_t, scans, poses = _random_scene(c, seed)
        try:
            ref = O.lidar_depth(int(c["image_t"][2]), c["poses"][2], scan_t, scans, poses, c["lidar_transform"],
                                c["camera_transform"], c["G"], c["focal"], c["principal"], c["shape"], c["scale"],
                                c["cutout"], c["range"])
        except IndexError:
            with pytest.raises(IndexError):
                _device_depth(c, 2, scan_t, scans, poses)
            continue
        assert (ref > 0).sum() > 100
        out = _device_depth(c, 2, scan_t, scans, poses)
        assert np.array_equal(_bits(out), ref.view(np.uint32)), (name, seed)
        order = g.permutation(len(scan_t))
        shuffled = [scans[i][g.permutation(len(scans[i]))] for i in order]
        again = _device_depth(c, 2, [scan_t[i] for i in order], shuffled, [poses[i] for i in order])
        assert torch.equal(again, out)


def _many_keys(c, K):
    """K increasing image timestamps across the case's scans, each with one of the case's poses."""
    t = np.linspace(int(c["scan_t"][0]), int(c["scan_t"][-1]), K).astype(np.int64).tolist()
    return t, [c["poses"][i % len(c["poses"])] for i in range(K)]


def test_a_batch_equals_single_calls():
    """K = 37 key frames (three launches) in one targets call against one lidar_depth call per key frame."""
    from monorec_b200.robotcar import RobotCarLidar, lidar_depth
    c = CASES["overlap"]
    ts, poses = _many_keys(c, 37)
    ring = RobotCarLidar(**_kw(c))
    for t, s, p in zip(c["scan_t"].tolist(), c["scans"], c["lidar_poses"]):
        ring.add_scan(t, s, p)
    batch = ring.targets(ts, poses)
    ring.check()
    kw = _kw(c)
    for k, (t, p) in enumerate(zip(ts, poses)):
        one = lidar_depth(t, p, c["scan_t"].tolist(), c["scans"], c["lidar_poses"], **kw)
        assert torch.equal(batch[k], one), k
    assert (batch > 0).sum() > 1000


def test_ring_equals_lidar_depth_without_host_synchronisation():
    """A stream: scans added as they arrive (device and host arrays), targets in batches of 3 as soon as a key frame's
    window is complete, a ring of 64 rows that grows, and evicted scans; every target equals lidar_depth's, and targets
    makes no host synchronisation after the first call."""
    from monorec_b200.robotcar import RobotCarLidar, lidar_depth
    c = CASES["overlap"]
    ts, poses = _many_keys(c, 14)
    r = c["range"] * 1e6
    ring = RobotCarLidar(**_kw(c), capacity=64)
    scans = list(zip(c["scan_t"].tolist(), c["scans"], c["lidar_poses"]))
    got, i = [], 0
    for j in range(0, len(ts), 3):
        batch_t, batch_p = ts[j:j + 3], poses[j:j + 3]
        while i < len(scans) and scans[i][0] <= batch_t[-1] + r:
            t, s, p = scans[i]
            ring.add_scan(t, torch.from_numpy(s).to(DEV) if i % 2 else s, p)
            i += 1
        if j:
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
        try:
            got.append(ring.targets(batch_t, batch_p))
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert len(ring._times) <= len(scans) and (not ring._times or ring._times[0] >= batch_t[-1] - r)
    ring.check()
    assert ring.capacity > 64
    got = torch.cat(got)
    kw = _kw(c)
    for k, (t, p) in enumerate(zip(ts, poses)):
        assert torch.equal(got[k], lidar_depth(t, p, c["scan_t"].tolist(), c["scans"], c["lidar_poses"], **kw)), k


def test_ring_raises_index_error_later_and_refuses_decreasing_timestamps():
    from monorec_b200.robotcar import RobotCarLidar
    c = CASES["index_error"]
    ring = RobotCarLidar(**_kw(c))
    for t, s, p in zip(c["scan_t"].tolist(), c["scans"], c["lidar_poses"]):
        ring.add_scan(t, s, p)
    with pytest.raises(ValueError):
        ring.add_scan(int(c["scan_t"][-1]), c["scans"][0], c["lidar_poses"][0])
    k = int(c["keys"][0])
    ring.targets([int(c["image_t"][k])], [c["poses"][k]])
    with pytest.raises(IndexError, match=str(int(c["image_t"][k]))):
        ring.check()
    with pytest.raises(ValueError):
        ring.targets([int(c["image_t"][k])], [c["poses"][k]])


def test_robotcar_stream_evaluation_equals_the_loaders_targets():
    """eval_monorec_oxrc.json's metrics and max_distance over a 5-frame RobotCar stream (robotcar_layout, key frames 1-3):
    SequenceEvaluater fed the device targets gives, bit for bit, the log it gives when fed the loader's targets."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.robotcar import RobotCarLidar
    from monorec_b200.sequence import MonoRecSequence, robotcar_layout
    from monorec_b200.synthetic import make_sequence
    from tests.test_sequence_layouts_gpu import _bits as log_bits, _model
    c = CASES["half_nocut"]
    n, (H, W) = len(c["image_t"]), c["shape"]
    lay = robotcar_layout(n, 2)
    assert list(lay.keys) == c["keys"].tolist()
    names = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
             "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]
    images, vo, Ks = make_sequence(n, H, W, seed=11)
    ring = RobotCarLidar(**_kw(c))
    for t, s, p in zip(c["scan_t"].tolist(), c["scans"], c["lidar_poses"]):
        ring.add_scan(t, s, p)
    device_targets = ring.targets(c["image_t"].tolist(), list(c["poses"]))
    ring.check()
    golden = torch.zeros(n, 1, H, W)
    golden[c["keys"].tolist()] = torch.from_numpy(c["depth"])
    model = _model(7)
    logs = []
    with torch.no_grad():
        for targets in (device_targets, golden.to(DEV)):
            ev = SequenceEvaluater(MonoRecSequence(model, batch_size=4, layout=lay), names, 4, max_distance=80)
            for f in range(n):
                ev.push(images[f].to(DEV), vo[f].to(DEV), Ks[f].to(DEV), target=targets[f])
            ev.flush()
            logs.append(ev.log())
    assert logs[0]["valid_batches"] == 1
    assert log_bits(logs[0]) == log_bits(logs[1])
