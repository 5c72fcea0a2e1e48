"""One process driving several devices (monorec_b200.lanes) against one process on one device, and the point-cloud export
without host synchronisation.

Lanes [0, 0, 0] (three lanes taking turns on one GPU: the whole split, feed and merge logic) and, on a machine with two
GPUs, [0, 1].  The evaluation's log equals the one-lane SequenceEvaluater's bit for bit and the PLY bytes equal
sequence_pointcloud's, with median scaling on and off, dropout 0 and with fixed numbers, and index-masked key lists with
stereo frames.  Under torch.cuda.set_sync_debug_mode("error"), once the graphs are captured, the pushes and flushes of
both make no host synchronisation, and neither does a single-GPU sequence_pointcloud; a vertex buffer that starts small
and grows during the run holds the same vertices as one large buffer."""
import io

import numpy as np
import pytest
import torch

from tests import test_sequence_dist_gpu as D
from tests import test_sequence_keys_gpu as K

pytestmark = pytest.mark.gpu

LANES = [[0, 0, 0]] + ([[0, 1]] if torch.cuda.device_count() >= 2 else [])


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def _same_log(got, ref):
    assert got["valid_batches"] == ref["valid_batches"]
    for key in ("metrics", "metrics_correct"):
        np.testing.assert_array_equal(_bits(got[key]), _bits(ref[key]), err_msg=key)


def _lanes_evaluate(model, inputs, eval_batch, median_scaling, devices):
    from monorec_b200.lanes import MultiDeviceEvaluater
    seqs, targets, masks, _ = inputs
    run = MultiDeviceEvaluater(model, devices, D.LENGTHS, D.NAMES, eval_batch, seq_batch=D.BATCH, roi=D.ROI,
                               max_distance=D.MAX_D, median_scaling=median_scaling)
    with torch.no_grad():
        for s, n in run.order:
            images, poses, Ks = seqs[s]
            run.push(s, n, images[n], poses[n], Ks[n], targets[s][n], mvobj_mask=masks[s][n])
        run.flush()
    return run.log()


def _lanes_pointcloud(model, inputs, dropout, devices):
    from monorec_b200.lanes import MultiDevicePointCloud
    seqs, _, _, rands = inputs
    mov = D._MovingObject(model, step=float(seqs[0][1][1, 2, 3]))
    run = MultiDevicePointCloud(mov, devices, D.LENGTHS, D.H, D.W, seq_batch=D.BATCH, min_d=3, max_d=20, roi=D.PLY_ROI,
                                dropout=dropout)
    with torch.no_grad():
        for s, n in run.order:
            images, poses, Ks = seqs[s]
            run.push(s, n, images[n], poses[n], Ks[n], rand=rands[s][n] if dropout else None)
        run.flush()
    f = io.BytesIO()
    run.save(f)
    return run.vertices.cpu(), f.getvalue()


@pytest.fixture(scope="module")
def one_process():
    dev = torch.device("cuda", 0)
    model, pc_model = D._models(dev)
    inputs = D._inputs()
    logs = [D._evaluate(model, inputs, eb, ms, dev) for eb, ms in D.EVAL_CASES]
    verts = [D._pointcloud(pc_model, inputs, p, dev) for p in D.DROPOUTS]
    return model, pc_model, inputs, logs, verts


@pytest.mark.parametrize("devices", LANES, ids=lambda d: "-".join(map(str, d)))
def test_lanes_equal_one_process(one_process, devices):
    model, pc_model, inputs, logs, verts = one_process
    assert all(0 < log["valid_batches"] for log in logs) and all(v.shape[0] > 1000 for v, _ in verts)
    for (eb, ms), ref in zip(D.EVAL_CASES, logs):
        _same_log(_lanes_evaluate(model, inputs, eb, ms, devices), ref)
    for dropout, (ref, ref_ply) in zip(D.DROPOUTS, verts):
        got, ply = _lanes_pointcloud(pc_model, inputs, dropout, devices)
        np.testing.assert_array_equal(got.numpy(), ref.numpy(), err_msg=f"dropout {dropout}")
        assert ply == ref_ply, dropout


@pytest.mark.parametrize("devices", LANES, ids=lambda d: "-".join(map(str, d)))
def test_lanes_with_key_lists_and_stereo_equal_one_process(devices):
    from monorec_b200.lanes import MultiDeviceEvaluater, MultiDevicePointCloud
    dev = torch.device("cuda", 0)
    model, pc_model = K._models(dev)
    streams = [K._stream(n, seed=3 + s) for s, n in enumerate(K.LENGTHS)]
    keys = K._dist_keys()
    ref_log = K._evaluate(model, streams, keys, dev)
    ref_v, ref_ply = K._pointcloud(pc_model, streams, keys, dev)
    assert ref_log["valid_batches"] > 0 and ref_v.shape[0] > 0

    def feed(run, **extra):
        with torch.no_grad():
            for s, n in run.order:
                st = streams[s]
                run.push(s, n, st["images"][n], st["poses"][n], st["Ks"][n],
                         stereo=(st["right"][n], st["right_poses"][n], st["Ks"][n]), **{k: f(st, n) for k, f in extra.items()})
            run.flush()

    ev = MultiDeviceEvaluater(model, devices, K.LENGTHS, K.NAMES, 3, seq_batch=K.BATCH, keys=keys, roi=K.ROI,
                              max_distance=K.MAX_D, stereo=True)
    feed(ev, target=lambda st, n: st["target"][n], mvobj_mask=lambda st, n: st["mask"][n])
    _same_log(ev.log(), ref_log)
    pc = MultiDevicePointCloud(pc_model, devices, K.LENGTHS, K.H, K.W, seq_batch=K.BATCH, keys=keys, min_d=3, max_d=20,
                               roi=[8, 64, 8, 120], dropout=0.75, stereo=True)
    feed(pc, rand=lambda st, n: st["rand"][n])
    f = io.BytesIO()
    pc.save(f)
    np.testing.assert_array_equal(pc.vertices.cpu().numpy(), ref_v)
    assert f.getvalue() == ref_ply


def _sync_free_after_capture(run, push, sequences):
    """Feeds `run` in its order; once every lane's current sequence has its graph, the rest of the pushes and the flush run
    under sync debug mode "error".  Returns whether that mode was on for at least one push."""
    checked = False
    try:
        for s, n in run.order:
            if not checked and all(q is not None and q._graph is not None for q in sequences()):
                torch.cuda.set_sync_debug_mode("error")
                checked = True
            push(s, n)
        run.flush()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return checked


@pytest.mark.parametrize("devices,keyed", [(d, k) for k in (False, True) for d in LANES],
                         ids=["-".join(map(str, d)) + ("-index_masked" if k else "") for k in (False, True) for d in LANES])
def test_lanes_make_no_host_synchronisation(one_process, devices, keyed):
    """Every key frame, or an index-masked key list (key frames 5 ... 7 masked out, so frame 6 is skipped)."""
    from monorec_b200.lanes import MultiDeviceEvaluater, MultiDevicePointCloud
    from monorec_b200.sequence import loader_keys
    model, pc_model, inputs, _, _ = one_process
    seqs, targets, masks, rands = inputs
    lengths = [seqs[0][0].shape[0]]
    keys = [loader_keys(lengths[0], index_masks=[{str(k): not 5 <= k <= 7 for k in range(lengths[0])}])] if keyed else None
    with torch.no_grad():
        ev = MultiDeviceEvaluater(model, devices, lengths, D.NAMES, 2, seq_batch=2, keys=keys, roi=D.ROI,
                                  max_distance=D.MAX_D)
        push = lambda s, n: ev.push(s, n, seqs[s][0][n], seqs[s][1][n], seqs[s][2][n], targets[s][n],  # noqa: E731
                                    mvobj_mask=masks[s][n])
        assert _sync_free_after_capture(ev, push, lambda: [e.seq for e in ev.evaluaters if e is not None])
        assert ev.log()["valid_batches"] > 0
        mov = D._MovingObject(pc_model, step=float(seqs[0][1][1, 2, 3]))
        pc = MultiDevicePointCloud(mov, devices, lengths, D.H, D.W, seq_batch=2, keys=keys, min_d=3, max_d=20,
                                   dropout=0.75)
        push = lambda s, n: pc.push(s, n, seqs[s][0][n], seqs[s][1][n], seqs[s][2][n], rand=rands[s][n])  # noqa: E731
        assert _sync_free_after_capture(pc, push, lambda: [r.seq if r else None
                                                           for r, sl in zip(pc._runner, pc.plan.slices) if sl])
        assert pc.vertices.shape[0] > 0


def test_sequence_pointcloud_makes_no_host_synchronisation(one_process):
    """The one-GPU export: after the graph capture, pushes and the flush wait for nothing (the vertex count is read back
    asynchronously)."""
    from monorec_b200 import pointcloud as PC
    from monorec_b200.sequence import MonoRecSequence
    _, pc_model, inputs, _, _ = one_process
    images, poses, Ks = inputs[0][0]
    saver = PC.PLYSaver(D.H, D.W, min_d=3, max_d=20, roi=D.PLY_ROI)
    with torch.no_grad():
        mov = D._MovingObject(pc_model, step=float(poses[1, 2, 3]))
        pc = PC.sequence_pointcloud(MonoRecSequence(mov, batch_size=D.BATCH), saver)
        checked = False
        try:
            for n in range(images.shape[0]):
                if not checked and pc.seq._graph is not None:
                    torch.cuda.set_sync_debug_mode("error")
                    checked = True
                pc.push(images[n], poses[n], Ks[n])
            pc.flush()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert checked and len(saver) > 0


def test_vertex_buffer_grows_without_synchronisation():
    """Every pixel valid, so each add appends B*H*W vertices: a buffer of 100 vertices grows several times during the run,
    with stream-ordered copies and no read-back, and ends with the vertices of one large buffer filled at the host-passed
    positions (n_before >= 0, the C ABI's earlier form)."""
    from monorec_b200 import _lib
    from monorec_b200 import pointcloud as PC
    dev = torch.device("cuda", 0)
    B, H, W, calls = 2, 32, 64, 24
    g = torch.Generator().manual_seed(11)
    batches = []
    for _ in range(calls):
        inv = (torch.rand(B, 1, H, W, generator=g) * 0.2 + 0.06).to(dev)          # depths in [3.6, 16.7] m
        img = (torch.rand(B, 3, H, W, generator=g) - 0.5).to(dev)
        K_ = torch.eye(4).repeat(B, 1, 1)
        K_[:, 0, 0], K_[:, 1, 1], K_[:, 0, 2], K_[:, 1, 2] = 50.0, 50.0, W / 2, H / 2
        P = torch.eye(4).repeat(B, 1, 1)
        P[:, :3, 3] = torch.rand(B, 3, generator=g)
        batches.append((inv, img, K_.to(dev), P.to(dev)))
    total = calls * B * H * W
    small = PC.PLYSaver(H, W, min_d=3, max_d=20)
    small._buf = torch.empty(100, 6, device=dev)
    small._count = torch.zeros(1, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    try:
        torch.cuda.set_sync_debug_mode("error")
        for b in batches:
            small.add_depthmap(*b)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(small) == total and small._buf.shape[0] >= total

    lib = _lib.load()
    ref = torch.empty(total, 6, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    ws_bytes = lib.mr_pointcloud_workspace(B, H, W)
    ws = torch.empty((ws_bytes + 7) // 8, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    for i, (inv, img, K_, P) in enumerate(batches):
        _lib.check(lib.mr_pointcloud_add(inv.data_ptr(), img.data_ptr(), K_.data_ptr(), P.data_ptr(), None, 0, 1, B, H, W,
                                         3.0, 20.0, None, None, 0.0, ref.data_ptr(), total, i * B * H * W, count.data_ptr(),
                                         ws.data_ptr(), ws_bytes, stream), "mr_pointcloud_add")
    assert int(count.item()) == total
    assert torch.equal(small.vertices, ref)


def test_an_overflowing_add_writes_nothing():
    """The device count is the backstop: an add past the capacity leaves it negative, and later adds that take the position
    from it (n_before < 0) keep it negative and write nothing."""
    from monorec_b200 import _lib
    dev = torch.device("cuda", 0)
    B, H, W = 1, 8, 16
    lib = _lib.load()
    inv = torch.full((B, 1, H, W), 0.1, device=dev)
    img = torch.zeros(B, 3, H, W, device=dev)
    eye = torch.eye(4, device=dev).repeat(B, 1, 1)
    buf = torch.zeros(200, 6, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    ws_bytes = lib.mr_pointcloud_workspace(B, H, W)
    ws = torch.empty((ws_bytes + 7) // 8, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    seen = []
    for _ in range(3):
        _lib.check(lib.mr_pointcloud_add(inv.data_ptr(), img.data_ptr(), eye.data_ptr(), eye.data_ptr(), None, 0, 1, B, H,
                                         W, 3.0, 20.0, None, None, 0.0, buf.data_ptr(), 200, -1, count.data_ptr(),
                                         ws.data_ptr(), ws_bytes, stream), "mr_pointcloud_add")
        seen.append(int(count.item()))
    assert seen == [128, -256, -384]
    assert torch.count_nonzero(buf[128:]) == 0
