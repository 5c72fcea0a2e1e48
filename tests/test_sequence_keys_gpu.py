"""The KITTI loader's optional inputs over a frame stream on the GPU: stereo frames (`use_stereo`), moving-object masks
(`pretrain_mode=3`) and index-masked key-frame lists through MonoRecSequence, SequenceEvaluater and the sharded
evaluation / point-cloud export, against eager forwards of the loader's dicts, the evaluater's fold and one process.

Seeded MonoRecModels at 64x128, sequence batch 4."""
import datetime
import io
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from tests import eval_oracle as EO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 64, 128
BATCH = 4
LENGTHS = (19, 14)
NAMES = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
         "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric", "abs_rel_sparse_onlydynamic_metric",
         "a1_sparse_onlydynamic_metric", "abs_rel_metric", "sc_inv_metric"]
TENSOR_SIGNATURE = ("sc_inv_metric", "l1_rel_metric", "l1_inv_metric", "completeness_metric", "covered_gt_metric")
ROI, MAX_D = [4, 60, 8, 120], 80


def _model(dev=DEV, **kw):
    import monorec_b200.model as MM
    from monorec_b200.synthetic import seeded_state_dict
    m = MM.MonoRecModel(**kw)
    m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
    return m.to(dev).eval()


def _stream(n, seed):
    """A synthetic sequence with its right-camera frames (pose @ a 0.54 m baseline), targets (frame 4 without ground
    truth), moving-object masks and dropout numbers, on the host."""
    from monorec_b200.synthetic import make_sequence
    images, poses, Ks = make_sequence(n, H, W, seed=seed)
    right = make_sequence(n, H, W, seed=seed + 50)[0]
    base = torch.eye(4)
    base[0, 3] = 0.54
    g = torch.Generator().manual_seed(seed + 100)
    target = torch.rand(n, 1, H, W, generator=g) * 0.2 + 0.01
    target[torch.rand(n, 1, H, W, generator=g) > 0.25] = 0.0
    target[4] = 0.0
    mask = (torch.rand(n, 1, H, W, generator=g) > 0.7).float()
    rand = torch.rand(n, 1, H, W, generator=g)
    return dict(images=images, poses=poses, Ks=Ks, right=right, right_poses=poses @ base, target=target, mask=mask,
                rand=rand)


def _masked_keys(n, seed, lidar=False):
    """The loader's key frames of an index-masked sequence: two JSON-style masks drop about a third."""
    from monorec_b200.sequence import loader_keys
    g = np.random.default_rng(seed)
    masks = [{str(i): bool(g.random() < 0.8) for i in range(n)} for _ in range(2)]
    return loader_keys(n, 2, 1, lidar_depth=lidar, index_masks=masks)


def _push_kw(st, n, stereo, mvobj):
    kw = {}
    if stereo:
        kw["stereo"] = (st["right"][n], st["right_poses"][n], st["Ks"][n])
    if mvobj:
        kw["mvobj_mask"] = st["mask"][n]
    return kw


def _loader_dict(st, keys, offs, stereo, mvobj):
    """The loader's collated dict of these key frames (kitti_odometry_dataset.py:248-282), on cuda:0."""
    rows = lambda t, d: torch.stack([t[i + d] for i in keys]).to(DEV)              # noqa: E731
    data = {"keyframe": rows(st["images"], 0), "keyframe_pose": rows(st["poses"], 0), "keyframe_intrinsics": rows(st["Ks"], 0),
            "frames": [rows(st["images"], d) for d in offs], "poses": [rows(st["poses"], d) for d in offs],
            "intrinsics": [rows(st["Ks"], d) for d in offs]}
    if stereo:
        data.update(stereoframe=rows(st["right"], 0), stereoframe_pose=rows(st["right_poses"], 0),
                    stereoframe_intrinsics=rows(st["Ks"], 0))
    if mvobj:
        data["mvobj_mask"] = rows(st["mask"], 0)
    return data


@pytest.mark.parametrize("case", ["stereo", "mvobj", "index_masked", "stereo_index_masked"])
def test_outputs_equal_eager_forwards_of_the_loader_dicts(case):
    """Every key frame run by the sequence (graph replay, short last batch eager) equals, bit for bit, the same row of an
    eager forward of the loader's dict of the same batch of key frames; in pretrain_mode 3, cv_mask is the pushed mask."""
    from monorec_b200.sequence import MonoRecSequence, neighbour_offsets
    stereo, mvobj, masked = "stereo" in case, case == "mvobj", "index_masked" in case
    model = _model(use_stereo=stereo, pretrain_mode=3 if mvobj else 0)
    n_frames = 23
    st = _stream(n_frames, seed=3)
    keys = _masked_keys(n_frames, seed=1) if masked else None
    seq = MonoRecSequence(model, batch_size=BATCH, keys=keys, stereo=stereo, mvobj_masks=mvobj)
    offs = neighbour_offsets(2)
    seen, batches = [], []

    def check(emitted):
        if not emitted:
            return
        indices = [i for i, _ in emitted]
        batches.append(len(indices))
        with torch.no_grad():
            ref = model(_loader_dict(st, indices, offs, stereo, mvobj))
        for j, (i, o) in enumerate(emitted):
            for k in ("result", "cv_mask", "cost_volume"):
                assert torch.equal(o[k], ref[k][j:j + 1]), (i, k)
            for s in range(4):
                assert torch.equal(o["predicted_inverse_depths"][s], ref["predicted_inverse_depths"][s][j:j + 1]), (i, s)
            if mvobj:
                assert torch.equal(o["cv_mask"], st["mask"][i:i + 1].to(DEV)), i
            if stereo:
                assert torch.equal(o["stereoframe_pose"], st["right_poses"][i:i + 1].to(DEV)), i
        seen.extend(indices)
    with torch.no_grad():
        for n in range(n_frames):
            if not seq.needs(n):
                seq.skip()
                continue
            check(seq.push(st["images"][n], st["poses"][n], st["Ks"][n], **_push_kw(st, n, stereo, mvobj)))
        check(seq.flush())
    expected = keys if masked else list(range(1, n_frames - 1))
    assert seen == expected
    assert batches == [BATCH] * (len(expected) // BATCH) + ([len(expected) % BATCH] if len(expected) % BATCH else [])
    if mvobj:
        assert 0 < float(torch.stack([st["mask"][i] for i in seen]).mean()) < 1


def _evaluater_fold(result, target, mvobj, names, bs, roi, md):
    """Evaluater.eval's loop (evaluater.py:78-119) with this package's metric functions, batch by batch, folded by the
    float64 restatement pinned on the reference's logs (tests/eval_oracle.py)."""
    from monorec_b200 import metrics as M
    n, rows = result.shape[0], []
    for b in range(0, n, bs):
        d = {"result": result[b:b + bs], "target": target[b:b + bs], "mvobj_mask": mvobj[b:b + bs]}
        rows.append([float(getattr(M, name)(d["result"], d["target"], roi, md) if name in TENSOR_SIGNATURE
                           else getattr(M, name)(d, roi, md)) for name in names])
    return EO.log(EO.accumulate(np.array(rows, np.float32), EO.batch_sizes(n, bs)))


def _assert_same(got, ref, rtol=2e-6, atol=1e-7):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=rtol, atol=atol)


@pytest.mark.parametrize("pretrain_mode", [0, 3], ids=["mono", "mvobj_mask"])
@pytest.mark.parametrize("bs", [2, 3])
def test_index_masked_evaluation_equals_the_evaluater_fold(pretrain_mode, bs):
    """Two index-masked sequences (the second with the annotated-lidar range), frames no listed key frame needs skipped: the
    log equals the evaluater's fold over the same per-batch results, in the DataLoader's batches of the listed key frames
    across the sequence boundary.  The moving-object masks feed both pretrain_mode 3 and the onlydynamic metrics."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.sequence import MonoRecSequence
    model = _model(pretrain_mode=pretrain_mode)
    mv = pretrain_mode == 3
    streams = [_stream(n, seed=3 + s) for s, n in enumerate(LENGTHS)]
    keys = [_masked_keys(LENGTHS[0], seed=2), _masked_keys(LENGTHS[1], seed=3, lidar=True)]
    ev = SequenceEvaluater(None, NAMES, bs, roi=ROI, max_distance=MAX_D)
    results, order = [], []
    with torch.no_grad():
        for s, st in enumerate(streams):
            emitted = ev.next_sequence(MonoRecSequence(model, batch_size=BATCH, keys=keys[s], mvobj_masks=mv))
            results += [o["result"].clone() for _, o in emitted]
            order += [(s - 1, i) for i, _ in emitted]
            for n in range(LENGTHS[s]):
                if not ev.seq.needs(n):
                    ev.skip()
                    continue
                emitted = ev.push(st["images"][n], st["poses"][n], st["Ks"][n], st["target"][n], mvobj_mask=st["mask"][n])
                results += [o["result"].clone() for _, o in emitted]
                order += [(s, i) for i, _ in emitted]
        emitted = ev.flush()
        results += [o["result"].clone() for _, o in emitted]
        order += [(1, i) for i, _ in emitted]
    assert order == [(s, k) for s in range(2) for k in keys[s]]
    log = ev.log()
    pick = lambda key: torch.cat([streams[s][key][i:i + 1] for s, i in order]).to(DEV)    # noqa: E731
    ref = _evaluater_fold(torch.cat(results), pick("target"), pick("mask"), NAMES, bs, ROI, MAX_D)
    assert log["valid_batches"] == ref["valid_batches"] > 0
    _assert_same(log["metrics"], ref["metrics"])
    _assert_same(log["metrics_correct"], ref["metrics_correct"])


# ---- two ranks on one GPU ---------------------------------------------------------------------------------------------
def _dist_keys():
    return [_masked_keys(LENGTHS[0], seed=4), _masked_keys(LENGTHS[1], seed=5)]


def _evaluate(model, streams, keys, dev, group=None, rank=0, world=None):
    from monorec_b200.dist import shard_sequences
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.sequence import MonoRecSequence
    if world is None:
        slices, kw = [(s, 0, n, None) for s, n in enumerate(LENGTHS)], {}
    else:
        shard = shard_sequences(LENGTHS, 2, 1, BATCH, rank, world, eval_batch=3, keys=keys)
        slices, kw = [(sl.sequence, sl.frames[0], sl.frames[1], sl.run[1]) for sl in shard], dict(group=group, shard=shard)
    ev = SequenceEvaluater(None, NAMES, 3, roi=ROI, max_distance=MAX_D, **kw)
    with torch.no_grad():
        for s, f0, f1, key_end in slices:
            ev.next_sequence(MonoRecSequence(model, batch_size=BATCH, device=dev, first_frame=f0, key_end=key_end,
                                             keys=keys[s], stereo=True))
            st = streams[s]
            for n in range(f0, f1):
                if not ev.seq.needs(n):
                    ev.skip()
                    continue
                ev.push(st["images"][n], st["poses"][n], st["Ks"][n], st["target"][n], mvobj_mask=st["mask"][n],
                        stereo=(st["right"][n], st["right_poses"][n], st["Ks"][n]))
        ev.flush()
    return ev.log()


def _pointcloud(model, streams, keys, dev, group=None, rank=0, world=None):
    from monorec_b200 import pointcloud as PC
    from monorec_b200.dist import shard_sequences
    from monorec_b200.sequence import MonoRecSequence
    if world is None:
        slices = [(s, 0, n, None, None) for s, n in enumerate(LENGTHS)]
    else:
        slices = [(sl.sequence, sl.frames[0], sl.frames[1], sl.run[1], sl.emit)
                  for sl in shard_sequences(LENGTHS, 2, 1, BATCH, rank, world, buffer_length=5, keys=keys)]
    saver = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=[8, 64, 8, 120], dropout=0.75)
    with torch.no_grad():
        for s, f0, f1, key_end, emit in slices:
            st = streams[s]
            pc = PC.SequencePointCloud(MonoRecSequence(model, batch_size=BATCH, device=dev, first_frame=f0, key_end=key_end,
                                                       keys=keys[s], stereo=True), saver, emit=emit)
            for n in range(f0, f1):
                if not pc.seq.needs(n):
                    pc.skip()
                    continue
                pc.push(st["images"][n], st["poses"][n], st["Ks"][n], rand=st["rand"][n],
                        stereo=(st["right"][n], st["right_poses"][n], st["Ks"][n]))
            pc.flush()
    f = io.BytesIO() if rank == 0 else None
    if world is None:
        saver.save(f)
        return saver.vertices.cpu().numpy(), f.getvalue()
    v = saver.gather(group)
    saver.save(f, group=group)
    return None if v is None else (v.cpu().numpy(), f.getvalue())


def _models(dev):
    return _model(dev, use_stereo=True), _model(dev, use_stereo=True, pretrain_mode=1, inv_depth_min_max=(0.33, 0.06))


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    try:
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
        model, pc_model = _models(dev)
        streams, keys = [_stream(n, seed=3 + s) for s, n in enumerate(LENGTHS)], _dist_keys()
        log = _evaluate(model, streams, keys, dev, dist.group.WORLD, rank, world)
        ply = _pointcloud(pc_model, streams, keys, dev, dist.group.WORLD, rank, world)
        q.put((rank, log, ply, None))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, None, None, traceback.format_exc()))


def test_two_ranks_with_key_lists_and_stereo_equal_one_process():
    """Two gloo ranks on cuda:0, index-masked key lists and stereo frames: every rank's log and rank 0's PLY equal the
    one process's bit for bit."""
    model, pc_model = _models(torch.device(DEV))
    streams, keys = [_stream(n, seed=3 + s) for s, n in enumerate(LENGTHS)], _dist_keys()
    ref_log = _evaluate(model, streams, keys, DEV)
    ref_v, ref_ply = _pointcloud(pc_model, streams, keys, DEV)
    assert 0 < ref_log["valid_batches"] and ref_v.shape[0] > 1000
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    try:
        [p.start() for p in procs]
        out = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r[0])
        [p.join(timeout=120) for p in procs]
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    errors = [e for _, _, _, e in out if e]
    assert not errors, errors[0]
    bits = lambda x: np.asarray(x, np.float64).view(np.uint64)    # noqa: E731
    for rank, log, _, _ in out:
        assert log["valid_batches"] == ref_log["valid_batches"], rank
        for key in ("metrics", "metrics_correct"):
            np.testing.assert_array_equal(bits(log[key]), bits(ref_log[key]), err_msg=f"rank {rank} {key}")
    v, ply = out[0][2]
    np.testing.assert_array_equal(v, ref_v)
    assert ply == ref_ply and out[1][2] is None
