"""The sequence evaluation and point-cloud export split over ranks (dist.shard_sequences, MonoRecSequence slices, the
sharded SequenceEvaluater, SequencePointCloud(emit=...), PLYSaver.gather) against one process.

2 and 3 ranks on cuda:0 over gloo, a 1-rank group, and (on a machine with >= 2 GPUs) one rank per GPU over NCCL.  Every rank
runs its slices of two concatenated synthetic sequences of unequal length with seeded weights; every rank's log() equals the
one-process SequenceEvaluater's log bit for bit, and rank 0's gathered vertices equal the one-process sequence_pointcloud
vertex for vertex, in order."""
import datetime
import io
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

H, W = 64, 128
LENGTHS = (15, 11)                       # 13 + 9 key frames at frame_count 2
BATCH = 4                                # the sequences' model batch
NAMES = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
         "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric", "abs_rel_sparse_onlydynamic_metric",
         "a1_sparse_onlydynamic_metric", "abs_rel_metric", "sc_inv_metric", "completeness_metric"]
ROI, MAX_D = [4, 60, 8, 120], 80
# (evaluater batch, median scaling): 22 key frames, so every evaluater batch size here leaves a partial last batch
EVAL_CASES = [(3, False), (3, True), (5, False), (4, True)]
PLY_ROI, DROPOUTS = [8, 64, 8, 120], [0.0, 0.75]


class _MovingObject(torch.nn.Module):
    """A seeded MonoRecModel whose cv_mask is a 12x12 block moving 5 px right per frame (the sequence index is read back
    from the pose's z translation), so that the 5-frame vote removes a different region per key frame."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self, model, step):
        super().__init__()
        self.model, self.step = model, step

    def forward(self, data):
        data = self.model(data)
        B, _, h, w = data["result"].shape
        n = torch.round(data["keyframe_pose"][:, 2, 3] / self.step).view(B, 1, 1, 1)
        y = torch.arange(h, device=n.device).view(1, 1, h, 1)
        x = torch.arange(w, device=n.device).view(1, 1, 1, w)
        data["cv_mask"] = (((y - 32).abs() < 6) & ((x - 20 - 5 * n).abs() < 6)).to(torch.float32)
        return data


def _inputs():
    """The two sequences, their targets (key frame 4 of the first without ground truth), moving-object masks and dropout
    numbers: host tensors, the same in every process."""
    from monorec_b200.synthetic import make_sequence
    seqs = [make_sequence(n, H, W, seed=3 + s) for s, n in enumerate(LENGTHS)]
    g = torch.Generator().manual_seed(5)
    targets, masks, rands = [], [], []
    for n in LENGTHS:
        t = torch.rand(n, 1, H, W, generator=g) * 0.2 + 0.01
        t[torch.rand(n, 1, H, W, generator=g) > 0.25] = 0.0
        targets.append(t)
        masks.append((torch.rand(n, 1, H, W, generator=g) > 0.5).float())
        rands.append(torch.rand(n, 1, H, W, generator=g))
    targets[0][4] = 0.0
    return seqs, targets, masks, rands


def _models(dev):
    import monorec_b200.model as MM
    from monorec_b200.synthetic import seeded_state_dict
    m = MM.MonoRecModel()
    m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
    pc = MM.MonoRecModel(pretrain_mode=1, inv_depth_min_max=(0.33, 0.06))     # every depth inside [3, 20] m
    pc.load_state_dict(seeded_state_dict(pc, seed=7, gain=0.7))
    return m.to(dev).eval(), pc.to(dev).eval()


def _slices(world, rank, **kind):
    """(sequence, first frame, frame end, key_end, emit): the whole sequences in one process, the rank's slices else."""
    from monorec_b200.dist import shard_sequences
    if world is None:
        return [(s, 0, n, None, None) for s, n in enumerate(LENGTHS)]
    return [(sl.sequence, sl.frames[0], sl.frames[1], sl.run[1], sl.emit)
            for sl in shard_sequences(LENGTHS, 2, 1, BATCH, rank, world, **kind)]


def _evaluate(model, inputs, eval_batch, median_scaling, dev, group=None, rank=0, world=None):
    from monorec_b200.dist import shard_sequences
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.sequence import MonoRecSequence
    seqs, targets, masks, _ = inputs
    kw = {} if world is None else dict(group=group, shard=shard_sequences(LENGTHS, 2, 1, BATCH, rank, world,
                                                                          eval_batch=eval_batch))
    ev = SequenceEvaluater(None, NAMES, eval_batch, roi=ROI, max_distance=MAX_D, median_scaling=median_scaling, **kw)
    with torch.no_grad():
        for s, f0, f1, key_end, _ in _slices(world, rank, eval_batch=eval_batch):
            ev.next_sequence(MonoRecSequence(model, batch_size=BATCH, device=dev, first_frame=f0, key_end=key_end))
            images, poses, Ks = seqs[s]
            for n in range(f0, f1):
                ev.push(images[n], poses[n], Ks[n], targets[s][n], mvobj_mask=masks[s][n])
        ev.flush()
    return ev.log()


def _pointcloud(model, inputs, dropout, dev, group=None, rank=0, world=None):
    """(vertices, PLY file): the one process's, or rank 0's gathered ones and collective save (None on the other ranks)."""
    from monorec_b200 import pointcloud as PC
    from monorec_b200.sequence import MonoRecSequence
    seqs, _, _, rands = inputs
    saver = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=PLY_ROI, dropout=dropout)
    with torch.no_grad():
        for s, f0, f1, key_end, emit in _slices(world, rank, buffer_length=5):
            images, poses, Ks = seqs[s]
            mov = _MovingObject(model, step=float(poses[1, 2, 3]))
            pc = PC.SequencePointCloud(MonoRecSequence(mov, batch_size=BATCH, device=dev, first_frame=f0, key_end=key_end),
                                       saver, emit=emit)
            for n in range(f0, f1):
                pc.push(images[n], poses[n], Ks[n], rand=rands[s][n] if dropout else None)
            pc.flush()
    if world is None:
        f = io.BytesIO()
        saver.save(f)
        return saver.vertices.cpu(), f.getvalue()
    v = saver.gather(group)
    f = io.BytesIO() if rank == 0 else None
    saver.save(f, group=group)                       # the collective save: rank 0 writes every rank's vertices
    return None if v is None else (v.cpu(), f.getvalue())


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    try:
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
        group = dist.group.WORLD
        model, pc_model = _models(dev)
        inputs = _inputs()
        logs = [_evaluate(model, inputs, eb, ms, dev, group, rank, world) for eb, ms in EVAL_CASES]
        verts = [_pointcloud(pc_model, inputs, p, dev, group, rank, world) for p in DROPOUTS]
        q.put((rank, logs, [None if v is None else (v[0].numpy(), v[1]) for v in verts], None))
        dist.destroy_process_group()
    except Exception:
        q.put((rank, None, None, traceback.format_exc()))


def _spawn(world, backend):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
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
    return out


@pytest.fixture(scope="module")
def one_process():
    dev = torch.device("cuda", 0)
    model, pc_model = _models(dev)
    inputs = _inputs()
    logs = [_evaluate(model, inputs, eb, ms, dev) for eb, ms in EVAL_CASES]
    verts = [_pointcloud(pc_model, inputs, p, dev) for p in DROPOUTS]
    return logs, verts


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def _check(out, one_process):
    logs, verts = one_process
    # the one-process runs evaluate something: valid and NaN batches, and votes that remove moving-object pixels
    assert all(0 < log["valid_batches"] < -(-22 // eb) for log, (eb, _) in zip(logs, EVAL_CASES))
    assert all(v.shape[0] > 1000 for v, _ in verts)
    for rank, rank_logs, _, _ in out:
        for case, got, ref in zip(EVAL_CASES, rank_logs, logs):
            assert got["valid_batches"] == ref["valid_batches"], (rank, case)
            for key in ("metrics", "metrics_correct"):
                np.testing.assert_array_equal(_bits(got[key]), _bits(ref[key]), err_msg=f"rank {rank} {case} {key}")
    for dropout, (got, ply), (ref, ref_ply) in zip(DROPOUTS, out[0][2], verts):
        assert got.shape == tuple(ref.shape), dropout
        np.testing.assert_array_equal(got, ref.numpy(), err_msg=f"dropout {dropout}")
        assert ply == ref_ply, dropout
    assert all(v is None for _, _, vs, _ in out[1:] for v in vs)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ranks_sharing_a_gpu_equal_one_process(one_process, world):
    """world ranks on cuda:0 over gloo (world 1: a 1-rank group gives the one-process results)."""
    _check(_spawn(world, "gloo"), one_process)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_one_rank_per_gpu_over_nccl_equals_one_process(one_process):
    _check(_spawn(min(torch.cuda.device_count(), 3), "nccl"), one_process)
