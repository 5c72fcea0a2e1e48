"""The sequence path split over ranks, on the CPU: dist.shard_sequences' arithmetic (every emitted key frame exactly once,
whole evaluater batches, whole one-process model batches, only the frames a slice needs), MonoRecSequence run on a slice
(first_frame / key_end) with a fake model, the argument checks of the sharded SequenceEvaluater, and the variable-row
gathers of dist.py over gloo."""
import itertools
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from monorec_b200.dist import shard_sequences
from monorec_b200.sequence import MonoRecSequence, neighbour_offsets

LENGTHS = [[13, 10], [5], [3, 40, 1, 17], [64, 63, 2], [9, 9, 9], [2], []]
SHAPES = [(2, 1, 4), (2, 1, 8), (4, 1, 3), (4, 2, 4), (2, 2, 1), (1, 1, 2), (3, 1, 5)]   # frame_count, dilation, batch


def _keys(n, frame_count, dilation):
    """The loader's key frames of a sequence of n frames: those with all their neighbours."""
    offs = neighbour_offsets(frame_count, dilation)
    return list(range(max(0, -min(offs)), n - max(offs)))


def _model_batches(keys, bs):
    """The one-process MonoRecSequence's batches: batch_size at a time from the first key frame, the rest last."""
    return [keys[b:b + bs] for b in range(0, len(keys), bs)]


def _cases():
    for lengths, (fc, dil, bs) in itertools.product(LENGTHS, SHAPES):
        for world in range(1, 9):
            yield lengths, fc, dil, bs, world


@pytest.mark.parametrize("eval_batch", [1, 2, 3, 5])
def test_evaluater_shards_tile_the_run_in_whole_batches(eval_batch):
    for lengths, fc, dil, bs, world in _cases():
        offs = neighbour_offsets(fc, dil)
        lo, hi = min(0, min(offs)), max(offs)
        every = [(s, i) for s, n in enumerate(lengths) for i in _keys(n, fc, dil)]
        emitted, counts = [], []
        for rank in range(world):
            mine = []
            for sl in shard_sequences(lengths, fc, dil, bs, rank, world, eval_batch=eval_batch):
                keys = _keys(lengths[sl.sequence], fc, dil)
                assert sl.position == every.index((sl.sequence, sl.emit[0]))
                # run: whole batches of the one-process run; emit inside it; frames: exactly the run's neighbours
                batches = _model_batches(keys, bs)
                run = list(range(*sl.run))
                assert run == [i for b in batches if set(b) & set(run) for i in b]
                assert sl.run[0] <= sl.emit[0] < sl.emit[1] <= sl.run[1]
                assert sl.frames == (sl.run[0] + lo, sl.run[1] - 1 + hi + 1)
                # only frames within one model batch and the neighbour span of the emitted key frames
                assert sl.frames[0] >= sl.emit[0] + lo - (bs - 1) and sl.frames[1] - 1 <= sl.emit[1] - 1 + hi + (bs - 1)
                assert 0 <= sl.frames[0] and sl.frames[1] <= lengths[sl.sequence]
                mine += [(sl.sequence, i) for i in range(*sl.emit)]
            # consecutive in the global list, starting and ending on evaluater batch boundaries (or the run's end)
            if mine:
                a = every.index(mine[0])
                assert mine == every[a:a + len(mine)]
                assert a % eval_batch == 0 and ((a + len(mine)) % eval_batch == 0 or a + len(mine) == len(every))
            emitted += mine
            counts.append(len(mine))
        assert emitted == every, (lengths, fc, dil, bs, world)
        assert all(abs(c - len(every) / world) <= eval_batch for c in counts), counts   # the nearest batch boundaries


@pytest.mark.parametrize("buffer_length", [1, 3, 5])
def test_pointcloud_shards_add_the_one_process_key_frames_once(buffer_length):
    before, after = buffer_length // 2, buffer_length - 1 - buffer_length // 2
    for lengths, fc, dil, bs, world in _cases():
        offs = neighbour_offsets(fc, dil)
        lo, hi = min(0, min(offs)), max(offs)
        # SequencePointCloud adds the key frames whose whole window lies in their sequence
        every = [(s, k) for s, n in enumerate(lengths) for p, k in enumerate(_keys(n, fc, dil))
                 if before <= p < len(_keys(n, fc, dil)) - after]
        emitted, counts = [], []
        for rank in range(world):
            mine = []
            for sl in shard_sequences(lengths, fc, dil, bs, rank, world, buffer_length=buffer_length):
                keys = _keys(lengths[sl.sequence], fc, dil)
                assert sl.position == every.index((sl.sequence, sl.emit[0]))
                batches = _model_batches(keys, bs)
                run = list(range(*sl.run))
                assert run == [i for b in batches if set(b) & set(run) for i in b]
                # the run covers every emitted key frame's window
                assert sl.run[0] <= sl.emit[0] - before and sl.emit[1] - 1 + after < sl.run[1]
                assert sl.frames == (sl.run[0] + lo, sl.run[1] + hi)
                span = (bs - 1) + before
                assert sl.frames[0] >= sl.emit[0] + lo - span and sl.frames[1] - 1 <= sl.emit[1] - 1 + hi + (bs - 1) + after
                mine += [(sl.sequence, i) for i in range(*sl.emit)]
            emitted += mine
            counts.append(len(mine))
        assert emitted == every, (lengths, fc, dil, bs, world)
        assert max(counts) - min(counts) <= 1


def test_more_ranks_than_batches_leaves_ranks_empty():
    empty = [r for r in range(8) if not shard_sequences([7], 2, 1, 4, r, 8, eval_batch=2)]
    assert len(empty) == 5                                   # 5 key frames: three evaluater batches of 2
    assert shard_sequences([], 2, 1, 4, 0, 1, eval_batch=2) == []


def test_shard_sequences_arguments():
    with pytest.raises(ValueError):
        shard_sequences([10], 2, 1, 4, 0, 1)
    with pytest.raises(ValueError):
        shard_sequences([10], 2, 1, 4, 0, 1, eval_batch=2, buffer_length=5)
    with pytest.raises(ValueError):
        shard_sequences([10], 2, 1, 4, 2, 2, eval_batch=2)
    with pytest.raises(ValueError):
        shard_sequences([10], 2, 1, 0, 0, 1, eval_batch=2)


# ---- MonoRecSequence on a slice ----------------------------------------------------------------------------------------
class _FakeModel:
    """result = the key frame's image (filled with its sequence index); records each batch's key frames."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self):
        self.batches = []

    def __call__(self, data):
        self.batches.append([int(v) for v in data["keyframe"][:, 0, 0, 0]])
        data["result"] = data["keyframe"][:, :1] * 1.0
        data["cost_volume"] = torch.stack([f[:, 0, 0, 0] for f in data["frames"]], 1)
        return data


def _frame(n):
    return torch.full((3, 2, 3), float(n)), torch.eye(4), torch.eye(4)


def _run_slice(fc, dil, bs, frames, key_end, first_frame=None):
    model = _FakeModel()
    kw = {} if first_frame is None else dict(first_frame=first_frame, key_end=key_end)
    seq = MonoRecSequence(model, fc, dil, bs, graphed=False, device="cpu", **kw)
    out = []
    for n in range(*frames):
        out += seq.push(*_frame(n))
    out += seq.flush()
    return model.batches, out


@pytest.mark.parametrize("fc,dil,bs", SHAPES)
@pytest.mark.parametrize("lengths", [[13, 10], [3, 40, 1, 17], [64, 63, 2]], ids=["13-10", "3-40-1-17", "64-63-2"])
def test_sliced_sequences_run_the_one_process_batches(lengths, fc, dil, bs):
    """Every rank's MonoRecSequence, fed its slice's frames, runs only batches of the one-process run, each with the same
    key frames and the same source frames."""
    offs = neighbour_offsets(fc, dil)
    whole = {}
    for s, n in enumerate(lengths):
        batches, out = _run_slice(fc, dil, bs, (0, n), None)
        whole[s] = batches
        assert [i for i, _ in out] == _keys(n, fc, dil)
    for world, kind in itertools.product((1, 2, 3, 5, 8), ({"eval_batch": 3}, {"buffer_length": 5})):
        for rank in range(world):
            for sl in shard_sequences(lengths, fc, dil, bs, rank, world, **kind):
                batches, out = _run_slice(fc, dil, bs, sl.frames, sl.run[1], first_frame=sl.frames[0])
                assert all(b in whole[sl.sequence] for b in batches), (sl, batches)
                assert [i for i, _ in out] == list(range(*sl.run))
                for i, o in out:
                    assert o["cost_volume"].tolist() == [[float(i + d) for d in offs]]


def test_slice_arguments():
    seq = MonoRecSequence(_FakeModel(), 2, 1, 4, graphed=False, device="cpu", first_frame=8, key_end=12)
    assert (seq.key_begin, seq.key_end, seq.first_key, seq.n_pushed) == (9, 12, 1, 8)
    out = []
    for n in range(8, 13):
        out += seq.push(*_frame(n))
    assert [i for i, _ in out] == [9, 10, 11]                # the short batch runs at the push that completes it
    with pytest.raises(ValueError):
        seq.push(*_frame(13))                                # no key frame before key_end needs frame 13
    assert seq.flush() == []
    with pytest.raises(ValueError):
        MonoRecSequence(_FakeModel(), device="cpu", first_frame=-1)


def test_sharded_evaluater_arguments():
    from monorec_b200.evaluation import SequenceEvaluater
    names = ["abs_rel_sparse_metric"]
    shard = shard_sequences([20], 2, 1, 4, 1, 2, eval_batch=2)
    with pytest.raises(ValueError):
        SequenceEvaluater(None, names, 2, shard=shard)                  # a shard without a group
    with pytest.raises(ValueError):
        SequenceEvaluater(None, names, 2, group=object())                # a group without a shard
    with pytest.raises(ValueError):
        SequenceEvaluater(None, names, 3, group=object(), shard=shard)   # not cut for evaluater batches of 3
    seq = MonoRecSequence(_FakeModel(), 2, 1, 4, graphed=False, device="cpu", first_frame=0, key_end=shard[0].emit[0])
    with pytest.raises(ValueError):
        SequenceEvaluater(seq, names, 2, group=object(), shard=shard)    # a sequence that does not run the slice


# ---- variable-row gathers over gloo -------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gather_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from monorec_b200.dist import all_gather_rows, gather_rows
    counts = [3, 0, 5][:world]
    mine = torch.arange(counts[rank] * 4, dtype=torch.float64).view(-1, 4) + 100 * rank
    full = torch.cat([torch.arange(c * 4, dtype=torch.float64).view(-1, 4) + 100 * r for r, c in enumerate(counts)])
    ok = torch.equal(all_gather_rows(mine), full)
    got = gather_rows(mine, dst=0)
    ok = ok and (torch.equal(got, full) if rank == 0 else got is None)
    empty = all_gather_rows(mine[:0])
    ok = ok and tuple(empty.shape) == (0, 4)
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_row_gathers_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gather_worker, args=(r, 3, port, q)) for r in range(3)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(ok for _, ok in res), res
