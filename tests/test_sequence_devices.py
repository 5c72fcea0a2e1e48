"""The host side of one process driving several devices (monorec_b200.lanes): each lane's slices, the frames pushed to each
lane, the read order and the merge order of the evaluation rows, on the CPU with a stub model."""
import itertools
import random

import pytest
import torch

from monorec_b200.dist import shard_sequences
from monorec_b200.evaluation import LANE, SequenceEvaluater, sort_rows
from monorec_b200.lanes import LanePlan, _Lanes
from monorec_b200.sequence import MonoRecSequence, loader_keys


class _FakeModel:
    """result = the key frame's image (filled with its sequence index); records each batch's key frames."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self):
        self.batches = []

    def __call__(self, data):
        self.batches.append([int(v) for v in data["keyframe"][:, 0, 0, 0]])
        data["result"] = data["keyframe"][:, :1] * 1.0
        return data


class _Recorder:
    """A lane runner: a CPU MonoRecSequence for one slice that records the frames pushed to it and the key frames run."""

    def __init__(self, seq, log):
        self.seq, self.log = seq, log

    def push(self, image, pose, intrinsics):
        n = int(image[0, 0, 0])
        assert n == self.seq.n_pushed and self.seq.needs(n), (n, self.seq.n_pushed)
        self.log["pushed"].append((self.sequence, n))
        self.log["run"] += [(self.sequence, i) for i, _ in self.seq.push(image, pose, intrinsics)]

    def skip(self):
        self.seq.skip()

    def flush(self):
        self.log["run"] += [(self.sequence, i) for i, _ in self.seq.flush()]


class _CpuLanes(_Lanes):
    def __init__(self, plan, keys, batch):
        super().__init__(plan, ["cpu"] * plan.lanes)
        self.keys, self.batch = keys, batch
        self.logs = [{"pushed": [], "run": []} for _ in range(plan.lanes)]
        self.models = [_FakeModel() for _ in range(plan.lanes)]

    def _open(self, r, sl):
        if self._runner[r] is not None:
            self._runner[r].flush()
        keys = None if self.keys is None else self.keys[sl.sequence]
        seq = MonoRecSequence(self.models[r], 2, 1, self.batch, graphed=False, device="cpu", first_frame=sl.frames[0],
                              key_end=sl.run[1], keys=keys)
        rec = _Recorder(seq, self.logs[r])
        rec.sequence = sl.sequence
        return rec

    def _close(self, r):
        self._runner[r].flush()


def _frame(n):
    return torch.full((3, 2, 3), float(n)), torch.eye(4), torch.eye(4)


def _one_process_batches(lengths, keys, batch):
    out = []
    for s, n in enumerate(lengths):
        model = _FakeModel()
        seq = MonoRecSequence(model, 2, 1, batch, graphed=False, device="cpu", keys=None if keys is None else keys[s])
        for f in range(n):
            if seq.needs(f):
                seq.push(*_frame(f))
            else:
                seq.skip()
        seq.flush()
        out.append(model.batches)
    return out


def _key_lists(lengths, seed):
    rng = random.Random(seed)
    masks = [{str(k): rng.random() < 0.6 for k in range(n)} for n in lengths]
    return [loader_keys(n, 2, 1, index_masks=[m]) for n, m in zip(lengths, masks)]


CASES = [([40], None), ([13, 10], None), ([3, 40, 1, 17], None), ([30, 25], "keys"), ([9], None), ([6, 5], "keys")]


@pytest.mark.parametrize("lengths,keyed", CASES, ids=lambda v: "-".join(map(str, v)) if isinstance(v, list) else str(v))
@pytest.mark.parametrize("kind", [{"eval_batch": 3}, {"buffer_length": 5}], ids=["eval", "export"])
@pytest.mark.parametrize("lanes", [1, 2, 3, 5, 8])
def test_lanes_push_each_needed_frame_once(lengths, keyed, kind, lanes):
    batch = 4
    keys = _key_lists(lengths, seed=len(lengths)) if keyed else None
    plan = LanePlan(lengths, 2, 1, batch, lanes, keys=keys, **kind)
    # lane r's slices are rank r's
    for r in range(lanes):
        assert plan.slices[r] == shard_sequences(lengths, 2, 1, batch, r, lanes, keys=keys, **kind)
    # the read order visits every frame some lane needs, once
    assert len(plan.order) == len(set(plan.order)) == len(plan.users)
    assert set(plan.order) == set(plan.users)
    feed = _CpuLanes(plan, keys, batch)
    for s, n in plan.order:
        feed.push(s, n, *_frame(n))
    feed.flush()
    whole = _one_process_batches(lengths, keys, batch)
    for r in range(lanes):
        # every frame the lane's sequences need (`needs`) is pushed to it once, in order, and no other frame
        need = []
        for sl in plan.slices[r]:
            probe = MonoRecSequence(_FakeModel(), 2, 1, batch, graphed=False, device="cpu", first_frame=sl.frames[0],
                                    key_end=sl.run[1], keys=None if keys is None else keys[sl.sequence])
            need += [(sl.sequence, n) for n in range(*sl.frames) if probe.needs(n)]
        assert feed.logs[r]["pushed"] == need, r
        # the lane runs exactly its slices' key frames, in batches of the one-process run
        run = [(sl.sequence, k) for sl in plan.slices[r]
               for k in (range(*sl.run) if keys is None else [k for k in keys[sl.sequence] if sl.run[0] <= k < sl.run[1]])]
        assert feed.logs[r]["run"] == run, r
        assert all(any(b in w for w in whole) for b in feed.models[r].batches), r
    assert not feed._held


def test_a_lane_without_a_slice_and_more_lanes_than_batches():
    """9 key frames make 3 model batches of 4: with 8 lanes, some lanes get no slice and push nothing."""
    plan = LanePlan([11], 2, 1, 4, 8, eval_batch=2)
    assert any(not sl for sl in plan.slices) and any(plan.slices)
    feed = _CpuLanes(plan, None, 4)
    for s, n in plan.order:
        feed.push(s, n, *_frame(n))
    feed.flush()
    for r, sl in enumerate(plan.slices):
        if not sl:
            assert feed.logs[r] == {"pushed": [], "run": []}
    assert sorted({k for log in feed.logs for k in log["run"]}) == [(0, k) for k in range(1, 10)]


def test_push_out_of_order_and_early_flush_raise():
    plan = LanePlan([20], 2, 1, 4, 2, eval_batch=2)
    feed = _CpuLanes(plan, None, 4)
    s, n = plan.order[1]
    with pytest.raises(ValueError):
        feed.push(s, n, *_frame(n))
    with pytest.raises(ValueError):
        feed.flush()


@pytest.mark.parametrize("lengths,keyed", CASES, ids=lambda v: "-".join(map(str, v)) if isinstance(v, list) else str(v))
@pytest.mark.parametrize("lanes", [1, 2, 3, 8])
def test_merged_rows_come_out_in_global_batch_order(lengths, keyed, lanes):
    """Each lane tags its evaluater batches from its shard's position; gathered in any order, sort_rows puts them in global
    batch order, each once, and refuses rows that do not tile the run."""
    eb = 3
    keys = _key_lists(lengths, seed=1) if keyed else None
    total = sum(len(range(1, n - 1)) if keys is None else len(k) for n, k in zip(lengths, keys or [None] * len(lengths)))
    rows = []
    for r in range(lanes):
        shard = shard_sequences(lengths, 2, 1, 4, r, lanes, eval_batch=eb, keys=keys)
        emitted = sum(len(range(*sl.emit)) if keys is None else
                      len([k for k in keys[sl.sequence] if sl.emit[0] <= k < sl.emit[1]]) for sl in shard)
        if not shard:
            continue
        first = shard[0].position // eb
        for i in range(-(-emitted // eb)):
            g = first + i
            size = min(eb, total - g * eb)
            rows.append([g, size, 100.0 * g, -g])
    random.Random(lanes).shuffle(rows)
    got, tags = sort_rows(torch.tensor(rows, dtype=torch.float64).reshape(-1, 4))
    G = -(-total // eb)
    assert tags[:, 0].tolist() == list(range(G))
    assert tags[:, 1].tolist() == [eb] * (total // eb) + ([total % eb] if total % eb else [])
    assert got[:, 2].tolist() == [100.0 * g for g in range(G)]
    if G > 1:
        with pytest.raises(RuntimeError):
            sort_rows(torch.tensor([row for row in rows if row[0] != 0], dtype=torch.float64).reshape(-1, 4))
    with pytest.raises(RuntimeError):
        sort_rows(torch.tensor(rows + rows[:1], dtype=torch.float64).reshape(-1, 4))


def test_lane_evaluater_log_is_the_drivers():
    shard = shard_sequences([20], 2, 1, 4, 0, 2, eval_batch=2)
    ev = SequenceEvaluater(None, ["abs_rel_sparse_metric"], 2, group=LANE, shard=shard)
    with pytest.raises(ValueError):
        ev.log()
    assert tuple(ev.tagged_rows(torch.device("cpu")).shape) == (0, 3)


def test_plan_arguments():
    with pytest.raises(ValueError):
        LanePlan([10], 2, 1, 4, 0, eval_batch=2)
    with pytest.raises(ValueError):
        LanePlan([10], 2, 1, 4, 2)                      # neither eval_batch nor buffer_length
    assert list(itertools.chain(*LanePlan([10], 2, 1, 4, 1, eval_batch=2).frames)) == [(0, 0, n) for n in range(10)]
