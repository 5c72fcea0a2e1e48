"""evaluate.py's list of models split over lanes (lanes.MultiDeviceModelsEvaluater) and over ranks (MultiModelEvaluater with
`group` / `shard`) without a GPU: the argument checks, the sharing groups every lane runs with, and the split runs against
one process with stub models.

The metric passes and their fold are CUDA kernels; here they are CPU stand-ins whose rows depend on every key frame of an
evaluater batch and whose fold depends on the order of the batches, so a key frame evaluated twice, missed, cut into
another batch or folded out of order changes the log.  Everything else (the lanes' feed, the slices, the key frames each
slice evaluates, the batch tags, the row gather over gloo, the sort and the log) is the library's."""
import os
import socket
import types
import warnings

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from monorec_b200.dist import shard_sequences

NAMES = ["abs_rel_sparse_metric", "a1_sparse_metric", "abs_rel_metric", "sc_inv_metric"]
LENGTHS = [13, 10]                              # 11 + 8 key frames
H, W = 4, 6


def _model(**kw):
    from monorec_b200.model import MonoRecModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # (no ImageNet weights in the hub cache: randomly initialised trunk)
        return MonoRecModel(**kw).eval()


@pytest.fixture(scope="module")
def three():
    """Two checkpoints on one trunk (one cost-volume stage) and a use_ssim=2 model on the same trunk (its own)."""
    a = _model()
    b, c = _model(), _model(use_ssim=2)
    for m in (b, c):
        m._feature_extractor.load_state_dict(a._feature_extractor.state_dict())
    return [a, b, c]


# ---- arguments and sharing groups --------------------------------------------------------------------------------------
def test_arguments(three):
    from monorec_b200.lanes import MultiDeviceModelsEvaluater
    from monorec_b200.models_eval import MultiModelEvaluater
    with pytest.raises(ValueError, match="empty"):
        MultiDeviceModelsEvaluater([], ["cpu", "cpu"], LENGTHS, NAMES, 2)
    elsewhere = _model().to("meta")
    with pytest.raises(ValueError, match="meta"):
        MultiDeviceModelsEvaluater([three[0], elsewhere], ["cpu", "cpu"], LENGTHS, NAMES, 2)
    shard = shard_sequences(LENGTHS, 2, 1, 4, 1, 2, eval_batch=2)
    with pytest.raises(ValueError, match="group and shard"):
        MultiModelEvaluater(three, NAMES, 2, device="cpu", shard=shard)
    with pytest.raises(ValueError, match="group and shard"):
        MultiModelEvaluater(three, NAMES, 2, device="cpu", group=object())
    with pytest.raises(ValueError, match="eval_batch"):
        MultiModelEvaluater(three, NAMES, 3, device="cpu", group=object(), shard=shard)   # not cut for batches of 3
    with pytest.raises(ValueError, match="next_sequence"):
        MultiModelEvaluater(three, NAMES, 2, device="cpu", group=object(), shard=shard, keys=[1, 2, 3])
    ev = MultiModelEvaluater(three, NAMES, 2, device="cpu", group=object(), shard=shard, graphed=False)
    assert ev.seq is None
    with pytest.raises(ValueError, match="no sequence"):
        ev.push(torch.zeros(3, H, W), torch.eye(4), torch.eye(4), torch.zeros(1, H, W))
    sl = shard[0]
    with pytest.raises(ValueError, match="do not cover"):
        ev.next_sequence(first_frame=sl.frames[0], key_end=sl.emit[1] - 1)


def test_every_lane_runs_the_groups_of_the_given_models(three):
    from monorec_b200.lanes import MultiDeviceModelsEvaluater
    from monorec_b200.models_eval import share_groups
    groups = share_groups(three)
    assert groups == ([[0, 1], [2]], [[0, 1, 2]])
    run = MultiDeviceModelsEvaluater(three, ["cpu"] * 3, LENGTHS, NAMES, 2, seq_batch=4, graphed=False)
    assert (run.cv_groups, run.trunk_groups) == groups
    lanes = [ev for ev in run.evaluaters if ev is not None]
    assert len(lanes) == 3
    for ev in lanes:
        assert (ev.cv_groups, ev.trunk_groups) == groups
        assert ev._forward.cv_groups == groups[0] and ev._forward.trunk_groups == groups[1]
        assert ev.models == three                 # the models' own device: no copies


def test_replicas_that_share_otherwise_are_refused(three, monkeypatch):
    """A replica is a copy of its model, so its groups are the model's; the driver checks that instead of assuming it."""
    from monorec_b200 import lanes
    real, calls = lanes.share_groups, []

    def second_call_differs(models):
        calls.append(1)
        cv, trunk = real(models)
        return (cv, trunk) if len(calls) == 1 else ([[i] for i in range(len(models))], trunk)
    monkeypatch.setattr(lanes, "share_groups", second_call_differs)
    with pytest.raises(RuntimeError, match="replicas"):
        lanes.MultiDeviceModelsEvaluater(three, ["cpu", "cpu"], LENGTHS, NAMES, 2, graphed=False)


# ---- split runs with stub models and CPU stand-ins of the metric passes -------------------------------------------------
class _Stub(torch.nn.Module):
    """The three stages of a MonoRecModel in a few CPU operations: cost-volume configuration `cv`, trunk `trunk`, head
    weight `head`."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self, cv, trunk, head):
        super().__init__()
        self.cv, self.trunk = cv, trunk
        self.head = torch.nn.Parameter(torch.tensor(float(head)))

    def _stage_cost_volume(self, d):
        d["cost_volume"] = (d["keyframe"][:, :1] - sum(f[:, :1] for f in d["frames"])) * (1 + self.cv)
        return d

    def _stage_trunk(self, d):
        return {"image_features": d["keyframe"][:, 1:2] * self.trunk}

    def _stage_heads(self, d):
        d["result"] = (d["cost_volume"] * 0.5 + d["image_features"]).abs() + self.head.detach()
        return d


def _stubs():
    return [_Stub(0, 1, 0.25), _Stub(0, 1, 0.5), _Stub(1, 1, 0.75)]


def _groups_of_stubs():
    return dict(cost_volume_key=lambda m: m.cv, same_trunk=lambda a, b: a.trunk == b.trunk)


def _rows(pred, target, group, columns):
    """One row per group of `group` images: per column j, (j + 1) times the mean |pred - target| over the pixels with a
    target (NaN for a group without one)."""
    G = pred.shape[0] // group
    valid = (target > 0).reshape(G, -1).to(torch.float32)
    err = ((pred - target).abs().reshape(G, -1) * valid).sum(1) / valid.sum(1)
    return torch.stack([err * (j + 1) for j in range(columns)], 1)


def _accumulate(values, sizes, state):
    """An order-dependent fold of the rows into [totals, valid counts, running values, images]."""
    m = values.shape[1]
    for v, s in zip(values.to(torch.float64), sizes):
        ok = ~torch.isnan(v)
        state[:m] += torch.where(ok, v, 0)
        state[m:2 * m] += ok
        state[2 * m:3 * m] = state[2 * m:3 * m] * 0.5 + torch.where(ok, v, 0) * s
        state[3 * m] += s
    return state


def _add(self, result, target, mvobj_mask=None):
    """SequenceEvaluater.add's batching without its CUDA check."""
    parts = [result.to(torch.float32), target.to(torch.float32)]
    if self._open is not None:
        parts = [torch.cat([o, p]) for o, p in zip(self._open, parts)]
    n, bs = parts[0].shape[0], self.batch_size
    full = n // bs * bs
    if full:
        self._evaluate([p[:full] for p in parts], [bs] * (full // bs))
    self._open = [p[full:].clone() for p in parts] if full < n else None


def _stand_ins(setattr_):
    from monorec_b200 import evaluation, models_eval
    setattr_(evaluation, "M", types.SimpleNamespace(
        sparse_metrics_grouped_impl=lambda pred, gt, mask, roi, max_d, all_valid, g: _rows(pred, gt, g, 7),
        dense_metrics_grouped_impl=lambda pred, gt, roi, min_inv, g: _rows(pred, gt, g, 12),
        median_scaling_impl=lambda pred, gt: pred * 1.5,
        eval_accumulate_impl=_accumulate))
    setattr_(evaluation.SequenceEvaluater, "add", _add)
    for k, v in _groups_of_stubs().items():
        setattr_(models_eval, k, v)


def _stream(s, n):
    g = torch.Generator().manual_seed(40 + s)
    images = torch.rand(n, 3, H, W, generator=g) - 0.5
    targets = torch.rand(n, 1, H, W, generator=g) * 0.2 + 0.01
    targets[torch.rand(n, 1, H, W, generator=g) > 0.5] = 0.0
    targets[3] = 0.0                                    # a key frame without ground truth
    pose = torch.eye(4)
    return [(images[i], pose, pose, targets[i]) for i in range(n)]


STREAMS = [_stream(s, n) for s, n in enumerate(LENGTHS)]


def _one_process(eval_batch, median_scaling):
    from monorec_b200.models_eval import MultiModelEvaluater
    ev = MultiModelEvaluater(_stubs(), NAMES, eval_batch, median_scaling=median_scaling, seq_batch=4, device="cpu",
                             graphed=False)
    assert ev.cv_groups == [[0, 1], [2]] and ev.trunk_groups == [[0, 1, 2]]
    for s, frames in enumerate(STREAMS):
        if s:
            ev.next_sequence()
        for f in frames:
            ev.push(*f)
    ev.flush()
    return ev.logs()


def _same_logs(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert g["valid_batches"] == r["valid_batches"]
        for k in ("metrics", "metrics_correct"):
            torch.testing.assert_close(torch.tensor(g[k], dtype=torch.float64), torch.tensor(r[k], dtype=torch.float64),
                                       rtol=0, atol=0, equal_nan=True)


CASES = [(3, False), (2, True), (5, False)]


@pytest.mark.parametrize("eval_batch,median_scaling", CASES)
@pytest.mark.parametrize("lanes", [1, 2, 3, 5])
def test_lanes_equal_one_process(monkeypatch, eval_batch, median_scaling, lanes):
    from monorec_b200.lanes import MultiDeviceModelsEvaluater
    _stand_ins(monkeypatch.setattr)
    ref = _one_process(eval_batch, median_scaling)
    assert all(0 < log["valid_batches"] for log in ref) and ref[0]["metrics"] != ref[1]["metrics"]
    run = MultiDeviceModelsEvaluater(_stubs(), ["cpu"] * lanes, LENGTHS, NAMES, eval_batch, seq_batch=4,
                                     median_scaling=median_scaling, graphed=False)
    for s, n in run.order:
        run.push(s, n, *STREAMS[s][n])
    run.flush()
    _same_logs(run.logs(), ref)
    results = run.results({"dataset_dir": "data"})
    assert [r["result"]["metrics_info"] for r in results] == [NAMES] * 3
    _same_logs([r["result"] for r in results], ref)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from monorec_b200.models_eval import MultiModelEvaluater
    _stand_ins(setattr)
    out = []
    for eb, ms in CASES:
        shard = shard_sequences(LENGTHS, 2, 1, 4, rank, world, eval_batch=eb)
        ev = MultiModelEvaluater(_stubs(), NAMES, eb, median_scaling=ms, seq_batch=4, device="cpu", graphed=False,
                                 group=dist.group.WORLD, shard=shard)
        for sl in shard:
            ev.next_sequence(first_frame=sl.frames[0], key_end=sl.run[1])
            for n in range(*sl.frames):
                ev.push(*STREAMS[sl.sequence][n])
        ev.flush()
        out.append((ev.logs(), [r["result"] for r in ev.results({"dataset_dir": "data"})]))
    q.put((rank, out))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_ranks_over_gloo_equal_one_process(monkeypatch, world):
    """Every rank's logs() and results() are the one-process logs (world 3 with evaluater batch 5: a rank may emit no
    batch at all)."""
    _stand_ins(monkeypatch.setattr)
    refs = [_one_process(eb, ms) for eb, ms in CASES]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert sorted(r for r, _ in res) == list(range(world))
    for _, out in res:
        for (logs, results), ref in zip(out, refs):
            _same_logs(logs, ref)
            _same_logs(results, ref)
