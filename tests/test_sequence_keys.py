"""The KITTI loader's optional inputs over a frame stream, on the CPU: the key-frame list of `use_index_mask` / annotated lidar
(sequence.loader_keys, pinned on the unmodified loader: tests/golden/loader_keys.json), MonoRecSequence with a key list,
stereo frames and moving-object masks (with a fake model), and dist.shard_sequences with key lists."""
import json
import random

import pytest
import torch

from monorec_b200.dist import shard_sequences
from monorec_b200.sequence import MonoRecSequence, loader_keys, neighbour_offsets
from tests.helpers import GOLDEN


# ---- the loader's key frames -------------------------------------------------------------------------------------------
def test_loader_keys_equal_the_reference_loader():
    g = json.loads((GOLDEN / "loader_keys.json").read_text())
    assert len(g["cases"]) == 32
    for case in g["cases"]:
        got_ids, got_seqs = [], []
        for s, n in g["lengths"].items():
            masks = None if case["use_index_mask"] is None else [g["masks"][name][s] for name in case["use_index_mask"]]
            keys = loader_keys(n, case["frame_count"], case["dilation"], case["lidar_depth"], case["annotated_lidar"],
                               index_masks=masks)
            got_ids += keys
            got_seqs += [s] * len(keys)
        assert got_ids == case["image_id"] and got_seqs == case["sequence"], case


def test_loader_keys_examples():
    assert loader_keys(10) == list(range(1, 9)) == loader_keys(10, index_masks=())
    assert loader_keys(20, lidar_depth=True) == list(range(5, 15))             # eval_monorec.json's annotated lidar
    assert loader_keys(20, lidar_depth=True, annotated_lidar=False) == list(range(1, 19))
    assert loader_keys(12, 4, 2) == list(range(4, 8))
    assert loader_keys(10, index_masks=[{"3": True, "4": False, "5": 1}, {"3": True, "5": True, "8": True}]) == [3, 5]
    assert loader_keys(1) == []
    for fc, dil in ((1, 1), (2, 1), (3, 2), (4, 2)):
        offs = neighbour_offsets(fc, dil)
        assert loader_keys(30, fc, dil) == list(range(-min(0, min(offs)), 30 - max(offs)))


# ---- MonoRecSequence with a key list, stereo frames and masks -----------------------------------------------------------
class _FakeModel:
    """Records the batch dicts; result = the key frame's image (filled with its sequence index)."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self, **attrs):
        self.__dict__.update(attrs)
        self.batches = []

    def __call__(self, data):
        self.batches.append({k: ([t.clone() for t in v] if isinstance(v, list) else v.clone()) for k, v in data.items()})
        data["result"] = data["keyframe"][:, :1] * 1.0
        data["cv_mask"] = data["mvobj_mask"].clone() if self.pretrain_mode == 3 else data["result"] * 0
        return data


def _frame(n, H=2, W=3):
    pose, K = torch.eye(4), torch.eye(4)
    pose[0, 3], K[0, 2] = float(n), float(n)
    return torch.full((3, H, W), float(n)), pose, K


def _stereo(n, H=2, W=3):
    pose, K = torch.eye(4), torch.eye(4)
    pose[1, 3], K[1, 2] = float(n) + 0.5, float(n) + 0.25
    return torch.full((3, H, W), -float(n)), pose, K


def _mask(n, H=2, W=3):
    return torch.arange(H * W, dtype=torch.float32).view(1, H, W) + 100 * n


def _run(seq, n_frames, skip=False, stereo=False, mvobj=False, target=False):
    out = []
    for n in range(n_frames):
        if skip and not seq.needs(n):
            seq.skip()
            continue
        kw = {}
        if stereo:
            kw["stereo"] = _stereo(n)
        if mvobj:
            kw["mvobj_mask"] = _mask(n)
        if target:
            kw["target"] = _mask(n) * -1
        out += [(i, {k: v.clone() for k, v in o.items()}) for i, o in seq.push(*_frame(n), **kw)]
    return out + seq.flush()


@pytest.mark.parametrize("fc,dil,bs", [(2, 1, 4), (4, 2, 3), (1, 1, 2), (3, 1, 1)])
@pytest.mark.parametrize("skip", [False, True], ids=["push_all", "skip"])
def test_key_list_batches_and_inputs(fc, dil, bs, skip):
    """Listed key frames only, in list order, batch_size consecutive listed key frames per batch (the last one short, at the
    push that completes it), each with its own stereo frame, mask and target and its neighbours' frames."""
    offs = neighbour_offsets(fc, dil)
    rng = random.Random(fc * 10 + dil)
    every = loader_keys(60, fc, dil)
    keys = sorted(rng.sample(every, 17))
    model = _FakeModel(use_stereo=True, pretrain_mode=3)
    seq = MonoRecSequence(model, fc, dil, bs, graphed=False, device="cpu", keys=keys, stereo=True, mvobj_masks=True)
    out = _run(seq, 60, skip=skip, stereo=True, mvobj=True, target=True)
    assert [i for i, _ in out] == keys
    assert [[int(v) for v in b["keyframe"][:, 0, 0, 0]] for b in model.batches] == \
        [keys[b:b + bs] for b in range(0, len(keys), bs)]
    for b in model.batches:
        for j, k in enumerate(int(v) for v in b["keyframe"][:, 0, 0, 0]):
            img, pose, K = _stereo(k)
            assert torch.equal(b["stereoframe"][j], img) and torch.equal(b["stereoframe_pose"][j], pose)
            assert torch.equal(b["stereoframe_intrinsics"][j], K)
            assert torch.equal(b["mvobj_mask"][j], _mask(k)) and torch.equal(b["target"][j], -_mask(k))
            assert [float(f[j, 0, 0, 0]) for f in b["frames"]] == [k + d for d in offs]
            assert [float(p[j, 0, 3]) for p in b["poses"]] == [k + d for d in offs]
            assert [float(q[j, 0, 2]) for q in b["intrinsics"]] == [k + d for d in offs]
    for i, o in out:
        assert torch.equal(o["cv_mask"], _mask(i)[None]) and torch.equal(o["stereoframe"], _stereo(i)[0][None])
        assert o["mvobj_mask"].shape == (1, 1, 2, 3) and o["target"].shape == (1, 1, 2, 3)


def test_default_keys_give_the_loader_range_with_stereo_and_masks():
    model = _FakeModel()
    seq = MonoRecSequence(model, 2, 1, 4, graphed=False, device="cpu", stereo=True, mvobj_masks=True)
    out = _run(seq, 13, stereo=True, mvobj=True)
    assert [i for i, _ in out] == list(range(1, 12))
    assert all(torch.equal(o["mvobj_mask"], _mask(i)[None]) for i, o in out)
    assert all(torch.equal(o["stereoframe_pose"], _stereo(i)[1][None]) for i, o in out)


class _Watched(torch.Tensor):
    """A frame image that records the sequence indices it is copied from."""
    copied = []

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        if func is torch.Tensor.copy_ and isinstance(args[1], _Watched):
            with torch._C.DisableTorchFunctionSubclass():
                cls.copied.append(int(args[1].reshape(-1)[0]))
        return super().__torch_function__(func, types, args, kwargs or {})


def test_frames_no_key_frame_needs_are_not_copied():
    fc, dil, bs = 4, 2, 3
    offs = [0] + neighbour_offsets(fc, dil)
    keys = [4, 5, 20, 33, 34, 35, 36, 50]
    needed = sorted({k + d for k in keys for d in offs})
    seq = MonoRecSequence(_FakeModel(), fc, dil, bs, graphed=False, device="cpu", keys=keys)
    assert [n for n in range(60) if seq.needs(n)] == needed
    _Watched.copied = []
    out = []
    for n in range(60):
        image, pose, K = _frame(n)
        out += seq.push(image.as_subclass(_Watched), pose, K)
    out += seq.flush()
    assert [i for i, _ in out] == keys
    assert _Watched.copied == needed                            # each needed frame once, no other
    with pytest.raises(ValueError):
        MonoRecSequence(_FakeModel(), fc, dil, bs, graphed=False, device="cpu", keys=keys).skip()    # frame 0 is needed


@pytest.mark.parametrize("gap", [1, 7, 1000, 20000])
def test_ring_is_bounded_by_the_batch_for_any_gap(gap):
    """Key frames in clusters `gap` frames apart: the ring holds batch_size * (F + 1) + span frames whatever the gap, and
    never more frames than that are live."""
    fc, dil, bs = 2, 1, 4
    keys = sorted({c * (gap + 6) + 1 + d for c in range(5) for d in (0, 2, 3)})
    seq = MonoRecSequence(_FakeModel(), fc, dil, bs, graphed=False, device="cpu", keys=keys)
    assert seq.ring_len == bs * (fc + 1) + 2
    out, live = [], 0
    for n in range(keys[-1] + 2):
        if not seq.needs(n):
            seq.skip()
            continue
        out += seq.push(*_frame(n))
        live = max(live, len(seq._slot))
        assert seq._rings[0].shape[0] == seq.ring_len
    assert [i for i, _ in out] == keys and seq.flush() == []
    assert live <= seq.ring_len


def test_stereo_and_mask_arguments():
    with pytest.raises(NotImplementedError):
        MonoRecSequence(_FakeModel(use_stereo=True), device="cpu", mvobj_masks=True)
    with pytest.raises(NotImplementedError):
        MonoRecSequence(_FakeModel(pretrain_mode=3), device="cpu", stereo=True)
    MonoRecSequence(_FakeModel(use_stereo=True, pretrain_mode=3), device="cpu", stereo=True, mvobj_masks=True)
    seq = MonoRecSequence(_FakeModel(), 2, 1, 2, graphed=False, device="cpu")
    with pytest.raises(ValueError):
        seq.push(*_frame(0), stereo=_stereo(0))                 # stereo frames without stereo=True
    seq = MonoRecSequence(_FakeModel(), 2, 1, 2, graphed=False, device="cpu", stereo=True, mvobj_masks=True)
    seq.push(*_frame(0))                                        # frame 0 is no key frame: its stereo frame is not needed
    with pytest.raises(ValueError):
        seq.push(*_frame(1), mvobj_mask=_mask(1))               # key frame 1 without its stereo frame
    with pytest.raises(ValueError):
        seq.push(*_frame(1), stereo=_stereo(1), mvobj_mask=torch.zeros(1, 3, 3))
    with pytest.raises(ValueError):
        MonoRecSequence(_FakeModel(), 2, 1, 2, device="cpu", keys=[0, 3])          # key frame 0 lacks its neighbour
    with pytest.raises(ValueError):
        MonoRecSequence(_FakeModel(), 2, 1, 2, device="cpu", keys=[3, 3])


# ---- shard_sequences with key lists --------------------------------------------------------------------------------------
LENGTHS = [[13, 10], [5], [3, 40, 1, 17], [64, 63, 2], [9, 9, 9]]
SHAPES = [(2, 1, 4), (4, 2, 3), (2, 1, 1), (1, 1, 2)]


def _key_lists(lengths, fc, dil, seed):
    """Random sub-lists of each sequence's key frames (some empty, some whole), with the loader's lidar range for one."""
    rng = random.Random(seed)
    out = []
    for s, n in enumerate(lengths):
        keys = loader_keys(n, fc, dil, lidar_depth=s == 1)
        out.append(keys if s == 2 else sorted(rng.sample(keys, rng.randint(0, len(keys)))))
    return out


@pytest.mark.parametrize("kind", [dict(eval_batch=1), dict(eval_batch=3), dict(buffer_length=5), dict(buffer_length=3)],
                         ids=["eval1", "eval3", "vote5", "vote3"])
def test_shards_with_key_lists_cover_every_listed_key_frame_once(kind):
    for (lengths, (fc, dil, bs)), seed in zip([(a, b) for a in LENGTHS for b in SHAPES], range(100)):
        keys = _key_lists(lengths, fc, dil, seed)
        if "eval_batch" in kind:
            every = [(s, k) for s, ks in enumerate(keys) for k in ks]
        else:
            before, after = kind["buffer_length"] // 2, kind["buffer_length"] - 1 - kind["buffer_length"] // 2
            every = [(s, k) for s, ks in enumerate(keys) for p, k in enumerate(ks) if before <= p < len(ks) - after]
        for world in range(1, 9):
            emitted = []
            for rank in range(world):
                mine = []
                for sl in shard_sequences(lengths, fc, dil, bs, rank, world, keys=keys, **kind):
                    ks = keys[sl.sequence]
                    run = [k for k in ks if sl.run[0] <= k < sl.run[1]]
                    emit = [k for k in ks if sl.emit[0] <= k < sl.emit[1]]
                    # whole one-process model batches of listed key frames
                    p0 = ks.index(run[0])
                    assert p0 % bs == 0 and run == ks[p0:p0 + len(run)]
                    assert len(run) % bs == 0 or p0 + len(run) == len(ks)
                    assert sl.run == (run[0], run[-1] + 1) and sl.emit == (emit[0], emit[-1] + 1)
                    offs = neighbour_offsets(fc, dil)
                    assert sl.frames == (run[0] + min(0, min(offs)), run[-1] + max(offs) + 1)
                    assert sl.position == every.index((sl.sequence, emit[0]))
                    if "eval_batch" in kind:
                        # a rank starts on an evaluater batch boundary of the listed key frames
                        assert mine or sl.position % kind["eval_batch"] == 0
                    else:
                        q = ks.index(emit[0])
                        assert ks.index(run[0]) <= q - before and ks.index(emit[-1]) + after <= ks.index(run[-1])
                    mine += [(sl.sequence, k) for k in emit]
                emitted += mine
            assert emitted == every, (lengths, fc, dil, bs, world)


@pytest.mark.parametrize("fc,dil,bs", SHAPES)
def test_sliced_key_list_sequences_run_the_one_process_batches(fc, dil, bs):
    lengths = [3, 40, 1, 17]
    keys = _key_lists(lengths, fc, dil, seed=fc + bs)
    whole = {}
    for s, n in enumerate(lengths):
        model = _FakeModel()
        seq = MonoRecSequence(model, fc, dil, bs, graphed=False, device="cpu", keys=keys[s])
        assert [i for i, _ in _run(seq, n)] == keys[s]
        whole[s] = [[int(v) for v in b["keyframe"][:, 0, 0, 0]] for b in model.batches]
    for world, kind in ((2, dict(eval_batch=3)), (3, dict(buffer_length=5)), (5, dict(eval_batch=1))):
        for rank in range(world):
            for sl in shard_sequences(lengths, fc, dil, bs, rank, world, keys=keys, **kind):
                model = _FakeModel()
                seq = MonoRecSequence(model, fc, dil, bs, graphed=False, device="cpu", keys=keys[sl.sequence],
                                      first_frame=sl.frames[0], key_end=sl.run[1])
                out = []
                for n in range(*sl.frames):
                    out += seq.push(*_frame(n)) if seq.needs(n) else seq.skip() or []
                out += seq.flush()
                batches = [[int(v) for v in b["keyframe"][:, 0, 0, 0]] for b in model.batches]
                assert all(b in whole[sl.sequence] for b in batches), (sl, batches)
                assert [i for i, _ in out] == [k for k in keys[sl.sequence] if sl.run[0] <= k < sl.run[1]]


def test_shard_key_list_arguments():
    with pytest.raises(ValueError):
        shard_sequences([10, 12], 2, 1, 4, 0, 1, eval_batch=2, keys=[[1, 2]])       # one list for two sequences
    with pytest.raises(ValueError):
        shard_sequences([10], 2, 1, 4, 0, 1, eval_batch=2, keys=[[1, 9]])           # key frame 9 lacks frame 10
    assert shard_sequences([10], 2, 1, 4, 0, 1, eval_batch=2, keys=[None]) == \
        shard_sequences([10], 2, 1, 4, 0, 1, eval_batch=2)
