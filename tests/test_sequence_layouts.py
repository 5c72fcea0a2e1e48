"""Frame layouts of the reference's other loaders, on the CPU: kitti_layout (offset_d, max_length), tum_mono_vo_layout and
robotcar_layout against the unmodified loaders' items (tests/golden/loader_streams.json), the key frames whose sources
fall outside the sequence, MonoRecSequence fed by a recording stub model, and the sharded / laned splits (shard_sequences,
LanePlan, gloo worlds of 2 and 3 ranks) against one process."""
import itertools
import json
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from monorec_b200.dist import shard_sequences
from monorec_b200.lanes import LanePlan
from monorec_b200.sequence import (FrameLayout, MonoRecSequence, kitti_layout, loader_keys, needs_frame,
                                   neighbour_offsets, robotcar_layout, tum_mono_vo_layout)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return json.loads((golden_dir / "loader_streams.json").read_text())


def _kitti_layouts(g, case, drop):
    masks = case["use_index_mask"]
    return [kitti_layout(n, case["frame_count"], case["dilation"], offset_d=case["offset_d"], max_length=case["max_length"],
                         index_masks=None if masks is None else [g["masks"][m][s] for m in masks], drop_outside=drop)
            for s, n in g["lengths"].items()]


def _tum_layouts(g, case, drop=None):
    return [tum_mono_vo_layout(g["length"], case["frame_count"], case["dilation"], max_length=case["max_length"],
                               keyframe_indices=g["depth_frames"] if case["only_keyframes"] else None)]


def _robotcar_layouts(g, case, drop):
    return [robotcar_layout(n, case["frame_count"], case["dilation"], drop_outside=drop) for n in g["lengths"]]


LOADERS = {"kitti": _kitti_layouts, "tum_mono_vo": _tum_layouts, "robotcar": _robotcar_layouts}


def _lengths(g):
    return list(g["lengths"].values()) if isinstance(g.get("lengths"), dict) else g.get("lengths", [g.get("length")])


def _seq(g, it):
    names = list(g["lengths"]) if isinstance(g.get("lengths"), dict) else None
    return names.index(it["sequence"]) if names else it["sequence"]


def _split(g, case):
    """The case's items the loader reads inside the sequence, per sequence as (key, sources), and the others: those that
    read a wrapped frame or raise IndexError."""
    clean, outside = [[] for _ in _lengths(g)], []
    for it in case["items"]:
        if "error" in it or it["wrapped"]:
            outside.append(it)
        else:
            clean[_seq(g, it)].append((it["key"], it["sources"]))
    return clean, outside


@pytest.mark.parametrize("loader", list(LOADERS))
def test_layouts_reproduce_the_loaders_items(golden, loader):
    """The layout's key frames, each with its sources in list order, are the loader's items, bit for bit; the items the
    layout leaves out (drop_outside) are exactly those for which the loader reads a wrapped frame or fails, and a wrapped
    item holds the frames Python's negative index gives."""
    g = golden[loader]
    lengths = _lengths(g)
    n_outside = 0
    for case in g["cases"]:
        layouts = LOADERS[loader](g, case, True)
        clean, outside = _split(g, case)
        for s, lay in enumerate(layouts):
            assert isinstance(lay, FrameLayout)
            assert [(k, [k + u for u in lay.offsets]) for k in lay.keys] == clean[s], (case, s)
        assert len(case["items"]) == sum(len(lay.keys) for lay in layouts) + len(outside)
        for it in outside:
            if "error" not in it:
                s = _seq(g, it)
                offs = layouts[s].offsets
                assert it["sources"] == [(it["key"] + u) % lengths[s] for u in offs]
                assert min(it["key"] + u for u in offs) < 0
        n_outside += len(outside)
    assert (n_outside > 0) == (loader != "tum_mono_vo")      # the golden holds wrapped and failing items


@pytest.mark.parametrize("loader", ["kitti", "robotcar"])
def test_keys_outside_the_sequence_raise_or_are_dropped(golden, loader):
    """Without drop_outside, a case with a wrapped or failing item raises ValueError naming the first such key frame and
    the frame the loader reads in its place; a case without one gives the drop_outside layout."""
    g = golden[loader]
    lengths = _lengths(g)
    for case in g["cases"]:
        _, outside = _split(g, case)
        if not outside:
            assert LOADERS[loader](g, case, False) == LOADERS[loader](g, case, True)
            continue
        with pytest.raises(ValueError, match="drop_outside=True") as e:
            LOADERS[loader](g, case, False)
        first = outside[0]
        if "error" in first:
            assert "IndexError" in str(e.value)
        else:
            s, k = _seq(g, first), first["key"]
            lo = min(LOADERS[loader](g, case, True)[s].offsets)
            assert f"key frame {k} needs frame {k + lo}, before the sequence" in str(e.value)
            assert f"wraps to frame {k + lo + lengths[s]}" in str(e.value)
            assert k + lo + lengths[s] in first["sources"]


def test_default_layout_is_the_kitti_loaders():
    for n, fc, dil in itertools.product((0, 5, 23), (1, 2, 3, 4), (1, 2)):
        lay = kitti_layout(n, fc, dil)
        assert list(lay.offsets) == neighbour_offsets(fc, dil) and list(lay.keys) == loader_keys(n, fc, dil)
    masks = [{str(i): i % 3 != 0 for i in range(30)}]
    assert list(kitti_layout(30, 2, 1, index_masks=masks, lidar_depth=True).keys) == loader_keys(30, 2, 1, True, True, masks)
    assert kitti_layout(30, 2, 1, max_length=4).keys == (1, 2, 3, 4)
    assert robotcar_layout(10, 3, drop_outside=True).offsets == (-2, -1, 1, 2)
    assert tum_mono_vo_layout(10, 3, 1).offsets == (-1, 1, 2)
    with pytest.raises(ValueError):
        kitti_layout(10, max_length=-1)
    with pytest.raises(ValueError):
        MonoRecSequence(_Recorder(), device="cpu", keys=[1, 2], layout=kitti_layout(10))


# ---- MonoRecSequence fed by a recording stub ----------------------------------------------------------------------------
class _Recorder:
    """Records every batch's key frames and, per key frame, the frames and poses its dict holds, by the sequence index
    the pushed image and pose carry; result = the key frame's image."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self):
        self.batches = []

    def __call__(self, data):
        keys = [int(v) for v in data["keyframe"][:, 0, 0, 0]]
        self.batches.append(keys)
        data["result"] = data["keyframe"][:, :1] * 1.0
        data["cost_volume"] = torch.stack([f[:, 0, 0, 0] for f in data["frames"]], 1)
        data["cv_mask"] = torch.stack([p[:, 0, 3] for p in data["poses"]], 1)
        return data


def _frame(n, C=3):
    pose = torch.eye(4)
    pose[0, 3] = n
    return torch.full((C, 2, 3), float(n)), pose, torch.eye(4)


def _golden_layouts(golden):
    """(name, length, layout, {key: sources}) for a spread of the golden's layouts, dropped keys left out."""
    picks = [("kitti", lambda c: c["offset_d"] == -1 and c["frame_count"] == 2 and c["dilation"] == 1 and not c["max_length"]
              and c["use_index_mask"] is None),
             ("kitti", lambda c: c["offset_d"] == -2 and c["frame_count"] == 3 and c["dilation"] == 2 and c["max_length"] == 6
              and c["use_index_mask"] == ["mask_a"]),
             ("kitti", lambda c: c["offset_d"] == 1 and c["frame_count"] == 2 and c["dilation"] == 2 and not c["max_length"]
              and c["use_index_mask"] == ["mask_a"]),
             ("tum_mono_vo", lambda c: c["only_keyframes"] and c["frame_count"] == 3 and c["dilation"] == 1),
             ("tum_mono_vo", lambda c: not c["only_keyframes"] and c["frame_count"] == 2 and c["dilation"] == 2
              and c["max_length"] == 5),
             ("robotcar", lambda c: c["frame_count"] == 3 and c["dilation"] == 1),
             ("robotcar", lambda c: c["frame_count"] == 4 and c["dilation"] == 2)]
    out = []
    for loader, pick in picks:
        g = golden[loader]
        case = next(c for c in g["cases"] if pick(c))
        clean, _ = _split(g, case)
        for s, (n, lay) in enumerate(zip(_lengths(g), LOADERS[loader](g, case, True))):
            out.append((f"{loader}-{s}", n, lay, dict((k, src) for k, src in clean[s])))
    return out


@pytest.mark.parametrize("bs", [1, 3])
def test_sequence_feeds_each_key_the_loaders_frames(golden, bs):
    """Every key frame gets exactly the frames and poses the loader lists, in its order, and is emitted at the push of its
    batch's last key frame's latest frame (its own for a causal layout); flush runs nothing more."""
    for name, n, lay, expect in _golden_layouts(golden):
        model = _Recorder()
        seq = MonoRecSequence(model, batch_size=bs, graphed=False, device="cpu", layout=lay)
        hi = max(0, max(lay.offsets))
        got, at = {}, {}
        for f in range(n):
            if not seq.needs(f):
                seq.skip()
                continue
            for i, o in seq.push(*_frame(f)):
                got[i] = ([int(v) for v in o["cost_volume"][0]], [int(v) for v in o["cv_mask"][0]])
                at[i] = f
        assert seq.flush() == []
        assert list(got) == list(lay.keys) == list(expect), name
        for k, (frames, poses) in got.items():
            assert frames == poses == expect[k], (name, k)
        batches = [lay.keys[b:b + bs] for b in range(0, len(lay.keys), bs)]
        assert model.batches == [list(b) for b in batches], name
        for b in batches:
            assert all(at[k] == b[-1] + hi for k in b), (name, b)
        if max(lay.offsets) <= 0 and bs == 1:
            assert all(at[k] == k for k in lay.keys)          # causal: emitted on the push of the key frame itself


def test_causal_layout_with_grayscale_frames_and_graph_free_ring():
    lay = kitti_layout(40, 2, 1, offset_d=-1, drop_outside=True)
    assert lay.offsets == (-2, 0)
    seq = MonoRecSequence(_Recorder(), batch_size=4, graphed=False, device="cpu", layout=lay, use_color=False)
    out = []
    for f in range(40):
        out += seq.push(*_frame(f, C=1))
    assert [i for i, _ in out] == list(lay.keys)
    assert all(o["cost_volume"][0].tolist() == [i - 2, i] for i, o in out)
    assert all(torch.equal(o["keyframe"], torch.full((1, 1, 2, 3), float(i))) for i, o in out)


# ---- the split runs -------------------------------------------------------------------------------------------------------
def _layout_sets(golden):
    """Per-sequence layout lists over several sequences: causal and shifted KITTI, TUM, RobotCar."""
    k = golden["kitti"]
    lens = [31, 7, 24, 2]
    return {
        "kitti-causal": (lens, [kitti_layout(n, 2, 1, offset_d=-1, drop_outside=True) for n in lens]),
        "kitti-shift": (lens, [kitti_layout(n, 3, 2, offset_d=1, drop_outside=True,
                                            index_masks=[{str(i): i % 4 != 1 for i in range(n)}]) for n in lens]),
        "tum": (lens, [tum_mono_vo_layout(n, 3, 2) for n in lens]),
        "tum-keyframes": ([k["lengths"]["00"]], [tum_mono_vo_layout(k["lengths"]["00"], 2, 1,
                                                                    keyframe_indices=[0, 2, 3, 7, 8, 9, 12, 15])]),
        "robotcar": (lens, [robotcar_layout(n, 3, 2, drop_outside=True) for n in lens]),
    }


def _one_process(lengths, layouts, bs):
    whole = {}
    for s, (n, lay) in enumerate(zip(lengths, layouts)):
        model = _Recorder()
        seq = MonoRecSequence(model, batch_size=bs, graphed=False, device="cpu", layout=lay)
        out = []
        for f in range(n):
            out += seq.push(*_frame(f)) if seq.needs(f) else (seq.skip() or [])
        out += seq.flush()
        whole[s] = (model.batches, [(i, o["cost_volume"][0].tolist()) for i, o in out])
    return whole


def _run_slice(lay, bs, sl):
    model = _Recorder()
    seq = MonoRecSequence(model, batch_size=bs, graphed=False, device="cpu", layout=lay, first_frame=sl.frames[0],
                          key_end=sl.run[1])
    out = []
    for f in range(*sl.frames):
        out += seq.push(*_frame(f)) if seq.needs(f) else (seq.skip() or [])
    out += seq.flush()
    return model.batches, [(i, o["cost_volume"][0].tolist()) for i, o in out]


@pytest.mark.parametrize("name", ["kitti-causal", "kitti-shift", "tum", "tum-keyframes", "robotcar"])
def test_shards_and_lanes_run_the_one_process_batches(golden, name):
    """Every slice of shard_sequences(layout=...) runs only batches of the one-process run, with the same frames; the
    emitted key frames tile the one-process list (evaluater batches) or its vote windows (point cloud); LanePlan's
    frames are the slices' needed frames."""
    lengths, layouts = _layout_sets(golden)[name]
    for bs in (1, 3, 4):
        whole = _one_process(lengths, layouts, bs)
        every = [(s, k) for s, lay in enumerate(layouts) for k in lay.keys]
        for world, kind in itertools.product((1, 2, 3, 5), ({"eval_batch": 3}, {"buffer_length": 5})):
            emitted = []
            for rank in range(world):
                for sl in shard_sequences(lengths, 2, 1, bs, rank, world, layout=layouts, **kind):
                    lay = layouts[sl.sequence]
                    batches, out = _run_slice(lay, bs, sl)
                    assert all(b in whole[sl.sequence][0] for b in batches), (name, sl, batches)
                    assert [i for i, _ in out] == [k for k in lay.keys if sl.run[0] <= k < sl.run[1]]
                    ref = dict(whole[sl.sequence][1])
                    assert all(ref[i] == frames for i, frames in out)
                    assert 0 <= sl.frames[0] and sl.frames[1] <= lengths[sl.sequence]
                    emitted += [(sl.sequence, k) for k in lay.keys if sl.emit[0] <= k < sl.emit[1]]
            if "eval_batch" in kind:
                assert emitted == every, (name, bs, world)
            else:
                before, after = 2, 2
                assert emitted == [(s, k) for s, lay in enumerate(layouts) for p, k in enumerate(lay.keys)
                                   if before <= p < len(lay.keys) - after], (name, bs, world)
            plan = LanePlan(lengths, 2, 1, bs, world, layout=layouts, **kind)
            for r, sl_list in enumerate(plan.slices):
                want = []
                for k, sl in enumerate(sl_list):
                    lay = layouts[sl.sequence]
                    run = [x for x in lay.keys if sl.run[0] <= x < sl.run[1]]
                    want += [(k, sl.sequence, f) for f in range(*sl.frames) if needs_frame(run, lay.offsets, f)]
                assert plan.frames[r] == want
            assert sorted(set(plan.order)) == sorted({(s, f) for fr in plan.frames for _, s, f in fr})


def test_layout_arguments():
    lay = [kitti_layout(10)]
    with pytest.raises(ValueError):
        shard_sequences([10], 2, 1, 4, 0, 1, eval_batch=2, keys=[[1, 2]], layout=lay)
    with pytest.raises(ValueError):
        shard_sequences([10, 10], 2, 1, 4, 0, 1, eval_batch=2, layout=lay)
    with pytest.raises(ValueError):
        shard_sequences([5], 2, 1, 4, 0, 1, eval_batch=2, layout=lay)      # key frames past a shorter sequence


# ---- gloo worlds ----------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _world_case():
    lengths = [29, 11, 18]
    layouts = [kitti_layout(lengths[0], 2, 1, offset_d=-1, drop_outside=True), robotcar_layout(lengths[1], 3, 1, drop_outside=True),
               tum_mono_vo_layout(lengths[2], 3, 2)]
    return lengths, layouts


def _rows(lengths, layouts, bs, slices):
    """(sequence, key, frame values...) of every key frame the slices emit, as float64 rows."""
    rows = []
    for sl in slices:
        _, out = _run_slice(layouts[sl.sequence], bs, sl)
        rows += [[sl.sequence, i] + frames for i, frames in out if sl.emit[0] <= i < sl.emit[1]]
    width = 2 + max(len(lay.offsets) for lay in layouts)
    return torch.tensor([r + [-1.0] * (width - len(r)) for r in rows], dtype=torch.float64).reshape(-1, width)


def _world_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from monorec_b200.dist import all_gather_rows
        lengths, layouts = _world_case()
        got = []
        for kind in ({"eval_batch": 2}, {"buffer_length": 3}):
            slices = shard_sequences(lengths, 2, 1, 3, rank, world, layout=layouts, **kind)
            got.append(all_gather_rows(_rows(lengths, layouts, 3, slices)).tolist())
        q.put((rank, got, None))
    except Exception as e:                   # noqa: BLE001  (reported to the parent)
        q.put((rank, None, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_worlds_give_the_one_process_rows(world):
    lengths, layouts = _world_case()
    ref = []
    for kind in ({"eval_batch": 2}, {"buffer_length": 3}):
        ref.append(_rows(lengths, layouts, 3, shard_sequences(lengths, 2, 1, 3, 0, 1, layout=layouts, **kind)).tolist())
    assert len(ref[0]) == sum(len(lay.keys) for lay in layouts)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_world_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = [q.get(timeout=180) for _ in procs]
    [p.join(timeout=60) for p in procs]
    assert all(err is None for _, _, err in res), res
    for _, got, _ in res:
        assert got == ref
