"""MultiModelEvaluater on the device: every model's log and results equal, bit for bit, those of its own SequenceEvaluater
over its own MonoRecSequence, with the stages shared or not, over the loader's configurations; no host synchronisation
after capture; and the staged eager forward issues the library calls and computes the bits of the single-block forward
it replaces (tests/golden/forward_stages.json, recorded from that forward by make_golden_forward_stages.py)."""
import hashlib
import json
import warnings

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN, kitti_sample_dict

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
SPARSE7 = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
           "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]
NAMES = SPARSE7 + ["abs_rel_metric", "sc_inv_metric"]
H, W = 64, 128


# ---- recording the forward's library calls (shared with tests/golden/make_golden_forward_stages.py) --------------------
def record_calls(fn):
    """Runs fn() with every declared entry of the library wrapped: (fn's return value, names of the entries it called)."""
    from monorec_b200 import _lib
    lib = _lib.load()
    calls, saved = [], {}
    for name in _lib.SIGNATURES:
        f = getattr(lib, name)
        saved[name] = f

        def wrapper(*a, _f=f, _n=name):
            calls.append(_n)
            return _f(*a)
        setattr(lib, name, wrapper)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        for name, f in saved.items():
            setattr(lib, name, f)
    return out, [c for c in calls if c not in ("mr_last_error", "mr_launch_count")]


def output_digests(out):
    """sha256 of the bytes of every output tensor of a forward (trunk levels 0-3; cv_module_time is host time)."""
    items = []
    for k, v in out.items():
        if k == "cv_module_time":
            continue
        if k == "image_features":
            v = v[:4]
        if torch.is_tensor(v):
            items.append((k, v))
        elif isinstance(v, (list, tuple)):
            items += [(f"{k}[{i}]", t) for i, t in enumerate(v) if torch.is_tensor(t)]
    return {k: hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest() for k, t in sorted(items)}


def golden_inputs(which):
    """(model weight seed, input dict on the device) of the model_synth_small / model_kitti_sample goldens."""
    from monorec_b200.synthetic import make_inputs, to_device
    if which == "synth_small":
        g = np.load(GOLDEN / "model_synth_small.npz")
        B, nF, D, h, w, seed, wseed = [int(v) for v in g["cfg"]]
        return wseed, to_device(make_inputs(B, nF, h, w, seed=seed), DEV)
    g = np.load(GOLDEN / "model_kitti_sample.npz")
    return int(g["wseed"][0]), to_device(kitti_sample_dict()[0], DEV)


def seeded_model(model_cls, seed, **kw):
    from monorec_b200.synthetic import seeded_state_dict
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = model_cls(**kw)
    m.load_state_dict(seeded_state_dict(m, seed=seed, gain=0.7))
    return m.to(DEV).eval()


@pytest.mark.parametrize("which", ["synth_small", "kitti_sample"])
@pytest.mark.parametrize("mode", ["tf32", "f16"])
def test_staged_forward_is_the_single_block_forward(mode, which):
    """The same library entries in the same order and the same output bits as the forward before the split into stages;
    69 launches on the model_synth_small input."""
    from monorec_b200 import _lib
    from monorec_b200 import conv as C
    from monorec_b200.model import MonoRecModel
    ref = json.loads((GOLDEN / "forward_stages.json").read_text())[mode][which]
    saved = C.MODE
    C.set_mode(mode)
    try:
        wseed, d = golden_inputs(which)
        model = seeded_model(MonoRecModel, wseed)
        with torch.no_grad():
            model(dict(d))                               # packs the weights
            torch.cuda.synchronize()
            _lib.launch_count(reset=True)
            out, calls = record_calls(lambda: model(dict(d)))
            launches = _lib.launch_count(reset=True)
    finally:
        C.set_mode(saved)
    assert calls == ref["calls"]
    assert output_digests(out) == ref["sha256"]
    if which == "synth_small":
        assert launches == 69


# ---- the evaluater against one SequenceEvaluater per model --------------------------------------------------------------
@pytest.fixture(scope="module")
def models():
    """a; b: other heads on a's trunk (shares the cost volume and the trunk with a); c: use_ssim=2 on a's trunk (shares
    only the trunk); s: use_stereo on a's trunk; p3: pretrain_mode 3 (the given masks) on a's trunk."""
    from monorec_b200.model import MonoRecModel
    a = seeded_model(MonoRecModel, 7)
    out = {"a": a, "b": seeded_model(MonoRecModel, 8), "c": seeded_model(MonoRecModel, 9, use_ssim=2),
           "s": seeded_model(MonoRecModel, 10, use_stereo=True), "p3": seeded_model(MonoRecModel, 11, pretrain_mode=3)}
    for k in ("b", "c", "s", "p3"):
        out[k]._feature_extractor.load_state_dict(a._feature_extractor.state_dict())
    return out


def _stream(n, seed, stereo=False, masks=False):
    """Frames of one synthetic sequence with targets (a key frame without ground truth), stereo frames, moving-object masks."""
    from monorec_b200.synthetic import make_sequence
    images, poses, Ks = make_sequence(n, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    t = torch.rand(n, 1, H, W, generator=g) * 0.2 + 0.01
    t[torch.rand(n, 1, H, W, generator=g) > 0.25] = 0.0
    t[4] = 0.0
    frames = []
    for i in range(n):
        kw = {"target": t[i]}
        if masks:
            kw["mvobj_mask"] = (torch.rand(1, H, W, generator=g) > 0.8).float()
        if stereo:
            base = torch.eye(4)
            base[0, 3] = 0.54
            kw["stereo"] = (torch.roll(images[i], shifts=(1, 3), dims=(1, 2)), poses[i] @ base, Ks[i])
        frames.append((images[i], poses[i], Ks[i], kw))
    return frames


def _index_keys(n, drop):
    from monorec_b200.sequence import loader_keys
    return loader_keys(n, index_masks=[{str(k): k % 3 != drop for k in range(n)}])


def _drive(ev, seqs, next_seq):
    """Pushes every frame of every sequence (skipping those no key frame needs), moving on with next_seq(s); returns the
    key frames emitted in order as (sequence, index, emitted row)."""
    rows = []
    for s, frames in enumerate(seqs):
        if s:
            rows += [(s - 1, i, o) for i, o in next_seq(s)]
        for n, (img, pose, K, kw) in enumerate(frames):
            if ev.seq.needs(n):
                rows += [(s, i, o) for i, o in ev.push(img, pose, K, **kw)]
            else:
                ev.skip()
    rows += [(len(seqs) - 1, i, o) for i, o in ev.flush()]
    return rows


def _clone(rows, model=None):
    if model is None:
        return [(s, i, o["result"].clone()) for s, i, o in rows]
    return [(s, i, o["models"][model]["result"].clone()) for s, i, o in rows]


def _same_bits(x, y):
    return torch.equal(x.view(torch.int32), y.view(torch.int32))


def _assert_logs_equal(got, ref):
    assert list(got) == list(ref) and got["valid_batches"] == ref["valid_batches"]
    for k in ("metrics", "metrics_correct"):
        g, r = np.asarray(got[k], np.float64), np.asarray(ref[k], np.float64)
        np.testing.assert_array_equal(g.view(np.uint64), r.view(np.uint64))


def _run_both(ms, seqs, keys=None, stereo=False, mvobj_masks=False, median_scaling=False, bs=3, seq_batch=4):
    """MultiModelEvaluater over `ms` and one SequenceEvaluater(MonoRecSequence(model)) per model: (multi, its rows,
    [(log, rows) per model])."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.models_eval import MultiModelEvaluater
    from monorec_b200.sequence import MonoRecSequence
    kw = dict(max_distance=80, median_scaling=median_scaling, roi=[4, 60, 8, 120])
    with torch.no_grad():
        multi = MultiModelEvaluater(ms, NAMES, bs, seq_batch=seq_batch, keys=None if keys is None else keys[0],
                                    stereo=stereo, mvobj_masks=mvobj_masks, **kw)
        multi_rows = _drive(multi, seqs, lambda s: multi.next_sequence(None if keys is None else keys[s]))
        multi_rows = [_clone(multi_rows, m) for m in range(len(ms))]
        separate = []
        for model in ms:
            def seq(s, model=model):
                return MonoRecSequence(model, batch_size=seq_batch, keys=None if keys is None else keys[s], stereo=stereo,
                                       mvobj_masks=mvobj_masks)
            ev = SequenceEvaluater(seq(0), NAMES, bs, **kw)
            rows = _clone(_drive(ev, seqs, lambda s: ev.next_sequence(seq(s))))
            separate.append((ev.log(), rows))
    return multi, multi_rows, separate


def _assert_each_model_is_its_own_run(multi, multi_rows, separate):
    for m, (log, rows) in enumerate(separate):
        assert [(s, i) for s, i, _ in multi_rows[m]] == [(s, i) for s, i, _ in rows]
        assert all(_same_bits(x, y) for (_, _, x), (_, _, y) in zip(multi_rows[m], rows)), f"model {m}"
        _assert_logs_equal(multi.logs()[m], log)


@pytest.mark.parametrize("median_scaling", [False, True], ids=["plain", "median_scaling"])
def test_each_log_is_its_own_sequence_evaluation(models, median_scaling):
    """a and b share the cost volume and the trunk, c only the trunk; two sequences (13 and 10 frames: 11 + 8 key frames)
    at 4 key frames per forward, evaluater batch 3 (ragged, across the boundary)."""
    ms = [models["a"], models["b"], models["c"]]
    multi, multi_rows, separate = _run_both(ms, [_stream(13, 3), _stream(10, 4)], median_scaling=median_scaling)
    assert multi.cv_groups == [[0, 1], [2]] and multi.trunk_groups == [[0, 1, 2]]
    assert len(multi_rows[0]) == 19
    _assert_each_model_is_its_own_run(multi, multi_rows, separate)
    assert not _same_bits(multi_rows[0][0][2], multi_rows[1][0][2])       # the heads differ


@pytest.mark.parametrize("config", ["keys", "stereo", "mvobj_masks"])
def test_loader_configurations(models, config):
    """An index-masked key-frame list per sequence; stereo frames with a use_stereo model in the list; moving-object masks
    with a pretrain_mode 3 model in the list."""
    seqs_kw, kw, ms = {}, {}, [models["a"], models["b"], models["c"]]
    if config == "keys":
        kw["keys"] = [_index_keys(13, 1), _index_keys(10, 2)]
    elif config == "stereo":
        seqs_kw["stereo"], kw["stereo"] = True, True
        ms = ms + [models["s"]]
    else:
        seqs_kw["masks"], kw["mvobj_masks"] = True, True
        ms = ms + [models["p3"]]
    multi, multi_rows, separate = _run_both(ms, [_stream(13, 5, **seqs_kw), _stream(10, 6, **seqs_kw)], **kw)
    if config == "keys":
        assert [i for s, i, _ in multi_rows[0]] == kw["keys"][0] + kw["keys"][1]
    else:
        assert multi.trunk_groups == [list(range(len(ms)))] and len(multi.cv_groups) == 3
    _assert_each_model_is_its_own_run(multi, multi_rows, separate)


def test_shared_and_unshared_give_the_same_bits(models, monkeypatch):
    from monorec_b200 import models_eval
    ms = [models["a"], models["b"], models["c"]]
    seqs = [_stream(13, 7)]
    shared, shared_rows, _ = _run_both(ms, seqs)
    monkeypatch.setattr(models_eval, "share_groups", lambda m: ([[i] for i in range(len(m))], [[i] for i in range(len(m))]))
    alone, alone_rows, _ = _run_both(ms, seqs)
    assert shared.cv_groups == [[0, 1], [2]] and alone.cv_groups == [[0], [1], [2]] and alone.trunk_groups == [[0], [1], [2]]
    for m in range(3):
        assert all(_same_bits(x, y) for (_, _, x), (_, _, y) in zip(shared_rows[m], alone_rows[m]))
        _assert_logs_equal(shared.logs()[m], alone.logs()[m])


def test_push_and_flush_do_not_synchronise(models):
    """After the first batch (the graph's capture), push, next_sequence and flush issue no host synchronisation; logs()
    reads back once per model."""
    from monorec_b200.models_eval import MultiModelEvaluater
    ms = [models["a"], models["b"], models["c"]]
    frames = [(img.to(DEV), p.to(DEV), K.to(DEV), {"target": kw["target"].to(DEV)}) for img, p, K, kw in _stream(16, 8)]
    ev = MultiModelEvaluater(ms, SPARSE7 + ["sc_inv_metric"], 3, max_distance=80, median_scaling=True, seq_batch=4)
    with torch.no_grad():
        n = 0
        while not ev.push(*frames[n][:3], **frames[n][3]):
            n += 1
        emitted = 4
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for n in range(n + 1, 16):
                emitted += len(ev.push(*frames[n][:3], **frames[n][3]))
            emitted += len(ev.next_sequence())
            for n in range(5):                                   # shorter than one batch: its eager tail
                emitted += len(ev.push(*frames[n][:3], **frames[n][3]))
            emitted += len(ev.flush())
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert emitted == 14 + 3
    logs = ev.logs()
    assert len(logs) == 3 and all(log["valid_batches"] == 5 for log in logs)     # 17 key frames, the one without targets


def test_results_reproduce_the_reference_results_json():
    """The precomputed results of the two models of tests/golden/eval_models.npz, fed through each model's evaluater:
    results() holds the reference's logs within the metric gates, valid_batches and the NaN pattern exact."""
    from monorec_b200.model import MonoRecModel
    from monorec_b200.models_eval import MultiModelEvaluater
    g = np.load(GOLDEN / "eval_models.npz")
    ref = json.loads(str(g["results_json"]))
    cfg = json.loads(str(g["cfg"]))
    ms = [seeded_model(MonoRecModel, 7, use_ssim=r["model"]["use_ssim"]) for r in ref]
    ev = MultiModelEvaluater(ms, cfg["names"], cfg["batch_size"], max_distance=cfg["max_distance"])
    target = torch.from_numpy(g["target"]).to(DEV)
    for m, e in enumerate(ev.evaluaters):
        res = torch.from_numpy(g[f"result_{m}"]).to(DEV)
        for i in range(0, res.shape[0], 4):                          # chunks that do not follow the evaluater's batches
            e.add(res[i:i + 4], target[i:i + 4])
        e.flush()
    got = ev.results({"dataset_dir": "data/dataset"})
    for mine, theirs in zip(got, ref):
        a, b = mine["result"], theirs["result"]
        assert a["valid_batches"] == b["valid_batches"] and a["metrics_info"] == b["metrics_info"]
        assert a["loss"] == b["loss"] == 0.0 and a["loss_loss"] == b["loss_loss"] == 0.0
        for k in ("metrics", "metrics_correct"):
            x, y = np.asarray(a[k], np.float64), np.asarray(b[k], np.float64)
            np.testing.assert_array_equal(np.isnan(x), np.isnan(y))
            np.testing.assert_allclose(x[~np.isnan(y)], y[~np.isnan(y)], rtol=5e-6, atol=1e-7)
