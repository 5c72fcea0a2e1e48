"""MonoRecModel under torch.nn.DataParallel, as the reference's evaluate.py (base/base_trainer.py:26-29) and
create_pointcloud.py (:38-39) wrap it: gather-safe outputs, per-device kernel-layout caches keyed on the source parameters,
a re-entrant forward, and the cost-volume kernel's shared-memory opt-in on every device."""
import threading

import pytest
import torch

import monorec_b200.model as M
from monorec_b200 import conv as C
from monorec_b200.synthetic import make_inputs, seeded_state_dict, to_device

DEV = "cuda:0"
KEYS = ("result", "cv_mask", "cost_volume")
gpu = pytest.mark.gpu
two_gpus = pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the list type of image_features and the replica signature
# ---------------------------------------------------------------------------------------------------------------------
def test_trunk_features_rebuild_from_iterable_is_plain_list():
    """torch.nn.parallel.gather rebuilds every list output as type(out)(iterable): a _TrunkFeatures must come out of that as
    the list of the iterated items, with no lazy tail (and reset_tail must not drop its last entry)."""
    items = [torch.full((1, 2), float(i)) for i in range(5)]
    calls = []
    lazy = M._TrunkFeatures(items[:4], tail_fn=lambda t: calls.append(1) or items[4])
    rebuilt = type(lazy)(iter(lazy))
    assert calls == [1] and type(rebuilt) is M._TrunkFeatures and len(rebuilt) == 5
    assert all(a is b for a, b in zip(rebuilt, items)) and list.__getitem__(rebuilt, 4) is items[4]
    rebuilt.reset_tail()
    assert list.__getitem__(rebuilt, 4) is items[4]
    assert list(type(lazy)(iter([1, 2, 3]))) == [1, 2, 3] and type(lazy)() == []
    assert len(calls) == 1


def _cpu_replicate(module):
    """What torch.nn.parallel.replicate does to one replica, without a device: _replicate_for_data_parallel on every
    sub-module, children wired, parameters set as plain (copied) attributes, buffers copied."""
    mods = list(module.modules())
    copies = {m: m._replicate_for_data_parallel() for m in mods}
    for m in mods:
        r = copies[m]
        for k, c in m._modules.items():
            if c is not None:
                setattr(r, k, copies[c])
        for k, p in m._parameters.items():
            if p is None:
                r._parameters[k] = None
            else:
                setattr(r, k, p.detach().clone())
        for k, b in m._buffers.items():
            if b is not None:
                setattr(r, k, b.clone())
    return copies[module]


def _counting(monkeypatch, cls):
    calls = []
    orig = cls._build

    def build(self):
        calls.append(self)
        return orig(self)
    monkeypatch.setattr(cls, "_build", build)
    return calls


def test_replica_carries_the_original_parameter_signature(monkeypatch):
    """A replica has no registered parameters; its cache key is the original's parameter signature taken at replicate time,
    so it reuses the original's entry for its device (the folded trunk runs on the CPU: no launch needed)."""
    model = M.MonoRecModel(pretrain_mode=0)
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model.eval()
    for sub in (model._feature_extractor, model.att_module, model.depth_module):
        rep = _cpu_replicate(sub)
        assert list(rep.parameters()) == [] and rep._pack_sig() == sub._pack_sig()
        assert rep._packed is sub._packed
    calls = _counting(monkeypatch, M.ResnetEncoder)
    enc = model._feature_extractor
    x = torch.rand(2, 3, 64, 128)
    with torch.no_grad():
        ref = list(enc(x))
        outs = [list(_cpu_replicate(enc)(x)) for _ in range(3)]
    assert len(calls) == 1 and calls[0] is enc
    assert all(torch.equal(a, b) for out in outs for a, b in zip(out, ref))
    sd = {k: v.clone() for k, v in enc.state_dict().items()}
    sd["encoder.bn1.bias"] += 1.0
    enc.load_state_dict(sd)                                            # new signature: one more build, by the replica
    rep = _cpu_replicate(enc)
    with torch.no_grad():
        out = rep(x)[0]
        again = _cpu_replicate(enc)(x)[0]
    assert len(calls) == 2 and calls[1] is rep and not torch.equal(out, ref[0]) and torch.equal(out, again)
    assert len(enc._packed.entries) == 1


# ---------------------------------------------------------------------------------------------------------------------
# one GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=["tf32", "f16"])
def mode(request):
    saved = C.MODE
    C.set_mode(request.param)
    yield request.param
    C.set_mode(saved)


def _model(dev=DEV, **kw):
    model = M.MonoRecModel(**kw)
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    return model.to(dev).eval()


def _inputs(B, seed, dev=DEV, stereo=False):
    d = make_inputs(B, 2, 64, 128, seed=seed)
    if stereo:
        d["stereoframe"] = torch.roll(d["keyframe"], shifts=(1, 4), dims=(2, 3)).contiguous()
        pose = torch.eye(4).unsqueeze(0).repeat(B, 1, 1)
        pose[:, 0, 3] = 0.54
        d["stereoframe_pose"] = pose
        d["stereoframe_intrinsics"] = d["keyframe_intrinsics"].clone()
    return to_device(d, dev)


def _rows(d, lo, hi):
    return {k: ([t[lo:hi] for t in v] if isinstance(v, list) else v[lo:hi]) for k, v in d.items()}


def _assert_gathered(g, parts, pretrain_mode=0):
    """Every output of `g` equals torch.cat of the same output of `parts` along the batch, bit for bit."""
    cat = lambda key: torch.cat([p[key].to(DEV) for p in parts])                            # noqa: E731
    keys = ("result", "cv_mask") if pretrain_mode == 2 else KEYS
    for k in keys:
        assert torch.equal(g[k], cat(k)), k
    for f in range(len(parts[0]["single_frame_cvs"])):
        assert torch.equal(g["single_frame_cvs"][f], torch.cat([p["single_frame_cvs"][f].to(DEV) for p in parts])), f
    if pretrain_mode != 2:
        assert len(g["predicted_inverse_depths"]) == 4
        for s in range(4):
            assert torch.equal(g["predicted_inverse_depths"][s],
                               torch.cat([p["predicted_inverse_depths"][s].to(DEV) for p in parts])), s


@gpu
def test_gather_of_two_forwards_equals_cat(mode):
    model = _model()
    with torch.no_grad():
        o0 = model(_inputs(2, seed=1))
        o1 = model(_inputs(3, seed=2))
        g = torch.nn.parallel.gather([o0, o1], 0)
    _assert_gathered(g, [o0, o1])
    feats = g["image_features"]
    assert type(feats) is M._TrunkFeatures and len(feats) == 5
    for lvl in range(5):
        assert torch.equal(feats[lvl], torch.cat([o0["image_features"][lvl], o1["image_features"][lvl]])), lvl
    for k in ("inv_depth_min", "inv_depth_max", "cv_depth_steps", "cv_module_time"):
        assert g[k].shape == (2,), k                                   # one entry per replica, as with the reference


@gpu
@pytest.mark.parametrize("cfg", [dict(pretrain_mode=0), dict(pretrain_mode=2), dict(use_stereo=True)],
                         ids=["pretrain0", "pretrain2", "stereo"])
def test_two_replicas_on_one_device_equal_the_whole_batch(mode, cfg, monkeypatch):
    """Two replicas of one device (replicate + parallel_apply + gather, what DataParallel runs) on the two halves of a batch
    give the single-module forward of the whole batch, bit for bit; over three such forwards every pack builder runs once
    (the first single-module forward), and once more after load_state_dict."""
    counts = {cls: _counting(monkeypatch, cls) for cls in (M.ResnetEncoder, M.MaskModule, M.DepthModule)}
    model = _model(**cfg)
    stereo = bool(cfg.get("use_stereo"))
    data = _inputs(4, seed=11, stereo=stereo)
    pm = cfg.get("pretrain_mode", 0)
    with torch.no_grad():
        full = model(dict(data))

        def dp_forward():
            reps = torch.nn.parallel.replicate(model, [0], detach=True) + torch.nn.parallel.replicate(model, [0], detach=True)
            outs = torch.nn.parallel.parallel_apply(reps, [(_rows(data, 0, 2),), (_rows(data, 2, 4),)], devices=[0, 0])
            return torch.nn.parallel.gather(outs, 0)
        for _ in range(3):
            _assert_gathered(dp_forward(), [full], pm)
    built = [M.ResnetEncoder, M.MaskModule] + ([] if pm == 2 else [M.DepthModule])
    assert all(len(counts[cls]) == 1 for cls in built), {cls: len(counts[cls]) for cls in built}
    model.load_state_dict(seeded_state_dict(model, seed=8, gain=0.7))
    with torch.no_grad():
        full2 = model(dict(data))
        for _ in range(2):
            _assert_gathered(dp_forward(), [full2], pm)
    assert all(len(counts[cls]) == 2 for cls in built), {cls: len(counts[cls]) for cls in built}
    assert not torch.equal(full2["result"], full["result"])


@gpu
def test_concurrent_forwards_on_two_streams_and_a_standalone_depth_call(mode):
    """Two host threads on two streams run forwards of one model on different inputs while a third thread calls its
    DepthModule alone; every output equals its sequential run bit for bit, and the standalone call keeps returning the raw
    |tanh| heads while the model's forwards apply the inverse-depth affine."""
    model = _model()
    da, db = _inputs(2, seed=21), _inputs(2, seed=22)
    with torch.no_grad():
        ref_a, ref_b = model(dict(da)), model(dict(db))
        dd = {"keyframe": da["keyframe"], "cost_volume": ref_a["cost_volume"], "image_features": ref_a["image_features"][:4]}
        ref_d = model.depth_module(dict(dd))["predicted_inverse_depths"]
    assert all(float(p.max()) <= 1.0 for p in ref_d) and not torch.equal(ref_d[0], ref_a["result"])
    torch.cuda.synchronize()
    barrier, errors = threading.Barrier(3, timeout=300), []

    def run(fn, ref, keys):
        try:
            s = torch.cuda.Stream()
            barrier.wait()
            for _ in range(4):
                with torch.cuda.stream(s), torch.no_grad():
                    out = fn()
                s.synchronize()
                for k in keys:
                    a, b = out[k], ref[k]
                    same = all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(a, list) else torch.equal(a, b)
                    if not same:
                        errors.append(k)
        except Exception as e:          # noqa: BLE001  (reported below, in the main thread)
            errors.append(repr(e))
    keys = KEYS + ("single_frame_cvs", "predicted_inverse_depths")
    threads = [threading.Thread(target=run, args=(lambda: model(dict(da)), ref_a, keys)),
               threading.Thread(target=run, args=(lambda: model(dict(db)), ref_b, keys)),
               threading.Thread(target=run, args=(lambda: model.depth_module(dict(dd)), {"predicted_inverse_depths": ref_d},
                                                  ("predicted_inverse_depths",)))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert errors == []
    assert model.depth_module.out_range == (0.0, 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# two or more GPUs
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@two_gpus
@pytest.mark.parametrize("B", [2, 5])
def test_data_parallel_equals_single_device(mode, B):
    model = _model()
    data = _inputs(B, seed=31)
    dp = torch.nn.DataParallel(model, device_ids=[0, 1])
    with torch.no_grad():
        single = model(dict(data))
        for _ in range(2):
            _assert_gathered(dp(dict(data)), [single])


@gpu
@two_gpus
def test_evaluater_sequence_on_gathered_outputs():
    """The reference evaluater's loop (evaluater/evaluater.py:36-47) with median scaling and the metrics of
    configs/evaluate/eval_monorec.json gives the same numbers on the DataParallel output as on the single-device one."""
    from monorec_b200 import metrics as MT
    names = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
             "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]
    model = _model()
    data = _inputs(4, seed=41)
    g = torch.Generator().manual_seed(5)
    depth = 5.0 + 60.0 * torch.rand(4, 1, 64, 128, generator=g)
    target = torch.where(torch.rand(4, 1, 64, 128, generator=g) < 0.05, depth, torch.zeros_like(depth)).to(DEV)
    with torch.no_grad():
        single = model(dict(data))
        gathered = torch.nn.DataParallel(model, device_ids=[0, 1])(dict(data))
    vals = []
    for out in (single, gathered):
        d = dict(out, target=target)
        row = []
        for n in names:
            d = MT.median_scaling(d)
            row.append(float(getattr(MT, n)(d, None, 80)))
        vals.append(row)
    assert vals[0] == vals[1], vals


@gpu
@two_gpus
def test_model_moved_to_a_second_device_runs_the_cost_volume_there():
    """The cost-volume kernel's 227 KB shared-memory opt-in holds per device: a model that ran on cuda:0 runs on cuda:1 in
    the same process, with the same outputs."""
    model = _model()
    data = make_inputs(2, 2, 64, 128, seed=51)
    with torch.no_grad():
        first = model(to_device(data, DEV))
        model.to("cuda:1")
        second = model(to_device(data, "cuda:1"))
    torch.cuda.synchronize("cuda:1")
    assert second["cost_volume"].device == torch.device("cuda:1")
    for k in KEYS:
        assert torch.equal(second[k].to(DEV), first[k]), k
