"""evaluate.py's list of models over several lanes (lanes.MultiDeviceModelsEvaluater) against one device and against each
model's own multi-device run.

Lanes [0, 0] and [0, 0, 0] (lanes taking turns on one GPU) and, on a machine with several GPUs, one lane per GPU.  Three
models in two cost-volume groups: two checkpoints on one trunk and a use_ssim=2 model on that trunk (plus a use_stereo or a
pretrain_mode 3 model for the stereo and moving-object streams).  Each model's log equals, bit for bit, the one-device
MultiModelEvaluater's and that model's own MultiDeviceEvaluater's, with median scaling on and off, index-masked key
lists, stereo frames, moving-object masks and grayscale frames; results() equals the one-device results(); and once the
lanes have captured their graphs, push and flush make no host synchronisation."""
import json

import numpy as np
import pytest
import torch

from tests import test_eval_models_gpu as E
from tests import test_sequence_devices_gpu as SD

pytestmark = pytest.mark.gpu

LANES = [[0, 0], [0, 0, 0]] + ([list(range(torch.cuda.device_count()))] if torch.cuda.device_count() >= 2 else [])
LENGTHS = [13, 10]                           # 11 + 8 key frames
KW = dict(roi=[4, 60, 8, 120], max_distance=80)
BS, SEQ_BATCH = 3, 4


@pytest.fixture(scope="module")
def models():
    from monorec_b200.model import MonoRecModel
    a = E.seeded_model(MonoRecModel, 7)
    out = {"a": a, "b": E.seeded_model(MonoRecModel, 8), "c": E.seeded_model(MonoRecModel, 9, use_ssim=2),
           "s": E.seeded_model(MonoRecModel, 10, use_stereo=True), "p3": E.seeded_model(MonoRecModel, 11, pretrain_mode=3)}
    for k in ("b", "c", "s", "p3"):
        out[k]._feature_extractor.load_state_dict(a._feature_extractor.state_dict())
    return out


def _config(models, name):
    """(models, streams, keyword arguments of the evaluaters) of one stream configuration."""
    ms, seq_kw, kw = [models["a"], models["b"], models["c"]], {}, dict(KW)
    if name == "stereo":
        seq_kw["stereo"], kw["stereo"] = True, True
        ms.append(models["s"])
    elif name == "mvobj_masks":
        seq_kw["masks"], kw["mvobj_masks"] = True, True
        ms.append(models["p3"])
    streams = [E._stream(n, 11 + s, **seq_kw) for s, n in enumerate(LENGTHS)]
    if name == "gray":
        streams = [[(img.mean(0, keepdim=True), p, K, kw_) for img, p, K, kw_ in st] for st in streams]
        kw["use_color"] = False
    if name == "keys":
        kw["keys"] = [E._index_keys(13, 1), E._index_keys(10, 2)]
    if name == "median_scaling":
        kw["median_scaling"] = True
    return ms, streams, kw


def _one_device(ms, streams, kw):
    from monorec_b200.models_eval import MultiModelEvaluater
    keys = kw.get("keys")
    one = dict(kw, keys=None if keys is None else keys[0])
    with torch.no_grad():
        ev = MultiModelEvaluater(ms, E.NAMES, BS, seq_batch=SEQ_BATCH, **one)
        E._drive(ev, streams, lambda s: ev.next_sequence(None if keys is None else keys[s]))
    return ev


def _feed(run, streams):
    with torch.no_grad():
        for s, n in run.order:
            img, pose, K, kw = streams[s][n]
            run.push(s, n, img, pose, K, **kw)
        run.flush()
    return run


CONFIGS = ["plain", "median_scaling", "keys", "stereo", "mvobj_masks", "gray"]


@pytest.mark.parametrize("devices", LANES, ids=lambda d: "-".join(map(str, d)))
@pytest.mark.parametrize("config", CONFIGS)
def test_each_log_is_the_one_device_log_and_its_own_multi_device_log(models, config, devices):
    from monorec_b200.lanes import MultiDeviceEvaluater, MultiDeviceModelsEvaluater
    ms, streams, kw = _config(models, config)
    one = _one_device(ms, streams, kw)
    ref = one.logs()
    assert all(log["valid_batches"] > 0 for log in ref)
    run = _feed(MultiDeviceModelsEvaluater(ms, devices, LENGTHS, E.NAMES, BS, seq_batch=SEQ_BATCH, **kw), streams)
    assert (run.cv_groups, run.trunk_groups) == (one.cv_groups, one.trunk_groups)
    assert len(run.cv_groups) == len(ms) - 1 and run.trunk_groups == [list(range(len(ms)))]
    logs = run.logs()
    assert len(logs) == len(ms)
    for m, model in enumerate(ms):
        E._assert_logs_equal(logs[m], ref[m])
        own = _feed(MultiDeviceEvaluater(model, devices, LENGTHS, E.NAMES, BS, seq_batch=SEQ_BATCH, **kw), streams)
        E._assert_logs_equal(logs[m], own.log())
    assert logs[0]["metrics"] != logs[1]["metrics"]                # the heads differ


@pytest.mark.parametrize("devices", LANES, ids=lambda d: "-".join(map(str, d)))
def test_results_are_the_one_device_results(models, devices):
    from monorec_b200.lanes import MultiDeviceModelsEvaluater
    ms, streams, kw = _config(models, "plain")
    dataset = {"dataset_dir": "data/dataset", "frame_count": 2, "sequences": ["00", "04"], "_offset": 1,
               "depth_range": np.array([0.5, 80.0])}
    ref = _one_device(ms, streams, kw).results(dataset)
    got = _feed(MultiDeviceModelsEvaluater(ms, devices, LENGTHS, E.NAMES, BS, seq_batch=SEQ_BATCH, **kw),
                streams).results(dataset)
    assert len(got) == len(ref) == 3
    for mine, theirs in zip(got, ref):
        assert list(mine) == list(theirs) == ["model", "dataset", "result"]
        assert mine["model"] == theirs["model"] and mine["dataset"] == theirs["dataset"]
        E._assert_logs_equal({k: v for k, v in mine["result"].items() if k != "metrics_info"},
                             {k: v for k, v in theirs["result"].items() if k != "metrics_info"})
        assert mine["result"]["metrics_info"] == theirs["result"]["metrics_info"] == E.NAMES
    assert json.loads(json.dumps(got, allow_nan=True))                # evaluate.py writes it as JSON


@pytest.mark.parametrize("devices,keyed", [(d, k) for k in (False, True) for d in LANES],
                         ids=["-".join(map(str, d)) + ("-index_masked" if k else "") for k in (False, True) for d in LANES])
def test_lanes_make_no_host_synchronisation(models, devices, keyed):
    """Every key frame, or an index-masked key list (key frames 5 ... 7 masked out, so frame 6 is skipped)."""
    from monorec_b200.lanes import MultiDeviceModelsEvaluater
    from monorec_b200.sequence import loader_keys
    ms = [models["a"], models["b"], models["c"]]
    frames = E._stream(16, 8)
    lengths = [len(frames)]
    keys = [loader_keys(lengths[0], index_masks=[{str(k): not 5 <= k <= 7 for k in range(lengths[0])}])] if keyed else None
    with torch.no_grad():
        run = MultiDeviceModelsEvaluater(ms, devices, lengths, E.SPARSE7 + ["sc_inv_metric"], 2, seq_batch=2, keys=keys,
                                         median_scaling=True, **KW)

        def push(s, n):
            img, pose, K, kw = frames[n]
            run.push(s, n, img, pose, K, **kw)
        assert SD._sync_free_after_capture(run, push, lambda: [e.seq for e in run.evaluaters if e is not None])
    logs = run.logs()
    assert len(logs) == 3 and all(log["valid_batches"] > 0 for log in logs)
