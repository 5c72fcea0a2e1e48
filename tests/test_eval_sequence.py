"""The sequence form of evaluate.py (monorec_b200/evaluation.py) on the CPU: the float64 restatement of the evaluater's
bookkeeping against the reference's own logs (tests/golden/eval_sequence.npz, written by make_golden_eval_sequence.py from
the unmodified evaluater/evaluater.py), the metric-name table, and the argument checks of SequenceEvaluater and of the new C
entries (before any CUDA call)."""
import ctypes
import json

import numpy as np
import pytest

from tests import eval_oracle as EO
from tests.helpers import GOLDEN


def _golden():
    g = np.load(GOLDEN / "eval_sequence.npz")
    return g, json.loads(str(g["cases"]))


def _same(got, ref):
    """Bit for bit, NaN in the same places."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_array_equal(got[~np.isnan(ref)].view(np.uint64), ref[~np.isnan(ref)].view(np.uint64))


def test_golden_covers_ragged_batches_nan_batches_and_both_scalings():
    g, cases = _golden()
    assert any(c["median_scaling"] for c in cases.values()) and not all(c["median_scaling"] for c in cases.values())
    for tag, c in cases.items():
        sizes = EO.batch_sizes(c["n"], c["batch_size"])
        assert g[f"{tag}_raw"].shape == (len(sizes), len(c["names"]))
        assert sizes[-1] < c["batch_size"], tag                               # a ragged last batch
        assert 0 < g[f"{tag}_valid_batches"] < len(sizes), tag                 # a batch with a NaN metric
    names = {n for c in cases.values() for n in c["names"]}
    assert any("onlyvalid" in n for n in names) and "sc_inv_metric" in names and "a1_sparse_metric" in names


@pytest.mark.parametrize("tag", ["eval_config", "ms_roi_onlyvalid", "dense_sparse", "dense_ms"])
def test_restatement_reproduces_the_reference_log(tag):
    g, cases = _golden()
    c = cases[tag]
    state = EO.accumulate(g[f"{tag}_raw"], EO.batch_sizes(c["n"], c["batch_size"]))
    log = EO.log(state)
    _same(log["metrics"], g[f"{tag}_metrics"])
    _same(log["metrics_correct"], g[f"{tag}_metrics_correct"])
    assert log["valid_batches"] == g[f"{tag}_valid_batches"]


def test_restatement_in_pieces_equals_one_pass():
    """Accumulating batch after batch (as SequenceEvaluater does per emitted batch) is the same as one pass."""
    g, cases = _golden()
    c = cases["eval_config"]
    raw, sizes = g["eval_config_raw"], EO.batch_sizes(c["n"], c["batch_size"])
    state = None
    for i in range(len(sizes)):
        state = EO.accumulate(raw[i:i + 1], sizes[i:i + 1], state)
    one = EO.accumulate(raw, sizes)
    for a, b in zip(state[:3], one[:3]):
        _same(a, b)
    assert state[3] == one[3] == c["n"]


def test_metric_table_names_every_reference_metric():
    from monorec_b200 import evaluation as E
    from monorec_b200 import metrics as M
    assert len(E.METRICS) == 33
    assert sum(1 for n in E.METRICS if "_sparse" in n) == 21
    for n in E.METRICS:
        assert E.metric_name(n) == n and E.metric_name(getattr(M, n)) == n
    assert E.METRICS["rmse_sparse_onlyvalid_metric"] == (("sparse", False, False), 3)
    assert E.METRICS["a2_sparse_onlydynamic_metric"] == (("sparse", True, True), 1)
    assert E.METRICS["covered_gt_metric"] == (("dense",), 11)


@pytest.mark.parametrize("kw", [dict(metrics=["a1_sparse_metric", "a4_sparse_metric"]), dict(metrics=[len]),
                                dict(metrics="a1_sparse_metric"), dict(metrics=[]),
                                dict(batch_size=0), dict(batch_size=2.5), dict(batch_size=True),
                                dict(roi=[1, 2, 3]), dict(roi=[0, 10.5, 0, 10]), dict(max_distance=0)],
                         ids=lambda kw: next(iter(kw)) + "=" + repr(next(iter(kw.values()))))
def test_bad_arguments_raise_value_error_before_any_launch(kw):
    from monorec_b200.evaluation import SequenceEvaluater
    args = dict(metrics=["a1_sparse_metric"], batch_size=2)
    args.update(kw)
    with pytest.raises(ValueError):
        SequenceEvaluater(None, **args)


def _abi():
    from monorec_b200 import _lib
    return _lib.load()


def test_metric_groups_validation_without_gpu():
    lib = _abi()
    p, t, o, ws = 0x7F0000100000, 0x7F0000200000, 0x7F0000300000, 0x7F0000400000
    for kw, text in ((dict(group=0), "group=0"), (dict(group=-2), "group=-2"), (dict(p=None), "null pointer"),
                     (dict(B=0), "B=0"), (dict(ws=ws + 4), "aligned")):
        a = dict(p=p, B=4, group=2, ws=ws)
        a.update(kw)
        rc = lib.mr_sparse_metrics(a["p"], t, None, a["B"], a["group"], 8, 8, None, 80.0, 1, o, a["ws"], 1024, None)
        msg = lib.mr_last_error().decode()
        assert rc == -1 and msg.startswith("mr_sparse_metrics:") and text in msg, (kw, rc, msg)
        rc = lib.mr_dense_metrics(a["p"], t, a["B"], a["group"], 8, 8, None, 0.0, o, a["ws"], 1024, None)
        msg = lib.mr_last_error().decode()
        assert rc == -1 and msg.startswith("mr_dense_metrics:") and text in msg, (kw, rc, msg)
    assert lib.mr_sparse_metrics(p, t, None, 4, 2, 8, 8, None, 80.0, 1, o, ws, 8, None) == -3      # MR_ENOMEM
    assert b"workspace too small" in lib.mr_last_error()


def test_eval_accumulate_validation_without_gpu():
    lib = _abi()
    v, st = 0x7F0000100000, 0x7F0000200000
    sizes = (ctypes.c_int * 3)(2, 2, 1)
    for args, text in (((None, 3, 7, sizes, st), "null pointer"), ((v, 3, 7, None, st), "null pointer"),
                       ((v, 0, 7, sizes, st), "G=0"), ((v, 3, 0, sizes, st), "M=0"), ((v, 3, 1025, sizes, st), "M=1025"),
                       ((v, 3, 7, (ctypes.c_int * 3)(2, 0, 1), st), "group_sizes[1] = 0"),
                       ((v, 3, 7, sizes, st + 4), "aligned")):
        rc = lib.mr_eval_accumulate(*args, None)
        msg = lib.mr_last_error().decode()
        assert rc == -1 and msg.startswith("mr_eval_accumulate") and text in msg, (args, rc, msg)
