"""The sequence form of evaluate.py on the device: the grouped metric passes (`mr_sparse_metrics` / `mr_dense_metrics` with
several groups), the evaluater's accumulator (`mr_eval_accumulate`) and SequenceEvaluater, against the one-group
passes, the float64 restatement (tests/eval_oracle.py), the reference's own logs (tests/golden/eval_sequence.npz) and the
evaluater's loop over the same key frames."""
import json
import warnings

import numpy as np
import pytest
import torch

from tests import eval_oracle as EO
from tests.helpers import GOLDEN

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
TENSOR_SIGNATURE = ("sc_inv_metric", "l1_rel_metric", "l1_inv_metric", "completeness_metric", "covered_gt_metric")
SPARSE7 = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
           "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]


def _bits(x):
    return np.asarray(x, np.float32).view(np.int32).astype(np.int64)


def _assert_bitwise(got, ref):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    np.testing.assert_array_equal(_bits(got[ok]), _bits(ref[ok]))


def _assert_ulp(got, ref, ulp=1):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.all(np.abs(_bits(got[ok]) - _bits(ref[ok])) <= ulp), np.abs(_bits(got[ok]) - _bits(ref[ok])).max()


def _assert_same(got, ref, rtol=5e-6, atol=1e-7):
    """Equal within the metric gates of test_metrics_dense.py where finite; NaN and +-inf in the same places."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_array_equal(np.isinf(got), np.isinf(ref))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=rtol, atol=atol)


# ---- grouped passes -------------------------------------------------------------------------------------------------
def _dyadic(B, H, W, seed):
    """Inverse depths 2^-k (k = 0..3): every per-pixel term is exact or one fixed fp32 value, so every sum is exact and its
    order does not matter; a third of the targets are missing."""
    g = torch.Generator().manual_seed(seed)
    pred = torch.pow(2.0, -torch.randint(0, 4, (B, 1, H, W), generator=g).float())
    gt = torch.pow(2.0, -torch.randint(0, 4, (B, 1, H, W), generator=g).float())
    gt[torch.rand(B, 1, H, W, generator=g) < 0.33] = 0.0
    pred[torch.rand(B, 1, H, W, generator=g) < 0.02] = 0.0
    gt[2] = 0.0                                                  # an image without ground truth: NaN rmse in its group
    return pred.to(DEV), gt.to(DEV)


def _gaussian(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    pred = torch.rand(B, 1, H, W, generator=g) * 0.3 + 0.002
    gt = (pred * (1 + 0.2 * torch.randn(B, 1, H, W, generator=g))).clamp_min(1e-3)
    gt[torch.rand(B, 1, H, W, generator=g) > 0.05] = 0.0
    return pred.to(DEV), gt.to(DEV)


def _passes(M, pred, gt, mv, kind, kw, group=None):
    """kind 'sparse' / 'dense': the grouped pass when group is given, else the ungrouped one."""
    if kind == "sparse":
        args = (pred, gt, mv, kw.get("roi"), kw.get("max_distance", 0.0), kw.get("pred_all_valid", True))
        return M.sparse_metrics_impl(*args) if group is None else M.sparse_metrics_grouped_impl(*args, group)
    md = kw.get("max_distance")
    args = (pred, gt, kw.get("roi"), 0.0 if md is None else float(1 / md))
    return M.dense_metrics_impl(*args) if group is None else M.dense_metrics_grouped_impl(*args, group)


KWS = [dict(), dict(roi=[3, 60, 5, 120], max_distance=80.0), dict(max_distance=50.0, pred_all_valid=False)]


@pytest.mark.parametrize("kind", ["sparse", "dense"])
@pytest.mark.parametrize("data", ["dyadic", "gaussian"])
@pytest.mark.parametrize("B,group", [(10, 3), (8, 4), (7, 1), (5, 9)])
def test_grouped_rows_equal_the_ungrouped_pass_on_each_slice(kind, data, B, group):
    from monorec_b200 import metrics as M
    pred, gt = (_dyadic if data == "dyadic" else _gaussian)(B, 64, 128, seed=B * 10 + group)
    mv = (torch.rand(pred.shape, device=DEV) > 0.3).float() if kind == "sparse" else None
    for kw in KWS:
        if kind == "dense" and "pred_all_valid" in kw:
            continue
        for use_mv in ((False, True) if kind == "sparse" else (False,)):
            m = mv if use_mv else None
            rows = _passes(M, pred, gt, m, kind, kw, group).cpu().numpy()
            assert rows.shape == (-(-B // group), 7 if kind == "sparse" else 12)
            for gi in range(rows.shape[0]):
                sl = slice(gi * group, min(B, (gi + 1) * group))
                ref = _passes(M, pred[sl], gt[sl], None if m is None else m[sl], kind, kw).cpu().numpy()
                (_assert_bitwise if data == "dyadic" else _assert_ulp)(rows[gi], ref)
    if data == "dyadic" and kind == "sparse":
        assert np.isnan(_passes(M, pred, gt, None, kind, {}, group).cpu().numpy()[2 // group][3])


@pytest.mark.parametrize("kind", ["sparse", "dense"])
@pytest.mark.parametrize("data", ["dyadic", "golden"])
def test_one_group_is_the_existing_entry(kind, data):
    from monorec_b200 import metrics as M
    if data == "golden":
        g = np.load(GOLDEN / ("metrics.npz" if kind == "sparse" else "metrics_dense.npz"))
        pred, gt = torch.from_numpy(g["pred"]).to(DEV), torch.from_numpy(g["gt"]).to(DEV)
    else:
        pred, gt = _dyadic(6, 64, 128, seed=3)
    for kw in KWS[:2]:
        one = _passes(M, pred, gt, None, kind, kw, group=pred.shape[0]).cpu().numpy()
        assert one.shape[0] == 1
        _assert_bitwise(one[0], _passes(M, pred, gt, None, kind, kw).cpu().numpy())


# ---- accumulator ----------------------------------------------------------------------------------------------------
def test_eval_accumulate_equals_the_numpy_restatement_bit_for_bit():
    """70 batches (three launches of the accumulator) in three calls, NaN rows (the first one among them), inf values,
    ragged sizes: total, valid, running average and sample count equal the float64 restatement bit for bit."""
    from monorec_b200 import metrics as M
    gen = np.random.default_rng(11)
    G, m = 70, 9
    rows = (gen.standard_normal((G, m)) * 10 ** gen.uniform(-3, 2, (G, m))).astype(np.float32)
    rows[[0, 5, 6, 40], gen.integers(0, m, 4)] = np.nan
    rows[12, 3] = np.inf
    sizes = [int(s) for s in gen.integers(1, 9, G)]
    state = torch.zeros(3 * m + 1, dtype=torch.float64, device=DEV)
    ref = None
    for a, b in ((0, 1), (1, 33), (33, 70)):
        M.eval_accumulate_impl(torch.from_numpy(rows[a:b]).to(DEV), sizes[a:b], state)
        ref = EO.accumulate(rows[a:b], sizes[a:b], ref)
        s = state.cpu().numpy()
        for k in range(3):
            np.testing.assert_array_equal(s[k * m:(k + 1) * m].view(np.uint64), ref[k].view(np.uint64))
        assert s[3 * m] == ref[3] == sum(sizes[:b])
    assert ref[1][0] == G - 4


# ---- SequenceEvaluater on the reference's logs ------------------------------------------------------------------------
@pytest.mark.parametrize("chunks", [[1], [3, 1, 4], [9]], ids=["1", "3-1-4", "9"])
@pytest.mark.parametrize("tag", ["eval_config", "ms_roi_onlyvalid", "dense_sparse", "dense_ms"])
def test_add_reproduces_the_reference_log(tag, chunks):
    """The golden key frames fed through `add` in chunks that do not follow the evaluater's batches: log() is the
    reference's Evaluater.eval log within the metric gates, with valid_batches and the NaN pattern exact."""
    from monorec_b200 import metrics as M
    from monorec_b200.evaluation import SequenceEvaluater
    g = np.load(GOLDEN / "eval_sequence.npz")
    c = json.loads(str(g["cases"]))[tag]
    # the configured names, given as names and as this package's functions
    metrics = [n if i % 2 else getattr(M, n) for i, n in enumerate(c["names"])]
    ev = SequenceEvaluater(None, metrics, c["batch_size"], roi=c["roi"], max_distance=c["max_distance"],
                           median_scaling=c["median_scaling"])
    result, target = torch.from_numpy(g["result"]).to(DEV), torch.from_numpy(g["target"]).to(DEV)
    i, k = 0, 0
    while i < c["n"]:
        n = min(chunks[k % len(chunks)], c["n"] - i)
        ev.add(result[i:i + n], target[i:i + n])
        i, k = i + n, k + 1
    ev.flush()
    log = ev.log()
    assert ev.names == c["names"] and log["loss"] == 0.0 and log["loss_loss"] == 0.0
    assert log["valid_batches"] == g[f"{tag}_valid_batches"]
    _assert_same(log["metrics"], g[f"{tag}_metrics"])
    _assert_same(log["metrics_correct"], g[f"{tag}_metrics_correct"])


# ---- end to end over two sequences ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    import monorec_b200.model as MM
    from monorec_b200.synthetic import seeded_state_dict
    m = MM.MonoRecModel()
    m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
    return m.to(DEV).eval()


def _targets(n, H, W, seed, empty=()):
    g = torch.Generator().manual_seed(seed)
    t = torch.rand(n, 1, H, W, generator=g) * 0.2 + 0.01
    t[torch.rand(n, 1, H, W, generator=g) > 0.25] = 0.0
    for i in empty:
        t[i] = 0.0
    return t


def _evaluater_loop(result, target, names, bs, roi, md, ms):
    """Evaluater.eval's loop (evaluater.py:38-49, 78-119) with this package's metric functions, batch by batch."""
    from monorec_b200 import metrics as M
    n, rows = result.shape[0], []
    for b in range(0, n, bs):
        d = {"result": result[b:b + bs], "target": target[b:b + bs]}
        row = []
        for name in names:
            if ms:
                d = M.median_scaling(d)
            fn = getattr(M, name)
            row.append(float(fn(d["result"], d["target"], roi, md) if name in TENSOR_SIGNATURE else fn(d, roi, md)))
        rows.append(row)
    return EO.log(EO.accumulate(np.array(rows, np.float32), EO.batch_sizes(n, bs)))


def _loader_batch(seqs, keys, offs):
    """The loader's collated dict of key frames `keys` = [(sequence, index)] (kitti_odometry_dataset.py:248-269)."""
    rows = lambda which, d: torch.cat([seqs[s][which][i + d:i + d + 1] for s, i in keys]).to(DEV)   # noqa: E731
    return {"keyframe": rows(0, 0), "keyframe_pose": rows(1, 0), "keyframe_intrinsics": rows(2, 0),
            "frames": [rows(0, d) for d in offs], "poses": [rows(1, d) for d in offs], "intrinsics": [rows(2, d) for d in offs]}


@pytest.mark.parametrize("median_scaling", [False, True], ids=["plain", "median_scaling"])
@pytest.mark.parametrize("bs", [2, 3])
def test_sequence_evaluation_end_to_end(model, bs, median_scaling):
    """Two synthetic sequences (13 and 10 frames: 11 + 8 key frames) run at batch 4 with graph replay, evaluated at evaluater
    batch 2 (divides 4) and 3 (does not), with the sequence boundary inside an evaluater batch and a key frame without
    ground truth.  The log equals the evaluater's loop over the same results (within the rounding of the grouped pass), and
    an eager B 2 loop of the model over the loader's dicts of the same key frames within tolerance."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.sequence import MonoRecSequence, neighbour_offsets
    from monorec_b200.synthetic import make_sequence
    H, W = 64, 128
    names = SPARSE7 + ["abs_rel_metric", "sc_inv_metric"]
    roi, md = [4, 60, 8, 120], 80
    seqs = [make_sequence(13, H, W, seed=3), make_sequence(10, H, W, seed=4)]
    targets = [_targets(13, H, W, seed=5, empty=(4,)), _targets(10, H, W, seed=6)]
    ev = SequenceEvaluater(MonoRecSequence(model, batch_size=4), names, bs, roi=roi, max_distance=md,
                           median_scaling=median_scaling)
    results, keys = [], []
    with torch.no_grad():
        for s, (images, poses, Ks) in enumerate(seqs):
            if s:
                emitted = ev.next_sequence(MonoRecSequence(model, batch_size=4))
                results += [o["result"].clone() for _, o in emitted]
                keys += [(s - 1, i) for i, _ in emitted]
            for n in range(images.shape[0]):
                emitted = ev.push(images[n], poses[n], Ks[n], targets[s][n])
                results += [o["result"].clone() for _, o in emitted]
                keys += [(s, i) for i, _ in emitted]
        emitted = ev.flush()
        results += [o["result"].clone() for _, o in emitted]
        keys += [(1, i) for i, _ in emitted]
    assert keys == [(0, i) for i in range(1, 12)] + [(1, i) for i in range(1, 9)]
    log = ev.log()
    result = torch.cat(results)
    target = torch.cat([targets[s][i:i + 1] for s, i in keys]).to(DEV)
    ref = _evaluater_loop(result, target, names, bs, roi, md, median_scaling)
    n_batches = -(-len(keys) // bs)
    assert log["valid_batches"] == ref["valid_batches"] == n_batches - 1      # the batch with key frame (0, 4)
    _assert_same(log["metrics"], ref["metrics"], rtol=2e-6)
    _assert_same(log["metrics_correct"], ref["metrics_correct"], rtol=2e-6)
    # the reference's own path: eager forwards of the loader's batch-2 dicts (batches cross the sequence boundary)
    offs = neighbour_offsets(2)
    with torch.no_grad():
        eager = torch.cat([model(_loader_batch(seqs, keys[b:b + 2], offs))["result"] for b in range(0, len(keys), 2)])
    ref2 = _evaluater_loop(eager, target, names, bs, roi, md, median_scaling)
    assert log["valid_batches"] == ref2["valid_batches"]
    _assert_same(log["metrics"], ref2["metrics"], rtol=1e-3, atol=1e-3)
    _assert_same(log["metrics_correct"], ref2["metrics_correct"], rtol=1e-3, atol=1e-3)


def test_push_and_flush_do_not_synchronise(model):
    """Once the sequence has captured its graph (its first batch), push, next_sequence and flush issue no host
    synchronisation -- graph replays, the eager tail of each sequence, median scaling, the grouped passes and the
    accumulator included; log() issues one."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.sequence import MonoRecSequence
    from monorec_b200.synthetic import make_sequence
    H, W = 64, 128
    images, poses, Ks = [t.to(DEV) for t in make_sequence(16, H, W, seed=8)]
    target = _targets(16, H, W, seed=9).to(DEV)
    ev = SequenceEvaluater(MonoRecSequence(model, batch_size=4), SPARSE7 + ["sc_inv_metric"], 3, max_distance=80,
                           median_scaling=True)
    with torch.no_grad():
        n = 0
        while not ev.push(images[n], poses[n], Ks[n], target[n]):      # up to the first batch: its graph is captured
            n += 1
        emitted = 4
        second = MonoRecSequence(model, batch_size=4)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for n in range(n + 1, 16):
                emitted += len(ev.push(images[n], poses[n], Ks[n], target[n]))
            # a second sequence shorter than one batch: its key frames run in its eager tail
            emitted += len(ev.next_sequence(second))
            for n in range(5):
                emitted += len(ev.push(images[n], poses[n], Ks[n], target[n]))
            emitted += len(ev.flush())
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert emitted == 14 + 3
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            log = ev.log()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len([w for w in caught if "synchroniz" in str(w.message)]) == 1
    assert log["valid_batches"] == 6                                    # 17 key frames in batches of 3
