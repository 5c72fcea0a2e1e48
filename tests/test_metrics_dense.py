"""The dense and completeness depth metrics (`mr_dense_metrics`) and the evaluater's median scaling (`mr_median_scaling`).

CPU: the numpy oracle (tests/metrics_dense_oracle.py) against the reference's own outputs (tests/golden/metrics_dense.npz,
written by make_golden_metrics_dense.py from the unmodified model/metric_functions/ and utils/util.py), and the C ABI's
argument checks.  GPU: the twelve reference-named functions and median_scaling against the golden, the oracle and a torch
restatement of the reference on the device."""
import ctypes

import numpy as np
import pytest
import torch

from tests import metrics_dense_oracle as MO
from tests.helpers import GOLDEN

gpu = pytest.mark.gpu
CASES = {"plain": dict(), "md": dict(max_distance=80.0), "roi": dict(roi=[2, 20, 5, 37]),
         "roi_md": dict(roi=[3, 21, 4, 36], max_distance=50.0), "roi_neg_md": dict(roi=[-20, -2, 0, 40], max_distance=30.0)}
TENSOR_SIGNATURE = ("sc_inv", "l1_rel", "l1_inv", "completeness", "covered_gt")


def _golden():
    return np.load(GOLDEN / "metrics_dense.npz")


def _assert_same(got, ref, rtol=5e-6):
    """Equal within rtol where finite; NaN and +-inf in the same places."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_array_equal(np.isinf(got) & (got > 0), np.isinf(ref) & (ref > 0))
    np.testing.assert_array_equal(np.isinf(got) & (got < 0), np.isinf(ref) & (ref < 0))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=rtol, atol=1e-7)


def _assert_bitwise(got, ref):
    """NaN in the same places, every other value the same fp32 bits."""
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    nan = np.isnan(ref)
    np.testing.assert_array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32))


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_golden_covers_the_ieee_and_median_edge_cases():
    g = _golden()
    assert np.isnan(g["case_plain"]).any() and np.isfinite(g["case_md"]).all()
    assert (g["gt"] == 0).any() and (g["pred"] == 0).any()
    counts = [int((g["ms_gt"][b] > 0).sum()) for b in range(g["ms_gt"].shape[0])]
    assert counts == [37, 40, 0, 21, 50]
    nan_img = np.isnan(g["ms_result"]).reshape(len(counts), -1).all(1)
    assert nan_img.tolist() == [False, False, True, True, False]


@pytest.mark.parametrize("tag", list(CASES))
def test_dense_oracle_matches_reference_golden(tag):
    g = _golden()
    got = MO.dense_metrics(g["pred"], g["gt"], **CASES[tag])
    _assert_same([got[n] for n in MO.DENSE_NAMES], g[f"case_{tag}"], rtol=2e-6)


def test_median_scaling_oracle_matches_reference_golden():
    g = _golden()
    scaled, _ = MO.median_scaling(g["ms_pred"], g["ms_gt"])
    _assert_bitwise(scaled, g["ms_result"])


def test_lower_median_is_torch_median():
    gen = torch.Generator().manual_seed(4)
    for n in (1, 2, 5, 6, 101, 1000):
        x = (torch.randint(0, 7, (n,), generator=gen) * 0.25 - 0.5).float()
        assert MO.lower_median(x.numpy()) == torch.median(x).item()


def _abi():
    from monorec_b200 import _lib
    return _lib.load()


def test_dense_metrics_group_validation_without_gpu():
    """Bad arguments of mr_dense_metrics, the group size included, give MR_EINVAL and a message naming the field, before any
    CUDA call (fake, never dereferenced pointers)."""
    lib = _abi()
    p, t, o, ws = 0x7F0000100000, 0x7F0000200000, 0x7F0000300000, 0x7F0000400000
    assert lib.mr_dense_metrics_workspace(4) == 4 * 13 * 8 and lib.mr_dense_metrics_workspace(0) == 0

    def call(p=p, t=t, o=o, ws=ws, B=2, group=2, H=8, W=8, roi=None, ws_bytes=1024):
        rc = lib.mr_dense_metrics(p, t, B, group, H, W, roi, 0.0, o, ws, ws_bytes, None)
        return rc, lib.mr_last_error().decode()

    empty = (ctypes.c_int * 4)(5, 5, 0, 8)
    for kw, text in ((dict(p=None), "result"), (dict(t=None), "target"), (dict(o=None), "out_metrics"),
                     (dict(ws=None), "workspace"), (dict(B=0), "B=0"), (dict(H=0), "H=0"), (dict(W=-1), "W=-1"),
                     (dict(roi=empty), "roi"), (dict(ws=ws + 4), "aligned"), (dict(group=0), "group=0")):
        rc, msg = call(**kw)
        assert rc == -1 and text in msg, (kw, rc, msg)
    rc, msg = call(ws_bytes=8)
    assert rc != 0 and "workspace too small" in msg


def test_median_scaling_validation_without_gpu():
    lib = _abi()
    p, t, o, ws = 0x7F0000100000, 0x7F0000200000, 0x7F0000300000, 0x7F0000400000
    assert lib.mr_median_scaling_workspace(4, 256, 512) >= 2 * 4 * 256 * 512 * 4 + 4 * 12
    assert lib.mr_median_scaling_workspace(0, 256, 512) == 0

    def call(p=p, t=t, o=o, ws=ws, B=2, H=8, W=8, ws_bytes=1 << 20):
        rc = lib.mr_median_scaling(p, t, o, B, H, W, ws, ws_bytes, None)
        return rc, lib.mr_last_error().decode()

    for kw, text in ((dict(p=None), "result"), (dict(t=None), "target"), (dict(o=None), "out"), (dict(ws=None), "workspace"),
                     (dict(B=0), "B=0"), (dict(H=-2), "H=-2"), (dict(o=p), "alias"), (dict(ws=ws + 2), "aligned")):
        rc, msg = call(**kw)
        assert rc == -1 and text in msg, (kw, rc, msg)
    rc, msg = call(ws_bytes=64)
    assert rc != 0 and "workspace too small" in msg


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _call_all(M, pred, gt, kw, d=None):
    """The twelve reference-named functions with the reference's signatures -> list of 0-dim device tensors."""
    d = {"result": pred, "target": gt} if d is None else d
    return [getattr(M, f"{n}_metric")(pred, gt, **kw) if n in TENSOR_SIGNATURE else getattr(M, f"{n}_metric")(d, **kw)
            for n in MO.DENSE_NAMES]


@gpu
@pytest.mark.parametrize("tag", list(CASES))
def test_cuda_dense_metrics_match_reference_golden(tag):
    from monorec_b200 import _lib
    from monorec_b200 import metrics as M
    g = _golden()
    pred, gt = torch.from_numpy(g["pred"]).cuda(), torch.from_numpy(g["gt"]).cuda()
    d = {"result": pred, "target": gt}
    torch.cuda.synchronize()
    _lib.launch_count(reset=True)
    vals = torch.stack(_call_all(M, pred, gt, CASES[tag], d)).cpu().numpy()
    # the twelve reference-named functions share one pass: the sums kernel and the finalize kernel of mr_dense_metrics
    assert _lib.launch_count() == 2
    _assert_same(vals, g[f"case_{tag}"])
    out = M.dense_metrics(pred, gt, **CASES[tag])
    assert _lib.launch_count() == 2
    _assert_same(out.cpu().numpy(), g[f"case_{tag}"])


@gpu
def test_cuda_dense_metrics_cache_follows_the_tensors():
    """An in-place change of the prediction, another roi or max_distance, or a new tensor runs the pass again."""
    from monorec_b200 import metrics as M
    g = _golden()
    pred, gt = torch.from_numpy(g["pred"]).cuda(), torch.from_numpy(g["gt"]).cuda()
    d = {"result": pred, "target": gt}
    a = float(M.l1_inv_metric(pred, gt))
    assert float(M.a1_metric(d, max_distance=80.0)) == pytest.approx(g["case_md"][0], rel=5e-6)
    pred.mul_(0.5)
    assert float(M.l1_inv_metric(pred, gt)) != a
    ref = MO.dense_metrics(pred.cpu().numpy(), g["gt"], max_distance=80.0)
    assert float(M.a1_metric(d, max_distance=80.0)) == pytest.approx(ref["a1"], rel=5e-6)
    assert float(M.a1_metric(d, roi=[2, 20, 5, 37], max_distance=80.0)) == pytest.approx(
        MO.dense_metrics(pred.cpu().numpy(), g["gt"], roi=[2, 20, 5, 37], max_distance=80.0)["a1"], rel=5e-6)
    with pytest.raises(ZeroDivisionError):                     # 1 / max_distance, as in the reference
        M.a1_metric(d, max_distance=0)


@gpu
def test_cuda_dense_metrics_match_oracle_at_full_size():
    """B 4 at 256x512 with a LiDAR-like target (~5 % of the pixels) and zeros in the prediction."""
    from monorec_b200 import metrics as M
    gen = torch.Generator().manual_seed(6)
    B, H, W = 4, 256, 512
    pred = torch.rand(B, 1, H, W, generator=gen) * 0.3 + 0.002
    gt = (pred * (1 + 0.2 * torch.randn(B, 1, H, W, generator=gen))).clamp_min(1e-3)
    gt[torch.rand(B, 1, H, W, generator=gen) > 0.05] = 0.0
    pred[torch.rand(B, 1, H, W, generator=gen) < 0.01] = 0.0
    for kw in (dict(roi=[40, 250, 20, 500], max_distance=80.0), dict()):
        out = M.dense_metrics(pred.cuda(), gt.cuda(), **kw).cpu().numpy()
        ref = MO.dense_metrics(pred.numpy(), gt.numpy(), **kw)
        _assert_same(out, [ref[n] for n in MO.DENSE_NAMES])


def _torch_median_scaling(data_dict):
    """utils/util.py:135-142 restated with the same torch calls."""
    target, prediction = data_dict["target"], data_dict["result"]
    mask = target > 0
    ratios = mask.new_tensor([torch.median(target[i, mask[i]]) / torch.median(prediction[i, mask[i]])
                              for i in range(target.shape[0])], dtype=torch.float32)
    out = dict(data_dict)
    out["result"] = prediction * ratios.view(-1, 1, 1, 1)
    return out


@gpu
def test_cuda_median_scaling_matches_reference_golden():
    from monorec_b200 import metrics as M
    g = _golden()
    pred, gt = torch.from_numpy(g["ms_pred"]).cuda(), torch.from_numpy(g["ms_gt"]).cuda()
    p0, t0 = pred.clone(), gt.clone()
    d = {"result": pred, "target": gt, "other": 3}
    out = M.median_scaling(d)
    _assert_bitwise(out["result"].cpu().numpy(), g["ms_result"])
    assert out is not d and out["target"] is gt and out["other"] == 3 and out["result"].shape == pred.shape
    assert d["result"] is pred and set(d) == {"result", "target", "other"}
    assert torch.equal(pred.nan_to_num(-1), p0.nan_to_num(-1)) and torch.equal(gt.nan_to_num(-1), t0.nan_to_num(-1))


@gpu
def test_cuda_median_scaling_bitwise_at_full_size():
    """B 4 at 256x512: a sparse target, a dense one with ties, and an image without any target, against the reference's
    torch calls on the device and the numpy oracle."""
    from monorec_b200 import metrics as M
    gen = torch.Generator().manual_seed(8)
    B, H, W = 4, 256, 512
    pred = torch.rand(B, 1, H, W, generator=gen) * 0.3 + 0.002
    gt = (pred * (1 + 0.2 * torch.randn(B, 1, H, W, generator=gen))).clamp_min(1e-3)
    gt[0][torch.rand(1, H, W, generator=gen) > 0.05] = 0.0                       # LiDAR-like
    gt[1] = (gt[1] * 16).round() / 16                                            # dense, many ties and zeros
    gt[2] = 0.0
    gt[3][torch.rand(1, H, W, generator=gen) > 0.5] = -1.0
    d = {"result": pred.cuda(), "target": gt.cuda()}
    out = M.median_scaling(d)["result"].cpu().numpy()
    ref = _torch_median_scaling(d)["result"].cpu().numpy()
    _assert_bitwise(out, ref)
    _assert_bitwise(out, MO.median_scaling(pred.numpy(), gt.numpy())[0])
    assert np.isnan(out[2]).all() and np.isfinite(out[[0, 1, 3]]).all()
    # the evaluater applies it before every metric: the sparse-metric cache of the unscaled result does not carry over
    M.a1_sparse_metric(d)
    assert "_mr_metrics_cache" in d and "_mr_metrics_cache" not in M.median_scaling(d)


@gpu
def test_cuda_metrics_reject_cpu_and_bad_shapes():
    from monorec_b200 import _lib
    from monorec_b200 import metrics as M
    x = torch.rand(2, 1, 8, 8)
    with pytest.raises(_lib.MonorecLibraryError):
        M.sc_inv_metric(x, x)
    with pytest.raises(_lib.MonorecLibraryError):
        M.median_scaling({"result": x, "target": x})
    with pytest.raises(ValueError):
        M.l1_inv_metric(x.cuda(), x[:, :, :4].cuda())
    with pytest.raises(ValueError):
        M.median_scaling({"result": x.cuda().half(), "target": x.cuda()})
