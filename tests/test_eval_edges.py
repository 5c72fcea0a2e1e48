"""The IEEE and slicing edges of the sparse metrics and the point-cloud export, on the oracles (CPU).

tests/golden/eval_edges.npz holds the unmodified reference's outputs (make_golden_eval_edges.py) for NaN, +-inf, negative and
-0.0 inputs and for rois with negative or out-of-range bounds.  The oracles are the CPU side of tests/test_eval_edges_gpu.py:
NaN and inf must come out in the same places as in the reference, finite values within the gates of test_metrics.py and
test_pointcloud.py."""
import numpy as np
import pytest
import torch

from tests import eval_edges_cases as E
from tests.helpers import GOLDEN


def _golden():
    return np.load(GOLDEN / "eval_edges.npz")


def test_golden_covers_the_edges():
    g = _golden()
    pred, gt, mv = g["pred"], g["gt"], g["mvobj"]
    assert np.isnan(pred[0]).any() and np.isposinf(pred[0]).any() and (pred[0] < 0).any()
    assert ((pred[0] == 0) & np.signbit(pred[0])).any() and ((pred[0] == 0) & ~np.signbit(pred[0])).any()
    assert np.isnan(gt[1]).any() and np.isposinf(gt[1]).any() and (gt[1] < 0).any()
    assert np.isnan(pred[2]).any() and (gt[2][np.isnan(pred[2])] == 0).all()          # NaN only where masked
    assert np.isnan(mv).any()
    # the NaN rows: image 0 and 1 in every set, image 4 only where its NaN is inside the roi and not masked by mvobj
    for tag in E.SPARSE_CASES:
        rows = g[f"sparse_{tag}"]
        assert np.isnan(rows[1, 3:]).all() and np.isfinite(rows[2]).all(), tag
        assert np.isfinite(rows[:, :3]).all(), tag                                   # a NaN pixel is a miss in a1-a3
        assert np.isnan(rows[3, 3]) == (tag not in ("onlydynamic", "roi_neg_md")), tag
    inv = g["pc_inv_depth"]
    with np.errstate(divide="ignore"):
        depth = np.float32(1) / inv
    assert (depth == E.PC_MIN_D).any() and (depth == E.PC_MAX_D).any()
    assert np.isnan(inv).any() and np.isinf(inv).any() and (inv == 0).any() and (inv < 0).any()
    assert g["pc_vertices_empty"].shape == (0, 6) and g["pc_vertices_neg"].shape[0] > 500


@pytest.mark.parametrize("tag", list(E.SPARSE_CASES))
def test_sparse_oracle_matches_reference_edges(tag):
    from oracle import metrics_oracle as MO
    g = _golden()
    kw = E.sparse_kwargs(tag)
    use_mv = kw.pop("use_cvmask")
    for k, (lo, hi) in enumerate(E.SLICES):
        got = MO.sparse_metrics(g["pred"][lo:hi], g["gt"][lo:hi], mvobj_mask=g["mvobj"][lo:hi] if use_mv else None, **kw)
        E.assert_same([got[n] for n in E.NAMES], g[f"sparse_{tag}"][k], rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("tag", list(E.PC_ROIS))
def test_pointcloud_oracle_matches_reference_edges(tag):
    from oracle import pointcloud_oracle as PO
    g = _golden()
    t = [torch.from_numpy(g[f"pc_{k}"]) for k in ("inv_depth", "image", "K", "pose")]
    v = PO.add_depthmap(*t, min_d=E.PC_MIN_D, max_d=E.PC_MAX_D, roi=E.PC_ROIS[tag])
    ref = torch.from_numpy(g[f"pc_vertices_{tag}"])
    assert v.shape == ref.shape
    assert torch.isfinite(ref).all()
    assert torch.equal(v[:, 3:], ref[:, 3:]) and torch.allclose(v, ref, rtol=1e-6, atol=1e-5)
