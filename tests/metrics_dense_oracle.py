"""CPU restatement (numpy) of the reference's dense and completeness depth metrics and of the evaluater's median scaling --
test infrastructure, never imported by the product.

Follows model/metric_functions/sparse_metrics.py:6-78, dense_metrics.py and completeness_metrics.py with the helpers of
utils/util.py:36-65 (preprocess_roi, get_absolute_depth, get_positive_depth) and :110-118 (mask_mean), and utils/util.py:135-142
(median_scaling).  Pinned on tests/golden/metrics_dense.npz, which tests/golden/make_golden_metrics_dense.py writes by calling
the unmodified reference functions.
"""
import numpy as np

DENSE_NAMES = ("a1", "a2", "a3", "rmse", "rmse_log", "abs_rel", "sq_rel", "sc_inv", "l1_rel", "l1_inv", "completeness",
               "covered_gt")


def dense_metrics(pred, gt, roi=None, max_distance=None):
    """The twelve dense-ground-truth metrics: the *_metric functions of model/metric_functions/sparse_metrics.py:6-78,
    dense_metrics.py (sc_inv, l1_rel, l1_inv) and completeness_metrics.py (completeness, covered_gt).  pred, gt: [B,1,H,W]
    inverse depths -> dict (fp32 per-pixel terms, float64 sums).  Pinned on tests/golden/metrics_dense.npz."""
    pred = np.asarray(pred, np.float32)
    gt = np.asarray(gt, np.float32)
    B = pred.shape[0]
    out = {"completeness": float((pred != 0).mean(dtype=np.float64)),                   # completeness_metrics.py: no roi
           "covered_gt": float(((pred != 0) & ~(gt != 0)).sum(dtype=np.float64) / (~(gt != 0)).sum(dtype=np.float64))}
    if roi is not None:                                            # utils/util.py:36-43
        pred = pred[:, :, roi[0]:roi[1], roi[2]:roi[3]]
        gt = gt[:, :, roi[0]:roi[1], roi[2]:roi[3]]
    n = gt.shape[2] * gt.shape[3]
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.where(np.isnan(pred), pred, np.maximum(pred, np.float32(0)))           # relu keeps a NaN
        g = np.where(np.isnan(gt), gt, np.maximum(gt, np.float32(0)))
        out["l1_inv"] = float(np.abs(p - g).mean(dtype=np.float64))
        if max_distance is not None:                               # :46-56 (`is not None`, unlike get_mask)
            lo = np.float32(1 / max_distance)
            p = np.where(np.isnan(p), p, np.maximum(p, lo))
            g = np.where(np.isnan(g), g, np.maximum(g, lo))
        dp, dg = np.float32(1) / p, np.float32(1) / g
        a, b = dg / dp, dp / dg
        th = np.where(np.isnan(a) | np.isnan(b), np.float32(np.nan), np.maximum(a, b))  # torch.max propagates NaN
        diff = dp - dg
        se = diff * diff
        E = np.log(dp) - np.log(dg)
        sle = E * E
        E = np.where(np.isnan(E), np.float32(0), E)
        for name, t in (("a1", 1.25), ("a2", 1.25 ** 2), ("a3", 1.25 ** 3)):
            out[name] = float((th < np.float32(t)).mean(dtype=np.float64))
        out["rmse"] = float(np.mean(np.sqrt(se.reshape(B, -1).sum(1, dtype=np.float64) / n)))
        out["rmse_log"] = float(np.mean(np.sqrt(sle.reshape(B, -1).sum(1, dtype=np.float64) / n)))
        out["abs_rel"] = out["l1_rel"] = float((np.abs(diff) / dg).mean(dtype=np.float64))
        out["sq_rel"] = float((se / dg).mean(dtype=np.float64))
        s1 = E.reshape(B, -1).sum(1, dtype=np.float64)
        s2 = (E * E).reshape(B, -1).sum(1, dtype=np.float64)
        v = np.sqrt(s2 / n - s1 * s1 / (n * n))
        out["sc_inv"] = float(np.mean(np.where(np.isnan(v), 0.0, v)))
    return out


def lower_median(x):
    """torch.median of a 1-D fp32 set: element (n - 1) // 2 of the sorted values; NaN if empty or holding a NaN."""
    x = np.asarray(x, np.float32).ravel()
    if x.size == 0 or np.isnan(x).any():
        return np.float32(np.nan)
    return np.partition(x, (x.size - 1) // 2)[(x.size - 1) // 2]


def median_scaling(pred, gt):
    """utils/util.py:135-142: pred * (median(gt[gt > 0]) / median(pred[gt > 0])) per image, all in fp32 -> (scaled, ratios)."""
    pred = np.asarray(pred, np.float32)
    gt = np.asarray(gt, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratios = np.array([lower_median(gt[i][gt[i] > 0]) / lower_median(pred[i][gt[i] > 0]) for i in range(pred.shape[0])],
                          dtype=np.float32)
        return pred * ratios.reshape(-1, 1, 1, 1), ratios
