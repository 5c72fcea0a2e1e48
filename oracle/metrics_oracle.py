"""CPU restatement (numpy) of the reference's sparse depth metrics -- TEST INFRASTRUCTURE, never imported by the product.

Follows model/metric_functions/sparse_metrics.py:81-251 with the helpers of utils/util.py:36-65 (preprocess_roi,
get_absolute_depth, get_positive_depth), :101-107 (get_mask) and :110-118 (mask_mean).  Pinned on tests/golden/metrics.npz,
which tests/golden/make_golden.py --only-metrics writes by calling the unmodified reference functions.
"""
import numpy as np


def sparse_metrics(pred, gt, mvobj_mask=None, roi=None, max_distance=None, pred_all_valid=True):
    """pred, gt: [B,1,H,W] inverse depths -> dict of the seven metrics (float64 accumulation of fp32 per-pixel terms)."""
    pred = np.asarray(pred, np.float32)
    gt = np.asarray(gt, np.float32)
    if roi is not None:                                            # utils/util.py:36-43
        pred = pred[:, :, roi[0]:roi[1], roi[2]:roi[3]]
        gt = gt[:, :, roi[0]:roi[1], roi[2]:roi[3]]
        if mvobj_mask is not None:
            mvobj_mask = np.asarray(mvobj_mask)[:, :, roi[0]:roi[1], roi[2]:roi[3]]
    mask = gt == 0                                                 # :101-107 (True = excluded)
    if max_distance:
        mask |= gt < np.float32(1.0 / max_distance)
    if not pred_all_valid:
        mask |= pred == 0
    if mvobj_mask is not None:                                     # sparse_metrics.py:86 `mask |= ~(mvobj_mask > .5)`
        mask |= ~(np.asarray(mvobj_mask, np.float32) > 0.5)
    # :59-65, torch's relu: NaN and -0.0 pass through (np.maximum(-0.0, 0) would give +0.0, whose inverse is +inf, not -inf)
    p, g = np.where(pred < 0, np.float32(0), pred), np.where(gt < 0, np.float32(0), gt)
    if max_distance is not None:                                   # :46-56
        p = np.maximum(p, np.float32(1.0 / max_distance))
        g = np.maximum(g, np.float32(1.0 / max_distance))
    with np.errstate(divide="ignore", invalid="ignore"):
        dp, dg = np.float32(1) / p, np.float32(1) / g
        dp = np.where(mask, np.float32(1), dp)                     # the *_base functions set masked entries to 1 (or zero them later)
        dg = np.where(mask, np.float32(1), dg)
        th = np.maximum(dg / dp, dp / dg)
        se = (dp - dg) ** 2
        sle = (np.log(dp) - np.log(dg)) ** 2
        ar = np.abs(dp - dg) / dg
        sr = (dp - dg) ** 2 / dg
    keep = ~mask
    n_all = keep.sum(dtype=np.float64)
    n_img = keep.sum(axis=(1, 2, 3), dtype=np.float64)

    def mean_all(t):
        return float((t * keep).sum(dtype=np.float64) / n_all)

    def mean_of_roots(t):
        with np.errstate(divide="ignore", invalid="ignore"):
            return float(np.mean(np.sqrt((t * keep).sum(axis=(1, 2, 3), dtype=np.float64) / n_img)))

    return {"a1": mean_all((th < 1.25).astype(np.float32)), "a2": mean_all((th < 1.25 ** 2).astype(np.float32)),
            "a3": mean_all((th < 1.25 ** 3).astype(np.float32)), "rmse": mean_of_roots(se), "rmse_log": mean_of_roots(sle),
            "abs_rel": mean_all(ar), "sq_rel": mean_all(sr)}
