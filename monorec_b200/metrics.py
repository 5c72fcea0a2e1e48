"""Drop-ins for the reference's depth metrics (model/metric.py: model/metric_functions/sparse_metrics.py,
dense_metrics.py, completeness_metrics.py), the evaluater's median scaling (utils/util.py:135-142) and the loader's image
normalisation (data_loader/kitti_odometry_dataset.py:121-132), computed on the device by libmonorec_b200.so.

The reference's evaluater (evaluater/evaluater.py:78-112) calls the configured metric functions one after the other, each a
dozen elementwise torch kernels and a few reductions.  Here the 21 `*_sparse*` metrics come out of ONE fused pass
(`mr_sparse_metrics`) and the 12 dense and completeness metrics out of another (`mr_dense_metrics`); the functions below keep
the reference's names and signatures and share those passes through a small cache, so `model.metric` can be pointed at this
module unchanged.  Each pass writes one row of metrics per group of `group` consecutive images; the functions below take
the whole batch as one group, and the sequence evaluation (`evaluation.py`) takes one row per evaluater batch from the
`*_grouped_impl` functions.  No CPU fallback.
"""
import ctypes
import weakref
from typing import List, Optional

import torch
from torch import Tensor

from . import _lib

NAMES = ("a1", "a2", "a3", "rmse", "rmse_log", "abs_rel", "sq_rel")


def sparse_metrics(data_dict, roi=None, max_distance=None, pred_all_valid=True, use_cvmask=False):
    """-> device tensor [7]: a1, a2, a3, rmse, rmse_log, abs_rel, sq_rel (no host synchronisation)."""
    pred, gt = data_dict["result"], data_dict["target"]
    if not pred.is_cuda:
        raise _lib.MonorecLibraryError("monorec_b200.metrics needs CUDA tensors (no CPU fallback)")
    mv = data_dict["mvobj_mask"] if use_cvmask else None
    roi_l = None if roi is None else [int(v) for v in roi]
    max_d = float(max_distance) if max_distance else 0.0
    if torch.compiler.is_compiling():
        return torch.ops.monorec_b200.sparse_metrics(pred, gt, mv, roi_l, max_d, bool(pred_all_valid))
    key = (id(pred), pred._version, id(gt), gt._version, None if roi is None else tuple(int(v) for v in roi),
           None if max_distance is None else float(max_distance), bool(pred_all_valid), bool(use_cvmask))
    cache = data_dict.get("_mr_metrics_cache")
    if cache is not None and cache[0] == key:
        return cache[1]
    out = sparse_metrics_impl(pred, gt, mv, roi_l, max_d, bool(pred_all_valid))
    data_dict["_mr_metrics_cache"] = (key, out)
    return out


def sparse_metrics_impl(pred: Tensor, gt: Tensor, mvobj_mask: Optional[Tensor], roi: Optional[List[int]],
                        max_distance: float, pred_all_valid: bool) -> Tensor:
    """The fused sparse pass over the whole batch -> [7].  sparse_metrics calls this directly; under torch.compile it is the
    implementation of the `monorec_b200::sparse_metrics` op."""
    # group = B (an empty batch keeps group 1, so that the library reports it)
    return sparse_metrics_grouped_impl(pred, gt, mvobj_mask, roi, max_distance, pred_all_valid, max(pred.shape[0], 1))[0]


def sparse_metrics_grouped_impl(pred: Tensor, gt: Tensor, mvobj_mask: Optional[Tensor], roi: Optional[List[int]],
                                max_distance: float, pred_all_valid: bool, group: int) -> Tensor:
    """The fused sparse pass (mr_sparse_metrics) over groups of `group` images -> [G,7], G = ceil(B / group): row g holds the
    metrics of images [g * group, (g + 1) * group) (the last group may be shorter); max_distance 0 = none."""
    lib = _lib.load()
    pred = pred.to(torch.float32).contiguous()
    gt = gt.to(device=pred.device, dtype=torch.float32).contiguous()
    B, _, H, W = pred.shape
    mv = None if mvobj_mask is None else mvobj_mask.to(device=pred.device, dtype=torch.float32).contiguous()
    out = torch.empty(-(-B // group), 7, device=pred.device, dtype=torch.float32)
    ws_bytes = lib.mr_sparse_metrics_workspace(B)
    ws = torch.empty(ws_bytes // 8, device=pred.device, dtype=torch.float64)
    roi_c = None if roi is None else (ctypes.c_int * 4)(*roi)
    with torch.cuda.device(pred.device):
        _lib.check(lib.mr_sparse_metrics(pred.data_ptr(), gt.data_ptr(), None if mv is None else mv.data_ptr(), B, int(group),
                                         H, W, roi_c, max_distance, 1 if pred_all_valid else 0, out.data_ptr(), ws.data_ptr(),
                                         ws_bytes, torch.cuda.current_stream(pred.device).cuda_stream), "mr_sparse_metrics")
    return out


def _make(index, **fixed):
    def metric(data_dict, roi=None, max_distance=None, pred_all_valid=True, use_cvmask=False):
        kw = dict(pred_all_valid=pred_all_valid, use_cvmask=use_cvmask)
        kw.update(fixed)
        return sparse_metrics(data_dict, roi, max_distance, **kw)[index]
    return metric


for _i, _n in enumerate(NAMES):
    globals()[f"{_n}_sparse_metric"] = _make(_i)                                        # sparse_metrics.py:81-156
    globals()[f"{_n}_sparse_onlyvalid_metric"] = _make(_i, pred_all_valid=False)        # :159-184
    globals()[f"{_n}_sparse_onlydynamic_metric"] = _make(_i, use_cvmask=True)           # :187-212


DENSE_NAMES = NAMES + ("sc_inv", "l1_rel", "l1_inv", "completeness", "covered_gt")
# the last dense pass: (weakref to result, weakref to target, key, out).  Keyed on the tensors rather than on a data_dict, so
# that the data_dict functions and the tensor-signature functions of one call set share it, and weak, so that a freed
# tensor whose id is reused never matches
_dense_last = [None]


def _check_pair(pred, gt, what):
    if not pred.is_cuda:
        raise _lib.MonorecLibraryError(f"{what} needs CUDA tensors (no CPU fallback)")
    if pred.dim() != 4 or pred.shape[1] != 1 or tuple(gt.shape) != tuple(pred.shape):
        raise ValueError(f"{what}: result and target must both be [B,1,H,W], got {tuple(pred.shape)} and {tuple(gt.shape)}")


def dense_metrics(depth_prediction, depth_gt, roi=None, max_distance=None):
    """-> device tensor [12] in the order of DENSE_NAMES (no host synchronisation), from one fused pass (`mr_dense_metrics`).

    The pass is remembered for these two tensors at their current version and this (roi, max_distance), so the twelve
    reference-named functions below cost one launch group per call set."""
    pred, gt = depth_prediction, depth_gt
    _check_pair(pred, gt, "monorec_b200.metrics.dense_metrics")
    roi_l = None if roi is None else [int(v) for v in roi]
    # get_absolute_depth (utils/util.py:46-56) clamps at the fp32 rounding of 1 / max_distance (a ZeroDivisionError for 0)
    min_inv = 0.0 if max_distance is None else 1 / max_distance
    if torch.compiler.is_compiling():
        return torch.ops.monorec_b200.dense_metrics(pred, gt, roi_l, float(min_inv))
    key = (pred._version, gt._version, None if roi is None else tuple(int(v) for v in roi),
           None if max_distance is None else float(max_distance))
    hit = _dense_last[0]
    if hit is not None and hit[0]() is pred and hit[1]() is gt and hit[2] == key:
        return hit[3]
    out = dense_metrics_impl(pred, gt, roi_l, float(min_inv))
    _dense_last[0] = (weakref.ref(pred), weakref.ref(gt), key, out)
    return out


def dense_metrics_impl(pred: Tensor, gt: Tensor, roi: Optional[List[int]], min_inv: float) -> Tensor:
    """The fused dense pass over the whole batch -> [12].  dense_metrics calls this directly; under torch.compile it is the
    implementation of the `monorec_b200::dense_metrics` op."""
    # group = B (an empty batch keeps group 1, so that the library reports it)
    return dense_metrics_grouped_impl(pred, gt, roi, min_inv, max(pred.shape[0], 1))[0]


def dense_metrics_grouped_impl(pred: Tensor, gt: Tensor, roi: Optional[List[int]], min_inv: float, group: int) -> Tensor:
    """The fused dense pass (mr_dense_metrics) over groups of `group` images -> [G,12]: row g holds the metrics of images
    [g * group, (g + 1) * group)."""
    lib = _lib.load()
    p = pred.to(torch.float32).contiguous()
    g = gt.to(device=p.device, dtype=torch.float32).contiguous()
    B, _, H, W = p.shape
    out = torch.empty(-(-B // group), len(DENSE_NAMES), device=p.device, dtype=torch.float32)
    ws_bytes = lib.mr_dense_metrics_workspace(B)
    ws = torch.empty(ws_bytes // 8, device=p.device, dtype=torch.float64)
    roi_c = None if roi is None else (ctypes.c_int * 4)(*roi)
    with torch.cuda.device(p.device):
        _lib.check(lib.mr_dense_metrics(p.data_ptr(), g.data_ptr(), B, int(group), H, W, roi_c, min_inv, out.data_ptr(),
                                        ws.data_ptr(), ws_bytes, torch.cuda.current_stream(p.device).cuda_stream), "mr_dense_metrics")
    return out


def _make_dense_dict(index):
    def metric(data_dict, roi=None, max_distance=None):
        return dense_metrics(data_dict["result"], data_dict["target"], roi, max_distance)[index]
    metric.__name__ = f"{DENSE_NAMES[index]}_metric"
    return metric


def _make_dense_tensor(index, doc):
    def metric(depth_prediction, depth_gt, roi=None, max_distance=None):
        return dense_metrics(depth_prediction, depth_gt, roi, max_distance)[index]
    metric.__name__ = f"{DENSE_NAMES[index]}_metric"
    metric.__doc__ = doc
    return metric


# sparse_metrics.py:6-78: data_dict signature, every pixel of the roi counts
for _i, _n in enumerate(NAMES):
    globals()[f"{_n}_metric"] = _make_dense_dict(_i)
# dense_metrics.py and completeness_metrics.py: (depth_prediction, depth_gt, roi, max_distance)
sc_inv_metric = _make_dense_tensor(7, """Scale-invariant error: per image sqrt(sum E^2 / n - (sum E)^2 / n^2) with E = log of the
    predicted over the true depth (NaN -> 0) and n the roi's pixel count; an image whose value is NaN counts 0.  Sums in
    float64, where the reference sums in fp32: images whose E is nearly constant can differ by more than rounding.""")
l1_rel_metric = _make_dense_tensor(8, "Mean |d_pred - d_gt| / d_gt of the depths (the formula of abs_rel_metric).")
l1_inv_metric = _make_dense_tensor(9, "Mean |p - g| of the inverse depths after relu: no clamp at max_distance.")
completeness_metric = _make_dense_tensor(10, "Share of pixels with result != 0 over the whole tensor (ignores roi and "
                                             "max_distance).")
covered_gt_metric = _make_dense_tensor(11, """mask_mean((result != 0), target != 0) as written in the reference: mask_mean
    drops the masked entries, so this is the share of pixels with result != 0 among the pixels where target == 0 (NaN when
    there is none), not among the pixels with ground truth.  Ignores roi and max_distance.""")


def median_scaling(data_dict):
    """utils/util.py:135-142 on the device (`mr_median_scaling`): a shallow copy of `data_dict` whose "result" is the
    prediction times, per image, median(target[target > 0]) / median(result[target > 0]), in fp32 and bit for bit as the
    reference computes it, without a host synchronisation.  Each median is torch.median's lower median; an image with no
    target > 0, or a NaN among its selected predictions, gets a NaN ratio.  The input dict and its tensors are not modified."""
    pred, gt = data_dict["result"], data_dict["target"]
    _check_pair(pred, gt, "monorec_b200.metrics.median_scaling")
    if pred.dtype != torch.float32:
        raise ValueError(f"median_scaling: result must be float32, got {pred.dtype}")
    run = torch.ops.monorec_b200.median_scaling if torch.compiler.is_compiling() else median_scaling_impl
    scaled = dict(data_dict)
    scaled["result"] = run(pred, gt)
    # the sparse pass cached for the unscaled result is keyed on its id, which a later tensor may reuse once it is freed
    scaled.pop("_mr_metrics_cache", None)
    return scaled


def median_scaling_impl(pred: Tensor, gt: Tensor) -> Tensor:
    """mr_median_scaling: the scaled prediction.  median_scaling calls this directly; under torch.compile it is the
    implementation of the `monorec_b200::median_scaling` op."""
    lib = _lib.load()
    p = pred.contiguous()
    g = gt.to(device=p.device, dtype=torch.float32).contiguous()
    B, _, H, W = p.shape
    out = torch.empty_like(p)
    ws_bytes = lib.mr_median_scaling_workspace(B, H, W)
    ws = torch.empty(ws_bytes // 4, device=p.device, dtype=torch.float32)
    with torch.cuda.device(p.device):
        _lib.check(lib.mr_median_scaling(p.data_ptr(), g.data_ptr(), out.data_ptr(), B, H, W, ws.data_ptr(), ws_bytes,
                                         torch.cuda.current_stream(p.device).cuda_stream), "mr_median_scaling")
    return out


def eval_accumulate_impl(values: Tensor, group_sizes: List[int], state: Tensor) -> Tensor:
    """mr_eval_accumulate: folds the metric rows `values` [G,M] (fp32, device) of G evaluater batches of `group_sizes`
    images into `state` (float64 [3M+1] on the device: total, valid, running average, number of samples), in place, as
    evaluater.py:45-49, 94-103 does batch after batch.  Returns `state`."""
    lib = _lib.load()
    v = values.to(torch.float32).contiguous()
    G, M = v.shape
    if len(group_sizes) != G or state.dtype != torch.float64 or state.numel() != 3 * M + 1 or not state.is_contiguous():
        raise ValueError(f"eval_accumulate: {len(group_sizes)} group sizes and a {state.dtype} state of {state.numel()} "
                         f"values for metric rows {tuple(v.shape)} (float64 [3M+1] contiguous expected)")
    sizes = (ctypes.c_int * G)(*[int(n) for n in group_sizes])
    with torch.cuda.device(v.device):
        _lib.check(lib.mr_eval_accumulate(v.data_ptr(), G, M, sizes, state.data_ptr(),
                                          torch.cuda.current_stream(v.device).cuda_stream), "mr_eval_accumulate")
    return state


def images_u8_to_f32(images_u8, crop_box=None):
    """uint8 HWC images [B,Hs,Ws,3] on the device -> float CHW [B,3,H,W] = u / 255 - 0.5, optionally cropped to the PIL-style
    box (left, upper, right, lower) -- kitti_odometry_dataset.py:121-132 without the resize."""
    if not images_u8.is_cuda or images_u8.dtype != torch.uint8 or images_u8.dim() != 4 or images_u8.shape[3] != 3:
        raise _lib.MonorecLibraryError("images_u8_to_f32 expects a CUDA uint8 tensor [B,H,W,3]")
    lib = _lib.load()
    x = images_u8.contiguous()
    B, Hs, Ws, _ = x.shape
    left, top, right, bottom = (0, 0, Ws, Hs) if crop_box is None else [int(v) for v in crop_box]
    H, W = bottom - top, right - left
    out = torch.empty(B, 3, H, W, device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(lib.mr_images_u8_to_f32(x.data_ptr(), out.data_ptr(), B, Hs, Ws, top, left, H, W,
                                           torch.cuda.current_stream(x.device).cuda_stream), "mr_images_u8_to_f32")
    return out


from . import ops  # noqa: E402,F401  (registers the metric ops, which the functions above call under torch.compile)
