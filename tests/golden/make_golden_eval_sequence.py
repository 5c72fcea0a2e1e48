#!/usr/bin/env python
"""Writes tests/golden/eval_sequence.npz by running the UNMODIFIED reference evaluater on CPU fp32:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_eval_sequence.py

`Evaluater.eval` (evaluater/evaluater.py:54-119) runs on an instance built without its constructor (which wants a parsed
config and a logger directory): a data loader that yields seeded (data, target) batches of key frames in order, an identity
"model" that puts precomputed `result` tensors into the data dict, device "cpu", the reference's metric functions.  The
tensor-signature metrics of dense_metrics.py / completeness_metrics.py (sc_inv, l1_rel, l1_inv, completeness, covered_gt)
take (depth_prediction, depth_gt, roi, max_distance) rather than the data dict the evaluater passes, so they are called
through a one-line adapter that hands them data_dict["result"] and data_dict["target"].

Stored:
  result, target        [N,1,H,W] fp32 inverse depths of N key frames: a few exact zeros in the prediction, a LiDAR-like
                        target (~25 % of the pixels), and key frame 3 without any ground truth (its batch has a NaN metric)
  cases                 JSON: per case the metric names, batch_size, the number n of leading key frames evaluated, roi,
                        max_distance and median_scaling
  <tag>_raw             float32 [batches, M]: every metric value the evaluater computed, batch by batch (before its NaN rule)
  <tag>_metrics, <tag>_metrics_correct, <tag>_valid_batches: the log dict's entries (float64)
"""
import json
import logging
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)

SPARSE7 = ["abs_rel_sparse_metric", "sq_rel_sparse_metric", "rmse_sparse_metric", "rmse_log_sparse_metric",
           "a1_sparse_metric", "a2_sparse_metric", "a3_sparse_metric"]                 # configs/evaluate/eval_monorec.json
DENSE12 = ["a1_metric", "a2_metric", "a3_metric", "rmse_metric", "rmse_log_metric", "abs_rel_metric", "sq_rel_metric",
           "sc_inv_metric", "l1_rel_metric", "l1_inv_metric", "completeness_metric", "covered_gt_metric"]
TENSOR_SIGNATURE = {"sc_inv_metric", "l1_rel_metric", "l1_inv_metric", "completeness_metric", "covered_gt_metric"}

CASES = {
    # the shipped config: ragged last batch (9 = 4 x 2 + 1), batch 1 holds the key frame without ground truth
    "eval_config": dict(names=SPARSE7, batch_size=2, n=9, roi=None, max_distance=80, median_scaling=False),
    # median scaling before every metric, roi, the onlyvalid variants; 8 = 3 + 3 + 2
    "ms_roi_onlyvalid": dict(names=["a1_sparse_metric", "abs_rel_sparse_onlyvalid_metric", "rmse_sparse_metric",
                                    "rmse_log_sparse_onlyvalid_metric", "sq_rel_sparse_metric", "a3_sparse_onlyvalid_metric"],
                             batch_size=3, n=8, roi=[2, 14, 3, 22], max_distance=50, median_scaling=True),
    # all twelve dense / completeness names with sparse ones in one list; 9 = 4 + 4 + 1
    "dense_sparse": dict(names=DENSE12 + ["rmse_sparse_metric", "a2_sparse_onlyvalid_metric"], batch_size=4, n=9,
                         roi=[1, 15, 2, 20], max_distance=80, median_scaling=False),
    # dense and sparse names under median scaling, without a roi; 7 = 2 + 2 + 2 + 1
    "dense_ms": dict(names=["abs_rel_metric", "sc_inv_metric", "a1_sparse_metric", "l1_inv_metric", "rmse_metric",
                            "covered_gt_metric", "sq_rel_sparse_onlyvalid_metric"],
                     batch_size=2, n=7, roi=None, max_distance=30, median_scaling=True),
}


def inputs(N=9, H=16, W=24):
    g = torch.Generator().manual_seed(41)
    result = torch.rand(N, 1, H, W, generator=g) * 0.3 + 0.01
    result[torch.rand(N, 1, H, W, generator=g) < 0.03] = 0.0                 # predictions that are exactly 0
    target = (result * (1 + 0.2 * torch.randn(N, 1, H, W, generator=g))).clamp_min(2e-3)
    target[torch.rand(N, 1, H, W, generator=g) > 0.25] = 0.0                 # LiDAR-like coverage
    target[result == 0] = 0.01
    target[3] = 0.0                                                          # a key frame without ground truth
    return result, target


class _InsertResult(torch.nn.Module):
    """The identity "model": adds the precomputed result of the batch's key frames to the data dict."""

    def __init__(self, result):
        super().__init__()
        self.result = result

    def forward(self, data):
        data["result"] = self.result[data["index"]].clone()
        return data


def run_case(Evaluater, module_metric, result, target, cfg):
    n, bs = cfg["n"], cfg["batch_size"]
    raw = []

    def recorded(name):
        fn = getattr(module_metric, name)
        if name in TENSOR_SIGNATURE:
            call = lambda d, roi=None, max_distance=None: fn(d["result"], d["target"], roi, max_distance)  # noqa: E731
        else:
            call = fn

        def metric(data_dict, roi=None, max_distance=None):
            v = call(data_dict, roi, max_distance)
            raw.append(np.float32(v.item()))
            return v
        metric.__name__ = name
        return metric

    ev = Evaluater.__new__(Evaluater)
    ev.model = _InsertResult(result)
    ev.data_loader = [({"index": torch.arange(b, min(b + bs, n))}, target[b:min(b + bs, n)].clone()) for b in range(0, n, bs)]
    ev.len_data = len(ev.data_loader)
    ev.device = "cpu"
    ev.logger = logging.getLogger("make_golden_eval_sequence")
    ev.log_step = 1
    ev.metrics = [recorded(name) for name in cfg["names"]]
    ev.roi, ev.max_distance, ev.median_scaling = cfg["roi"], cfg["max_distance"], cfg["median_scaling"]
    log = ev.eval(0)
    raw = np.array(raw, np.float32).reshape(ev.len_data, len(cfg["names"]))
    return log, raw


def main():
    torch.manual_seed(0)
    import_reference()
    from evaluater import Evaluater  # noqa
    import model.metric as module_metric  # noqa
    result, target = inputs()
    out = {"result": result.numpy(), "target": target.numpy(), "cases": np.array(json.dumps(CASES))}
    for tag, cfg in CASES.items():
        log, raw = run_case(Evaluater, module_metric, result, target, cfg)
        assert log["loss"] == 0.0 and log["loss_loss"] == 0.0
        out[f"{tag}_raw"] = raw
        out[f"{tag}_metrics"] = np.array(log["metrics"], np.float64)
        out[f"{tag}_metrics_correct"] = np.array(log["metrics_correct"], np.float64)
        out[f"{tag}_valid_batches"] = np.float64(log["valid_batches"])
        print(tag, "valid batches", log["valid_batches"], "of", raw.shape[0], "metrics", log["metrics"])
    path = HERE / "eval_sequence.npz"
    np.savez_compressed(path, **out)
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
