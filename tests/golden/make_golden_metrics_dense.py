#!/usr/bin/env python
"""Writes tests/golden/metrics_dense.npz by calling the UNMODIFIED reference on CPU fp32:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_metrics_dense.py

Stored (inputs in fp32, the reference's outputs as it returns them):
  pred, gt                 [3,1,24,40] inverse depths: zeros in both (image 2 has none), so without max_distance the
                           reference's inf / NaN outcomes appear
  case_<tag>               float64 [12]: a1 ... sq_rel (model/metric_functions/sparse_metrics.py:6-78), sc_inv, l1_rel,
                           l1_inv (dense_metrics.py), completeness, covered_gt (completeness_metrics.py) for the
                           (roi, max_distance) set CASES[tag]
  ms_pred, ms_gt           [5,1,16,24] inputs of utils.median_scaling: per image 37 (odd), 40 (even), 0, 21 (one NaN
                           prediction among them) and 50 (even, values on five levels: ties) pixels with target > 0; negative
                           and NaN targets are not selected
  ms_result                the reference's scaled "result"
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)
from tests.metrics_dense_oracle import DENSE_NAMES  # noqa: E402

CASES = {"plain": dict(), "md": dict(max_distance=80.0), "roi": dict(roi=[2, 20, 5, 37]),
         "roi_md": dict(roi=[3, 21, 4, 36], max_distance=50.0), "roi_neg_md": dict(roi=[-20, -2, 0, 40], max_distance=30.0)}


def dense_inputs():
    g = torch.Generator().manual_seed(31)
    B, H, W = 3, 24, 40
    pred = torch.rand(B, 1, H, W, generator=g) * 0.3 + 0.002
    gt = (pred * (1 + 0.25 * torch.randn(B, 1, H, W, generator=g))).clamp_min(1e-3)
    pred[:2][torch.rand(2, 1, H, W, generator=g) < 0.03] = 0.0       # predictions that are exactly 0
    gt[:2][torch.rand(2, 1, H, W, generator=g) < 0.10] = 0.0         # holes in the ground truth
    return pred, gt


def median_inputs():
    g = torch.Generator().manual_seed(32)
    B, H, W = 5, 16, 24
    pred = torch.rand(B, 1, H, W, generator=g) * 0.3 + 0.01
    gt = torch.zeros(B, 1, H, W)
    for b, cnt in enumerate((37, 40, 0, 21, 50)):
        idx = torch.randperm(H * W, generator=g)
        gt.view(B, -1)[b, idx[:cnt]] = torch.rand(cnt, generator=g) * 0.2 + 0.005
        gt.view(B, -1)[b, idx[cnt:cnt + 5]] = -torch.rand(5, generator=g)      # not selected (target > 0 is False)
        if b == 0:
            gt.view(B, -1)[b, idx[cnt + 5]] = float("nan")                      # not selected either
        if b == 3:
            pred.view(B, -1)[b, idx[7]] = float("nan")
        if b == 4:
            sel = idx[:cnt]
            gt.view(B, -1)[b, sel] = (torch.randint(1, 6, (cnt,), generator=g) * 0.02).float()
            pred.view(B, -1)[b, sel] = (torch.randint(1, 6, (cnt,), generator=g) * 0.03).float()
    return pred, gt


def main():
    torch.manual_seed(0)
    import_reference()
    import model.metric_functions.completeness_metrics as CM  # noqa
    import model.metric_functions.dense_metrics as DM  # noqa
    import model.metric_functions.sparse_metrics as SM  # noqa
    from utils import median_scaling  # noqa
    pred, gt = dense_inputs()
    out = {"pred": pred.numpy(), "gt": gt.numpy()}
    for tag, kw in CASES.items():
        vals = []
        for n in DENSE_NAMES:
            if n in ("sc_inv", "l1_rel", "l1_inv", "completeness", "covered_gt"):
                mod = DM if n in ("sc_inv", "l1_rel", "l1_inv") else CM
                v = getattr(mod, f"{n}_metric")(pred.clone(), gt.clone(), **kw)
            else:
                v = getattr(SM, f"{n}_metric")({"result": pred.clone(), "target": gt.clone()}, **kw)
            vals.append(float(v))
        out[f"case_{tag}"] = np.array(vals, dtype=np.float64)
        print(tag, dict(zip(DENSE_NAMES, vals)))
    mp, mg = median_inputs()
    d = {"result": mp.clone(), "target": mg.clone()}
    r = median_scaling(d)
    assert torch.equal(d["result"].nan_to_num(-1), mp.nan_to_num(-1))      # the input is left as it was
    out.update(ms_pred=mp.numpy(), ms_gt=mg.numpy(), ms_result=r["result"].numpy())
    print("median scaling: NaN images", torch.isnan(r["result"]).flatten(1).all(1).tolist())
    path = HERE / "metrics_dense.npz"
    np.savez_compressed(path, **out)
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
