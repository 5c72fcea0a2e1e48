#!/usr/bin/env python
"""Writes tests/golden/cv_matching.npz by running the UNMODIFIED reference on CPU fp32 with its non-default cost-volume
options: use_ssim (model/monorec/monorec_model.py:227-243) and not_center_cv (:267-269).

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_cv_matching.py

The inputs are rebuilt by tests/cv_cases.make_matching_case (seeded images, the default planes or a band of per-pixel
depths), so only the reference's outputs are stored, in fp32:
  <tag>_cv, <tag>_sf      CostVolumeModule(use_ssim=..., not_center_cv=...) outputs for the cases of
                          cv_cases.MATCHING_CASES
  model_<gain>_cv_mask, model_<gain>_depth{1..3}
                          a full MonoRecModel(use_ssim=2) forward (seeded weights of model_synth_small.npz, gain 1 and 0.7)
                          on the default planes
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)
from monorec_b200.synthetic import make_inputs, seeded_state_dict  # noqa: E402
from tests.cv_cases import MATCHING_CASES, MATCHING_MODEL_CASE, make_matching_case, with_plane_range  # noqa: E402


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref_mod = import_reference()
    out = {}
    for tag in MATCHING_CASES:
        data, z, D, use_ssim, not_center = make_matching_case(tag)
        d = with_plane_range(data, D)
        if z is not None:
            d["cv_depths"] = z
        with torch.no_grad():
            d = ref_mod.CostVolumeModule(use_ssim=use_ssim, not_center_cv=not_center)(d)
        out[f"{tag}_cv"] = d["cost_volume"].numpy()
        out[f"{tag}_sf"] = np.stack([v.numpy() for v in d["single_frame_cvs"]])
        print(tag, "valid share per frame", [float(1 - (v == 0).all(1).float().mean()) for v in d["single_frame_cvs"]])
    B, nF, H, W, seed = MATCHING_MODEL_CASE
    for gain_tag, gain in (("g1", 1.0), ("g07", 0.7)):
        model = ref_mod.MonoRecModel(use_ssim=2)
        model.load_state_dict(seeded_state_dict(model, seed=7, gain=gain))
        model.eval()
        d = with_plane_range(make_inputs(B, nF, H, W, seed=seed), model.cv_depth_steps)
        with torch.no_grad():
            r = model(d)
        out[f"model_{gain_tag}_cv_mask"] = r["cv_mask"].numpy()
        for i, p in enumerate(r["predicted_inverse_depths"][1:], start=1):
            out[f"model_{gain_tag}_depth{i}"] = p.numpy()
        print("model", gain_tag, "result range", float(r["result"].min()), float(r["result"].max()))
    path = HERE / "cv_matching.npz"
    np.savez_compressed(path, **out)
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
