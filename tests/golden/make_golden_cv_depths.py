#!/usr/bin/env python
"""Writes tests/golden/cv_pixel_depths.npz by running the UNMODIFIED reference on CPU fp32 with per-pixel depth hypotheses
(data_dict["cv_depths"], model/monorec/monorec_model.py:181-185):

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_cv_depths.py

The inputs are rebuilt by tests/cv_cases.make_pixel_case (seeded images, depths evaluated in float64 numpy and rounded
once to fp32), so only the reference's outputs are stored, in fp32:
  <tag>_cv, <tag>_sf      CostVolumeModule outputs for the cases band, shuffled and wide
  model_<gain>_cv_mask, model_<gain>_depth{1..4}
                          a full MonoRecModel forward (seeded weights of model_synth_small.npz, gain 1 and 0.7) with band
                          hypotheses and D = cv_depth_steps = 32
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)
from monorec_b200.synthetic import seeded_state_dict  # noqa: E402
from tests.cv_cases import PIXEL_CASES, make_pixel_case  # noqa: E402


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref_mod = import_reference()
    out = {}
    for tag in PIXEL_CASES:
        data, z = make_pixel_case(tag)
        d = dict(data)
        d["cv_depths"] = z
        with torch.no_grad():
            d = ref_mod.CostVolumeModule()(d)
        out[f"{tag}_cv"] = d["cost_volume"].numpy()
        out[f"{tag}_sf"] = np.stack([v.numpy() for v in d["single_frame_cvs"]])
        print(tag, "valid share per frame", [float(1 - (v == 0).all(1).float().mean()) for v in d["single_frame_cvs"]])
    for gain_tag, gain in (("g1", 1.0), ("g07", 0.7)):
        data, z = make_pixel_case("model")
        model = ref_mod.MonoRecModel()
        model.load_state_dict(seeded_state_dict(model, seed=7, gain=gain))
        model.eval()
        d = dict(data)
        d["cv_depths"] = z
        with torch.no_grad():
            r = model(d)
        out[f"model_{gain_tag}_cv_mask"] = r["cv_mask"].numpy()
        for i, p in enumerate(r["predicted_inverse_depths"][1:], start=1):
            out[f"model_{gain_tag}_depth{i}"] = p.numpy()
        print("model", gain_tag, "result range", float(r["result"].min()), float(r["result"].max()))
    path = HERE / "cv_pixel_depths.npz"
    np.savez_compressed(path, **out)
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
