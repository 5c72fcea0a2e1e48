#!/usr/bin/env python
"""Generates tests/golden/residual_image.npz by running the UNMODIFIED reference's ResidualImage / ResidualImageModule
(model/layers.py:147-217) on CPU fp32:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_residual_image.py

The reference is imported in place with make_golden.import_reference.  One more shim is needed: ResidualImageModule reads
`Backprojection(...).pix_coords`, an attribute the reference's Backprojection does not define (it names the same
[N,3,H*W] grid of (x, y, 1) pixel coordinates `coord`), so the unshimmed module raises AttributeError.  The shim adds
`pix_coords` as a read-only alias of `coord` on the class; no reference source is changed.  The per-frame masks are
recorded by observing the reference's F.grid_sample outputs (layers.py:203-204: any_c(warped == 0)).

Cases (tests/residual_cases.py builds the images and poses from their seeds):
  synth         B 2, F 2, 40x64, a seeded smooth inverse depth, ResidualImage
  out_of_image  near points and points behind the camera: samples partly and wholly outside the frames
  edges         0, -0, +-inf, NaN, tiny, huge and negative inverse depths
  stereo        ResidualImageModule(use_mono=True, use_stereo=True) with a right-camera frame
  ragged        37x61 (W % 4 != 0, H and W not multiples of the kernel's tile)
  gray          three-channel images whose planes are equal (a grayscale stream replicated)
  model         ResidualImageModule on the reference MonoRecModel's output dict (seeded weights): the prediction is mapped
                by inv_depth_min / inv_depth_max a second time
Per case: `<name>_invd` (the inverse depth given: `depths` of ResidualImage, predicted_inverse_depths[0] of the module),
`<name>_residual` [B,1,H,W] and `<name>_masks` [B,F,H,W] (uint8).
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent.parent))

import make_golden  # noqa: E402
from monorec_b200.synthetic import seeded_state_dict  # noqa: E402
from tests.residual_cases import CASES, MODEL_GAIN, MODEL_SEED, inputs, inverse_depth  # noqa: E402


class _Recorder:
    """Stands in for the reference module's `F` (torch.nn.functional) and keeps every grid_sample output."""

    def __init__(self, functional):
        self._f, self.outputs = functional, []

    def __getattr__(self, name):
        return getattr(self._f, name)

    def grid_sample(self, *a, **kw):
        out = self._f.grid_sample(*a, **kw)
        self.outputs.append(out.clone())
        return out


def main():
    torch.manual_seed(0)
    ref_mod = make_golden.import_reference()
    import model.layers as ref_layers
    ref_layers.Backprojection.pix_coords = property(lambda self: self.coord)
    rec = _Recorder(ref_layers.F)
    ref_layers.F = rec
    out = {}
    for name, (B, nF, H, W, seed, stereo, gray) in CASES.items():
        data = inputs(name)
        rec.outputs.clear()
        with torch.no_grad():
            if name == "model":
                model = ref_mod.MonoRecModel()
                model.load_state_dict(seeded_state_dict(model, seed=MODEL_SEED, gain=MODEL_GAIN))
                model.eval()
                d = model(dict(data))
                rec.outputs.clear()                # (the cost volume samples through its own module's F)
                invd = d["predicted_inverse_depths"][0].clone()
                res = ref_layers.ResidualImageModule()(d)["residual_image"]
            elif stereo:
                invd = inverse_depth(name)
                d = dict(data, predicted_inverse_depths=[invd], inv_depth_max=0, inv_depth_min=1)
                res = ref_layers.ResidualImageModule(use_mono=True, use_stereo=True)(d)["residual_image"]
            else:
                invd = inverse_depth(name)
                res = ref_layers.ResidualImage()(data["keyframe"], data["keyframe_pose"], data["keyframe_intrinsics"], invd,
                                                  data["frames"], data["poses"], data["intrinsics"])
        n_frames = nF + (1 if stereo else 0)
        assert len(rec.outputs) == n_frames, (name, len(rec.outputs))
        masks = torch.stack([(w == 0).any(1) for w in rec.outputs], 1)
        out[f"{name}_invd"] = invd.numpy().astype(np.float32)
        out[f"{name}_residual"] = res.numpy().astype(np.float32)
        out[f"{name}_masks"] = masks.numpy().astype(np.uint8)
        r = res.numpy()
        print(f"{name}: residual range [{np.nanmin(r):.4f}, {np.nanmax(r):.4f}], NaN {int(np.isnan(r).sum())}, "
              f"zero {int((r == 0).sum())}, masked (frame, pixel) {int(masks.sum())} of {masks.numel()}", flush=True)
    np.savez_compressed(HERE / "residual_image.npz", **out)


if __name__ == "__main__":
    main()
