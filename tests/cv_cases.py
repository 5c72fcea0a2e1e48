"""Seeded inputs of the cost-volume golden files, rebuilt bit for bit on every machine.

* `make_pixel_case(tag)`: tests/golden/cv_pixel_depths.npz (written by make_golden_cv_depths.py from the reference), the
  reference with per-pixel depths (data_dict["cv_depths"], model/monorec/monorec_model.py:181-201).  The depths are
  evaluated in float64 numpy and rounded once to fp32.
* `make_matching_case(tag)`: tests/golden/cv_matching.npz (written by make_golden_cv_matching.py), the reference's
  non-default error modes (use_ssim, :227-243) and uncentred fused volume (not_center_cv, :267-269), on the default
  planes or a band of per-pixel depths.

The images are seeded ones from monorec_b200.synthetic.  Both restatements in oracle/cost_volume_oracle.py take these
inputs; the default planes as a (B, D, H, W) tensor are `broadcast_planes`.
"""
import numpy as np
import torch

from oracle import cost_volume_oracle as O

INV_RANGE = (0.33, 0.0025)    # (inv_depth_min, inv_depth_max) of the reference's defaults, monorec_model.py:184

# tag -> (B, F, D, H, W, seed)
# (small on purpose: the golden file stores every reference volume in full fp32)
PIXEL_CASES = {
    "band": (1, 2, 16, 16, 40, 41),       # x0.5 - x2 band (geometric) around a smooth 4-60 m surface
    "shuffled": (1, 2, 16, 16, 40, 42),   # the default linspace planes, permuted independently per pixel
    "wide": (1, 2, 40, 12, 42, 43),       # 2 lanes per pixel with a partial chunk (D % 32 != 0), W % 4 != 0 (gather),
                                          # per-pixel spans of 1-400 m
}
PIXEL_MODEL_CASE = (1, 2, 32, 64, 128, 5)   # full MonoRecModel forward: B, F, D = cv_depth_steps, H, W, image seed

# tag -> (B, F, D, H, W, image seed, use_ssim, not_center_cv, depth source: "planes" or "band")
MATCHING_CASES = {
    "ssim_l1": (1, 2, 8, 16, 40, 61, 2, False, "planes"),
    "box_l1": (1, 2, 8, 16, 40, 62, 3, False, "planes"),
    "uncentred": (1, 2, 8, 16, 40, 63, True, True, "planes"),
    "ssim_l1_band": (1, 2, 16, 16, 40, 64, 2, False, "band"),
    "ragged": (1, 2, 12, 12, 42, 65, 3, True, "planes"),      # W % 4 != 0 (the kernel gathers), box + uncentred
}
MATCHING_MODEL_CASE = (1, 2, 64, 128, 5)   # full MonoRecModel(use_ssim=2) forward: B, F, H, W, image seed (default planes)


def smooth_surface(B, H, W, seed, lo=4.0, hi=60.0):
    """(B, H, W) float64 depths in [lo, hi]: a few seeded low-frequency waves."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.arange(H) / H, np.arange(W) / W, indexing="ij")
    s = np.zeros((B, H, W))
    for b in range(B):
        for _ in range(4):
            fy, fx, ph = rng.uniform(0, 2), rng.uniform(0, 3), rng.uniform(0, 2 * np.pi)
            s[b] += rng.uniform(0.5, 1.0) * np.sin(2 * np.pi * (fy * yy + fx * xx) + ph)
        s[b] = (s[b] - s[b].min()) / (s[b].max() - s[b].min())
    return lo * (hi / lo) ** s                   # log-uniform spread


def band_depths(B, D, H, W, seed, rel=2.0):
    """z = s(y, x) exp(linspace(-log rel, log rel, D)) around a smooth seeded surface, fp32."""
    f = np.exp(np.linspace(-np.log(rel), np.log(rel), D))
    return torch.from_numpy((smooth_surface(B, H, W, seed)[:, None] * f[None, :, None, None]).astype(np.float32))


def shuffled_depths(B, D, H, W, seed):
    """The default planes 1 / linspace(0.0025, 0.33, D), permuted independently per pixel."""
    z = O.plane_depths(*INV_RANGE, D).numpy()
    rng = np.random.default_rng(seed)
    out = np.broadcast_to(z[None, :, None, None], (B, D, H, W)).copy()
    return torch.from_numpy(rng.permuted(out, axis=1))


def wide_depths(B, D, H, W, seed):
    """Per-pixel geometric spans from 1 m up to a seeded far end of 20-400 m: the far ends of some pixels project out of
    the source images (their validity flips), the near ends of others come close to the camera."""
    rng = np.random.default_rng(seed)
    far = np.exp(rng.uniform(np.log(20.0), np.log(400.0), size=(B, 1, H, W)))
    t = np.linspace(0.0, 1.0, D)[None, :, None, None]
    return torch.from_numpy((far ** t).astype(np.float32))


def step_depths(B, D, H, W, z_near=2.0, z_far=30.0, rel=4.0):
    """A x1/rel - x rel band around z_near left of a vertical edge at 0.43 W (through the middle of a 60-column tile) and
    around z_far right of it, fp32.  (A far side at hundreds of metres has flat costs over the whole band: its view weights
    vanish and the fused value is a ratio of rounding noise in the reference formula itself; 30 m keeps the fused volume
    comparable.)"""
    s = torch.full((B, 1, H, W), z_far)
    s[..., : int(0.43 * W)] = z_near
    f = torch.exp(torch.linspace(-np.log(rel), np.log(rel), D, dtype=torch.float64)).float()
    return (s * f.view(1, D, 1, 1)).contiguous()


def broadcast_planes(B, D, H, W):
    """The reference's default planes 1 / linspace(0.0025, 0.33, D) as a (B, D, H, W) broadcast."""
    return O.plane_depths(*INV_RANGE, D).view(1, D, 1, 1).expand(B, D, H, W)


def with_plane_range(data, D):
    """A copy of the dict with the reference's plane-range keys (monorec_model.py:184)."""
    d = dict(data)
    key = d["keyframe"]
    d["inv_depth_min"] = key.new_tensor([INV_RANGE[0]])
    d["inv_depth_max"] = key.new_tensor([INV_RANGE[1]])
    d["cv_depth_steps"] = key.new_tensor([D], dtype=torch.int32)
    return d


def make_pixel_case(tag):
    """(data dict on the CPU, cv_depths (B, D, H, W) fp32) of a case of PIXEL_CASES, or of "model"."""
    from monorec_b200.synthetic import make_inputs
    if tag == "model":
        B, nF, D, H, W, seed = PIXEL_MODEL_CASE
        return make_inputs(B, nF, H, W, seed=seed), band_depths(B, D, H, W, seed=44, rel=2.0)
    B, nF, D, H, W, seed = PIXEL_CASES[tag]
    data = make_inputs(B, nF, H, W, seed=seed)
    gen = {"band": band_depths, "shuffled": shuffled_depths, "wide": wide_depths}[tag]
    return data, gen(B, D, H, W, seed)


def make_matching_case(tag):
    """(data dict on the CPU, cv_depths (B, D, H, W) fp32 or None for the default planes, D, use_ssim, not_center_cv)."""
    from monorec_b200.synthetic import make_inputs
    B, nF, D, H, W, seed, use_ssim, not_center, src = MATCHING_CASES[tag]
    data = make_inputs(B, nF, H, W, seed=seed)
    z = band_depths(B, D, H, W, seed=seed, rel=2.0) if src == "band" else None
    return data, z, D, use_ssim, not_center
