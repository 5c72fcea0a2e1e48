"""The cost volume's non-default error modes (use_ssim, monorec_model.py:227-243) and the uncentred fused volume
(not_center_cv, :267-269) for the oracles, and the seeded golden cases of tests/golden/cv_matching.npz.

`cost_volume_torch` restates CostVolumeModule.forward in the reference's operation order with both options;
`cost_volume_closed_form` is the float64 closed form (SURVEY.md Appendix C) with the same options.  Both take the depths as
a (B, D, H, W) tensor, as tests/cv_depths_oracle.py does: the default planes are that tensor built as a broadcast.  Only the
difference and the epilogue differ from tests/cv_depths_oracle.py; every other step reuses oracle/cost_volume_oracle.py.

`make_case(tag)` rebuilds the inputs of the golden file (written by tests/golden/make_golden_cv_matching.py from the
reference): seeded images from monorec_b200.synthetic, and either the default planes or a band of per-pixel depths.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import cost_volume_oracle as O
from tests import cv_depths_oracle as PO

INV_RANGE = (0.33, 0.0025)    # (inv_depth_min, inv_depth_max) of the reference's defaults, monorec_model.py:184

# tag -> (B, F, D, H, W, image seed, use_ssim, not_center_cv, depth source: "planes" or "band")
# (small on purpose: the golden file stores every reference volume in full fp32)
CASES = {
    "ssim_l1": (1, 2, 8, 16, 40, 61, 2, False, "planes"),
    "box_l1": (1, 2, 8, 16, 40, 62, 3, False, "planes"),
    "uncentred": (1, 2, 8, 16, 40, 63, True, True, "planes"),
    "ssim_l1_band": (1, 2, 16, 16, 40, 64, 2, False, "band"),
    "ragged": (1, 2, 12, 12, 42, 65, 3, True, "planes"),      # W % 4 != 0 (the kernel gathers), box + uncentred
}
MODEL_CASE = (1, 2, 64, 128, 5)    # full MonoRecModel(use_ssim=2) forward: B, F, H, W, image seed (default planes)


def plane_depths(B, D, H, W):
    """The reference's default planes 1 / linspace(0.0025, 0.33, D) as a (B, D, H, W) broadcast."""
    return O.plane_depths(INV_RANGE[0], INV_RANGE[1], D).view(1, D, 1, 1).expand(B, D, H, W)


def with_plane_range(data, D):
    """A copy of the dict with the reference's plane-range keys (monorec_model.py:184)."""
    d = dict(data)
    key = d["keyframe"]
    d["inv_depth_min"] = key.new_tensor([INV_RANGE[0]])
    d["inv_depth_max"] = key.new_tensor([INV_RANGE[1]])
    d["cv_depth_steps"] = key.new_tensor([D], dtype=torch.int32)
    return d


def make_case(tag):
    """(data dict on the CPU, cv_depths (B, D, H, W) fp32 or None for the default planes, D, use_ssim, not_center_cv)."""
    from monorec_b200.synthetic import make_inputs
    B, nF, D, H, W, seed, use_ssim, not_center, src = CASES[tag]
    data = make_inputs(B, nF, H, W, seed=seed)
    z = PO.band_depths(B, D, H, W, seed=seed, rel=2.0) if src == "band" else None
    return data, z, D, use_ssim, not_center


def _difference(use_ssim, warped, key, n, C, H, W):
    """The per-pixel, per-channel difference of monorec_model.py:227-243, in its order of comparisons and operations."""
    if not use_ssim:
        raise NotImplementedError("use_ssim falsy")
    if use_ssim == True:  # noqa: E712  (the reference's comparison)
        return O._ssim_error(warped.reshape(n, C, H, W) + .5, key.expand(n, -1, -1, -1) + .5)
    if use_ssim == 2:
        d = O._ssim_error(warped.reshape(n, C, H, W) + .5, key.expand(n, -1, -1, -1) + .5)
        d = d.view(warped.shape)
        return (0.85 * d + 0.15 * torch.abs(warped - key)).reshape(n, C, H, W)
    return F.avg_pool2d(torch.abs(warped - key).reshape(n, C, H, W), kernel_size=3, stride=1, padding=1)


@torch.no_grad()
def cost_volume_torch(data, cv_depths, use_ssim=True, not_center_cv=False, use_mono=True, use_stereo=False, patch_size=3,
                      alpha=O.ALPHA, channel_weights=O.CHANNEL_WEIGHTS):
    """tests.cv_depths_oracle.cost_volume_torch with the reference's use_ssim and not_center_cv.

    Returns (cost_volume (B,D,H,W), [F x (B,D,H,W)] single-frame volumes, valid (B,F,H,W)).
    """
    key = data["keyframe"]
    dtype = key.dtype
    frames, intrinsics, poses = O.collect_frames(data, use_mono, use_stereo)
    B, C, H, W = key.shape
    nF = len(frames)
    D = cv_depths.shape[1]
    grid_px = O._pixel_grid(H, W, dtype)
    inside = O.interior_mask(H, W, patch_size // 2 + 1, dtype)
    sad_w = (torch.tensor(channel_weights, dtype=dtype) / patch_size ** 2).view(1, C, 1, 1, 1) \
        .repeat(1, 1, 1, patch_size, patch_size)
    out_cv, out_sf, out_valid = [], [[] for _ in range(nF)], []
    for b in range(B):
        kinv = torch.inverse(data["keyframe_intrinsics"][b])[:3, :3]
        rays = kinv @ grid_px
        pts = cv_depths[b].to(dtype).reshape(D, 1, H * W) * rays.unsqueeze(0)
        pts = torch.cat([pts, torch.ones(D, 1, H * W, dtype=dtype)], 1)
        warped, valid = [], []
        for f in range(nF):
            T = torch.inverse(poses[f][b]) @ data["keyframe_pose"][b]
            P = (intrinsics[f][b] @ T)[:3, :]
            cam = P.unsqueeze(0) @ pts
            uv = cam[:, :2] / (cam[:, 2:3] + 1e-7)
            uv = torch.stack([uv[:, 0] / (W - 1), uv[:, 1] / (H - 1)], 1)
            g = ((uv - 0.5) * 2).view(D, 2, H, W).permute(0, 2, 3, 1).clamp(-2, 2)
            img = frames[f][b:b + 1].expand(D, -1, -1, -1)
            warped.append(F.grid_sample(img, g, mode="bilinear", padding_mode="zeros", align_corners=False))
            hit = F.grid_sample(inside.expand(D, -1, -1, -1), g, mode="bilinear", padding_mode="zeros",
                                align_corners=False)
            valid.append(inside[0] * torch.min(hit != 0, dim=0)[0])
        warped = torch.stack(warped, 1)                                   # (D, F, C, H, W)
        valid = torch.stack(valid)
        n = D * nF
        err = _difference(use_ssim, warped, key[b], n, C, H, W)
        err = err.view(D, nF, C, H, W).permute(1, 2, 0, 3, 4)
        sad = F.conv3d(err, sad_w, padding=(0, patch_size // 2, patch_size // 2)).squeeze(1)
        sfcv = (1 - sad * 2) * valid
        for f in range(nF):
            out_sf[f].append(sfcv[f])
        spread = torch.exp(-alpha * (sad - sad.min(dim=1, keepdim=True)[0]) ** 2)
        wgt = (1 - (spread.sum(dim=1, keepdim=True) - 1) / (D - 1)) * valid
        num = (sad * wgt).sum(0)
        den = wgt.sum(0).squeeze(0)
        nz = den != 0
        cv = torch.zeros_like(num)
        cv[:, nz] = num[:, nz] / den[nz]                                  # :262-264
        if not not_center_cv:
            cv[:, nz] = 1 - 2 * cv[:, nz]                                 # :266-267
        out_cv.append(cv)
        out_valid.append(valid[:, 0])
    return torch.stack(out_cv), [torch.stack(v) for v in out_sf], torch.stack(out_valid)


def cost_volume_closed_form(data, cv_depths, use_ssim=True, not_center_cv=False, use_mono=True, use_stereo=False,
                            alpha=O.ALPHA, channel_weights=O.CHANNEL_WEIGHTS, dtype=np.float64):
    """tests.cv_depths_oracle.cost_volume_closed_form with use_ssim and not_center_cv.  The box of the L1 mode is a
    zero-padded 3x3 sum / 9 (avg_pool2d with its default count_include_pad); no valid pixel reads the padding.

    Returns (cv, [sfcv_f], valid (B,F,H,W)); the positions are evaluated in float64, the rest in `dtype`.
    """
    if not use_ssim:
        raise NotImplementedError("use_ssim falsy")
    frames, _, _ = O.collect_frames(data, use_mono, use_stereo)
    key = data["keyframe"].numpy().astype(dtype)
    B, C, H, W = key.shape
    nF, D = len(frames), int(cv_depths.shape[1])
    z_all = cv_depths.numpy().astype(np.float64)
    proj, kinv = O.projection_tables(data, use_mono, use_stereo, dtype=np.float64)
    vv, uu = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    inside = np.zeros((H, W), dtype=bool)
    inside[2:H - 2, 2:W - 2] = True
    cw = np.asarray(channel_weights, dtype=dtype).reshape(1, 3, 1, 1)
    cvs = np.zeros((B, D, H, W), dtype=dtype)
    sfs = np.zeros((nF, B, D, H, W), dtype=dtype)
    valids = np.zeros((B, nF, H, W), dtype=bool)
    for b in range(B):
        ray = np.einsum("ij,jhw->ihw", kinv[b], np.stack([uu, vv, np.ones_like(uu)]))
        Y = key[b] + dtype(0.5)
        mu_y = O._box3(Y) / dtype(9)
        s_y = O._box3(Y * Y) / dtype(9) - mu_y * mu_y
        num = np.zeros((D, H, W), dtype=dtype)
        den = np.zeros((H, W), dtype=dtype)
        for f in range(nF):
            img = frames[f][b].numpy().astype(dtype)
            P = proj[b, f]
            A = np.einsum("ij,jhw->ihw", P[:, :3], ray)
            c = A[None] * z_all[b][:, None] + P[:, 3][None, :, None, None]
            with np.errstate(divide="ignore", invalid="ignore"):
                px = c[:, 0] / (c[:, 2] + 1e-7)
                py = c[:, 1] / (c[:, 2] + 1e-7)
            gx = np.clip((px / (W - 1) - 0.5) * 2, -2, 2)
            gy = np.clip((py / (H - 1) - 0.5) * 2, -2, 2)
            sx = ((gx + 1) * W - 1) / 2
            sy = ((gy + 1) * H - 1) / 2
            X = O._bilinear_zero(img, sx, sy) + dtype(0.5)
            hit = O._bilinear_zero(inside[None].astype(dtype), sx, sy)[0] != 0
            valid = inside & hit.all(axis=0)
            X = np.moveaxis(X, 0, 1)                                      # (D, C, H, W)
            l1 = np.abs(X - Y[None])
            if use_ssim == 2 or use_ssim == True:  # noqa: E712
                mu_x = O._box3(X) / dtype(9)
                s_x = O._box3(X * X) / dtype(9) - mu_x * mu_x
                s_xy = O._box3(X * Y[None]) / dtype(9) - mu_x * mu_y[None]
                n_ = (2 * mu_x * mu_y[None] + dtype(O.SSIM_C1)) * (2 * s_xy + dtype(O.SSIM_C2))
                d_ = (mu_x * mu_x + (mu_y * mu_y)[None] + dtype(O.SSIM_C1)) * (s_x + s_y[None] + dtype(O.SSIM_C2))
                e = np.clip((1 - n_ / d_) / 2, 0, 1)
                if use_ssim != True:  # noqa: E712
                    e = dtype(0.85) * e + dtype(0.15) * l1
            else:
                e = O._box3(l1) / dtype(9)
            sad = O._box3((e * cw).sum(axis=1)) / dtype(9)
            valids[b, f] = valid
            sfs[f, b] = (1 - 2 * sad) * valid
            spread = np.exp(-dtype(alpha) * (sad - sad.min(axis=0, keepdims=True)) ** 2).sum(axis=0)
            w = (1 - (spread - 1) / dtype(D - 1)) * valid
            num += w[None] * sad
            den += w
        nz = den != 0
        cv = np.zeros((D, H, W), dtype=dtype)
        cv[:, nz] = num[:, nz] / den[nz] if not_center_cv else 1 - 2 * num[:, nz] / den[nz]
        cvs[b] = cv
    return cvs, [sfs[f] for f in range(nF)], valids
