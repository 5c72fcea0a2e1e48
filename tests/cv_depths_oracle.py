"""Per-pixel depth hypotheses (data_dict["cv_depths"]) for the cost-volume oracles, and the seeded golden cases.

The reference takes its depths from data_dict["cv_depths"], a (B, D, H, W) tensor, when the caller supplies it
(model/monorec/monorec_model.py:181-185, :194-201); the uniform inverse-depth planes are that tensor built as a broadcast
linspace.  `cost_volume_torch` and `cost_volume_closed_form` below are the two restatements of
oracle/cost_volume_oracle.py with that one change: the depth that multiplies K^-1 (x, y, 1) comes from the pixel, and D is
the tensor's.  Everything else reuses the oracle's primitives.

`make_case(tag)` rebuilds the inputs of tests/golden/cv_pixel_depths.npz (written by make_golden_cv_depths.py from the
reference): seeded images from monorec_b200.synthetic and depths evaluated in float64 numpy and rounded once to fp32, so
they are the same bits on every machine.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import cost_volume_oracle as O

# tag -> (B, F, D, H, W, seed)
# (small on purpose: the golden file stores every reference volume in full fp32)
CASES = {
    "band": (1, 2, 16, 16, 40, 41),       # x0.5 - x2 band (geometric) around a smooth 4-60 m surface
    "shuffled": (1, 2, 16, 16, 40, 42),   # the default linspace planes, permuted independently per pixel
    "wide": (1, 2, 40, 12, 42, 43),       # 2 lanes per pixel with a partial chunk (D % 32 != 0), W % 4 != 0 (gather),
                                          # per-pixel spans of 1-400 m
}
MODEL_CASE = (1, 2, 32, 64, 128, 5)       # full MonoRecModel forward: B, F, D = cv_depth_steps, H, W, image seed


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
    z = O.plane_depths(0.33, 0.0025, D).numpy()
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


def make_case(tag):
    """(data dict on the CPU, cv_depths (B, D, H, W) fp32) of a golden case."""
    from monorec_b200.synthetic import make_inputs
    if tag == "model":
        B, nF, D, H, W, seed = MODEL_CASE
        return make_inputs(B, nF, H, W, seed=seed), band_depths(B, D, H, W, seed=44, rel=2.0)
    B, nF, D, H, W, seed = CASES[tag]
    data = make_inputs(B, nF, H, W, seed=seed)
    gen = {"band": band_depths, "shuffled": shuffled_depths, "wide": wide_depths}[tag]
    return data, gen(B, D, H, W, seed)


@torch.no_grad()
def cost_volume_torch(data, cv_depths, use_mono=True, use_stereo=False, patch_size=3, alpha=O.ALPHA,
                      channel_weights=O.CHANNEL_WEIGHTS):
    """oracle.cost_volume_oracle.cost_volume_torch with the depths of data_dict["cv_depths"] (monorec_model.py:181-201).

    Returns (cost_volume (B,D,H,W), [F x (B,D,H,W)] single-frame volumes, valid (B,F,H,W)).
    """
    key = data["keyframe"]
    dtype = key.dtype
    frames, intrinsics, poses = O.collect_frames(data, use_mono, use_stereo)
    B, C, H, W = key.shape
    nF = len(frames)
    D = cv_depths.shape[1]                                               # :196
    grid_px = O._pixel_grid(H, W, dtype)
    inside = O.interior_mask(H, W, patch_size // 2 + 1, dtype)
    sad_w = (torch.tensor(channel_weights, dtype=dtype) / patch_size ** 2).view(1, C, 1, 1, 1) \
        .repeat(1, 1, 1, patch_size, patch_size)
    out_cv, out_sf, out_valid = [], [[] for _ in range(nF)], []
    for b in range(B):
        kinv = torch.inverse(data["keyframe_intrinsics"][b])[:3, :3]
        rays = kinv @ grid_px
        pts = cv_depths[b].to(dtype).reshape(D, 1, H * W) * rays.unsqueeze(0)   # :200
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
        warped = torch.stack(warped, 1)
        valid = torch.stack(valid)
        n = D * nF
        err = O._ssim_error(warped.reshape(n, C, H, W) + 0.5, key[b:b + 1].expand(n, -1, -1, -1) + 0.5)
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
        cv[:, nz] = 1 - 2 * (num[:, nz] / den[nz])
        out_cv.append(cv)
        out_valid.append(valid[:, 0])
    return torch.stack(out_cv), [torch.stack(v) for v in out_sf], torch.stack(out_valid)


def cost_volume_closed_form(data, cv_depths, use_mono=True, use_stereo=False, alpha=O.ALPHA,
                            channel_weights=O.CHANNEL_WEIGHTS, dtype=np.float64):
    """oracle.cost_volume_oracle.cost_volume_closed_form (SURVEY.md Appendix C) with per-pixel depths z[b, d, y, x].

    Returns (cv, [sfcv_f], valid (B,F,H,W)); the positions are evaluated in float64, the rest in `dtype`.
    """
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
            c = A[None] * z_all[b][:, None] + P[:, 3][None, :, None, None]                # (D,3,H,W)
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
            X = np.moveaxis(X, 0, 1)
            mu_x = O._box3(X) / dtype(9)
            s_x = O._box3(X * X) / dtype(9) - mu_x * mu_x
            s_xy = O._box3(X * Y[None]) / dtype(9) - mu_x * mu_y[None]
            n_ = (2 * mu_x * mu_y[None] + dtype(O.SSIM_C1)) * (2 * s_xy + dtype(O.SSIM_C2))
            d_ = (mu_x * mu_x + (mu_y * mu_y)[None] + dtype(O.SSIM_C1)) * (s_x + s_y[None] + dtype(O.SSIM_C2))
            e = np.clip((1 - n_ / d_) / 2, 0, 1)
            sad = O._box3((e * cw).sum(axis=1)) / dtype(9)
            valids[b, f] = valid
            sfs[f, b] = (1 - 2 * sad) * valid
            spread = np.exp(-dtype(alpha) * (sad - sad.min(axis=0, keepdims=True)) ** 2).sum(axis=0)
            w = (1 - (spread - 1) / dtype(D - 1)) * valid
            num += w[None] * sad
            den += w
        nz = den != 0
        cv = np.zeros((D, H, W), dtype=dtype)
        cv[:, nz] = 1 - 2 * num[:, nz] / den[nz]
        cvs[b] = cv
    return cvs, [sfs[f] for f in range(nF)], valids
