"""ORACLE (test infrastructure, not product code) -- CPU restatement of MonoRec's plane-sweep cost volume.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this file, and only as the checker / the CPU baseline.  The product path (monorec_b200/) never
imports anything from `oracle/`.

Reference being restated: the reference's model/monorec/monorec_model.py:150-284 (CostVolumeModule.forward,
create_mask) with model/layers.py:43-71 (Backprojection, point_projection) and :91-139 (SSIM).

Parity pin: the reference has no tests or golden vectors of its own ("parity unpinned" by the reference,
SURVEY.md §4/§8c).  This oracle is pinned instead against outputs of the *reference itself* run on the CPU
(tests/golden/make_golden*.py import it unmodified from a checkout of the reference and write
tests/golden/*.npz); tests/test_oracle_golden.py, tests/test_cv_pixel_depths.py and tests/test_cv_matching.py check
both restatements below against those files.

Two independent restatements, each with every option the kernel implements:

* `cost_volume_torch`  -- same library primitives as the reference (F.grid_sample, avg_pool2d, conv3d), so it
  has the reference's CPU performance characteristics; this is what `bench.py` times as the CPU baseline
  ("port").
* `cost_volume_closed_form` -- numpy, explicit bilinear gather and box sums following SURVEY.md Appendix C;
  shares no primitive with the first one and can run in float64 (used for tie margins).

The options, with the reference's defaults:
* the depths: uniform in inverse depth from (inv_depth_min, inv_depth_max, steps), or per pixel from
  `cv_depths` (B, D, H, W), the reference's data_dict["cv_depths"] (monorec_model.py:181-201);
* the difference, `use_ssim` (:227-243): True (SSIM), 2 (0.85 SSIM + 0.15 L1), any other truthy value (3x3 box of the
  L1 difference).  The plain L1 difference of a falsy value is not implemented by the kernel and raises here too;
* `not_center_cv` (:266-267): the fused volume as sum_f w_f sad_f / sum_f w_f instead of 1 - 2 x that.
"""
import numpy as np
import torch
import torch.nn.functional as F

CHANNEL_WEIGHTS = (5.0 / 32.0, 16.0 / 32.0, 11.0 / 32.0)  # monorec_model.py:133
ALPHA = 10.0                                                # monorec_model.py:133
SSIM_C1 = 0.01 ** 2                                         # layers.py:116
SSIM_C2 = 0.03 ** 2                                         # layers.py:117


def plane_depths(inv_depth_min, inv_depth_max, steps, dtype=torch.float32):
    """z_d = 1 / linspace(inv_depth_max_value, inv_depth_min_value, D)  (monorec_model.py:184-185).

    Note the reference's names are swapped w.r.t. their values: data_dict["inv_depth_max"] holds the
    *smaller* number (0.0025), so index 0 is the farthest plane (400 m).
    """
    return 1.0 / torch.linspace(float(inv_depth_max), float(inv_depth_min), int(steps), dtype=dtype)


def collect_frames(data, use_mono=True, use_stereo=False):
    """monorec_model.py:156-167."""
    frames, intrinsics, poses = [], [], []
    if use_mono:
        frames += list(data["frames"])
        intrinsics += list(data["intrinsics"])
        poses += list(data["poses"])
    if use_stereo:
        frames.append(data["stereoframe"])
        intrinsics.append(data["stereoframe_intrinsics"])
        poses.append(data["stereoframe_pose"])
    return frames, intrinsics, poses


def interior_mask(height, width, border, dtype=torch.float32):
    """1 inside, 0 in a `border`-pixel ring (monorec_model.py:282-284)."""
    m = torch.zeros(1, 1, height, width, dtype=dtype)
    m[:, :, border:height - border, border:width - border] = 1
    return m


def _pixel_grid(height, width, dtype):
    # layers.py:49-54: rows of [x; y; 1], row-major over (y, x)
    ys, xs = torch.meshgrid(torch.arange(height, dtype=dtype), torch.arange(width, dtype=dtype), indexing="ij")
    return torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(height * width, dtype=dtype)], 0)


def _ssim_error(x, y):
    """layers.py:119-137 with the default ctor (reflection pad 1, 3x3 average pools)."""
    x = F.pad(x, (1, 1, 1, 1), mode="reflect")
    y = F.pad(y, (1, 1, 1, 1), mode="reflect")
    mu_x = F.avg_pool2d(x, 3, 1)
    mu_y = F.avg_pool2d(y, 3, 1)
    mu_xx, mu_yy, mu_xy = mu_x ** 2, mu_y ** 2, mu_x * mu_y
    sig_x = F.avg_pool2d(x ** 2, 3, 1) - mu_xx
    sig_y = F.avg_pool2d(y ** 2, 3, 1) - mu_yy
    sig_xy = F.avg_pool2d(x * y, 3, 1) - mu_xy
    num = (2 * mu_xy + SSIM_C1) * (2 * sig_xy + SSIM_C2)
    den = (mu_xx + mu_yy + SSIM_C1) * (sig_x + sig_y + SSIM_C2)
    return torch.clamp((1 - num / den) / 2, 0, 1)


def _difference(use_ssim, warped, key, n, C, H, W):
    """The per-pixel, per-channel difference of monorec_model.py:227-243, in its order of comparisons and operations.
    warped (D, F, C, H, W), key (C, H, W); returns (D*F, C, H, W)."""
    if use_ssim == True:  # noqa: E712  (the reference's comparison)
        return _ssim_error(warped.reshape(n, C, H, W) + .5, key.expand(n, -1, -1, -1) + .5)
    if use_ssim == 2:
        d = _ssim_error(warped.reshape(n, C, H, W) + .5, key.expand(n, -1, -1, -1) + .5)
        d = d.view(warped.shape)
        return (0.85 * d + 0.15 * torch.abs(warped - key)).reshape(n, C, H, W)
    return F.avg_pool2d(torch.abs(warped - key).reshape(n, C, H, W), kernel_size=3, stride=1, padding=1)


@torch.no_grad()
def cost_volume_torch(data, inv_depth_min=0.33, inv_depth_max=0.0025, steps=32, use_mono=True, use_stereo=False,
                      patch_size=3, alpha=ALPHA, channel_weights=CHANNEL_WEIGHTS, return_valid=False,
                      cv_depths=None, use_ssim=True, not_center_cv=False):
    """Restates CostVolumeModule.forward (sfcv_mult_mask=True).  With `cv_depths` (B, D, H, W) the depths come from it
    and D is its D; otherwise from the planes of (inv_depth_min, inv_depth_max, steps).

    Returns (cost_volume (B,D,H,W), [F x (B,D,H,W)] single-frame volumes[, valid (B,F,H,W)]).
    """
    if not use_ssim:
        raise NotImplementedError("use_ssim falsy")
    key = data["keyframe"]
    dtype = key.dtype
    frames, intrinsics, poses = collect_frames(data, use_mono, use_stereo)
    B, C, H, W = key.shape
    nF = len(frames)
    if cv_depths is None:
        D = int(steps)
        z = plane_depths(inv_depth_min, inv_depth_max, D, dtype)        # (D,)
    else:
        D = cv_depths.shape[1]                                          # monorec_model.py:196
    border = patch_size // 2 + 1                                        # monorec_model.py:139
    grid_px = _pixel_grid(H, W, dtype)                                  # (3, HW)
    inside = interior_mask(H, W, border, dtype)
    sad_w = (torch.tensor(channel_weights, dtype=dtype) / patch_size ** 2).view(1, C, 1, 1, 1) \
        .repeat(1, 1, 1, patch_size, patch_size)                        # monorec_model.py:141-142

    out_cv, out_sf, out_valid = [], [[] for _ in range(nF)], []
    for b in range(B):                                                  # monorec_model.py:193
        kinv = torch.inverse(data["keyframe_intrinsics"][b])[:3, :3]
        rays = kinv @ grid_px                                           # (3, HW)
        depth = z.view(D, 1, 1) if cv_depths is None else cv_depths[b].to(dtype).reshape(D, 1, H * W)
        pts = depth * rays.unsqueeze(0)                                 # (D, 3, HW)   :199-200
        pts = torch.cat([pts, torch.ones(D, 1, H * W, dtype=dtype)], 1)  # homogeneous :201
        warped, valid = [], []
        for f in range(nF):
            T = torch.inverse(poses[f][b]) @ data["keyframe_pose"][b]   # :171,207
            P = (intrinsics[f][b] @ T)[:3, :]                           # layers.py:65
            cam = P.unsqueeze(0) @ pts                                  # (D, 3, HW)
            uv = cam[:, :2] / (cam[:, 2:3] + 1e-7)                      # layers.py:66
            uv = torch.stack([uv[:, 0] / (W - 1), uv[:, 1] / (H - 1)], 1)
            g = ((uv - 0.5) * 2).view(D, 2, H, W).permute(0, 2, 3, 1).clamp(-2, 2)   # :67-70, monorec :208
            img = frames[f][b:b + 1].expand(D, -1, -1, -1)
            warped.append(F.grid_sample(img, g, mode="bilinear", padding_mode="zeros", align_corners=False))
            hit = F.grid_sample(inside.expand(D, -1, -1, -1), g, mode="bilinear", padding_mode="zeros",
                                align_corners=False)
            valid.append(inside[0] * torch.min(hit != 0, dim=0)[0])     # :218-219  (1,H,W)
        warped = torch.stack(warped, 1)                                 # (D, F, C, H, W)
        valid = torch.stack(valid)                                      # (F, 1, H, W)
        n = D * nF
        err = _difference(use_ssim, warped, key[b], n, C, H, W)        # :227-243
        err = err.view(D, nF, C, H, W).permute(1, 2, 0, 3, 4)           # (F, C, D, H, W)
        sad = F.conv3d(err, sad_w, padding=(0, patch_size // 2, patch_size // 2)).squeeze(1)  # (F, D, H, W)
        sfcv = (1 - sad * 2) * valid                                    # :251
        for f in range(nF):
            out_sf[f].append(sfcv[f])
        spread = torch.exp(-alpha * (sad - sad.min(dim=1, keepdim=True)[0]) ** 2)   # :257
        wgt = 1 - (spread.sum(dim=1, keepdim=True) - 1) / (D - 1)       # :258
        wgt = wgt * valid                                               # :260
        num = (sad * wgt).sum(0)                                        # (D, H, W)
        den = wgt.sum(0).squeeze(0)                                     # (H, W)
        nz = den != 0
        cv = torch.zeros_like(num)
        fused = num[:, nz] / den[nz]                                    # :262-264
        cv[:, nz] = fused if not_center_cv else 1 - 2 * fused           # :266-267
        out_cv.append(cv)
        out_valid.append(valid[:, 0])
    cost_volume = torch.stack(out_cv)
    single = [torch.stack(v) for v in out_sf]
    if return_valid:
        return cost_volume, single, torch.stack(out_valid)
    return cost_volume, single


# ----------------------------------------------------------------------------------------------
# closed form (SURVEY.md Appendix C) -- numpy, explicit gather; dtype selectable
# ----------------------------------------------------------------------------------------------

def _box3(q):
    """3x3 box *sum* with zero padding over the last two axes."""
    p = np.pad(q, [(0, 0)] * (q.ndim - 2) + [(1, 1), (1, 1)])
    h = p[..., :, :-2] + p[..., :, 1:-1] + p[..., :, 2:]
    return h[..., :-2, :] + h[..., 1:-1, :] + h[..., 2:, :]


def _bilinear_zero(img, sx, sy):
    """img (C,H,W); sx, sy (...) source pixel coordinates; taps outside the image contribute 0."""
    C, H, W = img.shape
    x0 = np.floor(sx)
    y0 = np.floor(sy)
    fx = (sx - x0).astype(img.dtype)
    fy = (sy - y0).astype(img.dtype)
    x0 = x0.astype(np.int64)
    y0 = y0.astype(np.int64)
    out = np.zeros((C,) + sx.shape, dtype=img.dtype)
    for dy, wy in ((0, 1 - fy), (1, fy)):
        for dx, wx in ((0, 1 - fx), (1, fx)):
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
            v = img[:, np.clip(yi, 0, H - 1), np.clip(xi, 0, W - 1)]
            out += v * (wx * wy * ok)[None]
    return out


def _difference_closed_form(use_ssim, X, Y, mu_y, s_y, dtype):
    """monorec_model.py:227-243 on X (D,C,H,W) and Y (C,H,W), with the key's box mean and variance.  The box of the L1
    mode is a zero-padded 3x3 sum / 9 (avg_pool2d with its default count_include_pad); no valid pixel reads the padding."""
    if use_ssim == True or use_ssim == 2:  # noqa: E712
        mu_x = _box3(X) / dtype(9)
        s_x = _box3(X * X) / dtype(9) - mu_x * mu_x
        s_xy = _box3(X * Y[None]) / dtype(9) - mu_x * mu_y[None]
        n_ = (2 * mu_x * mu_y[None] + dtype(SSIM_C1)) * (2 * s_xy + dtype(SSIM_C2))
        d_ = (mu_x * mu_x + (mu_y * mu_y)[None] + dtype(SSIM_C1)) * (s_x + s_y[None] + dtype(SSIM_C2))
        e = np.clip((1 - n_ / d_) / 2, 0, 1)
        return e if use_ssim == True else dtype(0.85) * e + dtype(0.15) * np.abs(X - Y[None])  # noqa: E712
    return _box3(np.abs(X - Y[None])) / dtype(9)


def projection_tables(data, use_mono=True, use_stereo=False, dtype=np.float64):
    """proj[b,f] = (K_f . inv(pose_f) . pose_kf)[0:3, 0:4], kinv[b] = inv(K_kf)[0:3, 0:3]  (Appendix C)."""
    frames, intrinsics, poses = collect_frames(data, use_mono, use_stereo)
    B = data["keyframe"].shape[0]
    proj = np.zeros((B, len(frames), 3, 4), dtype=dtype)
    kinv = np.zeros((B, 3, 3), dtype=dtype)
    for b in range(B):
        kinv[b] = np.linalg.inv(data["keyframe_intrinsics"][b].numpy().astype(dtype))[:3, :3]
        for f in range(len(frames)):
            T = np.linalg.inv(poses[f][b].numpy().astype(dtype)) @ data["keyframe_pose"][b].numpy().astype(dtype)
            proj[b, f] = (intrinsics[f][b].numpy().astype(dtype) @ T)[:3, :]
    return proj, kinv


def _closed_form_depths(data, inv_depth_min, inv_depth_max, steps, cv_depths, dtype):
    """(B, D, 1, H or 1, W or 1) float64 depths of the closed form: `cv_depths`, or the planes of `dtype`."""
    B = data["keyframe"].shape[0]
    if cv_depths is not None:
        return cv_depths.numpy().astype(np.float64)[:, :, None]
    D = int(steps)
    if dtype == np.float32:
        z = plane_depths(inv_depth_min, inv_depth_max, D).numpy().astype(np.float64)
    else:
        z = 1.0 / np.linspace(float(inv_depth_max), float(inv_depth_min), D, dtype=np.float64)
    return np.broadcast_to(z.reshape(1, D, 1, 1, 1), (B, D, 1, 1, 1))


def _source_positions(P, ray, z, H, W, dtype):
    """Source pixel coordinates (sx, sy), each (D, H, W), of the rays `ray` (3, H, W) at depths `z` (D, 1, H|1, W|1) under
    the projection P (3, 4): layers.py:65-70 and grid_sample's un-normalisation, in float64 (rounded to fp32 where dtype is
    float32)."""
    A = np.einsum("ij,jhw->ihw", P[:, :3], ray)                                           # (3,H,W)
    c = A[None] * z + P[:, 3][None, :, None, None]                                         # (D,3,H,W)
    c = c.astype(dtype).astype(np.float64) if dtype == np.float32 else c
    with np.errstate(divide="ignore", invalid="ignore"):
        px = c[:, 0] / (c[:, 2] + 1e-7)
        py = c[:, 1] / (c[:, 2] + 1e-7)
    gx = np.clip((px / (W - 1) - 0.5) * 2, -2, 2)
    gy = np.clip((py / (H - 1) - 0.5) * 2, -2, 2)
    sx = ((gx + 1) * W - 1) / 2
    sy = ((gy + 1) * H - 1) / 2
    if dtype == np.float32:
        sx, sy = sx.astype(np.float32), sy.astype(np.float32)
    return sx, sy


def _key_rays(kinv, H, W):
    vv, uu = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    return np.einsum("ij,jhw->ihw", kinv, np.stack([uu, vv, np.ones_like(uu)]))           # (3,H,W)


def _interior(H, W):
    inside = np.zeros((H, W), dtype=bool)
    inside[2:H - 2, 2:W - 2] = True                                                        # monorec_model.py:282-284
    return inside


def validity_margin(data, inv_depth_min=0.33, inv_depth_max=0.0025, steps=32, use_mono=True, use_stereo=False,
                    cv_depths=None, dtype=np.float64):
    """Signed distance (B, F, H, W) float64, in source pixels, from each pixel's nearest sample to the edge of the
    validity region, at the positions `cost_volume_closed_form` uses with the same arguments.

    The interior mask covers rows and columns 2 .. n-3, so its bilinear sample (zero padding) is non-zero exactly when
    1 < sx < W-2 and 1 < sy < H-2.  A pixel is valid for a frame when that holds for all of its depths, so the margin is the
    minimum over the depths of min(sx - 1, W - 2 - sx, sy - 1, H - 2 - sy): `margin > 0` is the closed form's `valid`.
    It is -inf in the 2-px ring and where a sample is not finite.
    """
    frames, _, _ = collect_frames(data, use_mono, use_stereo)
    B, _, H, W = data["keyframe"].shape
    z = _closed_form_depths(data, inv_depth_min, inv_depth_max, steps, cv_depths, dtype)
    proj, kinv = projection_tables(data, use_mono, use_stereo, dtype=np.float64)
    inside = _interior(H, W)
    out = np.full((B, len(frames), H, W), -np.inf)
    for b in range(B):
        ray = _key_rays(kinv[b], H, W)
        for f in range(len(frames)):
            sx, sy = _source_positions(proj[b, f], ray, z[b], H, W, dtype)
            sx, sy = sx.astype(np.float64), sy.astype(np.float64)
            m = np.minimum(np.minimum(sx - 1, W - 2 - sx), np.minimum(sy - 1, H - 2 - sy))
            m = np.where(np.isfinite(m), m, -np.inf).min(axis=0)
            out[b, f] = np.where(inside, m, -np.inf)
    return out


def cost_volume_closed_form(data, inv_depth_min=0.33, inv_depth_max=0.0025, steps=32, use_mono=True,
                            use_stereo=False, alpha=ALPHA, channel_weights=CHANNEL_WEIGHTS, dtype=np.float32,
                            cv_depths=None, use_ssim=True, not_center_cv=False):
    """Direct evaluation of the Appendix-C formulas, with the options of `cost_volume_torch`.  The positions are
    evaluated in float64 (rounded to fp32 where dtype is float32), the rest in `dtype`.

    Returns (cv, [sfcv_f], valid (B,F,H,W), sad (B,F,D,H,W)).
    """
    if not use_ssim:
        raise NotImplementedError("use_ssim falsy")
    frames, _, _ = collect_frames(data, use_mono, use_stereo)
    key = data["keyframe"].numpy().astype(dtype)
    B, C, H, W = key.shape
    z = _closed_form_depths(data, inv_depth_min, inv_depth_max, steps, cv_depths, dtype)
    nF, D = len(frames), z.shape[1]
    proj, kinv = projection_tables(data, use_mono, use_stereo, dtype=np.float64)
    inside = _interior(H, W)
    cw = np.asarray(channel_weights, dtype=dtype).reshape(1, 3, 1, 1)

    cvs = np.zeros((B, D, H, W), dtype=dtype)
    sfs = np.zeros((nF, B, D, H, W), dtype=dtype)
    valids = np.zeros((B, nF, H, W), dtype=bool)
    sads = np.zeros((B, nF, D, H, W), dtype=dtype)
    for b in range(B):
        ray = _key_rays(kinv[b], H, W)
        Y = key[b] + dtype(0.5)
        mu_y = _box3(Y) / dtype(9)
        s_y = _box3(Y * Y) / dtype(9) - mu_y * mu_y
        num = np.zeros((D, H, W), dtype=dtype)
        den = np.zeros((H, W), dtype=dtype)
        for f in range(nF):
            img = frames[f][b].numpy().astype(dtype)
            sx, sy = _source_positions(proj[b, f], ray, z[b], H, W, dtype)
            X = _bilinear_zero(img, sx, sy) + dtype(0.5)                                   # (3,D,H,W)
            hit = _bilinear_zero(inside[None].astype(dtype), sx, sy)[0] != 0               # (D,H,W)
            valid = inside & hit.all(axis=0)
            e = _difference_closed_form(use_ssim, np.moveaxis(X, 0, 1), Y, mu_y, s_y, dtype)   # (D,3,H,W)
            sad = _box3((e * cw).sum(axis=1)) / dtype(9)                                   # (D,H,W)
            sads[b, f] = sad
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
    return cvs, [sfs[f] for f in range(nF)], valids, sads
