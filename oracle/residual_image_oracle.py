"""Oracle of the photometric residual image (reference: model/layers.py:147-217, ResidualImage / ResidualImageModule).

- `residual_image_torch`: the reference's arithmetic restated in torch, fp32, on the inputs' device (the CPU for the golden
  checks; tools/time_residual_image.py times it on the GPU): back-projection of every keyframe
  pixel with torch.inverse(K) divided by the inverse depth, point_projection (layers.py:63-71: +1e-7, the (W-1) / (H-1)
  normalisation, no clamp), F.grid_sample of frame + 1 (bilinear, zero padding, align_corners=False), the mask
  any_c(warped == 0), the reflection-padded 3x3-box SSIM of warped - 0.5 against keyframe + 0.5 (not comp mode), the channel
  mean, +inf where masked, the minimum over the frames, 0 where every frame is masked.
- `residual_image_closed_form`: the same quantity in numpy float64 from the projection matrices, with the per-frame masks
  and `margin`, the signed distance in source pixels from each sample to the edge of the region where its bilinear sample
  has a tap inside the image (-1 < sx < W, -1 < sy < H): a sample within a small margin may be masked in one fp32
  evaluation and not in another.

Both take the inverse depth p and map it as the reference does, (1 - p) inv_depth_max + p inv_depth_min in fp32, and read a
grayscale image [B,1,H,W] as its three-channel replica.
"""
import numpy as np
import torch
import torch.nn.functional as F

from .cost_volume_oracle import _bilinear_zero, _key_rays

SSIM_C1 = 0.01 ** 2
SSIM_C2 = 0.03 ** 2


def _rgb(t):
    return t.expand(-1, 3, -1, -1) if t.shape[1] == 1 else t


def map_inverse_depth(p, inv_depth_max=0, inv_depth_min=1):
    """layers.py:172 in fp32 torch, op by op."""
    return (1 - p) * inv_depth_max + p * inv_depth_min


def _ssim_error(x, y):
    """Reflection-padded 3x3-box SSIM error clamp((1 - SSIM) / 2, 0, 1), per channel (layers.py:119-137)."""
    x = F.pad(x, (1, 1, 1, 1), mode="reflect")
    y = F.pad(y, (1, 1, 1, 1), mode="reflect")
    box = lambda t: F.avg_pool2d(t, 3, 1)   # noqa: E731
    mu_x, mu_y = box(x), box(y)
    sig_x = box(x * x) - mu_x ** 2
    sig_y = box(y * y) - mu_y ** 2
    sig_xy = box(x * y) - mu_x * mu_y
    n = (2 * mu_x * mu_y + SSIM_C1) * (2 * sig_xy + SSIM_C2)
    d = (mu_x ** 2 + mu_y ** 2 + SSIM_C1) * (sig_x + sig_y + SSIM_C2)
    return torch.clamp((1 - n / d) / 2, 0, 1)


def residual_image_torch(keyframe, keyframe_pose, keyframe_intrinsics, inv_depth, frames, poses, intrinsics,
                         inv_depth_max=0, inv_depth_min=1, return_masks=False):
    """-> residual [B,1,H,W] fp32 (and the masks [B,F,H,W] bool with return_masks), on the inputs' device."""
    keyframe, frames = _rgb(keyframe.float()), [_rgb(f.float()) for f in frames]
    B, C, H, W = keyframe.shape
    depth = map_inverse_depth(inv_depth.float(), inv_depth_max, inv_depth_min)
    dev = keyframe.device
    vv, uu = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=dev), torch.arange(W, dtype=torch.float32, device=dev),
                            indexing="ij")
    pix = torch.stack([uu.reshape(-1), vv.reshape(-1), torch.ones(H * W, device=dev)]).unsqueeze(0).expand(B, 3, H * W)
    rays = torch.inverse(keyframe_intrinsics.float())[:, :3, :3] @ pix
    points = torch.cat([rays / depth.reshape(B, 1, -1), torch.ones(B, 1, H * W, device=dev)], 1)
    errors, masks = [], []
    for img, pose, K in zip(frames, poses, intrinsics):
        T = torch.inverse(pose.float()) @ keyframe_pose.float()
        cam = (K.float() @ T)[:, :3, :] @ points
        xy = cam[:, :2] / (cam[:, 2:3] + 1e-7)
        gx = (xy[:, 0] / (W - 1) - 0.5) * 2
        gy = (xy[:, 1] / (H - 1) - 0.5) * 2
        grid = torch.stack([gx, gy], -1).reshape(B, H, W, 2)
        warped = F.grid_sample(img + 1, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
        masks.append((warped == 0).any(1))
        errors.append(_ssim_error(warped - 0.5, keyframe + 0.5).mean(1))
    masks = torch.stack(masks, 1)
    errors = torch.where(masks, torch.full_like(errors[0][:, None], float("inf")), torch.stack(errors, 1))
    out = errors.min(1, keepdim=True)[0]
    out = torch.where(masks.all(1, keepdim=True), torch.zeros_like(out), out)
    return (out, masks) if return_masks else out


def residual_image_closed_form(keyframe, keyframe_pose, keyframe_intrinsics, inv_depth, frames, poses, intrinsics,
                               inv_depth_max=0, inv_depth_min=1):
    """-> dict of float64 / bool numpy arrays: residual [B,1,H,W], masks [B,F,H,W], margin [B,F,H,W] (-inf where the
    position is not finite)."""
    keyframe, frames = _rgb(keyframe.float()), [_rgb(f.float()) for f in frames]
    B, C, H, W = keyframe.shape
    nF = len(frames)
    z_inv = map_inverse_depth(inv_depth.float(), inv_depth_max, inv_depth_min).numpy().astype(np.float64)[:, 0]
    residual = np.zeros((B, 1, H, W))
    masks = np.zeros((B, nF, H, W), dtype=bool)
    margin = np.zeros((B, nF, H, W))

    def ssim_error(x, y):
        pad = lambda t: np.pad(t, ((0, 0), (1, 1), (1, 1)), mode="reflect")   # noqa: E731
        box = lambda t: sum(t[:, i:i + H, j:j + W] for i in range(3) for j in range(3)) / 9.0   # noqa: E731
        x, y = pad(x), pad(y)
        mu_x, mu_y = box(x), box(y)
        sig_x, sig_y, sig_xy = box(x * x) - mu_x ** 2, box(y * y) - mu_y ** 2, box(x * y) - mu_x * mu_y
        n = (2 * mu_x * mu_y + SSIM_C1) * (2 * sig_xy + SSIM_C2)
        d = (mu_x ** 2 + mu_y ** 2 + SSIM_C1) * (sig_x + sig_y + SSIM_C2)
        with np.errstate(invalid="ignore"):
            e = (1 - n / d) / 2
            return np.where(np.isnan(e), e, np.clip(e, 0, 1))

    for b in range(B):
        kinv = np.linalg.inv(keyframe_intrinsics[b].numpy().astype(np.float64))[:3, :3]
        ray = _key_rays(kinv, H, W)
        key = keyframe[b].numpy().astype(np.float64) + 0.5
        errs = np.zeros((nF, H, W))
        for f in range(nF):
            T = np.linalg.inv(poses[f][b].numpy().astype(np.float64)) @ keyframe_pose[b].numpy().astype(np.float64)
            P = (intrinsics[f][b].numpy().astype(np.float64) @ T)[:3]
            with np.errstate(divide="ignore", invalid="ignore"):
                c = np.einsum("ij,jhw->ihw", P[:, :3], ray / z_inv[b][None]) + P[:, 3][:, None, None]
                px, py = c[0] / (c[2] + 1e-7), c[1] / (c[2] + 1e-7)
                sx = ((px / (W - 1) - 0.5) * 2 + 1) * W / 2 - 0.5
                sy = ((py / (H - 1) - 0.5) * 2 + 1) * H / 2 - 0.5
            finite = np.isfinite(sx) & np.isfinite(sy)
            sxf, syf = np.where(finite, sx, -10.0), np.where(finite, sy, -10.0)
            img = frames[f][b].numpy().astype(np.float64) + 1
            v = _bilinear_zero(img, sxf, syf)
            v = np.where(finite[None], v, np.nan)
            masks[b, f] = (v == 0).any(0)
            margin[b, f] = np.where(finite, np.minimum(np.minimum(sxf + 1, W - sxf), np.minimum(syf + 1, H - syf)), -np.inf)
            errs[f] = ssim_error(v - 0.5, key).mean(0)
        errs = np.where(masks[b], np.inf, errs)
        with np.errstate(invalid="ignore"):
            r = np.where(np.isnan(errs).any(0), np.nan, errs.min(0))
        residual[b, 0] = np.where(masks[b].all(0), 0.0, r)
    return {"residual": residual, "masks": masks, "margin": margin}
