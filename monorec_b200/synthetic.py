"""Synthetic KITTI-shaped inputs for the MonoRec hot path.

The generator follows SURVEY.md §8(d): smooth textured images in [-0.5, 0.5], the
intrinsics of the bundled KITTI sample (reference: data_loader/kitti_odometry_dataset.py:318-374
scaled to the requested size), identity keyframe pose and source poses that translate
along z by {-0.8, +0.8, -1.6, +1.6, -2.4, +2.4} m with a <= 0.5 degree random rotation.

Everything is produced with a CPU torch.Generator so the same seed gives the same dict
on the dev container and on the GPU box (tests, bench.py and the golden script share it).
"""
import math

import torch

# fx, fy, cx, cy of example/data/kitti/sequences/07 after crop+resize to 256x512
KITTI_FX, KITTI_FY, KITTI_CX, KITTI_CY = 489.2307, 489.2307, 248.3112, 126.6926
Z_STEPS = (-0.8, 0.8, -1.6, 1.6, -2.4, 2.4)


def kitti_intrinsics(height, width, batch=1):
    k = torch.zeros(4, 4, dtype=torch.float32)
    k[0, 0] = KITTI_FX * width / 512.0
    k[1, 1] = KITTI_FY * height / 256.0
    k[0, 2] = KITTI_CX * width / 512.0
    k[1, 2] = KITTI_CY * height / 256.0
    k[2, 2] = 1.0
    k[3, 3] = 1.0
    return k.unsqueeze(0).repeat(batch, 1, 1)


def _texture(gen, batch, height, width, n_waves=6):
    """Sum of random low-frequency sinusoids per channel, normalised to [-0.45, 0.45]."""
    yy = torch.arange(height, dtype=torch.float32).view(1, 1, height, 1) / height
    xx = torch.arange(width, dtype=torch.float32).view(1, 1, 1, width) / width
    img = torch.zeros(batch, 3, height, width)
    for _ in range(n_waves):
        fy = torch.rand(batch, 3, 1, 1, generator=gen) * 12.0
        fx = torch.rand(batch, 3, 1, 1, generator=gen) * 24.0
        ph = torch.rand(batch, 3, 1, 1, generator=gen) * 2 * math.pi
        amp = torch.rand(batch, 3, 1, 1, generator=gen) + 0.3
        img += amp * torch.sin(2 * math.pi * (fy * yy + fx * xx) + ph)
    img = img / img.abs().amax(dim=(2, 3), keepdim=True) * 0.45
    return img


def _small_rotation(gen, batch, max_deg=0.5):
    ang = (torch.rand(batch, 3, generator=gen) * 2 - 1) * math.radians(max_deg)
    rx, ry, rz = ang[:, 0], ang[:, 1], ang[:, 2]
    one, zero = torch.ones(batch), torch.zeros(batch)
    Rx = torch.stack([one, zero, zero, zero, rx.cos(), -rx.sin(), zero, rx.sin(), rx.cos()], 1).view(batch, 3, 3)
    Ry = torch.stack([ry.cos(), zero, ry.sin(), zero, one, zero, -ry.sin(), zero, ry.cos()], 1).view(batch, 3, 3)
    Rz = torch.stack([rz.cos(), -rz.sin(), zero, rz.sin(), rz.cos(), zero, zero, zero, one], 1).view(batch, 3, 3)
    return Rz @ Ry @ Rx


def _quantise(img):
    """8-bit image levels, as the reference loader yields (kitti_odometry_dataset.py:126-127: uint8/255 - .5)."""
    return torch.round((img.clamp(-0.5, 0.5) + 0.5) * 255.0) / 255.0 - 0.5


def make_inputs(batch, frames, height, width, seed=0, noise=0.05, device="cpu"):
    """Returns a MonoRec data_dict (reference layout: kitti_odometry_dataset.py:260-269 after collate)."""
    gen = torch.Generator().manual_seed(seed)
    base = _texture(gen, batch, height, width)
    data = {}
    key = base + noise * (torch.rand(batch, 3, height, width, generator=gen) - 0.5)
    data["keyframe"] = _quantise(key).contiguous()
    data["keyframe_pose"] = torch.eye(4).unsqueeze(0).repeat(batch, 1, 1)
    data["keyframe_intrinsics"] = kitti_intrinsics(height, width, batch)
    data["frames"], data["poses"], data["intrinsics"] = [], [], []
    for f in range(frames):
        # a different (shifted) texture per source frame keeps the photometric cost non-trivial
        shift = int(3 * (f + 1))
        img = torch.roll(base, shifts=(shift // 2, shift), dims=(2, 3))
        img = img + noise * (torch.rand(batch, 3, height, width, generator=gen) - 0.5)
        data["frames"].append(_quantise(img).contiguous())
        pose = torch.eye(4).unsqueeze(0).repeat(batch, 1, 1)
        pose[:, :3, :3] = _small_rotation(gen, batch)
        pose[:, 2, 3] = Z_STEPS[f % len(Z_STEPS)] * (1 + f // len(Z_STEPS))
        data["poses"].append(pose)
        data["intrinsics"].append(kitti_intrinsics(height, width, batch))
    if device != "cpu":
        data = to_device(data, device)
    return data


def make_sequence(n_frames, height, width, seed=0, step=0.8, noise=0.05):
    """A synthetic KITTI-shaped video: camera n sits n * step m down the z axis (with a <= 0.5 degree random rotation) and
    sees the shared texture shifted by n pixels.  Returns images [N,3,H,W] in [-0.5, 0.5], cam -> world poses [N,4,4] and
    intrinsics [N,4,4], on the CPU."""
    gen = torch.Generator().manual_seed(seed)
    base = _texture(gen, 1, height, width)[0]
    images = torch.stack([_quantise(torch.roll(base, shifts=(n // 2, n), dims=(1, 2))
                                    + noise * (torch.rand(3, height, width, generator=gen) - 0.5)) for n in range(n_frames)])
    poses = torch.eye(4).repeat(n_frames, 1, 1)
    poses[:, :3, :3] = _small_rotation(gen, n_frames)
    poses[:, 2, 3] = step * torch.arange(n_frames, dtype=torch.float32)
    return images.contiguous(), poses, kitti_intrinsics(height, width, n_frames)


def to_device(data, device, non_blocking=False):
    out = {}
    for k, v in data.items():
        if isinstance(v, (list, tuple)):
            out[k] = [t.to(device, non_blocking=non_blocking) for t in v]
        elif torch.is_tensor(v):
            out[k] = v.to(device, non_blocking=non_blocking)
        else:
            out[k] = v
    return out


def seeded_state_dict(module, seed=0, gain=1.0):
    """Deterministic weights for parity tests (no pretrained checkpoint is available offline).

    Every floating-point entry of module.state_dict() is regenerated from (seed, key) so that the
    reference model (golden script) and the drop-in (tests) can be given identical parameters
    without shipping a 70 MB state_dict.  `gain` > 1 spreads activations so that |tanh| / sigmoid
    heads leave their linear range (SURVEY.md §8c, "random weights make the gate vacuous").
    """
    import zlib
    out = {}
    for key, val in module.state_dict().items():
        if not torch.is_floating_point(val):
            out[key] = val.clone()
            continue
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFF)
        if key.endswith("running_var"):
            t = torch.rand(val.shape, generator=g) + 0.5
        elif key.endswith("running_mean"):
            t = torch.randn(val.shape, generator=g) * 0.1
        elif val.dim() >= 2:
            fan_in = val[0].numel() if "conv2d_t" not in key else val.shape[0] * val.shape[2] * val.shape[3] / 4.0
            t = torch.randn(val.shape, generator=g) * (gain * math.sqrt(2.0 / max(fan_in, 1)))
        elif key.endswith("weight"):          # batch-norm scale
            t = torch.rand(val.shape, generator=g) + 0.5
        else:                                 # biases
            t = torch.randn(val.shape, generator=g) * 0.05 * gain
        out[key] = t.to(val.dtype)
    return out
