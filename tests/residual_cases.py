"""Seeded inputs of the residual-image cases shared by tests/golden/make_golden_residual_image.py and the tests
(tests/test_residual_image.py on the CPU, tests/test_residual_image_gpu.py on the GPU).  The images and poses come from
monorec_b200.synthetic.make_inputs; the inverse depths are stored in the golden file beside the reference's results."""
import math

import torch

from monorec_b200.synthetic import make_inputs

# name -> (batch, frames, height, width, seed, stereo, gray)
CASES = {
    "synth": (2, 2, 40, 64, 31, False, False),
    "out_of_image": (1, 3, 40, 64, 32, False, False),
    "edges": (1, 2, 24, 40, 33, False, False),
    "stereo": (2, 2, 40, 64, 34, True, False),
    "ragged": (1, 2, 37, 61, 35, False, False),
    "gray": (1, 3, 40, 64, 36, False, True),
    "model": (1, 2, 64, 128, 37, False, False),
}
MODEL_SEED, MODEL_GAIN = 5, 0.7


def smooth_inverse_depth(B, H, W, seed, lo=0.02, hi=0.3):
    """A seeded smooth inverse-depth map [B,1,H,W] in [lo, hi]."""
    g = torch.Generator().manual_seed(seed)
    yy = torch.arange(H, dtype=torch.float32).view(1, 1, H, 1) / H
    xx = torch.arange(W, dtype=torch.float32).view(1, 1, 1, W) / W
    t = torch.zeros(B, 1, H, W)
    for _ in range(4):
        fy, fx = torch.rand(B, 1, 1, 1, generator=g) * 3, torch.rand(B, 1, 1, 1, generator=g) * 3
        ph = torch.rand(B, 1, 1, 1, generator=g) * 2 * math.pi
        t = t + torch.sin(2 * math.pi * (fy * yy + fx * xx) + ph)
    t = (t - t.amin((2, 3), keepdim=True)) / (t.amax((2, 3), keepdim=True) - t.amin((2, 3), keepdim=True))
    return (lo + (hi - lo) * t).contiguous()


def inverse_depth(name):
    """The case's inverse depth as the golden script makes it ("model" takes the model's prediction instead)."""
    B, _, H, W, seed, _, _ = CASES[name]
    if name == "out_of_image":
        # near points (inverse depth up to 1.2) on the right half: their samples leave the frame 0.8 m ahead partly or wholly;
        # a strip of points behind the camera (negative inverse depth) is sampled at the mirrored projection
        d = smooth_inverse_depth(B, H, W, seed)
        ramp = torch.linspace(0, 1.2, W).clamp(min=0.3) * (torch.arange(W) >= W // 2)
        d = torch.maximum(d, ramp.view(1, 1, 1, W))
        d[..., 5:8, 4:20] = -0.1
        return d.contiguous()
    if name == "edges":
        # non-finite and non-positive inverse depths: 0, -0, +inf, -inf, NaN, tiny and negative values
        d = smooth_inverse_depth(B, H, W, seed)
        special = [0.0, -0.0, math.inf, -math.inf, math.nan, 1e-30, -1e-30, -0.05, -5.0, 1e30]
        for i, v in enumerate(special):
            d[0, 0, 4 + (i % 5) * 4, 6 + (i // 5) * 20] = v
        return d.contiguous()
    return smooth_inverse_depth(B, H, W, seed)


def inputs(name):
    """The case's data dict (CPU): keyframe, frames, poses, intrinsics, and for "stereo" the stereo frame; for "gray"
    three-channel images whose planes are equal (their first plane is the one-channel input)."""
    B, nF, H, W, seed, stereo, gray = CASES[name]
    data = make_inputs(B, nF, H, W, seed=seed)
    if gray:
        rep = lambda t: t[:, :1].expand(-1, 3, -1, -1).contiguous()   # noqa: E731
        data["keyframe"] = rep(data["keyframe"])
        data["frames"] = [rep(f) for f in data["frames"]]
    if stereo:
        extra = make_inputs(B, nF + 1, H, W, seed=seed + 1000)
        pose = torch.eye(4).repeat(B, 1, 1)
        pose[:, 0, 3] = 0.54                      # the KITTI baseline, right camera
        data["stereoframe"] = extra["frames"][nF]
        data["stereoframe_pose"] = pose
        data["stereoframe_intrinsics"] = data["intrinsics"][0].clone()
    return data


def gray(data):
    """The one-channel dict of a "gray" case: the first plane of every image."""
    out = dict(data)
    out["keyframe"] = data["keyframe"][:, :1].contiguous()
    out["frames"] = [f[:, :1].contiguous() for f in data["frames"]]
    return out
