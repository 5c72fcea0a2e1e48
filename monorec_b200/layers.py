"""Drop-in for the reference's photometric residual image (model/layers.py:147-217), computed on the device by one kernel
(csrc/residual_image.cu through libmonorec_b200.so).

Given an inverse depth, the residual image warps every source frame into the keyframe, takes the per-pixel SSIM error of
each warp (3x3 box, reflection padding) averaged over the channels, and keeps the minimum over the frames: a check of a
depth map that needs no ground truth.  A (frame, pixel) whose warped sample is exactly 0 in some channel (no tap inside
the frame) is left out of the minimum, and a pixel that every frame leaves out is 0.

- `ResidualImage()(keyframe, keyframe_pose, keyframe_intrinsics, depths, frames, poses, intrinsics)` -> [B,1,H,W]: `depths`
  is the inverse depth itself (the wrapper passes inv_depth_max = 0, inv_depth_min = 1).
- `ResidualImageModule(use_mono, use_stereo)(data_dict)` writes `data_dict["residual_image"]` from
  `data_dict["predicted_inverse_depths"][0]` = p, back-projected at the inverse depth (1 - p) inv_depth_max + p inv_depth_min,
  as the reference does.  On a MonoRecModel output dict, whose prediction is already mapped to that range, this maps it a
  second time: the reference's behaviour, kept so that the two agree (use ResidualImage on `result` for the map of the
  model's inverse depth itself).

The images are [B,3,H,W] or grayscale [B,1,H,W] (one plane, read as the three-channel image whose planes equal it; the
result is that of the replicated images bit for bit).  CUDA tensors only: a CPU tensor raises MonorecLibraryError.
"""
from typing import List, Optional

import torch
from torch import Tensor, nn

from . import _lib


def residual_image_impl(keyframe: Tensor, frames: List[Tensor], keyframe_pose: Tensor, keyframe_intrinsics: Tensor,
                        poses: List[Tensor], intrinsics: List[Tensor], inv_depth: Tensor,
                        inv_depth_range: Optional[Tensor]) -> Tensor:
    """Projection tables + mr_residual_image on fp32 contiguous CUDA tensors -> [B,1,H,W] fp32.  inv_depth_range: [2] =
    (inv_depth_max, inv_depth_min) on the device, or None for (0, 1)."""
    lib = _lib.load()
    B, C, H, W = keyframe.shape
    proj = L.projection(keyframe, keyframe_pose, keyframe_intrinsics, poses, intrinsics)
    out = torch.empty(B, 1, H, W, device=keyframe.device, dtype=torch.float32)
    with torch.cuda.device(keyframe.device):
        _lib.check(lib.mr_residual_image(keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(), inv_depth.data_ptr(),
                                         None if inv_depth_range is None else inv_depth_range.data_ptr(), B, len(frames), C,
                                         H, W, out.data_ptr(), torch.cuda.current_stream(keyframe.device).cuda_stream),
                   "mr_residual_image")
    return out


def _range(inv_depth_max, inv_depth_min, device):
    """(inv_depth_max, inv_depth_min) as the kernel's device [2] fp32 tensor, or None for the wrapper's (0, 1).  Python
    numbers and one-element tensors are accepted (the reference broadcasts them over the map)."""
    if not torch.is_tensor(inv_depth_max) and not torch.is_tensor(inv_depth_min) \
            and float(inv_depth_max) == 0.0 and float(inv_depth_min) == 1.0:
        return None
    parts = []
    for name, v in (("inv_depth_max", inv_depth_max), ("inv_depth_min", inv_depth_min)):
        if torch.is_tensor(v):
            if v.numel() != 1:
                raise ValueError(f"ResidualImageModule: {name} must be a number or a one-element tensor, got {tuple(v.shape)}")
            parts.append(v.reshape(1).to(device=device, dtype=torch.float32))
        else:
            parts.append(torch.full((1,), float(v), device=device, dtype=torch.float32))
    return torch.cat(parts)


def residual_image(keyframe, keyframe_pose, keyframe_intrinsics, inv_depth, frames, poses, intrinsics, inv_depth_max=0,
                   inv_depth_min=1):
    """The residual image [B,1,H,W] fp32 of `inv_depth` [B,1,H,W] (mapped through (1 - p) inv_depth_max + p inv_depth_min)."""
    if not keyframe.is_cuda:
        raise _lib.MonorecLibraryError("monorec_b200.layers needs CUDA tensors (no CPU fallback)")
    frames, poses, intrinsics = list(frames), list(poses), list(intrinsics)
    if not frames or not (len(frames) == len(poses) == len(intrinsics)):
        raise ValueError(f"ResidualImage: {len(frames)} frames, {len(poses)} poses, {len(intrinsics)} intrinsics")
    if len(frames) > 8:
        raise NotImplementedError(f"ResidualImage: at most 8 source frames are built (got {len(frames)})")
    if keyframe.dim() != 4 or keyframe.shape[1] not in (1, 3):
        raise NotImplementedError(f"ResidualImage: images [B,3,H,W] or grayscale [B,1,H,W] only, got a keyframe "
                                  f"{tuple(keyframe.shape)}")
    if any(tuple(f.shape) != tuple(keyframe.shape) for f in frames):
        raise ValueError(f"ResidualImage: keyframe {tuple(keyframe.shape)}, frames {[tuple(f.shape) for f in frames]}: every "
                         "frame must have the keyframe's shape")
    B, _, H, W = keyframe.shape
    if tuple(inv_depth.shape) != (B, 1, H, W):
        raise ValueError(f"ResidualImage: depths {tuple(inv_depth.shape)}, keyframe {tuple(keyframe.shape)}")
    dev = keyframe.device
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()   # noqa: E731
    args = (f32(keyframe), [f32(t) for t in frames], f32(keyframe_pose), f32(keyframe_intrinsics), [f32(t) for t in poses],
            [f32(t) for t in intrinsics], f32(inv_depth).detach(), _range(inv_depth_max, inv_depth_min, dev))
    if torch.compiler.is_compiling():
        return torch.ops.monorec_b200.residual_image(*args)
    return residual_image_impl(*args)


class ResidualImage(nn.Module):
    """layers.py:147-158."""

    def __init__(self):
        super().__init__()
        self.residual_image = ResidualImageModule()

    def forward(self, keyframe: Tensor, keyframe_pose: Tensor, keyframe_intrinsics: Tensor, depths: Tensor, frames: list,
                poses: list, intrinsics: list):
        data_dict = {"keyframe": keyframe, "keyframe_pose": keyframe_pose, "keyframe_intrinsics": keyframe_intrinsics,
                     "predicted_inverse_depths": [depths], "frames": frames, "poses": poses, "list": list,
                     "intrinsics": intrinsics, "inv_depth_max": 0, "inv_depth_min": 1}
        data_dict = self.residual_image(data_dict)
        return data_dict["residual_image"]


class ResidualImageModule(nn.Module):
    """layers.py:161-217: the frames are the mono frames (`use_mono`) followed by the stereo frame (`use_stereo`)."""

    def __init__(self, use_mono=True, use_stereo=False):
        super().__init__()
        self.use_mono = use_mono
        self.use_stereo = use_stereo

    def forward(self, data_dict):
        frames, poses, intrinsics = L._collect(data_dict, self.use_mono, self.use_stereo)
        data_dict["residual_image"] = residual_image(
            data_dict["keyframe"], data_dict["keyframe_pose"], data_dict["keyframe_intrinsics"],
            data_dict["predicted_inverse_depths"][0], frames, poses, intrinsics, data_dict["inv_depth_max"],
            data_dict["inv_depth_min"])
        return data_dict


# imported last: losses and ops import this module in turn (ops wraps residual_image_impl)
from . import losses as L  # noqa: E402
from . import ops  # noqa: E402,F401  (registers monorec_b200::residual_image, which residual_image calls under torch.compile)
