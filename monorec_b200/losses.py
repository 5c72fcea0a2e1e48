"""Drop-in for the reference's photometric reprojection loss (model/loss_functions/common_losses.py:16-114), forward and
backward on the device (csrc/reprojection.cu through libmonorec_b200.so).  SURVEY.md 8f row 4.

`reprojection_loss` keeps the reference's name, argument list and defaults, and supports the argument sets the reference's
own losses pass (model/loss_functions/monorec_loss.py:185-188, :264-265, :355, :361): `error_function=compute_errors`,
`combine_frames="min"`, `mono_auto=False`, `automasking` False / True, `border` 0 / n, `use_mono` / `use_stereo`,
`reduce` False / True.  Everything else raises NotImplementedError (no second code path, no CPU fallback).  The result is
differentiable w.r.t. `depth_prediction` through a torch.autograd.Function whose backward is one kernel; nothing but the
[B,H,W] index of the winning frame is kept between the passes (the reference keeps ~25 full-size temporaries per frame).
"""
from typing import List

import torch
from torch import Tensor

from . import _lib


def compute_errors(img0, img1, mask=None):
    """Marker for `error_function=`: 0.85 * SSIM (Gaussian window, zero padding, comp mode) + 0.15 * L1, channel means
    (common_losses.py:10-13).  The arithmetic lives inside the fused kernels; this function is never called."""
    raise NotImplementedError("compute_errors is evaluated inside mr_reprojection_loss_fwd; pass it as error_function only")


def _collect(data_dict, use_mono, use_stereo):
    frames, poses, intrinsics = [], [], []                                     # common_losses.py:23-34
    if use_mono:
        frames += list(data_dict["frames"]); poses += list(data_dict["poses"]); intrinsics += list(data_dict["intrinsics"])
    if use_stereo:
        frames.append(data_dict["stereoframe"]); poses.append(data_dict["stereoframe_pose"])
        intrinsics.append(data_dict["stereoframe_intrinsics"])
    return frames, poses, intrinsics


def projection(keyframe: Tensor, keyframe_pose: Tensor, keyframe_intrinsics: Tensor, poses: List[Tensor],
               intrinsics: List[Tensor]) -> Tensor:
    """[B,F,12] keyframe-to-frame projection tables (mr_projection_tables) from contiguous fp32 CUDA tensors."""
    lib = _lib.load()
    B, _, H, W = keyframe.shape
    dev = keyframe.device
    proj = torch.empty(B, len(poses), 12, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(lib.mr_projection_tables(keyframe_pose.data_ptr(), keyframe_intrinsics.data_ptr(), _lib.ptr_array(poses),
                                            _lib.ptr_array(intrinsics), B, len(poses), H, W, proj.data_ptr(), None, 0, 0.0,
                                            0.0, torch.cuda.current_stream(dev).cuda_stream), "mr_projection_tables")
    return proj


def errors_fwd(keyframe, frames, proj, invd, automasking, border):
    """mr_reprojection_loss_fwd on fp32 contiguous inputs (invd: [B,1,H,W] inverse depth) -> (errors, winner) [B,H,W]."""
    lib = _lib.load()
    B, _, H, W = keyframe.shape
    errors = torch.empty(B, H, W, device=keyframe.device, dtype=torch.float32)
    winner = torch.empty(B, H, W, device=keyframe.device, dtype=torch.int32)
    with torch.cuda.device(keyframe.device):
        _lib.check(lib.mr_reprojection_loss_fwd(keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(), invd.data_ptr(),
                                                B, len(frames), H, W, 1 if automasking else 0, int(border), errors.data_ptr(),
                                                winner.data_ptr(), torch.cuda.current_stream(keyframe.device).cuda_stream),
                   "mr_reprojection_loss_fwd")
    return errors, winner


def errors_bwd(keyframe, frames, proj, invd, grad_errors, winner):
    """mr_reprojection_loss_bwd -> the gradient [B,1,H,W] fp32 w.r.t. the inverse depth."""
    lib = _lib.load()
    B, _, H, W = keyframe.shape
    g = grad_errors.to(torch.float32).contiguous()
    out = torch.empty(B, 1, H, W, device=keyframe.device, dtype=torch.float32)
    with torch.cuda.device(keyframe.device):
        _lib.check(lib.mr_reprojection_loss_bwd(keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(), invd.data_ptr(),
                                                g.data_ptr(), winner.data_ptr(), B, len(frames), H, W, out.data_ptr(),
                                                torch.cuda.current_stream(keyframe.device).cuda_stream),
                   "mr_reprojection_loss_bwd")
    return out


class _ReprojectionErrors(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_prediction, keyframe, proj, automasking, border, *frames):
        invd = depth_prediction.detach().to(torch.float32).contiguous()
        errors, winner = errors_fwd(keyframe, frames, proj, invd, automasking, border)
        ctx.save_for_backward(invd, keyframe, proj, winner, *frames)
        ctx.mark_non_differentiable(winner)
        ctx.in_dtype = depth_prediction.dtype
        return errors, winner

    @staticmethod
    def backward(ctx, grad_errors, _grad_winner):
        invd, keyframe, proj, winner, *frames = ctx.saved_tensors
        out = errors_bwd(keyframe, frames, proj, invd, grad_errors, winner)
        return (out.to(ctx.in_dtype), None, None, None, None) + (None,) * len(frames)


def reprojection_errors(depth_prediction, data_dict, automasking=False, use_mono=True, use_stereo=False, border=0):
    """-> (errors [B,H,W], +inf where no source frame gives a usable sample; winner [B,H,W] int32, -1 there)."""
    keyframe = data_dict["keyframe"]
    if not keyframe.is_cuda:
        raise _lib.MonorecLibraryError("monorec_b200.losses needs CUDA tensors (no CPU fallback)")
    frames, poses, intrinsics = _collect(data_dict, use_mono, use_stereo)
    if not frames:
        raise ValueError("reprojection_loss: no source frames (use_mono / use_stereo)")
    B, C, H, W = keyframe.shape
    if C != 3 or tuple(depth_prediction.shape) != (B, 1, H, W):
        raise ValueError(f"reprojection_loss: keyframe {tuple(keyframe.shape)} / depth_prediction {tuple(depth_prediction.shape)}")
    if depth_prediction.device != keyframe.device:
        raise ValueError(f"reprojection_loss: depth_prediction on {depth_prediction.device}, keyframe on {keyframe.device}")
    dev = keyframe.device
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()   # noqa: E731
    keyframe = f32(keyframe)
    frames = [f32(t) for t in frames]
    kf_pose, kf_K = f32(data_dict["keyframe_pose"]), f32(data_dict["keyframe_intrinsics"])
    poses, intrinsics = [f32(t) for t in poses], [f32(t) for t in intrinsics]
    if torch.compiler.is_compiling():
        # one op for the tables and the forward pass; its autograd formula runs the backward op (monorec_b200/ops.py)
        errors, winner, _ = torch.ops.monorec_b200.reprojection_loss_fwd(depth_prediction, keyframe, frames, kf_pose, kf_K,
                                                                         poses, intrinsics, bool(automasking), int(border))
        return errors, winner
    proj = projection(keyframe, kf_pose, kf_K, poses, intrinsics)
    return _ReprojectionErrors.apply(depth_prediction, keyframe, proj, bool(automasking), int(border), *frames)


def mask_mean(t, m):
    """utils/util.py:110-118 over all dimensions (one fused expression, no host synchronisation)."""
    return torch.sum(torch.where(m, torch.zeros_like(t), t)) / (t.numel() - torch.sum(m.to(torch.float32)))


def reprojection_loss(depth_prediction, data_dict, automasking=False, error_function=compute_errors, error_function_weight=None,
                      use_mono=True, use_stereo=False, reduce=True, combine_frames="min", mono_auto=False, border=0):
    """common_losses.py:16-114.  `error_function` must be `compute_errors` (this module's marker or the reference's function of
    that name), alone or as a one-element list with an optional weight."""
    efs = error_function if isinstance(error_function, list) else [error_function]
    wts = error_function_weight if error_function_weight is not None else [1] * len(efs)
    if len(efs) != 1 or getattr(efs[0], "__name__", None) != "compute_errors":
        raise NotImplementedError("reprojection_loss: only error_function=compute_errors is built (common_losses.py:10-13)")
    if combine_frames != "min" or mono_auto:
        raise NotImplementedError("reprojection_loss: only combine_frames='min', mono_auto=False are built "
                                  "(the settings of model/loss_functions/monorec_loss.py)")
    errors, _ = reprojection_errors(depth_prediction, data_dict, automasking, use_mono, use_stereo, border)
    if reduce:                                                                  # :110-111
        return wts[0] * mask_mean(errors, torch.isinf(errors))
    return wts[0] * errors                                                      # :112-113


from . import ops  # noqa: E402,F401  (registers the loss ops, which reprojection_errors calls under torch.compile)
