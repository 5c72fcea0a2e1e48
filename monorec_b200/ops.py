"""PyTorch custom operators (namespace `monorec_b200`) over the library's launches, so that `torch.compile(model)` and
`torch.export` trace MonoRecModel.forward, the metrics, the median scaling and the reprojection loss as graphs.

Every launch goes through ctypes with `tensor.data_ptr()`, and the packed-weight caches key on `data_ptr()` / `_version`:
neither can be traced (a FakeTensor has no storage).  Each op below wraps one stage whose host code does that, and its
implementation is the very function the eager path calls, so both give the same bits by construction.  The wrappers
(`CostVolumeModule.forward`, `MaskModule.forward`, `DepthModule.forward`, `MonoRecModel`'s trunk call,
`conv.mask_volume`, the functions of `metrics` and `losses`) call the op only when `torch.compiler.is_compiling()`; eager
calls the implementation directly, with no dispatcher in front of its ~150 launches.

- `cost_volume`: projection tables + the fused cost-volume kernel (every error mode, centring, both depth sources, fp32 /
  half storage); it fills the MaskModule's NHWC input buffer when one is given (a declared mutation).  Returns the fused
  volume [B,D,H,W] and the [F,B,D,H,W] single-frame buffer.
- `resnet_trunk`: the folded cuDNN trunk with the model's TF32 setting (the cuDNN flags are set on real tensors, inside the
  op) and the stem pool kernel; returns the five levels (level 4 is computed, not lazy).
- `mask_module`, `depth_module`: the two convolution stacks on the wgmma engine.
- `mask_volume`: cost_volume * (1 - cv_mask).
- `sparse_metrics`, `dense_metrics`, `median_scaling`: the evaluation passes.
- `reprojection_loss_fwd` (projection tables + forward pass) and `reprojection_loss_bwd`, joined by
  `torch.library.register_autograd`, so that a compiled loss backpropagates to `depth_prediction`.
- `residual_image`: projection tables + the residual-image kernel (`layers.ResidualImage`, `ResidualImageModule`).

The Mask, Depth and trunk ops compute from the weights they are given: the module's parameters (and the trunk's BatchNorm
buffers) are tensor inputs, next to the module's configuration.  The implementation binds them into a module of that
configuration kept for the purpose (`_template`, its own parameters never used) and runs the eager code on it; the
packed-weight lookup keys on the given tensors (signature: data pointer, version, device, arithmetic mode), on real tensors
inside the op.  So `load_state_dict`, an optimizer step or `.to()` between two compiled calls is seen as in eager, and an
exported program computes with the weights it holds.  The shared cache keeps the packed copies of the last four weight sets
per configuration, and holds those weights until they are evicted.

Not wrapped: `mr_pointcloud_add`, whose output size depends on the data, and the host-buffer entries
(`mr_cost_volume_host*`), which take host memory.
"""
import contextlib
import threading
from typing import List, Optional, Tuple

import torch
from torch import Tensor

from . import conv as C
from . import cost_volume as CV
from . import layers as LY
from . import losses as L
from . import metrics as MT

_TEMPLATES = {}                       # (class name, configuration) -> (module, lock)
_TEMPLATE_LOCK = threading.Lock()


def _template(kind, *config):
    """The module of class `kind` and this configuration that the ops bind weights into (built once, on the meta device)."""
    key = (kind,) + config
    with _TEMPLATE_LOCK:
        if key not in _TEMPLATES:
            from . import model as M
            with torch.device("meta"):
                mod = getattr(M, kind)(*config).eval()
            mod._packed = M._PackedShared()
            _TEMPLATES[key] = (mod, threading.Lock())
        return _TEMPLATES[key]


@contextlib.contextmanager
def _bound(mod, tensors):
    """`mod` with the tensors of its `_source_names()` replaced by `tensors` (restored on exit)."""
    names = mod._source_names()
    if len(names) != len(tensors):
        raise ValueError(f"monorec_b200 op: {type(mod).__name__} takes {len(names)} weight tensors, got {len(tensors)}")
    saved = []
    try:
        for name, t in zip(names, tensors):
            owner_name, _, leaf = name.rpartition(".")
            owner = mod.get_submodule(owner_name)
            slots = owner._parameters if leaf in owner._parameters else owner._buffers
            saved.append((slots, leaf, slots[leaf]))
            slots[leaf] = t
        yield mod
    finally:
        for slots, leaf, old in reversed(saved):
            slots[leaf] = old


def _run_bound(kind, config, params, fn):
    mod, lock = _template(kind, *config)
    with lock, _bound(mod, params), torch.no_grad():
        return fn(mod)


# ---- cost volume ---------------------------------------------------------------------------------------------------
cost_volume = torch.library.custom_op("monorec_b200::cost_volume", CV.launch, mutates_args=("sfcv_nhwc",),
                                      device_types="cuda")


@cost_volume.register_fake
def _(keyframe, frames, intrinsics, poses, keyframe_pose, keyframe_intrinsics, cv_depths, sfcv_nhwc, lo, hi, steps, alpha,
      channel_weights, matching, center, half):
    B, _, H, W = keyframe.shape
    D = steps if cv_depths is None else cv_depths.shape[1]
    dt = torch.float16 if half else torch.float32
    return keyframe.new_empty(B, D, H, W, dtype=dt), keyframe.new_empty(len(frames), B, D, H, W, dtype=dt)


# ---- trunk ---------------------------------------------------------------------------------------------------------
@torch.library.custom_op("monorec_b200::resnet_trunk", mutates_args=(), device_types="cuda")
def resnet_trunk(image: Tensor, params: List[Tensor], allow_tf32: bool) -> List[Tensor]:
    from .model import trunk_features
    return _run_bound("ResnetEncoder", (18, False), params, lambda enc: list(trunk_features(enc, image, allow_tf32)))


@resnet_trunk.register_fake
def _(image, params, allow_tf32):
    half = C.MODE == "f16" and image.is_cuda          # (the folded trunk: eval mode, no grad)
    B, _, H, W = image.shape
    down = lambda n: (n - 1) // 2 + 1       # noqa: E731  (3x3 / 7x7 stride-2 convolutions and the 3x3 stride-2 pool)
    sizes = [(down(H), down(W))]
    sizes.append((down(sizes[0][0]), down(sizes[0][1])))
    for _ in range(3):
        sizes.append((down(sizes[-1][0]), down(sizes[-1][1])))
    chans = (64, 64, 128, 256, 512)
    return [torch.empty(B, c, h, w, device=image.device, dtype=torch.float16 if half else torch.float32,
                        memory_format=torch.channels_last) for c, (h, w) in zip(chans, sizes)]


# ---- convolution stacks --------------------------------------------------------------------------------------------
@torch.library.custom_op("monorec_b200::mask_module", mutates_args=(), device_types="cuda")
def mask_module(single_frame_cvs: List[Tensor], image_features: List[Tensor], sfcv_nhwc: Optional[Tensor],
                params: List[Tensor], depth_steps: int, feature_channels: List[int], use_cv: bool,
                use_features: bool) -> Tensor:
    return _run_bound("MaskModule", (depth_steps, tuple(feature_channels), use_cv, use_features), params,
                      lambda m: m._run(single_frame_cvs, image_features, sfcv_nhwc))


@mask_module.register_fake
def _(single_frame_cvs, image_features, sfcv_nhwc, params, depth_steps, feature_channels, use_cv, use_features):
    B, _, H, W = single_frame_cvs[0].shape
    return single_frame_cvs[0].new_empty(B, 1, H, W, dtype=torch.float32)


@torch.library.custom_op("monorec_b200::depth_module", mutates_args=(), device_types="cuda")
def depth_module(keyframe: Tensor, cost_volume: Tensor, image_features: List[Tensor], cv_mask: Optional[Tensor],
                 out_a: float, out_b: float, params: List[Tensor], depth_steps: int,
                 feature_channels: List[int]) -> List[Tensor]:
    return _run_bound("DepthModule", (depth_steps, tuple(feature_channels)), params,
                      lambda m: m._run(keyframe, cost_volume, image_features, cv_mask, (out_a, out_b)))


@depth_module.register_fake
def _(keyframe, cost_volume, image_features, cv_mask, out_a, out_b, params, depth_steps, feature_channels):
    B, _, H, W = cost_volume.shape
    half = lambda n: -(-n // 2)    # noqa: E731  (stride-2 same-padded encoder levels)
    hs, ws = [H], [W]
    for _ in range(4):
        hs.append(half(hs[-1]))
        ws.append(half(ws[-1]))
    # heads at the outputs of the four Refine layers (x2 of encoder levels 1..4), finest first
    return [cost_volume.new_empty(B, 1, 2 * hs[i], 2 * ws[i], dtype=torch.float32) for i in range(1, 5)]


# ---- element-wise --------------------------------------------------------------------------------------------------
mask_volume = torch.library.custom_op("monorec_b200::mask_volume", C.mask_volume_impl, mutates_args=(),
                                      device_types="cuda")


@mask_volume.register_fake
def _(volume, mask):
    return torch.empty(volume.shape, device=volume.device, dtype=volume.dtype)


# ---- evaluation ----------------------------------------------------------------------------------------------------
sparse_metrics = torch.library.custom_op("monorec_b200::sparse_metrics", MT.sparse_metrics_impl, mutates_args=(),
                                         device_types="cuda")


@sparse_metrics.register_fake
def _(pred, gt, mvobj_mask, roi, max_distance, pred_all_valid):
    return pred.new_empty(7, dtype=torch.float32)


dense_metrics = torch.library.custom_op("monorec_b200::dense_metrics", MT.dense_metrics_impl, mutates_args=(),
                                        device_types="cuda")


@dense_metrics.register_fake
def _(pred, gt, roi, min_inv):
    return pred.new_empty(len(MT.DENSE_NAMES), dtype=torch.float32)


median_scaling = torch.library.custom_op("monorec_b200::median_scaling", MT.median_scaling_impl, mutates_args=(),
                                         device_types="cuda")


@median_scaling.register_fake
def _(pred, gt):
    return torch.empty(pred.shape, device=pred.device, dtype=pred.dtype)


# ---- reprojection loss ---------------------------------------------------------------------------------------------
@torch.library.custom_op("monorec_b200::reprojection_loss_fwd", mutates_args=(), device_types="cuda")
def reprojection_loss_fwd(depth_prediction: Tensor, keyframe: Tensor, frames: List[Tensor], keyframe_pose: Tensor,
                          keyframe_intrinsics: Tensor, poses: List[Tensor], intrinsics: List[Tensor], automasking: bool,
                          border: int) -> Tuple[Tensor, Tensor, Tensor]:
    """-> (errors [B,H,W], winner [B,H,W] int32, projection tables [B,F,12]) on fp32 contiguous inputs."""
    proj = L.projection(keyframe, keyframe_pose, keyframe_intrinsics, poses, intrinsics)
    invd = depth_prediction.detach().to(torch.float32).contiguous()
    errors, winner = L.errors_fwd(keyframe, frames, proj, invd, automasking, border)
    return errors, winner, proj


@reprojection_loss_fwd.register_fake
def _(depth_prediction, keyframe, frames, keyframe_pose, keyframe_intrinsics, poses, intrinsics, automasking, border):
    B, _, H, W = keyframe.shape
    return (keyframe.new_empty(B, H, W), keyframe.new_empty(B, H, W, dtype=torch.int32),
            keyframe.new_empty(B, len(frames), 12))


@torch.library.custom_op("monorec_b200::reprojection_loss_bwd", mutates_args=(), device_types="cuda")
def reprojection_loss_bwd(keyframe: Tensor, frames: List[Tensor], proj: Tensor, depth_prediction: Tensor,
                          grad_errors: Tensor, winner: Tensor) -> Tensor:
    """-> the gradient [B,1,H,W] w.r.t. depth_prediction, in its dtype."""
    invd = depth_prediction.detach().to(torch.float32).contiguous()
    return L.errors_bwd(keyframe, frames, proj, invd, grad_errors, winner).to(depth_prediction.dtype)


@reprojection_loss_bwd.register_fake
def _(keyframe, frames, proj, depth_prediction, grad_errors, winner):
    B, _, H, W = keyframe.shape
    return depth_prediction.new_empty(B, 1, H, W)


def _loss_setup_context(ctx, inputs, output):
    depth_prediction, keyframe, frames, _, _, poses, intrinsics = inputs[:7]
    _, winner, proj = output
    ctx.list_sizes = (len(frames), len(poses), len(intrinsics))
    ctx.save_for_backward(depth_prediction, keyframe, proj, winner, *frames)
    ctx.mark_non_differentiable(winner, proj)


def _loss_backward(ctx, grad_errors, _grad_winner, _grad_proj):
    depth_prediction, keyframe, proj, winner, *frames = ctx.saved_tensors
    g = reprojection_loss_bwd(keyframe, frames, proj, depth_prediction, grad_errors, winner)
    nf, npose, nk = ctx.list_sizes
    return g, None, [None] * nf, None, None, [None] * npose, [None] * nk, None, None


torch.library.register_autograd("monorec_b200::reprojection_loss_fwd", _loss_backward, setup_context=_loss_setup_context)


# ---- residual image ------------------------------------------------------------------------------------------------
residual_image = torch.library.custom_op("monorec_b200::residual_image", LY.residual_image_impl, mutates_args=(),
                                         device_types="cuda")


@residual_image.register_fake
def _(keyframe, frames, keyframe_pose, keyframe_intrinsics, poses, intrinsics, inv_depth, inv_depth_range):
    B, _, H, W = keyframe.shape
    return keyframe.new_empty(B, 1, H, W, dtype=torch.float32)


OPS = {"cost_volume": cost_volume, "resnet_trunk": resnet_trunk, "mask_module": mask_module,
       "depth_module": depth_module, "mask_volume": mask_volume, "sparse_metrics": sparse_metrics,
       "dense_metrics": dense_metrics, "median_scaling": median_scaling, "reprojection_loss_fwd": reprojection_loss_fwd,
       "reprojection_loss_bwd": reprojection_loss_bwd, "residual_image": residual_image}
