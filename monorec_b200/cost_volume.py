"""Host-side mirror of the reference's CostVolumeModule (model/monorec/monorec_model.py:132-284).

Same constructor arguments, same data_dict keys in and out; the arithmetic runs in the fused sm_90a kernel of
libmonorec_b200.so (csrc/cost_volume.cu) through the C ABI.  No torch fallback.
"""
import time
from typing import List, Optional, Tuple

import torch
from torch import Tensor, nn

from . import _lib


# error modes of the kernel (include/monorec_b200.h MR_CV_*): the numbers are the reference's use_ssim values
CV_SSIM, CV_SSIM_L1, CV_BOX_L1 = 1, 2, 3


def cv_matching_mode(use_ssim):
    """The cost volume's difference for the reference's use_ssim, chosen with the reference's own comparisons in its order
    (monorec_model.py:227-243): falsy -> |w - k| (not implemented: NotImplementedError), == True -> SSIM, == 2 -> 0.85 SSIM
    + 0.15 |w - k|, anything else -> the 3x3 box average of |w - k|.  So 1.0 is SSIM, 2.0 is SSIM + L1, and 3, 0.5 or "sad"
    are the box average."""
    if not use_ssim:
        raise NotImplementedError("monorec_b200: use_ssim falsy (the plain |w - k| difference) is not implemented")
    if use_ssim == True:  # noqa: E712  (the reference's comparison: True, 1 and 1.0 all select SSIM)
        return CV_SSIM
    if use_ssim == 2:
        return CV_SSIM_L1
    return CV_BOX_L1


def check_volume_dtype(dtype):
    """The storage type of the cost volumes: torch.float32 or torch.float16; anything else is a ValueError."""
    if dtype is not torch.float32 and dtype is not torch.float16:
        raise ValueError(f"volume_dtype must be torch.float32 or torch.float16, got {dtype!r}")
    return dtype


def _as_f32c(t):
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.to(torch.float32).contiguous()
    return t


def check_channels(keyframe, frames):
    """The images' channel count C: 3, or 1 for grayscale frames (read as their three-channel replicas).  Another C is a
    NotImplementedError; a frame (mono or stereo) whose C differs from the keyframe's a ValueError."""
    C = keyframe.shape[1] if keyframe.dim() == 4 else None
    if C != 3 and C != 1:
        raise NotImplementedError(f"monorec_b200: images [B,3,H,W] or grayscale [B,1,H,W] only, got a keyframe "
                                  f"{tuple(keyframe.shape)}")
    if any(f.dim() != 4 or f.shape[1] != C for f in frames):
        raise ValueError(f"CostVolumeModule: a keyframe with {C} channel(s) and frames {[tuple(f.shape) for f in frames]}: "
                         "the keyframe, the mono frames and the stereo frame must all have 3 channels or all 1")
    return C


def fills_nhwc(nhwc, F, B, D, H, W):
    """Whether the kernel writes the MaskModule's NHWC input [F*B,H,W,D] (fp32 or half) beside the volumes."""
    return nhwc is not None and D <= 32 and D % 8 == 0 and tuple(nhwc.shape) == (F * B, H, W, D) \
        and nhwc.is_contiguous() and nhwc.dtype in (torch.float32, torch.float16)


def launch(keyframe: Tensor, frames: List[Tensor], intrinsics: List[Tensor], poses: List[Tensor], keyframe_pose: Tensor,
           keyframe_intrinsics: Tensor, cv_depths: Optional[Tensor], sfcv_nhwc: Optional[Tensor], lo: float, hi: float,
           steps: int, alpha: float, channel_weights: List[float], matching: int, center: bool,
           half: bool) -> Tuple[Tensor, Tensor]:
    """Projection tables and the fused cost-volume kernel on contiguous fp32 CUDA inputs -> (cost_volume [B,D,H,W],
    single-frame volumes [F,B,D,H,W]), half when `half`.  D is cv_depths.shape[1] with per-pixel hypotheses, else `steps`
    planes uniform in inverse depth over [lo, hi].  `sfcv_nhwc`, when given, must satisfy `fills_nhwc` and is filled with
    the single-frame volumes in the MaskModule's layout.  The keyframe and the frames have C = 3 channels, or C = 1
    (grayscale: the results are those of the frames replicated to three channels, bit for bit); the caller has checked
    that they agree.  CostVolumeModule.forward calls this directly; under torch.compile it is the implementation of the
    `monorec_b200::cost_volume` op (monorec_b200/ops.py)."""
    lib = _lib.load()
    B, C, H, W = keyframe.shape
    F = len(frames)
    D = steps if cv_depths is None else cv_depths.shape[1]
    vdt = torch.float16 if half else torch.float32
    nhwc = sfcv_nhwc
    nhwc_half = 1 if nhwc is not None and nhwc.dtype == torch.float16 else 0
    centre = 1 if center else 0
    dev = keyframe.device
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        proj = torch.empty(B, F, 3, 4, device=dev, dtype=torch.float32)
        depths = torch.empty(D, device=dev, dtype=torch.float32) if cv_depths is None else None
        cv = torch.empty(B, D, H, W, device=dev, dtype=vdt)
        sfcv = torch.empty(F, B, D, H, W, device=dev, dtype=vdt)
        _lib.check(lib.mr_projection_tables(keyframe_pose.data_ptr(), keyframe_intrinsics.data_ptr(), _lib.ptr_array(poses),
                                            _lib.ptr_array(intrinsics), B, F, H, W, proj.data_ptr(),
                                            None if depths is None else depths.data_ptr(), D, lo, hi, stream),
                   "mr_projection_tables")
        cw = (_lib.c_float * 3)(*channel_weights)
        if C == 1:
            # grayscale frames: one entry for every error mode, centring, depth source and storage type
            _lib.check(lib.mr_cost_volume_fwd_channels(
                keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(),
                None if depths is None else depths.data_ptr(), None if cv_depths is None else cv_depths.data_ptr(),
                cv.data_ptr(), sfcv.data_ptr(), nhwc.data_ptr() if nhwc is not None else None, nhwc_half,
                B, F, D, H, W, alpha, cw, matching, centre, 1 if half else 0, 1, stream), "mr_cost_volume_fwd_channels")
        elif half:
            # half volumes: one entry for every error mode, centring and depth source
            _lib.check(lib.mr_cost_volume_fwd_typed(
                keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(),
                None if depths is None else depths.data_ptr(), None if cv_depths is None else cv_depths.data_ptr(),
                cv.data_ptr(), sfcv.data_ptr(), nhwc.data_ptr() if nhwc is not None else None, nhwc_half,
                B, F, D, H, W, alpha, cw, matching, centre, 1, stream), "mr_cost_volume_fwd_typed")
        elif matching != CV_SSIM or not center:
            # the reference's non-default error modes and the uncentred volume, on either depth source
            _lib.check(lib.mr_cost_volume_fwd_matching(
                keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(),
                None if depths is None else depths.data_ptr(), None if cv_depths is None else cv_depths.data_ptr(),
                cv.data_ptr(), sfcv.data_ptr(), nhwc.data_ptr() if nhwc is not None else None, nhwc_half,
                B, F, D, H, W, alpha, cw, matching, centre, stream), "mr_cost_volume_fwd_matching")
        elif cv_depths is not None:
            # (one entry: it chooses TMA windows or the gather itself, like mr_cost_volume_fwd)
            _lib.check(lib.mr_cost_volume_fwd_depthmap(
                keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(), cv_depths.data_ptr(), cv.data_ptr(),
                sfcv.data_ptr(), nhwc.data_ptr() if nhwc is not None else None, nhwc_half, B, F, D, H, W, alpha, cw,
                stream), "mr_cost_volume_fwd_depthmap")
        elif nhwc is not None:
            _lib.check(lib.mr_cost_volume_fwd_nhwc(keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(),
                                                   depths.data_ptr(), cv.data_ptr(), sfcv.data_ptr(), nhwc.data_ptr(),
                                                   nhwc_half, B, F, D, H, W, alpha, cw, stream), "mr_cost_volume_fwd_nhwc")
        else:
            _lib.check(lib.mr_cost_volume_fwd(keyframe.data_ptr(), _lib.ptr_array(frames), proj.data_ptr(), depths.data_ptr(),
                                              cv.data_ptr(), sfcv.data_ptr(), B, F, D, H, W, alpha, cw, stream),
                       "mr_cost_volume_fwd")
    return cv, sfcv


class CostVolumeModule(nn.Module):
    """Drop-in for the reference class of the same name (monorec_model.py:132-148 for the ctor).

    Every shipped config uses use_ssim=True, patch_size=3, sfcv_mult_mask=True, not_center_cv=False (SURVEY.md §8a).
    use_ssim also takes the reference's other truthy values (see cv_matching_mode) and not_center_cv=True stores the
    uncentred fused volume, as the reference does.  use_mono / use_stereo select the frame lists exactly like the reference
    (:160-167).  use_ssim falsy, patch_size != 3 and sfcv_mult_mask=False raise NotImplementedError instead of silently
    running something else.

    volume_dtype (not a reference argument) is the storage type of `cost_volume` and `single_frame_cvs`: torch.float32 (the
    default) or torch.float16, which halves their memory and the bytes the kernel writes.  The arithmetic is fp32 either way:
    each single-frame value is rounded to half where it is stored, and the fused volume is computed in fp32 from the stored
    half single-frame values and rounded once.
    """

    def __init__(self, use_mono=True, use_stereo=False, use_ssim=True, patch_size=3,
                 channel_weights=(5 / 32, 16 / 32, 11 / 32), alpha=10, not_center_cv=False, sfcv_mult_mask=True,
                 volume_dtype=torch.float32):
        super().__init__()
        self.volume_dtype = check_volume_dtype(volume_dtype)
        self.use_mono = use_mono
        self.use_stereo = use_stereo
        self.use_ssim = use_ssim
        self.patch_size = patch_size
        self.border_radius = patch_size // 2 + 1
        self.channel_weights = None if channel_weights is None else tuple(float(c) for c in channel_weights)
        self.alpha = alpha
        self.not_center_cv = not_center_cv
        self.sfcv_mult_mask = sfcv_mult_mask
        self.matching = cv_matching_mode(use_ssim)
        if patch_size != 3 or not sfcv_mult_mask:
            raise NotImplementedError("monorec_b200: only patch_size=3, sfcv_mult_mask=True")

    def _gather(self, data_dict):
        frames, intrinsics, poses = [], [], []
        if self.use_mono:
            frames += list(data_dict["frames"])
            intrinsics += list(data_dict["intrinsics"])
            poses += list(data_dict["poses"])
        if self.use_stereo:
            frames += [data_dict["stereoframe"]]
            intrinsics += [data_dict["stereoframe_intrinsics"]]
            poses += [data_dict["stereoframe_pose"]]
        return frames, intrinsics, poses

    @torch.no_grad()
    def forward(self, data_dict):
        """data_dict["cv_depths"], when present, gives the depth hypotheses per pixel as in the reference (:181-182): a
        (B, D, H, W) tensor on the keyframe's device with 2 <= D <= 128, any order along D.  It replaces the uniform
        inverse-depth planes, and its D is the one of the view weight.  It is read as contiguous fp32: other dtypes and
        expanded or strided views (such as a broadcast of per-plane depths) are materialised first.
        """
        compiling = torch.compiler.is_compiling()
        start_time = None if compiling else time.time()
        keyframe = _as_f32c(data_dict["keyframe"])
        frames, intrinsics, poses = self._gather(data_dict)
        check_channels(keyframe, frames)
        if not keyframe.is_cuda:
            raise _lib.MonorecLibraryError("monorec_b200.CostVolumeModule needs CUDA tensors (no CPU fallback)")
        pixel_depths = None
        if "cv_depths" in data_dict:
            pixel_depths = self._check_cv_depths(data_dict["cv_depths"], keyframe)
        if not compiling:
            _lib.load()
        frames = [_as_f32c(f) for f in frames]
        intrinsics = [_as_f32c(k) for k in intrinsics]
        poses = [_as_f32c(p) for p in poses]
        kpose = _as_f32c(data_dict["keyframe_pose"])
        kK = _as_f32c(data_dict["keyframe_intrinsics"])
        B, C, H, W = keyframe.shape
        F = len(frames)
        if pixel_depths is not None:
            lo, hi, D = 0.0, 0.0, pixel_depths.shape[1]
        else:
            # .item()-free: the ranges are python floats on the model, mirrored into the dict as 1-element tensors
            lo, hi, D = self._plane_range(data_dict)
        # monorec_model.py:174-177 without channel weights
        cw = list(self.channel_weights) if self.channel_weights is not None else [1 / 3, 1 / 3, 1 / 3]
        nhwc = data_dict.get("_sfcv_nhwc")   # MonoRecModel: the MaskModule's input buffer [F*B,H,W,D], filled by the kernel
        fill_nhwc = fills_nhwc(nhwc, F, B, D, H, W)
        run = torch.ops.monorec_b200.cost_volume if compiling else launch
        cv, sfcv = run(keyframe, frames, intrinsics, poses, kpose, kK, pixel_depths, nhwc if fill_nhwc else None,
                       float(lo), float(hi), int(D), float(self.alpha), cw, int(self.matching), not self.not_center_cv,
                       self.volume_dtype == torch.float16)
        if fill_nhwc:
            data_dict["_sfcv_nhwc_filled"] = True
        data_dict["cost_volume"] = cv
        data_dict["single_frame_cvs"] = [sfcv[f] for f in range(F)]
        # host-side issue time (the reference's number includes its device work only because it synchronises implicitly);
        # 0 in a torch.compile / torch.export graph, where no host clock is read
        elapsed = 0.0 if compiling else time.time() - start_time
        data_dict["cv_module_time"] = torch.full((1,), elapsed, device=keyframe.device, dtype=torch.float32)
        return data_dict

    @staticmethod
    def _check_cv_depths(z, keyframe):
        """(B, D, H, W) per-pixel hypotheses as contiguous fp32 on the keyframe's device; ValueError before any launch."""
        B, _, H, W = keyframe.shape
        if not torch.is_tensor(z):
            raise ValueError(f"cv_depths must be a tensor, got {type(z).__name__}")
        if z.device != keyframe.device:
            raise ValueError(f"cv_depths is on {z.device}, the keyframe on {keyframe.device}")
        if z.dim() != 4 or z.shape[0] != B or z.shape[2] != H or z.shape[3] != W:
            raise ValueError(f"cv_depths must be shaped (B, D, H, W) = ({B}, D, {H}, {W}), got {tuple(z.shape)}")
        if not 2 <= z.shape[1] <= 128:
            raise ValueError(f"cv_depths needs 2 <= D <= 128 hypotheses per pixel, got D = {z.shape[1]}")
        if z.is_complex():
            raise ValueError("cv_depths must be real")
        return _as_f32c(z)

    @staticmethod
    def _plane_range(data_dict):
        """(inv_depth_lo, inv_depth_hi, D) from the dict (monorec_model.py:184: names are swapped w.r.t. values).

        The model stores python numbers next to the tensors (keys with a leading underscore) so that no device->host
        synchronisation is needed; a dict that only has the reference's tensors falls back to .item().
        """
        if "_cv_range" in data_dict:
            return data_dict["_cv_range"]
        return (float(data_dict["inv_depth_max"][0].item()), float(data_dict["inv_depth_min"][0].item()),
                int(data_dict["cv_depth_steps"][0].item()))

    def create_mask(self, c, height, width, border_radius, device=None):
        """Kept for API parity (monorec_model.py:282-284); the kernel never materialises this mask."""
        mask = torch.zeros(c, 1, height, width, device=device)
        mask[:, :, border_radius:height - border_radius, border_radius:width - border_radius] = 1
        return mask


from . import ops  # noqa: E402,F401  (registers monorec_b200::cost_volume, which forward calls under torch.compile)
