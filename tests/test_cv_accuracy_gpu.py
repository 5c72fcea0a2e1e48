"""The fused cost-volume kernel against the float64 closed form (oracle.cost_volume_closed_form), at the accuracy the kernel
actually has rather than at the north-star 1e-3.  Needs an H100.

The closed form is fed the device's own fp32 depths (the plane table of mr_projection_tables as a broadcast `cv_depths`, or
the per-pixel depths themselves), so the comparison measures the kernel's arithmetic and nothing else.  The cases reach the
kernel's distinct paths: TMA windows and the global gather, a one-column last tile, a last 16-row tile with one valid row,
plane groups below kMinGroup, partial and several kChunk groups of the per-pixel phase, F = 1 and F = MR_MAX_FRAMES, every
error mode and centring, per-pixel depths, and depths behind a source camera (whose mirrored projections the reference
samples like any other).

Gates (per case):
* single-frame volumes, where the kernel and the closed form agree on validity: max |d| <= 2e-4, RMS <= 1.5e-5, and the RMS
  of every output row and column holding >= 256 compared values (over B, F, D and the other axis) <= 3e-5.  The row and
  column gate is what finds an error confined to a tile seam, which hardly moves the global RMS;
* validity (a plane stack that is exactly 0): the two sides may disagree only where the float64 sample lies within 2e-3 px
  of the edge of the validity region (oracle.validity_margin), with no count allowance.  The kernel projects in fp32, so
  its sample positions are some 1e-4 px from the float64 ones;
* fused volume, on pixels where every valid frame's view weight is >= 0.05: the single-frame gates.  Smaller weights are
  differences of nearly equal numbers (1 - (sum - 1) / (D - 1) with the sum close to D) whose rounding is amplified by 1 / w,
  so on the other valid pixels the fused value only has to be a weighted mean: inside [min, max] of the valid frames'
  float64 values, +- 2e-4;
* the fused volume may be exactly 0 on one side only where the float64 sum of the view weights is < 1e-5 or a frame's
  validity flips.

Each case prints its figures (max, RMS, worst row / column RMS, flips and their largest |margin|).
"""
import numpy as np
import pytest
import torch

from oracle import cost_volume_oracle as O
from tests import cv_cases as CC

pytestmark = pytest.mark.gpu
DEV = "cuda"

MAX, RMS, LINE_RMS, LINE_MIN = 2e-4, 1.5e-5, 3e-5, 256
FLIP_MARGIN_PX, STABLE_WEIGHT, MEAN_SLACK, ZERO_WSUM = 2e-3, 0.05, 2e-4, 1e-5
USE_SSIM = {1: True, 2: 2, 3: 3}    # MR_CV_* -> the reference's use_ssim

# tag -> (entry, B, F, D, H, W, image seed, matching (MR_CV_*), centred, depths)
#   entry: the C entry point; depths: "planes" (the plane table) or a per-pixel builder of tests/cv_cases.py
CASES = {
    # TMA windows at the two measured shapes; D x F = 384 halves the tile height
    "planes_f4_d32": ("fwd", 1, 4, 32, 256, 512, 100, 1, 1, "planes"),
    "planes_f6_d64": ("fwd", 1, 6, 64, 256, 512, 101, 1, 1, "planes"),
    # ragged shapes (those of test_ragged_shapes_against_oracle and test_cost_volume_tiles_gpu.py, plus D = 40)
    "w61": ("fwd", 1, 2, 32, 37, 61, 31, 1, 1, "planes"),          # W = 60 + 1 odd: gather, scalar stores, 1-column tile
    "f1_b2_w333": ("fwd", 2, 1, 8, 48, 333, 32, 1, 1, "planes"),   # F = 1, B = 2, W odd
    "w500": ("fwd", 1, 3, 32, 100, 500, 33, 1, 1, "planes"),       # 9 tile columns, W % 60 = 20
    "d128": ("fwd", 1, 2, 128, 32, 64, 34, 1, 1, "planes"),        # four kChunk groups per pixel
    "d4_f8": ("fwd", 1, 8, 4, 24, 70, 35, 1, 1, "planes"),         # D < kMinGroup (global gather), F = MR_MAX_FRAMES
    "h67": ("fwd", 1, 4, 64, 67, 180, 43, 1, 1, "planes"),         # H = 16k + 3 on the TMA windows
    "h51_w123": ("fwd", 2, 3, 16, 51, 123, 44, 1, 1, "planes"),    # H = 16k + 3 on the gather, B = 2
    "d40": ("fwd", 1, 3, 40, 64, 128, 45, 1, 1, "planes"),         # a partial kChunk group
    # the global-gather entry on a shape the TMA windows could take
    "gather": ("gather", 2, 3, 32, 96, 200, 55, 1, 1, "planes"),
    # error modes and centring, on the planes and on a band of per-pixel depths
    "ssim_l1_planes": ("matching", 2, 3, 32, 96, 200, 71, 2, 1, "planes"),
    "ssim_l1_band": ("matching", 2, 3, 32, 96, 200, 72, 2, 1, "band"),
    "box_l1_planes": ("matching", 2, 3, 32, 96, 200, 73, 3, 1, "planes"),
    "box_l1_band": ("matching", 2, 3, 32, 96, 200, 74, 3, 1, "band"),
    "uncentred_planes": ("matching", 2, 3, 32, 96, 200, 75, 1, 0, "planes"),
    "uncentred_band": ("matching", 2, 3, 32, 96, 200, 76, 1, 0, "band"),
    # source cameras ahead of the scene's planes (FORWARD below)
    "behind_planes": ("fwd", 1, 2, 8, 64, 128, 46, 1, 1, "planes"),
    # per-pixel depths (wide: spans of 1 - 400 m whose far ends leave the source images and whose near ends lie behind the
    # fourth source camera, with a partial kChunk group)
    "pix_band": ("depthmap", 1, 4, 32, 256, 512, 100, 1, 1, "band"),
    "pix_shuffled": ("depthmap", 1, 4, 32, 256, 512, 100, 1, 1, "shuffled"),
    "pix_wide": ("depthmap", 1, 4, 40, 256, 512, 100, 1, 1, "wide"),
    "pix_step": ("depthmap", 1, 4, 32, 256, 512, 100, 1, 1, "step"),
}
# tag -> per source frame, metres its camera moves forward along the keyframe's optical axis.  Planes behind a source
# camera project mirrored (the reference divides by z + 1e-7 whatever its sign), and some of those projections land inside
# the image: frame 0 (50 m) has planes on both sides of its camera, frame 1 (1000 m) has all of them behind it.
FORWARD = {"behind_planes": (50.0, 1000.0)}


def _pixel_depths(kind, B, D, H, W):
    if kind == "band":
        return CC.band_depths(B, D, H, W, seed=7, rel=2.0)
    if kind == "shuffled":
        return CC.shuffled_depths(B, D, H, W, seed=8)
    if kind == "wide":
        return CC.wide_depths(B, D, H, W, seed=9)
    return CC.step_depths(B, D, H, W)


def _kernel(data, entry, D, matching, centred, z):
    """One launch of `entry` on the device copy of `data`; returns (cv (B,D,H,W), sf (F,B,D,H,W), fp32 plane table (D,))."""
    from monorec_b200 import _lib
    from monorec_b200.synthetic import to_device
    lib = _lib.load()
    d = to_device(data, DEV)
    key = d["keyframe"].contiguous()
    B, _, H, W = key.shape
    F = len(d["frames"])
    stream = torch.cuda.current_stream().cuda_stream
    proj = torch.empty(B, F, 3, 4, device=DEV)
    planes = torch.empty(D, device=DEV)
    _lib.check(lib.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                        _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H, W,
                                        proj.data_ptr(), planes.data_ptr(), D, 0.0025, 0.33, stream), "mr_projection_tables")
    cv = torch.full((B, D, H, W), float("nan"), device=DEV)
    sf = torch.full((F, B, D, H, W), float("nan"), device=DEV)
    zd = None if z is None else z.to(DEV).contiguous()
    head = (key.data_ptr(), _lib.ptr_array(d["frames"]), proj.data_ptr())
    if entry in ("fwd", "gather"):
        rc = getattr(lib, "mr_cost_volume_fwd" if entry == "fwd" else "mr_cost_volume_fwd_gather")(
            *head, planes.data_ptr(), cv.data_ptr(), sf.data_ptr(), B, F, D, H, W, O.ALPHA, None, stream)
    elif entry == "depthmap":
        rc = lib.mr_cost_volume_fwd_depthmap(*head, zd.data_ptr(), cv.data_ptr(), sf.data_ptr(), None, 0, B, F, D, H, W,
                                             O.ALPHA, None, stream)
    else:
        rc = lib.mr_cost_volume_fwd_matching(*head, planes.data_ptr() if zd is None else None,
                                             None if zd is None else zd.data_ptr(), cv.data_ptr(), sf.data_ptr(), None, 0,
                                             B, F, D, H, W, O.ALPHA, None, matching, centred, stream)
    _lib.check(rc, entry)
    torch.cuda.synchronize()
    return cv.cpu().numpy(), sf.cpu().numpy(), planes.cpu()


class _Case:
    """A case's inputs, the kernel's volumes and the float64 reference (closed form, view weights, validity margin)."""

    def __init__(self, tag):
        from monorec_b200.synthetic import make_inputs
        entry, B, F, D, H, W, seed, matching, centred, depths = CASES[tag]
        self.tag, self.centred = tag, bool(centred)
        data = make_inputs(B, F, H, W, seed=seed)
        if tag in FORWARD:
            data["poses"] = [data["keyframe_pose"].clone() for _ in range(F)]
            for p, tz in zip(data["poses"], FORWARD[tag]):
                p[:, 2, 3] += tz
        z = None if depths == "planes" else _pixel_depths(depths, B, D, H, W)
        self.cv, self.sf, planes = _kernel(data, entry, D, matching, centred, z)
        if z is None:                       # the device's fp32 planes, as the closed form's per-pixel depths
            z = planes.view(1, D, 1, 1).expand(B, D, H, W)
        ref_cv, ref_sf, self.valid, sad = O.cost_volume_closed_form(
            data, cv_depths=z, dtype=np.float64, use_ssim=USE_SSIM[matching], not_center_cv=not centred)
        self.ref_cv, self.ref_sf, self.sad = ref_cv, np.stack(ref_sf), sad
        self.margin = O.validity_margin(data, cv_depths=z)
        # view weights monorec_model.py:257-260, in float64 from the closed form's own sad and validity
        spread = np.exp(-O.ALPHA * (sad - sad.min(axis=2, keepdims=True)) ** 2).sum(axis=2)
        self.w = (1 - (spread - 1) / (D - 1)) * self.valid                 # (B,F,H,W)
        kvalid = ~(self.sf == 0).all(axis=2)                               # (F,B,H,W)
        self.kvalid = np.moveaxis(kvalid, 0, 1)                            # (B,F,H,W)
        self.flip = self.kvalid != self.valid


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    """Each case built once (the float64 closed form at 256x512 takes tens of seconds); pytest runs both tests of a case
    before it builds the next one."""
    return _Case(request.param)


def _error_stats(d, mask):
    """d: float64 differences (..., H, W) with the compared values `mask` (same shape).  Returns max, RMS, and the worst RMS
    over the output rows and over the output columns holding >= LINE_MIN compared values (0 where none does)."""
    n = int(mask.sum())
    if n == 0:
        return dict(n=0, max=0.0, rms=0.0, row=0.0, col=0.0)
    sq = np.where(mask, d * d, 0.0)
    axes = tuple(range(d.ndim - 2))
    out = dict(n=n, max=float(np.abs(np.where(mask, d, 0.0)).max()), rms=float(np.sqrt(sq.sum() / n)))
    for name, keep in (("row", -2), ("col", -1)):
        other = -1 if keep == -2 else -2
        s = sq.sum(axis=axes).sum(axis=other)
        c = mask.sum(axis=axes).sum(axis=other)
        sel = c >= LINE_MIN
        out[name] = float(np.sqrt(s[sel] / c[sel]).max()) if sel.any() else 0.0
        out[name + "_at"] = int(np.flatnonzero(sel)[np.argmax(np.sqrt(s[sel] / c[sel]))]) if sel.any() else -1
    return out


def _fmt(s):
    return (f"n {s['n']} max {s['max']:.2e} rms {s['rms']:.2e} worst row {s['row']:.2e} (#{s.get('row_at', -1)}) "
            f"worst col {s['col']:.2e} (#{s.get('col_at', -1)})")


def _check(s, what):
    assert s["max"] <= MAX, f"{what}: max |d| = {s['max']:.3e} > {MAX}"
    assert s["rms"] <= RMS, f"{what}: RMS = {s['rms']:.3e} > {RMS}"
    assert s["row"] <= LINE_RMS, f"{what}: RMS of output row {s['row_at']} = {s['row']:.3e} > {LINE_RMS}"
    assert s["col"] <= LINE_RMS, f"{what}: RMS of output column {s['col_at']} = {s['col']:.3e} > {LINE_RMS}"


def _flips(c):
    m = np.abs(c.margin[c.flip])
    worst = float(m.max()) if m.size else 0.0
    return int(c.flip.sum()), worst


def test_single_frame_against_float64(case):
    c, tag = case, case.tag
    nflip, worst = _flips(c)
    both = np.moveaxis(c.kvalid & c.valid, 1, 0)[:, :, None]               # (F,B,1,H,W)
    mask = np.broadcast_to(both, c.sf.shape)
    s = _error_stats(c.sf.astype(np.float64) - c.ref_sf, mask)
    print(f"{tag} single-frame: {_fmt(s)}; validity flips {nflip}, largest |margin| {worst:.2e} px")
    assert worst < FLIP_MARGIN_PX, f"{tag}: a validity flip {worst:.3e} px inside the validity region"
    assert s["n"] > 0
    if tag in FORWARD:                      # every source frame has valid pixels that sample planes behind its camera
        assert c.valid.any(axis=(0, 2, 3)).all()
    _check(s, f"{tag} single-frame")


def test_fused_against_float64(case):
    c, tag = case, case.tag
    flip_px = c.flip.any(axis=1)                                           # (B,H,W)
    wsum = c.w.sum(axis=1)
    kz, rz = (c.cv == 0).all(axis=1), (c.ref_cv == 0).all(axis=1)
    # exact zeros: only where the float64 weights (nearly) vanish or a frame's validity flips
    bad_zero = (kz != rz) & ~(wsum < ZERO_WSUM) & ~flip_px
    cmp = ~kz & ~rz & ~flip_px
    wmin = np.where(c.valid, c.w, np.inf).min(axis=1)
    stable = cmp & (wmin >= STABLE_WEIGHT)
    d = c.cv.astype(np.float64) - c.ref_cv
    s = _error_stats(d, np.broadcast_to(stable[:, None], d.shape))
    # the other compared pixels: a weighted mean of the valid frames' float64 values
    vals = np.moveaxis(1 - 2 * c.sad if c.centred else c.sad, 2, 1)       # (B,D,F,H,W)
    v = c.valid[:, None]
    lo = np.where(v, vals, np.inf).min(axis=2)
    hi = np.where(v, vals, -np.inf).max(axis=2)
    other = np.broadcast_to((cmp & ~stable)[:, None], d.shape)
    cvk = c.cv.astype(np.float64)
    outside = np.where(other, np.maximum(lo - cvk, 0) + np.maximum(cvk - hi, 0), 0.0)
    worst_out = float(outside.max()) if outside.size else 0.0
    print(f"{tag} fused (weights >= {STABLE_WEIGHT}): {_fmt(s)}; other pixels {int((cmp & ~stable).sum())}, "
          f"outside the frames' range by {worst_out:.2e}; zero-set disagreements {int((kz != rz).sum())} "
          f"({int(bad_zero.sum())} with weight sum >= {ZERO_WSUM} and no flip)")
    assert not bad_zero.any(), f"{tag}: {int(bad_zero.sum())} fused pixels exactly 0 on one side only"
    assert worst_out <= MEAN_SLACK, f"{tag}: fused value {worst_out:.3e} outside the valid frames' range"
    assert s["n"] > 0
    _check(s, f"{tag} fused")
