"""Half-precision cost volumes (volume_dtype=torch.float16, mr_cost_volume_fwd_typed with MR_DT_F16) on the GPU.

The march and the per-pixel phase compute in fp32 either way, so:
  * the half single-frame volumes are the fp32 ones rounded to half, bit for bit, in every error mode and on every path;
  * the half fused volume is the fusion of the widened half single-frame values, evaluated in fp32 and rounded once;
  * the goldens pass the existing volume gates widened by the rounding of the stored value;
  * the full model keeps its reduced-precision gates against the fp32-volume model, eager and graph-replayed.
"""
import numpy as np
import pytest
import torch

from tests import cv_cases as CC
from tests.helpers import GOLDEN, kitti_sample_dict, synth_small_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF_ROUND = 4.9e-4     # the half spacing just below 1 (2^-11): bounds the rounding of a stored value on [-1, 1]
DT = {torch.float32: 0, torch.float16: 1}


def _to(data):
    from monorec_b200.synthetic import to_device
    return to_device(data, DEV)


class _Abi:
    """mr_cost_volume_fwd_typed on one input dict."""

    def __init__(self, data, D):
        from monorec_b200 import _lib
        self.lib, self.L = _lib.load(), _lib
        self.data = data
        self.key = data["keyframe"].contiguous()
        self.B, _, self.H, self.W = self.key.shape
        self.F, self.D = len(data["frames"]), D
        self.proj = torch.empty(self.B, self.F, 3, 4, device=DEV)
        self.planes = torch.empty(D, device=DEV)
        self.stream = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.mr_projection_tables(
            data["keyframe_pose"].data_ptr(), data["keyframe_intrinsics"].data_ptr(), _lib.ptr_array(data["poses"]),
            _lib.ptr_array(data["intrinsics"]), self.B, self.F, self.H, self.W, self.proj.data_ptr(), self.planes.data_ptr(),
            D, 0.0025, 0.33, self.stream), "mr_projection_tables")

    def run(self, dtype, matching=1, centered=1, z=None, nhwc_dtype=None, frames=None):
        cv = torch.full((self.B, self.D, self.H, self.W), float("nan"), device=DEV, dtype=dtype)
        sf = torch.full((self.F, self.B, self.D, self.H, self.W), float("nan"), device=DEV, dtype=dtype)
        nh = None
        if nhwc_dtype is not None:
            nh = torch.full((self.F * self.B, self.H, self.W, self.D), float("nan"), device=DEV, dtype=nhwc_dtype)
        z = None if z is None else z.contiguous()
        self.L.check(self.lib.mr_cost_volume_fwd_typed(
            self.key.data_ptr(), self.L.ptr_array(frames or self.data["frames"]), self.proj.data_ptr(),
            self.planes.data_ptr() if z is None else None, None if z is None else z.data_ptr(), cv.data_ptr(), sf.data_ptr(),
            None if nh is None else nh.data_ptr(), 0 if nh is None else DT[nh.dtype], self.B, self.F, self.D, self.H, self.W,
            10.0, None, matching, centered, DT[dtype], self.stream), "mr_cost_volume_fwd_typed")
        torch.cuda.synchronize()
        return cv, sf, nh

    def run_matching(self, matching, centered, z=None, frames=None):
        """The existing fp32 entry, for the bit-for-bit comparison of the typed entry's fp32 output."""
        cv = torch.empty(self.B, self.D, self.H, self.W, device=DEV)
        sf = torch.empty(self.F, self.B, self.D, self.H, self.W, device=DEV)
        z = None if z is None else z.contiguous()
        self.L.check(self.lib.mr_cost_volume_fwd_matching(
            self.key.data_ptr(), self.L.ptr_array(frames or self.data["frames"]), self.proj.data_ptr(),
            self.planes.data_ptr() if z is None else None, None if z is None else z.data_ptr(), cv.data_ptr(), sf.data_ptr(),
            None, 0, self.B, self.F, self.D, self.H, self.W, 10.0, None, matching, centered, self.stream),
            "mr_cost_volume_fwd_matching")
        torch.cuda.synchronize()
        return cv, sf


def _unaligned(t):
    """The same values in a view 4 bytes past a 16-byte boundary: TMA cannot address it, every tap is gathered."""
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def fuse(sf, centered=True, alpha=10.0):
    """The reference fusion (oracle/cost_volume_oracle.py:160-168, monorec_model.py:251-269) of single-frame volumes
    sf [F,B,D,H,W] in fp32; a frame is invalid at a pixel whose plane stack is exactly 0.  Returns (cv, min weight of the
    valid frames per pixel)."""
    sf = sf.float()
    D = sf.shape[2]
    valid = ~(sf == 0).all(2, keepdim=True)
    sad = (1 - sf) / 2
    spread = torch.exp(-alpha * (sad - sad.min(dim=2, keepdim=True)[0]) ** 2)
    w = (1 - (spread.sum(dim=2, keepdim=True) - 1) / (D - 1)) * valid
    num, den = (sad * w).sum(0), w.sum(0)
    nz = den != 0
    fsad = torch.where(nz, num / torch.where(nz, den, torch.ones_like(den)), torch.zeros_like(num))
    cv = torch.where(nz, 1 - 2 * fsad, torch.zeros_like(fsad)) if centered else fsad
    wmin = torch.where(valid, w, torch.full_like(w, float("inf"))).amin(0)
    return cv, wmin


def half_ulp(x):
    a = x.float().abs()
    e = torch.floor(torch.log2(torch.clamp(a, min=2.0 ** -14)))
    return torch.pow(2.0, e - 10)


# (name, matching, centered, F, D, H, W, per-pixel depths, gather)
CASES = [
    ("ssim", 1, 1, 2, 32, 64, 128, False, False),
    ("ssim_l1", 2, 1, 2, 32, 64, 128, False, False),
    ("box_l1", 3, 1, 2, 32, 64, 128, False, False),
    ("uncentred", 1, 0, 2, 32, 64, 128, False, False),
    ("uncentred_box_l1", 3, 0, 3, 32, 64, 128, False, False),
    ("cv_depths", 1, 1, 2, 32, 64, 128, True, False),
    ("cv_depths_ssim_l1", 2, 1, 2, 32, 64, 128, True, True),
    ("gather_w_odd", 1, 1, 2, 32, 61, 133, False, False),
    ("gather_unaligned", 2, 1, 3, 32, 64, 128, False, True),
    ("f1", 1, 1, 1, 32, 64, 128, False, False),
    ("f6_d64", 1, 1, 6, 64, 64, 192, False, False),
    ("d128", 1, 1, 2, 128, 48, 128, False, False),
    ("d128_cv_depths_uncentred", 3, 0, 2, 128, 48, 128, True, False),
    ("d40", 2, 1, 3, 40, 64, 128, False, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_half_volumes_against_fp32_path(case):
    from monorec_b200.synthetic import make_inputs
    name, m, c, F, D, H, W, pix, gather = case
    B = 2
    data = _to(make_inputs(B, F, H, W, seed=90 + len(name)))
    abi = _Abi(data, D)
    z = None
    if pix:
        z = CC.band_depths(B, D, H, W, seed=91, rel=1.1).to(DEV)
    frames = [_unaligned(f) for f in data["frames"]] if gather else None
    nhwc = torch.float16 if D <= 32 and D % 8 == 0 else None
    cv32, sf32, _ = abi.run(torch.float32, m, c, z=z, frames=frames)
    cvh, sfh, nh = abi.run(torch.float16, m, c, z=z, nhwc_dtype=nhwc, frames=frames)
    # the typed entry's fp32 output is the existing entry's, bit for bit
    cvm, sfm = abi.run_matching(m, c, z=z, frames=frames)
    assert torch.equal(cv32, cvm) and torch.equal(sf32, sfm)
    assert cvh.dtype == torch.float16 and sfh.dtype == torch.float16
    assert torch.isfinite(cvh).all() and torch.isfinite(sfh).all()
    # single-frame volumes: the fp32 path's values rounded to half, bit for bit
    assert torch.equal(sfh, sf32.half()), name
    # the NHWC copy holds the stored half values
    if nh is not None:
        assert torch.equal(nh, torch.cat([sfh[f].permute(0, 2, 3, 1) for f in range(F)], 0)), name
    # fused volume: the reference fusion of the widened half values, in fp32, rounded once.  Where every valid frame's view
    # weight is > 0.05 the two fp32 evaluations (kernel: ex2.approx, Σ w v · (1 / Σ w); oracle: exp, 1 - 2 Σ w sad / Σ w) differ
    # by a few fp32 ulps, so the half results agree to one half ulp plus 1e-5 (the half ulp alone falls below that fp32 noise
    # for values near 0).  Smaller weights are differences of nearly equal numbers (w = 1 - (Σ - 1) / (D - 1)) whose last-bit
    # noise is amplified by 1 / w; there the fused value must still be a weighted mean of the frames' stored values.
    ref, wmin = fuse(sfh, centered=bool(c))
    zh, z32, zr = (cvh == 0).all(1), (cv32 == 0).all(1), (ref == 0).all(1)
    d = (cvh.float() - ref.half().float()).abs()
    ulp = half_ulp(torch.maximum(cvh.float().abs(), ref.abs()))
    nonzero = ~(zh | zr).unsqueeze(1)
    stable = (wmin > 0.05).expand_as(d) & nonzero
    excess = torch.where(stable, d - ulp - 1e-5, torch.zeros_like(d)).max().item()
    vals = sfh.float() if c else (1 - sfh.float()) / 2
    valid = ~(sfh == 0).all(2, keepdim=True)
    lo = torch.where(valid, vals, torch.full_like(vals, float("inf"))).amin(0)
    hi = torch.where(valid, vals, torch.full_like(vals, -float("inf"))).amax(0)
    outside = torch.where(nonzero.expand_as(d), torch.clamp(lo - cvh.float(), min=0) + torch.clamp(cvh.float() - hi, min=0) - ulp,
                          torch.zeros_like(d)).max().item()
    # exact zeros: invalid pixels are 0 as in the fp32 path; Σ w == 0 may move only on flat-cost pixels at the knife edge of
    # Σ_d exp(..) == D (rounding can make nearly equal single-frame values equal, or split them)
    invalid = (sf32 == 0).all(2).all(0)
    assert zh[invalid].all()
    knife = int((zh != z32).sum())
    print(name, "max ulps (stable)", (d / ulp * stable).max().item(), "stable share", stable.float().mean().item(),
          "max|d| (other)", (d * (~stable & nonzero)).max().item(), "zero flips vs fp32", knife, "vs fused oracle",
          int((zh != zr).sum()))
    assert excess <= 0.0, excess
    assert outside <= 0.0, outside
    assert knife <= max(4, zh.numel() // 500) and int((zh != zr).sum()) <= max(4, zh.numel() // 500)
    # arg-max over the planes: the fp32 path's wherever its top1 - top2 margin exceeds 2e-3
    top = torch.topk(cv32, 2, dim=1)[0]
    # (a narrow band of 128 hypotheses has no pixel with such a margin in its uncentred volume: nothing to compare there)
    sel = ((top[:, 0] - top[:, 1]) > 2e-3) & ~zh & ~z32
    assert sel.any() or name == "d128_cv_depths_uncentred"
    assert torch.equal(cvh.float().argmax(1)[sel], cv32.argmax(1)[sel]), name
    # against the fp32 fused volume: the rounding of the inputs and of the output
    both = ~(zh | z32).unsqueeze(1)
    print(name, "half vs fp32 fused max|d|", ((cvh.float() - cv32).abs() * both).max().item())


# ---- goldens of the unmodified reference, at the existing gates widened by the half rounding ---------------------------
def _run_module(data, D=None, z=None, **kw):
    from monorec_b200.cost_volume import CostVolumeModule
    d = _to(data)
    if z is not None:
        d["cv_depths"] = z.to(DEV)
    else:
        d["_cv_range"] = (0.0025, 0.33, D)
    out = CostVolumeModule(volume_dtype=torch.float16, **kw)(d)
    torch.cuda.synchronize()
    cv, sf = out["cost_volume"], out["single_frame_cvs"]
    assert cv.dtype == torch.float16 and all(s.dtype == torch.float16 for s in sf)
    # the single-frame volumes are views of one [F,B,D,H,W] buffer
    assert all(s._base is sf[0]._base and s._base is not None for s in sf)
    assert sf[0]._base.shape == (len(sf),) + tuple(cv.shape)
    return cv.float().cpu(), [s.float().cpu() for s in sf]


def compare_half(cv, sf, ref_cv, ref_sf, tol=1e-3 + HALF_ROUND, max_flip_px_per_frame=4):
    """tests/helpers.compare_volumes with the volume gates widened by the half rounding.  The single-frame volumes are held to
    tol.  The fused volume's view weights are computed from the rounded single-frame values, and a weight near 0 (a difference
    of nearly equal numbers) amplifies that rounding: it is held to tol on 99 % of its values and to 5e-3 everywhere.  Two
    volumes that agree to tol can only disagree on an arg-max whose top1 - top2 margin is below 2 tol: the arg-max gate is
    margin > 3e-3."""
    stats, worst, flips = {}, 0.0, 0
    for a, r in zip(sf, ref_sf):
        za, zr = (a == 0).all(1), (r == 0).all(1)
        fl = int((za != zr).sum())
        assert fl <= max_flip_px_per_frame * a.shape[0], f"{fl} validity flips"
        flips += fl
        worst = max(worst, ((a - r).abs() * ~(za | zr).unsqueeze(1)).max().item())
    assert worst <= tol, f"single-frame volume max|d| = {worst}"
    za, zr = (cv == 0).all(1), (ref_cv == 0).all(1)
    both = ~(za | zr)
    dd = (cv - ref_cv).abs() * both.unsqueeze(1)
    dcv, share = dd.max().item(), (dd <= tol).float().mean().item()
    assert dcv <= 5e-3 and share >= 0.99, f"cost volume max|d| = {dcv}, share within {tol}: {share}"
    top = torch.topk(ref_cv, 2, dim=1)[0]
    sel = both & ((top[:, 0] - top[:, 1]) > 3e-3)
    agree = (cv.argmax(1) == ref_cv.argmax(1))[sel].float().mean().item() if sel.any() else 1.0
    stats.update(sf_max_abs=worst, cv_max_abs=dcv, cv_share_within_tol=share, valid_flips=flips, argmax_agree_gated=agree)
    assert agree == 1.0
    return stats


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_golden_synth_small(tag):
    data, D, ref_cv, ref_sf = synth_small_dict(tag)
    cv, sf = _run_module(data, D)
    print(tag, compare_half(cv, sf, ref_cv, ref_sf))


def test_golden_kitti_sample():
    data, g = kitti_sample_dict()
    cv, sf = _run_module(data, 32)
    sub = (slice(None), slice(None), slice(2, None, 4), slice(1, None, 8))
    print("sub", compare_half(cv[sub], [s[sub] for s in sf], torch.from_numpy(g["cv_sub"]),
                              [torch.from_numpy(v) for v in g["sf_sub"]]))
    rows = (slice(None), slice(None), slice(100, 104))
    print("rows", compare_half(cv[rows], [s[rows] for s in sf], torch.from_numpy(g["cv_rows"]),
                               [torch.from_numpy(v) for v in g["sf_rows"]]))
    H, W = cv.shape[-2:]
    same = cv.argmax(1) == torch.from_numpy(g["argmax"].astype(np.int64))
    margin = torch.from_numpy(g["margin"].astype(np.float32))
    ref_zero = torch.from_numpy(np.unpackbits(g["cv_zero"])[: H * W].reshape(1, H, W).astype(bool))
    both = ~ref_zero & ~(cv == 0).all(1)
    # (a pixel whose view weights are close to 0 amplifies the rounding of its single-frame values, see compare_half: the
    # arg-max above the 3e-3 margin is held on all but 1 in 10^4 pixels)
    agree = same[both & (margin > 3e-3)].float().mean().item()
    print("kitti argmax margin > 3e-3", agree, "raw", same[both].float().mean().item())
    assert agree > 0.9999
    np.testing.assert_allclose(cv.double().sum((2, 3)).numpy(), g["cv_plane_sum"], rtol=0,
                               atol=(1e-4 + HALF_ROUND) * H * W)


@pytest.mark.parametrize("tag", list(CC.MATCHING_CASES))
def test_golden_matching_cases(tag):
    g = np.load(GOLDEN / "cv_matching.npz")
    data, z, D, use_ssim, not_center = CC.make_matching_case(tag)
    if z is None:
        cv, sf = _run_module(CC.with_plane_range(data, D), D, use_ssim=use_ssim, not_center_cv=not_center)
    else:
        cv, sf = _run_module(data, z=z, use_ssim=use_ssim, not_center_cv=not_center)
    print(tag, compare_half(cv, sf, torch.from_numpy(g[f"{tag}_cv"]), [torch.from_numpy(s) for s in g[f"{tag}_sf"]]))


@pytest.mark.parametrize("tag", list(CC.PIXEL_CASES))
def test_golden_pixel_depth_cases(tag):
    g = np.load(GOLDEN / "cv_pixel_depths.npz")
    data, z = CC.make_pixel_case(tag)
    cv, sf = _run_module(data, z=z)
    print(tag, compare_half(cv, sf, torch.from_numpy(g[f"{tag}_cv"]), [torch.from_numpy(s) for s in g[f"{tag}_sf"]]))


# ---- layout helpers of the model on half volumes -------------------------------------------------------------------------
def test_half_volume_layout_and_mask_helpers():
    from monorec_b200 import conv as C
    g = torch.Generator().manual_seed(5)
    for (B, D, H, W) in [(2, 32, 16, 24), (1, 20, 7, 13)]:
        x = (torch.rand(B, D, H, W, generator=g) * 2 - 1).half().to(DEV)
        m = torch.rand(B, 1, H, W, generator=g).to(DEV)
        ref = x.float().permute(0, 2, 3, 1)
        assert torch.equal(C.nchw_to_nhwc(x), ref)
        assert torch.equal(C.nchw_to_nhwc(x, dtype=torch.float16), ref.half())
        # into a channel slice with the (1 - mask) product: fp32 product of the widened value, rounded once
        for dt in (torch.float32, torch.float16):
            buf = torch.zeros(B, H, W, D + 8, device=DEV, dtype=dt)
            C.nchw_to_nhwc(x, out=buf, out_coff=0, one_minus=m)
            assert torch.equal(buf[..., :D], (x.float() * (1.0 - m)).permute(0, 2, 3, 1).to(dt))
            assert float(buf[..., D:].abs().max()) == 0.0
        out = C.mask_volume(x, m)
        assert out.dtype == torch.float16 and torch.equal(out, ((1.0 - m) * x.float()).half())


# ---- the full model ------------------------------------------------------------------------------------------------------
def _kitti_model(volume_dtype):
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import seeded_state_dict
    g = np.load(GOLDEN / "model_kitti_sample.npz")
    model = MonoRecModel(volume_dtype=volume_dtype)
    model.load_state_dict(seeded_state_dict(model, seed=int(g["wseed"][0]), gain=1.0))
    return model.to(DEV).eval()


@pytest.mark.parametrize("mode", ["f16", "tf32"])
def test_model_half_volumes(mode):
    """MonoRecModel(volume_dtype=torch.float16) on the bundled KITTI sample: result / cv_mask within the reduced-precision gates
    of tests/test_convnet_gpu.py against the fp32-volume model in the same mode; eager == CUDA-graph replay bit for bit;
    DataParallel runs it unchanged."""
    from monorec_b200 import conv as C
    from monorec_b200.model import GraphedMonoRec
    data, _ = kitti_sample_dict()
    data = _to(data)
    old = C.MODE
    C.set_mode(mode)
    try:
        with torch.no_grad():
            ref = _kitti_model(torch.float32)(dict(data))
            model = _kitti_model(torch.float16)
            out = model(dict(data))
            res, mask = out["result"].clone(), out["cv_mask"].clone()
            assert out["cost_volume"].dtype == torch.float16
            assert all(s.dtype == torch.float16 for s in out["single_frame_cvs"])
            assert res.dtype == torch.float32 and out["mask"].dtype == torch.float32
            assert ref["cost_volume"].dtype == torch.float32
            gr = GraphedMonoRec(model, data)
            rep = gr(data)
            torch.cuda.synchronize()
            assert torch.equal(rep["result"], res) and torch.equal(rep["cv_mask"], mask)
            dp = torch.nn.DataParallel(model, device_ids=[0])(dict(data))
            torch.cuda.synchronize()
            assert torch.equal(dp["result"], res) and dp["cost_volume"].dtype == torch.float16
    finally:
        C.set_mode(old)
    dr = (res - ref["result"]).abs()
    dm = (mask - ref["cv_mask"]).abs()
    share, mshare = (dr < 1e-3).float().mean().item(), (dm < 5e-3).float().mean().item()
    print(f"{mode}: half vs fp32 volumes: result max|d| {dr.max().item():.3e} share within 1e-3 {share:.5f}, "
          f"mask max|d| {dm.max().item():.3e} share within 5e-3 {mshare:.5f}")
    assert dr.max().item() < 1e-2 and share > 0.9
    assert dm.max().item() < 2e-2 and mshare > 0.99


def test_model_half_volumes_fp32_mode_and_no_cv():
    """fp32 engine mode (the MaskModule widens the half volumes itself) and no_cv (half zero volumes)."""
    from monorec_b200 import conv as C
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import make_inputs, seeded_state_dict
    data = _to(make_inputs(1, 2, 64, 128, seed=95))
    old = C.MODE
    C.set_mode("fp32")
    try:
        with torch.no_grad():
            ref = _kitti_model(torch.float32)(dict(data))
            out = _kitti_model(torch.float16)(dict(data))
            m = MonoRecModel(no_cv=True, volume_dtype=torch.float16)
            m.load_state_dict(seeded_state_dict(m, seed=3, gain=1.0))
            nc = m.to(DEV).eval()(dict(data))
        torch.cuda.synchronize()
    finally:
        C.set_mode(old)
    assert out["cost_volume"].dtype == torch.float16 and nc["cost_volume"].dtype == torch.float16
    assert torch.isfinite(nc["result"]).all()
    dr = (out["result"] - ref["result"]).abs()
    print("fp32 mode: result max|d|", dr.max().item())
    assert dr.max().item() < 1e-2 and (dr < 1e-3).float().mean().item() > 0.9


# ---- host entry ----------------------------------------------------------------------------------------------------------
def test_half_host_entry_matches_device_entry():
    """mr_cost_volume_host_f16 (host buffers, internal copies) == the device entry's half output, bit for bit."""
    from monorec_b200 import _lib
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 3, 2, 32, 64, 128
    data = make_inputs(B, F, H, W, seed=96)
    cv, sf = _run_module(data, D)
    lib = _lib.load()
    ws_bytes = lib.mr_cost_volume_host_f16_workspace(B, F, D, H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    frames = torch.stack(data["frames"]).contiguous().pin_memory()
    poses = torch.stack(data["poses"]).contiguous()
    intr = torch.stack(data["intrinsics"]).contiguous()
    out_cv = torch.empty(B, D, H, W, dtype=torch.float16).pin_memory()
    out_sf = torch.empty(F, B, D, H, W, dtype=torch.float16).pin_memory()
    _lib.check(lib.mr_cost_volume_host_f16(data["keyframe"].contiguous().data_ptr(), frames.data_ptr(),
                                           data["keyframe_pose"].contiguous().data_ptr(),
                                           data["keyframe_intrinsics"].contiguous().data_ptr(), poses.data_ptr(),
                                           intr.data_ptr(), out_cv.data_ptr(), out_sf.data_ptr(), B, F, D, H, W,
                                           0.0025, 0.33, 10.0, ws.data_ptr(), ws_bytes), "mr_cost_volume_host_f16")
    assert torch.equal(out_cv.float(), cv)
    assert all(torch.equal(out_sf[f].float(), sf[f]) for f in range(F))
    # the single-frame volumes left on the device, at the documented offset
    off = lib.mr_cost_volume_host_f16_sfcv_offset(B, F, D, H, W)
    dev_sf = ws[off:off + F * B * D * H * W * 2].view(torch.float16).view(F, B, D, H, W)
    assert torch.equal(dev_sf.cpu(), out_sf)
