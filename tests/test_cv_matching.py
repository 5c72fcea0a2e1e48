"""The cost volume's non-default error modes (use_ssim 2 and other truthy values) and the uncentred fused volume
(not_center_cv), monorec_model.py:227-243, :267-269.

CPU: the oracle restatements against the reference's outputs (tests/golden/cv_matching.npz), the use_ssim mapping and the
C ABI's argument checks.  GPU: the golden cases, the properties of every mode on both march paths, equality of the new entry
with the existing ones for the default mode, the uncentred volume, and the full model with use_ssim=2.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import cost_volume_oracle as O
from tests import cv_cases as CC
from tests.helpers import GOLDEN, compare_volumes

gpu = pytest.mark.gpu
DEV = "cuda"
MODES = {"ssim": 1, "ssim_l1": 2, "box_l1": 3}


def _golden():
    return np.load(GOLDEN / "cv_matching.npz")


def _depths(data, z, D):
    B, _, H, W = data["keyframe"].shape
    return CC.broadcast_planes(B, D, H, W) if z is None else z


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", list(CC.MATCHING_CASES))
def test_torch_restatement_matches_reference(tag):
    g = _golden()
    data, z, D, use_ssim, not_center = CC.make_matching_case(tag)
    cv, sf = O.cost_volume_torch(data, cv_depths=_depths(data, z, D), use_ssim=use_ssim, not_center_cv=not_center)
    # the single-frame volumes at the tolerance of tests/test_oracle_golden.py; the fused volume at the north-star 1e-3, as
    # in tests/test_cv_pixel_depths.py (view weights of flat-cost pixels are differences of nearly equal numbers)
    assert (cv - torch.from_numpy(g[f"{tag}_cv"])).abs().max().item() <= 1e-3
    for a, r in zip(sf, g[f"{tag}_sf"]):
        assert (a - torch.from_numpy(r)).abs().max().item() <= 5e-5


@pytest.mark.parametrize("tag", list(CC.MATCHING_CASES))
def test_closed_form_matches_reference(tag):
    g = _golden()
    data, z, D, use_ssim, not_center = CC.make_matching_case(tag)
    cv, sf, _, _ = O.cost_volume_closed_form(data, cv_depths=_depths(data, z, D), use_ssim=use_ssim,
                                             not_center_cv=not_center, dtype=np.float64)
    stats = compare_volumes(torch.from_numpy(cv).float(), [torch.from_numpy(s).float() for s in sf],
                            torch.from_numpy(g[f"{tag}_cv"]), [torch.from_numpy(s) for s in g[f"{tag}_sf"]])
    print(tag, stats)


def test_use_ssim_mapping():
    from monorec_b200.cost_volume import CV_BOX_L1, CV_SSIM, CV_SSIM_L1, CostVolumeModule, cv_matching_mode
    assert (CV_SSIM, CV_SSIM_L1, CV_BOX_L1) == (1, 2, 3)
    for v, mode in ((True, CV_SSIM), (1, CV_SSIM), (1.0, CV_SSIM), (2, CV_SSIM_L1), (2.0, CV_SSIM_L1), (3, CV_BOX_L1),
                    (0.5, CV_BOX_L1), ("sad", CV_BOX_L1)):
        assert cv_matching_mode(v) == mode, v
        assert CostVolumeModule(use_ssim=v).matching == mode, v
    for v in (False, 0, 0.0, None, ""):
        with pytest.raises(NotImplementedError):
            cv_matching_mode(v)
        with pytest.raises(NotImplementedError):
            CostVolumeModule(use_ssim=v)
    assert CostVolumeModule(not_center_cv=True).not_center_cv
    from monorec_b200.model import MonoRecModel
    assert MonoRecModel(use_ssim=2).cv_module.matching == CV_SSIM_L1


def test_matching_entry_validation_without_gpu():
    """Bad arguments of mr_cost_volume_fwd_matching give MR_EINVAL (or MR_ENOSUPPORT for the plain L1 difference) and a
    message naming the field, before any CUDA call (fake, never dereferenced, 16-byte-aligned pointers)."""
    from monorec_b200 import _lib
    lib = _lib.load()
    frames = (ctypes.c_void_p * 8)(*[0x7F0000400000 + 0x100000 * i for i in range(8)])
    key, proj, z, pz, cv, sf, nhwc = (0x7F0000100000, 0x7F0000200000, 0x7F0000300000, 0x7F0000380000, 0x7F0001000000,
                                      0x7F0002000000, 0x7F0003000000)

    def call(depths=z, pixel=None, nhwc=None, nhwc_dtype=0, F=2, D=32, matching=2, centered=1):
        rc = lib.mr_cost_volume_fwd_matching(key, frames, proj, depths, pixel, cv, sf, nhwc, nhwc_dtype, 1, F, D, 64, 64, 10.0,
                                             None, matching, centered, None)
        return rc, lib.mr_last_error().decode()

    rc, msg = call(matching=0)
    assert rc == -2 and "matching" in msg, (rc, msg)
    for kw, text in ((dict(matching=4), "matching"), (dict(matching=-1), "matching"), (dict(centered=2), "centered"),
                     (dict(pixel=pz), "pixel_depths"), (dict(depths=None), "pixel_depths"),
                     (dict(depths=None, pixel=pz + 2), "pixel_depths"), (dict(D=1), "D="), (dict(D=129), "D="),
                     (dict(F=0), "F="), (dict(F=9), "F="), (dict(nhwc=nhwc, nhwc_dtype=2), "nhwc_dtype"),
                     (dict(nhwc_dtype=-1), "nhwc_dtype")):
        rc, msg = call(**kw)
        assert rc == -1 and text in msg, (kw, rc, msg)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _to(data):
    from monorec_b200.synthetic import to_device
    return to_device(data, DEV)


def _module_run(data, D, z=None, nhwc=None, **kw):
    from monorec_b200.cost_volume import CostVolumeModule
    d = CC.with_plane_range(data, D)
    if z is not None:
        d["cv_depths"] = z
    if nhwc is not None:
        d["_sfcv_nhwc"] = nhwc
    out = CostVolumeModule(**kw)(d)
    torch.cuda.synchronize()
    return out


def _unaligned(t):
    """The same values in a view whose base is 4 bytes past a 16-byte boundary: TMA cannot address it, so the kernel
    gathers every tap from global memory (the rule of launch_cost_volume)."""
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


class _Abi:
    """Direct calls of mr_cost_volume_fwd_matching (and of the existing entries) on one input dict."""

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

    def outputs(self, nhwc_dtype=None):
        cv = torch.full((self.B, self.D, self.H, self.W), float("nan"), device=DEV)
        sf = torch.full((self.F, self.B, self.D, self.H, self.W), float("nan"), device=DEV)
        nh = None
        if nhwc_dtype is not None:
            nh = torch.full((self.F * self.B, self.H, self.W, self.D), float("nan"), device=DEV, dtype=nhwc_dtype)
        return cv, sf, nh

    def run(self, matching, centered=1, z=None, nhwc_dtype=None, frames=None):
        cv, sf, nh = self.outputs(nhwc_dtype)
        z = None if z is None else z.contiguous()
        rc = self.lib.mr_cost_volume_fwd_matching(
            self.key.data_ptr(), self.L.ptr_array(frames or self.data["frames"]), self.proj.data_ptr(),
            self.planes.data_ptr() if z is None else None, None if z is None else z.data_ptr(), cv.data_ptr(), sf.data_ptr(),
            None if nh is None else nh.data_ptr(), int(nh is not None and nh.dtype == torch.float16), self.B, self.F, self.D,
            self.H, self.W, 10.0, None, matching, centered, self.stream)
        self.L.check(rc, "mr_cost_volume_fwd_matching")
        torch.cuda.synchronize()
        return cv, sf, nh

    def broadcast(self):
        return self.planes.view(1, self.D, 1, 1).expand(self.B, self.D, self.H, self.W)


@gpu
@pytest.mark.parametrize("tag", list(CC.MATCHING_CASES))
def test_golden_cases(tag):
    g = _golden()
    data, z, D, use_ssim, not_center = CC.make_matching_case(tag)
    out = _module_run(_to(data), D, None if z is None else z.to(DEV), use_ssim=use_ssim, not_center_cv=not_center)
    stats = compare_volumes(out["cost_volume"].cpu(), [s.cpu() for s in out["single_frame_cvs"]],
                            torch.from_numpy(g[f"{tag}_cv"]), [torch.from_numpy(s) for s in g[f"{tag}_sf"]])
    print(tag, stats)


@gpu
@pytest.mark.parametrize("gain_tag,gain", [("g1", 1.0), ("g07", 0.7)])
def test_golden_model(gain_tag, gain):
    """MonoRecModel(use_ssim=2) vs the reference, at the fp32-mode gate of the existing model goldens."""
    from monorec_b200 import conv as C
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import make_inputs, seeded_state_dict
    g = _golden()
    noise = np.load(GOLDEN / "model_fp64.npz")[f"synth_{gain_tag}_noise"]
    B, nF, H, W, seed = CC.MATCHING_MODEL_CASE
    model = MonoRecModel(use_ssim=2)
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=gain))
    model = model.to(DEV).eval()
    old = C.MODE
    C.set_mode("fp32")
    try:
        out = model(_to(make_inputs(B, nF, H, W, seed=seed)))
        torch.cuda.synchronize()
    finally:
        C.set_mode(old)
    tol = max(1e-4, 4 * max(float(noise[0]), float(noise[1])))
    dm = np.abs(out["cv_mask"].cpu().numpy() - g[f"model_{gain_tag}_cv_mask"]).max()
    dd = [np.abs(p.cpu().numpy() - g[f"model_{gain_tag}_depth{i}"]).max()
          for i, p in enumerate(out["predicted_inverse_depths"]) if f"model_{gain_tag}_depth{i}" in g]
    assert len(dd) >= 3
    print(gain_tag, "mask max|d|", dm, "depth max|d|", dd, "tol", tol)
    assert dm < tol and max(dd) < tol


@gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("centered", [1, 0])
def test_mode_properties(mode, centered):
    """Per error mode and centring: TMA windows and the global gather agree, broadcast per-pixel depths reproduce the plane
    path bit for bit, the 2-px ring is exactly 0, batch elements are independent and frames permute exactly."""
    from monorec_b200.synthetic import make_inputs
    m = MODES[mode]
    B, F, D, H, W = 2, 3, 32, 96, 200
    data = _to(make_inputs(B, F, H, W, seed=71))
    abi = _Abi(data, D)
    cv, sf, _ = abi.run(m, centered)
    assert torch.isfinite(cv).all() and torch.isfinite(sf).all()
    # the gather path, forced by unaligned frame views
    cvg, sfg, _ = abi.run(m, centered, frames=[_unaligned(f) for f in data["frames"]])
    assert (cv - cvg).abs().max().item() <= 5e-5 and (sf - sfg).abs().max().item() <= 5e-5, mode
    # per-pixel depths that repeat the planes
    cvb, sfb, _ = abi.run(m, centered, z=abi.broadcast())
    assert torch.equal(cv, cvb) and torch.equal(sf, sfb), mode
    # a band of per-pixel depths on the TMA windows and on the gather (the per-pixel march of every mode, both paths)
    z = CC.band_depths(B, D, H, W, seed=78, rel=1.1).to(DEV)
    cvz, sfz, _ = abi.run(m, centered, z=z)
    cvzg, sfzg, _ = abi.run(m, centered, z=z, frames=[_unaligned(f) for f in data["frames"]])
    assert torch.isfinite(cvz).all() and (sfz != 0).any()
    assert (cvz - cvzg).abs().max().item() <= 5e-5 and (sfz - sfzg).abs().max().item() <= 5e-5, mode
    # ring
    for t in (cv, sf):
        assert t[..., :2, :].abs().max() == 0 and t[..., -2:, :].abs().max() == 0
        assert t[..., :2].abs().max() == 0 and t[..., -2:].abs().max() == 0
    # batch independence: a changed second element leaves the first one's bits alone
    d2 = dict(data)
    d2["keyframe"] = data["keyframe"].clone()
    d2["keyframe"][1] = d2["keyframe"][1].flip(-1)
    cv2, sf2, _ = _Abi(d2, D).run(m, centered)
    assert torch.equal(cv[0], cv2[0]) and torch.equal(sf[:, 0], sf2[:, 0])
    assert not torch.equal(cv[1], cv2[1])
    # frame permutation: the single-frame volumes permute exactly, the fused volume up to the summation order
    perm = [2, 0, 1]
    dp = dict(data)
    for k in ("frames", "poses", "intrinsics"):
        dp[k] = [data[k][i] for i in perm]
    cvp, sfp, _ = _Abi(dp, D).run(m, centered)
    assert torch.equal(sfp, sf[perm])
    assert (cvp - cv).abs().max().item() <= 1e-5


@gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_nhwc_copy(mode, dtype):
    """The MaskModule's NHWC copy equals the permuted single-frame volumes in every mode, on both depth sources."""
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 2, 2, 32, 64, 128
    abi = _Abi(_to(make_inputs(B, F, H, W, seed=72)), D)
    for z in (None, CC.band_depths(B, D, H, W, seed=73).to(DEV)):
        cv, sf, nh = abi.run(MODES[mode], 1, z=z, nhwc_dtype=dtype)
        ref = torch.cat([sf[f].permute(0, 2, 3, 1) for f in range(F)], 0).to(dtype)
        assert torch.equal(nh, ref), mode


@gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_tall_image_on_both_paths(mode):
    """H = 16k + 3 (a last tile of 3 rows) on the TMA windows and on the gather."""
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 1, 2, 16, 16 * 5 + 3, 128
    data = _to(make_inputs(B, F, H, W, seed=74))
    abi = _Abi(data, D)
    cv, sf, _ = abi.run(MODES[mode])
    cvg, sfg, _ = abi.run(MODES[mode], frames=[_unaligned(f) for f in data["frames"]])
    assert torch.isfinite(cv).all() and torch.isfinite(sf).all()
    assert (sf[..., H - 3:H - 2, 2:W - 2] != 0).any()
    assert (cv - cvg).abs().max().item() <= 5e-5 and (sf - sfg).abs().max().item() <= 5e-5


@gpu
def test_ssim_centred_equals_existing_entries():
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 2, 3, 32, 96, 200
    abi = _Abi(_to(make_inputs(B, F, H, W, seed=75)), D)
    cv, sf, _ = abi.run(1, 1)
    cv0, sf0, _ = abi.outputs()
    abi.L.check(abi.lib.mr_cost_volume_fwd(abi.key.data_ptr(), abi.L.ptr_array(abi.data["frames"]), abi.proj.data_ptr(),
                                           abi.planes.data_ptr(), cv0.data_ptr(), sf0.data_ptr(), B, F, D, H, W, 10.0, None,
                                           abi.stream), "mr_cost_volume_fwd")
    torch.cuda.synchronize()
    assert torch.equal(cv, cv0) and torch.equal(sf, sf0)
    z = CC.band_depths(B, D, H, W, seed=76).to(DEV)
    cv, sf, _ = abi.run(1, 1, z=z)
    cv1, sf1, _ = abi.outputs()
    abi.L.check(abi.lib.mr_cost_volume_fwd_depthmap(abi.key.data_ptr(), abi.L.ptr_array(abi.data["frames"]),
                                                    abi.proj.data_ptr(), z.data_ptr(), cv1.data_ptr(), sf1.data_ptr(), None,
                                                    0, B, F, D, H, W, 10.0, None, abi.stream), "mr_cost_volume_fwd_depthmap")
    torch.cuda.synchronize()
    assert torch.equal(cv, cv1) and torch.equal(sf, sf1)


@gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_uncentred_volume(mode):
    """not_center_cv: sum_f w_f sad_f / sum_f w_f == (1 - centred) / 2, and exactly 0 where the centred volume is 0 because
    sum_f w_f == 0 (invalid pixels and flat costs); the single-frame volumes do not change."""
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 1, 2, 32, 64, 128
    data = _to(make_inputs(B, F, H, W, seed=77))
    data["frames"][1] = torch.zeros_like(data["frames"][1])     # flat costs: zero view weight for frame 1
    abi = _Abi(data, D)
    cv, sf, _ = abi.run(MODES[mode], 1)
    cvu, sfu, _ = abi.run(MODES[mode], 0)
    assert torch.equal(sf, sfu)
    zero = (cv == 0).all(1, keepdim=True).expand_as(cv)
    assert zero.any() and (~zero).any()
    assert (cvu[zero] == 0).all()
    assert ((cvu - (1 - cv) / 2).abs() * ~zero).max().item() <= 1e-6
