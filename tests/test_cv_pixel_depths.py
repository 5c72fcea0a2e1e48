"""Per-pixel depth hypotheses (data_dict["cv_depths"], monorec_model.py:181-201) through the fused cost-volume kernel.

CPU: the oracle restatements against the reference's outputs (tests/golden/cv_pixel_depths.npz) and the C ABI's argument
checks.  GPU: the golden cases, bit-for-bit equality with the plane path for broadcast depths, hypotheses that are not
usable, batch independence, the full model, and the module's input checks.  The per-pixel path against the float64 closed
form, at the kernel's own accuracy, is in tests/test_cv_accuracy_gpu.py.
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


def _golden():
    return np.load(GOLDEN / "cv_pixel_depths.npz")


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", list(CC.PIXEL_CASES))
def test_torch_restatement_matches_reference(tag):
    g = _golden()
    data, z = CC.make_pixel_case(tag)
    cv, sf = O.cost_volume_torch(data, cv_depths=z)
    # same primitives, same order as the reference: the single-frame volumes at the tolerance of tests/test_oracle_golden.py.
    # The fused volume of a band has pixels whose view weights are small differences of nearly equal numbers
    # (1 - (sum - 1) / (D - 1) with sum close to D), where a different summation order of the same terms moves it: by
    # 3.6e-5 on the band case here, by 6e-4 on a +-25 % band.  The fused volume is therefore held to the north-star 1e-3.
    assert (cv - torch.from_numpy(g[f"{tag}_cv"])).abs().max().item() <= 1e-3
    for a, r in zip(sf, g[f"{tag}_sf"]):
        assert (a - torch.from_numpy(r)).abs().max().item() <= 5e-5


@pytest.mark.parametrize("tag", list(CC.PIXEL_CASES))
def test_closed_form_matches_reference(tag):
    g = _golden()
    data, z = CC.make_pixel_case(tag)
    cv, sf, _, _ = O.cost_volume_closed_form(data, cv_depths=z, dtype=np.float64)
    stats = compare_volumes(torch.from_numpy(cv).float(), [torch.from_numpy(s).float() for s in sf],
                            torch.from_numpy(g[f"{tag}_cv"]), [torch.from_numpy(s) for s in g[f"{tag}_sf"]])
    print(tag, stats)


def test_broadcast_planes_are_the_plane_oracle():
    """The default planes as a broadcast depth tensor are the reference's own default (monorec_model.py:184-185)."""
    from monorec_b200.synthetic import make_inputs
    data = make_inputs(1, 2, 24, 40, seed=3)
    z = O.plane_depths(0.33, 0.0025, 8).view(1, 8, 1, 1).expand(1, 8, 24, 40)
    cv, sf = O.cost_volume_torch(data, cv_depths=z)
    ref_cv, ref_sf = O.cost_volume_torch(data, steps=8)
    assert torch.equal(cv, ref_cv) and all(torch.equal(a, b) for a, b in zip(sf, ref_sf))


@pytest.mark.parametrize("not_center_cv", [False, True])
@pytest.mark.parametrize("use_ssim", [True, 2, 3])
def test_broadcast_planes_are_the_plane_oracle_in_every_mode(use_ssim, not_center_cv):
    """The same for every error mode and centring: the depth source and the options are independent in the oracle."""
    from monorec_b200.synthetic import make_inputs
    data = make_inputs(1, 2, 24, 40, seed=3)
    kw = dict(use_ssim=use_ssim, not_center_cv=not_center_cv)
    cv, sf = O.cost_volume_torch(data, cv_depths=CC.broadcast_planes(1, 8, 24, 40), **kw)
    ref_cv, ref_sf = O.cost_volume_torch(data, steps=8, **kw)
    assert torch.equal(cv, ref_cv) and all(torch.equal(a, b) for a, b in zip(sf, ref_sf))


def test_depthmap_validation_without_gpu():
    """Bad arguments of mr_cost_volume_fwd_depthmap give MR_EINVAL and a message naming the field, before any CUDA call
    (fake, never dereferenced, 16-byte-aligned pointers)."""
    from monorec_b200 import _lib
    lib = _lib.load()
    frames = (ctypes.c_void_p * 8)(*[0x7F0000400000 + 0x100000 * i for i in range(8)])
    key, proj, z, cv, sf, nhwc = 0x7F0000100000, 0x7F0000200000, 0x7F0000300000, 0x7F0001000000, 0x7F0002000000, 0x7F0003000000

    def call(z=z, nhwc=None, nhwc_dtype=0, F=2, D=32):
        rc = lib.mr_cost_volume_fwd_depthmap(key, frames, proj, z, cv, sf, nhwc, nhwc_dtype, 1, F, D, 64, 64, 10.0, None, None)
        return rc, lib.mr_last_error().decode()

    for kw, text in ((dict(z=None), "pixel_depths"), (dict(z=z + 2), "pixel_depths"), (dict(D=1), "D="),
                     (dict(D=129), "D="), (dict(nhwc=nhwc, nhwc_dtype=2), "nhwc_dtype"),
                     (dict(nhwc_dtype=-1), "nhwc_dtype"), (dict(F=9), "F="), (dict(F=0), "F=")):
        rc, msg = call(**kw)
        assert rc == -1 and text in msg, (kw, rc, msg)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _to(data):
    from monorec_b200.synthetic import to_device
    return to_device(data, DEV)


def _module_run(data, z, nhwc=None):
    from monorec_b200.cost_volume import CostVolumeModule
    d = dict(data)
    d["cv_depths"] = z
    if nhwc is not None:
        d["_sfcv_nhwc"] = nhwc
    out = CostVolumeModule()(d)
    torch.cuda.synchronize()
    return out


class _Abi:
    """Direct C-ABI calls on one input dict: projection tables, plane depths, and every cost-volume entry point."""

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

    def plane(self, nhwc_dtype=None):
        cv, sf, nh = self.outputs(nhwc_dtype)
        a = (self.key.data_ptr(), self.L.ptr_array(self.data["frames"]), self.proj.data_ptr(), self.planes.data_ptr(),
             cv.data_ptr(), sf.data_ptr())
        if nh is None:
            rc = self.lib.mr_cost_volume_fwd(*a, self.B, self.F, self.D, self.H, self.W, 10.0, None, self.stream)
        else:
            rc = self.lib.mr_cost_volume_fwd_nhwc(*a, nh.data_ptr(), int(nh.dtype == torch.float16), self.B, self.F, self.D,
                                                  self.H, self.W, 10.0, None, self.stream)
        self.L.check(rc, "plane path")
        torch.cuda.synchronize()
        return cv, sf, nh

    def depthmap(self, z, nhwc_dtype=None):
        cv, sf, nh = self.outputs(nhwc_dtype)
        z = z.contiguous()
        rc = self.lib.mr_cost_volume_fwd_depthmap(
            self.key.data_ptr(), self.L.ptr_array(self.data["frames"]), self.proj.data_ptr(), z.data_ptr(), cv.data_ptr(),
            sf.data_ptr(), None if nh is None else nh.data_ptr(), int(nh is not None and nh.dtype == torch.float16), self.B,
            self.F, self.D, self.H, self.W, 10.0, None, self.stream)
        self.L.check(rc, "mr_cost_volume_fwd_depthmap")
        torch.cuda.synchronize()
        return cv, sf, nh

    def broadcast(self):
        return self.planes.view(1, self.D, 1, 1).expand(self.B, self.D, self.H, self.W)


@gpu
@pytest.mark.parametrize("tag", list(CC.PIXEL_CASES))
def test_golden_cases(tag):
    g = _golden()
    data, z = CC.make_pixel_case(tag)
    out = _module_run(_to(data), z.to(DEV))
    stats = compare_volumes(out["cost_volume"].cpu(), [s.cpu() for s in out["single_frame_cvs"]],
                            torch.from_numpy(g[f"{tag}_cv"]), [torch.from_numpy(s) for s in g[f"{tag}_sf"]])
    print(tag, stats)


@gpu
@pytest.mark.parametrize("gain_tag,gain", [("g1", 1.0), ("g07", 0.7)])
def test_golden_model(gain_tag, gain):
    """MonoRecModel with band hypotheses vs the reference, at the fp32-mode gate of the existing model goldens."""
    from monorec_b200 import conv as C
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import seeded_state_dict
    g = _golden()
    noise = np.load(GOLDEN / "model_fp64.npz")[f"synth_{gain_tag}_noise"]
    data, z = CC.make_pixel_case("model")
    model = MonoRecModel()
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=gain))
    model = model.to(DEV).eval()
    old = C.MODE
    C.set_mode("fp32")
    try:
        d = _to(data)
        d["cv_depths"] = z.to(DEV)
        out = model(d)
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
@pytest.mark.parametrize("shape", [(1, 4, 32, 256, 512), (2, 3, 64, 96, 200), (1, 2, 32, 37, 61), (1, 2, 128, 32, 64)])
def test_broadcast_equals_plane_path_bitwise(shape):
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = shape
    abi = _Abi(_to(make_inputs(B, F, H, W, seed=11)), D)
    nhwc_dtypes = [None] + ([torch.float32, torch.float16] if D <= 32 and D % 8 == 0 else [])
    for dt in nhwc_dtypes:
        cv0, sf0, nh0 = abi.plane(dt)
        cv1, sf1, nh1 = abi.depthmap(abi.broadcast(), dt)
        assert torch.equal(cv0, cv1), (shape, dt, (cv0 - cv1).abs().max().item())
        assert torch.equal(sf0, sf1), (shape, dt, (sf0 - sf1).abs().max().item())
        if dt is not None:
            assert torch.equal(nh0, nh1), (shape, dt)


@gpu
def test_unusable_hypotheses_zero_their_pixels():
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 1, 2, 32, 64, 128
    data = _to(make_inputs(B, F, H, W, seed=12))
    abi = _Abi(data, D)
    good = CC.band_depths(B, D, H, W, seed=9, rel=1.1).to(DEV)
    bad = good.clone()
    spots = [(20, 30, 5, float("nan")), (40, 70, 0, float("inf")), (30, 100, 31, 0.0), (50, 15, 17, -1.0)]
    for y, x, d, v in spots:
        bad[0, d, y, x] = v
    cv0, sf0, _ = abi.depthmap(good)
    cv1, sf1, _ = abi.depthmap(bad)
    near = torch.zeros(H, W, dtype=torch.bool)
    for y, x, _d, _v in spots:
        assert (sf1[:, 0, :, y, x] == 0).all() and (cv1[0, :, y, x] == 0).all(), (y, x)
        near[max(y - 2, 0):y + 3, max(x - 2, 0):x + 3] = True
    far = ~near.to(DEV)
    assert torch.isfinite(cv1).all() and torch.isfinite(sf1).all()
    assert ((cv1 - cv0).abs() * far).max().item() <= 5e-5
    assert ((sf1 - sf0).abs() * far).max().item() <= 5e-5


@gpu
def test_batch_elements_are_independent():
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 2, 3, 32, 96, 200
    abi = _Abi(_to(make_inputs(B, F, H, W, seed=13)), D)
    z = CC.band_depths(B, D, H, W, seed=10).to(DEV)
    cv0, sf0, _ = abi.depthmap(z)
    z2 = z.clone()
    z2[1] = z2[1].flip(0) * 0.5
    z2[1, 3, 10, 10] = float("nan")
    cv1, sf1, _ = abi.depthmap(z2)
    assert torch.equal(cv0[0], cv1[0]) and torch.equal(sf0[:, 0], sf1[:, 0])
    assert not torch.equal(cv0[1], cv1[1])


@gpu
@pytest.mark.parametrize("mode", ["fp32", "tf32", "f16"])
def test_model_broadcast_equals_default_planes(mode):
    from monorec_b200 import conv as C
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import make_inputs, seeded_state_dict
    model = MonoRecModel()
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(DEV).eval()
    B, F, H, W = 2, 2, 64, 128
    data = _to(make_inputs(B, F, H, W, seed=14))
    planes = _Abi(data, model.cv_depth_steps).planes
    old = C.MODE
    C.set_mode(mode)
    try:
        ref = model(dict(data))
        d = dict(data)
        d["cv_depths"] = planes.view(1, -1, 1, 1).expand(B, -1, H, W)
        out = model(d)
        torch.cuda.synchronize()
    finally:
        C.set_mode(old)
    for k in ("cost_volume", "cv_mask", "result"):
        assert torch.equal(ref[k], out[k]), (mode, k)


@gpu
def test_module_rejects_bad_cv_depths():
    from monorec_b200.cost_volume import CostVolumeModule
    from monorec_b200.synthetic import make_inputs
    data = _to(make_inputs(2, 2, 32, 64, seed=1))
    m = CostVolumeModule()
    for z in (torch.ones(2, 8, 32, 63, device=DEV), torch.ones(1, 8, 32, 64, device=DEV), torch.ones(2, 8, 32, device=DEV),
              torch.ones(2, 8, 32, 64), torch.ones(2, 1, 32, 64, device=DEV), torch.ones(2, 129, 32, 64, device=DEV)):
        d = dict(data)
        d["cv_depths"] = z
        with pytest.raises(ValueError):
            m(d)
