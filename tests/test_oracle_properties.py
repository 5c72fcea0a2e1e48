"""Property tests of the oracle itself (SURVEY.md §4 item 3), hypothesis-driven on tiny problems (CPU)."""
import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

from monorec_b200.synthetic import make_inputs
from oracle import cost_volume_oracle as O


@settings(max_examples=6, deadline=None)
@given(seed=st.integers(0, 10_000), frames=st.integers(1, 3), planes=st.sampled_from([4, 8, 16]))
def test_ring_range_and_permutation(seed, frames, planes):
    data = make_inputs(2, frames, 24, 40, seed=seed)
    cv, sf = O.cost_volume_torch(data, steps=planes)
    for t in [cv] + sf:
        assert torch.isfinite(t).all() and t.abs().max() <= 1 + 1e-6
        assert (t[..., :2, :] == 0).all() and (t[..., -2:, :] == 0).all() and (t[..., :, :2] == 0).all() and (t[..., :, -2:] == 0).all()
    # batch independence: element 1 alone
    one = {k: ([t[1:2] for t in v] if isinstance(v, list) else v[1:2]) for k, v in data.items()}
    cv1, sf1 = O.cost_volume_torch(one, steps=planes)
    assert torch.allclose(cv1[0], cv[1], atol=1e-6) and all(torch.allclose(a[0], b[1], atol=1e-6) for a, b in zip(sf1, sf))
    if frames > 1:   # frame order: single-frame volumes permute, the fused volume is symmetric
        perm = list(reversed(range(frames)))
        pd = dict(data)
        for k in ("frames", "poses", "intrinsics"):
            pd[k] = [data[k][i] for i in perm]
        cvp, sfp = O.cost_volume_torch(pd, steps=planes)
        assert all(torch.allclose(sfp[j], sf[perm[j]], atol=1e-6) for j in range(frames))
        assert torch.allclose(cvp, cv, atol=1e-5)


@settings(max_examples=4, deadline=None)
@given(seed=st.integers(0, 10_000))
def test_closed_form_agrees_with_torch_restatement(seed):
    data = make_inputs(1, 2, 24, 40, seed=seed)
    cv, sf = O.cost_volume_torch(data, steps=8)
    cvc, sfc, valid, _ = O.cost_volume_closed_form(data, steps=8, dtype=np.float32)
    za, zb = (cv == 0).all(1), torch.from_numpy((cvc == 0).all(1))
    both = ~(za | zb)
    assert int((za != zb).sum()) <= 8
    assert ((cv - torch.from_numpy(cvc)).abs() * both.unsqueeze(1)).max() < 1e-3


def _margin_cases():
    from tests import cv_cases as CC
    yield "planes", make_inputs(2, 3, 24, 41, seed=17), dict(steps=8)
    yield "planes_d64", make_inputs(1, 2, 37, 61, seed=31), dict(steps=64)
    for tag in CC.PIXEL_CASES:
        data, z = CC.make_pixel_case(tag)
        yield tag, data, dict(cv_depths=z)
    data, z, D, _, _ = CC.make_matching_case("ssim_l1_band")
    yield "ssim_l1_band", data, dict(cv_depths=z)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_validity_margin_sign_is_the_closed_form_validity(dtype):
    """`validity_margin > 0` is exactly the closed form's `valid` (the bilinear sample of the interior mask is non-zero
    strictly inside 1 < s < n-2) on seeded planes and on the golden per-pixel cases, whose wide spans flip validity inside
    the band; the float32 mode rounds the positions as the closed form does."""
    for tag, data, kw in _margin_cases():
        _, _, valid, _ = O.cost_volume_closed_form(data, dtype=dtype, **kw)
        margin = O.validity_margin(data, dtype=dtype, **kw)
        assert margin.dtype == np.float64 and margin.shape == valid.shape, tag
        assert np.array_equal(margin > 0, valid), (tag, int(((margin > 0) != valid).sum()))
        assert valid.any() and (~valid[..., 2:-2, 2:-2]).any(), tag        # both sides of the edge are reached
        assert np.isneginf(margin[..., :2, :]).all() and np.isneginf(margin[..., :, -2:]).all(), tag


def test_validity_margin_is_the_distance_to_the_edge():
    """With the keyframe as its own source frame every depth projects pixel (u, v) onto itself, at the source position
    sx = u W / (W - 1) - 1/2 (point_projection normalises with W - 1, grid_sample un-normalises with W), so the margin is
    min(sx - 1, W - 2 - sx, sy - 1, H - 2 - sy) of that position."""
    data = make_inputs(1, 1, 20, 33, seed=3)
    data = dict(data, frames=[data["keyframe"].clone()], poses=[data["keyframe_pose"].clone()],
                intrinsics=[data["keyframe_intrinsics"].clone()])
    m = O.validity_margin(data, steps=4)[0, 0]
    H, W = m.shape
    v, u = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    sx = u * W / (W - 1) - 0.5
    sy = v * H / (H - 1) - 0.5
    want = np.minimum(np.minimum(sx - 1, W - 2 - sx), np.minimum(sy - 1, H - 2 - sy))
    inner = np.zeros((H, W), bool)
    inner[2:-2, 2:-2] = True
    assert np.allclose(m[inner], want[inner], rtol=0, atol=1e-5)


@settings(max_examples=3, deadline=None)
@given(seed=st.integers(0, 10_000))
def test_reprojection_loss_properties(seed):
    """Size-independent properties of the photometric reprojection loss (common_losses.py:16-114) on the oracle:
    without relative motion the error does not depend on the predicted depth; the minimum over the frames never exceeds a single frame's error; frame order does not
    matter; batch elements are independent; the closed form agrees with the torch restatement."""
    import warnings
    from oracle import reprojection_oracle as RO
    B, H, W = 2, 24, 40
    data = make_inputs(B, 2, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed)
    invd = 0.05 + 0.2 * torch.rand(B, 1, H, W, generator=g)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        same = dict(data, frames=[data["keyframe"].clone()], poses=[data["keyframe_pose"].clone()], intrinsics=[data["keyframe_intrinsics"].clone()])
        e_same, w_same = RO.reprojection_errors(invd, same)
        # (not 0: point_projection normalises with W-1 while grid_sample un-normalises with W, a shift of up to half a pixel --
        # SURVEY.md section 8a row 3) but with no relative motion the sample position does not depend on the depth at all
        e_same2, _ = RO.reprojection_errors(0.3 - invd, same)
        assert (w_same == 0).all() and float((e_same - e_same2).abs().max()) < 1e-5
        e_all, w_all = RO.reprojection_errors(invd, data)
        singles = []
        for f in range(2):
            one = dict(data, frames=[data["frames"][f]], poses=[data["poses"][f]], intrinsics=[data["intrinsics"][f]])
            singles.append(RO.reprojection_errors(invd, one)[0])
        assert torch.equal(e_all, torch.minimum(singles[0], singles[1]))
        swapped = dict(data, frames=data["frames"][::-1], poses=data["poses"][::-1], intrinsics=data["intrinsics"][::-1])
        e_sw, w_sw = RO.reprojection_errors(invd, swapped)
        assert torch.equal(e_sw, e_all)
        tie = singles[0] == singles[1]
        assert torch.equal((1 - w_sw)[(w_all >= 0) & ~tie], w_all[(w_all >= 0) & ~tie])
        one_b = {k: ([t[1:2] for t in v] if isinstance(v, list) else v[1:2]) for k, v in data.items()}
        assert torch.equal(RO.reprojection_errors(invd[1:2], one_b)[0][0], e_all[1])
        be, wi, _ = RO.reprojection_closed_form(invd, data, dtype="float32")
    fin = (torch.from_numpy(wi) == w_all) & (w_all >= 0)
    assert float(fin.float().mean()) > 0.99
    assert float((torch.from_numpy(be) - e_all)[fin].abs().max()) < 1e-4
