"""Parity of the fused sm_90a cost-volume kernel (through the C ABI) with the reference / oracle.  Needs an H100."""
import numpy as np
import pytest
import torch

from tests.helpers import compare_volumes, kitti_sample_dict, synth_small_dict

pytestmark = pytest.mark.gpu


def _run(data, steps=32, inv=(0.33, 0.0025), **kw):
    from monorec_b200.cost_volume import CostVolumeModule
    from monorec_b200.synthetic import to_device
    d = to_device(data, "cuda:0")
    key = d["keyframe"]
    d["inv_depth_min"] = key.new_tensor([inv[0]])
    d["inv_depth_max"] = key.new_tensor([inv[1]])
    d["cv_depth_steps"] = key.new_tensor([steps], dtype=torch.int32)
    out = CostVolumeModule(**kw)(d)
    torch.cuda.synchronize()
    return out["cost_volume"].cpu(), [s.cpu() for s in out["single_frame_cvs"]]


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_golden_small_full_tensors(tag):
    data, D, ref_cv, ref_sf = synth_small_dict(tag)
    cv, sf = _run(data, steps=D)
    stats = compare_volumes(cv, sf, ref_cv, ref_sf)
    print(tag, stats)


def test_golden_kitti_sample():
    data, g = kitti_sample_dict()
    cv, sf = _run(data)
    sub = (slice(None), slice(None), slice(2, None, 4), slice(1, None, 8))
    stats = compare_volumes(cv[sub], [s[sub] for s in sf], torch.from_numpy(g["cv_sub"]),
                            [torch.from_numpy(v) for v in g["sf_sub"]])
    rows = (slice(None), slice(None), slice(100, 104))
    stats_rows = compare_volumes(cv[rows], [s[rows] for s in sf], torch.from_numpy(g["cv_rows"]),
                                 [torch.from_numpy(v) for v in g["sf_rows"]])
    # "identical argmin depth indices" (= argmax of the centred volume) under the tie rule of SURVEY.md §8c
    ref_arg = torch.from_numpy(g["argmax"].astype(np.int64))
    margin = torch.from_numpy(g["margin"].astype(np.float32))
    H, W = ref_arg.shape[-2:]
    ref_zero = torch.from_numpy(np.unpackbits(g["cv_zero"])[: H * W].reshape(1, H, W).astype(bool))
    mine_zero = (cv == 0).all(1)
    # per-frame validity must agree too (a boundary pixel whose bilinear mask sample is +-0 flips valid_f, which changes
    # the fused value completely; SURVEY.md §8c allows a few such pixels per frame and excludes them from the gate)
    nF = len(sf)
    ref_sf_zero = np.unpackbits(g["sf_zero"])[: nF * H * W].reshape(nF, 1, H, W).astype(bool)
    masks_agree = torch.ones(1, H, W, dtype=torch.bool)
    mask_flips = 0
    for f in range(nF):
        mz = (sf[f] == 0).all(1)
        rz = torch.from_numpy(ref_sf_zero[f])
        masks_agree &= (mz == rz)
        mask_flips += int((mz != rz).sum())
    assert mask_flips <= 4 * nF, f"{mask_flips} validity flips"
    both = (~ref_zero) & (~mine_zero) & masks_agree
    same = cv.argmax(1) == ref_arg
    agree4 = same[both & (margin > 1e-4)].float().mean().item()
    agree3 = same[both & (margin > 1e-3)].float().mean().item()
    raw = same[both].float().mean().item()
    flips = int((ref_zero != mine_zero).sum())
    print("kitti", stats, stats_rows, "argmax margin>1e-3", agree3, "margin>1e-4", agree4, "raw", raw,
          "zero-set flips", flips, "validity flips", mask_flips)
    # fp32 noise floor of the reference itself (fp32 vs fp64 run of the unmodified reference, make_golden.py):
    # raw agreement 99.83 %, volume max|d| 8.9e-4.  Two volumes that agree to 1e-3 can only flip an argmax whose
    # top1-top2 margin is below 2e-3, so the hard gate is margin > 1e-3; the 1e-4 band is reported and bounded.
    assert agree3 == 1.0
    assert agree4 > 0.9999
    assert raw > 0.997
    assert flips <= 600  # flat-cost pixels (exact-zero weights) sit on an fp32 knife edge: reference fp32 vs fp64 differ on 234
    # per-plane checksums of the full-resolution volume
    # per-plane mean error below 1e-4
    np.testing.assert_allclose(cv.double().sum((2, 3)).numpy(), g["cv_plane_sum"], rtol=0, atol=1e-4 * H * W)


@pytest.mark.parametrize("cfg", [(2, 4, 32, 128, 256, 11), (1, 2, 64, 64, 160, 12), (1, 6, 16, 80, 200, 13)])
def test_against_oracle_seeded(cfg):
    from oracle import cost_volume_oracle as O
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W, seed = cfg
    data = make_inputs(B, F, H, W, seed=seed)
    ref_cv, ref_sf = O.cost_volume_torch(data, steps=D)
    cv, sf = _run(data, steps=D)
    print(cfg, compare_volumes(cv, sf, ref_cv, ref_sf))


def test_full_size_properties():
    """BASELINE config 2 (B=8, F=4, D=32, 256x512): size-independent properties (SURVEY.md §4 item 3)."""
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 8, 4, 32, 256, 512
    data = make_inputs(B, F, H, W, seed=0)
    cv, sf = _run(data, steps=D)
    assert torch.isfinite(cv).all() and all(torch.isfinite(s).all() for s in sf)
    assert cv.abs().max() <= 1.0 + 1e-6 and all(s.abs().max() <= 1.0 + 1e-6 for s in sf)
    for t in [cv] + sf:   # the 2-px ring is exactly zero (monorec_model.py:139, :282-284)
        assert (t[..., :2, :] == 0).all() and (t[..., -2:, :] == 0).all()
        assert (t[..., :, :2] == 0).all() and (t[..., :, -2:] == 0).all()
    # batch independence: element 3 alone gives bitwise the same result
    one = {k: ([t[3:4] for t in v] if isinstance(v, list) else v[3:4]) for k, v in data.items()}
    cv1, sf1 = _run(one, steps=D)
    assert torch.equal(cv1[0], cv[3]) and all(torch.equal(a[0], b[3]) for a, b in zip(sf1, sf))
    # frame-permutation: single-frame volumes permute exactly, fused volume up to summation order
    perm = [2, 0, 3, 1]
    pd = dict(data)
    for k in ("frames", "poses", "intrinsics"):
        pd[k] = [data[k][i] for i in perm]
    cvp, sfp = _run(pd, steps=D)
    assert all(torch.equal(sfp[j], sf[perm[j]]) for j in range(F))
    assert (cvp - cv).abs().max() <= 1e-5
    # the same source frame given twice: equal view weights, so the fused volume equals the single-frame volume
    # (1 - 2 sum_f w sad / sum_f w with identical terms) wherever the weight is non-zero
    dup = dict(one)
    for k in ("frames", "poses", "intrinsics"):
        dup[k] = [one[k][1], one[k][1]]
    cvd, sfd = _run(dup, steps=D)
    assert torch.equal(sfd[0], sfd[1])
    nz = ~(cvd == 0).all(1, keepdim=True)
    assert ((cvd - sfd[0]) * nz).abs().max() < 1e-5

def test_host_entry_matches_device_entry():
    """mr_cost_volume_host (host buffers, internal copies) == device-pointer path, bitwise."""
    import ctypes
    from monorec_b200 import _lib
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W = 3, 2, 32, 64, 128
    data = make_inputs(B, F, H, W, seed=4)
    cv, sf = _run(data, steps=D)
    lib = _lib.load()
    ws_bytes = lib.mr_cost_volume_host_workspace(B, F, D, H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda:0")
    frames = torch.stack(data["frames"]).contiguous().pin_memory()
    poses = torch.stack(data["poses"]).contiguous()
    intr = torch.stack(data["intrinsics"]).contiguous()
    out_cv = torch.empty(B, D, H, W).pin_memory()
    out_sf = torch.empty(F, B, D, H, W).pin_memory()
    _lib.check(lib.mr_cost_volume_host(data["keyframe"].contiguous().data_ptr(), frames.data_ptr(),
                                       data["keyframe_pose"].contiguous().data_ptr(),
                                       data["keyframe_intrinsics"].contiguous().data_ptr(), poses.data_ptr(),
                                       intr.data_ptr(), out_cv.data_ptr(), out_sf.data_ptr(), B, F, D, H, W,
                                       0.0025, 0.33, 10.0, ws.data_ptr(), ws_bytes), "mr_cost_volume_host")
    assert torch.equal(out_cv, cv)
    assert all(torch.equal(out_sf[f], sf[f]) for f in range(F))


def test_error_behaviour():
    from monorec_b200 import _lib
    from monorec_b200.cost_volume import CostVolumeModule
    from monorec_b200.synthetic import make_inputs
    with pytest.raises(NotImplementedError):
        CostVolumeModule(use_ssim=False)
    data = make_inputs(1, 9, 32, 64, seed=1)
    with pytest.raises(_lib.MonorecLibraryError):
        _run(data)   # F = 9 > MR_MAX_FRAMES
    with pytest.raises(KeyError):
        CostVolumeModule()({"keyframe": torch.zeros(1, 3, 32, 64, device="cuda:0")})


@pytest.mark.parametrize("cfg", [(1, 2, 32, 37, 61, 31), (2, 1, 8, 48, 333, 32), (1, 3, 32, 100, 500, 33), (1, 2, 128, 32, 64, 34),
                                 (1, 8, 4, 24, 70, 35)])
def test_ragged_shapes_against_oracle(cfg):
    """tile edges: W not a multiple of the 60-column tile (and odd: scalar stores), H not a multiple of 16, D from 4 to 128,
    F from 1 to MR_MAX_FRAMES"""
    from oracle import cost_volume_oracle as O
    from monorec_b200.synthetic import make_inputs
    B, F, D, H, W, seed = cfg
    data = make_inputs(B, F, H, W, seed=seed)
    ref_cv, ref_sf = O.cost_volume_torch(data, steps=D)
    cv, sf = _run(data, steps=D)
    print(cfg, compare_volumes(cv, sf, ref_cv, ref_sf))


def test_hires_config_small_batch():
    """BASELINE config 5 shape (512x1024, D=64, F=6) on one keyframe: properties only (the CPU oracle needs 42 GB here)"""
    from monorec_b200.synthetic import make_inputs
    data = make_inputs(1, 6, 512, 1024, seed=40)
    cv, sf = _run(data, steps=64)
    assert cv.shape == (1, 64, 512, 1024) and len(sf) == 6
    assert torch.isfinite(cv).all() and cv.abs().max() <= 1.0 + 1e-6
    for t in [cv] + sf:
        assert (t[..., :2, :] == 0).all() and (t[..., -2:, :] == 0).all() and (t[..., :, :2] == 0).all() and (t[..., :, -2:] == 0).all()
    # frame order must not matter for the single-frame volumes at this size either
    perm = [5, 3, 1, 0, 2, 4]
    pd = dict(data)
    for k in ("frames", "poses", "intrinsics"):
        pd[k] = [data[k][i] for i in perm]
    cvp, sfp = _run(pd, steps=64)
    assert all(torch.equal(sfp[j], sf[perm[j]]) for j in range(6))
    assert (cvp - cv).abs().max() <= 1e-5


@pytest.mark.parametrize("B,F,H,W", [(2, 3, 96, 200), (1, 4, 256, 512)])
def test_tma_windows_and_global_gather_agree(B, F, H, W):
    """mr_cost_volume_fwd (TMA-staged windows) == mr_cost_volume_fwd_gather (taps from global memory): same formula, same
    validity; the two interpolation code paths may differ in the last bits only."""
    from monorec_b200 import _lib
    from monorec_b200.cost_volume import CostVolumeModule
    from monorec_b200.synthetic import make_inputs, to_device
    D, dev = 32, "cuda:0"
    d = to_device(make_inputs(B, F, H, W, seed=55), dev)
    lib = _lib.load()
    m = CostVolumeModule()
    cw = (_lib.c_float * 3)(*m.channel_weights)
    stream = torch.cuda.current_stream().cuda_stream
    proj = torch.empty(B, F, 3, 4, device=dev)
    depths = torch.empty(D, device=dev)
    _lib.check(lib.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                        _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H, W,
                                        proj.data_ptr(), depths.data_ptr(), D, 0.0025, 0.33, stream), "mr_projection_tables")
    outs = []
    for name in ("mr_cost_volume_fwd", "mr_cost_volume_fwd_gather"):
        cv = torch.full((B, D, H, W), float("nan"), device=dev)
        sfcv = torch.full((F, B, D, H, W), float("nan"), device=dev)
        _lib.check(getattr(lib, name)(d["keyframe"].data_ptr(), _lib.ptr_array(d["frames"]), proj.data_ptr(), depths.data_ptr(),
                                      cv.data_ptr(), sfcv.data_ptr(), B, F, D, H, W, float(m.alpha), cw, stream), name)
        torch.cuda.synchronize()
        outs.append((cv.cpu(), list(sfcv.cpu())))
    for a, b in zip(outs[0][1], outs[1][1]):
        assert torch.equal((a == 0).all(1), (b == 0).all(1))   # same validity (a plane stack that is exactly 0)
        d = (a - b).abs()
        assert d.max() <= 5e-5, f"single-frame volumes differ by {d.max().item():.3e} ({int((d > 2e-6).sum())} values > 2e-6)"
    d = (outs[0][0] - outs[1][0]).abs()
    assert d.max() <= 1e-4, f"fused volumes differ by {d.max().item():.3e}"


def test_cost_volume_golden_d64_f6():
    """CUDA cost volume vs the reference's own output for 64 planes x 6 source frames (tests/golden/cv_synth_d64f6.npz,
    BASELINE config 5's plane and frame counts); the same gates as test_golden_small_full_tensors."""
    from tests.helpers import compare_volumes, synth_small_dict
    data, D, ref_cv, ref_sf = synth_small_dict("d")
    cv, sf = _run(data, steps=D)
    print(compare_volumes(cv, sf, ref_cv, ref_sf))


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_nhwc_copy_of_single_frame_volumes(dtype):
    """mr_cost_volume_fwd_nhwc: the engine-layout copy written by the per-pixel phase == the NCHW volumes permuted (and
    rounded to half), bit for bit, invalid pixels included."""
    from monorec_b200.cost_volume import CostVolumeModule
    from monorec_b200.synthetic import make_inputs, to_device
    B, F, H, W, D = 2, 3, 64, 128, 32
    d = to_device(make_inputs(B, F, H, W, seed=77), "cuda:0")
    d["_cv_range"] = (0.0025, 0.33, D)
    d["_sfcv_nhwc"] = torch.full((F * B, H, W, D), 7.0, device="cuda:0", dtype=dtype)
    out = CostVolumeModule()(d)
    torch.cuda.synchronize()
    assert out.get("_sfcv_nhwc_filled") is True
    ref = torch.cat([s.permute(0, 2, 3, 1) for s in out["single_frame_cvs"]], 0).to(dtype)
    assert torch.equal(out["_sfcv_nhwc"], ref)
    # the ring of invalid border pixels is zero in both
    assert float(out["_sfcv_nhwc"][:, :2].abs().max()) == 0.0


def test_golden_config2_full_size():
    """BASELINE config 2's geometry at full size (256x512, D=32, F=4; tests/golden/cv_config2.npz from the unmodified reference):
    sub-sampled volumes and full rows within 1e-3, validity maps (valid shares 96 / 53 / 97 / 22 % per frame), arg-max under the
    tie rule, per-plane checksums."""
    from monorec_b200.synthetic import make_inputs
    from tests.helpers import GOLDEN, compare_volumes
    g = np.load(GOLDEN / "cv_config2.npz")
    B, nF, D, H, W, seed = [int(v) for v in g["cfg"]]
    cv, sf = _run(make_inputs(B, nF, H, W, seed=seed), steps=D)
    sub = (slice(None), slice(None), slice(2, None, 4), slice(1, None, 8))
    stats = compare_volumes(cv[sub], [s[sub] for s in sf], torch.from_numpy(g["cv_sub"]), [torch.from_numpy(v) for v in g["sf_sub"]])
    rows = (slice(None), slice(None), slice(100, 104))
    stats_rows = compare_volumes(cv[rows], [s[rows] for s in sf], torch.from_numpy(g["cv_rows"]), [torch.from_numpy(v) for v in g["sf_rows"]])
    ref_sf_zero = np.unpackbits(g["sf_zero"])[: nF * H * W].reshape(nF, 1, H, W).astype(bool)
    masks_agree = torch.ones(1, H, W, dtype=torch.bool)
    flips = 0
    for f in range(nF):
        mz, rz = (sf[f] == 0).all(1), torch.from_numpy(ref_sf_zero[f])
        masks_agree &= (mz == rz)
        flips += int((mz != rz).sum())
    assert flips <= 4 * nF, f"{flips} validity flips"
    ref_zero = torch.from_numpy(np.unpackbits(g["cv_zero"])[: H * W].reshape(1, H, W).astype(bool))
    both = (~ref_zero) & (~(cv == 0).all(1)) & masks_agree
    same = cv.argmax(1) == torch.from_numpy(g["argmax"].astype(np.int64))
    margin = torch.from_numpy(g["margin"].astype(np.float32))
    agree3 = same[both & (margin > 1e-3)].float().mean().item()
    agree4 = same[both & (margin > 1e-4)].float().mean().item()
    print("config 2", stats, stats_rows, "argmax margin>1e-3", agree3, "margin>1e-4", agree4, "raw", same[both].float().mean().item(),
          "validity flips", flips)
    assert agree3 == 1.0 and agree4 > 0.9999
    np.testing.assert_allclose(cv.double().sum((2, 3)).numpy(), g["cv_plane_sum"], rtol=0, atol=1e-4 * H * W)
    for f in range(nF):
        np.testing.assert_allclose(sf[f].double().sum((2, 3)).numpy(), g["sf_plane_sum"][f], rtol=0, atol=1e-4 * H * W)
