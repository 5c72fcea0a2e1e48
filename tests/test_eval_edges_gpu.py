"""The evaluation and point-cloud kernels at their IEEE, slicing and size edges, against the reference and the oracles.

* mr_sparse_metrics on tests/golden/eval_edges.npz (the unmodified reference: NaN, +-inf, negative and -0.0 inputs, rois
  with negative and out-of-range bounds), for the whole batch and per group of 2 images, and its NaN rows through the
  evaluater's fold (mr_eval_accumulate): the batch with a NaN pixel is dropped as the reference drops it.
* mr_pointcloud_add / mr_pointcloud_add_windows on the same golden (Python-slice rois, depths exactly at min_d / max_d,
  0, NaN, inf), at full size against the oracle with a ring vote whose windows wrap, and the C ABI's overflow contract.
* mr_pointcloud_keep_mask bit for bit against the oracle, windows larger than the image and values at the threshold.
* mr_median_scaling bit for bit against the reference's torch calls on the device, at 2^21 selected values and on tiny
  sets."""
import ctypes

import numpy as np
import pytest
import torch

from tests import eval_edges_cases as E
from tests import eval_oracle
from tests.helpers import GOLDEN
from tests.test_metrics_dense import _assert_bitwise, _torch_median_scaling

gpu = pytest.mark.gpu
DEV = "cuda:0"
SPARSE_GATE = dict(rtol=5e-6, atol=1e-7)          # test_metrics.py
PC_GATE = dict(rtol=2e-6, atol=2e-5)              # test_pointcloud.py


def _golden():
    return np.load(GOLDEN / "eval_edges.npz")


# ---- sparse metrics --------------------------------------------------------------------------------------------------
def _sparse_inputs(g):
    return [torch.from_numpy(g[k]).to(DEV) for k in ("pred", "gt", "mvobj")]


def _sparse_args(tag):
    """SPARSE_CASES[tag] as the trailing arguments of sparse_metrics_impl / _grouped_impl after the mvobj mask."""
    kw = E.sparse_kwargs(tag)
    return kw["roi"], float(kw["max_distance"] or 0.0), kw["pred_all_valid"]


@gpu
@pytest.mark.parametrize("tag", list(E.SPARSE_CASES))
def test_cuda_sparse_metrics_match_reference_edges(tag):
    from monorec_b200 import metrics as M
    g = _golden()
    pred, gt, mv = _sparse_inputs(g)
    mvobj = mv if E.sparse_kwargs(tag)["use_cvmask"] else None
    ref = g[f"sparse_{tag}"]
    whole = M.sparse_metrics_impl(pred, gt, mvobj, *_sparse_args(tag))
    E.assert_same(whole.cpu().numpy(), ref[0], **SPARSE_GATE)
    rows = M.sparse_metrics_grouped_impl(pred, gt, mvobj, *_sparse_args(tag), E.GROUP)
    assert tuple(rows.shape) == (len(E.SLICES) - 1, 7)
    E.assert_same(rows.cpu().numpy(), ref[1:], **SPARSE_GATE)
    # the reference-named functions, called as the evaluater calls them
    suffix, roi, md = E.SPARSE_CASES[tag]
    d = {"result": pred, "target": gt, "mvobj_mask": mv}
    named = [float(getattr(M, f"{n}_sparse{suffix}_metric")(d, roi, md)) for n in E.NAMES]
    E.assert_same(named, ref[0], **SPARSE_GATE)


@gpu
def test_cuda_nan_batch_is_dropped_by_the_evaluater_fold():
    """evaluate.py's metrics at max_distance 80 over batches of 2: the first and the last batch hold a NaN pixel, so their
    rows are NaN and the fold drops them (valid 1, not 3); the totals are the one finite batch's."""
    from monorec_b200 import metrics as M
    g = _golden()
    pred, gt, _ = _sparse_inputs(g)
    rows = M.sparse_metrics_grouped_impl(pred, gt, None, *_sparse_args("md"), E.GROUP)
    sizes = [hi - lo for lo, hi in E.SLICES[1:]]
    state = torch.zeros(3 * 7 + 1, dtype=torch.float64, device=DEV)
    M.eval_accumulate_impl(rows, sizes, state)
    got = state.cpu().numpy()
    want = eval_oracle.accumulate(rows.cpu().numpy(), sizes)
    np.testing.assert_array_equal(got.view(np.uint64), np.concatenate([*want[:3], [want[3]]]).view(np.uint64))
    ref = eval_oracle.accumulate(g["sparse_md"][1:], sizes)                 # the reference's rows through the same fold
    np.testing.assert_array_equal(got[7:14], ref[1])
    assert got[7:14].tolist() == [1.0] * 7 and got[21] == sum(sizes)
    np.testing.assert_allclose(got[:7], ref[0], **SPARSE_GATE)
    np.testing.assert_allclose(got[14:21], ref[2], **SPARSE_GATE)


# ---- point cloud ------------------------------------------------------------------------------------------------------
def _assert_vertices(v, ref):
    """Same count and order; colours bit for bit, coordinates within the gate of test_pointcloud.py."""
    v, ref = v.cpu(), torch.as_tensor(ref)
    assert v.shape == ref.shape
    assert torch.equal(v[:, 3:], ref[:, 3:])
    assert torch.allclose(v[:, :3], ref[:, :3], **PC_GATE)


def _pc_inputs(g):
    return [torch.from_numpy(g[f"pc_{k}"]).to(DEV) for k in ("inv_depth", "image", "K", "pose")]


@gpu
@pytest.mark.parametrize("entry", ["add", "windows"])
@pytest.mark.parametrize("tag", list(E.PC_ROIS))
def test_cuda_pointcloud_matches_reference_edges(tag, entry):
    from monorec_b200 import pointcloud as PC
    g = _golden()
    inv, image, K, pose = _pc_inputs(g)
    B, _, H, W = inv.shape
    saver = PC.PLYSaver(H, W, min_d=E.PC_MIN_D, max_d=E.PC_MAX_D, batch_size=B, roi=E.PC_ROIS[tag], dropout=0)
    if entry == "add":
        saver.add_depthmap(inv, image, K, pose)
    else:                            # a one-mask ring of ones keeps every pixel (min_hits 1: 1 > 1 - 1)
        saver.add_depthmap_windows(inv, image, K, pose, torch.ones(1, 1, H, W, device=DEV), [0] * B, 1, min_hits=1)
    _assert_vertices(saver.vertices, g[f"pc_vertices_{tag}"])


def _full_size_scene(seed=11):
    """B 8 at 256x512 (create_pointcloud.py's size): inverse depths around [3, 20] m, key frames, K, poses, dropout numbers,
    and a ring of 7 keep masks made from moving-object masks with blobs (real holes, of different sizes per slot)."""
    from oracle import pointcloud_oracle as PO
    gen = torch.Generator().manual_seed(seed)
    B, H, W, R = 8, 256, 512, 7
    inv = torch.rand(B, 1, H, W, generator=gen) * 0.3 + 0.04
    image = torch.rand(B, 3, H, W, generator=gen) - 0.5
    K = torch.eye(4).repeat(B, 1, 1)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] = 250.0, 248.0, 255.5, 127.5
    pose = torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        a = 0.05 * b
        pose[b, :3, :3] = torch.tensor([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
        pose[b, :3, 3] = torch.tensor([0.1 * b, 0.02 * b, 0.8 * b])
    rand = torch.rand(B, 1, H, W, generator=gen)
    cv = torch.rand(R, 1, H, W, generator=gen) * 0.09                            # below the threshold
    for r in range(R):
        for _ in range(2 + r):
            y, x = int(torch.randint(0, H, (1,), generator=gen)), int(torch.randint(0, W, (1,), generator=gen))
            h, w = int(torch.randint(4, 40, (1,), generator=gen)), int(torch.randint(4, 60, (1,), generator=gen))
            cv[r, 0, y:y + h, x:x + w] = torch.rand(1, generator=gen) * 0.9 + 0.1
    return inv, image, K, pose, rand, PO.keep_mask(cv)


@gpu
@pytest.mark.parametrize("min_hits", [1, 3])
def test_cuda_pointcloud_ring_windows_match_oracle_at_full_size(min_hits):
    """create_pointcloud.py's settings (roi, max_d 20, dropout 0.75, 5-mask vote) for 8 key frames whose windows wrap the
    7-slot ring (starts 5, 6, 0, 1, ...), against the oracle's add_depthmap per key frame: 512 blocks per image through the
    ordered compaction."""
    from monorec_b200 import pointcloud as PC
    from oracle import pointcloud_oracle as PO
    inv, image, K, pose, rand, ring = _full_size_scene()
    B, _, H, W = inv.shape
    R, n_masks, roi = ring.shape[0], 5, [40, 256, 48, 464]
    assert 0.05 < float((ring == 0).float().mean()) < 0.5
    starts = [(5 + b) % R for b in range(B)]
    ref = torch.cat([PO.add_depthmap(inv[b:b + 1], image[b:b + 1], K[b:b + 1], pose[b:b + 1],
                                     keep_masks=[ring[(s + k) % R:(s + k) % R + 1] for k in range(n_masks)],
                                     min_hits=min_hits, min_d=3, max_d=20, roi=roi, dropout=0.75, rand=rand[b:b + 1])
                     for b, s in enumerate(starts)])
    assert ref.shape[0] > B * 216 * 416 * 0.25 * 0.3
    saver = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=roi, dropout=0.75)
    saver.add_depthmap_windows(*[t.to(DEV) for t in (inv, image, K, pose, ring)], starts, n_masks, min_hits=min_hits,
                               rand=rand.to(DEV))
    _assert_vertices(saver.vertices, ref)


@gpu
def test_cuda_pointcloud_overflow_contract():
    """mr_pointcloud_add through the C ABI: a capacity below the needed count gives n_after = -needed and writes nothing; a
    following call with n_before = -1 keeps the count negative and grows it by its own batch; an explicit n_before = k with
    room writes the vertices from row k on."""
    from monorec_b200 import _lib
    lib = _lib.load()
    g = _golden()
    inv, image, K, pose = _pc_inputs(g)
    B, _, H, W = inv.shape
    needed, more = g["pc_vertices_none"].shape[0], g["pc_vertices_neg"].shape[0]
    sentinel, k = -1234.5, 7
    buf = torch.full((k + needed + 64, 6), sentinel, device=DEV)
    n_after = torch.zeros(1, dtype=torch.int64, device=DEV)
    ws_bytes = lib.mr_pointcloud_workspace(B, H, W)
    ws = torch.empty((ws_bytes + 7) // 8, dtype=torch.int64, device=DEV)

    def add(n_before, capacity, roi=None):
        roi_c = None if roi is None else (ctypes.c_int * 4)(*roi)
        _lib.check(lib.mr_pointcloud_add(inv.data_ptr(), image.data_ptr(), K.data_ptr(), pose.data_ptr(), None, 0, 1, B, H, W,
                                         E.PC_MIN_D, E.PC_MAX_D, roi_c, None, 0.0, buf.data_ptr(), capacity, n_before,
                                         n_after.data_ptr(), ws.data_ptr(), ws_bytes,
                                         torch.cuda.current_stream().cuda_stream), "mr_pointcloud_add")
        torch.cuda.synchronize()
        return int(n_after.item())

    assert add(0, needed - 1) == -needed
    assert bool((buf == sentinel).all())
    assert add(-1, needed - 1, roi=E.PC_ROIS["neg"]) == -(needed + more)
    assert bool((buf == sentinel).all())
    assert add(k, k + needed) == k + needed
    assert bool((buf[:k] == sentinel).all()) and bool((buf[k + needed:] == sentinel).all())
    _assert_vertices(buf[k:k + needed], g["pc_vertices_none"])


def _keep_mask_input(H, W, seed=12):
    """Three images below the threshold 0.1 with: image 0, a few pixels exactly float32(0.1); image 1, a quarter of the
    pixels at the float just below it and one +inf; image 2, NaN and -inf pixels and one pixel at 0.1."""
    gen = torch.Generator().manual_seed(seed)
    cv = torch.rand(3, 1, H, W, generator=gen) * 0.09
    t = torch.tensor(0.1, dtype=torch.float32)
    below = torch.nextafter(t, torch.tensor(0.0))

    def pick(n):
        return torch.randperm(H * W, generator=gen)[:n]

    cv[0].view(-1)[pick(5)] = t
    cv[1].view(-1)[pick(H * W // 4)] = below
    cv[1].view(-1)[pick(1)] = float("inf")
    cv[2].view(-1)[pick(H * W // 8)] = float("nan")
    cv[2].view(-1)[pick(3)] = float("-inf")
    cv[2].view(-1)[pick(1)] = t
    return cv


@gpu
@pytest.mark.parametrize("mask_fill", [0, 2, 32])
@pytest.mark.parametrize("size", [(20, 24), (256, 512)], ids=["smaller_than_window", "full"])
def test_cuda_keep_mask_matches_oracle_bitwise(size, mask_fill):
    from monorec_b200 import pointcloud as PC
    from oracle import pointcloud_oracle as PO
    cv = _keep_mask_input(*size)
    ref = PO.keep_mask(cv, mask_fill=mask_fill, thresh=0.1)
    got = PC.keep_mask(cv.to(DEV), mask_fill=mask_fill, thresh=0.1).cpu()
    assert torch.equal(got, ref)
    hit = cv >= torch.tensor(0.1)
    assert bool((ref[hit] == 0).all())                             # the threshold value itself is a hit
    if mask_fill == 0:                                             # the float below it, NaN and -inf are not
        assert torch.equal(ref == 0, hit)
    assert bool((ref == 1).any()) and bool((ref == 0).any())


# ---- median scaling ---------------------------------------------------------------------------------------------------
def _median_check(pred, gt):
    from monorec_b200 import metrics as M
    d = {"result": pred.to(DEV), "target": gt.to(DEV)}
    out = M.median_scaling(d)["result"].cpu().numpy()
    _assert_bitwise(out, _torch_median_scaling(d)["result"].cpu().numpy())
    return out


@gpu
def test_cuda_median_scaling_bitwise_at_two_million_values():
    """[2,1,1024,2048]: image 0 selects every pixel (2^21 values, an even count: the lower median), image 1 all but one
    (odd).  Targets span denormals to 1e30; predictions hold negative values, +inf and many ties; image 1's median
    prediction is negative (a negative ratio)."""
    gen = torch.Generator().manual_seed(13)
    B, H, W = 2, 1024, 2048
    gt = (10.0 ** (torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64) * 74 - 44)).float()
    gt[gt == 0] = 1e-45                                            # the smallest denormal: still selected
    gt[:, :, ::3] = torch.randint(1, 5, (B, 1, (H + 2) // 3, W), generator=gen).float() * 1e-7   # ties near the median
    gt[1, 0, 5, 7] = 0.0
    pred = (10.0 ** (torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64) * 60 - 30)).float()
    pred[:, :, 1::2] = torch.randint(-3, 4, (B, 1, H // 2, W), generator=gen).float() * 0.25        # ties
    pred[1] = -pred[1].abs()
    pred[torch.rand(B, 1, H, W, generator=gen) < 1e-3] = float("inf")
    assert bool((gt[0] > 0).all()) and int((gt[1] > 0).sum()) == H * W - 1
    assert bool(((gt > 0) & (gt < torch.finfo(torch.float32).tiny)).any())
    out = _median_check(pred, gt)
    assert np.isposinf(out[0]).any() and np.isneginf(out[1]).any() and (out[1] > 0).any()


@gpu
def test_cuda_median_scaling_small_sets():
    """One selected value, two (the lower one), all equal, NaN predictions only at unselected pixels (a finite ratio),
    and denormal targets against huge predictions (a ratio that underflows)."""
    gen = torch.Generator().manual_seed(14)
    B, H, W = 5, 16, 24
    pred = torch.rand(B, 1, H, W, generator=gen) * 0.3 + 0.01
    gt = torch.zeros(B, 1, H, W)
    flat_p, flat_g = pred.view(B, -1), gt.view(B, -1)
    idx = torch.randperm(H * W, generator=gen)
    flat_g[0, idx[0]] = 0.07
    flat_g[1, idx[:2]] = torch.tensor([0.05, 0.2])
    flat_p[1, idx[:2]] = torch.tensor([0.3, 0.1])
    flat_g[2, idx[:9]], flat_p[2, idx[:9]] = 0.125, 0.5
    flat_g[3, idx[:9]] = torch.rand(9, generator=gen) + 0.1
    flat_g[3, idx[9:20]] = -1.0
    flat_p[3, idx[9:30]] = float("nan")
    flat_g[3, idx[30]] = float("nan")
    flat_g[4, idx[:6]] = torch.tensor([1e-45, 3e-44, 2e-40, 1e-39, 5e-42, 7e-45])
    flat_p[4, idx[:6]] = 1e30
    out = _median_check(pred, gt)
    sel3 = ~np.isnan(flat_p[3].numpy())
    assert np.isfinite(out[3].reshape(-1)[sel3]).all()
    assert np.isfinite(out).reshape(B, -1)[[0, 1, 2, 4]].all()
