"""Grayscale frames ([.., 1, H, W]) on the GPU: every output equals, bit for bit (torch.equal), the output for the same
frames replicated to three channels with expand(-1, 3, -1, -1).contiguous().  The cost-volume kernel through
mr_cost_volume_fwd_channels and CostVolumeModule (every error mode, centring, depth source, volume type and NHWC copy, both
march paths, ragged tiles, F = 1 .. 8, D = 2 .. 128), MonoRecModel (engine modes, pretrain modes, stereo; eager, graph
replay, torch.compile), and the frame-stream drivers (MonoRecSequence, SequenceEvaluater, sequence_pointcloud,
MultiModelEvaluater)."""
import io
import json

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DT = {torch.float32: 0, torch.float16: 1}


def rgb(t):
    return t.expand(-1, 3, -1, -1).contiguous()


def _gray_inputs(B, F, H, W, seed):
    """make_inputs' dict with one-channel images (the first plane of its frames), on the GPU."""
    from monorec_b200.synthetic import make_inputs, to_device
    d = to_device(make_inputs(B, F, H, W, seed=seed), DEV)
    d["keyframe"] = d["keyframe"][:, :1].contiguous()
    d["frames"] = [f[:, :1].contiguous() for f in d["frames"]]
    return d


def _rgb_dict(d):
    out = dict(d)
    for k in ("keyframe", "stereoframe"):
        if k in d:
            out[k] = rgb(d[k])
    out["frames"] = [rgb(f) for f in d["frames"]]
    return out


def _unaligned(t):
    """The same values 4 bytes past a 16-byte boundary: TMA cannot address it, every unit gathers."""
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


class _Abi:
    """mr_cost_volume_fwd_channels / mr_cost_volume_fwd_typed on one projection table."""

    def __init__(self, d, D):
        from monorec_b200 import _lib
        self.lib, self.L, self.d, self.D = _lib.load(), _lib, d, D
        self.B, _, self.H, self.W = d["keyframe"].shape
        self.F = len(d["frames"])
        self.proj = torch.empty(self.B, self.F, 3, 4, device=DEV)
        self.planes = torch.empty(D, device=DEV)
        self.stream = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.mr_projection_tables(
            d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(), _lib.ptr_array(d["poses"]),
            _lib.ptr_array(d["intrinsics"]), self.B, self.F, self.H, self.W, self.proj.data_ptr(), self.planes.data_ptr(), D,
            0.0025, 0.33, self.stream), "mr_projection_tables")

    def run(self, key, frames, dtype, matching, centered, z, nhwc_dtype, channels=None):
        """channels None: the typed entry; else the channels entry.  Outputs start as NaN, so every value is written."""
        cv = torch.full((self.B, self.D, self.H, self.W), float("nan"), device=DEV, dtype=dtype)
        sf = torch.full((self.F, self.B, self.D, self.H, self.W), float("nan"), device=DEV, dtype=dtype)
        nh = None if nhwc_dtype is None else torch.full((self.F * self.B, self.H, self.W, self.D), float("nan"), device=DEV,
                                                         dtype=nhwc_dtype)
        args = [key.data_ptr(), self.L.ptr_array(frames), self.proj.data_ptr(), None if z is not None else self.planes.data_ptr(),
                None if z is None else z.data_ptr(), cv.data_ptr(), sf.data_ptr(), None if nh is None else nh.data_ptr(),
                0 if nh is None else DT[nhwc_dtype], self.B, self.F, self.D, self.H, self.W, 10.0, None, matching, centered,
                DT[dtype]]
        if channels is None:
            self.L.check(self.lib.mr_cost_volume_fwd_typed(*args, self.stream), "mr_cost_volume_fwd_typed")
        else:
            self.L.check(self.lib.mr_cost_volume_fwd_channels(*args, channels, self.stream), "mr_cost_volume_fwd_channels")
        torch.cuda.synchronize()
        return cv, sf, nh


def _same(a, b):
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


# (B, F, D, H, W, unaligned): W % 4 == 0 (TMA windows) / W % 4 != 0 or an unaligned base (global gather), ragged tile edges
# (W not a multiple of 60, H not a multiple of the tile height), F = 1 and 8, D = 2, 32, 33 and 128
KERNEL_CASES = [
    (2, 2, 32, 64, 128, False),
    (1, 3, 32, 37, 61, False),
    (1, 2, 32, 48, 128, True),
    (1, 1, 2, 40, 92, False),
    (1, 8, 33, 35, 124, False),
    (1, 2, 128, 32, 64, False),
    (1, 8, 128, 24, 70, False),
]


@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: "B{}F{}D{}_{}x{}{}".format(*c[:5], "_unaligned" if c[5] else ""))
def test_kernel_gray_is_the_replicated_kernel(case):
    """Through the C entry: every error mode x centring x depth source x fp32 / half volumes x NHWC copy none / fp32 /
    half, gray against the replicated frames; the channels = 3 entry against mr_cost_volume_fwd_typed."""
    B, F, D, H, W, unaligned = case
    d = _gray_inputs(B, F, H, W, seed=200 + D + W)
    abi = _Abi(d, D)
    key1, fr1 = d["keyframe"], d["frames"]
    key3, fr3 = rgb(key1), [rgb(f) for f in fr1]
    if unaligned:
        key1, key3 = _unaligned(key1), _unaligned(key3)
        fr1, fr3 = [_unaligned(f) for f in fr1], [_unaligned(f) for f in fr3]
    g = torch.Generator(device=DEV).manual_seed(D)
    zp = (1.0 / torch.linspace(0.33, 0.0025, D, device=DEV)).view(1, D, 1, 1)
    zp = (zp * (1.0 + 0.05 * torch.rand(B, D, H, W, device=DEV, generator=g))).contiguous()
    nhwc_types = [None] + ([torch.float32, torch.float16] if D <= 32 and D % 8 == 0 else [])
    n = 0
    for matching in (1, 2, 3):
        for centered in (1, 0):
            for z in (None, zp):
                for dtype in (torch.float32, torch.float16):
                    for nh in nhwc_types:
                        gray = abi.run(key1, fr1, dtype, matching, centered, z, nh, channels=1)
                        rep = abi.run(key3, fr3, dtype, matching, centered, z, nh, channels=3)
                        typed = abi.run(key3, fr3, dtype, matching, centered, z, nh)
                        tag = (matching, centered, z is not None, dtype, nh)
                        assert not torch.isnan(gray[0]).any() and not torch.isnan(gray[1]).any(), tag
                        assert _same(gray, rep), tag
                        assert _same(rep, typed), tag
                        n += 1
    assert n == 3 * 2 * 2 * 2 * len(nhwc_types)


@pytest.mark.parametrize("kw", [dict(), dict(use_ssim=2), dict(use_ssim=3, not_center_cv=True),
                                dict(not_center_cv=True, volume_dtype=torch.float16), dict(use_stereo=True),
                                dict(use_mono=False, use_stereo=True, volume_dtype=torch.float16)], ids=str)
@pytest.mark.parametrize("pixel_depths", [False, True])
def test_module_gray_is_the_replicated_module(kw, pixel_depths):
    from monorec_b200.cost_volume import CostVolumeModule
    d = _gray_inputs(2, 2, 64, 124, seed=31)
    d["stereoframe"] = d["frames"][0].flip(-1).contiguous()
    d["stereoframe_pose"], d["stereoframe_intrinsics"] = d["poses"][1], d["intrinsics"][1]
    d["_cv_range"] = (0.0025, 0.33, 32)
    if pixel_depths:
        d["cv_depths"] = (1.0 / torch.linspace(0.33, 0.0025, 24, device=DEV)).view(1, 24, 1, 1).expand(2, 24, 64, 124)
    m = CostVolumeModule(**kw)
    a = m(dict(d))
    b = m(_rgb_dict(d))
    torch.cuda.synchronize()
    assert torch.equal(a["cost_volume"], b["cost_volume"])
    assert all(torch.equal(x, y) for x, y in zip(a["single_frame_cvs"], b["single_frame_cvs"]))


def test_module_gray_under_torch_compile():
    """The monorec_b200::cost_volume op with C = 1 in a fullgraph compiled module."""
    from monorec_b200.cost_volume import CostVolumeModule
    d = _gray_inputs(1, 2, 48, 96, seed=33)
    d["_cv_range"] = (0.0025, 0.33, 32)
    m = CostVolumeModule()
    keys = ("keyframe", "frames", "poses", "intrinsics", "keyframe_pose", "keyframe_intrinsics")

    def f(*xs):
        dd = dict(zip(keys, xs))
        dd["_cv_range"] = (0.0025, 0.33, 32)
        out = m(dd)
        return out["cost_volume"], out["single_frame_cvs"]
    cf = torch.compile(f, fullgraph=True)
    cv, sf = cf(*[d[k] for k in keys])
    ref = m(_rgb_dict(d))
    torch.cuda.synchronize()
    assert torch.equal(cv, ref["cost_volume"]) and all(torch.equal(x, y) for x, y in zip(sf, ref["single_frame_cvs"]))


# ---- the model -------------------------------------------------------------------------------------------------------------
MODEL_KEYS = ("cost_volume", "cv_mask", "result")


def _model(**kw):
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import seeded_state_dict
    m = MonoRecModel(**kw)
    m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
    return m.to(DEV).eval()


def _model_inputs(B=2, H=64, W=128, seed=41, stereo=False, mvobj=False):
    d = _gray_inputs(B, 2, H, W, seed)
    if stereo:
        d["stereoframe"] = d["frames"][1].flip(-1).contiguous()
        d["stereoframe_pose"], d["stereoframe_intrinsics"] = d["poses"][1], d["intrinsics"][1]
    if mvobj:
        d["mvobj_mask"] = (torch.rand(B, 1, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5)) > 0.7).float()
    return d


def _assert_same_outputs(a, b):
    for k in MODEL_KEYS:
        if k in b:
            assert torch.equal(a[k], b[k]), k
    assert all(torch.equal(x, y) for x, y in zip(a["single_frame_cvs"], b["single_frame_cvs"]))
    if "predicted_inverse_depths" in b:
        assert all(torch.equal(x, y) for x, y in zip(a["predicted_inverse_depths"], b["predicted_inverse_depths"]))


@pytest.mark.parametrize("mode", ["fp32", "tf32", "f16"])
@pytest.mark.parametrize("pretrain_mode,use_stereo", [(0, False), (1, False), (2, False), (3, False), (0, True)])
def test_model_gray_is_the_replicated_model(mode, pretrain_mode, use_stereo):
    """MonoRecModel eager and by CUDA-graph replay: every output of the gray dict is the replicated dict's; the keyframe
    given stays the one-channel tensor."""
    from monorec_b200 import conv as C
    from monorec_b200.model import GraphedMonoRec
    old = C.MODE
    C.set_mode(mode)
    try:
        m = _model(pretrain_mode=pretrain_mode, use_stereo=use_stereo)
        d = _model_inputs(stereo=use_stereo, mvobj=pretrain_mode == 3)
        with torch.no_grad():
            ref = m(_rgb_dict(d))
            got = m(dict(d))
            torch.cuda.synchronize()
            _assert_same_outputs(got, ref)
            assert got["keyframe"].shape[1] == 1 and "_keyframe_rgb" not in got
            gr = GraphedMonoRec(m, d)
            rep = gr(d)
            torch.cuda.synchronize()
            _assert_same_outputs(rep, ref)
            dp = torch.nn.DataParallel(m, device_ids=[0])(dict(d))
            torch.cuda.synchronize()
            _assert_same_outputs(dp, ref)
    finally:
        C.set_mode(old)


def test_model_gray_under_torch_compile():
    from monorec_b200 import conv as C
    old = C.MODE
    C.set_mode("f16")
    try:
        m = _model()
        d = _model_inputs()
        with torch.no_grad():
            ref = m(_rgb_dict(d))
            cm = torch.compile(m, fullgraph=True)
            got = cm(dict(d))
            torch.cuda.synchronize()
        _assert_same_outputs(got, ref)
    finally:
        C.set_mode(old)


# ---- frame streams ---------------------------------------------------------------------------------------------------------
SH, SW = 64, 128
NAMES = ["abs_rel_sparse_metric", "a1_sparse_metric", "rmse_sparse_metric", "abs_rel_sparse_onlydynamic_metric",
         "abs_rel_metric", "sc_inv_metric"]


def _stream(n, seed):
    from monorec_b200.synthetic import make_sequence
    images, poses, Ks = make_sequence(n, SH, SW, seed=seed)
    right = make_sequence(n, SH, SW, seed=seed + 50)[0]
    base = torch.eye(4)
    base[0, 3] = 0.54
    g = torch.Generator().manual_seed(seed + 100)
    target = torch.rand(n, 1, SH, SW, generator=g) * 0.2 + 0.01
    target[torch.rand(n, 1, SH, SW, generator=g) > 0.25] = 0.0
    mask = (torch.rand(n, 1, SH, SW, generator=g) > 0.7).float()
    # the grayscale stream: one plane per image, and its replica for the colour run
    return dict(gray=images[:, :1].contiguous(), rep=images[:, :1].expand(-1, 3, -1, -1).contiguous(), poses=poses, Ks=Ks,
                right=right[:, :1].contiguous(), right_rep=right[:, :1].expand(-1, 3, -1, -1).contiguous(),
                right_poses=poses @ base, target=target, mask=mask)


def _push(obj, st, n, color, stereo, mvobj, target=True):
    kw = {}
    if stereo:
        kw["stereo"] = (st["right_rep" if color else "right"][n], st["right_poses"][n], st["Ks"][n])
    if mvobj:
        kw["mvobj_mask"] = st["mask"][n]
    args = (st["rep" if color else "gray"][n], st["poses"][n], st["Ks"][n]) + ((st["target"][n],) if target else ())
    return obj.push(*args, **kw)


@pytest.mark.parametrize("stereo,mvobj,keys", [(False, False, False), (True, True, True)])
def test_sequence_gray_is_the_replicated_sequence(stereo, mvobj, keys):
    """MonoRecSequence(use_color=False) against the colour sequence on the replicated frames, key frame by key frame; the
    SequenceEvaluater logs of both are equal."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.sequence import MonoRecSequence
    m = _model(use_stereo=stereo, pretrain_mode=3 if mvobj else 0)
    st = _stream(17, seed=61)
    kl = [1, 2, 4, 5, 6, 9, 10, 11, 14] if keys else None
    runs = []
    for color in (False, True):
        seq = MonoRecSequence(m, batch_size=4, stereo=stereo, mvobj_masks=mvobj, keys=kl, use_color=color)
        ev = SequenceEvaluater(seq, NAMES, 3)
        outs = []
        with torch.no_grad():
            for n in range(17):
                if not seq.needs(n):
                    ev.skip()
                    continue
                outs += [(i, {k: v.clone() for k, v in o.items() if torch.is_tensor(v)})
                         for i, o in _push(ev, st, n, color, stereo, True)]
            outs += [(i, {k: v.clone() for k, v in o.items() if torch.is_tensor(v)}) for i, o in ev.flush()]
        torch.cuda.synchronize()
        runs.append((outs, ev.log()))
    (g_out, g_log), (c_out, c_log) = runs
    assert [i for i, _ in g_out] == [i for i, _ in c_out] and g_out
    for (_, a), (_, b) in zip(g_out, c_out):
        for k in ("result", "cv_mask", "cost_volume"):
            if k in b:
                assert torch.equal(a[k], b[k]), k
        assert a["keyframe"].shape[1] == 1 and torch.equal(rgb(a["keyframe"]), b["keyframe"])
    assert json.dumps(g_log, sort_keys=True) == json.dumps(c_log, sort_keys=True)


def test_pointcloud_gray_is_the_replicated_pointcloud():
    """sequence_pointcloud over the gray sequence writes the replicated sequence's PLY, byte for byte.  As in
    tests/test_sequence.py, the model runs without its MaskModule (pretrain_mode 1) and with a depth range inside the
    saver's [3, 20] m, so that the cloud has vertices."""
    from monorec_b200.pointcloud import PLYSaver, sequence_pointcloud
    from monorec_b200.sequence import MonoRecSequence
    m = _model(pretrain_mode=1, inv_depth_min_max=(0.33, 0.06))
    st = _stream(13, seed=71)
    plys = []
    for color in (False, True):
        saver = PLYSaver(SH, SW, min_d=3, max_d=20, batch_size=4)
        pc = sequence_pointcloud(MonoRecSequence(m, batch_size=4, use_color=color), saver)
        with torch.no_grad():
            for n in range(13):
                _push(pc, st, n, color, False, False, target=False)
            pc.flush()
        buf = io.BytesIO()
        saver.save(buf)
        plys.append(buf.getvalue())
    assert len(plys[0]) > 200 and plys[0] == plys[1]


def test_multi_model_gray_results_json():
    """MultiModelEvaluater(use_color=False): the results.json list equals the replicated stream's."""
    from monorec_b200.models_eval import MultiModelEvaluater
    ms = [_model(), _model(use_ssim=2)]
    st = _stream(13, seed=81)
    res = []
    for color in (False, True):
        ev = MultiModelEvaluater(ms, NAMES[:3], 3, seq_batch=4, use_color=color)
        with torch.no_grad():
            for n in range(13):
                _push(ev, st, n, color, False, False)
            ev.flush()
        res.append(json.dumps(ev.results({"dataset_dir": "data/dataset"}), sort_keys=True, default=str))
    assert res[0] == res[1]
