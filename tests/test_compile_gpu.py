"""MonoRecModel under torch.compile and torch.export: the library's launches as `monorec_b200::*` custom operators
(monorec_b200/ops.py).  The compiled forward is one graph, gives the eager forward's bits, follows weight reloads, and
leaves the eager path's launches as they were."""
import io

import numpy as np
import pytest
import torch

import monorec_b200.model as M
from monorec_b200 import _lib, ops
from monorec_b200 import conv as C
from monorec_b200.synthetic import make_inputs, seeded_state_dict, to_device
from tests.helpers import GOLDEN, kitti_sample_dict

DEV = "cuda:0"
pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_dynamo():
    torch._dynamo.reset()
    saved = C.MODE
    yield
    C.set_mode(saved)
    torch._dynamo.reset()


def _model(seed=7, gain=0.7, **kw):
    model = M.MonoRecModel(**kw)
    model.load_state_dict(seeded_state_dict(model, seed=seed, gain=gain))
    return model.to(DEV).eval()


def _synth():
    g = np.load(GOLDEN / "model_synth_small.npz")
    B, nF, D, H, W, seed, wseed = [int(v) for v in g["cfg"]]
    return to_device(make_inputs(B, nF, H, W, seed=seed), DEV)


def _kitti():
    return to_device(kitti_sample_dict()[0], DEV)


def _cv_depths(d, D=32, seed=3):
    B, _, H, W = d["keyframe"].shape
    g = torch.Generator().manual_seed(seed)
    planes = 1.0 / torch.linspace(0.0025, 0.33, D).view(1, D, 1, 1)
    return (planes * (1 + 0.05 * torch.rand(B, D, H, W, generator=g))).to(DEV)


def _fresh(d):
    """A new dict with the same tensors (the forward writes its outputs into the dict it is given)."""
    return {k: (list(v) if isinstance(v, list) else v) for k, v in d.items()}


def _tensors(out):
    """Every tensor of an output dict by name (lists flattened; cv_module_time is host time, 0 under compile)."""
    flat = {}
    for k, v in out.items():
        if k == "cv_module_time":
            continue
        if torch.is_tensor(v):
            flat[k] = v
        elif isinstance(v, list):
            for i, t in enumerate(list(v)):    # (evaluates the eager trunk's lazy level 4)
                flat[f"{k}[{i}]"] = t
    return flat


def _assert_bitwise(got, ref):
    g, r = _tensors(got), _tensors(ref)
    assert sorted(g) == sorted(r)
    for k in r:
        assert g[k].shape == r[k].shape and g[k].dtype == r[k].dtype, k
        assert torch.equal(g[k], r[k]), f"{k}: max|d| {(g[k].float() - r[k].float()).abs().max().item()}"


CASES = [  # (data, mode, volume dtype, use_ssim, per-pixel depths)
    ("kitti", "fp32", torch.float32, True, False),
    ("kitti", "tf32", torch.float32, True, False),
    ("kitti", "f16", torch.float32, True, False),
    ("kitti", "f16", torch.float16, True, False),
    ("synth", "tf32", torch.float32, True, True),
    ("synth", "f16", torch.float16, True, True),
    ("synth", "tf32", torch.float32, 2, False),
    ("synth", "f16", torch.float16, 2, True),
]


def _case(data, mode, vdt, use_ssim, depths):
    C.set_mode(mode)
    model = _model(volume_dtype=vdt, use_ssim=use_ssim)
    d = _kitti() if data == "kitti" else _synth()
    if depths:
        d["cv_depths"] = _cv_depths(d)
    return model, d


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-{c[1]}-{str(c[2])[6:]}-ssim{int(c[3])}-{'depths' if c[4] else 'planes'}")
def test_aot_eager_fullgraph_is_bitwise_eager(case):
    model, d = _case(*case)
    with torch.no_grad():
        ref = model(_fresh(d))
        got = torch.compile(model, fullgraph=True, backend="aot_eager")(_fresh(d))
    torch.cuda.synchronize()
    assert float(got["cv_module_time"][0]) == 0.0
    _assert_bitwise(got, ref)


@pytest.mark.parametrize("mode", ["fp32", "tf32", "f16"])
def test_inductor_fullgraph_within_golden_gates(mode):
    """Inductor compiles only the few element-wise ops around the library's ops: the result stays within the gates of
    tests/test_convnet_gpu.py against the reference, and equals eager bit for bit."""
    try:
        import triton  # noqa: F401
    except ImportError:
        pytest.skip("Inductor needs Triton, which cannot be imported here")
    from tests.test_convnet_gpu import _ref_noise
    g = np.load(GOLDEN / "model_kitti_sample.npz")
    C.set_mode(mode)
    model = _model(seed=int(g["wseed"][0]), gain=0.7)
    d = _kitti()
    with torch.no_grad():
        ref = model(_fresh(d))
        out = torch.compile(model, fullgraph=True)(_fresh(d))
    torch.cuda.synchronize()
    dr = np.abs(out["result"].float().cpu().numpy() - g["g07_result"])
    dmask = np.abs(out["cv_mask"].float().cpu().numpy() - g["g07_cv_mask"].astype(np.float32))
    n_res, n_mask = _ref_noise("kitti", "g07")
    share = float((dr < 1e-3).mean())
    same = all(torch.equal(a, b) for a, b in zip(_tensors(out).values(), _tensors(ref).values()))
    print(f"inductor {mode}: result max|d| {dr.max():.3e}, share within 1e-3 {share:.5f}, mask max|d| {dmask.max():.3e}, "
          f"bitwise equal to eager: {same}")
    if mode == "fp32":
        assert dr.max() < max(1e-4, 4 * n_res) and share > 0.999
        assert dmask.max() < max(1e-3, 4 * n_mask)
    else:
        assert dr.max() < max(1e-2, 4 * n_res) and share > 0.99
        assert dmask.max() < max(2e-2, 4 * n_mask) and float((dmask < 5e-3).mean()) > 0.99
    assert same


def test_one_graph_no_breaks_no_recompile():
    C.set_mode("f16")
    model, d = _model(volume_dtype=torch.float16), _synth()
    with torch.no_grad():
        ex = torch._dynamo.explain(model)(_fresh(d))
    assert ex.graph_count == 1 and ex.graph_break_count == 0, ex.break_reasons
    torch._dynamo.reset()
    compiled = []

    def backend(gm, example_inputs):
        compiled.append(gm)
        return gm.forward
    f = torch.compile(model, backend=backend, fullgraph=True)
    with torch.no_grad():
        a = f(_fresh(d))
        b = f(_fresh(d))
    torch.cuda.synchronize()
    assert len(compiled) == 1
    assert torch.equal(a["result"], b["result"])


def test_load_state_dict_between_compiled_calls():
    """The packed-weight lookup runs inside the ops on real tensors: new weights are seen by the next compiled call."""
    C.set_mode("tf32")
    model, d = _model(seed=7), _synth()
    f = torch.compile(model, fullgraph=True, backend="aot_eager")
    with torch.no_grad():
        first = f(_fresh(d))
        model.load_state_dict(seeded_state_dict(model, seed=8, gain=0.7))
        second = f(_fresh(d))
        ref = _model(seed=8)(_fresh(d))
    torch.cuda.synchronize()
    assert not torch.equal(first["result"], second["result"])
    _assert_bitwise(second, ref)


class _Wrap(torch.nn.Module):
    """Tensor-in / tensor-out face of the forward, as torch.export needs it."""

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, keyframe, keyframe_pose, keyframe_intrinsics, frames, poses, intrinsics):
        out = self.model({"keyframe": keyframe, "keyframe_pose": keyframe_pose, "keyframe_intrinsics": keyframe_intrinsics,
                          "frames": list(frames), "poses": list(poses), "intrinsics": list(intrinsics)})
        return out["result"], out["cv_mask"], out["cost_volume"], tuple(out["predicted_inverse_depths"])


def test_export_and_save_load_round_trip():
    """The exported program computes with the weights it holds: after a save, new weights in the original model change
    neither the loaded program's output nor the saved one's."""
    C.set_mode("f16")
    model, d = _model(), _synth()
    w = _Wrap(model)
    args = (d["keyframe"], d["keyframe_pose"], d["keyframe_intrinsics"], tuple(d["frames"]), tuple(d["poses"]),
            tuple(d["intrinsics"]))
    flat = lambda t: [x for v in t for x in (v if isinstance(v, tuple) else (v,))]   # noqa: E731
    with torch.no_grad():
        ref = w(*args)
        ep = torch.export.export(w, args)
        got = ep.module()(*args)
        buf = io.BytesIO()
        torch.export.save(ep, buf)
        model.load_state_dict(seeded_state_dict(model, seed=8, gain=0.7))     # the original moves on
        changed = w(*args)
        buf.seek(0)
        again = torch.export.load(buf).module()(*args)
    torch.cuda.synchronize()
    assert not torch.equal(changed[0], ref[0])
    for out in (got, again):
        assert all(torch.equal(a, b) for a, b in zip(flat(out), flat(ref)))


def test_compiled_reprojection_loss_gradient_is_bitwise_eager():
    from monorec_b200.losses import reprojection_loss
    from tests.helpers import reprojection_inputs
    d, invd, _ = reprojection_inputs()
    d = to_device(d, DEV)
    invd = invd.to(DEV)

    def loss(x):
        return reprojection_loss(x, d, automasking=True, use_stereo=True).sum() + reprojection_loss(x, d, border=3).sum()
    grads = []
    for fn in (loss, torch.compile(loss, fullgraph=True, backend="aot_eager")):
        x = invd.clone().requires_grad_(True)
        value = fn(x)
        value.backward()
        grads.append((value.detach(), x.grad))
    torch.cuda.synchronize()
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    assert grads[0][1].abs().sum() > 0


def test_compiled_metrics_are_bitwise_eager():
    from monorec_b200 import metrics as MT
    g = torch.Generator().manual_seed(5)
    pred = (torch.rand(2, 1, 48, 80, generator=g) * 0.3 + 0.01).to(DEV)
    gt = torch.where(torch.rand(2, 1, 48, 80, generator=g) < 0.3, 0.0, torch.rand(2, 1, 48, 80, generator=g) * 0.3 + 0.01).to(DEV)

    def evaluate(p, t):
        dd = {"result": p, "target": t}
        scaled = MT.median_scaling(dd)
        return MT.sparse_metrics(scaled, roi=[4, 44, 8, 72], max_distance=80.0), MT.dense_metrics(p, t, None, 80.0), \
            scaled["result"]
    ref = evaluate(pred, gt)
    MT._dense_last[0] = None
    got = torch.compile(evaluate, fullgraph=True, backend="aot_eager")(pred, gt)
    torch.cuda.synchronize()
    for a, b in zip(got, ref):
        assert torch.equal(torch.nan_to_num(a, 7.0), torch.nan_to_num(b, 7.0))


@pytest.mark.parametrize("B,H,W", [(1, 64, 128), (2, 96, 160)])
def test_opcheck_every_op(B, H, W):
    """torch.library.opcheck (schema, fake against real outputs, declared mutations, autograd registration) on every op,
    with small real inputs of two shapes."""
    from monorec_b200 import losses as L
    C.set_mode("f16")
    model = _model(volume_dtype=torch.float16)
    d = to_device(make_inputs(B, 2, H, W, seed=B), DEV)
    kf = d["keyframe"]
    nF = len(d["frames"])
    nhwc = torch.empty(nF * B, H, W, 32, device=DEV, dtype=torch.float16)
    cv_args = (kf, d["frames"], d["intrinsics"], d["poses"], d["keyframe_pose"], d["keyframe_intrinsics"], None, nhwc,
               0.0025, 0.33, 32, 10.0, [5 / 32, 16 / 32, 11 / 32], 1, True, True)
    torch.library.opcheck(ops.cost_volume, cv_args)
    torch.library.opcheck(ops.cost_volume, cv_args[:6] + (_cv_depths(d, 16), None) + cv_args[8:14] + (False, False))
    cv, sfcv = ops.cost_volume(*cv_args)
    enc, att, dep = model._feature_extractor, model.att_module, model.depth_module
    image = (kf + .5).contiguous(memory_format=torch.channels_last)
    fc = [64, 64, 128, 256, 512]
    with torch.no_grad():
        trunk_args = (image, [t.detach() for t in enc._source_tensors()], True)
        torch.library.opcheck(ops.resnet_trunk, trunk_args)
        feats = ops.resnet_trunk(*trunk_args)
        mp = [p.detach() for p in att.parameters()]
        for buf in (nhwc, None):
            torch.library.opcheck(ops.mask_module, ([s for s in sfcv], feats[:4], buf, mp, 32, fc, True, True))
        mask = ops.mask_module([s for s in sfcv], feats[:4], nhwc, mp, 32, fc, True, True)
        dp = [p.detach() for p in dep.parameters()]
        torch.library.opcheck(ops.depth_module, (kf, cv, feats[:3], mask, 0.0025, 0.3275, dp, 32, fc))
        torch.library.opcheck(ops.mask_volume, (cv, mask))
        torch.library.opcheck(ops.mask_volume, (cv.float(), mask))
        depth = 1.0 / ops.depth_module(kf, cv, feats[:3], mask, 0.0025, 0.3275, dp, 32, fc)[0]
        gt = torch.where(torch.rand_like(depth) < 0.5, torch.zeros_like(depth), depth * 1.1)
        torch.library.opcheck(ops.sparse_metrics, (depth, gt, mask, [0, H, 0, W], 80.0, False))
        torch.library.opcheck(ops.sparse_metrics, (depth, gt, None, None, 0.0, True))
        torch.library.opcheck(ops.dense_metrics, (depth, gt, [2, H - 2, 2, W - 2], 0.0125))
        torch.library.opcheck(ops.median_scaling, (depth, gt))
    invd = (0.05 + 0.2 * torch.rand(B, 1, H, W, device=DEV)).requires_grad_(True)
    loss_args = (invd, kf, d["frames"], d["keyframe_pose"], d["keyframe_intrinsics"], d["poses"], d["intrinsics"], True, 1)
    torch.library.opcheck(ops.reprojection_loss_fwd, loss_args)
    errors, winner, proj = ops.reprojection_loss_fwd(*loss_args)
    g = torch.where(torch.isinf(errors), 0.0, 1.0).detach()
    torch.library.opcheck(ops.reprojection_loss_bwd, (kf, d["frames"], proj.detach(), invd.detach(), g, winner))
    # the op's autograd formula is the eager autograd.Function's
    (errors.nan_to_num(0.0, 0.0, 0.0) * g).sum().backward()
    x = invd.detach().clone().requires_grad_(True)
    e, _ = L.reprojection_errors(x, d, automasking=True, border=1)
    (e.nan_to_num(0.0, 0.0, 0.0) * g).sum().backward()
    assert torch.equal(invd.grad, x.grad)


@pytest.mark.parametrize("mode", ["tf32", "f16"])
def test_eager_launch_count_unchanged(mode):
    """The eager forward issues the library launches it issued before the ops existed (no op dispatch, no extra work):
    the counts are those of the forward of the previous release on this input."""
    C.set_mode(mode)
    model, d = _model(), _synth()
    with torch.no_grad():
        model(_fresh(d))
        torch.cuda.synchronize()
        _lib.launch_count(reset=True)
        model(_fresh(d))
        n = _lib.launch_count(reset=True)
    assert n == EAGER_LAUNCHES[mode]


EAGER_LAUNCHES = {"tf32": 69, "f16": 69}     # the forward before the ops existed, on the model_synth_small input
