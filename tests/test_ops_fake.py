"""The fake (meta) implementations of the `monorec_b200::*` ops (monorec_b200/ops.py) give the shapes, dtypes and strides of
the eager outputs, and each op's schema is the signature of the function it runs.  CPU only: FakeTensorMode makes CUDA
tensors without a device."""
import inspect

import pytest
import torch
import torchvision
from torch._subclasses.fake_tensor import FakeTensorMode

import monorec_b200.model as M
from monorec_b200 import conv as C
from monorec_b200 import cost_volume as CV
from monorec_b200 import metrics as MT
from monorec_b200 import ops

GRID = [(1, 2, 32, 64, 128), (2, 3, 16, 96, 160), (3, 1, 8, 32, 64)]     # B, F, D, H, W


@pytest.fixture
def mode():
    saved = C.MODE
    yield C.set_mode
    C.set_mode(saved)


def _args(op):
    return [a.name for a in op._opoverload._schema.arguments]


def test_schemas_are_the_signatures_of_the_functions_they_run():
    assert _args(ops.cost_volume) == list(inspect.signature(CV.launch).parameters)
    assert _args(ops.mask_volume) == list(inspect.signature(C.mask_volume_impl).parameters)
    assert _args(ops.mask_module) == ["single_frame_cvs", "image_features", "sfcv_nhwc", "params", "depth_steps",
                                      "feature_channels", "use_cv", "use_features"]
    assert list(inspect.signature(M.MaskModule._run).parameters) == ["self", "sfcvs", "feats_nchw", "x"]
    assert _args(ops.depth_module) == ["keyframe", "cost_volume", "image_features", "cv_mask", "out_a", "out_b", "params",
                                       "depth_steps", "feature_channels"]
    assert list(inspect.signature(M.DepthModule._run).parameters) == ["self", "keyframe", "cv", "feats_nchw", "cv_mask",
                                                                       "out_range"]
    assert _args(ops.resnet_trunk) == ["image", "params", "allow_tf32"]
    assert _args(ops.sparse_metrics) == list(inspect.signature(MT.sparse_metrics_impl).parameters)
    assert _args(ops.dense_metrics) == list(inspect.signature(MT.dense_metrics_impl).parameters)
    assert _args(ops.median_scaling) == list(inspect.signature(MT.median_scaling_impl).parameters)
    for name, op in ops.OPS.items():
        schema = op._opoverload._schema
        assert schema.name == f"monorec_b200::{name}"
        mutated = [a.name for a in schema.arguments if a.alias_info is not None and a.alias_info.is_write]
        assert mutated == (["sfcv_nhwc"] if name == "cost_volume" else [])


@pytest.mark.parametrize("B,F,D,H,W", GRID)
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("pixel_depths", [False, True])
def test_cost_volume_fake(B, F, D, H, W, half, pixel_depths):
    with FakeTensorMode():
        e = lambda *s: torch.empty(*s, device="cuda")    # noqa: E731
        frames = [e(B, 3, H, W) for _ in range(F)]
        z = e(B, D, H, W) if pixel_depths else None
        nhwc = e(F * B, H, W, D).half() if D % 8 == 0 and D <= 32 else None
        cv, sf = torch.ops.monorec_b200.cost_volume(e(B, 3, H, W), frames, [e(B, 4, 4) for _ in range(F)],
                                                    [e(B, 4, 4) for _ in range(F)], e(B, 4, 4), e(B, 4, 4), z, nhwc,
                                                    0.0025, 0.33, 7 if pixel_depths else D, 10.0, [1 / 3] * 3, 1, True, half)
    dt = torch.float16 if half else torch.float32
    assert cv.shape == (B, D, H, W) and sf.shape == (F, B, D, H, W) and cv.dtype == sf.dtype == dt
    assert cv.is_contiguous() and sf.is_contiguous() and cv.device.type == "cuda"


@pytest.mark.parametrize("B,H,W", [(1, 64, 128), (2, 96, 160), (3, 37, 61)])
@pytest.mark.parametrize("m", ["fp32", "tf32", "f16"])
def test_resnet_trunk_fake_matches_torchvision(B, H, W, m, mode):
    """Shapes against torchvision's own ResNet-18 on the meta device; channels-last strides, half in f16 mode."""
    mode(m)
    r = torchvision.models.resnet18().to("meta").to(memory_format=torch.channels_last)
    x = torch.empty(B, 3, H, W, device="meta").contiguous(memory_format=torch.channels_last)
    ref = [r.relu(r.bn1(r.conv1(x)))]
    ref.append(r.layer1(r.maxpool(ref[-1])))
    for layer in (r.layer2, r.layer3, r.layer4):
        ref.append(layer(ref[-1]))
    with FakeTensorMode():
        image = torch.empty(B, 3, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
        feats = torch.ops.monorec_b200.resnet_trunk(image, [], m != "fp32")
    assert len(feats) == 5
    for f, g in zip(feats, ref):
        assert f.shape == g.shape
        assert f.stride() == torch.empty(g.shape, device="meta", memory_format=torch.channels_last).stride()
        assert f.dtype == (torch.float16 if m == "f16" else torch.float32)


@pytest.mark.parametrize("B,F,D,H,W", GRID)
def test_module_ops_fake(B, F, D, H, W):
    with FakeTensorMode():
        e = lambda *s: torch.empty(*s, device="cuda")    # noqa: E731
        feats = [e(B, c, H >> (i + 1), W >> (i + 1)) for i, c in enumerate((64, 64, 128, 256))]
        mask = torch.ops.monorec_b200.mask_module([e(B, D, H, W) for _ in range(F)], feats, None, [], D,
                                                   [64, 64, 128, 256, 512], True, True)
        preds = torch.ops.monorec_b200.depth_module(e(B, 3, H, W), e(B, D, H, W).half(), feats[:3], mask, 0.0025, 0.3, [], D,
                                                    [64, 64, 128, 256, 512])
        masked = torch.ops.monorec_b200.mask_volume(e(B, D, H, W).half(), mask)
    assert mask.shape == (B, 1, H, W) and mask.dtype == torch.float32 and mask.is_contiguous()
    assert [tuple(p.shape) for p in preds] == [(B, 1, H >> s, W >> s) for s in range(4)]
    assert all(p.dtype == torch.float32 and p.is_contiguous() for p in preds)
    assert masked.shape == (B, D, H, W) and masked.dtype == torch.float16 and masked.is_contiguous()


@pytest.mark.parametrize("B,F,H,W", [(1, 2, 48, 80), (3, 1, 32, 64)])
def test_metric_and_loss_fakes(B, F, H, W):
    with FakeTensorMode():
        e = lambda *s: torch.empty(*s, device="cuda")    # noqa: E731
        pred, gt = e(B, 1, H, W), e(B, 1, H, W)
        sparse = torch.ops.monorec_b200.sparse_metrics(pred, gt, None, [0, H, 0, W], 80.0, True)
        dense = torch.ops.monorec_b200.dense_metrics(pred, gt, None, 0.0125)
        scaled = torch.ops.monorec_b200.median_scaling(pred, gt)
        frames = [e(B, 3, H, W) for _ in range(F)]
        errors, winner, proj = torch.ops.monorec_b200.reprojection_loss_fwd(
            pred.half(), e(B, 3, H, W), frames, e(B, 4, 4), e(B, 4, 4), [e(B, 4, 4)] * F, [e(B, 4, 4)] * F, True, 2)
        grad = torch.ops.monorec_b200.reprojection_loss_bwd(e(B, 3, H, W), frames, proj, pred.half(), errors, winner)
    assert sparse.shape == (7,) and dense.shape == (12,) and scaled.shape == (B, 1, H, W)
    assert errors.shape == winner.shape == (B, H, W) and winner.dtype == torch.int32 and proj.shape == (B, F, 12)
    assert grad.shape == (B, 1, H, W) and grad.dtype == torch.float16
