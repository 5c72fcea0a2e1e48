"""Host-side logic that needs no GPU: checkpoint contract, padding arithmetic, descriptor ABI, weight packing."""
import ctypes
from pathlib import Path

import pytest
import torch


def test_reference_checkpoint_loads(tmp_path):
    """Checkpoint contract (base/base_trainer.py:142-150, utils/util.py:244-248): DataParallel-prefixed state_dict."""
    from monorec_b200.model import MonoRecModel
    from monorec_b200.synthetic import seeded_state_dict
    src = MonoRecModel()
    sd = seeded_state_dict(src, seed=3, gain=1.0)
    torch.save({"arch": "DataParallel", "state_dict": {"module." + k: v for k, v in sd.items()}}, tmp_path / "cp.pth")
    m = MonoRecModel(checkpoint_location=[tmp_path / "cp.pth"])
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    torch.save({"arch": "MonoRecModel", "state_dict": sd}, tmp_path / "cp2.pth")
    m2 = MonoRecModel(mask_cp_loc=tmp_path / "cp2.pth", depth_cp_loc=tmp_path / "cp2.pth")
    assert torch.equal(m2.att_module.classifier[0].weight, sd["att_module.classifier.0.weight"])
    assert torch.equal(m2.depth_module.dec[4][2].bias, sd["depth_module.dec.4.2.bias"])


def test_same_padding_matches_reference_formula():
    from monorec_b200.conv import same_pad_before
    from oracle.convnet_oracle import same_pad
    for n in (16, 17, 32, 33, 64, 255, 256):
        for k in (1, 2, 3, 5, 7):
            for s in (1, 2):
                assert same_pad_before(n, k, s) == same_pad(n, k, s)[0]


def test_conv_desc_abi_matches_library():
    from monorec_b200 import _lib
    from monorec_b200.conv import ConvDesc
    assert ctypes.sizeof(ConvDesc) == _lib.load().mr_sizeof_conv_desc()


def test_refine_and_upconv_phases_reproduce_reference_layers():
    """The phase convolutions refine_layer and upconv_layer build (packed weights, pad, out_off, activation) reproduce
    ConvTranspose2d(k4, s2) + LeakyReLU + centre crop (Refine, layers.py:380-400) and Upsample(x2) + pad(0,1,0,1) +
    Conv2d(k2) (Upconv, :338-356)."""
    import torch.nn.functional as F
    from monorec_b200 import conv as C
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 8, 6, 7, generator=g)
    convt, conv = torch.nn.ConvTranspose2d(8, 4, 4, stride=2), torch.nn.Conv2d(8, 4, 2)
    with torch.no_grad():
        for p in list(convt.parameters()) + list(conv.parameters()):
            p.copy_(torch.randn(p.shape, generator=g))
        refine = F.leaky_relu(F.conv_transpose2d(x, convt.weight, convt.bias, stride=2)[:, :, 1:-1, 1:-1], C.LEAKY_SLOPE)
        upconv = F.conv2d(F.pad(F.interpolate(x, scale_factor=2, mode="nearest"), (0, 1, 0, 1)), conv.weight, conv.bias)
    for layer, ref in ((C.refine_layer(convt, (8,)), refine), (C.upconv_layer(conv, (8,)), upconv)):
        assert len(layer.subs) == 4
        out = torch.full_like(ref, float("nan"))
        for L in layer.subs:
            assert L.out_step == (2, 2)
            (pt, pl), (oy, ox) = L.pad, L.out_off
            xp = F.pad(x, (pl, L.kw - 1 - pl, pt, L.kh - 1 - pt))         # pixels beyond the trailing border are zero
            y = F.conv2d(xp, L.w32.permute(3, 2, 0, 1), L.bias)           # w32: [kh][kw][Cin][Cout]
            out[:, :, oy::2, ox::2] = F.leaky_relu(y, L.act_a) if L.act == C.ACT_LEAKY else y
        assert torch.allclose(out, ref, atol=1e-5)


def test_unsupported_reference_options_raise():
    from monorec_b200.model import MonoRecModel
    for kw in ({"simple_mask": True}, {"depth_large_model": True}, {"augmentation": "depth"}, {"use_ssim": False},
               {"cv_patch_size": 5}, {"sfcv_mult_mask": False}):
        with pytest.raises(NotImplementedError):
            MonoRecModel(**kw)
    m = MonoRecModel(pretrain_mode=2)
    assert hasattr(m, "att_module") and not hasattr(m, "depth_module")
    m = MonoRecModel(pretrain_mode=1)
    assert hasattr(m, "depth_module") and not hasattr(m, "att_module")


def test_trunk_batchnorm_folding_matches_unfolded_eval():
    """ResnetEncoder's inference path folds eval-mode BatchNorm into the convolutions (monorec_model.py:118-129 semantics);
    the folded copy must track parameter updates."""
    from monorec_b200.model import ResnetEncoder
    torch.manual_seed(0)
    enc = ResnetEncoder(18, pretrained=False).eval()
    for m in enc.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.5)
            m.running_var.uniform_(0.5, 2.0)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    x = torch.rand(2, 3, 64, 128)
    with torch.enable_grad():
        ref = [t.detach().clone() for t in enc(x)]          # module-by-module path
    with torch.no_grad():
        out = [t.clone() for t in enc(x)]                    # folded path
    assert len(out) == 5
    for a, b in zip(ref, out):
        assert a.shape == b.shape and float((a - b).abs().max()) <= 1e-5 * float(a.abs().max())
    sd = {k: v.clone() for k, v in enc.state_dict().items()}
    sd["encoder.bn1.bias"] += 1.0
    enc.load_state_dict(sd)
    with torch.no_grad():
        out2 = enc(x)[0]
    with torch.enable_grad():
        ref2 = enc(x)[0].detach()
    assert float((out2 - ref2).abs().max()) < 1e-4 and float((out2 - out[0]).abs().max()) > 0.5


def test_tc_weight_packing_follows_source_chunk_widths():
    """Packed tensor-core weights: [taps][n_pad][k_pad], every source padded to whole K chunks; half sources of <= 32
    channels use 32-channel chunks (64-byte swizzle rows; the library derives the chunk width from k_pad:
    include/monorec_b200.h)."""
    from monorec_b200 import conv as C
    w = torch.randn(24, 32, 3, 3)
    wt, n_pad, k_pad = C.pack_tc_weight(w, (32,), half=False)
    assert wt.dtype == torch.float32 and wt.shape == (9, 32, 32) and (n_pad, k_pad) == (32, 32)
    assert torch.equal(wt[4, :24, :], _round_tf32(w[:, :, 1, 1])) and float(wt[:, 24:].abs().max()) == 0.0
    wt, n_pad, k_pad = C.pack_tc_weight(w, (32,), half=True)
    assert wt.dtype == torch.float16 and k_pad == 32 and wt.shape == (9, 32, k_pad)
    w2 = torch.randn(48, 96, 3, 3)
    wt, n_pad, k_pad = C.pack_tc_weight(w2, (32, 64), half=True)          # a 64-channel source keeps 64-channel chunks
    assert (n_pad, k_pad) == (48, 128) and torch.equal(wt[0, :, 64:128], w2[:, 32:, 0, 0].half())
    assert float(wt[:, :, 32:64].abs().max()) == 0.0
    s1 = C.PackedConv(w, None, (32,), stride=(1, 1))
    s2 = C.PackedConv(w, None, (32,), stride=(2, 1))
    assert s1.wtc(True)[2] == 32 and s2.wtc(True)[2] == 32


def _round_tf32(w):
    """Round-to-nearest onto the TF32 grid (10 explicit mantissa bits); the tensor core truncates the rest."""
    bits = w.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def _pack_tc_weight_torch(w, src_c, half):
    """The layout of mr_pack_conv_weights written with torch ops: [kh*kw][n_pad][k_pad], every source padded to whole K
    chunks (32 fp32 channels; 64 half channels, or 32 when every source has <= 32 channels)."""
    Cout, Cin, kh, kw = w.shape
    kc = (32 if all(c <= 32 for c in src_c) else 64) if half else 32
    n_pad = ((Cout + 15) // 16) * 16
    k_pad = sum(((c + kc - 1) // kc) * kc for c in src_c)
    out = torch.zeros(kh * kw, n_pad, k_pad, device=w.device, dtype=torch.float32)
    wt = w.detach().to(torch.float32).permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin)
    ci = ko = 0
    for c in src_c:
        out[:, :Cout, ko:ko + c] = wt[:, :, ci:ci + c]
        ci += c
        ko += ((c + kc - 1) // kc) * kc
    return (out.to(torch.float16).contiguous() if half else _round_tf32(out)), n_pad, k_pad


def test_c_packer_matches_layout_restatement():
    """mr_pack_conv_weights (host-side C, include/monorec_b200.h) == the torch restatement of the layout, fp32/TF32 and half,
    one to three concatenated sources, ragged channel counts; padding rows and columns are zero."""
    from monorec_b200 import conv as C
    g = torch.Generator().manual_seed(3)
    for cout, src_c, kh, kw in [(24, (32,), 3, 3), (48, (32, 64), 3, 3), (96, (64, 64, 96), 1, 1), (1, (24,), 3, 3), (13, (40,), 7, 1)]:
        w = torch.randn(cout, sum(src_c), kh, kw, generator=g)
        for half in (False, True):
            got, n_pad, k_pad = C.pack_tc_weight(w, src_c, half=half)
            ref, n_ref, k_ref = _pack_tc_weight_torch(w, src_c, half)
            assert (n_pad, k_pad) == (n_ref, k_ref) and got.dtype == ref.dtype and torch.equal(got, ref), (cout, src_c, half)


def test_c_subpixel_kernels_reproduce_reference_layers():
    """mr_subpixel_convt_k4s2 / mr_subpixel_upconv2: the four phase kernels reproduce ConvTranspose2d(k4, s2) + crop (Refine,
    model/layers.py:380-400) and Upsample(x2) + pad(0,1,0,1) + Conv2d(k2) (Upconv, :338-356)."""
    import ctypes
    import torch.nn.functional as F
    from monorec_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 5, 6, 7, generator=g)
    wt = torch.randn(5, 4, 4, 4, generator=g).contiguous()           # (Cin, Cout, 4, 4)
    ref = F.conv_transpose2d(x, wt, stride=2)[:, :, 1:-1, 1:-1]
    out = torch.zeros_like(ref)
    for py in (0, 1):
        for px in (0, 1):
            sub = torch.empty(4, 5, 2, 2)
            pt, pl = ctypes.c_int(-1), ctypes.c_int(-1)
            assert lib.mr_subpixel_convt_k4s2(wt.data_ptr(), 5, 4, py, px, sub.data_ptr(), ctypes.byref(pt), ctypes.byref(pl)) == 0
            assert (pt.value, pl.value) == (1 - py, 1 - px)
            xp = F.pad(x, (pl.value, 1 - pl.value, pt.value, 1 - pt.value))
            out[:, :, py::2, px::2] = F.conv2d(xp, sub)
    assert torch.allclose(out, ref, atol=1e-5)
    wu = torch.randn(3, 5, 2, 2, generator=g).contiguous()           # (Cout, Cin, 2, 2)
    up = F.interpolate(x, scale_factor=2, mode="nearest")
    ref = F.conv2d(F.pad(up, (0, 1, 0, 1)), wu)
    out = torch.zeros_like(ref)
    for py in (0, 1):
        for px in (0, 1):
            kh, kw = ctypes.c_int(0), ctypes.c_int(0)
            sub = torch.empty(3 * 5 * 4)
            assert lib.mr_subpixel_upconv2(wu.data_ptr(), 3, 5, py, px, sub.data_ptr(), ctypes.byref(kh), ctypes.byref(kw)) == 0
            sub = sub[:3 * 5 * kh.value * kw.value].view(3, 5, kh.value, kw.value)
            xp = F.pad(x, (0, kw.value - 1, 0, kh.value - 1))          # pixel o + 1 beyond the border is the reference's zero pad
            out[:, :, py::2, px::2] = F.conv2d(xp, sub)
    assert torch.allclose(out, ref, atol=1e-5)


def test_integration_builds_from_reference_eval_config(golden_dir):
    """INTEGRATION.md section 2: the reference's evaluation config names the model by type and constructor keywords, and its
    registry resolves it as getattr(module, type)(**args) (utils/parse_config.py, evaluate.py:29-31).  The "models" block of
    configs/evaluate/eval_monorec.json is stored in tests/golden/eval_monorec_models.json; resolved against the drop-in's
    module, every entry constructs the drop-in with the reference's keywords."""
    import json
    import monorec_b200.model as fast
    cfg = json.loads((golden_dir / "eval_monorec_models.json").read_text())
    assert cfg["models"]
    for m in cfg["models"]:
        args = {k: v for k, v in m["args"].items() if k != "checkpoint_location"}   # no checkpoint offline
        model = getattr(fast, m["type"])(**args)
        assert type(model) is fast.MonoRecModel and type(model).__module__ == "monorec_b200.model"
        assert model.use_mono is True and model.use_stereo is False and model.pretrain_mode == 0
        assert tuple(model.inv_depth_min_max) == (0.33, 0.0025)


def test_trunk_level4_is_lazy_and_matches_run_blocks():
    """The 512-channel trunk level has no consumer in the reference (monorec_model.py:372-380, :545 read levels 0-3): it is
    evaluated on first use.  Slices / indices the Mask and Depth modules use do not trigger it; index 4, iteration and
    concatenation do, with the same values as the eager evaluation."""
    import monorec_b200.model as M
    enc = M.ResnetEncoder(18, pretrained=False).eval()
    x = torch.rand(2, 3, 64, 128)
    with torch.no_grad():
        lazy = enc(x)
        assert isinstance(lazy, M._TrunkFeatures) and len(lazy) == 5
        assert len(lazy[:4]) == 4 and lazy[3].shape[1] == 256 and list.__getitem__(lazy, 4) is None      # not evaluated yet
        eager = lazy[:4] + [enc._run_blocks(lazy[3], enc._folded()["blocks"][3])]
    assert list.__getitem__(lazy, 4) is None
    assert torch.equal(lazy[4], eager[4]) and torch.equal(lazy[-1], eager[4])
    with torch.no_grad():
        lazy2 = enc(x)
    assert all(torch.equal(a, b) for a, b in zip(lazy2, eager))                                            # iteration evaluates
    lazy2.reset_tail()
    assert list.__getitem__(lazy2, 4) is None and torch.equal((lazy2 + [])[4], eager[4])
