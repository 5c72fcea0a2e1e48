"""The convolution engine checked bit for bit against an exact reference, on every kernel the host code can choose.

Activations are i * 2^-3 (|i| <= 32), weights and biases j * 2^-4 (|j| <= 8): every value lies on the TF32 and the half grid,
every product is exact in fp32 and every partial sum is a multiple of 2^-7 below 2^17 (oracle.convnet_oracle.conv_engine_ref
asserts it), so the kernel's pre-activation equals the float64 sum whatever the accumulation order.  With no activation or
LeakyReLU every stored element must equal the reference bit for bit; sigmoid / |tanh| go through expf / tanhf and are held to
4 fp32 ulp (1 TF32 / half ulp after output rounding).  Every call writes into a destination pre-filled with a NaN bit
pattern: everything outside the written channel slice and output placement must keep it, everything inside must be
overwritten.  Every tensor-core case also asks the library which kernel it runs (mr_conv2d_nhwc_tc_plan);
test_kernel_coverage fails if a heuristic change moves a path out of reach.
"""
import math
import os
import subprocess
import sys
import zlib
from collections import Counter

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAN32 = 0x7FC0DEAD                      # quiet-NaN payloads no kernel produces
NAN16 = 0x7E5B
HALO_ENV = os.environ.get("MONOREC_B200_TC_HALO")
STREAM_ENV = os.environ.get("MONOREC_B200_TC_STREAM")
NPADS = tuple(range(16, 257, 16))


# ---------------------------------------------------------------------------------------------------------------------
# cases.  ch: source channel counts; k: (kh, kw); s: stride; hw: input (H, W); out_hw: output grid (default: SAME);
# dst_c / coff / step / off / dst_extra: the placement inside the destination, which is dst_extra rows / columns larger than
# the placed output grid
# ---------------------------------------------------------------------------------------------------------------------
def _case(name, ch, cout, k=(3, 3), s=(1, 1), hw=(11, 19), B=2, act=1, act_a=0.1, act_b=1.0, bias=True, round_out=None,
          out_f32=False, coff=0, dst_c=None, dtypes=("tf32", "f16"), pad=None, out_hw=None, step=(1, 1), off=(0, 0), dst_extra=(0, 0)):
    return dict(name=name, ch=tuple(ch), cout=cout, k=k, s=s, hw=hw, B=B, act=act, act_a=act_a, act_b=act_b, bias=bias,
                round_out=round_out, out_f32=out_f32, coff=coff, dst_c=dst_c, dtypes=dtypes, pad=pad, out_hw=out_hw, step=step,
                off=off, dst_extra=dst_extra)


# MMA widths: every n_pad / 16 = 1..16 on the strided tap kernel and on a stride-1 layer, odd Cout among them
_W2 = [13, 17, 48, 64, 80, 96, 112, 128, 144, 160, 176, 192, 208, 224, 240, 241]
_W1 = [1, 32, 47, 64, 80, 96, 112, 128, 144, 160, 176, 192, 208, 224, 239, 256]
TC_CASES = [_case(f"width_s2_c{c}", (40,), c, k=(3, 3), s=(2, 2), hw=(13, 37), B=1) for c in _W2]
TC_CASES += [_case(f"width_s1_c{c}", (40,), c, k=(2, 1), hw=(11, 19), B=1) for c in _W1]
TC_CASES += [
    # sources: tail chunks in the first / middle / last source, 1..3 sources, <= 32 half channels (64-byte rows)
    _case("src_tf32_tail_first_last", (36, 64, 100), 48, dtypes=("tf32",)),
    _case("src_tf32_tail_middle", (64, 12, 32), 40, dtypes=("tf32",)),
    _case("src_tf32_tiny", (4,), 24, dtypes=("tf32",)),
    _case("src_tf32_two_tails_s2", (12, 36), 64, s=(2, 2), dtypes=("tf32",)),
    _case("src_f16_tail_first_last", (72, 64, 40), 48, dtypes=("f16",)),
    _case("src_f16_tail_middle", (64, 24, 128), 40, dtypes=("f16",)),
    _case("src_f16_tiny", (8,), 24, dtypes=("f16",)),
    _case("src_f16_k32_halo", (8, 24, 32), 64, dtypes=("f16",)),
    _case("src_f16_k32_halo_one", (24,), 32, k=(5, 5), dtypes=("f16",)),
    _case("src_f16_k32_tap_s2", (32, 16), 48, s=(2, 2), dtypes=("f16",)),
    _case("src_f16_k32_tap_s21", (24,), 24, k=(5, 1), s=(2, 1), dtypes=("f16",)),
    _case("src_f16_k32_stream", (32, 32, 32), 128, k=(3, 3), dtypes=("f16",)),
    # the model's concatenations (DepthModule, MaskModule decoders)
    _case("cat_depth_192_128_256", (192, 128, 256), 128, k=(3, 1), hw=(6, 10)),
    _case("cat_depth_128_64_128", (128, 64, 128), 64, k=(1, 3), hw=(9, 14)),
    _case("cat_depth_64_64_64", (64, 64, 64), 64, hw=(10, 18)),
    _case("cat_depth_48_48", (48, 48), 48, k=(3, 1), hw=(17, 33)),
    _case("cat_mask_96_256", (96, 256), 256, hw=(5, 9)),
    _case("cat_mask_96_128_96", (96, 128, 96), 128, hw=(7, 11)),
    _case("cat_mask_64_64_96", (64, 64, 96), 96, hw=(9, 17)),
    _case("cat_mask_48_64_96", (48, 64, 96), 64, hw=(12, 20)),
    _case("cat_mask_32_64", (32, 64), 32, hw=(17, 30)),
    # filters, halo limits, strides
    _case("k1x1", (64,), 48, k=(1, 1)),
    _case("k2x2", (32,), 32, k=(2, 2), hw=(12, 17)),
    _case("k5x5", (32,), 32, k=(5, 5)),
    _case("k7x1", (48,), 48, k=(7, 1), hw=(19, 21)),
    _case("k1x7", (48,), 48, k=(1, 7), hw=(13, 29)),
    _case("k3x9_halo_limit", (32,), 32, k=(3, 9), hw=(12, 30)),
    _case("k7x3_halo_limit", (32,), 32, k=(7, 3), hw=(20, 14)),
    _case("k1x10_tap_fallback", (32,), 32, k=(1, 10), hw=(9, 30)),
    _case("k8x1_tap_fallback", (32,), 32, k=(8, 1), hw=(21, 9)),
    _case("k7x7_stream", (64,), 64, k=(7, 7), hw=(14, 22)),
    _case("s21", (48,), 64, k=(5, 1), s=(2, 1), hw=(21, 23)),
    _case("s12", (48,), 64, k=(1, 5), s=(1, 2), hw=(21, 23)),
    _case("s22", (64,), 96, k=(3, 3), s=(2, 2), hw=(19, 35)),
    _case("s33", (32,), 32, k=(3, 3), s=(3, 3), hw=(22, 50)),
    _case("s44", (32,), 16, k=(5, 5), s=(4, 4), hw=(27, 70)),
    # sizes
    _case("out_1x1", (32,), 32, k=(3, 3), s=(4, 4), hw=(3, 4), B=1),
    _case("out_1x1_s1", (16,), 16, k=(3, 3), hw=(1, 1), B=3),
    _case("out_1xW", (32,), 48, k=(3, 3), hw=(1, 37), B=1),
    _case("out_Hx1", (32,), 48, k=(3, 3), hw=(29, 1), B=3),
    _case("out_Hx1_s2", (32,), 48, k=(3, 3), s=(2, 2), hw=(29, 2), B=3),
    _case("many_tiles_halo", (16,), 16, k=(3, 3), hw=(256, 512), B=3),
    _case("many_tiles_tap", (16,), 32, k=(3, 3), s=(2, 1), hw=(256, 1024), B=2),
    # epilogue: activations, output rounding, half / fp32 output, null bias, channel slices
    _case("act_none", (32,), 40, act=0),
    _case("act_leaky_03", (32,), 40, act=1, act_a=0.3, round_out=False),
    _case("act_sigmoid", (32,), 24, act=2, round_out=False),
    _case("act_sigmoid_round", (32,), 24, act=2, round_out=True),
    _case("act_abstanh", (32,), 1, act=3, act_a=0.0025, act_b=0.3275, out_f32=True),
    _case("act_abstanh_s2", (32,), 40, act=3, act_a=0.5, act_b=2.0, s=(2, 2)),
    _case("round_leaky", (32,), 40, round_out=True),
    _case("round_f16", (32,), 40, round_out=True, dtypes=("f16",)),
    _case("final_f32", (48,), 48, out_f32=True, dtypes=("f16",)),
    _case("null_bias", (32,), 40, bias=False),
    _case("slice_even", (32,), 40, coff=8, dst_c=64),
    _case("slice_odd", (32,), 41, coff=3, dst_c=50),
    _case("slice_odd_s2", (32,), 17, coff=5, dst_c=30, s=(2, 2)),
    _case("slice_odd_f32out", (32,), 21, coff=1, dst_c=24, out_f32=True, dtypes=("f16",)),
    # placement: output grid at an offset / step inside a larger destination
    _case("place_offset", (32,), 32, k=(3, 3), hw=(9, 13), off=(2, 5), dst_extra=(2, 3)),
    _case("place_step", (32,), 24, k=(2, 2), hw=(9, 13), step=(2, 3), off=(1, 2), dst_extra=(2, 4), pad=(0, 1)),
]


def _ids(cases):
    return [c["name"] for c in cases]


def _tc_params():
    return [pytest.param(c, dt, id=f"{c['name']}-{dt}") for c in TC_CASES for dt in c["dtypes"]]


# ---------------------------------------------------------------------------------------------------------------------
def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _data(case, key):
    from oracle.convnet_oracle import exact_grid_data
    g = _gen(key, case["name"])
    B, (H, W) = case["B"], case["hw"]
    srcs = [exact_grid_data((B, H, W, c), 32, 3, g) for c in case["ch"]]
    w = exact_grid_data((case["cout"], sum(case["ch"]), *case["k"]), 8, 4, g)
    b = exact_grid_data((case["cout"],), 8, 4, g) if case["bias"] else None
    return srcs, w, b


def _nan_fill(shape, half):
    t = torch.empty(shape, dtype=torch.int16 if half else torch.int32, device=DEV)
    t.fill_(NAN16 if half else NAN32)
    return t.view(torch.float16 if half else torch.float32)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _check_written(out, ref, ys, xs, coff, act, round_out, what):
    """out: destination (NaN-filled before the call); ref: reference values [B, Ho, Wo, Cout] in out's dtype, or float64
    activations for sigmoid / |tanh|; (ys, xs, coff): where they belong."""
    out = out.cpu()
    cout = ref.shape[3]
    inside = torch.zeros(out.shape, dtype=torch.bool)
    inside[:, ys.view(-1, 1), xs.view(1, -1), coff:coff + cout] = True
    nan = NAN16 if out.dtype == torch.float16 else NAN32
    outside = _bits(out)[~inside]
    assert bool((outside == nan).all()), f"{what}: {int((outside != nan).sum())} elements written outside the slice / placement"
    got = out[:, ys.view(-1, 1), xs.view(1, -1), coff:coff + cout]
    if act in (0, 1):
        bad = _bits(got) != _bits(ref)
        if bool(bad.any()):
            i = bad.nonzero()[0].tolist()
            pytest.fail(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at (b, y, x, c) = {i}: "
                        f"{float(got[tuple(i)])} != {float(ref[tuple(i)])}")
    else:
        g64 = got.to(torch.float64)
        if out.dtype == torch.float16:
            tol = 2.0 ** -10 * ref.abs() + 2.0 ** -24                          # 1 half ulp
        elif round_out:
            tol = 2.0 ** -10 * ref.abs() + 2.0 ** -126                         # 1 TF32 ulp
        else:
            tol = 4 * 2.0 ** -23 * ref.abs() + 2.0 ** -126                     # 4 fp32 ulp
        err = (g64 - ref).abs()
        assert bool(torch.isfinite(g64).all()), f"{what}: non-finite outputs (unwritten elements)"
        assert bool((err <= tol).all()), f"{what}: max err {float(err.max())} beyond {float(tol[err > tol].min())}"
    if round_out and out.dtype == torch.float32:
        assert bool(((_bits(got) & 0x1FFF) == 0).all()), f"{what}: stored TF32-mode activations with low mantissa bits set"


def _act64(pre, b, act, act_a, act_b):
    """float64 activation of the exact pre-activation (the fp32 bias add is exact on this data)."""
    v = pre + (b.to(torch.float64) if b is not None else 0.0)
    a, bb = float(torch.tensor(act_a, dtype=torch.float32)), float(torch.tensor(act_b, dtype=torch.float32))
    return torch.sigmoid(v) if act == 2 else a + bb * torch.tanh(v).abs()


def _unpack_check(wtc, w, src_c, half, k_pad):
    """The packed tensor-core weights hold exactly w (RN-to-TF32 / to-half is the identity on this data) and zeros elsewhere."""
    cout, cin, kh, kw = w.shape
    k64 = sum((c + 63) // 64 * 64 for c in src_c)
    kc = (32 if k_pad != k64 else 64) if half else 32
    wt = wtc.cpu().to(torch.float32)
    ref = torch.zeros_like(wt)
    wr = w.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin)
    ci = ko = 0
    for c in src_c:
        ref[:, :cout, ko:ko + c] = wr[:, :, ci:ci + c]
        ci, ko = ci + c, ko + (c + kc - 1) // kc * kc
    assert ko == k_pad and torch.equal(wt, ref), "the packer changed weights that lie on the TF32 / half grid"


def _setup_tc(case, dt):
    """Device tensors, the PackedConv and the NaN-filled destination of one tensor-core case."""
    from monorec_b200 import conv as C
    half = dt == "f16"
    srcs, w, b = _data(case, dt)
    L = C.PackedConv(w.to(DEV), None if b is None else b.to(DEV), case["ch"], stride=case["s"], act=case["act"],
                     act_a=case["act_a"], act_b=case["act_b"], pad=case["pad"], out_step=case["step"], out_off=case["off"])
    dsrcs = [s.to(DEV, torch.float16 if half else torch.float32) for s in srcs]
    Ho, Wo = C._tc_out_hw(dsrcs, L, case["out_hw"])
    dH, dW = [(n - 1) * st + o + 1 + e for n, st, o, e in zip((Ho, Wo), case["step"], case["off"], case["dst_extra"])]
    out_half = half and not case["out_f32"]
    out = _nan_fill((case["B"], dH, dW, case["dst_c"] or case["cout"]), out_half)
    return srcs, w, b, L, dsrcs, (Ho, Wo), out


def _plan(case, dt):
    from monorec_b200 import conv as C
    _, _, _, L, dsrcs, out_hw, out = _setup_tc(case, dt)
    return C.tc_plan(dsrcs, [L], out, out_hw, half=dt == "f16", out_coff=case["coff"])


@pytest.mark.parametrize("case,dt", _tc_params())
def test_tc_conv_exact(case, dt):
    from monorec_b200 import conv as C
    from oracle.convnet_oracle import conv_engine_ref
    half = dt == "f16"
    srcs, w, b, L, dsrcs, out_hw, out = _setup_tc(case, dt)
    wtc, n_pad, k_pad = L.wtc(half)
    _unpack_check(wtc, w, case["ch"], half, k_pad)
    round_out = (not half) if case["round_out"] is None else case["round_out"]
    C.conv2d_tc(dsrcs, L, out=out, out_hw=out_hw, round_out=round_out, half=half, out_f32=case["out_f32"], out_coff=case["coff"])
    torch.cuda.synchronize()
    pad = C._tc_pad(dsrcs, L)
    pre, ref, ys, xs = conv_engine_ref(srcs, w, b, *case["k"], case["s"], pad, out_hw, case["step"], case["off"], case["act"],
                                       case["act_a"], case["act_b"], round_out, out.dtype)
    if case["act"] in (2, 3):
        ref = _act64(pre, b, case["act"], case["act_a"], case["act_b"])
    _check_written(out, ref, ys, xs, case["coff"], case["act"], round_out, f"{case['name']} {dt}")


def test_tc_filter_size_limits_of_the_halo_kernel():
    """kh <= 7 and kw <= 9 reach the halo kernel; kh = 8 or kw = 10 fall back to the tap-refetch kernel."""
    from monorec_b200 import conv as C
    by_name = {c["name"]: c for c in TC_CASES}
    for dt in ("tf32", "f16"):
        for name in ("k3x9_halo_limit", "k7x3_halo_limit"):
            p = _plan(by_name[name], dt)
            assert p["halo_shape"] == (0 if HALO_ENV == "0" else 1)
        for name in ("k1x10_tap_fallback", "k8x1_tap_fallback"):
            p = _plan(by_name[name], dt)
            assert p["halo_shape"] == 0 and p["kernel"] == C.TC_KERNEL_TAP


# ---------------------------------------------------------------------------------------------------------------------
# sub-pixel phases: Refine / Upconv (4 phases) and 2 / 3 phases through the C ABI; the phases must tile the output once
# ---------------------------------------------------------------------------------------------------------------------
def _phase_run(name, dt, subs_w, pads, steps, offs, ch, cout, hw, B, act=1, act_a=0.1, bias=True):
    from monorec_b200 import conv as C
    from oracle.convnet_oracle import conv_engine_ref, exact_grid_data
    half = dt == "f16"
    g = _gen(name, dt)
    H, W = hw
    srcs = [exact_grid_data((B, H, W, c), 32, 3, g) for c in ch]
    b = exact_grid_data((cout,), 8, 4, g) if bias else None
    ws = [wf(g) for wf in subs_w]
    subs = [C.PackedConv(w.to(DEV), None if b is None else b.to(DEV), ch, act=act, act_a=act_a, pad=p, out_step=steps, out_off=o)
            for w, p, o in zip(ws, pads, offs)]
    dsrcs = [s.to(DEV, torch.float16 if half else torch.float32) for s in srcs]
    out = _nan_fill((B, H * steps[0], W * steps[1], cout), half)
    round_out = not half
    plan = C.tc_plan(dsrcs, subs, out, (H, W), half=half)
    assert plan["kernel"] == C.TC_KERNEL_TAP and plan["total_tiles"] % len(subs) == 0
    C.conv2d_tc_phases(dsrcs, subs, out, (H, W), round_out=round_out, half=half)
    torch.cuda.synchronize()
    expect = _bits(_nan_fill(out.shape, half).cpu()).clone()
    hit = torch.zeros(out.shape[1:3], dtype=torch.int32)
    for w, p, o in zip(ws, pads, offs):
        _, ref, ys, xs = conv_engine_ref(srcs, w, b, w.shape[2], w.shape[3], (1, 1), p, (H, W), steps, o, act, act_a, 1.0,
                                         round_out, out.dtype)
        expect[:, ys.view(-1, 1), xs.view(1, -1)] = _bits(ref)
        hit[ys.view(-1, 1), xs.view(1, -1)] += 1
    assert bool((hit == 1).all()), f"{name}: the phases do not tile the output exactly once"
    got = _bits(out.cpu())
    bad = got != expect
    assert not bool(bad.any()), f"{name} {dt}: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"
    return plan


def _w(cout, cin, kh, kw):
    from oracle.convnet_oracle import exact_grid_data
    return lambda g: exact_grid_data((cout, cin, kh, kw), 8, 4, g)


@pytest.mark.parametrize("dt", ["tf32", "f16"])
@pytest.mark.parametrize("ch,cout,hw,B", [((192, 128, 256), 128, (5, 9), 1), ((128, 64, 128), 64, (6, 11), 2),
                                          ((64, 64, 64), 48, (9, 13), 2), ((48, 48), 24, (17, 30), 1)])
def test_refine_phases_exact(dt, ch, cout, hw, B):
    """Refine = ConvTranspose2d(k4, s2) + crop as four 2x2 phases in one launch (the DepthModule's concatenations)."""
    from monorec_b200 import conv as C
    from oracle.convnet_oracle import exact_grid_data
    g = _gen("refine", ch, dt)
    wt = exact_grid_data((sum(ch), cout, 4, 4), 8, 4, g)
    ct = torch.nn.ConvTranspose2d(sum(ch), cout, 4, stride=2)
    with torch.no_grad():
        ct.weight.copy_(wt)
    layer = C.refine_layer(ct, ch)
    ws = [L._w_src.cpu() for L in layer.subs]
    _phase_run(f"refine{ch}", dt, [lambda g, w=w: w for w in ws], [L.pad for L in layer.subs], (2, 2),
               [L.out_off for L in layer.subs], ch, cout, hw, B)


@pytest.mark.parametrize("dt", ["tf32", "f16"])
def test_upconv_phases_exact_many_tiles(dt):
    """Upconv = nearest-x2 + 2x2 conv as 1x1 / 1x2 / 2x1 / 2x2 phases; enough tiles that every CTA runs several."""
    from monorec_b200 import conv as C
    from oracle.convnet_oracle import exact_grid_data
    g = _gen("upconv", dt)
    up = torch.nn.Conv2d(24, 32, 2)
    with torch.no_grad():
        up.weight.copy_(exact_grid_data((32, 24, 2, 2), 8, 4, g))
    layer = C.upconv_layer(up, (8, 16))
    ws = [L._w_src.cpu() for L in layer.subs]
    plan = _phase_run("upconv", dt, [lambda g, w=w: w for w in ws], [L.pad for L in layer.subs], (2, 2),
                      [L.out_off for L in layer.subs], (8, 16), 32, (128, 256), 3, act=0, bias=False)
    assert plan["total_tiles"] >= 4 * plan["grid"]


@pytest.mark.parametrize("dt", ["tf32", "f16"])
def test_two_and_three_phases_exact(dt):
    """2 phases side by side (ox_step 2) and 3 phases stacked (oy_step 3), each with its own filter and padding."""
    _phase_run("two_phases", dt, [_w(40, 32, 3, 3), _w(40, 32, 1, 2)], [(1, 1), (0, 0)], (1, 2), [(0, 0), (0, 1)],
               (32,), 40, (10, 21), 2)
    _phase_run("three_phases", dt, [_w(24, 72, 2, 2), _w(24, 72, 3, 1), _w(24, 72, 1, 1)], [(1, 0), (1, 0), (0, 0)], (3, 1),
               [(0, 0), (1, 0), (2, 0)], (40, 32), 24, (7, 19), 3)


# ---------------------------------------------------------------------------------------------------------------------
# CUDA-core kernel (fp32 storage, FMA): exact on the same data, with upsample-on-read and the single-channel head kernel
# ---------------------------------------------------------------------------------------------------------------------
FP32_CASES = [
    _case("fp32_3x3", (32,), 48), _case("fp32_cat3", (12, 36, 5), 70, k=(3, 1)),
    _case("fp32_s21", (24,), 64, k=(5, 1), s=(2, 1), hw=(21, 23)), _case("fp32_s12", (24,), 64, k=(1, 5), s=(1, 2)),
    _case("fp32_s22_odd", (7,), 13, s=(2, 2), hw=(13, 29)), _case("fp32_head_abstanh", (24,), 1, act=3, act_a=0.0025, act_b=0.3275),
    _case("fp32_head_sigmoid_1x1", (48,), 1, k=(1, 1), act=2), _case("fp32_sigmoid", (16,), 20, act=2),
    _case("fp32_none_nobias", (16,), 20, act=0, bias=False), _case("fp32_slice_odd", (16,), 9, coff=3, dst_c=17),
    _case("fp32_place", (16,), 16, k=(2, 2), step=(2, 2), off=(1, 0), dst_extra=(1, 3), pad=(0, 0)),
    _case("fp32_out_1x1", (8,), 8, s=(4, 4), hw=(3, 2), B=1), _case("fp32_B3", (8,), 8, hw=(30, 1), B=3),
]


@pytest.mark.parametrize("upsample2", [False, True])
@pytest.mark.parametrize("case", FP32_CASES, ids=_ids(FP32_CASES))
def test_cuda_core_conv_exact(case, upsample2):
    from monorec_b200 import conv as C
    from oracle.convnet_oracle import conv_engine_ref
    srcs, w, b = _data(case, "fp32")
    kh, kw = case["k"]
    H, W = case["hw"][0] * (2 if upsample2 else 1), case["hw"][1] * (2 if upsample2 else 1)
    sy, sx = case["s"]
    pad = case["pad"] or (C.same_pad_before(H, kh, sy), C.same_pad_before(W, kw, sx))
    Ho, Wo = math.ceil(H / sy), math.ceil(W / sx)
    dH, dW = [(n - 1) * st + o + 1 + e for n, st, o, e in zip((Ho, Wo), case["step"], case["off"], case["dst_extra"])]
    out = _nan_fill((case["B"], dH, dW, case["dst_c"] or case["cout"]), False)
    C.conv2d([s.to(DEV) for s in srcs], C.pack_conv_weight(w).to(DEV), None if b is None else b.to(DEV), kh, kw, stride=case["s"],
             act=case["act"], act_a=case["act_a"], act_b=case["act_b"], upsample2=upsample2, out=out, out_coff=case["coff"],
             pad=pad, out_hw=(Ho, Wo), out_step=case["step"], out_off=case["off"])
    torch.cuda.synchronize()
    pre, ref, ys, xs = conv_engine_ref(srcs, w, b, kh, kw, case["s"], pad, (Ho, Wo), case["step"], case["off"], case["act"],
                                       case["act_a"], case["act_b"], False, torch.float32, upsample2=upsample2)
    if case["act"] in (2, 3):
        ref = _act64(pre, b, case["act"], case["act_a"], case["act_b"])
    _check_written(out, ref, ys, xs, case["coff"], case["act"], False, f"{case['name']} upsample2={upsample2}")


# ---------------------------------------------------------------------------------------------------------------------
# Gaussian data: accumulation at fp32 precision (a half accumulator or a dropped partial sum would break the bound)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["tf32", "f16"])
def test_gaussian_accumulation_bound(dt):
    """|out - ref| <= K 2^-23 (sum |a w| + |b|) element-wise, K = the output's nonzero products: the textbook bound of
    truncating fp32 accumulation, on inputs already on the MMA's input grid.  How tight wgmma is against it is printed."""
    from monorec_b200 import conv as C
    from oracle.convnet_oracle import conv_engine_ref, round_tf32
    import torch.nn.functional as F
    half = dt == "f16"
    g = _gen("gauss", dt)
    ch, cout, kh, kw, B, H, W = (96, 128, 64), 96, 3, 3, 2, 14, 27
    srcs = [torch.randn(B, H, W, c, generator=g) for c in ch]
    srcs = [s.half().float() if half else round_tf32(s) for s in srcs]
    w = torch.randn(cout, sum(ch), kh, kw, generator=g) / math.sqrt(sum(ch) * kh * kw)
    w = w.half().float() if half else round_tf32(w)
    b = torch.randn(cout, generator=g)
    L = C.PackedConv(w.to(DEV), b.to(DEV), ch, act=C.ACT_NONE)
    dsrcs = [s.to(DEV, torch.float16 if half else torch.float32) for s in srcs]
    out = C.conv2d_tc(dsrcs, L, round_out=False, half=half, out_f32=True).cpu().to(torch.float64)
    pad = C._tc_pad(dsrcs, L)
    pre, _, _, _ = conv_engine_ref(srcs, w, None, kh, kw, (1, 1), pad, (H, W), exact=False)
    ref = pre + b.to(torch.float64)
    x = torch.cat(srcs, 3).permute(0, 3, 1, 2).to(torch.float64)
    xp = F.pad(x, (pad[1], kw - 1 - pad[1], pad[0], kh - 1 - pad[0]))
    mag = F.conv2d(xp.abs(), w.to(torch.float64).abs()).permute(0, 2, 3, 1) + b.abs().to(torch.float64)
    nz = F.conv2d((xp != 0).to(torch.float64), (w != 0).to(torch.float64)).permute(0, 2, 3, 1)
    bound = nz * 2.0 ** -23 * mag
    ratio = float(((out - ref).abs() / bound).max())
    print(f"gaussian {dt}: max |out - ref| / (K 2^-23 (sum|a w| + |b|)) = {ratio:.3e}, max |out - ref| = "
          f"{float((out - ref).abs().max()):.3e}")
    assert ratio <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# kernel coverage
# ---------------------------------------------------------------------------------------------------------------------
def _coverage():
    from monorec_b200 import conv as C
    seen, plans = Counter(), {}
    for case in TC_CASES:
        for dt in case["dtypes"]:
            p = _plan(case, dt)
            plans[(case["name"], dt)] = p
            seen[(C.TC_KERNEL_NAMES[p["kernel"]], dt, p["row_bytes"], p["n_pad"])] += 1
    return seen, plans


def _print_table(seen, plans):
    print("\ntensor-core cases per kernel x dtype x row bytes (columns: n_pad)")
    print(f"{'kernel':12s} {'dtype':5s} {'row':>4s} " + " ".join(f"{n:>3d}" for n in NPADS))
    for kern in ("tap", "halo", "halo-stream"):
        for dt in ("tf32", "f16"):
            for rb in (128, 64):
                row = [seen.get((kern, dt, rb, n), 0) for n in NPADS]
                if any(row):
                    print(f"{kern:12s} {dt:5s} {rb:>4d} " + " ".join(f"{v:>3d}" for v in row))
    for field in ("tap_reg_ctas", "halo_reg_ctas"):
        per_n = {p["n_pad"]: p[field] for p in plans.values()}
        print(f"{field:23s} " + " ".join(f"{per_n.get(n, 0):>3d}" for n in NPADS))


def test_kernel_coverage():
    """The sweep reaches every kernel the host code can choose, in both dtypes, with 64-byte rows, at every MMA width.
    Combinations the current heuristics cannot reach are listed with their reason, which is checked against the plans."""
    seen, plans = _coverage()
    _print_table(seen, plans)
    reached = {(k, dt, rb, n) for (k, dt, rb, n) in seen}
    kern_dt = {(k, dt) for (k, dt, _, _) in reached}
    kern_rb = {(k, rb) for (k, _, rb, _) in reached}
    halo_family = {(dt, n) for (k, dt, _, n) in reached if k != "tap"}
    tap_n = {(dt, n) for (k, dt, _, n) in reached if k == "tap"}
    all_n = {(dt, n) for dt in ("tf32", "f16") for n in NPADS}
    assert tap_n == all_n, f"tap kernel misses {sorted(all_n - tap_n)}"
    if HALO_ENV == "0":                                   # forced: every stride-1 layer on the tap kernel
        assert kern_dt == {("tap", "tf32"), ("tap", "f16")} and ("tap", 64) in kern_rb
        return
    if HALO_ENV == "1" and STREAM_ENV == "0":             # forced: halo kernel with resident weights, one CTA per SM allowed
        assert {k for k, _ in kern_dt} == {"tap", "halo"} and ("halo", 64) in kern_rb and ("tap", 64) in kern_rb
        assert halo_family == all_n, f"halo kernel misses {sorted(all_n - halo_family)}"
        return
    for k in ("tap", "halo", "halo-stream"):
        for dt in ("tf32", "f16"):
            assert (k, dt) in kern_dt, f"no case reaches the {k} kernel in {dt}"
        assert (k, 64) in kern_rb, f"no case reaches the {k} kernel with 64-byte rows"
    # The automatic choice wants at least two halo CTAs per SM (resident weights) and streams weights only with two.  From
    # MMA N = 144 on, the halo kernel's accumulator registers allow one CTA per SM, so wide stride-1 layers run on the tap
    # kernel: the halo kernels are out of reach there (checked on every plan below, so the list cannot go stale).
    unreachable = {(dt, n): "halo kernel registers allow one CTA per SM (halo_reg_ctas == 1)"
                   for dt in ("tf32", "f16") for n in range(144, 257, 16)}
    assert halo_family == all_n - set(unreachable), (
        f"halo kernels reach {sorted(halo_family)}; expected every n_pad but {sorted(unreachable)}")
    for (name, dt), p in plans.items():
        assert (p["halo_reg_ctas"] == 1) == ((dt, p["n_pad"]) in unreachable), (name, dt, p)


def test_forced_kernels_in_subprocesses():
    """The sweep once more with every stride-1 layer forced onto the tap-refetch kernel (MONOREC_B200_TC_HALO=0), and once with
    the halo kernel allowed at one CTA per SM and weight streaming off (MONOREC_B200_TC_HALO=1 MONOREC_B200_TC_STREAM=0).  The
    switches are read once per process, hence the subprocesses."""
    for extra in ({"MONOREC_B200_TC_HALO": "0"}, {"MONOREC_B200_TC_HALO": "1", "MONOREC_B200_TC_STREAM": "0"}):
        env = dict(os.environ, **extra)
        r = subprocess.run([sys.executable, "-m", "pytest", __file__, "-q", "-m", "gpu", "-p", "no:cacheprovider",
                            "-k", "tc_ or kernel_coverage or phases"],
                           env=env, capture_output=True, text=True, timeout=900, cwd=os.path.dirname(os.path.dirname(__file__)))
        assert r.returncode == 0, f"{extra}:\n{r.stdout[-4000:]}"
