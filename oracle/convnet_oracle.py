"""ORACLE (test infrastructure, not product code) -- functional CPU restatement of MonoRec's conv stacks.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this file.

Reference being restated (all from the reference's model/):
  layers.py:220-252   PadSameConv2d          TF-"SAME" asymmetric zero padding
  layers.py:289-335   ConvReLU2 / ConvReLU   (k,1) conv + LReLU + (1,k) conv + LReLU   /   kxk conv + LReLU
  layers.py:338-356   Upconv                 nearest x2, pad (0,1,0,1), 2x2 conv (no activation)
  layers.py:380-400   Refine                 ConvTranspose2d(k=4, s=2) + LReLU + centre crop to 2x
  monorec/monorec_model.py:287-385   MaskModule
  monorec/monorec_model.py:476-557   DepthModule
  monorec/monorec_model.py:672-729   MonoRecModel.forward (default pretrain_mode=0 routing)

Parity pin: tests/golden/model_synth_small.npz holds outputs of the unmodified reference model (seeded weights from
monorec_b200.synthetic.seeded_state_dict); tests/test_oracle_golden.py checks `monorec_forward` below against it.
Weights are addressed through the reference's own state_dict keys (SURVEY.md §8b checkpoint contract).
"""
import math

import torch
import torch.nn.functional as F

SLOPE = 0.1  # LeakyReLU negative slope everywhere (layers.py:290, 318, 381)


def same_pad(n, k, s):
    """(before, after) zero padding of PadSameConv2d along one axis (layers.py:249-251)."""
    total = s * (math.ceil(n / s) - 1) + k - n
    return math.floor(total / 2), math.ceil(total / 2)


def conv_same(x, w, b, stride=(1, 1)):
    kh, kw = w.shape[2], w.shape[3]
    pt, pb = same_pad(x.shape[2], kh, stride[0])
    pl, pr = same_pad(x.shape[3], kw, stride[1])
    return F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, b, stride=stride)


def lrelu(x):
    return F.leaky_relu(x, SLOPE)


def conv_relu(sd, prefix, x):
    """ConvReLU (layers.py:317-335)."""
    return lrelu(conv_same(x, sd[prefix + ".conv.weight"], sd[prefix + ".conv.bias"]))


def conv_relu2(sd, prefix, x, stride=1):
    """ConvReLU2 (layers.py:289-314): y-direction conv, LReLU, x-direction conv, LReLU."""
    t = lrelu(conv_same(x, sd[prefix + ".conv_y.weight"], sd[prefix + ".conv_y.bias"], (stride, 1)))
    return lrelu(conv_same(t, sd[prefix + ".conv_x.weight"], sd[prefix + ".conv_x.bias"], (1, stride)))


def upconv(sd, prefix, x):
    """Upconv (layers.py:338-356)."""
    t = F.interpolate(x, scale_factor=2, mode="nearest")
    return conv_same(t, sd[prefix + ".conv.weight"], sd[prefix + ".conv.bias"])


def refine(sd, prefix, x):
    """Refine (layers.py:380-400): transposed conv k4 s2 -> LReLU -> crop one pixel per side (oversize = -2)."""
    t = lrelu(F.conv_transpose2d(x, sd[prefix + ".conv2d_t.weight"], sd[prefix + ".conv2d_t.bias"], stride=2))
    return t[:, :, 1:-1, 1:-1]


def mask_module(sd, single_frame_cvs, image_features, prefix="att_module."):
    """MaskModule.forward (monorec_model.py:345-385), eval mode (dropout inactive)."""
    feats = None
    for cv in single_frame_cvs:
        x, cur = cv, []
        for lvl in range(5):
            if lvl > 0:
                x = F.max_pool2d(x, 2)
            a, b = (0, 1) if lvl == 0 else (1, 2)
            x = conv_relu(sd, f"{prefix}enc.{lvl}.{a}", x)
            x = conv_relu(sd, f"{prefix}enc.{lvl}.{b}", x)
            cur.append(x)
        feats = cur if feats is None else [torch.max(p, q) for p, q in zip(feats, cur)]
    x = feats[-1]
    for i in range(4):
        if i == 0:
            x = torch.cat([feats[-1], image_features[3]], 1)
        x = upconv(sd, f"{prefix}dec.{i}.0", x)
        if i == 0:
            x = torch.cat([feats[-2], image_features[2], x], 1)
        elif i == 3:
            x = torch.cat([feats[-(i + 2)], x], 1)
        else:
            x = torch.cat([feats[-(i + 2)], image_features[2 - i], x], 1)
        x = conv_relu(sd, f"{prefix}dec.{i}.1", x)
        x = conv_relu(sd, f"{prefix}dec.{i}.2", x)
    return torch.sigmoid(F.conv2d(x, sd[prefix + "classifier.0.weight"], sd[prefix + "classifier.0.bias"]))


def depth_module(sd, cost_volume, keyframe, image_features, prefix="depth_module."):
    """DepthModule.forward (monorec_model.py:526-557); returns predictions ordered [full, 1/2, 1/4, 1/8]."""
    x = torch.cat([cost_volume, keyframe], 1)
    strides = [1, 2, 2, 2, 2]
    feats = []
    for lvl in range(5):
        x = conv_relu2(sd, f"{prefix}enc.{lvl}.0", x, strides[lvl])
        x = conv_relu2(sd, f"{prefix}enc.{lvl}.1", x)
        feats.append(x)

    def head(i, t):
        w, b = sd[f"{prefix}predictors.{i}.1.weight"], sd[f"{prefix}predictors.{i}.1.bias"]
        return torch.abs(torch.tanh(conv_same(t, w, b)))

    preds = []
    x = refine(sd, f"{prefix}dec.0", feats[-1])                                    # 256 @ 1/8
    preds.insert(0, head(0, x))
    x = refine(sd, f"{prefix}dec.1.0", torch.cat([feats[-2], image_features[-3], x], 1))
    x = conv_relu2(sd, f"{prefix}dec.1.1", x)                                      # 128 @ 1/4
    preds.insert(0, head(1, x))
    x = refine(sd, f"{prefix}dec.2.0", torch.cat([feats[-3], image_features[-4], x], 1))
    x = conv_relu2(sd, f"{prefix}dec.2.1", x)                                      # 64 @ 1/2
    preds.insert(0, head(2, x))
    x = refine(sd, f"{prefix}dec.3", torch.cat([feats[-4], image_features[-5], x], 1))   # 48 @ full (no head)
    x = conv_relu2(sd, f"{prefix}dec.4.0", torch.cat([feats[0], x], 1))
    x = lrelu(conv_same(x, sd[f"{prefix}dec.4.2.weight"], sd[f"{prefix}dec.4.2.bias"]))  # 24 @ full
    preds.insert(0, head(3, x))
    return preds


ACT_NONE, ACT_LEAKY, ACT_SIGMOID, ACT_ABSTANH = 0, 1, 2, 3    # include/monorec_b200.h MR_ACT_*


def exact_grid_data(shape, lim, scale_log2, generator):
    """Integers in [-lim, lim] times 2^-scale_log2 (float32).  With |i| <= 32 at 2^-3 for activations and |j| <= 8 at 2^-4 for
    weights and biases every value lies on the TF32 and the half grid and every product is exact in fp32."""
    i = torch.randint(-lim, lim + 1, shape, generator=generator, dtype=torch.int64)
    return (i.to(torch.float64) * 2.0 ** -scale_log2).to(torch.float32)


def round_tf32(x):
    """The engine's round_out: (bits + 0x1000) & ~0x1FFF on float32 (round half away from zero onto 10 mantissa bits)."""
    bits = x.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def conv_engine_ref(srcs, w, bias, kh, kw, stride, pad, out_hw, out_step=(1, 1), out_off=(0, 0), act=ACT_NONE, act_a=0.0,
                    act_b=1.0, round_out=False, out_dtype=torch.float32, upsample2=False, exact=True):
    """Reference of one call of the convolution engine (include/monorec_b200.h, mr_conv_desc), in float64 on the CPU.

    srcs: NHWC tensors [B, Hs, Ws, C_i] concatenated along C; w: correlation kernel (Cout, sum C_i, kh, kw); bias: (Cout,) or
    None; pad = (pad_t, pad_l) leading zero padding, every tap outside the (optionally nearest-x2 upsampled) input reads 0;
    out_hw = (Ho, Wo).  Returns (pre, out, ys, xs): pre = the float64 sum of products [B, Ho, Wo, Cout] (exact);
    out = bias + activation + output rounding applied the way the kernels do it, in float32 (then out_dtype); output
    pixel (oy, ox) belongs at destination row ys[oy], column xs[ox].

    exact=True asserts that the data makes the engine's result exact whatever its accumulation order: every input a multiple
    of 2^-3 and every weight / bias a multiple of 2^-4 (so every product and partial sum is a multiple of 2^-7), and the sum
    of |products| + |bias| of every output below 2^17, so every partial sum fits the 24-bit fp32 significand."""
    x = torch.cat([s.to(torch.float64) for s in srcs], 3).permute(0, 3, 1, 2)          # NCHW float64
    if upsample2:
        x = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
    Ho, Wo = out_hw
    sy, sx = stride
    pt, pl = pad
    x = x[:, :, max(-pt, 0):, max(-pl, 0):]              # negative SAME padding (stride > kernel) crops, as PadSameConv2d does
    pt, pl = max(pt, 0), max(pl, 0)
    B, C, H, W = x.shape
    need_h, need_w = (Ho - 1) * sy + kh, (Wo - 1) * sx + kw
    xp = torch.zeros(B, C, max(need_h, pt + H), max(need_w, pl + W), dtype=torch.float64)
    xp[:, :, pt:pt + H, pl:pl + W] = x
    xp = xp[:, :, :need_h, :need_w]
    w64 = w.to(torch.float64)
    pre = F.conv2d(xp, w64, None, stride=stride)[:, :, :Ho, :Wo]
    if exact:
        assert torch.equal(torch.frac(x * 8), torch.zeros_like(x)), "inputs must be multiples of 2^-3"
        assert torch.equal(torch.frac(w64 * 16), torch.zeros_like(w64)), "weights must be multiples of 2^-4"
        mag = F.conv2d(xp.abs(), w64.abs(), None, stride=stride)[:, :, :Ho, :Wo]
        if bias is not None:
            b64 = bias.to(torch.float64)
            assert torch.equal(torch.frac(b64 * 16), torch.zeros_like(b64)), "biases must be multiples of 2^-4"
            mag = mag + b64.abs().view(1, -1, 1, 1)
        assert float(mag.max()) < 2.0 ** 17, f"partial sums reach {float(mag.max())}: not exact in fp32"
    pre = pre.permute(0, 2, 3, 1).contiguous()
    v = pre.to(torch.float32)                                                            # exact (see above)
    if bias is not None:
        v = v + bias.to(torch.float32)
    if act == ACT_LEAKY:
        v = torch.where(v >= 0, v, torch.tensor(act_a, dtype=torch.float32) * v)
    elif act == ACT_SIGMOID:
        v = torch.sigmoid(v.to(torch.float64)).to(torch.float32)
    elif act == ACT_ABSTANH:
        v = (act_a + act_b * torch.tanh(v.to(torch.float64)).abs()).to(torch.float32)
    else:
        assert act == ACT_NONE, act
    if round_out:
        v = round_tf32(v)
    out = v.to(out_dtype)
    ys = torch.arange(Ho) * out_step[0] + out_off[0]
    xs = torch.arange(Wo) * out_step[1] + out_off[1]
    return pre, out, ys, xs


def resnet_features(sd, keyframe_plus_half, prefix="_feature_extractor.encoder."):
    """ResnetEncoder.forward (monorec_model.py:118-129) on torchvision resnet18 weights held in `sd` (eval BN)."""
    import torchvision
    net = torchvision.models.resnet18(weights=None)
    net.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)})
    net.eval()
    x = (keyframe_plus_half - 0.45) / 0.225
    f0 = net.relu(net.bn1(net.conv1(x)))
    f1 = net.layer1(net.maxpool(f0))
    f2 = net.layer2(f1)
    f3 = net.layer3(f2)
    f4 = net.layer4(f3)
    return [f0, f1, f2, f3, f4]


@torch.no_grad()
def monorec_forward(sd, data, cost_volume, single_frame_cvs, inv_depth_min_max=(0.33, 0.0025)):
    """MonoRecModel.forward, pretrain_mode=0 (monorec_model.py:691-727), given the cost-volume stage's outputs."""
    feats = resnet_features(sd, data["keyframe"] + 0.5)
    cv_mask = mask_module(sd, single_frame_cvs, feats)
    masked = (1 - cv_mask) * cost_volume
    preds = depth_module(sd, masked, data["keyframe"], feats)
    lo, hi = inv_depth_min_max[1], inv_depth_min_max[0]
    inv = [(1 - p) * lo + p * hi for p in preds]
    return {"image_features": feats, "cv_mask": cv_mask, "cost_volume": masked, "predicted_inverse_depths": inv,
            "result": inv[0], "mask": cv_mask}
