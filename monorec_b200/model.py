"""Drop-in replacement of the reference's MonoRecModel and its sub-modules (model/monorec/monorec_model.py:95-729).

Same constructor keywords, same `forward(data_dict) -> data_dict` contract and dict keys, same attribute names
(`cv_module`, `att_module`, `depth_module`, `_feature_extractor`, ...) and -- the checkpoint contract -- the same
`state_dict()` keys and shapes, so a reference checkpoint loads unchanged (SURVEY.md §8b).  The modules below only
*hold* parameters in the reference's layout; the arithmetic runs in libmonorec_b200.so (fused cost-volume kernel +
convolution engine) through the C ABI.  The ResNet-18 trunk stays on torchvision/cuDNN (third-party arithmetic in the
reference too; SURVEY.md §8f "next" row 1) with its eval-mode BatchNorms folded, in half precision in half mode.  (Round 2
measured the trunk on the conv engine at 1.03 ms against cuDNN's 0.71 ms in half mode, so that variant was removed.)
"""
import threading
import warnings

import torch
import torch.nn.functional as F
from torch import nn

from . import conv as C
from . import ops
from .cost_volume import CostVolumeModule

__all__ = ["MonoRecModel", "CostVolumeModule", "MaskModule", "DepthModule", "ResnetEncoder"]

_CUDNN_FUSED = hasattr(torch, "cudnn_convolution_relu") and hasattr(torch, "cudnn_convolution_add_relu")
_PACK_LOCK = threading.Lock()   # every _Packed lookup and build (module-level: a lock in a module would break deepcopy / pickle)


# --------------------------------------------------------------------------------------------------------------------
# parameter holders with the reference's attribute names (model/layers.py:289-400)
# --------------------------------------------------------------------------------------------------------------------
class ConvReLU(nn.Module):
    """PadSame + Conv2d(k) + LeakyReLU(0.1)  (model/layers.py:317-335).  Key: `.conv.{weight,bias}`."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride)
        self.kernel_size, self.stride = kernel_size, stride


class ConvReLU2(nn.Module):
    """(k,1) conv + LReLU + (1,k) conv + LReLU  (model/layers.py:289-314).  Keys: `.conv_y.*`, `.conv_x.*`."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1):
        super().__init__()
        self.conv_y = nn.Conv2d(in_channels, out_channels, (kernel_size, 1), stride=(stride, 1))
        self.conv_x = nn.Conv2d(out_channels, out_channels, (1, kernel_size), stride=(1, stride))
        self.kernel_size, self.stride = kernel_size, stride


class Upconv(nn.Module):
    """nearest x2 + pad(0,1,0,1) + Conv2d(2)  (model/layers.py:338-356).  Key: `.conv.*`."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, 2, stride=1)


class Refine(nn.Module):
    """ConvTranspose2d(k4, s2) + LReLU + centre crop  (model/layers.py:380-400).  Key: `.conv2d_t.*`."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv2d_t = nn.ConvTranspose2d(in_channels, out_channels, kernel_size=4, stride=2)


def _source_sig(tensors):
    return (C.MODE,) + tuple((t.data_ptr(), t._version, str(t.device)) for t in tensors)


class _Packed:
    """Kernel-layout copies of a module's parameters, one per device, rebuilt when a parameter changes (load_state_dict, .to(),
    an optimizer step: anything that bumps the tensors' version counters or moves them).  In-place edits through `.data`
    (e.g. `p.data.copy_(ema)`) are invisible to autograd's version counter: call `invalidate()` (or the owning module's
    `invalidate_packed_weights()`) after such an edit.

    An entry is keyed on the device its tensors live on and holds the signature of the source parameters it was built from
    (`_PackedSource._pack_sig`).  DataParallel replicas share this object with the module they were replicated from (their
    `__dict__` is a shallow copy), so the replicas of every later forward find the entry of their device.  Lookups and builds
    hold one lock: concurrent forwards build an entry once and never see a half-built one.  A new signature drops the entries
    of the old one on every device."""

    def __init__(self):
        self.entries = {}     # str(device) -> (signature, packed data)

    def invalidate(self):
        with _PACK_LOCK:
            self.entries = {}

    def get(self, sig, device, builder):
        key = str(device)
        with _PACK_LOCK:
            entry = self.entries.get(key)
            if entry is None or entry[0] != sig:
                with torch.no_grad():
                    entry = (sig, builder())
                if device.type == "cuda":   # built on this thread's stream: complete before another stream reads it
                    torch.cuda.current_stream(device).synchronize()
                entries = {k: v for k, v in self.entries.items() if v[0] == sig}
                entries[key] = entry
                self.entries = entries
            return entry[1]


class _PackedShared(_Packed):
    """The cache of a module that packs weights it is handed (ops.py: the weights of any model of one configuration).  One
    entry per (device, signature), the last `keep` kept.  An entry holds its source tensors, so their memory cannot be
    freed and reused by other tensors that would then match the signature's data pointers and versions."""

    def __init__(self, keep=4):
        super().__init__()
        self.keep = keep

    def get(self, sig, device, builder, sources=()):
        key = (str(device), sig)
        with _PACK_LOCK:
            entry = self.entries.pop(key, None)
            if entry is None:
                with torch.no_grad():
                    entry = (builder(), list(sources))
                if device.type == "cuda":
                    torch.cuda.current_stream(device).synchronize()
            self.entries[key] = entry                  # most recent last
            while len(self.entries) > self.keep:
                self.entries.pop(next(iter(self.entries)))
            return entry[0]


class _PackedSource:
    """Where a module's kernel-layout copies come from.  The signature is that of the module's own parameters -- except in a
    DataParallel replica, which has no registered parameters (its copies on its device are plain attributes, broadcast anew
    for every forward): it carries the signature of the original's parameters, taken when it is replicated."""

    _src_sig = None

    def _source_tensors(self):
        return list(self.parameters())

    def _pack_sig(self):
        return self._src_sig if self._src_sig is not None else _source_sig(self._source_tensors())

    def _replicate_for_data_parallel(self):
        replica = super()._replicate_for_data_parallel()
        replica._src_sig = self._pack_sig()
        return replica

    def _packs(self, builder):
        """The entry of the device this module's weights are on, built by `builder` (from those weights) if missing."""
        if isinstance(self._packed, _PackedShared):
            src = self._source_tensors()
            return self._packed.get(_source_sig(src), self._pack_device(), builder, src)
        return self._packed.get(self._pack_sig(), self._pack_device(), builder)

    def _source_names(self):
        """Names (relative to this module) of `_source_tensors()`, in that order."""
        return [n for n, _ in self.named_parameters()]


def _leaky(conv, src_c, stride=(1, 1)):
    return C.PackedConv(conv.weight, conv.bias, src_c, stride=stride, act=C.ACT_LEAKY, act_a=C.LEAKY_SLOPE)


# --------------------------------------------------------------------------------------------------------------------
class ResnetEncoder(_PackedSource, nn.Module):
    """torchvision ResNet-18 trunk, 5 feature maps (monorec_model.py:95-129)."""

    def __init__(self, num_layers=18, pretrained=True):
        super().__init__()
        import numpy as np
        import torchvision
        if num_layers != 18:
            raise NotImplementedError("monorec_b200: the reference only ever instantiates ResnetEncoder(18)")
        self.num_ch_enc = np.array([64, 64, 128, 256, 512])
        # The reference asks torchvision for ImageNet weights (:104-113).  They are used only if already in the local hub
        # cache: a MonoRec checkpoint carries `_feature_extractor.encoder.*` anyway, and this code must stay silent and
        # offline-safe (no download attempt, nothing printed to stdout).
        weights = None
        self.pretrained_requested_but_missing = False
        if pretrained:
            import os
            w = torchvision.models.ResNet18_Weights.IMAGENET1K_V1
            cached = os.path.join(torch.hub.get_dir(), "checkpoints", os.path.basename(w.url))
            if os.path.isfile(cached):
                weights = w
            else:
                # the reference would download them here; MonoRecModel warns if no checkpoint supplies the encoder either
                self.pretrained_requested_but_missing = True
        self.encoder = torchvision.models.resnet18(weights=weights)
        self._packed = _Packed()

    # ---- inference fast path: BatchNorm (eval mode = a fixed per-channel affine) folded into the preceding convolution ----
    @staticmethod
    def _fold(conv, bn):
        scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
        w = (conv.weight * scale.view(-1, 1, 1, 1)).contiguous(memory_format=torch.channels_last)
        b = bn.bias - bn.running_mean * scale
        if conv.bias is not None:
            b = b + conv.bias * scale
        return w, b.contiguous()

    def invalidate_packed_weights(self):
        """Forget the folded / packed copies (needed only after in-place `.data` edits of the parameters or BatchNorm buffers)."""
        self._packed.invalidate()

    def _source_tensors(self):
        e = self.encoder
        return [t for n, t in list(e.named_parameters()) + list(e.named_buffers()) if not n.startswith("fc.")]

    def _source_names(self):
        e = self.encoder
        return ["encoder." + n for n, _ in list(e.named_parameters()) + list(e.named_buffers()) if not n.startswith("fc.")]

    def _pack_device(self):
        return self.encoder.conv1.weight.device

    def _build(self):
        e = self.encoder
        f = {"stem": self._fold(e.conv1, e.bn1), "blocks": []}
        for layer in (e.layer1, e.layer2, e.layer3, e.layer4):
            blocks = []
            for blk in layer:
                down = None if blk.downsample is None else self._fold(blk.downsample[0], blk.downsample[1]) + (
                    blk.downsample[0].stride,)
                blocks.append((self._fold(blk.conv1, blk.bn1), blk.conv1.stride, self._fold(blk.conv2, blk.bn2), down))
            f["blocks"].append(blocks)
        # in half mode the trunk runs in half as well (folded weights and activations): its NHWC outputs feed the conv engine
        # without casts (0.82 -> 0.71 ms at B=8)
        if C.MODE == "f16" and f["stem"][0].is_cuda:
            conv = lambda wb: (wb[0].half().contiguous(memory_format=torch.channels_last), wb[1].half())   # noqa: E731
            f = {"stem": conv(f["stem"]),
                 "blocks": [[(conv(a), s_, conv(b), None if d is None else conv(d[:2]) + (d[2],)) for a, s_, b, d in blocks]
                            for blocks in f["blocks"]]}
        return f

    def _folded(self):
        """The folded trunk weights the inference path runs on (half in f16 mode on CUDA), built once per parameter version
        and device."""
        return self._packs(self._build)

    # cuDNN's fused epilogues where the build offers them (conv + bias + ReLU, conv + residual + bias + ReLU: the ~24
    # element-wise add / clamp launches of the trunk disappear); the folded trunk also runs on the CPU, on F.conv2d
    @staticmethod
    def _conv_relu(t, w, bias, stride, padding):
        if t.is_cuda and _CUDNN_FUSED:
            return torch.cudnn_convolution_relu(t, w, bias, list(stride), list(padding), [1, 1], 1)
        return F.conv2d(t, w, bias, stride=stride, padding=padding).relu_()

    @staticmethod
    def _conv_add_relu(t, w, bias, z):
        if t.is_cuda and _CUDNN_FUSED:
            return torch.cudnn_convolution_add_relu(t, w, z, 1.0, bias, [1, 1], [1, 1], [1, 1], 1)
        return F.conv2d(t, w, bias, padding=1).add_(z).relu_()

    def _run_blocks(self, x, blocks):
        """The residual blocks of one trunk level, on the folded weights `blocks` (an entry of `_folded()["blocks"]`)."""
        for (w1, b1), stride, (w2, b2), down in blocks:
            idt = x if down is None else F.conv2d(x, down[0], down[1], stride=down[2])
            out = self._conv_relu(x, w1, b1, tuple(stride), (1, 1))
            x = self._conv_add_relu(out, w2, b2, idt)
        return x

    def _forward_folded(self, input_image):
        e, f = self.encoder, self._folded()
        x = (input_image - 0.45) / 0.225
        if f["stem"][0].dtype == torch.float16:
            x = x.half()
        x = self._conv_relu(x, f["stem"][0], f["stem"][1], tuple(e.conv1.stride), tuple(e.conv1.padding))
        feats = [x]
        mp = e.maxpool
        if (x.is_cuda and x.dtype in (torch.float16, torch.float32) and x.shape[1] % 8 == 0 and
                x.permute(0, 2, 3, 1).is_contiguous() and isinstance(mp, nn.MaxPool2d) and mp.kernel_size == 3 and mp.stride == 2 and
                mp.padding == 1 and mp.dilation == 1 and not mp.ceil_mode):
            x = C.maxpool3s2_channels_last(x)            # (ATen's channels-last max-pool: 75 us for this 33 MB tensor)
        else:
            x = mp(x)
        for blocks in f["blocks"][:3]:
            x = self._run_blocks(x, blocks)
            feats.append(x)
        # The 512-channel level (layer4, 23 % of the trunk's multiply-adds) has no consumer: the MaskModule reads levels 0-3
        # (monorec_model.py:372-380), the DepthModule levels 0-2 (:545), and nothing else in the reference touches
        # data_dict["image_features"].  It is computed when somebody asks for it.
        last = f["blocks"][3]
        self.features = _TrunkFeatures(feats, tail_fn=lambda t: self._run_blocks(t, last))
        return self.features

    def forward(self, input_image):
        e = self.encoder
        if not e.training and not torch.is_grad_enabled():
            return self._forward_folded(input_image)
        x = (input_image - 0.45) / 0.225
        self.features = [e.relu(e.bn1(e.conv1(x)))]
        self.features.append(e.layer1(e.maxpool(self.features[-1])))
        self.features.append(e.layer2(self.features[-1]))
        self.features.append(e.layer3(self.features[-1]))
        self.features.append(e.layer4(self.features[-1]))
        return self.features


def trunk_features(encoder, image, allow_tf32):
    """The trunk's levels of `image` with cuDNN's TF32 switch set as given (only TF32 is decided here: the caller's cuDNN
    benchmark / deterministic settings are passed through).  MonoRecModel.forward calls this directly; under torch.compile
    it is the implementation of the `monorec_b200::resnet_trunk` op, which returns all five levels."""
    with torch.backends.cudnn.flags(enabled=True, benchmark=torch.backends.cudnn.benchmark,
                                    deterministic=torch.backends.cudnn.deterministic, allow_tf32=allow_tf32):
        return encoder(image)


class _TrunkFeatures(list):
    """`image_features` (monorec_model.py:118-129) with its last entry evaluated on first use.  Slices and indices below 4 --
    everything the Mask / Depth modules do -- never trigger it; index 4 / -1, iteration, comparison, concatenation, copy do.

    Without `tail_fn` it is a plain list of `items`: `type(f)(iterable)` is how torch.nn.parallel.gather rebuilds it (after
    iterating the replicas' lists, which evaluates their level 4), so DataParallel gathers it like the reference's list."""

    def __init__(self, items=(), tail_fn=None):
        super().__init__(list(items) + [None] if tail_fn is not None else items)
        self._tail_fn = tail_fn

    def _fill(self):
        if self._tail_fn is not None and list.__getitem__(self, 4) is None:
            with torch.no_grad():
                list.__setitem__(self, 4, self._tail_fn(list.__getitem__(self, 3)))

    def reset_tail(self):
        """After a CUDA-graph replay rewrote level 3 in place: the cached level 4 is stale."""
        if self._tail_fn is not None:
            list.__setitem__(self, 4, None)

    def __getitem__(self, i):
        if isinstance(i, slice):
            if 4 in range(*i.indices(5)):
                self._fill()
        elif i in (4, -1):
            self._fill()
        return list.__getitem__(self, i)

    def __iter__(self):
        self._fill()
        return list.__iter__(self)

    def __reversed__(self):
        self._fill()
        return list.__reversed__(self)

    def __add__(self, other):
        self._fill()
        return list(list.__iter__(self)) + list(other)

    def __eq__(self, other):
        self._fill()
        return list.__eq__(self, other)

    __hash__ = None

    def __contains__(self, item):
        self._fill()
        return list.__contains__(self, item)

    def copy(self):
        self._fill()
        return list(list.__iter__(self))

    def __reduce__(self):
        self._fill()
        return (list, (list(list.__iter__(self)),))


class MaskModule(_PackedSource, nn.Module):
    """Moving-object mask U-Net over the single-frame volumes (monorec_model.py:287-385)."""

    def __init__(self, depth_steps=32, feature_channels=(64, 64, 128, 256, 512), use_cv=True, use_features=True):
        super().__init__()
        self.depth_steps = depth_steps
        self.feat_chns = tuple(int(c) for c in feature_channels)
        self._in_channels = depth_steps
        self._cv_enc_feat_chns = (self._in_channels, 48, 64, 96, 96)
        self._dec_feat_chns = (96, 96, 64, 48, 128)
        self.use_cv, self.use_features = use_cv, use_features
        e, d, fc = self._cv_enc_feat_chns, self._dec_feat_chns, self.feat_chns
        self.enc = nn.ModuleList([nn.Sequential(ConvReLU(self._in_channels, e[0], 3), ConvReLU(e[0], e[0], 3))] + [
            nn.Sequential(nn.MaxPool2d(kernel_size=2), ConvReLU(e[i - 1], e[i], 3), ConvReLU(e[i], e[i], 3))
            for i in range(1, 5)])
        self.dec = nn.ModuleList([
            nn.Sequential(Upconv(e[4] + fc[3], d[0]), ConvReLU(d[0] + e[3] + fc[2], d[0], 3), ConvReLU(d[0], d[0], 3)),
            nn.Sequential(Upconv(d[0], d[0]), ConvReLU(d[0] + e[2] + fc[1], d[1], 3), ConvReLU(d[1], d[1], 3)),
            nn.Sequential(Upconv(d[1], d[1]), ConvReLU(d[1] + e[1] + fc[0], d[2], 3), ConvReLU(d[2], d[2], 3)),
            nn.Sequential(Upconv(d[2], d[2]), ConvReLU(d[2] + e[0], d[3], 3), ConvReLU(d[3], d[3], 3))])
        self.classifier = nn.Sequential(nn.Conv2d(d[3], 1, kernel_size=1, stride=1), nn.Sigmoid())
        self._packed = _Packed()

    def invalidate_packed_weights(self):
        """After in-place `.data` edits of the parameters (not seen by the version counters): repack on the next call."""
        self._packed.invalidate()

    def _pack_device(self):
        return self.classifier[0].weight.device

    def _build(self):
        e, d, fc = self._cv_enc_feat_chns, self._dec_feat_chns, self.feat_chns
        p = {}
        for lvl, seq in enumerate(self.enc):
            mods = [m for m in seq if isinstance(m, ConvReLU)]
            p[f"enc{lvl}"] = [_leaky(m.conv, (m.conv.in_channels,)) for m in mods]
        up_src = [(e[4], fc[3]), (d[0],), (d[1],), (d[2],)]
        cat_src = [(e[3], fc[2], d[0]), (e[2], fc[1], d[0]), (e[1], fc[0], d[1]), (e[0], d[2])]
        for i, seq in enumerate(self.dec):
            p[f"dec{i}"] = [C.upconv_layer(seq[0].conv, up_src[i]), _leaky(seq[1].conv, cat_src[i]),
                            _leaky(seq[2].conv, (seq[2].conv.in_channels,))]
        cls = self.classifier[0]
        p["cls"] = C.PackedConv(cls.weight, cls.bias, (cls.in_channels,), act=C.ACT_SIGMOID)
        return p

    def forward(self, data_dict):
        sfcvs = data_dict["single_frame_cvs"]
        feats_nchw = data_dict["image_features"]
        if self.training:
            raise NotImplementedError("monorec_b200.MaskModule: inference only (dropout / autograd are not implemented)")
        x = data_dict.pop("_sfcv_nhwc", None) if data_dict.pop("_sfcv_nhwc_filled", False) else None
        if torch.compiler.is_compiling():
            m = torch.ops.monorec_b200.mask_module(list(sfcvs), list(feats_nchw[:4]), x, list(self.parameters()),
                                                   self.depth_steps, list(self.feat_chns), self.use_cv, self.use_features)
        else:
            m = self._run(sfcvs, feats_nchw, x)
        data_dict["cv_mask"] = m
        return data_dict

    def _run(self, sfcvs, feats_nchw, x):
        """The U-Net on the single-frame volumes and trunk levels 0-3 -> cv_mask [B,1,H,W].  x: the volumes already in the
        engine's NHWC layout (written by the cost-volume kernel) or None.  The implementation of the
        `monorec_b200::mask_module` op as well."""
        P = self._packs(self._build)
        nF = len(sfcvs)
        B, D, H, W = sfcvs[0].shape
        # all frames go through the encoder as one batch of F*B volumes (the reference loops, :357-365)
        if x is None or x.dtype != C.act_dtype() or tuple(x.shape) != (nF * B, H, W, D):
            # (standalone call, or a configuration the fused kernel does not write the engine layout for)
            x = torch.empty(nF * B, H, W, D, device=sfcvs[0].device, dtype=C.act_dtype())
            for f, v in enumerate(sfcvs):
                C.nchw_to_nhwc(v, out=x[f * B:(f + 1) * B])
        if not self.use_cv:
            x = torch.zeros_like(x)      # (x may be the caller's buffer: not written)
        cv_feats = []
        fused_pool = nF > 1 and H % 16 == 0 and W % 16 == 0   # (one pass writes the pooled tensor and the frame maximum)
        for lvl in range(5):
            for layer in P[f"enc{lvl}"]:
                x = layer([x])
            if lvl == 4:
                cv_feats.append(C.max_over_frames(x, nF))
            elif fused_pool:
                x, fm = C.pool_and_frame_max(x, nF)
                cv_feats.append(fm)
            else:
                cv_feats.append(C.max_over_frames(x, nF))
                x = C.maxpool2(x)
        img = [C.as_nhwc(f, C.act_dtype()) for f in feats_nchw[:4]]
        if not self.use_features:
            img = [torch.zeros_like(t) for t in img]
        x = None
        for i in range(4):
            up, c1, c2 = P[f"dec{i}"]
            x = up([cv_feats[4], img[3]] if i == 0 else [x])                        # Upconv: no activation
            if i == 0:
                cat = [cv_feats[3], img[2], x]
            elif i == 3:
                cat = [cv_feats[0], x]
            else:
                cat = [cv_feats[3 - i], img[2 - i], x]
            x = c2([c1(cat)])
        m = P["cls"]([x], final=True)                                                # [B,H,W,1]
        return m.view(B, 1, H, W)                                                    # C == 1: NHWC == NCHW


class DepthModule(_PackedSource, nn.Module):
    """Depth U-Net over (masked cost volume (+) keyframe) with 4 output scales (monorec_model.py:476-557)."""

    def __init__(self, depth_steps=32, feature_channels=(64, 64, 128, 256, 512), large_model=False):
        super().__init__()
        if large_model:
            raise NotImplementedError("monorec_b200: depth_large_model is an unused ablation of the reference")
        self.depth_steps = depth_steps
        self.feat_chns = tuple(int(c) for c in feature_channels)
        self._in_channels = depth_steps + 3
        e = self._cv_enc_feat_chns = (48, 64, 128, 192, 256)
        d = self._dec_feat_chns = (256, 128, 64, 48, 32, 24)
        fc = self.feat_chns
        ks = (7, 7, 5, 5, 3)
        self.enc = nn.ModuleList([
            nn.Sequential(ConvReLU2(self._in_channels if i == 0 else e[i - 1], e[i], ks[i], stride=1 if i == 0 else 2),
                          ConvReLU2(e[i], e[i], 3)) for i in range(5)])
        self.dec = nn.ModuleList([
            Refine(e[4], d[0]),
            nn.Sequential(Refine(e[3] + fc[2] + d[0], d[1]), ConvReLU2(d[1], d[1], 3)),
            nn.Sequential(Refine(e[2] + fc[1] + d[1], d[2]), ConvReLU2(d[2], d[2], 3)),
            Refine(e[1] + fc[0] + d[2], d[3]),
            nn.Sequential(ConvReLU2(e[0] + d[3], d[4], 3), nn.Identity(), nn.Conv2d(d[4], d[5], 3),
                          nn.LeakyReLU(negative_slope=0.1))])
        self.predictors = nn.ModuleList([nn.Sequential(nn.Identity(), nn.Conv2d(ch, 1, 3))
                                         for ch in d[:3] + d[-1:]])
        self._packed = _Packed()
        self.out_range = (0.0, 1.0)   # (a, b): heads emit a + b * |tanh| unless forward() is given another affine

    def invalidate_packed_weights(self):
        """After in-place `.data` edits of the parameters (not seen by the version counters): repack on the next call."""
        self._packed.invalidate()

    def _pack_device(self):
        return self.predictors[0][1].weight.device

    def _build(self):
        e, d, fc = self._cv_enc_feat_chns, self._dec_feat_chns, self.feat_chns

        def cr2(m, src_c, pad_in=0):
            wy = m.conv_y.weight
            if pad_in:   # zero input channels appended so that the NHWC input is 16-byte aligned per pixel
                wy = torch.cat([wy, wy.new_zeros(wy.shape[0], pad_in, wy.shape[2], wy.shape[3])], 1)
            return (C.PackedConv(wy, m.conv_y.bias, src_c, stride=(m.stride, 1), act=C.ACT_LEAKY, act_a=C.LEAKY_SLOPE),
                    _leaky(m.conv_x, (m.conv_x.in_channels,), stride=(1, m.stride)))
        cin0 = self._in_channels
        cpad = (-cin0) % (8 if C.MODE == "f16" else 4)   # NHWC pixel stride must be a multiple of 16 bytes
        p = {"enc": [], "cin0_pad": cpad}
        for i, s in enumerate(self.enc):
            first = cr2(s[0], (cin0 + cpad,), cpad) if i == 0 else cr2(s[0], (e[i - 1],))
            p["enc"].append((first, cr2(s[1], (e[i],))))
        p["dec0"] = C.refine_layer(self.dec[0].conv2d_t, (e[4],))
        p["dec1"] = (C.refine_layer(self.dec[1][0].conv2d_t, (e[3], fc[2], d[0])), cr2(self.dec[1][1], (d[1],)))
        p["dec2"] = (C.refine_layer(self.dec[2][0].conv2d_t, (e[2], fc[1], d[1])), cr2(self.dec[2][1], (d[2],)))
        p["dec3"] = C.refine_layer(self.dec[3].conv2d_t, (e[1], fc[0], d[2]))
        p["dec4"] = (cr2(self.dec[4][0], (e[0], d[3])), _leaky(self.dec[4][2], (d[4],)))
        p["heads"] = [C.PackedConv(s[1].weight, s[1].bias, (s[1].in_channels,), act=C.ACT_ABSTANH)
                      for s in self.predictors]
        return p

    @staticmethod
    def _cr2(srcs, pk):
        return pk[1]([pk[0](srcs)])

    @staticmethod
    def _head(x, head, out_range):
        y = head([x], final=True, act_ab=out_range)
        B, H, W, _ = y.shape
        return y.view(B, 1, H, W)

    def forward(self, data_dict, out_range=None):
        """out_range: (a, b) of the heads' a + b * |tanh| for this call (MonoRecModel passes the inverse-depth affine);
        default `self.out_range`, the reference's raw |tanh|.  Passed to the launches, never stored: concurrent calls with
        different ranges are independent."""
        if self.training:
            raise NotImplementedError("monorec_b200.DepthModule: inference only")
        out_range = tuple(self.out_range if out_range is None else out_range)
        keyframe = data_dict.get("_keyframe_rgb", data_dict["keyframe"])   # see rgb_keyframe
        cv = data_dict["cost_volume"]
        feats_nchw = data_dict["image_features"]
        cv_mask = data_dict.get("_cv_mask_for_depth")
        if torch.compiler.is_compiling():
            preds = torch.ops.monorec_b200.depth_module(keyframe, cv, list(feats_nchw[:3]), cv_mask, float(out_range[0]),
                                                        float(out_range[1]), list(self.parameters()), self.depth_steps,
                                                        list(self.feat_chns))
        else:
            preds = self._run(keyframe, cv, feats_nchw, cv_mask, out_range)
        data_dict["predicted_inverse_depths"] = preds
        return data_dict

    def _run(self, keyframe, cv, feats_nchw, cv_mask, out_range):
        """The U-Net on cat(cost volume * (1 - cv_mask), keyframe) and trunk levels 0-2 -> the four inverse-depth maps,
        finest first.  The implementation of the `monorec_b200::depth_module` op as well."""
        P = self._packs(self._build)
        B, D, H, W = cv.shape
        # cat(cost_volume, keyframe) (:531); when MonoRecModel passes the unmasked volume plus `_cv_mask_for_depth`
        # the (1 - cv_mask) product of :713 is applied during the layout change
        cpad = P["cin0_pad"]
        # (the pad channels behind cat(cost volume, keyframe) must be zero, not garbage; the two layout kernels below write
        # channels [0, D + 3), so only the pad channels are cleared -- not the whole 84 MB buffer)
        x = torch.empty(B, H, W, D + 3 + cpad, device=cv.device, dtype=C.act_dtype())
        if cpad:
            x[..., D + 3:].zero_()
        C.nchw_to_nhwc(cv, out=x, out_coff=0, one_minus=cv_mask)
        C.nchw_to_nhwc(keyframe.to(torch.float32), out=x, out_coff=D)
        img = [C.as_nhwc(f, C.act_dtype()) for f in feats_nchw[:3]]
        feats = []
        for (p0, p1) in P["enc"]:
            x = self._cr2([self._cr2([x], p0)], p1)
            feats.append(x)
        heads = P["heads"]
        preds = []
        x = P["dec0"]([feats[4]])                                                     # 256 @ 1/8
        preds.insert(0, self._head(x, heads[0], out_range))
        up, pk = P["dec1"]
        x = self._cr2([up([feats[3], img[2], x])], pk)                                # 128 @ 1/4
        preds.insert(0, self._head(x, heads[1], out_range))
        up, pk = P["dec2"]
        x = self._cr2([up([feats[2], img[1], x])], pk)                                # 64 @ 1/2
        preds.insert(0, self._head(x, heads[2], out_range))
        x = P["dec3"]([feats[1], img[0], x])                                          # 48 @ full
        pk, last = P["dec4"]
        x = last([self._cr2([feats[0], x], pk)])                                      # 24 @ full
        preds.insert(0, self._head(x, heads[3], out_range))
        return preds

    def predict_depth(self, x, scale):
        """API parity with the reference (:554-557); x is NHWC inside this implementation."""
        return self._head(x, self._packs(self._build)["heads"][scale], tuple(self.out_range))


def rgb_keyframe(data_dict):
    """The keyframe as three channels: data_dict["keyframe"] itself, or for a grayscale keyframe [B,1,H,W] its replica
    [B,3,H,W], made at the first call and kept in the dict as `_keyframe_rgb` for the later ones (the trunk and the
    DepthModule read it; MonoRecModel's heads stage drops it)."""
    key = data_dict["keyframe"]
    if key.shape[1] != 1:
        return key
    rgb = data_dict.get("_keyframe_rgb")
    if rgb is None:
        rgb = data_dict["_keyframe_rgb"] = key.expand(-1, 3, -1, -1).contiguous()
    return rgb


class MonoRecModel(nn.Module):
    """Drop-in for model.monorec.monorec_model.MonoRecModel (:560-729); see the module docstring."""

    def __init__(self, inv_depth_min_max=(0.33, 0.0025), cv_depth_steps=32, pretrain_mode=False, pretrain_dropout=0.0,
                 pretrain_dropout_mode=0, augmentation=None, use_mono=True, use_stereo=False, use_ssim=True,
                 sfcv_mult_mask=True, simple_mask=False, mask_use_cv=True, mask_use_feats=True, cv_patch_size=3,
                 depth_large_model=False, no_cv=False, freeze_resnet=True, freeze_module=(), checkpoint_location=None,
                 mask_cp_loc=None, depth_cp_loc=None, volume_dtype=torch.float32):
        super().__init__()
        self.inv_depth_min_max = inv_depth_min_max
        self.cv_depth_steps = cv_depth_steps
        self.use_mono, self.use_stereo, self.use_ssim = use_mono, use_stereo, use_ssim
        self.sfcv_mult_mask = sfcv_mult_mask
        self.pretrain_mode = int(pretrain_mode)
        self.pretrain_dropout, self.pretrain_dropout_mode = pretrain_dropout, pretrain_dropout_mode
        self.augmentation = augmentation
        self.simple_mask, self.mask_use_cv, self.mask_use_feats = simple_mask, mask_use_cv, mask_use_feats
        self.cv_patch_size = cv_patch_size
        self.no_cv = no_cv
        self.depth_large_model = depth_large_model
        self.checkpoint_location, self.mask_cp_loc, self.depth_cp_loc = checkpoint_location, mask_cp_loc, depth_cp_loc
        self.freeze_module, self.freeze_resnet = freeze_module, freeze_resnet
        if simple_mask:
            raise NotImplementedError("monorec_b200: simple_mask is an unused ablation of the reference")
        if augmentation not in (None, "none"):
            raise NotImplementedError("monorec_b200: training-time augmentation is out of scope (inference path)")

        self._feature_extractor = ResnetEncoder(num_layers=18, pretrained=True)
        if self.freeze_resnet:
            for p in self._feature_extractor.parameters(True):
                p.requires_grad_(False)
        self.cv_module = CostVolumeModule(use_mono=use_mono, use_stereo=use_stereo, use_ssim=use_ssim,
                                          sfcv_mult_mask=self.sfcv_mult_mask, patch_size=cv_patch_size,
                                          volume_dtype=volume_dtype)
        self.volume_dtype = volume_dtype
        if not (self.pretrain_mode == 1 or self.pretrain_mode == 3):
            self.att_module = MaskModule(self.cv_depth_steps, self._feature_extractor.num_ch_enc, use_cv=mask_use_cv,
                                         use_features=mask_use_feats)
        if not self.pretrain_mode == 2:
            self.depth_module = DepthModule(self.cv_depth_steps, feature_channels=self._feature_extractor.num_ch_enc,
                                            large_model=self.depth_large_model)
        self._load_checkpoints(checkpoint_location, mask_cp_loc, depth_cp_loc)
        for module_name in self.freeze_module:
            module = getattr(self, module_name + "_module")
            module.eval()
            for param in module.parameters(True):
                param.requires_grad_(False)
        self.augmenter = None
        # torchvision trunk on cuDNN: channels-last so that its outputs are already NHWC for the conv engine (the dict still
        # holds logical (B,C,H,W) tensors).  Done once here, not in forward: forward mutates no module state, so concurrent
        # calls and DataParallel replicas are safe.  load_state_dict / .to() keep the layout.
        self._feature_extractor.to(memory_format=torch.channels_last)

    def invalidate_packed_weights(self):
        """Forget every kernel-layout copy of the parameters (folded trunk, packed conv stacks).  Only needed after edits
        that bypass the tensors' version counters, e.g. `p.data.copy_(ema)`; load_state_dict / .to() / optimizer steps are
        detected automatically."""
        for m in self.modules():
            if m is not self and hasattr(m, "invalidate_packed_weights"):
                m.invalidate_packed_weights()

    # -- checkpoint loading: same key filtering as utils/util.py:244-248 + monorec_model.py:630-657 ------------------
    @staticmethod
    def filter_state_dict(state_dict, data_parallel=False):
        if data_parallel:
            state_dict = {k[7:]: v for k, v in state_dict.items()}
        digits = tuple(str(i) for i in range(1, 10))
        return {(k[2:] if k.startswith("0") else k): v for k, v in state_dict.items() if not k.startswith(digits)}

    def _load_checkpoints(self, checkpoint_location, mask_cp_loc, depth_cp_loc):
        def as_list(x):
            return x if isinstance(x, list) else [x]

        def read(cp):
            checkpoint = torch.load(cp, map_location=torch.device("cpu"), weights_only=False)
            return self.filter_state_dict(checkpoint["state_dict"], checkpoint["arch"] == "DataParallel")
        encoder_loaded = False
        if checkpoint_location is not None:
            for cp in as_list(checkpoint_location):
                sd = read(cp)
                res = self.load_state_dict(sd, strict=False)
                encoder_loaded = encoder_loaded or any(k.startswith("_feature_extractor.") for k in sd)
                if res.missing_keys:
                    warnings.warn(f"monorec_b200: {cp} leaves {len(res.missing_keys)} parameters at their initial values "
                                  f"(first: {res.missing_keys[0]})")
        if getattr(self._feature_extractor, "pretrained_requested_but_missing", False) and not encoder_loaded:
            # the reference always has ImageNet weights at this point (torchvision downloads them, monorec_model.py:104-113)
            warnings.warn("monorec_b200: ResnetEncoder(pretrained=True) found no ImageNet weights in the local hub cache and no "
                          "checkpoint supplied `_feature_extractor.*`: the trunk is randomly initialised")
        if mask_cp_loc is not None:
            for cp in as_list(mask_cp_loc):
                sd = read(cp)
                self.att_module.load_state_dict({k[11:]: v for k, v in sd.items() if k.startswith("att_module")},
                                                strict=False)
        if depth_cp_loc is not None:
            for cp in as_list(depth_cp_loc):
                sd = read(cp)
                self.depth_module.load_state_dict({k[13:]: v for k, v in sd.items() if k.startswith("depth_module")},
                                                  strict=False)

    def forward(self, data_dict):
        """The reference's forward on its data dict.  The images may also be grayscale, [B,1,H,W] (a loader's
        use_color=False, TUM Mono-VO): they mean the three-channel images whose three planes equal them, and every output is
        that of those replicas bit for bit.  The cost volume reads the one-channel frames; the trunk and the DepthModule read
        one three-channel copy of the keyframe, made once here."""
        rgb_keyframe(data_dict)
        data_dict = self._stage_cost_volume(data_dict)
        data_dict = self._stage_trunk(data_dict)
        return self._stage_heads(data_dict)

    # The forward's three stages.  Each adds its outputs to the dict it is given and returns it; the heads read what the
    # other two added and write no tensor they produced, so several models can run their own heads on one cost volume and
    # one trunk output (models_eval.MultiModelEvaluater, which shares them through shallow copies of the dict).
    def _writes_sfcv_nhwc(self):
        """Whether the cost-volume stage also writes the MaskModule's NHWC input (a buffer the heads then read)."""
        return (not self.no_cv and hasattr(self, "att_module") and self.att_module.use_cv and C.MODE in ("tf32", "f16")
                and self.cv_depth_steps <= 32 and self.cv_depth_steps % 8 == 0)

    def _stage_cost_volume(self, data_dict):
        """Stage A: the depth-range entries, `cost_volume`, `single_frame_cvs` (and the MaskModule's NHWC copy of them)."""
        keyframe = data_dict["keyframe"]
        lo, hi = float(self.inv_depth_min_max[1]), float(self.inv_depth_min_max[0])
        # 1-element tensors like the reference's (:675-677); torch.full is a fill kernel (CUDA-graph capturable, no H2D copy)
        data_dict["inv_depth_min"] = torch.full((1,), float(self.inv_depth_min_max[0]), device=keyframe.device, dtype=keyframe.dtype)
        data_dict["inv_depth_max"] = torch.full((1,), float(self.inv_depth_min_max[1]), device=keyframe.device, dtype=keyframe.dtype)
        data_dict["cv_depth_steps"] = torch.full((1,), int(self.cv_depth_steps), device=keyframe.device, dtype=torch.int32)
        data_dict["_cv_range"] = (lo, hi, int(self.cv_depth_steps))   # host copy: no .item() synchronisation

        with torch.no_grad():
            if not self.no_cv:
                if self._writes_sfcv_nhwc():
                    # the MaskModule's NHWC input is written by the cost-volume kernel's per-pixel phase (no layout-change launches)
                    nf = (len(data_dict["frames"]) if self.use_mono else 0) + (1 if self.use_stereo else 0)
                    data_dict["_sfcv_nhwc"] = torch.empty(nf * keyframe.shape[0], keyframe.shape[2], keyframe.shape[3],
                                                          self.cv_depth_steps, device=keyframe.device, dtype=C.act_dtype())
                data_dict = self.cv_module(data_dict)
            else:
                s = list(keyframe.shape)
                s[1] = self.cv_depth_steps
                data_dict["cost_volume"] = keyframe.new_zeros(s, dtype=self.volume_dtype)
                data_dict["single_frame_cvs"] = [data_dict["cost_volume"].clone() for _ in data_dict["poses"]]
        return data_dict

    def _stage_trunk(self, data_dict):
        """Stage B: `image_features`, the ResNet-18 trunk's levels of the key frame."""
        keyframe = rgb_keyframe(data_dict)
        with torch.no_grad():
            # torchvision trunk on cuDNN, fed channels-last; TF32 is allowed there unless the engine runs its fp32 parity mode
            image = (keyframe + .5).contiguous(memory_format=torch.channels_last)
            if torch.compiler.is_compiling():
                # the cuDNN flags and the folded-weight cache are host state: set and looked up inside the op
                enc = self._feature_extractor
                if enc.training or enc.encoder.training:
                    raise NotImplementedError("monorec_b200: a compiled forward runs the trunk in eval mode only")
                data_dict["image_features"] = torch.ops.monorec_b200.resnet_trunk(image, enc._source_tensors(),
                                                                                  C.MODE != "fp32")
            else:
                data_dict["image_features"] = trunk_features(self._feature_extractor, image, C.MODE != "fp32")
        return data_dict

    def _stage_heads(self, data_dict):
        """Stage C: the Mask and Depth stacks, the masking and the heads -> `cv_mask`, `predicted_inverse_depths`, the
        masked `cost_volume` (a new tensor), `result`, `mask`."""
        keyframe = data_dict["keyframe"]
        lo, hi = float(self.inv_depth_min_max[1]), float(self.inv_depth_min_max[0])
        with torch.no_grad():
            if self.pretrain_mode == 0 or self.pretrain_mode == 2:
                data_dict = self.att_module(data_dict)
            elif self.pretrain_mode == 1:
                b, c, h, w = keyframe.shape
                data_dict["cv_mask"] = keyframe.new_zeros(b, 1, h, w)      # eval branch of :706-707
            elif self.pretrain_mode == 3:
                data_dict["cv_mask"] = data_dict["mvobj_mask"].clone().detach()

            if not self.pretrain_mode == 2:
                # cost_volume * (1 - cv_mask) (:713): the product is fused into the depth module's layout change and
                # the masked volume is also materialised for callers that read data_dict["cost_volume"]
                data_dict["_cv_mask_for_depth"] = data_dict["cv_mask"]
                rgb_keyframe(data_dict)     # (the DepthModule reads the three-channel copy of a grayscale keyframe)
                # (1-p)*lo + p*hi (:717-718) in the heads' epilogue; a standalone DepthModule call returns the raw |tanh| heads
                data_dict = self.depth_module(data_dict, out_range=(lo, hi - lo))
                del data_dict["_cv_mask_for_depth"]
                data_dict["cost_volume"] = C.mask_volume(data_dict["cost_volume"], data_dict["cv_mask"])

        if self.pretrain_mode == 2:
            data_dict["result"] = data_dict["cv_mask"]
        else:
            data_dict["result"] = data_dict["predicted_inverse_depths"][0]
            data_dict["mask"] = data_dict["cv_mask"]
        data_dict.pop("_cv_range", None)
        data_dict.pop("_sfcv_nhwc", None)
        data_dict.pop("_sfcv_nhwc_filled", None)
        data_dict.pop("_keyframe_rgb", None)
        return data_dict



class GraphedMonoRec:
    """CUDA-graph replay of MonoRecModel.forward for a fixed input signature.

    The forward is ~150 small launches; issued from Python it is bound by the host (SURVEY.md §3.5 "hidden syncs" are gone,
    the launch overhead is not).  Capturing once and replaying removes the host from the loop.  Inputs are copied into
    static buffers, outputs are the static tensors of the captured run (valid until the next call).  A tensor that appears
    several times in `example` (a key frame that is also one of its own source frames) gets one static buffer, so the
    captured forward reads it through the same pointers as an eager one.
    """

    def __init__(self, model, example, warmup=2):
        self.model = model
        buffers = {}

        def static(t):
            if id(t) not in buffers:
                buffers[id(t)] = t.clone()
            return buffers[id(t)]
        self.static_in = {k: ([static(t) for t in v] if isinstance(v, (list, tuple)) else static(v))
                          for k, v in example.items() if torch.is_tensor(v) or isinstance(v, (list, tuple))}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(warmup):
                self.model(dict(self.static_in))
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.static_out = self.model(dict(self.static_in))

    def __call__(self, data):
        for k, v in self.static_in.items():
            if isinstance(v, list):
                for dst, src in zip(v, data[k]):
                    dst.copy_(src, non_blocking=True)
            else:
                v.copy_(data[k], non_blocking=True)
        return self.replay()

    def replay(self):
        """Runs the captured forward on whatever `static_in` holds now (for callers that write the inputs in place)."""
        self.graph.replay()
        feats = self.static_out.get("image_features")
        if isinstance(feats, _TrunkFeatures):
            feats.reset_tail()
        return self.static_out
