"""Device-side drop-ins for the reference's point-cloud export (create_pointcloud.py:65-105, utils/ply_utils.py:8-53).

`PLYSaver` keeps the reference's constructor, `add_depthmap(depth, image, intrinsics, extrinsics)` and `save(file)`; the
vertices stay in one growing device buffer (the reference does `.cpu().tolist()` per frame) and are written in the reference's
order.  `keep_mask` is the 33x33 dilation of the moving-object mask, `MaskVoter` the sliding-window vote of
create_pointcloud.py:80-104.  The arithmetic runs in libmonorec_b200.so (csrc/pointcloud.cu); no CPU fallback.
"""
import ctypes

import torch

from . import _lib


def keep_mask(cv_mask, mask_fill=32, thresh=0.1):
    """(conv2d(cv_mask >= thresh, ones(mask_fill+1), padding=mask_fill//2) < 1) as float  (create_pointcloud.py:77-78)."""
    if not cv_mask.is_cuda:
        raise _lib.MonorecLibraryError("monorec_b200.pointcloud needs CUDA tensors (no CPU fallback)")
    lib = _lib.load()
    m = cv_mask.to(torch.float32).contiguous()
    B, _, H, W = m.shape
    out = torch.empty_like(m)
    with torch.cuda.device(m.device):
        _lib.check(lib.mr_pointcloud_keep_mask(m.data_ptr(), out.data_ptr(), B, H, W, int(mask_fill), float(thresh),
                                               torch.cuda.current_stream(m.device).cuda_stream), "mr_pointcloud_keep_mask")
    return out


class PLYSaver(torch.nn.Module):
    """Drop-in for utils/ply_utils.py:8-53."""

    def __init__(self, height, width, min_d=3, max_d=400, batch_size=1, roi=None, dropout=0):
        super().__init__()
        self.height, self.width = height, width
        self.min_d, self.max_d, self.roi, self.dropout = min_d, max_d, roi, dropout
        self._buf = None            # device float [capacity, 6]
        self._count = None          # device int64 [1]: vertices stored (negative: last add did not fit)

    def __len__(self):
        return 0 if self._count is None else int(self._count.item())

    @property
    def vertices(self):
        """Device tensor [N, 6] (x, y, z, red, green, blue)."""
        n = len(self)
        return self._buf[:n] if n else torch.empty(0, 6)

    def add_depthmap(self, depth, image, intrinsics, extrinsics, keep_masks=(), min_hits=1, rand=None):
        """depth: inverse depth [B,1,H,W] (the reference's argument name); keep_masks: the voting window's masks (optional:
        the reference multiplies the depth by the voted mask before calling; passing the masks here fuses that product)."""
        if not depth.is_cuda:
            raise _lib.MonorecLibraryError("monorec_b200.pointcloud needs CUDA tensors (no CPU fallback)")
        lib = _lib.load()
        dev = depth.device
        d = depth.to(torch.float32).contiguous()
        img = image.to(torch.float32).contiguous()
        K = intrinsics.to(torch.float32).contiguous()
        P = extrinsics.to(torch.float32).contiguous()
        B, _, H, W = d.shape
        masks = [m.to(torch.float32).contiguous() for m in keep_masks]
        if self.dropout > 0 and rand is None:
            rand = torch.rand_like(d)                                     # ply_utils.py:44-45
        n_before, ws, ws_bytes, roi = self._reserve(lib, B, H, W, dev)
        with torch.cuda.device(dev):
            _lib.check(lib.mr_pointcloud_add(d.data_ptr(), img.data_ptr(), K.data_ptr(), P.data_ptr(),
                                             _lib.ptr_array(masks) if masks else None, len(masks), int(min_hits), B, H, W,
                                             float(self.min_d), float(self.max_d), roi,
                                             None if rand is None else rand.contiguous().data_ptr(), float(self.dropout),
                                             self._buf.data_ptr(), self._buf.shape[0], n_before, self._count.data_ptr(),
                                             ws.data_ptr(), ws_bytes, torch.cuda.current_stream(dev).cuda_stream),
                       "mr_pointcloud_add")

    def _reserve(self, lib, B, H, W, dev):
        """Room for B more depth maps: (n_before, workspace, its bytes, roi as a C array)."""
        if self._buf is None:
            self._buf = torch.empty(max(4 * B * H * W, 1 << 20), 6, device=dev)
            self._count = torch.zeros(1, dtype=torch.int64, device=dev)
        ws_bytes = lib.mr_pointcloud_workspace(B, H, W)
        ws = torch.empty(ws_bytes // 4, dtype=torch.int32, device=dev)
        roi = None if self.roi is None else (ctypes.c_int * 4)(*[int(v) for v in self.roi])
        # the buffer position of this batch is the count so far: one 8-byte D2H per batch (the reference copies every vertex)
        n_before = int(self._count.item())
        if n_before + B * H * W > self._buf.shape[0]:
            grown = torch.empty(2 * (n_before + B * H * W), 6, device=dev)
            grown[:n_before] = self._buf[:n_before]
            self._buf = grown
        return n_before, ws, ws_bytes, roi

    def add_depthmap_windows(self, depth, image, intrinsics, extrinsics, keep_ring, window_start, n_masks, min_hits=1,
                             rand=None):
        """`add_depthmap` of B consecutive key frames, each voted with its own window: key frame b keeps the pixels where
        more than n_masks - min_hits of the keep masks in ring slots window_start[b], window_start[b] + 1, ...
        (mod len(keep_ring)) are 1.  The vertices are those of B add_depthmap calls, in the same order.
        keep_ring: device [R,1,H,W]; window_start: B host ints."""
        if not depth.is_cuda:
            raise _lib.MonorecLibraryError("monorec_b200.pointcloud needs CUDA tensors (no CPU fallback)")
        lib = _lib.load()
        dev = depth.device
        d = depth.to(torch.float32).contiguous()
        img = image.to(torch.float32).contiguous()
        K = intrinsics.to(torch.float32).contiguous()
        P = extrinsics.to(torch.float32).contiguous()
        ring = keep_ring.to(torch.float32).contiguous()
        B, _, H, W = d.shape
        if len(window_start) != B or tuple(ring.shape[1:]) != (1, H, W):
            raise ValueError(f"add_depthmap_windows: {len(window_start)} window starts and a keep ring of "
                             f"{tuple(ring.shape)} for depth maps {tuple(d.shape)}")
        if self.dropout > 0 and rand is None:
            rand = torch.rand_like(d)                                     # ply_utils.py:44-45
        starts = (ctypes.c_int * B)(*[int(v) for v in window_start])
        n_before, ws, ws_bytes, roi = self._reserve(lib, B, H, W, dev)
        with torch.cuda.device(dev):
            _lib.check(lib.mr_pointcloud_add_windows(d.data_ptr(), img.data_ptr(), K.data_ptr(), P.data_ptr(), ring.data_ptr(),
                                                     ring.shape[0], starts, int(n_masks), int(min_hits), B, H, W,
                                                     float(self.min_d), float(self.max_d), roi,
                                                     None if rand is None else rand.contiguous().data_ptr(),
                                                     float(self.dropout), self._buf.data_ptr(), self._buf.shape[0], n_before,
                                                     self._count.data_ptr(), ws.data_ptr(), ws_bytes,
                                                     torch.cuda.current_stream(dev).cuda_stream),
                       "mr_pointcloud_add_windows")

    def gather(self, group=None, dst=0):
        """Every rank's vertices, in rank order, on rank `dst` of `group` (a torch.distributed process group; a collective:
        every rank calls it); None on the other ranks.  With ranks holding consecutive key frames (dist.shard_sequences),
        that is the one-process vertex order."""
        from .dist import gather_rows
        v = self.vertices.detach()
        if not v.is_cuda:                                # nothing added on this rank yet: an empty buffer on its device
            v = torch.empty(0, 6, device=torch.device("cuda", torch.cuda.current_device()) if self._buf is None
                            else self._buf.device)
        return gather_rows(v, dst=dst, group=group)

    def save(self, file, group=None):
        """Binary little-endian PLY, the reference's header (ply_utils.py:20-32).  With `group`, a collective: rank 0 of the
        group writes every rank's vertices (`gather`) to its `file`; the other ranks write nothing (their `file` may be
        None)."""
        if group is not None:
            v = self.gather(group)
            if v is None:
                return
        else:
            v = self.vertices
        v = v.detach().to("cpu", torch.float32).contiguous()
        header = ("ply\nformat binary_little_endian 1.0\n"
                  f"element vertex {v.shape[0]}\n"
                  "property float x\nproperty float y\nproperty float z\n"
                  "property float red\nproperty float green\nproperty float blue\nend_header\n")
        file.write(header.encode(encoding="ascii"))
        file.write(v.numpy().tobytes())


class MaskVoter:
    """The sliding window of create_pointcloud.py:80-104: push one frame's tensors, get back the key frame (the middle of the
    window) with the window's keep masks once `buffer_length` frames are in."""

    def __init__(self, buffer_length=5, min_hits=1, mask_fill=32, thresh=0.1):
        self.buffer_length, self.min_hits, self.mask_fill, self.thresh = buffer_length, min_hits, mask_fill, thresh
        self.frames = []

    def push(self, result, data):
        out = result["result"]
        cvm = result["cv_mask"] if "cv_mask" in result else out.new_zeros(out.shape)
        self.frames.append((keep_mask(cvm, self.mask_fill, self.thresh), data["keyframe_pose"], data["keyframe_intrinsics"],
                            data["keyframe"], out))
        if len(self.frames) < self.buffer_length:
            return None
        key = self.frames[self.buffer_length // 2]
        masks = [f[0] for f in self.frames]
        del self.frames[0]
        return {"depth": key[4], "keyframe": key[3], "intrinsics": key[2], "pose": key[1], "keep_masks": masks,
                "min_hits": self.min_hits}


class SequencePointCloud:
    """create_pointcloud.py:65-105 over a `MonoRecSequence`: push frames, and every key frame the sequence runs is voted with
    the keep masks of the `buffer_length` key frames around it and added to `saver`, as the reference's loop does at batch
    size 1.  The windows cross batch boundaries: this keeps its own ring of keep masks, and the last buffer_length // 2
    key frames of a batch wait for the next one.  One `mr_pointcloud_add_windows` call per batch.

    `push(image, pose, intrinsics, rand=None)` and `flush()` forward to the sequence and return what it returns.  `rand`
    [1,H,W] (or [1,1,H,W]): the dropout numbers of this frame's depth map, used if it is added (`add_depthmap`'s `rand`);
    uniform random numbers when None and `saver.dropout` > 0.

    The windows stay inside the sequence: a run over several sequences takes one SequencePointCloud per sequence, into one
    saver.  One rank's share of the export (see dist.shard_sequences(..., buffer_length=...)): `seq` runs a slice of the
    sequence (MonoRecSequence(first_frame=slice.frames[0], key_end=slice.run[1])), and only the key frames of `emit`
    (slice.emit, sequence indices [lo, hi)) are added; the slice's other key frames are run for their keep masks only.
    `saver.save(file, group)` then writes every rank's vertices into rank 0's file."""

    def __init__(self, seq, saver, buffer_length=5, min_hits=1, mask_fill=32, thresh=0.1, emit=None):
        if buffer_length < 1 or not 1 <= min_hits <= buffer_length:
            raise ValueError(f"buffer_length ({buffer_length}) >= 1 and 1 <= min_hits ({min_hits}) <= buffer_length needed")
        if seq.batch_size > 256:
            raise ValueError(f"sequence_pointcloud: batch_size {seq.batch_size} > 256 (mr_pointcloud_add_windows' limit)")
        self.seq, self.saver = seq, saver
        self.buffer_length, self.min_hits, self.mask_fill, self.thresh = buffer_length, min_hits, mask_fill, thresh
        self.key_index = buffer_length // 2
        # a batch's windows span its own key frames plus buffer_length - 1 earlier ones
        self.ring_len = seq.batch_size + buffer_length - 1
        self._keep = None          # [ring_len,1,H,W]: keep mask of the key frame at position n in slot n % ring_len
        self.emit = None if emit is None else (int(emit[0]), int(emit[1]))
        if self.emit is not None and (self.emit[0] < seq.key_begin
                                      or (seq.key_end is not None and self.emit[1] > seq.key_end)):
            raise ValueError(f"SequencePointCloud: emit {self.emit} outside the key frames the sequence runs "
                             f"({seq.key_begin} ... {seq.key_end})")
        self._n_run = seq.key_begin - seq.first_key    # position in the sequence's key frames of the next key frame run
        self._waiting = None       # (positions, depth, keyframe, intrinsics, pose) of run key frames whose window is open
        self._rand = {}            # sequence index -> dropout numbers of the key frame

    def push(self, image, pose, intrinsics, rand=None):
        if rand is not None:
            self._rand[self.seq.n_pushed] = rand.to(self.seq.device, torch.float32).reshape(1, 1, *rand.shape[-2:])
        emitted = self.seq.push(image, pose, intrinsics)
        self._add(emitted)
        return emitted

    def flush(self):
        emitted = self.seq.flush()
        self._add(emitted)
        return emitted

    def _add(self, emitted):
        if not emitted:
            return
        n, R = len(emitted), self.ring_len
        keep = keep_mask(torch.cat([o["cv_mask"] for _, o in emitted]), self.mask_fill, self.thresh)
        if self._keep is None:
            self._keep = torch.empty((R,) + tuple(keep.shape[1:]), device=keep.device)
        first = self._n_run % R                                   # at most two contiguous runs of slots
        k = min(n, R - first)
        self._keep[first:first + k] = keep[:k]
        self._keep[:n - k] = keep[k:]
        # the key frames with a complete window: positions key_index .. last - (buffer_length - 1 - key_index)
        pos = list(range(self._n_run, self._n_run + n))
        fields = [torch.cat([o[key] for _, o in emitted]) for key in ("result", "keyframe", "keyframe_intrinsics",
                                                                      "keyframe_pose")]
        index = [i for i, _ in emitted]
        if self._waiting is not None:
            pos = self._waiting[0] + pos
            index = self._waiting[1] + index
            fields = [torch.cat([w, f]) for w, f in zip(self._waiting[2], fields)]
        self._n_run += n
        last_ready = self._n_run - 1 - (self.buffer_length - 1 - self.key_index)
        e0, e1 = (index[0], index[-1] + 1) if self.emit is None else self.emit
        # never added: their window starts before the sequence, or they are before the emitted key frames
        lo = sum(1 for p, i in zip(pos, index) if p < self.key_index or i < e0)
        hi = sum(1 for p, i in zip(pos, index) if p <= last_ready and i < e1)
        end = sum(1 for i in index if i < e1)                        # the key frames after `emit` are never added
        if hi > lo:
            if self.saver.dropout > 0:
                shape = (1, 1) + tuple(fields[0].shape[-2:])
                rand = torch.cat([self._rand[i] if i in self._rand else torch.rand(shape, device=keep.device)
                                  for i in index[lo:hi]])
            else:
                rand = None
            self.saver.add_depthmap_windows(*[f[lo:hi] for f in fields], self._keep,
                                            [(p - self.key_index) % R for p in pos[lo:hi]], self.buffer_length,
                                            self.min_hits, rand=rand)
        # the rest waits for the next batch (`fields` are torch.cat copies: the next replay does not overwrite them)
        hi = max(hi, lo)
        self._waiting = (pos[hi:end], index[hi:end], [f[hi:end] for f in fields]) if hi < end else None
        upto = index[hi - 1] if hi > 0 else None
        if upto is not None:
            self._rand = {i: r for i, r in self._rand.items() if i > upto}


def sequence_pointcloud(seq, saver, buffer_length=5, min_hits=1, mask_fill=32):
    """The point-cloud export of create_pointcloud.py over `seq` (a MonoRecSequence) into `saver` (a PLYSaver); see
    `SequencePointCloud`."""
    return SequencePointCloud(seq, saver, buffer_length=buffer_length, min_hits=min_hits, mask_fill=mask_fill)
