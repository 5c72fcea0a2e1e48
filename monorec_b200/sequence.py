"""MonoRecModel over an image sequence, in batches of key frames.

The reference's callers build one data dict per key frame (data_loader/kitti_odometry_dataset.py:248-269), each with its
own copies of the neighbour frames, and create_pointcloud.py runs them at batch size 1.  `MonoRecSequence` takes the frames
one at a time instead: each is copied to the device once, into a ring of frames, poses and intrinsics, and every
`batch_size` ready key frames are gathered from the ring into one batch dict and run together, by CUDA-graph replay when
`graphed`.
"""
import torch

from .model import GraphedMonoRec


def neighbour_offsets(frame_count, dilation=1):
    """Sequence offsets of a key frame's source frames, in the order of its `frames` / `poses` / `intrinsics` lists
    (kitti_odometry_dataset.py:253-258)."""
    if frame_count < 1 or dilation < 1:
        raise ValueError(f"frame_count ({frame_count}) and dilation ({dilation}) must be >= 1")
    return [i for i in range(-(frame_count // 2) * dilation, ((frame_count + 1) // 2) * dilation + 1, dilation) if i != 0]


class MonoRecSequence:
    """Runs `model` on every key frame of a sequence pushed frame by frame.

    `push(image, pose, intrinsics)` takes frame n of the sequence: image [3,H,W] in [-0.5, 0.5], pose [4,4] camera -> world,
    intrinsics [4,4], on the host or the device.  Key frame i is run once frames i + min(offsets) ... i + max(offsets) are
    in; the key frames at the two ends of the sequence, which lack a neighbour, are never run (the loader's index range,
    kitti_odometry_dataset.py:54-58, 74).  Key frames are run in sequence order, `batch_size` at a time; `flush()` runs the
    rest eagerly at the end of the sequence.

    `push` and `flush` return a list of (sequence index, outputs), one per key frame run by that call, in order.  `outputs`
    holds views, with a batch dimension of 1, of the batch's `result`, `cv_mask`, `cost_volume`, `predicted_inverse_depths`
    (whichever the model's configuration produces) and of its inputs `keyframe`, `keyframe_pose`, `keyframe_intrinsics`.
    With `graphed`, these are the CUDA graph's static tensors: they stay valid until the next replay, i.e. the next
    `push` that runs a batch.  Clone what must outlive it.

    One slice of the sequence (one rank's share, see dist.shard_sequences): `first_frame` is the sequence index of the first
    frame pushed, and key frames from `key_begin` = first_frame + max(0, -min(offsets)) on are run (the first key frame
    whose earlier neighbours are all pushed); `key_end` ends the key frames run (None: the end of the sequence).  Batches
    are counted from the first key frame run, and the last one before key_end is run at the push that completes it,
    eagerly when it is short.  The frames to push are first_frame ... key_end - 1 + max(offsets); `push` refuses a frame
    after those.  Indices (`n_pushed`, the emitted ones) are sequence indices.  The defaults run the whole sequence.

    `model` is a MonoRecModel (or any callable that adds its outputs to the reference's data dict and returns that dict,
    as MonoRecModel.forward does); `device` defaults to the
    device of its parameters.  Stereo frames (`use_stereo`) and `pretrain_mode == 3` (moving-object masks) need inputs a
    frame stream does not carry and raise NotImplementedError.
    """

    def __init__(self, model, frame_count=2, dilation=1, batch_size=8, graphed=True, device=None, first_frame=0,
                 key_end=None):
        if getattr(model, "use_stereo", False):
            raise NotImplementedError("MonoRecSequence: use_stereo needs stereo frames, which a frame stream does not carry")
        if int(getattr(model, "pretrain_mode", 0)) == 3:
            raise NotImplementedError("MonoRecSequence: pretrain_mode 3 needs moving-object masks, which a frame stream "
                                      "does not carry")
        if batch_size < 1:
            raise ValueError(f"batch_size ({batch_size}) must be >= 1")
        if first_frame < 0:
            raise ValueError(f"first_frame ({first_frame}) must be >= 0")
        self.model = model
        self.offsets = neighbour_offsets(frame_count, dilation)
        self.batch_size = int(batch_size)
        self.graphed = bool(graphed)
        self.device = torch.device(device) if device is not None else next(model.parameters()).device
        lo, self._hi = min(0, min(self.offsets)), max(self.offsets)
        self.ring_len = self._hi - lo + 1 + self.batch_size
        self.first_key = -lo               # the sequence's first key frame with all its neighbours in the sequence
        self.key_begin = int(first_frame) - lo
        self.key_end = None if key_end is None else int(key_end)
        self.n_pushed = int(first_frame)   # sequence index of the next frame pushed
        self._next = self.key_begin        # the next key frame to run
        self._rings = None                 # (frames [R,3,H,W], poses [R,4,4], intrinsics [R,4,4])
        self._graph = None
        # ring slots of a batch, relative to its first key frame: row 0 the key frames, row 1 + f their f-th source frames
        rel = torch.tensor([0] + self.offsets).view(-1, 1) + torch.arange(self.batch_size).view(1, -1)
        self._rel = rel.to(self.device)

    def push(self, image, pose, intrinsics):
        if image.dim() != 3 or image.shape[0] != 3 or tuple(pose.shape) != (4, 4) or tuple(intrinsics.shape) != (4, 4):
            raise ValueError(f"MonoRecSequence.push: image [3,H,W], pose [4,4], intrinsics [4,4] expected, got "
                             f"{tuple(image.shape)}, {tuple(pose.shape)}, {tuple(intrinsics.shape)}")
        if self.key_end is not None and self.n_pushed >= self.key_end + self._hi:
            raise ValueError(f"MonoRecSequence.push: frame {self.n_pushed} is past the last frame the key frames before "
                             f"key_end={self.key_end} need ({self.key_end + self._hi - 1})")
        if self._rings is None:
            R, (_, H, W) = self.ring_len, image.shape
            self._rings = (torch.empty(R, 3, H, W, device=self.device), torch.empty(R, 4, 4, device=self.device),
                           torch.empty(R, 4, 4, device=self.device))
        elif image.shape[1:] != self._rings[0].shape[2:]:
            raise ValueError(f"MonoRecSequence.push: frame size {tuple(image.shape[1:])} differs from the sequence's "
                             f"{tuple(self._rings[0].shape[2:])}")
        slot = self.n_pushed % self.ring_len
        for ring, t in zip(self._rings, (image, pose, intrinsics)):
            ring[slot].copy_(t, non_blocking=True)
        self.n_pushed += 1
        n = self._ready()
        if n >= self.batch_size:
            return self._run(self.batch_size, self.graphed)
        if n > 0 and self.key_end is not None and self.n_pushed == self.key_end + self._hi:
            return self._run(n, False)                             # the short last batch before key_end
        return []

    def flush(self):
        """Runs the key frames that are ready but fewer than `batch_size`, eagerly (end of the sequence)."""
        n = self._ready()
        return self._run(n, False) if n > 0 else []

    def _ready(self):
        """Key frames not yet run (before key_end) whose neighbours have all been pushed."""
        ready = self.n_pushed - self._hi
        return (ready if self.key_end is None else min(ready, self.key_end)) - self._next

    def _assemble(self, idx, out=None):
        """The batch dict, with the reference's keys and list order, gathered from the rings at slots `idx` [1+F, n];
        written into `out`'s tensors when given (the graph's static inputs)."""
        frames, poses, intrinsics = self._rings
        data = {}
        for key, ring in (("keyframe", frames), ("keyframe_pose", poses), ("keyframe_intrinsics", intrinsics)):
            data[key] = torch.index_select(ring, 0, idx[0], out=None if out is None else out[key])
        for key, ring in (("frames", frames), ("poses", poses), ("intrinsics", intrinsics)):
            data[key] = [torch.index_select(ring, 0, idx[1 + f], out=None if out is None else out[key][f])
                         for f in range(len(self.offsets))]
        return data

    def _run(self, n, graphed):
        i0 = self._next
        idx = torch.remainder(self._rel[:, :n] + i0, self.ring_len)
        if not graphed:
            out = self.model(self._assemble(idx))
        elif self._graph is None:
            self._graph = GraphedMonoRec(self.model, self._assemble(idx))
            out = self._graph.replay()
        else:
            self._assemble(idx, out=self._graph.static_in)
            out = self._graph.replay()
        self._next += n
        return [(i0 + j, _row(out, j)) for j in range(n)]


_ROW_KEYS = ("result", "cv_mask", "cost_volume", "keyframe", "keyframe_pose", "keyframe_intrinsics")


def _row(out, j):
    v = {k: out[k][j:j + 1] for k in _ROW_KEYS if k in out}
    if "predicted_inverse_depths" in out:
        v["predicted_inverse_depths"] = [p[j:j + 1] for p in out["predicted_inverse_depths"]]
    return v
