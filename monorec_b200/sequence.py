"""MonoRecModel over an image sequence, in batches of key frames.

The reference's callers build one data dict per key frame (data_loader/kitti_odometry_dataset.py:248-269), each with its
own copies of the neighbour frames, and create_pointcloud.py runs them at batch size 1.  `MonoRecSequence` takes the frames
one at a time instead: each is copied to the device once, into a ring of frames, poses and intrinsics, and every
`batch_size` ready key frames are gathered from the ring into one batch dict and run together, by CUDA-graph replay when
`graphed`.

The reference's KITTI loader can also select the key frames (`use_index_mask`; `loader_keys` restates its list), add the
right camera's frame (`return_stereo`) and a moving-object mask (`return_mvobj_mask`) to every key frame's dict; the
sequence takes those as `keys=`, `stereo=True` and `mvobj_masks=True`.

The reference's other frame streams pick their key and source frames differently: KITTI with `offset_d` or `max_length`,
TUM Mono-VO and Oxford RobotCar.  A `FrameLayout` (`kitti_layout`, `tum_mono_vo_layout`, `robotcar_layout`) holds one
sequence's source-frame offsets in the loader's list order and its key frames; the sequence takes it as `layout=`.
"""
import bisect
import functools
import sys
from typing import NamedTuple, Tuple

import torch

from .model import GraphedMonoRec


def neighbour_offsets(frame_count, dilation=1):
    """Sequence offsets of a key frame's source frames, in the order of its `frames` / `poses` / `intrinsics` lists
    (kitti_odometry_dataset.py:253-258)."""
    if frame_count < 1 or dilation < 1:
        raise ValueError(f"frame_count ({frame_count}) and dilation ({dilation}) must be >= 1")
    return [i for i in range(-(frame_count // 2) * dilation, ((frame_count + 1) // 2) * dilation + 1, dilation) if i != 0]


def loader_keys(length, frame_count=2, dilation=1, lidar_depth=False, annotated_lidar=True, index_masks=None):
    """The sequence indices (`image_id`) of the loader's key frames of one sequence of `length` frames, in order
    (kitti_odometry_dataset.py:54-76, 216-219).

    The loader's range is [offset, length + offset - extra_frames) with offset = (frame_count // 2) * dilation and
    extra_frames = frame_count * dilation, raised to at least 5 and 10 when `lidar_depth` and `annotated_lidar` (the
    annotated depth maps of eval_monorec.json).  `index_masks`: the loaded JSON dicts of `use_index_mask` (str(index) ->
    bool); a key frame stays only if every mask lists it as true.  None and () give the same list, as in the loader."""
    if frame_count < 1 or dilation < 1:
        raise ValueError(f"frame_count ({frame_count}) and dilation ({dilation}) must be >= 1")
    offset, extra = (frame_count // 2) * dilation, frame_count * dilation
    if annotated_lidar and lidar_depth:
        offset, extra = max(offset, 5), max(extra, 10)
    keys = range(offset, int(length) + offset - extra)
    for m in index_masks or ():
        keys = [k for k in keys if m.get(str(k))]
    return list(keys)


class FrameLayout(NamedTuple):
    """One sequence's frame layout: which frames a key frame's dict holds, and which key frames the loader serves.

    `offsets`: the sequence offsets of the source frames from the key frame, in the order of the dict's `frames` / `poses`
    / `intrinsics` lists (the fused cost volume sums over the frames in that order).  They may include 0 (the key frame is
    one of its own source frames) and need not be symmetric.  `keys`: the key frames' sequence indices, increasing."""
    offsets: Tuple[int, ...]
    keys: Tuple[int, ...]


def _inside(keys, offsets, length, drop, loader):
    """The key frames whose source frames all lie in the sequence [0, length).  A key frame with a source frame outside
    raises ValueError, unless `drop`: the reference loader would read a frame before 0 at a negative index, which Python
    wraps to the end of the sequence, and a frame past the end raises IndexError there."""
    lo, hi = min(offsets), max(offsets)
    out = []
    for k in keys:
        if k + lo >= 0 and k + hi < length:
            out.append(k)
        elif not drop:
            if k + lo < 0:
                raise ValueError(f"{loader}: key frame {k} needs frame {k + lo}, before the sequence; the reference loader's "
                                 f"negative index wraps to frame {k + lo + length}.  drop_outside=True leaves such key "
                                 "frames out")
            raise ValueError(f"{loader}: key frame {k} needs frame {k + hi}, past the sequence of {length} frames (the "
                             "reference loader raises IndexError).  drop_outside=True leaves such key frames out")
    return out


def kitti_layout(length, frame_count=2, dilation=1, offset_d=0, max_length=None, lidar_depth=False, annotated_lidar=True,
                 index_masks=None, drop_outside=False):
    """The KITTI loader's layout of one sequence of `length` frames.

    The key frames are `loader_keys(length, frame_count, dilation, lidar_depth, annotated_lidar, index_masks)`, cut to the
    first `max_length` (kitti_odometry_dataset.py:78-79, after the index masks).  The source frames are at k + i + offset_d
    for i in neighbour_offsets(frame_count, dilation) (:253-258): `offset_d` shifts the sources, not the key range, so a
    negative one puts the key frame among its own sources (offset_d=-1, frame_count=2: k-2 and k) and makes the stream
    causal.  The key frames whose sources fall outside the sequence (a negative `offset_d` on the first key frames, a
    positive one on the last) raise ValueError unless `drop_outside` (see `_inside`).  The defaults give
    neighbour_offsets(frame_count, dilation) and loader_keys(length, frame_count, dilation)."""
    offsets = [i + int(offset_d) for i in neighbour_offsets(frame_count, dilation)]
    keys = loader_keys(length, frame_count, dilation, lidar_depth, annotated_lidar, index_masks)
    if max_length is not None:
        if max_length < 0:
            raise ValueError(f"max_length ({max_length}) must be None or >= 0")
        keys = keys[:int(max_length)]
    return FrameLayout(tuple(offsets), tuple(_inside(keys, offsets, int(length), drop_outside, "kitti_layout")))


def tum_mono_vo_layout(length, frame_count=2, dilation=1, max_length=None, keyframe_indices=None):
    """The TUM Mono-VO loader's layout of one sequence of `length` frames (the rows of its result.txt).

    With offset = (frame_count // 2) * dilation, the source frames are at k - offset + i for i in range(0, (frame_count + 1)
    * dilation, dilation) except i == offset, in that order (tum_mono_vo_dataset.py:115-139).  The key frames are offset
    ... offset + min(length - frame_count * dilation, max_length) - 1 (:64-72); with `keyframe_indices` (the loader's
    `only_keyframes`), those of the given sequence indices that pass the loader's border rule, k >= offset and
    k < length - (frame_count // 2 + 1) * dilation (:164-174), and `max_length` does not apply, as in the loader.

    `keyframe_indices` are the sequence indices of the frames with a depth map; the loader maps each
    images_depth/NNNNN_d.exr to the first result.txt row whose image is not before NNNNN (data loading, the caller's)."""
    if frame_count < 1 or dilation < 1:
        raise ValueError(f"frame_count ({frame_count}) and dilation ({dilation}) must be >= 1")
    offset = (frame_count // 2) * dilation
    offsets = [i - offset for i in range(0, (frame_count + 1) * dilation, dilation) if i != offset]
    length = int(length)
    if keyframe_indices is None:
        n = length - frame_count * dilation
        if max_length is not None:
            if max_length < 0:
                raise ValueError(f"max_length ({max_length}) must be None or >= 0")
            n = min(n, int(max_length))
        keys = list(range(offset, offset + max(n, 0)))
    else:
        border = length - (frame_count // 2 + 1) * dilation
        keys = [int(k) for k in keyframe_indices if offset <= int(k) < border]
    return FrameLayout(tuple(offsets), tuple(_inside(keys, offsets, length, False, "tum_mono_vo_layout")))


def robotcar_layout(length, frame_count=2, dilation=1, drop_outside=False):
    """The Oxford RobotCar loader's layout of one sequence of `length` frames (oxford_robotcar_dataset.py:55-61, :80-85).

    The source frames are at k + i * dilation for i in range(-frame_count // 2, (frame_count + 1) // 2 + 1), i != 0, with
    Python's floor division: an odd frame_count gives frame_count + 1 source frames (3: -2, -1, 1, 2).  The key frames are
    offset ... length - frame_count + offset - 1 with offset = (frame_count // 2) * dilation; the loader trims frame_count
    frames, not frame_count * dilation, so with dilation > 1 the last key frames need frames past the sequence, and an odd
    frame_count makes the first one need frame -1.  Those raise ValueError unless `drop_outside` (see `_inside`)."""
    if frame_count < 1 or dilation < 1:
        raise ValueError(f"frame_count ({frame_count}) and dilation ({dilation}) must be >= 1")
    offsets = [i * dilation for i in range(-frame_count // 2, (frame_count + 1) // 2 + 1) if i != 0]
    offset = (frame_count // 2) * dilation
    keys = range(offset, int(length) - frame_count + offset)
    return FrameLayout(tuple(offsets), tuple(_inside(keys, offsets, int(length), drop_outside, "robotcar_layout")))


def check_keys(keys, offsets, length=None):
    """`keys` as a list of ints, checked to be increasing sequence indices of key frames with all their neighbours (at
    `offsets`) in the sequence: from -min(offsets) on, and before length - max(offsets) when `length` is given (the key
    frame itself counts as offset 0)."""
    keys = [int(k) for k in keys]
    lo, hi = min(0, min(offsets)), max(0, max(offsets))
    end = None if length is None else int(length) - hi
    if any(b <= a for a, b in zip(keys, keys[1:])) or (keys and (keys[0] < -lo or (end is not None and keys[-1] >= end))):
        raise ValueError(f"key frames must be increasing sequence indices in [{-lo}, {'...' if end is None else end}): the "
                         "key frames with all their neighbours in the sequence")
    return keys


def needs_frame(keys, offsets, n):
    """Whether frame n is one of the key frames `keys` (sorted: a list or a range) or one of their neighbours at `offsets`."""
    return any(_listed(keys, n - u) for u in [0] + list(offsets))


def _listed(keys, k):
    """Whether k is in the sorted `keys`: a range answers by arithmetic, a list by bisection."""
    if isinstance(keys, range):
        return k in keys
    i = bisect.bisect_left(keys, k)
    return i < len(keys) and keys[i] == k


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

    `keys`: a sorted list of the sequence indices of the key frames to run (`loader_keys`: the loader's index-masked or
    annotated-lidar list) instead of every key frame with its neighbours.  Batches are `batch_size` consecutive listed key
    frames, counted from the first listed key frame run, and the short last batch runs at the push that completes the last
    listed key frame.  Only the frames a listed key frame needs (`needs(n)`) are copied; `push` accepts the others and
    copies nothing, and `skip()` passes one without its image, so the caller need not read it.  The ring then holds
    batch_size * (frame_count + 1) + the neighbour span frames, however far apart the listed key frames are.  With
    `first_frame` / `key_end`, the listed key frames in [key_begin, key_end) are run.

    `stereo=True`: `push(..., stereo=(image, pose, intrinsics))` takes the frame's right-camera image [3,H,W], pose (the
    left pose @ the baseline transform) and intrinsics, and the batch dict holds them as `stereoframe`, `stereoframe_pose`,
    `stereoframe_intrinsics` (kitti_odometry_dataset.py:271-278), as a `use_stereo` model needs.  `mvobj_masks=True`:
    `push(..., mvobj_mask=[1,H,W])`, and the batch dict holds `mvobj_mask` [B,1,H,W] (:280-282), as `pretrain_mode == 3`
    needs.  `push(..., target=[1,H,W])` puts the frame's ground truth into the batch dict as `target`, as evaluate.py does
    (SequenceEvaluater uses it); a mask or target given at the first push that copies a frame is then needed for every key
    frame.  These are copied for the key frames only, into rings next to the frames', gathered with them into the batch
    (the CUDA graph's static inputs) and returned in each key frame's outputs.

    `use_color=False` (the KITTI loader's name for its grayscale cameras; TUM Mono-VO is grayscale too): `push` takes
    one-channel images [1,H,W], and stereo images [1,H,W] too, and the frame rings hold one plane.  The model reads them as
    the three-channel images whose planes equal them (MonoRecModel.forward), so the outputs are those of a colour sequence
    fed the replicated frames, bit for bit; the key frame's `keyframe` output is the one-channel image.

    `residual_image=True`: each key frame's outputs also hold `residual_image` [1,1,H,W], the reference's photometric
    residual image (layers.ResidualImage) of its `result`, an inverse depth, against the frames and poses its cost volume
    used (the mono frames, then the stereo frame of a `use_stereo` model).  It is computed in the same forward, inside the
    graph replay when `graphed`, with no host synchronisation; the other outputs are those of residual_image=False bit for
    bit.

    `layout` (a FrameLayout: `kitti_layout` with `offset_d` / `max_length`, `tum_mono_vo_layout`, `robotcar_layout`)
    replaces frame_count, dilation and keys: each key frame's `frames` / `poses` / `intrinsics` are the frames at its
    layout offsets, in their order, and the layout's key frames are run as a `keys` list is.  Offset 0 gathers the key
    frame's own frame again.  A key frame is run once its largest offset (or itself, when all are negative) is pushed: a
    causal layout runs each key frame at the push of that frame.

    `model` is a MonoRecModel (or any callable that adds its outputs to the reference's data dict and returns that dict,
    as MonoRecModel.forward does); `device` defaults to the device of its parameters.  A `use_stereo` model without
    `stereo=True`, and `pretrain_mode == 3` without `mvobj_masks=True`, raise NotImplementedError: a plain frame stream
    does not carry their inputs.
    """

    def __init__(self, model, frame_count=2, dilation=1, batch_size=8, graphed=True, device=None, first_frame=0,
                 key_end=None, keys=None, stereo=False, mvobj_masks=False, use_color=True, residual_image=False,
                 layout=None):
        if getattr(model, "use_stereo", False) and not stereo:
            raise NotImplementedError("MonoRecSequence: use_stereo needs stereo frames: MonoRecSequence(stereo=True) and "
                                      "push(..., stereo=(image, pose, intrinsics))")
        if int(getattr(model, "pretrain_mode", 0)) == 3 and not mvobj_masks:
            raise NotImplementedError("MonoRecSequence: pretrain_mode 3 needs moving-object masks: "
                                      "MonoRecSequence(mvobj_masks=True) and push(..., mvobj_mask=...)")
        if residual_image and int(getattr(model, "pretrain_mode", 0)) == 2:
            raise NotImplementedError("MonoRecSequence: residual_image needs an inverse depth as `result`; pretrain_mode 2 "
                                      "returns the mask there")
        if batch_size < 1:
            raise ValueError(f"batch_size ({batch_size}) must be >= 1")
        if first_frame < 0:
            raise ValueError(f"first_frame ({first_frame}) must be >= 0")
        if layout is not None and keys is not None:
            raise ValueError("MonoRecSequence: give keys or layout, not both (a layout holds its key frames)")
        self.model = model
        self.layout = layout
        if layout is None:
            self.offsets = neighbour_offsets(frame_count, dilation)
        else:
            self.offsets, keys = [int(u) for u in layout.offsets], layout.keys
            if not self.offsets:
                raise ValueError("MonoRecSequence: the layout has no source frames")
        self.batch_size = int(batch_size)
        self.graphed = bool(graphed)
        self.stereo, self.mvobj_masks = bool(stereo), bool(mvobj_masks)
        self.use_color = bool(use_color)
        self.residual_image = bool(residual_image)
        # what a batch runs: the model, or the model and the residual image of its result.  A function of the model only,
        # not a method of the sequence: the CUDA graph keeps it, and a sequence -> graph -> sequence cycle would leave a
        # dropped sequence's graph to the cyclic collector, which may then destroy it during another graph's capture
        self._forward = functools.partial(_with_residual_image, model) if self.residual_image else model
        self.channels = 3 if self.use_color else 1
        self.device = torch.device(device) if device is not None else next(model.parameters()).device
        # the frames a key frame i uses are i + lo ... i + hi (its own frame included)
        lo, self._hi = min(0, min(self.offsets)), max(0, max(self.offsets))
        self.first_key = -lo               # the sequence's first key frame with all its neighbours in the sequence
        self.key_begin = int(first_frame) - lo
        self.key_end = None if key_end is None else int(key_end)
        self.n_pushed = int(first_frame)   # sequence index of the next frame pushed
        self._rings = None                 # (frames [R,3,H,W], poses [R,4,4], intrinsics [R,4,4])
        self._maps = None                  # key-frame inputs beside the frames: batch-dict key -> ring [R,...]
        self._graph = None
        self._uses = [0] + self.offsets    # a key frame's own frame, then its source frames
        if keys is None:
            # every key frame: when batch [k, k+B) runs, the live frames are k+lo ... k+B-1+hi (all earlier ones are freed)
            self.keys, listed = None, range(self.first_key, sys.maxsize)
            self.ring_len = self._hi - lo + 1 + self.batch_size
        else:
            self.keys = listed = check_keys(keys, self.offsets)
            self.ring_len = self.batch_size * len(self._uses) + self._hi - lo
        self.key_position = bisect.bisect_left(listed, self.key_begin)   # place of the first key frame run in the list
        end = len(listed) if self.key_end is None else bisect.bisect_left(listed, self.key_end)
        self._run_keys = listed[self.key_position:end]
        self._next = 0                     # the next key frame to run: its place in _run_keys
        self._slot = {}                    # sequence index of a copied frame -> (ring slot, last key frame that uses it)
        self._free = list(range(self.ring_len))[::-1]

    def needs(self, n):
        """Whether `push` copies frame n: it is a key frame this sequence runs or a neighbour of one."""
        return needs_frame(self._run_keys, self.offsets, n)

    def runs(self, n):
        """Whether key frame n is one this sequence runs (for keys=None: any frame in [key_begin, key_end))."""
        return _listed(self._run_keys, n)

    def skip(self):
        """Passes the next frame without its data; only a frame that no key frame run needs (`needs`) can be skipped."""
        if self.needs(self.n_pushed):
            raise ValueError(f"MonoRecSequence.skip: frame {self.n_pushed} is needed by a key frame the sequence runs")
        self.n_pushed += 1

    def push(self, image, pose, intrinsics, stereo=None, mvobj_mask=None, target=None):
        C = self.channels
        if image.dim() != 3 or image.shape[0] != C or tuple(pose.shape) != (4, 4) or tuple(intrinsics.shape) != (4, 4):
            raise ValueError(f"MonoRecSequence.push: image [{C},H,W], pose [4,4], intrinsics [4,4] expected, got "
                             f"{tuple(image.shape)}, {tuple(pose.shape)}, {tuple(intrinsics.shape)}")
        if self.key_end is not None and self.n_pushed >= self.key_end + self._hi:
            raise ValueError(f"MonoRecSequence.push: frame {self.n_pushed} is past the last frame the key frames before "
                             f"key_end={self.key_end} need ({self.key_end + self._hi - 1})")
        if stereo is not None and not self.stereo:
            raise ValueError("MonoRecSequence.push: stereo frames need MonoRecSequence(stereo=True)")
        n = self.n_pushed
        if not self.needs(n):
            self.n_pushed += 1
            return []
        H, W = image.shape[1:]
        maps = self._key_inputs(H, W, stereo, mvobj_mask, target)
        if self._rings is None:
            R = self.ring_len
            self._rings = (torch.empty(R, self.channels, H, W, device=self.device), torch.empty(R, 4, 4, device=self.device),
                           torch.empty(R, 4, 4, device=self.device))
            # the key-frame inputs the sequence is built for, and the optional ones this first push gives
            shapes = {}
            if self.stereo:
                shapes.update(stereoframe=(self.channels, H, W), stereoframe_pose=(4, 4), stereoframe_intrinsics=(4, 4))
            if self.mvobj_masks or "mvobj_mask" in maps:
                shapes["mvobj_mask"] = (1, H, W)
            if "target" in maps:
                shapes["target"] = (1, H, W)
            self._maps = {k: torch.empty((R,) + v, device=self.device) for k, v in shapes.items()}
        elif image.shape[1:] != self._rings[0].shape[2:]:
            raise ValueError(f"MonoRecSequence.push: frame size {tuple(image.shape[1:])} differs from the sequence's "
                             f"{tuple(self._rings[0].shape[2:])}")
        slot = self._store(n)
        for ring, t in zip(self._rings, (image, pose, intrinsics)):
            ring[slot].copy_(t, non_blocking=True)
        if self.runs(n):
            if set(maps) != set(self._maps):
                raise ValueError(f"MonoRecSequence.push: key frame {n} comes with {sorted(maps)}, the sequence's key frames "
                                 f"with {sorted(self._maps)}")
            for k, t in maps.items():
                self._maps[k][slot].copy_(t, non_blocking=True)
        self.n_pushed += 1
        n = self._ready()
        if n >= self.batch_size:
            return self._run(self.batch_size, self.graphed)
        if n > 0 and n == self._remaining():
            return self._run(n, False)                             # the short last batch before key_end / of `keys`
        return []

    def flush(self):
        """Runs the key frames that are ready but fewer than `batch_size`, eagerly (end of the sequence)."""
        n = self._ready()
        return self._run(n, False) if n > 0 else []

    def _key_inputs(self, H, W, stereo, mvobj_mask, target):
        """The key-frame inputs given to this push, shaped as one row of their rings."""
        maps = {}
        if self.stereo and stereo is not None:
            image, pose, intrinsics = stereo
            C = self.channels
            if tuple(image.shape) != (C, H, W) or tuple(pose.shape) != (4, 4) or tuple(intrinsics.shape) != (4, 4):
                raise ValueError(f"MonoRecSequence.push: stereo image [{C},{H},{W}], pose [4,4], intrinsics [4,4] expected, "
                                 f"got {tuple(image.shape)}, {tuple(pose.shape)}, {tuple(intrinsics.shape)}")
            maps.update(stereoframe=image, stereoframe_pose=pose, stereoframe_intrinsics=intrinsics)
        for key, t in (("mvobj_mask", mvobj_mask), ("target", target)):
            if t is not None:
                if t.numel() != H * W or tuple(t.shape[-2:]) != (H, W):
                    raise ValueError(f"MonoRecSequence.push: {key} [1,H,W] of the image's size {(H, W)} expected, got "
                                     f"{tuple(t.shape)}")
                maps[key] = t.reshape(1, H, W)
        if (self.stereo and stereo is None) or (self.mvobj_masks and mvobj_mask is None):
            if self.runs(self.n_pushed):
                raise ValueError(f"MonoRecSequence.push: key frame {self.n_pushed} needs "
                                 f"{'stereo=(image, pose, intrinsics)' if self.stereo and stereo is None else 'mvobj_mask'}")
        return maps

    def _store(self, n):
        """The ring slot of frame n."""
        if not self._free:
            raise RuntimeError("MonoRecSequence: the frame ring is full (a bookkeeping error)")
        self._slot[n] = (self._free.pop(), max(n - u for u in self._uses if _listed(self._run_keys, n - u)))
        return self._slot[n][0]

    def _ready(self):
        """Key frames not yet run (before key_end) whose neighbours have all been pushed."""
        return bisect.bisect_left(self._run_keys, self.n_pushed - self._hi) - self._next

    def _remaining(self):
        """Key frames left to run."""
        return len(self._run_keys) - self._next

    def _assemble(self, idx, out=None):
        """The batch dict, with the reference's keys and list order, gathered from the rings at slots `idx` [1+F, n];
        written into `out`'s tensors when given (the graph's static inputs).  A source frame at offset 0 is the key frame's
        own tensor (its image, pose and intrinsics): gathered once, read twice (GraphedMonoRec keeps that aliasing)."""
        frames, poses, intrinsics = self._rings
        data = {}
        for key, ring in (("keyframe", frames), ("keyframe_pose", poses), ("keyframe_intrinsics", intrinsics)):
            data[key] = torch.index_select(ring, 0, idx[0], out=None if out is None else out[key])
        for key, own, ring in (("frames", "keyframe", frames), ("poses", "keyframe_pose", poses),
                               ("intrinsics", "keyframe_intrinsics", intrinsics)):
            data[key] = [data[own] if u == 0 else
                         torch.index_select(ring, 0, idx[1 + f], out=None if out is None else out[key][f])
                         for f, u in enumerate(self.offsets)]
        for key, ring in self._maps.items():
            data[key] = torch.index_select(ring, 0, idx[0], out=None if out is None else out[key])
        return data

    def _run(self, n, graphed):
        index = self._run_keys[self._next:self._next + n]
        idx = torch.tensor([[self._slot[k + u][0] for k in index] for u in self._uses], dtype=torch.int64)
        # a pinned copy does not synchronise; the host allocator keeps the block until the copy is done
        idx = idx.pin_memory().to(self.device, non_blocking=True) if self.device.type == "cuda" else idx
        if not graphed:
            out = self._forward(self._assemble(idx))
        elif self._graph is None:
            self._graph = GraphedMonoRec(self._forward, self._assemble(idx))
            out = self._graph.replay()
        else:
            self._assemble(idx, out=self._graph.static_in)
            out = self._graph.replay()
        self._next += n
        # frames no later key frame uses go back to the free slots (their next writes follow this batch's gathers)
        for f in [f for f, (_, last) in self._slot.items() if last <= index[-1]]:
            self._free.append(self._slot.pop(f)[0])
        return [(i, _row(out, j)) for j, i in enumerate(index)]


def _with_residual_image(model, data):
    """`model` on one batch dict, and the residual image (layers.ResidualImage) of its `result` against the frames its
    cost volume used, as `residual_image`."""
    from .layers import residual_image
    from .losses import _collect
    out = model(data)
    frames, poses, intrinsics = _collect(out, getattr(model, "use_mono", True), getattr(model, "use_stereo", False))
    out["residual_image"] = residual_image(out["keyframe"], out["keyframe_pose"], out["keyframe_intrinsics"], out["result"],
                                           frames, poses, intrinsics)
    return out


_ROW_KEYS = ("result", "cv_mask", "cost_volume", "keyframe", "keyframe_pose", "keyframe_intrinsics", "stereoframe",
             "stereoframe_pose", "stereoframe_intrinsics", "mvobj_mask", "target", "residual_image")


def _row(out, j):
    v = {k: out[k][j:j + 1] for k in _ROW_KEYS if k in out}
    if "predicted_inverse_depths" in out:
        v["predicted_inverse_depths"] = [p[j:j + 1] for p in out["predicted_inverse_depths"]]
    if "models" in out:          # several models over one batch (models_eval): one output dict per model
        v["models"] = [_row(o, j) for o in out["models"]]
    return v
