"""One process driving several devices: the sequence evaluation and the point-cloud export over N lanes from one thread.

The reference's evaluate.py and create_pointcloud.py are single-process programs (their configs ask for several GPUs,
which `DataParallel` would use).  `dist.shard_sequences` splits both loops over a world of N; under `torchrun` each rank is
a process.  Here lane r of N runs rank r's slices on `devices[r]` instead, all from the calling thread: every CUDA call
returns once it is queued, the evaluation and the export make no host synchronisation per batch, so one thread keeps every
lane's device busy.  Devices may repeat (`devices=[0, 0, 0]`: three lanes taking turns on one GPU).

`LanePlan` is the host side: each lane's slices, the frames each lane needs (in its order) and one read order of every
needed (sequence, frame) across lanes.  `MultiDeviceEvaluater` and `MultiDevicePointCloud` run the unchanged
`SequenceEvaluater` / `SequencePointCloud` on each lane and merge the results: the same row sort and fold as the
`torchrun` path, and the vertices in lane order, which is key-frame order.  Both give the one-process log and PLY bit for
bit (the two alignment rules of `shard_sequences`).  `MultiDeviceModelsEvaluater` runs evaluate.py's list of models the
same way, with a `MultiModelEvaluater` on each lane.

    runner = MultiDeviceEvaluater(model, [0, 1, 2, 3], lengths, metrics, batch_size=2, ...)
    for s, n in runner.order:              # the (sequence, frame) to read next
        image, pose, K, target = read(s, n)
        runner.push(s, n, image, pose, K, target)
    runner.flush()
    log = runner.log()
"""
import contextlib
import copy

import torch

from .dist import shard_sequences
from .evaluation import LANE, SequenceEvaluater, fold_rows, log_dict
from .models_eval import MultiModelEvaluater, results_list, share_groups
from .pointcloud import PLYSaver, SequencePointCloud, write_ply
from .sequence import MonoRecSequence, needs_frame, neighbour_offsets


class LanePlan:
    """Which frames go to which lane, and the order to read them, for `lanes` lanes (dist.shard_sequences' world).

    `slices[r]`: lane r's SequenceSlice list, `shard_sequences(..., rank=r, world=lanes)` with `eval_batch` or
    `buffer_length` and `keys` as given.  `frames[r]`: the (slice number, sequence, frame) lane r's sequences copy, in
    push order: the frames of each slice that `MonoRecSequence.needs` accepts (the others are passed with `skip`).
    `order`: every (sequence, frame) some lane needs, once.  Lanes take turns, each reading up to `batch_size` frames it
    needs that no lane has read yet, so every lane gets about one model batch per turn; a frame a later lane has already
    read (a boundary frame two lanes run) is held until this lane reaches it.

    `layout`: one sequence.FrameLayout per sequence, in place of frame_count, dilation and `keys` (shard_sequences')."""

    def __init__(self, lengths, frame_count, dilation, batch_size, lanes, eval_batch=None, buffer_length=None, keys=None,
                 layout=None):
        if lanes < 1:
            raise ValueError(f"LanePlan: lanes ({lanes}) must be >= 1")
        self.lanes, self.keys, self.layout = int(lanes), keys, layout
        self.slices = [shard_sequences(lengths, frame_count, dilation, batch_size, r, lanes, eval_batch=eval_batch,
                                       buffer_length=buffer_length, keys=keys, layout=layout) for r in range(lanes)]
        offsets = neighbour_offsets(frame_count, dilation)
        self.frames = []
        for sl in self.slices:
            mine = []
            for k, s in enumerate(sl):
                if layout is not None:
                    listed, offs = layout[s.sequence].keys, layout[s.sequence].offsets
                else:
                    listed = range(*s.run) if keys is None or keys[s.sequence] is None else keys[s.sequence]
                    offs = offsets
                run = [int(x) for x in listed if s.run[0] <= int(x) < s.run[1]]
                mine += [(k, s.sequence, n) for n in range(*s.frames) if needs_frame(run, offs, n)]
            self.frames.append(mine)
        self.users = {}                    # (sequence, frame) -> the lanes that need it
        for r, mine in enumerate(self.frames):
            for _, s, n in mine:
                self.users.setdefault((s, n), []).append(r)
        self.order, read, at = [], set(), [0] * self.lanes
        while any(a < len(f) for a, f in zip(at, self.frames)):
            for r, mine in enumerate(self.frames):
                taken = 0
                while at[r] < len(mine) and taken < batch_size:
                    f = mine[at[r]][1:]
                    at[r] += 1
                    if f not in read:
                        read.add(f)
                        self.order.append(f)
                        taken += 1

    def sequence_kw(self, sequence):
        """MonoRecSequence's key-frame argument for sequence `sequence`: its `keys` list or its `layout`."""
        if self.layout is not None:
            return dict(layout=self.layout[sequence])
        return dict(keys=None if self.keys is None else self.keys[sequence])


class _Lanes:
    """Feeds the lanes of a LanePlan: `push(sequence, frame, ...)` in `order`, then `flush()`.  Subclasses open a lane's
    runner for a slice (`_open`: an object with `seq`, `push`, `skip`) and close a lane's last one (`_close`)."""

    def __init__(self, plan, devices):
        if len(devices) != plan.lanes:
            raise ValueError(f"{len(devices)} devices for a plan of {plan.lanes} lanes")
        self.plan = plan
        self.devices = [_device(d) for d in devices]
        self.order = plan.order
        self._read = 0                     # frames of `order` pushed so far
        self._held = {}                    # (sequence, frame) -> (args, kwargs, lanes still to get it)
        self._at = [0] * plan.lanes        # next place in plan.frames[r]
        self._runner = [None] * plan.lanes
        self._slice = [None] * plan.lanes

    def _context(self, r):
        dev = self.devices[r]
        return torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()

    def push(self, sequence, frame, *args, **kwargs):
        """Frame `frame` of sequence `sequence`, which must be `order`'s next, with the arguments of the lane runners'
        `push`.  Host tensors are staged in pinned memory once, so the copies to every lane's device are asynchronous."""
        if self._read >= len(self.order) or self.order[self._read] != (sequence, frame):
            expect = self.order[self._read] if self._read < len(self.order) else "no frame"
            raise ValueError(f"push: (sequence, frame) {(sequence, frame)} given, {expect} expected next (`order`)")
        self._read += 1
        if any(d.type == "cuda" for d in self.devices):
            args, kwargs = _pinned(args), {k: _pinned(v) for k, v in kwargs.items()}
        users = self.plan.users[(sequence, frame)]
        self._held[(sequence, frame)] = [args, kwargs, len(users)]
        for r in users:
            self._deliver(r)

    def _deliver(self, r):
        """Pushes to lane r, in its order, every frame it needs next that has been read."""
        mine = self.plan.frames[r]
        while self._at[r] < len(mine) and mine[self._at[r]][1:] in self._held:
            k, s, n = mine[self._at[r]]
            self._at[r] += 1
            held = self._held[(s, n)]
            with self._context(r):
                if self._slice[r] != k:
                    self._runner[r] = self._open(r, self.plan.slices[r][k])
                    self._slice[r] = k
                runner = self._runner[r]
                while runner.seq.n_pushed < n:
                    runner.skip()
                self._push(r, runner, held[0], held[1])
            held[2] -= 1
            if held[2] == 0:
                del self._held[(s, n)]

    def _push(self, r, runner, args, kwargs):
        runner.push(*args, **kwargs)

    def flush(self):
        """Runs what every lane still holds; every frame of `order` must have been pushed."""
        if self._read != len(self.order):
            raise ValueError(f"flush: {self._read} of the {len(self.order)} frames of `order` pushed")
        for r in range(self.plan.lanes):
            if self._runner[r] is not None:
                with self._context(r):
                    self._close(r)


def _device(d):
    d = torch.device("cuda", d) if isinstance(d, int) else torch.device(d)
    return torch.device("cuda", torch.cuda.current_device()) if d.type == "cuda" and d.index is None else d


def _pinned(x):
    if torch.is_tensor(x):
        return x.pin_memory() if x.device.type == "cpu" and not x.is_pinned() else x
    if isinstance(x, (tuple, list)):
        return type(x)(_pinned(v) for v in x)
    return x


def _replicas(model, devices):
    """One model per distinct device: `model` itself on its own device, a copy on every other one (each packs its weights
    once, in its own per-device caches)."""
    home = next(model.parameters()).device
    out = {}
    for d in devices:
        if d not in out:
            out[d] = model if d == home else copy.deepcopy(model).to(d)
    return out


class MultiDeviceEvaluater(_Lanes):
    """`SequenceEvaluater` over the concatenated sequences of `lengths` frames, split over one lane per entry of `devices`.

    Lane r runs `shard_sequences(lengths, frame_count, dilation, seq_batch, r, len(devices), eval_batch=batch_size,
    keys=keys)` on devices[r]: a `MonoRecSequence(first_frame=, key_end=, keys=)` per slice, with `graphed` CUDA-graph
    replay (each lane captures its own graph), under a `SequenceEvaluater(group=LANE, shard=)`.  `metrics`, `batch_size`,
    `roi`, `max_distance` and `median_scaling` are the evaluater's; `stereo` / `mvobj_masks` / `use_color` the sequences'.
    `layout`: one sequence.FrameLayout per sequence, in place of frame_count, dilation and keys.

    `push(sequence, frame, image, pose, intrinsics, target, mvobj_mask=None, stereo=None)` in `order`, then `flush()`.
    `log()` brings every lane's closed evaluater-batch rows to devices[0], sorts them by global batch index and runs the
    one-process fold (`evaluation.fold_rows`, as the `torchrun` path): `Evaluater.eval`'s dict, equal to one process's."""

    def __init__(self, model, devices, lengths, metrics, batch_size, frame_count=2, dilation=1, seq_batch=8, keys=None,
                 roi=None, max_distance=None, median_scaling=False, graphed=True, stereo=False, mvobj_masks=False,
                 use_color=True, layout=None):
        plan = LanePlan(lengths, frame_count, dilation, seq_batch, len(devices), eval_batch=batch_size, keys=keys,
                        layout=layout)
        super().__init__(plan, devices)
        self._models = _replicas(model, self.devices)
        self._seq_kw = dict(frame_count=frame_count, dilation=dilation, batch_size=seq_batch, graphed=graphed,
                            stereo=stereo, mvobj_masks=mvobj_masks, use_color=use_color)
        self.evaluaters = [SequenceEvaluater(None, metrics, batch_size, roi=roi, max_distance=max_distance,
                                             median_scaling=median_scaling, group=LANE, shard=sl) if sl else None
                           for sl in plan.slices]

    def _open(self, r, sl):
        ev = self.evaluaters[r]
        ev.next_sequence(MonoRecSequence(self._models[self.devices[r]], device=self.devices[r], first_frame=sl.frames[0],
                                         key_end=sl.run[1], **self.plan.sequence_kw(sl.sequence), **self._seq_kw))
        return ev

    def _close(self, r):
        self.evaluaters[r].flush()

    def log(self):
        """The one-process log dict (one device-to-host read; call after `flush`)."""
        dev = self.devices[0]
        lanes = [ev for ev in self.evaluaters if ev is not None]
        m = len(lanes[0].names)
        with self._context(0):
            rows = torch.cat([ev.tagged_rows(dev) for ev in lanes])
            return log_dict(fold_rows(rows, m), m)


class MultiDeviceModelsEvaluater(_Lanes):
    """evaluate.py's list of models over the concatenated sequences of `lengths` frames, split over one lane per entry of
    `devices`: `MultiDeviceEvaluater` with `models` (MonoRecModels in eval mode on one device) in place of `model`.

    Lane r runs the slices of MultiDeviceEvaluater's lane r with a `MultiModelEvaluater(group=LANE, shard=)` on devices[r],
    over replicas of every model on that device, so each lane reads and copies every frame it needs once and shares the
    cost-volume and trunk stages as one device does.  The sharing (`cv_groups`, `trunk_groups`) is decided once, on
    `models`; every lane runs with it, and each device's replicas are checked to give the same groups.  Every lane holds
    every model and one captured graph of their shared forward.

    `order`, `push(sequence, frame, image, pose, intrinsics, target, mvobj_mask=None, stereo=None)` and `flush()` are
    MultiDeviceEvaluater's (each lane skips the frames of its slices that it does not need), and so is `layout`.  `logs()`: one log per model, in list order, each the one-process log bit for bit (every
    lane's rows of that model folded on devices[0]); `results(dataset_dict)`: evaluate.py's results.json list."""

    def __init__(self, models, devices, lengths, metrics, batch_size, frame_count=2, dilation=1, seq_batch=8, keys=None,
                 roi=None, max_distance=None, median_scaling=False, graphed=True, stereo=False, mvobj_masks=False,
                 use_color=True, layout=None):
        self.models = list(models)
        if not self.models:
            raise ValueError("MultiDeviceModelsEvaluater: models is empty")
        home = next(self.models[0].parameters()).device
        for m in self.models:
            if next(m.parameters()).device != home:
                raise ValueError(f"MultiDeviceModelsEvaluater: a model is on {next(m.parameters()).device}, not {home}")
        plan = LanePlan(lengths, frame_count, dilation, seq_batch, len(devices), eval_batch=batch_size, keys=keys,
                        layout=layout)
        super().__init__(plan, devices)
        self.cv_groups, self.trunk_groups = share_groups(self.models)
        replicas = [_replicas(m, self.devices) for m in self.models]
        self._models = {}
        for d in replicas[0]:
            self._models[d] = [rep[d] for rep in replicas]
            groups = share_groups(self._models[d])
            if groups != (self.cv_groups, self.trunk_groups):
                raise RuntimeError(f"MultiDeviceModelsEvaluater: the replicas on {d} share stages as {groups}, the models "
                                   f"as {(self.cv_groups, self.trunk_groups)}")
        kw = dict(roi=roi, max_distance=max_distance, median_scaling=median_scaling, frame_count=frame_count,
                  dilation=dilation, seq_batch=seq_batch, stereo=stereo, mvobj_masks=mvobj_masks, use_color=use_color,
                  graphed=graphed, group=LANE, groups=(self.cv_groups, self.trunk_groups))
        self.evaluaters = [MultiModelEvaluater(self._models[d], metrics, batch_size, device=d, shard=sl, **kw) if sl
                           else None for d, sl in zip(self.devices, plan.slices)]
        self.names = next(ev for ev in self.evaluaters if ev is not None).names

    def _open(self, r, sl):
        ev = self.evaluaters[r]
        ev.next_sequence(first_frame=sl.frames[0], key_end=sl.run[1], **self.plan.sequence_kw(sl.sequence))
        return ev

    def _close(self, r):
        self.evaluaters[r].flush()

    def logs(self):
        """The one-process log of every model, in list order (one device-to-host read each; call after `flush`)."""
        dev = self.devices[0]
        lanes = [ev for ev in self.evaluaters if ev is not None]
        m = len(self.names)
        out = []
        with self._context(0):
            for k in range(len(self.models)):
                rows = torch.cat([ev.evaluaters[k].tagged_rows(dev) for ev in lanes])
                out.append(log_dict(fold_rows(rows, m), m))
        return out

    def results(self, dataset_dict):
        """evaluate.py's results.json list: per model {"model", "dataset", "result"}, as MultiModelEvaluater.results."""
        return results_list(self.models, self.names, self.logs(), dataset_dict)


class MultiDevicePointCloud(_Lanes):
    """create_pointcloud.py's export (`SequencePointCloud`) over the sequences of `lengths` frames, split over one lane per
    entry of `devices`.

    Lane r runs `shard_sequences(..., r, len(devices), buffer_length=buffer_length, keys=keys)` on devices[r]: per slice a
    `MonoRecSequence` (with `stereo`, `mvobj_masks`, `use_color`) and a `SequencePointCloud(emit=slice.emit)` into the
    lane's own `PLYSaver(height, width, min_d, max_d, roi=roi, dropout=dropout)`.  `layout`: one sequence.FrameLayout per
    sequence, in place of frame_count, dilation and keys.

    `push(sequence, frame, image, pose, intrinsics, rand=None, stereo=None, mvobj_mask=None)` in `order`, then `flush()`;
    `rand` are the frame's dropout numbers, keyed by sequence index as in `SequencePointCloud`.  `vertices` (on
    devices[0]) and `save(file)` give every lane's vertices in lane order, which is the one-process key-frame order."""

    def __init__(self, model, devices, lengths, height, width, frame_count=2, dilation=1, seq_batch=8, keys=None,
                 buffer_length=5, min_hits=1, mask_fill=32, min_d=3, max_d=400, roi=None, dropout=0, graphed=True,
                 stereo=False, mvobj_masks=False, use_color=True, layout=None):
        plan = LanePlan(lengths, frame_count, dilation, seq_batch, len(devices), buffer_length=buffer_length, keys=keys,
                        layout=layout)
        super().__init__(plan, devices)
        self._models = _replicas(model, self.devices)
        self._seq_kw = dict(frame_count=frame_count, dilation=dilation, batch_size=seq_batch, graphed=graphed,
                            stereo=stereo, mvobj_masks=mvobj_masks, use_color=use_color)
        self._pc_kw = dict(buffer_length=buffer_length, min_hits=min_hits, mask_fill=mask_fill)
        self.savers = [PLYSaver(height, width, min_d=min_d, max_d=max_d, roi=roi, dropout=dropout)
                       for _ in self.devices]

    def _open(self, r, sl):
        if self._runner[r] is not None:
            self._runner[r].flush()
        seq = MonoRecSequence(self._models[self.devices[r]], device=self.devices[r], first_frame=sl.frames[0],
                              key_end=sl.run[1], **self.plan.sequence_kw(sl.sequence), **self._seq_kw)
        return SequencePointCloud(seq, self.savers[r], emit=sl.emit, **self._pc_kw)

    def _push(self, r, runner, args, kwargs):
        rand = kwargs.get("rand")
        if rand is not None:          # a key frame's dropout numbers go to its lane's device without a synchronising copy
            kwargs = dict(kwargs, rand=rand.to(self.devices[r], torch.float32, non_blocking=True)
                          if runner.seq.runs(runner.seq.n_pushed) else None)
        runner.push(*args, **kwargs)

    def _close(self, r):
        self._runner[r].flush()

    @property
    def vertices(self):
        """Every lane's vertices [N, 6] in lane order, on devices[0] (a host synchronisation per lane)."""
        dev = self.devices[0]
        return torch.cat([s.vertices.to(dev) for s in self.savers])

    def save(self, file):
        """The binary PLY of `vertices`, with the reference's header (`PLYSaver.save`)."""
        write_ply(file, torch.cat([s.vertices.cpu() for s in self.savers]))
