"""evaluate.py's list of models (`config["models"]`, evaluate.py:27-64) over one frame stream.

The reference evaluates each model of the list with a full `Evaluater.eval` over the same loader: every frame is read, copied
to the device and put through the cost volume and the trunk once per model.  `MultiModelEvaluater` runs all models over one
`MonoRecSequence`: one frame ring, one copy of each frame, and per batch of key frames one forward of every model in which

  * models whose cost-volume configuration is equal (`cost_volume_key`) share one cost-volume stage,
  * models whose trunk weights and BatchNorm buffers are equal (`same_trunk`) share one trunk stage,
  * every model runs its own Mask / Depth stacks and heads on those shared tensors (stage C never writes them),

and each model's results are folded by its own `SequenceEvaluater` (the device-side metric rows and `mr_eval_accumulate`).
Each model's log is bit for bit that of a `SequenceEvaluater` over `MonoRecSequence(model, batch_size=seq_batch)`: the
shared stages compute what each model's own stages would, on the same inputs.
"""
import pathlib

import numpy as np
import torch

from .evaluation import LANE, SequenceEvaluater, check_slice, emitted_in_slice, fold_rows, log_dict
from .model import rgb_keyframe
from .sequence import MonoRecSequence

__all__ = ["MultiModelEvaluater", "cost_volume_key", "same_trunk", "share_groups"]

_OUT_KEYS = ("result", "cv_mask", "cost_volume", "predicted_inverse_depths")


def cost_volume_key(model):
    """What a MonoRecModel's cost-volume stage depends on besides the batch: models with equal keys produce the same
    `cost_volume`, `single_frame_cvs`, depth-range entries and MaskModule NHWC copy.  Beyond the frame selection, the matching
    mode, the depth planes, the storage type, `no_cv` and whether the NHWC copy is written, the key holds the cost-volume
    module's centring, view-weight alpha and channel weights, which change the volume too."""
    cv = model.cv_module
    return (bool(model.use_mono), bool(model.use_stereo), bool(cv.use_mono), bool(cv.use_stereo), int(cv.matching),
            bool(cv.not_center_cv), float(cv.alpha), cv.channel_weights, int(model.cv_depth_steps),
            tuple(float(v) for v in model.inv_depth_min_max), cv.volume_dtype, bool(model.no_cv),
            model._writes_sfcv_nhwc())


def same_trunk(a, b):
    """Whether two MonoRecModels' ResNet-18 trunks hold equal parameters and BatchNorm buffers (torch.equal, one by one)."""
    ta, tb = a._feature_extractor._source_tensors(), b._feature_extractor._source_tensors()
    return len(ta) == len(tb) and all(x.shape == y.shape and x.dtype == y.dtype and x.device == y.device and torch.equal(x, y)
                                      for x, y in zip(ta, tb))


def share_groups(models):
    """(cost-volume groups, trunk groups) of `models`: lists of lists of indices into `models`, each group in list order and
    the groups in the order of their first member.  The first member of a group runs the shared stage."""
    def group(same):
        groups = []
        for i, m in enumerate(models):
            for g in groups:
                if same(models[g[0]], m):
                    g.append(i)
                    break
            else:
                groups.append([i])
        return groups
    return group(lambda a, b: cost_volume_key(a) == cost_volume_key(b)), group(same_trunk)


class _SharedForward:
    """The forward of several MonoRecModels on one batch dict, with the stages shared as `groups` say.  Returns the batch's
    `target` / `mvobj_mask` and under `models` one dict per model of its outputs (`_OUT_KEYS`).  MonoRecSequence runs it as
    it runs one model, captured in one CUDA graph per batch shape."""

    def __init__(self, models, cv_groups, trunk_groups):
        self.models, self.cv_groups, self.trunk_groups = models, cv_groups, trunk_groups

    def __call__(self, batch):
        batch = dict(batch)
        rgb_keyframe(batch)                   # a grayscale keyframe's three-channel copy: one for every stage and model
        cv, feats = {}, {}
        for g in self.cv_groups:
            d = self.models[g[0]]._stage_cost_volume(dict(batch))
            cv.update((i, d) for i in g)
        for g in self.trunk_groups:
            f = self.models[g[0]]._stage_trunk(dict(batch))["image_features"]
            feats.update((i, f) for i in g)
        outs = []
        for i, model in enumerate(self.models):
            d = dict(cv[i])                   # a shallow copy: the heads pop and replace entries of their own dict only
            d["image_features"] = feats[i]
            d = model._stage_heads(d)
            outs.append({k: d[k] for k in _OUT_KEYS if k in d})
        out = {k: batch[k] for k in ("target", "mvobj_mask") if k in batch}
        out["models"] = outs
        return out


def public_dict(obj):
    """evaluate.py's dict of a model or a dataset (:36-52): its attributes without the `_`-prefixed ones, ndarrays as lists
    and paths as strings.  A torch.dtype (MonoRecModel.volume_dtype, which the reference's model does not have) becomes its
    name, so that the dict can be written as JSON."""
    d = {}
    for k, v in (obj if isinstance(obj, dict) else vars(obj)).items():
        if k.startswith("_"):
            continue
        if type(v) == np.ndarray:         # noqa: E721  (evaluate.py's test: subclasses stay as they are)
            v = list(v)
        elif isinstance(v, pathlib.PurePath):
            v = str(v)
        elif isinstance(v, torch.dtype):
            v = str(v)
        d[k] = v
    return d


class MultiModelEvaluater:
    """`Evaluater.eval` of every model of `models` (MonoRecModels in eval mode on one device) over one frame stream.

    `metrics`, `batch_size`, `roi`, `max_distance`, `median_scaling` are SequenceEvaluater's (the same for every model, as
    in evaluate.py); `frame_count`, `dilation`, `seq_batch` (the key frames per forward), `keys`, `stereo`, `mvobj_masks`,
    `device` and `use_color` (False: grayscale [1,H,W] frames) build the MonoRecSequence the models run over.  A
    `use_stereo` model needs `stereo=True`, a `pretrain_mode == 3` model `mvobj_masks=True`; the stereo frames and masks are copied to the device once, and only if
    a model (or an `*_onlydynamic` metric, for the masks) reads them.

    `push(image, pose, intrinsics, target, mvobj_mask=None, stereo=None)`, `skip()` and `flush()` are SequenceEvaluater's
    and return what the sequence emits: per key frame (index, outputs), where `outputs["models"][m]` holds model m's
    `result`, `cv_mask`, `cost_volume`, `predicted_inverse_depths` and `outputs` the key frame's `target` (and
    `mvobj_mask`).  `next_sequence(keys=None, first_frame=0, key_end=None)` runs the rest of the current sequence and
    continues on a new one with the same settings and key-frame list `keys`; the totals and open evaluater batches carry
    over.  Once the sequence has captured its graph (its first full batch), `push` and `flush` never synchronise with the
    host.

    `layout` (a sequence.FrameLayout: `kitti_layout` with `offset_d` / `max_length`, `tum_mono_vo_layout`,
    `robotcar_layout`) replaces frame_count, dilation and keys, for the first sequence; `next_sequence(layout=...)` gives
    the next one's.

    The sharing is decided once, here (`share_groups`; `cv_groups` / `trunk_groups` hold it), and like GraphedMonoRec a
    sequence's captured graph keeps running on the weights it was captured with.  Build a new evaluater after changing a
    model's weights or options.  `groups` gives that sharing instead, decided on models equal to these (the lanes of
    lanes.MultiDeviceModelsEvaluater, which checks it).  `graphed=False` runs the sequences without CUDA-graph replay.

    `logs()`: one log per model, in list order.  `results(dataset_dict)`: evaluate.py's results.json list.

    One slice of a split run (one rank under `torchrun`, or one lane): `group` and `shard` as on SequenceEvaluater, a
    process group (or evaluation.LANE) and this rank's slices, `dist.shard_sequences(..., eval_batch=batch_size)`.  The
    evaluater then opens no sequence itself: `next_sequence(keys, first_frame=slice.frames[0], key_end=slice.run[1])`
    starts each slice in turn (and refuses a sequence that does not run the slice's key frames), the slice's frames
    slice.frames[0] ... slice.frames[1] - 1 are pushed (or skipped), and only the key frames of the slice's `emit` range
    are evaluated.  `logs()` is then a collective: every rank calls it and gets every model's log of the whole run, the
    one-process logs bit for bit.  A lane's logs are folded by its driver.
    """

    def __init__(self, models, metrics, batch_size, roi=None, max_distance=None, median_scaling=False, frame_count=2,
                 dilation=1, seq_batch=8, keys=None, stereo=False, mvobj_masks=False, device=None, use_color=True,
                 graphed=True, group=None, shard=None, groups=None, layout=None):
        self.models = list(models)
        if not self.models:
            raise ValueError("MultiModelEvaluater: models is empty")
        if shard is not None and (keys is not None or layout is not None):
            raise ValueError("MultiModelEvaluater: with a shard, each slice's key list or layout goes to "
                             "next_sequence(keys, ...) / next_sequence(layout=...)")
        self.device = torch.device(device) if device is not None else next(self.models[0].parameters()).device
        for m in self.models:
            if next(m.parameters()).device != self.device:
                raise ValueError(f"MultiModelEvaluater: a model is on {next(m.parameters()).device}, not {self.device}")
            if m.use_stereo and not stereo:
                raise NotImplementedError("MultiModelEvaluater: a use_stereo model needs stereo=True and "
                                          "push(..., stereo=(image, pose, intrinsics))")
            if int(m.pretrain_mode) == 3 and not mvobj_masks:
                raise NotImplementedError("MultiModelEvaluater: a pretrain_mode 3 model needs mvobj_masks=True and "
                                          "push(..., mvobj_mask=...)")
        self.evaluaters = [SequenceEvaluater(None, metrics, batch_size, roi=roi, max_distance=max_distance,
                                             median_scaling=median_scaling, group=group, shard=shard) for _ in self.models]
        self.names = self.evaluaters[0].names
        self.stereo = bool(stereo)
        self.group, self._slices, self._slice = group, None if shard is None else list(shard), 0
        self.cv_groups, self.trunk_groups = share_groups(self.models) if groups is None else groups
        self._forward = _SharedForward(self.models, self.cv_groups, self.trunk_groups)
        self._seq_args = dict(frame_count=frame_count, dilation=dilation, batch_size=seq_batch, device=self.device,
                              use_color=use_color, graphed=graphed,
                              stereo=self.stereo and any(m.use_stereo for m in self.models),
                              mvobj_masks=bool(mvobj_masks) and any(int(m.pretrain_mode) == 3 for m in self.models))
        self.seq = None if shard is not None else MonoRecSequence(self._forward, keys=keys, layout=layout,
                                                                  **self._seq_args)

    def push(self, image, pose, intrinsics, target, mvobj_mask=None, stereo=None):
        if self.seq is None:
            raise ValueError("MultiModelEvaluater.push: no sequence open (with a shard, next_sequence starts each slice)")
        ev = self.evaluaters[0]
        ev._check_frame(image, target, mvobj_mask)
        if stereo is not None and not self.stereo:
            raise ValueError("MultiModelEvaluater.push: stereo frames need MultiModelEvaluater(stereo=True)")
        keep_mask = ev._needs_mvobj or self.seq.mvobj_masks
        emitted = self.seq.push(image, pose, intrinsics, stereo=stereo if self.seq.stereo else None,
                                mvobj_mask=mvobj_mask if keep_mask else None, target=target)
        self._consume(emitted)
        return emitted

    def skip(self):
        """Passes a frame that no key frame of the sequence needs, without reading it (`MonoRecSequence.skip`)."""
        self.seq.skip()

    def flush(self):
        emitted = self.seq.flush() if self.seq is not None else []
        self._consume(emitted)
        for ev in self.evaluaters:
            ev.flush()
        return emitted

    def next_sequence(self, keys=None, first_frame=0, key_end=None, layout=None):
        """Runs the key frames the current sequence still holds, then continues on a new one with key-frame list `keys`
        (or frame layout `layout`), starting at frame `first_frame` and running the key frames before `key_end`
        (MonoRecSequence's; the defaults run the whole sequence).  Returns what the current sequence's flush returns."""
        emitted = self.seq.flush() if self.seq is not None else []
        self._consume(emitted)
        if self._slices is not None and self.seq is not None:
            self._slice += 1
        self.seq = None                   # (the old graph's memory is released before the new sequence captures one)
        seq = MonoRecSequence(self._forward, keys=keys, first_frame=first_frame, key_end=key_end, layout=layout,
                              **self._seq_args)
        check_slice(self._slices, self._slice, seq)
        self.seq = seq
        return emitted

    def _consume(self, emitted):
        emitted = emitted_in_slice(self._slices, self._slice, emitted)
        if not emitted:
            return
        # cut into evaluater batches as SequenceEvaluater._consume does, once per model, on the shared targets (and masks)
        target = torch.cat([o["target"] for _, o in emitted])
        mask = torch.cat([o["mvobj_mask"] for _, o in emitted]) if self.evaluaters[0]._needs_mvobj else None
        for m, ev in enumerate(self.evaluaters):
            ev.add(torch.cat([o["models"][m]["result"] for _, o in emitted]), target, mask)

    def logs(self):
        """Evaluater.eval's dict of every model, in list order (one device-to-host read each).  With a process group, a
        collective that gathers every rank's rows (SequenceEvaluater.log)."""
        if self.group is None or self.group is LANE:
            return [ev.log() for ev in self.evaluaters]
        from .dist import all_gather_rows
        m = len(self.names)
        return [log_dict(fold_rows(all_gather_rows(ev.tagged_rows(self.device), self.group), m), m)
                for ev in self.evaluaters]

    def results(self, dataset_dict):
        """evaluate.py's results.json list: per model {"model": its public attributes, "dataset": those of
        `dataset_dict` (the dataset's `__dict__`), "result": its log with `metrics_info`, the metric names}.  With a process
        group, a collective as `logs()` is."""
        return results_list(self.models, self.names, self.logs(), dataset_dict)


def results_list(models, names, logs, dataset_dict):
    """evaluate.py's results.json list of `models` with their `logs` over the metrics `names`."""
    dataset = public_dict(dataset_dict)
    out = []
    for model, log in zip(models, logs):
        log["metrics_info"] = list(names)
        out.append({"model": public_dict(model), "dataset": dict(dataset), "result": log})
    return out
