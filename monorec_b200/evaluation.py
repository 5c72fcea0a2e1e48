"""evaluate.py's evaluation (evaluater/evaluater.py:78-119) over a MonoRecSequence, without host synchronisation.

The reference's loop takes the loader's batches of key-frame dicts (batch size 2 in configs/evaluate/eval_monorec.json), runs
an eager forward per batch and turns every metric of every batch into a Python float.  `SequenceEvaluater` takes the frames
of a sequence and their targets one at a time instead: the model runs through the `MonoRecSequence` (rings, CUDA-graph
replay), every batch of key frames it emits is cut into the evaluater's batches, and per emitted batch one grouped metric
pass (`mr_sparse_metrics_grouped` / `mr_dense_metrics_grouped`) and one `mr_eval_accumulate` update the evaluater's float64
totals on the device.  `log()` reads them back once and returns `Evaluater.eval`'s dict.
"""
import numpy as np
import torch

from . import metrics as M

_SPARSE_VARIANTS = (("sparse", dict(pred_all_valid=True, use_cvmask=False)),
                    ("sparse_onlyvalid", dict(pred_all_valid=False, use_cvmask=False)),
                    ("sparse_onlydynamic", dict(pred_all_valid=True, use_cvmask=True)))

# reference metric name (model/metric.py) -> (pass, column of the pass's output): pass ("sparse", pred_all_valid,
# use_cvmask) is mr_sparse_metrics' seven columns, ("dense",) mr_dense_metrics' twelve
METRICS = {}
for _suffix, _kw in _SPARSE_VARIANTS:
    for _i, _n in enumerate(M.NAMES):
        METRICS[f"{_n}_{_suffix}_metric"] = (("sparse", _kw["pred_all_valid"], _kw["use_cvmask"]), _i)
for _i, _n in enumerate(M.DENSE_NAMES):
    METRICS[f"{_n}_metric"] = (("dense",), _i)
_BY_FUNCTION = {getattr(M, _n): _n for _n in METRICS}


def metric_name(metric):
    """The reference name of `metric`: one of METRICS, or the monorec_b200.metrics function of that name."""
    if isinstance(metric, str):
        if metric not in METRICS:
            raise ValueError(f"unknown metric {metric!r}: expected one of the {len(METRICS)} names of model/metric.py")
        return metric
    try:
        return _BY_FUNCTION[metric]
    except (KeyError, TypeError):
        raise ValueError(f"unknown metric {metric!r}: expected a name of model/metric.py or the monorec_b200.metrics "
                         "function of that name") from None


class SequenceEvaluater:
    """`Evaluater.eval` over the key frames of `seq` (a MonoRecSequence), in evaluater batches of `batch_size` key frames.

    `metrics`: reference metric names or this package's functions of those names (the 21 sparse and 12 dense / completeness
    metrics of model/metric.py); `roi` [r0, r1, c0, c1], `max_distance` and `median_scaling` are the evaluater's settings.

    `push(image, pose, intrinsics, target, mvobj_mask=None)` forwards the frame to `seq`; `target` [1,H,W] is the frame's
    inverse-depth ground truth (host or device), copied once into a ring next to the sequence's.  Every batch of key frames
    the sequence emits is cut into evaluater batches in key-frame order, as the loader's DataLoader batches them with
    shuffle=False; a partial batch waits for the next emitted one.  `next_sequence(seq)` runs the rest of the current
    sequence and continues on the next one with the same totals and the same open batch (the loader's batches run across
    the boundary of concatenated sequences); `flush()` runs the rest of the sequence and closes the last partial batch.
    `push`, `flush` and `next_sequence` return what the sequence returns, and never synchronise with the host once the
    sequence has captured its graph.  `mvobj_mask` [1,H,W] is needed by the `*_sparse_onlydynamic_metric` names only.

    `add(result, target, mvobj_mask=None)` is the part after the model: the batching and accumulation of results already
    computed ([n,1,H,W] each, key frames in order); `seq` may be None when only `add` is used.

    `log()` makes the one device-to-host read and returns the evaluater's dict: `loss` and `loss_loss` 0.0, `metrics` (total
    over valid batches: NaN for a metric no batch was valid for), `metrics_correct` (the running average over samples) and
    `valid_batches`.  Batches still open are not in it: call `flush()` first.

    Several processes (one per GPU, or several on one GPU) evaluate one run together with `group` (a torch.distributed
    process group) and `shard`, this rank's slices of the sequences (`dist.shard_sequences(..., eval_batch=batch_size)`):
    `seq` and every sequence given to `next_sequence` run `shard`'s slices in order (MonoRecSequence(first_frame=
    slice.frames[0], key_end=slice.run[1]), fed frames slice.frames[0] ... slice.frames[1] - 1), and only the key frames
    of each slice's `emit` range are evaluated.  Each evaluater batch's metric row stays on the device, tagged with the
    batch's index in the whole run, instead of being folded at once.  `log()` is then a collective: every rank of `group`
    calls it, the rows of all ranks are gathered, and the one-process fold runs over them in global batch order on every
    rank, so every rank returns the one-process log (the same device state, bit for bit).
    """

    def __init__(self, seq, metrics, batch_size, roi=None, max_distance=None, median_scaling=False, group=None, shard=None):
        if isinstance(metrics, (str, bytes)) or not hasattr(metrics, "__iter__"):
            raise ValueError(f"metrics must be a list of metric names or functions, got {metrics!r}")
        self.names = [metric_name(m) for m in metrics]
        if not self.names:
            raise ValueError("metrics is empty")
        if isinstance(batch_size, bool) or int(batch_size) != batch_size or batch_size < 1:
            raise ValueError(f"batch_size ({batch_size!r}) must be an integer >= 1")
        if roi is not None:
            if len(roi) != 4 or any(isinstance(v, bool) or int(v) != v for v in roi):
                raise ValueError(f"roi must be four integers [r0, r1, c0, c1], got {roi!r}")
            roi = [int(v) for v in roi]
        if max_distance is not None and not max_distance > 0:
            raise ValueError(f"max_distance ({max_distance!r}) must be None or > 0")
        self.seq, self.batch_size, self.roi = seq, int(batch_size), roi
        self.max_distance, self.median_scaling = max_distance, bool(median_scaling)
        self._specs = [METRICS[n] for n in self.names]
        self._needs_mvobj = any(key[0] == "sparse" and key[2] for key, _ in self._specs)
        self._state = None         # device float64 [3M+1]: total, valid, running average, num_samples
        self._open = None          # (result, target, mvobj_mask) of the key frames of the open evaluater batch
        self._rings = None         # device [R,1,H,W] targets (and moving-object masks) of the sequence's frames
        if (group is None) != (shard is None):
            raise ValueError("SequenceEvaluater: group and shard go together (shard: dist.shard_sequences(...)'s slices)")
        self.group, self._slices, self._slice = group, None if shard is None else list(shard), 0
        if self._slices:
            if self._slices[0].position % self.batch_size:
                raise ValueError(f"SequenceEvaluater: the shard starts at key frame {self._slices[0].position}, inside an "
                                 f"evaluater batch of {self.batch_size} (shard_sequences(..., eval_batch={self.batch_size}))")
            self._check_slice(seq)
        # sharded: the metric rows of this rank's closed evaluater batches, their sizes and their global batch indices
        self._rows, self._row_sizes, self._row_index = [], [], []
        self._batch_index = self._slices[0].position // self.batch_size if self._slices else 0

    # ---- the sequence side ---------------------------------------------------------------------------------------------
    def push(self, image, pose, intrinsics, target, mvobj_mask=None):
        if self.seq is None:
            raise ValueError("SequenceEvaluater.push needs a sequence (seq is None)")
        H, W = image.shape[-2:]
        if self._needs_mvobj and mvobj_mask is None:
            raise ValueError(f"{[n for n in self.names if 'onlydynamic' in n]} need the frame's mvobj_mask")
        maps = [target] + ([mvobj_mask] if self._needs_mvobj else [])
        for t in maps:
            if t.numel() != H * W or tuple(t.shape[-2:]) != (H, W):
                raise ValueError(f"SequenceEvaluater.push: target / mvobj_mask [1,H,W] of the image's size {(H, W)} expected, "
                                 f"got {tuple(t.shape)}")
        R = self.seq.ring_len
        if self._rings is None or self._rings[0].shape[0] != R or tuple(self._rings[0].shape[2:]) != (H, W):
            self._rings = [torch.empty(R, 1, H, W, device=self.seq.device) for _ in maps]
        slot = self.seq.n_pushed % R
        for ring, t in zip(self._rings, maps):
            ring[slot].copy_(t.reshape(1, H, W), non_blocking=True)
        emitted = self.seq.push(image, pose, intrinsics)
        self._consume(emitted)
        return emitted

    def flush(self):
        emitted = self.seq.flush() if self.seq is not None else []
        self._consume(emitted)
        if self._open is not None:
            self._evaluate(self._open, [self._open[0].shape[0]])
            self._open = None
        return emitted

    def next_sequence(self, seq):
        """Runs the key frames the current sequence still holds, then continues on `seq`: the totals and the open evaluater
        batch carry over.  Returns what the current sequence's flush returns."""
        emitted = self.seq.flush() if self.seq is not None else []
        self._consume(emitted)
        if self._slices is not None and self.seq is not None:
            self._slice += 1
        self.seq = seq
        self._check_slice(seq)
        return emitted

    def _check_slice(self, seq):
        if seq is None or self._slices is None:
            return
        if self._slice >= len(self._slices):
            raise ValueError(f"SequenceEvaluater: a sequence after the shard's {len(self._slices)} slices")
        emit = self._slices[self._slice].emit
        if seq.key_begin > emit[0] or (seq.key_end is not None and seq.key_end < emit[1]):
            raise ValueError(f"SequenceEvaluater: the sequence runs key frames {seq.key_begin} ... {seq.key_end}, which "
                             f"do not cover the shard's key frames {emit[0]} ... {emit[1] - 1}")

    def _consume(self, emitted):
        if self._slices is not None:
            e0, e1 = self._slices[self._slice].emit if self._slice < len(self._slices) else (0, 0)
            emitted = [(i, o) for i, o in emitted if e0 <= i < e1]
        if not emitted:
            return
        result = torch.cat([o["result"] for _, o in emitted])
        R, n = self._rings[0].shape[0], len(emitted)
        first = emitted[0][0] % R                                 # the key frames' slots: at most two contiguous runs
        k = min(n, R - first)
        maps = [torch.cat([ring[first:first + k], ring[:n - k]]) for ring in self._rings]
        self.add(result, *maps)

    # ---- batching and accumulation ---------------------------------------------------------------------------------------
    def add(self, result, target, mvobj_mask=None):
        if result.dim() != 4 or result.shape[1] != 1 or tuple(target.shape) != tuple(result.shape):
            raise ValueError(f"SequenceEvaluater.add: result and target [n,1,H,W] expected, got {tuple(result.shape)} and "
                             f"{tuple(target.shape)}")
        if not result.is_cuda:
            raise M._lib.MonorecLibraryError("SequenceEvaluater needs CUDA tensors (no CPU fallback)")
        if self._needs_mvobj:
            if mvobj_mask is None or tuple(mvobj_mask.shape) != tuple(result.shape):
                raise ValueError(f"{[n for n in self.names if 'onlydynamic' in n]} need mvobj_mask of the result's shape")
        else:
            mvobj_mask = None
        H, W = result.shape[2:]
        if self.roi is not None and (not len(range(H)[self.roi[0]:self.roi[1]]) or not len(range(W)[self.roi[2]:self.roi[3]])):
            raise ValueError(f"roi {self.roi} leaves no pixel of a {H}x{W} depth map")
        parts = [result.to(torch.float32), target.to(result.device, torch.float32)]
        if mvobj_mask is not None:
            parts.append(mvobj_mask.to(result.device, torch.float32))
        if self._open is not None:
            parts = [torch.cat([o, p]) for o, p in zip(self._open, parts)]
        n, bs = parts[0].shape[0], self.batch_size
        full = n // bs * bs
        if full:
            self._evaluate([p[:full] for p in parts], [bs] * (full // bs))
        # the rest waits for the next key frames (a copy: the sequence's outputs are overwritten by its next replay)
        self._open = [p[full:].clone() for p in parts] if full < n else None

    def _evaluate(self, parts, sizes):
        """One accumulation of len(sizes) evaluater batches; parts = [result, target(, mvobj_mask)] hold their key frames in
        order."""
        result, target = parts[0], parts[1]
        mvobj_mask = parts[2] if len(parts) > 2 else None
        group = sizes[0]
        if self._state is None:
            self._state = torch.zeros(3 * len(self.names) + 1, dtype=torch.float64, device=result.device)

        def run(key, pred):
            if key[0] == "dense":
                min_inv = 0.0 if self.max_distance is None else 1 / self.max_distance
                return M.dense_metrics_grouped_impl(pred, target, self.roi, float(min_inv), group)
            max_d = float(self.max_distance) if self.max_distance else 0.0
            return M.sparse_metrics_grouped_impl(pred, target, mvobj_mask if key[2] else None, self.roi, max_d, key[1], group)

        if not self.median_scaling:
            passes = {}
            for key, _ in self._specs:
                if key not in passes:
                    passes[key] = run(key, result)
            cols = [passes[key][:, col] for key, col in self._specs]
        else:
            # evaluater.py:40-42 scales the data dict again before every metric: metric k sees the result scaled k + 1 times
            cols, cur = [], result
            for key, col in self._specs:
                cur = M.median_scaling_impl(cur, target)
                cols.append(run(key, cur)[:, col])
        if self._slices is None:
            M.eval_accumulate_impl(torch.stack(cols, 1), sizes, self._state)
            return
        self._rows.append(torch.stack(cols, 1).to(torch.float32))
        self._row_sizes += sizes
        self._row_index += range(self._batch_index, self._batch_index + len(sizes))
        self._batch_index += len(sizes)

    def _gathered_state(self):
        """The one-process device state from every rank's rows: gathered (a collective), put in global batch order and
        folded by the same accumulator.  Rows travel as float64, which holds their float32 values (NaN and inf included)
        and the integer tags exactly."""
        from .dist import all_gather_rows
        m = len(self.names)
        dev = self.seq.device if self.seq is not None else (self._rows[0].device if self._rows else
                                                            torch.device("cuda", torch.cuda.current_device()))
        rows = torch.cat(self._rows) if self._rows else torch.zeros(0, m, device=dev)
        tags = torch.tensor([self._row_index, self._row_sizes], dtype=torch.float64).reshape(2, len(self._row_index)).t()
        rows = all_gather_rows(torch.cat([tags.to(rows.device), rows.to(torch.float64)], 1), self.group)
        if rows.shape[0] == 0:
            return None
        rows = rows[torch.argsort(rows[:, 0])]
        tags = rows[:, :2].cpu().to(torch.int64)
        if not torch.equal(tags[:, 0], torch.arange(rows.shape[0])):
            raise RuntimeError(f"SequenceEvaluater.log: the ranks hold evaluater batches {tags[:, 0].tolist()}, not each of "
                               f"0 ... {rows.shape[0] - 1} once: the ranks' shards do not tile the run")
        state = torch.zeros(3 * m + 1, dtype=torch.float64, device=rows.device)
        return M.eval_accumulate_impl(rows[:, 2:].to(torch.float32), tags[:, 1].tolist(), state)

    def log(self):
        m = len(self.names)
        state = self._state if self._slices is None else self._gathered_state()
        s = np.zeros(3 * m + 1) if state is None else state.cpu().numpy()
        total, valid, avg = s[:m], s[m:2 * m], s[2 * m:3 * m]
        with np.errstate(divide="ignore", invalid="ignore"):
            metrics = (total / valid).tolist()
        return {"loss": 0.0, "metrics": metrics, "metrics_correct": avg.tolist(), "valid_batches": valid[0],
                "loss_loss": 0.0}
