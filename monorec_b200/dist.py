"""Batch sharding for the one-process-per-GPU layout (replaces the reference's single-process
torch.nn.DataParallel scatter/gather: base/base_trainer.py:26-29, evaluater/evaluater.py:29-30).

Every keyframe is independent end to end (SURVEY.md §8e), so the path shards on dim 0 with no data-path collective;
the only exchange is the optional all-gather of the per-rank result maps.

`shard_sequences` is the same split for the sequence path (MonoRecSequence, SequenceEvaluater, SequencePointCloud): each
rank runs a contiguous slice of the key frames of one or more concatenated sequences and pushes only the frames that slice
needs; `all_gather_rows` / `gather_rows` move the few per-rank results at the end.
"""
from typing import NamedTuple, Tuple

import torch
import torch.distributed as dist


def shard_bounds(batch, rank, world):
    """Contiguous, balanced [lo, hi) of a batch of `batch` keyframes for `rank` of `world`."""
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class SequenceSlice(NamedTuple):
    """One sequence's part of a rank's work (sequence indices, [lo, hi) ranges)."""
    sequence: int                  # index into the list of sequence lengths
    frames: Tuple[int, int]        # the frames to push: MonoRecSequence(first_frame=frames[0]) and push frames[0] .. frames[1]-1
    run: Tuple[int, int]           # the key frames the model runs (whole batches of the one-process run): key_end=run[1]
    emit: Tuple[int, int]          # the key frames evaluated / added to the point cloud, inside `run`
    position: int                  # place of emit[0] in the concatenated list of emitted key frames of all sequences


def shard_sequences(lengths, frame_count, dilation, batch_size, rank, world, eval_batch=None, buffer_length=None,
                    keys=None, layout=None):
    """The slices of sequences of `lengths` frames that `rank` of `world` runs, in sequence order (sequences it does not
    touch are left out; a rank may get none).  Exactly one of:

    `eval_batch` (SequenceEvaluater's batch_size): every key frame with all its neighbours (the loader's index range) is
    emitted by one rank.  A rank emits whole evaluater batches of the concatenated key-frame list, as the loader batches it
    across sequence boundaries (only the globally last batch can be partial), so no evaluater batch is split between ranks.
    `position` counts key frames over all sequences; rank r's first batch has global index position // eval_batch.

    `buffer_length` (SequencePointCloud's vote window): the key frames the one-process export adds (those whose whole
    window of buffer_length key frames lies in their sequence) are split evenly, and a rank also runs the buffer_length // 2
    key frames on either side of its slice for their keep masks.  `position` counts added key frames.

    Either way, `run` is made of whole model batches of the one-process run: multiples of `batch_size` from the sequence's
    first key frame, and the short last batch at its end, so every key frame's outputs come from the same batch of the same
    inputs as in one process.

    `keys`: one key-frame list per sequence (MonoRecSequence's `keys`, e.g. sequence.loader_keys with index masks; None in
    the list, or keys=None, for every key frame with its neighbours).  Everything above is then counted in listed key
    frames: positions, evaluater batches, model batches and the vote windows' neighbours.  `run` and `emit` stay sequence
    indices ([first, last + 1) of the listed key frames in them), and `frames` spans the run's neighbours; a rank passes the
    frames in it that no listed key frame needs with MonoRecSequence.skip.

    `layout`: one sequence.FrameLayout per sequence (MonoRecSequence's `layout`), in place of frame_count, dilation and
    `keys`.  Its key frames are counted as a `keys` list is, and `frames` spans the run's frames at the layout's offsets."""
    if (eval_batch is None) == (buffer_length is None):
        raise ValueError("shard_sequences: give exactly one of eval_batch and buffer_length")
    if batch_size < 1 or world < 1 or not 0 <= rank < world:
        raise ValueError(f"shard_sequences: batch_size ({batch_size}) >= 1 and 0 <= rank ({rank}) < world ({world}) needed")
    from .sequence import check_keys, neighbour_offsets
    if keys is not None and layout is not None:
        raise ValueError("shard_sequences: give keys or layout, not both (a layout holds its key frames)")
    if keys is not None and len(keys) != len(lengths):
        raise ValueError(f"shard_sequences: {len(keys)} key lists for {len(lengths)} sequences")
    if layout is None:
        offs = neighbour_offsets(frame_count, dilation)
        lo, hi = min(0, min(offs)), max(offs)
        spread = [(lo, hi)] * len(lengths)
        # the key frames of each sequence: the listed ones, or -lo .. n - hi - 1
        K = [range(-lo, int(n) - hi) if keys is None or keys[s] is None else check_keys(keys[s], offs, n)
             for s, n in enumerate(lengths)]
    else:
        if len(layout) != len(lengths):
            raise ValueError(f"shard_sequences: {len(layout)} layouts for {len(lengths)} sequences")
        # the frames key frame i uses are i + lo ... i + hi, its own included
        spread = [(min(0, min(lay.offsets)), max(0, max(lay.offsets))) for lay in layout]
        K = [check_keys(lay.keys, lay.offsets, n) for lay, n in zip(layout, lengths)]
    n_keys = [len(k) for k in K]
    if eval_batch is not None:
        if eval_batch < 1:
            raise ValueError(f"shard_sequences: eval_batch ({eval_batch}) must be >= 1")
        before, after = 0, 0
        # the emitted positions of sequence s: its key frames, all of them
        spans = [(0, k) for k in n_keys]
        # rank r starts at the evaluater batch boundary nearest r / world of the key frames
        total = sum(n_keys)
        cut = lambda r: min(total, (2 * total * r + world * eval_batch) // (2 * world * eval_batch) * eval_batch)  # noqa: E731
        mine = (cut(rank), total if rank == world - 1 else cut(rank + 1))
    else:
        if buffer_length < 1:
            raise ValueError(f"shard_sequences: buffer_length ({buffer_length}) must be >= 1")
        before, after = buffer_length // 2, buffer_length - 1 - buffer_length // 2
        spans = [(before, max(before, k - after)) for k in n_keys]
        mine = shard_bounds(sum(e - b for b, e in spans), rank, world)
    out, offset = [], 0
    for s, ((p0, p1), k) in enumerate(zip(spans, n_keys)):
        a, b = max(p0, mine[0] - offset + p0), min(p1, mine[1] - offset + p0)   # emitted positions (from the first key frame)
        if a < b:
            r0 = (a - before) // batch_size * batch_size
            r1 = min(k, -(-(b + after) // batch_size) * batch_size)
            key = K[s]
            lo, hi = spread[s]
            out.append(SequenceSlice(s, (key[r0] + lo, key[r1 - 1] + hi + 1), (key[r0], key[r1 - 1] + 1),
                                     (key[a], key[b - 1] + 1), offset + a - p0))
        offset += p1 - p0
    return out


def shard_data_dict(data, rank, world):
    """Slices every tensor (and every tensor in a list) of a MonoRec data_dict on dim 0."""
    batch = data["keyframe"].shape[0]
    lo, hi = shard_bounds(batch, rank, world)
    out = {}
    for k, v in data.items():
        if isinstance(v, (list, tuple)):
            out[k] = [t[lo:hi] if torch.is_tensor(t) and t.dim() > 0 and t.shape[0] == batch else t for t in v]
        elif torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == batch:
            out[k] = v[lo:hi]
        else:
            out[k] = v
    return out


def all_gather_batch(t, group=None, equal_shards=False):
    """All-gather of per-rank (b_r, ...) maps into (sum b_r, ...) on every rank (one ncclAllGather when the shards
    are equal, a padded gather otherwise).  `equal_shards=True` asserts the caller knows every rank holds the same b_r
    (a batch divisible by the world size) and skips the size exchange and its host synchronisation."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return t
    world = dist.get_world_size(group)
    if equal_shards:
        out = t.new_empty((world * t.shape[0],) + tuple(t.shape[1:]))
        dist.all_gather_into_tensor(out, t.contiguous(), group=group)
        return out
    sizes = torch.tensor([t.shape[0]], device=t.device, dtype=torch.int64)
    all_sizes = [torch.zeros_like(sizes) for _ in range(world)]
    dist.all_gather(all_sizes, sizes, group=group)
    all_sizes = [int(s.item()) for s in all_sizes]
    if len(set(all_sizes)) == 1:
        out = t.new_empty((world * t.shape[0],) + tuple(t.shape[1:]))
        dist.all_gather_into_tensor(out, t.contiguous(), group=group)
        return out
    mx = max(all_sizes)
    pad = t.new_zeros((mx,) + tuple(t.shape[1:]))
    pad[: t.shape[0]] = t
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    return torch.cat([b[:n] for b, n in zip(bufs, all_sizes)], 0)


def _exchange_device(t, group):
    """NCCL moves CUDA tensors between GPUs; any other backend (gloo: ranks sharing a GPU, or a CPU group) goes through host
    memory."""
    return t.device if t.is_cuda and "nccl" in str(dist.get_backend(group)).lower() else torch.device("cpu")


def _row_counts(x, group):
    n = torch.tensor([x.shape[0]], device=x.device, dtype=torch.int64)
    counts = [torch.zeros_like(n) for _ in range(dist.get_world_size(group))]
    dist.all_gather(counts, n, group=group)
    return [int(c.item()) for c in counts]


def all_gather_rows(t, group=None):
    """Every rank's rows (b_r, ...) of a variable count, concatenated in rank order, on every rank (on t's device).  A
    collective: every rank of `group` calls it, with b_r = 0 allowed."""
    x = t.to(_exchange_device(t, group)).contiguous()
    counts = _row_counts(x, group)
    if max(counts) == 0:
        return t[:0]
    pad = x.new_zeros((max(counts),) + tuple(x.shape[1:]))
    pad[:x.shape[0]] = x
    bufs = [torch.empty_like(pad) for _ in counts]
    dist.all_gather(bufs, pad, group=group)
    return torch.cat([b[:n] for b, n in zip(bufs, counts)]).to(t.device)


def gather_rows(t, dst=0, group=None):
    """Every rank's rows (b_r, ...) concatenated in rank order on rank `dst` of `group` (on t's device); None on the other
    ranks.  A collective, as all_gather_rows."""
    x = t.to(_exchange_device(t, group)).contiguous()
    counts = _row_counts(x, group)
    me = dist.get_rank(group)
    if max(counts) == 0:
        return t[:0] if me == dst else None
    pad = x.new_zeros((max(counts),) + tuple(x.shape[1:]))
    pad[:x.shape[0]] = x
    bufs = [torch.empty_like(pad) for _ in counts] if me == dst else None
    dist.gather(pad, bufs, dst=dist.get_global_rank(group, dst) if group is not None else dst, group=group)
    return torch.cat([b[:n] for b, n in zip(bufs, counts)]).to(t.device) if me == dst else None
