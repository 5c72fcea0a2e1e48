"""Key frames per second of the sequence evaluation and point-cloud export split over ranks, one process per rank.

    torchrun --nproc_per_node N tools/time_sequence_dist.py [--frames=F] [--sequences=S] [--rounds=R] [--mode=f16|tf32|fp32]

The synthetic KITTI-shaped stream of tools/time_eval_sequence.py / tools/time_sequence.py: S sequences of F frames (256x512,
host tensors as a loader yields them), frame_count 2, model batch 8 with CUDA-graph replay, random-init weights.  Every rank
takes its slices (dist.shard_sequences) and pushes only their frames.
  eval    SequenceEvaluater with eval_monorec.json's settings (evaluater batch 2, the seven sparse metrics, max_distance 80,
          a LiDAR-like target covering ~5 % of the pixels), ending with the collective log()
  export  SequencePointCloud with create_pointcloud.py's settings (roi, max_d 20, dropout 0.75, 5-frame vote), ending with
          PLYSaver.gather of every rank's vertices on rank 0
One GPU per rank over NCCL when there are as many GPUs as local ranks, else every rank on cuda:0 over gloo.  A round's number
is the key frames of the whole run (the one-process count) over the slowest rank's host time from a barrier to the end of
the collective, for fresh sequences (their graph captures included); the report is the median over R rounds, after one
warm-up round.  Rank 0 prints one JSON line with the card name and power limit.
"""
import argparse
import datetime
import json
import os
import statistics
import sys
import time
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import monorec_b200.model as MM  # noqa: E402
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200 import pointcloud as PC  # noqa: E402
from monorec_b200.dist import shard_sequences  # noqa: E402
from monorec_b200.evaluation import SequenceEvaluater  # noqa: E402
from monorec_b200.sequence import MonoRecSequence  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402
from tools.time_eval_sequence import BATCH, MAX_D, NAMES  # noqa: E402
from tools.time_sequence import DROPOUT, ROI, power_limit  # noqa: E402
from tools.time_sequence import MAX_D as PLY_MAX_D  # noqa: E402

H, W = 256, 512
SEQ_BATCH, BUFFER = 8, 5


def run_eval(model, dev, data, lengths, rank, world):
    shard = shard_sequences(lengths, 2, 1, SEQ_BATCH, rank, world, eval_batch=BATCH)
    ev = SequenceEvaluater(None, NAMES, BATCH, max_distance=MAX_D, group=dist.group.WORLD, shard=shard)
    for sl in shard:
        images, poses, Ks, targets = data[sl.sequence]
        ev.next_sequence(MonoRecSequence(model, batch_size=SEQ_BATCH, device=dev, first_frame=sl.frames[0],
                                         key_end=sl.run[1]))
        for n in range(*sl.frames):
            ev.push(images[n], poses[n], Ks[n], targets[n])
    ev.flush()
    return ev.log()


def run_export(model, dev, data, lengths, rank, world):
    saver = PC.PLYSaver(H, W, max_d=PLY_MAX_D, roi=ROI, dropout=DROPOUT)
    for sl in shard_sequences(lengths, 2, 1, SEQ_BATCH, rank, world, buffer_length=BUFFER):
        images, poses, Ks, _ = data[sl.sequence]
        pc = PC.SequencePointCloud(MonoRecSequence(model, batch_size=SEQ_BATCH, device=dev, first_frame=sl.frames[0],
                                                   key_end=sl.run[1]), saver, buffer_length=BUFFER, emit=sl.emit)
        for n in range(*sl.frames):
            pc.push(images[n], poses[n], Ks[n])
        pc.flush()
    v = saver.gather(dist.group.WORLD)
    torch.cuda.synchronize(dev)
    return 0 if v is None else v.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--sequences", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local_rank, local_world = int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("LOCAL_WORLD_SIZE", 1))
    own_gpu = torch.cuda.device_count() >= local_world
    dev = torch.device("cuda", local_rank if own_gpu else 0)
    torch.cuda.set_device(dev)
    backend = "nccl" if own_gpu else "gloo"
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600),
                            **({"device_id": dev} if own_gpu else {}))
    C.set_mode(args.mode)
    models = {}
    for name, kw in (("eval", {}), ("export", dict(inv_depth_min_max=(0.33, 0.06)))):
        m = MM.MonoRecModel(**kw)
        m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
        models[name] = m.to(dev).eval()
    lengths = [args.frames] * args.sequences
    data = []
    for s in range(args.sequences):
        gen = torch.Generator().manual_seed(2 + s)
        targets = torch.rand(args.frames, 1, H, W, generator=gen) * 0.3 + 0.0125
        targets[torch.rand(args.frames, 1, H, W, generator=gen) > 0.05] = 0.0
        data.append(make_sequence(args.frames, H, W, seed=1 + s) + (targets,))
    keyframes = sum(sl.emit[1] - sl.emit[0] for r in range(world)
                    for sl in shard_sequences(lengths, 2, 1, SEQ_BATCH, r, world, eval_batch=BATCH))
    mine = {k: sum(sl.emit[1] - sl.emit[0] for sl in shard_sequences(lengths, 2, 1, SEQ_BATCH, rank, world, **kw))
            for k, kw in (("eval", dict(eval_batch=BATCH)), ("export", dict(buffer_length=BUFFER)))}
    variants = {"eval": run_eval, "export": run_export}
    rates, results = {k: [] for k in variants}, {}
    with torch.no_grad():
        for r in range(args.rounds + 1):                 # round 0: warm-up (packing, cuDNN algorithms, graph capture)
            for name, fn in variants.items():
                dist.barrier()
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                results[name] = fn(models[name], dev, data, lengths, rank, world)
                dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64,
                                  device=dev if backend == "nccl" else "cpu")
                dist.all_reduce(dt, op=dist.ReduceOp.MAX)
                if r:
                    rates[name].append(keyframes / float(dt.item()))
    per_rank = [None] * world
    dist.all_gather_object(per_rank, mine)
    if rank == 0:
        med = {k: statistics.median(v) for k, v in rates.items()}
        print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "mode": args.mode,
                          "world": world, "backend": backend, "gpus": torch.cuda.device_count(), "size": [H, W],
                          "frames": lengths, "frame_count": 2, "batch": SEQ_BATCH, "eval_batch": BATCH,
                          "keyframes": keyframes, "keyframes_per_rank": per_rank, "keyframes_per_s": med, "rounds": rates,
                          "valid_batches": results["eval"]["valid_batches"], "vertices": results["export"]}), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
