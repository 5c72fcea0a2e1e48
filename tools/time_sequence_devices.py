"""Key frames per second of the sequence evaluation and point-cloud export run by one process over several lanes
(lanes.MultiDeviceEvaluater / MultiDevicePointCloud), against the torchrun path, and of the one-GPU export with and
without a read-back of the vertex count per batch.

    python tools/time_sequence_devices.py [--frames=F] [--rounds=R] [--mode=f16|tf32|fp32] [--shared=2,3] [--no-torchrun]

The synthetic 256x512 stream of tools/time_sequence_dist.py (one sequence of F frames on the host, frame_count 2, model
batch 8 by CUDA-graph replay, random-init weights; eval_monorec.json's evaluation settings, create_pointcloud.py's export
settings).  Prints one JSON line per measurement, each with the card name and power limit:
  lanes      1 ... N lanes on N GPUs (N = the GPUs visible), and --shared lanes taking turns on cuda:0.  A round is a fresh
             run (graph captures included) from the first push to the log / the vertex count; the median of R rounds.
  torchrun   tools/time_sequence_dist.py under torchrun with as many ranks, on the same devices (--no-torchrun: skipped)
  readback   the one-GPU export (MonoRecSequence + sequence_pointcloud) with PLYSaver as it is against a PLYSaver that reads
             the count back before every add, as the saver did before (`item()` per batch), alternated round by round
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import monorec_b200.model as MM  # noqa: E402
from monorec_b200 import conv as C  # noqa: E402
from monorec_b200 import pointcloud as PC  # noqa: E402
from monorec_b200.lanes import MultiDeviceEvaluater, MultiDevicePointCloud  # noqa: E402
from monorec_b200.sequence import MonoRecSequence  # noqa: E402
from monorec_b200.synthetic import make_sequence, seeded_state_dict  # noqa: E402
from tools.time_eval_sequence import BATCH, MAX_D, NAMES  # noqa: E402
from tools.time_sequence import DROPOUT, ROI, power_limit  # noqa: E402
from tools.time_sequence import MAX_D as PLY_MAX_D  # noqa: E402

H, W = 256, 512
SEQ_BATCH, BUFFER = 8, 5


class _ReadBackSaver(PC.PLYSaver):
    """PLYSaver sized as before: the count read back (a host synchronisation) before every add."""

    def _reserve(self, lib, B, H, W, dev):
        self._in_flight.clear()
        if self._count is not None:
            self._known = int(self._count.item())
        return super()._reserve(lib, B, H, W, dev)

    def _track(self, worst, dev):
        self._in_flight.append((None, None, worst))


def run_eval(model, devices, data):
    images, poses, Ks, targets = data
    run = MultiDeviceEvaluater(model, devices, [images.shape[0]], NAMES, BATCH, seq_batch=SEQ_BATCH, max_distance=MAX_D)
    for s, n in run.order:
        run.push(s, n, images[n], poses[n], Ks[n], targets[n])
    run.flush()
    return run.log()["valid_batches"]


def run_export(model, devices, data):
    images, poses, Ks, _ = data
    run = MultiDevicePointCloud(model, devices, [images.shape[0]], H, W, seq_batch=SEQ_BATCH, buffer_length=BUFFER,
                                max_d=PLY_MAX_D, roi=ROI, dropout=DROPOUT)
    for s, n in run.order:
        run.push(s, n, images[n], poses[n], Ks[n])
    run.flush()
    return sum(len(s) for s in run.savers)


def run_one_gpu_export(model, data, saver_class):
    images, poses, Ks, _ = data
    saver = saver_class(H, W, max_d=PLY_MAX_D, roi=ROI, dropout=DROPOUT)
    pc = PC.sequence_pointcloud(MonoRecSequence(model, batch_size=SEQ_BATCH), saver)
    n = 0
    for f in range(images.shape[0]):
        n += len(pc.push(images[f], poses[f], Ks[f]))
    n += len(pc.flush())
    return n, len(saver)


def timed(fn, devices):
    for d in set(devices):
        torch.cuda.synchronize(d)
    t0 = time.perf_counter()
    out = fn()
    for d in set(devices):
        torch.cuda.synchronize(d)
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--mode", default="f16", choices=["f16", "tf32", "fp32"])
    ap.add_argument("--shared", default="2,3", help="lane counts to run on cuda:0 alone")
    ap.add_argument("--no-torchrun", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sequence_devices.py needs a GPU")
    C.set_mode(args.mode)
    gpus = torch.cuda.device_count()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "gpus": gpus, "mode": args.mode,
            "size": [H, W], "frames": args.frames, "batch": SEQ_BATCH, "eval_batch": BATCH}
    models = {}
    for name, kw in (("eval", {}), ("export", dict(inv_depth_min_max=(0.33, 0.06)))):
        m = MM.MonoRecModel(**kw)
        m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
        models[name] = m.to("cuda:0").eval()
    gen = torch.Generator().manual_seed(2)
    targets = torch.rand(args.frames, 1, H, W, generator=gen) * 0.3 + 0.0125
    targets[torch.rand(args.frames, 1, H, W, generator=gen) > 0.05] = 0.0
    data = make_sequence(args.frames, H, W, seed=1) + (targets,)
    keyframes = args.frames - 2

    layouts = [("gpus", list(range(n))) for n in range(1, gpus + 1)]
    layouts += [("shared", [0] * int(n)) for n in args.shared.split(",") if n]
    with torch.no_grad():
        # the export's read-back per batch, before and after, alternated on one GPU
        variants = {"no_readback": PC.PLYSaver, "readback_per_batch": _ReadBackSaver}
        for cls in variants.values():
            run_one_gpu_export(models["export"], data, cls)
        rates, verts = {k: [] for k in variants}, {}
        for _ in range(args.rounds):
            for name, cls in variants.items():
                dt, (n, v) = timed(lambda: run_one_gpu_export(models["export"], data, cls), [0])
                rates[name].append(n / dt)
                verts[name] = v
        print(json.dumps(dict(card, measurement="readback", keyframes_per_s={k: statistics.median(v) for k, v in
                                                                              rates.items()}, rounds=rates,
                              vertices=verts)), flush=True)

        for kind, devices in layouts:
            rates, results = {"eval": [], "export": []}, {}
            for r in range(args.rounds + 1):               # round 0: warm-up (packing on every device, algorithms)
                for name, fn in (("eval", run_eval), ("export", run_export)):
                    dt, results[name] = timed(lambda: fn(models[name], devices, data), devices)
                    if r:
                        rates[name].append(keyframes / dt)
            print(json.dumps(dict(card, measurement="lanes", layout=kind, devices=devices, keyframes=keyframes,
                                  keyframes_per_s={k: statistics.median(v) for k, v in rates.items()}, rounds=rates,
                                  valid_batches=results["eval"], vertices=results["export"])), flush=True)

    if args.no_torchrun:
        return
    for kind, devices in layouts:
        env = dict(os.environ, CUDA_VISIBLE_DEVICES=",".join(str(d) for d in sorted(set(devices))))
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", str(len(devices)),
               str(ROOT / "tools" / "time_sequence_dist.py"), f"--frames={args.frames}", f"--rounds={args.rounds}",
               f"--mode={args.mode}"]
        res = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=1800)
        line = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
        out = json.loads(line[-1]) if line else {"error": (res.stderr or res.stdout)[-2000:]}
        print(json.dumps(dict(card, measurement="torchrun", layout=kind, devices=devices, result=out)), flush=True)


if __name__ == "__main__":
    main()
