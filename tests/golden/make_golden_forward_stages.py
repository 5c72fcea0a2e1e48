#!/usr/bin/env python
"""Writes tests/golden/forward_stages.json on an H100: per conv mode (tf32, f16) and input (the model_synth_small and
model_kitti_sample goldens' inputs and weight seeds), the names of the library entries one eager MonoRecModel.forward
calls, in order, and the sha256 of the bytes of each of its output tensors.

    python tests/golden/make_golden_forward_stages.py --model-source FILE

FILE is the monorec_b200/model.py whose forward is recorded, loaded inside the package in place of the installed one.  The
stored golden is the single-block forward that MonoRecModel.forward had before it was split into the cost-volume, trunk
and heads stages (commit 64b7af2: `git show 64b7af2:monorec_b200/model.py > FILE`), so tests/test_eval_models_gpu.py checks
that the staged forward issues the same calls and computes the same bits.
"""
import argparse
import importlib.util
import json
import sys
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from tests.test_eval_models_gpu import golden_inputs, output_digests, record_calls, seeded_model  # noqa: E402


def load_model_module(path):
    spec = importlib.util.spec_from_file_location("monorec_b200._recorded_model", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-source", required=True)
    ap.add_argument("--out", default=str(HERE / "forward_stages.json"))
    args = ap.parse_args()
    import monorec_b200  # noqa: F401
    from monorec_b200 import conv as C
    mod = load_model_module(args.model_source)
    out = {}
    for mode in ("tf32", "f16"):
        C.set_mode(mode)
        out[mode] = {}
        for which in ("synth_small", "kitti_sample"):
            wseed, d = golden_inputs(which)
            model = seeded_model(mod.MonoRecModel, wseed)
            with torch.no_grad():
                model(dict(d))
                res, calls = record_calls(lambda: model(dict(d)))
            out[mode][which] = {"calls": calls, "sha256": output_digests(res)}
            print(mode, which, len(calls), "calls", flush=True)
    Path(args.out).write_text(json.dumps(out, indent=1) + "\n")
    print("wrote", args.out)


if __name__ == "__main__":
    main()
