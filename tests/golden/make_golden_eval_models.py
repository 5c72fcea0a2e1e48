#!/usr/bin/env python
"""Writes tests/golden/eval_models.npz by running the UNMODIFIED reference evaluate.py `main` on CPU fp32 over a list of
two models:

    MONOREC_REFERENCE=<path to the MonoRec checkout> python tests/golden/make_golden_eval_models.py

`main` takes a parsed config; it gets a stand-in with the pieces main reads (`config["models"]` without "arch", the loss and
metric names, a logger, `log_dir`), whose `initialize` returns the stub loader of make_golden_eval_sequence.py (seeded
(data, target) batches of key frames, batch size 2, with a stub dataset holding public, private, path and ndarray
attributes) and whose `initialize_list` returns two reference MonoRecModels built with the arguments of
configs/evaluate/eval_monorec.json's model (the second with use_ssim=2), each with a forward that puts precomputed results
into the data dict.  `Evaluater.eval` runs unmodified on an instance whose constructor (which wants a full trainer
config) is replaced by the field set-up of make_golden_eval_sequence.py.  The evaluate.py modules main only passes to the
config (data_loader.data_loaders, model.model) are stubbed, so that their third-party imports are not needed.

Stored:
  result_0, result_1, target   [N,1,H,W] fp32: each model's inverse depths and the ground truth of the N key frames
  cfg                          JSON: metric names, batch size, max_distance
  results_json                 the results.json main wrote
"""
import json
import logging
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE))

from make_golden import import_reference  # noqa: E402  (same shims, same reference import)
from make_golden_eval_sequence import SPARSE7, inputs  # noqa: E402

CFG = dict(names=SPARSE7, batch_size=2, max_distance=80)
MODEL_ARGS = [dict(inv_depth_min_max=[0.33, 0.0025], pretrain_mode=0, pretrain_dropout=0, use_stereo=False, use_mono=True,
                   use_ssim=1),
              dict(inv_depth_min_max=[0.33, 0.0025], pretrain_mode=0, pretrain_dropout=0, use_stereo=False, use_mono=True,
                   use_ssim=2)]


class _Dataset:
    """Stands in for the KITTI dataset: public values of the kinds evaluate.py converts, and private ones it drops."""

    def __init__(self):
        self.dataset_dir = Path("data/dataset")
        self.frame_count = 2
        self.sequences = ["00", "04"]
        self.depth_range = np.array([0.5, 80.0])
        self.use_color = True
        self._offset = 1


class _Loader:
    def __init__(self, batches):
        self.batches, self.batch_size, self.dataset = batches, CFG["batch_size"], _Dataset()

    def __iter__(self):
        return iter(self.batches)

    def __len__(self):
        return len(self.batches)


def main():
    torch.manual_seed(0)
    ref_mod = import_reference()
    for name in ("data_loader.data_loaders", "model.model"):
        sys.modules[name] = types.ModuleType(name)
    import evaluate  # noqa
    from evaluater import Evaluater  # noqa

    result, target = inputs()
    results = [result, (result * 0.9 + 0.004 * torch.rand(result.shape, generator=torch.Generator().manual_seed(5)))]
    n, bs = result.shape[0], CFG["batch_size"]
    batches = [({"index": torch.arange(b, min(b + bs, n))}, target[b:min(b + bs, n)].clone()) for b in range(0, n, bs)]

    class StubModel(ref_mod.MonoRecModel):
        def forward(self, data):
            data["result"] = self._results[data["index"]].clone()
            return data

    models = []
    for args, res in zip(MODEL_ARGS, results):
        m = StubModel(**args)
        m._results = res
        models.append(m)

    class StubEvaluater(Evaluater):
        def __init__(self, model, loss, metrics, config, data_loader):
            self.model, self.loss, self.metrics, self.data_loader = model, loss, metrics, data_loader
            self.len_data = len(data_loader)
            self.device, self.log_step = "cpu", 1
            self.logger = logging.getLogger("make_golden_eval_models")
            self.roi, self.max_distance, self.median_scaling = None, CFG["max_distance"], False

    evaluate.Evaluater = StubEvaluater
    tmp = tempfile.mkdtemp()

    class Config:
        config = {"models": [{"type": "MonoRecModel", "args": a} for a in MODEL_ARGS]}
        log_dir = tmp

        def __getitem__(self, key):
            return {"loss": next(n for n in dir(evaluate.module_loss) if not n.startswith("_")),
                    "metrics": CFG["names"]}[key]

        def get_logger(self, name):
            return logging.getLogger(name)

        def initialize(self, name, module):
            return _Loader(batches)

        def initialize_list(self, name, module):
            return models

    evaluate.main(Config())
    text = (Path(tmp) / "results.json").read_text()
    out = {"result_0": results[0].numpy(), "result_1": results[1].numpy(), "target": target.numpy(),
           "cfg": np.array(json.dumps(CFG)), "results_json": np.array(text)}
    path = HERE / "eval_models.npz"
    np.savez_compressed(path, **out)
    for r in json.loads(text):
        print(sorted(r), sorted(r["result"]), r["result"]["valid_batches"], r["result"]["metrics"][:2])
    print(path.name, path.stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
