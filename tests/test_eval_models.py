"""MultiModelEvaluater without a GPU: which models share the cost-volume and trunk stages, and evaluate.py's results.json
structure, pinned on the reference's own results.json for two models (tests/golden/eval_models.npz)."""
import json
import pathlib
import warnings

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN


def _model(**kw):
    from monorec_b200.model import MonoRecModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")          # (no ImageNet weights in the hub cache: randomly initialised trunk)
        return MonoRecModel(**kw).eval()


@pytest.fixture(scope="module")
def base():
    return _model()


def _like(base, **kw):
    """A model built with `kw` that holds base's weights wherever the shapes agree."""
    m = _model(**kw)
    own = m.state_dict()
    m.load_state_dict({k: v for k, v in base.state_dict().items() if k in own and own[k].shape == v.shape}, strict=False)
    return m


# every field of the cost-volume key, changed one at a time: each model gets a cost-volume stage of its own
CV_VARIANTS = {
    "use_ssim": dict(use_ssim=2),
    "use_stereo": dict(use_stereo=True),
    "use_mono": dict(use_mono=False, use_stereo=True),
    "cv_depth_steps": dict(cv_depth_steps=24),
    "inv_depth_min_max": dict(inv_depth_min_max=(0.25, 0.0025)),
    "volume_dtype": dict(volume_dtype=torch.float16),
    "no_cv": dict(no_cv=True),
    "nhwc_copy": dict(mask_use_cv=False),
}


@pytest.mark.parametrize("field", sorted(CV_VARIANTS))
def test_each_cost_volume_field_splits_the_cost_volume_group(base, field):
    from monorec_b200.models_eval import cost_volume_key, share_groups
    other = _like(base, **CV_VARIANTS[field])
    same = _like(base)
    assert cost_volume_key(other) != cost_volume_key(base)
    cv_groups, trunk_groups = share_groups([base, other, same])
    assert cv_groups == [[0, 2], [1]]
    assert trunk_groups == [[0, 1, 2]]                # the trunk weights are base's in all three


def test_cost_volume_module_options_split_the_group(base):
    """Options of the cost-volume module outside the constructor's keywords change the volume as well."""
    from monorec_b200.models_eval import share_groups
    for attr, value in (("not_center_cv", True), ("alpha", 5), ("channel_weights", (1 / 3, 1 / 3, 1 / 3))):
        other = _like(base)
        setattr(other.cv_module, attr, value)
        assert share_groups([base, other])[0] == [[0], [1]], attr


def test_nhwc_copy_follows_the_mask_module(base):
    """A model without a MaskModule reading the volumes does not write the NHWC copy: it shares only with its kind."""
    from monorec_b200 import conv as C
    from monorec_b200.models_eval import share_groups
    p1, p3 = _like(base, pretrain_mode=1), _like(base, pretrain_mode=3)
    groups = share_groups([base, p1, p3])[0]
    assert groups == ([[0], [1, 2]] if C.MODE in ("tf32", "f16") else [[0, 1, 2]])


def test_trunk_groups_follow_the_weights(base):
    from monorec_b200.models_eval import share_groups
    equal = _like(base, use_ssim=2)
    moved = _like(base)
    with torch.no_grad():
        moved._feature_extractor.encoder.layer3[1].conv2.weight[0, 0, 0, 0] += 1e-6
    bn = _like(base)
    with torch.no_grad():
        bn._feature_extractor.encoder.bn1.running_var[5] *= 1.5   # a BatchNorm buffer, not a parameter
    fresh = _model()                                              # its own random trunk
    cv_groups, trunk_groups = share_groups([base, equal, moved, bn, fresh])
    assert trunk_groups == [[0, 1], [2], [3], [4]]
    assert cv_groups == [[0, 2, 3, 4], [1]]


def test_unsupported_inputs_raise(base):
    from monorec_b200.models_eval import MultiModelEvaluater
    with pytest.raises(NotImplementedError, match="stereo"):
        MultiModelEvaluater([base, _like(base, use_stereo=True)], ["a1_sparse_metric"], 2, device="cpu")
    with pytest.raises(NotImplementedError, match="mvobj_masks"):
        MultiModelEvaluater([base, _like(base, pretrain_mode=3)], ["a1_sparse_metric"], 2, device="cpu")
    with pytest.raises(ValueError, match="empty"):
        MultiModelEvaluater([], ["a1_sparse_metric"], 2, device="cpu")
    with pytest.raises(ValueError, match="unknown metric"):
        MultiModelEvaluater([base], ["nope"], 2, device="cpu")


class _Dataset:
    """The stub dataset of make_golden_eval_models.py, restated."""

    def __init__(self):
        self.dataset_dir = pathlib.Path("data/dataset")
        self.frame_count = 2
        self.sequences = ["00", "04"]
        self.depth_range = np.array([0.5, 80.0])
        self.use_color = True
        self._offset = 1


def test_results_have_the_reference_structure():
    """results(): one entry per model with the reference's keys; the model dict holds the reference MonoRecModel's public
    attributes with its values (plus volume_dtype, by name), the dataset dict is evaluate.py's, `metrics_info` the names;
    the whole list is JSON."""
    from monorec_b200.models_eval import MultiModelEvaluater
    g = np.load(GOLDEN / "eval_models.npz")
    ref = json.loads(str(g["results_json"]))
    cfg = json.loads(str(g["cfg"]))
    args = [r["model"] for r in ref]
    kw = [{k: args[i][k] for k in ("inv_depth_min_max", "pretrain_mode", "pretrain_dropout", "use_stereo", "use_mono",
                                   "use_ssim")} for i in range(2)]
    models = [_model(**k) for k in kw]
    ev = MultiModelEvaluater(models, cfg["names"], cfg["batch_size"], max_distance=cfg["max_distance"], device="cpu")
    got = json.loads(json.dumps(ev.results(vars(_Dataset()))))
    assert len(got) == len(ref) == 2
    for mine, theirs in zip(got, ref):
        assert list(mine) == list(theirs) == ["model", "dataset", "result"]
        assert list(mine["result"]) == list(theirs["result"])
        assert mine["result"]["metrics_info"] == theirs["result"]["metrics_info"] == cfg["names"]
        assert mine["dataset"] == theirs["dataset"]
        assert set(mine["model"]) == set(theirs["model"]) | {"volume_dtype"}
        assert mine["model"]["volume_dtype"] == "torch.float32"
        # the reference's dict is taken before Evaluater.eval puts the model in eval mode
        assert {k: v for k, v in mine["model"].items() if k not in ("volume_dtype", "training")} == \
            {k: v for k, v in theirs["model"].items() if k != "training"}
        assert mine["result"]["valid_batches"] == 0.0          # nothing evaluated yet
