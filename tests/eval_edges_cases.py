"""The parameter sets of tests/golden/eval_edges.npz, shared by make_golden_eval_edges.py and the tests that read it."""
import numpy as np

NAMES = ("a1", "a2", "a3", "rmse", "rmse_log", "abs_rel", "sq_rel")
# sparse metrics: tag -> (reference name suffix, roi, max_distance), called as metric(data_dict, roi, max_distance)
SPARSE_CASES = {"plain": ("", None, None), "md": ("", None, 80.0), "onlyvalid": ("_onlyvalid", None, 50.0),
                "onlydynamic": ("_onlydynamic", None, 80.0), "roi_neg_md": ("", [-20, -2, 3, -3], 80.0),
                "roi_wide": ("", [0, 100, -100, 40], None)}
# the images of each stored row: the whole batch, then the rows of group = 2 (a ragged last group)
SLICES = ((0, 5), (0, 2), (2, 4), (4, 5))
GROUP = 2
# PLYSaver(min_d=PC_MIN_D, max_d=PC_MAX_D, roi=PC_ROIS[tag])
PC_MIN_D, PC_MAX_D = 3.0, 20.0
PC_ROIS = {"neg": [-20, -2, 6, -6], "wide": [4, 100, -100, 40], "empty": [10, 5, 0, 48], "none": None}


def sparse_kwargs(tag):
    """SPARSE_CASES[tag] as keyword arguments of the device pass / the oracle: (roi, max_distance, pred_all_valid,
    use_cvmask)."""
    suffix, roi, md = SPARSE_CASES[tag]
    return dict(roi=roi, max_distance=md, pred_all_valid=suffix != "_onlyvalid", use_cvmask=suffix == "_onlydynamic")


def assert_same(got, ref, rtol, atol):
    """NaN and +-inf in the same places; finite values within rtol / atol."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_array_equal(np.isposinf(got), np.isposinf(ref))
    np.testing.assert_array_equal(np.isneginf(got), np.isneginf(ref))
    fin = np.isfinite(ref)
    np.testing.assert_allclose(got[fin], ref[fin], rtol=rtol, atol=atol)
