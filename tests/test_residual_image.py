"""The residual image without a GPU: both oracles (oracle/residual_image_oracle.py) against the reference's results in
tests/golden/residual_image.npz, the argument checks of mr_residual_image (made before any CUDA call), the CPU refusal
of the Python layer and the sequence option's checks."""
import ctypes
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import residual_image_oracle as O
from tests import residual_cases as RC

GOLDEN = np.load(Path(__file__).resolve().parent / "golden" / "residual_image.npz")
EDGE = 1e-3          # px: a sample this close to the edge of the all-zero region may be masked in one evaluation only


def case_args(name):
    """(data dict, inverse depth, module arguments) of a golden case."""
    data = RC.inputs(name)
    invd = torch.from_numpy(GOLDEN[f"{name}_invd"])
    frames, poses, intr = list(data["frames"]), list(data["poses"]), list(data["intrinsics"])
    if RC.CASES[name][5]:
        frames.append(data["stereoframe"]); poses.append(data["stereoframe_pose"])
        intr.append(data["stereoframe_intrinsics"])
    rng = (torch.tensor([0.0025]), torch.tensor([0.33])) if name == "model" else (0, 1)
    return (data["keyframe"], data["keyframe_pose"], data["keyframe_intrinsics"], invd, frames, poses, intr) + rng


@pytest.mark.parametrize("name", list(RC.CASES))
def test_torch_oracle_matches_the_reference(name):
    out, masks = O.residual_image_torch(*case_args(name), return_masks=True)
    ref = torch.from_numpy(GOLDEN[f"{name}_residual"])
    assert torch.equal(masks, torch.from_numpy(GOLDEN[f"{name}_masks"]).bool())
    assert torch.equal(torch.isnan(out), torch.isnan(ref))
    assert torch.allclose(out, ref, rtol=0, atol=2e-6, equal_nan=True), (out - ref).abs().nan_to_num().max()


@pytest.mark.parametrize("name", list(RC.CASES))
def test_closed_form_matches_the_reference(name):
    cf = O.residual_image_closed_form(*case_args(name))
    ref = GOLDEN[f"{name}_residual"].astype(np.float64)
    near = (np.abs(cf["margin"]) < EDGE)
    flips = (cf["masks"] != GOLDEN[f"{name}_masks"].astype(bool))
    assert not (flips & ~near).any(), int((flips & ~near).sum())
    # pixels whose window holds a near-edge sample of some frame are compared only for their NaN pattern
    ring = near.any(1)
    ring = ring | np.pad(ring, ((0, 0), (1, 1), (1, 1)))[:, :-2, 1:-1] | np.pad(ring, ((0, 0), (1, 1), (1, 1)))[:, 2:, 1:-1]
    ring = ring | np.pad(ring, ((0, 0), (1, 1), (1, 1)))[:, 1:-1, :-2] | np.pad(ring, ((0, 0), (1, 1), (1, 1)))[:, 1:-1, 2:]
    got = cf["residual"][:, 0]
    assert np.array_equal(np.isnan(got), np.isnan(ref[:, 0]))
    keep = ~ring & ~np.isnan(got)
    assert np.abs(got - ref[:, 0])[keep].max() < 1e-4


def test_gray_case_is_a_replicated_plane():
    data = RC.inputs("gray")
    g = RC.gray(data)
    assert g["keyframe"].shape[1] == 1 and torch.equal(g["keyframe"].expand(-1, 3, -1, -1), data["keyframe"])
    args = list(case_args("gray"))
    args[0], args[4] = g["keyframe"], g["frames"]
    assert torch.equal(O.residual_image_torch(*args), torch.from_numpy(GOLDEN["gray_residual"]))


def _entry(lib, null=None, align=None, **over):
    """mr_residual_image on fake (never dereferenced) aligned pointers; `null` names one to pass as NULL, `align` one to
    misalign by 2 bytes."""
    p = {k: 0x7F0000100000 + 0x10000 * i for i, k in enumerate(("keyframe", "frame0", "frame1", "proj", "invd", "range", "out"))}
    if align is not None:
        p[align] += 2
    p = {k: ctypes.c_void_p(v) for k, v in p.items()}
    if null is not None:
        p[null] = None
    frames = (ctypes.c_void_p * 2)(p["frame0"], p["frame1"])
    a = dict(B=1, F=2, C=3, H=32, W=48)
    a.update(over)
    return lib.mr_residual_image(p["keyframe"], None if null == "frames" else frames, p["proj"], p["invd"], p["range"],
                                 a["B"], a["F"], a["C"], a["H"], a["W"], p["out"], None)


@pytest.mark.parametrize("null", ["keyframe", "frames", "frame1", "proj", "invd", "out"])
def test_entry_rejects_null_pointers(null):
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _entry(lib, null=null) == -1
    assert b"null" in lib.mr_last_error()


@pytest.mark.parametrize("align", ["keyframe", "frame0", "proj", "invd", "range", "out"])
def test_entry_rejects_misaligned_pointers(align):
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _entry(lib, align=align) == -1
    assert b"aligned" in lib.mr_last_error()


@pytest.mark.parametrize("over,text", [(dict(F=0), b"F"), (dict(F=9), b"F"), (dict(C=2), b"channels"), (dict(C=0), b"channels"),
                                       (dict(C=4), b"channels"), (dict(H=1), b"size"), (dict(W=1), b"size"),
                                       (dict(B=0), b"batch")])
def test_entry_checks_sizes(over, text):
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _entry(lib, **over) == -1
    msg = lib.mr_last_error()
    assert text in msg and b"mr_residual_image" in msg, msg


def test_layers_refuse_cpu_tensors():
    from monorec_b200 import _lib
    from monorec_b200 import ResidualImage, ResidualImageModule
    d = RC.inputs("synth")
    invd = RC.inverse_depth("synth")
    with pytest.raises(_lib.MonorecLibraryError):
        ResidualImage()(d["keyframe"], d["keyframe_pose"], d["keyframe_intrinsics"], invd, d["frames"], d["poses"],
                        d["intrinsics"])
    with pytest.raises(_lib.MonorecLibraryError):
        ResidualImageModule()(dict(d, predicted_inverse_depths=[invd], inv_depth_max=0, inv_depth_min=1))


def test_sequence_refuses_residual_image_for_a_mask_only_model():
    from monorec_b200.sequence import MonoRecSequence

    class _MaskOnly:
        use_stereo, pretrain_mode = False, 2

    with pytest.raises(NotImplementedError):
        MonoRecSequence(_MaskOnly(), device="cpu", residual_image=True)
    assert MonoRecSequence(_MaskOnly(), device="cpu").residual_image is False
