"""Grayscale frame streams ([.., 1, H, W], the KITTI loader's use_color=False and TUM Mono-VO) without a GPU: the
MonoRecSequence rings and push checks with a fake model, the channel checks of CostVolumeModule and the argument checks of
mr_cost_volume_fwd_channels (made before any CUDA call)."""
import ctypes

import pytest
import torch

from monorec_b200.sequence import MonoRecSequence, neighbour_offsets


class _FakeModel:
    """Records the batch dicts' image shapes and returns the keyframe's first plane as `result`."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self):
        self.shapes = []

    def __call__(self, data):
        self.shapes.append({k: tuple(data[k].shape) for k in ("keyframe", "stereoframe") if k in data})
        self.shapes[-1]["frames"] = [tuple(f.shape) for f in data["frames"]]
        data["result"] = data["keyframe"][:, :1] * 1.0
        return data


def _frame(n, C, H=4, W=6):
    pose, K = torch.eye(4), torch.eye(4)
    pose[0, 3], K[0, 2] = float(n), float(n)
    return torch.full((C, H, W), float(n)), pose, K


@pytest.mark.parametrize("stereo", [False, True])
def test_gray_sequence_rings_and_batches(stereo):
    """use_color=False: one-plane rings, [1,H,W] images (and stereo images) in, the same key frames and batches as a colour
    sequence, and every key frame's keyframe / stereoframe are its own one-channel images."""
    model = _FakeModel()
    model.use_stereo = stereo
    seq = MonoRecSequence(model, 2, 1, 3, graphed=False, device="cpu", stereo=stereo, use_color=False)
    ref = MonoRecSequence(_FakeModel(), 2, 1, 3, graphed=False, device="cpu")
    got, want = [], []
    for n in range(11):
        kw = {"stereo": _frame(100 + n, 1)} if stereo else {}
        got += seq.push(*_frame(n, 1), **kw)
        want += ref.push(*_frame(n, 3))
        if n == 0:
            assert tuple(seq._rings[0].shape[1:]) == (1, 4, 6)
            assert all(seq._maps[k].shape[1] == 1 for k in seq._maps if k == "stereoframe")
    got += seq.flush()
    want += ref.flush()
    assert [i for i, _ in got] == [i for i, _ in want] == list(range(1, 10))
    for i, o in got:
        assert tuple(o["keyframe"].shape) == (1, 1, 4, 6) and bool((o["keyframe"] == i).all())
        if stereo:
            assert tuple(o["stereoframe"].shape) == (1, 1, 4, 6) and bool((o["stereoframe"] == 100 + i).all())
    for s in model.shapes:
        assert s["keyframe"][1] == 1 and all(f[1] == 1 for f in s["frames"])
        assert not stereo or s["stereoframe"][1] == 1


def test_channel_count_of_push_follows_use_color():
    gray = MonoRecSequence(_FakeModel(), graphed=False, device="cpu", use_color=False)
    color = MonoRecSequence(_FakeModel(), graphed=False, device="cpu")
    assert color.use_color and not gray.use_color
    with pytest.raises(ValueError):
        gray.push(*_frame(0, 3))
    with pytest.raises(ValueError):
        color.push(*_frame(0, 1))
    gray.push(*_frame(0, 1))
    color.push(*_frame(0, 3))
    m = _FakeModel()
    m.use_stereo = True
    st = MonoRecSequence(m, graphed=False, device="cpu", stereo=True, use_color=False)
    with pytest.raises(ValueError):
        st.push(*_frame(0, 1), stereo=_frame(0, 3))
    st.push(*_frame(0, 1), stereo=_frame(0, 1))
    assert neighbour_offsets(2) == st.offsets


def _cv_dict(C_key, C_frames):
    B, H, W = 1, 16, 20
    return {"keyframe": torch.zeros(B, C_key, H, W), "frames": [torch.zeros(B, c, H, W) for c in C_frames],
            "poses": [torch.eye(4).expand(B, 4, 4)] * len(C_frames), "intrinsics": [torch.eye(4).expand(B, 4, 4)] * len(C_frames),
            "keyframe_pose": torch.eye(4).expand(B, 4, 4), "keyframe_intrinsics": torch.eye(4).expand(B, 4, 4),
            "stereoframe": torch.zeros(B, C_frames[0], H, W), "stereoframe_pose": torch.eye(4).expand(B, 4, 4),
            "stereoframe_intrinsics": torch.eye(4).expand(B, 4, 4)}


def test_cost_volume_channel_checks():
    """C = 2 (or any C but 1 and 3) is NotImplementedError; a mono or stereo frame whose C differs from the keyframe's is a
    ValueError.  Both are raised before anything touches a device."""
    from monorec_b200.cost_volume import CostVolumeModule, check_channels
    with pytest.raises(NotImplementedError):
        CostVolumeModule()(_cv_dict(2, [2, 2]))
    with pytest.raises(NotImplementedError):
        CostVolumeModule()(_cv_dict(4, [4]))
    with pytest.raises(ValueError):
        CostVolumeModule()(_cv_dict(1, [1, 3]))
    with pytest.raises(ValueError):
        CostVolumeModule()(_cv_dict(3, [1, 1]))
    d = _cv_dict(1, [1, 1])
    d["stereoframe"] = torch.zeros(1, 3, 16, 20)
    with pytest.raises(ValueError):
        CostVolumeModule(use_stereo=True)(d)
    CostVolumeModule(use_mono=False, use_stereo=True)           # (constructs; the stereo frame alone must agree too)
    with pytest.raises(ValueError):
        CostVolumeModule(use_mono=False, use_stereo=True)(d)
    assert check_channels(torch.zeros(1, 1, 8, 8), [torch.zeros(1, 1, 8, 8)]) == 1
    assert check_channels(torch.zeros(1, 3, 8, 8), [torch.zeros(1, 3, 8, 8)] * 2) == 3


def _channels_entry(lib, channels=1, null=None, **over):
    """mr_cost_volume_fwd_channels on fake (never dereferenced) 16-byte-aligned pointers; `null` names one to pass as NULL."""
    p = {k: ctypes.c_void_p(0x7F0000100000 + 0x10000 * i) for i, k in
         enumerate(("keyframe", "frame0", "frame1", "proj", "depths", "cv", "sfcv"))}
    if null is not None:
        p[null] = None
    frames = (ctypes.c_void_p * 2)(p["frame0"], p["frame1"])
    a = dict(B=1, F=2, D=32, H=64, W=128, matching=1, centered=1, out_dtype=0)
    a.update(over)
    return lib.mr_cost_volume_fwd_channels(p["keyframe"], frames, p["proj"], p["depths"], None, p["cv"], p["sfcv"], None, 0,
                                           a["B"], a["F"], a["D"], a["H"], a["W"], 10.0, None, a["matching"], a["centered"],
                                           a["out_dtype"], channels, None)


@pytest.mark.parametrize("channels", [0, 2, 4, -1, 9])
def test_channels_entry_rejects_other_channel_counts(channels):
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _channels_entry(lib, channels) == -1
    assert b"channels must be 1 or 3" in lib.mr_last_error()


@pytest.mark.parametrize("null", ["keyframe", "frame1", "proj", "depths", "cv", "sfcv"])
@pytest.mark.parametrize("channels", [1, 3])
def test_channels_entry_rejects_null_pointers(null, channels):
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _channels_entry(lib, channels, null=null) == -1
    msg = lib.mr_last_error()
    assert b"null" in msg or b"non-null" in msg or b"exactly one of depths" in msg, msg


def test_channels_entry_checks_the_other_arguments_as_the_typed_entry():
    from monorec_b200 import _lib
    lib = _lib.load()
    for over, text in ((dict(D=1), b"D"), (dict(F=9), b"F"), (dict(matching=5), b"matching"), (dict(centered=2), b"centered"),
                       (dict(out_dtype=3), b"out_dtype")):
        assert _channels_entry(lib, 1, **over) == -1
        assert text in lib.mr_last_error() and b"mr_cost_volume_fwd_channels" in lib.mr_last_error()
    assert _channels_entry(lib, 1, matching=0) == -2          # use_ssim falsy: not implemented, as in the typed entry
