"""MonoRecSequence (monorec_b200/sequence.py): key frames of a frame stream run in batches from a device ring, and the
sequence's point-cloud export (SequencePointCloud, mr_pointcloud_add_windows).

CPU: the neighbour offsets, the bookkeeping with a fake model, the argument checks of the new C entry.  GPU: every key frame's
outputs against an eager forward of a batch dict built by hand, and the batched point cloud against the per-key-frame
MaskVoter + PLYSaver loop of create_pointcloud.py."""
import ctypes

import pytest
import torch

from monorec_b200.sequence import MonoRecSequence, neighbour_offsets

DEV = "cuda:0"
gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dilation", [1, 2, 3])
@pytest.mark.parametrize("frame_count", [1, 2, 3, 4, 5, 6])
def test_neighbour_offsets_follow_the_loader(frame_count, dilation):
    """The loader (kitti_odometry_dataset.py:253-258) takes frame_count // 2 frames before the key frame and the rest after
    it, `dilation` apart, in increasing order."""
    before = [-k * dilation for k in range(frame_count // 2, 0, -1)]
    after = [k * dilation for k in range(1, (frame_count + 1) // 2 + 1)]
    assert neighbour_offsets(frame_count, dilation) == before + after
    assert len(neighbour_offsets(frame_count, dilation)) == frame_count


def test_neighbour_offsets_examples():
    assert neighbour_offsets(1) == [1]
    assert neighbour_offsets(2) == [-1, 1]
    assert neighbour_offsets(3) == [-1, 1, 2]
    assert neighbour_offsets(4, 2) == [-4, -2, 2, 4]
    with pytest.raises(ValueError):
        neighbour_offsets(0)
    with pytest.raises(ValueError):
        neighbour_offsets(2, 0)


class _FakeModel:
    """Adds outputs that name the frames the batch was built from: frame n's image is filled with n, its pose translates
    by n in x and its intrinsics hold n in K[0,2]; cost_volume channel f is source frame f's value."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self):
        self.batch_sizes = []

    def __call__(self, data):
        self.batch_sizes.append(data["keyframe"].shape[0])
        data["result"] = data["keyframe"][:, :1] * 1.0
        data["cv_mask"] = data["keyframe_pose"][:, 0, 3].view(-1, 1, 1, 1).expand_as(data["result"]) * 1.0
        data["cost_volume"] = torch.cat([f[:, :1] for f in data["frames"]], 1)
        sources = torch.stack([torch.stack([p[:, 0, 3], k[:, 0, 2]], 1) for p, k in zip(data["poses"], data["intrinsics"])], 1)
        data["predicted_inverse_depths"] = [data["result"] + s for s in range(4)] + [sources]
        return data


def _frame(n, H=4, W=6):
    pose, K = torch.eye(4), torch.eye(4)
    pose[0, 3], K[0, 2] = float(n), float(n)
    return torch.full((3, H, W), float(n)), pose, K


@pytest.mark.parametrize("n_frames", [1, 2, 3, 5, 9, 10, 17, 40, 61])
@pytest.mark.parametrize("frame_count,dilation,batch_size", [(2, 1, 8), (1, 1, 3), (4, 2, 4), (3, 1, 1), (5, 3, 2)])
def test_bookkeeping_with_a_fake_model(frame_count, dilation, batch_size, n_frames):
    """Emitted indices, their order, the batch boundaries, the flush tail and the ring wrap-around, for sequences from
    shorter than one window to several rings."""
    model = _FakeModel()
    seq = MonoRecSequence(model, frame_count, dilation, batch_size, graphed=False, device="cpu")
    offs = neighbour_offsets(frame_count, dilation)
    lo, hi = min(0, min(offs)), max(offs)
    assert seq.ring_len == hi - lo + 1 + batch_size
    expected = list(range(-lo, n_frames - hi))              # the loader's index range: key frames with every neighbour
    got, calls = [], []
    for n in range(n_frames):
        out = seq.push(*_frame(n))
        if out:
            calls.append((n, [i for i, _ in out]))
        got += out
    tail = seq.flush()
    got += tail
    assert [i for i, _ in got] == expected
    # a batch runs at the push of its last key frame's last neighbour; the flush runs the rest
    full = len(expected) // batch_size
    assert calls == [(expected[(b + 1) * batch_size - 1] + hi, expected[b * batch_size:(b + 1) * batch_size])
                     for b in range(full)]
    assert [i for i, _ in tail] == expected[full * batch_size:]
    assert model.batch_sizes == [batch_size] * full + ([len(expected) % batch_size] if len(expected) % batch_size else [])
    assert seq.flush() == []
    for i, o in got:
        assert o["result"].shape == (1, 1, 4, 6) and bool((o["result"] == i).all())
        assert bool((o["cv_mask"] == i).all()) and float(o["keyframe_pose"][0, 0, 3]) == i
        assert float(o["keyframe_intrinsics"][0, 0, 2]) == i and bool((o["keyframe"] == i).all())
        assert [float(o["cost_volume"][0, f, 0, 0]) for f in range(len(offs))] == [i + d for d in offs]
        assert o["predicted_inverse_depths"][4][0].tolist() == [[i + d, i + d] for d in offs]


def test_unsupported_configurations_raise():
    for attrs in ({"use_stereo": True}, {"pretrain_mode": 3}):
        model = _FakeModel()
        for k, v in attrs.items():
            setattr(model, k, v)
        with pytest.raises(NotImplementedError):
            MonoRecSequence(model, device="cpu")
    seq = MonoRecSequence(_FakeModel(), graphed=False, device="cpu")
    with pytest.raises(ValueError):
        seq.push(torch.zeros(1, 3, 4, 6), torch.eye(4), torch.eye(4))
    seq.push(*_frame(0))
    with pytest.raises(ValueError):
        seq.push(*_frame(1, H=5))


def _add_windows(lib, B=2, H=8, W=8, ring_len=6, starts=(0, 5), n_masks=5, min_hits=1, null=None, ws_bytes=1 << 20):
    p = {k: ctypes.c_void_p(0x1000) for k in ("inv_depth", "keyframe", "K", "pose", "keep_ring", "vertices", "n_after",
                                               "workspace")}
    if null in p:
        p[null] = None
    win = None if null == "window_start" else (ctypes.c_int * max(len(starts), 1))(*starts)
    return lib.mr_pointcloud_add_windows(p["inv_depth"], p["keyframe"], p["K"], p["pose"], p["keep_ring"], ring_len, win,
                                         n_masks, min_hits, B, H, W, 3.0, 20.0, None, None, 0.0, p["vertices"], 1 << 20, 0,
                                         p["n_after"], p["workspace"], ws_bytes, None)


@pytest.mark.parametrize("case,field", [
    (dict(null="inv_depth"), b"inv_depth"), (dict(null="keyframe"), b"keyframe"), (dict(null="K"), b"null pointer K"),
    (dict(null="pose"), b"pose"), (dict(null="keep_ring"), b"keep_ring"), (dict(null="window_start"), b"window_start"),
    (dict(null="vertices"), b"vertices"), (dict(null="n_after"), b"n_after"), (dict(null="workspace"), b"workspace"),
    (dict(B=0, starts=()), b"B = 0"), (dict(B=-3, starts=()), b"B = -3"), (dict(B=257, starts=(0,) * 257), b"B = 257"),
    (dict(n_masks=0), b"n_masks = 0"), (dict(n_masks=-1), b"n_masks = -1"), (dict(n_masks=7), b"n_masks = 7"),
    (dict(min_hits=0), b"min_hits = 0"), (dict(min_hits=6), b"min_hits = 6"), (dict(min_hits=-2), b"min_hits = -2"),
    (dict(starts=(0, 6)), b"window_start[1] = 6"), (dict(starts=(-1, 0)), b"window_start[0] = -1"),
    (dict(ring_len=0, starts=(0, 0), n_masks=1), b"ring_len = 0"), (dict(H=0), b"H = 0"),
], ids=lambda v: v.decode() if isinstance(v, bytes) else None)
def test_add_windows_rejects_bad_arguments_without_a_gpu(case, field):
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _add_windows(lib, **case) == -1                   # MR_EINVAL, before any CUDA call
    msg = lib.mr_last_error()
    assert msg.startswith(b"mr_pointcloud_add_windows") and field in msg, msg


def test_add_windows_workspace_too_small_without_a_gpu():
    from monorec_b200 import _lib
    lib = _lib.load()
    assert _add_windows(lib, ws_bytes=4) == -3               # MR_ENOMEM
    assert b"workspace too small" in lib.mr_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    """A seeded MonoRecModel on cuda:0."""
    import monorec_b200.model as M
    from monorec_b200.synthetic import seeded_state_dict
    m = M.MonoRecModel()
    m.load_state_dict(seeded_state_dict(m, seed=7, gain=0.7))
    return m.to(DEV).eval()


@pytest.fixture(params=["fp32", "tf32", "f16"])
def mode(request):
    from monorec_b200 import conv as C
    saved = C.MODE
    C.set_mode(request.param)
    yield request.param
    C.set_mode(saved)


def _by_hand(images, poses, Ks, indices, offsets):
    """The reference loader's dict for these key frames, collated (kitti_odometry_dataset.py:248-269), on cuda:0."""
    rows = lambda t, d: torch.stack([t[i + d] for i in indices]).to(DEV)              # noqa: E731
    return {"keyframe": rows(images, 0), "keyframe_pose": rows(poses, 0), "keyframe_intrinsics": rows(Ks, 0),
            "frames": [rows(images, d) for d in offsets], "poses": [rows(poses, d) for d in offsets],
            "intrinsics": [rows(Ks, d) for d in offsets]}


@gpu
@pytest.mark.parametrize("graphed", [True, False], ids=["graphed", "eager"])
@pytest.mark.parametrize("frame_count,dilation,batch_size", [(2, 1, 8), (4, 2, 4)], ids=["F2", "F4d2"])
@pytest.mark.parametrize("size", [(64, 128), (256, 512)], ids=["64x128", "256x512"])
def test_outputs_equal_an_eager_forward_of_the_batch(model, mode, size, frame_count, dilation, batch_size, graphed):
    """23 frames: every key frame's result, cv_mask, four inverse depths and cost volume equal, bit for bit, the same row of
    an eager forward of the batch's dict built by hand from the same frames (partial final batch included)."""
    from monorec_b200.synthetic import make_sequence
    H, W = size
    images, poses, Ks = make_sequence(23, H, W, seed=3)
    seq = MonoRecSequence(model, frame_count, dilation, batch_size, graphed=graphed)
    offs = neighbour_offsets(frame_count, dilation)
    seen = []

    def check(emitted):
        if not emitted:
            return
        indices = [i for i, _ in emitted]
        with torch.no_grad():
            ref = model(_by_hand(images, poses, Ks, indices, offs))
        for j, (i, o) in enumerate(emitted):
            for k in ("result", "cv_mask", "cost_volume"):
                assert torch.equal(o[k], ref[k][j:j + 1]), (i, k)
            assert len(o["predicted_inverse_depths"]) == 4
            for s in range(4):
                assert torch.equal(o["predicted_inverse_depths"][s], ref["predicted_inverse_depths"][s][j:j + 1]), (i, s)
        seen.extend(indices)
    with torch.no_grad():
        for n in range(23):
            check(seq.push(images[n], poses[n], Ks[n]))         # compared before the next push replays the graph
        tail = seq.flush()
        assert 0 < len(tail) < batch_size
        check(tail)
    assert seen == list(range(-min(offs), 23 - max(offs)))


class _MovingObject(torch.nn.Module):
    """A seeded MonoRecModel whose cv_mask is replaced by a 40x40 block that moves 12 px right per frame (the sequence index
    is read back from the pose's z translation), so that the 5-frame vote removes a different region per key frame."""
    use_stereo, pretrain_mode = False, 0

    def __init__(self, model, step):
        super().__init__()
        self.model, self.step = model, step

    def forward(self, data):
        data = self.model(data)
        B, _, H, W = data["result"].shape
        n = torch.round(data["keyframe_pose"][:, 2, 3] / self.step).view(B, 1, 1, 1)
        y = torch.arange(H, device=n.device).view(1, 1, H, 1)
        x = torch.arange(W, device=n.device).view(1, 1, 1, W)
        data["cv_mask"] = (((y - 120).abs() < 20) & ((x - 60 - 12 * n).abs() < 20)).to(torch.float32)
        return data


@gpu
@pytest.mark.parametrize("moving", [False, True], ids=["no_moving_object", "moving_object"])
def test_sequence_pointcloud_equals_the_per_keyframe_loop(moving):
    """create_pointcloud.py's settings (configs/test/pointcloud_monorec.json: roi, max_d 20, dropout 0.75, 5-frame vote):
    sequence_pointcloud at B 4 gives exactly the vertices, in the same order, of MaskVoter + PLYSaver.add_depthmap called
    once per key frame on the same outputs with the same dropout numbers.  The model is seeded, without its MaskModule
    (pretrain_mode 1: cv_mask is zero), and its inverse-depth range keeps every depth inside [3, 20] m."""
    import monorec_b200.model as M
    from monorec_b200 import pointcloud as PC
    from monorec_b200.synthetic import make_sequence, seeded_state_dict
    H, W, N = 256, 512, 23
    roi = [40, 256, 48, 464]
    model = M.MonoRecModel(pretrain_mode=1, inv_depth_min_max=(0.33, 0.06))
    model.load_state_dict(seeded_state_dict(model, seed=7, gain=0.7))
    model = model.to(DEV).eval()
    images, poses, Ks = make_sequence(N, H, W, seed=5)
    if moving:
        model = _MovingObject(model, step=float(poses[1, 2, 3]))
    gen = torch.Generator().manual_seed(9)
    rand = torch.rand(N, 1, H, W, generator=gen)
    seq = MonoRecSequence(model, frame_count=2, batch_size=4, graphed=True)
    saver = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=roi, dropout=0.75)
    pc = PC.sequence_pointcloud(seq, saver)
    outputs = []
    with torch.no_grad():
        for n in range(N):
            outputs += [(i, {k: (v.clone() if torch.is_tensor(v) else v) for k, v in o.items()})
                        for i, o in pc.push(images[n], poses[n], Ks[n], rand=rand[n])]
        outputs += pc.flush()
    assert [i for i, _ in outputs] == list(range(1, N - 1))
    assert all(bool(o["cv_mask"].any()) == moving for _, o in outputs)
    ref = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=roi, dropout=0.75)
    voter = PC.MaskVoter(buffer_length=5, min_hits=1, mask_fill=32)
    for p, (i, o) in enumerate(outputs):
        key = voter.push(o, o)
        if key is not None:
            ref.add_depthmap(key["depth"], key["keyframe"], key["intrinsics"], key["pose"], keep_masks=key["keep_masks"],
                             min_hits=key["min_hits"], rand=rand[outputs[p - 2][0]].unsqueeze(0).to(DEV))
    n = len(ref)
    # 17 voted key frames, a quarter of each roi pixel survives the dropout
    assert n > 17 * 0.2 * (216 * 416) * (0.8 if moving else 1) and len(saver) == n
    assert torch.equal(saver.vertices, ref.vertices)
