"""The reference's other frame layouts over a frame stream on the GPU: KITTI with offset_d (a causal stream whose key frame
is one of its own source frames) and max_length, TUM Mono-VO and Oxford RobotCar.  MonoRecSequence, SequenceEvaluater,
MultiModelEvaluater and the point-cloud export against eager MonoRecModel forwards of the loader's dicts, the lanes against
one device, no host synchronisation after the capture, and the cost-volume kernel with the key frame as its own source
frame (one device tensor read twice) against the float64 closed form at tests/test_cv_accuracy_gpu.py's gates.

Seeded MonoRecModels at 64x128, sequence batch 4."""
import io

import numpy as np
import pytest
import torch

from tests import test_cv_accuracy_gpu as A

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 64, 128
BATCH = 4
N_FRAMES = 21
NAMES = ["abs_rel_sparse_metric", "rmse_sparse_metric", "a1_sparse_metric", "abs_rel_metric", "sc_inv_metric"]
EVAL_KW = dict(roi=[4, 60, 8, 120], max_distance=80)


def _layout(name, n):
    from monorec_b200 import sequence as S
    if name == "kitti_causal":
        return S.kitti_layout(n, 2, 1, offset_d=-1, drop_outside=True)                 # sources k-2, k
    if name == "kitti_shifted":
        masks = [{str(i): i % 5 != 3 for i in range(n)}]
        return S.kitti_layout(n, 2, 2, offset_d=1, max_length=12, index_masks=masks, drop_outside=True)
    if name == "tum":
        return S.tum_mono_vo_layout(n, 3, 1)                                          # sources k-1, k+1, k+2
    if name == "tum_keyframes":
        return S.tum_mono_vo_layout(n, 2, 2, keyframe_indices=[0, 2, 3, 5, 8, 9, 10, 13, 15, 16, 19])
    if name == "robotcar":
        return S.robotcar_layout(n, 3, 1, drop_outside=True)                          # sources k-2, k-1, k+1, k+2
    raise KeyError(name)


LAYOUTS = ["kitti_causal", "kitti_shifted", "tum", "tum_keyframes", "robotcar"]


def _model(seed=7, **kw):
    import monorec_b200.model as MM
    from monorec_b200.synthetic import seeded_state_dict
    m = MM.MonoRecModel(**kw)
    m.load_state_dict(seeded_state_dict(m, seed=seed, gain=0.7))
    return m.to(DEV).eval()


def _pc_model():
    """A point-cloud model whose every depth lies inside [3, 20] m (the exports' min_d / max_d)."""
    return _model(pretrain_mode=1, inv_depth_min_max=(0.33, 0.06))


def _stream(n, seed):
    from monorec_b200.synthetic import make_sequence
    images, poses, Ks = make_sequence(n, H, W, seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    target = torch.rand(n, 1, H, W, generator=g) * 0.2 + 0.01
    target[torch.rand(n, 1, H, W, generator=g) > 0.25] = 0.0
    rand = torch.rand(n, 1, H, W, generator=g)
    return dict(images=images, poses=poses, Ks=Ks, target=target, rand=rand)


def _loader_dict(st, keys, offsets, alias=True):
    """The loader's collated dict of these key frames, the sources in the layout's order.  With `alias`, a source at offset
    0 is the key frame's own device tensor; without, a second copy (the loader reads the frame twice)."""
    rows = lambda t, d: torch.stack([t[i + d] for i in keys]).to(DEV)              # noqa: E731
    data = {"keyframe": rows(st["images"], 0), "keyframe_pose": rows(st["poses"], 0), "keyframe_intrinsics": rows(st["Ks"], 0)}
    for key, own, src in (("frames", "keyframe", "images"), ("poses", "keyframe_pose", "poses"),
                          ("intrinsics", "keyframe_intrinsics", "Ks")):
        data[key] = [data[own] if d == 0 and alias else rows(st[src], d) for d in offsets]
    return data


def _drive(runner, st, n, **kw):
    """Pushes frames 0 .. n-1 (skipping those no key frame needs) and flushes; returns the emitted batches as index
    lists."""
    batches = []

    def take(emitted):
        if emitted:
            batches.append([i for i, _ in emitted])
    seq = runner.seq
    for f in range(n):
        if not seq.needs(f):
            runner.skip()
            continue
        extra = {k: st[v][f] for k, v in kw.items()}
        take(runner.push(st["images"][f], st["poses"][f], st["Ks"][f], **extra))
    take(runner.flush())
    return batches


@pytest.mark.parametrize("name", LAYOUTS)
def test_sequence_outputs_equal_forwards_of_the_loader_dicts(name):
    """Every key frame (graph replay, and the short last batch eager) equals, bit for bit, its row of an eager forward of
    the loader's dict of the same batch, with the key frame passed once or twice as a source; the batches are the layout's
    key frames four at a time; after the capture, push makes no host synchronisation."""
    from monorec_b200.sequence import MonoRecSequence
    model = _model()
    lay = _layout(name, N_FRAMES)
    st = _stream(N_FRAMES, seed=3)
    dev = {k: st[k].to(DEV) for k in ("images", "poses", "Ks")}
    seq = MonoRecSequence(model, batch_size=BATCH, layout=lay)
    batches, rows = [], {}
    with torch.no_grad():
        for f in range(N_FRAMES):
            if not seq.needs(f):
                seq.skip()
                continue
            captured = seq._graph is not None
            if captured:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
            try:
                emitted = seq.push(dev["images"][f], dev["poses"][f], dev["Ks"][f])
                if emitted:
                    batches.append([i for i, _ in emitted])
                    for i, o in emitted:
                        rows[i] = {k: o[k].clone() for k in ("result", "cv_mask", "cost_volume")}
                        rows[i]["pid"] = [p.clone() for p in o["predicted_inverse_depths"]]
            finally:
                torch.cuda.set_sync_debug_mode(0)
        assert seq.flush() == []
        assert seq._graph is not None
        assert [i for b in batches for i in b] == list(lay.keys)
        assert [len(b) for b in batches] == [len(c) for c in (lay.keys[j:j + BATCH] for j in range(0, len(lay.keys), BATCH))]
        aliased = 0 in lay.offsets
        for b in batches:
            for alias in ((True, False) if aliased else (True,)):
                ref = model(_loader_dict(st, b, lay.offsets, alias))
                for j, i in enumerate(b):
                    for k in ("result", "cv_mask", "cost_volume"):
                        assert torch.equal(rows[i][k], ref[k][j:j + 1]), (name, i, k, alias)
                    for s in range(4):
                        assert torch.equal(rows[i]["pid"][s], ref["predicted_inverse_depths"][s][j:j + 1]), (name, i, s)


def _fold(model, st, batches, lay, bs):
    """The evaluater's device fold (SequenceEvaluater.add, no sequence) of the eager forwards of the loader's dicts, added
    batch by batch as the sequence emits them."""
    from monorec_b200.evaluation import SequenceEvaluater
    ev = SequenceEvaluater(None, NAMES, bs, **EVAL_KW)
    with torch.no_grad():
        for c in batches:
            ev.add(model(_loader_dict(st, c, lay.offsets))["result"], torch.cat([st["target"][i:i + 1] for i in c]).to(DEV))
    ev.flush()
    return ev.log()


def _bits(log):
    return {k: np.asarray(log[k], np.float64).view(np.uint64).tolist() for k in ("metrics", "metrics_correct")}, \
        log["valid_batches"]


@pytest.mark.parametrize("name", ["kitti_causal", "tum", "robotcar"])
def test_evaluater_logs_equal_the_fold_of_eager_forwards(name):
    """SequenceEvaluater and MultiModelEvaluater (two models on one trunk) over a layout: every log equals, bit for bit, the
    evaluater's fold of the eager forwards' results in the sequence's batches."""
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.models_eval import MultiModelEvaluater
    from monorec_b200.sequence import MonoRecSequence
    a, b = _model(7), _model(8)
    b._feature_extractor.load_state_dict(a._feature_extractor.state_dict())
    lay = _layout(name, N_FRAMES)
    st = _stream(N_FRAMES, seed=4)
    with torch.no_grad():
        ev = SequenceEvaluater(MonoRecSequence(a, batch_size=BATCH, layout=lay), NAMES, 3, **EVAL_KW)
        batches = _drive(ev, st, N_FRAMES, target="target")
        mm = MultiModelEvaluater([a, b], NAMES, 3, seq_batch=BATCH, layout=lay, **EVAL_KW)
        mm_batches = _drive(mm, st, N_FRAMES, target="target")
    assert batches == mm_batches and [i for c in batches for i in c] == list(lay.keys)
    ref_a, ref_b = _fold(a, st, batches, lay, 3), _fold(b, st, batches, lay, 3)
    assert ref_a["valid_batches"] > 0
    assert _bits(ev.log()) == _bits(ref_a)
    logs = mm.logs()
    assert _bits(logs[0]) == _bits(ref_a) and _bits(logs[1]) == _bits(ref_b)


@pytest.mark.parametrize("name", ["kitti_causal", "tum_keyframes", "robotcar"])
def test_point_cloud_equals_the_reference_loop_on_eager_forwards(name):
    """sequence_pointcloud over a layout writes, byte for byte, the PLY of create_pointcloud.py's loop (MaskVoter, then
    PLYSaver.add_depthmap per key frame) over the eager forwards' rows."""
    from monorec_b200 import pointcloud as PC
    from monorec_b200.sequence import MonoRecSequence
    model = _pc_model()
    lay = _layout(name, N_FRAMES)
    st = _stream(N_FRAMES, seed=5)
    saver = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=[8, 64, 8, 120], dropout=0.5)
    with torch.no_grad():
        pc = PC.sequence_pointcloud(MonoRecSequence(model, batch_size=BATCH, layout=lay), saver)
        batches = _drive(pc, st, N_FRAMES, rand="rand")
        ref = PC.PLYSaver(H, W, min_d=3, max_d=20, roi=[8, 64, 8, 120], dropout=0.5)
        voter = PC.MaskVoter(buffer_length=5)
        keys = [i for c in batches for i in c]
        for c in batches:
            data = _loader_dict(st, c, lay.offsets)
            out = model(dict(data))
            for j, i in enumerate(c):
                row = {k: out[k][j:j + 1] for k in ("result", "cv_mask")}
                v = voter.push(row, {k: data[k][j:j + 1] for k in ("keyframe", "keyframe_pose", "keyframe_intrinsics")})
                if v is not None:
                    k = keys[keys.index(i) - 2]
                    ref.add_depthmap(v["depth"], v["keyframe"], v["intrinsics"], v["pose"], keep_masks=v["keep_masks"],
                                     min_hits=v["min_hits"], rand=st["rand"][k].reshape(1, 1, H, W).to(DEV))
    assert len(ref) > 1000
    got, want = io.BytesIO(), io.BytesIO()
    saver.save(got)
    ref.save(want)
    assert got.getvalue() == want.getvalue()


@pytest.mark.parametrize("name", ["kitti_causal", "robotcar"])
def test_lanes_on_one_device_equal_one_device(name):
    """Lanes [0, 0] over two sequences with their own layouts: MultiDeviceEvaluater, MultiDeviceModelsEvaluater and
    MultiDevicePointCloud give the one-device logs and PLY bit for bit."""
    from monorec_b200 import pointcloud as PC
    from monorec_b200.evaluation import SequenceEvaluater
    from monorec_b200.lanes import MultiDeviceEvaluater, MultiDeviceModelsEvaluater, MultiDevicePointCloud
    from monorec_b200.models_eval import MultiModelEvaluater
    from monorec_b200.sequence import MonoRecSequence
    a, b, pc_model = _model(7), _model(8), _pc_model()
    lengths = [19, 14]
    layouts = [_layout(name, n) for n in lengths]
    streams = [_stream(n, seed=10 + s) for s, n in enumerate(lengths)]

    def feed(runner):
        for s, f in runner.order:
            st = streams[s]
            yield s, f, st

    with torch.no_grad():
        ev = SequenceEvaluater(None, NAMES, 3, **EVAL_KW)
        mm = MultiModelEvaluater([a, b], NAMES, 3, seq_batch=BATCH, layout=layouts[0], **EVAL_KW)
        saver = PC.PLYSaver(H, W, min_d=3, max_d=20)
        for s, (n, lay, st) in enumerate(zip(lengths, layouts, streams)):
            ev.next_sequence(MonoRecSequence(a, batch_size=BATCH, layout=lay))
            if s:
                mm.next_sequence(layout=lay)
            pc = PC.sequence_pointcloud(MonoRecSequence(pc_model, batch_size=BATCH, layout=lay), saver)
            for runner in (ev, mm, pc):
                extra = {} if runner is pc else dict(target="target")
                for f in range(n):
                    if not runner.seq.needs(f):
                        runner.skip()
                        continue
                    runner.push(st["images"][f], st["poses"][f], st["Ks"][f], **{k: st[v][f] for k, v in extra.items()})
                if runner is pc:
                    pc.flush()
        ev.flush()
        mm.flush()
        ref_log, ref_logs = ev.log(), mm.logs()
        ref_ply = io.BytesIO()
        saver.save(ref_ply)

        lane_ev = MultiDeviceEvaluater(a, [0, 0], lengths, NAMES, 3, seq_batch=BATCH, layout=layouts, **EVAL_KW)
        lane_mm = MultiDeviceModelsEvaluater([a, b], [0, 0], lengths, NAMES, 3, seq_batch=BATCH, layout=layouts, **EVAL_KW)
        lane_pc = MultiDevicePointCloud(pc_model, [0, 0], lengths, H, W, seq_batch=BATCH, min_d=3, max_d=20, layout=layouts)
        for runner in (lane_ev, lane_mm):
            for s, f, st in feed(runner):
                runner.push(s, f, st["images"][f], st["poses"][f], st["Ks"][f], st["target"][f])
            runner.flush()
        for s, f, st in feed(lane_pc):
            lane_pc.push(s, f, st["images"][f], st["poses"][f], st["Ks"][f])
        lane_pc.flush()
    assert ref_log["valid_batches"] > 0
    assert _bits(lane_ev.log()) == _bits(ref_log)
    assert [_bits(x) for x in lane_mm.logs()] == [_bits(x) for x in ref_logs]
    ply = io.BytesIO()
    lane_pc.save(ply)
    assert len(ref_ply.getvalue()) > 10000 and ply.getvalue() == ref_ply.getvalue()


# ---- the key frame as its own source frame, against the float64 closed form ----------------------------------------------
# tag -> (entry, B, F, D, H, W, image seed, index of the source frame that is the key frame)
SELF_CASES = {"self_tma_f2": ("fwd", 1, 2, 32, 256, 512, 100, 1),
              "self_gather_f3": ("gather", 2, 3, 32, 96, 200, 55, 1)}


class _SelfCase(A._Case):
    """test_cv_accuracy_gpu's case with source frame `s` replaced by the key frame: its image is the key frame's own device
    tensor (one pointer passed twice) and its pose and intrinsics the key frame's (the identity relative pose)."""

    def __init__(self, tag):
        from monorec_b200 import _lib
        from monorec_b200.synthetic import make_inputs, to_device
        entry, B, F, D, H_, W_, seed, s = SELF_CASES[tag]
        self.tag, self.centred = tag, True
        data = make_inputs(B, F, H_, W_, seed=seed)
        data["frames"][s], data["poses"][s] = data["keyframe"], data["keyframe_pose"]
        data["intrinsics"][s] = data["keyframe_intrinsics"]
        lib = _lib.load()
        d = to_device(data, DEV)
        key = d["keyframe"].contiguous()
        d["frames"][s] = key                                         # the same device tensor, read twice
        stream = torch.cuda.current_stream().cuda_stream
        proj, planes = torch.empty(B, F, 3, 4, device=DEV), torch.empty(D, device=DEV)
        _lib.check(lib.mr_projection_tables(d["keyframe_pose"].data_ptr(), d["keyframe_intrinsics"].data_ptr(),
                                            _lib.ptr_array(d["poses"]), _lib.ptr_array(d["intrinsics"]), B, F, H_, W_,
                                            proj.data_ptr(), planes.data_ptr(), D, 0.0025, 0.33, stream),
                   "mr_projection_tables")
        cv = torch.full((B, D, H_, W_), float("nan"), device=DEV)
        sf = torch.full((F, B, D, H_, W_), float("nan"), device=DEV)
        fn = lib.mr_cost_volume_fwd if entry == "fwd" else lib.mr_cost_volume_fwd_gather
        _lib.check(fn(key.data_ptr(), _lib.ptr_array(d["frames"]), proj.data_ptr(), planes.data_ptr(), cv.data_ptr(),
                      sf.data_ptr(), B, F, D, H_, W_, A.O.ALPHA, None, stream), entry)
        torch.cuda.synchronize()
        self.cv, self.sf = cv.cpu().numpy(), sf.cpu().numpy()
        z = planes.cpu().view(1, D, 1, 1).expand(B, D, H_, W_)
        ref_cv, ref_sf, self.valid, sad = A.O.cost_volume_closed_form(data, cv_depths=z, dtype=np.float64, use_ssim=True,
                                                                    not_center_cv=False)
        self.ref_cv, self.ref_sf, self.sad = ref_cv, np.stack(ref_sf), sad
        self.margin = A.O.validity_margin(data, cv_depths=z)
        spread = np.exp(-A.O.ALPHA * (sad - sad.min(axis=2, keepdims=True)) ** 2).sum(axis=2)
        self.w = (1 - (spread - 1) / (D - 1)) * self.valid
        self.kvalid = np.moveaxis(~(self.sf == 0).all(axis=2), 0, 1)
        self.flip = self.kvalid != self.valid


@pytest.fixture(scope="module", params=list(SELF_CASES))
def self_case(request):
    return _SelfCase(request.param)


def test_self_source_single_frame_against_float64(self_case):
    A.test_single_frame_against_float64(self_case)
    s = SELF_CASES[self_case.tag][7]
    assert np.isfinite(self_case.sf[s]).all()


def test_self_source_fused_against_float64(self_case):
    """test_cv_accuracy_gpu's fused gates, with one change: the key frame's own view weight is 0 (its cost is the same on
    every plane), so it adds nothing to the fused volume, and the stable pixels are those where the other valid frames'
    weights are >= 0.05."""
    c, tag = self_case, self_case.tag
    s = SELF_CASES[tag][7]
    assert np.abs(c.w[:, s]).max() < 1e-6
    flip_px = c.flip.any(axis=1)
    wsum = c.w.sum(axis=1)
    kz, rz = (c.cv == 0).all(axis=1), (c.ref_cv == 0).all(axis=1)
    bad_zero = (kz != rz) & ~(wsum < A.ZERO_WSUM) & ~flip_px
    cmp = ~kz & ~rz & ~flip_px
    others = np.delete(np.where(c.valid, c.w, np.inf), s, axis=1)
    stable = cmp & (others.min(axis=1) >= A.STABLE_WEIGHT)
    d = c.cv.astype(np.float64) - c.ref_cv
    st = A._error_stats(d, np.broadcast_to(stable[:, None], d.shape))
    vals = np.moveaxis(1 - 2 * c.sad, 2, 1)                                # (B,D,F,H,W)
    v = c.valid[:, None]
    lo = np.where(v, vals, np.inf).min(axis=2)
    hi = np.where(v, vals, -np.inf).max(axis=2)
    other = np.broadcast_to((cmp & ~stable)[:, None], d.shape)
    cvk = c.cv.astype(np.float64)
    worst_out = float(np.where(other, np.maximum(lo - cvk, 0) + np.maximum(cvk - hi, 0), 0.0).max())
    print(f"{tag} fused (other frames' weights >= {A.STABLE_WEIGHT}): {A._fmt(st)}; other pixels "
          f"{int((cmp & ~stable).sum())}, outside the frames' range by {worst_out:.2e}; zero-set disagreements "
          f"{int((kz != rz).sum())} ({int(bad_zero.sum())} with weight sum >= {A.ZERO_WSUM} and no flip)")
    assert not bad_zero.any(), f"{tag}: {int(bad_zero.sum())} fused pixels exactly 0 on one side only"
    assert worst_out <= A.MEAN_SLACK, f"{tag}: fused value {worst_out:.3e} outside the valid frames' range"
    assert st["n"] > 0
    A._check(st, f"{tag} fused")
