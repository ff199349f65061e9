"""Tracking with one sensor: one feature stack (0 image, 1 LiDAR, 2 fused) computed alone, without the absent modality's
input or work.

Every output of a stack depends on that stack's features only (w_det with folded BatchNorm works per column, the affinity
MLP treats each stack as its own GroupNorm sample, stacks 0 and 1 are not mixed), and every engine and tile choice depends
on the per-pair shape only, so the oracle is exact: the full three-stack forward, sliced to the stack, bit for bit.

GPU: forward_stack against forward on every eval golden configuration (VGG / ResNet trunks, SkipPool / FPN heads, widths,
xyz / xyzr points, K = 3 frames); forward_batch / predict_batch(stack=s) against the full call over the engine thresholds;
independence from the absent sensor's values; the skipped stages' launches; TrackingModule.predict with a missing sensor.
CPU: argument errors before any launch, the one-stack workspace queries, the new entry points' exports."""
import ctypes
import glob
import os

import pytest
import torch

from helpers import GOLDEN_DIR, golden_cases
from kernel_kit import eval_net
import mmmot_b200
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict

STACKS = (0, 1, 2)
gpu = pytest.mark.gpu


@pytest.fixture(params=["fp32", "tcgen05"])
def engine(request):
    mmmot_b200.set_engine(request.param)
    yield request.param
    mmmot_b200.set_engine("auto")


# ------------------------------------------------------------------------------------------------ golden configurations
def _net(sd, **kw):
    net = mmmot_b200.TrackingNet(kw.pop("seq_len", 2), score_arch="branch_cls", test_mode=2, dropblock=0, **kw)
    net.load_state_dict(sd, strict=True)
    return net.cuda().eval()


def _golden_configs():
    """(id, make_net, make_sample) for every eval golden; make_sample -> (dets, det_info, dets_split)."""
    out = []
    for g in golden_cases():
        name, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = g["case"]
        out.append((name, lambda f=fusion, s=seed, o=op, x=sm, t=thr: eval_net(f, s, affinity_op=o, softmax_mode=x,
                                                                              neg_threshold=t)[0],
                    lambda a=(n, m, pts, hw, seed, ragged): synthetic_pair(*a[:4], seed=a[4], ragged=a[5])))
    for f in sorted(glob.glob(os.path.join(GOLDEN_DIR, "width", "w*.pt"))):
        name, arch, head, width, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = torch.load(f)["case"][:14]
        out.append((name, lambda a=(arch, head, width, fusion, op, sm, thr, seed): _net(
            synthetic_state_dict(a[3], seed=a[7], appear_arch=a[0], appear_head=a[1], width=a[2]), appear_len=a[2],
            point_len=a[2], appear_arch=a[0], appear_skippool=a[1] == "skippool", appear_fpn=a[1] == "fpn",
            score_fusion_arch=a[3], affinity_op=a[4], softmax_mode=a[5], neg_threshold=a[6]),
            lambda a=(n, m, pts, hw, seed, ragged): synthetic_pair(*a[:4], seed=a[4], ragged=a[5])))
    for sub, head in (("resnet", "skippool"), ("resnet_fpn", "fpn")):
        for f in sorted(glob.glob(os.path.join(GOLDEN_DIR, sub, "*.pt"))):
            name, arch, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = torch.load(f)["case"]
            out.append((name, lambda a=(arch, head, fusion, op, sm, thr, seed): _net(
                synthetic_state_dict(a[2], seed=a[6], appear_arch=a[0], appear_head=a[1]), appear_arch=a[0],
                appear_skippool=a[1] == "skippool", appear_fpn=a[1] == "fpn", score_fusion_arch=a[2], affinity_op=a[3],
                softmax_mode=a[4], neg_threshold=a[5]),
                lambda a=(n, m, pts, hw, seed, ragged): synthetic_pair(*a[:4], seed=a[4], ragged=a[5])))
    for f in sorted(glob.glob(os.path.join(GOLDEN_DIR, "xyzr", "xyzr_*.pt"))):
        name, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = torch.load(f)["case"]
        out.append((name, lambda a=(fusion, op, sm, thr, seed): _net(
            synthetic_state_dict(a[0], seed=a[4], point_in=4), appear_skippool=True, without_reflectivity=False,
            score_fusion_arch=a[0], affinity_op=a[1], softmax_mode=a[2], neg_threshold=a[3]),
            lambda a=(n, m, pts, hw, seed, ragged): synthetic_pair(*a[:4], seed=a[4], ragged=a[5], reflectance=True)))
    # K = 3 frames (test_gpu_parity.py::test_multi_frame_sample_and_end_mode_max), both end modes
    for end_mode in ("avg", "max"):
        out.append((f"k3_{end_mode}", lambda e=end_mode: _net(
            synthetic_state_dict("C", seed=13), seq_len=3, appear_skippool=True, score_fusion_arch="C",
            affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2, end_mode=e),
            lambda: synthetic_pair(5, 11, 24, 32, seed=61, ragged=True)[:2] + ([torch.tensor([k]) for k in (5, 7, 4)],)))
    return out


GOLDEN = _golden_configs()


def _cuda(info):
    return {k: v.cuda() for k, v in info.items()}


@gpu
@pytest.mark.parametrize("cfg", GOLDEN, ids=[c[0] for c in GOLDEN])
def test_forward_stack_equals_forward_slice(cfg, engine):
    """forward_stack(s) with the absent modality left out == forward(...)[s:s+1], bit for bit, for every stack."""
    _, make_net, make_sample = cfg
    net = make_net()
    dets, info, split = make_sample()
    dets, info = dets.cuda(), _cuda(info)
    det, links, new, end, trans = net(dets, info, split)
    for s in STACKS:
        o = net.forward_stack(None if s == 1 else dets, [] if s == 0 else info, split, s)
        assert o[0].shape == (1, det.shape[1]) and len(o[1]) == len(links), f"stack {s}"
        assert torch.equal(o[0], det[s:s + 1]), f"det, stack {s}"
        for k, (a, b) in enumerate(zip(o[1], links)):
            assert torch.equal(a, b[s:s + 1]), f"link {k}, stack {s}"
        assert torch.equal(o[2], new[s:s + 1]) and torch.equal(o[3], end[s:s + 1]), f"new / end, stack {s}"
        assert all(torch.equal(a, b) for a, b in zip(o[4], trans))
    # det_info None or without points is the same absent LiDAR
    o = net.forward_stack(dets, {"points_split": info["points_split"]}, split, 0)
    assert torch.equal(o[0], det[:1]) and torch.equal(o[2], new[:1])
    assert torch.equal(net.forward_stack(dets, None, split, 0)[3], end[:1])


# ------------------------------------------------------------------------------------------------ batched calls
def _batch(B, n, m, pts, hw, seed):
    """B frame-pairs of n and m detections packed for forward_batch: crops, points, points_split (CPU int64)."""
    ds, ps, sp, off = [], [], [torch.zeros(1, dtype=torch.int64)], 0
    for b in range(B):
        d, info, _ = synthetic_pair(n, m, pts, hw, seed=seed + b, ragged=True)
        ds.append(d)
        ps.append(info["points"][0])
        s_ = info["points_split"][0].long()
        sp.append(s_[1:] + off)
        off += int(s_[-1])
    return torch.cat(ds).cuda(), torch.cat(ps).cuda(), torch.cat(sp)


SHAPES = [(1, 1), (3, 7), (8, 8), (7, 9), (20, 45), (128, 128)]
HEADS = [("A", "multiply", "none"), ("B", "minus_abs", "single"), ("C", "minus", "dual"), ("A", "minus_abs", "dual_add"),
         ("B", "multiply", "dual_max"), ("C", "minus_abs", "dual_add")]
BATCH = [(n, m, B) + HEADS[(2 * i + j) % len(HEADS)] for i, (n, m) in enumerate(SHAPES) for j, B in enumerate((1, 5))]


@gpu
@pytest.mark.parametrize("n,m,B,fusion,op,sm", BATCH)
@pytest.mark.parametrize("eng", ["fp32", "tcgen05", "auto"])
def test_forward_batch_stack_equals_slice(n, m, B, fusion, op, sm, eng):
    """forward_batch(stack=s) == forward_batch()[:, s:s+1] bit for bit (features included), and predict_batch(stack=s)
    gives the assignment of predict_batch() of a net with test_mode = s.  "auto" crosses the engine thresholds
    n*m >= 64 (affinity) and L >= 64 (fusion / w_det) with the shapes."""
    net, _ = eval_net(fusion, 3, affinity_op=op, softmax_mode=sm, neg_threshold=0.2)
    crops, pts, split = _batch(B, n, m, 16, 32, seed=100 + n + m)
    mmmot_b200.set_engine(eng)
    try:
        full = net.forward_batch(crops, pts, split, n, m, keep_feats=True)
        for s in STACKS:
            one = net.forward_batch(None if s == 1 else crops, None if s == 0 else pts, None if s == 0 else split, n, m,
                                    keep_feats=True, stack=s)
            for k in ("det", "link", "new", "end", "feats"):
                assert one[k].shape[1] == 1 and torch.equal(one[k], full[k][:, s:s + 1]), f"{k}, stack {s}"
            assert int(one["status"]) == 0
            got = net.predict_batch(None if s == 1 else crops, None if s == 0 else pts, None if s == 0 else split, n, m,
                                    stack=s)
            net.test_mode = s
            ref = net.predict_batch(crops, pts, split, n, m)
            net.test_mode = 2
            for k in ("match", "assign_det", "assign_link", "assign_new", "assign_end"):
                assert torch.equal(got[k], ref[k]), f"{k}, stack {s}"
    finally:
        mmmot_b200.set_engine("auto")


# ------------------------------------------------------------------------------------------------ independence
@gpu
def test_lidar_stack_ignores_the_image_range():
    """Crops scaled by 1e6 make the full call report MMMOT_E_RANGE on the tensor cores; the LiDAR stack never looks at
    them (no appearance trunk, no fusion) and equals stack 1 of the unscaled full call."""
    net, _ = eval_net("C", 3, affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2)
    n = 16
    crops, pts, split = _batch(2, n, n, 32, 32, seed=8)
    mmmot_b200.set_engine("tcgen05")
    try:
        ref = net.forward_batch(crops, pts, split, n)
        with pytest.raises(_lib.MmmotError, match="MMMOT_E_RANGE"):
            net.forward_batch(crops * 1e6, pts, split, n)
        one = net.forward_batch(crops * 1e6, pts, split, n, stack=1)
        assert int(one["status"]) == 0
        for k in ("det", "link", "new", "end"):
            assert torch.equal(one[k], ref[k][:, 1:2]), k
    finally:
        mmmot_b200.set_engine("auto")


@gpu
def test_image_stack_ignores_the_points(engine):
    """NaN points do not reach the image stack (no PointNet, no fusion)."""
    net, _ = eval_net("B", 4, affinity_op="multiply", softmax_mode="single", neg_threshold=0.2)
    n = 12
    crops, pts, split = _batch(3, n, n, 24, 32, seed=20)
    ref = net.forward_batch(crops, pts, split, n)
    one = net.forward_batch(crops, torch.full_like(pts, float("nan")), split, n, stack=0)
    for k in ("det", "link", "new", "end"):
        assert torch.equal(one[k], ref[k][:, :1]), k


# ------------------------------------------------------------------------------------------------ skipped work
def _tags(run):
    """Per-tag (launches, FLOPs) of the timed launches of run()."""
    lib = _lib.load()
    T = lib.mmmot_timing_tag_count()
    names = [lib.mmmot_timing_tag_name(t).decode() for t in range(T)]
    flop, cnt = (ctypes.c_double * T)(), (ctypes.c_long * T)()
    assert lib.mmmot_timing_enable(1) == 0
    try:
        lib.mmmot_timing_collect_tags(None, None, None, None)
        run()
        torch.cuda.synchronize()
        assert lib.mmmot_timing_collect_tags(None, flop, None, cnt) == 0
    finally:
        lib.mmmot_timing_enable(0)
    return {nm: (cnt[t], flop[t]) for t, nm in enumerate(names) if cnt[t]}


@gpu
@pytest.mark.parametrize("arch,head", [("vgg", "skippool"), ("resnet50", "fpn")])
def test_absent_sensor_stages_are_not_launched(arch, head):
    """stack 1 launches no appearance kernel, stack 0 no PointNet kernel; the affinity stage of one stack does a third
    of the full call's algorithmic FLOPs at the same B, n, m."""
    net = _net(synthetic_state_dict("C", seed=5, appear_arch=arch, appear_head=head), appear_arch=arch,
               appear_skippool=head == "skippool", appear_fpn=head == "fpn", score_fusion_arch="C",
               affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2)
    n = 32
    crops, pts, split = _batch(3, n, n, 24, 64, seed=30)
    full = _tags(lambda: net.forward_batch(crops, pts, split, n))
    assert any(k.startswith("pointnet.") for k in full) and any(k.startswith(("vgg.", "resnet.")) for k in full)
    aff = lambda t: sum(f for k, (c, f) in t.items() if k.startswith("affinity."))
    assert aff(full) > 0
    for s in STACKS:
        one = _tags(lambda: net.forward_batch(None if s == 1 else crops, None if s == 0 else pts,
                                              None if s == 0 else split, n, stack=s))
        if s == 1:
            assert not [k for k in one if k.startswith(("vgg.", "resnet.", "fpn."))], one
        if s == 0:
            assert not [k for k in one if k.startswith("pointnet.")], one
        assert aff(one) * 3 == pytest.approx(aff(full), rel=1e-12), s


# ------------------------------------------------------------------------------------------------ TrackingModule
@gpu
def test_predict_with_one_sensor():
    """TrackingModule.predict with the reference's 2-D loader output (det_info = []) at test_mode 0, and without
    images at test_mode 1, returns what it returns with both inputs; test_mode 2 names the missing sensor."""
    from mmmot_b200.tracking_model import TrackingModule
    from helpers import stitch_scenario
    frames, _ = stitch_scenario(seed=3)
    for t in (0, 1):
        net, _ = eval_net("C", 9, affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2)
        net.test_mode = t
        both, one = TrackingModule(net), TrackingModule(net)
        for a in range(3):
            na, nb = int(frames[a]["bbox"].shape[1]), int(frames[a + 1]["bbox"].shape[1])
            dets, info, split = synthetic_pair(na, nb, 24, 32, seed=40 + a, ragged=True)
            dets, info = dets.cuda(), _cuda(info)
            r_both = both.predict(dets, info, [frames[a], frames[a + 1]], split)
            r_one = one.predict(None if t == 1 else dets, [] if t == 0 else info, [frames[a], frames[a + 1]], split)
            assert r_both[2] == r_one[2]
            assert len(r_both[0]) == len(r_one[0])
            for x, y in zip(r_both[0], r_one[0]):
                assert list(map(int, x)) == list(map(int, y))
            for x, y in zip(r_both[1], r_one[1]):
                assert x.keys() == y.keys() and all(torch.equal(torch.as_tensor(x[k]), torch.as_tensor(y[k])) for k in x)
    net, _ = eval_net("C", 9, affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2)
    dets, info, split = synthetic_pair(4, 5, 24, 32, seed=1)
    with pytest.raises(_lib.MmmotError, match="LiDAR"):
        TrackingModule(net).predict(dets.cuda(), [], [frames[0], frames[1]], split)
    with pytest.raises(_lib.MmmotError, match="image"):
        TrackingModule(net).predict(None, _cuda(info), [frames[0], frames[1]], split)


# ------------------------------------------------------------------------------------------------ CPU
def _cpu_net(training=False):
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", test_mode=2, dropblock=0)
    return net.train() if training else net.eval()


def test_argument_errors_before_any_launch(lib_built):
    """A stack outside {0, 1, 2} is a ValueError, a missing input the stack needs an MmmotError naming the sensor,
    training mode a NotImplementedError: all raised before the net reaches the device (it is on the CPU here)."""
    net = _cpu_net()
    crops, pts, split = torch.zeros(8, 3, 32, 32), torch.zeros(10, 3), torch.arange(9)
    dets, info, ds = synthetic_pair(4, 4, 8, 32, seed=0)
    for bad in (3, -1, "1", 1.5):
        with pytest.raises(ValueError):
            net.forward_batch(crops, pts, split, 4, stack=bad)
        with pytest.raises(ValueError):
            net.predict_batch(crops, pts, split, 4, stack=bad)
        with pytest.raises(ValueError):
            net.forward_stack(dets, info, ds, bad)
    with pytest.raises(ValueError):
        net.forward_stack(dets, info, ds, None)
    for s, args, sensor in ((0, (None, pts, split), "image"), (1, (crops, None, None), "LiDAR"),
                            (1, (crops, pts, None), "LiDAR"), (2, (None, pts, split), "image"),
                            (2, (crops, None, None), "LiDAR")):
        with pytest.raises(_lib.MmmotError, match=f"stack {s} needs the {sensor}"):
            net.forward_batch(*args, 4, stack=s)
    for s, args, sensor in ((0, (None, info), "image"), (1, (dets, []), "LiDAR"), (1, (dets, None), "LiDAR"),
                            (2, (dets, {"points_split": info["points_split"]}), "LiDAR"), (2, (None, info), "image")):
        with pytest.raises(_lib.MmmotError, match=f"stack {s} needs the {sensor}"):
            net.forward_stack(*args, ds, s)
    train = _cpu_net(training=True)
    for s in STACKS:
        with pytest.raises(NotImplementedError):
            train.forward_batch(crops, pts, split, 4, stack=s)
        with pytest.raises(NotImplementedError):
            train.forward_stack(dets, info, ds, s)


def test_predict_names_the_missing_sensor(lib_built):
    from mmmot_b200.tracking_model import TrackingModule
    dets, info, ds = synthetic_pair(3, 3, 8, 32, seed=0)
    for t, args, sensor in ((2, (dets, []), "LiDAR"), (2, (None, info), "image"), (0, (None, info), "image"),
                            (1, (dets, None), "LiDAR"), (1, (dets, {}), "LiDAR")):
        net = _cpu_net()
        net.test_mode = t
        with pytest.raises(_lib.MmmotError, match=f"test_mode {t} needs the {sensor}"):
            TrackingModule(net).predict(*args, [{}, {}], ds)


@pytest.mark.parametrize("pairs,n,m", [(1, 1, 1), (5, 3, 7), (32, 128, 128), (2, 20, 45)])
def test_one_stack_workspaces_are_smaller(lib_built, pairs, n, m):
    lib = _lib.load()
    assert lib.mmmot_affinity_stack_workspace(pairs, n, m) < lib.mmmot_affinity_workspace(pairs, n, m)
    assert lib.mmmot_fusion_det_stack_workspace(pairs, n + m) < lib.mmmot_fusion_det_workspace(pairs, n + m)
    net = _cpu_net()
    for s in STACKS:        # the feature stages a stack still runs may need more than the affinity stage: <=, not <
        assert net._workspace_bytes(pairs, [(n, m)], n + m, 100 * pairs, 64, 64, s) <= \
            net._workspace_bytes(pairs, [(n, m)], n + m, 100 * pairs, 64, 64)
    # the LiDAR stack needs no room for the appearance trunk
    assert net._workspace_bytes(pairs, [(n, m)], n + m, 1, 224, 224, 1) == net._workspace_bytes(pairs, [(n, m)], n + m, 1, 8, 8, 1)


def test_stack_entry_points_reject_bad_stacks(lib_built):
    """MMMOT_E_ARG before any CUDA call for a stack outside 0..2 (dummy non-null pointers: nothing is dereferenced)."""
    lib = _lib.load()
    w = _lib.Weights()
    p = ctypes.c_void_p(16)
    for s in (-1, 3):
        assert lib.mmmot_affinity_stack_fwd(ctypes.byref(w), 0, 1, 0, 1, s, 4, 4, p, p, p, p, p, 1 << 20, None) == -1
        assert lib.mmmot_fusion_det_stack_fwd(ctypes.byref(w), 2, 3, 0.0, 1, 8, s, p, p, p, 1 << 20, None) == -1
