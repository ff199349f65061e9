"""Nets on xyz + LiDAR reflectance points (reference ``without_reflectivity: False``: PointNet on 4 input channels,
modules/tracking_net.py:41, modules/point_net.py:93-100), from the checkpoint to the kernels.

CPU: the 4-channel state_dict against the reference's own key -> shape list; the STN1 fold of a 4x4 transform; the
oracle against the fixtures of the UNMODIFIED reference (tests/golden/xyzr/, oracle/make_xyzr_goldens.py), eval and
training; ABI v3 and the argument checks that need no device.

GPU: the forward against those fixtures on both engines; a 4-channel net whose reflectance channel is switched off
(zero conv1 column, block-diagonal T1) reproducing the 3-channel net bit for bit; layer 1 of both PointNet paths against
fp64, on the stage's own workspace (test_pointnet_stage.py's method); the loader's output through forward_batch and
HostPipeline.
"""
import ctypes
import glob
import json
import os
import types

import numpy as np
import pytest
import torch

import mmmot_b200
from helpers import GOLDEN_DIR, LOSS_KW, TOL, case_tol, det_close, relerr, synthetic_gt
from kernel_kit import (U, Workspace, affine_bound, case_seed, contraction_bound, gn_apply, gn_stats, lib_state, nan_output,
                        nan_workspace, report, stage_layout, vp, worst_ratio)
from mmmot_b200 import _lib
from mmmot_b200.schema import state_schema
from mmmot_b200.synthetic import synthetic_batch, synthetic_pair, synthetic_state_dict
from mmmot_b200.weights import prepare
from oracle import torch_ref

gpu = pytest.mark.gpu
XYZR = os.path.join(GOLDEN_DIR, "xyzr")
EVAL = [torch.load(f) for f in sorted(glob.glob(os.path.join(XYZR, "xyzr_*.pt")))]
TRAIN = [torch.load(f) for f in sorted(glob.glob(os.path.join(XYZR, "train_*.pt")))]
PF = "point_net.feat"
# the keys whose shape depends on the point width
WIDTH_KEYS = {f"{PF}.stn1.idt": (4, 4), f"{PF}.stn1.conv1.weight": (64, 4, 1), f"{PF}.stn1.output.weight": (16, 256),
              f"{PF}.stn1.output.bias": (16,), f"{PF}.conv1.weight": (64, 4, 1)}


def net_of(fusion, sd, **kw):
    """TrackingNet(2) with the SkipPool heads, its point width from sd, loaded with sd (strict), eval mode, on the CPU."""
    c = sd[f"{PF}.conv1.weight"].shape[1]
    kw = dict(dict(affinity_op="multiply", softmax_mode="none", neg_threshold=0.2), **kw)
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch=fusion, test_mode=2,
                                 dropblock=0, without_reflectivity=(c == 3), **kw)
    net.load_state_dict(sd, strict=True)
    return net.eval()


def embed_xyz(sd3, seed=0):
    """A 4-channel checkpoint that computes exactly what the 3-channel sd3 does: conv1's reflectance column zero and
    T1 block-diagonal (STN1 output rows and bias zero for every entry of row or column 3 but (3, 3)).  What channel 3
    alone reaches, the STN1 convs and T1[3][3], is random: the reflectance must add nothing through it."""
    g = torch.Generator().manual_seed(7000 + seed)
    sd = dict(sd3)
    sd[f"{PF}.stn1.idt"] = torch.eye(4)
    sd[f"{PF}.stn1.conv1.weight"] = torch.cat([sd3[f"{PF}.stn1.conv1.weight"], torch.randn(64, 1, 1, generator=g)], 1)
    ow, ob = torch.zeros(16, 256), torch.zeros(16)
    for i in range(3):
        for j in range(3):
            ow[i * 4 + j] = sd3[f"{PF}.stn1.output.weight"][i * 3 + j]
            ob[i * 4 + j] = sd3[f"{PF}.stn1.output.bias"][i * 3 + j]
    ow[15] = torch.randn(256, generator=g) * 0.01
    ob[15] = 0.25
    sd[f"{PF}.stn1.output.weight"], sd[f"{PF}.stn1.output.bias"] = ow, ob
    sd[f"{PF}.conv1.weight"] = torch.cat([sd3[f"{PF}.conv1.weight"], torch.zeros(64, 1, 1)], 1)
    return sd


# ------------------------------------------------------------------------------------------------ CPU
def test_state_dict_matches_reference_schema():
    """The 263 keys of the reference's without_reflectivity=False net with its shapes; strict load; the 3-channel
    schema unchanged (only the five width-dependent keys differ)."""
    ref = json.load(open(os.path.join(XYZR, "schema_C.json")))
    sch = state_schema("C", point_in=4)
    assert [[k, list(s)] for k, (s, _) in sch.items()] == ref
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", without_reflectivity=False)
    assert net.point_channels == 4
    sd = net.state_dict()
    assert [[k, list(v.shape)] for k, v in sd.items()] == ref
    for k, s in WIDTH_KEYS.items():
        assert tuple(sd[k].shape) == s, k
    assert torch.equal(sd[f"{PF}.stn1.idt"], torch.eye(4))
    res = net.load_state_dict(synthetic_state_dict("C", seed=3, point_in=4), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    s3, s4 = state_schema("C"), state_schema("C", point_in=4)
    assert list(s3) == list(s4) and state_schema("C") == state_schema("C", 3)
    assert {k for k in s3 if s3[k] != s4[k]} == set(WIDTH_KEYS)
    assert mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls").point_channels == 3
    cfg = dict(sample_max_len=2, without_reflectivity=False, dropblock=5, use_dropout=True,
               model=dict(point_arch="v1", point_len=512, appear_arch="vgg", appear_len=512, appear_skippool=True,
                          appear_fpn=False, end_arch="v2", end_mode="avg", affinity_op="minus_abs", softmax_mode="dual_add",
                          score_arch="branch_cls", neg_threshold=0.2, score_fusion_arch="C", test_mode=2))
    assert mmmot_b200.build_model({"common": cfg}).point_channels == 4


def test_prepare_folds_4x4_stn():
    """conv1(T1^T x) == (W1 T1^T) x on random 4-channel points; trans1 is the 4x4 STN constant; PN_L1 is Wt[4][64]."""
    sd = synthetic_state_dict("C", seed=2, point_in=4)
    w, t1, t2, _ = prepare(sd, "C")
    assert t1.shape == (4, 4) and w[_lib.W["PN_L1"]].shape == (4, 64)
    assert torch.allclose(t1, torch_ref.stn_constant(sd, f"{PF}.stn1", 4)[0], rtol=0, atol=1e-6)
    pts = torch.randn(1, 4, 50, generator=torch.Generator().manual_seed(1))
    ref = torch.nn.functional.conv1d(torch.bmm(pts.transpose(2, 1), t1.unsqueeze(0)).transpose(2, 1), sd[f"{PF}.conv1.weight"])
    got = torch.einsum("kc,bkp->bcp", w[_lib.W["PN_L1"]], pts)
    assert (got - ref).abs().max() < 1e-5


def test_prepare_of_switched_off_reflectance_equals_xyz():
    """embed_xyz's checkpoint prepares to the 3-channel net's operands bit for bit, plus a zero PN_L1 row."""
    sd3 = synthetic_state_dict("C", seed=5)
    w3, t13, t23, s3 = prepare(sd3, "C")
    w4, t14, t24, s4 = prepare(embed_xyz(sd3), "C")
    l1 = _lib.W["PN_L1"]
    for i, (a, b) in enumerate(zip(w3, w4)):
        if i != l1:
            assert (a is None and b is None) or torch.equal(a, b), i
    assert torch.equal(w4[l1][:3], w3[l1]) and not w4[l1][3].any()
    assert torch.equal(t14[:3, :3], t13) and not t14[3, :3].any() and not t14[:3, 3].any()
    assert torch.equal(t24, t23) and s3 == s4


def test_synthetic_reflectance_leaves_xyz_draws_alone():
    d3, i3, _ = synthetic_pair(5, 6, 20, 32, seed=8, ragged=True)
    d4, i4, _ = synthetic_pair(5, 6, 20, 32, seed=8, ragged=True, reflectance=True)
    assert torch.equal(d3, d4) and torch.equal(i3["points_split"], i4["points_split"])
    assert i4["points"].shape[-1] == 4 and torch.equal(i4["points"][..., :3], i3["points"])
    r = i4["points"][0, :, 3]
    assert float(r.min()) >= 0 and float(r.max()) <= 1
    # per-detection structure: the spread of the detection means dwarfs the spread inside a detection
    s = i4["points_split"][0].long()
    means = torch.stack([r[s[d]:s[d + 1]].mean() for d in range(11)])
    assert float(means.std()) > 3 * 0.05
    c, p, sp = synthetic_batch(2, 3, pts=8, hw=32, seed=1, reflectance=True)
    assert p.shape == (int(sp[-1]), 4) and torch.equal(p[:48, :3], synthetic_batch(2, 3, pts=8, hw=32, seed=1)[1][:48])


def test_fixture_set_covers_the_cases():
    fus = {(g["case"][1], g["case"][2], g["case"][3]) for g in EVAL}
    assert {("C", "minus_abs", "dual_add"), ("A", "multiply", "none")} <= fus
    assert any(g["case"][9] for g in EVAL if g["case"][1] == "C") and any(g["case"][5] != g["case"][6] for g in EVAL)
    assert all(g["trans1"].shape[-1] == 4 for g in EVAL + TRAIN)
    assert len(TRAIN) == 1 and TRAIN[0]["drop"] == dict(dropblock=5, use_dropout=True)


@pytest.mark.parametrize("g", EVAL, ids=[c["case"][0] for c in EVAL])
def test_oracle_matches_reference_golden(g):
    name, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = g["case"]
    sd = synthetic_state_dict(fusion, seed=seed, point_in=4)
    dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged, reflectance=True)
    (det, link, new, end, trans), st = torch_ref.forward(sd, dets, info, split, fusion, op, sm, thr, return_stages=True)
    tol = case_tol(g["case"])
    assert relerr(st["feats"], g["feats"]) < tol
    assert relerr(det, g["det"]) < tol and relerr(link[0], g["link"]) < tol
    assert relerr(new, g["new"]) < tol and relerr(end, g["end"]) < tol
    assert relerr(trans[0], g["trans1"]) < 1e-5 and relerr(trans[1], g["trans2"]) < 1e-5


@pytest.mark.parametrize("g", TRAIN, ids=[c["case"][0] for c in TRAIN])
def test_train_oracle_matches_reference_golden(g):
    from oracle import train_ref
    name, fusion, op, sm, n, m, pts, hw, ragged, seed = g["case"]
    sd = synthetic_state_dict(fusion, seed=seed, point_in=4)
    dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged, reflectance=True)
    torch.manual_seed(seed)
    (det, link, new, end, trans), stats = train_ref.forward_train(sd, dets, info, split, fusion, op, sm, **g["drop"])
    assert relerr(det, g["det"]) < 5e-5 and relerr(link[0], g["link"]) < 5e-5
    assert relerr(new, g["new"]) < 5e-5 and relerr(end, g["end"]) < 5e-5
    for k, v in train_ref.running_after(sd, stats).items():
        assert relerr(v, g["running"][k]) < 1e-5, k
    cls, ids = synthetic_gt(n, m, seed)
    tm = mmmot_b200.TrackingModule(types.SimpleNamespace(test_mode=2), None, mmmot_b200.TrackingLoss(**LOSS_KW))
    gt_det, gt_link, gt_new, gt_end = tm.generate_gt(g["det"][0], cls, ids, split)
    args = (split, gt_det, gt_link, gt_new, gt_end, g["det"], [g["link"]], g["new"], g["end"], [g["trans1"], g["trans2"]])
    kw = {k: LOSS_KW[k] for k in ("det_ratio", "trans_ratio", "trans_last")}
    assert abs(float(train_ref.tracking_loss(*args, **kw)) - float(g["loss"])) < 1e-6 * abs(float(g["loss"]))
    assert abs(float(tm.criterion(*args)) - float(g["loss"])) < 1e-6 * abs(float(g["loss"]))


def test_abi_v3_point_channels(lib_built):
    lib = _lib.load()
    hdr = open(_lib.HEADER_PATH).read()
    assert lib.mmmot_abi_version() == _lib.ABI_VERSION == 3 and "#define MMMOT_ABI_VERSION 3" in hdr
    assert "int point_channels;" in hdr
    assert _lib.Weights.point_channels.offset == ctypes.sizeof(ctypes.c_void_p * _lib.W["COUNT"]) + 4 * _lib.W["COUNT"]
    # argument checks before any CUDA call: a width other than 3 or 4, or 4-channel points off a 16-byte boundary
    fake = lambda a: ctypes.c_void_p(a)
    hs = (ctypes.c_int * 3)(0, 4, 8)
    for pc, pts in ((5, 4096), (0, 4096), (2, 4096), (4, 4100)):
        w = _lib.Weights()
        w.point_channels = pc
        ptr = ctypes.pointer(w)
        assert lib.mmmot_pointnet_fwd(ptr, fake(pts), fake(8192), hs, 1, 2, fake(12288), fake(16384), 1 << 20, None) == -1
        assert lib.mmmot_pointnet_train_fwd(ptr, fake(pts), fake(8192), hs, 1, 2, None, fake(12288), fake(16384), 1 << 20,
                                            None) == -1


def test_width_checks_raise():
    """forward needs at least C columns; forward_batch / predict_batch exactly C (a [P][4] tensor must not be read as
    [4P/3][3]).  The checks come before anything touches a device."""
    net4 = net_of("C", synthetic_state_dict("C", seed=1, point_in=4))
    net3 = net_of("C", synthetic_state_dict("C", seed=1))
    dets, info3, split = synthetic_pair(2, 2, 6, 32, seed=1)
    _, info4, _ = synthetic_pair(2, 2, 6, 32, seed=1, reflectance=True)
    with pytest.raises(_lib.MmmotError, match="at least 4 columns"):
        net4(dets, info3, split)
    with pytest.raises(_lib.MmmotError, match=r"\[P\]\[4\]"):
        net4.forward_batch(dets, info3["points"][0], info3["points_split"][0], 2)
    with pytest.raises(_lib.MmmotError, match=r"\[P\]\[3\]"):
        net3.forward_batch(dets, info4["points"][0], info4["points_split"][0], 2)
    with pytest.raises(_lib.MmmotError, match=r"\[P\]\[3\]"):
        net3.predict_batch(dets, info4["points"][0], info4["points_split"][0], 2)
    with pytest.raises(_lib.MmmotError, match=r"\[P\]\[4\]"):
        net4.forward_batch(dets, info4["points"][0].reshape(-1), info4["points_split"][0], 2)
    # a 3-channel net takes the first 3 columns of wider points (the reference's loader layout): it gets as far as the
    # device check
    with pytest.raises(_lib.MmmotError, match="CUDA"):
        net3(dets, info4, split)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(params=["fp32", "tcgen05"])
def engine(request):
    mmmot_b200.set_engine(request.param)
    yield request.param
    mmmot_b200.set_engine("auto")


@gpu
@pytest.mark.parametrize("g", EVAL, ids=[c["case"][0] for c in EVAL])
def test_forward_matches_reference_golden(g, engine):
    name, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = g["case"]
    net = net_of(fusion, synthetic_state_dict(fusion, seed=seed, point_in=4), affinity_op=op, softmax_mode=sm,
                 neg_threshold=thr).cuda()
    dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged, reflectance=True)
    det, link, new, end, trans = net(dets.cuda(), {k: v.cuda() for k, v in info.items()}, split)
    tol = case_tol(g["case"])
    assert link[0].shape == g["link"].shape and det.shape == g["det"].shape
    assert relerr(link[0], g["link"]) < tol
    assert relerr(new, g["new"]) < tol and relerr(end, g["end"]) < tol
    assert det_close(det, g["det"], thr, tol)
    assert trans[0].shape == (1, 4, 4)
    assert relerr(trans[0], g["trans1"]) < 1e-5 and relerr(trans[1], g["trans2"]) < 1e-5
    assert torch.all(new[:, :n] == 0) and torch.all(end[:, n:] == 0)


@gpu
@pytest.mark.parametrize("g", TRAIN, ids=[c["case"][0] for c in TRAIN])
def test_training_forward_and_loss_match_reference_golden(g):
    name, fusion, op, sm, n, m, pts, hw, ragged, seed = g["case"]
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch=fusion, affinity_op=op,
                                 softmax_mode=sm, neg_threshold=0.2, test_mode=2, without_reflectivity=False, **g["drop"])
    net.load_state_dict(synthetic_state_dict(fusion, seed=seed, point_in=4))
    net.cuda().train()
    # the fixture's Dropout mask came from the CPU generator: draw it there
    net._dropout_mask = lambda shape, dev, p=0.5: torch.nn.functional.dropout(torch.ones(shape), p=p, training=True).to(dev)
    dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged, reflectance=True)
    cls, ids = synthetic_gt(n, m, seed)
    tm = mmmot_b200.TrackingModule(net, None, mmmot_b200.TrackingLoss(**LOSS_KW))
    dinfo = {k: v.cuda() for k, v in info.items()}
    torch.manual_seed(seed)
    det, link, new, end, trans = net(dets.cuda(), dinfo, split)
    assert det.shape == (3, n + m) and new.shape == (3, m) and end.shape == (3, n) and trans[0].shape == (1, 4, 4)
    assert relerr(det, g["det"]) < TOL and relerr(link[0], g["link"]) < TOL
    assert relerr(new, g["new"]) < TOL and relerr(end, g["end"]) < TOL
    sd_after = net.state_dict()
    for k, v in g["running"].items():
        if k.startswith("appearance.layers") or k.startswith("w_det"):
            if k.endswith("num_batches_tracked"):
                assert int(sd_after[k]) == int(v), k
            else:
                assert relerr(sd_after[k], v) < 1e-4, k
    torch.manual_seed(seed)
    loss = tm.step(dets.cuda(), dinfo, ids, cls, split)
    assert abs(float(loss) - float(g["loss"])) < 2e-4 * abs(float(g["loss"]))


@gpu
@pytest.mark.parametrize("eng", ["fp32", "tcgen05"])
@pytest.mark.parametrize("n", [4, 10])
def test_switched_off_reflectance_is_bit_identical_to_xyz(n, eng):
    """embed_xyz(sd3) on xyz + random reflectance == the 3-channel net on the same xyz, every output bit for bit
    (L = 8 < 16 and L = 20 >= 16, each engine forced)."""
    sd3 = synthetic_state_dict("C", seed=17)
    kw = dict(affinity_op="minus_abs", softmax_mode="dual_add")
    net3, net4 = net_of("C", sd3, **kw).cuda(), net_of("C", embed_xyz(sd3, 17), **kw).cuda()
    crops, pts4, split = synthetic_batch(2, n, pts=40, hw=32, seed=60 + n, reflectance=True)
    g = torch.Generator().manual_seed(n)
    pts4[:, 3] = torch.rand(pts4.shape[0], generator=g)                  # reflectance with no structure at all
    mmmot_b200.set_engine(eng)
    try:
        o4 = net4.forward_batch(crops.cuda(), pts4.cuda(), split, n, keep_feats=True)
        o3 = net3.forward_batch(crops.cuda(), pts4[:, :3].contiguous().cuda(), split, n, keep_feats=True)
    finally:
        mmmot_b200.set_engine("auto")
    for k in ("feats", "det", "link", "new", "end"):
        assert torch.equal(o4[k], o3[k]), k
    assert torch.equal(o4["trans"][0][0, :3, :3], o3["trans"][0][0]) and torch.equal(o4["trans"][1], o3["trans"][1])


# layer 1 on 4-channel points, kernel level
def l1_ref4(pts, W1, b1):
    """y = fma(w3, r, fma(w2, z, fma(w1, y, fma(w0, x, b)))) as pn_l1_*_kernel evaluate it -> (y [P][64], T), T = 1.01 u
    times the sum of the |prefix sums| (each fma rounds once)."""
    s, T = b1, 0.0
    for k in range(4):
        s = s + pts[:, k:k + 1] * W1[k]
        T = T + s.abs()
    return s, 1.01 * U * T


def _l1_points(kind, counts, g):
    """xyz as test_pointnet_stage.py draws them ("far": detections 63.5-66.5 m ahead with 0.5 m spread), reflectance
    per kind: "zero", "const" (0.37 everywhere) or a per-detection base plus noise."""
    P, nd = sum(counts), len(counts)
    if kind == "far":
        centre = torch.rand(nd, 3, generator=g) * torch.tensor([3.0, 2.0, 0.5]) + torch.tensor([63.5, -1.0, -1.5])
        spread = torch.tensor([0.5, 0.5, 0.5])
    else:
        centre = torch.rand(nd, 3, generator=g) * torch.tensor([60.0, 40.0, 2.0]) + torch.tensor([0.0, -20.0, -2.0])
        spread = torch.tensor([2.0, 1.0, 0.8])
    rep = torch.tensor(counts)
    xyz = torch.randn(P, 3, generator=g) * spread + centre.repeat_interleave(rep, 0)
    if kind == "zero":
        r = torch.zeros(P)
    elif kind == "const":
        r = torch.full((P,), 0.37)
    else:
        r = ((torch.rand(nd, generator=g) * 0.8 + 0.1).repeat_interleave(rep) + torch.randn(P, generator=g) * 0.05).clamp(0, 1)
    return torch.cat([xyz, r[:, None]], 1).contiguous()


# (name, pairs, L, points kind, count kind); every case runs on both paths
L1_CASES = [("far", 1, 32, "far", "r64"), ("zero", 2, 16, "zero", "r64"), ("const", 1, 20, "const", "r48"),
            ("ragged", 2, 24, "noisy", "ones")]


@gpu
@pytest.mark.parametrize("path", ["tc", "fp32"])
@pytest.mark.parametrize("case", L1_CASES, ids=[c[0] for c in L1_CASES])
def test_layer1_vs_fp64(case, path):
    """mmmot_pointnet_fwd on a NaN-filled workspace, then layer 1 against fp64 of the points: on the tensor cores x1p
    (the 4-term chain, fp64 statistics of it, gn_apply, the FP16 split), on the FP32 path y1 (K = 4 chain of the FP32
    engine, kernel_kit.contraction_bound) and sc1 / sh1 from the stored y1; xt stays untouched there (4-channel points
    are transposed into t1)."""
    name, pairs, L, kind, ck = case
    lib = _lib.load()
    net = net_of("C", synthetic_state_dict("C", seed=31, point_in=4)).cuda()
    t = prepare(net.state_dict(), "C")[0]
    W1, b1, g1, be1 = (t[_lib.W["PN_L1"] + i].double().cuda() for i in range(4))
    g = torch.Generator().manual_seed(case_seed("reflectance layer 1", *case))
    if ck == "ones":                              # runs of 1-point detections between larger ones
        counts = [1 if (d % 3) else int(torch.randint(2, 90, (1,), generator=g)) for d in range(pairs * L)]
    else:
        counts = torch.randint(1, 2 * int(ck[1:]), (pairs * L,), generator=g).tolist()
        counts[0] = counts[-1] = 1
    pts = _l1_points(kind, counts, g).cuda()
    split = [0] + np.cumsum(counts).tolist()
    P = split[-1]
    hs = np.asarray(split, dtype=np.int32)
    feats = nan_output(pairs * 3 * 512 * L)
    with lib_state(lib, engine=path):
        lay, tc = stage_layout(lib, 2, pairs, L, P)
        nbytes = int(lib.mmmot_pointnet_workspace(pairs, L, P))
        ws = nan_workspace(lib, nbytes)
        rc = lib.mmmot_pointnet_fwd(net.prepared().ptr, vp(pts), vp(torch.tensor(hs, device="cuda")),
                                    ctypes.c_void_p(hs.ctypes.data), pairs, L, vp(feats), vp(ws), nbytes, None)
        torch.cuda.synchronize()
    assert rc == 0 and tc == (path == "tc")
    assert lib.mmmot_status_check(vp(ws), None) == 0
    f = feats[:pairs * 3 * 512 * L].view(pairs, 3, 512, L)
    assert bool(torch.isfinite(f[:, 1]).all())
    W = Workspace(ws, lay)
    grp = torch.tensor(np.repeat(np.arange(pairs * L), counts), device="cuda") // L
    x = pts.double()
    r = {}
    if tc:
        y, T = l1_ref4(x, W1, b1)
        st = gn_stats(y, grp, pairs, T, kappa=False)
        cond = float((st[0].abs() / st[1].clamp_min(1e-300).sqrt()).max())
        z, Tz, _ = gn_apply(y, T, grp, st, g1, be1)
        h = W.owned("x1p", 2 * P * 64, torch.float16).view(2, P, 64)
        x1 = h[0].double() + h[1].double()
        r["x1p"] = worst_ratio(x1, z.clamp_min(0), Tz + 2.0 ** -22 * z.abs() + 2.0 ** -25)
    else:
        assert W.untouched_after("xt", 0), "xt written by a 4-channel run"
        y1 = W.owned("y1", 64 * P).view(64, P)
        ref, T = contraction_bound(W1, x.T.contiguous(), b1)
        r["y1"] = worst_ratio(y1, ref, T)
        y = y1.double().T
        st = gn_stats(y, grp, pairs)
        cond = float((st[0].abs() / st[1].clamp_min(1e-300).sqrt()).max())
        a, sh, Ta, Tsh = affine_bound(st, g1, be1)
        sc1 = W.owned("sc1", pairs * 64).view(pairs, 64)
        sh1 = W.owned("sh1", pairs * 64).view(pairs, 64)
        r["sc1_sh1"] = max(worst_ratio(sc1, a, Ta), worst_ratio(sh1, sh, Tsh))
    report(f"reflectance layer 1 {name} [{path}] pairs={pairs} L={L} P={P} (err / bound)", **r, layer1_mean_over_std=cond)
    if name == "far":
        assert cond >= 30, cond
    assert all(v <= 1.0 for v in r.values()), r


def _prep_pair():
    """Two frames of the reference loader's 3-D box fixture (tests/golden/prep_3d.npz: KITTI calibration, 4-feature scan)
    as prep_points_batch frames; the second frame's scan is the first one shifted 0.4 m ahead."""
    from mmmot_b200.lidar_crop import prep_points_batch
    gz = np.load(os.path.join(GOLDEN_DIR, "prep_3d.npz"))
    info = {"calib/P2": gz["P2"], "calib/R0_rect": gz["R0_rect"], "calib/Tr_velo_to_cam": gz["Tr_velo_to_cam"],
            "img_shape": gz["img_shape"]}
    dets = {k: gz[k] for k in ("location", "dimensions", "rotation_y", "bbox")}
    scan = torch.from_numpy(gz["points"].astype(np.float32)).cuda()
    scan2 = scan.clone()
    scan2[:, 0] += 0.4
    frames = [(scan, info, dets, None), (scan2, info, dets, None)]
    return frames, prep_points_batch, len(dets["bbox"])


@gpu
def test_loader_output_feeds_the_forward():
    """prep_points_batch(without_reflectivity=False) -> forward_batch of a 4-channel net, its 3-column output -> a
    3-channel net, each against the oracle; HostPipeline on pinned [P][4] points equals predict_batch, and refuses
    [P][3]."""
    frames, prep, n = _prep_pair()
    out = {}
    for c in (4, 3):
        pts, split = prep(frames, without_reflectivity=(c == 3))
        assert pts.shape[1] == c and split.numel() == 2 * n + 1
        out[c] = (pts, split)
    assert torch.equal(out[4][0][:, :3], out[3][0]) and torch.equal(out[4][1], out[3][1])
    fusion, op, sm = "C", "minus_abs", "dual_add"
    crops = torch.randn(2 * n, 3, 32, 32, generator=torch.Generator().manual_seed(3))
    for c, (pts, split) in out.items():
        sd = synthetic_state_dict(fusion, seed=29, point_in=c)
        net = net_of(fusion, sd, affinity_op=op, softmax_mode=sm).cuda()
        o = net.forward_batch(crops.cuda(), pts, split, n, keep_feats=True)
        info = {"points": pts.cpu()[None], "points_split": split.float()[None]}
        ds = [torch.tensor([n]), torch.tensor([n])]
        (rdet, rlink, rnew, rend, _), st = torch_ref.forward(sd, crops, info, ds, fusion, op, sm, 0.2, return_stages=True)
        assert relerr(o["feats"][0, 1], st["feats"][1]) < TOL, c
        assert relerr(o["link"][0], rlink[0]) < TOL and relerr(o["new"][0], rnew[:, n:]) < TOL, c
        assert relerr(o["end"][0], rend[:, :n]) < TOL and det_close(o["det"][0], rdet, 0.2, TOL), c
    # HostPipeline: 4 pairs of the 4-channel loader output, pinned
    pts, split = out[4]
    net = net_of(fusion, synthetic_state_dict(fusion, seed=29, point_in=4), affinity_op=op, softmax_mode=sm).cuda()
    B, P = 4, int(split[-1])
    h_pts = torch.cat([pts.cpu()] * B).pin_memory()
    h_split = torch.cat([split[:1]] + [split[1:] + b * P for b in range(B)])
    h_crops = torch.cat([crops] * B).pin_memory()
    ref = net.predict_batch(h_crops.cuda(), h_pts.cuda(), h_split, n)
    pipe = mmmot_b200.HostPipeline(net, n, sub_batches=2)
    res = pipe.run(h_crops, h_pts, h_split)
    assert torch.equal(res["match"], ref["match"].cpu())
    for k in ("assign_det", "assign_new", "assign_end"):
        assert torch.equal(res[k], ref[k].cpu()), k
    with pytest.raises(_lib.MmmotError, match=r"\[P\]\[4\]"):
        pipe.run(h_crops, h_pts[:, :3].contiguous().pin_memory(), h_split)
