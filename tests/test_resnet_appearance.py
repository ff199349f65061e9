"""Nets with a ResNet-50/101/152 appearance trunk (reference appear_arch resnet50 | resnet101 | resnet152 with skip
pooling, modules/appear_net.py:60-83,213-256), from the checkpoint to the kernels.

CPU: each arch's state_dict against the reference's own key -> shape list (tests/golden/resnet/, written by
oracle/make_resnet_goldens.py from the UNMODIFIED reference); strict loads; the BatchNorm fold and the K orders against
fp64 convolutions; workspace queries and the argument checks that need no device; the constructor's guards; the
reference net built offline without touching torch.hub (where a reference checkout is present).

GPU: the whole trunk against an fp64 restatement with torch.nn.functional at 64 x 64 and 224 x 224 crops on both engines;
the forward against the reference fixtures (scores, and LP assignments wherever the fixture's optimum has a gap larger
than the score perturbation) on both engines; forward_batch bit-identical to looped forward.
"""
import ctypes
import glob
import json
import os

import pytest
import torch
import torch.nn.functional as F

import mmmot_b200
from helpers import GOLDEN_DIR, TOL, det_close, relerr
from mmmot_b200 import _lib
from mmmot_b200.schema import RESNET_BLOCKS, resnet_convs, state_schema
from mmmot_b200.synthetic import synthetic_batch, synthetic_pair, synthetic_state_dict
from mmmot_b200.weights import prepare, prepare_resnet

gpu = pytest.mark.gpu
RES = os.path.join(GOLDEN_DIR, "resnet")
EVAL = [torch.load(f) for f in sorted(glob.glob(os.path.join(RES, "res*.pt")))]
ARCHS = tuple(RESNET_BLOCKS)


def net_of(arch, fusion, sd, **kw):
    kw = dict(dict(affinity_op="multiply", softmax_mode="none", neg_threshold=0.2), **kw)
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, appear_arch=arch, score_arch="branch_cls",
                                 score_fusion_arch=fusion, test_mode=2, dropblock=0, **kw)
    net.load_state_dict(sd, strict=True)
    return net.eval()


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("arch", ARCHS)
def test_state_dict_matches_reference_schema(arch):
    ref = json.load(open(os.path.join(RES, f"schema_{arch}.json")))
    sch = state_schema("C", 3, arch)
    assert [[k, list(s)] for k, (s, _) in sch.items()] == ref
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, appear_arch=arch, score_arch="branch_cls")
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
    res = net.load_state_dict(synthetic_state_dict("C", seed=3, appear_arch=arch), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert not any(".fc." in k and "global_pool" not in k for k in sch)          # the wrapper drops torchvision's fc
    convs = resnet_convs(arch)
    assert len(convs) == 1 + 3 * sum(RESNET_BLOCKS[arch]) + 4 <= _lib.RESNET_MAX_CONVS
    # everything outside the appearance trunk and its heads is the VGG net's
    vgg = state_schema("C")
    assert {k: v for k, v in sch.items() if not k.startswith("appearance.")} == \
        {k: v for k, v in vgg.items() if not k.startswith("appearance.")}


def test_vgg_schema_and_draws_unchanged():
    assert state_schema("C") == state_schema("C", 3, "vgg")
    a, b = synthetic_state_dict("C", seed=9), synthetic_state_dict("C", seed=9, appear_arch="vgg")
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    w, _, _, _ = prepare(a, "C")
    assert sum(t is not None for t in w) == _lib.W["COUNT"]
    r, _, _, _ = prepare(synthetic_state_dict("C", seed=9, appear_arch="resnet50"), "C", "resnet50")
    vgg_ids = {i for k, i in _lib.W.items() if k.startswith("VGG") for i in range(i, i + (2 if k == "VGG_WPX0" else 13))}
    vgg_ids |= set(range(_lib.W["SKIP0"], _lib.W["SKIP0"] + 40))
    assert {i for i, t in enumerate(r) if t is None} == vgg_ids
    with pytest.raises(ValueError):
        state_schema("C", 3, "resnet34")


def _fold64(sd, conv, bn):
    """fp64 BatchNorm(conv(x)) as a function of x."""
    w = sd[f"{conv}.weight"].double()
    rm, rv = sd[f"{bn}.running_mean"].double(), sd[f"{bn}.running_var"].double()
    g, b = sd[f"{bn}.weight"].double(), sd[f"{bn}.bias"].double()
    return lambda x, stride, pad: F.batch_norm(F.conv2d(x, w, stride=stride, padding=pad), rm, rv, g, b, False, 0.0, 1e-5)


def _unpack(packed, scale, M, K):
    """pack_tc's tiles -> (hi + lo) * scale as W [M][K] fp64 (the inverse of the packing permutation)."""
    mt, kc = (M + 127) // 128, (K + 31) // 32
    t = packed.view(torch.float16).view(kc, mt, 2, 4, 16, 8, 8).permute(2, 1, 4, 5, 0, 3, 6).reshape(2, mt * 128, kc * 32)
    return (t[0].double() + t[1].double()) * scale


def test_bn_fold_and_k_order_vs_fp64():
    """prepare_resnet: every conv's folded Wt (K order of mmmot_resnet_weights) and bias reproduce fp64 conv + BatchNorm
    on a random input, for the stem, a strided 3x3, a 1x1 and a strided downsample; the packed tiles hold the same
    matrix (hi + lo) zero-padded to K = 160 for the stem."""
    arch = "resnet50"
    sd = synthetic_state_dict("C", seed=4, appear_arch=arch)
    convs, heads = prepare_resnet(sd, arch)
    spec = resnet_convs(arch)
    g = torch.Generator().manual_seed(5)
    picks = [0, 1, 4, spec.index(next(c for c in spec if c[0] == "appearance.layers.layer2.0.conv2")),
             spec.index(next(c for c in spec if c[0] == "appearance.layers.layer3.0.downsample.0"))]
    for i in picks:
        conv, bn, cin, cout, k, stride = spec[i]
        wt, b, packed, scale = convs[i]
        assert wt.shape == (k * k * cin, cout) and b.shape == (cout,)
        x = torch.randn(2, cin, 16, 16, generator=g, dtype=torch.float64)
        ref = _fold64(sd, conv, bn)(x, stride, k // 2)
        w = wt.double().reshape(k, k, cin, cout).permute(3, 2, 0, 1)      # [(ky*k+kx)*cin + ci][co] -> [co][ci][ky][kx]
        got = F.conv2d(x, w, b.double(), stride=stride, padding=k // 2)
        assert relerr(got, ref) < 1e-6, conv
        W = _unpack(packed, scale, cout, k * k * cin)
        Kp = (k * k * cin + 31) // 32 * 32
        assert W.shape[1] == Kp and (i != 0 or Kp == 160)
        assert not W[:, k * k * cin:].any() and not W[cout:].any()
        assert float((W[:cout, :k * k * cin] - wt.double().t()).abs().max()) <= 2.0 ** -22 * float(wt.abs().max()), conv
    assert len(heads) == 40 and heads[2].shape == (256, 64) and heads[30 + 2].shape == (2048, 512)
    assert heads[6].shape == (64, 128) and heads[36].shape == (512, 128)


def test_workspace_and_argument_checks(lib_built):
    lib = _lib.load()
    ws = lib.mmmot_appearance_resnet_workspace(16, 64, 64)
    assert ws > 16 * 64 * 64 * (16 * 3 + 8 * 2 + 40) * 4
    assert lib.mmmot_appearance_resnet_workspace(16, 224, 224) > ws
    fake = lambda a: ctypes.c_void_p(a)
    rw = _lib.ResnetWeights()
    rw.blocks[:] = RESNET_BLOCKS["resnet50"]
    args = lambda r, n=4, H=64, W=64, L=2: (None, ctypes.pointer(r) if r is not None else None, fake(4096), n, H, W, L,
                                             fake(8192), fake(1 << 20), ws, None)
    assert lib.mmmot_appearance_resnet_fwd(*args(None)) == -1
    bad = _lib.ResnetWeights()
    for blocks in ((0, 4, 6, 3), (3, 4, 6, -1), (3, 8, 60, 3)):
        bad.blocks[:] = blocks
        assert lib.mmmot_appearance_resnet_fwd(*args(bad)) == -1, blocks
    assert lib.mmmot_appearance_resnet_fwd(*args(rw, H=48)) == -3
    assert lib.mmmot_appearance_resnet_fwd(*args(rw, W=80)) == -3
    assert lib.mmmot_appearance_resnet_fwd(*args(rw, n=5, L=2)) == -3
    assert lib.mmmot_appearance_resnet_fwd(*args(rw, L=0)) == -1
    assert lib.mmmot_appearance_resnet_fwd(*args(rw)) == -1            # good shapes, but no conv pointers
    names = [lib.mmmot_timing_tag_name(t).decode() for t in range(lib.mmmot_timing_tag_count())]
    assert [n for n in names if n.startswith("resnet.")] == ["resnet.stem", "resnet.maxpool", "resnet.conv1x1",
                                                             "resnet.conv3x3", "resnet.stride2", "resnet.residual",
                                                             "resnet.mean_heads"]


def test_constructor_guards():
    for kw in (dict(appear_arch="resnet50", appear_skippool=False), dict(appear_arch="resnet101", appear_fpn=True),
               dict(appear_arch="resnet34"), dict(appear_arch="resnet50", appear_len=256)):
        kw = dict(dict(appear_skippool=True), **kw)
        with pytest.raises(NotImplementedError):
            mmmot_b200.TrackingNet(2, score_arch="branch_cls", **kw)
    net = net_of("resnet50", "C", synthetic_state_dict("C", seed=1, appear_arch="resnet50")).train()
    dets, info, split = synthetic_pair(2, 2, 6, 32, seed=1)
    with pytest.raises(NotImplementedError, match="training-mode"):
        net(dets, info, split)
    cfg = dict(sample_max_len=2, without_reflectivity=True, dropblock=5, use_dropout=False,
               model=dict(point_arch="v1", point_len=512, appear_arch="resnet152", appear_len=512, appear_skippool=True,
                          appear_fpn=False, end_arch="v2", end_mode="avg", affinity_op="minus_abs", softmax_mode="dual_max",
                          score_arch="branch_cls", neg_threshold=0.2, score_fusion_arch="B", test_mode=2))
    assert mmmot_b200.build_model({"common": cfg}).appear_arch == "resnet152"


def test_fixture_set_covers_the_cases():
    cases = {(g["case"][1], g["case"][2], g["case"][3], g["case"][4]) for g in EVAL}
    assert cases == {("resnet50", "C", "minus_abs", "dual_add"), ("resnet101", "A", "multiply", "none"),
                     ("resnet152", "B", "minus_abs", "dual_max")}
    assert all(g["case"][6] != g["case"][7] and g["case"][9] == 64 for g in EVAL)
    assert all(os.path.getsize(f) < 150_000 for f in glob.glob(os.path.join(RES, "*")))


def test_reference_resnet_net_builds_offline():
    """The oracle's recipe builds the reference ResNet nets without any hub call: downloads raise and are recorded,
    torchvision's builders ignore pretrained=True."""
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("no reference checkout (MMMOT_REFERENCE)")
    import torch.hub
    import torchvision
    from oracle import make_resnet_goldens as mrg
    mrg.offline_torchvision()
    before = len(mrg.BLOCKED)
    for arch in ARCHS:
        net = mrg.reference_net(arch, "C", "minus_abs", "dual_add", 0.2)
        ref = json.load(open(os.path.join(RES, f"schema_{arch}.json")))
        assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
        assert torchvision.models.__dict__[arch](pretrained=True).fc.out_features == 1000
    assert len(mrg.BLOCKED) == before == 0
    with pytest.raises(RuntimeError, match="network access refused"):
        torch.hub.load_state_dict_from_url("http://127.0.0.1/none.pth")
    assert len(mrg.BLOCKED) == 1
    mrg.BLOCKED.clear()


# ------------------------------------------------------------------------------------------------ GPU
def trunk64(sd, arch, crops):
    """fp64 restatement of the ResNet trunk + SkipPool heads (eval) with torch.nn.functional: stack 0 [L][512]."""
    x = crops.double()
    spec = resnet_convs(arch)
    f = lambda i, x: _fold64(sd, spec[i][0], spec[i][1])(x, spec[i][5], spec[i][4] // 2)
    x = F.max_pool2d(F.relu(f(0, x)), 3, 2, 1)
    i, pooled = 1, []
    for s, nb in enumerate(RESNET_BLOCKS[arch]):
        for b in range(nb):
            y = f(i + 2, F.relu(f(i + 1, F.relu(f(i, x)))))
            idt = f(i + 3, x) if b == 0 else x
            x = F.relu(y + idt)
            i += 4 if b == 0 else 3
        pooled.append(x.mean(dim=(2, 3), keepdim=True))
    outs = []
    for s, v in enumerate(pooled):
        p = lambda k: sd[f"appearance.global_pool.{s}.fc.{k}"].double().to(v.device)
        h = F.group_norm(v, 1, p("0.weight"), p("0.bias"), 1e-5)
        h = F.relu(F.group_norm(F.conv2d(h, p("1.weight"), p("1.bias")), 1, p("2.weight"), p("2.bias"), 1e-5))
        h = F.relu(F.group_norm(F.conv2d(h, p("4.weight"), p("4.bias")), 1, p("5.weight"), p("5.bias"), 1e-5))
        outs.append(h.flatten(1))
    return torch.cat(outs, 1)


@pytest.fixture(params=["fp32", "tcgen05"])
def engine(request):
    mmmot_b200.set_engine(request.param)
    yield request.param
    mmmot_b200.set_engine("auto")


# (M, K) of every FP32-engine contraction of the trunks (resnet.cu through mm_simt_direct, XM_DIRECT on uniform
# tiling): the stem (K = 147 gathered taps), 1x1 convs, 3x3 convs on gathered taps, downsamples
SIMT_SHAPES = sorted({(cout, k * k * cin) for arch in ARCHS for _, _, cin, cout, k, _ in resnet_convs(arch)})


def test_simt_shapes_listed():
    assert (64, 147) in SIMT_SHAPES and (512, 4608) in SIMT_SHAPES and (2048, 1024) in SIMT_SHAPES
    assert all(m % 64 == 0 for m, _ in SIMT_SHAPES)


@gpu
@pytest.mark.parametrize("relu", [0, 1])
def test_fp32_engine_contractions_vs_fp64(relu):
    """Every (M, K) the FP32 path of the trunk runs, through mmmot_debug_simt_op (mode DIRECT, the launch
    mm_simt_direct makes), against fp64 within kernel_kit.contraction_bound; 300 columns (two full 128-column tiles and
    a partial one), x_ks = 300 as the trunk's [K][pixels] operands."""
    from kernel_kit import XM, case_seed, contraction_bound, nan_output, vp, worst_ratio
    lib = _lib.load()
    S = 300
    worst = 0.0
    for M, K in SIMT_SHAPES:
        g = torch.Generator().manual_seed(case_seed("resnet simt", M, K, relu))
        wt = (torch.randn(K, M, generator=g) * (2.0 / K) ** 0.5).cuda()
        b = (torch.rand(M, generator=g) * 0.2 - 0.1).cuda()
        x = torch.randn(K, S, generator=g).clamp_min(-0.5).cuda()
        Y = nan_output(M * S)
        rc = lib.mmmot_debug_simt_op(XM.DIRECT, M, K, vp(wt), vp(b), relu, vp(x), 0, S, None, None, 0, 0, 0, 0, 0, 0, S, 1,
                                     None, 0, None, None, 0, vp(Y), 0, S, None, None)
        torch.cuda.synchronize()
        assert rc == 0, (M, K)
        assert bool(torch.isfinite(Y[:M * S]).all()) and bool(torch.isnan(Y[M * S:]).all())
        ref, T = contraction_bound(wt.double(), x.double(), b.double(), relu=bool(relu))
        r = worst_ratio(Y[:M * S].view(M, S), ref, T)
        worst = max(worst, r)
        assert r <= 1.0, (M, K, r)
    print(f"\nresnet FP32-engine contractions relu={relu}: worst err / bound {worst:.3g} over {len(SIMT_SHAPES)} shapes")


@gpu
@pytest.mark.parametrize("arch,hw,L", [("resnet50", 64, 6), ("resnet101", 64, 4), ("resnet152", 64, 4),
                                       ("resnet50", 224, 2), ("resnet152", 224, 2)])
def test_trunk_vs_fp64(arch, hw, L, engine):
    """mmmot_appearance_resnet_fwd's stack 0 against the fp64 trunk, max-norm relative error per image."""
    lib = _lib.load()
    sd = synthetic_state_dict("C", seed=21, appear_arch=arch)
    net = net_of(arch, "C", sd).cuda()
    wts = net.prepared()
    crops, _, _ = synthetic_pair(L // 2, L - L // 2, 4, hw, seed=hw + L)
    crops = crops.cuda()
    n = crops.shape[0]
    feats = torch.full((1, 3, 512, L), float("nan"), device="cuda")
    nbytes = lib.mmmot_appearance_resnet_workspace(n, hw, hw)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    assert lib.mmmot_status_reset(ctypes.c_void_p(ws.data_ptr()), None) == 0
    rc = lib.mmmot_appearance_resnet_fwd(wts.ptr, wts.rptr, ctypes.c_void_p(crops.data_ptr()), n, hw, hw, L,
                                         ctypes.c_void_p(feats.data_ptr()), ctypes.c_void_p(ws.data_ptr()), nbytes, None)
    assert rc == 0
    assert lib.mmmot_status_check(ctypes.c_void_p(ws.data_ptr()), None) == 0
    got = feats[0, 0].T
    assert bool(torch.isfinite(got).all()) and bool(torch.isnan(feats[0, 1:]).all())
    ref = trunk64({k: v.cuda() for k, v in sd.items()}, arch, crops)
    err = max(relerr(got[i], ref[i]) for i in range(n))
    print(f"\nresnet trunk {arch} {hw}x{hw} [{engine}]: max-norm rel err {err:.3g}")
    assert err < TOL, err


@gpu
@pytest.mark.parametrize("g", EVAL, ids=[c["case"][0] for c in EVAL])
def test_forward_matches_reference_golden(g, engine):
    from oracle import lp_ref
    name, arch, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = g["case"]
    net = net_of(arch, fusion, synthetic_state_dict(fusion, seed=seed, appear_arch=arch), affinity_op=op, softmax_mode=sm,
                 neg_threshold=thr).cuda()
    dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged)
    dinfo = {k: v.cuda() for k, v in info.items()}
    det, link, new, end, trans = net(dets.cuda(), dinfo, split)
    o = net.forward_batch(dets.cuda(), info["points"][0].cuda(), info["points_split"][0].long(), n, m, keep_feats=True)
    errs = {"feats0": relerr(o["feats"][0, 0], g["feats"][0]), "link": relerr(link[0], g["link"]),
            "new": relerr(new, g["new"]), "end": relerr(end, g["end"])}
    print(f"\n{name} [{engine}]: {errs}")
    assert all(e < TOL for e in errs.values()), errs
    assert det_close(det, g["det"], thr, TOL)
    assert relerr(trans[1], g["trans2"]) < 1e-5
    # LP assignments: identical to the fixture's wherever its optimum beats the second best by more than the perturbation
    t = 2
    a = mmmot_b200.ortools_solve(det[t], [link[0][t:t + 1]], new[t], end[t], split)
    a = (a[0].cpu(), [a[1][0].cpu()], a[2].cpu(), a[3].cpu())
    rdet, rlink, rnew, rend = g["det"][t], g["link"][t:t + 1], g["new"][t], g["end"][t]
    mil, obj, y = lp_ref.milp_solve(rdet, [rlink], rnew, rend, [n, m])
    _, obj2, _ = lp_ref.milp_solve(rdet, [rlink], rnew, rend, [n, m], exclude=y)
    perturb = float((det[t].cpu() - rdet).abs().sum() + (link[0][t].cpu() - rlink[0]).abs().sum()
                    + (new[t].cpu() - rnew).abs().sum() + (end[t].cpu() - rend).abs().sum())
    same = all(torch.equal(p, q) for p, q in ((a[0], mil[0]), (a[1][0], mil[1][0]), (a[2], mil[2]), (a[3], mil[3])))
    print(f"{name}: LP gap {obj - obj2:.3e}, perturbation {perturb:.3e}, identical {same}")
    if obj - obj2 > perturb:
        assert same


@gpu
@pytest.mark.parametrize("eng", ["auto", "fp32", "tcgen05"])
def test_forward_batch_equals_looped_forward(eng):
    """Three pairs in one forward_batch == each pair through forward, bit for bit, at L = 6 and L = 16 on 64 x 64 crops:
    auto mode takes the FP32 engine for L*H*W = 24576 < 32768 and the tensor cores for 65536."""
    arch = "resnet50"
    sd = synthetic_state_dict("C", seed=23, appear_arch=arch)
    net = net_of(arch, "C", sd, affinity_op="minus_abs", softmax_mode="dual_add").cuda()
    mmmot_b200.set_engine(eng)
    try:
        for n in (3, 8):
            crops, pts, split = synthetic_batch(3, n, pts=16, hw=64, seed=70 + n)
            o = net.forward_batch(crops.cuda(), pts.cuda(), split, n, keep_feats=True)
            L = 2 * n
            for b in range(3):
                d, info, sp = synthetic_pair(n, n, 16, 64, seed=70 + n + b)
                det, link, new, end, _ = net(d.cuda(), {k: v.cuda() for k, v in info.items()}, sp)
                assert torch.equal(o["link"][b], link[0]) and torch.equal(o["det"][b], det)
                assert torch.equal(o["new"][b], new[:, n:]) and torch.equal(o["end"][b], end[:, :n])
            assert o["feats"].shape == (3, 3, 512, L)
    finally:
        mmmot_b200.set_engine("auto")
