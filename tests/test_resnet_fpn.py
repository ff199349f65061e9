"""Nets with a ResNet-50/101/152 appearance trunk and the FPN head (reference appear_arch resnetXX with
appear_skippool False, appear_fpn True: modules/appear_net.py:83-104,192-210), from the checkpoint to the kernels.

CPU: each arch's state_dict against the reference's own key -> shape list (tests/golden/resnet_fpn/, written by
oracle/make_resnet_fpn_goldens.py from the UNMODIFIED reference); strict loads; the identity the head is computed by
(the literal bilinear top-down chain + avgpool == the sum of the per-level means, for H and W multiples of 32), in fp64,
also on the reference's own AppearanceNet where a reference checkout is present; the BatchNorm folds and the packed
tiles; workspace queries and argument checks that need no device; the constructor's guards.

GPU, on both engines: every lateral shape and the head against fp64 through mmmot_debug_fpn_op; the whole appearance
stage against an fp64 restatement with the literal interpolate chain; the forward against the reference fixtures;
forward_batch bit-identical to looped forward, with odd L at 224 x 224 (image boundaries inside the laterals' 32-column
chunks) and L on each side of auto mode's engine switch at 64 x 64.
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
from mmmot_b200.schema import RES_SKIP_CHANNELS, RESNET_BLOCKS, resnet_convs, state_schema
from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from mmmot_b200.weights import prepare_fpn

gpu = pytest.mark.gpu
FPN = os.path.join(GOLDEN_DIR, "resnet_fpn")
EVAL = [torch.load(f) for f in sorted(glob.glob(os.path.join(FPN, "fpn*.pt")))]
ARCHS = tuple(RESNET_BLOCKS)


def fpn_sd(arch, seed, fusion="C"):
    return synthetic_state_dict(fusion, seed=seed, appear_arch=arch, appear_head="fpn")


def net_of(arch, fusion, sd, **kw):
    kw = dict(dict(affinity_op="multiply", softmax_mode="none", neg_threshold=0.2), **kw)
    net = mmmot_b200.TrackingNet(2, appear_skippool=False, appear_fpn=True, appear_arch=arch, score_arch="branch_cls",
                                 score_fusion_arch=fusion, test_mode=2, dropblock=0, **kw)
    net.load_state_dict(sd, strict=True)
    return net.eval()


def fpn_chain64(feats, lat):
    """The reference's head up to avgpool, literally (appear_net.py:192-210): lat(k, f) the lateral of level k."""
    out = lat(3, feats[3])
    for k in (2, 1, 0):
        c = lat(k, feats[k])
        out = F.interpolate(out, size=c.shape[2:], mode="bilinear", align_corners=False) + c
    return out.mean(dim=(2, 3))


def bn64(sd, p, x):
    g = lambda k: sd[f"{p}.{k}"].double().to(x.device)
    return F.batch_norm(x, g("running_mean"), g("running_var"), g("weight"), g("bias"), False, 0.0, 1e-5)


def lateral64(sd, k, f):
    w = sd[f"appearance.fpn_in.{k}.0.weight"].double().to(f.device)
    return F.relu(bn64(sd, f"appearance.fpn_in.{k}.1", F.conv2d(f, w)))


def head64(sd, v):
    """conv_last.1 + conv_last.2 + ReLU on the pooled [n][512]."""
    w = sd["appearance.conv_last.1.weight"].double().to(v.device)
    b = sd["appearance.conv_last.1.bias"].double().to(v.device)
    return F.relu(bn64(sd, "appearance.conv_last.2", F.conv2d(v[:, :, None, None], w, b))).flatten(1)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("arch", ARCHS)
def test_state_dict_matches_reference_schema(arch):
    ref = json.load(open(os.path.join(FPN, f"schema_{arch}.json")))
    sch = state_schema("C", 3, arch, "fpn")
    assert [[k, list(s)] for k, (s, _) in sch.items()] == ref
    net = mmmot_b200.TrackingNet(2, appear_skippool=False, appear_fpn=True, appear_arch=arch, score_arch="branch_cls")
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
    res = net.load_state_dict(fpn_sd(arch, 3), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert not any("global_pool" in k for k in sch)
    vgg = state_schema("C")
    assert {k: v for k, v in sch.items() if not k.startswith("appearance.")} == \
        {k: v for k, v in vgg.items() if not k.startswith("appearance.")}
    skip = state_schema("C", 3, arch)
    assert [k for k in sch if k.startswith("appearance.layers.")] == [k for k in skip if k.startswith("appearance.layers.")]


def test_default_schema_and_draws_unchanged():
    for arch in ("vgg",) + ARCHS:
        assert state_schema("C", 3, arch) == state_schema("C", 3, arch, "skippool")
        a, b = synthetic_state_dict("C", seed=9, appear_arch=arch), synthetic_state_dict("C", 9, 3, arch, "skippool")
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    for bad in (("vgg", "fpn"), ("resnet50", "pooled")):
        with pytest.raises(ValueError):
            state_schema("C", 3, *bad)


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (96, 160), (224, 224)])
def test_top_down_chain_is_sum_of_level_means(H, W):
    """With H, W multiples of 32 every interpolate is an exact 2x bilinear upsample (align_corners=False), whose every
    source row and column gets total weight 2, so the global mean of the chain is the sum of the levels' means."""
    g = torch.Generator().manual_seed(H * 1000 + W)
    lv = [torch.rand(2, 8, H >> (k + 2), W >> (k + 2), generator=g, dtype=torch.float64) * (k + 1) for k in range(4)]
    got = fpn_chain64(lv, lambda k, f: f)
    ident = sum(x.mean(dim=(2, 3)) for x in lv)
    assert float((got - ident).abs().max() / ident.abs().max()) < 1e-14


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (96, 160), (224, 224)])
def test_reference_appearance_net_is_sum_of_level_means(H, W):
    """The reference's own AppearanceNet (resnet50, FPN head, random BatchNorm statistics) in fp64 against the trunk's
    four stage outputs through Σ_k mean(lateral_k) + conv_last."""
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("no reference checkout (MMMOT_REFERENCE)")
    from oracle import make_resnet_fpn_goldens as mfg
    net = mfg.reference_net("resnet50", "C", "minus_abs", "dual_add", 0.2)
    sd = fpn_sd("resnet50", 5)
    net.load_state_dict(sd, strict=True)
    app = net.appearance.double().eval()
    x = torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(H + W), dtype=torch.float64)
    with torch.no_grad():
        ref = app(x)
        feats = app.layers(x, return_feature_maps=True)
        got = head64(sd, sum(lateral64(sd, k, f).mean(dim=(2, 3)) for k, f in enumerate(feats)))
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-12


def _unpack(packed, scale, M, K):
    """pack_tc's tiles -> (hi + lo) * scale as W [M][K] fp64 (the inverse of the packing permutation)."""
    mt, kc = (M + 127) // 128, (K + 31) // 32
    t = packed.view(torch.float16).view(kc, mt, 2, 4, 16, 8, 8).permute(2, 1, 4, 5, 0, 3, 6).reshape(2, mt * 128, kc * 32)
    return (t[0].double() + t[1].double()) * scale


def test_fpn_folds_and_packing_vs_fp64():
    sd = fpn_sd("resnet50", 4)
    lats, (wl, bl) = prepare_fpn(sd)
    g = torch.Generator().manual_seed(6)
    for k, c in enumerate(RES_SKIP_CHANNELS):
        wt, b, packed, scale = lats[k]
        assert wt.shape == (c, 512) and b.shape == (512,)
        x = torch.randn(2, c, 3, 5, generator=g, dtype=torch.float64)
        ref = bn64(sd, f"appearance.fpn_in.{k}.1", F.conv2d(x, sd[f"appearance.fpn_in.{k}.0.weight"].double()))
        got = torch.einsum("kc,nkhw->nchw", wt.double(), x) + b.double()[:, None, None]
        assert relerr(got, ref) < 1e-6, k
        Wu = _unpack(packed, scale, 512, c)
        assert float((Wu - wt.double().t()).abs().max()) <= 2.0 ** -22 * float(wt.abs().max()), k
    v = torch.randn(3, 512, generator=g, dtype=torch.float64)
    ref = head64(sd, v)
    got = torch.relu(v @ wl.double() + bl.double())
    assert relerr(got, ref) < 1e-6


def test_workspace_and_argument_checks(lib_built):
    lib = _lib.load()
    ws = lib.mmmot_appearance_resnet_fpn_workspace(16, 64, 64, 4)
    assert ws > lib.mmmot_appearance_resnet_workspace(16, 64, 64)
    assert lib.mmmot_appearance_resnet_fpn_workspace(16, 224, 224, 4) > ws
    assert lib.mmmot_appearance_resnet_fpn_workspace(16, 64, 64, 0) == 0
    fake = lambda a: ctypes.c_void_p(a)
    rw = _lib.ResnetWeights()
    rw.blocks[:] = RESNET_BLOCKS["resnet50"]
    fw = _lib.FpnWeights()
    P = lambda s: ctypes.pointer(s) if s is not None else None
    ws4 = lib.mmmot_appearance_resnet_fpn_workspace(4, 64, 64, 2)          # exactly what the calls below carve
    args = lambda r, f, n=4, H=64, W=64, L=2, nb=ws4: (P(r), P(f), fake(4096), n, H, W, L, fake(8192), fake(1 << 20), nb,
                                                      None)
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(None, fw)) == -1
    bad = _lib.ResnetWeights()
    bad.blocks[:] = (0, 4, 6, 3)
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(bad, fw)) == -1
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw, H=48)) == -3
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw, W=80)) == -3
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw, n=5, L=2)) == -3
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw, L=0)) == -1
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw)) == -1              # no conv pointers
    for i in range(1 + 3 * 16 + 4):
        rw.wt[i] = rw.bias[i] = rw.wp[i] = 4096
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, None)) == -1
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw)) == -1              # no FPN pointers
    for k in range(4):
        fw.lat_wt[k] = fw.lat_bias[k] = fw.lat_wp[k] = 4096
    fw.last_wt = fw.last_bias = 4096
    assert lib.mmmot_appearance_resnet_fpn_fwd(*args(rw, fw, nb=ws4 - 1)) == -2
    # the test hook
    hook = lambda op, f, level=0, n=4, h=16, w=16, L=2, nb=ws4: lib.mmmot_debug_fpn_op(op, P(f), level, n, h, w, L, fake(4096),
                                                                                    fake(8192), fake(1 << 20), nb, None)
    assert hook(2, fw) == -1 and hook(-1, fw) == -1 and hook(0, None) == -1 and hook(1, None) == -1
    assert hook(0, fw, level=4) == -1 and hook(0, fw, n=5) == -1 and hook(0, fw, L=0) == -1
    assert hook(0, fw, nb=ws4 - 1) == -2 and hook(0, fw, level=2, h=4, w=4, nb=ws4 - 1) == -2
    names = [lib.mmmot_timing_tag_name(t).decode() for t in range(lib.mmmot_timing_tag_count())]
    assert [n for n in names if n.startswith("fpn.")] == ["fpn.lateral", "fpn.head"]


def test_constructor_guards():
    for arch in ARCHS:
        net = mmmot_b200.TrackingNet(2, appear_skippool=False, appear_fpn=True, appear_arch=arch, score_arch="branch_cls")
        assert net.appear_head == "fpn"
    for kw in (dict(appear_arch="vgg", appear_skippool=False, appear_fpn=True), dict(appear_arch="vgg", appear_skippool=False),
               dict(appear_arch="resnet50", appear_skippool=True, appear_fpn=True),
               dict(appear_arch="resnet152", appear_skippool=False, appear_fpn=False),
               dict(appear_arch="resnet34", appear_skippool=False, appear_fpn=True)):
        with pytest.raises(NotImplementedError):
            mmmot_b200.TrackingNet(2, score_arch="branch_cls", **kw)
    net = net_of("resnet50", "C", fpn_sd("resnet50", 1)).train()
    dets, info, split = synthetic_pair(2, 2, 6, 32, seed=1)
    with pytest.raises(NotImplementedError, match="training-mode"):
        net(dets, info, split)
    cfg = dict(sample_max_len=2, without_reflectivity=True, dropblock=5, use_dropout=False,
               model=dict(point_arch="v1", point_len=512, appear_arch="resnet101", appear_len=512, appear_skippool=False,
                          appear_fpn=True, end_arch="v2", end_mode="avg", affinity_op="minus_abs", softmax_mode="dual_max",
                          score_arch="branch_cls", neg_threshold=0.2, score_fusion_arch="B", test_mode=2))
    net = mmmot_b200.build_model({"common": cfg})
    assert net.appear_arch == "resnet101" and net.appear_head == "fpn"


def test_fixture_set_covers_the_cases():
    cases = {(g["case"][1], g["case"][2], g["case"][3], g["case"][4], g["case"][9]) for g in EVAL}
    assert cases == {("resnet50", "C", "minus_abs", "dual_add", 64), ("resnet101", "A", "multiply", "none", 64),
                     ("resnet152", "B", "minus_abs", "dual_max", 64), ("resnet50", "C", "minus_abs", "dual_add", 224)}
    assert all(g["case"][6] != g["case"][7] for g in EVAL)
    assert all(os.path.getsize(f) < 150_000 for f in glob.glob(os.path.join(FPN, "*")))


def test_reference_fpn_net_builds_offline():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("no reference checkout (MMMOT_REFERENCE)")
    from oracle import make_resnet_fpn_goldens as mfg
    from oracle import make_resnet_goldens as mrg
    before = len(mrg.BLOCKED)
    for arch in ARCHS:
        net = mfg.reference_net(arch, "C", "minus_abs", "dual_add", 0.2)
        ref = json.load(open(os.path.join(FPN, f"schema_{arch}.json")))
        assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
    assert len(mrg.BLOCKED) == before == 0


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(params=["fp32", "tcgen05"])
def engine(request):
    mmmot_b200.set_engine(request.param)
    yield request.param
    mmmot_b200.set_engine("auto")


def _fold64(sd, conv, bn):
    w = sd[f"{conv}.weight"].double()
    return lambda x, stride, pad: bn64(sd, bn, F.conv2d(x, w.to(x.device), stride=stride, padding=pad))


def fpn_stage64(sd, arch, crops):
    """fp64 restatement of the ResNet trunk + FPN head (eval) with torch.nn.functional and the literal interpolate
    chain: stack 0 [n][512]."""
    x = crops.double()
    spec = resnet_convs(arch)
    f = lambda i, x: _fold64(sd, spec[i][0], spec[i][1])(x, spec[i][5], spec[i][4] // 2)
    x = F.max_pool2d(F.relu(f(0, x)), 3, 2, 1)
    i, feats = 1, []
    for s, nb in enumerate(RESNET_BLOCKS[arch]):
        for b in range(nb):
            y = f(i + 2, F.relu(f(i + 1, F.relu(f(i, x)))))
            idt = f(i + 3, x) if b == 0 else x
            x = F.relu(y + idt)
            i += 4 if b == 0 else 3
        feats.append(x)
    return head64(sd, fpn_chain64(feats, lambda k, t: lateral64(sd, k, t)))


@gpu
@pytest.mark.parametrize("hw", [64, 224])
@pytest.mark.parametrize("level", [0, 1, 2, 3])
def test_lateral_vs_fp64(level, hw, engine):
    """One lateral (K = 256 << level -> 512, folded BatchNorm, ReLU) reduced to per-image means, through the hook, on
    3 images of the level's size at hw x hw crops, L = 3 (one pair; at 224 image boundaries fall inside 32-column
    chunks).  Bound: the mean of the per-element bounds (ReLU is 1-Lipschitz; tensor cores: TAU |W||x|, FP32 engine:
    kernel_kit.contraction_bound) plus an fp32 chain of hw terms for the mean."""
    from kernel_kit import TAU, U, contraction_bound, fp16_split, report, vp, worst_ratio
    lib = _lib.load()
    net = net_of("resnet50", "C", fpn_sd("resnet50", 30 + level)).cuda()
    wts = net.prepared()
    lats, _ = prepare_fpn(net.state_dict())
    wt, b = lats[level][0].double().cuda(), lats[level][1].double().cuda()
    n, L, C, h = 3, 3, 256 << level, hw >> (level + 2)
    g = torch.Generator().manual_seed(1000 * level + hw)
    x = (torch.rand(n, C, h, h, generator=g) * 2).cuda()            # a stage output: non-negative
    nbytes = lib.mmmot_appearance_resnet_fpn_workspace(n, hw, hw, L)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    assert lib.mmmot_status_reset(vp(ws), None) == 0
    Y = torch.full((n * 512 + 256,), float("nan"), device="cuda")
    cols = lambda t: t.permute(1, 0, 2, 3).reshape(C, n * h * h)    # [C][n*hw]
    if engine == "tcgen05":
        hi, lo = fp16_split(x.permute(0, 2, 3, 1).contiguous())
        X = torch.stack([hi.reshape(-1), lo.reshape(-1)]).contiguous()
        xe = cols((hi.double() + lo.double()).permute(0, 3, 1, 2))
        ref = (wt.t() @ xe + b[:, None])
        T = TAU * (wt.abs().t() @ xe.abs() + b.abs()[:, None])
        ref = ref.clamp_min(0)
    else:
        X = cols(x).contiguous()
        ref, T = contraction_bound(wt, cols(x.double()), b, relu=True)
    rc = lib.mmmot_debug_fpn_op(0, wts.fptr, level, n, h, h, L, vp(X), vp(Y), vp(ws), nbytes, None)
    torch.cuda.synchronize()
    assert rc == 0
    assert lib.mmmot_status_check(vp(ws), None) == 0
    assert bool(torch.isnan(Y[n * 512:]).all())
    hw2 = h * h
    per = lambda t: t.view(512, n, hw2).mean(-1).t()                # [n][512]
    mref = per(ref)
    Tm = per(T) + 1.01 * U * ((hw2 + 6) * per(ref.abs()) + mref.abs()) + 2.0 ** -30
    r = worst_ratio(Y[:n * 512].view(n, 512).double(), mref, Tm)
    report(f"fpn lateral {level} K={C} {h}x{h} [{engine}] (err / bound)", mean=r)
    assert r <= 1.0, r


@gpu
def test_head_vs_fp64(engine):
    """Level sum + conv_last (folded) + ReLU through the hook against fp64: an fp32 chain of 512 terms after a 4-term
    sum, |err| <= 1.01 u (sum_c |w_c| |v_c| (c + 4) + |b|) + the sum's own rounding."""
    from kernel_kit import U, report, vp, worst_ratio
    lib = _lib.load()
    sd = fpn_sd("resnet101", 40)
    net = net_of("resnet101", "C", sd).cuda()
    wts = net.prepared()
    _, (wl, bl) = prepare_fpn(net.state_dict())
    n, L = 6, 3
    means = (torch.rand(4, n, 512, generator=torch.Generator().manual_seed(7)) * 3).cuda()
    feats = torch.full((n // L, 3, 512, L), float("nan"), device="cuda")
    rc = lib.mmmot_debug_fpn_op(1, wts.fptr, 0, n, 0, 0, L, vp(means), vp(feats), None, 0, None)
    torch.cuda.synchronize()
    assert rc == 0
    assert bool(torch.isnan(feats[:, 1:]).all())
    got = feats[:, 0].permute(0, 2, 1).reshape(n, 512).double()
    v = means.double().sum(0)
    w, b = wl.double().cuda(), bl.double().cuda()
    ref = torch.relu(v @ w + b)
    k = torch.arange(1, 513, dtype=torch.float64, device="cuda")
    T = 1.01 * U * ((v.abs()[:, :, None] * w.abs() * (k[:, None] + 4)).sum(1) + b.abs()) + 2.0 ** -40
    r = worst_ratio(got, ref, T)
    report(f"fpn head [{engine}] (err / bound)", head=r)
    assert r <= 1.0, r


@gpu
@pytest.mark.parametrize("arch,H,W,L", [("resnet50", 64, 64, 6), ("resnet101", 64, 64, 4), ("resnet152", 64, 64, 4),
                                        ("resnet50", 224, 224, 3), ("resnet152", 224, 224, 2), ("resnet50", 64, 96, 5)])
def test_fpn_stage_vs_fp64(arch, H, W, L, engine):
    """mmmot_appearance_resnet_fpn_fwd's stack 0 against fp64 with the literal interpolate chain, max-norm relative error
    per image; the status word stays clear."""
    from kernel_kit import vp
    lib = _lib.load()
    sd = fpn_sd(arch, 21)
    net = net_of(arch, "C", sd).cuda()
    wts = net.prepared()
    g = torch.Generator().manual_seed(H + W + L)
    crops = (torch.randn(L, 3, H, W, generator=g) + torch.randn(L, 3, 1, 1, generator=g)).cuda()
    feats = torch.full((1, 3, 512, L), float("nan"), device="cuda")
    nbytes = lib.mmmot_appearance_resnet_fpn_workspace(L, H, W, L)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    assert lib.mmmot_status_reset(vp(ws), None) == 0
    rc = lib.mmmot_appearance_resnet_fpn_fwd(wts.rptr, wts.fptr, vp(crops), L, H, W, L, vp(feats), vp(ws), nbytes, None)
    assert rc == 0
    assert lib.mmmot_status_check(vp(ws), None) == 0
    got = feats[0, 0].T
    assert bool(torch.isfinite(got).all()) and bool(torch.isnan(feats[0, 1:]).all())
    ref = fpn_stage64({k: v.cuda() for k, v in sd.items()}, arch, crops)
    err = max(relerr(got[i], ref[i]) for i in range(L))
    print(f"\nresnet fpn {arch} {H}x{W} [{engine}]: max-norm rel err {err:.3g}")
    assert err < TOL, err


@gpu
@pytest.mark.parametrize("g", EVAL, ids=[c["case"][0] for c in EVAL])
def test_forward_matches_reference_golden(g, engine):
    from oracle import lp_ref
    name, arch, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = g["case"]
    net = net_of(arch, fusion, fpn_sd(arch, seed, fusion), affinity_op=op, softmax_mode=sm, neg_threshold=thr).cuda()
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
    """Three pairs in one forward_batch == each pair through forward, bit for bit: (n, m) = (2, 1) on 224 x 224 crops
    (L = 3: 9408, 2352 and 147 pixels per pair on the four levels, so the second and third pairs start inside a
    256-column tile of a uniform tiling), and (3, 2) / (5, 4) on 64 x 64 (L*H*W = 20480 < 32768 <= 36864: auto mode
    takes the FP32 engine for the first, the tensor cores for the second)."""
    arch = "resnet50"
    net = net_of(arch, "C", fpn_sd(arch, 23), affinity_op="minus_abs", softmax_mode="dual_add").cuda()
    mmmot_b200.set_engine(eng)
    try:
        for n, m, hw in ((2, 1, 224), (3, 2, 64), (5, 4, 64)):
            pairs = [synthetic_pair(n, m, 16, hw, seed=80 + n + b) for b in range(3)]
            crops = torch.cat([p[0] for p in pairs]).cuda()
            pts = torch.cat([p[1]["points"][0] for p in pairs]).cuda()
            sp, off = [torch.zeros(1, dtype=torch.int64)], 0
            for p in pairs:
                s = p[1]["points_split"][0].long()
                sp.append(s[1:] + off)
                off += int(s[-1])
            o = net.forward_batch(crops, pts, torch.cat(sp), n, m, keep_feats=True)
            assert int(o["status"]) == 0
            for b, (d, info, split) in enumerate(pairs):
                det, link, new, end, _ = net(d.cuda(), {k: v.cuda() for k, v in info.items()}, split)
                assert torch.equal(o["link"][b], link[0]) and torch.equal(o["det"][b], det), (n, m, hw, b)
                assert torch.equal(o["new"][b], new[:, n:]) and torch.equal(o["end"][b], end[:, :n])
            assert o["feats"].shape == (3, 3, 512, n + m)
    finally:
        mmmot_b200.set_engine("auto")
