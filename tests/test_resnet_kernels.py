"""The ResNet trunk's kernels (csrc/resnet.cu), each on its own inputs against fp64, through mmmot_debug_resnet_op, which
runs every launch kind through the code mmmot_appearance_resnet_fwd runs, on both engines.

  gathers (the stem's 7x7 taps of the crops, the strided 1x1 / 3x3 taps of the activations) and the 3x3 / 2 max-pool:
      bit-exact (they copy values, or split them into the FP16 (hi, lo) pair as fp16_split does);
  contractions at every (Cin, M, kernel, stride) of ResNet-50/101/152, the stem included: tensor cores within
      TAU * S (S = |W| |X| + |b|, kernel_kit.TAU; the K >= 2304 3x3 convs K-segmented as in the trunk), the FP32 engine
      within kernel_kit.contraction_bound;
  residual add + ReLU: one fp32 rounding and the FP16 split; the FP16 range flag on a sum >= 65504 and on NaN;
  per-image plane means; the wide SkipPool heads (C = 256 .. 2048, mid = C / 4) against F.group_norm / F.conv2d in fp64
      to a bound derived like tests/test_heads.py's, with the reduction depth of the 512-thread kernel.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_kit import TAU, U, EPS, case_seed, contraction_bound, fp16_split, lib_state, report, vp, worst_ratio
from mmmot_b200 import _lib
from mmmot_b200.schema import RESNET_BLOCKS, resnet_convs
from mmmot_b200.synthetic import synthetic_state_dict
from mmmot_b200.weights import pack_tc

gpu = pytest.mark.gpu
ENGINES = ["tc", "fp32"]
OP = dict(gather=0, stem_gather=1, stem=2, conv=3, maxpool=4, add_relu=5, mean=6, heads=7)
# every (Cin, M, kernel, stride) of the three trunks' convs after the stem
CONV_SHAPES = sorted({(cin, cout, k, s) for a in RESNET_BLOCKS for _, _, cin, cout, k, s in resnet_convs(a)[1:]})


def op(lib, name, *, rw=None, conv=0, n=1, H=1, W=1, C=0, ks=1, stride=1, M=0, relu=0, L=1, X=None, id=None, Y=None,
       cols=None, kseg=None, status=None):
    rwp = ctypes.pointer(rw) if rw is not None else None
    rc = lib.mmmot_debug_resnet_op(OP[name], rwp, conv, n, H, W, C, ks, stride, M, relu, L, vp(X), vp(id), vp(Y), vp(cols),
                                   vp(kseg), vp(status), None)
    torch.cuda.synchronize()
    return rc


def guarded(count, dtype=torch.float32):
    """count elements + a NaN guard band (0xFFFF for fp16)."""
    return torch.full((count + 256,), float("nan"), dtype=dtype, device="cuda")


def planes(x_nhwc):
    """fp32 NHWC -> the (hi, lo) planes [2][numel] fp16 and their value hi + lo (fp64, same shape)."""
    hi, lo = fp16_split(x_nhwc)
    return torch.stack([hi.reshape(-1), lo.reshape(-1)]).contiguous(), hi.double() + lo.double()


def taps(x_nchw, ks, stride):
    """[n][C][H][W] -> the conv's taps [K = ks*ks*C][n*Ho*Wo], k = (ky*ks+kx)*C + ci, zero padding ks // 2."""
    n, C = x_nchw.shape[:2]
    u = F.unfold(x_nchw, ks, padding=ks // 2, stride=stride)            # [n][C*ks*ks][P], (ci, ky, kx)
    P = u.shape[-1]
    return u.view(n, C, ks * ks, P).permute(2, 1, 0, 3).reshape(ks * ks * C, n * P)


def rw_with(i, wt, b):
    """A weight struct holding one conv at index i: fp32 Wt [K][M] (FP32 engine), its packed tiles (tensor cores), bias.
    Returns (struct, tensors to keep alive)."""
    packed, scale = pack_tc(wt)
    wt_d, b_d, p_d = wt.float().cuda().contiguous(), b.float().cuda().contiguous(), packed.cuda()
    rw = _lib.ResnetWeights()
    rw.wt[i], rw.bias[i], rw.wp[i] = wt_d.data_ptr(), b_d.data_ptr(), p_d.data_ptr()
    rw.wp_scale[i] = scale
    return rw, (wt_d, b_d, p_d)


# ------------------------------------------------------------------------------------------------ CPU
def test_conv_shapes_cover_the_trunks():
    assert (64, 64, 1, 1) in CONV_SHAPES and (64, 256, 1, 1) in CONV_SHAPES      # layer1 conv1, downsample
    assert (128, 128, 3, 2) in CONV_SHAPES and (512, 512, 3, 2) in CONV_SHAPES     # strided conv2
    assert (1024, 2048, 1, 2) in CONV_SHAPES and (512, 512, 3, 1) in CONV_SHAPES   # strided downsample, K = 4608
    assert all(c % 32 == 0 and m % 64 == 0 for c, m, _, _ in CONV_SHAPES)


def test_hook_rejects_bad_arguments(lib_built):
    lib = _lib.load()
    f = lambda a: ctypes.c_void_p(a)
    rw = _lib.ResnetWeights()
    call = lambda o, **k: lib.mmmot_debug_resnet_op(o, ctypes.pointer(rw), k.get("conv", 0), k.get("n", 2), k.get("H", 8),
                                                    k.get("W", 8), k.get("C", 64), k.get("ks", 3), k.get("stride", 2),
                                                    k.get("M", 64), 1, k.get("L", 2), f(4096), f(8192), f(12288), f(16384),
                                                    None, None, None)
    assert call(8) == -1 and call(-1) == -1
    assert call(0, C=48) == -1 and call(0, ks=5) == -1 and call(0, stride=3) == -1 and call(0, H=7) == -1
    assert call(3) == -1                                    # no weights at conv 0
    assert call(4, C=128) == -1 and call(7, L=3) == -1 and call(6, C=4096) == -1


# ------------------------------------------------------------------------------------------------ GPU
@gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("C,ks,stride,H", [(64, 3, 1, 16), (128, 3, 2, 16), (256, 1, 2, 8), (512, 3, 2, 8), (1024, 1, 2, 4)])
def test_gather_exact(C, ks, stride, H, engine):
    lib = _lib.load()
    n = 3
    g = torch.Generator().manual_seed(case_seed("resnet gather", C, ks, stride, H))
    x = torch.randn(n, C, H, H, generator=g)
    Ho = H // stride
    K, P = ks * ks * C, n * Ho * Ho
    with lib_state(lib, engine=engine):
        if engine == "tc":
            X, xv = planes(x.permute(0, 2, 3, 1).contiguous())
            Y = guarded(2 * P * K, torch.float16)
            assert op(lib, "gather", n=n, H=H, W=H, C=C, ks=ks, stride=stride, X=X.cuda(), Y=Y) == 0
            hi, lo = fp16_split(x.permute(0, 2, 3, 1).contiguous())
            for pl, ref in enumerate((hi, lo)):
                want = taps(ref.float().permute(0, 3, 1, 2), ks, stride).t().contiguous()      # [P][K]
                assert torch.equal(Y[pl * P * K:(pl + 1) * P * K].view(P, K).cpu().float(), want), pl
            assert bool(torch.isnan(Y[2 * P * K:].float()).all())
        else:
            X = x.permute(1, 0, 2, 3).contiguous().cuda()           # [C][n][H][W]
            Y = guarded(K * P)
            assert op(lib, "gather", n=n, H=H, W=H, C=C, ks=ks, stride=stride, X=X, Y=Y) == 0
            assert torch.equal(Y[:K * P].view(K, P).cpu(), taps(x, ks, stride))
            assert bool(torch.isnan(Y[K * P:]).all())


@gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_stem_gather_exact_and_range_flag(engine):
    lib = _lib.load()
    n, H = 2, 32
    x = torch.randn(n, 3, H, H, generator=torch.Generator().manual_seed(11)) * 3
    P = n * (H // 2) ** 2
    want = taps(x, 7, 2)                                            # [147][P], k = (ky*7+kx)*3 + ci
    with lib_state(lib, engine=engine):
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        if engine == "tc":
            Y = guarded(2 * P * 160, torch.float16)
            assert op(lib, "stem_gather", n=n, H=H, W=H, X=x.cuda(), Y=Y, status=status) == 0
            hi, lo = fp16_split(torch.cat([want.t(), torch.zeros(P, 13)], 1).contiguous())
            assert torch.equal(Y[:P * 160].view(P, 160).cpu(), hi) and torch.equal(Y[P * 160:2 * P * 160].view(P, 160).cpu(), lo)
            assert int(status) == 0
            x[1, 2, 5, 7] = 70000.0                                 # outside FP16's range: flagged, not silently clamped
            assert op(lib, "stem_gather", n=n, H=H, W=H, X=x.cuda(), Y=Y, status=status) == 0
            assert int(status) & 1
        else:
            Y = guarded(147 * P)
            assert op(lib, "stem_gather", n=n, H=H, W=H, X=x.cuda(), Y=Y) == 0
            assert torch.equal(Y[:147 * P].view(147, P).cpu(), want) and bool(torch.isnan(Y[147 * P:]).all())


@gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("H", [16, 32])
def test_maxpool_exact(H, engine):
    """3x3 / 2 / pad 1: the winner's value (tensor cores: its (hi, lo) pair) exactly; negative inputs make the -inf
    padding matter at the borders."""
    lib = _lib.load()
    n, C = 2, 64
    x = torch.randn(n, C, H, H, generator=torch.Generator().manual_seed(H)) - 0.5
    Ho = H // 2
    with lib_state(lib, engine=engine):
        if engine == "tc":
            X, xv = planes(x.permute(0, 2, 3, 1).contiguous())
            Y = guarded(2 * n * Ho * Ho * C, torch.float16)
            assert op(lib, "maxpool", n=n, H=H, W=H, C=C, X=X.cuda(), Y=Y) == 0
            m = n * Ho * Ho * C
            v = xv.permute(0, 3, 1, 2)
            ref, idx = F.max_pool2d(v, 3, 2, 1, return_indices=True)
            hi, lo = (X[p].view(n, H, H, C).permute(0, 3, 1, 2).reshape(n, C, -1) for p in (0, 1))
            whi = hi.gather(2, idx.reshape(n, C, -1)).view(n, C, Ho, Ho).permute(0, 2, 3, 1).reshape(-1)
            wlo = lo.gather(2, idx.reshape(n, C, -1)).view(n, C, Ho, Ho).permute(0, 2, 3, 1).reshape(-1)
            assert torch.equal(Y[:m].cpu(), whi) and torch.equal(Y[m:2 * m].cpu(), wlo)
            assert bool(torch.isnan(Y[2 * m:].float()).all())
        else:
            X = x.permute(1, 0, 2, 3).contiguous().cuda()
            Y = guarded(C * n * Ho * Ho)
            assert op(lib, "maxpool", n=n, H=H, W=H, C=C, X=X, Y=Y) == 0
            want = F.max_pool2d(x, 3, 2, 1).permute(1, 0, 2, 3).reshape(-1)
            assert torch.equal(Y[:want.numel()].cpu(), want)


def _conv_case(lib, engine, i, wt, b, x, ks, stride, relu):
    """Runs conv (op 3, or the stem, op 2, at i = 0 with ks = 7) of x [n][C][H][W] fp32 -> (y [M][P] fp64, ref, bound)."""
    n, C, H, W = x.shape
    K, M = wt.shape
    Ho, Wo = H // stride, W // stride
    P = n * Ho * Wo
    rw, keep = rw_with(i, wt, b)
    cols = torch.empty(2 * 40 * n * H * W + 2 * P * K + 1024, dtype=torch.float32, device="cuda")
    kseg = torch.empty(64 * 256 * M, dtype=torch.float32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    name = "stem" if ks == 7 else "conv"
    kw = dict(rw=rw, conv=i, n=n, H=H, W=W, C=C, ks=ks, stride=stride, M=M, relu=relu, cols=cols, kseg=kseg, status=status)
    if engine == "tc":
        X, xv = planes(x.permute(0, 2, 3, 1).contiguous())
        xeff = xv.permute(0, 3, 1, 2)
        Y = guarded(2 * P * M, torch.float16)
        assert op(lib, name, X=X.cuda() if ks != 7 else x.cuda(), Y=Y, **kw) == 0
        assert bool(torch.isnan(Y[2 * P * M:].float()).all())
        y = (Y[:P * M].double() + Y[P * M:2 * P * M].double()).view(P, M).t()
        if ks == 7:
            xeff = sum(t.double() for t in fp16_split(x))
        Xc = taps(xeff, ks, stride).cuda()
        ref = wt.double().cuda().t() @ Xc + b.double().cuda()[:, None]
        S = wt.double().abs().cuda().t() @ Xc.abs() + b.double().abs().cuda()[:, None]
        ref = ref.clamp_min(0) if relu else ref
        T = TAU * S
    else:
        X = x.permute(1, 0, 2, 3).contiguous().cuda() if ks != 7 else x.cuda()
        Y = guarded(M * P)
        assert op(lib, name, X=X, Y=Y, **kw) == 0
        assert bool(torch.isnan(Y[M * P:]).all())
        y = Y[:M * P].view(M, P)
        ref, T = contraction_bound(wt.double().cuda(), taps(x.double(), ks, stride).cuda(), b.double().cuda(), relu=bool(relu))
    assert int(status) == 0
    return y, ref, T


@gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("C,M,ks,stride", CONV_SHAPES, ids=[f"{c}to{m}_k{k}s{s}" for c, m, k, s in CONV_SHAPES])
def test_conv_vs_fp64(C, M, ks, stride, engine):
    """Every conv shape of the trunks on 3 images of 8 x 8 (a partial column tile), the layer1 shapes also on 16 x 16;
    relu as the trunk uses it (conv1 / conv2 with, conv3 / downsample without)."""
    lib = _lib.load()
    relu = int(not (ks == 1 and (M > C or stride == 2)))       # conv3 and downsample: no ReLU before the add
    r = {}
    for H in ((8, 16) if C <= 256 else (8,)):
        g = torch.Generator().manual_seed(case_seed("resnet conv", C, M, ks, stride, H))
        K = ks * ks * C
        wt = torch.randn(K, M, generator=g) * (2.0 / K) ** 0.5
        b = torch.rand(M, generator=g) * 0.2 - 0.1
        x = torch.randn(3, C, H, H, generator=g).clamp_min(-0.3)
        with lib_state(lib, engine=engine):
            y, ref, T = _conv_case(lib, engine, 5, wt, b, x, ks, stride, relu)
        r[f"H{H}"] = worst_ratio(y, ref, T)
    report(f"resnet conv {C}->{M} k{ks} s{stride} relu={relu} [{engine}] (err / bound)", **r)
    assert max(r.values()) <= 1.0, r


@gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_stem_vs_fp64(engine):
    """The stem (7x7 / 2 / pad 3, K = 147; packed K 160) with bias and ReLU on 3 crops of 32 x 32 and 64 x 64."""
    lib = _lib.load()
    r = {}
    for H in (32, 64):
        g = torch.Generator().manual_seed(case_seed("resnet stem", H))
        wt = torch.randn(147, 64, generator=g) * (2.0 / 147) ** 0.5
        b = torch.rand(64, generator=g) * 0.2 - 0.1
        x = torch.randn(3, 3, H, H, generator=g) * 1.5
        with lib_state(lib, engine=engine):
            y, ref, T = _conv_case(lib, engine, 0, wt, b, x, 7, 2, 1)
        r[f"H{H}"] = worst_ratio(y, ref, T)
    report(f"resnet stem [{engine}] (err / bound)", **r)
    assert max(r.values()) <= 1.0, r


@gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_add_relu(engine):
    """relu(y + id): tensor cores within one fp32 rounding of the exact sum of the two (hi, lo) values plus the FP16 split
    of the result (2^-22 relative, 2^-25 absolute); the FP32 engine exactly torch's fp32 relu(y + id).  Range flag: a sum
    >= 65504 and a NaN sum raise it; a sum <= -65504 is stored exactly as 0 and does not."""
    lib = _lib.load()
    n, H, C = 2, 8, 256
    g = torch.Generator().manual_seed(5)
    a, b = torch.randn(n, H, H, C, generator=g) * 2, torch.randn(n, H, H, C, generator=g) * 2
    N = a.numel()
    with lib_state(lib, engine=engine):
        if engine == "fp32":
            Y, I = a.reshape(-1).cuda().clone(), b.reshape(-1).cuda()
            assert op(lib, "add_relu", n=n, H=H, W=H, C=C, Y=Y, id=I) == 0
            assert torch.equal(Y.cpu(), torch.relu(a.reshape(-1) + b.reshape(-1)))
            return
        status = torch.zeros(1, dtype=torch.int32, device="cuda")

        def run(a, b):
            A, av = planes(a)
            B, bv = planes(b)
            A = A.cuda()
            status.zero_()
            assert op(lib, "add_relu", n=n, H=H, W=H, C=C, Y=A, id=B.cuda(), status=status) == 0
            return A, (av + bv).reshape(-1), int(status)
        A, s, st = run(a, b)
        got = A[0].double() + A[1].double()
        T = 2.0 ** -24 * s.abs() + 2.0 ** -22 * s.abs() * (1 + 2.0 ** -24) + 2.0 ** -25
        ratio = worst_ratio(got.cpu(), s.clamp_min(0), T)
        assert st == 0 and ratio <= 1.0, (st, ratio)
        report("resnet add_relu [tc] (err / bound)", add_relu=ratio)
        for va, vb, flagged in ((40000.0, 40000.0, True), (-40000.0, -40000.0, False), (float("nan"), 1.0, True)):
            a2, b2 = a.clone(), b.clone()
            a2[1, 3, 4, 17], b2[1, 3, 4, 17] = va, vb
            A, _, st = run(a2, b2)
            assert bool(st & 1) == flagged, (va, vb, st)
            if not flagged:
                assert float(A[0].view(-1)[a2.reshape(-1).abs().argmax()]) == 0.0
    assert N == A.shape[1]


@gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("C,H", [(256, 16), (2048, 2), (1024, 7 * 2)])
def test_plane_means(C, H, engine):
    """Per-image channel means: each an fp32 chain of hw terms, so |err| <= 1.01 u ((hw + 6) mean|x| + |mean|)."""
    lib = _lib.load()
    n = 3
    x = torch.rand(n, C, H, H, generator=torch.Generator().manual_seed(C + H)) * 4
    with lib_state(lib, engine=engine):
        if engine == "tc":
            X, xv = planes(x.permute(0, 2, 3, 1).contiguous())
            xv = xv.permute(0, 3, 1, 2)
            X = X.cuda()
        else:
            X, xv = x.permute(1, 0, 2, 3).contiguous().cuda(), x.double()
        Y = guarded(n * C)
        assert op(lib, "mean", n=n, H=H, W=H, C=C, X=X, Y=Y) == 0
    ref = xv.mean(dim=(2, 3))
    T = 1.01 * U * ((H * H + 6) * xv.abs().mean(dim=(2, 3)) + ref.abs())
    r = worst_ratio(Y[:n * C].view(n, C).cpu(), ref, T)
    assert bool(torch.isnan(Y[n * C:]).all())
    report(f"resnet plane means C={C} {H}x{H} [{engine}] (err / bound)", mean=r)
    assert r <= 1.0, r


# ---- wide SkipPool heads: the bound of tests/test_heads.py (chain_bound, gn_propagate) with skip_head_wide's reduction
def _chain(wt, x, Tx, b):
    prod = x[:, :, None] * wt[None]
    pre = prod.cumsum(1) + b
    return pre[:, -1], Tx @ wt.abs() + 1.01 * U * pre.abs().sum(1)


def _gn(y, T, gamma, beta):
    """GroupNorm(1, C) of each row of y (fp64) with kernel errors T, as skip_head_wide_kernel forms it: per-thread
    sequential sums of ceil(C/512) values, a 5-level warp tree, 16 warp partials summed in order."""
    C = y.shape[1]
    ns = math.ceil(C / 512) + 5 + 16 + 4
    m = y.mean(1, keepdim=True)
    dev = y - m
    v = (dev * dev).sum(1, keepdim=True) / C
    tm = T.mean(1, keepdim=True) + ns * U * (y.abs() + T).mean(1, keepdim=True) + U * m.abs()
    tv = 2 * (dev.abs() * T).mean(1, keepdim=True) + ((T + tm) ** 2).mean(1, keepdim=True) + (ns + 4) * U * v
    rstd = 1 / torch.sqrt(v + EPS)
    rr = (tv + U * (v + EPS)) / (2 * (v + EPS)) + 4 * U
    zd = dev * rstd * gamma
    z = zd + beta
    return z, gamma.abs() * rstd * (T + tm + dev.abs() * (U + rr)) + 3 * U * (zd.abs() + z.abs())


def _head_ref(sd, s, x):
    p = f"appearance.global_pool.{s}.fc"
    f = lambda k: sd[f"{p}.{k}"].double().cuda()
    z, T = _gn(x, torch.zeros_like(x), f("0.weight"), f("0.bias"))
    w1 = f("1.weight").flatten(1)
    y, T = _chain(w1.t().contiguous(), z, T, f("1.bias"))
    z, T = _gn(y, T, f("2.weight"), f("2.bias"))
    y, T = _chain(f("4.weight").flatten(1).t().contiguous(), z.clamp_min(0), T, f("4.bias"))
    z, T = _gn(y, T, f("5.weight"), f("5.bias"))
    # the same chain with torch.nn.functional, as the reference's SkipPool.fc computes it
    q = x[:, :, None, None]
    q = F.group_norm(q, 1, f("0.weight"), f("0.bias"), EPS)
    q = F.relu(F.group_norm(F.conv2d(q, f("1.weight"), f("1.bias")), 1, f("2.weight"), f("2.bias"), EPS))
    q = F.relu(F.group_norm(F.conv2d(q, f("4.weight"), f("4.bias")), 1, f("5.weight"), f("5.bias"), EPS))
    assert torch.allclose(q.flatten(1), z.clamp_min(0), rtol=1e-10, atol=1e-12)
    return z.clamp_min(0), T


@gpu
@pytest.mark.parametrize("kind", ["mixed", "offset"])
def test_wide_heads_vs_fp64(kind):
    lib = _lib.load()
    sd = synthetic_state_dict("C", seed=13, appear_arch="resnet50")
    from mmmot_b200.weights import prepare_resnet
    _, heads = prepare_resnet(sd, "resnet50")
    heads = [t.cuda() for t in heads]
    rw = _lib.ResnetWeights()
    for s in range(4):
        for j in range(10):
            rw.head[s][j] = heads[10 * s + j].data_ptr()
    n, L = 6, 3
    g = torch.Generator().manual_seed(case_seed("resnet heads", kind))
    pooled = []
    for s in range(4):
        C = 256 << s
        if kind == "mixed":
            pooled.append(torch.randn(n, C, generator=g).abs() * 10 ** (torch.rand(n, C, generator=g) * 3 - 2))
        else:
            pooled.append(10 ** (torch.rand(n, 1, generator=g) * 2 - 1) * (20 + torch.randn(n, C, generator=g)))
    X = torch.cat([p.reshape(-1) for p in pooled]).cuda()
    Y = torch.full((n // L, 3, 512, L), float("nan"), device="cuda")
    assert op(lib, "heads", rw=rw, n=n, H=1, W=1, L=L, X=X, Y=Y) == 0
    assert bool(torch.isnan(Y[:, 1:]).all())
    got = Y[:, 0].permute(0, 2, 1).reshape(n, 512)
    r = {}
    for s in range(4):
        ref, T = _head_ref(sd, s, pooled[s].double().cuda())
        r[f"head{s}_C{256 << s}"] = worst_ratio(got[:, s * 128:(s + 1) * 128], ref, T)
    report(f"resnet wide heads {kind} (err / bound)", **r)
    assert max(r.values()) <= 1.0, r
