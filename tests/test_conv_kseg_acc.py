"""K-segmented launches of the channel-major conv kernel (csrc/gemm_tma.cuh): the epilogue from the wgmma accumulators,
which folds each segment's partial sums from the registers through the K-segment scratch (seg_fold), against the
accumulator-image epilogue that debug bit 11 keeps.  Both compute S = RN(v0 s), then S = fmaf(vk, s, S) per later
segment, then S + b and the ReLU, so the FP16 hi/lo planes (pooled or not, with their guard bands) must be
byte-identical and the range flag the same; SkipPool's per-image sums are held to the bound test_conv_acc_epilogue.py
derives for the two epilogues' different fp32 groupings.  The scratch must hold the documented [tiles * 256][M] floats
and nothing past them is written.

The cases cover 2 to 5 segments (uneven last segments included), fused pools with box rows of 2, 4, 8, 16 and 32
pixels, partial boxes and image slabs, empty tile halves, a 64-channel layer, 147 (tile, row group) units on 132 SMs,
and a ResNet 3x3 conv at K = 4608.  Output widths that are not a multiple of 64 keep the image epilogue (the partial
sums are kept in whole m64 blocks); their K-segmented launches are checked against fp64 and for writes past the
scratch.  The plan checks at the end run without a GPU."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from kernel_kit import TAU, case_seed, fp16_split, lib_state, vp
from mmmot_b200 import _lib
from mmmot_b200.weights import pack_tc

NAN16 = 0x7E00
GUARD = 4096
BIT_IMAGE_EPI = 2048
BIT_CM64 = 64
PLAN_KEYS = ("px", "halo", "pool", "bx", "by", "bi", "ksegs", "tiles")

gpu = pytest.mark.gpu

# (name, cin, cout, H, W, n_img, debug bits, kseg (None: default), want_pool, expected plan subset)
CASES = [
    ("seg2_pool_bx16", 256, 256, 16, 16, 2, 0, None, True, dict(pool=1, bx=16, ksegs=2)),
    ("seg4_pool_bx8", 512, 512, 8, 8, 4, 0, None, True, dict(pool=1, bx=8, ksegs=4)),
    ("seg4_pool_bx4", 512, 512, 4, 4, 16, 0, None, True, dict(pool=1, bx=4, ksegs=4)),
    ("seg4_pool_bx2", 512, 512, 2, 2, 64, 0, None, True, dict(pool=1, bx=2, ksegs=4)),
    ("seg4_pool_bx4_partial_n17", 512, 512, 2, 2, 17, 0, None, True, dict(pool=1, bx=4, ksegs=4)),
    ("seg3_pool_bx32", 128, 128, 32, 32, 2, 0, 12, True, dict(pool=1, bx=32, ksegs=3)),
    ("seg4_pool_partial_14", 512, 512, 14, 14, 1, 0, None, True, dict(pool=1, ksegs=4)),
    ("seg4_pool_partial_6_n3", 512, 512, 6, 6, 3, 0, None, True, dict(pool=1, ksegs=4)),
    ("seg3_pool_slab_half_empty", 64, 128, 8, 8, 5, 0, 8, True, dict(pool=1, bi=4, ksegs=3)),
    ("seg4_uneven_pool", 64, 128, 16, 16, 2, 0, 5, True, dict(pool=1, ksegs=4)),
    ("seg2_partial_12", 256, 512, 12, 12, 2, 0, None, False, dict(pool=0, ksegs=2)),
    ("seg2_slab_n3", 256, 512, 8, 8, 3, 0, None, False, dict(pool=0, ksegs=2)),
    ("seg4_partial_28", 512, 512, 28, 28, 1, 0, None, False, dict(pool=0, ksegs=4)),
    ("seg5_uneven", 512, 512, 8, 8, 2, 0, 35, False, dict(pool=0, ksegs=5)),
    ("seg5_uneven_pool", 128, 128, 8, 8, 4, 0, 8, True, dict(pool=1, ksegs=5)),
    ("seg2_uneven", 32, 128, 16, 16, 2, 0, 5, False, dict(pool=0, ksegs=2)),
    ("seg3_m64", 64, 64, 16, 16, 2, BIT_CM64, 8, False, dict(pool=0, ksegs=3)),
    ("seg3_m64_pool_bx32", 64, 64, 32, 32, 2, BIT_CM64, 8, True, dict(pool=1, bx=32, ksegs=3)),
    ("seg2_uneven_units_147", 32, 384, 112, 112, 1, 0, 5, False, dict(pool=0, ksegs=2, tiles=49)),
]
CASE_IDS = [c[0] for c in CASES]


def _plan(lib, n, H, W, C, M, want_pool):
    arr = (ctypes.c_int * 8)()
    assert lib.mmmot_debug_conv_plan(n, H, W, C, M, int(want_pool), 1, arr) == 0
    return dict(zip(PLAN_KEYS, list(arr)))


def _scratch(tiles, M):
    """The documented [tiles * 256][M] fp32 scratch, NaN, followed by a guard band of a bit pattern no fp32 sum has."""
    scr = torch.full((tiles * 256 * M + GUARD,), float("nan"), device="cuda")
    scr[tiles * 256 * M:].view(torch.int32).fill_(0x7FA5A5A5)
    return scr


def _run(lib, Wp, wps, b, X, n, H, W, C, M, want_pool, tiles):
    """One mmmot_debug_conv_layer call on NaN-filled buffers -> (raw output buffer, pool sums or None, status, did_pool,
    pooled plane distance)."""
    full, pooled = n * H * W * M, n * (H // 2) * (W // 2) * M
    y_plane, p_plane = full + GUARD, pooled + GUARD
    Y = torch.full((2 * y_plane,), NAN16, dtype=torch.int16, device="cuda")
    psum = None
    if want_pool:
        psum = torch.full((n * M + GUARD,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
        psum[:n * M] = 0
    scr = _scratch(tiles, M)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    did = ctypes.c_int(-1)
    rc = lib.mmmot_debug_conv_layer(vp(Wp), None, wps, vp(b), vp(X), X[0].numel(), n, H, W, C, M, vp(Y), y_plane,
                                    p_plane if want_pool else 0, ctypes.byref(did) if want_pool else None, vp(psum),
                                    vp(scr), vp(status), None, None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    assert bool((scr[tiles * 256 * M:].view(torch.int32) == 0x7FA5A5A5).all()), "K-segment scratch written past its end"
    return Y.cpu(), None if psum is None else psum.cpu(), int(status.item()), did.value if want_pool else 0, p_plane


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_seg_acc_epilogue_matches_image_epilogue(case):
    name, C, M, H, W, n, dbg, kseg, want_pool, expect = case
    lib = _lib.load()
    g = torch.Generator().manual_seed(case_seed("kseg acc", name))
    w = torch.randn(M, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    b = torch.randn(M, generator=g) * 0.1
    x_hi, x_lo = fp16_split(torch.randn(n, H, W, C, generator=g))
    X = torch.stack([x_hi, x_lo]).contiguous().cuda()
    Wp, wps = pack_tc(w.permute(2, 3, 1, 0).reshape(9 * C, M).contiguous())
    Wp, bd = Wp.cuda(), b.cuda()
    runs = {}
    for bits in (dbg, dbg | BIT_IMAGE_EPI):
        with lib_state(lib, dbg=bits, kseg=kseg):
            plan = _plan(lib, n, H, W, C, M, want_pool)
            assert not plan["px"] and plan["ksegs"] > 1
            for k, v in expect.items():
                assert plan[k] == v, (name, k, plan)
            seg_acc = lib.mmmot_debug_conv_seg_epilogue(n, H, W, C, M, int(want_pool), 1)
            assert seg_acc == (0 if bits & BIT_IMAGE_EPI else 1)
            runs[bits] = _run(lib, Wp, wps, bd, X, n, H, W, C, M, want_pool, plan["tiles"])
    (y_new, ps_new, st_new, did_new, p_plane), (y_old, ps_old, st_old, did_old, _) = runs[dbg], runs[dbg | BIT_IMAGE_EPI]
    assert did_new == did_old == expect["pool"]
    assert st_new == st_old
    diff = int((y_new != y_old).sum())
    assert diff == 0, f"{diff} output halves differ between the two epilogues"
    if want_pool:
        assert torch.equal(ps_new[n * M:], ps_old[n * M:]), "pool sums written past [n][M]"
        Hp, Wp_ = H // 2, W // 2
        ext = n * Hp * Wp_ * M
        v = (y_new[:ext].view(torch.float16).double() + y_new[p_plane:p_plane + ext].view(torch.float16).double())
        ref = v.reshape(n, Hp * Wp_, M).sum(dim=1).reshape(-1)
        # the bound of test_conv_acc_epilogue.py: fp32 runs of at most Hp*Wp terms (<= m 2^-24 of the sum each), flushed
        # as 2^-32 fixed point (<= 2^-33 per flush, at most Hp*Wp flushes), in each epilogue
        m = Hp * Wp_
        tol = 2 * (m * 2.0 ** -24 * ref * (1 + 2.0 ** -10) + m * 2.0 ** -33)
        got_new, got_old = ps_new[:n * M].double() * 2.0 ** -32, ps_old[:n * M].double() * 2.0 ** -32
        worst = float(((got_new - got_old).abs() / tol).max())
        assert worst <= 1.0, worst


@gpu
def test_resnet_k4608_conv_matches_image_epilogue():
    """A ResNet layer4 3x3 conv (512 -> 512, K = 4608: four segments) through mmmot_debug_resnet_op as the trunk runs it:
    byte-identical planes and the same range flag under both epilogues."""
    lib = _lib.load()
    n, H, W, C, M = 3, 8, 8, 512, 512
    g = torch.Generator().manual_seed(case_seed("kseg acc resnet", C, M))
    wt = torch.randn(9 * C, M, generator=g) * (2.0 / (9 * C)) ** 0.5
    b = torch.rand(M, generator=g) * 0.2 - 0.1
    x_hi, x_lo = fp16_split(torch.randn(n, H, W, C, generator=g).clamp_min(-0.3))
    X = torch.stack([x_hi.reshape(-1), x_lo.reshape(-1)]).contiguous().cuda()
    packed, scale = pack_tc(wt)
    b_d, p_d, wt_d = b.cuda(), packed.cuda(), wt.cuda()
    rw = _lib.ResnetWeights()
    rw.wt[5], rw.bias[5], rw.wp[5] = wt_d.data_ptr(), b_d.data_ptr(), p_d.data_ptr()
    rw.wp_scale[5] = scale
    P = n * H * W
    cols = torch.empty(1024, dtype=torch.float32, device="cuda")
    out = {}
    for bits in (0, BIT_IMAGE_EPI):
        with lib_state(lib, engine="tc", dbg=bits):
            plan = _plan(lib, n, H, W, C, M, False)
            assert plan["ksegs"] == 4 and not plan["px"]
            assert lib.mmmot_debug_conv_seg_epilogue(n, H, W, C, M, 0, 1) == (0 if bits else 1)
            Y = torch.full((2 * P * M + 256,), NAN16, dtype=torch.int16, device="cuda")
            scr = _scratch(plan["tiles"], M)
            status = torch.zeros(1, dtype=torch.int32, device="cuda")
            rc = lib.mmmot_debug_resnet_op(3, ctypes.pointer(rw), 5, n, H, W, C, 3, 1, M, 1, 1, vp(X), None, vp(Y),
                                           vp(cols), vp(scr), vp(status), None)
            torch.cuda.synchronize()
            assert rc == 0, rc
            assert bool((scr[plan["tiles"] * 256 * M:].view(torch.int32) == 0x7FA5A5A5).all())
            out[bits] = (Y.cpu(), int(status.item()))
    assert out[0][1] == out[BIT_IMAGE_EPI][1]
    diff = int((out[0][0] != out[BIT_IMAGE_EPI][0]).sum())
    assert diff == 0, f"{diff} output halves differ between the two epilogues"


@gpu
@pytest.mark.parametrize("M,want_pool", [(96, False), (160, True)], ids=["m96", "m160_pool"])
def test_kseg_partial_m64_block_keeps_image_epilogue(M, want_pool):
    """K-segmented launches whose M is not a multiple of 64 take the image epilogue: within TAU * S of fp64 (pooled
    like y), the range flag clear, and nothing written past the [tiles * 256][M] scratch or the output planes."""
    lib = _lib.load()
    n, H, W, C = 2, 16, 16, 256
    g = torch.Generator().manual_seed(case_seed("kseg acc partial m64", M))
    w = torch.randn(M, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5
    b = torch.randn(M, generator=g) * 0.1
    x_hi, x_lo = fp16_split(torch.randn(n, H, W, C, generator=g))
    X = torch.stack([x_hi, x_lo]).contiguous().cuda()
    Wp, wps = pack_tc(w.permute(2, 3, 1, 0).reshape(9 * C, M).contiguous())
    with lib_state(lib):
        plan = _plan(lib, n, H, W, C, M, want_pool)
        assert not plan["px"] and plan["ksegs"] == 2 and plan["pool"] == int(want_pool)
        assert lib.mmmot_debug_conv_seg_epilogue(n, H, W, C, M, int(want_pool), 1) == 0
        Y, _, status, did, p_plane = _run(lib, Wp.cuda(), wps, b.cuda(), X, n, H, W, C, M, want_pool, plan["tiles"])
    assert status == 0 and did == int(want_pool)
    Ho, Wo = (H // 2, W // 2) if want_pool else (H, W)
    plane = p_plane if want_pool else n * H * W * M + GUARD
    ext = n * Ho * Wo * M
    assert bool((Y[ext:plane] == NAN16).all()) and bool((Y[plane + ext:] == NAN16).all()), "output written past its plane"
    y = Y[:ext].view(torch.float16).double() + Y[plane:plane + ext].view(torch.float16).double()
    y = y.view(n, Ho, Wo, M).permute(0, 3, 1, 2)
    xv = (x_hi.double() + x_lo.double()).permute(0, 3, 1, 2)
    ref = F.relu(F.conv2d(xv, w.double(), b.double(), padding=1))
    S = F.conv2d(xv.abs(), w.double().abs(), b.double().abs(), padding=1)
    if want_pool:
        ref, S = F.max_pool2d(ref, 2), F.max_pool2d(S, 2)
    worst = float(((y - ref).abs() / (TAU * S)).max())
    assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------ CPU: plans
PLAN_GRID = [
    # (n, H, W, C, M, want_pool)
    (2, 16, 16, 256, 256, 1), (4, 8, 8, 512, 512, 1), (2, 16, 16, 256, 256, 0), (3, 8, 8, 512, 512, 0),
    (2, 16, 16, 64, 64, 0), (2, 64, 64, 64, 64, 1), (2, 32, 32, 128, 128, 1), (1, 112, 112, 32, 384, 0),
    (2, 16, 16, 32, 128, 0), (5, 8, 8, 64, 128, 1), (2, 16, 16, 256, 96, 0), (2, 16, 16, 256, 160, 1),
]


def test_seg_epilogue_plan_needs_no_gpu(lib_built):
    """seg_epilogue is 1 exactly for K-segmented channel-major plans with M a multiple of 64 and without debug bit 11,
    and never together with the single-pass accumulator epilogue."""
    lib = _lib.load()
    seen = set()
    for dbg in (0, BIT_CM64, BIT_IMAGE_EPI, BIT_CM64 | BIT_IMAGE_EPI):
        for kseg in (0, 5, 8, 12, None):
            with lib_state(lib, dbg=dbg, kseg=kseg):
                for n, H, W, C, M, pool in PLAN_GRID:
                    p = _plan(lib, n, H, W, C, M, pool)
                    seg = lib.mmmot_debug_conv_seg_epilogue(n, H, W, C, M, pool, 1)
                    single = lib.mmmot_debug_conv_epilogue(n, H, W, C, M, pool, 1)
                    want = int(not p["px"] and p["ksegs"] > 1 and M % 64 == 0 and not dbg & BIT_IMAGE_EPI)
                    assert seg == want, (dbg, kseg, n, H, W, C, M, pool, p)
                    assert not (seg and single)
                    # without scratch there are no K segments
                    assert lib.mmmot_debug_conv_seg_epilogue(n, H, W, C, M, pool, 0) == 0
                    seen.add((bool(p["px"]), p["ksegs"] > 1, bool(dbg & BIT_IMAGE_EPI)))
    assert {(False, True, False), (False, True, True), (True, False, False), (False, False, False)} <= seen
    assert lib.mmmot_debug_conv_seg_epilogue(2, 16, 16, 48, 64, 0, 1) == -1      # MMMOT_E_ARG: C not a multiple of 32
    assert lib.mmmot_debug_conv_seg_epilogue(0, 16, 16, 64, 64, 0, 1) == -1


def test_seg_cases_plan_as_named(lib_built):
    """Every GPU case above is K-segmented on the channel-major kernel, and together they cover every fused-pool box
    width and 2 to 5 segments, uneven last segments included."""
    lib = _lib.load()
    widths, segs, uneven = set(), set(), 0
    for name, C, M, H, W, n, dbg, kseg, want_pool, expect in CASES:
        with lib_state(lib, dbg=dbg, kseg=kseg):
            p = _plan(lib, n, H, W, C, M, want_pool)
            assert lib.mmmot_debug_conv_seg_epilogue(n, H, W, C, M, int(want_pool), 1) == 1, name
        for k, v in expect.items():
            assert p[k] == v, (name, k, p)
        kc = 9 * C // 32
        per = -(-kc // p["ksegs"])
        uneven += kc != per * p["ksegs"]
        segs.add(p["ksegs"])
        if p["pool"]:
            widths.add(p["bx"])
    assert {2, 4, 8, 16, 32} <= widths
    assert {2, 3, 4, 5} <= segs
    assert uneven >= 3
