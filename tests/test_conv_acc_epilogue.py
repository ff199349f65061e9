"""The channel-major conv kernel's two epilogues against each other (csrc/gemm_tma.cuh): the epilogue from the wgmma
accumulators in registers (TMA stores; single-pass K launches) and the accumulator-image epilogue that debug bit 11
keeps.  Both apply the same fp32 operations in the same order, so the FP16 hi/lo planes
(pooled or not, with their guard bands) must be byte-identical and the range flag the same.  SkipPool's per-image sums
are fp32 runs of a different grouping (at most 32 terms each in the accumulator epilogue), so they are held to the bound
such runs obey against the fp64 sums of the pooled map both epilogues wrote.

The cases cover fused pools with box rows of 2, 4, 8, 16 and 32 pixels, partial boxes and image slabs, empty tile
halves, a 256-pixel-wide box and a 64-channel layer (K segmentation off, so the deep layers take the accumulator
epilogue too).  The plan checks at the end run without a GPU: K-segmented launches keep the image epilogue."""
import ctypes

import pytest
import torch

from kernel_kit import fp16_split, lib_state, vp
from mmmot_b200 import _lib
from mmmot_b200.weights import pack_tc

NAN16 = 0x7E00
GUARD = 4096
BIT_IMAGE_EPI = 2048
PLAN_KEYS = ("px", "halo", "pool", "bx", "by", "bi", "ksegs", "tiles")

gpu = pytest.mark.gpu

# (name, cin, cout, H, W, n_img, debug bits, kseg (None: default), want_pool, expected plan subset)
CASES = [
    ("pool_bx32", 128, 128, 32, 32, 2, 0, None, True, dict(pool=1, bx=32)),
    ("pool_bx16", 256, 256, 16, 16, 2, 0, 0, True, dict(pool=1, bx=16)),
    ("pool_bx8", 512, 512, 8, 8, 4, 0, 0, True, dict(pool=1, bx=8)),
    ("pool_bx4", 512, 512, 4, 4, 16, 0, 0, True, dict(pool=1, bx=4)),
    ("pool_bx2", 512, 512, 2, 2, 64, 0, 0, True, dict(pool=1, bx=2)),
    ("pool_bx4_partial_n17", 512, 512, 2, 2, 17, 0, 0, True, dict(pool=1, bx=4)),
    ("pool_partial_14", 512, 512, 14, 14, 1, 0, 0, True, dict(pool=1)),
    ("pool_partial_6_n3", 512, 512, 6, 6, 3, 0, 0, True, dict(pool=1)),
    ("pool_slab_half_empty", 64, 128, 8, 8, 5, 0, None, True, dict(pool=1, bi=4)),
    ("partial_12", 256, 512, 12, 12, 2, 0, 0, False, dict(pool=0)),
    ("slab_n3", 256, 512, 8, 8, 3, 0, 0, False, dict(pool=0)),
    ("partial_28", 512, 512, 28, 28, 1, 0, 0, False, dict(pool=0)),
    ("bx32_32x8", 64, 128, 32, 32, 1, 0, None, False, dict(pool=0, bx=32)),
    ("m64_16x16", 64, 64, 16, 16, 2, 64, None, False, dict(pool=0)),
    ("m64_pool_bx32", 64, 64, 32, 32, 2, 64, None, True, dict(pool=1, bx=32)),
    ("width_300", 32, 128, 1, 300, 1, 0, None, False, dict(pool=0, bx=256)),
    ("odd_units_147", 32, 384, 112, 112, 1, 0, None, False, dict(pool=0)),
]
CASE_IDS = [c[0] for c in CASES]


def _plan(lib, n, H, W, C, M, want_pool):
    arr = (ctypes.c_int * 8)()
    assert lib.mmmot_debug_conv_plan(n, H, W, C, M, int(want_pool), 1, arr) == 0
    return dict(zip(PLAN_KEYS, list(arr)))


def _run(lib, Wp, wps, b, X, n, H, W, C, M, want_pool, tiles):
    """One mmmot_debug_conv_layer call on NaN-filled buffers -> (raw output buffer, pool sums or None, status, did_pool)."""
    full, pooled = n * H * W * M, n * (H // 2) * (W // 2) * M
    y_plane, p_plane = full + GUARD, pooled + GUARD
    Y = torch.full((2 * y_plane,), NAN16, dtype=torch.int16, device="cuda")
    psum = None
    if want_pool:
        psum = torch.full((n * M + GUARD,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
        psum[:n * M] = 0
    scr = torch.full((tiles * 256 * M,), float("nan"), device="cuda")     # the documented [tiles * 256][M] scratch
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    did = ctypes.c_int(-1)
    rc = lib.mmmot_debug_conv_layer(vp(Wp), None, wps, vp(b), vp(X), X[0].numel(), n, H, W, C, M, vp(Y), y_plane,
                                    p_plane if want_pool else 0, ctypes.byref(did) if want_pool else None, vp(psum),
                                    vp(scr), vp(status), None, None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return Y.cpu(), None if psum is None else psum.cpu(), int(status.item()), did.value if want_pool else 0, p_plane


@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_acc_epilogue_matches_image_epilogue(case):
    name, C, M, H, W, n, dbg, kseg, want_pool, expect = case
    lib = _lib.load()
    g = torch.Generator().manual_seed(sum(map(ord, name)))
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
            assert not plan["px"] and plan["ksegs"] == 1
            for k, v in expect.items():
                assert plan[k] == v, (name, k, plan)
            assert lib.mmmot_debug_conv_epilogue(n, H, W, C, M, int(want_pool), 1) == (0 if bits & BIT_IMAGE_EPI else 1)
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
        # Each epilogue sums the same fp32 pooled values in fp32 runs (of at most Hp*Wp terms in the image epilogue, of at
        # most 32 in the accumulator one: <= m 2^-24 of the sum each) flushed as 2^-32 fixed point (<= 2^-33 per flush,
        # at most Hp*Wp flushes).  ref (hi + lo, within 2^-10 of the fp32 values) only scales the relative part.
        m = Hp * Wp_
        tol = 2 * (m * 2.0 ** -24 * ref * (1 + 2.0 ** -10) + m * 2.0 ** -33)
        got_new, got_old = ps_new[:n * M].double() * 2.0 ** -32, ps_old[:n * M].double() * 2.0 ** -32
        worst = float(((got_new - got_old).abs() / tol).max())
        assert worst <= 1.0, worst


# ------------------------------------------------------------------------------------------------ CPU: plans
def test_acc_epilogue_plan_needs_no_gpu(lib_built):
    lib = _lib.load()
    with lib_state(lib):
        for name, C, M, H, W, n, dbg, kseg, want_pool, expect in CASES:
            with lib_state(lib, dbg=dbg, kseg=kseg):
                assert lib.mmmot_debug_conv_epilogue(n, H, W, C, M, int(want_pool), 1) == 1, name
            with lib_state(lib, dbg=dbg | BIT_IMAGE_EPI, kseg=kseg):
                assert lib.mmmot_debug_conv_epilogue(n, H, W, C, M, int(want_pool), 1) == 0, name
        # the pixel-major kernel (64 -> 64 without bit 6) has no channel-major epilogue
        assert lib.mmmot_debug_conv_epilogue(2, 64, 64, 64, 64, 1, 1) == 0
        # K-segmented launches (K = 2304 at the default segment length) keep the accumulator-image epilogue
        assert lib.mmmot_debug_conv_epilogue(2, 16, 16, 256, 256, 0, 1) == 0
        assert lib.mmmot_debug_conv_epilogue(2, 16, 16, 256, 256, 0, 0) == 1
        assert lib.mmmot_debug_conv_epilogue(2, 16, 16, 48, 64, 0, 0) == -1      # MMMOT_E_ARG: C not a multiple of 32


def test_acc_epilogue_cases_cover_every_pool_width(lib_built):
    lib = _lib.load()
    widths = set()
    for name, C, M, H, W, n, dbg, kseg, want_pool, expect in CASES:
        with lib_state(lib, dbg=dbg, kseg=kseg):
            p = _plan(lib, n, H, W, C, M, want_pool)
        assert p["ksegs"] == 1, name
        if p["pool"]:
            widths.add(p["bx"])
    assert {2, 4, 8, 16, 32} <= widths
