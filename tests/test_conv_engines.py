"""Kernel-level parity of the VGG trunk's convolutions (csrc/gemm_tma.cuh, csrc/gemm_tma_px.cuh, the first-layer
variants of appearance.cu) against fp64 references, element by element, at every launch plan the product uses.

The end-to-end tests see the trunk only through SkipPool's global averages, which hide a wrong border tap, a wrong
pixel of a partial box or image slab, a misplaced pooled pixel or a missing lo term.  These tests run one layer through
the product's own launch code (mmmot_debug_conv_layer / mmmot_debug_vgg_conv0) and bound every output element by

    |y - y_ref| <= TAU * S,   S = conv2d(|X|, |W|) + |b|   (max-pooled like y for pooled outputs; TAU = 2^-18, see
                                                            kernel_kit.TAU),

the forward-error form of a dot product: meaningful at ReLU zeros and cancellations, where a bound relative to |y| is
not.  X is exactly what the kernel reads (hi + lo of the input planes, or the fp32 crops), W the fp32 weights handed
to pack_tc, and the outputs are read back as hi + lo in fp64.

Output buffers are filled with FP16 NaN (0x7E00) before each call, so an element the kernel never wrote fails, and
carry a guard band past the valid extent of each plane that must come back unchanged (a store past a partial box or
image slab shows up there without relying on a fault).

The launch-plan tests at the end run without a GPU: mmmot_debug_conv_plan computes the plan on the host.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_kit import KSEG_DEFAULT, TAU, bench_n_imgs, fp16_split, lib_state, vp
from mmmot_b200 import _lib
from mmmot_b200.schema import VGG_STAGES
from mmmot_b200.weights import pack_px, pack_tc

NAN16 = 0x7E00
GUARD = 4096                       # guard band (elements) after every output plane
PLAN_KEYS = ("px", "halo", "pool", "bx", "by", "bi", "ksegs", "tiles")
SMS = 132                          # H100 SXM: the persistent grid of the channel-major kernel is min(units, SMs)

gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ case table
# One entry per conv-layer case: (name, cin, cout, H, W, n_img, debug bits, kseg, want_pool, compact Wpx, check).
# `check(plan)` asserts the path the case is named after; the GPU test runs every case, and the CPU coverage guard
# requires every plan class of the benchmark configurations to appear among these cases' plans.
def _partial_x(p):
    return p["bx"] * math.ceil(p["W"] / p["bx"]) > p["W"]


def _partial_y(p):
    return p["by"] * math.ceil(p["H"] / p["by"]) > p["H"]


def _partial_slab(p):
    return p["bi"] > 1 and p["n"] % p["bi"] != 0


def half_dim(p):
    """The box dimension that separates a tile's two 128-column halves (columns (ii*by + yy)*bx + xx): the outermost
    one larger than 1."""
    return "bi" if p["bi"] > 1 else "by" if p["by"] > 1 else "bx"


def empty_halves(p):
    """Column tiles of a conv plan whose half 1 lies wholly outside the image."""
    d = half_dim(p)
    lim = {"bi": p["n"], "by": p["H"], "bx": p["W"]}[d]
    count = {"bi": math.ceil(p["n"] / p["bi"]), "by": math.ceil(p["H"] / p["by"]), "bx": math.ceil(p["W"] / p["bx"])}[d]
    others = p["tiles"] // count
    return others * sum(1 for k in range(count) if k * p[d] + p[d] // 2 >= lim)


def units(p, M):
    return p["tiles"] * math.ceil(M / 128)


CASES = [
    # pixel-major kernel (64 -> 64, VGG conv 1)
    ("px_halo_pool_64", 64, 64, 64, 64, 2, 0, None, True, True, lambda p: p["px"] and p["halo"] and p["pool"]),
    ("px_halo_pool_224", 64, 64, 224, 224, 1, 0, None, True, True, lambda p: p["px"] and p["halo"] and p["pool"]),
    ("px_halo_96", 64, 64, 96, 96, 1, 0, None, False, True, lambda p: p["px"] and p["halo"] and not p["pool"]),
    ("px_nohalo_pool_32", 64, 64, 32, 32, 3, 256, None, True, True, lambda p: p["px"] and not p["halo"] and p["pool"]),
    ("px_noncompact_32", 64, 64, 32, 32, 2, 0, None, True, False, lambda p: p["px"] and p["pool"]),
    ("px_noncompact_nohalo_32", 64, 64, 32, 32, 1, 256, None, False, False, lambda p: p["px"] and not p["halo"]),
    ("px_slab_n3", 64, 64, 8, 8, 3, 0, None, True, True, lambda p: p["px"] and p["pool"] and _partial_slab(p)),
    ("px_partial_24x40", 64, 64, 24, 40, 1, 0, None, False, True, lambda p: p["px"] and (_partial_x(p) or _partial_y(p))),
    # channel-major kernel, fused pools of every box width
    ("cm_pool32_64", 128, 128, 32, 32, 2, 0, None, True, False, lambda p: not p["px"] and p["pool"] and p["bx"] == 32),
    ("cm_pool16_kseg2_64", 256, 256, 16, 16, 2, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and p["bx"] == 16 and p["ksegs"] == 2),
    ("cm_pool8_kseg4_64", 512, 512, 8, 8, 4, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and p["bx"] == 8 and p["bi"] == 4 and p["ksegs"] == 4),
    ("cm_pool4_kseg4_64", 512, 512, 4, 4, 16, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and p["bx"] == 4 and p["bi"] == 16 and p["ksegs"] == 4),
    ("cm_pool2_64", 512, 512, 2, 2, 64, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and p["bx"] == 2 and p["bi"] == 64),
    # 2 x 2 maps of 17 images: the 4 x 2 x 32 box (tied in waste, wider first) pads x and the image slab
    ("cm_pool4_partial_n17", 512, 512, 2, 2, 17, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and p["bx"] == 4 and _partial_x(p) and _partial_slab(p)),
    # channel-major kernel without a fused pool
    ("cm_32x8_32", 64, 128, 16, 16, 3, 0, None, False, False, lambda p: not p["px"] and not p["pool"] and p["ksegs"] == 1),
    ("cm_32x8_64", 64, 128, 32, 32, 1, 0, None, False, False,
     lambda p: not p["px"] and not p["pool"] and p["bx"] == 32 and p["ksegs"] == 1),
    ("cm_kseg2_64", 256, 256, 16, 16, 2, 0, None, False, False, lambda p: not p["px"] and not p["pool"] and p["ksegs"] == 2),
    ("cm_kseg4_8x8x4_64", 512, 512, 8, 8, 4, 0, None, False, False,
     lambda p: not p["px"] and not p["pool"] and p["ksegs"] == 4 and p["bi"] == 4),
    ("cm_16x16_64", 128, 256, 16, 16, 2, 0, None, False, False,
     lambda p: not p["px"] and not p["pool"] and p["bx"] == 16 and p["ksegs"] == 1),
    ("cm_unfused_bit512", 128, 128, 32, 32, 1, 512, None, True, False, lambda p: not p["px"] and not p["pool"]),
    # 64-channel layers on the channel-major kernel (rows 64-127 of the tile masked)
    ("cm_m64_pool32", 64, 64, 32, 32, 2, 64, None, True, False, lambda p: not p["px"] and p["pool"] and p["bx"] == 32),
    ("cm_m64_kseg8", 64, 64, 16, 16, 2, 64, 8, False, False, lambda p: not p["px"] and p["ksegs"] == 3),
    # partial boxes (96 and 224 crops) and partial image slabs
    ("cm_partial_12_96", 256, 512, 12, 12, 2, 0, None, False, False,
     lambda p: not p["px"] and p["ksegs"] == 2 and (_partial_x(p) or _partial_y(p) or _partial_slab(p))),
    ("cm_partial_6_96", 512, 512, 6, 6, 3, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and (_partial_x(p) or _partial_y(p) or _partial_slab(p))),
    ("cm_partial_pool_14_224", 512, 512, 14, 14, 1, 0, None, True, False,
     lambda p: not p["px"] and p["pool"] and _partial_x(p) and _partial_y(p) and p["ksegs"] == 4),
    ("cm_partial_28_224", 512, 512, 28, 28, 1, 0, None, False, False,
     lambda p: not p["px"] and _partial_x(p) and _partial_y(p)),
    ("cm_slab_n3", 256, 512, 8, 8, 3, 0, None, False, False, lambda p: not p["px"] and _partial_slab(p) and p["ksegs"] == 2),
    ("cm_slab_n6_pool", 512, 512, 4, 4, 6, 0, None, True, False, lambda p: not p["px"] and p["pool"] and _partial_slab(p)),
    # one 4 x 4 image: the 64 x 4 box (tied in waste) is too wide for a fused pool, the pooled map comes separately
    ("cm_wide_box_n1", 512, 512, 4, 4, 1, 0, None, True, False,
     lambda p: not p["px"] and not p["pool"] and p["bx"] == 64 and _partial_x(p)),
    # K segmentation: many middle segments (kseg 8 on K = 1152: five segments)
    ("cm_kseg8_pool", 128, 128, 8, 8, 4, 0, 8, True, False,
     lambda p: not p["px"] and p["pool"] and p["ksegs"] == 5),
    # The edges of the channel-major kernel's work schedule: the persistent grid of min(units, SMs) CTAs walks
    # (column tile, M group) units, each in K segments, and consumer warpgroup h takes column half h of every tile.
    # One 16 x 16 box: a single unit, halves split along the box rows, fused pool
    ("one_tile_pool", 64, 128, 16, 16, 1, 0, None, True, False,
     lambda p: not p["px"] and p["tiles"] == 1 and half_dim(p) == "by" and p["pool"]),
    # 49 boxes x 3 M groups = 147 units on 132 CTAs: odd, not a multiple of the grid
    ("odd_units_147", 32, 384, 112, 112, 1, 0, None, False, False,
     lambda p: not p["px"] and units(p, 384) == 147 and p["ksegs"] == 1),
    # 3 boxes (odd) and 2, 3, 4, 5 K segments per half, fused pool
    ("kseg2_tiles3", 128, 128, 16, 16, 3, 0, 18, True, False,
     lambda p: not p["px"] and p["tiles"] == 3 and p["ksegs"] == 2 and p["pool"] and half_dim(p) == "by"),
    ("kseg3_tiles3", 128, 128, 16, 16, 3, 0, 12, True, False,
     lambda p: not p["px"] and p["tiles"] == 3 and p["ksegs"] == 3 and p["pool"]),
    ("kseg4_tiles3", 128, 128, 16, 16, 3, 0, 9, True, False,
     lambda p: not p["px"] and p["tiles"] == 3 and p["ksegs"] == 4 and p["pool"]),
    ("kseg5_tiles3", 128, 128, 16, 16, 3, 0, 8, True, False,
     lambda p: not p["px"] and p["tiles"] == 3 and p["ksegs"] == 5 and p["pool"]),
    # halves split along the image slab (8 x 8 x 4 box): 5 images leave the second box's half 1 (images 6, 7) empty
    ("slab_half_empty_pool", 64, 128, 8, 8, 5, 0, None, True, False,
     lambda p: not p["px"] and half_dim(p) == "bi" and p["pool"] and empty_halves(p) == 1),
    ("slab_half_empty_pool_kseg3", 64, 128, 8, 8, 5, 0, 8, True, False,
     lambda p: not p["px"] and half_dim(p) == "bi" and p["pool"] and p["ksegs"] == 3 and empty_halves(p) == 1),
    # halves split along the box width (256 x 1 x 1 box on one-row images); 300 columns leave the second box's half 1
    # empty
    ("width_half_256", 32, 128, 1, 256, 2, 0, None, False, False,
     lambda p: not p["px"] and half_dim(p) == "bx" and p["tiles"] == 2 and empty_halves(p) == 0),
    ("width_half_empty_300", 32, 128, 1, 300, 1, 0, None, False, False,
     lambda p: not p["px"] and half_dim(p) == "bx" and p["tiles"] == 2 and empty_halves(p) == 1),
]
CASE_IDS = [c[0] for c in CASES]


def _plan(lib, n, H, W, C, M, want_pool, use_kseg=True):
    arr = (ctypes.c_int * 8)()
    assert lib.mmmot_debug_conv_plan(n, H, W, C, M, int(want_pool), int(use_kseg), arr) == 0
    return _plan_dict(arr, n, H, W)


def _plan_dict(arr, n, H, W):
    d = dict(zip(PLAN_KEYS, list(arr)))
    d.update(n=n, H=H, W=W)
    return d


def plan_class(p):
    """What decides which code of the two kernels runs: the kernel, halo boxes, the fused pool (and for the
    channel-major kernel its box width: bx == 32 and pool_chunk<bx> are different code), the number of K segments
    (1, 2, or >= 3 with middle segments) and whether a box spans several images."""
    return (p["px"], p["halo"], p["pool"], p["bx"] if p["pool"] and not p["px"] else 0, min(p["ksegs"], 3), p["bi"] > 1)


# ------------------------------------------------------------------------------------------------ helpers
def _weights(g, M, C, scale=1.0):
    w = torch.randn(M, C, 3, 3, generator=g) * (2.0 / (9 * C)) ** 0.5 * scale
    b = torch.randn(M, generator=g) * 0.1 * scale
    return w, b


def _w_terms(wt):
    """(W_hi, W_lo) in fp64 exactly as pack_tc splits Wt[K][M] (including its power-of-two pre-scale)."""
    _, scale = pack_tc(wt)
    w = (wt.double() / scale).float()
    hi = w.half()
    lo = (w - hi.float()).half()
    return hi.double() * scale, lo.double() * scale


def _zero_hi_tiles(packed, M, K):
    """pack_tc layout [k chunk][m tile][hi|lo][k group 4][m group 16][8][8]: the hi tiles set to zero."""
    t = packed.clone().view(torch.int16).view((K + 31) // 32, (M + 127) // 128, 2, 4, 16, 8, 8)
    t[:, :, 0] = 0
    return t.reshape(-1).view(torch.uint8)


def _zero_px_tiles(packed_px, K, which):
    """pack_px layout [k chunk][k group 4][hi|lo][row group 8][8][8]: the hi (0) or lo (1) tiles set to zero."""
    t = packed_px.clone().view(torch.int16).view((K + 31) // 32, 4, 2, 8, 8, 8)
    t[:, :, which] = 0
    return t.reshape(-1).view(torch.uint8)


def _out_buffer(plane, extra=0):
    """Two planes `plane` elements apart (valid extent + GUARD each), every element FP16 NaN."""
    return torch.full((2 * plane + extra,), NAN16, dtype=torch.int16, device="cuda")


def _read_planes(buf, plane, ext, shape):
    """-> fp64 hi + lo of the valid extent (CPU); asserts every valid element was written and every other element
    (guard bands) still holds the NaN fill."""
    b = buf.cpu()
    mask = torch.zeros(b.numel(), dtype=torch.bool)
    mask[:ext] = True
    mask[plane:plane + ext] = True
    untouched = b[~mask]
    assert bool((untouched == NAN16).all()), f"{int((untouched != NAN16).sum())} elements written outside the output planes"
    h = b[:ext].view(torch.float16).double()
    l = b[plane:plane + ext].view(torch.float16).double()
    y = h + l
    assert bool(torch.isfinite(y).all()), f"{int((~torch.isfinite(y)).sum())} output elements never written"
    return y.reshape(shape)


def _ratio(y, ref, S):
    return float(((y - ref).abs() / (TAU * S)).max())


def _conv_ref(x, w, b, pool):
    """fp64 reference (NCHW) of relu(conv3x3(x) + b) and its error scale S, both optionally 2x2 max-pooled."""
    y = torch.relu(F.conv2d(x, w, b, padding=1))
    S = F.conv2d(x.abs(), w.abs(), None if b is None else b.abs(), padding=1)
    if pool:
        y, S = F.max_pool2d(y, 2), F.max_pool2d(S, 2)
    return y, S


def _pool_planar_host(y_hi, y_lo):
    """maxpool2_planar_kernel on the host: per 2x2 window the (hi, lo) pair with the largest hi + lo, first in
    (0,0), (0,1), (1,0), (1,1) order on ties.  NHWC fp16 planes [n][H][W][C] -> fp64 hi + lo [n][H/2][W/2][C]."""
    v = y_hi.double() + y_lo.double()
    n, H, W, C = v.shape
    win = v.reshape(n, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(n, H // 2, W // 2, 4, C)
    return win.max(dim=3).values


class ConvRun:
    """One call of mmmot_debug_conv_layer on fresh buffers."""

    def __init__(self, lib, Wp, Wpx, wps, b, x_hi, x_lo, n, H, W, C, M, want_pool):
        self.plan_q = _plan(lib, n, H, W, C, M, want_pool)
        full, pooled = n * H * W * M, n * (H // 2) * (W // 2) * M
        self.y_plane, self.p_plane = full + GUARD, pooled + GUARD
        self.Y = _out_buffer(self.y_plane)
        X = torch.stack([x_hi, x_lo]).contiguous().cuda()
        self.Wp_d, self.Wpx_d, self.b_d = Wp.cuda(), None if Wpx is None else Wpx.cuda(), b.cuda()
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.psum = None
        if want_pool:
            self.psum = torch.full((n * M + GUARD,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
            self.psum[:n * M] = 0
        self.scr = torch.full((self.plan_q["tiles"] * 256 * M,), float("nan"), device="cuda")
        did = ctypes.c_int(-1)
        plan = (ctypes.c_int * 8)()
        rc = lib.mmmot_debug_conv_layer(vp(self.Wp_d), vp(self.Wpx_d), wps, vp(self.b_d), vp(X), X[0].numel(), n, H, W, C, M,
                                        vp(self.Y), self.y_plane, self.p_plane if want_pool else 0,
                                        ctypes.byref(did) if want_pool else None, vp(self.psum), vp(self.scr),
                                        vp(self.status), plan, None)
        torch.cuda.synchronize()
        assert rc == 0, rc
        self.plan = _plan_dict(plan, n, H, W)
        self.did_pool = did.value if want_pool else 0
        assert self.plan == self.plan_q, (self.plan, self.plan_q)
        assert self.did_pool == self.plan["pool"]
        self.n, self.H, self.W, self.M = n, H, W, M

    def output(self):
        n, H, W, M = self.n, self.H, self.W, self.M
        if self.did_pool:
            shape = (n, H // 2, W // 2, M)
            y = _read_planes(self.Y, self.p_plane, n * (H // 2) * (W // 2) * M, shape)
        else:
            y = _read_planes(self.Y, self.y_plane, n * H * W * M, (n, H, W, M))
        return y.permute(0, 3, 1, 2)       # NCHW

    def planes_nhwc(self):
        b = self.Y.cpu()
        ext = self.n * self.H * self.W * self.M
        shape = (self.n, self.H, self.W, self.M)
        return b[:ext].view(torch.float16).reshape(shape), b[self.y_plane:self.y_plane + ext].view(torch.float16).reshape(shape)


def _case_inputs(g, n, H, W, C, M):
    w, b = _weights(g, M, C)
    x = torch.randn(n, H, W, C, generator=g)
    x_hi, x_lo = fp16_split(x)
    return w, b, x_hi, x_lo


def _packed(w, compact):
    """[M][C][3][3] fp32 -> (Wt, pack_tc tiles, pack_px tiles or None, out_scale); K order (ky*3+kx)*C + ci."""
    M, C = w.shape[:2]
    wt = w.permute(2, 3, 1, 0).reshape(9 * C, M).contiguous()
    Wp, wps = pack_tc(wt)
    return wt, Wp, pack_px(Wp, 64, 9 * C) if compact and M == 64 else None, wps


# ------------------------------------------------------------------------------------------------ GPU: conv layers
@gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_conv_layer_vs_fp64(case):
    """Every plan class of the two conv kernels against fp64 conv2d (+ bias, ReLU, 2x2 max-pool when fused), and the
    fused pool's per-image sums (pool_sum) against the fp64 sums of the pooled map.

    pool_sum tolerance: each (image, channel) sum is built from fp32 running sums that one thread keeps over at most
    m = Hp*Wp pooled values (each rounding <= 2^-24 of the running sum, so <= m 2^-24 sum|v| in all), flushed as
    round-to-nearest 2^-32 fixed point (<= 2^-33 per flush, at most m flushes), on top of the pooled values' own error
    (<= TAU * S per value): |sum - ref| <= TAU * sum S + m 2^-24 sum ref + m 2^-33 (+ 2^-24 sum TAU*S, negligible)."""
    name, C, M, H, W, n, dbg, kseg, want_pool, compact, check = case
    lib = _lib.load()
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    w, b, x_hi, x_lo = _case_inputs(g, n, H, W, C, M)
    _, Wp, Wpx, wps = _packed(w, compact)
    with lib_state(lib, dbg=dbg, kseg=kseg):
        r = ConvRun(lib, Wp, Wpx, wps, b, x_hi, x_lo, n, H, W, C, M, want_pool)
    assert check(r.plan), (name, r.plan)
    x = (x_hi.double() + x_lo.double()).permute(0, 3, 1, 2)
    ref, S = _conv_ref(x, w.double(), b.double(), r.did_pool)
    y = r.output()
    ratio = _ratio(y, ref, S)
    print(f"\n{name}: plan {dict((k, r.plan[k]) for k in PLAN_KEYS)} worst err/(tau S) = {ratio:.3g}", end="")
    assert ratio <= 1.0, (name, ratio)
    assert int(r.status.item()) == 0
    if r.psum is not None:
        ps = r.psum.cpu()
        if r.plan["pool"] and not r.plan["px"]:
            got = ps[:n * M].double().reshape(n, M) * 2.0 ** -32
            want = ref.sum(dim=(2, 3))
            m = (H // 2) * (W // 2)
            tol = TAU * S.sum(dim=(2, 3)) + m * 2.0 ** -24 * want + m * 2.0 ** -33
            worst = float(((got - want).abs() / tol).max())
            print(f"; pool_sum err/tol = {worst:.3g}", end="")
            assert worst <= 1.0, (name, worst)
        else:
            assert bool((ps[:n * M] == 0).all()), "pool_sum written although the channel-major pool did not run"
        assert bool((ps[n * M:] == 0x5A5A5A5A5A5A5A5A).all()), "pool_sum written past [n_img][M]"


@gpu
@pytest.mark.parametrize("C,M,H,W,n", [(64, 64, 64, 64, 2), (128, 128, 32, 32, 2), (512, 512, 8, 8, 4), (64, 64, 8, 8, 3)],
                         ids=["px", "cm_pool32", "cm_pool8_kseg", "px_slab"])
def test_fused_pool_matches_unfused(C, M, H, W, n):
    """The fused 2x2 max-pool equals the unfused path (bit 512: full map, then the planar max-pool) to 2^-21 |v|.  Max
    commutes with bias and ReLU, so the two differ only where two window entries tie to within the hi/lo residual."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(C + M + H + n)
    w, b, x_hi, x_lo = _case_inputs(g, n, H, W, C, M)
    _, Wp, Wpx, wps = _packed(w, True)
    with lib_state(lib):
        fused = ConvRun(lib, Wp, Wpx, wps, b, x_hi, x_lo, n, H, W, C, M, True)
    with lib_state(lib, dbg=512):
        unf = ConvRun(lib, Wp, Wpx, wps, b, x_hi, x_lo, n, H, W, C, M, True)
    assert fused.did_pool and not unf.did_pool
    yf = fused.output().permute(0, 2, 3, 1)
    yu = _pool_planar_host(*unf.planes_nhwc())
    diff = float(((yf - yu).abs() - 2.0 ** -21 * yu.abs()).max())
    print(f"\nfused vs unfused pool {fused.plan}: max |d| - 2^-21|v| = {diff:.3g}", end="")
    assert diff <= 0.0


@gpu
@pytest.mark.parametrize("kind", ["cm", "px", "px_noncompact"])
def test_conv_split_terms_alone(kind):
    """The two split terms of D += Xhi Whi + Xhi Wlo + Xlo Whi, each alone against its own fp64 reference:
    input planes (0, r) leave only Xlo Whi; packed weights with zeroed hi tiles leave only Xhi Wlo.  Each term is about
    2^-11 of the output, below what an end-to-end test sees; a missing or mis-addressed term fails by orders of
    magnitude here.  Bias 0, so the output is the term alone.

    Each term is given outputs of order one (lo plane r of order one; inputs scaled by 2^12, exactly, for Xhi Wlo): a
    term of natural size (~1e-4) would be stored with a subnormal lo plane, whose fixed 2^-24 resolution exceeds TAU S."""
    lib = _lib.load()
    C, M, H, W, n = (128, 128, 16, 16, 2) if kind == "cm" else (64, 64, 32, 32, 2)
    compact = kind == "px"
    g = torch.Generator().manual_seed(7 + len(kind))
    w, _, x_hi, x_lo = _case_inputs(g, n, H, W, C, M)
    x_hi, x_lo = x_hi * 2 ** 12, x_lo * 2 ** 12
    wt, Wp, Wpx, wps = _packed(w, compact)
    b = torch.zeros(M)
    w_hi, w_lo = _w_terms(wt)
    to_nchw = lambda t: t.permute(0, 3, 1, 2)
    wk = lambda t: t.reshape(3, 3, C, M).permute(3, 2, 0, 1)           # Wt layout -> [M][C][3][3]
    with lib_state(lib):
        # (0, r): only Xlo * Whi contributes
        r = torch.randn(n, H, W, C, generator=g).half()
        run = ConvRun(lib, Wp, Wpx, wps, b, torch.zeros_like(r), r, n, H, W, C, M, False)
        assert run.plan["px"] == (kind != "cm")
        ref, S = _conv_ref(to_nchw(r.double()), wk(w_hi), None, False)
        ratio_lo = _ratio(run.output(), ref, S)
        # W hi tiles zeroed: only Xhi * Wlo contributes
        Wpz = _zero_hi_tiles(Wp, M, 9 * C)
        Wpxz = None if Wpx is None else _zero_px_tiles(Wpx, 9 * C, 0)
        run = ConvRun(lib, Wpz, Wpxz, wps, b, x_hi, x_lo, n, H, W, C, M, False)
        ref, S = _conv_ref(to_nchw(x_hi.double()), wk(w_lo), None, False)
        ratio_hi = _ratio(run.output(), ref, S)
    print(f"\n{kind}: Xlo*Whi alone err/(tau S) = {ratio_lo:.3g}; Xhi*Wlo alone = {ratio_hi:.3g}", end="")
    assert ratio_lo <= 1.0 and ratio_hi <= 1.0, (ratio_lo, ratio_hi)


@gpu
def test_matrix_split_terms_alone():
    """As test_conv_split_terms_alone, on the matrix hook (mmmot_debug_linear_planar, fp32 channels-last out)."""
    lib = _lib.load()
    M, K, rows = 128, 256, 700
    g = torch.Generator().manual_seed(3)
    wt = torch.randn(K, M, generator=g) * K ** -0.5
    Wp, wps = pack_tc(wt)
    w_hi, w_lo = _w_terms(wt)
    b = torch.zeros(M, device="cuda")
    x_hi, x_lo = fp16_split(torch.randn(rows, K, generator=g))
    r = torch.randn(rows, K, generator=g).half() * 2.0 ** -11
    ratios = []
    for (xh, xl, Wpk, x_ref, w_ref) in ((torch.zeros_like(r), r, Wp, r, w_hi),
                                         (x_hi, x_lo, _zero_hi_tiles(Wp, M, K), x_hi, w_lo)):
        X = torch.stack([xh, xl]).contiguous().cuda()
        Y = torch.full((rows, M), float("nan"), device="cuda")
        assert lib.mmmot_debug_linear_planar(vp(Wpk.cuda()), wps, vp(b), vp(X), vp(Y), M, K, rows, None) == 0
        torch.cuda.synchronize()
        ref = x_ref.double() @ w_ref
        S = x_ref.double().abs() @ w_ref.abs()
        ratios.append(_ratio(Y.double().cpu(), ref, S))
    print(f"\nmatrix: Xlo*Whi alone err/(tau S) = {ratios[0]:.3g}; Xhi*Wlo alone = {ratios[1]:.3g}", end="")
    assert max(ratios) <= 1.0, ratios


@gpu
@pytest.mark.parametrize("C,H,W,n", [(256, 16, 16, 2), (512, 8, 8, 4)], ids=["K2304", "K4608"])
def test_kseg_record(C, H, W, n):
    """Records the error of the long-K layers with one pass (kseg 0) and with the default K segmentation.  How the
    wgmma accumulator rounds decides which is smaller; both must meet the bound, neither is asserted to beat the other."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(C)
    M = C
    w, b, x_hi, x_lo = _case_inputs(g, n, H, W, C, M)
    _, Wp, _, wps = _packed(w, False)
    x = (x_hi.double() + x_lo.double()).permute(0, 3, 1, 2)
    ref, S = _conv_ref(x, w.double(), b.double(), False)
    out = {}
    for kseg in (0, KSEG_DEFAULT):
        with lib_state(lib, dbg=0, kseg=kseg):
            r = ConvRun(lib, Wp, None, wps, b, x_hi, x_lo, n, H, W, C, M, False)
        y = r.output()
        nz = ref > 0
        out[kseg] = (r.plan["ksegs"], _ratio(y, ref, S), float(((y - ref).abs() / S)[nz].mean()))
    print(f"\nK={9 * C}: " + "; ".join(f"kseg {k}: {s} segment(s), worst err/(tau S) {a:.3g}, mean err/S {m:.3g}"
                                   for k, (s, a, m) in out.items()), end="")
    assert out[0][0] == 1 and out[KSEG_DEFAULT][0] > 1
    assert max(v[1] for v in out.values()) <= 1.0


@gpu
@pytest.mark.parametrize("C,M,H,W,n,dbg,kseg", [(64, 64, 16, 16, 2, 0, None), (64, 64, 16, 16, 1, 256, None),
                                                 (128, 128, 8, 8, 2, 0, None), (256, 256, 8, 8, 4, 0, None),
                                                 (128, 128, 8, 8, 4, 0, 8)],
                         ids=["px", "px_nohalo", "cm", "cm_kseg", "cm_pool_kseg8"])
def test_conv_range_flag(C, M, H, W, n, dbg, kseg):
    """An output at or above 65504 (FP16's range) raises bit 0 of the status word; the same case scaled just below
    does not.  (The inputs of these layers are FP16 planes already: they cannot leave the range.)"""
    lib = _lib.load()
    g = torch.Generator().manual_seed(C + n + dbg)
    w, b, x_hi, x_lo = _case_inputs(g, n, H, W, C, M)
    x = (x_hi.double() + x_lo.double()).permute(0, 3, 1, 2)
    peak = float(_conv_ref(x, w.double(), b.double(), False)[0].max())
    for target, flagged in ((70000.0, 1), (64000.0, 0)):
        f = target / peak
        ws, bs = (w * f).float(), (b * f).float()
        _, Wp, Wpx, wps = _packed(ws, True)
        want_pool = kseg is not None
        with lib_state(lib, dbg=dbg, kseg=kseg):
            r = ConvRun(lib, Wp, Wpx, wps, bs, x_hi, x_lo, n, H, W, C, M, want_pool)
        top = float(_conv_ref(x, ws.double(), bs.double(), False)[0].max())
        assert (top >= 65504.0) == bool(flagged) and top < 65504 * 1.2
        assert int(r.status.item()) & 1 == flagged, (target, r.plan)


# ------------------------------------------------------------------------------------------------ GPU: first layer
CONV0_SHAPES = [(32, 32, 2), (64, 64, 2), (96, 96, 2), (224, 224, 2), (64, 32, 3), (32, 512, 2)]
VARIANTS = {"gen27": (0, 0), "im2col": (16384, 1), "ffma": (32, 2)}


def _conv0_inputs(g, n, H, W, scale_x=1.0, scale_w=1.0):
    x = torch.randn(n, 3, H, W, generator=g) * scale_x
    w = torch.randn(64, 3, 3, 3, generator=g) * (2.0 / 27) ** 0.5 * scale_w
    b = torch.randn(64, generator=g) * 0.1 * scale_w
    return x, w, b


def _run_conv0(lib, x, w, b, dbg, w_packed=None, wpx=None):
    n, _, H, W = x.shape
    wt_ffma = w.permute(2, 3, 1, 0).reshape(27, 64).contiguous()     # [(ky*3+kx)*3 + ci][co]
    Wp, wps = pack_tc(w.reshape(64, 27).t())                           # k = ci*9 + ky*3 + kx
    if w_packed is not None:
        Wp = w_packed
    Wpx = pack_px(Wp, 64, 27) if wpx is None else wpx
    ext = n * H * W * 64
    plane = ext + GUARD
    Y = _out_buffer(plane)
    cols = torch.empty(2 * n * H * W * 32, dtype=torch.float16, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    variant = ctypes.c_int(-1)
    xd = x.contiguous().cuda()
    keep = [t.cuda() for t in (wt_ffma, b, Wp, Wpx)]
    with lib_state(lib, dbg=dbg):
        rc = lib.mmmot_debug_vgg_conv0(vp(xd), n, H, W, vp(keep[0]), vp(keep[1]), vp(keep[2]), wps, vp(keep[3]), vp(Y), plane,
                                       vp(cols), vp(status), ctypes.byref(variant), None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    return _read_planes(Y, plane, ext, (n, H, W, 64)).permute(0, 3, 1, 2), variant.value, int(status.item())


@gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("H,W,n", CONV0_SHAPES + [(32, 544, 1), (64, 64, 20)], ids=lambda v: str(v))
def test_vgg_conv0_vs_fp64(variant, H, W, n):
    """The first layer's three variants (taps generated in the kernel, im2col + the compact-weight pixel-major matrix
    kernel, FP32 FFMA) against fp64 conv2d of the fp32 crops.  Border pixels are where the producers' staging and
    padding predicates live; 32x512 is the widest staging span the producers take, 32x544 falls back to im2col, and
    64x64 x 20 images (320 tiles) makes both producer groups wrap the stage ring."""
    lib = _lib.load()
    dbg, expect = VARIANTS[variant]
    if variant == "gen27" and W > 512:
        expect = 1
    g = torch.Generator().manual_seed(H * 1000 + W + n)
    x, w, b = _conv0_inputs(g, n, H, W)
    y, got, status = _run_conv0(lib, x, w, b, dbg)
    assert got == expect, (variant, got)
    ref, S = _conv_ref(x.double(), w.double(), b.double(), False)
    ratio = _ratio(y, ref, S)
    print(f"\nconv0 {variant} {H}x{W} n={n}: worst err/(tau S) = {ratio:.3g}", end="")
    assert ratio <= 1.0 and status == 0


@gpu
@pytest.mark.parametrize("variant", ["gen27", "im2col"])
def test_vgg_conv0_split_terms_alone(variant):
    """The first layer's split terms alone.  Packed weights with zeroed hi tiles leave Xhi Wlo; with zeroed lo tiles
    the output is (Xhi + Xlo) Whi, which fails by ~2^-11 of the output if the Xlo Whi MMA is missing.  The crops of the
    Xhi Wlo run are scaled by 2^12 so that the term's outputs are of order one (see test_conv_split_terms_alone)."""
    lib = _lib.load()
    dbg, _ = VARIANTS[variant]
    g = torch.Generator().manual_seed(5)
    n, H, W = 2, 64, 64
    x, w, _ = _conv0_inputs(g, n, H, W)
    b = torch.zeros(64)
    wt = w.reshape(64, 27).t()
    Wp, _ = pack_tc(wt)
    w_hi, w_lo = _w_terms(wt)
    wk = lambda t: t.t().reshape(64, 3, 3, 3)
    x12 = x * 2 ** 12
    ratios = []
    for which, xin, x_ref, w_ref in ((0, x12, x12.half().double(), w_lo), (1, x, x.double(), w_hi)):
        t = Wp.clone().view(torch.int16).view(1, 1, 2, 4, 16, 8, 8)
        t[:, :, which] = 0
        Wz = t.reshape(-1).view(torch.uint8)
        y, _, _ = _run_conv0(lib, xin, w, b, dbg, w_packed=Wz, wpx=_zero_px_tiles(pack_px(Wp, 64, 27), 27, which))
        ref, S = _conv_ref(x_ref, wk(w_ref), None, False)
        ratios.append(_ratio(y, ref, S))
    print(f"\nconv0 {variant}: Xhi*Wlo alone err/(tau S) = {ratios[0]:.3g}; X*Whi = {ratios[1]:.3g}", end="")
    assert max(ratios) <= 1.0, ratios


@gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_vgg_conv0_range_flag(variant):
    """Status bit 0 on the first layer: an output at or above 65504 raises it, just below does not; so does an input
    at or above 65504 on the variants that convert the crops to FP16 (the FFMA variant reads them as fp32)."""
    lib = _lib.load()
    dbg, _ = VARIANTS[variant]
    g = torch.Generator().manual_seed(11)
    n, H, W = 1, 32, 32
    x, w, b = _conv0_inputs(g, n, H, W)
    peak = float(_conv_ref(x.double(), w.double(), b.double(), False)[0].max())
    for target, flagged in ((70000.0, 1), (64000.0, 0)):
        f = target / peak
        _, _, status = _run_conv0(lib, x, (w * f).float(), (b * f).float(), dbg)
        assert status & 1 == flagged, ("output", target, status)
    if variant != "ffma":
        for top, flagged in ((70000.0, 1), (65000.0, 0)):
            xs = x / x.abs().max() * top
            _, _, status = _run_conv0(lib, xs, w * 1e-3, b * 1e-3, dbg)
            assert status & 1 == flagged, ("input", top, status)


# ------------------------------------------------------------------------------------------------ CPU: launch plans
def _candidates():
    for cx in (256, 128, 64, 32, 16, 8, 4, 2, 1):
        cy = 256 // cx
        while cy >= 1:
            yield cx, cy, 256 // (cx * cy)
            cy //= 2


def _waste(n, H, W, bx, by, bi):
    return math.ceil(W / bx) * bx / W * math.ceil(H / by) * by / H * math.ceil(n / bi) * bi / n


POOL_AFTER = (1, 3, 6, 9, 12)      # VGG16 "D": conv layers followed by a 2x2 max-pool (appearance.cu kPoolAfter)


def _vgg_layers(hw):
    """(cin, cout, H, W, pool after) of VGG conv layers 1..12 at crop size hw."""
    out, h = [], hw
    for i, (_, cin, cout) in enumerate(l for stage in VGG_STAGES for l in stage):
        if i > 0:
            out.append((cin, cout, h, h, i in POOL_AFTER))
        if i in POOL_AFTER:
            h //= 2
    return out


def test_vgg_layer_table():
    layers = _vgg_layers(64)
    assert [(c, m) for c, m, *_ in layers] == [(64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256),
                                                (256, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512)]
    assert [h for _, _, h, _, _ in layers] == [64, 32, 32, 16, 16, 16, 8, 8, 8, 4, 4, 4]
    assert [p for *_, p in layers] == [True, False, True, False, False, True, False, False, True, False, False, True]


@pytest.mark.parametrize("dbg,kseg", [(0, 36), (0, 0), (0, 8), (64, 36), (256, 36), (512, 36), (64, 8)])
def test_conv_plans_well_formed(lib_built, dbg, kseg):
    """Every plan over the VGG layers at crop sizes 32..224 and odd image counts is well formed, and its box has the
    least padding waste of all candidates (the pixel-major kernel may take 16 x 16 x 1 when it wastes no more)."""
    lib = _lib.load()
    with lib_state(lib, dbg=dbg, kseg=kseg):
        for hw in (32, 64, 96, 224):
            for C, M, H, W, pool in _vgg_layers(hw) + [(64, 64, 24, 40, False), (512, 512, 2, 2, True)]:
                for n in (1, 3, 6, 17, 64, 256):
                    for want_pool in {pool, False}:
                        for use_kseg in (True, False):
                            p = _plan(lib, n, H, W, C, M, want_pool, use_kseg)
                            bx, by, bi = p["bx"], p["by"], p["bi"]
                            ctx = (hw, C, M, H, W, n, want_pool, use_kseg, p)
                            assert all(v > 0 and v & (v - 1) == 0 for v in (bx, by, bi)) and bx * by * bi == 256, ctx
                            assert not p["halo"] or (p["px"] and bi == 1 and bx >= 8 and not dbg & 256), ctx
                            assert not p["pool"] or (want_pool and H % 2 == 0 and W % 2 == 0 and not dbg & 512), ctx
                            assert p["px"] == (M == 64 and not dbg & 64 and not (use_kseg and 0 < kseg < 9 * C // 32)), ctx
                            kc = 9 * C // 32
                            want_segs = math.ceil(kc / kseg) if use_kseg and 0 < kseg < kc else 1
                            assert p["ksegs"] == want_segs, ctx
                            assert p["tiles"] == math.ceil(W / bx) * math.ceil(H / by) * math.ceil(n / bi), ctx
                            best = min(_waste(n, H, W, *c) for c in _candidates())
                            assert _waste(n, H, W, bx, by, bi) <= best + 1e-9, ctx


def test_conv_plan_needs_no_gpu(lib_built):
    lib = _lib.load()
    arr = (ctypes.c_int * 8)()
    assert lib.mmmot_debug_conv_plan(4, 8, 8, 64, 64, 1, 1, arr) == 0
    E_ARG = -1
    assert lib.mmmot_debug_conv_plan(4, 8, 8, 48, 64, 0, 0, arr) == E_ARG     # C not a multiple of 32
    assert lib.mmmot_debug_conv_plan(0, 8, 8, 64, 64, 0, 0, arr) == E_ARG
    assert lib.mmmot_debug_conv_plan(4, 8, 8, 64, 64, 0, 0, None) == E_ARG


def test_case_table_takes_named_paths(lib_built):
    """Each GPU case's plan, computed on the host, is the path the case is named after."""
    lib = _lib.load()
    for name, C, M, H, W, n, dbg, kseg, want_pool, _, check in CASES:
        with lib_state(lib, dbg=dbg, kseg=kseg):
            p = _plan(lib, n, H, W, C, M, want_pool)
        assert check(p), (name, p)
    assert 147 % SMS and 147 % 2


def test_gpu_cases_cover_bench_plans(lib_built):
    """Coverage guard: every conv-layer plan class the benchmark configurations (cfg2, cfg3, cfg4: 64x64 crops) can
    launch is exercised by a case of test_conv_layer_vs_fp64."""
    import bench
    lib = _lib.load()
    covered = set()
    for name, C, M, H, W, n, dbg, kseg, want_pool, _, _ in CASES:
        with lib_state(lib, dbg=dbg, kseg=kseg):
            covered.add(plan_class(_plan(lib, n, H, W, C, M, want_pool)))
    missing = {}
    with lib_state(lib):
        for cfg in ("cfg2", "cfg3", "cfg4"):
            c = bench.CONFIGS[cfg]
            assert c["hw"] == 64
            for n_img in bench_n_imgs(c["pairs"], 2 * c["n"]):
                for C, M, H, W, pool in _vgg_layers(c["hw"]):
                    k = plan_class(_plan(lib, n_img, H, W, C, M, pool))
                    if k not in covered:
                        missing.setdefault(k, (cfg, n_img, C, M, H, W))
    assert not missing, missing
