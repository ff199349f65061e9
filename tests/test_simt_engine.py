"""The FP32 FFMA engine (csrc/gemm_simt.cuh) in every operand mode, element by element against fp64.

The engine runs every training-mode forward (the 13 VGG convolutions as XM_CONV3, w_det, PointNet with its per-detection
head addend) and the eval path of small frame-pairs (VGG when L.H.W < 32768, PointNet at L < 16, affinity layer 1 at
N.M < 64, fusion and w_det at L < 64).  Each GPU case below runs one launch through mmmot_debug_simt_op at the shapes
and strides one of those call sites passes, or at the edges the kernel's index arithmetic has to get right: column tiles
spanning 8 or 32 images of a 4x4 or 2x2 map, where the 9-tap validity mask is all that keeps a tap out of the
neighbouring image; K = 27, not a multiple of the 16-wide k-tile; the TM = 64 instantiation; odd maps (5x9), whose
4-column store groups straddle images and take the scalar store branch; partial last tiles; the pairwise column
decoding s = i*m + j at n or m = 1; the addend lookup addend[co*ld_add + seg[c]] on ragged tile tables.

Reference.  The operand is formed in fp32 exactly as the loader forms it (torch's fp32 elementwise ops are IEEE):
x (XM_DIRECT), relu(fma(x, sc, sh)) (XM_NORM_RELU; the fma as one fp64 multiply-add rounded to fp32), a*b, (a-b)*0.5
and its absolute value (XM_PAIR_*), the zero-padded im2col with k = (ky*3 + kx)*Cin + ci (XM_CONV3).  The contraction
is then done in fp64.

Bound.  Every output against the chain bound of the engine's sequential fma accumulation, kernel_kit.contraction_bound
(derived there, not measured); the CPU self-test below shows with an fp32 emulation of the kernel's arithmetic that a
single dropped or wrong tap at K = 4608 misses it by far more than an order of magnitude.

Every launch also fills Y and the partials with NaN first: every element the launch owns must be written and every
other element of the buffer (gaps of padded strides and a guard band past the end) must stay NaN.  The GroupNorm
partials are checked against fp64 statistics of the kernel's own stored Y, to the bound of kernel_kit.stats_ratios.
"""
import ctypes
import dataclasses
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_kit import (CSRC, XM, case_seed, contraction_bound, nan_output, norm_operand, pair_operand, reduce_parts,
                        report, stats_ratios, vp, worst_ratio)
from mmmot_b200 import _lib

gpu = pytest.mark.gpu
TN = 128        # the engine's column tile
GUARD = 512     # NaN floats past the end of every output buffer


# ------------------------------------------------------------------------------------------------ reference
def im2col(x):
    """x [n_img][Cin][H][W] -> the zero-padded 3x3 operand [9*Cin][n_img*H*W], row (ky*3 + kx)*Cin + ci."""
    n_img, cin, h, w = x.shape
    cols = F.unfold(x, 3, padding=1).view(n_img, cin, 9, h * w)
    return cols.permute(2, 1, 0, 3).reshape(9 * cin, n_img * h * w)


def emulate_fp32(wt, xin, bias=None, add=None, relu=False):
    """The kernel's arithmetic in numpy: acc = fma(w_k, x_k, acc) for k = 0..K-1 (an fp64 multiply-add rounded to fp32),
    then + bias, + addend and ReLU in fp32.  wt [K][M], xin [K][C] float32."""
    w, x = wt.astype(np.float64), xin.astype(np.float64)
    acc = np.zeros((wt.shape[1], xin.shape[1]), np.float32)
    for k in range(wt.shape[0]):
        acc = (acc.astype(np.float64) + w[k][:, None] * x[k][None, :]).astype(np.float32)
    if bias is not None:
        acc = acc + bias[:, None]
    if add is not None:
        acc = acc + add
    return np.maximum(acc, np.float32(0)) if relu else acc


# ------------------------------------------------------------------------------------------------ CPU: bound self-test
def test_bound_self_test():
    """The bound holds for an fp32 emulation of the kernel's arithmetic and rejects two one-element faults by more than
    an order of magnitude: a conv at K = 4608 (512 -> 64, two 3x3 images) with one valid tap of an edge pixel dropped,
    and a NORM_RELU head contraction (K = 64, ragged detections) with one column taking the neighbouring detection's
    addend.  Also: im2col's k order reproduces torch's conv2d in fp64."""
    g = torch.Generator().manual_seed(5)
    # conv, K = 4608
    cin, M, h, w = 512, 64, 3, 3
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(9 * cin, M, generator=g) * (9 * cin) ** -0.5
    b = torch.randn(M, generator=g) * 0.5
    xin = im2col(x)
    w4 = wt.double().view(3, 3, cin, M).permute(3, 2, 0, 1)              # [co][ci][ky][kx]
    conv = F.conv2d(x.double(), w4, b.double(), padding=1).permute(1, 0, 2, 3).reshape(M, -1)
    ref, T = contraction_bound(wt.double(), xin.double(), b.double())
    assert float((conv - ref).abs().max()) <= 1e-12 * float(conv.abs().max())
    good = emulate_fp32(wt.numpy(), xin.numpy(), b.numpy())
    r_ok = worst_ratio(torch.from_numpy(good), ref, T)
    col, tap = 1 * h * w + 0 * w + (w - 1), 3                            # image 1, top-right pixel; its left neighbour
    ci = int(x[1, :, 0, w - 2].abs().argmax())
    bad = xin.clone()
    bad[tap * cin + ci, col] = 0
    r_bad = worst_ratio(torch.from_numpy(emulate_fp32(wt.numpy(), bad.numpy(), b.numpy())), ref, T)
    report("emulation conv K=4608", err_over_bound=r_ok, dropped_tap=r_bad)
    assert r_ok <= 1.0 and r_bad > 10.0, (r_ok, r_bad)
    # NORM_RELU with the per-detection addend
    K, M = 64, 64
    counts = [1, 5, 1, 30, 2, 1, 17]
    seg = torch.tensor(np.repeat(np.arange(len(counts)), counts))
    P = len(seg)
    v = torch.randn(K, P, generator=g)
    sc, sh = torch.randn(K, 1, generator=g), torch.randn(K, 1, generator=g) * 0.5
    xin = norm_operand(v, sc.expand(K, P), sh.expand(K, P))
    wt = torch.randn(K, M, generator=g) * K ** -0.5
    b = torch.randn(M, generator=g) * 0.5
    addend = torch.randn(M, len(counts), generator=g)
    add = addend[:, seg]
    ref, T = contraction_bound(wt.double(), xin.double(), b.double(), add.double(), relu=True)
    good = emulate_fp32(wt.numpy(), xin.numpy(), b.numpy(), add.numpy(), relu=True)
    r_ok = worst_ratio(torch.from_numpy(good), ref, T)
    wrong = add.clone()
    c = int(np.cumsum(counts)[2])                                         # first point of detection 3
    wrong[:, c] = addend[:, 4]
    bad = emulate_fp32(wt.numpy(), xin.numpy(), b.numpy(), wrong.numpy(), relu=True)
    r_bad = worst_ratio(torch.from_numpy(bad), ref, T)
    report("emulation head addend", err_over_bound=r_ok, neighbour_addend=r_bad)
    assert r_ok <= 1.0 and r_bad > 10.0, (r_ok, r_bad)


# ------------------------------------------------------------------------------------------------ cases
@dataclasses.dataclass
class Case:
    """One launch.  tiling "uniform": `groups` groups of S columns; "table" / "table+addend": the ragged per-pair tile
    table PointNet builds (128-column tiles over each pair's points), counts[pair] = points per detection, or, with
    ne = (G, n, m), the table ne_tiles_kernel builds for the affinity stage's new/end MLP (groups (g, new | end))."""
    name: str
    mode: int
    M: int
    K: int
    tiling: str = "uniform"
    S: int = 0
    groups: int = 1
    x_gs: int = 0
    x_ks: int = 0
    y_gs: int = 0
    y_ms: int = 0
    n: int = 0
    m: int = 0
    Lf: int = 0
    H: int = 0
    W: int = 0
    counts: tuple = ()
    ne: tuple = ()
    bias: bool = True
    relu: bool = False
    part: bool = True

    @property
    def key(self):
        return (self.mode, self.M, self.K, self.tiling)


def conv_case(cin, cout, h, w, n_img, bias=True, relu=False, part=True):
    return Case(f"conv{cin}-{cout}-{h}x{w}x{n_img}{'-relu' if relu else ''}", XM.CONV, cout, 9 * cin, S=n_img * h * w, H=h,
                W=w, bias=bias, relu=relu, part=part)


def pair_case(op, n, m, G, M=1024, pad=0):
    name = ("mul", "abs", "sub")[op - XM.MUL]
    return Case(f"{name}-{n}x{m}-G{G}-M{M}", op, M, 512, S=n * m, groups=G, n=n, m=m, Lf=n + m + pad, y_gs=M * n * m,
                y_ms=n * m)


def strided_case(name, mode, M, K, S, groups, x_gs, x_ks, y_gs, y_ms, **kw):
    return Case(name, mode, M, K, S=S, groups=groups, x_gs=x_gs, x_ks=x_ks, y_gs=y_gs, y_ms=y_ms, **kw)


# Ragged detections of two pairs (L = 8): 1-point detections, detections across the 128-column tile boundaries, and a
# pair boundary inside a tile row of the other pair's table.
PN_COUNTS = ((1, 130, 1, 64, 127, 1, 3, 250), (128, 1, 77, 1, 1, 300, 2, 9))
PN_P = sum(map(sum, PN_COUNTS))


def table_case(name, mode, M, K, ld_pad=0, addend=False, relu=False):
    ld = PN_P + ld_pad
    return Case(name, mode, M, K, tiling="table+addend" if addend else "table", x_ks=ld, y_ms=ld, counts=PN_COUNTS,
                relu=relu)


def ne_case(name, mode, M, G, n, m):
    """affinity.cu's FP32 new/end MLP: V [512][ldv], ldv = G (n + m), column g (n + m) + r of pair g is new vector r < m
    or end vector r - m; tiles of group 2g over the m new columns, then of group 2g + 1 over the n end columns."""
    ld = G * (n + m)
    return Case(name, mode, M, 512, tiling="table", x_ks=ld, y_ms=ld, ne=(G, n, m))


def table_tiles(c):
    """-> (tiles [(group, first absolute column, length)], group of each column 0..P-1) of a table case."""
    if c.ne:
        G, n, m = c.ne
        tiles = [(2 * g + e, g * (n + m) + e * m + t0, min(TN, cnt - t0)) for g in range(G)
                 for e, cnt in ((0, m), (1, n)) for t0 in range(0, cnt, TN)]
    else:
        pair_pts = [sum(cp) for cp in c.counts]
        starts = np.concatenate([[0], np.cumsum(pair_pts)])
        tiles = [(p, int(starts[p]) + t0, min(TN, pair_pts[p] - t0)) for p in range(len(pair_pts)) for t0 in range(0, pair_pts[p], TN)]
    grp = np.zeros(max(c0 + ln for _, c0, ln in tiles), np.int64)
    for gi, c0, ln in tiles:
        grp[c0:c0 + ln] = gi
    return tiles, torch.from_numpy(grp)


CONV_CASES = [
    conv_case(3, 64, 224, 224, 2, relu=True, part=False),   # K = 27, TM = 64: eval layer 0 at full crop size
    conv_case(3, 64, 5, 9, 3, bias=False),                  # odd map: scalar stores, vectors straddling images
    conv_case(64, 64, 224, 224, 2),                         # training layer 1
    conv_case(64, 64, 64, 64, 3, relu=True, part=False),
    conv_case(64, 128, 64, 64, 4),
    conv_case(128, 128, 14, 14, 5, relu=True),
    conv_case(128, 256, 7, 7, 9),                           # 441 columns: a 57-column last tile
    conv_case(256, 256, 14, 14, 3, bias=False, relu=True),
    conv_case(256, 512, 4, 4, 26),                          # 8 images per tile, a 32-column last tile
    conv_case(256, 512, 2, 2, 24, relu=True, part=False),   # 24 images in one partial tile
    conv_case(512, 512, 2, 2, 40),                          # K = 4608, 32 images per tile
    conv_case(512, 512, 7, 7, 3, relu=True),
    conv_case(512, 512, 5, 9, 4, relu=True),                # odd map at K = 4608
]
PAIR_SHAPES = [(1, 1, 3), (1, 7, 6), (7, 1, 3), (6, 8, 6), (5, 13, 3), (12, 16, 6), (128, 128, 3)]
PAIR_CASES = ([pair_case(op, n, m, G) for op in (XM.MUL, XM.ABS, XM.SUB) for n, m, G in PAIR_SHAPES]
              + [pair_case(XM.MUL, 5, 13, 3, M=64, pad=2), pair_case(XM.ABS, 1, 7, 6, M=64), pair_case(XM.SUB, 12, 16, 3, M=64, pad=1)])
TABLE_CASES = [
    table_case("pn-l1", XM.DIRECT, 64, 3),                     # PointNet trunk (FP32 path: training, or L < 16)
    table_case("pn-l2", XM.NORM, 64, 64),
    table_case("pn-l4", XM.NORM, 128, 64, relu=True),
    table_case("pn-l5", XM.NORM, 1024, 128),
    table_case("pn-head", XM.NORM, 512, 64, addend=True),      # + U[:, det(p)], ld_add = ndet
    table_case("pn-head-relu", XM.NORM, 512, 64, addend=True, relu=True),
    ne_case("ne-l1-G3-7x130", XM.DIRECT, 512, 3, 7, 130),      # affinity new/end MLP (FP32 path: N.M < 64 in eval)
    ne_case("ne-l1-G2-1x1", XM.DIRECT, 512, 2, 1, 1),
    ne_case("ne-l2-G2-129x1", XM.NORM, 128, 2, 129, 1),
    table_case("pn-l5-padded", XM.NORM, 1024, 128, ld_pad=5),  # x_ks = y_ms > columns: the gap columns stay NaN
]
STRIDED_CASES = (
    [strided_case(f"wdet1-L{L}", XM.DIRECT, 512, 512, L, 3, 512 * L, L, 512 * L, L, relu=L % 2 == 1) for L in (1, 5, 127, 128, 129, 300)]
    + [strided_case(f"wdet2-L{L}", XM.NORM, 256, 512, L, 3, 512 * L, L, 256 * L, L) for L in (1, 5, 127, 128, 129, 300)]
    + [strided_case(f"wdet2-eval-L{L}", XM.DIRECT, 256, 512, L, 3, 512 * L, L, 256 * L, L, relu=True, part=False) for L in (5, 63)]
    + [strided_case(f"pn-conv2-L{L}", XM.DIRECT, 512, 512, L, 3, L, 3 * L, L, 3 * L) for L in (5, 130)]
    + [strided_case(f"pn-U-{nd}", XM.DIRECT, 512, 1024, nd, 1, 0, nd, 0, nd, bias=False, part=False) for nd in (48, 200)]
    + [strided_case(f"fusion-K{K}-L{L}", XM.DIRECT, 512, K, L, 2, 1536 * L, L, 512 * L, L) for K in (512, 1024) for L in (16, 63)]
    + [strided_case(f"aff-l2-{nm}", XM.NORM, 512, 512, nm, 3, 1024 * nm, nm, 512 * nm, nm) for nm in (48, 65)]
    + [strided_case(f"aff-l3-{nm}", XM.NORM, 128, 512, nm, 3, 512 * nm, nm, 128 * nm, nm) for nm in (48, 65)]
    + [strided_case("padded-rows", XM.NORM, 192, 96, 130, 2, 140 * 96, 140, 192 * 150, 150, relu=True)]   # gaps stay NaN
)
CASES = CONV_CASES + PAIR_CASES + TABLE_CASES + STRIDED_CASES

# Every gemm_simt_launch call site of the product: (file, what, mode, M, K, tiling).
CALL_SITES = (
    [("appearance.cu", f"VGG conv {ci}->{co}, eval and training", XM.CONV, co, 9 * ci, "uniform") for ci, co in
     ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 512), (512, 512))]
    + [("train.cu", "w_det layer 1", XM.DIRECT, 512, 512, "uniform"), ("train.cu", "w_det layer 2", XM.NORM, 256, 512, "uniform"),
       ("affinity.cu", "layer 1 multiply", XM.MUL, 1024, 512, "uniform"),
       ("affinity.cu", "layer 1 minus_abs", XM.ABS, 1024, 512, "uniform"),
       ("affinity.cu", "layer 1 minus", XM.SUB, 1024, 512, "uniform"),
       ("affinity.cu", "new/end layer 1", XM.DIRECT, 512, 512, "table"),
       ("affinity.cu", "new/end layer 2", XM.NORM, 128, 512, "table"),
       ("affinity.cu", "layer 2", XM.NORM, 512, 512, "uniform"), ("affinity.cu", "layer 3", XM.NORM, 128, 512, "uniform"),
       ("fusion_det.cu", "fusion A input", XM.DIRECT, 512, 1024, "uniform"),
       ("fusion_det.cu", "fusion B/C inputs and gates", XM.DIRECT, 512, 512, "uniform"),
       ("fusion_det.cu", "w_det layer 1", XM.DIRECT, 512, 512, "uniform"),
       ("fusion_det.cu", "w_det layer 2", XM.DIRECT, 256, 512, "uniform"),
       ("pointnet.cu", "trunk layer 1", XM.DIRECT, 64, 3, "table"), ("pointnet.cu", "trunk layers 2, 3", XM.NORM, 64, 64, "table"),
       ("pointnet.cu", "trunk layer 4", XM.NORM, 128, 64, "table"), ("pointnet.cu", "trunk layer 5", XM.NORM, 1024, 128, "table"),
       ("pointnet.cu", "U", XM.DIRECT, 512, 1024, "uniform"), ("pointnet.cu", "head", XM.NORM, 512, 64, "table+addend"),
       ("pointnet.cu", "conv2", XM.DIRECT, 512, 512, "uniform")]
)
# gemm_simt_launch expressions per source file (the test hooks in api.cu aside); a new call site changes these counts
LAUNCH_EXPRESSIONS = {"appearance.cu": 1, "train.cu": 2, "affinity.cu": 7, "fusion_det.cu": 3, "pointnet.cu": 5}


def test_simt_cases_cover_call_sites():
    """Coverage guard: every call site of gemm_simt_launch appears among the GPU cases with its (mode, M, K, tiling),
    and the list above is every call site the sources hold."""
    found = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh")) and f != "api.cu":
            k = len(re.findall(r"gemm_simt_launch<", open(os.path.join(CSRC, f)).read()))
            if k and f != "gemm_simt.cuh":
                found[f] = k
    assert found == LAUNCH_EXPRESSIONS, found
    assert {s[0] for s in CALL_SITES} == set(LAUNCH_EXPRESSIONS)
    covered = {c.key for c in CASES}
    missing = [s for s in CALL_SITES if s[2:] not in covered]
    assert not missing, missing
    assert len({c.name for c in CASES}) == len(CASES)


def test_simt_op_hook_rejects_bad_arguments(lib_built):
    """mmmot_debug_simt_op validates its arguments before any CUDA call (without a GPU a CUDA call would return a CUDA
    error, not MMMOT_E_ARG)."""
    lib = _lib.load()
    z = ctypes.c_void_p(8)
    zi = ctypes.c_void_p(16)

    def call(mode=XM.DIRECT, M=64, K=64, X=z, x_gs=0, sc=None, sh=None, n=0, m=0, Lf=0, H=0, W=0, Cin=0, S=64, groups=1,
             tt=None, nt=0, addend=None, seg=None, ld_add=0, y_gs=0, Wt=z):
        return lib.mmmot_debug_simt_op(mode, M, K, Wt, None, 0, X, x_gs, 64, sc, sh, n, m, Lf, H, W, Cin, S, groups, tt, nt,
                                       addend, seg, ld_add, z, y_gs, 64, None, None)

    bad = [dict(mode=6), dict(mode=-1), dict(M=96), dict(M=0), dict(K=0), dict(X=None), dict(Wt=None),
           dict(mode=XM.NORM, sc=z), dict(addend=z), dict(addend=z, seg=zi, ld_add=0),
           dict(S=0), dict(groups=0), dict(tt=zi, nt=0), dict(tt=zi, nt=2, x_gs=64), dict(tt=zi, nt=2, y_gs=64),
           dict(mode=XM.MUL, n=0, m=8, Lf=8, S=0), dict(mode=XM.ABS, n=2, m=4, Lf=5, S=8), dict(mode=XM.SUB, n=2, m=4, Lf=6, S=9),
           dict(mode=XM.MUL, n=2, m=4, Lf=6, S=8, tt=zi, nt=1),
           dict(mode=XM.CONV, K=63, H=4, W=4, Cin=8, S=32), dict(mode=XM.CONV, K=72, H=4, W=4, Cin=8, S=33),
           dict(mode=XM.CONV, K=72, H=4, W=4, Cin=8, S=32, groups=2), dict(mode=XM.CONV, K=72, H=0, W=4, Cin=8, S=32),
           dict(mode=XM.CONV, K=72, H=4, W=4, Cin=8, S=32, x_gs=16), dict(mode=XM.CONV, K=72, H=4, W=4, Cin=8, S=32, tt=zi, nt=1)]
    for kw in bad:
        assert call(**kw) == -1, kw


# ------------------------------------------------------------------------------------------------ GPU
def build(c, g):
    """Inputs, launch arguments and the fp32 operand of case c.  -> dict with the device tensors for the launch, xin
    [K][C] fp32 (columns in the order groups, then columns), yidx [M][C] (flat Y offset of each output), ysize, grp [C]
    (group of each column), tile_group [num_tiles], add [M][C] or None."""
    K, M = c.K, c.M
    d = dict(sc=None, sh=None, tt=None, nt=0, addend=None, seg=None, ld_add=0, add=None, Cin=0)
    co = torch.arange(M)[:, None]
    if c.mode == XM.CONV:
        cin, hw = K // 9, c.H * c.W
        n_img = c.S // hw
        x = torch.randn(n_img, cin, c.H, c.W, generator=g).cuda()
        d["X"], d["xin"], d["Cin"] = x, im2col(x), cin
        s = torch.arange(c.S)[None]
        d["yidx"] = ((s // hw) * M + co) * hw + s % hw
        d["grp"] = torch.zeros(c.S, dtype=torch.long)
        d["tile_group"] = torch.zeros(-(-c.S // TN), dtype=torch.long)
        d["G"] = 1
    elif c.mode in (XM.MUL, XM.ABS, XM.SUB):
        f = torch.randn(c.groups, K, c.Lf, generator=g).cuda()
        d["X"], d["xin"] = f, pair_operand(f, c.mode, c.n, c.m)
    elif c.tiling == "uniform":
        size = (c.groups - 1) * c.x_gs + (K - 1) * c.x_ks + c.S
        x = torch.randn(size, generator=g).cuda()
        gi, k, s = torch.arange(c.groups)[None, :, None], torch.arange(K)[:, None, None], torch.arange(c.S)[None, None]
        d["X"], d["xin"] = x, x[(gi * c.x_gs + k * c.x_ks + s).reshape(K, -1).cuda()]
    else:
        tiles, grp = table_tiles(c)
        P = len(grp)
        d["tt"] = torch.tensor([[p, c0, ln, 0] for p, c0, ln in tiles], dtype=torch.int32).cuda()
        d["nt"] = len(tiles)
        d["tile_group"] = torch.tensor([t[0] for t in tiles])
        d["grp"] = grp
        d["G"] = int(grp.max()) + 1
        x = torch.randn((K - 1) * c.x_ks + P, generator=g).cuda()
        d["X"], d["xin"] = x, x[(torch.arange(K)[:, None] * c.x_ks + torch.arange(P)[None]).cuda()]
        d["yidx"] = co * c.y_ms + torch.arange(P)[None]
        if c.tiling == "table+addend":
            counts = [np.asarray(cp) for cp in c.counts]
            ndet = len(counts) * len(counts[0])
            seg = torch.tensor(np.repeat(np.arange(ndet), np.concatenate(counts)), dtype=torch.int32).cuda()
            d["addend"] = torch.randn(M, ndet, generator=g).cuda()
            d["seg"], d["ld_add"] = seg, ndet
            d["add"] = d["addend"][:, seg.long()]
    if c.tiling == "uniform" and c.mode != XM.CONV:
        G, S = c.groups, c.S
        d["G"] = G
        d["grp"] = torch.arange(G).repeat_interleave(S)
        d["tile_group"] = torch.arange(G).repeat_interleave(-(-S // TN))
        gi, s = torch.arange(G)[:, None], torch.arange(S)[None]
        d["yidx"] = (gi * c.y_gs)[None] + co[:, :, None] * c.y_ms + s[None]
        d["yidx"] = d["yidx"].reshape(M, G * S)
    if c.mode == XM.NORM:
        G = d["G"]
        d["sc"] = (torch.randn(G, K, generator=g)).cuda()
        d["sh"] = (torch.randn(G, K, generator=g) * 0.5).cuda()
        gc = d["grp"].cuda()
        d["xin"] = norm_operand(d["xin"], d["sc"].T[:, gc], d["sh"].T[:, gc])
    d["ysize"] = int(d["yidx"].max()) + 1
    return d


@gpu
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_simt_vs_fp64(c):
    """One mmmot_debug_simt_op launch against the fp64 contraction of the fp32 operand, every output element to the
    bound of the module docstring; NaN-filled outputs: every owned element written, every other one untouched; the
    partials against fp64 statistics of the stored Y."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(case_seed("simt", c.name))
    d = build(c, g)
    wt = (torch.randn(c.K, c.M, generator=g) * c.K ** -0.5).cuda()
    bias = (torch.randn(c.M, generator=g) * 0.5).cuda() if c.bias else None
    nt = d["nt"] if d["tt"] is not None else len(d["tile_group"])
    Y = nan_output(d["ysize"], guard=GUARD)
    part = torch.full((nt + 1, c.M, 2), float("nan"), dtype=torch.float64, device="cuda") if c.part else None
    rc = lib.mmmot_debug_simt_op(c.mode, c.M, c.K, vp(wt), vp(bias), int(c.relu), vp(d["X"]), c.x_gs, c.x_ks, vp(d["sc"]),
                                 vp(d["sh"]), c.n, c.m, c.Lf, c.H, c.W, d["Cin"], c.S, c.groups, vp(d["tt"]), d["nt"],
                                 vp(d["addend"]), vp(d["seg"]), d["ld_add"], vp(Y), c.y_gs, c.y_ms, vp(part), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    yidx = d["yidx"].cuda()
    owned = torch.zeros_like(Y, dtype=torch.bool)
    owned[yidx.reshape(-1)] = True
    assert int(owned.sum()) == yidx.numel(), "two outputs share an element"
    assert bool(torch.isnan(Y[~owned]).all()), "an element outside the outputs was written"
    got = Y[yidx]
    assert bool(torch.isfinite(got).all()), "an output was not written"
    add = None if d["add"] is None else d["add"].double()
    ref, T = contraction_bound(wt.double(), d["xin"].double(), None if bias is None else bias.double(), add, c.relu)
    ratio = worst_ratio(got, ref, T)
    stats = {}
    if c.relu:
        assert bool((got == 0).any()) and bool((got > 0).any()), "ReLU case without zeros and positives"
    if c.part:
        assert bool(torch.isfinite(part[:nt]).all()), "a partial was not written"
        assert bool(torch.isnan(part[nt:]).all()), "a partial past the last tile was written"
        S1, S2 = reduce_parts(part[:nt], d["tile_group"].cuda(), d["G"])
        rv, rm, _ = stats_ratios(S1, S2, got.T.double(), d["grp"].cuda(), d["G"])
        stats = dict(var_err_over_bound=rv, mean_err_over_bound=rm)
    report(f"simt {c.name}", err_over_bound=ratio, **stats)
    assert ratio <= 1.0, ratio
    assert all(v <= 1.0 for v in stats.values()), stats
