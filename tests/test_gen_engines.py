"""Kernel-level parity of the tensor-core contractions outside the VGG trunk against fp64, element by element: the
generated-operand engine (csrc/gemm_gen.cuh, all five producers) and the TMA-fed engine in matrix mode over PointNet's
ragged detections (csrc/gemm_tma.cuh), at the launches the affinity, PointNet and fusion stages issue.

The end-to-end tests see these contractions only through GroupNorm, softmax and per-detection means, which hide a wrong
tail column, a wrong source row or a missing addend in a few elements.  These tests run one contraction through the
product's own launch code (mmmot_debug_gen / mmmot_debug_pn_contraction) and bound every output element by

    |y - y_ref| <= TAU * S,   S = |W| A + |b|,

with A the magnitude of the operand the producer forms, from the exact fp32 inputs (MUL |f_i||g_j|; ABS, SUB
(|f_i| + |g_j|)/2; NORM |y||sc| + |sh|, which covers the fp32 fma at the ReLU cut; COPY and the FP16 planes |x|).
The reference is fp64 on the GPU.  Outputs start as NaN; rows outside every tile (a guard band after the buffer, the
gaps between groups and the rows the tests' own tile tables skip) must come back unchanged.  The GroupNorm partials,
the per-detection segment sums and PointNet's device-built tables are checked as well (see the tests).

The coverage guard at the end runs without a GPU: it classifies every launch site of the three stages at the benchmark
shapes and requires each class among the GPU cases.
"""
import ctypes

import numpy as np
import pytest
import torch

from kernel_kit import (BN, GEN, GUARD_ROWS, LAYOUTS, TAU, Cols, bench_n_imgs, check_part, check_rows, fp16_split,
                        gen_weights, lib_state, ne_table, ne_tiles_host, nan_output, pn_host_tables, pn_tiles_host,
                        ref_linear, report, run_gen, vp)
from mmmot_b200 import _lib

gpu = pytest.mark.gpu
SEG_FILL = 0x5A5A5A5A5A5A5A5A      # guard pattern after the segment sums


# ------------------------------------------------------------------------------------------------ layouts
def tail_class(length):
    """Fill of a 256-column tile: full, at least half (the second epilogue half has columns) or less than half."""
    return "full" if length == BN else "half+" if length >= BN // 2 else "lt_half"


def uniform_lengths(S):
    return [BN] * (S // BN) + ([S % BN] if S % BN else [])


# ------------------------------------------------------------------------------------------------ GPU: pairwise layer 1
# affinity.cu affinity_tc layer 1: [conv1.0 ; new/end conv0] 512 -> 1024 on the generated pairwise tensor, uniform tiling, S = n*m
PAIR_SHAPES = [(128, 128, 3), (127, 128, 4), (1, 128, 6), (20, 45, 5), (8, 8, 6), (2, 300, 4), (256, 256, 3)]
PAIR_CASES = [(op, n, m, G) for op in (GEN.MUL, GEN.ABS, GEN.SUB) for n, m, G in PAIR_SHAPES]


@gpu
@pytest.mark.parametrize("op,n,m,G", PAIR_CASES, ids=[f"{GEN.NAMES[c[0]]}-{c[1]}x{c[2]}" for c in PAIR_CASES])
def test_pairwise_vs_fp64(op, n, m, G):
    """GEN_PAIR_MUL / ABS / SUB at M = 1024, K = 512: m = 128 takes the prefetching producers (two whole rows per tile;
    127 x 128 and 1 x 128 end on a half tile), 20 x 45 tiles span rows with a tail, 8 x 8 is a quarter tile, 2 x 300 rows
    span tiles.  Features are signed; for MUL some reach 255.8, near the 255.9 range guard (products near 65504)."""
    lib = _lib.load()
    K, M, Lf, NM = 512, 1024, n + m, n * m
    g = torch.Generator().manual_seed(op * 1000 + n * 7 + m)
    wt, b, Wp, wps = gen_weights(g, K, M)
    F = torch.randn(G, Lf, K, generator=g) * (1.0 if op == GEN.MUL else 2.0)
    if op == GEN.MUL:
        hot = torch.randint(0, K, (16,), generator=g)
        F[:, :, hot] = torch.sign(torch.randn(G, Lf, 16, generator=g)) * 255.8
    gap = 7
    cols = Cols.uniform(NM, G, 0, NM + gap)
    Fd = F.cuda()
    Y, P, pref = run_gen(lib, op, wt, b, Wp, wps, Fd, cols, G * (NM + gap), n=n, m=m, Lf=Lf, S=NM, groups=G, y_gs=NM + gap)
    assert pref == (m == 128)
    F64 = Fd.double()
    a, d = F64[:, :n, None, :], F64[:, None, n:, :]
    if op == GEN.MUL:
        X, A = a * d, a.abs() * d.abs()
    else:
        X = (a - d).abs() / 2 if op == GEN.ABS else (a - d) / 2
        A = (a.abs() + d.abs()) / 2
    ref, S = ref_linear(X.reshape(-1, K), A.reshape(-1, K), wt, b)
    del X, A
    r = check_rows(Y, cols, ref, S)
    rp = check_part(P, cols, ref, S)
    report(f"pair {GEN.NAMES[op]} {n}x{m} G={G} prefetch={pref}", err_over_bound=r, part_err_over_tol=rp)
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------ GPU: GEN_NORM
# (M, K, ld_src, S, groups, dbg).  affinity.cu affinity_tc layer 2 (K = 512, M = 512, ld_src = 1024 reads y01's first
# 512 channels) and layer 3 (M = 128, ld_src = 512).  Enough groups that persistent CTAs see several groups
# (the per-group affine staging).  The last five are the engine's former single-group linear test (ld_src = K).
NORM_UNIFORM = [(512, 512, 1024, 300, 48, 0), (512, 512, 1024, 512, 36, 0), (512, 512, 1024, 400, 40, 4096),
                (512, 512, 512, 300, 48, 4096), (128, 512, 512, 300, 80, 0), (128, 512, 512, 512, 80, 0),
                (128, 512, 1024, 400, 80, 4096),
                (128, 32, 32, 256, 1, 0), (256, 96, 96, 512, 1, 0), (64, 64, 64, 300, 1, 0), (512, 512, 512, 4099, 1, 0),
                (1024, 128, 128, 1000, 1, 0)]


def _norm_inputs(g, rows, ld_src, K, groups):
    src = torch.randn(rows, ld_src, generator=g) * 1.5
    gsc = (torch.rand(groups, K, generator=g) + 0.5) * torch.sign(torch.randn(groups, K, generator=g))
    gsh = torch.randn(groups, K, generator=g) * 0.5
    return src, gsc, gsh


def _norm_ref(src, gsc, gsh, cols, K):
    y = src.cuda().double()[cols.src_row.cuda(), :K]
    sc, sh = gsc.cuda().double()[cols.grp.cuda()], gsh.cuda().double()[cols.grp.cuda()]
    return torch.relu(y * sc + sh), y.abs() * sc.abs() + sh.abs()


@gpu
@pytest.mark.parametrize("M,K,ld,S,G,dbg", NORM_UNIFORM, ids=[f"M{c[0]}_K{c[1]}_ld{c[2]}_S{c[3]}_G{c[4]}_dbg{c[5]}" for c in NORM_UNIFORM])
def test_gen_norm_uniform_vs_fp64(M, K, ld, S, G, dbg):
    """GEN_NORM over uniform tiling, default and prefetching (bit 4096) producers, with source rows wider than K."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(M + K + ld + S + G + dbg)
    wt, b, Wp, wps = gen_weights(g, K, M)
    x_gs, gap = S + 3, 5
    src, gsc, gsh = _norm_inputs(g, G * x_gs, ld, K, G)
    cols = Cols.uniform(S, G, x_gs, S + gap)
    sd, scd, shd = src.cuda(), gsc.cuda(), gsh.cuda()
    Y, P, pref = run_gen(lib, GEN.NORM, wt, b, Wp, wps, sd, cols, G * (S + gap), ld_src=ld, gsc=scd, gsh=shd, S=S, groups=G,
                         x_gs=x_gs, y_gs=S + gap, dbg=dbg)
    assert pref == bool(dbg & 4096)
    X, A = _norm_ref(src, gsc, gsh, cols, K)
    ref, Sb = ref_linear(X, A, wt, b)
    r, rp = check_rows(Y, cols, ref, Sb), check_part(P, cols, ref, Sb)
    report(f"norm uniform M={M} K={K} ld={ld} S={S} G={G} dbg={dbg}", err_over_bound=r, part_err_over_tol=rp)
    assert r <= 1.0


def _ragged_split(seed, pairs, L, lo, hi, ones=0):
    g = torch.Generator().manual_seed(seed)
    cnt = torch.randint(lo, hi, (pairs * L,), generator=g)
    cnt[:ones] = 1
    return [0] + np.cumsum(cnt.numpy()).tolist()


def _table_with_gaps(tiles, every):
    """Drops every `every`-th tile: its rows stay outside the launch and must come back unchanged."""
    return [t for i, t in enumerate(tiles) if i % every != every - 1]


# (name, M, K, tiles builder, dbg): pointnet_tc (layers 3, 4: GEN_NORM over ragged per-pair point ranges, K = 64,
# M = 64 / 128), affinity_tc (new/end layer 2: K = 512, M = 128, groups 2g / 2g+1 of lengths m / n)
def _pn_table(seed, pairs=40, L=8):
    split = _ragged_split(seed, pairs, L, 1, 200, ones=3)
    tiles = _table_with_gaps(pn_tiles_host(split, pairs, L), 7)
    return tiles, split[-1], pairs



NORM_TABLE = [("pn_l3", 64, 64, lambda: _pn_table(1), 0), ("pn_l4", 128, 64, lambda: _pn_table(2), 0),
              ("pn_l4_prefetch", 128, 64, lambda: _pn_table(3), 4096), ("ne_l2", 128, 512, ne_table, 0),
              ("ne_l2_400x20", 128, 512, lambda: ne_table(G=6, n=400, m=20), 0)]


@gpu
@pytest.mark.parametrize("name,M,K,build,dbg", NORM_TABLE, ids=[c[0] for c in NORM_TABLE])
def test_gen_norm_table_vs_fp64(name, M, K, build, dbg):
    """GEN_NORM over a tile table (absolute rows, one GroupNorm affine per group), with tiles left out on purpose."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(len(name) * 31 + M)
    tiles, rows, groups = build()
    wt, b, Wp, wps = gen_weights(g, K, M)
    src, gsc, gsh = _norm_inputs(g, rows, K, K, groups)
    cols = Cols.table(tiles)
    Y, P, pref = run_gen(lib, GEN.NORM, wt, b, Wp, wps, src.cuda(), cols, rows, ld_src=K, gsc=gsc.cuda(), gsh=gsh.cuda(), dbg=dbg)
    X, A = _norm_ref(src, gsc, gsh, cols, K)
    ref, Sb = ref_linear(X, A, wt, b)
    r, rp = check_rows(Y, cols, ref, Sb), check_part(P, cols, ref, Sb)
    report(f"norm table {name} ({cols.ntiles} tiles) prefetch={pref}", err_over_bound=r, part_err_over_tol=rp)
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------ GPU: GEN_COPY
# (name, M, K, ld_src, src offset, relu, layout): layout = ("table", builder) or ("uniform", S, groups, x_gs)
COPY_CASES = [
    ("ne_l1", 512, 512, 512, 0, 0, ("table", ne_table)),                               # affinity_tc new/end layer 1
    ("ne_l1_256", 512, 512, 512, 0, 0, ("table", lambda: ne_table(G=4, n=256, m=200))),
    ("pn_u_120", 512, 1024, 1024, 0, 0, ("uniform", 120, 1, 120)),                       # pointnet_tc U, S = pairs*L
    ("pn_u_400", 512, 1024, 1024, 0, 0, ("uniform", 400, 1, 400)),
    ("pn_conv2_L40", 512, 512, 512, 0, 0, ("uniform", 40, 5, 40)),                       # pointnet_tc conv2, groups = pairs
    ("pn_conv2_L400", 512, 512, 512, 0, 0, ("uniform", 400, 2, 400)),
    ("fusion_a", 512, 1024, 1536, 0, 0, ("uniform", 64, 3, 64)),                          # fusion_det_tc inputs, stacks 0+1
    ("fusion_bc_img", 512, 512, 1536, 0, 0, ("uniform", 128, 3, 128)),                    # fusion_det_tc inputs, stack 0
    ("fusion_bc_lidar", 512, 512, 1536, 512, 0, ("uniform", 256, 2, 256)),                # fusion_det_tc inputs, stack 1
    ("wdet_1", 512, 512, 512, 0, 1, ("uniform", 420, 1, 420)),                           # fusion_det_tc w_det1, 3 rows per det
    ("wdet_1_576", 512, 512, 512, 0, 1, ("uniform", 576, 1, 576)),
    ("wdet_2", 256, 512, 512, 0, 1, ("uniform", 400, 1, 400)),                           # fusion_det_tc w_det2
]


@gpu
@pytest.mark.parametrize("case", COPY_CASES, ids=[c[0] for c in COPY_CASES])
def test_gen_copy_vs_fp64(case):
    """GEN_COPY (always the prefetching producers) at the new/end, PointNet per-detection, fusion and w_det launches:
    tile tables, K = 1024, source rows of 1536 floats read at a stack offset, ReLU in the epilogue."""
    name, M, K, ld, off, relu, lay = case
    lib = _lib.load()
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    wt, b, Wp, wps = gen_weights(g, K, M)
    if lay[0] == "table":
        tiles, rows, _ = lay[1]()
        cols = Cols.table(tiles)
        kw = {}
        y_rows = rows
    else:
        _, S, G, x_gs = lay
        gap = 3
        cols = Cols.uniform(S, G, x_gs, S + gap)
        rows, y_rows = G * x_gs, G * (S + gap)
        kw = dict(S=S, groups=G, x_gs=x_gs, y_gs=S + gap)
    src = torch.randn(rows * ld, generator=g) * 2.0
    sd = src.cuda()
    Y, P, pref = run_gen(lib, GEN.COPY, wt, b, Wp, wps, sd[off:], cols, y_rows, ld_src=ld, relu=relu, **kw)
    assert pref == 1
    X = sd.double().view(rows, ld)[cols.src_row.cuda(), off:off + K]
    ref, Sb = ref_linear(X, X.abs(), wt, b)
    r = check_rows(Y, cols, ref, Sb, relu=bool(relu))
    rp = check_part(P, cols, torch.relu(ref) if relu else ref, Sb)
    report(f"copy {name} ({cols.ntiles} tiles)", err_over_bound=r, part_err_over_tol=rp)
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------ GPU: matrix mode
# The point layouts of kernel_kit.LAYOUTS and two at the edges of the persistent kernel's work schedule, in which
# consumer warpgroup h takes column half h of every tile: in `ends` the pair totals 257, 384 and 385 leave the pairs'
# last tiles 1, 128 and 129 columns (half 1 empty, empty, one column); `single` is one pair of 129 points, a launch of
# one tile.
PN_LAYOUTS = dict(LAYOUTS, ends=(3, 4, [100, 100, 56, 1, 128, 128, 64, 64, 1, 255, 1, 128]), single=(1, 2, [60, 69]))
# kind -> (M, K, Y, part, addend, segsum), in pointnet.cu: layer 2 in pointnet_tc; pass 1 of layer 5 and of the head in
# pn_wide_stats (debug bit 4), pass 2 in pn_wide_layer
MAT_KINDS = {"l2": (64, 64, True, True, False, False), "l5_pass1": (1024, 128, False, True, False, False),
             "l5_pass2": (1024, 128, False, False, False, True), "head_pass1": (512, 64, False, True, True, False),
             "head_pass2": (512, 64, False, False, True, True)}
MAT_CASES = [(lay, kind) for lay in PN_LAYOUTS for kind in MAT_KINDS]


def _runs_per_det(tiles, seg, ndet):
    """Per detection: the 32-column chunks its points fall in (one fixed-point flush per chunk and run)."""
    keys = set()
    for t, (_, c0, ln) in enumerate(tiles):
        for c in range(ln):
            keys.add((int(seg[c0 + c]), t, c // 32))
    runs = np.zeros(ndet)
    for d, _, _ in keys:
        runs[d] += 1
    return torch.tensor(runs, dtype=torch.float64)


@gpu
@pytest.mark.parametrize("layout,kind", MAT_CASES, ids=[f"{a}-{b}" for a, b in MAT_CASES])
def test_pn_matrix_vs_fp64(layout, kind):
    """One PointNet matrix-mode launch (gemm_tma_launch_mat over the device-built tile table) on FP16 planes X[2][P][K].
    Tables: tiles, counts, first tiles, point -> detection map and chunk descriptors equal the host-built ones.
    Y / partials: as the gen tests, with the addend in S.  Segment sums: against fp64
    sum_p relu((W x_p + b + add_d) sc + sh), to |sc| TAU sum_p S_p (the values' error) + 40 2^-24 sum_p (|y_p sc| + |sh|)
    (the fp32 fmas that apply bias, addend and affine, at most three roundings, and the <= 32-term fp32 run sums) +
    2^-33 per fixed-point flush (one per 32-column chunk the detection touches)."""
    pairs, L, counts = PN_LAYOUTS[layout]
    M, K, want_y, want_part, want_add, want_seg = MAT_KINDS[kind]
    lib = _lib.load()
    ndet = pairs * L
    split = [0] + np.cumsum(counts).tolist()
    P = split[-1]
    tiles_h, seg_h, ctab_h, cnt_h, gstart_h = pn_host_tables(split, pairs, L)
    nt = len(tiles_h)
    g = torch.Generator().manual_seed(P + M + K)
    wt, b, Wp, wps = gen_weights(g, K, M)
    x = torch.randn(P, K, generator=g)
    hi, lo = fp16_split(x)
    X = torch.stack([hi, lo]).contiguous().cuda()
    add = torch.randn(ndet, M, generator=g) * 0.5 if want_add else None
    sc = (torch.rand(pairs, M, generator=g) + 0.5) * torch.sign(torch.randn(pairs, M, generator=g))
    sh = torch.randn(pairs, M, generator=g) * 0.3
    d_split = torch.tensor(split, dtype=torch.int32, device="cuda")
    h_split = torch.tensor(split, dtype=torch.int32)
    cap = nt + 3
    tiles = torch.full((cap, 4), -7, dtype=torch.int32, device="cuda")
    ctab = torch.full((2 * cap, 4), -7, dtype=torch.int32, device="cuda")
    cnt = torch.full((pairs + 2,), -7, dtype=torch.int32, device="cuda")
    gstart = torch.full((pairs + 3,), -7, dtype=torch.int32, device="cuda")
    segd = torch.full((P + 64,), -7, dtype=torch.int32, device="cuda")
    Y = nan_output(P, M, guard=GUARD_ROWS) if want_y else None
    part = torch.full((2 * nt + 4, M, 2), float("nan"), dtype=torch.float64, device="cuda") if want_part else None
    ss = None
    if want_seg:
        ss = torch.full((ndet * M + 512,), SEG_FILL, dtype=torch.int64, device="cuda")
        ss[:ndet * M] = 0
    keep = (Wp.cuda(), b.cuda(), None if add is None else add.cuda(), sc.cuda(), sh.cuda())
    n_tiles = ctypes.c_long(-1)
    rc = lib.mmmot_debug_pn_contraction(vp(d_split), vp(h_split), pairs, L, cap, vp(tiles), vp(cnt), vp(gstart), vp(segd),
                                        vp(ctab), ctypes.byref(n_tiles), vp(keep[0]), wps, vp(keep[1]), M, K, vp(X), vp(Y),
                                        vp(part), vp(keep[2]), M, vp(ss), vp(keep[3]), vp(keep[4]), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    # ---- tables
    assert n_tiles.value == nt
    tl = tiles.cpu()
    assert tl[:nt].tolist() == [[p, c, ln, 0] for p, c, ln in tiles_h] and bool((tl[nt:] == -7).all())
    assert ctab.cpu()[:2 * nt].tolist() == ctab_h and bool((ctab.cpu()[2 * nt:] == -7).all())
    assert cnt.cpu()[:pairs].tolist() == cnt_h and gstart.cpu()[:pairs + 1].tolist() == gstart_h
    assert segd.cpu()[:P].tolist() == seg_h.tolist() and bool((segd.cpu()[P:] == -7).all())
    # ---- reference
    cols = Cols.table(tiles_h)
    xr = (hi.double() + lo.double()).cuda()
    seg_t = torch.tensor(seg_h, device="cuda")
    ref, S = ref_linear(xr, xr.abs(), wt, b)
    if want_add:
        a64 = add.double().cuda()[seg_t]
        ref, S = ref + a64, S + a64.abs()
    out = {}
    if want_y:
        out["y_err_over_bound"] = check_rows(Y, cols, ref, S)
    if want_part:
        out["part_err_over_tol"] = check_part(part, cols, ref, S)
    if want_seg:
        pair_of = seg_t // L
        scp, shp = sc.double().cuda()[pair_of], sh.double().cuda()[pair_of]
        r = torch.relu(ref * scp + shp)
        acc = lambda v: torch.zeros(ndet, M, dtype=torch.float64, device="cuda").index_add_(0, seg_t, v)
        want = acc(r)
        runs = _runs_per_det(tiles_h, seg_h, ndet).cuda()[:, None]
        tol = acc(scp.abs() * TAU * S) + 40 * 2.0 ** -24 * acc((ref * scp).abs() + shp.abs()) + runs * 2.0 ** -33
        got = ss[:ndet * M].view(ndet, M).double() * 2.0 ** -32
        w = float(((got - want).abs() / tol).max())
        out["segsum_err_over_tol"] = w
        assert bool((ss[ndet * M:] == SEG_FILL).all()), "segment sums written past [det][M]"
        assert w <= 1.0, w
    report(f"matrix {layout} {kind} ({nt} tiles, P={P})", **out)
    assert out.get("y_err_over_bound", 0.0) <= 1.0


# ------------------------------------------------------------------------------------------------ CPU: coverage guard
def site_classes(lib, gen, M, K, ld_src, tiling, lengths, m=0, kind=None, dbg=0):
    """The classes of one launch: (engine, producer variant, tiling, ld_src != K, M < 128, K > 512, tile fill)."""
    if gen == "mat":
        pre = kind
    else:
        with lib_state(lib, dbg=dbg):
            pre = lib.mmmot_debug_gen_prefetch(gen, m)
            assert pre in (0, 1)
    return {(gen, pre, tiling, ld_src != K, M < 128, K > 512, tail_class(ln)) for ln in lengths}


def bench_site_classes(lib):
    """Every gemm_gen / matrix-mode launch of the affinity, PointNet and fusion stages at the benchmark shapes, with
    the stage's own use of the tensor cores (affinity n*m >= 64, PointNet L >= 16, fusion L >= 64)."""
    import bench
    out = {}

    def add(site, classes):
        for c in classes:
            out.setdefault(c, site)

    for cfg in ("cfg2", "cfg3", "cfg4", "cfg5"):
        c = bench.CONFIGS[cfg]
        op = {"multiply": GEN.MUL, "minus_abs": GEN.ABS, "minus": GEN.SUB}[c["affinity_op"]]
        ns = bench.SWEEP_N if cfg == "cfg5" else (c["n"],)
        for n in ns:
            NM = n * n
            if NM < 64:
                continue
            lengths = uniform_lengths(NM)
            add(("affinity.cu affinity_tc l1", cfg, n), site_classes(lib, op, 1024, 512, 512, "uniform", lengths, m=n))
            ne = [t[2] for t in ne_tiles_host(1, n, n, 0)[0]]
            add(("affinity.cu affinity_tc ne_l1", cfg, n), site_classes(lib, GEN.COPY, 512, 512, 512, "table", ne))
            add(("affinity.cu affinity_tc ne_l2", cfg, n), site_classes(lib, GEN.NORM, 128, 512, 512, "table", ne))
            add(("affinity.cu affinity_tc l2", cfg, n), site_classes(lib, GEN.NORM, 512, 512, 1024, "uniform", lengths))
            add(("affinity.cu affinity_tc l3", cfg, n), site_classes(lib, GEN.NORM, 128, 512, 512, "uniform", lengths))
        if cfg == "cfg5":
            continue
        L = 2 * c["n"]
        for pairs in bench_n_imgs(c["pairs"], 1):          # forward_batch's chunk sizes
            if L >= 16:
                pn = uniform_lengths(L * c["pts"])            # every detection has `pts` points: per-pair tiles
                for kind, (M, K, *_rest) in MAT_KINDS.items():
                    fn = "pointnet_tc" if kind == "l2" else "pn_wide_stats" if kind.endswith("pass1") else "pn_wide_layer"
                    add((f"pointnet.cu {fn} {kind}", cfg, pairs),
                        site_classes(lib, "mat", M, K, K, "table", pn, kind=kind))
                add(("pointnet.cu pointnet_tc l3", cfg, pairs), site_classes(lib, GEN.NORM, 64, 64, 64, "table", pn))
                add(("pointnet.cu pointnet_tc l4", cfg, pairs), site_classes(lib, GEN.NORM, 128, 64, 64, "table", pn))
                add(("pointnet.cu pointnet_tc U", cfg, pairs), site_classes(lib, GEN.COPY, 512, 1024, 1024, "uniform", uniform_lengths(pairs * L)))
                add(("pointnet.cu pointnet_tc conv2", cfg, pairs), site_classes(lib, GEN.COPY, 512, 512, 512, "uniform", uniform_lengths(L)))
            if L >= 64:
                Kf = (1024,) if c["fusion"] == "A" else (512,)
                for K in Kf:
                    add(("fusion_det.cu fusion_det_tc inputs", cfg, pairs), site_classes(lib, GEN.COPY, 512, K, 1536, "uniform", uniform_lengths(L)))
                rows = uniform_lengths(pairs * L * 3)
                add(("fusion_det.cu fusion_det_tc w_det1", cfg, pairs), site_classes(lib, GEN.COPY, 512, 512, 512, "uniform", rows))
                add(("fusion_det.cu fusion_det_tc w_det2", cfg, pairs), site_classes(lib, GEN.COPY, 256, 512, 512, "uniform", rows))
    return out


def gpu_case_classes(lib):
    cov = set()
    for op, n, m, G in PAIR_CASES:
        cov |= site_classes(lib, op, 1024, 512, 512, "uniform", uniform_lengths(n * m), m=m)
    for M, K, ld, S, G, dbg in NORM_UNIFORM:
        cov |= site_classes(lib, GEN.NORM, M, K, ld, "uniform", uniform_lengths(S), dbg=dbg)
    for _, M, K, build, dbg in NORM_TABLE:
        cov |= site_classes(lib, GEN.NORM, M, K, K, "table", [t[2] for t in build()[0]], dbg=dbg)
    for _, M, K, ld, _, _, lay in COPY_CASES:
        lengths = [t[2] for t in lay[1]()[0]] if lay[0] == "table" else uniform_lengths(lay[1])
        cov |= site_classes(lib, GEN.COPY, M, K, ld, lay[0], lengths)
    for layout, kind in MAT_CASES:
        pairs, L, counts = PN_LAYOUTS[layout]
        split = [0] + np.cumsum(counts).tolist()
        M, K, *_ = MAT_KINDS[kind]
        cov |= site_classes(lib, "mat", M, K, K, "table", [t[2] for t in pn_tiles_host(split, pairs, L)], kind=kind)
    return cov


def test_gpu_cases_cover_bench_launches(lib_built):
    """Coverage guard: every class of gemm_gen / matrix-mode launch the benchmark configurations (cfg2-cfg5) issue
    appears among the GPU cases above."""
    lib = _lib.load()
    sites = bench_site_classes(lib)
    assert len(sites) >= 10
    covered = gpu_case_classes(lib)
    missing = {k: v for k, v in sites.items() if k not in covered}
    assert not missing, missing


def test_gen_prefetch_query(lib_built):
    """gen_prefetch through the library, no GPU: pairwise producers pipeline only at m == 128, GEN_COPY always,
    GEN_NORM only with debug bit 12; bit 10 turns every pipeline off."""
    lib = _lib.load()
    with lib_state(lib):
        assert [lib.mmmot_debug_gen_prefetch(op, m) for op in (GEN.MUL, GEN.ABS, GEN.SUB) for m in (1, 127, 128, 129, 256)] == \
               [0, 0, 1, 0, 0] * 3
        assert lib.mmmot_debug_gen_prefetch(GEN.COPY, 0) == 1 and lib.mmmot_debug_gen_prefetch(GEN.NORM, 0) == 0
        assert lib.mmmot_debug_gen_prefetch(5, 0) == -1 and lib.mmmot_debug_gen_prefetch(-1, 0) == -1
    with lib_state(lib, dbg=4096):
        assert lib.mmmot_debug_gen_prefetch(GEN.NORM, 0) == 1 and lib.mmmot_debug_gen_prefetch(GEN.MUL, 64) == 0
    with lib_state(lib, dbg=1024 | 4096):
        assert all(lib.mmmot_debug_gen_prefetch(gn, 128) == 0 for gn in range(5))


def test_host_tables():
    """The host-built tables the GPU tests compare against: tiles cover each pair's points once, in order, without
    straddling pairs; a chunk descriptor marks single-detection only for complete chunks."""
    for pairs, L, counts in PN_LAYOUTS.values():
        split = [0] + np.cumsum(counts).tolist()
        tiles, seg, ctab, cnt, gstart = pn_host_tables(split, pairs, L)
        assert sum(t[2] for t in tiles) == split[-1] and len(ctab) == 2 * len(tiles) and gstart[-1] == len(tiles)
        covered = np.concatenate([np.arange(c, c + ln) for _, c, ln in tiles])
        assert (covered == np.arange(split[-1])).all()
        for p, c, ln in tiles:
            assert split[p * L] <= c and c + ln <= split[(p + 1) * L] and 0 < ln <= BN
    pairs, L, counts = LAYOUTS["edges"]
    split = [0] + np.cumsum(counts).tolist()
    assert {32, 128, 256} <= set(split) and split[-1] % BN and max(counts) > BN
    assert counts[3:6] == [1, 1, 1] and 256 <= split[3] and split[6] <= 288
    pairs, L, counts = LAYOUTS["two"]
    split = [0] + np.cumsum(counts).tolist()
    assert split[L] == 700 and counts[L - 1] >= 60
    tiles, _, ctab, _, _ = pn_host_tables(split, pairs, L)
    # pair 0's last tile: 188 points, its chunk 160..191 partial and inside the last detection -> not single
    assert tiles[2] == (0, 512, 188) and ctab[5][1] & 1 == 0 and ctab[5][0] & 1 == 1


def test_pn_layouts_end_as_named():
    """The schedule layouts' tiles end with 1, 128 and 129 columns, and `single` is one tile."""
    pairs, L, counts = PN_LAYOUTS["ends"]
    ends = [ln for _, _, ln in pn_tiles_host([0] + np.cumsum(counts).tolist(), pairs, L)]
    assert sorted(ln for ln in ends if ln < BN) == [1, 128, 129]
    pairs, L, counts = PN_LAYOUTS["single"]
    assert [ln for _, _, ln in pn_tiles_host([0] + np.cumsum(counts).tolist(), pairs, L)] == [129]
