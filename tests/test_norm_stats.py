"""GroupNorm statistics of the three contraction epilogues on channels whose mean dwarfs their spread.

Each epilogue (csrc/gemm_gen.cuh, csrc/gemm_tma.cuh matrix mode, csrc/gemm_simt.cuh) sums its outputs per channel in
fp32 runs (32 columns of a tensor-core epilogue thread, the 8 columns of an FP32-engine thread) and hands fp64
partials (sum y, sum y^2) to stats_reduce and gn_finalize, which form mean = S1/n and var = S2/n - mean^2.  Summed as
they are, the fp32 runs round S2 by about k 2^-24 (var + mean^2), so var loses (mean/std)^2 of relative accuracy,
while GroupNorm itself is conditioned only like mean/std.  The runs are therefore summed as differences from their
fp32 mean, and each run is folded into the fp64 partial exactly (stat_fold in common.cuh).

Bound.  The statistics are held to
    |dvar| <= KAPPA u (|ybar| mean|delta| + mean delta^2),   |dmean| <= KAPPA1 u mean|y|,   KAPPA = 64, KAPPA1 = 40,
u = 2^-24, ybar the mean, delta = y - ybar (kernel_kit.stats_ratios, where the constants are derived from the rounding
counts of a run).  They are empirical, not proven; what they rest on is measured by the CPU test below (an emulation of
the gemm_gen epilogue's summation order) and the GPU cases.  The bound is linear in R = |ybar|/std; the unshifted sums
err by about sqrt(k) u ybar^2, R / KAPPA times its first term, and the CPU test shows the bound rejects them at
R >= 100.

Kernel-level tests (GPU) run one contraction through the product's launch code and compare the statistics of its own
partials, reduced in fp64 as stats_reduce does, with a two-pass fp64 mean and variance over the kernel's own stored Y,
which keeps the contraction's error out of the check.  The common mode comes either from the inputs (a component all
columns share, as look-alike detections produce) or from the bias.  Every activation stays far inside FP16's range.
"""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

from kernel_kit import (GEN, KAPPA, KAPPA1, LAYOUTS, U, Cols, case_seed, eval_net, fp16_split, lib_state, ne_table,
                        pn_host_tables, reduce_parts, report, run_gen, stats_ratios, vp)
from mmmot_b200 import _lib
from mmmot_b200.weights import pack_tc

gpu = pytest.mark.gpu
RS = (1, 20, 100, 300)
SOURCES = ("input", "bias")


# ------------------------------------------------------------------------------------------------ CPU: emulation
def emulate_chunk_stats(Y, shifted):
    """The gemm_gen epilogue's partials of one group, Y [C][n] fp32 (numpy): 32-column runs in fp32 (sum y and an
    fma sum of y^2, or the sums of d = y - (the run's fp32 mean) folded into fp64), four runs per 128-column half."""
    C, n = Y.shape
    nch = -(-n // 32)
    X = np.zeros((C, nch * 32), np.float32)
    X[:, :n] = Y
    X = X.reshape(C, nch, 32)
    valid = (np.arange(nch * 32) < n).reshape(nch, 32)
    k = valid.sum(1)
    p = np.zeros((C, nch), np.float32)
    if shifted:   # the run's fp32 mean: a sequential fp32 sum of its valid values over their count
        for j in range(32):
            p = (p + np.where(valid[:, j], X[:, :, j], np.float32(0))).astype(np.float32)
        p = (p / k.astype(np.float32)).astype(np.float32)
    s1 = np.zeros((C, nch), np.float32)
    s2 = np.zeros((C, nch), np.float32)
    for j in range(32):
        d = np.where(valid[:, j], (X[:, :, j] - p).astype(np.float32), np.float32(0))
        s1 = (s1 + d).astype(np.float32)
        s2 = (s2.astype(np.float64) + d.astype(np.float64) ** 2).astype(np.float32)   # one rounding: an fma
    if shifted:
        pd, a = p.astype(np.float64), s1.astype(np.float64)
        return (k * pd + a).sum(1), (pd * (k * pd + 2 * a) + s2).sum(1)
    nh = -(-nch // 4)
    f1 = np.zeros((C, nh), np.float32)
    f2 = np.zeros((C, nh), np.float32)
    S1 = np.zeros((C, nh * 4), np.float32)
    S2 = np.zeros((C, nh * 4), np.float32)
    S1[:, :nch], S2[:, :nch] = s1, s2
    for c in range(4):
        f1 = (f1 + S1.reshape(C, nh, 4)[:, :, c]).astype(np.float32)
        f2 = (f2 + S2.reshape(C, nh, 4)[:, :, c]).astype(np.float32)
    return f1.astype(np.float64).sum(1), f2.astype(np.float64).sum(1)


@pytest.mark.parametrize("n", [16, 40, 128, 300])
def test_bound_separates_one_pass_from_shifted(n):
    """At R >= 100 the bound rejects the unshifted fp32 sums and accepts the shifted ones with a wide margin (ratio <=
    0.1); at every R the shifted sums stay inside it.  Channels of log-normal spread, signed means R std, 512 per case."""
    rng = np.random.default_rng(n)
    for R in RS:
        sd = np.exp(rng.normal(size=(512, 1)))
        Y = (R * sd * np.sign(rng.normal(size=(512, 1))) + sd * rng.normal(size=(512, n))).astype(np.float32)
        y = torch.from_numpy(Y.astype(np.float64)).T.contiguous()
        grp = torch.zeros(n, dtype=torch.long)
        out = {}
        for form in ("one_pass", "shifted"):
            S1, S2 = emulate_chunk_stats(Y, form == "shifted")
            out[form] = stats_ratios(torch.from_numpy(S1)[None], torch.from_numpy(S2)[None], y, grp, 1)
        report(f"emulation n={n} R={R}", one_pass_var=out["one_pass"][0], shifted_var=out["shifted"][0],
                shifted_mean=out["shifted"][1])
        assert out["shifted"][0] <= 1.0 and out["shifted"][1] <= 1.0, out
        assert out["one_pass"][1] <= 1.0, out
        if R >= 100:
            assert out["one_pass"][0] > 1.0 and out["shifted"][0] <= 0.1, out


# ------------------------------------------------------------------------------------------------ conditioned inputs
def conditioned_weights(g, K, M, R, source, sigma=1.0):
    """Wt [K][M], bias [M] and the operand's common vector c [K] (all >= 4 sigma, so a ReLU or |.| on the operand
    leaves it alone) such that y = (c + e) Wt + b, e iid with std sigma, has |mean| / std = R in every channel.
    source "input": b = 0 and w_m = s_m a u + r_m, u = c / |c|, r_m a unit vector orthogonal to u, a = R / sqrt(|c|^2 /
    sigma^2 - R^2), so mean = s_m a |c| and std = sigma sqrt(a^2 + 1).  source "bias": c = 0, w random, b_m = s_m R
    sigma |w_m|."""
    s = torch.sign(torch.randn(M, generator=g))
    if source == "bias":
        wt = torch.randn(K, M, generator=g) * K ** -0.5
        return wt, s * R * sigma * wt.norm(dim=0), torch.zeros(K)
    gam = max(4.0 * sigma, 3.0 * R * sigma / math.sqrt(K))
    c = gam * (1.0 + 0.5 * torch.rand(K, generator=g))
    u = c / c.norm()
    r = torch.randn(K, M, generator=g)
    r = r - u[:, None] * (u @ r)[None]
    r = r / r.norm(dim=0)
    a = R / math.sqrt((c.norm() / sigma) ** 2 - R * R)
    return (s * a)[None] * u[:, None] + r, torch.zeros(M), c


def pair_features(g, G, n, m, K, c, op):
    """Feature stacks [G][n + m][K] whose pairwise operand has the common vector c: SUB / ABS objects 2c + sqrt2 e,
    detections sqrt2 e' (operand c + (e - e')/sqrt2, |.| leaves it alone since c >= 4); MUL objects c / 8 + e / 8,
    detections 8 + e' / 8 (operand ~ c + e + small terms)."""
    e1, e2 = torch.randn(G, n, K, generator=g), torch.randn(G, m, K, generator=g)
    if op == GEN.MUL:
        return torch.cat([(c + e1) / 8, 8 + e2 / 8], 1)
    return torch.cat([2 * c + math.sqrt(2) * e1, math.sqrt(2) * e2], 1)


def _slot_groups(cols):
    """Partial slot (tile*2 + half) -> group, over the slots that hold columns."""
    sg = torch.full((cols.ntiles * 2,), -1, dtype=torch.long)
    sg[cols.hid] = cols.grp
    return sg


def check_partials(P, Y, cols, G, name):
    """The partials of the slots with columns, reduced per group in fp64, against the two-pass statistics of the stored
    Y; empty slots are zero."""
    sg = _slot_groups(cols).cuda()
    live = sg >= 0
    part = P[:cols.ntiles * 2]
    assert bool((part[~live] == 0).all()), "an empty half-tile has nonzero partials"
    S1, S2 = reduce_parts(part[live], sg[live], G)
    y = Y[cols.y_row.cuda()].double()
    rv, rm, cond = stats_ratios(S1, S2, y, cols.grp.cuda(), G)
    report(name, var_err_over_bound=rv, mean_err_over_bound=rm, max_mean_over_std=cond)
    return rv, rm, cond


# ------------------------------------------------------------------------------------------------ GPU: gemm_gen
# (name, gen, M, K, layout): layout ("uniform", S, groups) or ("table", builder) or ("pair", n, m, groups).  Uniform
# S = 16 (fusion at L = 16: half a run), 300 (a full tile and a 44-column tile whose second half is empty), 600 (three
# tiles per group, the last a 88-column tail); tables with per-group counts (the new/end MLP); pairs: 8 x 8 (N.M = 64),
# 20 x 45 (tiles across rows, tail) and 2 x 128 (the pipelined producers, two whole rows per tile).  Names ending in
# _relu take ReLU in the epilogue: its zeros count as values and can be a run's pivot.
GEN_LAYOUTS = [("copy_S16", GEN.COPY, 512, 512, ("uniform", 16, 5)), ("copy_S300", GEN.COPY, 512, 512, ("uniform", 300, 3)),
               ("copy_S600", GEN.COPY, 256, 512, ("uniform", 600, 2)), ("copy_ne", GEN.COPY, 512, 512, ("table", ne_table)),
               ("norm_S300", GEN.NORM, 512, 512, ("uniform", 300, 3)),
               ("norm_ne", GEN.NORM, 128, 512, ("table", lambda: ne_table(G=6, n=400, m=20))),
               ("mul_8x8", GEN.MUL, 1024, 512, ("pair", 8, 8, 3)), ("abs_20x45", GEN.ABS, 1024, 512, ("pair", 20, 45, 2)),
               ("sub_2x128", GEN.SUB, 1024, 512, ("pair", 2, 128, 2)), ("abs_2x128", GEN.ABS, 1024, 512, ("pair", 2, 128, 2)),
               ("mul_2x128", GEN.MUL, 1024, 512, ("pair", 2, 128, 2)),
               ("copy_S300_relu", GEN.COPY, 512, 512, ("uniform", 300, 3)), ("copy_ne_relu", GEN.COPY, 512, 512, ("table", ne_table))]
GEN_CASES = [(lay, R, src) for lay in GEN_LAYOUTS for R in RS for src in SOURCES]


@gpu
@pytest.mark.parametrize("lay,R,source", GEN_CASES, ids=[f"{c[0][0]}-R{c[1]}-{c[2]}" for c in GEN_CASES])
def test_gen_stats_conditioned(lay, R, source):
    """gemm_gen through mmmot_debug_gen on conditioned channels: every producer, uniform and table tiling."""
    name, gen, M, K, shape = lay
    lib = _lib.load()
    g = torch.Generator().manual_seed(case_seed(name, R, source))
    wt, b, c = conditioned_weights(g, K, M, R, source)
    Wp, wps = pack_tc(wt)
    kw = {}
    if shape[0] == "pair":
        _, n, m, G = shape
        src = pair_features(g, G, n, m, K, c, gen)
        cols = Cols.uniform(n * m, G, 0, n * m)
        kw = dict(n=n, m=m, Lf=n + m, S=n * m, groups=G, y_gs=n * m)
        y_rows = G * n * m
    else:
        if shape[0] == "uniform":
            _, S, G = shape
            cols = Cols.uniform(S, G, S, S)
            rows = y_rows = S * G
            kw = dict(S=S, groups=G, x_gs=S, y_gs=S)
        else:
            tiles, rows, G = shape[1]()
            cols = Cols.table(tiles)
            y_rows = rows
        src = c + torch.randn(rows, K, generator=g)
        kw["ld_src"] = K
        if gen == GEN.NORM:
            kw["gsc"], kw["gsh"] = torch.ones(G, K).cuda(), torch.zeros(G, K).cuda()
    relu = int(name.endswith("_relu"))
    Y, P, _ = run_gen(lib, gen, wt, b, Wp, wps, src.cuda(), cols, y_rows, relu=relu, **kw)
    if relu:
        assert bool((Y[cols.y_row.cuda()] == 0).any()), "no ReLU zero among the outputs"
    rv, rm, cond = check_partials(P, Y, cols, G, f"gen {name} R={R} {source}")
    assert cond >= 0.5 * R
    assert rv <= 1.0 and rm <= 1.0, (rv, rm)


# ------------------------------------------------------------------------------------------------ GPU: gemm_tma
# (M, K, addend): PointNet layer 2 (Y and partials) and a 512-wide contraction with a per-detection addend, whose
# partial chunks take the slow epilogue path.
TMA_KINDS = {"l2": (64, 64, False), "add512": (512, 64, True)}
TMA_CASES = [(lay, kind, R, src) for lay in LAYOUTS for kind in TMA_KINDS for R in RS for src in SOURCES]


@gpu
@pytest.mark.parametrize("layout,kind,R,source", TMA_CASES, ids=[f"{c[0]}-{c[1]}-R{c[2]}-{c[3]}" for c in TMA_CASES])
def test_tma_stats_conditioned(layout, kind, R, source):
    """gemm_tma matrix mode through mmmot_debug_pn_contraction on the ragged layouts of kernel_kit.LAYOUTS (group =
    pair)."""
    pairs, L, counts = LAYOUTS[layout]
    M, K, want_add = TMA_KINDS[kind]
    lib = _lib.load()
    ndet = pairs * L
    split = [0] + np.cumsum(counts).tolist()
    Pn = split[-1]
    tiles_h = pn_host_tables(split, pairs, L)[0]
    nt = len(tiles_h)
    g = torch.Generator().manual_seed(case_seed(layout, kind, R, source))
    wt, b, c = conditioned_weights(g, K, M, R, source)
    Wp, wps = pack_tc(wt)
    X = torch.stack(fp16_split(c + torch.randn(Pn, K, generator=g))).contiguous().cuda()
    add = torch.randn(ndet, M, generator=g) * 0.25 if want_add else None
    cap = nt + 3
    tiles = torch.zeros((cap, 4), dtype=torch.int32, device="cuda")
    ctab = torch.zeros((2 * cap, 4), dtype=torch.int32, device="cuda")
    cnt = torch.zeros((pairs + 2,), dtype=torch.int32, device="cuda")
    gstart = torch.zeros((pairs + 3,), dtype=torch.int32, device="cuda")
    segd = torch.zeros((Pn + 64,), dtype=torch.int32, device="cuda")
    Y = torch.full((Pn, M), float("nan"), device="cuda")
    part = torch.full((2 * nt, M, 2), float("nan"), dtype=torch.float64, device="cuda")
    keep = (Wp.cuda(), b.cuda(), None if add is None else add.cuda())
    d_split = torch.tensor(split, dtype=torch.int32, device="cuda")
    h_split = torch.tensor(split, dtype=torch.int32)
    n_tiles = ctypes.c_long(-1)
    rc = lib.mmmot_debug_pn_contraction(vp(d_split), vp(h_split), pairs, L, cap, vp(tiles), vp(cnt),
                                        vp(gstart), vp(segd), vp(ctab), ctypes.byref(n_tiles), vp(keep[0]), wps,
                                        vp(keep[1]), M, K, vp(X), vp(Y), vp(part), vp(keep[2]), M, None, None, None, None)
    torch.cuda.synchronize()
    assert rc == 0 and n_tiles.value == nt, (rc, n_tiles.value)
    cols = Cols.table(tiles_h)
    rv, rm, cond = check_partials(part, Y, cols, pairs, f"tma {layout} {kind} R={R} {source}")
    assert cond >= 0.5 * R
    assert rv <= 1.0 and rm <= 1.0, (rv, rm)


# ------------------------------------------------------------------------------------------------ GPU: gemm_simt
TN = 128   # the FP32 engine's column tile
# (name, mode, M, K, layout): uniform (S, groups) or a table of per-group column counts (ragged, <= 128 per tile)
SIMT_LAYOUTS = [("direct_S16", 0, 512, 512, ("uniform", 16, 4)), ("direct_S300", 0, 256, 512, ("uniform", 300, 3)),
                ("norm_S48", 1, 512, 512, ("uniform", 48, 4)), ("norm_S300", 1, 128, 512, ("uniform", 300, 2)),
                ("direct_tab", 0, 512, 64, ("table", [37, 100, 1, 200, 129])),
                ("norm_tab", 1, 64, 64, ("table", [5, 300, 64, 128, 33])),
                ("direct_S48_relu", 0, 512, 512, ("uniform", 48, 4)), ("norm_tab_relu", 1, 64, 64, ("table", [5, 300, 1, 33]))]
SIMT_CASES = [(lay, R, src) for lay in SIMT_LAYOUTS for R in RS for src in SOURCES]


@gpu
@pytest.mark.parametrize("lay,R,source", SIMT_CASES, ids=[f"{c[0][0]}-R{c[1]}-{c[2]}" for c in SIMT_CASES])
def test_simt_stats_conditioned(lay, R, source):
    """gemm_simt through mmmot_debug_simt_op (XM_DIRECT, XM_NORM_RELU with sc = 1, sh = 0), uniform and table tiling; the
    partials are one per (tile, channel)."""
    name, mode, M, K, shape = lay
    relu = int(name.endswith("_relu"))
    lib = _lib.load()
    g = torch.Generator().manual_seed(case_seed(name, R, source))
    wt, b, c = conditioned_weights(g, K, M, R, source)
    if shape[0] == "uniform":
        _, S, G = shape
        lens = [S] * G
    else:
        lens = shape[1]
        G = len(lens)
    start = np.concatenate([[0], np.cumsum(lens)])
    P = int(start[-1])
    tiles = [(gi, int(start[gi]) + c0, min(TN, lens[gi] - c0)) for gi in range(G) for c0 in range(0, lens[gi], TN)]
    x = (c[:, None] + torch.randn(K, P, generator=g)).cuda()            # [K][P] channel-major, groups back to back
    Y = torch.full((M, P), float("nan"), device="cuda")
    part = torch.full((len(tiles), M, 2), float("nan"), dtype=torch.float64, device="cuda")
    wd, bd = wt.cuda(), b.cuda()
    sc, sh = torch.ones(G, K, device="cuda"), torch.zeros(G, K, device="cuda")
    if shape[0] == "uniform":
        # uniform tiling reads X + g*x_gs + k*x_ks + col: the same [K][P] buffer with x_gs = S, x_ks = P
        rc = lib.mmmot_debug_simt_op(mode, M, K, vp(wd), vp(bd), relu, vp(x), S, P, vp(sc), vp(sh), 0, 0, 0, 0, 0, 0, S, G,
                                     None, 0, None, None, 0, vp(Y), S, P, vp(part), None)
    else:
        tt = torch.tensor([[gi, c0, ln, 0] for gi, c0, ln in tiles], dtype=torch.int32, device="cuda")
        rc = lib.mmmot_debug_simt_op(mode, M, K, vp(wd), vp(bd), relu, vp(x), 0, P, vp(sc), vp(sh), 0, 0, 0, 0, 0, 0, 0, 0,
                                     vp(tt), len(tiles), None, None, 0, vp(Y), 0, P, vp(part), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    assert bool(torch.isfinite(Y).all())
    if relu:
        assert bool((Y == 0).any()), "no ReLU zero among the outputs"
    grp = torch.tensor(np.repeat(np.arange(G), lens), device="cuda")
    tile_group = torch.tensor([t[0] for t in tiles], device="cuda")
    S1, S2 = reduce_parts(part, tile_group, G)
    rv, rm, cond = stats_ratios(S1, S2, Y.T.double(), grp, G)
    report(f"simt {name} R={R} {source}", var_err_over_bound=rv, mean_err_over_bound=rm, max_mean_over_std=cond)
    assert cond >= 0.5 * R
    assert rv <= 1.0 and rm <= 1.0, (rv, rm)


# ------------------------------------------------------------------------------------------------ GPU: affinity stage
# N.M on both sides of 64 (the tensor cores take the pairwise layer from N.M >= 64)
AFF_CASES = [(op, sm, n, m) for op in ("multiply", "minus_abs", "minus") for sm in ("none", "dual_add")
             for n, m in ((6, 8), (12, 16))]


@gpu
@pytest.mark.parametrize("op,sm,n,m", AFF_CASES, ids=[f"{c[0]}-{c[1]}-{c[2]}x{c[3]}" for c in AFF_CASES])
def test_affinity_lookalike_vs_fp64(op, sm, n, m):
    """associate_batch on look-alike detections (every feature column = one shared column + 2 % noise, as near-identical
    cars give) against torch_ref.associate in float64: the effect a user sees of the statistics above."""
    from helpers import TOL, check_close
    from oracle import torch_ref
    net, sd = eval_net("C", 23, affinity_op=op, softmax_mode=sm, neg_threshold=0.2)
    g = torch.Generator().manual_seed(case_seed(op, sm, n, m))
    base = torch.relu(torch.randn(1, 3, 512, 1, generator=g)) + 0.5
    feats = base * (1 + 0.02 * torch.randn(1, 3, 512, n + m, generator=g))
    link, new, end = net.associate_batch(feats.cuda(), n, m)
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    f64 = feats.double()
    rl, rn, re = torch_ref.associate(sd64, f64[0, :, :, :n], f64[0, :, :, n:], op, sm)
    # Every output: max-norm error < 1e-4 and no element beyond 4x the element-wise bound.  Every output but the raw
    # link logits of softmax "none" also has no element past that bound; for those logits the fraction past it is
    # reported only: near-zero logits of look-alike pairs miss it in any fp32 implementation (the fp32 oracle differs
    # from the fp64 one by 2.7e-5 max-norm on these inputs).
    rep = []
    check_close(link[0], rl.squeeze(1), TOL, "link", rep, max_outside=1.0 if sm == "none" else 0.0)
    check_close(new[0], rn, TOL, "new", rep)
    check_close(end[0], re, TOL, "end", rep)
    report(f"affinity {op} {sm} {n}x{m}", **{f"{w}_{k}": v for w, e, fo, wr in rep
                                             for k, v in (("err", e), ("outside", fo), ("worst", wr))})


# ------------------------------------------------------------------------------------------------ GPU: fusion, w_det
# The stage tests below make their contractions exact so that the statistics are all that is left to check: weights
# and biases are multiples of 2^-6 of magnitude <= 1/4, inputs integers of magnitude < 1024.  Every product and partial
# sum is then a multiple of 2^-6 below 2^18, exact in fp32 and in the FP16 hi/lo tensor-core path, in any order.
def _dyadic(t):
    return (t * 64).round().clamp(-16, 16) / 64


def _int_features(g, shape, R):
    """Integer features c_k + e, e uniform on {-2..2} (std sqrt 2), c_k ~ R sqrt2 (1 + U/2) shared by every detection:
    a channel w.x then has |mean| / std ~ 1.25 R |N(0, 1)| (up to ~4R over 512 channels)."""
    K = shape[-2]
    gam = R * math.sqrt(2)
    c = (gam * (1 + 0.5 * torch.rand(K, 1, generator=g))).round()
    return c + torch.randint(-2, 3, shape, generator=g).float()


def _exact_net(arch, seed):
    """A network whose fusion and w_det layer-1 weights are dyadic (see above); fusion C's gates have zero weights (a
    per-channel constant sigmoid(bias)), so that saturating gates cannot make 0/0."""
    def dyadic(sd):
        g = torch.Generator().manual_seed(seed)
        for k, v in sd.items():
            if (k.startswith("fusion_module.") and ".0." in k) or k.startswith("w_det.0."):
                sd[k] = _dyadic(torch.randn(v.shape, generator=g) * 3 / 64)
                if ".gate_" in k and k.endswith("weight"):
                    sd[k] = torch.zeros_like(v)

    net, sd = eval_net(arch, seed, edit=dyadic)
    return net, {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}


def _gn_bound(y, gamma, beta):
    """GroupNorm(C, C) over y [C][L] (fp64, exact): -> (z, per-element bound on the kernel's error in z).  The bound
    carries the statistics bound above through GroupNorm, |gamma| rstd (dmean + |y - ybar| dvar / (2 (var + eps))), and
    the fp32 roundings of sc, sh and y sc + sh, 8 u (|y sc| + |sh| + |z|): GroupNorm's own conditioning."""
    m = y.mean(1, keepdim=True)
    dev = y - m
    v = (dev * dev).mean(1, keepdim=True)
    tv = KAPPA * U * (m.abs() * dev.abs().mean(1, keepdim=True) + v)
    tm = KAPPA1 * U * y.abs().mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(v + 1e-5)
    sc = gamma[:, None] * rstd
    sh = beta[:, None] - m * sc
    z = y * sc + sh
    T = gamma.abs()[:, None] * rstd * (tm + dev.abs() * tv / (2 * (v + 1e-5))) + 8 * U * ((y * sc).abs() + sh.abs() + z.abs())
    return z, T, float((m.abs() * torch.sqrt(1 / v.clamp_min(1e-300))).max())


FUSION_CASES = [(arch, L, pairs, eng, R) for arch in "ABC" for L in (16, 48, 64, 128, 300) for pairs in (1, 3)
                for eng in ("auto", "fp32", "tc") for R in (20, 300)]


@functools.lru_cache(maxsize=None)
def _fusion_net(arch):
    return _exact_net(arch, 29)


@gpu
@pytest.mark.parametrize("arch,L,pairs,eng,R", FUSION_CASES, ids=[f"{a}-L{b}-p{c}-{d}-R{e}" for a, b, c, d, e in FUSION_CASES])
def test_fusion_stage_conditioned(arch, L, pairs, eng, R):
    """mmmot_fusion_det_fwd on crafted stacks 0 and 1 (look-alike detections: a shared component R std large) under
    the automatic engine choice (tensor cores from L = 64) and each engine forced; stack 2 element by element against
    torch_ref.fusion in float64, to the bound of _gn_bound summed over the GroupNorm branches (plus 8 u of their
    magnitudes for the gate and sum arithmetic)."""
    from oracle import torch_ref
    lib = _lib.load()
    net, sd64 = _fusion_net(arch)
    wts = net.prepared()
    g = torch.Generator().manual_seed(case_seed(arch, L, pairs, eng, R))
    feats = torch.full((pairs, 3, 512, L), float("nan"))
    feats[:, :2] = _int_features(g, (pairs, 2, 512, L), R)
    fd = feats.cuda()
    det = torch.empty(pairs, 3, L, device="cuda")
    ws = torch.empty(int(lib.mmmot_fusion_det_workspace(pairs, L)), dtype=torch.uint8, device="cuda")
    with lib_state(lib, engine=eng):
        rc = lib.mmmot_fusion_det_fwd(wts.ptr, _lib.FUSION[arch], 0, 0.0, pairs, L, vp(fd), vp(det), vp(ws), ws.numel(), None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    got = fd[:, 2].double().cpu()
    f64 = feats[:, :2].double()
    f = "fusion_module"
    lin = lambda name, x: torch.nn.functional.conv1d(x[None], sd64[f"{f}.{name}.0.weight"], sd64[f"{f}.{name}.0.bias"])[0]
    worst, cond = 0.0, 0.0
    for p in range(pairs):
        ref = torch_ref.fusion(sd64, arch, f64[p].reshape(1, 1024, L))[2]
        branches = [("input_w", f64[p].reshape(1024, L))] if arch == "A" else [("input_p", f64[p, 0]), ("input_i", f64[p, 1])]
        T = torch.zeros(512, L, dtype=torch.float64)
        for name, x in branches:
            z, Tb, cb = _gn_bound(lin(name, x), sd64[f"{f}.{name}.1.weight"], sd64[f"{f}.{name}.1.bias"])
            T += Tb + 8 * U * z.abs()
            cond = max(cond, cb)
        worst = max(worst, float(((got[p] - ref).abs() / T).max()))
    report(f"fusion {arch} L={L} pairs={pairs} {eng} R={R}", err_over_bound=worst, max_mean_over_std=cond)
    assert cond >= 0.5 * R
    assert worst <= 1.0, worst


W_DET_CASES = [(L, R) for L in (16, 48, 300) for R in RS]


@gpu
@pytest.mark.parametrize("L,R", W_DET_CASES, ids=[f"L{L}-R{R}" for L, R in W_DET_CASES])
def test_w_det_train_batch_stats(L, R):
    """mmmot_w_det_train_fwd: layer 1's exported BatchNorm batch mean and biased variance (one domain over the 3L
    columns of the three stacks, gemm_simt partials -> stats_reduce -> bn_export_kernel) against fp64 over the exact
    layer-1 outputs, to the statistics bound above plus the float conversion (u of the value).  Layer 2, whose input
    already carries layer 1's normalisation error, is reported: its worst relative variance error."""
    lib = _lib.load()
    net, sd64 = _fusion_net("C")
    wts = net.prepared()
    g = torch.Generator().manual_seed(case_seed("w_det", L, R))
    feats = _int_features(g, (3, 512, L), R)
    det = torch.empty(3, L, device="cuda")
    bn = torch.full((2, 2, 512), float("nan"), device="cuda")
    ws = torch.empty(int(lib.mmmot_w_det_train_workspace(L)), dtype=torch.uint8, device="cuda")
    fd = feats.cuda()
    rc = lib.mmmot_w_det_train_fwd(wts.ptr, L, vp(fd), vp(det), vp(bn), vp(ws), ws.numel(), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    bn = bn.double().cpu()
    F = torch.nn.functional
    y = F.conv1d(feats.double(), sd64["w_det.0.weight"], sd64["w_det.0.bias"]).transpose(0, 1).reshape(512, 3 * L)
    m = y.mean(1)
    dev = y - m[:, None]
    v = (dev * dev).mean(1)
    tv = KAPPA * U * (m.abs() * dev.abs().mean(1) + v) + U * v
    tm = KAPPA1 * U * y.abs().mean(1) + U * m.abs()
    rm = float(((bn[0, 0] - m).abs() / tm).max())
    rv = float(((bn[0, 1] - v).abs() / tv).max())
    cond = float((m.abs() / v.sqrt()).max())
    h = F.relu((y - m[:, None]) / torch.sqrt(v[:, None] + 1e-5) * sd64["w_det.1.weight"][:, None] + sd64["w_det.1.bias"][:, None])
    y2 = F.conv1d(h.reshape(512, 3, L).transpose(0, 1), sd64["w_det.3.weight"], sd64["w_det.3.bias"]).transpose(0, 1)
    v2 = y2.reshape(256, -1).var(1, unbiased=False)
    l2 = float(((bn[1, 1, :256] - v2).abs() / v2).max())
    report(f"w_det train L={L} R={R}", var_err_over_bound=rv, mean_err_over_bound=rm, max_mean_over_std=cond,
            layer2_var_rel_err=l2)
    assert cond >= 0.5 * R
    assert rv <= 1.0 and rm <= 1.0, (rv, rm)
