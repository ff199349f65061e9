"""The kernels between the contractions -- affinity tail, detection score, SkipPool heads -- element by element against fp64.

Each GPU case runs the real stage (mmmot_affinity_fwd, mmmot_fusion_det_fwd) with its own workspace, filled with NaN
first, then reads the intermediates the stage left there at the offsets mmmot_debug_stage_layout reports (the same carve
the stage runs) and checks every kernel after the last contraction against fp64 computed from that kernel's own stored
inputs, so no contraction error enters a bound.  The SkipPool heads run through mmmot_debug_skip_heads on pooled vectors
the test chooses.  Outputs start as NaN with a NaN guard band past their end: every element a kernel owns must be
written, every other one must come back NaN.  Every case prints err / bound per kernel (_report).

With u = 2^-24, T = 2^-126 and r = relu(fmaf(y, sc, sh)) formed from the stored y, sc, sh exactly as the kernels form
it (one fp64 multiply-add rounded to fp32):

New/end means (rowcol_mean_kernel, FP32 path, V[c][ldv]; newend_mean_cl_kernel, tensor-core path, V[col][512]): new
    column j = mean_i r, end column i = mean_j r over cnt = n or m terms of the stored y01[..., 512:] with sc0 / sh0.
    avg: |V - V_ref| <= (cnt + 2) u mean|r| + u |V_ref|   (cnt - 1 fp32 additions in any order, the division)
    max: |V - V_ref| <= u |V_ref|                         (the maximum of the same fp32 values: in fact exact)
Final new/end layer (ne_final_kernel / ne_final_cl_kernel) from the stored h2 with nsc2 / nsh2 of the column's group
    2g + (end): a = b3 + sum_c w3 r over 128 terms in any order,
    |a - a_ref| <= Ta = 1.01 * 130 u (sum |w3 r| + |b3|),
    then s = 1 / (1 + expf(-a)): expf is within 2 ulp (4u relative), the add and the division round once each, and
    d s / d a = s (1 - s), so  |s - s_ref| <= s (1 - s) Ta + 6 u s + 4T,
    scattered into new[g][j] / end[g][i] of the column's own pair and stack.
Link logits (link_logit_kernel / link_logit_cl_kernel) from the stored y3 with sc3 / sh3: z = b4 + sum_c w4 r over 128
    terms, |z - z_ref| <= 1.01 * 130 u (sum |w4 r| + |b4|).
Softmax (softmax_stats_kernel, softmax_apply_kernel) from the stored z (link itself for mode none): rmax / cmax are the
    maxima of fp32 values and must match bit for bit.  Term t of a row sum is expf(fl(z_t - max)): the subtraction
    rounds once (|z_t - max| u in the exponent) and expf adds 2 ulp, so e_t = |z_t - max| u + 4u relative, T absolute
    where it underflows; the cnt terms are added in fp32 (at most cnt - 1 roundings in any order):
    |rsum - rsum_ref| <= sum_t (e_t exp_t + T) + cnt u rsum_ref,  R_row = that bound / rsum_ref.
    p_row = expf(z - rmax) / rsum then errs by e_p = |z - rmax| u + 4u + R_row + u relative, p_col likewise, and link =
    single p_row: e_row;  dual p_row p_col: e_row + e_col + u;  dual_add (p_row + p_col) / 2: max + u;  dual_max: max,
    times the link value, plus 4T where results underflow.  A softmax over one element (n or m = 1) is exactly 1.
Detection score (det_score_kernel, FP32 path, h2 [g][256][L]; det_score_rows_kernel, tensor-core path, h2
    [(pair L + l) 3 + stack][256]) from the stored post-ReLU h2: a = b3 + sum_c w3 h2 over 256 terms,
    Ta = 1.01 * 258 u (sum |w3 h2| + |b3|); with MMMOT_SCORE_SIGMOID s carries the sigmoid bound above (Ts), else s = a.
    With MMMOT_SCORE_THRESHOLD the output is s - [s < thr]: where |s_ref - thr| > Ts the step must match the
    reference (bound Ts + u |out|, the rounding of s - 1); inside that band either side is accepted.
    Tensor-core path: stacks 0 and 1 of F3 are the transpose of feats bit for bit, stack 2 of F3 equals the stack 2
    written to feats; the FP32 path leaves F3 untouched.
SkipPool heads (skip_head_kernel: GN(1,C) -> 1x1 conv C->mid -> GN(1,mid) -> ReLU -> 1x1 conv mid->128 -> GN(1,128) ->
    ReLU, one CTA per image) against torch_ref.skip_pool's fc chain in fp64.  Contractions: acc = bias, then fma over
    the K inputs in order, one rounding per step; with the fp64 prefix sums s_k (bias included) and the input's own
    bound Tx,  Ty = |W| Tx + 1.01 u sum_k |s_k|.
    GroupNorm over the C channels of one image (gn_propagate), ns = ceil(C/128) + 8 fp32 roundings per block sum (the
    strided per-thread terms, the 5-level shuffle tree, the 4 warp totals): the kernel's mean m^ and, from the
    centred d = fl(y - m^), its variance
        |dmean| <= tm = mean(Ty) + ns u mean(|y| + Ty) + u |mean|,
        |dvar|  <= tv = 2 mean(|y - mean| Ty) + mean((Ty + tm)^2) + (ns + 4) u var
    (sum_c (y_c - mean) = 0 cancels the mean's error in the cross term); rsqrtf is within 2 ulp, so rstd errs by
    rr = (tv + u (var + eps)) / (2 (var + eps)) + 4u relative, and z = d rstd gamma + beta by
        Tz = |gamma| rstd (Ty + tm + |y - mean| (u + rr)) + 3u (|gamma d rstd| + |z|).
    A constant vector (zero variance) makes GN return beta up to the rounding of m^ times rstd = eps^-1/2.

CPU tests: the layout query (no device), a guard that the case lists cover what they must, and a sensitivity check:
each bound accepts a plain fp32 evaluation and rejects a planted defect -- a mean divided by m instead of n, a row sum
missing one column, a logit without its bias, each by more than 10x, and a head's last GroupNorm variance taken over
C - 1 = 127 channels by more than 2x.  The head's margin is the small one: its worst-case bound carries |W| through two
contractions and three GroupNorms and sits about 10^3 above a plain fp32 evaluation, while the planted variance moves
the output by 1/256 of its spread.  (The same defect in the first or second GroupNorm is largely normalised away by the
GroupNorm after it; only beta and the conv bias carry it to the output.)
"""
import ctypes
import functools
import math

import pytest
import torch

from kernel_kit import (AF_BUFS, ENGINE, EPS, TINY, U, Workspace, assert_written, case_seed, eval_net, lib_state,
                        nan_output, nan_workspace, norm_operand, report, stage_layout, vp, worst_ratio)
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_state_dict

gpu = pytest.mark.gpu
FLOOR = 4 * TINY
MODES = ("none", "single", "dual", "dual_add", "dual_max")
OPS = ("multiply", "minus_abs", "minus")
SKIP_C = (128, 256, 512, 512)
PEAKY = 25.0     # scale of w_link.conv1.9 (weight and bias) that spreads the synthetic link logits over about +-100
# the benchmark configurations' per-pair head shapes: N detections per frame (L = 2N); cfg5 is the N sweep's top
CFG_N = {"cfg2": 32, "cfg3": 64, "cfg4": 128, "cfg5": 256}


# ------------------------------------------------------------------------------------------------ layout
def af_sizes(pairs, n, m):
    """Bytes of each affinity intermediate (the shapes and types the header documents; part, npart and tiles sized for
    the larger of the two paths' tilings)."""
    G, NM, ldv = 3 * pairs, n * m, 3 * pairs * (n + m)
    cd = lambda a, b: -(-a // b)
    ntile = G * (cd(n, 128) + cd(m, 128))
    f32 = dict(y01=G * 1024 * NM, y3=G * 128 * NM, z=G * NM, fcl=G * (n + m) * 512, sc0=G * 512, sh0=G * 512,
               sc3=G * 128, sh3=G * 128, v=512 * ldv, h2=128 * ldv, nsc2=2 * G * 128, nsh2=2 * G * 128,
               rmax=G * n, rsum=G * n, cmax=G * m, csum=G * m, y2=G * 512 * NM, sc1=G * 512, sh1=G * 512, sc2=G * 512,
               sh2=G * 512, h1=512 * ldv, nsc1=2 * G * 512, nsh1=2 * G * 512)
    size = {k: 4 * v for k, v in f32.items()}
    size.update(stats=8 * G * 1024 * 2, nstats=8 * 2 * G * 512 * 2, part=16 * G * 2 * cd(NM, 256) * 1024,
                npart=16 * 2 * ntile * 512, tiles=16 * ntile, cnt=4 * 2 * G, gstart=4 * (2 * G + 1))
    return size


def fd_sizes(pairs, L):
    """Bytes of each fusion / detection-score intermediate (the header's shapes; part holds two partials per 128
    columns, room for either path's tiling)."""
    n, pc = pairs * 512 * L, pairs * 512
    return dict(f3=12 * n, h2=6 * n, yp=4 * n, yi=4 * n, gp=4 * n, gi=4 * n, scp=4 * pc, shp=4 * pc, sci=4 * pc, shi=4 * pc,
                h1=12 * n, stats=16 * pc, part=16 * pc * 2 * -(-L // 128))


# ------------------------------------------------------------------------------------------------ fp64 bounds
def mean_bound(r, cnt, mx):
    """New/end reduction of the fp32 values r (fp64, the reduced axis last) -> (V_ref, bound)."""
    if mx:
        v = r.amax(-1)
        return v, U * v
    v = r.sum(-1) / cnt
    return v, (cnt + 2) * U * r.abs().mean(-1) + U * v.abs()


def logit_bound(x, w, b, nterm):
    """b + x @ w over the last axis of x (fp64) -> (a_ref, Ta)."""
    a = x @ w + b
    return a, 1.01 * (nterm + 2) * U * (x.abs() @ w.abs() + abs(b))


def sigmoid_bound(a, Ta):
    s = torch.sigmoid(a)
    return s, s * (1 - s) * Ta + 6 * U * s + FLOOR


def softmax_sums(z, dim):
    """Row (dim=-1) or column (dim=-2) statistics of z (fp64 holding fp32) -> (max, sum, bound of sum, per-term relative
    error e_t of expf(fl(z - max)) without the sum's)."""
    mx = z.amax(dim, keepdim=True)
    t = torch.exp(z - mx)
    et = (z - mx).abs() * U + 4 * U
    cnt = z.shape[dim]
    s = t.sum(dim, keepdim=True)
    ts = (et * t).sum(dim, keepdim=True) + cnt * TINY + cnt * U * s
    return mx, s, ts, et


def softmax_link(z, mode):
    """link of softmax mode `mode` from z [G][n][m] (fp64 holding fp32) -> (link_ref, bound, stats) with stats the
    (max, sum, bound) of rows and columns."""
    rmx, rs, trs, ert = softmax_sums(z, -1)
    cmx, cs, tcs, ect = softmax_sums(z, -2)
    pr, pc = torch.exp(z - rmx) / rs, torch.exp(z - cmx) / cs
    er = ert + trs / rs + U
    ec = ect + tcs / cs + U
    if mode == "single":
        out, rel = pr, er
    elif mode == "dual":
        out, rel = pr * pc, er + ec + U
    elif mode == "dual_add":
        out, rel = (pr + pc) / 2, torch.maximum(er, ec) + U
    else:
        out, rel = torch.maximum(pr, pc), torch.maximum(er, ec)
    return out, out * rel + FLOOR, ((rmx, rs, trs), (cmx, cs, tcs))


def chain_bound(wt, x, Tx, b):
    """acc = b, then acc = fma(w_k, x_k, acc) for k in order: x [n][K], wt [K][M], b [M] (fp64) -> (y [n][M], Ty)."""
    prod = x[:, :, None] * wt[None]
    pre = prod.cumsum(1) + b
    y = pre[:, -1]
    return y, Tx @ wt.abs() + 1.01 * U * pre.abs().sum(1)


def gn_propagate(y, T, gamma, beta, over=None):
    """GroupNorm(1, C) of each row of y [n][C] (fp64) whose kernel values err by at most T, as skip_head_kernel forms it
    (module docstring) -> (z, Tz).  over: divisor of the variance (C by definition; the sensitivity check plants C - 1)."""
    C = y.shape[1]
    ns = math.ceil(C / 128) + 8
    m = y.mean(1, keepdim=True)
    dev = y - m
    v = (dev * dev).sum(1, keepdim=True) / (C if over is None else over)
    tm = T.mean(1, keepdim=True) + ns * U * (y.abs() + T).mean(1, keepdim=True) + U * m.abs()
    tv = 2 * (dev.abs() * T).mean(1, keepdim=True) + ((T + tm) ** 2).mean(1, keepdim=True) + (ns + 4) * U * v
    rstd = 1 / torch.sqrt(v + EPS)
    rr = (tv + U * (v + EPS)) / (2 * (v + EPS)) + 4 * U
    zd = dev * rstd * gamma
    z = zd + beta
    return z, gamma.abs() * rstd * (T + tm + dev.abs() * (U + rr)) + 3 * U * (zd.abs() + z.abs())


def skip_head_ref(sd, s, x, last_var_over=None):
    """SkipPool head s on pooled x [n][C] (fp64) -> (out [n][128], bound).  last_var_over: divisor of the last
    GroupNorm's variance (the sensitivity check plants 127)."""
    p = f"appearance.global_pool.{s}.fc"
    f = lambda k: sd[f"{p}.{k}"].double().to(x.device)
    z, T = gn_propagate(x, torch.zeros_like(x), f("0.weight"), f("0.bias"))
    w1 = f("1.weight").reshape(f("1.weight").shape[0], -1)
    y, T = chain_bound(w1.T.contiguous(), z, T, f("1.bias"))
    z, T = gn_propagate(y, T, f("2.weight"), f("2.bias"))
    h = z.clamp_min(0)
    w2 = f("4.weight").reshape(128, -1)
    y, T = chain_bound(w2.T.contiguous(), h, T, f("4.bias"))
    z, T = gn_propagate(y, T, f("5.weight"), f("5.bias"), over=last_var_over)
    return z.clamp_min(0), T


# ------------------------------------------------------------------------------------------------ cases
# affinity: (n, m, pairs, engine, op, softmax mode, end mode, peaky)
AF_CASES = [
    (1, 1, 2, "fp32", "multiply", "single", "avg", False), (1, 1, 2, "tc", "minus_abs", "dual", "max", False),
    (1, 64, 1, "fp32", "minus", "dual_max", "avg", False), (1, 64, 1, "tc", "multiply", "none", "max", False),
    (64, 1, 1, "fp32", "minus_abs", "none", "max", False), (64, 1, 1, "tc", "minus", "dual_add", "avg", False),
    (7, 9, 3, "fp32", "multiply", "dual", "avg", False), (7, 9, 3, "tc", "minus_abs", "single", "max", False),
    (7, 9, 3, "auto", "minus", "dual_add", "avg", False),
    (8, 8, 2, "fp32", "minus", "dual_add", "max", False), (8, 8, 2, "tc", "multiply", "dual_max", "avg", False),
    (8, 8, 2, "auto", "minus_abs", "dual", "max", False),
    (37, 29, 3, "fp32", "minus_abs", "dual_max", "max", False), (37, 29, 3, "tc", "minus", "none", "avg", False),
    (257, 40, 1, "fp32", "multiply", "dual_add", "avg", False), (257, 40, 1, "tc", "minus_abs", "dual", "max", False),
    (40, 300, 1, "fp32", "minus", "single", "max", False), (40, 300, 1, "tc", "multiply", "dual_max", "avg", False),
    (32, 32, 1, "tc", "minus_abs", "none", "avg", False), (32, 32, 1, "fp32", "minus", "dual", "max", False),
    (64, 64, 1, "tc", "multiply", "single", "max", False), (64, 64, 1, "fp32", "minus_abs", "dual_add", "avg", False),
    (128, 128, 1, "tc", "minus_abs", "dual_add", "avg", False), (128, 128, 1, "tc", "minus", "dual_max", "max", False),
    (256, 256, 1, "tc", "minus_abs", "dual_add", "max", False), (256, 256, 1, "fp32", "multiply", "none", "avg", False),
    # peaky link logits (about +-100): underflowing softmax tails and dual products
    (37, 29, 3, "tc", "multiply", "dual", "max", True), (37, 29, 3, "fp32", "minus", "dual", "avg", True),
    (1, 64, 1, "tc", "minus_abs", "single", "avg", True), (64, 1, 1, "fp32", "multiply", "dual_add", "max", True),
    (128, 128, 1, "tc", "minus", "dual_max", "avg", True),
]
DET_LS = (1, 2, 31, 63, 64, 65, 128, 256, 300)
# detection score: (L, pairs, engine, score flags, fusion); the flags and fusion architectures rotate over the cases
DET_CASES = [(L, p, e, k % 4, "ABC"[(k // 3) % 3])
             for k, (L, p, e) in enumerate((L, p, e) for L in DET_LS for p in (1, 3) for e in ("fp32", "tc", "auto"))]
# SkipPool heads: (pooled kind, offset R, n_img, L)
SKIP_CASES = [("mixed", 0, 1, 1), ("mixed", 0, 5, 5), ("mixed", 0, 64, 16), ("offset", 1, 5, 1), ("offset", 30, 5, 5),
              ("offset", 300, 64, 64), ("offset", 300, 1, 1), ("const", 0, 5, 5), ("const", 0, 64, 32),
              ("mixed", 0, 128, 128), ("offset", 30, 256, 256)]


def af_path(n, m, engine):
    """The path a case must take: 'tc' or 'fp32' (auto: tensor cores from N.M = 64)."""
    return engine if engine != "auto" else ("tc" if n * m >= 64 else "fp32")


def det_path(L, engine):
    return engine if engine != "auto" else ("tc" if L >= 64 else "fp32")


def _af_id(c):
    return f"{c[0]}x{c[1]}x{c[2]}-{c[3]}-{c[4]}-{c[5]}-{c[6]}" + ("-peaky" if c[7] else "")


# ------------------------------------------------------------------------------------------------ CPU
def test_stage_layout_without_device():
    """mmmot_debug_stage_layout works on the host: every buffer lies inside the stage's workspace, behind the status
    block, and no two overlap; the path it reports follows the engine setting; bad arguments are refused."""
    lib = _lib.load()
    for engine in ("auto", "fp32", "tc"):
        with lib_state(lib, engine=engine):
            for pairs, n, m in ((1, 1, 1), (2, 7, 9), (2, 8, 8), (3, 37, 29), (1, 257, 40), (1, 256, 256)):
                lay, tc = stage_layout(lib, 0, pairs, n, m)
                assert tc == (af_path(n, m, engine) == "tc"), (engine, n, m)
                _disjoint_inside(lay, af_sizes(pairs, n, m), int(lib.mmmot_affinity_workspace(pairs, n, m)))
            for pairs, L in ((1, 1), (3, 63), (3, 64), (1, 300)):
                lay, tc = stage_layout(lib, 1, pairs, L)
                assert tc == (det_path(L, engine) == "tc"), (engine, L)
                _disjoint_inside(lay, fd_sizes(pairs, L), int(lib.mmmot_fusion_det_workspace(pairs, L)))
    off = (ctypes.c_size_t * 32)()
    for args in ((3, 1, 4, 4), (0, 0, 4, 4), (0, 1, 0, 4), (0, 1, 4, 0), (1, 1, 0, 0), (-1, 1, 4, 4)):
        assert lib.mmmot_debug_stage_layout(*args, off, None) == -1, args
    assert lib.mmmot_debug_stage_layout(0, 1, 4, 4, None, None) == -1
    # the SkipPool hook checks its shape before any CUDA call: images must fill whole pairs
    w = ctypes.pointer(_lib.Weights())
    feats = ctypes.c_void_p(256)
    for n_img, L in ((5, 2), (0, 1), (4, 0)):
        assert lib.mmmot_debug_skip_heads(w, None, None, None, None, n_img, L, feats, None) == -1, (n_img, L)


def _disjoint_inside(lay, sizes, ws_bytes):
    spans = sorted((lay[k], lay[k] + sizes[k], k) for k in lay)
    assert spans[0][0] >= 256, spans[0]
    assert spans[-1][1] <= ws_bytes, (spans[-1], ws_bytes)
    for (a0, a1, ka), (b0, b1, kb) in zip(spans, spans[1:]):
        assert a1 <= b0, (ka, kb)
    assert all(o % 16 == 0 for o in lay.values())


def test_case_coverage():
    """The GPU case lists cover: every softmax mode on both paths, on a non-square multi-pair shape and at n or m = 1;
    both end modes on every shape; every affinity op; the peaky weights; auto on both sides of N.M = 64; every
    detection-score flag combination on both paths; the cfg2-cfg5 per-pair head shapes in all three heads."""
    for mode in MODES:
        cs = [c for c in AF_CASES if c[5] == mode]
        assert {af_path(c[0], c[1], c[3]) for c in cs} == {"fp32", "tc"}, mode
        assert any(c[0] != c[1] and c[2] > 1 for c in cs), mode
        assert any(c[0] == 1 or c[1] == 1 for c in cs), mode
    for shape in {c[:3] for c in AF_CASES}:
        assert {c[6] for c in AF_CASES if c[:3] == shape} == {"avg", "max"}, shape
    assert {c[4] for c in AF_CASES} == set(OPS)
    assert {c[5] for c in AF_CASES if c[7]} >= {"single", "dual", "dual_add", "dual_max"}
    assert {af_path(c[0], c[1], "auto") for c in AF_CASES if c[3] == "auto"} == {"fp32", "tc"}
    assert {(det_path(c[0], c[2]), c[3]) for c in DET_CASES} == {(p, f) for p in ("fp32", "tc") for f in range(4)}
    assert {c[0] for c in DET_CASES} >= {1, 2, 31, 63, 64, 65, 300} and {c[1] for c in DET_CASES} == {1, 3}
    assert {c[2] for c in DET_CASES} == set(ENGINE)
    assert {c[0] for c in SKIP_CASES} == {"mixed", "offset", "const"}
    assert {c[1] for c in SKIP_CASES if c[0] == "offset"} == {1, 30, 300}
    assert {c[2] for c in SKIP_CASES} >= {1, 5, 64}
    for cfg, N in CFG_N.items():
        assert any(c[0] == N and c[1] == N for c in AF_CASES), cfg
        if cfg != "cfg5":       # the N sweep runs the affinity stage alone
            assert 2 * N in {c[0] for c in DET_CASES}, cfg
            assert 2 * N in {c[3] for c in SKIP_CASES}, cfg


def test_bounds_reject_planted_defects():
    """Each bound accepts a plain fp32 evaluation and misses a planted defect by at least 10x."""
    from oracle import torch_ref
    g = torch.Generator().manual_seed(7)
    out = {}
    # new/end mean over n = 37 objects (columns j of a 37 x 29 map) divided by m
    n, m = 37, 29
    r = (torch.randn(512, n, m, generator=g) * 0.7 + 0.2).clamp_min(0)
    ref, T = mean_bound(r.double().transpose(1, 2), n, False)
    out["mean fp32"] = worst_ratio(r.sum(1) / n, ref, T)
    out["mean / m"] = worst_ratio(r.double().sum(1) / m, ref, T)
    # row sum of a softmax missing its last column
    z = torch.randn(3, n, m, generator=g) * 2
    (rmx, rs, trs), _ = softmax_link(z.double(), "dual")[2]
    out["rsum fp32"] = worst_ratio(torch.exp(z - z.amax(-1, keepdim=True)).sum(-1, keepdim=True), rs, trs)
    out["rsum short"] = worst_ratio(torch.exp(z.double() - rmx)[..., :-1].sum(-1, keepdim=True), rs, trs)
    # link logit without its bias
    sd = synthetic_state_dict("C", seed=7)
    w4, b4 = sd["w_link.conv1.9.weight"].reshape(-1), float(sd["w_link.conv1.9.bias"])
    x = (torch.randn(4096, 128, generator=g) * 0.8 + 0.1).clamp_min(0)
    ref, T = logit_bound(x.double(), w4.double(), b4, 128)
    out["logit fp32"] = worst_ratio(x @ w4 + b4, ref, T)
    out["logit no bias"] = worst_ratio(x.double() @ w4.double(), ref, T)
    # SkipPool head whose last GroupNorm variance divides by 127 (C - 1)
    worst_ok, worst_bad = 0.0, float("inf")
    for s, C in enumerate(SKIP_C):
        pooled = torch.rand(16, C, generator=g) * 10 ** (torch.rand(16, C, generator=g) * 3 - 2)
        ref, T = skip_head_ref(sd, s, pooled.double())
        o32 = torch_ref.skip_pool(sd, s, pooled[:, :, None, None])
        bad, _ = skip_head_ref(sd, s, pooled.double(), last_var_over=127)
        worst_ok = max(worst_ok, worst_ratio(o32, ref, T))
        worst_bad = min(worst_bad, worst_ratio(bad, ref, T))
    out["skip fp32"], out["skip var / (C-1)"] = worst_ok, worst_bad
    report("planted defects (err / bound)", **out)
    assert max(out["mean fp32"], out["rsum fp32"], out["logit fp32"], out["skip fp32"]) <= 1.0, out
    assert min(out["mean / m"], out["rsum short"], out["logit no bias"]) > 10.0, out
    # the head's bound compounds |W| through two contractions and three GroupNorms (about 1e3 times the fp32 error), and
    # a variance 1/128 off moves the output by 1/256 of its spread: the head's margin is smaller (2.4x measured)
    assert out["skip var / (C-1)"] > 2.0, out


# ------------------------------------------------------------------------------------------------ GPU
def _peaky(sd):
    for k in ("w_link.conv1.9.weight", "w_link.conv1.9.bias"):
        sd[k] = sd[k] * PEAKY


@functools.lru_cache(maxsize=None)
def _net(fusion, peaky=False):
    return eval_net(fusion, 29, edit=_peaky if peaky else None)


@gpu
@pytest.mark.parametrize("n,m,pairs,engine,op,sm,end,peaky", AF_CASES, ids=[_af_id(c) for c in AF_CASES])
def test_affinity_tail_vs_fp64(n, m, pairs, engine, op, sm, end, peaky):
    """mmmot_affinity_fwd, then every kernel after the last contraction against fp64 of its own stored inputs."""
    lib = _lib.load()
    net, sd = _net("C", peaky)
    wts = net.prepared()
    G, NM, L = 3 * pairs, n * m, n + m
    g = torch.Generator().manual_seed(case_seed("affinity tail", n, m, pairs, engine, op, sm, end, peaky))
    feats = torch.relu(torch.randn(pairs, 3, 512, L, generator=g)).cuda()
    link, new, end_s = nan_output(G * NM), nan_output(G * m), nan_output(G * n)
    with lib_state(lib, engine=engine):
        lay, tc = stage_layout(lib, 0, pairs, n, m)
        assert tc == (af_path(n, m, engine) == "tc")
        ws = nan_workspace(lib, int(lib.mmmot_affinity_workspace(pairs, n, m)))
        rc = lib.mmmot_affinity_fwd(wts.ptr, _lib.AFFINITY[op], _lib.SOFTMAX[sm], _lib.END_MODE[end], pairs, n, m, vp(feats),
                                    vp(link), vp(new), vp(end_s), vp(ws), ws.numel(), None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    assert lib.mmmot_status_check(vp(ws), None) == 0
    for buf, cnt, what in ((link, G * NM, "link"), (new, G * m, "new"), (end_s, G * n, "end")):
        assert_written(buf, cnt, what)
    size = af_sizes(pairs, n, m)
    wsv = Workspace(ws, lay)
    B = {k: wsv.view(k, size[k] // 4) for k in AF_BUFS[:16]}     # the fp32 buffers this test reads
    r = {}
    # fcl: the channels-last copy of the feature stacks on the tensor-core path, untouched on the FP32 path
    if tc:
        assert torch.equal(B["fcl"].view(G, L, 512), feats.view(G, 512, L).transpose(1, 2)), "fcl"
    else:
        assert bool(torch.isnan(B["fcl"]).all()), "fcl written on the FP32 path"
    # new / end reductions of relu(GN(y0)), y0 = channels 512.. of layer 1
    if tc:
        y0 = B["y01"].view(G, n, m, 1024)[..., 512:]
    else:
        y0 = B["y01"].view(G, 1024, n, m)[:, 512:].permute(0, 2, 3, 1)
    rr0 = norm_operand(y0, B["sc0"].view(G, 1, 1, 512), B["sh0"].view(G, 1, 1, 512)).double()
    mx = end == "max"
    vn, tn = mean_bound(rr0.permute(0, 2, 3, 1), n, mx)       # new column j: over i
    ve, te = mean_bound(rr0.permute(0, 1, 3, 2), m, mx)       # end column i: over j
    del rr0, y0
    V = B["v"].view(G, L, 512) if tc else B["v"].view(512, G, L).permute(1, 2, 0)
    assert bool(torch.isfinite(V).all()), "V"
    r["new_end_mean"] = max(worst_ratio(V[:, :m], vn, tn), worst_ratio(V[:, m:], ve, te))
    # final new/end layer and its scatter
    h2 = B["h2"].view(G, L, 128) if tc else B["h2"].view(128, G, L).permute(1, 2, 0)
    grp = torch.arange(G, device="cuda")[:, None] * 2 + (torch.arange(L, device="cuda") >= m)[None]
    r2 = norm_operand(h2, B["nsc2"].view(2 * G, 128)[grp], B["nsh2"].view(2 * G, 128)[grp]).double()
    a, Ta = logit_bound(r2, sd["w_link.w_new_end.conv1.6.weight"].reshape(-1).double().cuda(),
                        float(sd["w_link.w_new_end.conv1.6.bias"]), 128)
    s, Ts = sigmoid_bound(a, Ta)
    r["new_end_sigmoid"] = max(worst_ratio(new[:G * m].view(G, m), s[:, :m], Ts[:, :m]),
                               worst_ratio(end_s[:G * n].view(G, n), s[:, m:], Ts[:, m:]))
    # link logits
    y3 = B["y3"].view(G, NM, 128) if tc else B["y3"].view(G, 128, NM).transpose(1, 2)
    r3 = norm_operand(y3, B["sc3"].view(G, 1, 128), B["sh3"].view(G, 1, 128)).double()
    zr, Tz = logit_bound(r3, sd["w_link.conv1.9.weight"].reshape(-1).double().cuda(), float(sd["w_link.conv1.9.bias"]), 128)
    zk = (link if sm == "none" else B["z"])[:G * NM].view(G, NM)
    r["link_logit"] = worst_ratio(zk, zr, Tz)
    if sm == "none":
        for k in ("z", "rmax", "rsum", "cmax", "csum"):
            assert bool(torch.isnan(B[k]).all()), f"{k} written in softmax mode none"
    else:
        z = B["z"].view(G, n, m).double()
        ref, T, ((rmx, rs, trs), (cmx, cs, tcs)) = softmax_link(z, sm)
        assert torch.equal(B["rmax"].view(G, n).double(), rmx[..., 0]) and torch.equal(B["cmax"].view(G, m).double(), cmx[:, 0]), \
            "softmax maxima"
        r["softmax_sums"] = max(worst_ratio(B["rsum"].view(G, n), rs[..., 0], trs[..., 0]),
                                worst_ratio(B["csum"].view(G, m), cs[:, 0], tcs[:, 0]))
        got = link[:G * NM].view(G, n, m)
        r["softmax_link"] = worst_ratio(got, ref, T)
        if m == 1:
            assert bool((B["rsum"].view(G, n) == 1).all())
        if n == 1:
            assert bool((B["csum"].view(G, m) == 1).all())
        one = {"single": m == 1, "dual": n == 1 and m == 1, "dual_add": n == 1 and m == 1, "dual_max": n == 1 or m == 1}[sm]
        if one:
            assert bool((got == 1).all()), "a softmax over one element is not exactly 1"
        if peaky:
            r["underflowed"] = float((ref < TINY).double().mean())
    report(f"affinity {_af_id((n, m, pairs, engine, op, sm, end, peaky))} [{'tc' if tc else 'fp32'}] (err / bound)",
            **r, logit_span=float(zr.abs().max()))
    assert all(v <= 1.0 for k, v in r.items() if k != "underflowed"), r


@gpu
@pytest.mark.parametrize("L,pairs,engine,flags,fusion", DET_CASES,
                         ids=[f"L{c[0]}-p{c[1]}-{c[2]}-flags{c[3]}-{c[4]}" for c in DET_CASES])
def test_det_score_vs_fp64(L, pairs, engine, flags, fusion):
    """mmmot_fusion_det_fwd: det against fp64 w3 . h2 + b3 of the stored h2, through the sigmoid and the threshold step
    of the case's flags; F3 and the stack 2 the stage writes, bit for bit."""
    lib = _lib.load()
    net, sd = _net(fusion)
    wts = net.prepared()
    g = torch.Generator().manual_seed(case_seed("det score", L, pairs, engine, flags, fusion))
    feats0 = torch.randn(pairs, 3, 512, L, generator=g).cuda()
    feats0[:, 2] = float("nan")                                  # stack 2 is the fusion's output
    w3, b3 = sd["w_det.6.weight"].reshape(-1).double().cuda(), float(sd["w_det.6.bias"])
    with lib_state(lib, engine=engine):
        lay, tc = stage_layout(lib, 1, pairs, L)
        assert tc == (det_path(L, engine) == "tc")
        thr = 0.0
        if flags & _lib.SCORE_THRESHOLD:     # a threshold at the median score, so both sides of the step are populated
            raw = _run_det(lib, wts, fusion, 0, 0.0, pairs, L, feats0.clone())[0]
            raw = raw[:pairs * 3 * L].double()
            thr = float((torch.sigmoid(raw) if flags & _lib.SCORE_SIGMOID else raw).median())
        det, feats, ws = _run_det(lib, wts, fusion, flags, thr, pairs, L, feats0.clone())
    assert_written(det, pairs * 3 * L, "det")
    assert torch.equal(feats[:, :2], feats0[:, :2]), "feature stacks 0, 1 changed"
    assert bool(torch.isfinite(feats[:, 2]).all()), "stack 2 not written"
    size = fd_sizes(pairs, L)
    wsv = Workspace(ws, lay)
    f3, h2 = wsv.view("f3", size["f3"] // 4), wsv.view("h2", size["h2"] // 4)
    if tc:
        f3 = f3.view(pairs, L, 3, 512)
        for s in range(3):
            assert torch.equal(f3[:, :, s], feats[:, s].transpose(1, 2)), f"F3 stack {s}"
        h2 = h2.view(pairs, L, 3, 256).permute(0, 2, 1, 3)
    else:
        assert bool(torch.isnan(f3).all()), "F3 written on the FP32 path"
        h2 = h2.view(pairs, 3, 256, L).transpose(2, 3)
    a, Ta = logit_bound(h2.double(), w3, b3, 256)
    s, Ts = sigmoid_bound(a, Ta) if flags & _lib.SCORE_SIGMOID else (a, Ta)
    got = det[:pairs * 3 * L].view(pairs, 3, L).double()
    r = {}
    if flags & _lib.SCORE_THRESHOLD:
        step = (s < thr).double()
        clear = (s - thr).abs() > Ts
        exp = s - step
        err = torch.where(clear, (got - exp).abs(), torch.minimum((got - s).abs(), (got - s + 1).abs()))
        bound = Ts + U * torch.where(clear, exp.abs(), s.abs() + 1)
        r["det"] = float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())
        r["stepped"] = float(step.mean())
        assert 0 < float(step.sum()) < step.numel() or step.numel() == 1
    else:
        r["det"] = worst_ratio(got, s, Ts)
    report(f"det score L={L} pairs={pairs} {engine} flags={flags} {fusion} [{'tc' if tc else 'fp32'}] (err / bound)", **r)
    assert r["det"] <= 1.0, r


def _run_det(lib, wts, fusion, flags, thr, pairs, L, feats):
    det = nan_output(pairs * 3 * L)
    ws = nan_workspace(lib, int(lib.mmmot_fusion_det_workspace(pairs, L)))
    rc = lib.mmmot_fusion_det_fwd(wts.ptr, _lib.FUSION[fusion], flags, thr, pairs, L, vp(feats), vp(det), vp(ws), ws.numel(),
                                  None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    assert lib.mmmot_status_check(vp(ws), None) == 0
    return det, feats, ws


def _pooled(kind, R, n_img, C, g):
    if kind == "mixed":      # non-negative, channels of mixed scale (10^-2 .. 10)
        return torch.randn(n_img, C, generator=g).abs() * 10 ** (torch.rand(n_img, C, generator=g) * 3 - 2)
    if kind == "offset":     # a common offset R times the spread, spread of per-image scale 10^-1 .. 10
        sd = 10 ** (torch.rand(n_img, 1, generator=g) * 2 - 1)
        return sd * (R + torch.randn(n_img, C, generator=g))
    return (torch.rand(n_img, 1, generator=g) * 2 + 0.1).expand(n_img, C).contiguous()   # zero variance


@gpu
@pytest.mark.parametrize("kind,R,n_img,L", SKIP_CASES, ids=[f"{c[0]}{c[1] or ''}-n{c[2]}-L{c[3]}" for c in SKIP_CASES])
def test_skip_heads_vs_fp64(kind, R, n_img, L):
    """mmmot_debug_skip_heads on chosen pooled vectors: each head alone writes its own 128 channels of stack 0 and nothing
    else; all four together give the same, against torch_ref.skip_pool's fc chain in fp64 to the derived bound."""
    lib = _lib.load()
    net, sd = _net("C")
    wts = net.prepared()
    sdd = {k: v.double().cuda() for k, v in sd.items() if k.startswith("appearance.global_pool")}
    g = torch.Generator().manual_seed(case_seed("skip heads", kind, R, n_img, L))
    pooled = [_pooled(kind, R, n_img, C, g).cuda() for C in SKIP_C]
    pairs = n_img // L
    r = {}
    alone = []
    for s in range(4):
        feats = torch.full((pairs, 3, 512, L), float("nan"), device="cuda")
        ps = [pooled[k] if k == s else None for k in range(4)]
        assert lib.mmmot_debug_skip_heads(wts.ptr, *map(vp, ps), n_img, L, vp(feats), None) == 0
        torch.cuda.synchronize()
        mine = torch.zeros(512, dtype=torch.bool, device="cuda")
        mine[s * 128:(s + 1) * 128] = True
        assert bool(torch.isfinite(feats[:, 0, mine]).all()), f"head {s}: an owned element was not written"
        assert bool(torch.isnan(feats[:, 0, ~mine]).all()) and bool(torch.isnan(feats[:, 1:]).all()), f"head {s} wrote elsewhere"
        alone.append(feats[:, 0, mine].clone())
        got = feats[:, 0, mine].permute(0, 2, 1).reshape(n_img, 128)
        ref, T = skip_head_ref(sdd, s, pooled[s].double())
        assert torch.allclose(ref, _oracle_head(sdd, s, pooled[s]), rtol=1e-10, atol=1e-12)
        r[f"head{s}"] = worst_ratio(got, ref, T)
    feats = torch.full((pairs, 3, 512, L), float("nan"), device="cuda")
    assert lib.mmmot_debug_skip_heads(wts.ptr, *map(vp, pooled), n_img, L, vp(feats), None) == 0
    torch.cuda.synchronize()
    assert torch.equal(feats[:, 0], torch.cat(alone, 1)) and bool(torch.isnan(feats[:, 1:]).all())
    report(f"skip heads {kind} R={R} n_img={n_img} L={L} (err / bound)", **r)
    assert max(r.values()) <= 1.0, r


def _oracle_head(sdd, s, x):
    from oracle import torch_ref
    return torch_ref.skip_pool(sdd, s, x.double()[:, :, None, None])
