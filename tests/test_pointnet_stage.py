"""PointNet (csrc/pointnet.cu) kernel by kernel against fp64, each kernel on its own stored inputs.

Each GPU case runs the real mmmot_pointnet_fwd once with a workspace filled with NaN (0xFF bytes, status reset) and
feats filled with NaN plus a NaN guard band, then reads the intermediates the stage left in the workspace at the
offsets mmmot_debug_stage_layout(2, ...) reports (the same carve the stage runs).  Every kernel is checked against
fp64 (computed on the GPU) from the inputs it read, as stored, so no upstream error enters a bound wherever that input
survives.  Every element a kernel owns must be written; the padding after each buffer, the buffers the path does not
use, stacks 0 and 2 of feats and its guard band must come back untouched.  Every case prints err / bound (_report).

Notation: u = 2^-24, TAU = 2^-18 (the tensor-core contraction bound, kernel_kit.TAU: |y - y_ref| <= TAU S,
S = |W| A + |b| with A the magnitude of the operand the producer forms), a = gamma / sqrt(var + eps) and
sh = beta - mean a the fp64 GroupNorm affine of the reference statistics, FP64 = 2^-40 (fp64 summation and
cancellation, far below every other term).

GroupNorm statistics (gn_stats).  The kernel's mean and variance of values y_k that err from the reference y by at
most T differ from the two-pass fp64 mean / var of y by
    tm = mean(T) + [KAPPA1 u mean|y|] + FP64 mean|y|,
    tv = 2 mean(|y - mean| T) + mean(T^2) + [KAPPA u (|mean| mean|y - mean| + var)] + FP64 (mean^2 + var),
the bracketed terms only where the sums come from a contraction epilogue's fp32 runs (kernel_kit.stats_ratios).  From
the input moments (layer 5 and the head on the tensor cores, test_pn_moments.py): S2 errs by 2^-18 |X|^T |X|, so
    tv = 1.01 2^-18 mean_p (|x_p| . |w|)^2 + FP64 (mean^2 + var)  (+ (2/n) sum_d |a_d - abar| n_d 2^-33 sum_k |w_k|,
the head's cross term with the 2^-33-rounded per-detection sums of x), and tm = FP64 (mean(|x| . |w|) + mean|y|).
GroupNorm application (gn_apply): relu(fmaf(y_k, sc_k, sh_k)) with sc_k = fl(a_k), sh_k = fl(beta - mean_k a_k) and
|a_k - a| <= |a| er, er = tv / (2 (var + eps)) + FP64, errs before the ReLU (1-Lipschitz) by
    Tz = |a| (T + tm + |y - mean| er) + 8u (|y a| + |sh| + |z|),
the last term the fp32 roundings of sc, sh and the fma; |y a| ~ |mean| / std is GroupNorm's own conditioning.  FP16
hi/lo planes add 2^-22 |z| + 2^-25 (the split's residual; lo may be subnormal).

Tensor-core path (L >= 16 under auto, or mmmot_set_engine(2)):
  tables      tiles, cnt, gstart, seg, ctab equal _pn_host_tables exactly.
  x1p         layer 1 from the points: y = fma(w2, z, fma(w1, y, fma(w0, x, b))) carries T = 1.01 u (|s1| + |s2| + |y|)
              (the fp64 prefix sums), the statistics are fp64 sums of those y (no fp32 runs), then gn_apply and the split.
  t1          layers 2 and 3 from x1p (layer 2's output does not survive): y2 = W2 x1 + b2 to TAU S2, its epilogue
              statistics carrying that, gn_apply, then layer 3 (GEN_NORM) to TAU S3 + |W3|^T Tz2.
  t0          layer 4 from the stored t1: layer 3's statistics recomputed from t1 (epilogue bound), gn_apply, then
              GEN_NORM to TAU S4 + |W4|^T Tz3.
  xp          norm_split of the stored t0 with layer 4's statistics (epilogue bound), gn_apply, the split.
  gmean       layer 5 from xp (hi + lo exact): y5 to TAU S5; statistics from the moments; gn_apply; the per-detection
              mean of the recompute epilogue: fp32 fmas and <= 32-term runs, 40 u sum(|y a| + |sh|), at most one
              2^-33 fixed-point rounding per point, the division u |mean|:
                  T = (sum_p Tz + 40 u sum_p (|y a| + |sh|)) / n_d + 2^-33 + u |mean|.
  ut          U = gmean WhG (GEN_COPY, no bias) to TAU S.
  hmean       as gmean from x1p, the stored ut (addend) and Wh[:, :64], bh, with the addend in S and in the statistics.
  o           conv2 from the stored hmean (GEN_COPY with bias) to TAU S.
  conv2       stats (the stored fp64 sums) against two-pass fp64 over the stored o (the epilogue bound, stats_ratios);
              sc / sh against gn_finalize in fp64 from the stored stats (32 channels per group, count L), one fp32
              rounding each: u |sc| + FP64 |a| (mean^2 + var) / (var + eps), and likewise for sh.
  feats       feats[pair][1][c][l] = relu(fmaf(o, sc, sh)) to u |ref| + 2^-126, from the stored o, sc, sh.
FP32 path (L < 16 under auto, or mmmot_set_engine(1)): the FP32 engine's chain bound (kernel_kit.contraction_bound)
replaces TAU S; y1 from the points (xt equals them transposed bit for bit); sc1 / sh1 from y1
(|sc1 - a| <= |a| er + u |a|, |sh1 - sh| <= |a| tm + |mean a| er + u (|sh| + |mean a|)); t1 from y1 through layer 2
recomputed; t0 from t1; big (the head) from y1, sc1 / sh1 and the addend u; gmean from t0 through layer 5 recomputed
(its output is overwritten by the head), its statistics carrying the contraction bound, and segment_mean's fp32 lane
sums (cnt + 2) u mean|r|; u from gmean; hmean from big with the head's statistics recomputed; o, conv2 and feats as above.

CPU tests: the layout query without a device, a coverage guard over every launch of the stage, and planted
defects: each bound accepts a plain fp32 evaluation and rejects pn_l1_apply taking the next pair's sc / sh, a
per-detection mean divided by n_d + 1, the head taking the neighbouring detection's U row, conv2's GroupNorm taken
over 16 channels per group instead of 32, and pointnet_out_cl with l and c swapped inside a 32 x 32 tile.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

from kernel_kit import (ENGINE, EPS, FP64, PN_BUFS, TAU, TINY, U, Workspace, affine_bound, case_seed,
                        contraction_bound, eval_net, gn_affine, gn_apply, gn_stats, group_moments, group_sum, impl_launches,
                        lib_state, nan_output, nan_workspace, norm_operand, pn_host_tables, ref_linear, report,
                        stage_layout, stats_ratios, vp, worst_ratio)
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_state_dict
from mmmot_b200.weights import prepare

gpu = pytest.mark.gpu
MOM = 2.0 ** -18                   # S2 of the moments kernel (test_pn_moments.py)
FIX = 2.0 ** -33                   # one rounding to 2^-32 fixed point
W = _lib.W
TC_CHECKS = ("tables", "x1p", "t1", "t0", "xp", "gmean", "ut", "hmean", "o", "conv2_stats", "conv2_affine", "feats")
FP32_CHECKS = ("tables", "xt", "y1", "sc1_sh1", "t1", "t0", "big", "gmean", "u", "hmean", "o", "conv2_stats",
               "conv2_affine", "feats")


# ------------------------------------------------------------------------------------------------ layout
def pn_sizes(pairs, L, P, tc):
    """Bytes of each buffer as the header documents them, on the path tc (True: tensor cores)."""
    nd, mt = pairs * L, P // 128 + 2 * pairs + 2
    part16 = max(mt * 1024, ((mt // 32 + pairs) * (128 * 128 + 128) + 1) // 2) if tc else mt * 1024
    fp = lambda v: 0 if tc else v
    tcv = lambda v: v if tc else 0
    return dict(xt=fp(12 * P), y1=fp(256 * P), t0=512 * P, t1=256 * P, big=fp(4096 * P), segsum=8192 * nd,
                x1p=256 * P, xp=512 * P, gmean=4096 * nd, u=fp(2048 * nd), ut=tcv(2048 * nd),
                hmean=2048 * nd, o=2048 * nd, sc1=256 * pairs, sh1=256 * pairs, sc=4096 * pairs, sh=4096 * pairs,
                stats=16384 * pairs, mom=tcv(8 * pairs * (128 * 128 + 128)), part=16 * part16, gstart=4 * (pairs + 1),
                sstart=tcv(4 * (pairs + 1)), seg=4 * P, cnt=4 * pairs, tiles=16 * mt, ctab=32 * mt)


def _align(n):
    return (n + 255) // 256 * 256


# ------------------------------------------------------------------------------------------------ fp64 bounds
def mom_stats(y, XW, grp, G, cross=None):
    """Statistics from the input moments: y [n][C] the fp64 reference, XW = |x| @ |W| -> (mean, var, tm, tv)."""
    n, mean, var, _, may = group_moments(y, grp, G)
    tv = 1.01 * MOM * group_sum(XW * XW, grp, G) / n + FP64 * (mean * mean + var)
    if cross is not None:
        tv = tv + cross
    return mean, var, FP64 * (group_sum(XW, grp, G) / n + may), tv


def split_bound(z):
    return 2.0 ** -22 * z.abs() + 2.0 ** -25


def seg_mean_tc(z, Tz, mag, seg, cnt):
    """Per-detection mean of relu(z) through the 2^-32 fixed-point segment sums -> (ref [ndet][C], bound)."""
    nd = cnt.shape[0]
    ref = group_sum(z.clamp_min(0), seg, nd) / cnt
    return ref, (group_sum(Tz, seg, nd) + 40 * U * group_sum(mag, seg, nd)) / cnt + FIX + U * ref.abs()


def seg_mean_fp32(z, Tz, seg, cnt):
    """segment_mean_kernel: fp32 lane sums of relu(z) over the detection, then the division."""
    nd = cnt.shape[0]
    r = z.clamp_min(0)
    ref = group_sum(r, seg, nd) / cnt
    return ref, group_sum(Tz, seg, nd) / cnt + (cnt + 2) * U * group_sum(r, seg, nd) / cnt + U * ref.abs()


def out_ref(o, sc, sh):
    """relu(o sc + sh) in fp64 of the stored fp32 values (o [pairs][L][512]) -> ([pairs][512][L], bound)."""
    ref = (o.double() * sc.double()[:, None] + sh.double()[:, None]).clamp_min(0).transpose(1, 2)
    return ref, U * ref.abs() + TINY


def l1_ref(pts, W1, b1):
    """Layer 1 as pn_l1_*_kernel evaluate it, y = fma(w2, z, fma(w1, y, fma(w0, x, b))) -> (y [P][64], T)."""
    s1 = b1 + pts[:, :1] * W1[0]
    s2 = s1 + pts[:, 1:2] * W1[1]
    y = s2 + pts[:, 2:3] * W1[2]
    return y, 1.01 * U * (s1.abs() + s2.abs() + y.abs())


# ------------------------------------------------------------------------------------------------ cases
# (name, pairs, L, points, engine): points "rN" ragged 1..2N-1 per detection with two 1-point detections, "uN" N per
# detection (the benchmark shapes), "skew" pair totals 255 / 257 / 9000 (the last spans two 8192-point moment slices),
# "far" detections at 63.5-66.5 m with 0.5 m spread (layer-1 channels at |mean| / std >= 30), "same" one point
# repeated (every trunk GroupNorm has zero variance), "one" a single point.
TC_CASES = [("L16", 1, 16, "r64", "auto"), ("cfg2", 2, 64, "u128", "auto"), ("cfg3", 1, 128, "u512", "auto"),
            ("cfg4", 1, 256, "u512", "auto"), ("L300", 1, 300, "r96", "auto"), ("skew", 3, 16, "skew", "auto"),
            ("far", 1, 32, "far", "auto"), ("same", 1, 16, "same", "auto"),
            ("L1-tc", 2, 1, "r200", "tc"), ("L2-tc", 3, 2, "r100", "tc"), ("L7-tc", 2, 7, "r60", "tc")]
FP32_CASES = [("L1-P1", 1, 1, "one", "auto"), ("L2", 2, 2, "r50", "auto"), ("L15", 1, 15, "r100", "auto"),
              ("L40-fp32", 2, 40, "r300", "fp32")]


def pn_path(L, engine):
    return engine if engine != "auto" else ("tc" if L >= 16 else "fp32")


def _counts(kind, pairs, L, g):
    if kind == "one":
        return [1] * (pairs * L)
    if kind[0] == "u":
        return [int(kind[1:])] * (pairs * L)
    if kind == "skew":
        out = []
        for total in (255, 257, 9000):
            w = torch.rand(L - 1, generator=g) + 0.05
            c = (1 + (w / w.sum() * (total - 2 * L + 1)).floor()).long()
            c[-1] += total - 1 - int(c.sum())
            out += [1] + c.tolist()
        return out
    n = int(kind[1:]) if kind[0] == "r" else 128
    c = torch.randint(1, 2 * n, (pairs * L,), generator=g)
    c[torch.randperm(pairs * L, generator=g)[:2]] = 1
    return c.tolist()


def _points(kind, counts, g):
    P = sum(counts)
    if kind in ("same", "one"):
        return torch.tensor([[12.25, -3.5, -1.0]]).expand(P, 3).contiguous()
    nd = len(counts)
    if kind == "far":
        centre = torch.rand(nd, 3, generator=g) * torch.tensor([3.0, 2.0, 0.5]) + torch.tensor([63.5, -1.0, -1.5])
        spread = torch.tensor([0.5, 0.5, 0.5])
    else:
        centre = torch.rand(nd, 3, generator=g) * torch.tensor([60.0, 40.0, 2.0]) + torch.tensor([0.0, -20.0, -2.0])
        spread = torch.tensor([2.0, 1.0, 0.8])
    return torch.randn(P, 3, generator=g) * spread + centre.repeat_interleave(torch.tensor(counts), 0)


@functools.lru_cache(maxsize=None)
def _net():
    net, sd = eval_net("C", 31)
    t = prepare(sd, "C")[0]
    w = lambda k: t[W[k]].double().cuda()
    wt = dict(layers=[tuple(t[W["PN_L1"] + 4 * j + i].double().cuda() for i in range(4)) for j in range(5)])
    for k in ("PN_WHAT", "PN_WHGT", "PN_BH", "PN_GHW", "PN_GHB", "PN_WOT", "PN_BO", "PN_GOW", "PN_GOB"):
        wt[k] = w(k)
    return net, wt


def _run(lib, case):
    name, pairs, L, kind, engine = case
    net, wt = _net()
    g = torch.Generator().manual_seed(case_seed("pointnet stage", *case))
    counts = _counts(kind, pairs, L, g)
    pts = _points(kind, counts, g).cuda()
    split = [0] + np.cumsum(counts).tolist()
    P = split[-1]
    hs = np.asarray(split, dtype=np.int32)
    feats = nan_output(pairs * 3 * 512 * L)
    with lib_state(lib, engine=engine):
        lay, tc = stage_layout(lib, 2, pairs, L, P)
        nbytes = int(lib.mmmot_pointnet_workspace(pairs, L, P))
        ws = nan_workspace(lib, nbytes)
        rc = lib.mmmot_pointnet_fwd(net.prepared().ptr, vp(pts), vp(torch.tensor(hs, device="cuda")),
                                    ctypes.c_void_p(hs.ctypes.data), pairs, L, vp(feats), vp(ws), nbytes, None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    assert tc == (pn_path(L, engine) == "tc")
    assert lay["end"] == nbytes
    assert lib.mmmot_status_check(vp(ws), None) == 0, "status word raised"
    nf = pairs * 3 * 512 * L
    f = feats[:nf].view(pairs, 3, 512, L)
    assert bool(torch.isfinite(f[:, 1]).all()), "feats stack 1: an element was not written"
    assert bool(torch.isnan(f[:, 0]).all() and torch.isnan(f[:, 2]).all()), "feats stacks 0 / 2 written"
    assert bool(torch.isnan(feats[nf:]).all()), "feats written past its end"
    seg = torch.tensor(np.repeat(np.arange(pairs * L), counts), device="cuda")
    cnt = torch.tensor(counts, dtype=torch.float64, device="cuda")[:, None]
    return dict(pairs=pairs, L=L, P=P, split=split, pts=pts.double(), seg=seg, grp=seg // L, cnt=cnt, wt=wt,
                W=Workspace(ws, lay), f=f, tc=tc)


def _planes(W, name, P, C):
    h = W.owned(name, 2 * P * C, torch.float16).view(2, P, C)
    return h[0].double() + h[1].double()


def _check_tables(d, tw):
    W, pairs, L, P, split = d["W"], d["pairs"], d["L"], d["P"], d["split"]
    tiles = [(p, c, min(tw, split[(p + 1) * L] - c)) for p in range(pairs) for c in range(split[p * L], split[(p + 1) * L], tw)]
    nt = len(tiles)
    got = W.owned("tiles", 4 * nt, torch.int32).view(nt, 4).tolist()
    assert got == [[p, c, ln, 0] for p, c, ln in tiles], "tiles"
    cnt = [split[(p + 1) * L] - split[p * L] for p in range(pairs)]
    assert W.owned("cnt", pairs, torch.int32).tolist() == cnt, "cnt"
    gstart = np.concatenate([[0], np.cumsum([-(-c // tw) for c in cnt])]).tolist()
    assert W.owned("gstart", pairs + 1, torch.int32).tolist() == gstart, "gstart"
    assert torch.equal(W.owned("seg", P, torch.int32).long(), d["seg"]), "seg"
    if d["tc"]:
        ctab = pn_host_tables(split, pairs, L)[2]
        assert W.owned("ctab", 4 * len(ctab), torch.int32).view(-1, 4).tolist() == ctab, "ctab"
    else:
        assert W.untouched_after("ctab", 0), "ctab written on the FP32 path"
    return 0.0


def _check_conv2(d, o, r):
    """conv2's statistics, GroupNorm(16, 512) affine and the output transpose; o [ndet][512] as stored."""
    W, pairs, L, wt = d["W"], d["pairs"], d["L"], d["wt"]
    nd = pairs * L
    stats = W.view("stats", pairs * 1024 * 2, torch.float64)[:pairs * 512 * 2].view(pairs, 512, 2)
    assert bool(torch.isfinite(stats).all()), "conv2 stats not written"
    pg = torch.arange(nd, device="cuda") // L
    rv, rm, _ = stats_ratios(stats[..., 0], stats[..., 1], o.double(), pg, pairs)
    r["conv2_stats"] = max(rv, rm)
    sc = W.view("sc", pairs * 1024)[:pairs * 512].view(pairs, 512)
    sh = W.view("sh", pairs * 1024)[:pairs * 512].view(pairs, 512)
    a, b, Ta, Tb = gn_affine(stats, wt["PN_GOW"], wt["PN_GOB"], L, 32)
    r["conv2_affine"] = max(worst_ratio(sc, a, Ta), worst_ratio(sh, b, Tb))
    ref, T = out_ref(o.view(pairs, L, 512), sc, sh)
    r["feats"] = worst_ratio(d["f"][:, 1], ref, T)


def check_tc(d):
    W, pairs, L, P, wt, grp, seg, cnt = (d[k] for k in ("W", "pairs", "L", "P", "wt", "grp", "seg", "cnt"))
    nd = pairs * L
    lay = W.lay
    lyr = wt["layers"]
    r = {"tables": _check_tables(d, 256)}
    for k in ("xt", "y1", "big", "u"):                  # zero-sized on this path
        assert lay[k] == lay[PN_BUFS[PN_BUFS.index(k) + 1]], k
    for k in ("sc1", "sh1"):
        assert W.untouched_after(k, 0), f"{k} written on the tensor-core path"
    # x1p: layer 1 from the points
    W1, b1, g1, be1 = lyr[0]
    y, T = l1_ref(d["pts"], W1, b1)
    st = gn_stats(y, grp, pairs, T, kappa=False)
    d["cond"] = float((st[0].abs() / st[1].clamp_min(1e-300).sqrt()).max())
    z, Tz, _ = gn_apply(y, T, grp, st, g1, be1)
    x1 = _planes(W, "x1p", P, 64)
    r["x1p"] = worst_ratio(x1, z.clamp_min(0), Tz + split_bound(z))
    # t1: layers 2, 3 from x1p
    W2, b2, g2, be2 = lyr[1]
    W3, b3, g3, be3 = lyr[2]
    y2, S2 = ref_linear(x1, x1.abs(), W2, b2)
    st = gn_stats(y2, grp, pairs, TAU * S2)
    z, Tz, mag = gn_apply(y2, TAU * S2, grp, st, g2, be2)
    y3, S3 = ref_linear(z.clamp_min(0), mag, W3, b3)
    t1 = W.owned("t1", 64 * P).view(P, 64)
    r["t1"] = worst_ratio(t1, y3, TAU * S3 + Tz @ W3.abs())
    # t0: layer 4 from the stored t1
    W4, b4, g4, be4 = lyr[3]
    y = t1.double()
    z, Tz, mag = gn_apply(y, None, grp, gn_stats(y, grp, pairs), g3, be3)
    y4, S4 = ref_linear(z.clamp_min(0), mag, W4, b4)
    t0 = W.owned("t0", 128 * P).view(P, 128)
    r["t0"] = worst_ratio(t0, y4, TAU * S4 + Tz @ W4.abs())
    # xp: norm_split of the stored t0
    y = t0.double()
    z, Tz, _ = gn_apply(y, None, grp, gn_stats(y, grp, pairs), g4, be4)
    xp = _planes(W, "xp", P, 128)
    r["xp"] = worst_ratio(xp, z.clamp_min(0), Tz + split_bound(z))
    del y, z, Tz, mag, y2, S2, y3, S3, y4, S4
    # gmean: layer 5 from xp, statistics from the moments, the per-detection means
    W5, b5, g5, be5 = lyr[4]
    gm = W.owned("gmean", nd * 1024).view(nd, 1024)
    r["gmean"] = 0.0
    for c0 in range(0, 1024, 128):
        cs = slice(c0, c0 + 128)
        y, S = ref_linear(xp, xp.abs(), W5[:, cs], b5[cs])
        st = mom_stats(y, xp.abs() @ W5[:, cs].abs(), grp, pairs)
        z, Tz, mag = gn_apply(y, TAU * S, grp, st, g5[cs], be5[cs])
        ref, T = seg_mean_tc(z, Tz, mag, seg, cnt)
        r["gmean"] = max(r["gmean"], worst_ratio(gm[:, cs], ref, T))
    del y, S, z, Tz, mag
    # ut: U = gmean WhG
    ut = W.owned("ut", nd * 512).view(nd, 512)
    ref, S = ref_linear(gm.double(), gm.double().abs(), wt["PN_WHGT"], torch.zeros(512, dtype=torch.float64, device="cuda"))
    r["ut"] = worst_ratio(ut, ref, TAU * S)
    # hmean: the head from x1p and the stored addend ut
    hm = W.owned("hmean", nd * 512).view(nd, 512)
    WhA, bh = wt["PN_WHAT"], wt["PN_BH"]
    ad = ut.double() + bh                                             # a_d of the moments kernel
    n_p = group_sum(cnt, torch.arange(nd, device="cuda") // L, pairs)
    abar = group_sum(cnt * ad, torch.arange(nd, device="cuda") // L, pairs) / n_p
    cross = 2 * group_sum(cnt * (ad - abar[torch.arange(nd, device="cuda") // L]).abs(), torch.arange(nd, device="cuda") // L,
                     pairs) / n_p * FIX * WhA.abs().sum(0)
    r["hmean"] = 0.0
    for c0 in range(0, 512, 128):
        cs = slice(c0, c0 + 128)
        y, S = ref_linear(x1, x1.abs(), WhA[:, cs], bh[cs])
        add = ut[:, cs].double()[seg]
        y, S = y + add, S + add.abs()
        st = mom_stats(y, x1.abs() @ WhA[:, cs].abs(), grp, pairs, cross[:, cs])
        z, Tz, mag = gn_apply(y, TAU * S, grp, st, wt["PN_GHW"][cs], wt["PN_GHB"][cs])
        ref, T = seg_mean_tc(z, Tz, mag, seg, cnt)
        r["hmean"] = max(r["hmean"], worst_ratio(hm[:, cs], ref, T))
    del y, S, z, Tz, mag, add
    # o: conv2 from the stored hmean
    o = W.owned("o", nd * 512).view(nd, 512)
    ref, S = ref_linear(hm.double(), hm.double().abs(), wt["PN_WOT"], wt["PN_BO"])
    r["o"] = worst_ratio(o, ref, TAU * S)
    _check_conv2(d, o, r)
    return r


def check_fp32(d):
    W, pairs, L, P, wt, grp, seg, cnt = (d[k] for k in ("W", "pairs", "L", "P", "wt", "grp", "seg", "cnt"))
    nd = pairs * L
    lay = W.lay
    lyr = wt["layers"]
    r = {"tables": _check_tables(d, 128)}
    for k in ("ut", "mom", "sstart"):                  # zero-sized on this path
        assert lay[k] == lay[PN_BUFS[PN_BUFS.index(k) + 1]], k
    for k in ("segsum", "x1p", "xp"):
        assert W.untouched_after(k, 0), f"{k} written on the FP32 path"
    xt = W.owned("xt", 3 * P).view(3, P)
    assert torch.equal(xt.double(), d["pts"].T), "xt"
    r["xt"] = 0.0
    # y1 and its GroupNorm affine
    W1, b1, g1, be1 = lyr[0]
    y1 = W.owned("y1", 64 * P).view(64, P)
    ref, T = contraction_bound(W1, d["pts"].T.contiguous(), b1)
    r["y1"] = worst_ratio(y1, ref, T)
    y = y1.double().T
    a, sh, Ta, Tsh = affine_bound(gn_stats(y, grp, pairs), g1, be1)
    sc1 = W.owned("sc1", pairs * 64).view(pairs, 64)
    sh1 = W.owned("sh1", pairs * 64).view(pairs, 64)
    r["sc1_sh1"] = max(worst_ratio(sc1, a, Ta), worst_ratio(sh1, sh, Tsh))
    # t1: layers 2 (recomputed from the stored y1, sc1, sh1) and 3
    W2, b2, g2, be2 = lyr[1]
    W3, b3, g3, be3 = lyr[2]
    x2 = norm_operand(y1, sc1.T[:, grp], sh1.T[:, grp]).double()
    y2, T2 = contraction_bound(W2, x2, b2)
    st = gn_stats(y2.T, grp, pairs, T2.T)
    z, Tz, _ = gn_apply(y2.T, T2.T, grp, st, g2, be2)
    y3, T3 = contraction_bound(W3, z.clamp_min(0).T.contiguous(), b3)
    t1 = W.owned("t1", 64 * P).view(64, P)
    r["t1"] = worst_ratio(t1, y3, T3 + (Tz @ W3.abs()).T)
    # t0: layer 4 from the stored t1
    W4, b4, g4, be4 = lyr[3]
    y = t1.double().T
    z, Tz, _ = gn_apply(y, None, grp, gn_stats(y, grp, pairs), g3, be3)
    y4, T4 = contraction_bound(W4, z.clamp_min(0).T.contiguous(), b4)
    t0 = W.owned("t0", 128 * P).view(128, P)
    r["t0"] = worst_ratio(t0, y4, T4 + (Tz @ W4.abs()).T)
    # big: the head from y1, sc1, sh1 and the addend u
    u = W.owned("u", 512 * nd).view(512, nd)
    big = W.owned("big", 1024 * P)[:512 * P].view(512, P)     # rows 512.. still hold layer 5's output
    ref, T = contraction_bound(wt["PN_WHAT"], x2, wt["PN_BH"], u.double()[:, seg])
    r["big"] = worst_ratio(big, ref, T)
    del x2, y2, T2, y3, T3, y4, T4, ref, T
    # gmean: layer 5 recomputed from the stored t0, its statistics, segment_mean
    W5, b5, g5, be5 = lyr[4]
    y = t0.double().T
    z4, Tz4, _ = gn_apply(y, None, grp, gn_stats(y, grp, pairs), g4, be4)
    x5 = z4.clamp_min(0).T.contiguous()
    gm = W.owned("gmean", 1024 * nd).view(1024, nd)
    r["gmean"] = 0.0
    for c0 in range(0, 1024, 128):
        cs = slice(c0, c0 + 128)
        y5, T5 = contraction_bound(W5[:, cs], x5, b5[cs])
        y5, T5 = y5.T, T5.T + Tz4 @ W5[:, cs].abs()
        z, Tz, _ = gn_apply(y5, T5, grp, gn_stats(y5, grp, pairs, T5), g5[cs], be5[cs])
        ref, T = seg_mean_fp32(z, Tz, seg, cnt)
        r["gmean"] = max(r["gmean"], worst_ratio(gm[cs].T, ref, T))
    del z4, Tz4, x5, y5, T5, z, Tz
    # u from gmean
    ref, T = contraction_bound(wt["PN_WHGT"], gm.double())
    r["u"] = worst_ratio(u, ref, T)
    # hmean from big, the head's statistics recomputed
    y = big.double().T
    z, Tz, _ = gn_apply(y, None, grp, gn_stats(y, grp, pairs), wt["PN_GHW"], wt["PN_GHB"])
    hm = W.owned("hmean", 512 * nd).view(512, nd)
    ref, T = seg_mean_fp32(z, Tz, seg, cnt)
    r["hmean"] = worst_ratio(hm.T, ref, T)
    # o: conv2 from the stored hmean
    o = W.owned("o", 512 * nd).view(512, nd)
    ref, T = contraction_bound(wt["PN_WOT"], hm.double(), wt["PN_BO"])
    r["o"] = worst_ratio(o, ref, T)
    _check_conv2(d, o.T.contiguous(), r)
    return r


# ------------------------------------------------------------------------------------------------ GPU
@gpu
@pytest.mark.parametrize("case", TC_CASES + FP32_CASES, ids=[c[0] for c in TC_CASES + FP32_CASES])
def test_pointnet_stage_vs_fp64(case):
    """mmmot_pointnet_fwd, then every kernel against fp64 of its own stored inputs (module docstring)."""
    lib = _lib.load()
    d = _run(lib, case)
    r = check_tc(d) if d["tc"] else check_fp32(d)
    assert set(r) == set(TC_CHECKS if d["tc"] else FP32_CHECKS), sorted(r)
    extra = {"layer1_mean_over_std": d["cond"]} if "cond" in d else {}
    report(f"pointnet {case[0]} pairs={d['pairs']} L={d['L']} P={d['P']} [{'tc' if d['tc'] else 'fp32'}] (err / bound)",
            **r, **extra)
    if case[0] == "far":
        assert d["cond"] >= 30, d["cond"]
    assert all(v <= 1.0 for v in r.values()), r


# ------------------------------------------------------------------------------------------------ CPU
def test_pointnet_layout_without_device():
    """mmmot_debug_stage_layout(2, ...) on the host: the offsets are the carve order, every buffer holds exactly its
    documented size on the path the engine setting selects (xt, y1, big, u empty on the tensor cores, ut on the FP32
    path), and `end` is mmmot_pointnet_workspace."""
    lib = _lib.load()
    for engine in ENGINE:
        with lib_state(lib, engine=engine):
            for pairs, L, P in ((1, 1, 1), (2, 2, 100), (1, 15, 900), (1, 16, 1000), (3, 16, 9512), (2, 64, 16384),
                                (1, 256, 131072), (1, 300, 28800)):
                lay, tc = stage_layout(lib, 2, pairs, L, P)
                assert tc == (pn_path(L, engine) == "tc"), (engine, L)
                assert lay["end"] == int(lib.mmmot_pointnet_workspace(pairs, L, P))
                size = pn_sizes(pairs, L, P, tc)
                assert lay["xt"] == 256
                for a, b in zip(PN_BUFS, PN_BUFS[1:]):
                    assert lay[b] - lay[a] == _align(size[a]), (engine, pairs, L, P, a)
                for k in (("xt", "y1", "big", "u") if tc else ("ut", "sstart", "mom")):
                    assert size[k] == 0
    off = (ctypes.c_size_t * 32)()
    for args in ((2, 1, 4, 0), (2, 0, 4, 10), (2, 1, 0, 10)):
        assert lib.mmmot_debug_stage_layout(*args, off, None) == -1, args


# The functions the stage runs and, per function, every kernel launch and helper call in its body, in source order, with
# the checks above that hold its output.  A call of pn_wide_layer counts as a site of the layer it runs.
LAUNCH_SITES = {
    "pointnet_impl": [("pn_tables", ("tables",))],
    "pointnet_tc": [
        ("pn_l1_stats_kernel", ("x1p",)),
        ("stats_reduce", ("x1p",)),
        ("gn_finalize", ("x1p",)),
        ("pn_l1_apply_kernel", ("x1p",)),
        ("gemm_gen_launch", ("t1", "t0")),              # layers 3, 4 (GEN_NORM)
        ("gemm_tma_launch_mat", ("t1",)),               # layer 2 from x1p
        ("stats_reduce", ("t1", "t0", "xp")),
        ("gn_finalize", ("t1", "t0", "xp")),
        ("norm_split", ("xp",)),
        ("pn_wide_layer", ("gmean",)),                  # layer 5
        ("gemm_gen_launch", ("ut",)),
        ("pn_wide_layer", ("hmean",)),                  # head
        ("gemm_gen_launch", ("o",)),
        ("stats_reduce", ("conv2_stats",)),
        ("gn_finalize", ("conv2_affine",)),
        ("pointnet_out_cl_kernel", ("feats",)),
    ],
    "pn_wide_layer": [
        ("pn_wide_stats", ("gmean", "hmean")),          # statistics from the moments
        ("gn_finalize", ("gmean", "hmean")),
        ("gemm_tma_launch_mat", ("gmean", "hmean")),    # recompute + per-detection sums
        ("segsum_mean_cl_kernel", ("gmean", "hmean")),
    ],
    "pointnet_fp32": [
        ("transpose_points_kernel", ("xt",)),
        ("gemm_simt_launch", ("y1",)),
        ("gemm_simt_launch", ("t1", "t0", "gmean")),
        ("stats_reduce", ("sc1_sh1", "t1", "t0", "gmean")),
        ("gn_finalize", ("sc1_sh1", "t1", "t0", "gmean")),
        ("segment_mean_kernel", ("gmean",)),
        ("gemm_simt_launch", ("u",)),
        ("gemm_simt_launch", ("big",)),
        ("stats_reduce", ("hmean",)),
        ("gn_finalize", ("hmean",)),
        ("segment_mean_kernel", ("hmean",)),
        ("gemm_simt_launch", ("o",)),
        ("stats_reduce", ("conv2_stats",)),
        ("gn_finalize", ("conv2_affine",)),
        ("pointnet_out_kernel", ("feats",)),
    ],
}


PN_HELPERS = (r"gemm_\w+_launch\w*", "norm_split", "stats_reduce", "gn_finalize", "pn_wide_stats", "pn_wide_layer",
              "pn_tables")


def test_stage_launch_coverage_guard():
    """Every launch in the functions the stage runs maps to a check of this file: a launch added, removed or reordered
    without its entry in LAUNCH_SITES fails here, and every check named there is one the GPU test fills."""
    for func, sites in LAUNCH_SITES.items():
        assert impl_launches("pointnet.cu", func, PN_HELPERS) == [s[0] for s in sites], func
    named = {c for sites in LAUNCH_SITES.values() for _, cs in sites for c in cs}
    assert named <= set(TC_CHECKS) | set(FP32_CHECKS), named - set(TC_CHECKS) - set(FP32_CHECKS)
    assert (set(TC_CHECKS) | set(FP32_CHECKS)) - {"tables"} <= named


def test_case_coverage():
    """The GPU cases take both paths under auto and under each forced engine, run the cfg2-cfg4 per-pair shapes, the
    engine boundary L = 16, a 12-column tail tile of pointnet_out_cl (L = 300), GroupNorm over 1, 2 and 7 detections
    on the tensor cores, several pairs on both paths, and 1-point detections."""
    cases = TC_CASES + FP32_CASES
    assert {(pn_path(c[2], c[4]), c[4]) for c in cases} == {("tc", "auto"), ("tc", "tc"), ("fp32", "auto"), ("fp32", "fp32")}
    assert {16, 64, 128, 256, 300} <= {c[2] for c in TC_CASES} and 300 % 32 == 12
    assert {1, 2, 7} <= {c[2] for c in TC_CASES if c[4] == "tc"}
    assert any(c[1] > 1 for c in TC_CASES) and any(c[1] > 1 for c in FP32_CASES)
    assert {15, 1} <= {c[2] for c in FP32_CASES}
    g = torch.Generator().manual_seed(0)
    sk = _counts("skew", 3, 16, g)
    assert [sum(sk[p * 16:(p + 1) * 16]) for p in range(3)] == [255, 257, 9000] and min(sk) == 1
    assert 8192 < 9000 and min(_counts("r64", 1, 16, g)) == 1


def _weights_cpu():
    t = prepare(synthetic_state_dict("C", seed=31), "C")[0]
    return lambda k, i=0: t[W[k] + i].double()


def _fp32_gn(y32, grp, G, gamma, beta):
    """The plain fp32 evaluation of GroupNorm + ReLU: fp64 statistics of the fp32 values, fp32 affine, fp32 fma."""
    _, mean, var, _, _ = group_moments(y32.double(), grp, G)
    a = gamma / torch.sqrt(var + EPS)
    sc, sh = a.float(), (beta - mean * a).float()
    return sc, sh


def test_bounds_reject_planted_defects():
    """Each bound accepts a plain fp32 evaluation and rejects its planted defect by at least 10x."""
    w = _weights_cpu()
    g = torch.Generator().manual_seed(11)
    out = {}
    # pn_l1_apply taking the next pair's sc / sh
    pairs, L = 2, 16
    counts = [int(c) for c in torch.randint(1, 200, (pairs * L,), generator=g)]
    pts = _points("r", counts, g)
    grp = torch.tensor(np.repeat(np.arange(pairs * L), counts)) // L
    W1, b1, g1, be1 = (w("PN_L1", i) for i in range(4))
    y, T = l1_ref(pts.double(), W1, b1)
    z, Tz, _ = gn_apply(y, T, grp, gn_stats(y, grp, pairs, T, kappa=False), g1, be1)
    p32, w32 = pts.float(), W1.float()
    y32 = b1.float().expand(len(pts), 64)
    for k in range(3):
        y32 = (p32[:, k:k + 1].double() * w32[k].double() + y32.double()).float()
    sc, sh = _fp32_gn(y32, grp, pairs, g1, be1)
    T = Tz + split_bound(z)
    def ev(s):                                          # relu(fmaf(y, sc, sh)) as FP16 hi + lo
        v = (y32.double() * sc[s].double() + sh[s].double()).float().clamp_min(0)
        hi = v.half()
        return hi.double() + (v - hi.float()).half().double()
    out["l1 fp32"] = worst_ratio(ev(grp), z.clamp_min(0), T)
    out["l1 next pair"] = worst_ratio(ev((grp + 1) % pairs), z.clamp_min(0), T)
    # a per-detection mean divided by n_d + 1 (layer 5 on the tensor cores, 128 channels)
    nd = pairs * L
    seg = torch.tensor(np.repeat(np.arange(nd), counts))
    cnt = torch.tensor(counts, dtype=torch.float64)[:, None]
    x = torch.relu(torch.randn(len(seg), 128, generator=g) + 0.3).double()
    W5, b5 = w("PN_L1", 16)[:, :128], w("PN_L1", 17)[:128]
    y = x @ W5 + b5
    S = x.abs() @ W5.abs() + b5.abs()
    st = mom_stats(y, x.abs() @ W5.abs(), grp, pairs)
    z, Tz, mag = gn_apply(y, TAU * S, grp, st, w("PN_L1", 18)[:128], w("PN_L1", 19)[:128])
    ref, T = seg_mean_tc(z, Tz, mag, seg, cnt)
    a = w("PN_L1", 18)[:128] / torch.sqrt(st[1] + EPS)
    sc32, sh32 = a.float(), (w("PN_L1", 19)[:128] - st[0] * a).float()
    y32 = x.float() @ W5.float() + b5.float()
    r32 = (y32.double() * sc32[grp].double() + sh32[grp].double()).float().clamp_min(0)
    s32 = torch.zeros(nd, 128).index_add_(0, seg, r32).double()
    out["mean fp32"] = worst_ratio((s32 / cnt).float(), ref, T)
    out["mean / (n+1)"] = worst_ratio(s32 / (cnt + 1), ref, T)
    # the head taking the neighbouring detection's U row (every point of detection 3 takes detection 4's)
    x1 = torch.relu(torch.randn(len(seg), 64, generator=g) + 0.2).double()
    WhA, bh = w("PN_WHAT")[:, :128], w("PN_BH")[:128]
    ut = torch.randn(nd, 128, generator=g).double() * 0.5
    y = x1 @ WhA + bh + ut[seg]
    S = x1.abs() @ WhA.abs() + bh.abs() + ut[seg].abs()
    st = mom_stats(y, x1.abs() @ WhA.abs(), grp, pairs)
    z, Tz, mag = gn_apply(y, TAU * S, grp, st, w("PN_GHW")[:128], w("PN_GHB")[:128])
    ref, T = seg_mean_tc(z, Tz, mag, seg, cnt)
    a = w("PN_GHW")[:128] / torch.sqrt(st[1] + EPS)
    sc32, sh32 = a.float(), (w("PN_GHB")[:128] - st[0] * a).float()

    def head(useg):
        h = (x1.float() @ WhA.float() + bh.float() + ut.float()[useg])
        r = (h.double() * sc32[grp].double() + sh32[grp].double()).float().clamp_min(0)
        return torch.zeros(nd, 128).index_add_(0, seg, r).double() / cnt
    out["head fp32"] = worst_ratio(head(seg), ref, T)
    bad = seg.clone()
    bad[seg == 3] = 4
    out["head neighbour U"] = worst_ratio(head(bad), ref, T)
    # conv2's GroupNorm over 16 channels per group instead of 32
    L2 = 40
    o = torch.randn(pairs * L2, 512, generator=g) * 0.7 + torch.randn(512, generator=g) * 0.3
    stats = torch.stack([group_sum(o.double(), torch.arange(pairs * L2) // L2, pairs),
                         group_sum(o.double() ** 2, torch.arange(pairs * L2) // L2, pairs)], -1)
    a, b, Ta, Tb = gn_affine(stats, w("PN_GOW"), w("PN_GOB"), L2, 32)
    a16, b16, _, _ = gn_affine(stats, w("PN_GOW"), w("PN_GOB"), L2, 16)
    out["conv2 fp32"] = max(worst_ratio(a.float(), a, Ta), worst_ratio(b.float(), b, Tb))
    out["conv2 16 per group"] = max(worst_ratio(a16.float(), a, Ta), worst_ratio(b16.float(), b, Tb))
    # pointnet_out_cl with l and c swapped inside each 32 x 32 tile (L = 40: one full tile and an 8-column tail)
    sc, sh = a.float().view(pairs, 512), b.float().view(pairs, 512)
    ref, T = out_ref(o.view(pairs, L2, 512), sc, sh)
    good = (o.view(pairs, L2, 512).double() * sc.double()[:, None] + sh.double()[:, None]).float().clamp_min(0).transpose(1, 2)
    swapped = good.clone()
    for c0 in range(0, 512, 32):
        for l0 in range(0, L2, 32):
            n = min(32, L2 - l0)
            swapped[:, c0:c0 + n, l0:l0 + n] = good[:, c0:c0 + n, l0:l0 + n].transpose(1, 2)
    out["out fp32"] = worst_ratio(good, ref, T)
    out["out l/c swapped"] = worst_ratio(swapped, ref, T)
    report("planted defects (err / bound)", **out)
    assert max(out["l1 fp32"], out["mean fp32"], out["head fp32"], out["conv2 fp32"], out["out fp32"]) <= 1.0, out
    assert min(out["l1 next pair"], out["mean / (n+1)"], out["head neighbour U"], out["conv2 16 per group"],
               out["out l/c swapped"]) > 10.0, out
