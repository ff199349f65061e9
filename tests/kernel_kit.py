"""Shared machinery of the kernel-level fp64 tests: ctypes plumbing, the library's process-wide knobs, NaN-filled
buffers and stage workspaces, seeds and report lines, the error bounds more than one test module uses, and the runner
and checks of the generated-operand tensor-core engine.  (tests/helpers.py holds the golden and oracle helpers of the
end-to-end tests.)

Nothing here needs a GPU to import; the helpers that allocate do so on cuda.
"""
import contextlib
import ctypes
import math
import os
import re
import zlib

import numpy as np
import torch

from mmmot_b200.weights import pack_tc

U = 2.0 ** -24                     # fp32 unit roundoff
TINY = 2.0 ** -126                 # smallest normal fp32
EPS = 1e-5                         # GroupNorm / BatchNorm epsilon
# TAU = 2^-18, the tensor-core contractions' bound |y - y_ref| <= TAU S, S = |W| A + |b| (A the magnitude of the operand
# the producer forms): with the fp32 accumulator truncating at every K=16 step, about 216 roundings per 36-chunk K
# segment with random-sign partial sums give ~1e-6 S at K = 4608.  Measured on an H100 80GB HBM3 (400 W power limit):
# the worst err / (TAU S) of the VGG convolutions over all cases is 0.51 (K = 4608 in one pass), 0.28 over the product's
# plans.
TAU = 2.0 ** -18
KAPPA, KAPPA1 = 64, 40             # the GroupNorm statistics bound of stats_ratios
FP64 = 2.0 ** -40                  # fp64 summation and cancellation, far below every other term of a bound
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mmmot_b200", "csrc")
KSEG_DEFAULT = 36                  # mmmot_set_kseg default (api.cu)
ENGINE = {"auto": 0, "fp32": 1, "tc": 2}
NAN_GUARD = 256                    # NaN elements after every output buffer of nan_output
BN = 256                           # column tile of the tensor-core contractions
GUARD_ROWS = 64                    # rows of NaN after every output buffer of run_gen


class GEN:
    """Producer ids of the generated-operand engine (gen::GEN_*, mmmot_debug_gen)."""
    MUL, ABS, SUB, NORM, COPY = range(5)
    NAMES = ("mul", "abs", "sub", "norm", "copy")


class XM:
    """Operand modes of the FP32 FFMA engine (XM_*, mmmot_debug_simt_op)."""
    DIRECT, NORM, MUL, ABS, SUB, CONV = range(6)


def vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def case_seed(*key):
    """A generator seed from a case's key (stable across runs and machines)."""
    return zlib.crc32(repr(key).encode())


def report(name, **ratios):
    """One line of err / bound figures, printed under -s."""
    print(f"\n{name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()), end="")


# ------------------------------------------------------------------------------------------------ library state
@contextlib.contextmanager
def lib_state(lib, engine="auto", dbg=0, kseg=None):
    """Sets the library's process-wide knobs for the body: the contraction engine (a key of ENGINE), the debug bits and
    the K-segment length (None: the default).  Restores the defaults of all three whatever happens, so that no test
    leaks a knob into the tests after it."""
    try:
        assert lib.mmmot_set_engine(ENGINE[engine]) == 0
        assert lib.mmmot_set_debug(dbg) == 0
        assert lib.mmmot_set_kseg(KSEG_DEFAULT if kseg is None else kseg) == 0
        yield
    finally:
        lib.mmmot_set_engine(0)
        lib.mmmot_set_debug(0)
        lib.mmmot_set_kseg(KSEG_DEFAULT)


def eval_net(fusion, seed, edit=None, **kw):
    """TrackingNet(2) with the SkipPool appearance heads and score fusion `fusion`, loaded with the synthetic weights of
    `seed` (after edit(state dict), if given), on the GPU in eval mode; kw: further TrackingNet arguments.
    -> (net, state dict)."""
    import mmmot_b200
    from mmmot_b200.synthetic import synthetic_state_dict
    sd = synthetic_state_dict(fusion, seed=seed)
    if edit is not None:
        edit(sd)
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch=fusion, test_mode=2,
                                 dropblock=0, **kw)
    net.load_state_dict(sd)
    return net.cuda().eval(), sd


# ------------------------------------------------------------------------------------------------ buffers
def fp16_split(x):
    """fp32 -> the FP16 (hi, lo) pair of the tensor-core operands: hi = fl16(x), lo = fl16(x - hi)."""
    hi = x.half()
    return hi, (x - hi.float()).half()


def fp16_planes(x):
    """fp32 -> the planes [2][...] (hi, lo) of fp16_split, contiguous."""
    return torch.stack(fp16_split(x)).contiguous()


def nan_output(rows, *cols, guard=NAN_GUARD):
    """An fp32 output buffer [rows + guard][*cols] on the GPU, every element NaN: the `guard` rows past the end must
    come back NaN."""
    return torch.full((rows + guard, *cols), float("nan"), device="cuda")


def assert_written(buf, count, what):
    """The first `count` elements of a nan_output buffer are written (finite), the guard band after them is not."""
    assert bool(torch.isfinite(buf[:count]).all()), f"{what}: an owned element was not written"
    assert bool(torch.isnan(buf[count:]).all()), f"{what}: written past its end"


def nan_workspace(lib, nbytes):
    """A stage workspace of nbytes whose every float and double is NaN (0xFF bytes), its status block reset."""
    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda")
    assert lib.mmmot_status_reset(vp(ws), None) == 0
    return ws


# Buffers of mmmot_debug_stage_layout, in the header's order: stage 0 = mmmot_affinity_fwd, 1 = mmmot_fusion_det_fwd,
# 2 = mmmot_pointnet_fwd (its last entry, `end`, is the workspace size).
AF_BUFS = ("y01", "y3", "z", "fcl", "sc0", "sh0", "sc3", "sh3", "v", "h2", "nsc2", "nsh2", "rmax", "rsum", "cmax", "csum",
           "y2", "sc1", "sh1", "sc2", "sh2", "h1", "nsc1", "nsh1", "stats", "nstats", "part", "npart", "tiles", "cnt",
           "gstart")
FD_BUFS = ("f3", "h2")
PN_BUFS = ("xt", "y1", "t0", "t1", "big", "segsum", "x1p", "xp", "gmean", "u", "ut", "hmean", "o", "sc1", "sh1", "sc",
           "sh", "stats", "mom", "part", "gstart", "sstart", "seg", "cnt", "tiles", "ctab", "end")
STAGE_BUFS = (AF_BUFS, FD_BUFS, PN_BUFS)


def stage_layout(lib, stage, pairs, n, m=0):
    """mmmot_debug_stage_layout -> ({buffer: byte offset}, tensor-core path?)."""
    off = (ctypes.c_size_t * 32)()
    tc = ctypes.c_int(-1)
    assert lib.mmmot_debug_stage_layout(stage, pairs, n, m, off, ctypes.byref(tc)) == 0
    return {k: int(off[i]) for i, k in enumerate(STAGE_BUFS[stage])}, bool(tc.value)


class Workspace:
    """Typed views of one stage run's nan_workspace at the offsets stage_layout reports."""

    def __init__(self, ws, lay):
        self.ws, self.lay = ws, lay

    def view(self, name, count, dtype=torch.float32):
        off = self.lay[name]
        nbytes = count * torch.empty(0, dtype=dtype).element_size()
        return self.ws[off:off + nbytes].view(dtype)

    def untouched_after(self, name, nbytes):
        """The bytes of buffer `name` past its first nbytes, up to the next buffer (or the workspace's end), still hold
        the 0xFF fill."""
        off = self.lay[name]
        nxt = min((v for v in self.lay.values() if v > off), default=self.ws.numel())
        return bool((self.ws[off + nbytes:nxt] == 255).all())

    def owned(self, name, count, dtype=torch.float32):
        """The first `count` elements of buffer `name`, all written (finite), the rest of the buffer untouched."""
        v = self.view(name, count, dtype)
        finite = torch.isfinite(v.float() if dtype == torch.float16 else v)
        assert bool(finite.all()), f"{name}: an owned element was not written"
        assert self.untouched_after(name, v.numel() * v.element_size()), f"{name}: written past its end"
        return v


# ------------------------------------------------------------------------------------------------ bounds
def worst_ratio(got, ref, T):
    """max |got - ref| / T, an exact match counting 0 wherever T is."""
    err = (got.double() - ref).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / T).max())


def contraction_bound(wt, xin, bias=None, add=None, relu=False, chunk=1 << 25):
    """fp64 reference and error bound of the FP32 FFMA engine's outputs (csrc/gemm_simt.cuh).  wt [K][M] and xin [K][C]
    hold fp32 values as fp64, bias [M] or None, add [M][C] the addend of each output or None.  Chunked over the columns,
    on the inputs' device.  -> (y64 [M][C], T [M][C]).

    Output (co, c) is the sequential chain acc = fma(w_k, x_k, acc) over k = 0..K-1, then + bias, + addend and ReLU,
    each an fp32 rounding.  With u = 2^-24 and s_k the fp64 prefix sum of w_j x_j, j <= k, in that order, the rounding of
    step k is at most u |s_k| to first order, so
        |y - y64| <= 1.01 u (sum_k |s_k| + |s_K + b| + |y^| [addend]) + u sum_k |w_k x_k|,
    y^ the value after the addend.  The factor 1.01 covers the second-order terms (K u < 10^-3 here); the last term
    covers the rare double rounding of the fp64 emulation of fma in the NORM_RELU operand.  ReLU is 1-Lipschitz.  The
    bound is derived, not measured: no case needs a looser constant.  On random data sum_k |s_k| grows like K^1.5 while
    one term of the chain is of order 1/K of it at most, so a single dropped or wrong tap at K = 4608 misses the bound by
    far more than an order of magnitude (test_simt_engine.py's CPU self-test shows it with an fp32 emulation of the
    kernel's arithmetic)."""
    K, M = wt.shape
    C = xin.shape[1]
    y = torch.empty(M, C, dtype=torch.float64, device=xin.device)
    T = torch.empty_like(y)
    step = max(1, chunk // (K * M))
    for c0 in range(0, C, step):
        c1 = min(C, c0 + step)
        prod = wt[:, :, None] * xin[:, None, c0:c1]          # [K][M][c], exact in fp64
        t = U * prod.abs().sum(0)
        prod.cumsum_(0)
        s = prod[-1] + (0.0 if bias is None else bias[:, None])
        acc = prod.abs_().sum(0) + s.abs()
        if add is not None:
            s = s + add[:, c0:c1]
            acc += s.abs()
        T[:, c0:c1] = 1.01 * U * acc + t
        y[:, c0:c1] = s.clamp_min(0) if relu else s
    return y, T


def norm_operand(v, sc, sh):
    """relu(fmaf(v, sc, sh)) in fp32: the product of two fp32 values is exact in fp64, the add rounds once, then to fp32."""
    return (v.double() * sc.double() + sh.double()).float().clamp_min(0)


def pair_operand(f, op, n, m):
    """f [G][K][Lf] fp32 -> the FP32 engine's pairwise operand [K][G*n*m] (XM.MUL / ABS / SUB), column g*n*m + i*m + j
    from object i and detection n + j, formed in fp32 as the engine's loader forms it."""
    s = torch.arange(n * m, device=f.device)
    a, b = f[:, :, s // m], f[:, :, n + s % m]
    x = a * b if op == XM.MUL else (a - b) * 0.5
    if op == XM.ABS:
        x = x.abs()
    return x.permute(1, 0, 2).reshape(f.shape[1], -1)


def ref_linear(X, A, wt, b):
    """fp64 X W^T + b and S = A |W|^T + |b| (X, A [cols][K] fp64, on their device): the reference and scale of the TAU
    bound."""
    w = wt.double().to(X.device)
    bb = b.double().to(X.device)
    return X @ w + bb, A @ w.abs() + bb.abs()


def group_moments(y, grp, G):
    """Two-pass fp64 over y [cols][M] (fp64) grouped by grp [cols] -> count, mean, var, mean|delta|, mean|y|."""
    acc = lambda v: torch.zeros(G, y.shape[1], dtype=torch.float64, device=y.device).index_add_(0, grp, v)
    n = torch.bincount(grp, minlength=G).double()[:, None]
    mean = acc(y) / n
    dev = y - mean[grp]
    return n, mean, acc(dev * dev) / n, acc(dev.abs()) / n, acc(y.abs()) / n


def stats_ratios(S1, S2, y, grp, G):
    """gn_finalize's mean and var from the fp64 group sums (S1, S2) [G][M] of a contraction epilogue's partials against
    the two-pass values over y: -> (worst dvar / bound, worst dmean / bound, largest |mean| / std over the channels).

    The epilogues sum their outputs per channel in fp32 runs (32 columns of a tensor-core epilogue thread, the 8 columns
    of an FP32-engine thread) as differences from the run's fp32 mean, each run folded into the fp64 partial exactly
    (stat_fold in common.cuh).  With u = 2^-24, ybar, delta = y - ybar, and run c of k <= 32 valid columns with pivot p_c
    (its fp32 mean):
        d = fl(y - p_c) carries u|d|; sum d takes k - 1 further roundings, sum d^2 k fma roundings, so in the worst case
        |e1_c| <= 32 u sum_c |d|  and  |e2_c| <= 34 u sum_c d^2.
      The fold (k p + s1, k p^2 + 2 p s1 + s2) is fp64, as are stats_reduce and gn_finalize: each adds a relative 2^-53
      of n (ybar^2 + var), below 2^-29 u (R^2 + 1) var -- invisible up to R = 10^4.  To first order
        dvar = (1/n) sum_c [2 (p_c - ybar) e1_c + e2_c],      dmean = (1/n) sum_c e1_c,
      with |d| <= |delta| + |p_c - ybar|.  A worst-case bound from this needs the largest deviation of a run's mean from
      the group's, which structured data can make several std, and would be several times the var term below.  The
      statistics are instead held to
        |dvar| <= KAPPA u (|ybar| mean|delta| + mean delta^2),   |dmean| <= KAPPA1 u mean|y|,   KAPPA = 64, KAPPA1 = 40,
      constants set from the rounding counts above (2 x 32 for the cross term, about 36 roundings for a run's sum) on the
      argument that the k roundings of a run are independent, so their sum grows like sqrt(k) and stays well below the
      coherent worst case.  They are empirical in that sense, not proven; what they rest on is measured by
      test_norm_stats.py (an emulation of the gemm_gen epilogue's summation order on the CPU, and the GPU cases).  (A
      pivot taken from the run's values, its first say, fails this bound at R = 1 once ReLU zeros surround a rare
      positive pivot.)  The bound is linear in R = |ybar|/std; the unshifted sums err by about sqrt(k) u ybar^2, R / KAPPA
      times its first term, and the bound rejects them at R >= 100."""
    n, mean, var, mad, may = group_moments(y, grp, G)
    keep = n[:, 0] > 0
    m = S1 / n
    v = S2 / n - m * m
    tv = KAPPA * U * (mean.abs() * mad + var)
    tm = KAPPA1 * U * may
    rv = ((v - var).abs() / tv.clamp_min(1e-300))[keep]
    rm = ((m - mean).abs() / tm.clamp_min(1e-300))[keep]
    cond = (mean.abs() / var.clamp_min(1e-300).sqrt())[keep]
    return float(rv.max()), float(rm.max()), float(cond.max())


def group_sum(v, idx, G):
    """Rows of v [n][C] summed in fp64 into their groups idx [n] -> [G][C]."""
    return torch.zeros(G, v.shape[1], dtype=torch.float64, device=v.device).index_add_(0, idx, v)


def gn_stats(y, grp, G, T=None, kappa=True, cpg=1):
    """GroupNorm statistics per group of y [n][C] (fp64 reference of the values the kernel summed, which err by at most
    T), normalisation groups of cpg adjacent channels -> (mean, var, tm, tv) [G][C], each channel carrying its
    normalisation group's values.

    Per channel the kernel's mean and variance differ from the two-pass fp64 values by at most
        tm = mean(T) + [KAPPA1 u mean|y|] + FP64 mean|y|,
        tv = 2 mean(|y - mean| T) + mean(T^2) + [KAPPA u (|mean| mean|y - mean| + var)] + FP64 (mean^2 + var),
    the bracketed terms (kappa) only where the sums come from a contraction epilogue's fp32 runs (stats_ratios).
    gn_finalize adds the cpg channel sums of a normalisation group in fp64.  Every channel has the same count, so the
    group's mean M is the mean over its channels of the channel means m_c and its variance is
    mean_c [v_c + (m_c - M)^2].  With the channel errors dm_c, dv_c:
        dM = mean_c dm_c,    dV = mean_c [dv_c + 2 (m_c - M) dm_c] + (mean_c dm_c^2 - (mean_c dm_c)^2),
    the last bracket in [0, mean_c dm_c^2], so
        tm_G = mean_c tm_c,  tv_G = mean_c [tv_c + 2 |m_c - M| tm_c + tm_c^2].
    The channels' FP64 (m_c^2 + v_c) average to FP64 (M^2 + V), which also covers the fp64 sums over the cpg channels."""
    n, mean, var, mad, may = group_moments(y, grp, G)
    tm = FP64 * may
    tv = FP64 * (mean * mean + var)
    if kappa:
        tm = tm + KAPPA1 * U * may
        tv = tv + KAPPA * U * (mean.abs() * mad + var)
    if T is not None:
        dev = y - mean[grp]
        tm = tm + group_sum(T, grp, G) / n
        tv = tv + (2 * group_sum(dev.abs() * T, grp, G) + group_sum(T * T, grp, G)) / n
    if cpg == 1:
        return mean, var, tm, tv
    C = y.shape[1]
    per = lambda v: v.view(G, C // cpg, cpg)
    wide = lambda v: v.repeat_interleave(cpg, 1)
    M = per(mean).mean(2, keepdim=True)
    V = (per(var) + (per(mean) - M) ** 2).mean(2)
    TV = (per(tv) + 2 * (per(mean) - M).abs() * per(tm) + per(tm) ** 2).mean(2)
    return wide(M[..., 0]), wide(V), wide(per(tm).mean(2)), wide(TV)


def gn_apply(y, T, grp, st, gamma, beta):
    """fmaf(y, sc, sh) of a kernel's GroupNorm before the ReLU, from y [n][C] that errs by at most T (None: exact) and
    the statistics st of gn_stats -> (z [n][C], Tz, |y a| + |sh|).

    With a = gamma / sqrt(var + eps), sh = beta - mean a, sc_k = fl(a_k), sh_k = fl(beta - mean_k a_k) and
    |a_k - a| <= |a| er, er = tv / (2 (var + eps)) + FP64, the value errs before the ReLU (1-Lipschitz) by
        Tz = |a| (T + tm + |y - mean| er) + 8u (|y a| + |sh| + |z|),
    the last term the fp32 roundings of sc, sh and the fma; |y a| ~ |mean| / std is GroupNorm's own conditioning."""
    mean, var, tm, tv = st
    a = gamma / torch.sqrt(var + EPS)
    sh = beta - mean * a
    er = tv / (2 * (var + EPS)) + FP64
    A, SH = a[grp], sh[grp]
    z = y * A + SH
    Tz = A.abs() * ((0.0 if T is None else T) + tm[grp] + (y - mean[grp]).abs() * er[grp])
    mag = (y * A).abs() + SH.abs()
    return z, Tz + 8 * U * (mag + z.abs()), mag


def affine_bound(st, gamma, beta):
    """gn_finalize's fp32 sc / sh from statistics whose mean and variance err by at most (tm, tv) of st = gn_stats(...)
    -> (a, sh, Ta, Tsh) [G][C]: the fp64 affine of the reference statistics and the bounds
        |sc - a| <= |a| (er + u),   |sh - sh_ref| <= |a| tm + |mean a| er + u (|sh| + |mean a|),
    er = tv / (2 (var + eps)) + FP64 (the relative error of 1 / sqrt(var + eps)), u the final fp32 rounding."""
    mean, var, tm, tv = st
    a = gamma / torch.sqrt(var + EPS)
    er = tv / (2 * (var + EPS)) + FP64
    sh = beta - mean * a
    ma = (mean * a).abs()
    return a, sh, a.abs() * (er + U), a.abs() * tm + ma * er + U * (sh.abs() + ma)


def gn_affine(stats, gamma, beta, count, cpg=1):
    """gn_finalize of GroupNorm(C / cpg, C) from the stored fp64 stats [G][C][2] (sum, sum of squares) over `count`
    columns per group (a number, or a tensor [G]) -> (sc, sh, Tsc, Tsh) [G][C]: fp64 from the stored sums, the kernel
    then rounds each once to fp32 (u |sc|, u |sh|); its fp64 arithmetic adds FP64 |a| (mean^2 + var) / (var + eps) and
    likewise for sh."""
    G, C = stats.shape[:2]
    s = stats.view(G, C // cpg, cpg, 2).sum(2)
    n = (count.double().view(G, 1) if torch.is_tensor(count) else float(count)) * cpg
    mean = s[..., 0] / n
    var = (s[..., 1] / n - mean * mean).clamp_min(0)
    mean, var = mean.repeat_interleave(cpg, 1), var.repeat_interleave(cpg, 1)
    a = gamma / torch.sqrt(var + EPS)
    sh = beta - mean * a
    cond = (mean * mean + var) / (var + EPS)
    return a, sh, U * a.abs() + FP64 * a.abs() * cond, U * sh.abs() + FP64 * (mean * a).abs() * (1 + cond)


def reduce_parts(part, slot_group, G):
    """Partials [slots][M][2] (sum, sum of squares) summed in fp64 into their groups -> (S1, S2) [G][M]."""
    M = part.shape[1]
    acc = lambda v: torch.zeros(G, M, dtype=torch.float64, device="cuda").index_add_(0, slot_group, v)
    return acc(part[:, :, 0]), acc(part[:, :, 1])


# ------------------------------------------------------------------------------------------------ tile tables
class Cols:
    """The columns (operand rows) of one generated-operand launch in a fixed order: per column its output row, source
    row, group and partial slot tile*2 + half; plus the tile table (table tiling) and the tile count."""

    def __init__(self, y_row, src_row, grp, hid, ntiles, tiles=None):
        self.y_row, self.src_row, self.grp, self.hid = (torch.tensor(v, dtype=torch.long) for v in (y_row, src_row, grp, hid))
        self.ntiles, self.tiles = ntiles, tiles

    @staticmethod
    def uniform(S, groups, x_gs, y_gs):
        y, s, g, h = [], [], [], []
        tpg = math.ceil(S / BN)
        for gi in range(groups):
            c = np.arange(S)
            y.append(gi * y_gs + c); s.append(gi * x_gs + c); g.append(np.full(S, gi))
            h.append((gi * tpg + c // BN) * 2 + (c % BN) // 128)
        return Cols(*(np.concatenate(v) for v in (y, s, g, h)), tpg * groups)

    @staticmethod
    def table(tiles):
        """tiles: list of (group, first absolute row, length)."""
        y, g, h = [], [], []
        for t, (gi, r0, ln) in enumerate(tiles):
            c = np.arange(ln)
            y.append(r0 + c); g.append(np.full(ln, gi)); h.append(t * 2 + c // 128)
        y = np.concatenate(y)
        tt = torch.tensor([[gi, r0, ln, 0] for gi, r0, ln in tiles], dtype=torch.int32)
        return Cols(y, y, np.concatenate(g), np.concatenate(h), len(tiles), tt)


def pn_tiles_host(split, pairs, L):
    """PointNet's tensor-core tile table on the host: (pair, first point, length <= BN) over each pair's points."""
    return [(p, c, min(BN, split[(p + 1) * L] - c)) for p in range(pairs) for c in range(split[p * L], split[(p + 1) * L], BN)]


def pn_host_tables(split, pairs, L):
    """Every table PointNet's tensor-core trunk builds, on the host: tiles, point -> detection map, chunk descriptors,
    points per pair and first tile of each pair."""
    P = split[-1]
    seg = np.zeros(P, dtype=np.int64)
    for d in range(pairs * L):
        seg[split[d]:split[d + 1]] = d
    tiles = pn_tiles_host(split, pairs, L)
    ctab = []
    for _, c0, ln in tiles:
        for half in range(2):
            v = []
            for c in range(4):
                col0 = half * 128 + c * 32
                if col0 >= ln:
                    v.append(0)
                    continue
                first, last = seg[c0 + col0], seg[c0 + min(col0 + 31, ln - 1)]
                v.append(int(first) << 1 | int(col0 + 32 <= ln and first == last))
            ctab.append(v)
    cnt = [split[(p + 1) * L] - split[p * L] for p in range(pairs)]
    gstart = np.concatenate([[0], np.cumsum([math.ceil(c / BN) for c in cnt])]).tolist()
    return tiles, seg, ctab, cnt, gstart


def ne_tiles_host(G, n, m, gap, tw=BN):
    """The new/end MLP's table (affinity.cu ne_tiles_kernel) in tiles of tw columns (BN on the tensor cores, 128 on the
    FP32 engine): group 2g = the m new columns, 2g+1 = the n end columns of pair-stack g, here with `gap` unused rows
    after every g."""
    tiles = []
    for g in range(G):
        base = g * (n + m + gap)
        tiles += [(2 * g, base + c, min(tw, m - c)) for c in range(0, m, tw)]
        tiles += [(2 * g + 1, base + m + c, min(tw, n - c)) for c in range(0, n, tw)]
    return tiles, G * (n + m + gap)


def ne_table(G=80, n=100, m=37):
    """-> (tiles, rows, groups) of a new/end MLP launch over G pair-stacks of n objects and m detections."""
    tiles, rows = ne_tiles_host(G, n, m, 5)
    return tiles, rows, 2 * G


def _layouts():
    edges = [32, 96, 128, 1, 1, 1, 29, 300, 40, 17, 5, 64, 1, 33, 7, 50]
    two = [100, 28, 128, 1, 1, 1, 1, 60, 100, 50, 40, 30, 50, 20, 30, 60] + \
          [5, 27, 64, 256, 3, 1, 1, 1, 90, 33, 31, 70, 12, 200, 9, 100]
    g = torch.Generator().manual_seed(5)
    three = torch.randint(1, 80, (60,), generator=g)
    three[10:15] = 1
    six = torch.randint(1, 200, (192,), generator=g)
    six[40:44] = 1
    return {"edges": (1, 16, edges), "two": (2, 16, two), "three": (3, 20, three.tolist()), "six": (6, 32, six.tolist())}


# PointNet point layouts (pairs, L, counts per detection).  edges: detection boundaries exactly at 32, 128 and 256, three
# one-point detections inside one chunk, a 300-point detection across a tile edge, a total (805) that ends mid-box.
# two: pair 0 ends at 700 (not a multiple of 256, its last 32-column chunk partial and inside one detection) and is
# followed by pair 1.  three / six: seeded ragged counts, with runs of one-point detections.
LAYOUTS = _layouts()


def bench_n_imgs(pairs, L):
    """Image counts forward_batch can launch for `pairs` frame-pairs of L detections: its chunk size halves from the
    whole batch until the workspace fits the free memory, so every size of that chain (and its remainder) can occur."""
    sizes, c = {pairs}, pairs
    while c > 1:
        c = (c + 1) // 2
        sizes.add(c)
    chunks = set()
    for c in sizes:
        chunks.add(c)
        if pairs % c:
            chunks.add(pairs % c)
    return sorted(k * L for k in chunks)


# ------------------------------------------------------------------------------------------------ launch sites
def impl_launches(src_file, func, helpers):
    """(name) of every `kernel<<<` launch and every call of one of `helpers` (regular expressions of function names) in
    the body of the function func of csrc/src_file, in source order, comments skipped."""
    src = open(os.path.join(CSRC, src_file)).read()
    defs = list(re.finditer(rf'^(?:static |extern "C" )?int {func}\([^;{{]*\)\s*{{', src, re.M))
    assert len(defs) == 1, (func, len(defs))
    body = src[defs[0].end():src.index("\n}\n", defs[0].end())]
    body = re.sub(r"//[^\n]*", "", body)
    pat = rf"\b(\w+)(?:<[^<>;()]*>)?<<<|\b({'|'.join(helpers)})\s*[<(]"
    return [m.group(1) or m.group(2) for m in re.finditer(pat, body)]


# ------------------------------------------------------------------------------------------------ generated-operand engine
def gen_weights(g, K, M, scale=1.0):
    """Wt [K][M], bias [M] and the packed tensor-core tiles of W -> (wt, b, Wp, wp_scale)."""
    wt = torch.randn(K, M, generator=g) * K ** -0.5 * scale
    b = torch.randn(M, generator=g) * 0.2
    Wp, wps = pack_tc(wt)
    return wt, b, Wp, wps


def check_rows(Y, cols, ref, S, relu=False):
    """Y [rows + guard][M]: the columns' rows against ref / S (fp64, cuda, column order); every other row still NaN.
    -> worst err / (TAU S)."""
    written = torch.zeros(Y.shape[0], dtype=torch.bool, device="cuda")
    yr = cols.y_row.cuda()
    written[yr] = True
    stray = torch.isfinite(Y[~written]).any(dim=1)
    assert not bool(stray.any()), f"{int(stray.sum())} rows written outside the launch's columns"
    y = Y[yr].double()
    assert bool(torch.isfinite(y).all()), f"{int((~torch.isfinite(y)).sum())} output elements never written"
    if relu:
        ref = torch.relu(ref)
    return float(((y - ref).abs() / (TAU * S)).max())


def check_part(part, cols, ref, S):
    """GroupNorm partials part[tile*2 + half][co] = (sum, sum of squares) of the half-tile's valid columns against fp64
    sums of y_ref.  Each y carries |e| <= TAU S; the kernel sums a thread's 32-column chunks sequentially in fp32 and
    adds the four chunk sums (36 roundings, each <= 2^-24 of a partial sum <= sum |y|), hence 64 2^-24 sum|y| (and
    sum y^2 for the squares, whose element error is <= 2|y| TAU S + (TAU S)^2).  Half-tiles without columns must be 0."""
    hid = cols.hid.cuda()
    nslot = cols.ntiles * 2
    M = ref.shape[1]
    acc = lambda v: torch.zeros(nslot, M, dtype=torch.float64, device="cuda").index_add_(0, hid, v)
    e = TAU * S
    want1, want2 = acc(ref), acc(ref * ref)
    tol1 = acc(e) + 64 * 2.0 ** -24 * acc(ref.abs())
    tol2 = acc(2 * ref.abs() * e + e * e) + 64 * 2.0 ** -24 * want2
    got = part[:nslot]
    assert bool(torch.isfinite(got).all()), "partials not written"
    # an empty half-tile has tolerance 0: any nonzero value there gives a huge ratio
    w1 = float(((got[..., 0] - want1).abs() / tol1.clamp_min(1e-300)).max())
    w2 = float(((got[..., 1] - want2).abs() / tol2.clamp_min(1e-300)).max())
    assert w1 <= 1.0 and w2 <= 1.0, (w1, w2)
    assert bool(torch.isnan(part[nslot:]).all()), "partials written past the launch's tiles"
    return max(w1, w2)


def run_gen(lib, gen, wt, b, Wp, wps, src, cols, y_rows, *, ld_src=0, gsc=None, gsh=None, n=0, m=0, Lf=0, S=0, groups=0,
            x_gs=0, y_gs=0, relu=0, part=True, dbg=0):
    """One mmmot_debug_gen launch over `cols` into NaN-filled outputs -> (Y [y_rows + GUARD_ROWS][M], partials or None,
    the producer variant taken)."""
    K, M = wt.shape
    Y = nan_output(y_rows, M, guard=GUARD_ROWS)
    P = torch.full((cols.ntiles * 2 + 4, M, 2), float("nan"), dtype=torch.float64, device="cuda") if part else None
    tiles = None if cols.tiles is None else cols.tiles.cuda()
    pref = ctypes.c_int(-1)
    keep = (Wp.cuda(), b.cuda())
    with lib_state(lib, dbg=dbg):
        want = lib.mmmot_debug_gen_prefetch(gen, m)
        rc = lib.mmmot_debug_gen(gen, M, K, vp(keep[0]), wps, vp(keep[1]), relu, vp(src), ld_src, vp(gsc), vp(gsh), n, m, Lf,
                                 S, groups, x_gs, y_gs, vp(tiles), cols.ntiles if tiles is not None else 0, vp(Y), M, vp(P),
                                 ctypes.byref(pref), None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    assert pref.value == want, (pref.value, want)
    return Y, P, pref.value
