"""GroupNorm statistics of PointNet's two widest tensor-core layers (128 -> 1024 and the 64 -> 512 head) from the moments
of their input (csrc/pointnet.cu, pnm), run through the product's launch code (mmmot_debug_pn_stats).

Moments: S2 = sum x x^T, S1 = sum x per pair and, for the head, the per-detection sums of x, against fp64 over the
exact inputs x = hi + lo.  S2 is bounded element by element by 2^-18 (|X|^T |X|): per 256-point tile the fp32
accumulator takes 16 k-steps x 3 MMAs (hi hi, hi lo, lo hi), each truncating once by < 2^-23 of a running sum that is at
most k/16 of the tile's sum of |x_i x_j|, so at most 3 * 8.5 * 2^-23 = 2^-18.3 of it; the dropped lo lo term adds
<= 2^-22, and the fp64 sums over tiles add nothing visible.  S1 is summed in fp64 (2^-40 bound), the per-detection
sums in 2^-32 fixed point (each value rounded once: n_d 2^-33).

Statistics: sc / sh of GroupNorm(M, M) per pair against fp64 y = x Wt + b (+ U[det]) on the host, on the default path
and on the statistics-only contraction of debug bit 4.  One output channel has |mean| / std >= 30: its variance is
exact in the centred form of the moments path, while the bit-4 path sums y^2 in fp32 and loses about mean^2 / var of
relative accuracy there (reported, not asserted).

Determinism: the same batch twice is bit-identical, and a pair's statistics and PointNet features are bit-identical
whether it runs alone or inside a larger batch.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from kernel_kit import LAYOUTS, eval_net, fp16_split, lib_state, report, vp
from mmmot_b200 import _lib
from mmmot_b200.weights import pack_tc

gpu = pytest.mark.gpu
TWO_PASS = 16                      # mmmot_set_debug bit 4
PTXAS_LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mmmot_b200", "csrc", "build",
                         "pointnet.ptxas.log")
# the matrix-mode layouts of kernel_kit.LAYOUTS, plus pairs of very different sizes: 11200 points (two 32-tile
# slices, the second partial) between pairs of 16 one-point detections and of 16 x 37 points
MOM_LAYOUTS = dict(LAYOUTS, skew=(3, 16, [1] * 16 + [700] * 16 + [37] * 16))


def _inputs(layout, K, seed):
    pairs, L, counts = MOM_LAYOUTS[layout]
    split = [0] + np.cumsum(counts).tolist()
    P = split[-1]
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(P, K, generator=g) + 0.3)     # post-ReLU-like activations, many exact zeros
    hi, lo = fp16_split(x)
    return pairs, L, split, hi, lo, g


def _run(lib, pairs, L, split, hi, lo, K, M, wt, b, add, gamma, beta, dbg=0):
    P = split[-1]
    d_split = torch.tensor(split, dtype=torch.int32, device="cuda")
    h_split = torch.tensor(split, dtype=torch.int32)
    X = torch.stack([hi, lo]).contiguous().cuda()
    Wp, wps = pack_tc(wt)
    ws = torch.empty(int(lib.mmmot_pointnet_workspace(pairs, L, P)), dtype=torch.uint8, device="cuda")
    sc = torch.full((pairs, M), float("nan"), device="cuda")
    sh = torch.full((pairs, M), float("nan"), device="cuda")
    stats = torch.full((pairs, M, 2), float("nan"), dtype=torch.float64, device="cuda")
    mom = torch.full((pairs, K * K + K), float("nan"), dtype=torch.float64, device="cuda")
    det = torch.zeros((pairs * L, 64), dtype=torch.int64, device="cuda") if K == 64 else None
    keep = [t.cuda() if t is not None else None for t in (wt, Wp, b, add, gamma, beta)]
    with lib_state(lib, dbg=dbg):
        rc = lib.mmmot_debug_pn_stats(vp(d_split), vp(h_split), pairs, L, vp(X), K, vp(keep[0]), vp(keep[1]), wps,
                                      vp(keep[2]), M, vp(keep[3]), vp(keep[4]), vp(keep[5]), vp(sc), vp(sh), vp(stats),
                                      vp(mom), vp(det), vp(ws), ws.numel(), None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    return dict(sc=sc.cpu(), sh=sh.cpu(), stats=stats.cpu(), mom=mom.cpu(), det=None if det is None else det.cpu())


def _layer(K, g, heavy):
    M = 1024 if K == 128 else 512
    wt = torch.randn(K, M, generator=g) * K ** -0.5
    b = torch.randn(M, generator=g) * 0.2
    b[heavy] = 0.0
    gamma = torch.rand(M, generator=g) + 0.5
    beta = torch.randn(M, generator=g) * 0.3
    return M, wt, b, gamma, beta


# ------------------------------------------------------------------------------------------------ moments
@gpu
@pytest.mark.parametrize("layout,K", [(lay, K) for lay in MOM_LAYOUTS for K in (64, 128)])
def test_moments_vs_fp64(layout, K):
    lib = _lib.load()
    pairs, L, split, hi, lo, g = _inputs(layout, K, seed=len(MOM_LAYOUTS[layout][2]) + K)
    M, wt, b, gamma, beta = _layer(K, g, 0)
    add = torch.randn(pairs * L, M, generator=g) * 0.5 if K == 64 else None
    out = _run(lib, pairs, L, split, hi, lo, K, M, wt, b, add, gamma, beta)
    x = hi.double() + lo.double()
    res = {}
    for p in range(pairs):
        xp = x[split[p * L]:split[(p + 1) * L]]
        S2 = xp.t() @ xp
        A = xp.abs().t() @ xp.abs()
        got = out["mom"][p]
        e2 = float(((got[:K * K].view(K, K) - S2).abs() / (2.0 ** -18 * A).clamp_min(1e-300)).max())
        e1 = float(((got[K * K:] - xp.sum(0)).abs() / (2.0 ** -40 * xp.abs().sum(0)).clamp_min(1e-300)).max())
        res[f"S2_p{p}"], res[f"S1_p{p}"] = e2, e1
        assert e2 <= 1.0 and e1 <= 1.0, (p, e2, e1)
    if K == 64:
        seg = np.repeat(np.arange(pairs * L), np.diff(split))
        want = torch.zeros(pairs * L, 64, dtype=torch.float64).index_add_(0, torch.tensor(seg), x)
        n_d = torch.tensor(np.diff(split), dtype=torch.float64)[:, None]
        got = out["det"].double() * 2.0 ** -32
        e = float(((got - want).abs() / (n_d * 2.0 ** -33 + 2.0 ** -40 * want.abs())).max())
        res["det"] = e
        assert e <= 1.0, e
    report(f"moments {layout} K={K}", **res)


# ------------------------------------------------------------------------------------------------ statistics
def _ref_stats(x, split, pairs, L, wt, b, add, gamma, beta):
    y = x @ wt.double() + b.double()
    if add is not None:
        seg = np.repeat(np.arange(pairs * L), np.diff(split))
        y = y + add.double()[torch.tensor(seg)]
    sc, sh, mean_sc = [], [], []
    for p in range(pairs):
        yp = y[split[p * L]:split[(p + 1) * L]]
        m = yp.mean(0)
        v = ((yp - m) ** 2).mean(0)
        a = gamma.double() / torch.sqrt(v + 1e-5)
        sc.append(a); sh.append(beta.double() - m * a); mean_sc.append((m * a).abs())
    return torch.stack(sc), torch.stack(sh), torch.stack(mean_sc), y


@gpu
@pytest.mark.parametrize("dbg", [0, TWO_PASS], ids=["moments", "two_pass"])
@pytest.mark.parametrize("K", [128, 64])
@pytest.mark.parametrize("layout", ["two", "skew"])
def test_stats_vs_fp64(layout, K, dbg):
    """sc, sh to 2e-5 relative (sh: of |beta| + |mean sc|) on every channel on the moments path; the bit-4 path, whose
    fp32 sums of y^2 lose (1 + mean^2 / var) 2^-19 or so, to 1e-4 on every channel but the heavy one (|mean| / std >= 30,
    from its bias), which is only reported there."""
    lib = _lib.load()
    pairs, L, split, hi, lo, g = _inputs(layout, K, seed=11 + K)
    heavy = 5
    M, wt, b, gamma, beta = _layer(K, g, heavy)
    add = torch.randn(pairs * L, M, generator=g) * 0.5 if K == 64 else None
    x = hi.double() + lo.double()
    *_, y0 = _ref_stats(x, split, pairs, L, wt, b, add, gamma, beta)
    parts = [y0[split[p * L]:split[(p + 1) * L], heavy] for p in range(pairs)]
    b[heavy] = float(max(v.abs().max() + 31.0 * v.std(unbiased=False) for v in parts))   # mean >= 30 std in every pair
    sc_r, sh_r, msc, y = _ref_stats(x, split, pairs, L, wt, b, add, gamma, beta)
    for p in range(pairs):
        yp = y[split[p * L]:split[(p + 1) * L], heavy]
        if yp.numel() > 1:
            assert float(yp.mean().abs() / yp.std(unbiased=False).clamp_min(1e-300)) >= 30
    out = _run(lib, pairs, L, split, hi, lo, K, M, wt, b, add, gamma, beta, dbg=dbg)
    esc = (out["sc"].double() - sc_r).abs() / sc_r.abs()
    esh = (out["sh"].double() - sh_r).abs() / (beta.double().abs() + msc)
    rest = torch.ones(M, dtype=torch.bool)
    rest[heavy] = False
    r = dict(sc_rel=float(esc[:, rest].max()), sh_rel=float(esh[:, rest].max()),
             heavy_sc_rel=float(esc[:, heavy].max()), heavy_sh_rel=float(esh[:, heavy].max()))
    report(f"stats {layout} K={K} {'two-pass' if dbg else 'moments'}", **r)
    tol = 1e-4 if dbg else 2e-5
    assert r["sc_rel"] <= tol and r["sh_rel"] <= tol, r
    if not dbg:
        assert r["heavy_sc_rel"] <= 2e-5 and r["heavy_sh_rel"] <= 2e-5, r


# ------------------------------------------------------------------------------------------------ determinism
@gpu
@pytest.mark.parametrize("K", [128, 64])
def test_stats_deterministic_and_batch_independent(K):
    lib = _lib.load()
    pairs, L, split, hi, lo, g = _inputs("skew", K, seed=23 + K)
    M, wt, b, gamma, beta = _layer(K, g, 0)
    add = torch.randn(pairs * L, M, generator=g) * 0.5 if K == 64 else None
    a = _run(lib, pairs, L, split, hi, lo, K, M, wt, b, add, gamma, beta)
    a2 = _run(lib, pairs, L, split, hi, lo, K, M, wt, b, add, gamma, beta)
    for k in ("sc", "sh", "stats", "mom"):
        assert torch.equal(a[k].view(torch.uint8), a2[k].view(torch.uint8)), k
    for p in range(pairs):
        s0, s1 = split[p * L], split[(p + 1) * L]
        sub = [v - s0 for v in split[p * L:(p + 1) * L + 1]]
        one = _run(lib, 1, L, sub, hi[s0:s1], lo[s0:s1], K, M, wt, b, None if add is None else add[p * L:(p + 1) * L],
                   gamma, beta)
        for k in ("sc", "sh", "stats", "mom"):
            assert torch.equal(one[k][0].contiguous().view(torch.uint8), a[k][p].contiguous().view(torch.uint8)), (p, k)


@gpu
def test_pointnet_features_batch_independent():
    """mmmot_pointnet_fwd on a batch of three pairs of different sizes and on its middle pair alone: that pair's
    features are bit-identical."""
    lib = _lib.load()
    net, _ = eval_net("C", 0)
    wts = net.prepared()
    L = 16
    g = torch.Generator().manual_seed(3)
    counts = [torch.randint(1, 40, (L,), generator=g), torch.randint(300, 900, (L,), generator=g),
              torch.randint(1, 200, (L,), generator=g)]
    split = np.concatenate([[0], np.cumsum(torch.cat(counts).numpy())]).astype(np.int32)
    points = torch.randn(int(split[-1]), 3, generator=g).cuda() * 5

    def fwd(pts, sp, pairs):
        feats = torch.full((pairs, 3, 512, L), float("nan"), device="cuda")
        ws = torch.empty(int(lib.mmmot_pointnet_workspace(pairs, L, int(sp[-1]))), dtype=torch.uint8, device="cuda")
        d = torch.tensor(sp, device="cuda")
        _lib.check(lib.mmmot_pointnet_fwd(wts.ptr, vp(pts), vp(d), ctypes.c_void_p(sp.ctypes.data), pairs, L, vp(feats),
                                          vp(ws), ws.numel(), None), "mmmot_pointnet_fwd")
        torch.cuda.synchronize()
        return feats.cpu()

    with lib_state(lib, engine="tc"):
        full = fwd(points, split, 3)
        full2 = fwd(points, split, 3)
        s0, s1 = int(split[L]), int(split[2 * L])
        one = fwd(points[s0:s1].contiguous(), (split[L:2 * L + 1] - s0).astype(np.int32), 1)
    assert torch.equal(full.view(torch.int32), full2.view(torch.int32))
    assert torch.equal(one[0, 1].view(torch.int32), full[1, 1].view(torch.int32))


# ------------------------------------------------------------------------------------------------ CPU
def test_moments_kernels_do_not_spill():
    """ptxas -v of pointnet.cu (written by the Makefile): both moments instantiations, pn_moments_kernel<64, true> and
    <128, false>, report no spill stores or loads."""
    if not os.path.exists(PTXAS_LOG):
        pytest.skip("no ptxas log: the library was not built in this tree")
    log = open(PTXAS_LOG).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(\w*pn_moments_kernelILi(\d+)ELb([01])E\w*)'.*?\n(.*?\n.*?)\n", log):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", m.group(4))
        assert spill, m.group(0)
        found[(int(m.group(2)), int(m.group(3)))] = (int(spill.group(1)), int(spill.group(2)))
    assert found == {(64, 1): (0, 0), (128, 0): (0, 0)}, found
