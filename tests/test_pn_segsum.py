"""PointNet's per-detection-sum passes (layer 5, K = 128 -> M = 1024; the head, K = 64 -> M = 512 with the addend U) on
the dedicated kernel (csrc/gemm_segsum.cuh) and on the general TMA-fed kernel it replaces (debug bit 16, 65536).

Kernel level: one launch through mmmot_debug_pn_contraction, the segment sums of each kernel held to the fp64 bound of
test_gen_engines.py's matrix tests,

    |got - want| <= |sc| TAU sum_p S_p + 40 2^-24 sum_p (|y_p sc| + |sh|) + 2^-33 (fixed-point flushes),

on point layouts that put detection boundaries inside 32-column chunks and on chunk and half-tile edges, leave tile
halves without columns, end a pair on a partial tile, make a launch of one tile, and at the benchmark configurations'
detection sizes (cfg2: 64 detections of 128 points per pair, cfg3 / cfg4: 128 / 256 detections of 512 points; one
pair each).  The launch sizes also run both work schedules of the new kernel: all m-groups of a tile in one unit
(at least as many tiles as SMs, here with a unit count that is not a multiple of the grid) and m-groups split over
several units (fewer tiles than SMs).  Nothing may be written past [ndet][M].

Stage level: mmmot_pointnet_fwd with and without the bit.  Everything before layer 5's recompute is the same code, so
the per-detection means of layer 5 (gmean) may differ only by the fp32 order inside each <= 32-term run of ReLU
outputs (non-negative terms: 2 x 31 roundings relative to the sum) and the 2^-32 fixed point of each flush; the head's
means (hmean) inherit that through U and its GroupNorm statistics, and are held to the stage's TAU scale.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from kernel_kit import (BN, LAYOUTS, TAU, U, Workspace, case_seed, fp16_split, gen_weights, lib_state, nan_workspace,
                        pn_host_tables, pn_tiles_host, ref_linear, report, stage_layout, vp)
from mmmot_b200 import _lib

gpu = pytest.mark.gpu
OLD = 65536                         # debug bit 16: the per-detection-sum passes on gemm_tma_kernel
SEG_FILL = 0x5A5A5A5A5A5A5A5A       # guard pattern after the segment sums
PTXAS_LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mmmot_b200", "csrc", "build",
                         "pointnet.ptxas.log")


def _seeded(seed, n, lo, hi, ones):
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(lo, hi, (n,), generator=g)
    c[ones] = 1
    return c.tolist()


# (pairs, L, points per detection).  ends: pair totals 257, 384, 385 leave last tiles of 1, 128 and 129 columns (half 1
# empty, empty, one column); single: one tile; halves: boundaries on chunk edges (32, 64, 96) and on the half-tile edge
# (128, 384) with one-point detections straddling none of them; many: 1 pair, 201 tiles (more than the SMs: one unit
# per tile, 201 units on a 132-SM H100 grid), ragged.
LAYOUTS_SS = dict(
    LAYOUTS,
    ends=(3, 4, [100, 100, 56, 1, 128, 128, 64, 64, 1, 255, 1, 128]),
    single=(1, 2, [60, 69]),
    halves=(1, 16, [32, 32, 32, 32, 256, 1, 31, 64, 32, 1, 1, 30, 128, 64, 64, 100]),
    many=(1, 128, _seeded(7, 128, 310, 510, [5, 6, 40])),
    cfg2=(1, 64, [128] * 64),
    cfg3=(1, 128, [512] * 128),
    cfg4=(1, 256, [512] * 256),
)
KINDS = {"l5": (1024, 128, False), "head": (512, 64, True)}     # kind -> (M, K, addend)
CASES = [(lay, kind) for lay in LAYOUTS_SS for kind in KINDS]


def _runs_per_det(tiles, seg, ndet):
    """Per detection: the 32-column chunks its points fall in (one fixed-point flush per chunk and run)."""
    tile_of = np.concatenate([np.full(ln, t) for t, (_, _, ln) in enumerate(tiles)])
    chunk = np.concatenate([np.arange(ln) // 32 for _, _, ln in tiles])
    keys = np.unique(np.stack([seg, tile_of, chunk]), axis=1)
    return torch.tensor(np.bincount(keys[0], minlength=ndet), dtype=torch.float64)


@gpu
@pytest.mark.parametrize("layout,kind", CASES, ids=[f"{a}-{b}" for a, b in CASES])
def test_segsum_kernels_vs_fp64(layout, kind):
    """Both kernels' per-detection sums of one PointNet segsum launch against fp64, and the guard after them intact."""
    pairs, L, counts = LAYOUTS_SS[layout]
    M, K, want_add = KINDS[kind]
    lib = _lib.load()
    ndet = pairs * L
    split = [0] + np.cumsum(counts).tolist()
    P = split[-1]
    tiles_h, seg_h, _, _, _ = pn_host_tables(split, pairs, L)
    nt = len(tiles_h)
    g = torch.Generator().manual_seed(case_seed("segsum", layout, kind))
    wt, b, Wp, wps = gen_weights(g, K, M)
    x = torch.randn(P, K, generator=g)
    hi, lo = fp16_split(x)
    X = torch.stack([hi, lo]).contiguous().cuda()
    add = (torch.randn(ndet, M, generator=g) * 0.5).cuda() if want_add else None
    sc = ((torch.rand(pairs, M, generator=g) + 0.5) * torch.sign(torch.randn(pairs, M, generator=g))).cuda()
    sh = (torch.randn(pairs, M, generator=g) * 0.3).cuda()
    d_split = torch.tensor(split, dtype=torch.int32, device="cuda")
    h_split = torch.tensor(split, dtype=torch.int32)
    Wd, bd = Wp.cuda(), b.cuda()

    # fp64 reference and bound, shared by both kernels
    seg_t = torch.tensor(seg_h, device="cuda")
    xr = (hi.double() + lo.double()).cuda()
    ref, S = ref_linear(xr, xr.abs(), wt, b)
    del xr
    if want_add:
        a64 = add.double()[seg_t]
        ref, S = ref + a64, S + a64.abs()
        del a64
    pair_of = seg_t // L
    scp, shp = sc.double()[pair_of], sh.double()[pair_of]
    acc = lambda v: torch.zeros(ndet, M, dtype=torch.float64, device="cuda").index_add_(0, seg_t, v)
    want = acc(torch.relu(ref * scp + shp))
    runs = _runs_per_det(tiles_h, np.asarray(seg_h), ndet).cuda()[:, None]
    tol = acc(scp.abs() * TAU * S) + 40 * U * acc((ref * scp).abs() + shp.abs()) + runs * 2.0 ** -33
    del ref, S, scp, shp

    out = {}
    for dbg, name in ((0, "new"), (OLD, "old")):
        cap = nt + 3
        tiles = torch.full((cap, 4), -7, dtype=torch.int32, device="cuda")
        ctab = torch.full((2 * cap, 4), -7, dtype=torch.int32, device="cuda")
        cnt = torch.full((pairs + 2,), -7, dtype=torch.int32, device="cuda")
        gstart = torch.full((pairs + 3,), -7, dtype=torch.int32, device="cuda")
        segd = torch.full((P + 64,), -7, dtype=torch.int32, device="cuda")
        ss = torch.full((ndet * M + 512,), SEG_FILL, dtype=torch.int64, device="cuda")
        ss[:ndet * M] = 0
        n_tiles = ctypes.c_long(-1)
        with lib_state(lib, dbg=dbg):
            assert lib.mmmot_debug_segsum_kernel(K, 0, 0, 0) == (1 if dbg == 0 else 0)
            rc = lib.mmmot_debug_pn_contraction(vp(d_split), vp(h_split), pairs, L, cap, vp(tiles), vp(cnt), vp(gstart),
                                                vp(segd), vp(ctab), ctypes.byref(n_tiles), vp(Wd), wps, vp(bd), M, K,
                                                vp(X), None, None, vp(add), M, vp(ss), vp(sc), vp(sh), None)
            torch.cuda.synchronize()
        assert rc == 0, rc
        assert n_tiles.value == nt
        assert bool((ss[ndet * M:] == SEG_FILL).all()), f"{name}: segment sums written past [det][M]"
        got = ss[:ndet * M].view(ndet, M).double() * 2.0 ** -32
        out[f"{name}_err_over_tol"] = float(((got - want).abs() / tol).max())
    report(f"segsum {layout} {kind} ({nt} tiles, P={P})", **out)
    assert max(out.values()) <= 1.0, out


# ------------------------------------------------------------------------------------------------ GPU: stage level
def _stage(lib, net, pts, counts, pairs, L, dbg):
    split = [0] + np.cumsum(counts).tolist()
    P = split[-1]
    hs = np.asarray(split, dtype=np.int32)
    feats = torch.full((pairs * 3 * 512 * L,), float("nan"), device="cuda")
    with lib_state(lib, dbg=dbg):
        lay, tc = stage_layout(lib, 2, pairs, L, P)
        nbytes = int(lib.mmmot_pointnet_workspace(pairs, L, P))
        ws = nan_workspace(lib, nbytes)
        rc = lib.mmmot_pointnet_fwd(net.prepared().ptr, vp(pts), vp(torch.tensor(hs, device="cuda")),
                                    ctypes.c_void_p(hs.ctypes.data), pairs, L, vp(feats), vp(ws), nbytes, None)
        torch.cuda.synchronize()
        taken = lib.mmmot_debug_segsum_kernel(128, 0, 0, 0), lib.mmmot_debug_segsum_kernel(64, 0, 0, 0)
    assert rc == 0, rc
    assert tc, "PointNet took the FP32 path"
    assert lib.mmmot_status_check(vp(ws), None) == 0, "status word raised"
    W = Workspace(ws, lay)
    nd = pairs * L
    return dict(gmean=W.owned("gmean", nd * 1024).view(nd, 1024).double(),
                hmean=W.owned("hmean", nd * 512).view(nd, 512).double()), taken


STAGE_CASES = [("cfg4-xyz", 3, 1, 256, 512), ("xyzr", 4, 2, 32, 300)]


@gpu
@pytest.mark.parametrize("name,C,pairs,L,pts", STAGE_CASES, ids=[c[0] for c in STAGE_CASES])
def test_pointnet_stage_both_kernels(name, C, pairs, L, pts):
    """mmmot_pointnet_fwd with the dedicated kernel (the default, reported by mmmot_debug_segsum_kernel) and with debug
    bit 16: gmean within the fp32 run-order bound, hmean within the stage's TAU scale."""
    import mmmot_b200 as mb
    from mmmot_b200.synthetic import synthetic_state_dict
    lib = _lib.load()
    g = torch.Generator().manual_seed(case_seed("segsum stage", name))
    nd = pairs * L
    counts = (torch.randint(pts // 2, pts * 3 // 2, (nd,), generator=g) if name != "cfg4-xyz"
              else torch.full((nd,), pts)).tolist()
    counts[1] = 1
    P = sum(counts)
    centre = torch.rand(nd, 3, generator=g) * torch.tensor([60.0, 40.0, 2.0]) + torch.tensor([0.0, -20.0, -2.0])
    xyz = torch.randn(P, 3, generator=g) * torch.tensor([2.0, 1.0, 0.8]) + centre.repeat_interleave(torch.tensor(counts), 0)
    pts_t = torch.cat([xyz, torch.rand(P, 1, generator=g)], 1) if C == 4 else xyz
    net = mb.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch="C", test_mode=2, dropblock=0,
                         without_reflectivity=(C == 3))
    net.load_state_dict(synthetic_state_dict("C", seed=3, point_in=C))
    net.cuda().eval()
    pts_d = pts_t.contiguous().cuda()
    new, taken_new = _stage(lib, net, pts_d, counts, pairs, L, 0)
    old, taken_old = _stage(lib, net, pts_d, counts, pairs, L, OLD)
    assert taken_new == (1, 1) and taken_old == (0, 0)
    # gmean: per detection, the mean of <= 32-term fp32 runs of non-negative terms, each run summed in two orders
    # (<= 2 x 31 roundings of the run's sum) and flushed in 2^-32 fixed point; a detection of n points has at most
    # n / 32 + 2 runs per 256-column tile it touches
    cnt = torch.tensor(counts, dtype=torch.float64, device="cuda")[:, None]
    runs = cnt / 32 + 2 * (cnt / BN + 2)
    tol_g = 64 * U * (new["gmean"] + old["gmean"]) / 2 + runs * 2.0 ** -31 / cnt
    r_g = float(((new["gmean"] - old["gmean"]).abs() / tol_g).max())
    # hmean: U and the head's statistics shift with gmean; the stage's scale TAU x the channel's largest mean
    scale = torch.maximum(new["hmean"].abs().amax(0, keepdim=True), torch.tensor(1e-30, device="cuda"))
    r_h = float(((new["hmean"] - old["hmean"]).abs() / (TAU * scale)).max())
    report(f"stage {name} (P={P})", gmean_diff_over_tol=r_g, hmean_diff_over_tau_scale=r_h)
    assert r_g <= 1.0 and r_h <= 1.0, (r_g, r_h)


# ------------------------------------------------------------------------------------------------ CPU
def test_pointnet_shapes_route_to_segsum_kernel(lib_built):
    """The per-detection-sum passes PointNet issues at cfg2-cfg4 (cfg5 has no PointNet) take the dedicated kernel: layer
    5 (K = 128) and the head (K = 64), no Y, no partials, no ReLU, at any detection count.  Launches with an output,
    partials, a ReLU or another K (the FPN laterals, K >= 256), and every launch under debug bit 16, do not."""
    import bench
    lib = _lib.load()
    for cfg in ("cfg2", "cfg3", "cfg4"):
        assert bench.CONFIGS[cfg]["pts"] > 0 and 2 * bench.CONFIGS[cfg]["n"] >= 16   # the tensor-core PointNet path
    assert bench.CONFIGS["cfg5"]["pts"] == 0
    with lib_state(lib):
        assert lib.mmmot_debug_segsum_kernel(128, 0, 0, 0) == 1 and lib.mmmot_debug_segsum_kernel(64, 0, 0, 0) == 1
        assert [lib.mmmot_debug_segsum_kernel(128, y, p, r) for y, p, r in ((1, 0, 0), (0, 1, 0), (0, 0, 1))] == [0, 0, 0]
        assert [lib.mmmot_debug_segsum_kernel(k, 0, 0, 0) for k in (32, 96, 256, 512, 1024, 2048)] == [0] * 6
        assert lib.mmmot_debug_segsum_kernel(0, 0, 0, 0) < 0 and lib.mmmot_debug_segsum_kernel(100, 0, 0, 0) < 0
    with lib_state(lib, dbg=OLD):
        assert lib.mmmot_debug_segsum_kernel(128, 0, 0, 0) == 0 and lib.mmmot_debug_segsum_kernel(64, 0, 0, 0) == 0
    with lib_state(lib, dbg=16 | 8192):
        assert lib.mmmot_debug_segsum_kernel(128, 0, 0, 0) == 1


def test_segsum_layouts_as_named():
    """The layouts hold the cases the docstring names."""
    tiles = lambda lay: pn_tiles_host([0] + np.cumsum(LAYOUTS_SS[lay][2]).tolist(), *LAYOUTS_SS[lay][:2])
    assert sorted(ln for _, _, ln in tiles("ends") if ln < BN) == [1, 128, 129]
    assert [ln for _, _, ln in tiles("single")] == [129]
    split = set(np.cumsum(LAYOUTS_SS["halves"][2]).tolist())
    assert {32, 64, 96, 128, 384} <= split
    assert len(tiles("many")) == 201
    assert [len(tiles(c)) for c in ("cfg2", "cfg3", "cfg4")] == [32, 256, 512]


def test_segsum_kernels_do_not_spill():
    """ptxas -v of pointnet.cu (written by the Makefile): gemm_segsum_kernel<64> and <128> report no spill stores or
    loads and no wgmma serialisation (C75xx) remark."""
    if not os.path.exists(PTXAS_LOG):
        pytest.skip("no ptxas log: the library was not built in this tree")
    log = open(PTXAS_LOG).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(\w*gemm_segsum_kernelILi(\d+)E\w*)'.*?\n(.*?\n.*?)\n", log):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", m.group(3))
        assert spill, m.group(0)
        found[int(m.group(2))] = (int(spill.group(1)), int(spill.group(2)))
    assert found == {64: (0, 0), 128: (0, 0)}, found
    assert not re.search(r"C75\d\d\).*gemm_segsum_kernel", log)


def test_tma_kernels_do_not_spill():
    """ptxas -v of appearance.cu (written by the Makefile): every gemm_tma_kernel instantiation (matrix, conv through the
    accumulator image, conv from the accumulators) reports no spill stores or loads."""
    log_path = os.path.join(os.path.dirname(PTXAS_LOG), "appearance.ptxas.log")
    if not os.path.exists(log_path):
        pytest.skip("no ptxas log: the library was not built in this tree")
    log = open(log_path).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(\w*gemm_tma_kernelILi(\d+)E\w*)'.*?\n(.*?\n.*?)\n", log):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", m.group(3))
        assert spill, m.group(0)
        found[int(m.group(2))] = (int(spill.group(1)), int(spill.group(2)))
    assert found == {0: (0, 0), 1: (0, 0), 2: (0, 0)}, found
