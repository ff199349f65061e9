"""The GroupNorm + ReLU producers of the generated-operand engine (csrc/gemm_gen.cuh, GEN_NORM), which by default stage
each chunk's [256 rows x 32 channels] fp32 source box in shared memory by TMA (128-byte swizzle), two boxes ahead and
across tile boundaries, instead of loading it into registers.

GPU cases run one launch through mmmot_debug_gen (kernel_kit.run_gen: NaN-filled outputs with guard rows) with the
staged producers and one with the plain producers (debug bit 10) on the same inputs; Y and the GroupNorm partials must
agree bit for bit: the operand is the same function of the same fp32 values and the MMA order is the same.  The shapes
are the launches of the affinity MLP (layers 2 and 3 over uniform tiling; boxes that run into the next group and past
the end of the tensor), the new/end MLP's layer 2 and PointNet's layers 3 and 4 (tile tables over ragged groups of 1,
255, 257 and 9000 rows whose last tile ends at the end of the tensor), a single-tile launch and launches of more tiles
than there are SMs.  Element-wise accuracy against fp64 of the default (staged) producers is test_gen_engines.py's.

The CPU tests pin the variant query and check that the staged instantiation compiles without register spills.
"""
import os
import re

import numpy as np
import pytest
import torch

from kernel_kit import GEN, Cols, gen_weights, lib_state, ne_table, pn_tiles_host, run_gen
from mmmot_b200 import _lib

gpu = pytest.mark.gpu
PLAIN, PREFETCH = 1024, 4096       # mmmot_set_debug bits 10 and 12
BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mmmot_b200", "csrc", "build")


def _inputs(seed, rows, ld, K, groups):
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(rows, ld, generator=g) * 1.5
    gsc = (torch.rand(groups, K, generator=g) + 0.5) * torch.sign(torch.randn(groups, K, generator=g))
    gsh = torch.randn(groups, K, generator=g) * 0.5
    return g, src.cuda(), gsc.cuda(), gsh.cuda()


def _both(lib, seed, M, K, ld, rows, n_groups, cols, y_rows, **kw):
    g, src, gsc, gsh = _inputs(seed, rows, ld, K, n_groups)
    wt, b, Wp, wps = gen_weights(g, K, M)
    out = []
    for dbg in (0, PLAIN):
        Y, P, pref = run_gen(lib, GEN.NORM, wt, b, Wp, wps, src, cols, y_rows, ld_src=ld, gsc=gsc, gsh=gsh, dbg=dbg, **kw)
        assert pref == 0
        out.append((Y, P))
    (Y0, P0), (Y1, P1) = out
    assert bool(torch.isfinite(Y0[cols.y_row.cuda()]).all())
    assert torch.equal(Y0.view(torch.int32), Y1.view(torch.int32))
    assert torch.equal(P0.view(torch.int64), P1.view(torch.int64))


# (M, K, ld_src, S, groups): affinity layer 2 (K = 512 of 1024 floats per row), layer 3 (M = 128), a single tile, and
# one group of 64 tiles (more tiles than SMs with four 128-row blocks of M).  Source rows = groups * S exactly
# (x_gs = S, as the affinity stage lays them out), so the last box of every group but the last reads into the next
# group and the last one past the end of the tensor.
UNIFORM = [(512, 512, 1024, 300, 48), (512, 512, 1024, 400, 40), (512, 512, 1024, 16384, 3), (128, 512, 512, 300, 80),
           (128, 64, 64, 100, 1), (512, 512, 512, 16384, 1)]


@gpu
@pytest.mark.parametrize("M,K,ld,S,G", UNIFORM, ids=[f"M{c[0]}_K{c[1]}_ld{c[2]}_S{c[3]}_G{c[4]}" for c in UNIFORM])
def test_staged_norm_uniform_equals_plain(M, K, ld, S, G):
    lib = _lib.load()
    cols = Cols.uniform(S, G, S, S + 5)
    _both(lib, M * 7 + K + ld + S + G, M, K, ld, G * S, G, cols, G * (S + 5), S=S, groups=G, x_gs=S, y_gs=S + 5)


def _pn_ragged():
    """PointNet's table over four pairs of one detection each with 1, 255, 257 and 9000 points: the last tile ends at
    the last of the tensor's 9513 rows."""
    split = np.cumsum([0, 1, 255, 257, 9000]).tolist()
    return pn_tiles_host(split, 4, 1), split[-1], 4


# (name, M, K, tiles builder): new/end layer 2 (K = 512, M = 128, groups of m = 37 and n = 100 rows), PointNet layers
# 3 and 4 (K = 64: two chunks per tile, so the source ring runs across tiles)
TABLE = [("ne_l2", 128, 512, ne_table), ("pn_l3", 64, 64, _pn_ragged), ("pn_l4", 128, 64, _pn_ragged)]


@gpu
@pytest.mark.parametrize("name,M,K,build", TABLE, ids=[c[0] for c in TABLE])
def test_staged_norm_table_equals_plain(name, M, K, build):
    lib = _lib.load()
    tiles, rows, groups = build()
    _both(lib, len(name) * 31 + M, M, K, K, rows, groups, Cols.table(tiles), rows)


# ------------------------------------------------------------------------------------------------ CPU
def test_gen_norm_staged_query(lib_built):
    """Staged by default; bit 10 keeps the plain producers, bit 12 the prefetching ones; the other queries as before."""
    lib = _lib.load()
    assert [lib.mmmot_debug_gen_norm_staged(d) for d in (0, PLAIN, PREFETCH, PLAIN | PREFETCH)] == [1, 0, 0, 0]
    assert lib.mmmot_debug_gen_norm_staged(1 | 2 | 4 | 8) == 1
    for dbg, pre in ((0, 0), (PLAIN, 0), (PREFETCH, 1), (PLAIN | PREFETCH, 0)):
        with lib_state(lib, dbg=dbg):
            assert lib.mmmot_debug_gen_prefetch(GEN.NORM, 0) == pre
            assert lib.mmmot_debug_gen_staged(GEN.NORM, 128) == 0


@pytest.mark.parametrize("unit", ["affinity", "pointnet"])
def test_staged_norm_kernel_does_not_spill(unit):
    """ptxas -v (written by the Makefile) of the units that launch GEN_NORM: gemm_gen_kernel<GEN_NORM, false, true>
    reports no spill stores or loads and no wgmma serialization."""
    path = os.path.join(BUILD, f"{unit}.ptxas.log")
    if not os.path.exists(path):
        pytest.skip("no ptxas log: the library was not built in this tree")
    log = open(path).read()
    found = []
    for m in re.finditer(r"Compiling entry function '(_ZN3gen15gemm_gen_kernelILi3ELb0ELb1E\w*)'.*?\n(.*?\n.*?)\n", log):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", m.group(2))
        assert spill, m.group(0)
        found.append((int(spill.group(1)), int(spill.group(2))))
        assert not re.search(r"C7520[^\n]*" + re.escape(m.group(1)), log), m.group(1)
    assert found == [(0, 0)], found
