"""The work schedule of the channel-major TMA-fed kernel (csrc/gemm_tma.cuh, gemm_tma_kernel) at its edges, against
fp64, element by element, through the product's launch code.

The persistent kernel walks (column tile, M group) units with a grid of min(units, SMs) CTAs, each unit in K segments,
and consumer warpgroup h takes column half h of every tile.  The cases below aim at the edges of that schedule: a launch
of one unit, an odd number of units that is no multiple of the grid, 2 to 5 K segments on an odd tile count, each of
the three box dimensions that can separate a tile's two column halves (image slab, box rows, box width) with the fused
pool and its per-image sums, and column halves that hold no column at all (a PointNet tile of <= 128 points, a conv
half wholly outside the image).  Any rework of the schedule has to keep these.

The checks themselves (|y - y_ref| <= 2^-18 S, NaN-initialised outputs, guard bands, pool sums, GroupNorm partials,
segment sums, device tables) are those of test_conv_engines.py and test_gen_engines.py, run on these shapes.
"""
import math

import pytest

import test_conv_engines as conv
import test_gen_engines as gen
from mmmot_b200 import _lib

gpu = pytest.mark.gpu
SMS = 132       # H100 SXM: the persistent grid is min(units, SMs)


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


# (name, cin, cout, H, W, n_img, debug bits, kseg, want_pool, compact Wpx, check) as test_conv_engines.CASES
CONV_CASES = [
    # one 16 x 16 box: a single (tile, M group) unit, halves split along the box rows, fused pool
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

# PointNet point layouts (pairs, L, points per detection).  ends: pair totals 257, 384 and 385, so the pairs' last
# tiles hold 1, 128 and 129 columns (half 1 empty, empty, one column).  single: one pair of 129 points, a launch of
# one tile.
PN_LAYOUTS = {"ends": (3, 4, [100, 100, 56, 1, 128, 128, 64, 64, 1, 255, 1, 128]),
              "single": (1, 2, [60, 69])}
PN_CASES = [(lay, kind) for lay in PN_LAYOUTS for kind in gen.MAT_KINDS]


@gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_schedule_vs_fp64(case):
    conv.test_conv_layer_vs_fp64(case)


@gpu
@pytest.mark.parametrize("layout,kind", PN_CASES, ids=[f"{a}-{b}" for a, b in PN_CASES])
def test_pn_schedule_vs_fp64(layout, kind, monkeypatch):
    monkeypatch.setitem(gen.LAYOUTS, layout, PN_LAYOUTS[layout])
    gen.test_pn_matrix_vs_fp64(layout, kind)


def test_conv_cases_take_named_schedules(lib_built):
    """Each conv case's plan, computed on the host, has the shape the case is named after."""
    lib = _lib.load()
    for name, C, M, H, W, n, dbg, kseg, want_pool, _, check in CONV_CASES:
        with conv._State(lib, dbg, kseg):
            p = conv._plan(lib, n, H, W, C, M, want_pool)
        assert check(p), (name, p)
    assert 147 % SMS and 147 % 2


def test_pn_layouts_end_as_named():
    """The PointNet layouts' tiles end with 1, 128 and 129 columns, and `single` is one tile."""
    ends = [ln for _, _, ln in gen.pn_tiles_host([0] + list(_cumsum(PN_LAYOUTS["ends"][2])), 3, 4)]
    assert sorted(ln for ln in ends if ln < gen.BN) == [1, 128, 129]
    single = gen.pn_tiles_host([0] + list(_cumsum(PN_LAYOUTS["single"][2])), 1, 2)
    assert [ln for _, _, ln in single] == [129]


def _cumsum(xs):
    s = 0
    for x in xs:
        s += x
        yield s
