"""The pairwise producers of the generated-operand engine at m == 128 (csrc/gemm_gen.cuh, PAIRED GEN_PAIR_*), which
stage each chunk's sources in shared memory by TMA: the [128 detections x 32 channels] fp32 box (128-byte swizzle) and
the tile's two object rows.

GPU cases use the fp64 element-wise harness of the generated-operand tests (kernel_kit.run_gen: |y - y_ref| <= 2^-18 S,
partials to their stated tolerance, NaN-filled outputs with guard rows) at the edges of the staging: a last tile of one object row (its second
row is the group's first detection row, masked), many groups (the detection box never starts at row 0), a stack whose
G * Lf rows end exactly at the last box, one- and two-chunk K (fewer chunks than the source look-ahead), and enough
tiles per CTA that the ring wraps many times.  The staged and the plain producers (debug bit 10) must give bit-identical
outputs: the operand is the same function of the same fp32 values and the MMA order is the same.

The CPU tests check the variant query and that the staged instantiations compile without register spills.
"""
import os
import re

import pytest
import torch

from kernel_kit import GEN, Cols, check_part, check_rows, gen_weights, lib_state, ref_linear, report, run_gen
from mmmot_b200 import _lib

gpu = pytest.mark.gpu
PLAIN = 1024                       # mmmot_set_debug bit 10: producers without the pipeline (no staging)
PTXAS_LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mmmot_b200", "csrc", "build",
                         "affinity.ptxas.log")

# (n, G, M, K): n object rows against m = 128 detections, G groups (feature stacks of Lf = n + 128 rows)
STAGE_SHAPES = [(128, 3, 1024, 512), (127, 4, 1024, 512), (1, 6, 1024, 512), (128, 12, 1024, 512), (3, 40, 1024, 512),
                (64, 5, 256, 32), (65, 2, 128, 64)]
STAGE_CASES = [(op,) + s for op in (GEN.MUL, GEN.ABS, GEN.SUB) for s in STAGE_SHAPES]


def _pair_inputs(op, n, G, K, seed):
    g = torch.Generator().manual_seed(seed)
    F = torch.randn(G, n + 128, K, generator=g) * (1.0 if op == GEN.MUL else 2.0)
    if op == GEN.MUL:
        hot = torch.randint(0, K, (min(16, K),), generator=g)
        F[:, :, hot] = torch.sign(torch.randn(G, n + 128, hot.numel(), generator=g)) * 255.8
    return g, F


def _run(lib, op, n, G, M, K, seed, dbg=0):
    g, F = _pair_inputs(op, n, G, K, seed)
    wt, b, Wp, wps = gen_weights(g, K, M)
    NM, gap = n * 128, 5
    cols = Cols.uniform(NM, G, 0, NM + gap)
    Fd = F.cuda().contiguous()      # exactly G * Lf rows: the last detection box ends at the end of the tensor
    Y, P, pref = run_gen(lib, op, wt, b, Wp, wps, Fd, cols, G * (NM + gap), n=n, m=128, Lf=n + 128, S=NM, groups=G,
                         y_gs=NM + gap, dbg=dbg)
    return Fd, wt, b, cols, Y, P, pref


@gpu
@pytest.mark.parametrize("op,n,G,M,K", STAGE_CASES,
                         ids=[f"{GEN.NAMES[c[0]]}-n{c[1]}-G{c[2]}-M{c[3]}-K{c[4]}" for c in STAGE_CASES])
def test_staged_pairwise_vs_fp64(op, n, G, M, K):
    lib = _lib.load()
    with lib_state(lib):
        assert lib.mmmot_debug_gen_staged(op, 128) == 1
    Fd, wt, b, cols, Y, P, pref = _run(lib, op, n, G, M, K, seed=op * 1000 + n * 7 + G * 13 + K)
    assert pref == 1
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
    report(f"staged pair {GEN.NAMES[op]} n={n} G={G} M={M} K={K}", err_over_bound=r, part_err_over_tol=rp)
    assert r <= 1.0


BITWISE_CASES = [(op, 127, 4, 1024, 512) for op in (GEN.MUL, GEN.ABS, GEN.SUB)] + [(GEN.MUL, 1, 9, 256, 64)]


@gpu
@pytest.mark.parametrize("op,n,G,M,K", BITWISE_CASES,
                         ids=[f"{GEN.NAMES[c[0]]}-n{c[1]}-G{c[2]}-M{c[3]}-K{c[4]}" for c in BITWISE_CASES])
def test_staged_equals_plain_bitwise(op, n, G, M, K):
    """The staged producers and the plain ones (bit 10) on the same launch: Y and the partials agree bit for bit."""
    lib = _lib.load()
    seed = 77 + op * 31 + n
    *_, Y0, P0, pref0 = _run(lib, op, n, G, M, K, seed)
    *_, Y1, P1, pref1 = _run(lib, op, n, G, M, K, seed, dbg=PLAIN)
    assert (pref0, pref1) == (1, 0)
    assert torch.equal(Y0.view(torch.int32), Y1.view(torch.int32))
    assert torch.equal(P0.view(torch.int64), P1.view(torch.int64))


def test_gen_staged_query(lib_built):
    """gen_staged through the library, no GPU: only the pairwise producers at m == 128, never with bit 10."""
    lib = _lib.load()
    ms = (1, 64, 127, 128, 129, 256)
    with lib_state(lib):
        assert [lib.mmmot_debug_gen_staged(op, m) for op in (GEN.MUL, GEN.ABS, GEN.SUB) for m in ms] == [0, 0, 0, 1, 0, 0] * 3
        assert all(lib.mmmot_debug_gen_staged(gn, m) == 0 for gn in (GEN.NORM, GEN.COPY) for m in ms)
        assert lib.mmmot_debug_gen_staged(5, 128) == -1 and lib.mmmot_debug_gen_staged(-1, 128) == -1
        # the staged path is the pipelined one at exactly those shapes
        assert all(lib.mmmot_debug_gen_prefetch(op, 128) == 1 for op in (GEN.MUL, GEN.ABS, GEN.SUB))
    with lib_state(lib, dbg=4096):
        assert [lib.mmmot_debug_gen_staged(op, m) for op in (GEN.MUL, GEN.ABS, GEN.SUB) for m in ms] == [0, 0, 0, 1, 0, 0] * 3
    for dbg in (PLAIN, PLAIN | 4096):
        with lib_state(lib, dbg=dbg):
            assert all(lib.mmmot_debug_gen_staged(gn, m) == 0 for gn in range(5) for m in ms)


def test_staged_kernels_do_not_spill():
    """ptxas -v of affinity.cu (written by the Makefile): the staged instantiations gemm_gen_kernel<0|1|2, true>
    report no spill stores or loads and no wgmma serialization."""
    if not os.path.exists(PTXAS_LOG):
        pytest.skip("no ptxas log: the library was not built in this tree")
    log = open(PTXAS_LOG).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(_ZN3gen15gemm_gen_kernelILi([0-2])ELb1E\w*)'.*?\n(.*?\n.*?)\n", log):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", m.group(3))
        assert spill, m.group(0)
        found[int(m.group(2))] = (int(spill.group(1)), int(spill.group(2)))
        assert not re.search(r"C7520[^\n]*" + re.escape(m.group(1)), log), m.group(1)
    assert found == {0: (0, 0), 1: (0, 0), 2: (0, 0)}, found
