"""The affinity stage (csrc/affinity.cu mmmot_affinity_fwd) from its input features to y3 and h2, kernel by kernel
against fp64, each kernel on its own stored inputs.

Each GPU case runs the real mmmot_affinity_fwd once with a workspace filled with NaN (0xFF bytes, status reset), then
reads the intermediates the stage left there at the offsets mmmot_debug_stage_layout(0, ...) reports (the same carve
the stage runs).  Every kernel is checked against fp64 (computed on the GPU) from the inputs it read, as stored, so no
upstream error enters a bound.  Every element a kernel owns must be written and the rest of each buffer must still hold
the fill (Workspace.owned).  Every case prints err / bound per check.  The kernels after the last contraction (the
new/end means and final layer, the link logits, the softmax) are tests/test_heads.py's.

Notation: u = 2^-24, TAU = 2^-18 (the tensor-core contraction bound, kernel_kit.TAU: |y - y_ref| <= TAU S,
S = |W| A + |b| with A the magnitude of the operand the producer forms), FP64 = 2^-40 (fp64 summation and
cancellation).  G = 3 pairs groups g = pair*3 + stack, NM = n m columns per g, the new/end table's groups 2g (the m new
columns) and 2g + 1 (the n end columns).  Weights come from the state dict by name (w_link.conv1.*,
w_link.w_new_end.*), so the checks also pin which packed weight each launch uses.

Contractions.  TC: the reference is X W^T + b in fp64 of the operand the producer forms from the stored input, to
TAU S: layer 1 (GEN_PAIR_*) from the stored fcl with X = f_i g_j, A = |f_i||g_j| (multiply), X = |f_i - g_j| / 2 or
(f_i - g_j) / 2, A = (|f_i| + |g_j|) / 2 (minus_abs, minus), as test_gen_engines.test_pairwise_vs_fp64; GEN_NORM (layers
2, 3 and new/end 2) X = relu(y sc + sh), A = |y||sc| + |sh| from the stored y, sc, sh of the column's group; GEN_COPY
(new/end 1) X = V, A = |V|.  FP32: the operand as the engine's loader forms it in fp32 (kernel_kit.pair_operand,
norm_operand, V itself), then the chain bound of kernel_kit.contraction_bound.  The layer-1 references are chunked
(several GB in fp64 at 256 x 256 otherwise).

GroupNorm statistics.  The sums come from the contraction epilogues' fp32 runs, so the stored output y is what they
summed; per channel, the kernel's mean and variance differ from the two-pass fp64 values over y by kernel_kit.gn_stats's
tm, tv with the epilogue terms (KAPPA, KAPPA1) and T = 0.  GroupNorm(1, 512) (new/end conv0 on channels 512..1023 of
y01, both new/end layers) adds the 512 channel sums of a group: gn_stats's combination, derived there,
    tm_g = mean_c tm_c,   tv_g = mean_c [tv_c + 2 |m_c - m_g| tm_c + tm_c^2]   (+ the FP64 terms, which average).
The affine then follows kernel_kit.affine_bound: with er = tv / (2 (var + eps)) + FP64,
    |sc - a| <= |a| (er + u),   |sh - sh_ref| <= |a| tm + |mean a| er + u (|sh| + |mean a|).
  sc1 / sh1   GroupNorm(512, 512) over NM columns of the stored y01[..., :512].
  sc0 / sh0   GroupNorm(1, 512) over 512 NM values of the stored y01[..., 512:].
  sc2 / sh2   GroupNorm(512, 512) of the stored y2.
  nsc1 / nsh1 GroupNorm(1, 512) of the stored h1 per table group, m columns (new) or n (end).
Statistics that survive the stage.  stats (layer 3, [G][128][2]) and nstats (new/end layer 2, [2G][128][2]) must equal
bit for bit stats_reduce's fixed-order fp64 sum of the stored partials part / npart (stripe y sums slots t0 + y,
t0 + y + 8, ... in order from 0, then the 8 stripes are added 0..7; slots g tpg k .. (g + 1) tpg k for layer 3 and
gstart[i] k .. gstart[i + 1] k for the table, k = 2 partials per tile on TC, 1 on FP32), and match the two-pass moments
of the stored y3 / h2 to kernel_kit.stats_ratios.  sc3 / sh3 and nsc2 / nsh2 are gn_finalize in fp64 of those stored
sums (cpg 1, count NM; cpg 128, count m or n), one fp32 rounding each (kernel_kit.gn_affine).
Tables.  tiles, cnt and gstart equal the host table (kernel_kit.ne_tiles_host, tile width 256 on TC and 128 on FP32, no
gap) exactly; the rest of the tiles buffer is untouched.  fcl (TC) is the transpose of the features bit for bit, and
untouched on FP32.

CPU tests: the layout query is tests/test_heads.py's; here a guard that the cases cover what they must, a guard that
every launch and helper call of mmmot_affinity_fwd maps to a named check, and planted defects: each bound accepts a
plain fp32 evaluation and rejects, by more than 10x, a per-channel variance over NM - 1 columns, conv0's GroupNorm
finalised per channel, the new group's statistics taken with the end group's count, layer 2 reading y01's channels
512.. instead of 0.., new/end layer 2 taking the neighbouring group's affine and stats_reduce dropping a group's last
tile.  The NM - 1 defect moves sc by 1/(2 NM) relative while the statistics bound is about 32 u (1 + |mean| / std), so
its margin falls as 1/NM: it is planted at NM = 1073 (37 x 29), where it is 237x, which puts it near 4x at the
benchmark's NM = 65536 (256 x 256) -- the one defect here whose detection depends on the shape.
"""
import functools
import os

import numpy as np
import pytest
import torch

from kernel_kit import (BN, TAU, XM, Workspace, affine_bound, case_seed, contraction_bound, eval_net, gn_affine,
                        gn_stats, group_moments, impl_launches, lib_state, nan_output, nan_workspace, ne_tiles_host,
                        norm_operand, pair_operand, ref_linear, report, stage_layout, stats_ratios, vp, worst_ratio)
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_state_dict

gpu = pytest.mark.gpu
XMODE = {"multiply": XM.MUL, "minus_abs": XM.ABS, "minus": XM.SUB}
CHECKS = ("fcl", "y01", "sc1_sh1", "sc0_sh0", "tables", "h1", "nsc1_nsh1", "h2", "nstats", "nsc2_nsh2", "y2", "sc2_sh2",
          "y3", "stats", "sc3_sh3")
HEAD_CHECKS = ("new_end_mean", "new_end_sigmoid", "link_logit", "softmax_sums", "softmax_link")   # tests/test_heads.py
ROWS = 16384                       # columns per chunk of the fp64 contraction references


# ------------------------------------------------------------------------------------------------ cases
# (name, n, m, pairs, engine, op, end mode, features): "relu" relu(randn); "alike" look-alike detections, every feature
# column one shared column plus 2 % noise (layer-1 channels at |mean| / std >= 100)
CASES = [
    ("1x1-fp32", 1, 1, 2, "fp32", "multiply", "avg", "relu"), ("1x1-tc", 1, 1, 2, "tc", "minus_abs", "max", "relu"),
    ("1x64-tc", 1, 64, 1, "tc", "minus", "avg", "relu"), ("64x1-fp32", 64, 1, 1, "fp32", "minus_abs", "max", "relu"),
    ("7x9-auto", 7, 9, 3, "auto", "minus", "avg", "relu"), ("8x8-auto", 8, 8, 2, "auto", "minus_abs", "max", "relu"),
    ("37x29-tc", 37, 29, 3, "tc", "multiply", "avg", "relu"), ("37x29-fp32", 37, 29, 3, "fp32", "minus", "max", "relu"),
    ("20x45-tc", 20, 45, 1, "tc", "minus", "max", "relu"), ("20x45-fp32", 20, 45, 1, "fp32", "multiply", "avg", "relu"),
    ("257x40-tc", 257, 40, 1, "tc", "minus_abs", "avg", "relu"), ("40x300-tc", 40, 300, 1, "tc", "multiply", "max", "relu"),
    ("257x40-fp32", 257, 40, 1, "fp32", "multiply", "max", "relu"),
    ("40x300-fp32", 40, 300, 1, "fp32", "minus_abs", "avg", "relu"),
    ("cfg2", 32, 32, 1, "auto", "minus_abs", "avg", "relu"), ("cfg3", 64, 64, 1, "auto", "multiply", "max", "relu"),
    ("cfg4", 128, 128, 1, "auto", "minus", "avg", "relu"), ("cfg5", 256, 256, 1, "auto", "minus_abs", "max", "relu"),
    ("alike-tc", 37, 29, 3, "tc", "multiply", "avg", "alike"), ("alike-fp32", 20, 45, 1, "fp32", "multiply", "max", "alike"),
]


def af_path(n, m, engine):
    """The path a case must take: 'tc' or 'fp32' (auto: tensor cores from N.M = 64)."""
    return engine if engine != "auto" else ("tc" if n * m >= 64 else "fp32")


def _feats(kind, pairs, L, g):
    if kind == "alike":
        base = torch.relu(torch.randn(pairs, 3, 512, 1, generator=g)) + 0.5
        return base * (1 + 0.02 * torch.randn(pairs, 3, 512, L, generator=g))
    return torch.relu(torch.randn(pairs, 3, 512, L, generator=g))


# ------------------------------------------------------------------------------------------------ references
def weights(sd, device):
    """The stage's weights from the state dict by name, fp64: W*T [K][M] (transposed), biases, GroupNorm gamma / beta."""
    f = lambda k: sd[k].double().to(device)
    c, ne = "w_link.conv1", "w_link.w_new_end"
    lin = lambda k, M: f(f"{k}.weight").reshape(M, 512).T.contiguous()
    return dict(W01=torch.cat([lin(f"{c}.0", 512), lin(f"{ne}.conv0.0", 512)], 1),
                b01=torch.cat([f(f"{c}.0.bias"), f(f"{ne}.conv0.0.bias")]),
                g1=f(f"{c}.1.weight"), be1=f(f"{c}.1.bias"), g0=f(f"{ne}.conv0.1.weight"), be0=f(f"{ne}.conv0.1.bias"),
                W2=lin(f"{c}.3", 512), b2=f(f"{c}.3.bias"), g2=f(f"{c}.4.weight"), be2=f(f"{c}.4.bias"),
                W3=lin(f"{c}.6", 128), b3=f(f"{c}.6.bias"), g3=f(f"{c}.7.weight"), be3=f(f"{c}.7.bias"),
                Wn1=lin(f"{ne}.conv1.0", 512), bn1=f(f"{ne}.conv1.0.bias"), gn1=f(f"{ne}.conv1.1.weight"),
                ben1=f(f"{ne}.conv1.1.bias"), Wn2=lin(f"{ne}.conv1.3", 128), bn2=f(f"{ne}.conv1.3.bias"),
                gn2=f(f"{ne}.conv1.4.weight"), ben2=f(f"{ne}.conv1.4.bias"))


def pair_tc(F, op, n, m, s0, s1):
    """GEN_PAIR_* operand and its magnitude A for columns s0..s1 of one group from F [n + m][512] (fp64)."""
    s = torch.arange(s0, s1, device=F.device)
    a, d = F[s // m], F[n + s % m]
    if op == "multiply":
        return a * d, a.abs() * d.abs()
    X = (a - d).abs() / 2 if op == "minus_abs" else (a - d) / 2
    return X, (a.abs() + d.abs()) / 2


def norm_tc(y, sc, sh):
    """GEN_NORM operand relu(y sc + sh) and A = |y||sc| + |sh| (fp64, sc / sh per row)."""
    return torch.relu(y * sc + sh), y.abs() * sc.abs() + sh.abs()


def gn_check(y, grp, G, gamma, beta, sc, sh, cpg=1):
    """sc / sh [G][C] of a GroupNorm over the stored y [cols][C] (fp64) -> worst err / bound of both."""
    a, b, Ta, Tb = affine_bound(gn_stats(y, grp, G, cpg=cpg), gamma, beta)
    return max(worst_ratio(sc, a, Ta), worst_ratio(sh, b, Tb))


def reduce_ref(part, ranges):
    """stats_reduce's fixed-order fp64 sum of part [slots][M][2] over each group's slot range [t0, t1) -> [G][M][2]."""
    out = []
    for t0, t1 in ranges:
        tot = torch.zeros_like(part[0])
        for y in range(8):
            s = torch.zeros_like(part[0])
            for t in range(t0 + y, t1, 8):
                s = s + part[t]
            tot = tot + s
        out.append(tot)
    return torch.stack(out)


def ne_groups(G, n, m, device):
    """Table group 2g + (end) of every new/end column col = g (n + m) + r."""
    L = n + m
    col = torch.arange(G * L, device=device)
    return 2 * (col // L) + (col % L >= m).long()


# ------------------------------------------------------------------------------------------------ GPU
@functools.lru_cache(maxsize=None)
def _net():
    return eval_net("C", 37)


def _run(lib, case):
    name, n, m, pairs, engine, op, end, kind = case
    net, sd = _net()
    G, NM, L = 3 * pairs, n * m, n + m
    g = torch.Generator().manual_seed(case_seed("affinity stage", *case))
    feats = _feats(kind, pairs, L, g).cuda()
    link, new, end_s = nan_output(G * NM), nan_output(G * m), nan_output(G * n)
    with lib_state(lib, engine=engine):
        lay, tc = stage_layout(lib, 0, pairs, n, m)
        nbytes = int(lib.mmmot_affinity_workspace(pairs, n, m))
        ws = nan_workspace(lib, nbytes)
        rc = lib.mmmot_affinity_fwd(net.prepared().ptr, _lib.AFFINITY[op], _lib.SOFTMAX["single"], _lib.END_MODE[end],
                                    pairs, n, m, vp(feats), vp(link), vp(new), vp(end_s), vp(ws), nbytes, None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    assert tc == (af_path(n, m, engine) == "tc")
    assert lib.mmmot_status_check(vp(ws), None) == 0, "status word raised"
    return dict(n=n, m=m, G=G, NM=NM, L=L, op=op, tc=tc, feats=feats, W=Workspace(ws, lay), wt=weights(sd, "cuda"))


def check_layer1(d, r):
    """fcl, y01 and the two GroupNorm affines formed from it."""
    W, wt, G, n, m, NM, L, tc = (d[k] for k in ("W", "wt", "G", "n", "m", "NM", "L", "tc"))
    feats = d["feats"].view(G, 512, L)
    if tc:
        fcl = W.owned("fcl", G * L * 512).view(G, L, 512)
        assert torch.equal(fcl, feats.transpose(1, 2)), "fcl"
    else:
        assert W.untouched_after("fcl", 0), "fcl written on the FP32 path"
    r["fcl"] = 0.0
    y01 = W.owned("y01", G * 1024 * NM)
    y01 = y01.view(G, NM, 1024) if tc else y01.view(G, 1024, NM)
    sc1, sh1 = (W.owned(k, G * 512).view(G, 512) for k in ("sc1", "sh1"))
    sc0, sh0 = (W.owned(k, G * 512).view(G, 512) for k in ("sc0", "sh0"))
    r["y01"] = r["sc1_sh1"] = r["sc0_sh0"] = 0.0
    one = torch.zeros(NM, dtype=torch.long, device="cuda")
    cond = 0.0
    for gi in range(G):
        if tc:
            F = fcl[gi].double()
            for s0 in range(0, NM, ROWS):
                s1 = min(NM, s0 + ROWS)
                X, A = pair_tc(F, d["op"], n, m, s0, s1)
                ref, S = ref_linear(X, A, wt["W01"], wt["b01"])
                r["y01"] = max(r["y01"], worst_ratio(y01[gi, s0:s1], ref, TAU * S))
            y = y01[gi].double()
        else:
            x = pair_operand(feats[gi:gi + 1], XMODE[d["op"]], n, m).double()
            ref, T = contraction_bound(wt["W01"], x, wt["b01"])
            r["y01"] = max(r["y01"], worst_ratio(y01[gi], ref, T))
            y = y01[gi].double().T
        del ref
        r["sc1_sh1"] = max(r["sc1_sh1"], gn_check(y[:, :512], one, 1, wt["g1"], wt["be1"], sc1[gi:gi + 1], sh1[gi:gi + 1]))
        r["sc0_sh0"] = max(r["sc0_sh0"], gn_check(y[:, 512:], one, 1, wt["g0"], wt["be0"], sc0[gi:gi + 1], sh0[gi:gi + 1],
                                                  cpg=512))
        _, mean, var, _, _ = group_moments(y[:, :512], one, 1)
        spread = var > 0                                       # NM = 1: no spread, nothing to condition
        if bool(spread.any()):
            cond = max(cond, float((mean.abs()[spread] / var[spread].sqrt()).max()))
    d["cond"] = cond
    return y01, sc1, sh1


def check_layers23(d, r, y01, sc1, sh1):
    """y2, sc2 / sh2, y3, the surviving statistics and sc3 / sh3."""
    W, wt, G, NM, tc = (d[k] for k in ("W", "wt", "G", "NM", "tc"))
    y2 = W.owned("y2", G * 512 * NM)
    y2 = y2.view(G, NM, 512) if tc else y2.view(G, 512, NM)
    y3 = W.owned("y3", G * 128 * NM)
    y3 = y3.view(G, NM, 128) if tc else y3.view(G, 128, NM)
    sc2, sh2 = (W.owned(k, G * 512).view(G, 512) for k in ("sc2", "sh2"))
    r["y2"] = r["sc2_sh2"] = r["y3"] = 0.0
    one = torch.zeros(NM, dtype=torch.long, device="cuda")
    for gi in range(G):
        for src, sc, sh, Wt, b, dst, key in ((y01, sc1, sh1, wt["W2"], wt["b2"], y2, "y2"),
                                             (y2, sc2, sh2, wt["W3"], wt["b3"], y3, "y3")):
            if tc:
                for s0 in range(0, NM, ROWS):
                    s1 = min(NM, s0 + ROWS)
                    X, A = norm_tc(src[gi, s0:s1, :512].double(), sc[gi].double(), sh[gi].double())
                    ref, S = ref_linear(X, A, Wt, b)
                    r[key] = max(r[key], worst_ratio(dst[gi, s0:s1], ref, TAU * S))
            else:
                x = norm_operand(src[gi, :512], sc[gi, :, None], sh[gi, :, None]).double()
                ref, T = contraction_bound(Wt, x, b)
                r[key] = max(r[key], worst_ratio(dst[gi], ref, T))
            del ref
            if key == "y2":
                y = y2[gi].double() if tc else y2[gi].double().T
                r["sc2_sh2"] = max(r["sc2_sh2"], gn_check(y, one, 1, wt["g2"], wt["be2"], sc2[gi:gi + 1], sh2[gi:gi + 1]))
    # layer 3's statistics: bit for bit from the stored partials, against the stored y3, then its affine
    k = 2 if tc else 1
    tpg = -(-NM // (BN if tc else 128))
    part = W.owned("part", G * tpg * k * 1024 * 2, torch.float64)[:G * tpg * k * 128 * 2].view(G * tpg * k, 128, 2)
    stats = W.owned("stats", G * 1024 * 2, torch.float64)[:G * 128 * 2].view(G, 128, 2)
    want = reduce_ref(part, [(gi * tpg * k, (gi + 1) * tpg * k) for gi in range(G)])
    assert torch.equal(stats, want), "stats: not stats_reduce's fixed-order sum of the stored partials"
    yy = (y3.double() if tc else y3.double().transpose(1, 2)).reshape(G * NM, 128)
    grp = torch.arange(G, device="cuda").repeat_interleave(NM)
    rv, rm, _ = stats_ratios(stats[..., 0], stats[..., 1], yy, grp, G)
    r["stats"] = max(rv, rm)
    sc3, sh3 = (W.owned(k2, G * 128).view(G, 128) for k2 in ("sc3", "sh3"))
    a, b, Ta, Tb = gn_affine(stats, wt["g3"], wt["be3"], NM)
    r["sc3_sh3"] = max(worst_ratio(sc3, a, Ta), worst_ratio(sh3, b, Tb))


def check_new_end(d, r):
    """The tile table, h1, nsc1 / nsh1, h2, nstats and nsc2 / nsh2."""
    W, wt, G, n, m, L, tc = (d[k] for k in ("W", "wt", "G", "n", "m", "L", "tc"))
    tw = BN if tc else 128
    tiles, _ = ne_tiles_host(G, n, m, 0, tw)
    nt = len(tiles)
    assert W.owned("tiles", 4 * nt, torch.int32).view(nt, 4).tolist() == [[gi, r0, ln, 0] for gi, r0, ln in tiles], "tiles"
    assert W.owned("cnt", 2 * G, torch.int32).tolist() == [m, n] * G, "cnt"
    per = [0] * (2 * G)
    for gi, _, _ in tiles:
        per[gi] += 1
    gstart = np.concatenate([[0], np.cumsum(per)]).tolist()
    assert W.owned("gstart", 2 * G + 1, torch.int32).tolist() == gstart, "gstart"
    r["tables"] = 0.0
    ldv = G * L
    grp = ne_groups(G, n, m, "cuda")
    V = W.owned("v", 512 * ldv)
    h1 = W.owned("h1", 512 * ldv)
    h2 = W.owned("h2", 128 * ldv)
    nsc1, nsh1 = (W.owned(k, 2 * G * 512).view(2 * G, 512) for k in ("nsc1", "nsh1"))
    if tc:
        V, h1, h2 = V.view(ldv, 512), h1.view(ldv, 512), h2.view(ldv, 128)
        ref, S = ref_linear(V.double(), V.double().abs(), wt["Wn1"], wt["bn1"])
        r["h1"] = worst_ratio(h1, ref, TAU * S)
        X, A = norm_tc(h1.double(), nsc1[grp].double(), nsh1[grp].double())
        ref, S = ref_linear(X, A, wt["Wn2"], wt["bn2"])
        r["h2"] = worst_ratio(h2, ref, TAU * S)
        h1r, h2r = h1.double(), h2.double()
    else:
        V, h1, h2 = V.view(512, ldv), h1.view(512, ldv), h2.view(128, ldv)
        ref, T = contraction_bound(wt["Wn1"], V.double(), wt["bn1"])
        r["h1"] = worst_ratio(h1, ref, T)
        x = norm_operand(h1, nsc1[grp].T, nsh1[grp].T).double()
        ref, T = contraction_bound(wt["Wn2"], x, wt["bn2"])
        r["h2"] = worst_ratio(h2, ref, T)
        h1r, h2r = h1.double().T, h2.double().T
    r["nsc1_nsh1"] = gn_check(h1r, grp, 2 * G, wt["gn1"], wt["ben1"], nsc1, nsh1, cpg=512)
    k = 2 if tc else 1
    npart = W.owned("npart", nt * k * 512 * 2, torch.float64)[:nt * k * 128 * 2].view(nt * k, 128, 2)
    nstats = W.owned("nstats", 2 * G * 512 * 2, torch.float64)[:2 * G * 128 * 2].view(2 * G, 128, 2)
    want = reduce_ref(npart, [(gstart[i] * k, gstart[i + 1] * k) for i in range(2 * G)])
    assert torch.equal(nstats, want), "nstats: not stats_reduce's fixed-order sum of the stored partials"
    rv, rm, _ = stats_ratios(nstats[..., 0], nstats[..., 1], h2r, grp, 2 * G)
    r["nstats"] = max(rv, rm)
    nsc2, nsh2 = (W.owned(k2, 2 * G * 128).view(2 * G, 128) for k2 in ("nsc2", "nsh2"))
    cnt = torch.tensor([m, n] * G, device="cuda")
    a, b, Ta, Tb = gn_affine(nstats, wt["gn2"], wt["ben2"], cnt, 128)
    r["nsc2_nsh2"] = max(worst_ratio(nsc2, a, Ta), worst_ratio(nsh2, b, Tb))


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_affinity_stage_vs_fp64(case):
    """mmmot_affinity_fwd, then every kernel up to y3 and h2 against fp64 of its own stored inputs (module docstring)."""
    lib = _lib.load()
    d = _run(lib, case)
    r = {}
    y01, sc1, sh1 = check_layer1(d, r)
    check_new_end(d, r)
    check_layers23(d, r, y01, sc1, sh1)
    assert set(r) == set(CHECKS), sorted(r)
    name, n, m, pairs = case[:4]
    report(f"affinity stage {name} {n}x{m} pairs={pairs} {case[5]} [{'tc' if d['tc'] else 'fp32'}] (err / bound)", **r,
           layer1_mean_over_std=d["cond"])
    if case[7] == "alike":
        assert d["cond"] >= 100, d["cond"]
    assert all(v <= 1.0 for v in r.values()), r


# ------------------------------------------------------------------------------------------------ CPU
def test_case_coverage():
    """The GPU cases take both paths, forced and under auto on both sides of N.M = 64 (7 x 9, 8 x 8), every op on each
    path, new or end groups of one column and GroupNorm over one row (n or m = 1), tail tiles under half (37 x 29, G = 9)
    and over half (20 x 45) of 256 columns, a 1-column end tile and two new tiles per group on the tensor cores
    (257 x 40, 40 x 300) and 128 + 128 + 1 table tiles on FP32, the cfg2-cfg5 square shapes, and look-alike features
    on each path."""
    path = {c[0]: af_path(c[1], c[2], c[4]) for c in CASES}
    assert {(path[c[0]], c[4]) for c in CASES} == {("tc", "tc"), ("tc", "auto"), ("fp32", "fp32"), ("fp32", "auto")}
    auto = {(c[1], c[2]): path[c[0]] for c in CASES if c[4] == "auto"}
    assert auto[(7, 9)] == "fp32" and auto[(8, 8)] == "tc" and 7 * 9 < 64 == 8 * 8
    for p in ("tc", "fp32"):
        cs = [c for c in CASES if path[c[0]] == p]
        assert {c[5] for c in cs} == set(XMODE), p
        assert any(c[1] == 1 for c in cs) or any(c[2] == 1 for c in cs), p
        assert any(c[1] == 1 and c[2] == 1 for c in cs), p
        assert any(c[7] == "alike" for c in cs), p
        for nm in ((37, 29), (20, 45), (257, 40), (40, 300)):
            assert any((c[1], c[2]) == nm for c in cs), (p, nm)
    assert any((c[1], c[2], c[3]) == (37, 29, 3) for c in CASES)
    assert 37 * 29 % BN < BN // 2 <= 20 * 45 % BN
    assert 257 % BN == 1 and -(-300 // BN) == 2 and 257 % 128 == 1 and -(-300 // 128) == 3
    assert {c[1] for c in CASES if c[1] == c[2] and path[c[0]] == "tc" and c[4] == "auto"} >= {32, 64, 128, 256}


# Every kernel launch and helper call of mmmot_affinity_fwd, in source order (both paths), with the checks that hold
# its output: this file's CHECKS or tests/test_heads.py's HEAD_CHECKS.  feats_range_kernel's only output is the status
# word, which every case requires clear.
AF_HELPERS = ("launch_gen", "gemm_simt_launch", "transpose_f32", "stats_reduce", "gn_finalize")
LAUNCH_SITES = [
    ("transpose_f32", ("fcl",)), ("feats_range_kernel", ("y01",)),
    ("launch_gen", ("y01",)), ("launch_gen", ("y01",)), ("launch_gen", ("y01",)),                    # TC layer 1, per op
    ("gemm_simt_launch", ("y01",)), ("gemm_simt_launch", ("y01",)), ("gemm_simt_launch", ("y01",)),  # FP32 layer 1
    ("stats_reduce", ("sc1_sh1", "sc0_sh0")), ("gn_finalize", ("sc1_sh1",)), ("gn_finalize", ("sc0_sh0",)),
    ("newend_mean_cl_kernel", ("new_end_mean",)), ("rowcol_mean_kernel", ("new_end_mean",)),
    ("ne_tiles_kernel", ("tables",)),
    # new / end MLP, tensor cores
    ("launch_gen", ("h1",)), ("stats_reduce", ("nsc1_nsh1",)), ("gn_finalize", ("nsc1_nsh1",)),
    ("launch_gen", ("h2",)), ("stats_reduce", ("nstats",)), ("gn_finalize", ("nsc2_nsh2",)),
    ("ne_final_cl_kernel", ("new_end_sigmoid",)),
    # new / end MLP, FP32
    ("gemm_simt_launch", ("h1",)), ("stats_reduce", ("nsc1_nsh1",)), ("gn_finalize", ("nsc1_nsh1",)),
    ("gemm_simt_launch", ("h2",)), ("stats_reduce", ("nstats",)), ("gn_finalize", ("nsc2_nsh2",)),
    ("ne_final_kernel", ("new_end_sigmoid",)),
    # affinity layers 2, 3, tensor cores then FP32
    ("launch_gen", ("y2",)), ("stats_reduce", ("sc2_sh2",)), ("gn_finalize", ("sc2_sh2",)),
    ("launch_gen", ("y3",)), ("stats_reduce", ("stats",)), ("gn_finalize", ("sc3_sh3",)),
    ("gemm_simt_launch", ("y2",)), ("stats_reduce", ("sc2_sh2",)), ("gn_finalize", ("sc2_sh2",)),
    ("gemm_simt_launch", ("y3",)), ("stats_reduce", ("stats",)), ("gn_finalize", ("sc3_sh3",)),
    ("link_logit_cl_kernel", ("link_logit",)), ("link_logit_kernel", ("link_logit",)),
    ("softmax_stats_kernel", ("softmax_sums",)), ("softmax_apply_kernel", ("softmax_link",)),
]


def test_stage_launch_coverage_guard():
    """Every launch of mmmot_affinity_fwd maps to a check: a launch added, removed or reordered without its entry in
    LAUNCH_SITES fails here; every check named there is one the GPU tests fill, and every check is named."""
    assert impl_launches("affinity.cu", "mmmot_affinity_fwd", AF_HELPERS) == [s[0] for s in LAUNCH_SITES]
    named = {c for _, cs in LAUNCH_SITES for c in cs}
    assert named == set(CHECKS) | set(HEAD_CHECKS), named ^ (set(CHECKS) | set(HEAD_CHECKS))
    heads = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_heads.py")).read()
    for c in HEAD_CHECKS:
        assert f'r["{c}"]' in heads, c


def _fp32_affine(y32, grp, G, gamma, beta, cpg=1, count=None):
    """The plain fp32 evaluation of a GroupNorm affine: fp64 statistics of the fp32 values, rounded once to fp32;
    count overrides the per-group column count (a planted defect)."""
    n, mean, var, _, _ = group_moments(y32.double(), grp, G)
    if count is not None:                     # the same sums divided by another count
        s1, s2 = mean * n, (var + mean * mean) * n
        mean = s1 / count
        var = s2 / count - mean * mean
    if cpg > 1:
        C = y32.shape[1]
        M = mean.view(G, C // cpg, cpg).mean(2, keepdim=True)
        V = (var.view(G, C // cpg, cpg) + (mean.view(G, C // cpg, cpg) - M) ** 2).mean(2)
        mean, var = M[..., 0].repeat_interleave(cpg, 1), V.repeat_interleave(cpg, 1)
    a = gamma / torch.sqrt(var + 1e-5)
    return a.float(), (beta - mean * a).float()


def test_bounds_reject_planted_defects():
    """Each bound accepts a plain fp32 evaluation and rejects its planted defect by more than 10x (module docstring)."""
    wt = weights(synthetic_state_dict("C", seed=37), "cpu")
    g = torch.Generator().manual_seed(13)
    out = {}
    n, m = 37, 29
    NM, L = n * m, n + m
    F = torch.relu(torch.randn(L, 512, generator=g))
    X, A = pair_tc(F.double(), "multiply", n, m, 0, NM)
    y01 = (X.float() @ wt["W01"].float() + wt["b01"].float())          # plain fp32 layer 1
    one = torch.zeros(NM, dtype=torch.long)
    y = y01.double()
    # sc1: per-channel variance over NM - 1 columns
    a, b, Ta, Tb = affine_bound(gn_stats(y[:, :512], one, 1), wt["g1"], wt["be1"])
    sc, sh = _fp32_affine(y01[:, :512], one, 1, wt["g1"], wt["be1"])
    out["sc1 fp32"] = max(worst_ratio(sc, a, Ta), worst_ratio(sh, b, Tb))
    _, mean, var, _, _ = group_moments(y[:, :512], one, 1)
    ab = wt["g1"] / torch.sqrt(var * NM / (NM - 1) + 1e-5)                 # the variance over NM - 1, the mean over NM
    out["sc1 var / (NM-1)"] = max(worst_ratio(ab.float(), a, Ta), worst_ratio((wt["be1"] - mean * ab).float(), b, Tb))
    # sc0: GroupNorm(1, 512) finalised per channel
    a, b, Ta, Tb = affine_bound(gn_stats(y[:, 512:], one, 1, cpg=512), wt["g0"], wt["be0"])
    sc, sh = _fp32_affine(y01[:, 512:], one, 1, wt["g0"], wt["be0"], cpg=512)
    out["sc0 fp32"] = max(worst_ratio(sc, a, Ta), worst_ratio(sh, b, Tb))
    sc, sh = _fp32_affine(y01[:, 512:], one, 1, wt["g0"], wt["be0"], cpg=1)
    out["sc0 per channel"] = max(worst_ratio(sc, a, Ta), worst_ratio(sh, b, Tb))
    # layer 2 reading y01's channels 512.. instead of 0.. (TC and FP32 bounds)
    sc1, sh1 = _fp32_affine(y01[:, :512], one, 1, wt["g1"], wt["be1"])
    X2, A2 = norm_tc(y[:, :512], sc1.double(), sh1.double())
    ref, S = ref_linear(X2, A2, wt["W2"], wt["b2"])
    ev = lambda v: norm_operand(v, sc1, sh1) @ wt["W2"].float() + wt["b2"].float()
    out["y2 fp32"] = worst_ratio(ev(y01[:, :512]), ref, TAU * S)
    out["y2 channels 512.."] = worst_ratio(ev(y01[:, 512:]), ref, TAU * S)
    c = slice(0, 64)                                                    # the chain bound on 64 columns
    refc, T = contraction_bound(wt["W2"], norm_operand(y01[c, :512], sc1, sh1).double().T.contiguous(), wt["b2"])
    out["y2 chain fp32"] = worst_ratio(ev(y01[c, :512]).T, refc, T)
    out["y2 chain channels 512.."] = worst_ratio(ev(y01[c, 512:]).T, refc, T)
    # new/end layer 1 statistics with the end group's count; layer 2 with the neighbouring group's affine
    G = 3
    grp = ne_groups(G, n, m, "cpu")
    V = torch.relu(torch.randn(G * L, 512, generator=g) * 0.6 + 0.3)
    h1 = V @ wt["Wn1"].float() + wt["bn1"].float()
    st = gn_stats(h1.double(), grp, 2 * G, cpg=512)
    a, b, Ta, Tb = affine_bound(st, wt["gn1"], wt["ben1"])
    nsc1, nsh1 = _fp32_affine(h1, grp, 2 * G, wt["gn1"], wt["ben1"], cpg=512)
    out["nsc1 fp32"] = max(worst_ratio(nsc1, a, Ta), worst_ratio(nsh1, b, Tb))
    cnt = torch.tensor([m, n] * G, dtype=torch.float64)[:, None]
    wrong = cnt.clone()
    wrong[0::2] = n                                                    # the new groups take the end group's count
    scb, shb = _fp32_affine(h1, grp, 2 * G, wt["gn1"], wt["ben1"], cpg=512, count=wrong)
    out["nsc1 end count"] = max(worst_ratio(scb, a, Ta), worst_ratio(shb, b, Tb))
    X2, A2 = norm_tc(h1.double(), nsc1[grp].double(), nsh1[grp].double())
    ref, S = ref_linear(X2, A2, wt["Wn2"], wt["bn2"])
    ev = lambda gg: norm_operand(h1, nsc1[gg], nsh1[gg]) @ wt["Wn2"].float() + wt["bn2"].float()
    out["h2 fp32"] = worst_ratio(ev(grp), ref, TAU * S)
    out["h2 neighbour affine"] = worst_ratio(ev(grp ^ 1), ref, TAU * S)
    refc, T = contraction_bound(wt["Wn2"], norm_operand(h1, nsc1[grp], nsh1[grp]).double().T.contiguous(), wt["bn2"])
    out["h2 chain fp32"] = worst_ratio(ev(grp).T, refc, T)
    out["h2 chain neighbour affine"] = worst_ratio(ev(grp ^ 1).T, refc, T)
    # stats_reduce dropping a group's last tile: layer 3 partials per 128-column half-tile of 256-column tiles
    y3 = torch.randn(G * NM, 128, generator=g) * 0.8 + torch.randn(128, generator=g)
    tpg = -(-NM // BN)
    slot = torch.arange(NM).repeat(G) // 128 + torch.arange(G).repeat_interleave(NM) * 2 * tpg
    y3d = y3.double()
    part = torch.stack([torch.zeros(G * 2 * tpg, 128, dtype=torch.float64).index_add_(0, slot, v) for v in (y3d, y3d * y3d)], -1)
    grp3 = torch.arange(G).repeat_interleave(NM)
    full = reduce_ref(part, [(gi * 2 * tpg, (gi + 1) * 2 * tpg) for gi in range(G)])
    short = reduce_ref(part, [(gi * 2 * tpg, (gi + 1) * 2 * tpg - (2 if gi == 1 else 0)) for gi in range(G)])
    out["stats fp32"] = max(stats_ratios(full[..., 0], full[..., 1], y3d, grp3, G)[:2])
    out["stats last tile dropped"] = max(stats_ratios(short[..., 0], short[..., 1], y3d, grp3, G)[:2])
    report("planted defects (err / bound)", **out)
    ok = [k for k in out if "fp32" in k]
    assert max(out[k] for k in ok) <= 1.0, out
    assert min(v for k, v in out.items() if k not in ok) > 10.0, out
