"""The fusion and detection-score stage (csrc/fusion_det.cu mmmot_fusion_det_fwd) from its input stacks to h2, kernel by
kernel against fp64, each kernel on its own stored inputs.

Each GPU case runs the real mmmot_fusion_det_fwd once with a workspace filled with NaN (0xFF bytes, status reset) and
feats whose stack 2 (the fusion's output) is NaN, followed by a NaN guard band, then reads the intermediates the stage
left in the workspace at the offsets mmmot_debug_stage_layout(1, ...) reports (the same carve the stage runs).  Every
kernel is checked against fp64 (computed on the GPU) from the inputs it read, as stored, so no upstream error enters a
bound.  Every element a kernel owns must be written and the rest of each buffer must still hold the fill
(Workspace.owned); the buffers the fusion architecture does not use (yi, gi, sci, shi for A; gp, gi for B) and F3 on the
FP32 path stay untouched, and stacks 0 and 1 of feats come back bit for bit.  Every case prints err / bound per check.
The detection score from h2 is tests/test_heads.py's.

Notation: u = 2^-24, TAU = 2^-18 (the tensor-core contraction bound, kernel_kit.TAU: |y - y_ref| <= TAU S,
S = |W| |X| + |b|), FP64 = 2^-40, T0 = 2^-126 (an absolute floor for results near the subnormal range).  Weights are
the fp32 tensors the kernels are handed (the device table of net.prepared()), pinned to the state dict by name.

Layouts (the header's): TC (tensor cores; L >= 64 under auto) the fusion buffers are channels-last [pair*L + l][512]
and F3, h1, h2 detection-major rows [(pair*L + l)*3 + stack][512 | 512 | 256]; FP32 the fusion buffers are
[pair][512][L] and h1, h2 [pair*3 + stack][512 | 256][L].

Linears.  yp = input_w [stack 0; stack 1] (A, K = 1024) or input_p stack 0 (B, C), yi = input_i stack 1, gp = gate_p
stack 0, gi = gate_i stack 1 (C), each W x + b over 512 outputs.  TC: from the stored F3 rows (stacks 0 and 1 the
transpose of feats bit for bit), X W^T + b in fp64 to TAU S.  FP32: from feats, kernel_kit.contraction_bound (the
sequential fma chain).
GroupNorm(512, 512) per pair over the L detections.  The sums come from the contraction epilogues' fp32 runs over the
stored y, so scp / shp (from yp) and sci / shi (from yi) follow kernel_kit.gn_stats (KAPPA terms, T = 0) and
affine_bound:  |sc - a| <= |a| (er + u),  |sh - sh_ref| <= |a| tm + |mean a| er + u (|sh| + |mean a|),
er = tv / (2 (var + eps)) + FP64.  The stats and part buffers end as the last branch's (yp for A, yi for B and C):
stats must equal bit for bit stats_reduce's fixed-order fp64 sum of the stored partials (slots pair*tpg*k ..
(pair + 1)*tpg*k, k = 2 per 256-column tile on TC, 1 per 128-column tile on FP32), match the two-pass moments of the
stored y to kernel_kit.stats_ratios, and give that branch's sc / sh as gn_finalize in fp64 with one fp32 rounding each
(kernel_kit.gn_affine).
Combine (fusion_combine_rows_kernel on TC, fusion_combine_kernel on FP32) from the stored y, g, sc, sh; feats[:, 2] is
checked, and on TC F3's stack 2 must equal it bit for bit.  With v = yp scp + shp and w = yi sci + shi in fp64 (exact
products of fp32 values; one fp64 rounding, far below u), fmaf rounds each once:
  A   out = fl(v):             |out - v| <= 1.01 u |v|       (1.01 here and below: second-order and fp64 terms)
  B   out = fl(fl(v) + fl(w)): |out - (v + w)| <= 1.01 u (|v| + |w| + |v + w|)
  C   a = mm_sigmoid(gp) = 1 / (1 + expf(-gp)).  The build does not use fast-math, so expf is within 2 ulp (4u
      relative) and the add and the division round once each: a = s_p (1 + e_a), |e_a| <= 4u (1 - s_p) + 2u, s_p the
      fp64 sigmoid of the stored gp (d/dE of 1/(1 + E) is -s (1 - s) / E).  Likewise b for gi.  The numerator
      a*v + b*w rounds at most three times (two products and the sum), or twice where nvcc contracts it into an fma
      either way: within u (a|v| + b|w| + |num|) in every case.  a + b (both positive) and the division round once
      each.  To first order, with D = s_p + s_i and r = (s_p v + s_i w) / D,
          |out - r| <= 1.01 ([s_p |v| (e_a + 2u) + s_i |w| (e_b + 2u) + |r| (s_p e_a + s_i e_b)] / D + 3u |r|) + T0.
      The saturating cases drive the gate logits to about +-30 with opposite signs per channel: one sigmoid rounds to
      exactly 1 in fp32 (logit > 17.4) while the other is near 1e-13, and the fp32 sigmoids stay normal numbers.  Both
      logits below about -88 would make both sigmoids 0 in fp32 and the combine 0/0, as in the fp32 model; that regime
      is not tested (every stored logit is asserted within +-80).
w_det layers 1 and 2 (eval BatchNorm folded, ReLU in the epilogue; ReLU is 1-Lipschitz).  TC: h1 from the stored F3
rows (one matrix of 3 pairs L rows whose 256-row tiles cross detections, stacks and pairs), h2 from the stored h1, each
to TAU S.  FP32: h1 per (pair, stack) from the stored feats, h2 from the stored h1, contraction_bound with ReLU.

CPU tests: the layout query is tests/test_heads.py's; here a guard that the cases cover every architecture on each
path and every tail class, a guard that every launch of mmmot_fusion_det_fwd maps to a named check, and planted
defects: each bound accepts a plain fp32 evaluation and rejects, by more than 10x, a linear missing one 32-wide K
chunk (TC and FP32 bounds), gp and gi swapped in the combine (at ordinary and at saturating gates), a GroupNorm variance
over L - 1 instead of L (at L = 300; its margin falls as 1/L), w_det reading stack 2 of the neighbouring detection's
F3 row, and one 256-row w_det tile reading its rows shifted by one stack.
"""
import functools
import math
import os

import pytest
import torch

from kernel_kit import (BN, TAU, TINY, U, Workspace, affine_bound, assert_written, case_seed, contraction_bound,
                        eval_net, gn_affine, gn_stats, group_moments, impl_launches, lib_state, nan_output,
                        nan_workspace, reduce_ref, ref_linear, report, stage_layout, stats_ratios, vp, worst_ratio)
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_state_dict
from mmmot_b200.weights import prepare

gpu = pytest.mark.gpu
W = _lib.W
SAT = 22.0           # gate bias offset of the saturating nets (+-SAT by channel, opposite signs for gate_p and gate_i)
SAT_SCALE = 4.0      # their gate weight scale: logits spread about +-17 around +-SAT
# (buffer, weight id, bias id, input stacks, state-dict module) of each linear, per fusion architecture
LINEARS = {"A": [("yp", "FU_WPT", "FU_BP", (0, 1), "input_w")],
           "B": [("yp", "FU_WPT", "FU_BP", (0,), "input_p"), ("yi", "FU_WIT", "FU_BI", (1,), "input_i")]}
LINEARS["C"] = LINEARS["B"] + [("gp", "FU_GATE_PT", "FU_GATE_PB", (0,), "gate_p"),
                               ("gi", "FU_GATE_IT", "FU_GATE_IB", (1,), "gate_i")]
# (branch, gamma id, beta id, state-dict module) of each GroupNorm
NORMS = {"A": [("p", "FU_GPW", "FU_GPB", "input_w")],
         "B": [("p", "FU_GPW", "FU_GPB", "input_p"), ("i", "FU_GIW", "FU_GIB", "input_i")]}
NORMS["C"] = NORMS["B"]
CHECKS = {a: ("f3",) + tuple(k for k, *_ in LINEARS[a]) + tuple(f"sc{b}_sh{b}" for b, *_ in NORMS[a])
          + ("stats", "stats_affine", "combine", "h1", "h2") for a in "ABC"}
HEAD_CHECKS = ("det",)                                   # tests/test_heads.py


# ------------------------------------------------------------------------------------------------ cases
# (name, fusion, L, pairs, engine, saturating gates).  The L grid: one detection, two, a 32-column transpose tile +-1,
# the automatic engine switch at 64 +-1, and 300 = one 256-row tile plus a 44-row tail (ragged 32 x 32 transposes);
# the architecture rotates so that each (L, pairs) runs a different one on each engine.
LS = (1, 2, 31, 33, 63, 64, 65, 300)
GRID = [(L, p, e) for L in LS for p in (1, 3) for e in ("fp32", "tc", "auto")]
CASES = [(f"{'ABC'[(k + k // 3) % 3]}-L{L}-p{p}-{e}", "ABC"[(k + k // 3) % 3], L, p, e, False)
         for k, (L, p, e) in enumerate(GRID)]
CASES += [("cfg2", "A", 64, 2, "auto", False), ("cfg3", "C", 128, 3, "auto", False), ("cfg4", "C", 256, 4, "auto", False),
          ("sat-tc", "C", 65, 3, "tc", True), ("sat-fp32", "C", 33, 3, "fp32", True), ("sat-auto", "C", 300, 1, "auto", True)]


def fd_path(L, engine):
    """The path a case must take: 'tc' or 'fp32' (auto: tensor cores from L = 64)."""
    return engine if engine != "auto" else ("tc" if L >= 64 else "fp32")


# ------------------------------------------------------------------------------------------------ references
def combine_ref(arch, v, w=None, gp=None, gi=None):
    """The fused stack from v = yp scp + shp and w = yi sci + shi (fp64 of the stored values) and the stored gate logits
    -> (ref, bound) (module docstring)."""
    if arch == "A":
        return v, 1.01 * U * v.abs() + TINY
    if arch == "B":
        s = v + w
        return s, 1.01 * U * (v.abs() + w.abs() + s.abs()) + TINY
    a, b = torch.sigmoid(gp), torch.sigmoid(gi)
    ea, eb = 4 * U * torch.sigmoid(-gp) + 2 * U, 4 * U * torch.sigmoid(-gi) + 2 * U
    D = a + b
    r = (a * v + b * w) / D
    T = ((a * v.abs() * (ea + 2 * U) + b * w.abs() * (eb + 2 * U) + r.abs() * (a * ea + b * eb)) / D + 3 * U * r.abs())
    return r, 1.01 * T + TINY


def combine_fp32(arch, yp, scp, shp, yi=None, sci=None, shi=None, gp=None, gi=None, fma=False):
    """The combine kernel's arithmetic in fp32 (fma: the numerator contracted into one fma)."""
    f = lambda y, sc, sh: (y.double() * sc.double() + sh.double()).float()
    v = f(yp, scp, shp)
    if arch == "A":
        return v
    w = f(yi, sci, shi)
    if arch == "B":
        return v + w
    sig = lambda g: 1.0 / (1.0 + torch.exp(-g))
    a, b = sig(gp), sig(gi)
    num = (a.double() * v.double() + (b * w).double()).float() if fma else a * v + b * w
    return num / (a + b)


def _saturate(sd):
    sign = torch.ones(512)
    sign[1::2] = -1
    for k, s in (("gate_p", 1.0), ("gate_i", -1.0)):
        sd[f"fusion_module.{k}.0.weight"] = sd[f"fusion_module.{k}.0.weight"] * SAT_SCALE
        sd[f"fusion_module.{k}.0.bias"] = s * SAT * sign


# ------------------------------------------------------------------------------------------------ GPU
@functools.lru_cache(maxsize=None)
def _net(arch, sat):
    """The net of a case and the fp64 weights the kernels are handed, checked against the state dict by name."""
    net, sd = eval_net(arch, 43, edit=_saturate if sat else None)
    wts = net.prepared()
    base = wts.flat.data_ptr()

    def handed(wid, *shape):
        o = (wts.table.w[W[wid]] - base) // 4
        return wts.flat[o:o + math.prod(shape)].view(*shape).double()
    wt = {}
    for _, wid, bid, stacks, mod in LINEARS[arch]:
        wt[wid], wt[bid] = handed(wid, 512 * len(stacks), 512), handed(bid, 512)
        assert torch.equal(wt[wid], sd[f"fusion_module.{mod}.0.weight"][..., 0].T.double().cuda()), wid
        assert torch.equal(wt[bid], sd[f"fusion_module.{mod}.0.bias"].double().cuda()), bid
    for _, gid, bid, mod in NORMS[arch]:
        wt[gid], wt[bid] = handed(gid, 512), handed(bid, 512)
        assert torch.equal(wt[gid], sd[f"fusion_module.{mod}.1.weight"].double().cuda()), gid
        assert torch.equal(wt[bid], sd[f"fusion_module.{mod}.1.bias"].double().cuda()), bid
    wt.update(WD_W1T=handed("WD_W1T", 512, 512), WD_B1=handed("WD_B1", 512), WD_W2T=handed("WD_W2T", 512, 256),
              WD_B2=handed("WD_B2", 256))
    return net, wt


def _run(lib, case):
    name, arch, L, pairs, engine, sat = case
    net, wt = _net(arch, sat)
    g = torch.Generator().manual_seed(case_seed("fusion stage", *case))
    nf = pairs * 3 * 512 * L
    feats = nan_output(nf)
    f = feats[:nf].view(pairs, 3, 512, L)
    f[:, :2] = torch.relu(torch.randn(pairs, 2, 512, L, generator=g)).cuda()
    f01 = f[:, :2].clone()
    det = nan_output(pairs * 3 * L)
    with lib_state(lib, engine=engine):
        lay, tc = stage_layout(lib, 1, pairs, L)
        nbytes = int(lib.mmmot_fusion_det_workspace(pairs, L))
        ws = nan_workspace(lib, nbytes)
        rc = lib.mmmot_fusion_det_fwd(net.prepared().ptr, _lib.FUSION[arch], 0, 0.0, pairs, L, vp(feats), vp(det), vp(ws),
                                      nbytes, None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    assert tc == (fd_path(L, engine) == "tc")
    assert lib.mmmot_status_check(vp(ws), None) == 0, "status word raised"
    assert_written(det, pairs * 3 * L, "det")
    assert torch.equal(f[:, :2], f01), "feature stacks 0, 1 changed"
    assert bool(torch.isfinite(f[:, 2]).all()), "stack 2: an element was not written"
    assert bool(torch.isnan(feats[nf:]).all()), "feats written past its end"
    return dict(arch=arch, L=L, pairs=pairs, tc=tc, f=f, wt=wt, W=Workspace(ws, lay),
                grp=torch.arange(pairs * L, device="cuda") // L)


def cl(d, v, tc):
    """A fusion buffer, channels-last (tc) or [pair][512][L] -> channels-last [pair*L][512]."""
    return v.view(-1, 512) if tc else v.view(d["pairs"], 512, d["L"]).transpose(1, 2).reshape(-1, 512)


def check_f3(d, r):
    """F3: stacks 0..2 the transpose of feats bit for bit on TC, untouched on FP32 -> F3 [pair*L*3][512] or None."""
    W, pairs, L = d["W"], d["pairs"], d["L"]
    r["f3"] = 0.0
    if not d["tc"]:
        assert W.untouched_after("f3", 0), "F3 written on the FP32 path"
        return None
    f3 = W.owned("f3", pairs * L * 3 * 512)
    rows = f3.view(pairs, L, 3, 512)
    for s in range(3):
        assert torch.equal(rows[:, :, s], d["f"][:, s].transpose(1, 2)), f"F3 stack {s}"
    return f3.view(pairs * L * 3, 512)


def check_linears(d, r, f3):
    """The five linears -> {buffer: stored output, channels-last [pair*L][512]}."""
    W, wt, pairs, L, arch = d["W"], d["wt"], d["pairs"], d["L"], d["arch"]
    ys = {}
    for key, wid, bid, stacks, _ in LINEARS[arch]:
        y = W.owned(key, pairs * L * 512)
        K = 512 * len(stacks)
        if d["tc"]:
            X = f3.view(pairs * L, 3, 512)[:, stacks[0]:stacks[-1] + 1].reshape(pairs * L, K).double()
            ref, S = ref_linear(X, X.abs(), wt[wid], wt[bid])
            r[key] = worst_ratio(y.view(pairs * L, 512), ref, TAU * S)
        else:
            x = d["f"][:, stacks[0]:stacks[-1] + 1].reshape(pairs, K, L).transpose(0, 1).reshape(K, pairs * L)
            ref, T = contraction_bound(wt[wid], x.double(), wt[bid])
            r[key] = worst_ratio(y.view(pairs, 512, L).transpose(0, 1).reshape(512, pairs * L), ref, T)
        ys[key] = cl(d, y, d["tc"])
    for key in ("yp", "yi", "gp", "gi"):
        if key not in ys:
            assert W.untouched_after(key, 0), f"{key} written by fusion {arch}"
    return ys


def check_norms(d, r, ys):
    """Both GroupNorm affines from the stored y, the surviving statistics -> {branch: (sc, sh) [pairs][512]}."""
    W, wt, pairs, L, arch, grp = d["W"], d["wt"], d["pairs"], d["L"], d["arch"], d["grp"]
    aff = {}
    for b, gid, bid, _ in NORMS[arch]:
        sc, sh = (W.owned(f"{k}{b}", pairs * 512).view(pairs, 512) for k in ("sc", "sh"))
        a, s, Ta, Ts = affine_bound(gn_stats(ys[f"y{b}"].double(), grp, pairs), wt[gid], wt[bid])
        r[f"sc{b}_sh{b}"] = max(worst_ratio(sc, a, Ta), worst_ratio(sh, s, Ts))
        aff[b] = (sc, sh)
    if arch == "A":
        for k in ("sci", "shi"):
            assert W.untouched_after(k, 0), f"{k} written by fusion A"
    # the last branch's statistics survive: bit for bit from the stored partials, against the stored y, then its affine
    b, gid, bid, _ = NORMS[arch][-1]
    k, tpg = (2, -(-L // BN)) if d["tc"] else (1, -(-L // 128))
    part = W.owned("part", pairs * tpg * k * 512 * 2, torch.float64).view(pairs * tpg * k, 512, 2)
    stats = W.owned("stats", pairs * 512 * 2, torch.float64).view(pairs, 512, 2)
    want = reduce_ref(part, [(p * tpg * k, (p + 1) * tpg * k) for p in range(pairs)])
    assert torch.equal(stats, want), "stats: not stats_reduce's fixed-order sum of the stored partials"
    rv, rm, _ = stats_ratios(stats[..., 0], stats[..., 1], ys[f"y{b}"].double(), grp, pairs)
    r["stats"] = max(rv, rm)
    a, s, Ta, Ts = gn_affine(stats, wt[gid], wt[bid], L)
    r["stats_affine"] = max(worst_ratio(aff[b][0], a, Ta), worst_ratio(aff[b][1], s, Ts))
    return aff


def check_combine(d, r, ys, aff):
    """The fused stack 2 from the stored y, g, sc, sh; F3's stack 2 equals it (check_f3)."""
    arch, grp = d["arch"], d["grp"]
    nv = lambda b: ys[f"y{b}"].double() * aff[b][0][grp].double() + aff[b][1][grp].double()
    gates = {}
    if arch == "C":
        gates = dict(gp=ys["gp"].double(), gi=ys["gi"].double())
        assert float(torch.maximum(gates["gp"].abs(), gates["gi"].abs()).max()) < 80, "gate logits outside +-80"
        one = ((gates["gp"] > 17.4) & (gates["gi"] < -27.6)) | ((gates["gi"] > 17.4) & (gates["gp"] < -27.6))
        d["saturated"] = float(one.double().mean())
    ref, T = combine_ref(arch, nv("p"), nv("i") if arch != "A" else None, **gates)
    r["combine"] = worst_ratio(cl(d, d["f"][:, 2], False), ref, T)


def check_wdet(d, r, f3):
    """w_det layers 1 and 2: h1 from the stored F3 (TC) or feats (FP32), h2 from the stored h1."""
    W, wt, pairs, L = d["W"], d["wt"], d["pairs"], d["L"]
    rows = pairs * L * 3
    h1 = W.owned("h1", rows * 512)
    h2 = W.owned("h2", rows * 256)
    if d["tc"]:
        h1, h2 = h1.view(rows, 512), h2.view(rows, 256)
        for key, x, y, w, b in (("h1", f3, h1, "WD_W1T", "WD_B1"), ("h2", h1, h2, "WD_W2T", "WD_B2")):
            X = x.double()
            ref, S = ref_linear(X, X.abs(), wt[w], wt[b])
            r[key] = worst_ratio(y, ref.clamp_min(0), TAU * S)
    else:
        G = 3 * pairs
        cm = lambda v, C: v.view(G, C, L).transpose(0, 1).reshape(C, G * L)        # [C][g*L + l]
        for key, x, y, w, b, C in (("h1", d["f"].reshape(-1), h1, "WD_W1T", "WD_B1", 512),
                                   ("h2", h1, h2, "WD_W2T", "WD_B2", 256)):
            ref, T = contraction_bound(wt[w], cm(x, 512).double(), wt[b], relu=True)
            r[key] = worst_ratio(cm(y, C), ref, T)


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fusion_stage_vs_fp64(case):
    """mmmot_fusion_det_fwd, then every kernel up to h2 against fp64 of its own stored inputs (module docstring)."""
    lib = _lib.load()
    d = _run(lib, case)
    r = {}
    f3 = check_f3(d, r)
    ys = check_linears(d, r, f3)
    aff = check_norms(d, r, ys)
    check_combine(d, r, ys, aff)
    check_wdet(d, r, f3)
    assert set(r) == set(CHECKS[d["arch"]]), sorted(r)
    extra = {"saturated": d["saturated"]} if "saturated" in d else {}
    report(f"fusion stage {case[0]} {d['arch']} L={d['L']} pairs={d['pairs']} [{'tc' if d['tc'] else 'fp32'}] (err / bound)",
           **r, **extra)
    if case[5]:
        assert d["saturated"] > 0, "no element with one gate rounding to 1 and the other below 1e-12"
    assert all(v <= 1.0 for v in r.values()), r


# ------------------------------------------------------------------------------------------------ CPU
def test_case_coverage():
    """The GPU cases run every architecture on each path and each engine setting, every L of the grid with 1 and 3
    pairs on both paths, auto on both sides of L = 64, 300 = 256 + 44 rows and 9 x 32 + 12 columns, the cfg2-cfg4
    per-pair shapes, and the saturating gates on both paths."""
    path = {c[0]: fd_path(c[2], c[4]) for c in CASES}
    assert {(c[1], path[c[0]], c[4]) for c in CASES} >= {(a, p, e) for a in "ABC" for p, e in
                                                        (("fp32", "fp32"), ("tc", "tc"), ("fp32", "auto"), ("tc", "auto"))}
    for p in ("fp32", "tc"):
        assert {(c[2], c[3]) for c in CASES if path[c[0]] == p} >= {(L, n) for L in LS for n in (1, 3)}, p
        assert {c[1] for c in CASES if c[5] and path[c[0]] == p} == {"C"}, p
    auto = {c[2]: path[c[0]] for c in CASES if c[4] == "auto"}
    assert auto[63] == "fp32" and auto[64] == "tc"
    assert 300 % BN == 44 and 300 % 32 == 12 and 31 % 32 == 31 and 33 % 32 == 1
    assert {(c[1], c[2], path[c[0]]) for c in CASES if c[0].startswith("cfg")} == {("A", 64, "tc"), ("C", 128, "tc"),
                                                                                   ("C", 256, "tc")}
    assert all(2 <= c[3] <= 4 for c in CASES if c[0].startswith("cfg"))


# The functions the stage runs and, per function, every kernel launch and helper call in its body, in source order, with
# the checks that hold its output: this file's CHECKS or tests/test_heads.py's HEAD_CHECKS.
FD_HELPERS = ("gemm_gen_launch", "gemm_simt_launch", "stats_reduce", "gn_finalize")
LINEAR_CHECKS = ("yp", "yi", "gp", "gi")
NORM_CHECKS = ("scp_shp", "sci_shi", "stats_affine")
LAUNCH_SITES = {
    "fusion_det_tc": [
        ("feats_to_rows_kernel", ("f3",)), ("gemm_gen_launch", LINEAR_CHECKS), ("stats_reduce", ("stats",)),
        ("gn_finalize", NORM_CHECKS), ("fusion_combine_rows_kernel", ("combine", "f3")),
        ("gemm_gen_launch", ("h1",)), ("gemm_gen_launch", ("h2",)), ("det_score_rows_kernel", ("det",)),
    ],
    "fusion_det_fp32": [
        ("gemm_simt_launch", LINEAR_CHECKS), ("stats_reduce", ("stats",)), ("gn_finalize", NORM_CHECKS),
        ("fusion_combine_kernel", ("combine",)), ("gemm_simt_launch", ("h1",)), ("gemm_simt_launch", ("h2",)),
        ("det_score_kernel", ("det",)),
    ],
}


def test_stage_functions_launch_coverage_guard():
    """Every launch in the functions the stage runs maps to a check: a launch added, removed or reordered without its
    entry in LAUNCH_SITES fails here; every check named there is one the GPU test fills, and every check is named."""
    for func, sites in LAUNCH_SITES.items():
        assert impl_launches("fusion_det.cu", func, FD_HELPERS) == [s[0] for s in sites], func
    named = {c for sites in LAUNCH_SITES.values() for _, cs in sites for c in cs}
    every = set(CHECKS["C"]) | set(HEAD_CHECKS)
    assert named == every, named ^ every
    heads = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_heads.py")).read()
    for c in HEAD_CHECKS:
        assert f'r["{c}"]' in heads, c


def _fp32_affine(y32, grp, G, gamma, beta, unbiased=False):
    """GroupNorm(C, C)'s affine in plain fp32 evaluation (fp64 statistics of the fp32 values, rounded once); unbiased:
    the variance over n - 1 (a planted defect)."""
    n, mean, var, _, _ = group_moments(y32.double(), grp, G)
    if unbiased:
        var = var * n / (n - 1)
    a = gamma / torch.sqrt(var + 1e-5)
    return a.float(), (beta - mean * a).float()


def test_bounds_reject_planted_defects():
    """Each bound accepts a plain fp32 evaluation and rejects its planted defect by more than 10x (module docstring)."""
    t = prepare(synthetic_state_dict("C", seed=43), "C")[0]
    w = lambda k: t[W[k]].double()
    g = torch.Generator().manual_seed(17)
    out = {}
    # a linear missing K chunk 32..63 (input_p over 64 detections), against the TC and the FP32 bounds
    X = torch.relu(torch.randn(64, 512, generator=g))
    Wp, bp = w("FU_WPT"), w("FU_BP")
    ref, S = ref_linear(X.double(), X.double().abs(), Wp, bp)
    refc, T = contraction_bound(Wp, X.double().T.contiguous(), bp)
    drop = X.clone()
    drop[:, 32:64] = 0
    for tag, x in (("fp32", X), ("K chunk dropped", drop)):
        y = x @ Wp.float() + bp.float()
        out[f"linear {tag}"] = worst_ratio(y, ref, TAU * S)
        out[f"linear chain {tag}"] = worst_ratio(y.T, refc, T)
    # GroupNorm(512, 512) over L = 300 detections of two pairs with the variance over L - 1
    L, pairs = 300, 2
    grp = torch.arange(pairs * L) // L
    y = (torch.randn(pairs * L, 512, generator=g) * 0.7 + torch.randn(512, generator=g)).float()
    a, s, Ta, Ts = affine_bound(gn_stats(y.double(), grp, pairs), w("FU_GPW"), w("FU_GPB"))
    for tag, unb in (("fp32", False), ("var / (L-1)", True)):
        sc, sh = _fp32_affine(y, grp, pairs, w("FU_GPW"), w("FU_GPB"), unbiased=unb)
        out[f"affine {tag}"] = max(worst_ratio(sc, a, Ta), worst_ratio(sh, s, Ts))
    # the combine C with gp and gi swapped, at ordinary gates and at gates near +-30 of opposite signs
    sign = torch.ones(512)
    sign[1::2] = -1
    yp, yi = (torch.randn(256, 512, generator=g) * 0.8 + 0.3 for _ in range(2))
    scp, shp, sci, shi = (torch.rand(512, generator=g) + 0.5 for _ in range(4))
    for gates, (gp, gi) in (("", (torch.randn(256, 512, generator=g) * 2 for _ in range(2))),
                            (" saturating", (torch.randn(256, 512, generator=g) * 4 + SAT * s * sign for s in (1, -1)))):
        v = yp.double() * scp.double() + shp.double()
        u = yi.double() * sci.double() + shi.double()
        ref, T = combine_ref("C", v, u, gp.double(), gi.double())
        for fma in (False, True):
            got = combine_fp32("C", yp, scp, shp, yi, sci, shi, gp, gi, fma=fma)
            out[f"combine fp32{gates}{' fma' if fma else ''}"] = worst_ratio(got, ref, T)
        out[f"combine gp, gi swapped{gates}"] = worst_ratio(combine_fp32("C", yp, scp, shp, yi, sci, shi, gi, gp), ref, T)
    for arch in ("A", "B"):
        ref, T = combine_ref(arch, v, u)
        out[f"combine fp32 {arch}"] = worst_ratio(combine_fp32(arch, yp, scp, shp, yi, sci, shi), ref, T)
    # w_det layer 1 over the F3 rows of 2 pairs x 50 detections (300 rows: a 256-row tile and a 44-row tail)
    pairs, L = 2, 50
    F3 = torch.relu(torch.randn(pairs, L, 3, 512, generator=g))
    W1, b1 = w("WD_W1T"), w("WD_B1")
    X = F3.reshape(-1, 512)
    ref, S = ref_linear(X.double(), X.double().abs(), W1, b1)
    ref = ref.clamp_min(0)
    h1 = lambda x: torch.relu(x @ W1.float() + b1.float())
    out["h1 fp32"] = worst_ratio(h1(X), ref, TAU * S)
    nb = F3.clone()
    nb[:, :, 2] = F3[:, :, 2].roll(-1, 1)                               # stack 2 of detection l + 1
    out["h1 stack 2 of the next detection"] = worst_ratio(h1(nb.reshape(-1, 512)), ref, TAU * S)
    sh1 = X.clone()
    sh1[:BN] = X[1:BN + 1]                                              # the first tile one stack late
    out["h1 tile shifted by one stack"] = worst_ratio(h1(sh1), ref, TAU * S)
    report("planted defects (err / bound)", **out)
    ok = [k for k in out if "fp32" in k]
    assert max(out[k] for k in ok) <= 1.0, {k: out[k] for k in ok}
    assert min(v for k, v in out.items() if k not in ok) > 10.0, out
