"""Training-mode stages on the FP32 engine against oracle/train_ref.py in float64, per channel and element by element.

In training every contraction runs on the FP32 FFMA engine: the 13 VGG convolutions (XM_CONV3) with their BatchNorm
batch statistics, and w_det (XM_DIRECT, then XM_NORM_RELU) with its two BatchNorm1d layers and raw logits.  The
statistics are compared per channel, each against its own scale (|dmean| against the channel's mean |y|, |dvar|
against its own variance), so a channel whose variance is far below the layer's largest is held as tightly as any.

w_det: derived bound.  Layer 1's outputs carry at most T1, the contraction bound of the FP32 engine
(kernel_kit.contraction_bound).  BatchNorm over n = 3L columns then gives, to first order and with the statistics bound
of kernel_kit.stats_ratios for the fp32 runs of the partials and u for the export to fp32,
    |dmean| <= mean(T) + KAPPA1 u mean|y| + u |mean|,
    |dvar|  <= 2 mean(|y - mean| T) + mean(T^2) + KAPPA u (|mean| mean|y - mean| + var) + u var,
and the normalised, rectified output h = relu(gamma (y - mean) rstd + beta) carries
    Th = |gamma| rstd (T + |dmean| + |y - mean| |dvar| / (2 (var + eps))) + 8 u (|y sc| + |sh| + |z|),
the last term the fp32 roundings of sc, sh and the fma (as in test_norm_stats._gn_bound).  Layer 2 carries |W2|^T Th
plus its own contraction bound, and the logits (det_logit_kernel: b3, then 256 fmas) |w3|^T Th2 + 1.01 * 257 u (|b3| +
sum |w3 h2|).

VGG trunk: measured tolerance.  The same first-order propagation through 13 convolutions multiplies the bound by
sum_k |w| (about 0.8 sqrt(K), up to 54 at K = 4608) per layer while the error itself grows like the weights' spectral
scale, so a derived bound is useless past the first layers.  The trunk's statistics are therefore held to TAU_MEAN and
TAU_VAR, relative per channel, set at about 20 times the worst ratio measured on an H100 SXM (700 W limit) over the
cases below (printed by every case).  A channel 1 % off fails them by two orders of magnitude (CPU check below).

PointNet at L >= 16 runs on the FP32 engine only in training (the eval path takes the tensor cores from L = 16): its
output is held to the project's parity metric (helpers.check_close, 1e-4) against torch_ref.pointnet in float64 with the
same head Dropout mask.  The running averages after one TrackingNet.train() forward are checked per element and per
channel against train_ref.running_after, with the batch tolerances above scaled by the update's weights.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import mmmot_b200
from kernel_kit import EPS, KAPPA, KAPPA1, U, case_seed, contraction_bound, eval_net, report, vp, worst_ratio
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict

gpu = pytest.mark.gpu
TAU_MEAN, TAU_VAR = 2e-5, 6e-5     # measured worst: 1.1e-6 (mean, 64 px, L = 24), 3.0e-6 (var)


def _net(seed=17):
    net, sd = eval_net("C", seed)
    return net, {k: v.double().cuda() if v.is_floating_point() else v for k, v in sd.items()}


def bn_propagate(y, T, gamma, beta):
    """Training BatchNorm + ReLU over y [C][n] (fp64 reference) whose kernel values err by at most T [C][n] -> mean,
    var, their bounds tm, tv, h = relu(BN(y)) and its bound Th (module docstring)."""
    m = y.mean(1, keepdim=True)
    dev = y - m
    v = (dev * dev).mean(1, keepdim=True)
    tm = T.mean(1, keepdim=True) + KAPPA1 * U * y.abs().mean(1, keepdim=True) + U * m.abs()
    tv = (2 * (dev.abs() * T).mean(1, keepdim=True) + (T * T).mean(1, keepdim=True)
          + KAPPA * U * (m.abs() * dev.abs().mean(1, keepdim=True) + v) + U * v)
    rstd = 1 / torch.sqrt(v + EPS)
    sc = gamma[:, None] * rstd
    sh = beta[:, None] - m * sc
    z = y * sc + sh
    Th = gamma.abs()[:, None] * rstd * (T + tm + dev.abs() * tv / (2 * (v + EPS))) + 8 * U * ((y * sc).abs() + sh.abs() + z.abs())
    return m[:, 0], v[:, 0], tm[:, 0], tv[:, 0], z.clamp_min(0), Th


def channel_ratios(mean_k, var_k, mean, var, mean_abs):
    """Worst |dmean| / mean|y| and |dvar| / var over the channels: each channel against its own scale."""
    return float(((mean_k - mean).abs() / mean_abs).max()), float(((var_k - var).abs() / var).max())


def _record_mean_abs(monkeypatch, mabs):
    """Make train_ref's training BatchNorm also record each layer's per-channel mean |y| into mabs[prefix]."""
    from oracle import train_ref
    bn_train = train_ref._bn_train

    def recording(x, sd_, p, st):
        mabs[p] = x.abs().mean([d for d in range(x.dim()) if d != 1])
        return bn_train(x, sd_, p, st)

    monkeypatch.setattr(train_ref, "_bn_train", recording)


def test_channel_tolerance_rejects_one_percent():
    """The per-channel tolerance accepts statistics rounded to fp32 and rejects a 1 % error in the mean or the variance of
    the channel with the smallest variance (10^-6 of the largest) by more than two orders of magnitude, where the
    whole-vector metric max|a - b| / max|ref| stays below 10^-4 and would not see it."""
    g = torch.Generator().manual_seed(3)
    sd = 10 ** (-3 * torch.rand(512, generator=g, dtype=torch.float64))
    sd[7] = 1e-3
    mean = torch.randn(512, generator=g, dtype=torch.float64) * sd * 3
    var = sd * sd
    mabs = mean.abs() + 0.8 * sd                      # mean |y| of a normal channel, near enough for the test
    rm, rv = channel_ratios(mean.float().double(), var.float().double(), mean, var, mabs)
    assert rm <= 0.01 * TAU_MEAN and rv <= 0.01 * TAU_VAR, (rm, rv)
    bad_v = var.clone()
    bad_v[7] *= 1.01
    bad_m = mean.clone()
    bad_m[7] += 0.01 * mabs[7]
    rv = channel_ratios(mean, bad_v, mean, var, mabs)[1]
    rm = channel_ratios(bad_m, var, mean, var, mabs)[0]
    whole = float((bad_v - var).abs().max() / var.abs().max())
    report("tolerance check", var_1pct_over_tol=rv / TAU_VAR, mean_1pct_over_tol=rm / TAU_MEAN, whole_vector_relerr=whole)
    assert rv > 100 * TAU_VAR and rm > 100 * TAU_MEAN and whole < 1e-4


W_DET_LS = (1, 2, 127, 128, 129, 300)


@gpu
@pytest.mark.parametrize("L", W_DET_LS)
def test_w_det_train_vs_fp64(L):
    """mmmot_w_det_train_fwd: both BatchNorm layers' exported batch mean and biased variance per channel, and the raw
    logits element by element, against train_ref.determine_det_train in float64, to the derived bound."""
    from oracle import train_ref
    lib = _lib.load()
    net, sd = _net()
    wts = net.prepared()
    g = torch.Generator().manual_seed(case_seed("w_det train", L))
    feats = torch.randn(3, 512, L, generator=g).cuda()
    det = torch.full((3, L), float("nan"), device="cuda")
    bn = torch.full((2, 2, 512), float("nan"), device="cuda")
    ws = torch.empty(int(lib.mmmot_w_det_train_workspace(L)), dtype=torch.uint8, device="cuda")
    rc = lib.mmmot_w_det_train_fwd(wts.ptr, L, vp(feats), vp(det), vp(bn), vp(ws), ws.numel(), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    stats = {}
    ref = train_ref.determine_det_train(sd, feats.double(), stats)
    # the bound chain, columns (stack, detection)
    x = feats.double().permute(1, 0, 2).reshape(512, 3 * L)
    w1 = sd["w_det.0.weight"][:, :, 0]
    y1, T1 = contraction_bound(w1.T.contiguous(), x, sd["w_det.0.bias"])
    m1, v1, tm1, tv1, h1, Th1 = bn_propagate(y1, T1, sd["w_det.1.weight"], sd["w_det.1.bias"])
    w2 = sd["w_det.3.weight"][:, :, 0]
    y2, T2 = contraction_bound(w2.T.contiguous(), h1, sd["w_det.3.bias"])
    T2 = T2 + w2.abs() @ Th1
    m2, v2, tm2, tv2, h2, Th2 = bn_propagate(y2, T2, sd["w_det.4.weight"], sd["w_det.4.bias"])
    w3, b3 = sd["w_det.6.weight"][0, :, 0], sd["w_det.6.bias"]
    T3 = w3.abs() @ Th2 + 1.01 * 257 * U * (b3.abs() + w3.abs() @ h2)
    for p, (m, v) in (("w_det.1", (m1, v1)), ("w_det.4", (m2, v2))):     # the bound chain computes what the oracle does
        assert torch.allclose(stats[p][0], m, rtol=1e-12, atol=1e-12) and torch.allclose(stats[p][1], v, rtol=1e-12, atol=1e-12)
    got = det.double()
    assert bool(torch.isfinite(got).all())
    r = dict(mean1=float(((bn[0, 0].double() - m1).abs() / tm1).max()), var1=float(((bn[0, 1].double() - v1).abs() / tv1).max()),
             mean2=float(((bn[1, 0, :256].double() - m2).abs() / tm2).max()),
             var2=float(((bn[1, 1, :256].double() - v2).abs() / tv2).max()),
             logits=worst_ratio(got.reshape(-1), ref.reshape(-1), T3))
    report(f"w_det train L={L} (err / bound)", **r)
    assert all(val <= 1.0 for val in r.values()), r


APP_CASES = [(64, 24, 0), (64, 24, 5), (224, 6, 0), (224, 6, 5)]


@gpu
@pytest.mark.parametrize("hw,L,drop", APP_CASES, ids=[f"{a}px-L{b}-drop{c}" for a, b, c in APP_CASES])
def test_appearance_train_vs_fp64(hw, L, drop, monkeypatch):
    """mmmot_appearance_train_fwd: all 13 layers' exported batch mean and biased variance per channel against
    train_ref.appearance_train in float64 (TAU_MEAN, TAU_VAR), and the stack-0 features with check_close; DropBlock
    masks of the two deepest heads drawn as the reference draws them."""
    from helpers import TOL, check_close
    from oracle import train_ref
    lib = _lib.load()
    net, sd = _net()
    wts = net.prepared()
    crops = synthetic_pair(L // 2, L - L // 2, 16, hw, seed=case_seed("app", hw, L) % 1000)[0].float().cuda()
    dm2 = dm3 = None
    if drop:
        torch.manual_seed(case_seed("drop", hw, L))
        dm2 = net._dropblock_weights(L, hw // 16, hw // 16, drop).cuda()
        dm3 = net._dropblock_weights(L, hw // 32, hw // 32, drop).cuda()
    feats = torch.full((1, 3, 512, L), float("nan"), device="cuda")
    bn = torch.full((13, 2, 512), float("nan"), device="cuda")
    ws = torch.empty(int(lib.mmmot_appearance_train_workspace(L, hw, hw)), dtype=torch.uint8, device="cuda")
    rc = lib.mmmot_appearance_train_fwd(wts.ptr, vp(crops), L, hw, hw, L, vp(feats), vp(bn), vp(dm2), vp(dm3), vp(ws),
                                        ws.numel(), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    stats, mabs = {}, {}
    _record_mean_abs(monkeypatch, mabs)
    if drop:
        torch.manual_seed(case_seed("drop", hw, L))
    ref = train_ref.appearance_train(sd, crops.double(), stats, drop)
    worst_m = worst_v = 0.0
    per_layer = {}
    for i, p in enumerate(net._VGG_BN):
        m, v, _ = stats[p]
        C = m.numel()
        rm, rv = channel_ratios(bn[i, 0, :C].double(), bn[i, 1, :C].double(), m, v, mabs[p])
        per_layer[f"L{i}"] = max(rm / TAU_MEAN, rv / TAU_VAR)
        worst_m, worst_v = max(worst_m, rm), max(worst_v, rv)
    rep = []
    check_close(feats[0, 0], ref.T, TOL, "stack 0", rep)
    report(f"appearance train {hw}px L={L} dropblock={drop}", mean_rel=worst_m, var_rel=worst_v,
           stack0_err=rep[0][1], stack0_worst=rep[0][3])
    report("  per layer (worst ratio to tolerance)", **per_layer)
    assert worst_m <= TAU_MEAN and worst_v <= TAU_VAR, per_layer


PN_CASES = [(L, mask) for L in (16, 40) for mask in (False, True)]


@gpu
@pytest.mark.parametrize("L,mask", PN_CASES, ids=[f"L{L}-{'mask' if k else 'nomask'}" for L, k in PN_CASES])
def test_pointnet_train_vs_fp64(L, mask, monkeypatch):
    """mmmot_pointnet_train_fwd at L >= 16, where only training runs PointNet on the FP32 engine (the eval path takes the
    tensor cores): about 512 points per detection, ragged, with 1-point detections; stack 1 against torch_ref.pointnet in
    float64 with the same head Dropout mask, by check_close (the project's 1e-4 parity metric, element-wise too)."""
    from helpers import TOL, check_close
    from oracle import torch_ref
    lib = _lib.load()
    net, sd = _net()
    wts = net.prepared()
    g = torch.Generator().manual_seed(case_seed("pointnet train", L, mask))
    cnt = torch.randint(1, 1024, (L,), generator=g)
    cnt[[0, L // 2, L - 1]] = 1
    split = torch.zeros(L + 1, dtype=torch.int32)
    split[1:] = torch.cumsum(cnt, 0)
    P = int(split[-1])
    centre = torch.rand(L, 3, generator=g) * torch.tensor([60.0, 40.0, 2.0]) + torch.tensor([0.0, -20.0, -2.0])
    points = (torch.randn(P, 3, generator=g) * torch.tensor([2.0, 1.0, 0.8]) + centre.repeat_interleave(cnt, 0)).cuda()
    hmask = None
    if mask:
        torch.manual_seed(case_seed("head mask", L))
        hmask = F.dropout(torch.ones(512, P, device="cuda"), p=0.5, training=True)
    feats = torch.full((1, 3, 512, L), float("nan"), device="cuda")
    ws = torch.empty(int(lib.mmmot_pointnet_train_workspace(1, L, P)), dtype=torch.uint8, device="cuda")
    hs = split.numpy()
    rc = lib.mmmot_pointnet_train_fwd(wts.ptr, vp(points), vp(split.cuda()), ctypes.c_void_p(hs.ctypes.data), 1, L,
                                      vp(hmask), vp(feats), vp(ws), ws.numel(), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    if mask:   # the reference's nn.Dropout, applied with the same mask
        m64 = hmask.double()
        monkeypatch.setattr(F, "dropout", lambda x, p=0.5, training=True: x * m64)
    ref = torch_ref.pointnet(sd, points.double().T[None], split.long().cuda(), dropout=mask)[0]
    assert bool(torch.isfinite(feats[0, 1]).all())
    rep = []
    check_close(feats[0, 1], ref.T, TOL, "stack 1", rep)
    report(f"pointnet train L={L} P={P} mask={mask}", err=rep[0][1], outside=rep[0][2], worst=rep[0][3])


# running-average update: per-layer count L h w (VGG) or 3 L (w_det), unbiased factor count / (count - 1), momentum 0.1
RUN_CASES = [(224, 3, 3), (64, 12, 12)]
TAU_WDET = 1.5e-4    # measured worst 6.7e-6 (w_det.4, 224 px): about 20x, as TAU_MEAN / TAU_VAR


@gpu
@pytest.mark.parametrize("hw,n,m", RUN_CASES, ids=[f"{a}px-{b}x{c}" for a, b, c in RUN_CASES])
def test_running_averages_vs_fp64(hw, n, m, monkeypatch):
    """One TrackingNet.train() forward: all 15 BatchNorm layers' running_mean / running_var element by element against
    train_ref.running_after over train_ref.forward_train in float64, and num_batches_tracked == 1.  Per channel, the
    batch part of the update (0.1 of the batch statistic, times count / (count - 1) for the variance) to the batch
    tolerance relative to the channel's own mean |y| or variance, plus 4 u of the fp32 update's operands: TAU_MEAN /
    TAU_VAR for the VGG trunk, TAU_WDET for w_det, whose input features carry the whole forward's error."""
    from oracle import train_ref
    sd0 = synthetic_state_dict("C", seed=23)
    net = mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch="C",
                                 affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2, test_mode=2,
                                 dropblock=0, use_dropout=False)
    net.load_state_dict(sd0)
    net.cuda().train()
    dets, info, split = synthetic_pair(n, m, 64, hw, seed=case_seed("running", hw) % 1000, ragged=True)
    net(dets.cuda(), {k: v.cuda() for k, v in info.items()}, split)
    torch.cuda.synchronize()
    after = net.state_dict()
    sd = {k: v.double().cuda() if v.is_floating_point() else v for k, v in sd0.items()}
    mabs = {}
    _record_mean_abs(monkeypatch, mabs)
    _, stats = train_ref.forward_train(sd, dets.double().cuda(), {k: v.double().cuda() for k, v in info.items()}, split, "C",
                                       "minus_abs", "dual_add", dropblock=0, use_dropout=False)
    run = train_ref.running_after(sd, stats)
    prefixes = net._VGG_BN + ["w_det.1", "w_det.4"]
    assert set(stats) == set(prefixes)
    worst = {}
    for p in prefixes:
        mean, var, cnt = stats[p]
        f = cnt / (cnt - 1)
        tm_, tv_ = (TAU_WDET, TAU_WDET) if p.startswith("w_det") else (TAU_MEAN, TAU_VAR)
        r0m, r0v = sd[p + ".running_mean"], sd[p + ".running_var"]
        bm = 0.1 * tm_ * mabs[p] + 4 * U * (r0m.abs() + mean.abs())
        bv = 0.1 * f * tv_ * var + 4 * U * (r0v.abs() + f * var)
        rm = float(((after[p + ".running_mean"].double() - run[p + ".running_mean"]).abs() / bm).max())
        rv = float(((after[p + ".running_var"].double() - run[p + ".running_var"]).abs() / bv).max())
        worst[p] = max(rm, rv)
        assert int(after[p + ".num_batches_tracked"]) == int(sd0[p + ".num_batches_tracked"]) + 1, p
    report(f"running averages {hw}px L={n + m} (err / bound)", **{p.replace("appearance.layers.", "vgg"): v for p, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst
