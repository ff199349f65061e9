"""Checkpoint -> prepared device weights (one-time, per load_state_dict / .cuda()).

Takes the reference-format ``state_dict`` (263 keys, see schema.py) and produces the tensors the
C ABI expects (``enum mmmot_weight_id`` in include/mmmot_b200.h):

* eval-mode BatchNorm folded into the preceding conv (VGG trunk: modules/vgg.py:67-80; w_det:
  modules/tracking_net.py:92-100);
* the two STN transforms, which are input-independent constants at inference (SURVEY F4;
  modules/point_net.py:63-66,72-86), folded into PointNet conv1, conv2 and the head conv;
* the 1088-wide head conv (modules/point_net.py:13,27-28) split into its 64 local and 1024
  per-detection-global columns (SURVEY B-9);
* affinity conv1.0 and new/end conv0 stacked into one 512 -> 1024 matrix (same input tensor);
* every matrix transposed to Wt[K][Cout];
* a net narrower than 512 (appear_len = point_len = 256 or 128) embedded in an equivalent 512-wide one first
  (embed_width), so the same operands and kernels run it.

The folding is done once in fp64 on the host and rounded to fp32; it is checkpoint conversion,
not part of the per-frame path.
"""
import ctypes

import torch

from . import _lib
from .schema import D, RES_SKIP_CHANNELS, RESNET_BLOCKS, SKIP_CHANNELS, SKIP_OUT, VGG_STAGES, resnet_convs, state_schema

EPS = 1e-5
W = _lib.W


def stn_constant(sd, p, k):
    """I + reshape(W_out relu(beta_fc_bn2) + b_out): what STN3d.forward returns for ANY input at
    batch size 1 (modules/point_net.py:80-86 with fc_bn2 = GroupNorm(256,256) on one value/group)."""
    v = torch.relu(sd[f"{p}.fc_bn2.bias"].double())
    out = sd[f"{p}.output.weight"].double() @ v + sd[f"{p}.output.bias"].double()
    return out.reshape(k, k) + sd[f"{p}.idt"].double()


def _fold_bn(sd, conv, bn):
    w = sd[f"{conv}.weight"].double()
    b = sd[f"{conv}.bias"].double()
    s = sd[f"{bn}.weight"].double() / torch.sqrt(sd[f"{bn}.running_var"].double() + EPS)
    w = w * s.reshape(-1, *([1] * (w.dim() - 1)))
    b = (b - sd[f"{bn}.running_mean"].double()) * s + sd[f"{bn}.bias"].double()
    return w, b


def pack_tc(wt):
    """Wt[K][M] (fp32/fp64) -> (uint8 tensor, out_scale): the tensor-core operand tiles of W = Wt^T,
    [k chunk 32][m tile 128][hi|lo][k group 4][m group 16][8 rows][8 k] fp16, zero padded.
    W is pre-scaled by 2^s (max |W 2^s| <= 2048) so that lo = fp16(w - hi) stays in fp16's normal
    range; hi = fp16(w) (round-to-nearest-even): w = hi + lo to 2^-22 relative.  out_scale = 2^-s
    is applied to the fp32 accumulators in the epilogue (exact)."""
    import math
    w = wt.t().double().contiguous()                      # [M][K]
    M, K = w.shape
    amax = float(w.abs().max())
    sexp = int(math.floor(math.log2(2048.0 / amax))) if amax > 0 else 0
    w = (w * (2.0 ** sexp)).float()
    mt, kc = (M + 127) // 128, (K + 31) // 32
    pad = torch.zeros(mt * 128, kc * 32, dtype=torch.float32)
    pad[:M, :K] = w
    hi = pad.to(torch.float16)
    lo = (pad - hi.float()).to(torch.float16)
    both = torch.stack([hi, lo], 0).view(2, mt, 16, 8, kc, 4, 8)      # hl, mt, mg, r, kc, kg, e
    both = both.permute(4, 1, 0, 5, 2, 3, 6).contiguous()              # kc, mt, hl, kg, mg, r, e
    return both.view(torch.int16).reshape(-1).view(torch.uint8), 2.0 ** (-sexp)


def pack_px(packed_u8, M, K):
    """The compact N = 64 form of a pack_tc() result for the pixel-major kernel (64-output layers): rows 0..63 only,
    [k chunk][k group 4][hi rows | lo rows][row group 8][8 rows][8 k] fp16 = 8 KB per k chunk.  One bulk copy per chunk,
    and per k group the 64 hi rows are followed by the 64 lo rows (one copy for both).  The pixel-major kernel
    (csrc/gemm_tma_px.cuh) issues X_hi * W_hi and X_hi * W_lo as two m64n64 wgmmas whose B descriptors start at the
    hi rows and 8 row groups later at the lo rows."""
    assert M == 64
    kc = (K + 31) // 32
    t = packed_u8.view(torch.int16).view(kc, 1, 2, 4, 16, 8, 8)          # kc, mt, hl, kg, mg, r, e
    return t[:, 0, :, :, :8].permute(0, 2, 1, 3, 4, 5).contiguous().reshape(-1).view(torch.uint8)   # kc, kg, hl, mg, r, e


def _skip_heads(sd, out, channels):
    """The four SkipPool heads' 10 tensors each (the layout of MMMOT_W_SKIP0) -> out[10 s + j]."""
    f64 = lambda k: sd[k].double()
    for s, c in enumerate(channels):
        p = f"appearance.global_pool.{s}.fc"
        base = 10 * s
        out[base + 0] = f64(f"{p}.0.weight"); out[base + 1] = f64(f"{p}.0.bias")
        out[base + 2] = f64(f"{p}.1.weight").reshape(-1, c).t(); out[base + 3] = f64(f"{p}.1.bias")
        out[base + 4] = f64(f"{p}.2.weight"); out[base + 5] = f64(f"{p}.2.bias")
        w2 = f64(f"{p}.4.weight")
        out[base + 6] = w2.reshape(w2.shape[0], -1).t(); out[base + 7] = f64(f"{p}.4.bias")
        out[base + 8] = f64(f"{p}.5.weight"); out[base + 9] = f64(f"{p}.5.bias")


def fold_bn_nobias(sd, conv, bn):
    """Eval BatchNorm folded into a bias-free conv (torchvision's): w * s, bias = beta - mean * s, in fp64."""
    w = sd[f"{conv}.weight"].double()
    s = sd[f"{bn}.weight"].double() / torch.sqrt(sd[f"{bn}.running_var"].double() + EPS)
    return w * s.reshape(-1, 1, 1, 1), sd[f"{bn}.bias"].double() - sd[f"{bn}.running_mean"].double() * s


def _resnet_trunk(sd, arch):
    convs = []
    for conv, bn, cin, cout, k, _ in resnet_convs(arch):
        w, b = fold_bn_nobias(sd, conv, bn)
        wt = w.permute(2, 3, 1, 0).reshape(k * k * cin, cout)       # [co][ci][ky][kx] -> [(ky*k+kx)*cin + ci][co]
        packed, scale = pack_tc(wt)
        convs.append((wt.contiguous().float(), b.float(), packed, scale))
    return convs


def prepare_resnet(state_dict, arch):
    """ResNet appearance trunk -> (convs, heads): convs in execution order (schema.resnet_convs), each (Wt [K][Cout] fp32,
    bias [Cout] fp32, packed tiles uint8, out_scale) with every BatchNorm folded and the K order of
    mmmot_resnet_weights (1x1: ci; 3x3: (ky*3+kx)*Cin + ci; stem: (ky*7+kx)*3 + ci, packed K zero-padded 147 -> 160);
    heads: the 40 fp32 tensors of the four SkipPool heads, head s at [10 s, 10 s + 10)."""
    sd = {k: v.detach().cpu() for k, v in state_dict.items()}
    convs = _resnet_trunk(sd, arch)
    heads = [None] * 40
    _skip_heads(sd, heads, RES_SKIP_CHANNELS)
    return convs, [t.contiguous().float() for t in heads]


def prepare_fpn(state_dict):
    """The FPN head (mmmot_fpn_weights) -> (laterals, last): laterals[k] = (Wt [C_k][512] fp32, bias [512] fp32, packed
    tiles uint8, out_scale) of fpn_in[k] with its BatchNorm folded (C_k = 256 << k); last = (Wt [512][512] fp32,
    bias [512] fp32) of conv_last.1 with conv_last.2 folded."""
    sd = {k: v.detach().cpu() for k, v in state_dict.items()}
    lats = []
    for k, c in enumerate(RES_SKIP_CHANNELS):
        w, b = fold_bn_nobias(sd, f"appearance.fpn_in.{k}.0", f"appearance.fpn_in.{k}.1")
        wt = w.reshape(-1, c).t()
        packed, scale = pack_tc(wt)
        lats.append((wt.contiguous().float(), b.float(), packed, scale))
    w, b = _fold_bn(sd, "appearance.conv_last.1", "appearance.conv_last.2")
    return lats, (w.reshape(w.shape[0], -1).t().contiguous().float(), b.float())


def prepare(state_dict, fusion, appear_arch="vgg"):
    """-> (list of fp32 CPU tensors indexed by weight id (None = unused), trans1 CxC (C = 3 xyz or 4 xyz +
    reflectance: the checkpoint's point width), trans2 64x64, per-id tensor-core output scales).  With a ResNet
    appearance trunk the VGG and SkipPool ids stay None (prepare_resnet holds that stage's operands)."""
    sd = {k: v.detach().cpu() for k, v in state_dict.items()}
    out = [None] * W["COUNT"]
    f64 = lambda k: sd[k].double()
    vgg = appear_arch == "vgg"

    # VGG trunk
    i = 0
    for s, stage in enumerate(VGG_STAGES if vgg else ()):
        for idx, cin, cout in stage:
            w, b = _fold_bn(sd, f"appearance.layers.{s}.{idx}", f"appearance.layers.{s}.{idx + 1}")
            # [co][ci][ky][kx] -> Wt[(ky*3+kx)*cin + ci][co]
            out[W["VGG_WT0"] + i] = w.permute(2, 3, 1, 0).reshape(9 * cin, cout)
            out[W["VGG_B0"] + i] = b
            i += 1
    # SkipPool heads
    if vgg:
        heads = [None] * 40
        _skip_heads(sd, heads, SKIP_CHANNELS)
        out[W["SKIP0"]:W["SKIP0"] + 40] = heads
    # PointNet trunk with the constant STN transforms folded in:
    #   x' = T1^T x  => conv1(x') = (W1 T1^T) x ;  x_local = T2^T x1 => conv2(x_local) = (W2 T2^T) x1
    pf = "point_net.feat"
    t1 = stn_constant(sd, f"{pf}.stn1", sd[f"{pf}.stn1.idt"].shape[0])     # 3x3 on xyz, 4x4 with reflectance
    t2 = stn_constant(sd, f"{pf}.stn2", 64)
    ws = [f64(f"{pf}.conv{j}.weight").squeeze(-1) for j in range(1, 6)]
    ws[0] = ws[0] @ t1.t()
    ws[1] = ws[1] @ t2.t()
    for j in range(5):
        base = W["PN_L1"] + 4 * j
        out[base + 0] = ws[j].t()
        out[base + 1] = f64(f"{pf}.conv{j + 1}.bias")
        out[base + 2] = f64(f"{pf}.bn{j + 1}.weight")
        out[base + 3] = f64(f"{pf}.bn{j + 1}.bias")
    wh = f64("point_net.conv1.weight").squeeze(-1)            # [512][1088] = [local 64 | global 1024]
    out[W["PN_WHAT"]] = (wh[:, :64] @ t2.t()).t()
    out[W["PN_WHGT"]] = wh[:, 64:].t()
    out[W["PN_BH"]] = f64("point_net.conv1.bias")
    out[W["PN_GHW"]] = f64("point_net.bn1.weight"); out[W["PN_GHB"]] = f64("point_net.bn1.bias")
    out[W["PN_WOT"]] = f64("point_net.conv2.weight").squeeze(-1).t()
    out[W["PN_BO"]] = f64("point_net.conv2.bias")
    out[W["PN_GOW"]] = f64("point_net.bn2.weight"); out[W["PN_GOB"]] = f64("point_net.bn2.bias")
    # fusion
    fm = "fusion_module"

    def lin(name, wt, b, gw=None, gb=None):
        out[W[wt]] = f64(f"{fm}.{name}.0.weight").squeeze(-1).t()
        out[W[b]] = f64(f"{fm}.{name}.0.bias")
        if gw:
            out[W[gw]] = f64(f"{fm}.{name}.1.weight"); out[W[gb]] = f64(f"{fm}.{name}.1.bias")
    if fusion == "A":
        lin("input_w", "FU_WPT", "FU_BP", "FU_GPW", "FU_GPB")
    else:
        lin("input_p", "FU_WPT", "FU_BP", "FU_GPW", "FU_GPB")
        lin("input_i", "FU_WIT", "FU_BI", "FU_GIW", "FU_GIB")
        if fusion == "C":
            lin("gate_p", "FU_GATE_PT", "FU_GATE_PB")
            lin("gate_i", "FU_GATE_IT", "FU_GATE_IB")
    # w_det
    w1, b1 = _fold_bn(sd, "w_det.0", "w_det.1")
    w2, b2 = _fold_bn(sd, "w_det.3", "w_det.4")
    out[W["WD_W1T"]] = w1.squeeze(-1).t(); out[W["WD_B1"]] = b1
    out[W["WD_W2T"]] = w2.squeeze(-1).t(); out[W["WD_B2"]] = b2
    out[W["WD_W3"]] = f64("w_det.6.weight").reshape(-1); out[W["WD_B3"]] = f64("w_det.6.bias")
    # affinity + new/end
    c10 = f64("w_link.conv1.0.weight").reshape(512, 512)
    c0 = f64("w_link.w_new_end.conv0.0.weight").reshape(512, 512)
    out[W["AF_W01T"]] = torch.cat([c10, c0], 0).t()
    out[W["AF_B01"]] = torch.cat([f64("w_link.conv1.0.bias"), f64("w_link.w_new_end.conv0.0.bias")])
    out[W["AF_G1W"]] = f64("w_link.conv1.1.weight"); out[W["AF_G1B"]] = f64("w_link.conv1.1.bias")
    out[W["AF_G0W"]] = f64("w_link.w_new_end.conv0.1.weight"); out[W["AF_G0B"]] = f64("w_link.w_new_end.conv0.1.bias")
    out[W["AF_W2T"]] = f64("w_link.conv1.3.weight").reshape(512, 512).t(); out[W["AF_B2"]] = f64("w_link.conv1.3.bias")
    out[W["AF_G2W"]] = f64("w_link.conv1.4.weight"); out[W["AF_G2B"]] = f64("w_link.conv1.4.bias")
    out[W["AF_W3T"]] = f64("w_link.conv1.6.weight").reshape(128, 512).t(); out[W["AF_B3"]] = f64("w_link.conv1.6.bias")
    out[W["AF_G3W"]] = f64("w_link.conv1.7.weight"); out[W["AF_G3B"]] = f64("w_link.conv1.7.bias")
    out[W["AF_W4"]] = f64("w_link.conv1.9.weight").reshape(-1); out[W["AF_B4"]] = f64("w_link.conv1.9.bias")
    ne = "w_link.w_new_end.conv1"
    out[W["NE_W1T"]] = f64(f"{ne}.0.weight").squeeze(-1).t(); out[W["NE_B1"]] = f64(f"{ne}.0.bias")
    out[W["NE_G1W"]] = f64(f"{ne}.1.weight"); out[W["NE_G1B"]] = f64(f"{ne}.1.bias")
    out[W["NE_W2T"]] = f64(f"{ne}.3.weight").squeeze(-1).t(); out[W["NE_B2"]] = f64(f"{ne}.3.bias")
    out[W["NE_G2W"]] = f64(f"{ne}.4.weight"); out[W["NE_G2B"]] = f64(f"{ne}.4.bias")
    out[W["NE_W3"]] = f64(f"{ne}.6.weight").reshape(-1); out[W["NE_B3"]] = f64(f"{ne}.6.bias")

    # training-mode operands (SURVEY 8f N4): unfolded conv weights + BatchNorm affines of the layers whose BatchNorm
    # uses batch statistics in .train() (VGG trunk, w_det)
    i = 0
    for s_, stage in enumerate(VGG_STAGES if vgg else ()):
        for idx, cin, cout in stage:
            cp, bp = f"appearance.layers.{s_}.{idx}", f"appearance.layers.{s_}.{idx + 1}"
            out[W["VGG_RAWW0"] + i] = f64(f"{cp}.weight").permute(2, 3, 1, 0).reshape(9 * cin, cout)
            out[W["VGG_RAWB0"] + i] = f64(f"{cp}.bias")
            out[W["VGG_BNW0"] + i] = f64(f"{bp}.weight")
            out[W["VGG_BNB0"] + i] = f64(f"{bp}.bias")
            i += 1
    r0 = W["WD_RAW0"]
    out[r0 + 0] = f64("w_det.0.weight").squeeze(-1).t(); out[r0 + 1] = f64("w_det.0.bias")
    out[r0 + 2] = f64("w_det.1.weight"); out[r0 + 3] = f64("w_det.1.bias")
    out[r0 + 4] = f64("w_det.3.weight").squeeze(-1).t(); out[r0 + 5] = f64("w_det.3.bias")
    out[r0 + 6] = f64("w_det.4.weight"); out[r0 + 7] = f64("w_det.4.bias")

    out = [None if t is None else t.contiguous().float() for t in out]
    # tensor-core operand tiles (bytes, viewed as float32 words for the flat buffer)
    scales = [0.0] * W["COUNT"]

    def put(wid, wt):
        out[wid], scales[wid] = pack_tc(wt)
    i = 0
    for s_, stage in enumerate(VGG_STAGES if vgg else ()):
        for idx, cin, cout in stage:
            w, _ = _fold_bn(sd, f"appearance.layers.{s_}.{idx}", f"appearance.layers.{s_}.{idx + 1}")
            if i == 0:
                put(W["VGG_WP0"] + i, w.reshape(cout, cin * 9).t())    # fp32 NCHW input: K order ci*9 + tap
            else:
                put(W["VGG_WP0"] + i, out[W["VGG_WT0"] + i])          # packed NHWC input: K order tap*Cin + ci
            i += 1
    if vgg:
        out[W["VGG_WPX0"]] = pack_px(out[W["VGG_WP0"]], 64, 27)
        out[W["VGG_WPX0"] + 1] = pack_px(out[W["VGG_WP0"] + 1], 64, 576)
    for j in range(5):
        put(W["PN_WP1"] + j, out[W["PN_L1"] + 4 * j])
    put(W["PN_WHAP"], out[W["PN_WHAT"]])
    put(W["AF_W01P"], out[W["AF_W01T"]])
    put(W["AF_W2P"], out[W["AF_W2T"]])
    put(W["AF_W3P"], out[W["AF_W3T"]])
    for wid, src in (("FU_WPP", "FU_WPT"), ("FU_WIP", "FU_WIT"), ("FU_GATE_PP", "FU_GATE_PT"), ("FU_GATE_IP", "FU_GATE_IT"),
                     ("WD_W1P", "WD_W1T"), ("WD_W2P", "WD_W2T"), ("NE_W1P", "NE_W1T"), ("NE_W2P", "NE_W2T"),
                     ("PN_WHGP", "PN_WHGT"), ("PN_WOP", "PN_WOT")):
        if out[W[src]] is not None:
            put(W[wid], out[W[src]])
    out = [t.view(torch.float32) if (t is not None and t.dtype == torch.uint8) else t for t in out]
    return out, t1.float(), t2.float(), scales


def stack_index(width):
    """pi: channel i of a 512-wide feature stack of the embedded net carries channel pi(i) of the width-``width`` net's
    stack.  The SkipPool heads write head s to channels [128 s, 128 s + 128), so pi maps that block onto copies of head
    s's width / 4 channels: pi(i) = (i // 128) * width / 4 + i % (width / 4).  Each aligned 32-channel block then holds
    one whole group of PointNet's GroupNorm(16 // r, width) (groups of 32), which GroupNorm(16, 512) sees unchanged."""
    q = width // 4
    i = torch.arange(D)
    return (i // SKIP_OUT) * q + i % q


def _channel_index(red, pad, width):
    """The channels of a width-``red`` activation of the narrow net in its ``pad``-wide copy (pad / red copies of each):
    the feature stacks (and every other width-``width`` activation) by stack_index, any other one tiled."""
    if red == pad:
        return None
    if red == width and pad == D:
        return stack_index(width)
    return torch.arange(pad) % red


def embed_width(state_dict, fusion, width, appear_arch="vgg", appear_head="skippool"):
    """The state_dict of a width-``width`` net (appear_len = point_len in {256, 128}, the reference's key names and
    shapes) -> an fp64 state_dict of the 512-wide net that computes it exactly, each activation as k identical copies
    (k = its 512-wide width over its own: 1, 2 or 4, so every division below is exact).  A layer whose input grows
    k_in-fold gets W_pad[i][j] = W[pi_out(i)][pi_in(j)] / k_in and bias b[pi_out(i)]; per-channel parameters (BatchNorm,
    GroupNorm affines and running statistics) are gathered by pi.  Per-channel operations keep the copies equal, and
    GroupNorm(1, C) or GroupNorm(G, C) over whole copies of its groups sees the narrow net's statistics.

    Two inputs are concatenations (fusion A's input_w: image | LiDAR stack; PointNet's head conv: local 64 | global 1024
    features) and are indexed piecewise.  STN2's output row (a, b) is T2[pi(a)][pi(b)]: its output layer and idt are
    embedded as T2_pad = T2[pi][pi] / k, which turns x T2 on the narrow features into x_pad T2_pad on their copies."""
    sd = {k: v.detach().cpu() for k, v in state_dict.items()}
    point_in = sd["point_net.feat.conv1.weight"].shape[1]
    wide = state_schema(fusion, point_in, appear_arch, appear_head)
    ix = lambda red, pad: _channel_index(red, pad, width)
    out = {}
    for key, (shape, _) in wide.items():
        t = sd[key].double() if sd[key].is_floating_point() else sd[key].clone()
        if t.dim() >= 1 and t.shape[0] != shape[0]:
            t = t[ix(t.shape[0], shape[0])]
        if t.dim() >= 2 and t.shape[1] != shape[1]:
            c = t.shape[1]
            if key == "fusion_module.input_w.0.weight":
                j = torch.cat([ix(c // 2, D), c // 2 + ix(c // 2, D)])
            elif key == "point_net.conv1.weight":
                c64 = sd["point_net.feat.conv1.weight"].shape[0]
                j = torch.cat([ix(c64, 64), c64 + ix(c - c64, 1024)])
            else:
                j = ix(c, shape[1])
            t = t[:, j] / (shape[1] // c)
        out[key] = t
    # STN2 emits the 64/r x 64/r matrix T2 flattened: row a * 64/r + b of its output layer; idt was gathered and divided
    # above like a matrix [a][b] (rows by pi, columns by pi over k)
    k2 = sd["point_net.feat.stn2.idt"].shape[0]
    if k2 != 64:
        p = ix(k2, 64)
        rows = (p[:, None] * k2 + p[None, :]).reshape(-1)
        s = "point_net.feat.stn2"
        kk = 64 // k2
        out[f"{s}.output.weight"] = sd[f"{s}.output.weight"].double()[rows][:, ix(256 * k2 // 64, 256)] / (kk * kk)
        out[f"{s}.output.bias"] = sd[f"{s}.output.bias"].double()[rows] / kk
    return out


class DeviceWeights:
    """All prepared tensors in ONE flat device buffer (256-byte aligned slices) + the pointer table
    handed to the C ABI."""

    def __init__(self, state_dict, fusion, device, appear_arch="vgg", appear_head="skippool", width=D):
        self.width = width
        narrow = None
        if width != D:
            # a narrow net runs as its 512-wide embedding; trans keeps the narrow net's T2, features its channels
            narrow = state_dict
            state_dict = embed_width(state_dict, fusion, width, appear_arch, appear_head)
            pi = stack_index(width)
            self.widen_index = pi.to(device)
            self.narrow_index = (pi[:, None] == torch.arange(width)).int().argmax(0).to(device)     # first copy
        tensors, self.trans1, self.trans2, scales = prepare(state_dict, fusion, appear_arch)
        if narrow is not None:
            k2 = narrow["point_net.feat.stn2.idt"].shape[0]
            self.trans2 = stn_constant({k: v.detach().cpu() for k, v in narrow.items()}, "point_net.feat.stn2", k2).float()
        nmain = len(tensors)
        self.resnet = self.fpn = None
        if appear_arch != "vgg":
            # the ResNet trunk's operands (and its head's) ride in the same flat buffer, behind the weight-id table's
            if appear_head == "fpn":
                convs = _resnet_trunk({k: v.detach().cpu() for k, v in state_dict.items()}, appear_arch)
                lats, last = prepare_fpn(state_dict)
                heads = [t for c in lats for t in (c[0], c[1], c[2].view(torch.float32))] + list(last)
            else:
                convs, heads = prepare_resnet(state_dict, appear_arch)
            tensors = tensors + [t for c in convs for t in (c[0], c[1], c[2].view(torch.float32))] + heads
        offs, total = [], 0
        for t in tensors:
            offs.append(total)
            if t is not None:
                total += (t.numel() + 63) // 64 * 64
        flat = torch.zeros(total, dtype=torch.float32)
        for t, o in zip(tensors, offs):
            if t is not None:
                flat[o:o + t.numel()] = t.reshape(-1)
        self.flat = flat.to(device)
        self.table = _lib.Weights()
        base = self.flat.data_ptr()
        for i, (t, o) in enumerate(zip(tensors[:nmain], offs)):
            self.table.w[i] = None if t is None else base + 4 * o
            self.table.tc_scale[i] = scales[i]
        if appear_arch != "vgg":
            r = self.resnet = _lib.ResnetWeights()
            r.blocks[:] = RESNET_BLOCKS[appear_arch]
            for i, c in enumerate(convs):
                o = offs[nmain + 3 * i: nmain + 3 * i + 3]
                r.wt[i], r.bias[i], r.wp[i] = (base + 4 * x for x in o)
                r.wp_scale[i] = c[3]
            ho = offs[nmain + 3 * len(convs):]
            if appear_head == "fpn":
                f = self.fpn = _lib.FpnWeights()
                for k in range(4):
                    f.lat_wt[k], f.lat_bias[k], f.lat_wp[k] = (base + 4 * x for x in ho[3 * k:3 * k + 3])
                    f.lat_wp_scale[k] = lats[k][3]
                f.last_wt, f.last_bias = base + 4 * ho[12], base + 4 * ho[13]
                self.fptr = ctypes.pointer(f)
            else:
                for s in range(4):
                    for j in range(10):
                        r.head[s][j] = base + 4 * ho[10 * s + j]
            self.rptr = ctypes.pointer(r)
        self.table.point_channels = int(state_dict["point_net.feat.conv1.weight"].shape[1])
        self.ptr = ctypes.pointer(self.table)
        self.trans1 = self.trans1.to(device)
        self.trans2 = self.trans2.to(device)

    def narrow(self, feats):
        """B x 3 x 512 x L features of the embedded net -> B x 3 x width x L, the narrow net's channels in its order."""
        return feats if self.width == D else feats.index_select(2, self.narrow_index)

    def widen(self, feats):
        """B x 3 x width x L features of the narrow net -> their 512-wide embedding (narrow's inverse)."""
        return feats if self.width == D else feats.index_select(2, self.widen_index).contiguous()
