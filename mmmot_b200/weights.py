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
* every matrix transposed to Wt[K][Cout].

The folding is done once in fp64 on the host and rounded to fp32; it is checkpoint conversion,
not part of the per-frame path.
"""
import ctypes

import torch

from . import _lib
from .schema import SKIP_CHANNELS, VGG_STAGES

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


def prepare(state_dict, fusion):
    """-> (list of fp32 CPU tensors indexed by weight id (None = unused), trans1 CxC (C = 3 xyz or 4 xyz +
    reflectance: the checkpoint's point width), trans2 64x64, per-id tensor-core output scales)."""
    sd = {k: v.detach().cpu() for k, v in state_dict.items()}
    out = [None] * W["COUNT"]
    f64 = lambda k: sd[k].double()

    # VGG trunk
    i = 0
    for s, stage in enumerate(VGG_STAGES):
        for idx, cin, cout in stage:
            w, b = _fold_bn(sd, f"appearance.layers.{s}.{idx}", f"appearance.layers.{s}.{idx + 1}")
            # [co][ci][ky][kx] -> Wt[(ky*3+kx)*cin + ci][co]
            out[W["VGG_WT0"] + i] = w.permute(2, 3, 1, 0).reshape(9 * cin, cout)
            out[W["VGG_B0"] + i] = b
            i += 1
    # SkipPool heads
    for s, c in enumerate(SKIP_CHANNELS):
        p = f"appearance.global_pool.{s}.fc"
        base = W["SKIP0"] + 10 * s
        out[base + 0] = f64(f"{p}.0.weight"); out[base + 1] = f64(f"{p}.0.bias")
        out[base + 2] = f64(f"{p}.1.weight").reshape(-1, c).t(); out[base + 3] = f64(f"{p}.1.bias")
        out[base + 4] = f64(f"{p}.2.weight"); out[base + 5] = f64(f"{p}.2.bias")
        w2 = f64(f"{p}.4.weight")
        out[base + 6] = w2.reshape(w2.shape[0], -1).t(); out[base + 7] = f64(f"{p}.4.bias")
        out[base + 8] = f64(f"{p}.5.weight"); out[base + 9] = f64(f"{p}.5.bias")
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
    for s_, stage in enumerate(VGG_STAGES):
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
    for s_, stage in enumerate(VGG_STAGES):
        for idx, cin, cout in stage:
            w, _ = _fold_bn(sd, f"appearance.layers.{s_}.{idx}", f"appearance.layers.{s_}.{idx + 1}")
            if i == 0:
                put(W["VGG_WP0"] + i, w.reshape(cout, cin * 9).t())    # fp32 NCHW input: K order ci*9 + tap
            else:
                put(W["VGG_WP0"] + i, out[W["VGG_WT0"] + i])          # packed NHWC input: K order tap*Cin + ci
            i += 1
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


class DeviceWeights:
    """All prepared tensors in ONE flat device buffer (256-byte aligned slices) + the pointer table
    handed to the C ABI."""

    def __init__(self, state_dict, fusion, device):
        tensors, self.trans1, self.trans2, scales = prepare(state_dict, fusion)
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
        for i, (t, o) in enumerate(zip(tensors, offs)):
            self.table.w[i] = None if t is None else base + 4 * o
            self.table.tc_scale[i] = scales[i]
        self.table.point_channels = int(state_dict["point_net.feat.conv1.weight"].shape[1])
        self.ptr = ctypes.pointer(self.table)
        self.trans1 = self.trans1.to(device)
        self.trans2 = self.trans2.to(device)
