"""Checkpoint schema of the association hot path.

The drop-in contract includes the 263 ``state_dict`` key names of the reference
``TrackingNet`` (reference: modules/tracking_net.py:17-104, utils/train_util.py:157-188
``load_state`` uses ``load_state_dict(strict=False)``).  This module is the single table
of those names and shapes; the parameter holder (``tracking_net.py``), the weight packer
(``weights.py``) and the synthetic weight generator (``synthetic.py``) are all driven by it.

Key order follows module registration order of the reference so that
``list(state_dict())`` matches too (fusion_module, appearance, point_net, w_link, w_det).
"""
from collections import OrderedDict

# VGG16 (configuration "D", reference: modules/vgg.py:87-90) split into the four stages
# that modules/appear_net.py:130-157 builds: the first max-pool does NOT close a stage.
# Entries: (index inside the stage's Sequential, cin, cout) for convs; BN sits at index+1.
VGG_STAGES = (
    ((0, 3, 64), (3, 64, 64), (7, 64, 128), (10, 128, 128)),   # pools at 6 and 13
    ((0, 128, 256), (3, 256, 256), (6, 256, 256)),             # pool at 9
    ((0, 256, 512), (3, 512, 512), (6, 512, 512)),
    ((0, 512, 512), (3, 512, 512), (6, 512, 512)),
)
# conv index after which a 2x2 max-pool follows, per stage
VGG_POOL_AFTER = ((3, 10), (6,), (6,), (6,))
SKIP_CHANNELS = (128, 256, 512, 512)          # channels of the four skip maps
SKIP_OUT = 128                                # each SkipPool head emits 128 -> concat 512
D = 512
# ResNet trunks of appear_arch resnet50 / resnet101 / resnet152 (reference modules/appear_net.py:60-83): bottleneck
# blocks of layer1..layer4 (torchvision resnet.py), widths 64 << s, outputs 4x that, one SkipPool head per layer
RESNET_BLOCKS = {"resnet50": (3, 4, 6, 3), "resnet101": (3, 4, 23, 3), "resnet152": (3, 8, 36, 3)}
RES_SKIP_CHANNELS = (256, 512, 1024, 2048)
APPEAR_ARCHS = ("vgg",) + tuple(RESNET_BLOCKS)
# appear_len = point_len of the nets the reference builds: vgg16_bn_512 / _256 / _128 (modules/vgg.py:83-98, configs D,
# D_256, D_128) and every PointNet, fusion, affinity and w_det width divided by 512 // width (modules/point_net.py:10-19)
WIDTHS = (512, 256, 128)


def vgg_stages(width=D):
    """VGG_STAGES of the width-``width`` trunk: every conv's channels divided by 512 // width, the image's 3 kept."""
    r = D // width
    return tuple(tuple((idx, cin if cin == 3 else cin // r, cout // r) for idx, cin, cout in st) for st in VGG_STAGES)


def skip_mid(c):
    """Hidden width of a SkipPool head (reference: modules/appear_net.py:22)."""
    return max(c // 4, 64)


def _conv_bn(sd, prefix, idx, cin, cout, k):
    shape = (cout, cin, k, k) if k else (cout, cin, 1)
    sd[f"{prefix}.{idx}.weight"] = (shape, "conv")
    sd[f"{prefix}.{idx}.bias"] = ((cout,), "bias")
    sd[f"{prefix}.{idx + 1}.weight"] = ((cout,), "norm_w")
    sd[f"{prefix}.{idx + 1}.bias"] = ((cout,), "norm_b")
    sd[f"{prefix}.{idx + 1}.running_mean"] = ((cout,), "run_mean")
    sd[f"{prefix}.{idx + 1}.running_var"] = ((cout,), "run_var")
    sd[f"{prefix}.{idx + 1}.num_batches_tracked"] = ((), "nbt")


def _bn(sd, prefix, c, w_kind="norm_w"):
    sd[f"{prefix}.weight"] = ((c,), w_kind)
    sd[f"{prefix}.bias"] = ((c,), "norm_b")
    sd[f"{prefix}.running_mean"] = ((c,), "run_mean")
    sd[f"{prefix}.running_var"] = ((c,), "run_var")
    sd[f"{prefix}.num_batches_tracked"] = ((), "nbt")


def resnet_convs(arch):
    """The convs of a ResNet trunk in execution order (mmmot_resnet_weights, include/mmmot_b200.h): (conv key, its
    BatchNorm's key, cin, cout, kernel size, stride) -- the stem, then per bottleneck block conv1, conv2, conv3 and, on
    block 0 of every layer, downsample."""
    p = "appearance.layers"
    out = [(f"{p}.conv1", f"{p}.bn1", 3, 64, 7, 2)]
    cin = 64
    for s, nb in enumerate(RESNET_BLOCKS[arch]):
        w = 64 << s
        for b in range(nb):
            stride = 2 if (b == 0 and s > 0) else 1
            q = f"{p}.layer{s + 1}.{b}"
            out += [(f"{q}.conv1", f"{q}.bn1", cin, w, 1, 1), (f"{q}.conv2", f"{q}.bn2", w, w, 3, stride),
                    (f"{q}.conv3", f"{q}.bn3", w, 4 * w, 1, 1)]
            if b == 0:
                out.append((f"{q}.downsample.0", f"{q}.downsample.1", cin, 4 * w, 1, stride))
            cin = 4 * w
    return out


def _resnet(sd, arch):
    """torchvision's resnetXX minus avgpool / fc (the reference's Resnet wrapper keeps conv1 .. layer4): bias-free convs,
    each followed by a BatchNorm2d.  Registration order: conv1, bn1, then per block conv1, bn1, conv2, bn2, conv3, bn3,
    downsample.  bn3 closes a residual branch (kind res_norm_w)."""
    for conv, bn, cin, cout, k, _ in resnet_convs(arch):
        sd[f"{conv}.weight"] = ((cout, cin, k, k), "conv")
        _bn(sd, bn, cout, "res_norm_w" if conv.endswith("conv3") else "norm_w")


def _lin_gn(sd, conv, norm, cin, cout, wshape):
    sd[f"{conv}.weight"] = (wshape, "conv")
    sd[f"{conv}.bias"] = ((cout,), "bias")
    if norm is not None:
        sd[f"{norm}.weight"] = ((cout,), "norm_w")
        sd[f"{norm}.bias"] = ((cout,), "norm_b")


def _stn(sd, p, cin, k, r=1):
    sd[f"{p}.idt"] = ((k, k), "eye")
    _lin_gn(sd, f"{p}.conv1", f"{p}.bn1", cin, 64 // r, (64 // r, cin, 1))
    _lin_gn(sd, f"{p}.conv2", f"{p}.bn2", 64 // r, 128 // r, (128 // r, 64 // r, 1))
    _lin_gn(sd, f"{p}.conv3", f"{p}.bn3", 128 // r, 1024 // r, (1024 // r, 128 // r, 1))
    _lin_gn(sd, f"{p}.fc1", f"{p}.fc_bn1", 1024 // r, 512 // r, (512 // r, 1024 // r))
    _lin_gn(sd, f"{p}.fc2", f"{p}.fc_bn2", 512 // r, 256 // r, (256 // r, 512 // r))
    sd[f"{p}.output.weight"] = ((k * k, 256 // r), "stn_out")
    sd[f"{p}.output.bias"] = ((k * k,), "stn_out")


def _fpn(sd, D=D):
    """The FPN head (reference modules/appear_net.py:83-104): per ResNet stage a bias-free 1x1 lateral C -> D and its
    BatchNorm2d (fpn_in.k.0 / .1), then conv_last.1 (1x1, D -> D, with bias) and its BatchNorm2d conv_last.2."""
    for k, c in enumerate(RES_SKIP_CHANNELS):
        sd[f"appearance.fpn_in.{k}.0.weight"] = ((D, c, 1, 1), "conv")
        _bn(sd, f"appearance.fpn_in.{k}.1", D)
    sd["appearance.conv_last.1.weight"] = ((D, D, 1, 1), "conv")
    sd["appearance.conv_last.1.bias"] = ((D,), "bias")
    _bn(sd, "appearance.conv_last.2", D)


APPEAR_HEADS = ("skippool", "fpn")


def state_schema(fusion="C", point_in=3, appear_arch="vgg", appear_head="skippool", width=D):
    """OrderedDict key -> (shape, kind).  ``kind`` drives init / synthetic generation:
    conv, bias, norm_w, res_norm_w, norm_b, run_mean, run_var, nbt, eye, stn_out.
    appear_arch: "vgg" (VGG16-BN) or a key of RESNET_BLOCKS; appear_head: "skippool" (four SkipPool heads,
    appear_skippool) or "fpn" (the FPN head, appear_fpn; ResNet trunks only); width: appear_len = point_len, one of
    WIDTHS (the reference divides every width of the net below 512 by r = 512 // width)."""
    if appear_head not in APPEAR_HEADS or (appear_head == "fpn" and appear_arch == "vgg"):
        raise ValueError(f"unsupported appearance head {appear_head!r} on {appear_arch!r}")
    if width not in WIDTHS:
        raise ValueError(f"unsupported width {width!r} (appear_len = point_len must be one of {WIDTHS})")
    d, r = width, D // width
    sd = OrderedDict()
    # --- fusion_module (modules/fusion_net.py) ---
    f = "fusion_module"
    if fusion == "C":
        for g in ("gate_p", "gate_i"):
            _lin_gn(sd, f"{f}.{g}.0", None, d, d, (d, d, 1))
        for g in ("input_p", "input_i"):
            _lin_gn(sd, f"{f}.{g}.0", f"{f}.{g}.1", d, d, (d, d, 1))
    elif fusion == "B":
        for g in ("input_p", "input_i"):
            _lin_gn(sd, f"{f}.{g}.0", f"{f}.{g}.1", d, d, (d, d, 1))
    elif fusion == "A":
        _lin_gn(sd, f"{f}.input_w.0", f"{f}.input_w.1", 2 * d, d, (d, 2 * d, 1))
    else:
        raise ValueError(f"unknown fusion arch {fusion!r}")
    # --- appearance (modules/appear_net.py, modules/vgg.py or torchvision's ResNet) ---
    if appear_arch == "vgg":
        for s, stage in enumerate(vgg_stages(width)):
            for idx, cin, cout in stage:
                _conv_bn(sd, f"appearance.layers.{s}", idx, cin, cout, 3)
    elif appear_arch in RESNET_BLOCKS:
        _resnet(sd, appear_arch)
    else:
        raise ValueError(f"unknown appearance arch {appear_arch!r}")
    if appear_head == "fpn":
        _fpn(sd, d)
    skip = () if appear_head == "fpn" else tuple(c // r for c in SKIP_CHANNELS) if appear_arch == "vgg" else RES_SKIP_CHANNELS
    for s, c in enumerate(skip):
        p = f"appearance.global_pool.{s}.fc"
        m = skip_mid(c)
        sd[f"{p}.0.weight"] = ((c,), "norm_w")
        sd[f"{p}.0.bias"] = ((c,), "norm_b")
        _lin_gn(sd, f"{p}.1", f"{p}.2", c, m, (m, c, 1, 1))
        _lin_gn(sd, f"{p}.4", f"{p}.5", m, d // 4, (d // 4, m, 1, 1))
    # --- point_net (modules/point_net.py) ---
    p = "point_net.feat"
    c64, c128, c1024, c512 = 64 // r, 128 // r, 1024 // r, 512 // r
    _stn(sd, f"{p}.stn1", point_in, point_in, r)
    _lin_gn(sd, f"{p}.conv1", f"{p}.bn1", point_in, c64, (c64, point_in, 1))
    _lin_gn(sd, f"{p}.conv2", f"{p}.bn2", c64, c64, (c64, c64, 1))
    _stn(sd, f"{p}.stn2", c64, c64, r)
    _lin_gn(sd, f"{p}.conv3", f"{p}.bn3", c64, c64, (c64, c64, 1))
    _lin_gn(sd, f"{p}.conv4", f"{p}.bn4", c64, c128, (c128, c64, 1))
    _lin_gn(sd, f"{p}.conv5", f"{p}.bn5", c128, c1024, (c1024, c128, 1))
    sd["point_net.conv1.weight"] = ((c512, c64 + c1024, 1), "conv")
    sd["point_net.conv1.bias"] = ((c512,), "bias")
    sd["point_net.conv2.weight"] = ((d, c512, 1), "conv")
    sd["point_net.conv2.bias"] = ((d,), "bias")
    for n, c in (("bn1", c512), ("bn2", d), ("avg_bn", c512)):
        sd[f"point_net.{n}.weight"] = ((c,), "norm_w")
        sd[f"point_net.{n}.bias"] = ((c,), "norm_b")
    # --- w_link (modules/gcn.py, modules/new_end.py) ---
    ne = "w_link.w_new_end"
    _lin_gn(sd, f"{ne}.conv0.0", f"{ne}.conv0.1", d, d, (d, d, 1, 1))
    _lin_gn(sd, f"{ne}.conv1.0", f"{ne}.conv1.1", d, d, (d, d, 1))
    _lin_gn(sd, f"{ne}.conv1.3", f"{ne}.conv1.4", d, d // 4, (d // 4, d, 1))
    _lin_gn(sd, f"{ne}.conv1.6", None, d // 4, 1, (1, d // 4, 1))
    _lin_gn(sd, "w_link.conv1.0", "w_link.conv1.1", d, d, (d, d, 1, 1))
    _lin_gn(sd, "w_link.conv1.3", "w_link.conv1.4", d, d, (d, d, 1, 1))
    _lin_gn(sd, "w_link.conv1.6", "w_link.conv1.7", d, d // 4, (d // 4, d, 1, 1))
    _lin_gn(sd, "w_link.conv1.9", None, d // 4, 1, (1, d // 4, 1, 1))
    # --- w_det (modules/tracking_net.py:91-100) ---
    _conv_bn(sd, "w_det", 0, d, d, 0)
    _conv_bn(sd, "w_det", 3, d, d // 2, 0)
    sd["w_det.6.weight"] = ((1, d // 2, 1), "conv")
    sd["w_det.6.bias"] = ((1,), "bias")
    return sd


BUFFER_KINDS = ("run_mean", "run_var", "nbt")
