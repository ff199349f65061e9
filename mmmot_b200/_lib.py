"""ctypes binding of libmmmot_sm90a.so (the C ABI declared in include/mmmot_b200.h).

There is no fallback: if the shared library is missing or cannot be loaded, every product entry
point raises.  Nothing here touches torch; callers pass raw device pointers and a stream handle.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmmmot_sm90a.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "mmmot_b200.h")

ABI_VERSION = 3
SCORE_SIGMOID, SCORE_THRESHOLD = 1, 2
FUSION = {"A": 0, "B": 1, "C": 2}
AFFINITY = {"multiply": 0, "minus_abs": 1, "minus": 2}
SOFTMAX = {"none": 0, "single": 1, "dual": 2, "dual_add": 3, "dual_max": 4}
END_MODE = {"avg": 0, "max": 1}

# weight ids: mirrors `enum mmmot_weight_id` (tests/test_abi.py parses the header and compares)
W = dict(
    VGG_WT0=0, VGG_B0=13, SKIP0=26, PN_L1=66, PN_WHAT=86, PN_WHGT=87, PN_BH=88, PN_GHW=89, PN_GHB=90,
    PN_WOT=91, PN_BO=92, PN_GOW=93, PN_GOB=94,
    FU_WPT=95, FU_BP=96, FU_GPW=97, FU_GPB=98, FU_WIT=99, FU_BI=100, FU_GIW=101, FU_GIB=102,
    FU_GATE_PT=103, FU_GATE_PB=104, FU_GATE_IT=105, FU_GATE_IB=106,
    WD_W1T=107, WD_B1=108, WD_W2T=109, WD_B2=110, WD_W3=111, WD_B3=112,
    AF_W01T=113, AF_B01=114, AF_G1W=115, AF_G1B=116, AF_G0W=117, AF_G0B=118,
    AF_W2T=119, AF_B2=120, AF_G2W=121, AF_G2B=122, AF_W3T=123, AF_B3=124, AF_G3W=125, AF_G3B=126,
    AF_W4=127, AF_B4=128,
    NE_W1T=129, NE_B1=130, NE_G1W=131, NE_G1B=132, NE_W2T=133, NE_B2=134, NE_G2W=135, NE_G2B=136,
    NE_W3=137, NE_B3=138,
    VGG_WP0=139, PN_WP1=152, PN_WHAP=157, AF_W01P=158, AF_W2P=159, AF_W3P=160,
    VGG_RAWW0=161, VGG_RAWB0=174, VGG_BNW0=187, VGG_BNB0=200, WD_RAW0=213,
    FU_WPP=221, FU_WIP=222, FU_GATE_PP=223, FU_GATE_IP=224, WD_W1P=225, WD_W2P=226, VGG_WPX0=227, NE_W1P=229, NE_W2P=230, PN_WHGP=231, PN_WOP=232, COUNT=233,
)


class Weights(ctypes.Structure):
    _fields_ = [("w", ctypes.c_void_p * W["COUNT"]), ("tc_scale", ctypes.c_float * W["COUNT"]), ("point_channels", ctypes.c_int)]


class MmmotError(RuntimeError):
    pass


_vp, _i, _l, _f, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_size_t
_wp = ctypes.POINTER(Weights)

# name -> (restype, argtypes); every symbol the header declares
SIGNATURES = {
    "mmmot_abi_version": (_i, []),
    "mmmot_device_info": (_i, [ctypes.POINTER(_i)] * 3),
    "mmmot_launch_count": (ctypes.c_ulonglong, []),
    "mmmot_set_engine": (_i, [_i]),
    "mmmot_set_debug": (_i, [_i]),
    "mmmot_set_kseg": (_i, [_i]),
    "mmmot_debug_simt_op": (_i, [_i, _i, _i, _vp, _vp, _i, _vp, _l, _l, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _i,
                                 _vp, _vp, _i, _vp, _l, _l, _vp, _vp]),
    "mmmot_debug_linear_planar": (_i, [_vp, _f, _vp, _vp, _vp, _i, _i, _l, _vp]),
    "mmmot_debug_conv_plan": (_i, [_i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(_i)]),
    "mmmot_debug_conv_layer": (_i, [_vp, _vp, _f, _vp, _vp, _l, _i, _i, _i, _i, _i, _vp, _l, _l, ctypes.POINTER(_i), _vp, _vp,
                                    _vp, ctypes.POINTER(_i), _vp]),
    "mmmot_debug_vgg_conv0": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _l, _vp, _vp, ctypes.POINTER(_i), _vp]),
    "mmmot_timing_enable": (_i, [_i]),
    "mmmot_timing_tag_count": (_i, []),
    "mmmot_timing_tag_name": (ctypes.c_char_p, [_i]),
    "mmmot_timing_collect_tags": (_i, [ctypes.POINTER(ctypes.c_double)] * 3 + [ctypes.POINTER(ctypes.c_long)]),
    "mmmot_status_reset": (_i, [_vp, _vp]),
    "mmmot_status_check": (_i, [_vp, _vp]),
    "mmmot_fetch_pinned_i32": (_i, [_vp, _vp, _l, _vp]),
    "mmmot_debug_gen_prefetch": (_i, [_i, _i]),
    "mmmot_debug_gen_staged": (_i, [_i, _i]),
    "mmmot_debug_gen": (_i, [_i, _i, _i, _vp, _f, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _l, _l, _vp, _i, _vp, _l, _vp,
                             ctypes.POINTER(_i), _vp]),
    "mmmot_debug_pn_contraction": (_i, [_vp, _vp, _i, _i, _l, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_l), _vp, _f, _vp, _i, _i,
                                        _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "mmmot_debug_pn_stats": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  _sz, _vp]),
    "mmmot_debug_stage_layout": (_i, [_i, _i, _i, _i, ctypes.POINTER(_sz), ctypes.POINTER(_i)]),
    "mmmot_debug_skip_heads": (_i, [_wp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "mmmot_timing_collect": (_i, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_long)]),
    "mmmot_appearance_workspace": (_sz, [_i, _i, _i]),
    "mmmot_appearance_fwd": (_i, [_wp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "mmmot_appearance_train_workspace": (_sz, [_i, _i, _i]),
    "mmmot_appearance_train_fwd": (_i, [_wp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_pointnet_train_workspace": (_sz, [_i, _i, _l]),
    "mmmot_pointnet_train_fwd": (_i, [_wp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_w_det_train_workspace": (_sz, [_i]),
    "mmmot_w_det_train_fwd": (_i, [_wp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_pointnet_workspace": (_sz, [_i, _i, _l]),
    "mmmot_pointnet_fwd": (_i, [_wp, _vp, _vp, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    "mmmot_fusion_det_workspace": (_sz, [_i, _i]),
    "mmmot_fusion_det_fwd": (_i, [_wp, _i, _i, _f, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_affinity_workspace": (_sz, [_i, _i, _i]),
    "mmmot_affinity_fwd": (_i, [_wp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_crop_workspace": (_sz, [_i, _i]),
    "mmmot_crop_count": (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    "mmmot_crop_scatter": (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "mmmot_prep_workspace": (_sz, [_i, _i, _i]),
    "mmmot_prep_count": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _sz, _vp]),
    "mmmot_prep_scatter": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "mmmot_crop_resize_max_taps": (_i, []),
    "mmmot_crop_resize_workspace": (_sz, [_i, _l, _i, _i]),
    "mmmot_crop_resize": (_i, [_vp, _i, _i, _vp, _vp, _i, _l, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_lp_workspace": (_sz, [_i, _i, _i]),
    "mmmot_lp_assign": (_i, [_vp, _l, _vp, _l, _vp, _l, _vp, _l, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mmmot_flow_workspace": (_sz, [_i, _i, ctypes.POINTER(_i)]),
    "mmmot_flow_assign": (_i, [_vp, _l, _vp, _l, _vp, _l, _vp, _l, _i, _i, ctypes.POINTER(_i), _vp, _vp, _vp, _vp, _vp,
                               _vp, _sz, _vp]),
}

_lib = None


def header_functions():
    """Names of all functions declared in include/mmmot_b200.h."""
    src = open(HEADER_PATH).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mmmot_[a-z_0-9]+)\s*\(", src)))


def load():
    """Load the shared library (once).  Raises MmmotError when it is absent: the product has no
    CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MmmotError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(mmmot_b200 has no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.mmmot_abi_version() != ABI_VERSION:
        raise MmmotError("ABI version mismatch between mmmot_b200/_lib.py and libmmmot_sm90a.so")
    _lib = lib
    return lib


def check(code, what):
    if code == 0:
        return
    names = {-1: "MMMOT_E_ARG", -2: "MMMOT_E_WORKSPACE", -3: "MMMOT_E_SHAPE",
             -4: "MMMOT_E_RANGE (an activation reached |x| >= 65504, FP16's range, on the tensor-core path; the outputs are "
                 "clamped and must not be used — run with mmmot_b200.set_engine('fp32') for such checkpoints)"}
    msg = names.get(code, f"cudaError {code}" if code > 0 else str(code))
    raise MmmotError(f"{what} failed: {msg}")
