"""The fused first VGG block (csrc/vgg_conv01.cuh: layers 0 and 1 and the 2x2 max-pool in one launch) against the
two-launch path it replaces, through the product's own launch code (mmmot_debug_vgg_conv01, which runs the block exactly
as mmmot_appearance_fwd does; debug bit 15 forces the two launches).

The fused kernel keeps the two-launch path's accumulation order, so its pooled planes must be byte-identical to it.  They
are also bounded against fp64 conv1 + bias + ReLU + pool of the layer-0 planes the two-launch path stores, by
|y - y_ref| <= TAU * S (kernel_kit.TAU, S = the pooled conv2d(|X|, |W|) + |b|), and the FP16 range flag must be raised
as the two-launch path raises it.  The plan test at the end runs without a GPU (mmmot_debug_vgg_conv01_plan).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from kernel_kit import KSEG_DEFAULT, TAU, bench_n_imgs, lib_state, vp
from mmmot_b200 import _lib
from mmmot_b200.weights import pack_px, pack_tc

NAN16 = 0x7E00
TWO_LAUNCH = 1 << 15               # debug bit 15
gpu = pytest.mark.gpu


def _weights(g, b0_shift=0.0):
    w0 = torch.randn(64, 3, 3, 3, generator=g) * (2.0 / 27) ** 0.5
    b0 = torch.randn(64, generator=g) * 0.1 + b0_shift
    w1 = torch.randn(64, 64, 3, 3, generator=g) * (2.0 / 576) ** 0.5
    b1 = torch.randn(64, generator=g) * 0.1
    return w0, b0, w1, b1


def _run(lib, x, w0, b0, w1, b1, dbg):
    """-> (pooled hi, pooled lo) int16 [n][H/2][W/2][64], layer-0 planes (hi, lo) [n][H][W][64] or None, fused, status."""
    n, _, H, W = x.shape
    wt0 = w0.permute(2, 3, 1, 0).reshape(27, 64).contiguous()
    Wp0, s0 = pack_tc(w0.reshape(64, 27).t())
    Wp1, s1 = pack_tc(w1.permute(2, 3, 1, 0).reshape(576, 64).contiguous())
    keep = [t.contiguous().cuda() for t in (x, wt0, b0, Wp0, pack_px(Wp0, 64, 27), b1, Wp1, pack_px(Wp1, 64, 576))]
    plane, plane_p = n * H * W * 64, n * H * W * 16
    bufs = [torch.full((2 * plane,), NAN16, dtype=torch.int16, device="cuda") for _ in range(2)]
    scratch = torch.empty((n + 16) * H * W * 16, dtype=torch.float32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out, fused = ctypes.c_int(-1), ctypes.c_int(-1)
    with lib_state(lib, dbg=dbg):
        rc = lib.mmmot_debug_vgg_conv01(vp(keep[0]), n, H, W, vp(keep[1]), vp(keep[2]), vp(keep[3]), s0, vp(keep[4]),
                                        vp(keep[5]), vp(keep[6]), s1, vp(keep[7]), vp(bufs[0]), vp(bufs[1]), vp(scratch),
                                        vp(status), ctypes.byref(out), ctypes.byref(fused), None)
        torch.cuda.synchronize()
    assert rc == 0, rc
    y = bufs[out.value].cpu()
    shape = (n, H // 2, W // 2, 64)
    l0 = None
    if not fused.value:
        b = bufs[0].cpu() if out.value == 1 else None
        l0 = None if b is None else (b[:plane].reshape(n, H, W, 64), b[plane:].reshape(n, H, W, 64))
    return (y[:plane_p].reshape(shape), y[plane_p:2 * plane_p].reshape(shape)), l0, fused.value, int(status.item())


def _both(lib, x, w0, b0, w1, b1):
    fa, _, f1, st1 = _run(lib, x, w0, b0, w1, b1, 0)
    tw, l0, f2, st2 = _run(lib, x, w0, b0, w1, b1, TWO_LAUNCH)
    assert (f1, f2) == (1, 0), (f1, f2)
    return fa, tw, l0, st1, st2


def _pooled_ref(l0, w1, b1):
    """fp64 relu(conv1(X) + b) max-pooled, and its error scale S, X = hi + lo of the stored layer-0 planes."""
    x = (l0[0].view(torch.float16).double() + l0[1].view(torch.float16).double()).permute(0, 3, 1, 2)
    w, b = w1.double(), b1.double()
    y = F.max_pool2d(torch.relu(F.conv2d(x, w, b, padding=1)), 2)
    S = F.max_pool2d(F.conv2d(x.abs(), w.abs(), b.abs(), padding=1), 2)
    return y.permute(0, 2, 3, 1), S.permute(0, 2, 3, 1)


@gpu
@pytest.mark.parametrize("H,W,n", [(64, 64, 1), (64, 64, 2), (64, 64, 24), (32, 32, 2), (64, 96, 2), (128, 128, 1)],
                         ids=lambda v: str(v))
def test_fused_block_equals_two_launches(H, W, n):
    """Pooled hi and lo planes byte for byte, at the benchmark's 64x64 crops (64x64 x 24 images: 384 tiles, so every CTA
    of the persistent grid runs several tiles and wraps the weight ring), and at 32x32, 64x96 and 128x128; then the
    fused output against fp64 conv1 + pool of the two-launch path's stored layer-0 planes."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(H * 1000 + W + n)
    x = torch.randn(n, 3, H, W, generator=g)
    w0, b0, w1, b1 = _weights(g)
    fa, tw, l0, st1, st2 = _both(lib, x, w0, b0, w1, b1)
    for p in range(2):
        diff = int((fa[p] != tw[p]).sum())
        assert diff == 0, f"plane {p}: {diff} elements differ"
    y = fa[0].view(torch.float16).double() + fa[1].view(torch.float16).double()
    assert bool(torch.isfinite(y).all())
    ref, S = _pooled_ref(l0, w1, b1)
    ratio = float(((y - ref).abs() / (TAU * S)).max())
    print(f"\nvgg block 0+1 {H}x{W} n={n}: worst err/(tau S) = {ratio:.3g}", end="")
    assert ratio <= 1.0 and st1 == st2 == 0


@gpu
def test_fused_block_zero_padding():
    """A large positive layer-0 bias: relu(bias) written for the layer-0 pixels outside the image instead of layer 1's
    zero padding would change every border output."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 64, 64, generator=g)
    w0, b0, w1, b1 = _weights(g, b0_shift=4.0)
    fa, tw, l0, _, _ = _both(lib, x, w0, b0, w1, b1)
    assert torch.equal(fa[0], tw[0]) and torch.equal(fa[1], tw[1])
    y = fa[0].view(torch.float16).double() + fa[1].view(torch.float16).double()
    ref, S = _pooled_ref(l0, w1, b1)
    assert float(((y - ref).abs() / (TAU * S)).max()) <= 1.0


@gpu
def test_fused_block_range_flag():
    """Status bit 0: a layer-0 output at or above 65504 raises it, just below does not; so does a crop value at or above
    65504; and a layer-1 output.  The fused launch raises it exactly when the two launches do."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(11)
    n, H, W = 1, 32, 32
    x = torch.randn(n, 3, H, W, generator=g)
    w0, b0, w1, b1 = _weights(g)
    peak0 = float(torch.relu(F.conv2d(x.double(), w0.double(), b0.double(), padding=1)).max())
    small = (w1 * 1e-3).float(), (b1 * 1e-3).float()
    cases = []
    for target, flagged in ((70000.0, 1), (64000.0, 0)):                  # layer-0 outputs
        f = target / peak0
        cases.append((x, (w0 * f).float(), (b0 * f).float(), *small, flagged))
    for top, flagged in ((70000.0, 1), (65000.0, 0)):                     # crop values
        cases.append((x / x.abs().max() * top, w0 * 1e-3, b0 * 1e-3, *small, flagged))
    cases.append((x, w0, b0, (w1 * 3e4).float(), b1, 1))                  # layer-1 outputs
    for xc, a, b, c, d, flagged in cases:
        _, _, f1, st1 = _run(lib, xc, a, b, c, d, 0)
        _, _, f2, st2 = _run(lib, xc, a, b, c, d, TWO_LAUNCH)
        assert (f1, f2) == (1, 0)
        assert st1 & 1 == st2 & 1 == flagged, (st1, st2, flagged)


# ------------------------------------------------------------------------------------------------ CPU: plan selection
def _fused(lib, n, H, W, dbg=0, kseg=None):
    f = ctypes.c_int(-1)
    with lib_state(lib, dbg=dbg, kseg=kseg):
        assert lib.mmmot_debug_vgg_conv01_plan(n, H, W, ctypes.byref(f)) == 0
    return f.value


BENCH = {"cfg2": (64, 32), "cfg3": (256, 64), "cfg4": (128, 128)}   # (frame-pairs, detections per frame), 64x64 crops


def test_fused_block_plan():
    """Every image count the cfg2-cfg4 forwards can launch at 64x64 takes the fused launch; shapes the 16x16 tiles do not
    cover, widths past layer 0's in-kernel taps, debug bit 15 and K segments shorter than layer 1's 18 chunks fall back
    to the two launches."""
    lib = _lib.load()
    for name, (pairs, n) in BENCH.items():
        for imgs in bench_n_imgs(pairs, 2 * n):
            assert _fused(lib, imgs, 64, 64) == 1, (name, imgs)
    for H, W in ((32, 32), (64, 96), (128, 128), (224, 224)):
        assert _fused(lib, 2, H, W) == 1, (H, W)
    assert _fused(lib, 2, 40, 40) == 0                       # not a multiple of 16
    assert _fused(lib, 2, 64, 72) == 0
    assert _fused(lib, 1, 32, 544) == 0                      # layer 0 without in-kernel taps
    assert _fused(lib, 2, 64, 64, dbg=TWO_LAUNCH) == 0
    assert _fused(lib, 2, 64, 64, dbg=512) == 0              # no fused pool in layer 1
    assert _fused(lib, 2, 64, 64, kseg=16) == 0
    assert _fused(lib, 2, 64, 64, kseg=KSEG_DEFAULT) == 1
