"""Probe the fp32 accumulation rounding of the tensor-core engine's FP16 MMAs (signed error vs fp64)."""
import ctypes, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mmmot_b200 import _lib
from mmmot_b200.weights import pack_tc
lib = _lib.load()
vp = lambda t: ctypes.c_void_p(t.data_ptr())
g = torch.Generator().manual_seed(0)
M, S = 128, 1024
for K in (512, 1152, 2304, 4608):
    for name, fw, fx in (("pos*pos", 1, 1), ("neg*pos", -1, 1), ("mixed", 0, 0)):
        Wt = torch.rand(K, M, generator=g) + 0.5 if fw else torch.randn(K, M, generator=g)
        X = torch.rand(K, S, generator=g) + 0.5 if fx else torch.randn(K, S, generator=g)
        if fw == -1: Wt = -Wt
        ref = Wt.double().t() @ X.double()
        Wp, wps = pack_tc(Wt)
        res = {}
        for eng in (1, 2):
            if eng == 1:
                Y = torch.zeros(M, S, device="cuda")
                lib.mmmot_debug_simt_op(0, M, K, vp(Wt.cuda()), None, 0, vp(X.cuda()), 0, S, None, None, 0, 0, 0, 0, 0, 0, S, 1,
                                        None, 0, None, None, 0, vp(Y), 0, S, None, None)
            else:       # TMA-fed tensor-core engine: channels-last FP16 hi/lo planes in, Y[S][M] out
                Xc = X.t().contiguous()
                hi = Xc.half()
                Xp = torch.stack([hi, (Xc - hi.float()).half()]).contiguous().cuda()
                Yt = torch.zeros(S, M, device="cuda")
                lib.mmmot_debug_linear_planar(vp(Wp.cuda()), wps, None, vp(Xp), vp(Yt), M, K, S, None)
                Y = Yt.t()
            torch.cuda.synchronize()
            e = (Y.double().cpu() - ref)
            rel = e / ref.abs().clamp_min(1e-30)
            if name == "mixed":
                res[eng] = (float((e * ref.sign()).mean() / ref.abs().mean()), float(e.abs().max() / ref.abs().max()))
            else:
                res[eng] = (float(rel.mean()), float(rel.abs().max()))
        print(f"K={K:5d} {name:8s} simt mean_signed_rel={res[1][0]:+.2e} max={res[1][1]:.2e} | tc mean_signed_rel={res[2][0]:+.2e} max={res[2][1]:.2e}  steps={3*K//16} steps*2^-25={3*K/16*2**-25:.2e}")
