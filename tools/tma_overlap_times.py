"""Where the time of the TMA-fed channel-major contraction (tma::gemm_tma_kernel) goes, per tagged launch of the cfg4
forward, under three mmmot_set_debug settings:
    dbg 0  the real kernel
    dbg 8  MMA issue skipped: loader (weights + operand boxes from L2) + epilogue
    dbg 6  weight and operand loads skipped: MMA + epilogue without L2 traffic
next to the ideal MMA time 3 * algorithmic FLOPs / (132 SMs * 4096 FLOP/clk * median SM clock of the run).
Bits 2-8 give wrong results by design: this is timing only, so the forward stops before the assignment LP and neither
the status word nor the outputs are looked at.
Run on a GPU box:  python tools/tma_overlap_times.py [pairs] [steps]"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb          # noqa: E402
from mmmot_b200 import _lib      # noqa: E402
import bench                     # noqa: E402

# tags whose launches run tma::gemm_tma_kernel (vgg.conv0 / conv1 and PointNet l3 / l4 run the pixel-major kernel)
# (PointNet's l5 / head statistics-only passes run it only under debug bit 4, which this tool does not set)
TAGS = [f"vgg.conv{i}" for i in range(2, 13)] + ["pointnet.l2_64to64", "pointnet.l5_128to1024_segsum",
                                                  "pointnet.head_64to512_segsum"]
DBG = (0, 8, 6)
SM_COUNT, FLOP_PER_CLK = 132, 4096      # H100 SXM: SMs, dense FP16 tensor FLOP per clock per SM


def card():
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=10).stdout.strip()
        return o or torch.cuda.get_device_name(0)
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    pairs = int(sys.argv[1]) if len(sys.argv) > 1 else bench.CFG["pairs"]
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    dev = torch.device("cuda:0")
    c = bench.CFG
    n, pts, hw = c["n"], c["pts"], c["hw"]
    L = 2 * n
    net = mb.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch=c["fusion"],
                         affinity_op=c["affinity_op"], softmax_mode=c["softmax_mode"],
                         neg_threshold=c["neg_threshold"], test_mode=2, dropblock=0)
    from mmmot_b200.synthetic import synthetic_state_dict
    net.load_state_dict(synthetic_state_dict(c["fusion"], seed=0))
    net.cuda(dev).eval()
    g = torch.Generator(device=dev).manual_seed(1234)
    crops = torch.randn(pairs * L, 3, hw, hw, device=dev, generator=g)
    points = torch.randn(pairs * L * pts, 3, device=dev, generator=g)
    split = torch.arange(0, pairs * L * pts + 1, pts, dtype=torch.int32)
    lib = _lib.load()
    sampler = bench.ClockSampler(0)
    sampler.start()
    times = {}
    for dbg in DBG:
        lib.mmmot_set_debug(dbg)
        net.forward_batch(crops, points, split, n, check=False)      # warm-up
        torch.cuda.synchronize(dev)
        lib.mmmot_timing_enable(1)
        for _ in range(steps):
            net.forward_batch(crops, points, split, n, check=False)
        torch.cuda.synchronize(dev)
        lib.mmmot_timing_enable(0)
        times[dbg] = bench.collect_tags(lib)
    lib.mmmot_set_debug(0)
    clk = sampler.summary()
    mhz = clk["sm_mhz"]
    print(f"card: {card()}   SM clock median {mhz} MHz (max {clk['sm_max_mhz']}, throttle {clk['reasons']}, "
          f"power {clk['power_w']} W)   cfg4, {pairs} pairs, ms per step over {steps} steps")
    print(f"{'tag':32s} {'dbg0':>8s} {'dbg8':>8s} {'dbg6':>8s} {'mma':>8s}  {'dbg0-mma':>8s}  {'dbg8/dbg0':>9s}")
    tot = [0.0] * 5
    for t in TAGS:
        if t not in times[0]:
            continue
        ms = [times[d][t][0] / steps if t in times[d] else float("nan") for d in DBG]
        flop = times[0][t][1] / steps
        ideal = 3 * flop / (SM_COUNT * FLOP_PER_CLK * mhz * 1e6) * 1e3 if mhz else float("nan")
        row = ms + [ideal, ms[0] - ideal]
        tot = [a + b for a, b in zip(tot, row)]
        print(f"{t:32s} {row[0]:8.2f} {row[1]:8.2f} {row[2]:8.2f} {row[3]:8.2f}  {row[4]:8.2f}  {ms[1] / ms[0]:9.2f}")
    print(f"{'total':32s} {tot[0]:8.2f} {tot[1]:8.2f} {tot[2]:8.2f} {tot[3]:8.2f}  {tot[4]:8.2f}  {tot[1] / tot[0]:9.2f}")


if __name__ == "__main__":
    main()
