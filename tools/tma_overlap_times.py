"""Where the time of the TMA-fed channel-major contraction (tma::gemm_tma_kernel) goes, per tagged launch of the cfg4
forward, under three mmmot_set_debug settings:
    dbg 0  the real kernel
    dbg 8  MMA issue skipped: loader (weights + operand boxes from L2) + epilogue
    dbg 6  weight and operand loads skipped: MMA + epilogue without L2 traffic
next to the ideal MMA time 3 * algorithmic FLOPs / (132 SMs * 4096 FLOP/clk * median SM clock of the run).
Each setting runs once per conv epilogue: the extra debug bits of --epi-bits are OR'd into it (default "0,2048": the
epilogue from the accumulators, then debug bit 11's accumulator-image epilogue), and the epilogues alternate in
--rounds rounds in one process, so both see the same clocks; a table per epilogue (times averaged over the rounds)
and the per-tag dbg-0 ratio follow.
Bits 2-8 give wrong results by design: this is timing only, so the forward stops before the assignment LP and neither
the status word nor the outputs are looked at.
Run on a GPU box:  python tools/tma_overlap_times.py [pairs] [steps] [--epi-bits 0,2048] [--rounds 2] [--json out]"""
import argparse
import json
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
    ap = argparse.ArgumentParser()
    ap.add_argument("pairs", nargs="?", type=int, default=bench.CFG["pairs"])
    ap.add_argument("steps", nargs="?", type=int, default=2)
    ap.add_argument("--epi-bits", default="0,2048", help="comma-separated debug bits OR'd into every setting, one epilogue each")
    ap.add_argument("--rounds", type=int, default=2, help="rounds over the epilogues, alternating")
    ap.add_argument("--json", default=None, help="also write the tables as JSON here")
    args = ap.parse_args()
    pairs, steps = args.pairs, args.steps
    epis = [int(b) for b in args.epi_bits.split(",")]
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
    times = {e: {d: {} for d in DBG} for e in epis}       # epi -> dbg -> tag -> [ms, flop] summed over rounds
    for _ in range(args.rounds):
        for e in epis:
            for dbg in DBG:
                lib.mmmot_set_debug(dbg | e)
                net.forward_batch(crops, points, split, n, check=False)      # warm-up
                torch.cuda.synchronize(dev)
                lib.mmmot_timing_enable(1)
                for _ in range(steps):
                    net.forward_batch(crops, points, split, n, check=False)
                torch.cuda.synchronize(dev)
                lib.mmmot_timing_enable(0)
                for t, v in bench.collect_tags(lib).items():
                    acc = times[e][dbg].setdefault(t, [0.0, 0.0])
                    acc[0] += v[0]
                    acc[1] += v[1]
    lib.mmmot_set_debug(0)
    clk = sampler.summary()
    mhz = clk["sm_mhz"]
    nsteps = steps * args.rounds
    print(f"card: {card()}   SM clock median {mhz} MHz (max {clk['sm_max_mhz']}, throttle {clk['reasons']}, "
          f"power {clk['power_w']} W)   cfg4, {pairs} pairs, ms per step over {steps} steps x {args.rounds} rounds")
    out = {"card": card(), "clocks": clk, "pairs": pairs, "steps": steps, "rounds": args.rounds, "epilogues": {}}
    for e in epis:
        print(f"\nextra debug bits {e}")
        print(f"{'tag':32s} {'dbg0':>8s} {'dbg8':>8s} {'dbg6':>8s} {'mma':>8s}  {'dbg0-mma':>8s}  {'dbg8/dbg0':>9s}")
        tot = [0.0] * 5
        rows = {}
        for t in TAGS:
            if t not in times[e][0]:
                continue
            ms = [times[e][d][t][0] / nsteps if t in times[e][d] else float("nan") for d in DBG]
            flop = times[e][0][t][1] / nsteps
            ideal = 3 * flop / (SM_COUNT * FLOP_PER_CLK * mhz * 1e6) * 1e3 if mhz else float("nan")
            row = ms + [ideal, ms[0] - ideal]
            rows[t] = [round(x, 3) for x in row]
            tot = [a + b for a, b in zip(tot, row)]
            print(f"{t:32s} {row[0]:8.2f} {row[1]:8.2f} {row[2]:8.2f} {row[3]:8.2f}  {row[4]:8.2f}  {ms[1] / ms[0]:9.2f}")
        print(f"{'total':32s} {tot[0]:8.2f} {tot[1]:8.2f} {tot[2]:8.2f} {tot[3]:8.2f}  {tot[4]:8.2f}  {tot[1] / tot[0]:9.2f}")
        rows["total"] = [round(x, 3) for x in tot]
        out["epilogues"][str(e)] = rows
    if len(epis) > 1:
        e0, e1 = epis[0], epis[1]
        print(f"\ndbg 0 time, extra bits {e0} / extra bits {e1}")
        for t in TAGS + ["total"]:
            if t in out["epilogues"][str(e0)] and t in out["epilogues"][str(e1)]:
                a, b = out["epilogues"][str(e0)][t][0], out["epilogues"][str(e1)][t][0]
                print(f"{t:32s} {a:8.2f} {b:8.2f}  {a / b:6.3f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
