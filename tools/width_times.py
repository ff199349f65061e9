"""The 256- and 128-wide nets (appear_len = point_len, run as their 512-wide embedding) against the 512-wide net at cfg4's
shape (Fusion C, minus_abs, dual_add, N = M = 128, P = 512, 64 x 64 crops): one ``predict_batch`` call of `pairs`
frame-pairs per width, the widths alternated round by round in one process so drift on a shared host hits all three
alike.  Each round times a window of `reps` back-to-back calls with device events after warm-up; the figure per width is
the median over rounds of ms per call.  Card name, power limit and SM clock are read in the same run.  Prints one JSON line (also written to the path given as the first argument).
Run on a GPU box:  python tools/width_times.py [out.json] [pairs] [rounds] [reps]"""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb                                      # noqa: E402
from bench import CFG                                        # noqa: E402
from mmmot_b200.synthetic import synthetic_batch, synthetic_state_dict  # noqa: E402

WIDTHS = (512, 256, 128)


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 32
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    reps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
    assert torch.cuda.is_available(), "width_times.py needs a CUDA device"
    c = CFG
    n = c["n"]
    crops, pts, split = synthetic_batch(pairs, n, pts=c["pts"], hw=c["hw"], seed=5)
    crops, pts = crops.cuda(), pts.cuda()
    nets = {}
    for w in WIDTHS:
        net = mb.TrackingNet(2, appear_len=w, point_len=w, appear_skippool=True, score_arch="branch_cls",
                             score_fusion_arch=c["fusion"], affinity_op=c["affinity_op"], softmax_mode=c["softmax_mode"],
                             neg_threshold=c["neg_threshold"], test_mode=2, dropblock=0)
        net.load_state_dict(synthetic_state_dict(c["fusion"], seed=7, width=w))
        nets[w] = net.cuda().eval()
    call = lambda w: nets[w].predict_batch(crops, pts, split, n)
    for w in WIDTHS:                                          # warm-up: every shape of the timed windows
        for _ in range(2):
            call(w)
    torch.cuda.synchronize()
    times = {w: [] for w in WIDTHS}
    for r in range(rounds):
        order = WIDTHS if r % 2 == 0 else WIDTHS[::-1]
        for w in order:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                call(w)
            b.record()
            b.synchronize()
            times[w].append(a.elapsed_time(b) / reps)
    med = {w: statistics.median(times[w]) for w in WIDTHS}
    res = {
        "tool": "width_times", "config": "cfg4", "pairs_per_call": pairs, "rounds": rounds, "calls_per_window": reps,
        "gpu": smi("name"), "power_limit": smi("power.limit"), "max_sm_clock": smi("clocks.max.sm"),
        "ms_per_call": {str(w): round(med[w], 3) for w in WIDTHS},
        "ms_per_call_all_rounds": {str(w): [round(t, 3) for t in times[w]] for w in WIDTHS},
        "ratio_to_512": {str(w): round(med[w] / med[512], 4) for w in WIDTHS},
    }
    line = json.dumps(res)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
