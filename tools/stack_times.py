"""One feature stack alone (``predict_batch(stack=s)``: 0 image, 1 LiDAR, 2 fused) against the full three-stack call at
cfg4's and cfg3's shapes (BASELINE configs; 64 x 64 crops, P = 512 points per detection).  One ``predict_batch`` call of
`pairs` frame-pairs per variant, the variants alternated round by round in one process so drift on a shared host hits all
alike.  Each round times a window of `reps` back-to-back calls with device events after warm-up; the figure per variant is
the median over rounds of ms per call.  The one-stack calls are given only the input their stack needs (crops for 0,
points for 1).  Card name, power limit and SM clock are read in the same run.  Prints one JSON line (also written to the
path given as the first argument).
Run on a GPU box:  python tools/stack_times.py [out.json] [pairs] [rounds] [reps]"""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb                                      # noqa: E402
from bench import CONFIGS                                    # noqa: E402
from mmmot_b200.synthetic import synthetic_batch, synthetic_state_dict  # noqa: E402

VARIANTS = ("full", "stack0", "stack1", "stack2")


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]


def time_config(name, pairs, rounds, reps):
    c = CONFIGS[name]
    n = c["n"]
    crops, pts, split = synthetic_batch(pairs, n, pts=c["pts"], hw=c["hw"], seed=5)
    crops, pts = crops.cuda(), pts.cuda()
    net = mb.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch=c["fusion"],
                         affinity_op=c["affinity_op"], softmax_mode=c["softmax_mode"], neg_threshold=c["neg_threshold"],
                         test_mode=2, dropblock=0)
    net.load_state_dict(synthetic_state_dict(c["fusion"], seed=7))
    net.cuda().eval()
    calls = {
        "full": lambda: net.predict_batch(crops, pts, split, n),
        "stack0": lambda: net.predict_batch(crops, None, None, n, stack=0),
        "stack1": lambda: net.predict_batch(None, pts, split, n, stack=1),
        "stack2": lambda: net.predict_batch(crops, pts, split, n, stack=2),
    }
    for v in VARIANTS:                                        # warm-up: every shape of the timed windows
        for _ in range(2):
            calls[v]()
    torch.cuda.synchronize()
    times = {v: [] for v in VARIANTS}
    for r in range(rounds):
        for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                calls[v]()
            b.record()
            b.synchronize()
            times[v].append(a.elapsed_time(b) / reps)
    med = {v: statistics.median(times[v]) for v in VARIANTS}
    return {
        "n": n, "pairs_per_call": pairs,
        "ms_per_call": {v: round(med[v], 3) for v in VARIANTS},
        "ms_per_call_all_rounds": {v: [round(t, 3) for t in times[v]] for v in VARIANTS},
        "ratio_to_full": {v: round(med[v] / med["full"], 4) for v in VARIANTS},
    }


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 32
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    reps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
    assert torch.cuda.is_available(), "stack_times.py needs a CUDA device"
    res = {"tool": "stack_times", "rounds": rounds, "calls_per_window": reps,
           "gpu": smi("name"), "power_limit": smi("power.limit"), "max_sm_clock": smi("clocks.max.sm")}
    for name in ("cfg4", "cfg3"):
        res[name] = time_config(name, pairs, rounds, reps)
    res["sm_clock_after"] = smi("clocks.sm")
    line = json.dumps(res)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
