"""Association programme of K-frame samples: solve_frames (csrc/flow_assign.cu, min-cost flow) per call of B samples,
from device events after warm-up, for K in {3, 5, 8} and n in {8, 16, 32, 64, 128} detections per frame; next to it
mmmot_lp_assign (solve_batch) at K = 2 for the same n and B, and the host MILP restatement (oracle/lp_ref.py, HiGHS)
per sample.  Card name, power limit and SM clock are read in the same run.  Prints one JSON line (also written to the
path given as the first argument).
--cap: instead, one sample of dense random scores per call at L = 2048 (16 frames of 128) and at L = 4469 (64 frames,
the most detections one sample's shared-memory state admits), one timed call each: what a single launch costs there.
Run on a GPU box:  python tools/flow_times.py [out.json] [B] [reps]      python tools/flow_times.py --cap [out.json]"""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb          # noqa: E402
from oracle import lp_ref        # noqa: E402


def scores(g, counts, B):
    """Random continuous scores in the forward's layout (new zero on frame 0, end zero on the last frame)."""
    L = sum(counts)
    det = torch.rand(B, L, generator=g) - (torch.rand(B, L, generator=g) < 0.3).float()
    links = [torch.rand(B, a, b, generator=g) - 0.25 for a, b in zip(counts[:-1], counts[1:])]
    new, end = torch.rand(B, L, generator=g) - 0.2, torch.rand(B, L, generator=g) - 0.2
    new[:, :counts[0]] = 0
    end[:, L - counts[-1]:] = 0
    return det, links, new, end


def device_ms(fn, reps, warm=True):
    if warm:
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]


def cap(out):
    card = smi("name,power.limit,clocks.max.sm")
    g = torch.Generator().manual_seed(4469)
    det, links, new, end = scores(g, [8, 8, 8], 1)
    mb.solve_frames(det.cuda(), [l.cuda() for l in links], new.cuda(), end.cuda(), [8, 8, 8])     # loads the module
    rows = []
    for counts in ([128] * 16, [70] * 63 + [59]):
        det, links, new, end = scores(g, counts, 1)
        dd, dn, de = det.cuda(), new.cuda(), end.cuda()
        dl = [l.cuda() for l in links]
        ms = device_ms(lambda: mb.solve_frames(dd, dl, dn, de, counts), 1, warm=False)
        rows.append({"K": len(counts), "L": sum(counts), "B": 1, "solver": "mmmot_flow_assign",
                     "ms_per_call": round(ms, 1), "sm_clock": smi("clocks.sm")})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    line = json.dumps({"tool": "flow_times --cap", "card": card, "statistic": "one call, module already loaded",
                       "rows": rows})
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--cap":
        return cap(sys.argv[2] if len(sys.argv) > 2 else None)
    out = sys.argv[1] if len(sys.argv) > 1 else None
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 128
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    card = smi("name,power.limit,clocks.max.sm")
    rows, sm_clocks = [], []
    for n in (8, 16, 32, 64, 128):
        g = torch.Generator().manual_seed(n)
        det, links, new, end = scores(g, [n, n], B)
        dd, dl, dn, de = det.cuda(), links[0].cuda(), new.cuda(), end.cuda()
        ms = device_ms(lambda: mb.solve_batch(dd, dl, dn, de, n, n), reps)
        rows.append({"K": 2, "n": n, "B": B, "solver": "mmmot_lp_assign", "ms_per_call": round(ms, 4)})
        for K in (3, 5, 8):
            counts = [n] * K
            det, links, new, end = scores(g, counts, B)
            dd, dn, de = det.cuda(), new.cuda(), end.cuda()
            dl = [l.cuda() for l in links]
            r = mb.solve_frames(dd, dl, dn, de, counts)
            ms = device_ms(lambda: mb.solve_frames(dd, dl, dn, de, counts), reps)
            sm_clocks.append(smi("clocks.sm"))
            hs = 1 if K * n > 256 else 3
            t0 = time.perf_counter()
            objs = [lp_ref.milp_solve(det[b], [l[b:b + 1] for l in links], new[b], end[b], counts)[1] for b in range(hs)]
            host_s = (time.perf_counter() - t0) / hs
            got = [lp_ref.objective(det[b], [l[b:b + 1] for l in links], new[b], end[b],
                                    (r["assign_det"][b].cpu(), [x[b:b + 1].cpu() for x in r["assign_link"]],
                                     r["assign_new"][b].cpu(), r["assign_end"][b].cpu())) for b in range(hs)]
            rows.append({"K": K, "n": n, "B": B, "solver": "mmmot_flow_assign", "ms_per_call": round(ms, 4),
                         "milp_host_s_per_sample": round(host_s, 4), "milp_samples": hs,
                         "objective_equals_milp": all(abs(a - b) < 1e-8 for a, b in zip(got, objs))})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    line = json.dumps({"tool": "flow_times", "card": card, "sm_clock_after_each_flow_shape": sm_clocks,
                       "reps": reps, "statistic": "median device time per call after one warm-up call", "rows": rows})
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
