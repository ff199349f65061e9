"""Batched K-frame windows (``predict_batch(counts=...)``, ``forward_batch(counts=...)``) against a loop over the same
samples of ``forward`` + ``ortools_solve`` (what ``TrackingModule.predict`` runs per window before its id bookkeeping) and
of ``forward`` alone.  K = 3, 4 and 8 frames at KITTI-like counts (4-16 detections per frame, B = 32 windows per call)
and at 128 detections per frame (B = 4), on the VGG16-BN and the ResNet-50 SkipPool trunk; cfg4's heads (Fusion C,
minus_abs, dual_add), 64 x 64 crops, 512 LiDAR points per detection.

The four variants of a shape are alternated round by round in one process (order reversed every other round), so drift
on a shared host hits all alike; each round times `reps` back-to-back runs with device events after warm-up, and the
figure per variant is the median over rounds of ms per run (one run = all B windows).  Also recorded: the device time of
the copies that put each transition's feature columns into a contiguous slab for the affinity stage (the same copies
``forward_batch`` makes, timed alone on a tensor of the window's shape), and whether the batched call's assignments equal
the loop's.  Card name, power limit and SM clock are read in the same run.  Prints one JSON line (also written to the
path given as the first argument).
Run on a GPU box:  python tools/window_times.py [out.json] [rounds]"""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb                                      # noqa: E402
from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict  # noqa: E402

KITTI = {3: (9, 12, 7), 4: (6, 14, 9, 11), 8: (8, 4, 12, 16, 9, 5, 13, 10)}
SHAPES = [(f"k{K}_kitti", c, 32, 3) for K, c in KITTI.items()] + [(f"k{K}_128", (128,) * K, 4, 1) for K in (3, 4, 8)]
ARCHS = ("vgg", "resnet50")
VARIANTS = ("predict_batch", "loop_forward_ortools", "forward_batch", "loop_forward")
PTS, HW = 512, 64


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]


def make_net(arch):
    sd = synthetic_state_dict("C", seed=7, appear_arch=arch)
    net = mb.TrackingNet(3, appear_arch=arch, appear_skippool=True, score_arch="branch_cls", score_fusion_arch="C",
                         affinity_op="minus_abs", softmax_mode="dual_add", neg_threshold=0.2, test_mode=2, dropblock=0)
    net.load_state_dict(sd)
    return net.cuda().eval()


def windows(B, counts, seed):
    """B windows: per-sample (dets, det_info, dets_split) on the device, and their packing for the batched calls."""
    L = sum(counts)
    one, ds, ps, sp, off = [], [], [], [torch.zeros(1, dtype=torch.int64)], 0
    for b in range(B):
        d, info, _ = synthetic_pair(counts[0], L - counts[0], PTS, HW, seed=seed + b, ragged=True)
        one.append((d.cuda(), {k: v.cuda() for k, v in info.items()}, [torch.tensor([k]) for k in counts]))
        ds.append(d)
        ps.append(info["points"][0])
        s_ = info["points_split"][0].long()
        sp.append(s_[1:] + off)
        off += int(s_[-1])
    return one, (torch.cat(ds).cuda(), torch.cat(ps).cuda(), torch.cat(sp))


def loop_predict(net, one):
    t, res = net.test_mode, []
    for d, info, split in one:
        det, links, new, end, _ = net(d, info, split)
        res.append(mb.ortools_solve(det[t], [l[t:t + 1] for l in links], new[t], end[t], split))
    return res


def slab_copy_ms(B, counts, reps=20):
    """Device time of one window batch's transition-slab copies (B x 3 x 512 x (n_k + n_k+1) each)."""
    feats = torch.randn(B, 3, 512, sum(counts), device="cuda")
    spans, s = [], 0
    for a, b in zip(counts[:-1], counts[1:]):
        spans.append((s, a + b))
        s += a
    copy = lambda: [feats[:, :, :, s:s + w].contiguous() for s, w in spans]
    copy()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        copy()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def time_shape(net, counts, B, reps, rounds, seed):
    one, (crops, pts, split) = windows(B, counts, seed)
    runs = {
        "predict_batch": lambda: net.predict_batch(crops, pts, split, counts=counts),
        "loop_forward_ortools": lambda: loop_predict(net, one),
        "forward_batch": lambda: net.forward_batch(crops, pts, split, counts=counts),
        "loop_forward": lambda: [net(d, info, s) for d, info, s in one],
    }
    batched, looped = runs["predict_batch"](), runs["loop_forward_ortools"]()      # warm-up, and the assignments
    same = all(torch.equal(batched["assign_det"][b], r[0]) and torch.equal(batched["assign_new"][b], r[2])
               and torch.equal(batched["assign_end"][b], r[3])
               and all(torch.equal(x[b], y.reshape(x[b].shape)) for x, y in zip(batched["assign_link"], r[1]))
               for b, r in enumerate(looped))
    runs["forward_batch"](), runs["loop_forward"]()
    torch.cuda.synchronize()
    times = {v: [] for v in VARIANTS}
    for r in range(rounds):
        for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                runs[v]()
            b.record()
            b.synchronize()
            times[v].append(a.elapsed_time(b) / reps)
    med = {v: statistics.median(times[v]) for v in VARIANTS}
    copy_ms = slab_copy_ms(B, counts)
    return {
        "counts": list(counts), "windows_per_call": B, "detections_per_window": sum(counts),
        "ms_per_run": {v: round(med[v], 3) for v in VARIANTS},
        "ms_per_run_all_rounds": {v: [round(t, 3) for t in times[v]] for v in VARIANTS},
        "speedup_predict": round(med["loop_forward_ortools"] / med["predict_batch"], 3),
        "speedup_forward": round(med["loop_forward"] / med["forward_batch"], 3),
        "slab_copy_ms": round(copy_ms, 4),
        "slab_copy_share_of_forward_batch": round(copy_ms / med["forward_batch"], 5),
        "assignments_equal_loop": bool(same),
    }


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    assert torch.cuda.is_available(), "window_times.py needs a CUDA device"
    res = {"tool": "window_times", "rounds": rounds, "crop_px": HW, "points_per_detection": PTS,
           "gpu": smi("name"), "power_limit": smi("power.limit"), "max_sm_clock": smi("clocks.max.sm")}
    clocks = []
    for arch in ARCHS:
        net = make_net(arch)
        res[arch] = {}
        for i, (name, counts, B, reps) in enumerate(SHAPES):
            res[arch][name] = time_shape(net, counts, B, reps, rounds, seed=100 * i)
            clocks.append(smi("clocks.sm"))
            print(arch, name, res[arch][name]["ms_per_run"], flush=True)
        del net
        torch.cuda.empty_cache()
    res["sm_clock_after_each_shape"] = clocks
    line = json.dumps(res)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
