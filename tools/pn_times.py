"""PointNet stage alone: per-kernel device times from the library's tagged timing hook.
Run on a GPU box:  python tools/pn_times.py [n] [pts] [pairs] [channels]     TC_DBG=... sets mmmot_set_debug bits.

channels: the point width, 3 (xyz) or 4 (xyz + reflectance, a without_reflectivity=False net), or a comma list such as
3,4: one net per width on the same xyz, measured in ROUNDS alternating rounds (default 5) in this one process.  Each
round times the stage over REPS untimed-hook calls (default 20) with CUDA events (median per call), then one call with
the tagged timing hook on for the per-kernel lines (every round for layer 1 and the per-detection-sum passes, round 0
for the rest).  TC_DBG takes a comma list too, alternated within each round in this one process: TC_DBG=0,65536 sets
the dedicated per-detection-sum kernel against the general TMA-fed one.  The card's name, power limit and max SM clock
come first."""
import ctypes
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb          # noqa: E402
from mmmot_b200 import _lib      # noqa: E402
from mmmot_b200.synthetic import synthetic_state_dict   # noqa: E402
from tools.aff_times import collect                     # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    pts = int(sys.argv[2]) if len(sys.argv) > 2 else 512
    pairs = int(sys.argv[3]) if len(sys.argv) > 3 else 32
    widths = [int(c) for c in (sys.argv[4] if len(sys.argv) > 4 else "3").split(",")]
    rounds = int(os.environ.get("ROUNDS", "5"))
    reps = int(os.environ.get("REPS", "20"))
    L = 2 * n
    print(f"card: {card()}")
    lib = _lib.load()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(1)
    xyzr = torch.randn(pairs * L * pts, 4, device=dev, generator=g)
    xyzr[:, 3].uniform_(0.0, 1.0, generator=g)
    split = torch.arange(0, pairs * L * pts + 1, pts, dtype=torch.int32)
    split_d = split.to(dev)
    hs = split.numpy()
    feats = torch.empty(pairs, 3, 512, L, device=dev)
    ws = torch.empty(int(lib.mmmot_pointnet_workspace(pairs, L, pairs * L * pts)), dtype=torch.uint8, device=dev)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    nets, points = {}, {}
    for c in widths:
        net = mb.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", score_fusion_arch="C", test_mode=2, dropblock=0,
                             without_reflectivity=(c == 3))
        net.load_state_dict(synthetic_state_dict("C", seed=0, point_in=c))
        nets[c] = net.cuda().eval().prepared()
        points[c] = xyzr[:, :c].contiguous()

    def run(c):
        _lib.check(lib.mmmot_pointnet_fwd(nets[c].ptr, vp(points[c]), vp(split_d), ctypes.c_void_p(hs.ctypes.data), pairs, L,
                                          vp(feats), vp(ws), ws.numel(), st), "mmmot_pointnet_fwd")
    stage = {(dbg, c): [] for dbg in [int(x) for x in os.environ.get("TC_DBG", "0").split(",")] for c in widths}
    for dbg, c in stage:
        lib.mmmot_set_debug(dbg)
        for _ in range(2):
            run(c)
    torch.cuda.synchronize()
    for r in range(rounds):
        for (dbg, c), times in stage.items():
            lib.mmmot_set_debug(dbg)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
            ev[0].record()
            for i in range(reps):
                run(c)
                ev[i + 1].record()
            torch.cuda.synchronize()
            ms = statistics.median(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
            times.append(ms)
            lib.mmmot_timing_enable(1)
            run(c)
            torch.cuda.synchronize()
            lib.mmmot_timing_enable(0)
            tags = collect(lib)
            print(f"round {r} n={n} pts={pts} pairs={pairs} channels={c} dbg={dbg}: PointNet stage {ms:.3f} ms "
                  f"(median of {reps})")
            for name, (tms, fl, by, cnt) in tags.items():
                if r == 0 or name.startswith("pointnet.l1") or name.endswith("_segsum"):
                    print(f"   {name:32s} {tms:8.3f} ms  {fl / tms / 1e9 if tms else 0:8.1f} TFLOP/s  "
                          f"{by / tms / 1e6 if tms else 0:8.1f} GB/s")
    lib.mmmot_set_debug(0)
    for (dbg, c), times in stage.items():
        print(f"summary channels={c} dbg={dbg}: stage ms per round {[round(t, 3) for t in times]}, "
              f"median {statistics.median(times):.3f}")


if __name__ == "__main__":
    main()
