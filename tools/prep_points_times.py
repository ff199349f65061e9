"""Per-frame LiDAR preparation (prep_points_batch) at KITTI scale: wall time of whole calls (host plane geometry,
uploads, the one sync, kernels), measured with device events after warm-up, against the same frames one
prep_points call each, plus the library launches per call.  Card name and power limit on the first line.
Run on a GPU box:  python tools/prep_points_times.py [frames] [points] [reps]"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb          # noqa: E402
from mmmot_b200 import _lib      # noqa: E402


def kitti_info(seed):
    p2, rect, v2c = np.eye(4), np.eye(4), np.eye(4)
    p2[:3] = [[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]]
    rect[:3, :3] = [[0.9999239, 0.00983776, -0.007445048], [-0.009869795, 0.9999421, -0.004278459],
                    [0.007402527, 0.004351614, 0.9999631]]
    v2c[:3] = [[0.007533745, -0.9999714, -0.000616602, -0.004069766], [0.01480249, 0.0007280733, -0.9998902, -0.07631618],
               [0.9998621, 0.00752379, 0.01480755, -0.2718806]]
    shape = np.array([375, 1242]) if seed % 2 == 0 else np.array([370, 1224])
    return {"calib/P2": p2, "calib/R0_rect": rect, "calib/Tr_velo_to_cam": v2c, "img_shape": shape}


def frame(P, n, seed, dev):
    """360-degree scan, ranges 1..120 m, and n detections ahead of the car (3-D boxes and 2-D image boxes)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    az = torch.rand(P, device=dev, generator=g) * 6.2832 - 3.1416
    r = 1 + torch.rand(P, device=dev, generator=g) * 119
    z = torch.rand(P, device=dev, generator=g) * 4 - 2.5
    pts = torch.stack([r * torch.cos(az), r * torch.sin(az), z, torch.rand(P, device=dev, generator=g)], 1)
    rng = np.random.default_rng(seed)
    loc = np.stack([rng.uniform(-15, 15, n), rng.uniform(1.4, 1.8, n), rng.uniform(4, 60, n)], 1)
    x1, y1 = rng.uniform(0, 1150, n), rng.uniform(120, 250, n)
    dets = {"location": loc, "dimensions": rng.uniform([3.5, 1.4, 1.6], [4.5, 1.8, 2.0], size=(n, 3)),
            "rotation_y": rng.uniform(-3.1, 3.1, n),
            "bbox": np.stack([x1, y1, x1 + rng.uniform(20, 120, n), y1 + rng.uniform(20, 100, n)], 1)}
    return pts.contiguous(), kitti_info(seed), dets, None


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts))


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    P = int(sys.argv[2]) if len(sys.argv) > 2 else 120000
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    dev = torch.device("cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}   frames {F} x {P} points, median / min of {reps} calls after warm-up")
    lib = _lib.load()
    for n in (64, 128):
        frames = [frame(P, n, 1000 * n + i, dev) for i in range(F)]
        for name, kw in (("box3d", dict(det_type="3D")), ("frustum", dict(use_frustum=True))):
            before = lib.mmmot_launch_count()
            out, split = mb.prep_points_batch(frames, **kw)
            launches = lib.mmmot_launch_count() - before
            med, mn = timed(lambda: mb.prep_points_batch(frames, **kw), reps)
            smed, smn = timed(lambda: [mb.prep_points(*f[:3], **kw) for f in frames], max(1, reps // 2))
            kept = int(split[-1])
            print(f"{name:8s} n={n:3d}: batch {med:8.2f} ms (min {mn:8.2f})  {F} single calls {smed:8.2f} ms "
                  f"(min {smn:8.2f})  launches/call {launches}  points out {kept}  "
                  f"mean/max per det {kept / (F * n):.0f}/{int((split[1:] - split[:-1]).max())}")
    # the device part alone: the batch with host geometry done once (kernels + uploads + the one sync)
    frames = [frame(P, 128, 7 + i, dev) for i in range(F)]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        mb.prep_points_batch(frames, use_frustum=True)
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if "crop_" in e.key:
            print(f"kernel {e.key[:60]:60s} {e.device_time_total / 1e3:8.3f} ms  x{e.count}")


if __name__ == "__main__":
    main()
