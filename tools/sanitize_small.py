"""Small runs of every device path for compute-sanitizer (memcheck / racecheck): eval forward + LP on both engines
(N=M=8, 32x32 crops; the tensor-core engine forced so that its kernels, incl. the first layer's in-kernel operand
producers and VGG conv5-conv12's K-segmented accumulator epilogue with its fused pools, are the ones checked), all fusion / softmax / affinity variants, end_mode max, a three-frame sample and its
assignment programme, the training-mode forward with DropBlock + Dropout, the pinned-host pipeline, LiDAR cropping in
both precisions and image crop-and-resize.
  compute-sanitizer --tool memcheck  python tools/sanitize_small.py
  compute-sanitizer --tool racecheck python tools/sanitize_small.py"""
import os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mmmot_b200
from mmmot_b200.synthetic import synthetic_batch, synthetic_pair, synthetic_state_dict


def make(fusion, op, sm, **kw):
    net = mmmot_b200.TrackingNet(kw.pop("seq", 2), appear_skippool=True, score_arch="branch_cls", score_fusion_arch=fusion,
                                 affinity_op=op, softmax_mode=sm, neg_threshold=0.2, test_mode=2,
                                 **dict(dict(dropblock=0), **kw))
    net.load_state_dict(synthetic_state_dict(fusion, seed=3))
    return net.cuda().eval()


crops, pts, split = synthetic_batch(2, 8, pts=24, hw=32, seed=5)
for engine in ("tcgen05", "fp32"):
    mmmot_b200.set_engine(engine)
    for fusion, op, sm in (("C", "minus_abs", "dual_add"), ("A", "multiply", "none"), ("B", "minus", "dual_max"),
                           ("C", "multiply", "single"), ("C", "minus_abs", "dual")):
        out = make(fusion, op, sm).predict_batch(crops.cuda(), pts.cuda(), split, 8)
    torch.cuda.synchronize()
    print(engine, "match", out["match"].cpu().tolist(), "status", int(out["status"]))
mmmot_b200.set_engine("auto")

# end_mode max + a three-frame sample through forward
net = make("C", "minus_abs", "dual_add", seq=3, end_mode="max")
dets, info, _ = synthetic_pair(5, 11, 24, 32, seed=61, ragged=True)
o = net(dets.cuda(), {k: v.cuda() for k, v in info.items()}, [torch.tensor([5]), torch.tensor([7]), torch.tensor([4])])
print("multi-frame link shapes", [tuple(l.shape) for l in o[1]])
a = mmmot_b200.ortools_solve(o[0][2], [l[2:3] for l in o[1]], o[2][2], o[3][2], [5, 7, 4])
print("multi-frame assignment kept", int(a[0].sum()))

# training-mode forward with DropBlock / Dropout
net = make("C", "minus_abs", "dual_add", dropblock=5, use_dropout=True).train()
dets, info, ds = synthetic_pair(9, 6, 40, 64, seed=23, ragged=True)
torch.manual_seed(0)
o = net(dets.cuda(), {k: v.cuda() for k, v in info.items()}, ds)
print("train det", tuple(o[0].shape))

# pinned-host pipeline
net = make("C", "minus_abs", "dual_add")
crops, pts, split = synthetic_batch(8, 8, pts=24, hw=32, seed=7)
r = mmmot_b200.HostPipeline(net, 8, sub_batches=4).run(crops.pin_memory(), pts.pin_memory(), split)
print("pipeline match rows", r["match"].shape[0])

# LiDAR cropping (fp32 and fp64 predicate) and image crops
rng = np.random.default_rng(3)
P, n = 20000, 16
centers = rng.uniform([0, -30, -2], [70, 30, 0], size=(n, 3)).astype(np.float32)
pc = np.concatenate([centers[rng.integers(0, n, P)] + rng.normal(size=(P, 3)) * [3.0, 2.0, 1.0], rng.uniform(size=(P, 1))], 1).astype(np.float32)
boxes = np.concatenate([centers, rng.uniform([1.2, 2.5, 1.2], [2.2, 5.0, 2.0], size=(n, 3)), rng.uniform(-3.14, 3.14, size=(n, 1))], 1)
for b in (boxes.astype(np.float32), boxes.astype(np.float64)):
    out, sp = mmmot_b200.crop_points(torch.from_numpy(pc).cuda(), b)
print("crop points", tuple(out.shape))
from tools.prep_points_times import frame   # noqa: E402
prep_frames = [frame(P, k, 50 + k, torch.device("cuda")) for k in (3, 1, 9)]   # several frames, image shapes, counts
for kw in (dict(det_type="3D"), dict(use_frustum=True, without_reflectivity=True)):
    out, sp = mmmot_b200.prep_points_batch(prep_frames, **kw)
print("prep points", tuple(out.shape))
img = torch.from_numpy(rng.integers(0, 256, size=(120, 200, 3), dtype=np.uint8)).cuda()
bb = np.array([[10.2, 5.5, 80.9, 70.1], [-4.0, 30.0, 60.0, 130.0], [150.0, 20.0, 199.0, 119.0]], np.float32)
print("crop_resize", tuple(mmmot_b200.crop_resize(img, bb, out_size=32).shape))
torch.cuda.synchronize()
