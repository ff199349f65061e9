"""Per-frame LiDAR preparation (SURVEY.md §8f N1): field-of-view cull + 3-D boxes or 2-D frustums, many frames per call.
Oracle and host plane coefficients vs fixtures of the UNMODIFIED reference read_and_prep_points (CPU); the GPU path vs
the fixtures, the oracle and itself (single-frame calls vs one batched call)."""
import ctypes
import glob
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN_DIR
from kernel_kit import vp
from mmmot_b200.lidar_crop import box_camera_to_lidar, detection_planes, fov_planes
from oracle.crop_ref import crop_points_ref
from oracle.make_prep_goldens import kitti_calib, synthetic_scan
from oracle.prep_ref import prep_points_batch_ref, prep_points_ref, remove_outside_ref

GOLD = sorted(glob.glob(os.path.join(GOLDEN_DIR, "prep_*.npz")))
IDS = [os.path.basename(p) for p in GOLD]


def load(path):
    g = np.load(path)
    info = {"calib/P2": g["P2"], "calib/R0_rect": g["R0_rect"], "calib/Tr_velo_to_cam": g["Tr_velo_to_cam"],
            "img_shape": g["img_shape"]}
    dets = {k: g[k] for k in ("location", "dimensions", "rotation_y", "bbox")}
    kw = dict(use_frustum=bool(g["use_frustum"]), det_type=str(g["det_type"]),
              without_reflectivity=bool(g["without_reflectivity"]),
              shift_bbox=g["shift_bbox"] if "shift_bbox" in g.files else None)
    return g, info, dets, kw


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_fixture_set_covers_the_cases():
    cases = [load(p) for p in GOLD]
    assert len(cases) == 4
    assert {str(g["det_type"]) for g, *_ in cases} == {"3D", "2D"}
    assert {bool(g["use_frustum"]) for g, *_ in cases} == {True, False}
    assert {bool(g["without_reflectivity"]) for g, *_ in cases} == {True, False}
    frustum = [(g, d, kw) for g, _, d, kw in cases if kw["use_frustum"] or kw["det_type"] == "2D"]
    boxes = [kw["shift_bbox"] if kw["shift_bbox"] is not None else d["bbox"] for _, d, kw in frustum]
    assert {b.dtype for b in boxes} == {np.dtype(np.float32), np.dtype(np.float64)}


@pytest.mark.parametrize("path", GOLD, ids=IDS)
def test_oracle_matches_reference_golden(path):
    g, info, dets, kw = load(path)
    out, split = prep_points_ref(g["points"], info, dets, **kw)
    assert out.dtype == g["out"].dtype and out.shape == g["out"].shape           # float64 once a detection is empty
    assert np.array_equal(out, g["out"]) and np.array_equal(split, g["split"])
    keep = np.unpackbits(g["fov_keep"])[:len(g["points"])].astype(bool)
    fov = remove_outside_ref(g["points"], info)
    assert len(fov) == int(g["fov_count"]) and np.array_equal(fov, g["points"][keep])


@pytest.mark.parametrize("path", GOLD, ids=IDS)
def test_host_planes_match_reference_bit_for_bit(path):
    g, info, dets, kw = load(path)
    assert same_bits(fov_planes(info, info["img_shape"]), g["fov_planes"])
    assert same_bits(detection_planes(info, dets, kw["use_frustum"], kw["det_type"], kw["shift_bbox"]), g["det_planes"])


def test_fixtures_exercise_what_they_claim():
    g, info, dets, kw = load(os.path.join(GOLDEN_DIR, "prep_3d.npz"))
    rect, v2c = info["calib/R0_rect"].astype(np.float32), info["calib/Tr_velo_to_cam"].astype(np.float32)
    boxes = box_camera_to_lidar(np.concatenate([dets["location"], dets["dimensions"], dets["rotation_y"][:, None]],
                                               1).astype(np.float32), rect, v2c)
    ref = np.diff(g["split"])
    raw = np.diff(crop_points_ref(g["points"], boxes)[1])                      # the 3-D box test without the cull
    assert ref[3] < raw[3] and ref[4] < raw[4]                                 # straddling the left / right image edge
    assert ref[6] < raw[6]                                                     # straddling the far clip (depth 100)
    assert ref[7] == 1 and raw[7] > 100                                        # behind the camera: culled to empty
    assert np.array_equal(ref[:3], raw[:3])                                    # boxes well inside the image
    keep = np.unpackbits(g["fov_keep"])[:len(g["points"])].astype(bool)
    assert (g["points"][~keep, 0] > 100).any()                                 # far points ahead are dropped
    for p in GOLD:
        g, info, dets, kw = load(p)
        n = np.diff(g["split"])
        assert (~g["out"][g["split"][:-1][n == 1]].any(1)).any()                # an empty detection: one zero point
        if kw["use_frustum"] or kw["det_type"] == "2D":
            bb = kw["shift_bbox"] if kw["shift_bbox"] is not None else dets["bbox"]
            w, h = info["img_shape"][1], info["img_shape"][0]
            across = (bb[:, 0] < 0) | (bb[:, 2] > w) | (bb[:, 1] < 0) | (bb[:, 3] > h)
            assert (n[across] > 100).any()                                     # a frustum across the border holds points
            if kw["shift_bbox"] is None:
                assert n[bb[:, 0] == bb[:, 2]].tolist() == [1]                 # degenerate box: empty


# ---------------------------------------------------------------- GPU

def calib_1224():
    """A second KITTI-like camera (370 x 1224 image, different intrinsics)."""
    info = kitti_calib()
    info["calib/P2"] = info["calib/P2"].copy()
    info["calib/P2"][:3] = [[7.070493e+02, 0.0, 6.040814e+02, 4.575831e+01], [0.0, 7.070493e+02, 1.805066e+02, -0.3454157],
                            [0.0, 0.0, 1.0, 4.981016e-03]]
    info["img_shape"] = np.array([370, 1224])
    return info


def random_frame(P, n, seed, info, all_empty=False):
    """A 360-degree scan with n detections: 3-D boxes ahead of the car and 2-D boxes in and around the image
    (all_empty: boxes behind the camera and degenerate 2-D boxes)."""
    rng = np.random.default_rng(seed)
    loc = np.stack([rng.uniform(-15, 15, n), rng.uniform(1.4, 1.8, n), rng.uniform(4, 60, n)], 1)
    if all_empty:
        loc[:, 2] = -rng.uniform(10, 30, n)
    clusters = np.concatenate([loc, rng.uniform([3.5, 1.4, 1.6], [4.5, 1.8, 2.0], size=(n, 3))], 1)
    pts = synthetic_scan(P, seed, info, clusters=clusters)
    x1 = rng.uniform(-80, 1200, n)
    y1 = rng.uniform(100, 250, n)
    bbox = np.stack([x1, y1, x1 + rng.uniform(0 if all_empty else 10, 150, n), y1 + rng.uniform(10, 100, n)], 1)
    if all_empty:
        bbox[:, 2] = bbox[:, 0]
    dets = {"location": loc, "dimensions": clusters[:, 3:6], "rotation_y": rng.uniform(-3.1, 3.1, n),
            "bbox": bbox.astype(np.float32 if seed % 2 else np.float64)}
    return pts, dets


def gpu_frames(spec):
    frames, host = [], []
    for P, n, seed, info, empty in spec:
        pts, dets = random_frame(P, n, seed, info, empty)
        frames.append((torch.from_numpy(pts).cuda(), info, dets, None))
        host.append((pts, info, dets, None))
    return frames, host


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLD, ids=IDS)
def test_gpu_prep_points_matches_reference_golden(path):
    import mmmot_b200
    g, info, dets, kw = load(path)
    # host planes first: a numpy / LAPACK difference is reported as that, not as a kernel fault
    assert same_bits(fov_planes(info, info["img_shape"]), g["fov_planes"])
    assert same_bits(detection_planes(info, dets, kw["use_frustum"], kw["det_type"], kw["shift_bbox"]), g["det_planes"])
    out, split = mmmot_b200.prep_points(torch.from_numpy(g["points"]).cuda(), info, dets, **kw)
    assert out.dtype == torch.float32 and split.dtype == torch.int64
    assert torch.equal(split, torch.from_numpy(g["split"]))
    o = out.cpu().numpy()
    assert o.shape == g["out"].shape and np.array_equal(o.astype(g["out"].dtype), g["out"])


@pytest.mark.gpu
@pytest.mark.parametrize("branch", [dict(det_type="3D"), dict(use_frustum=True), dict(det_type="2D")],
                         ids=["box3d", "frustum", "det2d"])
@pytest.mark.parametrize("without_reflectivity", [False, True])
def test_gpu_batch_equals_single_frames_and_oracle(branch, without_reflectivity):
    import mmmot_b200
    spec = [(24000, 8, 11, kitti_calib(), False), (5000, 3, 12, calib_1224(), False),
            (60000, 40, 13, calib_1224(), False), (700, 2, 14, kitti_calib(), True),
            (30000, 70, 15, kitti_calib(), False), (1, 1, 16, calib_1224(), False)]
    frames, host = gpu_frames(spec)
    kw = dict(branch, without_reflectivity=without_reflectivity)
    out, split = mmmot_b200.prep_points_batch(frames, **kw)
    singles = [mmmot_b200.prep_points(p, i, d, shift_bbox=s, **kw) for p, i, d, s in frames]
    cat_out = torch.cat([o for o, _ in singles])
    cat_split = [torch.zeros(1, dtype=torch.int64)]
    for _, s in singles:
        cat_split.append(s[1:] + cat_split[-1][-1])
    assert torch.equal(split, torch.cat(cat_split)) and torch.equal(out, cat_out)
    ro, rs = prep_points_batch_ref(host, **kw)
    assert out.shape[1] == (3 if without_reflectivity else 4)
    assert torch.equal(split, torch.from_numpy(rs)) and np.array_equal(out.cpu().numpy(), ro)
    n = np.diff(rs)
    lo, hi = int(rs[sum(s[1] for s in spec[:3])]), int(rs[sum(s[1] for s in spec[:4])])
    assert hi - lo == 2 and not out[lo:hi].any()                               # the all-empty frame: zero points
    assert (n > 1).sum() > 20


@pytest.mark.gpu
@pytest.mark.parametrize("use_frustum", [False, True], ids=["box3d", "frustum"])
def test_gpu_kitti_scale_batch_matches_oracle(use_frustum):
    import mmmot_b200
    spec = [(120000, 128, 21 + i, kitti_calib() if i % 2 == 0 else calib_1224(), False) for i in range(3)]
    frames, host = gpu_frames(spec)
    out, split = mmmot_b200.prep_points_batch(frames, use_frustum=use_frustum, without_reflectivity=True)
    ro, rs = prep_points_batch_ref(host, use_frustum=use_frustum, without_reflectivity=True)
    assert torch.equal(split, torch.from_numpy(rs)) and np.array_equal(out.cpu().numpy(), ro)


@pytest.mark.gpu
def test_gpu_launch_count_does_not_grow_with_frames():
    import mmmot_b200
    from mmmot_b200 import _lib
    lib = _lib.load()
    frames, _ = gpu_frames([(3000, 4, 100 + i, kitti_calib(), False) for i in range(256)])
    grow = []
    for fs in (frames[:1], frames):
        mmmot_b200.prep_points_batch(fs, use_frustum=True)              # warm
        before = lib.mmmot_launch_count()
        mmmot_b200.prep_points_batch(fs, use_frustum=True)
        grow.append(lib.mmmot_launch_count() - before)
    assert grow[0] == grow[1] == 5


@pytest.mark.gpu
def test_gpu_frame_without_detections_raises():
    import mmmot_b200
    frames, _ = gpu_frames([(2000, 3, 200, kitti_calib(), False), (2000, 1, 201, kitti_calib(), False)])
    p, info, dets, _ = frames[1]
    dets = {k: v[:0] for k, v in dets.items()}
    with pytest.raises(ValueError):
        mmmot_b200.prep_points_batch([frames[0], (p, info, dets, None)])
    with pytest.raises(ValueError):
        mmmot_b200.prep_points(p, info, dets, use_frustum=True)


@pytest.mark.gpu
def test_gpu_bad_arguments_are_rejected():
    from mmmot_b200 import _lib
    lib = _lib.load()
    pts = torch.zeros(100, 4, device="cuda")
    planes = torch.zeros(3, 24, dtype=torch.float64, device="cuda")
    split = torch.zeros(3, dtype=torch.int32, device="cuda")
    out = torch.zeros(10, 4, device="cuda")
    ws = torch.empty(int(lib.mmmot_prep_workspace(60, 2, 2)), dtype=torch.uint8, device="cuda")
    ints = lambda *v: (ctypes.c_int * len(v))(*v)

    def count(offs, det_frame, stride=4):
        return lib.mmmot_prep_count(vp(pts), ints(*offs), 2, stride, vp(planes), vp(planes), ints(*det_frame), 2,
                                    vp(split), vp(ws), ws.numel(), None)

    def scatter(out_c):
        return lib.mmmot_prep_scatter(vp(pts), ints(0, 40, 100), 2, 4, vp(planes), vp(planes), ints(0, 1), 2,
                                      vp(split), out_c, vp(out), vp(ws), ws.numel(), None)
    E_ARG = -1
    assert count((0, 60, 50), (0, 1)) == E_ARG           # non-monotone frame offsets
    assert count((5, 40, 100), (0, 1)) == E_ARG          # offsets not starting at 0
    assert count((0, 40, 100), (0, 2)) == E_ARG          # frame index out of range
    assert count((0, 40, 100), (1, 0)) == E_ARG          # detections not grouped in frame order
    assert count((0, 40, 100), (0, 1), stride=5) == E_ARG
    assert scatter(2) == E_ARG and scatter(5) == E_ARG   # channels outside 3..4
    assert count((0, 40, 100), (0, 1)) == 0
    assert scatter(4) == 0
    torch.cuda.synchronize()
