"""ORACLE fixture generator for the per-frame LiDAR preparation (SURVEY.md §8f N1) — needs a checkout of the reference:

    MMMOT_REFERENCE=<path to ZwwWayne/mmMOT> python -m oracle.make_prep_goldens

Runs the UNMODIFIED reference ``point_cloud.preprocess.read_and_prep_points`` (numba) on seeded synthetic 360-degree
scans, written to a temporary ``velodyne/<seq>/<frame>`` file as the reference reads them, with a KITTI calibration,
and stores under tests/golden/prep_*.npz: the scan, calibration and detections, the reference's output and split,
the output of its ``remove_outside_points`` (as the packed mask of the scan points it keeps, checked against it),
and the reference's own plane coefficients (``surface_equ_3d`` on its surfaces) for the field of view and every
detection's region.
"""
import os
import sys
import tempfile

import numpy as np

from mmmot_b200.lidar_crop import box_camera_to_lidar
from oracle import ref_loader

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

IMG_SHAPE = np.array([375, 1242], dtype=np.int64)


def kitti_calib():
    """Calibration of KITTI tracking sequence 0000 (public devkit values), as 4x4 float64 like the KITTI infos."""
    p2, rect, v2c = np.eye(4), np.eye(4), np.eye(4)
    p2[:3] = [[7.215377e+02, 0.0, 6.095593e+02, 4.485728e+01], [0.0, 7.215377e+02, 1.728540e+02, 2.163791e-01],
              [0.0, 0.0, 1.0, 2.745884e-03]]
    rect[:3, :3] = [[9.999239e-01, 9.837760e-03, -7.445048e-03], [-9.869795e-03, 9.999421e-01, -4.278459e-03],
                    [7.402527e-03, 4.351614e-03, 9.999631e-01]]
    v2c[:3] = [[7.533745e-03, -9.999714e-01, -6.166020e-04, -4.069766e-03],
               [1.480249e-02, 7.280733e-04, -9.998902e-01, -7.631618e-02],
               [9.998621e-01, 7.523790e-03, 1.480755e-02, -2.717806e-01]]
    return {"calib/P2": p2, "calib/R0_rect": rect, "calib/Tr_velo_to_cam": v2c, "img_shape": IMG_SHAPE}


# camera-frame 3-D boxes (x, y, z, l, h, w): inside the image, straddling its left and right edges (x/z = -0.845 and
# +0.876 at u = 0 and 1242), straddling the far clip (depth 100), and behind the camera
BOXES_3D = np.array([[2.0, 1.6, 15.0, 4.0, 1.6, 1.8], [-3.0, 1.7, 25.0, 4.2, 1.5, 1.7], [5.0, 1.6, 40.0, 3.9, 1.6, 1.7],
                     [-12.7, 1.6, 15.0, 4.0, 1.6, 1.8], [13.1, 1.6, 15.0, 4.0, 1.6, 1.8],
                     [-25.0, 1.6, 30.0, 4.5, 1.7, 1.9], [1.0, 1.6, 99.5, 4.0, 1.6, 1.8],
                     [0.0, 1.6, -10.0, 4.0, 1.6, 1.8]])
# image boxes (x1, y1, x2, y2): inside, across the left / right / top borders, degenerate (x1 == x2), and a sliver at
# the top of the image that holds no point
BBOXES = np.array([[550.0, 150.0, 650.0, 220.0], [300.0, 160.0, 420.0, 230.0], [800.5, 140.25, 900.75, 260.5],
                   [-60.0, 150.0, 60.0, 230.0], [1180.0, 150.0, 1300.0, 230.0], [600.0, -40.0, 700.0, 30.0],
                   [700.0, 150.0, 700.0, 250.0], [100.0, 0.0, 101.0, 1.0]])


def synthetic_scan(n_points, seed, info=None, clusters=BOXES_3D):
    """[P][4] float32: a 360-degree scan with ranges out to 130 m plus point clusters around the camera-frame boxes
    (so that the boxes and the frustums through them hold points)."""
    info = info or kitti_calib()
    rng = np.random.default_rng(seed)
    n_bg = n_points * 3 // 5
    az = rng.uniform(-np.pi, np.pi, n_bg)
    rr = rng.uniform(1.0, 130.0, n_bg)
    bg = np.stack([rr * np.cos(az), rr * np.sin(az), rng.uniform(-2.5, 1.5, n_bg)], 1)
    cam = np.concatenate([clusters[:, :3], clusters[:, 3:6], np.zeros((len(clusters), 1))], 1)
    lid = box_camera_to_lidar(cam, info["calib/R0_rect"], info["calib/Tr_velo_to_cam"])
    centres = lid[:, :3] + np.stack([np.zeros(len(lid)), np.zeros(len(lid)), lid[:, 5] / 2], 1)
    n_cl = n_points - n_bg
    cl = centres[rng.integers(0, len(centres), n_cl)] + rng.normal(size=(n_cl, 3)) * [1.5, 1.2, 0.6]
    xyz = np.concatenate([bg, cl])[rng.permutation(n_points)]
    return np.concatenate([xyz, rng.uniform(size=(n_points, 1))], 1).astype(np.float32)


def dets_for(seed, bbox_dtype):
    rng = np.random.default_rng(seed)
    return {"location": BOXES_3D[:, :3].copy(), "dimensions": BOXES_3D[:, 3:6].copy(),
            "rotation_y": rng.uniform(-3.1, 3.1, len(BOXES_3D)), "bbox": BBOXES.astype(bbox_dtype)}


# (name, seed, use_frustum, det_type, without_reflectivity, bbox dtype, shift_bbox)
CASES = [
    ("prep_3d", 1, False, "3D", False, np.float64, False),
    ("prep_frustum_f32", 3, True, "3D", True, np.float32, False),
    ("prep_frustum_shift_f64", 5, True, "3D", False, np.float64, True),
    ("prep_2d", 6, False, "2D", True, np.float64, False),
]


def reference_planes(surfaces):
    from point_cloud.geometry import surface_equ_3d
    n, d = surface_equ_3d(surfaces[:, :, :3, :])
    return np.concatenate([n, d[..., None]], axis=-1)


def prep_goldens(n_points=24000):
    sys.path.insert(0, ref_loader.REF)
    from point_cloud import box_np_ops as B
    from point_cloud.preprocess import read_and_prep_points
    info = kitti_calib()
    rect = info["calib/R0_rect"].astype(np.float32)
    v2c = info["calib/Tr_velo_to_cam"].astype(np.float32)
    p2 = info["calib/P2"].astype(np.float32)
    for name, seed, use_frustum, det_type, wo_refl, bdt, shift in CASES:
        pts = synthetic_scan(n_points, seed, info)
        dets = dets_for(seed, bdt)
        shift_bbox = (dets["bbox"] + np.random.default_rng(seed).uniform(-8, 8, dets["bbox"].shape)).astype(bdt) \
            if shift else None
        with tempfile.TemporaryDirectory() as root:
            os.makedirs(os.path.join(root, "velodyne", "0000"))
            pts.tofile(os.path.join(root, "velodyne", "0000", "000000.bin"))
            ex = read_and_prep_points(info, root, "0000-000000.bin", dets, use_frustum=use_frustum,
                                      num_point_features=4, without_reflectivity=wo_refl, det_type=det_type,
                                      shift_bbox=shift_bbox)
        # the reference's own plane coefficients, through its own functions
        c, r, t = B.projection_matrix_to_CRT_kitti(p2)
        fr = B.get_frustum([0, 0, info["img_shape"][1], info["img_shape"][0]], c)
        fr -= t
        fr_lidar = B.camera_to_lidar((np.linalg.inv(r) @ fr.T).T, rect, v2c)
        fov_planes = reference_planes(B.corner_to_surfaces_3d_jit(fr_lidar[np.newaxis]))[0]
        fov_pts = B.remove_outside_points(pts, rect, v2c, p2, info["img_shape"])
        # remove_outside_points keeps a subsequence of the scan: stored as its packed keep-mask (a few KB)
        keep = B.points_in_convex_polygon_3d_jit(pts[:, :3], B.corner_to_surfaces_3d_jit(fr_lidar[np.newaxis]))[:, 0]
        assert np.array_equal(pts[keep], fov_pts)
        if det_type == "3D" and not use_frustum:
            boxes = np.concatenate([dets["location"], dets["dimensions"], dets["rotation_y"][:, None]],
                                   1).astype(np.float32)
            boxes = B.box_camera_to_lidar(boxes, rect, v2c)
            det_planes = reference_planes(B.corner_to_surfaces_3d(B.center_to_corner_box3d(
                boxes[:, :3], boxes[:, 3:6], boxes[:, 6], origin=[0.5, 0.5, 0], axis=2)))
        else:
            bb = shift_bbox if shift_bbox is not None else dets["bbox"]
            det_planes = []
            for i in range(len(bb)):                     # one box at a time, as get_frustum_points is called
                fs = B.get_frustum_v2(bb[i:i + 1], c)
                fs -= t
                fs = B.camera_to_lidar(np.einsum('ij, akj->aki', np.linalg.inv(r), fs), rect, v2c)
                det_planes.append(reference_planes(B.corner_to_surfaces_3d_jit(fs))[0])
            det_planes = np.stack(det_planes)
        extra = {"shift_bbox": shift_bbox} if shift_bbox is not None else {}
        np.savez_compressed(os.path.join(OUT, name + ".npz"), points=pts, P2=info["calib/P2"],
                            R0_rect=info["calib/R0_rect"], Tr_velo_to_cam=info["calib/Tr_velo_to_cam"],
                            img_shape=info["img_shape"], location=dets["location"], dimensions=dets["dimensions"],
                            rotation_y=dets["rotation_y"], bbox=dets["bbox"], use_frustum=use_frustum,
                            det_type=det_type, without_reflectivity=wo_refl, out=ex["points"],
                            split=np.asarray(ex["points_split"], np.int64), fov_keep=np.packbits(keep),
                            fov_count=len(fov_pts),
                            fov_planes=fov_planes, det_planes=det_planes, **extra)
        print(name, "fov", len(fov_pts), "out", ex["points"].shape, ex["points"].dtype,
              "per det", np.diff(ex["points_split"]))


if __name__ == "__main__":
    prep_goldens()
