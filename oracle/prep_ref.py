"""ORACLE — test infrastructure, NOT product code.

CPU restatement of the reference's per-frame LiDAR preparation (SURVEY.md §8f N1), point_cloud/preprocess.py:45-106
without the file read: the field-of-view cull (box_np_ops.py:629-640), then per detection its 3-D box
(preprocess.py:66-84) or the frustum of its 2-D box (preprocess.py:85-93), empty detection -> one zero point,
reflectivity popped at :96-99.  The membership predicate of geometry.py:96-114 is vectorised numpy float64 over the
host planes of mmmot_b200.lidar_crop (whose coefficients the fixtures pin against the reference's own).  Pinned by
tests/golden/prep_*.npz, produced by the UNMODIFIED reference read_and_prep_points in oracle/make_prep_goldens.py.
"""
import numpy as np

from mmmot_b200.lidar_crop import detection_planes, fov_planes


def inside_planes(points, planes, chunk=16):
    """bool [P][n]: x*nx + y*ny + z*nz + d < 0 for all six planes, summed left to right in float64 on the float32
    coordinates (numba's evaluation with float64 planes)."""
    p = np.asarray(points, dtype=np.float32)[:, :3].astype(np.float64)
    x, y, z = p[:, None, None, 0], p[:, None, None, 1], p[:, None, None, 2]
    out = np.empty((p.shape[0], planes.shape[0]), dtype=bool)
    for b0 in range(0, planes.shape[0], chunk):
        pl = planes[None, b0:b0 + chunk]
        s = (x * pl[..., 0] + y * pl[..., 1]) + z * pl[..., 2]
        out[:, b0:b0 + chunk] = ((s + pl[..., 3]) < 0).all(-1)
    return out


def remove_outside_ref(points, info):
    """The field-of-view cull alone (remove_outside_points)."""
    points = np.asarray(points, dtype=np.float32)
    return points[inside_planes(points, fov_planes(info, info['img_shape'])[None])[:, 0]]


def prep_points_ref(points, info, dets, use_frustum=False, num_point_features=4, without_reflectivity=False,
                    det_type='3D', shift_bbox=None):
    """(points [P_out][3 or C], points_split int64 [n+1]) exactly as read_and_prep_points returns them, including its
    dtype: float64 when a detection is empty (its zero point is np.zeros((1, 4))), float32 otherwise."""
    points = remove_outside_ref(np.asarray(points, dtype=np.float32).reshape(-1, num_point_features), info)
    mask = inside_planes(points, detection_planes(info, dets, use_frustum, det_type, shift_bbox))
    out, split = [], [0]
    for b in range(mask.shape[1]):
        sel = points[mask[:, b]]
        if sel.shape[0] == 0:
            sel = np.zeros(shape=(1, 4))
        split.append(split[-1] + sel.shape[0])
        out.append(sel)
    out = np.concatenate(out, axis=0)
    if without_reflectivity:
        keep = list(range(num_point_features))
        keep.pop(3)
        out = out[:, keep]
    return out, np.asarray(split, dtype=np.int64)


def prep_points_batch_ref(frames, **kw):
    """Frames concatenated in order, splits shifted to global offsets (test_seq_dataset.py:237-244)."""
    outs, splits = [], [np.zeros(1, np.int64)]
    for points, info, dets, shift_bbox in frames:
        o, s = prep_points_ref(points, info, dets, shift_bbox=shift_bbox, **kw)
        outs.append(o.astype(np.float32))
        splits.append(s[1:] + splits[-1][-1])
    return np.concatenate(outs), np.concatenate(splits)
