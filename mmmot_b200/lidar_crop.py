"""Per-detection LiDAR preparation on the GPU (SURVEY.md §8f N1 — the step right before the hot path).

``prep_points`` / ``prep_points_batch`` mirror reference point_cloud/preprocess.py:45-106
(``read_and_prep_points`` without the file read): the scan is culled to camera 2's field of view
(box_np_ops.py:629-640), then every detection keeps the surviving points inside its region, in scan order —
its rotated 3-D box (camera frame: location, dimensions l-h-w, rotation_y; preprocess.py:66-84) when
``det_type == '3D'`` and not ``use_frustum``, otherwise the view frustum of its 2-D image box
(``shift_bbox`` or ``dets['bbox']``; preprocess.py:85-93, box_np_ops.py:643-653).  An empty detection
contributes one all-zero point, and the result is the packed ``points`` + ``points_split`` pair that
``TrackingNet.forward`` / ``forward_batch`` take.  ``crop_points`` is the 3-D box test alone, on an
already culled cloud and LiDAR-frame boxes.

Each region is six plane equations, prepared here with the same numpy operations, in the same dtypes, as the
reference so that the coefficients are identical (float64 for every plane set of the real pipeline, where
``camera_to_lidar``'s ``np.ones`` promotes them; float32 for float32 boxes handed to ``crop_points``).  That is
microseconds of host work per frame; the O(P x n) membership test and the stable compaction run in
libmmmot_sm90a.so (csrc/lidar_crop.cu), many frames per call.  There is no CPU path for the membership test.
"""
import ctypes

import numpy as np
import torch

from . import _lib

# corner order of a unit box (x0y0z0, x0y0z1, x0y1z1, x0y1z0, x1y0z0, x1y0z1, x1y1z1, x1y1z0) and the six faces
# listed so that their normals (cross of consecutive edges) point inward (box_np_ops.py:161-178, 702-720)
_CORNER_ORDER = [0, 1, 3, 2, 4, 5, 7, 6]
_FACES = [[0, 1, 2, 3], [7, 6, 5, 4], [0, 3, 7, 4], [1, 5, 6, 2], [0, 4, 5, 1], [3, 2, 6, 7]]


def box_camera_to_lidar(boxes_cam, r_rect, velo2cam):
    """[x, y, z, l, h, w, ry] camera frame -> [x, y, z, w, l, h, ry] LiDAR frame
    (reference box_np_ops.py:584-589, 613-618)."""
    xyz = boxes_cam[:, 0:3]
    l, h, w = boxes_cam[:, 3:4], boxes_cam[:, 4:5], boxes_cam[:, 5:6]
    r = boxes_cam[:, 6:7]
    return np.concatenate([camera_to_lidar(xyz, r_rect, velo2cam), w, l, h, r], axis=1)


def camera_to_lidar(xyz, r_rect, velo2cam):
    """[..., 3] camera frame -> LiDAR frame, float64: the homogeneous ``np.ones`` column promotes
    (reference box_np_ops.py:584-589)."""
    hom = np.concatenate([xyz, np.ones(list(xyz.shape[:-1]) + [1])], axis=-1)
    return (hom @ np.linalg.inv((r_rect @ velo2cam).T))[..., :3]


def surface_planes(surf):
    """[n][6][4][3] faces (corners ordered so that the normals point inward) -> [n][6][4] plane equations
    (nx, ny, nz, d) in the faces' dtype; geometry.py:84-93 (``surface_equ_3d``)."""
    vec = surf[:, :, :2, :] - surf[:, :, 1:3, :]
    normal = np.cross(vec[:, :, 0, :], vec[:, :, 1, :])
    d = -np.einsum('aij, aij->ai', normal, surf[:, :, 0, :])
    return np.concatenate([normal, d[..., None]], axis=-1)


def box_planes(boxes_lidar):
    """[n][7] LiDAR-frame boxes (x, y, z, w, l, h, yaw; origin (0.5, 0.5, 0), rotation about z) ->
    [n][6][4] inward plane equations (nx, ny, nz, d) in the boxes' dtype (float32 or float64).  Same numpy
    operations, in the same order, as reference box_np_ops.py:147-178 (corners), :236-254 (rotation), :312-337,
    :702-720 (faces) and geometry.py:84-93 (plane equations), so the results are identical."""
    rb = np.asarray(boxes_lidar)
    centers, dims, angles = rb[:, :3], rb[:, 3:6], rb[:, 6]
    unit = np.stack(np.unravel_index(np.arange(8), [2] * 3), axis=1).astype(dims.dtype)[_CORNER_ORDER]
    unit = unit - np.array([0.5, 0.5, 0], dtype=dims.dtype)
    corners = dims.reshape([-1, 1, 3]) * unit.reshape([1, 8, 3])
    rot_sin, rot_cos = np.sin(angles), np.cos(angles)
    ones, zeros = np.ones_like(rot_cos), np.zeros_like(rot_cos)
    rot_t = np.stack([[rot_cos, -rot_sin, zeros], [rot_sin, rot_cos, zeros], [zeros, zeros, ones]])
    corners = np.einsum('aij,jka->aik', corners, rot_t)
    corners += centers.reshape([-1, 1, 3])
    surf = np.array([[corners[:, i] for i in f] for f in _FACES]).transpose([2, 0, 1, 3])   # [n][6][4][3]
    return surface_planes(surf).astype(rb.dtype if rb.dtype == np.float64 else np.float32)


def crop_points(points, boxes_lidar, without_reflectivity=True):
    """points: CUDA float32 [P][C>=3] scene cloud; boxes_lidar: [n][7] (numpy / CPU tensor, LiDAR frame).
    Returns (points_out CUDA [P_out][3 or C], points_split CPU int64 [n+1]) — the layout of
    ``det_info['points'][0]`` / ``det_info['points_split'][0]``."""
    lib = _lib.load()
    if points.device.type != "cuda":
        raise _lib.MmmotError("mmmot_b200.crop_points runs on CUDA only (no CPU fallback)")
    points = points.contiguous().float()
    P, C = points.shape
    boxes = np.asarray(boxes_lidar)
    f64 = boxes.dtype == np.float64         # the reference evaluates the predicate in the boxes' precision
    boxes = boxes.astype(np.float64 if f64 else np.float32).reshape(-1, 7)
    n = boxes.shape[0]
    dev = points.device
    with torch.cuda.device(dev):            # the library works on the CURRENT device
        planes = torch.from_numpy(np.ascontiguousarray(box_planes(boxes))).to(dev)
        ws = torch.empty(int(lib.mmmot_crop_workspace(P, n)), dtype=torch.uint8, device=dev)
        split = torch.empty(n + 1, dtype=torch.int32, device=dev)
        vp = lambda t: ctypes.c_void_p(t.data_ptr())
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.mmmot_crop_count(vp(points), P, C, vp(planes), int(f64), n, vp(split), vp(ws), ws.numel(), st), "mmmot_crop_count")
        split_h = split.cpu()                      # output size is data dependent: one sync, like the reference's host loop
        out_c = 3 if without_reflectivity else min(C, 4)
        out = torch.empty(int(split_h[-1]), out_c, device=dev)
        _lib.check(lib.mmmot_crop_scatter(vp(points), P, C, vp(planes), int(f64), n, vp(split), out_c, vp(out), vp(ws), ws.numel(), st),
                   "mmmot_crop_scatter")
    return out, split_h.long()


# ---- per-frame preparation: field-of-view cull + 3-D boxes or 2-D frustums (preprocess.py:45-106) ----

_FACE_IDX = np.array(_FACES)        # corner_to_surfaces_3d's face order (box_np_ops.py:724-743)
NEAR_CLIP, FAR_CLIP = 0.001, 100    # the reference's frustum depth range (box_np_ops.py:456)


def calib_f32(info):
    """(R0_rect, Tr_velo_to_cam, P2) cast to float32 as preprocess.py:59-61 does."""
    return (info['calib/R0_rect'].astype(np.float32), info['calib/Tr_velo_to_cam'].astype(np.float32),
            info['calib/P2'].astype(np.float32))


def projection_to_crt(p2):
    """P2 = C @ [R | T] with C upper triangular: inverse, QR, inverse (box_np_ops.py:442-453)."""
    rinv, cinv = np.linalg.qr(np.linalg.inv(p2[0:3, 0:3]))
    return np.linalg.inv(cinv), np.linalg.inv(rinv), cinv @ p2[0:3, 3]


def _frustum_corners(box_corners, c):
    """[..., 4, 2] image-plane corners -> [..., 8, 3] camera-frame frustum corners (near face then far face),
    box_np_ops.py:456-493; the corners' dtype carries through ``box_corners - u0v0``."""
    fku, fkv, u0v0 = c[0, 0], -c[1, 1], c[0:2, 2]
    z = np.array([NEAR_CLIP] * 4 + [FAR_CLIP] * 4, dtype=c.dtype)[:, np.newaxis]
    near = (box_corners - u0v0) / np.array([fku / NEAR_CLIP, -fkv / NEAR_CLIP], dtype=c.dtype)
    far = (box_corners - u0v0) / np.array([fku / FAR_CLIP, -fkv / FAR_CLIP], dtype=c.dtype)
    xy = np.concatenate([near, far], axis=-2)
    return np.concatenate([xy, np.broadcast_to(z, xy.shape[:-1] + (1,))], axis=-1)


def fov_planes(info, img_shape):
    """[6][4] float64 planes of camera 2's image frustum in the LiDAR frame (remove_outside_points,
    box_np_ops.py:629-636): the corners stay float32 until camera_to_lidar."""
    rect, trv2c, p2 = calib_f32(info)
    c, r, t = projection_to_crt(p2)
    h, w = img_shape[0], img_shape[1]
    frustum = _frustum_corners(np.array([[0, 0], [0, h], [w, h], [w, 0]], dtype=c.dtype), c)
    frustum -= t
    frustum = np.linalg.inv(r) @ frustum.T
    frustum = camera_to_lidar(frustum.T, rect, trv2c)
    return surface_planes(frustum[np.newaxis][:, _FACE_IDX])[0]


def frustum_planes(bboxes, info):
    """[n][4] image boxes (x1, y1, x2, y2; float32 or float64) -> [n][6][4] float64 planes of their view frustums
    in the LiDAR frame (get_frustum_points, box_np_ops.py:643-649)."""
    rect, trv2c, p2 = calib_f32(info)
    c, r, t = projection_to_crt(p2)
    corners = bboxes[..., [0, 1, 0, 3, 2, 3, 2, 1]].reshape(-1, 4, 2)    # minmax_to_corner_2d_v2
    frustums = _frustum_corners(corners, c)
    frustums -= t
    frustums = np.einsum('ij, akj->aki', np.linalg.inv(r), frustums)
    frustums = camera_to_lidar(frustums, rect, trv2c)
    return surface_planes(frustums[:, _FACE_IDX])


def detection_planes(info, dets, use_frustum=False, det_type='3D', shift_bbox=None):
    """[n][6][4] float64 planes of each detection's region: its 3-D box (preprocess.py:66-77) when
    ``det_type == '3D'`` and not ``use_frustum``, else the frustum of its 2-D box (preprocess.py:85-87)."""
    if det_type == '3D' and not use_frustum:
        rect, trv2c, _ = calib_f32(info)
        boxes = np.concatenate([dets['location'], dets['dimensions'], dets['rotation_y'][..., np.newaxis]],
                               axis=1).astype(np.float32)
        return box_planes(box_camera_to_lidar(boxes, rect, trv2c))
    bboxes = np.asarray(shift_bbox if shift_bbox is not None else dets['bbox'])
    return frustum_planes(bboxes, info)


def prep_points_batch(frames, use_frustum=False, num_point_features=4, without_reflectivity=False, det_type='3D'):
    """frames: list of (points, info, dets, shift_bbox) — points a CUDA float32 [P_f][num_point_features] raw scan,
    info the frame's KITTI info (``calib/P2``, ``calib/R0_rect``, ``calib/Tr_velo_to_cam``, ``img_shape``), dets its
    detections, shift_bbox None or [n_f][4] image boxes replacing ``dets['bbox']``.
    Returns (points CUDA float32 [P_out][3 or C], points_split CPU int64 [1 + sum n_f]): every frame's
    ``read_and_prep_points`` result concatenated in frame order with global offsets — ``det_info['points']`` /
    ``['points_split']`` before ``align_points``.  One launch sequence and one host sync for all frames."""
    lib = _lib.load()
    if not frames:
        raise ValueError("prep_points_batch: no frames")
    pts, fov, dets_pl, det_frame, offs = [], [], [], [], [0]
    for f, (points, info, dets, shift_bbox) in enumerate(frames):
        if points.device.type != "cuda":
            raise _lib.MmmotError("mmmot_b200.prep_points runs on CUDA only (no CPU fallback)")
        if points.dim() != 2 or points.shape[1] != num_point_features or num_point_features not in (3, 4):
            raise ValueError(f"frame {f}: points must be [P][num_point_features] with 3 or 4 features, "
                             f"got {tuple(points.shape)}")
        pl = detection_planes(info, dets, use_frustum, det_type, shift_bbox)
        if pl.shape[0] == 0:
            raise ValueError(f"frame {f} has no detections (the reference fails on it too)")
        pts.append(points)
        fov.append(fov_planes(info, info['img_shape']))
        dets_pl.append(pl)
        det_frame += [f] * pl.shape[0]
        offs.append(offs[-1] + points.shape[0])
    if offs[-1] >= 2 ** 31:
        raise ValueError("prep_points_batch: more than 2^31 - 1 points in one call")
    dev = pts[0].device
    points = torch.cat([p.to(dev).float() for p in pts]).contiguous() if len(pts) > 1 else pts[0].contiguous().float()
    C, F, D = num_point_features, len(frames), len(det_frame)
    out_c = 3 if without_reflectivity else C
    offs_h = (ctypes.c_int * (F + 1))(*offs)
    det_frame_h = (ctypes.c_int * D)(*det_frame)
    max_p = max(offs[i + 1] - offs[i] for i in range(F))
    if max_p == 0:      # nothing to crop: every detection is one zero point (the kernels need points)
        return torch.zeros(D, out_c, device=dev), torch.arange(D + 1, dtype=torch.int64)
    with torch.cuda.device(dev):            # the library works on the CURRENT device
        planes = np.ascontiguousarray(np.concatenate([np.stack(fov)] + dets_pl), dtype=np.float64)
        planes = torch.from_numpy(planes).to(dev)              # [F + D][6][4]: fields of view, then detections
        fov_d, det_d = planes[:F], planes[F:]
        ws = torch.empty(int(lib.mmmot_prep_workspace(max_p, F, D)), dtype=torch.uint8, device=dev)
        split = torch.empty(D + 1, dtype=torch.int32, device=dev)
        vp = lambda t: ctypes.c_void_p(t.data_ptr())
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.mmmot_prep_count(vp(points), offs_h, F, C, vp(fov_d), vp(det_d), det_frame_h, D, vp(split),
                                        vp(ws), ws.numel(), st), "mmmot_prep_count")
        split_h = split.cpu()                      # output size is data dependent: the call's one host sync
        out = torch.empty(int(split_h[-1]), out_c, device=dev)
        _lib.check(lib.mmmot_prep_scatter(vp(points), offs_h, F, C, vp(fov_d), vp(det_d), det_frame_h, D, vp(split),
                                          out_c, vp(out), vp(ws), ws.numel(), st), "mmmot_prep_scatter")
    return out, split_h.long()


def prep_points(points, info, dets, use_frustum=False, num_point_features=4, without_reflectivity=False,
                det_type='3D', shift_bbox=None):
    """``read_and_prep_points`` (preprocess.py:45-106) on a scan already in memory: points CUDA float32
    [P][num_point_features]; returns (points CUDA float32 [P_out][3 or C], points_split CPU int64 [n+1]),
    the layout of ``crop_points``.  ``prep_points_batch`` with one frame."""
    return prep_points_batch([(points, info, dets, shift_bbox)], use_frustum=use_frustum,
                             num_point_features=num_point_features, without_reflectivity=without_reflectivity,
                             det_type=det_type)
