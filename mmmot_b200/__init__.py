"""mmmot_b200 — CUDA-native (sm_90a, H100) implementation of mmMOT's per-frame-pair association
forward behind the reference's own Python surface.  See DESIGN.md."""
from .config import build_model, model_kwargs  # noqa: F401
from .solvers import ortools_solve, solve_batch, solve_frames  # noqa: F401
from .tracking_net import TrackingNet  # noqa: F401
from .lidar_crop import box_camera_to_lidar, box_planes, crop_points, prep_points, prep_points_batch  # noqa: F401
from .image_crop import crop_boxes, crop_resize  # noqa: F401
from .tracking_model import TrackingModule, kitti_result_line, write_kitti_result  # noqa: F401
from .cost import DetLoss, LinkLoss, TrackingLoss  # noqa: F401
from .pipeline import HostPipeline  # noqa: F401


def set_engine(engine):
    """Contraction engine: "auto" (default), "fp32" (FFMA engine) or "tcgen05" (the tensor-core engine; on sm_90a
    it issues wgmma — the name is kept for callers)."""
    from . import _lib
    code = {"auto": 0, "fp32": 1, "tcgen05": 2}[engine]
    _lib.check(_lib.load().mmmot_set_engine(code), "mmmot_set_engine")
