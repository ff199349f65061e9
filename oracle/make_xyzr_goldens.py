"""ORACLE fixture generator for nets on xyz + reflectance points (reference ``without_reflectivity: False``) — needs a
checkout of the reference:

    MMMOT_REFERENCE=<path to ZwwWayne/mmMOT> python -m oracle.make_xyzr_goldens

Runs the UNMODIFIED reference ``modules.TrackingNet(without_reflectivity=False)`` (PointNet on 4 input channels,
modules/tracking_net.py:41, modules/point_net.py:93-100) on seeded 4-channel frame-pairs
(``synthetic_pair(..., reflectance=True)``) with seeded 4-channel weights (``synthetic_state_dict(..., point_in=4)``),
in eval mode and, for the rrc config, in training mode with its loss, exactly as oracle/make_goldens.py does for xyz
nets.  Writes tests/golden/xyzr/: a subdirectory, because the xyz parity tests glob tests/golden/*.pt.  Also stores the
reference's own state_dict key -> shape list of the 4-channel net.
"""
import contextlib
import io
import json
import os
import sys
import types

import torch

from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from oracle import ref_loader
from oracle.make_goldens import LOSS_KW, synthetic_gt

# (name, fusion, affinity_op, softmax_mode, neg_threshold, N, M, pts, hw, ragged, seed): the layout of make_goldens.CASES
CASES = [
    ("xyzr_subabs_dualadd_C_n8", "C", "minus_abs", "dual_add", 0.2, 8, 8, 32, 32, True, 41),
    ("xyzr_mul_A_n6", "A", "multiply", "none", 0.2, 6, 6, 24, 32, False, 42),
    ("xyzr_subabs_dualadd_C_n5x9", "C", "minus_abs", "dual_add", 0.0, 5, 9, 20, 32, True, 43),
]
# training mode, experiments/rrc_pfv_40e_subabs_dualadd_C/config.yaml:32-33 (dropblock 5, use_dropout True):
# (name, fusion, affinity_op, softmax_mode, N, M, pts, hw, ragged, seed), the layout of make_goldens.TRAIN_CASES
TRAIN_CASES = [("train_xyzr_drop_subabs_dualadd_C_n7x5", "C", "minus_abs", "dual_add", 7, 5, 40, 64, True, 44)]
TRAIN_DROP = dict(dropblock=5, use_dropout=True)

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "xyzr")


def _net(fusion, op, sm, thr, **kw):
    return ref_loader.load_tracking_net(
        seq_len=2, score_arch="branch_cls", appear_arch="vgg", appear_len=512, appear_skippool=True, appear_fpn=False,
        point_arch="v1", point_len=512, without_reflectivity=False, softmax_mode=sm, affinity_op=op, end_arch="v2",
        end_mode="avg", test_mode=2, score_fusion_arch=fusion, neg_threshold=thr, **kw)


def eval_goldens():
    for case in CASES:
        name, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = case
        net = _net(fusion, op, sm, thr, dropblock=0, use_dropout=False)
        net.load_state_dict(synthetic_state_dict(fusion, seed=seed, point_in=4), strict=True)
        dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged, reflectance=True)
        with torch.no_grad():
            feats, _ = net.feature(dets, info)
            det, link, new, end, trans = net(dets, info, split)
        out = {"det": det, "link": link[0], "new": new, "end": end, "trans1": trans[0], "trans2": trans[1], "feats": feats}
        out = {k: v.clone().contiguous() for k, v in out.items()}
        out["case"] = case
        torch.save(out, os.path.join(OUT, name + ".pt"))
        print(name, {k: tuple(v.shape) for k, v in out.items() if hasattr(v, "shape")})


def train_goldens():
    """As make_goldens.train_goldens (same shims), on the 4-channel net."""
    sys.path.insert(0, ref_loader.REF)
    sys.modules.setdefault("pyproj", types.ModuleType("pyproj"))
    if "solvers" not in sys.modules:
        sys.modules["solvers"] = types.SimpleNamespace(ortools_solve=None)
    with contextlib.redirect_stdout(io.StringIO()):
        import tracking_model as ref_tm
        from cost import TrackingLoss
    for case in TRAIN_CASES:
        name, fusion, op, sm, n, m, pts, hw, ragged, seed = case
        net = _net(fusion, op, sm, 0.2, **TRAIN_DROP)
        net.load_state_dict(synthetic_state_dict(fusion, seed=seed, point_in=4), strict=True)
        net.train()
        dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged, reflectance=True)
        torch.manual_seed(seed)              # the DropBlock / Dropout draws (CPU generator) start from here
        with torch.no_grad():
            det, link, new, end, trans = net(dets, info, split)
        after = {k: v.clone() for k, v in net.state_dict().items() if "running_" in k or "num_batches" in k}
        cls, ids = synthetic_gt(n, m, seed)
        with contextlib.redirect_stdout(io.StringIO()):
            tm = ref_tm.TrackingModule(net, None, TrackingLoss(**LOSS_KW))
        gt_det, gt_link, gt_new, gt_end = tm.generate_gt(det[0], cls, ids, split)
        orig_eq = torch.Tensor.eq
        torch.Tensor.eq = lambda a, b: orig_eq(a, b).to(torch.uint8)
        try:
            with torch.no_grad():
                loss = tm.criterion(split, gt_det, gt_link, gt_new, gt_end, det, link, new, end, trans)
        finally:
            torch.Tensor.eq = orig_eq
        out = {"case": case, "det": det, "link": link[0], "new": new, "end": end, "trans1": trans[0], "trans2": trans[1],
               "running": after, "gt_det": gt_det, "gt_link": gt_link[0], "gt_new": gt_new, "gt_end": gt_end,
               "loss": loss.detach().clone(), "drop": dict(TRAIN_DROP)}
        torch.save(out, os.path.join(OUT, name + ".pt"))
        print(name, float(loss), tuple(det.shape), tuple(trans[0].shape))


def schema_golden():
    """The reference's own key -> shape list of the 4-channel Fusion C net, in registration order."""
    net = _net("C", "minus_abs", "dual_add", 0.2, dropblock=0, use_dropout=False)
    keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(os.path.join(OUT, "schema_C.json"), "w") as f:
        json.dump(keys, f)
    print("schema_C", len(keys))


def main():
    os.makedirs(OUT, exist_ok=True)
    schema_golden()
    train_goldens()
    eval_goldens()


if __name__ == "__main__":
    main()
