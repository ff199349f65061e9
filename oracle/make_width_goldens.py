"""ORACLE fixture generator for the reference's narrower nets (``appear_len = point_len`` 256 or 128: ``vgg16_bn_256`` /
``vgg16_bn_128``, every PointNet, fusion, affinity and w_det width divided by 512 // width) — needs a checkout of the
reference:

    MMMOT_REFERENCE=<path to ZwwWayne/mmMOT> python -m oracle.make_width_goldens

The recipe of oracle/make_goldens.py and oracle/make_resnet_goldens.py at the other widths: the UNMODIFIED reference
``modules.TrackingNet`` is built (ResNet trunks offline through ``make_resnet_goldens.offline_torchvision``), loaded
strictly with ``synthetic_state_dict(..., width=...)`` and run on the CPU in eval mode on seeded frame-pairs.  Writes
tests/golden/width/: each width's state_dict key -> shape list (schema_<arch>_<head>_<width>.json, Fusion C) and the eval
fixtures of CASES.
"""
import json
import os

import torch

from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from oracle import make_resnet_goldens as mrg
from oracle import ref_loader

# (name, arch, head, width, fusion, affinity_op, softmax_mode, neg_threshold, N, M, pts, hw, ragged, seed)
CASES = [
    ("w256_subabs_dualadd_C_n5x3", "vgg", "skippool", 256, "C", "minus_abs", "dual_add", 0.2, 5, 3, 24, 64, True, 91),
    ("w256_mul_A_n4x6", "vgg", "skippool", 256, "A", "multiply", "none", 0.2, 4, 6, 20, 64, True, 92),
    ("w256_minus_B_n1x1", "vgg", "skippool", 256, "B", "minus", "dual_max", 0.2, 1, 1, 16, 64, True, 93),
    ("w128_subabs_single_C_n6x4", "vgg", "skippool", 128, "C", "minus_abs", "single", 0.2, 6, 4, 24, 64, True, 94),
    ("w128_minus_A_n3x5", "vgg", "skippool", 128, "A", "minus", "dual", 0.2, 3, 5, 20, 64, True, 95),
    ("w128_mul_B_n1x1", "vgg", "skippool", 128, "B", "multiply", "single", 0.2, 1, 1, 16, 64, True, 96),
    ("w256_res50_subabs_dualadd_C_n4x3", "resnet50", "skippool", 256, "C", "minus_abs", "dual_add", 0.2, 4, 3, 24, 64, True,
     97),
    ("w128_res50_minus_B_n3x4", "resnet50", "skippool", 128, "B", "minus", "dual_max", 0.2, 3, 4, 16, 64, True, 98),
    ("w256_fpn50_mul_A_n3x5", "resnet50", "fpn", 256, "A", "multiply", "none", 0.2, 3, 5, 20, 64, True, 99),
    ("w256_fpn50_224_subabs_dualadd_C_n3x2", "resnet50", "fpn", 256, "C", "minus_abs", "dual_add", 0.2, 3, 2, 16, 224, True,
     100),
]
SCHEMAS = [("vgg", "skippool", 256), ("vgg", "skippool", 128), ("resnet50", "skippool", 256), ("resnet50", "fpn", 256),
           ("resnet50", "skippool", 128), ("resnet50", "fpn", 128)]
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "width")


def reference_net(arch, head, width, fusion, op, sm, thr):
    """The reference TrackingNet at appear_len = point_len = width, eval mode (ResNet trunks built offline)."""
    if arch != "vgg":
        mrg.offline_torchvision()
    return ref_loader.load_tracking_net(
        seq_len=2, score_arch="branch_cls", appear_arch=arch, appear_len=width, appear_skippool=head == "skippool",
        appear_fpn=head == "fpn", point_arch="v1", point_len=width, without_reflectivity=True, softmax_mode=sm,
        affinity_op=op, end_arch="v2", end_mode="avg", test_mode=2, score_fusion_arch=fusion, neg_threshold=thr,
        dropblock=0, use_dropout=False)


def schema_goldens():
    for arch, head, width in SCHEMAS:
        net = reference_net(arch, head, width, "C", "minus_abs", "dual_add", 0.2)
        keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
        name = f"schema_{arch}_{head}_{width}"
        with open(os.path.join(OUT, name + ".json"), "w") as f:
            json.dump(keys, f)
        print(name, len(keys))


def eval_goldens():
    for case in CASES:
        name, arch, head, width, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = case
        net = reference_net(arch, head, width, fusion, op, sm, thr)
        net.load_state_dict(synthetic_state_dict(fusion, seed=seed, appear_arch=arch, appear_head=head, width=width),
                            strict=True)
        dets, info, split = synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged)
        with torch.no_grad():
            feats, _ = net.feature(dets, info)
            det, link, new, end, trans = net(dets, info, split)
        out = {"det": det, "link": link[0], "new": new, "end": end, "trans1": trans[0], "trans2": trans[1], "feats": feats}
        out = {k: v.clone().contiguous() for k, v in out.items()}
        out["case"] = case
        torch.save(out, os.path.join(OUT, name + ".pt"))
        print(name, {k: tuple(v.shape) for k, v in out.items() if hasattr(v, "shape")})


def main():
    os.makedirs(OUT, exist_ok=True)
    schema_goldens()
    eval_goldens()
    assert not mrg.BLOCKED, mrg.BLOCKED


if __name__ == "__main__":
    main()
