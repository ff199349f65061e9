"""ORACLE fixture generator for nets with a ResNet appearance trunk and the FPN head (reference ``appear_arch: resnet50 |
resnet101 | resnet152`` with ``appear_skippool: False, appear_fpn: True``) — needs a checkout of the reference:

    MMMOT_REFERENCE=<path to ZwwWayne/mmMOT> python -m oracle.make_resnet_fpn_goldens

The recipe of oracle/make_resnet_goldens.py with the other head: the UNMODIFIED reference ``modules.TrackingNet`` is built
offline (``make_resnet_goldens.offline_torchvision``: hub downloads raise and are recorded, torchvision's builders get
``weights=None``), loaded strictly with ``synthetic_state_dict(..., appear_head="fpn")`` and run on the CPU in eval mode
on seeded frame-pairs.  Writes tests/golden/resnet_fpn/: each arch's state_dict key -> shape list (schema_<arch>.json)
and the eval fixtures of CASES, three at 64 x 64 and one at 224 x 224 (where the 784-, 196- and 49-pixel levels put
image boundaries inside the laterals' 32-column chunks).
"""
import json
import os

import torch

from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from oracle import make_resnet_goldens as mrg
from oracle import ref_loader

# (name, arch, fusion, affinity_op, softmax_mode, neg_threshold, N, M, pts, hw, ragged, seed): make_resnet_goldens.CASES
CASES = [
    ("fpn50_subabs_dualadd_C_n4x3", "resnet50", "C", "minus_abs", "dual_add", 0.2, 4, 3, 24, 64, True, 61),
    ("fpn101_mul_A_n3x5", "resnet101", "A", "multiply", "none", 0.2, 3, 5, 20, 64, True, 62),
    ("fpn152_dualmax_B_n5x4", "resnet152", "B", "minus_abs", "dual_max", 0.2, 5, 4, 16, 64, True, 63),
    ("fpn50_224_subabs_dualadd_C_n3x2", "resnet50", "C", "minus_abs", "dual_add", 0.2, 3, 2, 16, 224, True, 64),
]
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "resnet_fpn")


def reference_net(arch, fusion, op, sm, thr):
    """The reference TrackingNet with a ResNet trunk and the FPN head, eval mode, built offline."""
    mrg.offline_torchvision()
    return ref_loader.load_tracking_net(
        seq_len=2, score_arch="branch_cls", appear_arch=arch, appear_len=512, appear_skippool=False, appear_fpn=True,
        point_arch="v1", point_len=512, without_reflectivity=True, softmax_mode=sm, affinity_op=op, end_arch="v2",
        end_mode="avg", test_mode=2, score_fusion_arch=fusion, neg_threshold=thr, dropblock=0, use_dropout=False)


def schema_goldens():
    for arch in mrg.ARCHS:
        net = reference_net(arch, "C", "minus_abs", "dual_add", 0.2)
        keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
        with open(os.path.join(OUT, f"schema_{arch}.json"), "w") as f:
            json.dump(keys, f)
        print(f"schema_{arch}", len(keys))


def eval_goldens():
    for case in CASES:
        name, arch, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = case
        net = reference_net(arch, fusion, op, sm, thr)
        net.load_state_dict(synthetic_state_dict(fusion, seed=seed, appear_arch=arch, appear_head="fpn"), strict=True)
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
