"""ORACLE fixture generator for nets with a ResNet appearance trunk (reference ``appear_arch: resnet50 | resnet101 |
resnet152`` with ``appear_skippool: True``) — needs a checkout of the reference:

    MMMOT_REFERENCE=<path to ZwwWayne/mmMOT> python -m oracle.make_resnet_goldens

Runs the UNMODIFIED reference ``modules.TrackingNet(appear_arch=resnetXX)`` (modules/appear_net.py:60-83,213-256) on the
CPU, in eval mode, on seeded frame-pairs (``synthetic_pair``, 64 x 64 crops) with seeded weights
(``synthetic_state_dict(..., appear_arch=...)``), as oracle/make_goldens.py does for VGG nets.  Writes
tests/golden/resnet/: each arch's state_dict key -> shape list (schema_<arch>.json) and one eval fixture per arch.

The reference builds its trunk with ``torchvision.models.resnetXX(pretrained=True)``, which in current torchvision
means ImageNet weights fetched from the network.  ``offline_torchvision()`` runs first: every hub download raises (and is
recorded in BLOCKED), and the three builders on ``torchvision.models`` are replaced by ones that pass ``weights=None``.
The synthetic state_dict then overwrites every parameter and buffer (strict load), so no pretrained value could matter
anyway.  ``reference_net`` is the one place that constructs the reference ResNet net.
"""
import json
import os

import torch

from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from oracle import ref_loader

ARCHS = ("resnet50", "resnet101", "resnet152")
# (name, arch, fusion, affinity_op, softmax_mode, neg_threshold, N, M, pts, hw, ragged, seed): the layout of
# make_goldens.CASES with the arch second
CASES = [
    ("res50_subabs_dualadd_C_n4x3", "resnet50", "C", "minus_abs", "dual_add", 0.2, 4, 3, 24, 64, True, 51),
    ("res101_mul_A_n3x5", "resnet101", "A", "multiply", "none", 0.2, 3, 5, 20, 64, True, 52),
    ("res152_dualmax_B_n5x4", "resnet152", "B", "minus_abs", "dual_max", 0.2, 5, 4, 16, 64, True, 53),
]
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "resnet")

BLOCKED = []      # (function, args) of every download attempt offline_torchvision refused


def offline_torchvision():
    """Make every torch.hub download raise, and torchvision.models.resnet50/101/152 ignore ``pretrained`` (build with
    weights=None).  Idempotent."""
    import torch.hub
    import torchvision.models
    import torchvision.models._api as tv_api

    def refuse(name):
        def f(*a, **k):
            BLOCKED.append((name, a))
            raise RuntimeError(f"{name}: network access refused while building the reference net offline")
        f.offline_guard = True
        return f
    for mod in (torch.hub, tv_api):
        for name in ("load_state_dict_from_url", "download_url_to_file"):
            if hasattr(mod, name) and not getattr(getattr(mod, name), "offline_guard", False):
                setattr(mod, name, refuse(f"{mod.__name__}.{name}"))
    for arch in ARCHS:
        fn = getattr(torchvision.models, arch)
        if getattr(fn, "offline_guard", False):
            continue

        def build(*a, _fn=fn, **k):
            k.pop("pretrained", None)
            k.pop("weights", None)
            return _fn(weights=None)
        build.offline_guard = True
        setattr(torchvision.models, arch, build)


def reference_net(arch, fusion, op, sm, thr):
    """The reference TrackingNet with a ResNet appearance trunk, eval mode, built offline."""
    offline_torchvision()
    return ref_loader.load_tracking_net(
        seq_len=2, score_arch="branch_cls", appear_arch=arch, appear_len=512, appear_skippool=True, appear_fpn=False,
        point_arch="v1", point_len=512, without_reflectivity=True, softmax_mode=sm, affinity_op=op, end_arch="v2",
        end_mode="avg", test_mode=2, score_fusion_arch=fusion, neg_threshold=thr, dropblock=0, use_dropout=False)


def schema_goldens():
    for arch in ARCHS:
        net = reference_net(arch, "C", "minus_abs", "dual_add", 0.2)
        keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
        with open(os.path.join(OUT, f"schema_{arch}.json"), "w") as f:
            json.dump(keys, f)
        print(f"schema_{arch}", len(keys))


def eval_goldens():
    for case in CASES:
        name, arch, fusion, op, sm, thr, n, m, pts, hw, ragged, seed = case
        net = reference_net(arch, fusion, op, sm, thr)
        net.load_state_dict(synthetic_state_dict(fusion, seed=seed, appear_arch=arch), strict=True)
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
    assert not BLOCKED, BLOCKED


if __name__ == "__main__":
    main()
