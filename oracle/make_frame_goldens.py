"""ORACLE fixture generator for samples of more than two frames — needs a checkout of the reference:

    MMMOT_REFERENCE=<path to ZwwWayne/mmMOT> python -m oracle.make_frame_goldens

Runs the UNMODIFIED reference ``modules.TrackingNet`` (imported in place, as oracle/make_goldens.py does) in eval mode on
seeded synthetic samples of K = 3 and 4 frames: one feature pass over the sample's L detections, then ``associate`` on
every pair of consecutive frames (modules/tracking_net.py:165-193).  The L crops and point clouds come from
``synthetic_pair(n_0, L - n_0)``; ``dets_split`` holds the K frame counts.  Writes tests/golden/frames/, a subdirectory,
because the two-frame parity tests glob tests/golden/*.pt.
"""
import os

import torch

from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from oracle import ref_loader

# (name, fusion, affinity_op, softmax_mode, neg_threshold, counts, pts, hw, ragged, seed)
CASES = [
    ("k3_subabs_dualadd_C_n4x7x3", "C", "minus_abs", "dual_add", 0.2, (4, 7, 3), 24, 32, True, 71),
    ("k4_mul_A_n5x3x6x4", "A", "multiply", "none", 0.2, (5, 3, 6, 4), 20, 32, True, 72),
]

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "frames")


def sample(case):
    """The case's sample in the reference's forward layout: (dets, det_info, dets_split)."""
    name, fusion, op, sm, thr, counts, pts, hw, ragged, seed = case
    dets, info, _ = synthetic_pair(counts[0], sum(counts) - counts[0], pts, hw, seed=seed, ragged=ragged)
    return dets, info, [torch.tensor([k]) for k in counts]


def reference_forward(case):
    name, fusion, op, sm, thr, counts, pts, hw, ragged, seed = case
    net = ref_loader.load_tracking_net(
        seq_len=len(counts), score_arch="branch_cls", appear_arch="vgg", appear_len=512, appear_skippool=True,
        appear_fpn=False, point_arch="v1", point_len=512, without_reflectivity=True, softmax_mode=sm, affinity_op=op,
        end_arch="v2", end_mode="avg", test_mode=2, score_fusion_arch=fusion, neg_threshold=thr, dropblock=0,
        use_dropout=False)
    net.load_state_dict(synthetic_state_dict(fusion, seed=seed), strict=True)
    dets, info, split = sample(case)
    with torch.no_grad():
        det, links, new, end, trans = net(dets, info, split)
    return {"det": det, "links": [l.clone().contiguous() for l in links], "new": new, "end": end,
            "trans1": trans[0], "trans2": trans[1]}


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for case in CASES:
        out = reference_forward(case)
        out = {k: v if isinstance(v, list) else v.clone().contiguous() for k, v in out.items()}
        out["case"] = case
        torch.save(out, os.path.join(OUT, case[0] + ".pt"))
        print(case[0], tuple(out["det"].shape), [tuple(l.shape) for l in out["links"]], tuple(out["new"].shape))


if __name__ == "__main__":
    main()
