"""Deterministic synthetic weights and frame-pair inputs (SURVEY.md §8d).

No checkpoints, detections or KITTI frames exist offline, so parity and throughput are both
measured on seeded synthetic data.  Everything here is CPU ``torch.Generator`` driven, hence
identical on any machine and inside the golden-fixture script.
"""
import math

import torch

from .schema import state_schema


def synthetic_state_dict(fusion="C", seed=0, point_in=3):
    """A non-degenerate ``state_dict`` for ``TrackingNet`` with the reference's key names; point_in = 4 for a net on
    xyz + reflectance points (``without_reflectivity=False``).

    Default inits make every GroupNorm the identity affine and both STN output layers zero
    (reference: modules/point_net.py:69-70), which hides bugs; so norm affines, BN running
    statistics and the STN output layers are all randomised."""
    g = torch.Generator().manual_seed(1000 + seed)
    sd = {}
    for key, (shape, kind) in state_schema(fusion, point_in).items():
        if kind == "conv":
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_in)
        elif kind == "bias":
            t = torch.rand(shape, generator=g) * 0.2 - 0.1
        elif kind == "norm_w":
            t = torch.rand(shape, generator=g) + 0.5
        elif kind == "norm_b":
            t = torch.rand(shape, generator=g) * 0.4 - 0.2
        elif kind == "run_mean":
            t = torch.randn(shape, generator=g) * 0.1
        elif kind == "run_var":
            t = torch.rand(shape, generator=g) + 0.5
        elif kind == "nbt":
            t = torch.zeros(shape, dtype=torch.int64)
        elif kind == "eye":
            t = torch.eye(shape[0])
        elif kind == "stn_out":
            t = torch.randn(shape, generator=g) * 0.01
        else:
            raise AssertionError(kind)
        sd[key] = t
    return sd


def structured_crops(noise, gen):
    """Image crops are mean/std-normalised pixels (reference utils/build_util.py:111-112), i.e.
    ~N(0,1) per pixel, but different detections show different objects.  Pure white noise makes
    every crop's pooled VGG feature nearly identical, so the fusion GroupNorm (per channel over the
    L detections) divides by a ~zero spread and amplifies fp32 round-off ~20-100x for ANY
    implementation.  Give each detection its own contrast, brightness and low-frequency content,
    like real crops have (|mean|/std of the pre-norm fusion channels drops from ~18 to ~4)."""
    L, hw = noise.shape[0], noise.shape[-1]
    lf = torch.nn.functional.interpolate(torch.randn(L, 3, 4, 4, generator=gen), size=hw, mode="bilinear",
                                         align_corners=False)
    contrast = torch.rand(L, 1, 1, 1, generator=gen) + 0.25
    bright = torch.randn(L, 3, 1, 1, generator=gen) * 0.5
    return noise * contrast + 1.5 * lf + bright


def synthetic_pair(n, m=None, pts=128, hw=64, seed=0, ragged=False, reflectance=False):
    """One frame-pair in the exact layout ``TestSequence.__getitem__`` + the DataLoader hand to
    ``TrackingNet.forward`` (reference: dataset/test_seq_dataset.py:227-246, eval_seq.py:144-153):

    dets ``L x 3 x H x W``; det_info['points'] ``1 x P_t x 3`` (``1 x P_t x 4`` with reflectance);
    det_info['points_split'] ``1 x (L+1)`` **float**; dets_split = list of shape-(1,) int tensors.

    reflectance: a fourth column in [0, 1], a per-detection base (surfaces differ between objects) plus per-point
    noise, drawn after every other value so the xyz outputs of a seed are the same with or without it.  A column
    without detection-level structure would be a degenerate GroupNorm input (see ``structured_crops``).
    """
    m = n if m is None else m
    L = n + m
    g = torch.Generator().manual_seed(1234 + seed)
    dets = structured_crops(torch.randn(L, 3, hw, hw, generator=g), g)
    if ragged:
        cnt = torch.randint(1, 2 * pts, (L,), generator=g)
    else:
        cnt = torch.full((L,), pts, dtype=torch.int64)
    split = torch.zeros(L + 1, dtype=torch.int64)
    split[1:] = torch.cumsum(cnt, 0)
    pt = int(split[-1])
    centre = torch.rand(L, 3, generator=g) * torch.tensor([60.0, 40.0, 2.0]) + torch.tensor(
        [0.0, -20.0, -2.0])
    which = torch.repeat_interleave(torch.arange(L), cnt)
    points = torch.randn(pt, 3, generator=g) * torch.tensor([2.0, 1.0, 0.8]) + centre[which]
    if reflectance:
        base = torch.rand(L, generator=g) * 0.8 + 0.1
        refl = (base[which] + torch.randn(pt, generator=g) * 0.05).clamp(0.0, 1.0)
        points = torch.cat([points, refl[:, None]], 1)
    det_info = {
        "points": points.unsqueeze(0).contiguous(),
        "points_split": split.float().unsqueeze(0),
    }
    dets_split = [torch.tensor([n]), torch.tensor([m])]
    return dets, det_info, dets_split


def synthetic_batch(b, n, pts=128, hw=64, seed=0, reflectance=False):
    """``b`` frame-pairs with equal ``n`` detections per frame, packed for ``forward_batch``:
    dets ``(b*2n) x 3 x H x W``, points ``P_total x 3`` (``x 4`` with reflectance), points_split ``(b*2n+1,)``
    int64."""
    ds, ps, sp = [], [], [torch.zeros(1, dtype=torch.int64)]
    off = 0
    for p in range(b):
        d, info, _ = synthetic_pair(n, n, pts, hw, seed=seed + p, reflectance=reflectance)
        ds.append(d)
        ps.append(info["points"][0])
        s = info["points_split"][0].long()
        sp.append(s[1:] + off)
        off += int(s[-1])
    return torch.cat(ds), torch.cat(ps), torch.cat(sp)
