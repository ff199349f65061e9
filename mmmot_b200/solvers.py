"""Association solver with the reference's ``ortools_solve`` signature.

Mirrors reference solvers.py:9-138: same arguments (``link_score`` is a list holding one ``1 x n_i x n_{i+1}``
tensor per pair of consecutive frames, ``det_split`` a list of ints / 1-element tensors), same outputs — four fp32
0/1 tensors ``(assign_det (L,), [assign_link 1 x n_i x n_{i+1}, ...], assign_new (L,), assign_end (L,))`` on the
input device — so reference tracking_model.py:72-81 (``predict`` -> ``assign_det_id``) works on them unchanged.
The programme is solved exactly on the GPU: two-frame samples by ``mmmot_lp_assign`` (csrc/lp_assign.cu, an
assignment problem), samples of more frames by ``mmmot_flow_assign`` (csrc/flow_assign.cu, a min-cost flow).
There is no CPU solver in the product.
"""
import ctypes

import torch

from . import _lib


def solve_batch(det, link, new, end, n, m):
    """det B x L, link B x n x m, new/end B x L (zero-padded as the forward returns them); CUDA,
    arbitrary strides between pairs (views into the forward outputs are fine).  Returns a dict of
    assign_det/new/end (B x L), assign_link (B x n x m), match (B x n int32, -1 = no link)."""
    lib = _lib.load()
    if det.device.type != "cuda":
        raise _lib.MmmotError("mmmot_b200 solver runs on CUDA only (no CPU fallback)")
    B, L = det.shape[0], n + m

    def rowview(t, inner):
        # one pair's data must be contiguous; the stride between pairs is free
        if t.dtype != torch.float32 or t[0].numel() != inner or not t[0].is_contiguous():
            t = t.float().contiguous()
        return t, (t.stride(0) if B > 1 else inner)
    det, sd = rowview(det, L)
    link, sl = rowview(link, n * m)
    new, sn = rowview(new, L)
    end, se = rowview(end, L)
    dev = det.device
    a_det = torch.empty(B, L, device=dev)
    a_new = torch.empty(B, L, device=dev)
    a_end = torch.empty(B, L, device=dev)
    a_link = torch.empty(B, n, m, device=dev)
    match = torch.empty(B, n, dtype=torch.int32, device=dev)
    ws = torch.empty(int(lib.mmmot_lp_workspace(B, n, m)), dtype=torch.uint8, device=dev)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    with torch.cuda.device(dev):            # the library works on the CURRENT device
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.mmmot_lp_assign(vp(det), sd, vp(link), sl, vp(new), sn, vp(end), se, B, n, m,
                                       vp(a_det), vp(a_link), vp(a_new), vp(a_end), vp(match),
                                       vp(ws), ws.numel(), st), "mmmot_lp_assign")
    return {"assign_det": a_det, "assign_link": a_link, "assign_new": a_new, "assign_end": a_end,
            "match": match}


def solve_frames(det, links, new, end, counts):
    """Samples of K >= 2 frames sharing the detection counts ``counts`` (K ints): det, new, end B x L (L = sum of
    counts, zero-padded as the forward returns them), links a list of K - 1 tensors B x n_i x n_{i+1}; CUDA,
    arbitrary strides between samples for det / new / end.  Returns a dict of assign_det/new/end (B x L),
    assign_link (a list of K - 1 tensors B x n_i x n_{i+1}) and match (B x (L - n_{K-1}) int32: each detection's
    successor in the next frame, -1 = none)."""
    lib = _lib.load()
    if det.device.type != "cuda":
        raise _lib.MmmotError("mmmot_b200 solver runs on CUDA only (no CPU fallback)")
    counts = [int(c) for c in counts]
    K, B, L = len(counts), det.shape[0], sum(counts)
    if len(links) != K - 1:
        raise ValueError(f"{K} frames need {K - 1} link matrices, got {len(links)}")

    def rowview(t):
        # one sample's data must be contiguous; the stride between samples is free
        if t.dtype != torch.float32 or t[0].numel() != L or not t[0].is_contiguous():
            t = t.float().contiguous()
        return t, (t.stride(0) if B > 1 else L)
    det, sd = rowview(det)
    new, sn = rowview(new)
    end, se = rowview(end)
    sizes = [a * b for a, b in zip(counts[:-1], counts[1:])]
    packed = torch.cat([l.reshape(B, s).float() for l, s in zip(links, sizes)], 1).contiguous()
    dev = det.device
    a_det = torch.empty(B, L, device=dev)
    a_new = torch.empty(B, L, device=dev)
    a_end = torch.empty(B, L, device=dev)
    a_links = torch.empty(B, sum(sizes), device=dev)
    match = torch.empty(B, L - counts[-1], dtype=torch.int32, device=dev)
    c_counts = (ctypes.c_int * K)(*counts)
    ws = torch.empty(int(lib.mmmot_flow_workspace(B, K, c_counts)), dtype=torch.uint8, device=dev)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    with torch.cuda.device(dev):            # the library works on the CURRENT device
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.mmmot_flow_assign(vp(det), sd, vp(packed), packed.shape[1], vp(new), sn, vp(end), se, B, K,
                                         c_counts, vp(a_det), vp(a_links), vp(a_new), vp(a_end), vp(match), vp(ws),
                                         ws.numel(), st), "mmmot_flow_assign")
    assign_link = [a.reshape(B, n, m) for a, n, m in zip(a_links.split(sizes, 1), counts[:-1], counts[1:])]
    return {"assign_det": a_det, "assign_link": assign_link, "assign_new": a_new, "assign_end": a_end, "match": match}


def ortools_solve(det_score, link_score, new_score, end_score, det_split, gt=None):
    """Drop-in for reference solvers.py:9, for samples of any number of frames.  The loss-augmented ``gt`` branch
    (:50-81) is never used on the predict path and is not implemented.  A ``link_score`` that does not hold one matrix
    per pair of consecutive frames raises ValueError (the reference fails with a KeyError)."""
    if gt is not None:
        raise NotImplementedError("loss-augmented solve (gt != None) is training-only; not implemented")
    if len(det_split) < 2 or len(link_score) != len(det_split) - 1:
        raise ValueError(f"{len(det_split)} frames need {len(det_split) - 1} link matrices, got {len(link_score)}")
    if len(det_split) == 2:
        n, m = int(det_split[0]), int(det_split[1])
        r = solve_batch(det_score.reshape(1, -1), link_score[0].reshape(1, n, m),
                        new_score.reshape(1, -1), end_score.reshape(1, -1), n, m)
        return r["assign_det"][0], [r["assign_link"]], r["assign_new"][0], r["assign_end"][0]
    counts = [int(s) for s in det_split]
    r = solve_frames(det_score.reshape(1, -1), [l.reshape(1, a, b) for l, a, b in zip(link_score, counts[:-1], counts[1:])],
                     new_score.reshape(1, -1), end_score.reshape(1, -1), counts)
    return r["assign_det"][0], r["assign_link"], r["assign_new"][0], r["assign_end"][0]
