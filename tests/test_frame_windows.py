"""Batched windows of K > 2 frames: ``forward_batch`` / ``predict_batch`` / ``HostPipeline`` with ``counts``.

B samples share the per-frame detection counts (n_0, ..., n_{K-1}).  Each sample is its own GroupNorm domain and every
engine and tile choice depends on the per-sample (per-transition) shape only, so the oracle is exact: a loop of
``forward`` over the samples, bit for bit, and ``ortools_solve`` per sample on those outputs.  Against the unmodified
reference: the K = 3 and K = 4 goldens of oracle/make_frame_goldens.py, within the project's 1e-4 bound.

GPU: identity with the looped forward for K = 3, 4, 8 (1-detection frames, unequal neighbours, several chunks, ragged
points, every stack) on both engines, and on a 256-wide, a ResNet-50 SkipPool and an xyz + reflectance net; the reference
goldens; the assignments against ortools_solve; counts = (n, m) against (n, m); HostPipeline against predict_batch.
CPU: argument errors before any device work, the window's workspace, the chunk budget."""
import glob
import os

import pytest
import torch

from helpers import GOLDEN_DIR, TOL, det_close, relerr
import mmmot_b200
from mmmot_b200 import _lib
from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict

gpu = pytest.mark.gpu
FRAME_GOLDENS = sorted(glob.glob(os.path.join(GOLDEN_DIR, "frames", "*.pt")))


@pytest.fixture(params=["fp32", "tcgen05"])
def engine(request):
    mmmot_b200.set_engine(request.param)
    yield request.param
    mmmot_b200.set_engine("auto")


def _net(fusion="C", seed=3, op="minus_abs", sm="dual_add", sd=None, **kw):
    sd = synthetic_state_dict(fusion, seed=seed) if sd is None else sd
    kw = dict(dict(appear_skippool=True), **kw)
    net = mmmot_b200.TrackingNet(3, score_arch="branch_cls", score_fusion_arch=fusion, affinity_op=op, softmax_mode=sm,
                                 neg_threshold=0.2, test_mode=2, dropblock=0, **kw)
    net.load_state_dict(sd, strict=True)
    return net


def _samples(B, counts, pts=16, hw=32, seed=0, reflectance=False):
    """B K-frame samples: the list of (dets, det_info, dets_split) for ``forward`` and their packing for forward_batch
    (crops (B*L) x 3 x hw x hw, points, points_split (B*L + 1,) CPU int64)."""
    L = sum(counts)
    one, ds, ps, sp, off = [], [], [], [torch.zeros(1, dtype=torch.int64)], 0
    for b in range(B):
        d, info, _ = synthetic_pair(counts[0], L - counts[0], pts, hw, seed=seed + b, ragged=True, reflectance=reflectance)
        one.append((d, info, [torch.tensor([k]) for k in counts]))
        ds.append(d)
        ps.append(info["points"][0])
        s_ = info["points_split"][0].long()
        sp.append(s_[1:] + off)
        off += int(s_[-1])
    return one, (torch.cat(ds), torch.cat(ps), torch.cat(sp))


def _cuda(info):
    return {k: v.cuda() for k, v in info.items()}


def _assert_equals_loop(net, counts, one, o, stack=None):
    """o (forward_batch(counts=...)) == forward / forward_stack per sample, bit for bit; new / end compared after the
    zero padding forward applies."""
    n0, nl, L = counts[0], counts[-1], sum(counts)
    assert len(o["link"]) == len(counts) - 1
    for b, (d, info, ds) in enumerate(one):
        d, info = d.cuda(), _cuda(info)
        ref = net(d, info, ds) if stack is None else net.forward_stack(d, info, ds, stack)
        det, links, new, end, trans = ref
        assert torch.equal(o["det"][b], det), f"det, sample {b}"
        for k, (a, r) in enumerate(zip(o["link"], links)):
            assert torch.equal(a[b], r), f"link {k}, sample {b}"
        assert torch.equal(o["new"][b], new[:, n0:]) and not new[:, :n0].any(), f"new, sample {b}"
        assert torch.equal(o["end"][b], end[:, :L - nl]) and not end[:, L - nl:].any(), f"end, sample {b}"
        assert all(torch.equal(x, y) for x, y in zip(o["trans"], trans))


# ------------------------------------------------------------------------------------------------ GPU: looped forward
WINDOWS = [((4, 1, 6), 5), ((7, 3, 1, 5), 5), ((2, 5, 1, 3, 6, 4, 1, 2), 3)]


@gpu
@pytest.mark.parametrize("counts,B", WINDOWS, ids=["k3", "k4", "k8"])
@pytest.mark.parametrize("stack", [None, 0, 1, 2])
def test_windows_equal_looped_forward(counts, B, stack, engine):
    """forward_batch(counts=...) over B samples, cut into chunks of 2, == B calls of forward (forward_stack with a
    stack), bit for bit: det, every link, new / end, trans, and the features with keep_feats."""
    net = _net(seed=5).cuda().eval()
    one, (crops, pts, split) = _samples(B, counts, seed=10 * len(counts))
    L = sum(counts)
    net.chunk_pairs = 2
    o = net.forward_batch(None if stack == 1 else crops.cuda(), None if stack == 0 else pts.cuda(),
                          None if stack == 0 else split, counts=counts, stack=stack, keep_feats=True)
    net.chunk_pairs = None
    ns = 3 if stack is None else 1
    assert o["det"].shape == (B, ns, L) and o["new"].shape == (B, ns, L - counts[0]) and \
        o["end"].shape == (B, ns, L - counts[-1]) and int(o["status"]) == 0
    assert [tuple(x.shape) for x in o["link"]] == [(B, ns, a, b) for a, b in zip(counts[:-1], counts[1:])]
    _assert_equals_loop(net, counts, one, o, stack)
    # the features of an unchunked call are the chunked call's
    whole = net.forward_batch(crops.cuda(), pts.cuda(), split, counts=counts, keep_feats=True)
    assert torch.equal(whole["feats"] if stack is None else whole["feats"][:, stack:stack + 1], o["feats"])


@gpu
@pytest.mark.parametrize("kind", ["w256", "resnet50", "xyzr"])
def test_windows_equal_looped_forward_other_nets(kind, engine):
    """The same identity on a 256-wide net (K = 4), a ResNet-50 SkipPool net (K = 3, 64-px crops) and a net on
    xyz + reflectance points (K = 5)."""
    if kind == "w256":
        net, counts, hw, refl = _net("A", 7, "multiply", "none", sd=synthetic_state_dict("A", seed=7, width=256),
                                     appear_len=256, point_len=256), (3, 6, 2, 5), 32, False
    elif kind == "resnet50":
        net, counts, hw, refl = _net("C", 8, sd=synthetic_state_dict("C", seed=8, appear_arch="resnet50"),
                                     appear_arch="resnet50"), (5, 2, 4), 64, False
    else:
        net, counts, hw, refl = _net("B", 9, "minus", "single", sd=synthetic_state_dict("B", seed=9, point_in=4),
                                     without_reflectivity=False), (3, 1, 4, 6, 2), 32, True
    net = net.cuda().eval()
    B = 3
    one, (crops, pts, split) = _samples(B, counts, hw=hw, seed=200, reflectance=refl)
    net.chunk_pairs = 2
    o = net.forward_batch(crops.cuda(), pts.cuda(), split, counts=counts)
    net.chunk_pairs = None
    _assert_equals_loop(net, counts, one, o)


# ------------------------------------------------------------------------------------------------ GPU: reference goldens
@gpu
@pytest.mark.parametrize("path", FRAME_GOLDENS, ids=[os.path.basename(f)[:-3] for f in FRAME_GOLDENS])
def test_windows_match_reference_golden(path, engine):
    """forward on the golden's K-frame sample, and forward_batch(counts=...) on three copies of it, against the
    unmodified reference's eval forward (oracle/make_frame_goldens.py)."""
    g = torch.load(path)
    name, fusion, op, sm, thr, counts, pts, hw, ragged, seed = g["case"]
    counts = list(counts)
    L = sum(counts)
    net = _net(fusion, seed, op, sm).cuda().eval()
    dets, info, _ = synthetic_pair(counts[0], L - counts[0], pts, hw, seed=seed, ragged=ragged)
    det, links, new, end, trans = net(dets.cuda(), _cuda(info), [torch.tensor([k]) for k in counts])
    assert [tuple(x.shape) for x in links] == [tuple(x.shape) for x in g["links"]]
    for a, r in zip(links, g["links"]):
        assert relerr(a, r) < TOL
    assert relerr(new, g["new"]) < TOL and relerr(end, g["end"]) < TOL and det_close(det, g["det"], thr, TOL)
    assert relerr(trans[0], g["trans1"]) < 1e-5 and relerr(trans[1], g["trans2"]) < 1e-5
    B = 3
    s_ = info["points_split"][0].long()
    P = int(s_[-1])
    split = torch.cat([s_[:1]] + [s_[1:] + b * P for b in range(B)])
    o = net.forward_batch(dets.repeat(B, 1, 1, 1).cuda(), info["points"][0].repeat(B, 1).cuda(), split, counts=counts)
    zn, zl = g["new"].new_zeros(3, counts[0]), g["end"].new_zeros(3, counts[-1])
    for b in range(B):
        for a, r in zip(o["link"], g["links"]):
            assert relerr(a[b], r) < TOL
        assert relerr(torch.cat([zn, o["new"][b].cpu()], 1), g["new"]) < TOL
        assert relerr(torch.cat([o["end"][b].cpu(), zl], 1), g["end"]) < TOL
        assert det_close(o["det"][b], g["det"], thr, TOL)


# ------------------------------------------------------------------------------------------------ GPU: assignments
@gpu
@pytest.mark.parametrize("counts,B", WINDOWS + [((20, 45, 30), 3)], ids=["k3", "k4", "k8", "k3_wide"])
def test_predict_windows_equal_ortools_per_sample(counts, B, engine):
    """predict_batch(counts=...) solves every sample's programme in one call: its 0/1 tensors equal ortools_solve on
    each sample's own forward outputs, bit for bit, and match agrees with assign_link."""
    net = _net("A", 11, "multiply", "none").cuda().eval()
    one, (crops, pts, split) = _samples(B, counts, seed=300 + len(counts))
    L, t = sum(counts), net.test_mode
    r = net.predict_batch(crops.cuda(), pts.cuda(), split, counts=counts)
    assert r["match"].shape == (B, L - counts[-1]) and r["assign_det"].shape == (B, L)
    off = [sum(counts[:k]) for k in range(len(counts))]
    linked = 0
    for b, (d, info, ds) in enumerate(one):
        det, links, new, end, _ = net(d.cuda(), _cuda(info), ds)
        a_det, a_links, a_new, a_end = mmmot_b200.ortools_solve(det[t], [l[t:t + 1] for l in links], new[t], end[t], ds)
        assert torch.equal(r["assign_det"][b], a_det) and torch.equal(r["assign_new"][b], a_new)
        assert torch.equal(r["assign_end"][b], a_end)
        for k, (x, y) in enumerate(zip(r["assign_link"], a_links)):
            assert torch.equal(x[b], y.reshape(x[b].shape)), f"assign_link {k}, sample {b}"
            mt, al = r["match"][b, off[k]:off[k] + counts[k]].cpu(), x[b].cpu()
            assert torch.equal(mt >= 0, al.sum(1) > 0)
            assert torch.equal(mt[mt >= 0].long(), al.argmax(1)[mt >= 0])
            linked += int((mt >= 0).sum())
    assert linked > 0


# ------------------------------------------------------------------------------------------------ GPU: two frames
@gpu
@pytest.mark.parametrize("n,m", [(1, 1), (7, 9), (20, 45)])
def test_two_frame_counts_equal_n_m(n, m, engine):
    """counts = (n, m) gives the tensors of (n, m) (link and assign_link in a one-element list); the two-frame
    HostPipeline is unchanged by the counts form."""
    net = _net("C", 4).cuda().eval()
    B = 4
    _, (crops, pts, split) = _samples(B, (n, m), seed=400 + n)
    crops, pts = crops.cuda(), pts.cuda()
    a = net.forward_batch(crops, pts, split, n, m, keep_feats=True)
    c = net.forward_batch(crops, pts, split, counts=(n, m), keep_feats=True)
    assert isinstance(c["link"], list) and len(c["link"]) == 1 and torch.equal(c["link"][0], a["link"])
    for k in ("det", "new", "end", "feats", "status"):
        assert torch.equal(c[k], a[k]), k
    assert all(torch.equal(x, y) for x, y in zip(a["trans"], c["trans"]))
    pa = net.predict_batch(crops, pts, split, n, m)
    pc = net.predict_batch(crops, pts, split, counts=[n, m])
    assert torch.equal(pc["assign_link"][0], pa["assign_link"])
    for k in ("match", "assign_det", "assign_new", "assign_end"):
        assert torch.equal(pc[k], pa[k]), k
    h_crops, h_pts = crops.cpu().pin_memory(), pts.cpu().pin_memory()
    ra = mmmot_b200.HostPipeline(net, n, m, sub_batches=2).run(h_crops, h_pts, split)
    rc = mmmot_b200.HostPipeline(net, counts=(n, m), sub_batches=2).run(h_crops, h_pts, split)
    for k in ("match", "assign_det", "assign_new", "assign_end", "match_device"):
        assert torch.equal(ra[k], rc[k]), k
    assert torch.equal(ra["match"], pa["match"].cpu())


# ------------------------------------------------------------------------------------------------ GPU: HostPipeline
@gpu
def test_host_pipeline_windows_equal_predict_batch():
    """HostPipeline(counts=...) on pinned host windows returns predict_batch(counts=...)'s results, across repeated runs
    and for a batch that cannot be cut into sub-batches; the FP16 range flag is raised through it."""
    net = _net("C", 6).cuda().eval()
    counts = (4, 1, 6, 3)
    for B, seed in ((8, 500), (3, 600)):
        _, (crops, pts, split) = _samples(B, counts, seed=seed)
        ref = net.predict_batch(crops.cuda(), pts.cuda(), split, counts=counts)
        pipe = mmmot_b200.HostPipeline(net, counts=counts, sub_batches=4)
        h_crops, h_pts = crops.pin_memory(), pts.pin_memory()
        for _ in range(2):
            r = pipe.run(h_crops, h_pts, split)
            assert r["match"].shape == (B, sum(counts) - counts[-1])
            assert torch.equal(r["match"], ref["match"].cpu()) and torch.equal(r["match_device"], ref["match"])
            for k in ("assign_det", "assign_new", "assign_end"):
                assert torch.equal(r[k], ref[k].cpu()), k
        assert pipe.nsub == (4 if B == 8 else 1)
    mmmot_b200.set_engine("tcgen05")
    try:
        o = net.forward_batch((crops * 1e6).cuda(), pts.cuda(), split, counts=counts, check=False)
        assert int(o["status"]) & 1
        with pytest.raises(_lib.MmmotError, match="MMMOT_E_RANGE"):
            pipe.run((h_crops * 1e6).pin_memory(), h_pts, split)
    finally:
        mmmot_b200.set_engine("auto")


# ------------------------------------------------------------------------------------------------ CPU
def test_argument_errors_before_any_device_work(lib_built):
    """Both counts and n / m, fewer than two frames, a count below one or not an int: ValueError; crops or
    points_split that do not hold whole windows: MmmotError naming counts.  The net is on the CPU, so any of these
    reaching the device would raise the no-CPU-fallback error instead."""
    net = _net().eval()
    crops, pts, split = torch.zeros(12, 3, 32, 32), torch.zeros(20, 3), torch.arange(13)
    for kw in (dict(n=4, counts=(4, 4, 4)), dict(n=4, m=4, counts=(4, 4, 4)), dict(m=4, counts=(4, 4, 4)),
               dict(counts=(12,)), dict(counts=()), dict(counts=(4, 0, 8)), dict(counts=(6, -1, 7)),
               dict(counts=(4, 4.0, 4)), dict(counts=(4, "4", 4)), dict()):
        with pytest.raises(ValueError):
            net.forward_batch(crops, pts, split, **kw)
        with pytest.raises(ValueError):
            net.predict_batch(crops, pts, split, **kw)
        with pytest.raises(ValueError):
            mmmot_b200.HostPipeline(net, **kw)
    with pytest.raises(_lib.MmmotError, match="do not match counts"):
        net.forward_batch(crops[:10], pts, split[:11], counts=(2, 2, 2))            # 10 rows, windows of 6
    with pytest.raises(_lib.MmmotError, match="do not match counts"):
        net.forward_batch(crops, pts, split, counts=(2, 3, 2))                       # 12 rows, windows of 7
    with pytest.raises(_lib.MmmotError, match="do not match counts"):
        net.forward_batch(crops, pts, split[:12], counts=(2, 2, 2))                  # 12 crops, 11 point ranges
    with pytest.raises(_lib.MmmotError, match="do not match counts"):
        net.forward_batch(None, pts, split[:11], counts=(1, 2, 4), stack=1)          # LiDAR alone: 10 ranges, windows of 7
    with pytest.raises(_lib.MmmotError, match="runs on CUDA"):                      # a valid call gets as far as the device
        net.forward_batch(crops, pts, split, counts=(2, 2, 2))
    with pytest.raises(NotImplementedError):
        net.train().forward_batch(crops, pts, split, counts=(2, 2, 2))


COUNTS = [(4, 1, 6), (7, 3, 1, 5), (2, 5, 1, 3, 6, 4, 1, 2), (128,) * 8, (16, 4, 9), (128, 64)]


@pytest.mark.parametrize("counts", COUNTS)
@pytest.mark.parametrize("stack", [None, 0, 1, 2])
def test_window_workspace_is_the_max_over_its_stages(lib_built, counts, stack):
    """The workspace of a chunk of K-frame windows is the largest of its stages: the affinity stage of each pair of
    consecutive frames and the feature stages on the window's L detections."""
    lib = _lib.load()
    net = _net().eval()
    L, pairs, P, hw = sum(counts), 6, 6 * sum(counts) * 20, 64
    trans = list(zip(counts[:-1], counts[1:]))
    aff = lib.mmmot_affinity_workspace if stack is None else lib.mmmot_affinity_stack_workspace
    stages = [aff(pairs, a, b) for a, b in trans]
    stages.append(lib.mmmot_fusion_det_workspace(pairs, L) if stack is None else lib.mmmot_fusion_det_stack_workspace(pairs, L))
    if stack != 1:
        stages.append(lib.mmmot_appearance_workspace(pairs * L, hw, hw))
    if stack != 0:
        stages.append(lib.mmmot_pointnet_workspace(pairs, L, P))
    ws = net._workspace_bytes(pairs, trans, L, P, hw, hw, stack)
    assert ws == max(stages)
    for a, b in trans:      # never less than a frame-pair of any of its transitions alone would ask for
        assert ws >= net._workspace_bytes(pairs, [(a, b)], 0, 0, hw, hw, stack)


@pytest.mark.parametrize("counts", COUNTS)
def test_pick_chunk_stays_within_its_budget(lib_built, monkeypatch, counts):
    """_pick_chunk halves the chunk until a chunk's workspace (every transition and the feature stages) fits half the
    free memory, for any free memory; a chunk of one sample is the floor; chunk_pairs overrides it."""
    net = _net().eval()
    B, L, per, hw = 64, sum(counts), 37.5, 64
    trans = list(zip(counts[:-1], counts[1:]))
    need = lambda c: net._workspace_bytes(c, trans, L, int(per * c) + 1, hw, hw)
    for free in (1e5, 1e8, need(1) * 2.5, need(7) * 2.01, need(B) * 2, 1e11, 2e12):
        monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev, f=free: (int(f), int(f)))
        c = net._pick_chunk(B, counts, per, hw, hw, "cuda:0")
        budget = min(int(free) * 0.5, 48e9)
        assert 1 <= c <= B
        assert c == 1 or need(c) <= budget, (free, c)
        assert c == B or need(min(B, 2 * c)) > budget, (free, c)     # halving stopped at the first chunk that fits
    net.chunk_pairs = 5
    assert net._pick_chunk(B, counts, per, hw, hw, "cuda:0") == 5 and net._pick_chunk(3, counts, per, hw, hw, "cuda:0") == 3
