"""The reference's narrower nets (appear_len = point_len = 256 or 128: vgg16_bn_256 / _128, modules/vgg.py:83-98, and every
PointNet, fusion, affinity and w_det width divided by 512 // width), run exactly as their 512-wide embedding
(weights.embed_width), from the checkpoint to the kernels.

CPU: each width's state_dict against the reference's own key -> shape list (tests/golden/width/, written by
oracle/make_width_goldens.py from the UNMODIFIED reference); the layout of the stack channels; the embedding identity --
the embedded 512-wide state_dict through the fp32 restatement of the 512-wide net (oracle/torch_ref.py, and a ResNet trunk
restated here) reproduces every reduced fixture; the default width's schema and draws unchanged; the constructor guards.

GPU, on both engines: the forward against every fixture; forward_batch bit-identical to looped forward; the returned
features in the reference's channel order and associate_batch on them; predict_batch's assignment against the one solved
from the fixture's scores.
"""
import glob
import json
import os

import pytest
import torch
import torch.nn.functional as F

import mmmot_b200
from helpers import GOLDEN_DIR, TOL, TOL_DEGENERATE, det_close, relerr
from mmmot_b200.schema import RESNET_BLOCKS, WIDTHS, resnet_convs, state_schema
from mmmot_b200.synthetic import synthetic_pair, synthetic_state_dict
from mmmot_b200.weights import embed_width, pack_tc, stack_index, stn_constant
from oracle import torch_ref

gpu = pytest.mark.gpu
WIDTH = os.path.join(GOLDEN_DIR, "width")
EVAL = [torch.load(f) for f in sorted(glob.glob(os.path.join(WIDTH, "w*.pt")))]
SCHEMAS = sorted(glob.glob(os.path.join(WIDTH, "schema_*.json")))
ORACLE_TOL = 2e-5          # the oracle restatement against the reference's fixtures, away from degenerate GroupNorms


def case_tol(case, tol):
    """GroupNorm over the 2-detection grid of N*M = 1 is ill-conditioned (helpers.TOL_DEGENERATE)."""
    return TOL_DEGENERATE if case[8] * case[9] <= 4 else tol


def sd_of(case, seed=None):
    _, arch, head, width, fusion = case[:5]
    return synthetic_state_dict(fusion, seed=case[13] if seed is None else seed, appear_arch=arch, appear_head=head,
                                width=width)


def net_of(case, seed=None, **kw):
    _, arch, head, width, fusion, op, sm, thr = case[:8]
    net = mmmot_b200.TrackingNet(2, appear_len=width, point_len=width, appear_arch=arch, appear_skippool=head == "skippool",
                                 appear_fpn=head == "fpn", score_arch="branch_cls", score_fusion_arch=fusion, affinity_op=op,
                                 softmax_mode=sm, neg_threshold=thr, test_mode=2, dropblock=0, **kw)
    net.load_state_dict(sd_of(case, seed), strict=True)
    return net.eval()


def pair_of(case):
    n, m, pts, hw, ragged, seed = case[8:14]
    return synthetic_pair(n, m, pts, hw, seed=seed, ragged=ragged)


# ------------------------------------------------------------------------------------------------ fp32 restatement
def _conv_bn(sd, conv, bn, x, stride, pad):
    return torch_ref._bn_eval(F.conv2d(x, sd[f"{conv}.weight"], stride=stride, padding=pad), sd, bn)


def resnet_maps(sd, arch, x):
    """torchvision's ResNet trunk (eval) as the reference's Resnet wrapper runs it: the four stage outputs."""
    spec = resnet_convs(arch)
    f = lambda i, x: _conv_bn(sd, spec[i][0], spec[i][1], x, spec[i][5], spec[i][4] // 2)
    x = F.max_pool2d(F.relu(f(0, x)), 3, 2, 1)
    i, maps = 1, []
    for nb in RESNET_BLOCKS[arch]:
        for b in range(nb):
            y = f(i + 2, F.relu(f(i + 1, F.relu(f(i, x)))))
            x = F.relu(y + (f(i + 3, x) if b == 0 else x))
            i += 4 if b == 0 else 3
        maps.append(x)
    return maps


def fpn_head(sd, maps):
    """modules/appear_net.py:192-210: laterals, the bilinear top-down chain, conv_last."""
    lat = lambda k: F.relu(_conv_bn(sd, f"appearance.fpn_in.{k}.0", f"appearance.fpn_in.{k}.1", maps[k], 1, 0))
    out = lat(3)
    for k in (2, 1, 0):
        c = lat(k)
        out = F.interpolate(out, size=c.shape[2:], mode="bilinear", align_corners=False) + c
    v = F.conv2d(out.mean(dim=(2, 3), keepdim=True), sd["appearance.conv_last.1.weight"], sd["appearance.conv_last.1.bias"])
    return F.relu(torch_ref._bn_eval(v, sd, "appearance.conv_last.2")).flatten(1)


def forward512(sd, case, dets, info, split):
    """The 512-wide net's eval forward in fp32 on the CPU (torch_ref's stages; the ResNet trunks restated above)."""
    _, arch, head, _, fusion, op, sm, thr = case[:8]
    if arch == "vgg":
        app = torch_ref.appearance(sd, dets)
    else:
        maps = resnet_maps(sd, arch, dets)
        app = fpn_head(sd, maps) if head == "fpn" else torch.cat([torch_ref.skip_pool(sd, s, x) for s, x in enumerate(maps)], -1)
    pts, trans = torch_ref.pointnet(sd, info["points"].transpose(-1, -2), info["points_split"].long().squeeze(0))
    feats = torch_ref.fusion(sd, fusion, torch.cat([app, pts], dim=-1).t().unsqueeze(0))
    det = torch_ref.determine_det(sd, feats, thr)
    n = int(split[0])
    link, new, end = torch_ref.associate(sd, feats[:, :, :n], feats[:, :, n:], op, sm)
    new = torch.cat([new.new_zeros(3, n), new], 1)              # eval-mode zero padding (tracking_net.py:183-189)
    end = torch.cat([end, end.new_zeros(3, int(split[1]))], 1)
    return feats, det, link.squeeze(1), new, end, trans


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("path", SCHEMAS, ids=[os.path.basename(p)[7:-5] for p in SCHEMAS])
def test_state_dict_matches_reference_schema(path):
    arch, head, width = os.path.basename(path)[7:-5].split("_")
    width = int(width)
    ref = json.load(open(path))
    assert [[k, list(s)] for k, (s, _) in state_schema("C", 3, arch, head, width).items()] == ref
    net = mmmot_b200.TrackingNet(2, appear_len=width, point_len=width, appear_arch=arch, appear_skippool=head == "skippool",
                                 appear_fpn=head == "fpn", score_arch="branch_cls")
    assert net.width == width
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
    res = net.load_state_dict(synthetic_state_dict("C", seed=3, appear_arch=arch, appear_head=head, width=width), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert list(state_schema("C", 3, arch, head, width)) == list(state_schema("C", 3, arch, head))


def test_default_width_schema_and_draws_unchanged():
    for arch, head in (("vgg", "skippool"), ("resnet50", "skippool"), ("resnet101", "fpn")):
        for fusion in "ABC":
            assert state_schema(fusion, 3, arch, head) == state_schema(fusion, 3, arch, head, 512)
        a = synthetic_state_dict("C", seed=9, appear_arch=arch, appear_head=head)
        b = synthetic_state_dict("C", 9, 3, arch, head, 512)
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    for bad in (64, 384, 1024):
        with pytest.raises(ValueError):
            state_schema("C", width=bad)


@pytest.mark.parametrize("width", WIDTHS[1:])
def test_stack_layout(width):
    """pi maps SkipPool head s's 128 channels onto copies of its width / 4 channels, each aligned 32-channel block onto one
    whole group of PointNet's GroupNorm(16 // r, width), and every channel of the narrow stack to 512 / width copies."""
    pi = stack_index(width)
    q, r = width // 4, 512 // width
    for s in range(4):
        assert set(pi[128 * s:128 * s + 128].tolist()) == set(range(q * s, q * s + q))
    for b in range(16):
        blk = pi[32 * b:32 * b + 32]
        assert sorted(blk.tolist()) == list(range(int(blk[0]) // 32 * 32, int(blk[0]) // 32 * 32 + 32))
    assert torch.equal(torch.bincount(pi, minlength=width), torch.full((width,), r))
    assert torch.equal(stack_index(512), torch.arange(512))


@pytest.mark.parametrize("width", WIDTHS[1:])
def test_embedding_scales_by_powers_of_two(width):
    """Each embedded weight is a narrow one divided by 1, 2 or 4, so the tensor-core hi/lo tiles are the narrow weight's
    tiles with a shifted out_scale: hi and lo are exact copies, scale divided by k."""
    sd = synthetic_state_dict("C", seed=4, width=width)
    e = embed_width(sd, "C", width)
    assert set(e) == set(state_schema("C"))
    assert all(tuple(e[k].shape) == s for k, (s, _) in state_schema("C").items())
    w = sd["w_link.conv1.3.weight"].double().reshape(width, width)
    we = e["w_link.conv1.3.weight"].reshape(512, 512)
    pi = stack_index(width)
    assert torch.equal(we, w[pi][:, pi] / (512 // width))
    p1, s1 = pack_tc(w.t())
    p2, s2 = pack_tc(we.t())
    assert s2 == s1 / (512 // width)
    assert torch.equal(p2.view(torch.float16).unique(), p1.view(torch.float16).unique())


@pytest.mark.parametrize("g", EVAL, ids=[c["case"][0] for c in EVAL])
def test_embedding_reproduces_reference_fixture(g):
    """The embedding identity: the reduced checkpoint embedded in the 512-wide net (weights.embed_width), run through the
    fp32 restatement of the 512-wide net, reproduces the reference's reduced net; its stacks carry the reference's
    features at every copy, and STN2 is T2 embedded."""
    case = g["case"]
    _, arch, head, width, fusion = case[:5]
    sd = sd_of(case)
    e = {k: v.float() if v.is_floating_point() else v for k, v in embed_width(sd, fusion, width, arch, head).items()}
    dets, info, split = pair_of(case)
    with torch.no_grad():
        feats, det, link, new, end, trans = forward512(e, case, dets, info, split)
    tol = case_tol(case, ORACLE_TOL)
    pi = stack_index(width)
    errs = {"feats": relerr(feats, g["feats"][:, pi]), "det": relerr(det, g["det"]),
            "link": relerr(link, g["link"]), "new": relerr(new, g["new"]), "end": relerr(end, g["end"])}
    print(f"\n{case[0]}: {errs}")
    assert all(v < tol for v in errs.values()), errs
    k2 = 64 * width // 512
    t2 = stn_constant(sd, "point_net.feat.stn2", k2)
    assert relerr(t2.float(), g["trans2"][0]) < 1e-6
    p = torch.arange(64) % k2                  # PointNet's 64/r local channels tiled over 64
    assert relerr(trans[1][0], t2[p][:, p].float() / (512 // width)) < 1e-6
    assert relerr(trans[0], g["trans1"]) < 1e-5


def test_fixture_set_covers_the_cases():
    cases = {(c[1], c[2], c[3]) for c in (g["case"] for g in EVAL)}
    assert cases >= {("vgg", "skippool", 256), ("vgg", "skippool", 128), ("resnet50", "skippool", 256),
                     ("resnet50", "fpn", 256)}
    vgg = [g["case"] for g in EVAL if g["case"][1] == "vgg"]
    for w in (256, 128):
        assert {c[4] for c in vgg if c[3] == w} == set("ABC")
        assert any(c[8] * c[9] == 1 for c in vgg if c[3] == w) and any(c[8] != c[9] for c in vgg if c[3] == w)
    assert {c[5] for c in vgg} == {"multiply", "minus_abs", "minus"} and all(c[12] for c in vgg)
    assert any(g["case"][2] == "fpn" and g["case"][11] == 224 for g in EVAL)
    assert all(os.path.getsize(f) < 150_000 for f in glob.glob(os.path.join(WIDTH, "*")))


def test_constructor_guards():
    for kw in (dict(appear_len=256), dict(point_len=128), dict(appear_len=256, point_len=128),
               dict(appear_len=64, point_len=64), dict(appear_len=0, point_len=0)):
        with pytest.raises(NotImplementedError, match="appear_len/point_len"):
            mmmot_b200.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", **kw)
    case = EVAL[0]["case"]
    net = net_of(case).train()
    dets, info, split = pair_of(case)
    with pytest.raises(NotImplementedError, match="training-mode"):
        net(dets, info, split)
    cfg = dict(sample_max_len=2, without_reflectivity=True, dropblock=5, use_dropout=False,
               model=dict(point_arch="v1", point_len=128, appear_arch="vgg", appear_len=128, appear_skippool=True,
                          appear_fpn=False, end_arch="v2", end_mode="avg", affinity_op="minus_abs", softmax_mode="dual_add",
                          score_arch="branch_cls", neg_threshold=0.2, score_fusion_arch="C", test_mode=2))
    net = mmmot_b200.build_model({"common": cfg})
    assert net.width == 128 and net.state_dict()["w_det.0.weight"].shape == (128, 128, 1)


def test_reference_reduced_nets_build():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("no reference checkout (MMMOT_REFERENCE)")
    from oracle import make_width_goldens as mwg
    for path in SCHEMAS:
        arch, head, width = os.path.basename(path)[7:-5].split("_")
        net = mwg.reference_net(arch, head, int(width), "C", "minus_abs", "dual_add", 0.2)
        assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == json.load(open(path))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(params=["fp32", "tcgen05"])
def engine(request):
    mmmot_b200.set_engine(request.param)
    yield request.param
    mmmot_b200.set_engine("auto")


@gpu
@pytest.mark.parametrize("g", EVAL, ids=[c["case"][0] for c in EVAL])
def test_forward_matches_reference_golden(g, engine):
    from oracle import lp_ref
    case = g["case"]
    name, width, thr, n, m = case[0], case[3], case[7], case[8], case[9]
    net = net_of(case).cuda()
    dets, info, split = pair_of(case)
    det, link, new, end, trans = net(dets.cuda(), {k: v.cuda() for k, v in info.items()}, split)
    o = net.predict_batch(dets.cuda(), info["points"][0].cuda(), info["points_split"][0].long(), n, m)
    ob = net.forward_batch(dets.cuda(), info["points"][0].cuda(), info["points_split"][0].long(), n, m, keep_feats=True)
    tol = case_tol(case, TOL)
    assert ob["feats"].shape == (1, 3, width, n + m) and trans[1].shape == (1, width // 8, width // 8)
    errs = {"feats": relerr(ob["feats"][0], g["feats"]), "link": relerr(link[0], g["link"]), "new": relerr(new, g["new"]),
            "end": relerr(end, g["end"])}
    print(f"\n{name} [{engine}]: {errs}")
    assert all(e < tol for e in errs.values()), errs
    assert det_close(det, g["det"], thr, tol)
    assert relerr(trans[1], g["trans2"]) < 1e-5 and relerr(trans[0], g["trans1"]) < 1e-5
    # associate_batch on the returned (reference-order) features reproduces the forward's scores
    lk, nw, en = net.associate_batch(ob["feats"], n, m)
    assert relerr(lk[0], link[0]) < 1e-5 and relerr(nw[0], new[:, n:]) < 1e-5 and relerr(en[0], end[:, :n]) < 1e-5
    # predict_batch's assignment: the fixture's own optimum wherever it beats the second best by more than the perturbation
    t = 2
    rdet, rlink, rnew, rend = g["det"][t], g["link"][t:t + 1], g["new"][t], g["end"][t]
    mil, obj, y = lp_ref.milp_solve(rdet, [rlink], rnew, rend, [n, m])
    _, obj2, _ = lp_ref.milp_solve(rdet, [rlink], rnew, rend, [n, m], exclude=y)
    perturb = float((o["det"][0, t].cpu() - rdet).abs().sum() + (o["link"][0, t].cpu() - rlink[0]).abs().sum()
                    + (o["new"][0, t].cpu() - rnew[n:]).abs().sum() + (o["end"][0, t].cpu() - rend[:n]).abs().sum())
    got = (o["assign_det"][0].cpu(), o["assign_link"][0].cpu(), o["assign_new"][0].cpu(), o["assign_end"][0].cpu())
    flat = lambda t: t.float().reshape(-1)
    same = all(torch.equal(flat(a), flat(b)) for a, b in zip(got, (mil[0], mil[1][0], mil[2], mil[3])))
    print(f"{name}: LP gap {obj - obj2:.3e}, perturbation {perturb:.3e}, identical {same}")
    if obj - obj2 > perturb:
        assert same


@gpu
@pytest.mark.parametrize("eng", ["auto", "fp32", "tcgen05"])
@pytest.mark.parametrize("arch,head,width", [("vgg", "skippool", 256), ("vgg", "skippool", 128), ("resnet50", "fpn", 256)])
def test_forward_batch_equals_looped_forward(arch, head, width, eng):
    """Three pairs in one forward_batch == each pair through forward, bit for bit, at (n, m) = (3, 2) and (6, 6)."""
    case = ("b", arch, head, width, "C", "minus_abs", "dual_add", 0.2)
    net = net_of(case, seed=59).cuda()
    mmmot_b200.set_engine(eng)
    try:
        for n, m in ((3, 2), (6, 6)):
            pairs = [synthetic_pair(n, m, 16, 64, seed=60 + n + b, ragged=True) for b in range(3)]
            crops = torch.cat([p[0] for p in pairs]).cuda()
            pts = torch.cat([p[1]["points"][0] for p in pairs]).cuda()
            sp, off = [torch.zeros(1, dtype=torch.int64)], 0
            for p in pairs:
                s = p[1]["points_split"][0].long()
                sp.append(s[1:] + off)
                off += int(s[-1])
            o = net.forward_batch(crops, pts, torch.cat(sp), n, m, keep_feats=True)
            assert int(o["status"]) == 0 and o["feats"].shape == (3, 3, width, n + m)
            for b, (d, info, split) in enumerate(pairs):
                det, link, new, end, trans = net(d.cuda(), {k: v.cuda() for k, v in info.items()}, split)
                assert torch.equal(o["link"][b], link[0]) and torch.equal(o["det"][b], det), (n, m, b)
                assert torch.equal(o["new"][b], new[:, n:]) and torch.equal(o["end"][b], end[:, :n])
            assert torch.equal(o["trans"][1], trans[1]) and trans[1].shape == (1, width // 8, width // 8)
    finally:
        mmmot_b200.set_engine("auto")
