"""ORACLE — test infrastructure, NOT product code.

CPU fp32 restatement (functional PyTorch, no nn.Module) of the reference's association
forward ``TrackingNet.forward`` in eval mode.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu_baseline / ``--impl reference`` legs may import this file; the product
(``mmmot_b200``) never does.

Every function names the reference lines it restates (paths relative to the reference checkout).
It deliberately keeps the reference's *work* (dead STN branches, the 1088-wide head conv,
the materialised 3xDxNxM pairwise tensor), because it doubles as the CPU baseline.

Pinned against the real reference modules: ``oracle/make_goldens.py`` runs the unmodified
reference (imported in place by oracle/make_goldens.py) on seeded inputs and commits
the outputs under tests/golden/; tests/test_oracle.py checks this file against them.
"""
import torch
import torch.nn.functional as F

from mmmot_b200.schema import SKIP_CHANNELS, VGG_POOL_AFTER, VGG_STAGES

EPS = 1e-5


def group_norm(x, groups, w, b):
    """torch.nn.GroupNorm forward (eps 1e-5, biased variance) written out, so that the
    1-value-per-group case returns beta like reference-era torch (SURVEY F3) without
    patching torch.nn.functional._verify_batch_size."""
    n, c = x.shape[:2]
    xg = x.reshape(n, groups, -1)
    mean = xg.mean(-1, keepdim=True)
    var = xg.var(-1, unbiased=False, keepdim=True) if xg.shape[-1] > 1 else torch.zeros_like(mean)
    y = ((xg - mean) * torch.rsqrt(var + EPS)).reshape(x.shape)
    shape = (1, c) + (1,) * (x.dim() - 2)
    return y * w.reshape(shape) + b.reshape(shape)


def _bn_eval(x, sd, p):
    """BatchNorm (eval: running statistics)."""
    shape = (1, -1) + (1,) * (x.dim() - 2)
    inv = torch.rsqrt(sd[p + ".running_var"] + EPS) * sd[p + ".weight"]
    return (x - sd[p + ".running_mean"].reshape(shape)) * inv.reshape(shape) + sd[p + ".bias"].reshape(shape)


# ---------------------------------------------------------------- appearance
def vgg_maps(sd, dets):
    """modules/appear_net.py:166-172 (vgg_forward) over the stages built at :130-157 from
    modules/vgg.py:67-80 cfg 'D': conv3x3 pad1 + BN(eval) + ReLU, 2x2 max-pools."""
    x = dets
    maps = []
    for s, stage in enumerate(VGG_STAGES):
        p = f"appearance.layers.{s}"
        for idx, _, _ in stage:
            x = F.conv2d(x, sd[f"{p}.{idx}.weight"], sd[f"{p}.{idx}.bias"], padding=1)
            x = F.relu(_bn_eval(x, sd, f"{p}.{idx + 1}"))
            if idx in VGG_POOL_AFTER[s]:
                x = F.max_pool2d(x, 2, 2)
        maps.append(x)
    return maps


def drop_block(x, block_size, drop_prob=0.1):
    """modules/dropblock.py:28-67 (DropBlock2D.forward in training): seeds from the CPU generator, max-pooled into
    blocks, inverted, rescaled by numel / sum."""
    mask = (torch.rand(x.shape[0], *x.shape[2:]) < drop_prob / (block_size ** 2)).float().to(x.device)
    bm = F.max_pool2d(mask[:, None], kernel_size=(block_size, block_size), stride=(1, 1), padding=block_size // 2)
    if block_size % 2 == 0:
        bm = bm[:, :, :-1, :-1]
    bm = 1 - bm.squeeze(1)
    return x * bm[:, None] * bm.numel() / bm.sum()


def skip_pool(sd, s, fmap, dropblock=0):
    """modules/appear_net.py:27-32 with fc from :18-25 (dropblock is identity in eval; in training the two deepest heads
    carry one when the config sets dropblock, appear_net.py:143-152)."""
    p = f"appearance.global_pool.{s}.fc"
    if dropblock:
        fmap = drop_block(fmap, dropblock)
    o = fmap.mean(dim=(2, 3), keepdim=True)
    o = group_norm(o, 1, sd[f"{p}.0.weight"], sd[f"{p}.0.bias"])
    o = F.conv2d(o, sd[f"{p}.1.weight"], sd[f"{p}.1.bias"])
    o = F.relu(group_norm(o, 1, sd[f"{p}.2.weight"], sd[f"{p}.2.bias"]))
    o = F.conv2d(o, sd[f"{p}.4.weight"], sd[f"{p}.4.bias"])
    o = F.relu(group_norm(o, 1, sd[f"{p}.5.weight"], sd[f"{p}.5.bias"]))
    return o.reshape(fmap.shape[0], -1)


def appearance(sd, dets):
    """modules/appear_net.py:178-190: four SkipPool heads concatenated -> L x 512."""
    maps = vgg_maps(sd, dets)
    assert tuple(m.shape[1] for m in maps) == SKIP_CHANNELS
    return torch.cat([skip_pool(sd, s, m) for s, m in enumerate(maps)], dim=-1)


# ---------------------------------------------------------------- point net
def stn(sd, p, x, k):
    """modules/point_net.py:72-86 (STN3d.forward), executed as written."""
    def cgr(x, c, n):
        y = F.conv1d(x, sd[f"{p}.{c}.weight"], sd[f"{p}.{c}.bias"])
        return F.relu(group_norm(y, y.shape[1], sd[f"{p}.{n}.weight"], sd[f"{p}.{n}.bias"]))
    x = cgr(cgr(cgr(x, "conv1", "bn1"), "conv2", "bn2"), "conv3", "bn3")
    x = torch.max(x, -1, keepdim=True)[0].reshape(-1, 1024)
    for fc, bn in (("fc1", "fc_bn1"), ("fc2", "fc_bn2")):
        x = F.linear(x, sd[f"{p}.{fc}.weight"], sd[f"{p}.{fc}.bias"])
        x = F.relu(group_norm(x, x.shape[1], sd[f"{p}.{bn}.weight"], sd[f"{p}.{bn}.bias"]))
    x = F.linear(x, sd[f"{p}.output.weight"], sd[f"{p}.output.bias"]).reshape(-1, k, k)
    return x + sd[f"{p}.idt"]


def stn_constant(sd, p, k):
    """SURVEY F4: at batch 1 fc_bn1/fc_bn2 see one value per group, so STN3d returns the
    input-independent constant I + reshape(W_out relu(beta_fc_bn2) + b_out)."""
    v = F.relu(sd[f"{p}.fc_bn2.bias"])
    return (sd[f"{p}.output.weight"] @ v + sd[f"{p}.output.bias"]).reshape(1, k, k) + sd[f"{p}.idt"]


def _segment_mean(x, split):
    """The Python loops at modules/point_net.py:33-37 / :140-146: AdaptiveAvgPool1d(1) of every
    detection's slice (variables are *named* max_feat but the pooling is a mean, SURVEY F5)."""
    return torch.cat([x[:, :, int(split[i]):int(split[i + 1])].mean(-1, keepdim=True)
                      for i in range(len(split) - 1)], dim=-1)


def pointnet_feat(sd, x, split):
    """modules/point_net.py:115-153 (PointNetfeatGN.forward)."""
    p = "point_net.feat"

    def cgr(x, i):
        y = F.conv1d(x, sd[f"{p}.conv{i}.weight"], sd[f"{p}.conv{i}.bias"])
        return F.relu(group_norm(y, y.shape[1], sd[f"{p}.bn{i}.weight"], sd[f"{p}.bn{i}.bias"]))
    t1 = stn(sd, f"{p}.stn1", x, x.shape[1])
    x = torch.bmm(x.transpose(2, 1), t1).transpose(2, 1)
    x = cgr(x, 1)
    t2 = stn(sd, f"{p}.stn2", x, 64)
    x = torch.bmm(x.transpose(2, 1), t2).transpose(2, 1)
    local = x
    x = cgr(cgr(cgr(cgr(x, 2), 3), 4), 5)
    seg = _segment_mean(x, split)                                   # 1 x 1024 x L
    cnt = (split[1:] - split[:-1]).long()
    glob = torch.repeat_interleave(seg, cnt, dim=-1)                # broadcast back (:143-146)
    assert glob.shape[-1] == x.shape[-1]
    return [local, glob], [t1, t2]


def pointnet(sd, points_t, split, dropout=False):
    """modules/point_net.py:25-44 (PointNet_v1.forward); points_t is 1 x 3 x P_t.  dropout: the training-mode
    nn.Dropout(0.5) of :29-30."""
    feats, trans = pointnet_feat(sd, points_t, split)
    x = torch.cat(feats, dim=1)
    x = F.conv1d(x, sd["point_net.conv1.weight"], sd["point_net.conv1.bias"])
    x = F.relu(group_norm(x, 512, sd["point_net.bn1.weight"], sd["point_net.bn1.bias"]))
    if dropout:
        x = F.dropout(x, p=0.5, training=True)
    seg = _segment_mean(x, split)                                   # 1 x 512 x L
    o = F.conv1d(seg, sd["point_net.conv2.weight"], sd["point_net.conv2.bias"])
    o = F.relu(group_norm(o, 16, sd["point_net.bn2.weight"], sd["point_net.bn2.bias"]))
    return o.transpose(-1, -2).squeeze(0), trans


# ---------------------------------------------------------------- fusion / det score
def fusion(sd, arch, objs):
    """modules/fusion_net.py: A :85-92, B :62-70, C :31-42.  objs is 1 x 2D x L; returns 3 x D x L
    (note input_p / gate_p act on stack 0 = image: the names are swapped in the reference)."""
    f = "fusion_module"
    L = objs.shape[-1]
    feats = objs.reshape(2, -1, L)

    def lin_gn(name, x):
        y = F.conv1d(x, sd[f"{f}.{name}.0.weight"], sd[f"{f}.{name}.0.bias"])
        return group_norm(y, y.shape[1], sd[f"{f}.{name}.1.weight"], sd[f"{f}.{name}.1.bias"])
    if arch == "A":
        fused = lin_gn("input_w", objs)
    elif arch == "B":
        fused = lin_gn("input_p", feats[:1]) + lin_gn("input_i", feats[1:])
    elif arch == "C":
        gp = torch.sigmoid(F.conv1d(feats[:1], sd[f"{f}.gate_p.0.weight"], sd[f"{f}.gate_p.0.bias"]))
        gi = torch.sigmoid(F.conv1d(feats[1:], sd[f"{f}.gate_i.0.weight"], sd[f"{f}.gate_i.0.bias"]))
        fused = (gp * lin_gn("input_p", feats[:1]) + gi * lin_gn("input_i", feats[1:])) / (gp + gi)
    else:
        raise ValueError(arch)
    return torch.cat([feats, fused], dim=0)


def determine_det(sd, feats, neg_threshold, score_arch="branch_cls"):
    """modules/tracking_net.py:149-163 with w_det from :91-100, eval mode."""
    x = F.conv1d(feats, sd["w_det.0.weight"], sd["w_det.0.bias"])
    x = F.relu(_bn_eval(x, sd, "w_det.1"))
    x = F.conv1d(x, sd["w_det.3.weight"], sd["w_det.3.bias"])
    x = F.relu(_bn_eval(x, sd, "w_det.4"))
    s = F.conv1d(x, sd["w_det.6.weight"], sd["w_det.6.bias"]).squeeze(1)
    if "cls" in score_arch:
        s = torch.sigmoid(s)
    return s - (s < neg_threshold).float()


# ---------------------------------------------------------------- association
def pairwise(op, objs, dets):
    """modules/gcn.py:6-41."""
    if op == "multiply":
        return torch.einsum("bci,bcj->bcij", objs, dets)
    d = (objs.unsqueeze(-1) - dets.unsqueeze(-2)) / 2
    if op == "minus_abs":
        return d.abs()
    if op == "minus":
        return d
    raise ValueError(op)


def new_end(sd, x, mode="avg"):
    """modules/new_end.py:62-82 (NewEndIndicator_v2.forward)."""
    p = "w_link.w_new_end"
    y = F.conv2d(x, sd[f"{p}.conv0.0.weight"], sd[f"{p}.conv0.0.bias"])
    y = F.relu(group_norm(y, 1, sd[f"{p}.conv0.1.weight"], sd[f"{p}.conv0.1.bias"]))
    if mode == "avg":
        new_vec, end_vec = y.mean(dim=-2), y.mean(dim=-1)
    else:
        new_vec, end_vec = y.max(dim=-2)[0], y.max(dim=-1)[0]

    def mlp(v):
        v = F.conv1d(v, sd[f"{p}.conv1.0.weight"], sd[f"{p}.conv1.0.bias"])
        v = F.relu(group_norm(v, 1, sd[f"{p}.conv1.1.weight"], sd[f"{p}.conv1.1.bias"]))
        v = F.conv1d(v, sd[f"{p}.conv1.3.weight"], sd[f"{p}.conv1.3.bias"])
        v = F.relu(group_norm(v, 1, sd[f"{p}.conv1.4.weight"], sd[f"{p}.conv1.4.bias"]))
        v = F.conv1d(v, sd[f"{p}.conv1.6.weight"], sd[f"{p}.conv1.6.bias"])
        return torch.sigmoid(v).squeeze(1)
    return mlp(new_vec), mlp(end_vec)


def affinity(sd, x):
    """modules/gcn.py:59-66 (conv1 stack), applied at :80."""
    p = "w_link.conv1"
    for i, n in ((0, 1), (3, 4), (6, 7)):
        x = F.conv2d(x, sd[f"{p}.{i}.weight"], sd[f"{p}.{i}.bias"])
        x = F.relu(group_norm(x, x.shape[1], sd[f"{p}.{n}.weight"], sd[f"{p}.{n}.bias"]))
    return F.conv2d(x, sd[f"{p}.9.weight"], sd[f"{p}.9.bias"])


def associate(sd, objs, dets, affinity_op, softmax_mode, end_mode="avg"):
    """modules/gcn.py:68-82 then modules/tracking_net.py:106-126."""
    x = pairwise(affinity_op, objs, dets)
    new_score, end_score = new_end(sd, x, end_mode)
    link = affinity(sd, x)
    if softmax_mode == "single":
        link = F.softmax(link, dim=-1)
    elif softmax_mode == "dual":
        link = F.softmax(link, dim=-1) * F.softmax(link, dim=-2)
    elif softmax_mode == "dual_add":
        link = (F.softmax(link, dim=-1) + F.softmax(link, dim=-2)) / 2
    elif softmax_mode == "dual_max":
        link = torch.max(F.softmax(link, dim=-1), F.softmax(link, dim=-2))
    return link, new_score, end_score


def features(sd, dets, det_info, fusion_arch):
    """modules/tracking_net.py:128-147."""
    app = appearance(sd, dets)
    pts, trans = pointnet(sd, det_info["points"].transpose(-1, -2),
                          det_info["points_split"].long().squeeze(0))
    feats = torch.cat([app, pts], dim=-1).t().unsqueeze(0)
    return fusion(sd, fusion_arch, feats), trans, app, pts


@torch.no_grad()
def forward(sd, dets, det_info, dets_split, fusion_arch="C", affinity_op="multiply",
            softmax_mode="single", neg_threshold=0.0, end_mode="avg", return_stages=False):
    """modules/tracking_net.py:165-193 in eval mode.  Returns the reference's 5-tuple
    (det_scores 3xL, [link 3xNxM], new 3xL, end 3xL, trans)."""
    feats, trans, app, pts = features(sd, dets, det_info, fusion_arch)
    det_scores = determine_det(sd, feats, neg_threshold)
    start, links, news, ends = 0, [], [], []
    for i in range(len(dets_split) - 1):
        prev_end = start + int(dets_split[i])
        end = prev_end + int(dets_split[i + 1])
        link, new_s, end_s = associate(sd, feats[:, :, start:prev_end], feats[:, :, prev_end:end],
                                       affinity_op, softmax_mode, end_mode)
        links.append(link.squeeze(1))
        news.append(new_s)
        ends.append(end_s)
        start = prev_end
    fake_new = det_scores.new_zeros((det_scores.size(0), links[0].size(-2)))
    fake_end = det_scores.new_zeros((det_scores.size(0), links[-1].size(-1)))
    new_scores = torch.cat([fake_new] + news, dim=1)
    end_scores = torch.cat(ends + [fake_end], dim=1)
    if return_stages:
        return (det_scores, links, new_scores, end_scores, trans), {
            "appear": app, "points": pts, "feats": feats}
    return det_scores, links, new_scores, end_scores, trans
