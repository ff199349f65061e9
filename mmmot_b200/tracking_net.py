"""Drop-in ``TrackingNet`` — the reference's Python boundary for the association forward.

Mirrors reference modules/tracking_net.py:15-193: same constructor keywords (:17-35), same
``forward(dets, det_info, dets_split)`` signature and 5-tuple return (:165-193), same
``state_dict`` key names (schema.py), ``.test_mode`` / ``.eval()`` / ``.cuda()`` behaviour — so it
can be handed to the reference's ``TrackingModule`` / ``eval_seq.py`` unchanged.  All arithmetic
runs in libmmmot_sm90a.so through the C ABI (``_lib.py``); torch is used for device memory,
streams and the parameter container only.  There is no CPU path: ``forward`` raises unless the
module lives on a CUDA device and the shared library loads.

New relative to the reference (which handles one frame-pair per call, SURVEY F12):
``forward_batch`` runs B independent frame-pairs in one pass with per-pair semantics identical
to ``forward``, and ``predict_batch`` also solves the association programme on the device.
"""
import ctypes

import torch
import torch.nn as nn

from . import _lib
from .schema import BUFFER_KINDS, VGG_POOL_AFTER, VGG_STAGES, state_schema

# conv k of the 13 is followed by a 2x2 max-pool (so the map of conv k+1 is 4x smaller)
VGG_POOLED_BEFORE = [idx in VGG_POOL_AFTER[s] for s, stage in enumerate(VGG_STAGES) for idx, _, _ in stage]
from .weights import DeviceWeights


def _vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _aligned_rows(points):
    """4-channel points are read as 16-byte rows (one float4 per point): a tensor that does not start on a 16-byte
    boundary (a view at an odd storage offset) is copied."""
    return points.clone() if points.shape[1] == 4 and points.data_ptr() % 16 else points


class _Holder(nn.Module):
    """Empty module used to build the reference's parameter tree (names only)."""


def _register(root, key, tensor, is_buffer):
    parts = key.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Holder())
        mod = mod._modules[p]
    if is_buffer:
        mod.register_buffer(parts[-1], tensor)
    else:
        mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=tensor.is_floating_point()))


def _default_init(shape, kind, gen):
    if kind == "conv":
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        return torch.randn(shape, generator=gen) * (2.0 / fan_in) ** 0.5
    if kind in ("norm_w", "run_var"):
        return torch.ones(shape)
    if kind == "eye":
        return torch.eye(shape[0])
    if kind == "nbt":
        return torch.zeros(shape, dtype=torch.int64)
    return torch.zeros(shape)          # biases, norm_b, run_mean, stn_out (reference point_net.py:69-70)


class TrackingNet(nn.Module):

    def __init__(self, seq_len, appear_len=512, appear_skippool=False, appear_fpn=False,
                 score_arch='vgg', score_fusion_arch='C', appear_arch='vgg', point_arch='v1',
                 point_len=512, softmax_mode='single', test_mode=0, affinity_op='multiply',
                 dropblock=5, end_arch='v2', end_mode='avg', without_reflectivity=True,
                 neg_threshold=0, use_dropout=False):
        super().__init__()
        # the value space of the shipped experiments/*/config.yaml (SURVEY §8b); anything else is
        # rejected loudly instead of silently computing something different
        unsupported = []
        if appear_len != 512 or point_len != 512: unsupported.append("appear_len/point_len != 512")
        if appear_arch != 'vgg' or not appear_skippool or appear_fpn: unsupported.append("appearance must be vgg + skippool")
        if point_arch != 'v1': unsupported.append("point_arch must be v1")
        if end_arch != 'v2' or end_mode not in _lib.END_MODE: unsupported.append("end_arch must be v2, end_mode avg or max")
        if score_arch not in ('branch_cls', 'branch_reg'): unsupported.append("score_arch must be branch_cls/branch_reg")
        if score_fusion_arch not in _lib.FUSION: unsupported.append(f"score_fusion_arch {score_fusion_arch!r}")
        if affinity_op not in _lib.AFFINITY: unsupported.append(f"affinity_op {affinity_op!r}")
        if unsupported:
            raise NotImplementedError("mmmot_b200.TrackingNet: " + "; ".join(unsupported))
        self.seq_len = seq_len
        self.score_arch = score_arch
        self.neg_threshold = neg_threshold
        self.test_mode = test_mode          # 0:image; 1:LiDAR; 2:fusion (tracking_net.py:40)
        self.softmax_mode = softmax_mode
        self.affinity_op = affinity_op
        self.end_mode = end_mode
        self.score_fusion_arch = score_fusion_arch
        # dropblock / use_dropout are identity in eval mode; accepted for config compatibility
        self.dropblock, self.use_dropout = dropblock, use_dropout
        # PointNet's input width (tracking_net.py:41): xyz, or xyz + LiDAR reflectance
        self.point_channels = 4 - int(bool(without_reflectivity))
        gen = torch.Generator().manual_seed(0)
        for key, (shape, kind) in state_schema(score_fusion_arch, self.point_channels).items():
            _register(self, key, _default_init(shape, kind, gen), kind in BUFFER_KINDS)
        for name, prm in self.named_parameters():
            if name.endswith(".idt"):           # reference point_net.py:62: requires_grad=False
                prm.requires_grad_(False)
        self._prepared = None
        self._ws = None
        self.chunk_pairs = None             # None: pick from free memory

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, *a, **k):
        self._prepared = None
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self._prepared = None
        self._ws = None
        return super()._apply(fn, *a, **k)

    def prepared(self):
        """Device-resident prepared weights (rebuilt after load_state_dict / .cuda() / .to())."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise _lib.MmmotError("mmmot_b200.TrackingNet runs on CUDA (sm_90a) only: call .cuda() first "
                                  "(there is no CPU fallback)")
        if self._prepared is None or self._prepared.flat.device != dev:
            _lib.load()
            self._prepared = DeviceWeights(self.state_dict(), self.score_fusion_arch, dev)
        return self._prepared

    def _split_to_device(self, s_host, dev):
        """CSR offsets host -> device without blocking the calling thread and without the copy engine: staged in a small
        ring of pinned buffers that a kernel reads over PCIe (mmmot_fetch_pinned_i32).  A pageable copy would make the
        host wait for everything already enqueued on the stream; a cudaMemcpyAsync from pinned memory queues on the
        copy engine behind the bulk input copies of a pipelined caller (HostPipeline) and stalls the compute stream for
        milliseconds per sub-batch (measured: 7 % of cfg4's e2e).  A slot is reused only after its fetch has executed."""
        n = s_host.numel()
        ring = getattr(self, "_pin_ring", None)
        if ring is None or ring[0][0].numel() < n:
            for old in ring or []:              # a fetch kernel may still be reading the old (smaller) pinned buffers
                if old[1] is not None:
                    old[1].synchronize()
            cap = max(n, 1024)
            ring = self._pin_ring = [[torch.empty(cap, dtype=torch.int32, pin_memory=True), None] for _ in range(4)]
            self._pin_next = 0
        slot = ring[self._pin_next]
        self._pin_next = (self._pin_next + 1) % len(ring)
        if slot[1] is not None:
            slot[1].synchronize()
        slot[0][:n].copy_(s_host)
        out = torch.empty(n, dtype=torch.int32, device=dev)
        cur = torch.cuda.current_stream(dev)
        _lib.check(_lib.load().mmmot_fetch_pinned_i32(ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(slot[0].data_ptr()), n,
                                                      ctypes.c_void_p(cur.cuda_stream)), "mmmot_fetch_pinned_i32")
        slot[1] = torch.cuda.Event()
        slot[1].record(cur)
        return out

    def _workspace(self, nbytes, dev):
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = None
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
        return self._ws

    # ------------------------------------------------------------------ core
    def _workspace_bytes(self, pairs, transitions, L=0, P=0, H=0, W=0):
        """Workspace of one call on `pairs` samples: the affinity stage on every (n, m) of `transitions` and, when L > 0,
        the feature stages on L detections, P points and H x W crops (their training variants in training mode)."""
        lib = _lib.load()
        need = [lib.mmmot_affinity_workspace(pairs, n, m) for n, m in transitions]
        if L:
            if self.training:
                need += [lib.mmmot_appearance_train_workspace(pairs * L, H, W), lib.mmmot_pointnet_train_workspace(pairs, L, P),
                         lib.mmmot_w_det_train_workspace(L)]
            else:
                need += [lib.mmmot_appearance_workspace(pairs * L, H, W), lib.mmmot_pointnet_workspace(pairs, L, P)]
            need.append(lib.mmmot_fusion_det_workspace(pairs, L))
        return max(need)

    def _features(self, wts, ws, st, crops, points, split, pairs, L, feats, det):
        """Appearance, PointNet and fusion / detection score of `pairs` samples of L detections on stream `st`:
        feats pairs x 3 x 512 x L, det pairs x 3 x L.  split: the CSR point offsets, CPU int32.

        In training mode (reference TrackingNet.forward with self.training, modules/tracking_net.py:152-162) the
        BatchNorm layers (VGG trunk, w_det) normalise with the statistics of this call and det scores are raw logits
        without the neg_threshold step; DropBlock (the two deepest SkipPool heads) and the PointNet head's Dropout
        (rrc_pfv config: dropblock 5, use_dropout True) draw their masks from torch's generators exactly as the
        reference does (_dropblock_weights / _dropout_mask) and the library applies them.  Returns the batch statistics
        (bn_vgg 13 x 2 x 512, bn_det 2 x 2 x 512) in training mode, else None."""
        lib = _lib.load()
        dev = feats.device
        H, W = crops.shape[-2:]
        wsp, wsn = _vp(ws), ctypes.c_size_t(ws.numel())
        train = self.training
        if train:
            # random masks, in the reference's draw order: appearance heads 2 and 3 (CPU generator), then the PointNet head
            dm2 = dm3 = hmask = None
            if self.dropblock:
                dm2 = self._dropblock_weights(L, H // 16, W // 16, int(self.dropblock)).to(dev)
                dm3 = self._dropblock_weights(L, H // 32, W // 32, int(self.dropblock)).to(dev)
            if self.use_dropout:
                hmask = self._dropout_mask((512, int(split[-1])), dev).contiguous()
            bn_vgg = torch.zeros(13, 2, 512, device=dev)
            bn_det = torch.zeros(2, 2, 512, device=dev)
            _lib.check(lib.mmmot_appearance_train_fwd(wts.ptr, _vp(crops), pairs * L, H, W, L, _vp(feats), _vp(bn_vgg), _vp(dm2),
                                                      _vp(dm3), wsp, wsn, st), "mmmot_appearance_train_fwd")
        else:
            _lib.check(lib.mmmot_appearance_fwd(wts.ptr, _vp(crops), pairs * L, H, W, L, _vp(feats), wsp, wsn, st),
                       "mmmot_appearance_fwd")
        split_dev = self._split_to_device(split, dev)
        hs = ctypes.c_void_p(split.numpy().ctypes.data)
        if train:
            _lib.check(lib.mmmot_pointnet_train_fwd(wts.ptr, _vp(points), _vp(split_dev), hs, pairs, L, _vp(hmask), _vp(feats),
                                                    wsp, wsn, st), "mmmot_pointnet_train_fwd")
        else:
            _lib.check(lib.mmmot_pointnet_fwd(wts.ptr, _vp(points), _vp(split_dev), hs, pairs, L, _vp(feats), wsp, wsn, st),
                       "mmmot_pointnet_fwd")
        flags, thr = (0, 0.0) if train else (self._score_flags(), float(self.neg_threshold))
        _lib.check(lib.mmmot_fusion_det_fwd(wts.ptr, _lib.FUSION[self.score_fusion_arch], flags, thr, pairs, L, _vp(feats),
                                            _vp(det), wsp, wsn, st), "mmmot_fusion_det_fwd")
        if not train:
            return None
        _lib.check(lib.mmmot_w_det_train_fwd(wts.ptr, L, _vp(feats), _vp(det), _vp(bn_det), wsp, wsn, st), "mmmot_w_det_train_fwd")
        return bn_vgg, bn_det

    def _associate(self, wts, ws, st, pairs, n, m, feats, link, new, end):
        """Affinity / start-end / softmax stage on stream `st`: feats pairs x 3 x 512 x (n+m), contiguous ->
        link pairs x 3 x n x m, new pairs x 3 x m, end pairs x 3 x n."""
        _lib.check(_lib.load().mmmot_affinity_fwd(wts.ptr, _lib.AFFINITY[self.affinity_op], _lib.SOFTMAX.get(self.softmax_mode, 0),
                                                  _lib.END_MODE[self.end_mode], pairs, n, m, _vp(feats), _vp(link), _vp(new),
                                                  _vp(end), _vp(ws), ctypes.c_size_t(ws.numel()), st), "mmmot_affinity_fwd")

    def _score_flags(self):
        """reference tracking_net.py:153-162: sigmoid only when 'cls' is in score_arch; the neg_threshold step is
        the eval branch."""
        return (_lib.SCORE_SIGMOID if "cls" in self.score_arch else 0) | _lib.SCORE_THRESHOLD

    def _check_points(self, points):
        """points [P][C] with C the net's point width (point_channels); raises MmmotError otherwise.  Any other width
        would be read as rows of C floats and silently regrouped."""
        if points.dim() != 2 or points.shape[1] != self.point_channels:
            raise _lib.MmmotError(f"points must be [P][{self.point_channels}] for this net "
                                  f"(without_reflectivity={self.point_channels == 3}), got {list(points.shape)}")

    @staticmethod
    def _raise_on_status(status):
        """`status`: the int32 word forward_batch returns (device tensor or int)."""
        if int(status) & 1:
            _lib.check(-4, "mmmot_b200.TrackingNet forward")

    def _pick_chunk(self, B, n, m, P_per_pair, H, W, dev):
        if self.chunk_pairs:
            return min(B, self.chunk_pairs)
        free, _ = torch.cuda.mem_get_info(dev)
        budget = min(free * 0.5, 48e9)
        c = B
        while c > 1 and self._workspace_bytes(c, [(n, m)], n + m, int(P_per_pair * c) + 1, H, W) > budget:
            c = (c + 1) // 2
        return c

    @torch.no_grad()
    def forward_batch(self, crops, points, points_split, n, m=None, keep_feats=False, check=True):
        """B independent frame-pairs, each with n previous and m next detections.

        crops         (B*(n+m)) x 3 x H x W  fp32, CUDA
        points        P_total x C            fp32, CUDA (detections concatenated in order); C = point_channels:
                                             xyz, or xyz + reflectance (without_reflectivity=False)
        points_split  (B*(n+m) + 1,) int     CSR offsets, CPU tensor (the reference reads it with
                                             .item() per detection: modules/point_net.py:33-35)
        returns dict: det B x 3 x L, link B x 3 x n x m, new B x 3 x m, end B x 3 x n (un-padded),
                      trans [1xCxC, 1x64x64]; per-pair semantics identical to ``forward``; "status": the library's
                      status word (int32 device tensor; bit 0 = an activation left FP16's range, MMMOT_E_RANGE).
        check=True (default) reads the status word back (one host sync) and raises MmmotError when it is set;
        pipelined callers pass check=False and test ``out["status"]`` together with the results they copy back.
        """
        if self.training:
            raise NotImplementedError("mmmot_b200.TrackingNet implements the eval-mode forward only (SURVEY §8f N4)")
        m = n if m is None else m
        L = n + m
        self._check_points(points)
        lib = _lib.load()
        wts = self.prepared()
        dev = wts.flat.device
        if crops.device != dev or points.device != dev:
            raise _lib.MmmotError("inputs must live on the module's CUDA device")
        crops = crops.contiguous().float()
        points = _aligned_rows(points.contiguous().float())
        split = points_split.detach().to("cpu", torch.int32).contiguous()
        if crops.shape[0] % L or split.numel() != crops.shape[0] + 1:
            raise _lib.MmmotError("crops / points_split do not match n, m")
        B = crops.shape[0] // L
        H, W = crops.shape[-2:]
        out = {
            "status": torch.zeros(1, dtype=torch.int32, device=dev),
            "feats": torch.empty(B, 3, 512, L, device=dev),
            "det": torch.empty(B, 3, L, device=dev),
            "link": torch.empty(B, 3, n, m, device=dev),
            "new": torch.empty(B, 3, m, device=dev),
            "end": torch.empty(B, 3, n, device=dev),
        }
        with torch.cuda.device(dev):        # the library works on the CURRENT device
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            chunk = self._pick_chunk(B, n, m, int(split[-1]) / B, H, W, dev)
            for p0 in range(0, B, chunk):
                pc = min(chunk, B - p0)
                s_host = split[p0 * L:(p0 + pc) * L + 1]
                off = int(s_host[0])
                s_host = (s_host - off).contiguous()
                P = int(s_host[-1])
                ws = self._workspace(self._workspace_bytes(pc, [(n, m)], L, P, H, W), dev)
                _lib.check(lib.mmmot_status_reset(_vp(ws), st), "mmmot_status_reset")
                feats = out["feats"][p0:p0 + pc]
                self._features(wts, ws, st, crops[p0 * L:(p0 + pc) * L], points[off:off + P], s_host, pc, L, feats,
                               out["det"][p0:p0 + pc])
                self._associate(wts, ws, st, pc, n, m, feats, out["link"][p0:p0 + pc], out["new"][p0:p0 + pc],
                                out["end"][p0:p0 + pc])
                # the status word (FP16 range flag) of this chunk, accumulated into out["status"] in stream order
                out["status"] |= ws[:4].view(torch.int32)
        out["trans"] = [wts.trans1.unsqueeze(0).clone(), wts.trans2.unsqueeze(0).clone()]
        if not keep_feats:
            del out["feats"]
        if check:
            self._raise_on_status(out["status"])
        return out

    @torch.no_grad()
    def associate_batch(self, feats, n, m=None):
        """Affinity / start-end / softmax stage alone (reference TrackingNet.associate on every
        stack): feats B x 3 x 512 x (n+m) CUDA -> (link B x 3 x n x m, new B x 3 x m, end B x 3 x n)."""
        m = n if m is None else m
        lib = _lib.load()
        wts = self.prepared()
        dev = wts.flat.device
        feats = feats.contiguous().float()
        B = feats.shape[0]
        assert feats.shape[1:] == (3, 512, n + m) and feats.device == dev
        link = torch.empty(B, 3, n, m, device=dev)
        new = torch.empty(B, 3, m, device=dev)
        end = torch.empty(B, 3, n, device=dev)
        with torch.cuda.device(dev):
            ws = self._workspace(self._workspace_bytes(B, [(n, m)]), dev)
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(lib.mmmot_status_reset(_vp(ws), st), "mmmot_status_reset")
            self._associate(wts, ws, st, B, n, m, feats, link, new, end)
            _lib.check(lib.mmmot_status_check(_vp(ws), st), "mmmot_affinity_fwd")
        return link, new, end

    @torch.no_grad()
    def predict_batch(self, crops, points, points_split, n, m=None, check=True):
        """forward_batch + association programme on the ``test_mode`` stack, all on the device.
        Returns forward_batch's dict plus assign_{det,link,new,end} and match (B x n int32)."""
        from .solvers import solve_batch
        m = n if m is None else m
        out = self.forward_batch(crops, points, points_split, n, m, check=check)
        B, t = out["det"].shape[0], self.test_mode
        zn = out["det"].new_zeros(B, 3, n)
        zm = out["det"].new_zeros(B, 3, m)
        new_p = torch.cat([zn, out["new"]], dim=2)      # tracking_net.py:183-189 zero padding
        end_p = torch.cat([out["end"], zm], dim=2)
        out.update(solve_batch(out["det"][:, t], out["link"][:, t], new_p[:, t], end_p[:, t], n, m))
        return out

    # ------------------------------------------------------------------ training-mode forward (SURVEY §8f N4)
    # (name in state_dict of the BatchNorm, number of channels) in the order of the bn_stats rows the library returns
    _VGG_BN = [f"appearance.layers.{s}.{idx + 1}" for s, stage in enumerate(VGG_STAGES) for idx, _, _ in stage]

    def _update_running(self, prefix, mean, var_biased, count, momentum=0.1):
        """torch.nn.BatchNorm semantics in .train(): running = (1 - m) * running + m * batch, with the UNBIASED batch
        variance; num_batches_tracked += 1."""
        mod = self
        for part in prefix.split("."):
            mod = mod._modules[part]
        unbiased = var_biased * (count / max(count - 1.0, 1.0))
        mod.running_mean.mul_(1 - momentum).add_(mean, alpha=momentum)
        mod.running_var.mul_(1 - momentum).add_(unbiased, alpha=momentum)
        mod.num_batches_tracked += 1

    @staticmethod
    def _dropblock_weights(n_img, h, w, block_size, drop_prob=0.1):
        """DropBlock2D (reference modules/dropblock.py:28-67): Bernoulli(gamma) seeds from torch's CPU generator (the
        reference calls torch.rand without a device and moves the mask afterwards), grown to block_size x block_size
        blocks by a max-pool, inverted, scaled by numel / sum.  Returns the per-pixel weights n_img x h x w (CPU)."""
        gamma = drop_prob / (block_size ** 2)
        seeds = (torch.rand(n_img, h, w) < gamma).float()
        grown = torch.nn.functional.max_pool2d(seeds[:, None], kernel_size=(block_size, block_size), stride=(1, 1),
                                               padding=block_size // 2)
        if block_size % 2 == 0:
            grown = grown[:, :, :-1, :-1]
        keep = 1 - grown.squeeze(1)
        return (keep * (keep.numel() / keep.sum())).contiguous()

    @staticmethod
    def _dropout_mask(shape, dev, p=0.5):
        """nn.Dropout(p) of the PointNet head (reference modules/point_net.py:23,29-30) as a multiplicative mask with
        values {0, 1/(1-p)}, drawn by torch's own dropout on the activation's device, i.e. from the generator the
        reference consumes for a tensor of this shape."""
        return torch.nn.functional.dropout(torch.ones(shape, device=dev), p=p, training=True)

    # ------------------------------------------------------------------ the reference's forward
    @torch.no_grad()
    def forward(self, dets, det_info, dets_split):
        """Reference signature (modules/tracking_net.py:165-193): one sample of K >= 2 frames.

        dets L x 3 x H x W; det_info['points'] 1 x P x C' (C' >= C, the net's point width: the first C columns are
        used, as the reference's loader keeps x, y, z and, with without_reflectivity=False, r); det_info['points_split']
        1 x (L+1) float;
        dets_split: K shape-(1,) int tensors, the detections of each frame.  The feature stages run once over all L
        detections of the sample (one GroupNorm domain, exactly like the reference), then the affinity stage on every
        pair of consecutive frames (mmmot_b200.ortools_solve solves the association programme of K > 2 frames as a
        min-cost flow).  Returns (det_scores 3xL, [link_scores 3 x n_k x n_k+1 per pair of frames], new_scores 3xL,
        end_scores 3xL, trans).

        In training mode (two-frame samples only) the reference's training branch is returned instead
        (tracking_net.py:183-192; see _features): raw det logits, new_scores 3 x m and end_scores 3 x n not zero-padded,
        and the BatchNorm layers' running averages are updated.  Forward only: no autograd graph is built through the
        CUDA library."""
        splits = [int(s) for s in dets_split]
        if self.training and len(splits) != 2:
            raise NotImplementedError("mmmot_b200.TrackingNet supports 2-frame samples (sample_max_len: 2)")
        L = sum(splits)
        C = self.point_channels
        raw = det_info['points']
        if raw.dim() < 2 or raw.shape[-1] < C:
            raise _lib.MmmotError(f"det_info['points'] must carry at least {C} columns per point for this net "
                                  f"(without_reflectivity={C == 3}), got {list(raw.shape)}")
        lib = _lib.load()
        if self.training:
            self._prepared = None                  # parameters move under an optimizer: re-derive the operands every step
        wts = self.prepared()
        dev = wts.flat.device
        crops = dets.contiguous().float()
        points = _aligned_rows(raw.reshape(-1, raw.shape[-1])[:, :C].contiguous().float())
        split = det_info['points_split'].reshape(-1).detach().to("cpu", torch.int32).contiguous()
        if (crops.device != dev or points.device != dev or crops.shape[0] != L or split.numel() != L + 1
                or len(splits) < 2 or min(splits) <= 0):
            raise _lib.MmmotError("inputs do not match the module's device / dets_split")
        H, W = crops.shape[-2:]
        transitions = list(zip(splits[:-1], splits[1:]))
        feats = torch.empty(1, 3, 512, L, device=dev)
        det = torch.empty(1, 3, L, device=dev)
        links, news, ends = [], [], []
        with torch.cuda.device(dev):
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            ws = self._workspace(self._workspace_bytes(1, transitions, L, int(split[-1]), H, W), dev)
            _lib.check(lib.mmmot_status_reset(_vp(ws), st), "mmmot_status_reset")
            bn = self._features(wts, ws, st, crops, points, split, 1, L, feats, det)
            start = 0
            for a, b in transitions:
                link = torch.empty(1, 3, a, b, device=dev)
                new = torch.empty(1, 3, b, device=dev)
                end = torch.empty(1, 3, a, device=dev)
                self._associate(wts, ws, st, 1, a, b, feats[:, :, :, start:start + a + b].contiguous(), link, new, end)
                links.append(link[0]); news.append(new[0]); ends.append(end[0])
                start += a
            _lib.check(lib.mmmot_status_check(_vp(ws), st),
                       "mmmot_b200.TrackingNet training forward" if self.training else "mmmot_b200.TrackingNet forward")
        trans = [wts.trans1.unsqueeze(0).clone(), wts.trans2.unsqueeze(0).clone()]
        if self.training:
            # running averages (reference: nn.BatchNorm2d / BatchNorm1d side effect of a training-mode forward)
            bn_vgg, bn_det = bn
            h, w_ = H, W
            for i, cout in enumerate(cout for stage in VGG_STAGES for _, _, cout in stage):
                self._update_running(self._VGG_BN[i], bn_vgg[i, 0, :cout], bn_vgg[i, 1, :cout], float(L * h * w_))
                if VGG_POOLED_BEFORE[i]:
                    h, w_ = h // 2, w_ // 2
            self._update_running("w_det.1", bn_det[0, 0, :512], bn_det[0, 1, :512], 3.0 * L)
            self._update_running("w_det.4", bn_det[1, 0, :256], bn_det[1, 1, :256], 3.0 * L)
            return det[0], links, news[0], ends[0], trans
        new_scores = torch.cat([det.new_zeros(3, splits[0])] + news, dim=1)        # tracking_net.py:183-189
        end_scores = torch.cat(ends + [det.new_zeros(3, splits[-1])], dim=1)
        return det[0], links, new_scores, end_scores, trans
