"""Host-side pipelining of the association path (new relative to the reference, whose eval loop copies one sample at a
time and synchronises 2+2L times per pair, SURVEY F12).

``HostPipeline`` owns a copy stream, device staging buffers and pinned result buffers.  ``run`` takes a batch of
frame-pairs that lives in (pinned) HOST memory, cuts it into sub-batches and overlaps the host->device copy of
sub-batch i+1 with ``TrackingNet.predict_batch`` of sub-batch i; the assignment results (and the library's range flag)
come back device->host asynchronously.  One host synchronisation per batch.  This is what ``bench.py`` times as ``e2e``.
The same holds for windows of K > 2 frames (``counts``), whose programmes ``predict_batch`` solves as min-cost flows.
"""
import torch

from . import _lib


class HostPipeline:

    def __init__(self, net, n=None, m=None, sub_batches=4, counts=None):
        """n, m: frame-pairs of n and m (default n) detections; counts (n_0, ..., n_{K-1}) in their place: windows of
        K frames with these detection counts (``TrackingNet.predict_batch``'s ``counts``)."""
        self.net = net
        self.counts = net._frame_counts(n, m, counts)
        self.frames = dict(counts=self.counts) if counts is not None else dict(n=self.counts[0], m=self.counts[1])
        self.L = sum(self.counts)
        self.sub = max(1, int(sub_batches))
        self.dev = next(net.parameters()).device
        if self.dev.type != "cuda":
            raise _lib.MmmotError("HostPipeline needs the module on a CUDA device")
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self._shape = None

    def _prepare(self, h_crops, h_points, pairs):
        key = (tuple(h_crops.shape), tuple(h_points.shape), pairs)
        if self._shape == key:
            return
        L, cols = self.L, self.L - self.counts[-1]      # match: one column per detection with a next frame
        nsub = self.sub if pairs % self.sub == 0 and pairs >= 2 * self.sub else 1
        self.nsub, self.sb = nsub, pairs // nsub
        self.d_crops = torch.empty(h_crops.shape, dtype=torch.float32, device=self.dev)
        self.d_points = torch.empty(h_points.shape, dtype=torch.float32, device=self.dev)
        self.d_match = torch.empty(pairs, cols, dtype=torch.int32, device=self.dev)       # whole-batch result on the device
        self.h_match = torch.empty(pairs, cols, dtype=torch.int32, pin_memory=True)
        self.h_flags = torch.empty(3, pairs, L, dtype=torch.float32, pin_memory=True)       # assign_det | new | end
        self.h_status = torch.zeros(nsub, dtype=torch.int32, pin_memory=True)
        self.ev_copied = [torch.cuda.Event() for _ in range(nsub)]
        self.ev_used = [torch.cuda.Event() for _ in range(nsub)]
        cur = torch.cuda.current_stream(self.dev)
        for e in self.ev_used:
            e.record(cur)
        self._shape = key

    def run(self, h_crops, h_points, points_split, sync=True):
        """h_crops (B*L) x 3 x H x W, h_points P x C (C the net's point width, else MmmotError): pinned host tensors;
        points_split (B*L + 1,) CPU int CSR offsets.
        Returns {"match": B x n int32, "assign_det" / "assign_new" / "assign_end": B x L} as pinned host tensors (valid
        after the synchronisation this call performs unless sync=False) and "match_device", the same B x n matches on the
        device (for a gather across ranks).  For K-frame windows match is B x (L - n_{K-1}), predict_batch's layout.
        Raises MmmotError (MMMOT_E_RANGE) if the library flagged an FP16 range overflow."""
        L = self.L
        self.net._check_points(h_points)
        pairs = h_crops.shape[0] // L
        self._prepare(h_crops, h_points, pairs)
        split = points_split.detach().to("cpu", torch.int64)
        cur = torch.cuda.current_stream(self.dev)
        sb, bounds = self.sb, []
        for i in range(self.nsub):
            c0, c1 = i * sb * L, (i + 1) * sb * L
            p0, p1 = int(split[c0]), int(split[c1])
            bounds.append((c0, c1, p0, p1))
            with torch.cuda.stream(self.copy_stream):
                self.copy_stream.wait_event(self.ev_used[i])         # the previous batch finished reading this slice
                self.d_crops[c0:c1].copy_(h_crops[c0:c1], non_blocking=True)
                self.d_points[p0:p1].copy_(h_points[p0:p1], non_blocking=True)
                self.ev_copied[i].record(self.copy_stream)
        out = None
        for i, (c0, c1, p0, p1) in enumerate(bounds):
            cur.wait_event(self.ev_copied[i])
            out = self.net.predict_batch(self.d_crops[c0:c1], self.d_points[p0:p1], split[c0:c1 + 1] - p0, check=False,
                                         **self.frames)
            self.ev_used[i].record(cur)
            q0, q1 = i * sb, (i + 1) * sb
            self.d_match[q0:q1].copy_(out["match"])
            self.h_match[q0:q1].copy_(out["match"], non_blocking=True)
            self.h_flags[0, q0:q1].copy_(out["assign_det"], non_blocking=True)
            self.h_flags[1, q0:q1].copy_(out["assign_new"], non_blocking=True)
            self.h_flags[2, q0:q1].copy_(out["assign_end"], non_blocking=True)
            self.h_status[i:i + 1].copy_(out["status"], non_blocking=True)    # the range flag travels with the results
        res = {"match": self.h_match, "assign_det": self.h_flags[0], "assign_new": self.h_flags[1],
               "assign_end": self.h_flags[2], "match_device": self.d_match}
        if sync:
            cur.synchronize()
            self.net._raise_on_status(int(self.h_status.max()))
        return res

    def bytes_per_batch(self, h_crops, h_points, points_split):
        """(host->device, device->host) bytes one ``run`` moves."""
        return (h_crops.numel() * 4 + h_points.numel() * 4 + points_split.numel() * 4,
                self.h_match.numel() * 4 + self.h_flags.numel() * 4 + self.h_status.numel() * 4)
