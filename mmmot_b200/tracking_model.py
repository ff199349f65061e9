"""Track-id assignment and stitching after the association programme (SURVEY.md §8f N3 — the step right
after the hot path), plus the KITTI result writer the evaluator reads.

Drop-in for the evaluation half of reference ``tracking_model.TrackingModule`` (tracking_model.py:8-46, 68-81
``predict``; :275-352 ``assign_det_id``; :109-272 ``align_id``) and ``utils.data_util.write_kitti_result``
(utils/data_util.py:41-128): same constructor, same attributes (``frames_id``, ``frames_det``, ``last_id``,
``used_id``, ``test_mode``), same return values, same text file.  The bookkeeping is host work on a few hundred
integers per frame and is written here as vectorised numpy/torch instead of nested Python loops; the network
forward and the assignment programme run on the GPU through ``mmmot_b200.TrackingNet`` / ``ortools_solve``.
Parity: tests/test_tracking_model.py replays goldens produced by the unmodified reference class.
"""
import os

import numpy as np
import torch

from .solvers import ortools_solve

_FIELDS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y")

LABEL = {"Car": 0, "Van": 1, "Truck": 2, "Pedestrian": 3, "Person": 4, "Cyclist": 5, "Tram": 6, "Misc": 7,
         "DontCare": -1}                                   # utils/data_util.py:14-24
LABEL_VERSE = {v: k for k, v in LABEL.items()}


def _flags(x):
    return np.asarray(x.detach().cpu() if isinstance(x, torch.Tensor) else x).reshape(-1) == 1


class TrackingModule(object):
    """Twin of the reference class: the evaluation side (predict / id stitching) and the forward half of the training
    ``step`` (training-mode forward, ground-truth generation, loss value; SURVEY §8f N4).  The CUDA library is forward
    only, so ``step`` returns the loss without calling backward / the optimizer."""

    def __init__(self, model, optimizer=None, criterion=None, det_type="3D"):
        self.model = model
        self.optimizer = optimizer
        self.criterion = criterion
        self.det_type = det_type
        self.test_mode = model[0].test_mode if isinstance(model, list) else model.test_mode
        self.clear_mem()

    def clear_mem(self):
        self.used_id = []
        self.last_id = 0
        self.frames_id = []
        self.frames_det = []
        self.track_feats = None

    def eval(self):
        for m in (self.model if isinstance(self.model, list) else [self.model]):
            m.eval()
        self.clear_mem()

    def train(self):
        for m in (self.model if isinstance(self.model, list) else [self.model]):
            m.train()
        self.clear_mem()

    # ------------------------------------------------------------------ training step (forward half)
    def step(self, det_img, det_info, det_id, det_cls, det_split):
        """tracking_model.py:50-66 up to the loss: training-mode forward -> generate_gt -> criterion.  The reference then
        calls loss.backward() and optimizer.step(); the CUDA library builds no autograd graph, so the loss VALUE is
        returned (a detached tensor) and the parameters are left untouched."""
        det_score, link_score, new_score, end_score, trans = self.model(det_img, det_info, det_split)
        gt_det, gt_link, gt_new, gt_end = self.generate_gt(det_score[0], det_cls, det_id, det_split)
        return self.criterion(det_split, gt_det, gt_link, gt_new, gt_end, det_score, link_score, new_score, end_score, trans)

    def generate_gt(self, det_score, det_cls, det_id, det_split):
        """tracking_model.py:294-351 without the per-detection Python loops: a detection is a positive when its class
        flag is 1; positives of consecutive frames with the same track id are linked (first match wins, as the
        reference's ``break``); a positive without successor ends, one without predecessor is new.  det_cls / det_id:
        per frame, tensors of shape 1 x n_i (the DataLoader layout)."""
        split = [int(s) for s in det_split]
        L = sum(split)
        dev, dt = det_score.device, det_score.dtype
        cls = [torch.as_tensor(c).reshape(-1).to(dev) == 1 for c in det_cls]
        ids = [torch.as_tensor(i).reshape(-1).to(dev) for i in det_id]
        gt_det = torch.cat(cls).to(dt)
        gt_new, gt_end, gt_link = torch.zeros(L, device=dev, dtype=dt), torch.zeros(L, device=dev, dtype=dt), []
        start = 0
        for i, n in enumerate(split):
            pos = cls[i]
            has_succ = torch.zeros(n, dtype=torch.bool, device=dev)
            if i + 1 < len(split):
                same = ids[i][:, None] == ids[i + 1][None, :]                    # any class on the next frame
                first = same & (same.cumsum(1) == 1)                             # the first match only
                link = (first & pos[:, None]).to(dt)
                gt_link.append(link.unsqueeze(0))
                has_succ = link.sum(1) > 0
            has_pred = torch.zeros(n, dtype=torch.bool, device=dev)
            if i > 0:
                has_pred = (ids[i][:, None] == ids[i - 1][None, :]).any(1)
            gt_end[start:start + n] = (pos & ~has_succ).to(dt)
            gt_new[start:start + n] = (pos & ~has_pred).to(dt)
            start += n
        return gt_det, gt_link, gt_new, gt_end

    # ------------------------------------------------------------------ predict
    @torch.no_grad()
    def predict(self, det_imgs, det_info, dets, det_split):
        """tracking_model.py:68-81: forward -> assignment programme on the ``test_mode`` stack -> ids.

        Samples of K > 2 frames pass every transition's link matrix to the programme.  (The reference passes only
        ``link_score[0]`` and fails there with a KeyError, solvers.py:91.)"""
        det_score, link_score, new_score, end_score, _ = self.model(det_imgs, det_info, det_split)
        t = self.test_mode
        if len(det_split) == 2:
            assign_det, assign_link, assign_new, assign_end = ortools_solve(
                det_score[t], [link_score[0][t:t + 1]], new_score[t], end_score[t], det_split)
        else:
            assign_det, assign_link, assign_new, assign_end = ortools_solve(
                det_score[t], [l[t:t + 1] for l in link_score], new_score[t], end_score[t], det_split)
        ids, boxes = self.assign_det_id(assign_det, assign_link, assign_new, assign_end, det_split, dets)
        return self.align_id(ids, boxes)

    # ------------------------------------------------------------------ per-sample ids
    def assign_det_id(self, assign_det, assign_link, assign_new, assign_end, det_split, dets):
        """Sample-local ids (0, 1, 2, ...) for the kept detections of every frame of the sample.

        Frame 0: kept detections are numbered in order.  Later frames: a kept detection flagged `new` takes the next
        free number, otherwise it inherits the number of the previous-frame detection its link column selects
        (tracking_model.py:275-352).  Returns (list of int arrays, list of per-frame detection dicts)."""
        keep_all, new_all = _flags(assign_det), _flags(assign_new)
        counts = [int(s.item()) if isinstance(s, torch.Tensor) else int(s) for s in det_split]
        next_id, start = 0, 0
        prev_local = None
        det_ids, dets_out = [], []
        for i, n in enumerate(counts):
            keep = keep_all[start:start + n]
            local = np.full(n, -1, np.int64)
            if i == 0:
                fresh = keep
            else:
                fresh = keep & new_all[start:start + n]
                linked = np.flatnonzero(keep & ~fresh)
                if linked.size:
                    link = np.asarray(assign_link[i - 1][0].detach().cpu() if isinstance(assign_link[i - 1], torch.Tensor)
                                      else assign_link[i - 1][0]) == 1          # [prev][cur]
                    col = link[:counts[i - 1], linked]
                    if not col.any(axis=0).all():
                        # the reference appends no id for such a detection and then trips its own
                        # `assert len(fake_id) == det_curr_num` (tracking_model.py:281): same exception type here
                        raise AssertionError("kept detection is neither new nor linked to the previous frame")
                    local[linked] = prev_local[col.argmax(axis=0)]               # first linked previous detection
            k = int(fresh.sum())
            local[fresh] = next_id + np.arange(k)
            next_id += k
            kept_idx = np.flatnonzero(keep)
            out = {}
            for f in _FIELDS:
                v = dets[i][f]
                out[f] = v[0][torch.from_numpy(kept_idx)] if kept_idx.size else torch.Tensor([])
                if kept_idx.size and out[f].dim() == 0:
                    out[f] = out[f].reshape(1)
            out["id"] = torch.from_numpy(local[kept_idx]).long() if kept_idx.size else torch.Tensor([])
            out["frame_idx"] = dets[i]["frame_idx"]
            det_ids.append(local[kept_idx])
            dets_out.append(out)
            prev_local = local
            start += n
        return det_ids, dets_out

    # ------------------------------------------------------------------ stitching across samples
    def _same_detection(self, a, b):
        """[na][nb] bool: exact equality of bbox (and location for 3-D detections), tracking_model.py:158-167."""
        eq = (a["bbox"][:, None, :] == b["bbox"][None, :, :]).all(-1)
        if self.det_type == "3D":
            eq &= (a["location"][:, None, :] == b["location"][None, :, :]).all(-1)
        return eq.numpy()

    def align_id(self, dets_ids, dets_out):
        """Map sample-local ids to sequence-global track ids (tracking_model.py:109-272).

        Three situations: the first sample of a sequence (ids kept), a sample that does not start on the last stored
        frame (ids shifted past ``last_id``), and the normal overlapping case — the sample's first frame IS the last
        stored frame: its detections are matched to the stored ones by exact box equality, matched ids carry over,
        everything else gets fresh ids; only the sample's later frames are appended.  Returns
        (ids per appended frame, detections per appended frame, frame_start)."""
        def top(ids_list):
            return max([int(np.max(x)) for x, d in zip(ids_list, dets_out) if d["id"].size(0)] + [0])

        if len(self.used_id) == 0:
            self.used_id += dets_ids
            self.frames_id += dets_ids
            self.frames_det += dets_out
            self.last_id = np.maximum(self.last_id, top(dets_ids))
            return dets_ids, dets_out, 0

        if self.frames_det[-1]["frame_idx"] != dets_out[0]["frame_idx"]:
            shift = self.last_id + 1
            moved = []
            for ids, d in zip(dets_ids, dets_out):
                if d["id"].size(0) == 0:
                    moved.append([])
                    continue
                moved.append(ids + shift)
                d["id"] += shift
            self.last_id = np.maximum(self.last_id, top(moved))
            self.frames_id += moved
            self.frames_det += dets_out
            return moved, dets_out, 0

        # overlapping sample
        mapping = {}
        first, stored = dets_out[0], self.frames_det[-1]
        if len(dets_ids[0]):
            if len(self.frames_id[-1]):
                eq = self._same_detection(first, stored)
                hit, where = eq.any(axis=1), eq.argmax(axis=1)
            else:
                hit = np.zeros(len(dets_ids[0]), bool)
                where = hit.astype(np.int64)
            for i, local in enumerate(dets_ids[0]):
                if hit[i]:
                    mapping[local] = self.frames_id[-1][where[i]]
                else:
                    self.last_id += 1
                    mapping[local] = self.last_id
            if len(set(mapping.values())) != len(mapping):
                print("ID pairs has duplicates!!!")
        aligned = []
        for i in range(1, len(dets_ids)):
            if dets_out[i]["id"].size(0) == 0:
                aligned.append([])
                continue
            new_id = dets_ids[i].copy()
            for j, local in enumerate(dets_ids[i]):
                if local not in mapping:
                    self.last_id += 1
                    mapping[local] = self.last_id
                new_id[j] = mapping[local]
            if len(set(new_id.tolist())) != len(new_id):
                raise AssertionError("duplicate track ids inside one frame")
            self.last_id = np.maximum(self.last_id, int(np.max(new_id)))
            aligned.append(new_id)
            dets_out[i]["id"] = torch.Tensor(new_id).long()
        kept = []
        if dets_out[1]["id"].size(0) != 0:       # the reference appends only when frame 1 kept something (:268-271)
            kept = dets_out[1:]
            self.frames_id += aligned
            self.frames_det += kept
        return aligned, kept, 1


# ---------------------------------------------------------------------- KITTI text
def kitti_result_line(result_dict, precision=4):
    """One line of a KITTI tracking result file (utils/data_util.py:41-86): frame id name truncated occluded alpha
    bbox(4) dimensions(3) location(3) rotation_y score; floats with `precision` decimals, `occluded` verbatim."""
    defaults = {"truncated": -1, "occluded": -1, "alpha": -10, "dimensions": [-1, -1, -1],
                "location": [-1000, -1000, -1000], "rotation_y": -10, "score": 0.0}
    order = ("frame", "id", "name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y",
             "score")
    for key in result_dict:
        if key not in order:
            raise ValueError("unknown key. supported key:{}".format(order))
    num = "{" + ":.{}f".format(precision) + "}"
    parts = []
    for key in order:
        val = result_dict.get(key)
        if val is None and key not in defaults:
            raise ValueError("you must specify a value for {}".format(key))
        if key in ("frame", "id"):
            parts.append(str(val))
        elif key == "name":
            parts.append(val)
        elif key == "occluded":
            parts.append(str(defaults[key]) if val is None else "{}".format(val))
        elif key in ("truncated", "alpha", "rotation_y", "score"):
            parts.append(str(defaults[key]) if val is None else num.format(val))
        else:
            parts += [str(v) for v in defaults[key]] if val is None else [num.format(v) for v in val]
    return " ".join(parts)


def write_kitti_result(root, seq_name, step, frames_id, frames_det, part="train"):
    """utils/data_util.py:89-128: one text line per kept detection of every stored frame, written to
    ``{root}/{step}/{part}/{seq_name}.txt``.  Like the reference this permutes each frame's ``dimensions`` in place
    (l h w -> h w l, the label-file order)."""
    assert len(frames_id) == len(frames_det)
    lines = []
    for ids, det in zip(frames_id, frames_det):
        n = det["id"].size(0)
        if n == 0:
            continue
        det["dimensions"] = det["dimensions"][:, [1, 2, 0]]
        frame = int(det["frame_idx"][0])
        for j in range(n):
            lines.append(kitti_result_line({
                "frame": frame, "id": ids[j], "name": LABEL_VERSE[det["name"][j].item()],
                "truncated": det["truncated"][j].item(), "occluded": det["occluded"][j].item(),
                "alpha": det["alpha"][j].item(), "bbox": det["bbox"][j].numpy(),
                "location": det["location"][j].numpy(), "dimensions": det["dimensions"][j].numpy(),
                "rotation_y": det["rotation_y"][j].item(), "score": 0.9}))
    path = f"{root}/{step}/{part}"
    os.makedirs(path, exist_ok=True)
    with open(f"{path}/{seq_name}.txt", "w") as f:
        f.write("\n".join(lines))
