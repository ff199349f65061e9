"""Appearance stage per crop: the ResNet-50/101/152 trunks with SkipPool heads (mmmot_appearance_resnet_fwd) and with the
FPN head (mmmot_appearance_resnet_fpn_fwd) against the VGG16-BN trunk (mmmot_appearance_fwd), heads included, at 64 x 64
and 224 x 224 crops, in auto engine mode (the tensor cores at these sizes).  Each figure is the median of 5 windows of >= 100 ms of back-to-back calls, from device events after
warm-up; achieved FLOP/s = the trunk's multiply-adds x 2 (computed from the conv shapes) over that time.  A second,
separate run with the per-launch timing hooks on gives the per-tag table.  Card name, power limit and SM clock are read
in the same run.  Prints one JSON line (also written to the path given as the first argument).
Run on a GPU box:  python tools/resnet_times.py [out.json]"""
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb                                               # noqa: E402
from mmmot_b200 import _lib                                           # noqa: E402
from mmmot_b200.schema import VGG_POOL_AFTER, VGG_STAGES, resnet_convs  # noqa: E402
from mmmot_b200.synthetic import synthetic_state_dict                 # noqa: E402

CONFIGS = (("vgg", "skippool"),) + tuple((a, h) for a in ("resnet50", "resnet101", "resnet152") for h in ("skippool", "fpn"))
SIZES = ((64, 256), (224, 32))          # (crop side, crops per call); L = 16 detections per pair


def macs_per_crop(arch, hw):
    """Multiply-adds of the trunk's convolutions for one hw x hw crop (heads and pools excluded)."""
    if arch == "vgg":
        tot, h = 0, hw
        for s, stage in enumerate(VGG_STAGES):
            for idx, cin, cout in stage:
                tot += 9 * cin * cout * h * h
                if idx in VGG_POOL_AFTER[s]:
                    h //= 2
        return tot
    tot, cur, out = 0, hw, hw // 4          # cur: the block input's side, out: its output's side
    for conv, _, cin, cout, k, stride in resnet_convs(arch):
        if conv.endswith("layers.conv1"):
            tot += k * k * cin * cout * (hw // 2) ** 2
            continue
        if conv.endswith(".conv1"):
            cur = out
            side = cur
        else:
            out = cur // stride if conv.endswith("conv2") else out
            side = out
        tot += k * k * cin * cout * side * side
    return tot


def fpn_lateral_macs_per_crop(hw):
    """Multiply-adds of the FPN head's four laterals (C_k -> 512 at hw / 2^(k+2)) for one hw x hw crop."""
    return sum((256 << k) * 512 * (hw >> (k + 2)) ** 2 for k in range(4))


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]


def main():
    assert torch.cuda.is_available(), "resnet_times needs a CUDA device"
    lib = _lib.load()
    out = {"card": smi("name"), "power_limit": smi("power.limit"), "sm_clock_max": smi("clocks.max.sm"), "rows": []}
    L = 16
    for arch, head in CONFIGS:
        fpn = head == "fpn"
        net = mb.TrackingNet(2, appear_skippool=not fpn, appear_fpn=fpn, appear_arch=arch, score_arch="branch_cls",
                             dropblock=0)
        net.load_state_dict(synthetic_state_dict("C", seed=1, appear_arch=arch, appear_head=head))
        net.cuda().eval()
        wts = net.prepared()
        for hw, n in SIZES:
            g = torch.Generator(device="cuda").manual_seed(hw)
            crops = torch.randn(n, 3, hw, hw, device="cuda", generator=g)
            feats = torch.empty(n // L, 3, 512, L, device="cuda")
            if arch == "vgg":
                nbytes = lib.mmmot_appearance_workspace(n, hw, hw)
            elif fpn:
                nbytes = lib.mmmot_appearance_resnet_fpn_workspace(n, hw, hw, L)
            else:
                nbytes = lib.mmmot_appearance_resnet_workspace(n, hw, hw)
            ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            a = [ctypes.c_void_p(t.data_ptr()) for t in (crops, feats, ws)]

            def call():
                if arch == "vgg":
                    rc = lib.mmmot_appearance_fwd(wts.ptr, a[0], n, hw, hw, L, a[1], a[2], nbytes, None)
                elif fpn:
                    rc = lib.mmmot_appearance_resnet_fpn_fwd(wts.rptr, wts.fptr, a[0], n, hw, hw, L, a[1], a[2], nbytes, None)
                else:
                    rc = lib.mmmot_appearance_resnet_fwd(wts.ptr, wts.rptr, a[0], n, hw, hw, L, a[1], a[2], nbytes, None)
                assert rc == 0, rc
            assert lib.mmmot_status_reset(a[2], None) == 0
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            reps = max(3, int(120.0 / max(e0.elapsed_time(e1), 1e-3)) + 1)
            wins = []
            for _ in range(5):
                e0.record()
                for _ in range(reps):
                    call()
                e1.record()
                torch.cuda.synchronize()
                wins.append(e0.elapsed_time(e1))
            assert lib.mmmot_status_check(a[2], None) == 0
            ms = sorted(wins)[2] / reps
            assert sorted(wins)[0] >= 100.0, wins
            macs = macs_per_crop(arch, hw)
            # per-launch tags, in a run of their own
            lib.mmmot_timing_collect_tags(None, None, None, None)
            lib.mmmot_timing_enable(1)
            call()
            lib.mmmot_timing_enable(0)
            k = lib.mmmot_timing_tag_count()
            tms, tfl = (ctypes.c_double * k)(), (ctypes.c_double * k)()
            cnt = (ctypes.c_long * k)()
            assert lib.mmmot_timing_collect_tags(tms, tfl, None, cnt) == 0
            tags = {lib.mmmot_timing_tag_name(t).decode(): {
                "ms_per_crop": round(tms[t] / n, 5), "launches": cnt[t],
                "tflops": round(tfl[t] / (tms[t] * 1e9), 1) if tfl[t] and tms[t] else None} for t in range(k) if cnt[t]}
            row = {"arch": arch, "head": head, "hw": hw, "crops_per_call": n, "window_ms": round(sorted(wins)[2], 1), "calls": reps,
                   "ms_per_crop": round(ms / n, 5), "gmacs_per_crop": round(macs / 1e9, 3),
                   "tflops": round(2.0 * macs * n / (ms * 1e9), 1), "tags": tags}
            if fpn:
                row["fpn_lateral_gmacs_per_crop"] = round(fpn_lateral_macs_per_crop(hw) / 1e9, 4)
            out["rows"].append(row)
            print(arch, head, hw, row["ms_per_crop"], "ms/crop", row["tflops"], "TFLOP/s", file=sys.stderr)
        del net, wts
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
