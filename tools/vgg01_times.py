"""The first VGG block at cfg4 (64 x 64 crops, 32,768 per 128-pair step): the fused launch (csrc/vgg_conv01.cuh) against
the two launches it replaces (debug bit 15), alternating, in one process.

Each round times, for each path, a window of back-to-back mmmot_appearance_fwd calls on 8,192 crops (L = 256; four calls
per step) with device events, then one call with the per-launch timing hooks on (the per-tag table).  Rounds repeat
ROUNDS times; medians are reported per step.  The card name, power limit and the median SM clock sampled during the
timed windows are read in the same run.  The outputs are compared byte for byte: the pooled conv-1 planes of the block
(mmmot_debug_vgg_conv01, which runs it as the forward does) and the appearance features of the whole trunk.
Prints one JSON line (also written to the path given as the first argument).
Run on a GPU box:  python tools/vgg01_times.py [out.json]"""
import ctypes
import json
import os
import statistics
import subprocess
import sys
import threading

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mmmot_b200 as mb                                   # noqa: E402
from mmmot_b200 import _lib                               # noqa: E402
from mmmot_b200.synthetic import synthetic_state_dict     # noqa: E402

HW, N, L, STEP_CROPS, ROUNDS = 64, 8192, 256, 32768, 3
TWO_LAUNCH = 1 << 15
PATHS = (("fused", 0), ("two_launch", TWO_LAUNCH))


def smi(fields):
    return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]


class ClockSampler:
    """SM clock (MHz) sampled every 0.2 s while active."""
    def __init__(self):
        self.samples, self.on, self.stop = [], threading.Event(), threading.Event()
        self.t = threading.Thread(target=self.run, daemon=True)
        self.t.start()

    def run(self):
        while not self.stop.is_set():
            if self.on.is_set():
                try:
                    self.samples.append(float(smi("clocks.sm")))
                except (ValueError, IndexError):
                    pass
            self.stop.wait(0.2)

    def close(self):
        self.stop.set()
        self.t.join()


def block_outputs(lib, wts, crops, n):
    """Pooled conv-1 planes of the first block on crops[:n] through mmmot_debug_vgg_conv01, as int16 (bytes)."""
    tab, W = wts.table, _lib.W
    plane = n * HW * HW * 64
    bufs = [torch.zeros(2 * plane, dtype=torch.int16, device="cuda") for _ in range(2)]
    scratch = torch.empty((n + 16) * HW * HW * 16, dtype=torch.float32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out, fused = ctypes.c_int(-1), ctypes.c_int(-1)
    p = lambda k, i=0: ctypes.c_void_p(tab.w[W[k] + i])
    sc = lambda k, i=0: tab.tc_scale[W[k] + i]
    rc = lib.mmmot_debug_vgg_conv01(ctypes.c_void_p(crops.data_ptr()), n, HW, HW, p("VGG_WT0"), p("VGG_B0"), p("VGG_WP0"),
                                    sc("VGG_WP0"), p("VGG_WPX0"), p("VGG_B0", 1), p("VGG_WP0", 1), sc("VGG_WP0", 1),
                                    p("VGG_WPX0", 1), ctypes.c_void_p(bufs[0].data_ptr()), ctypes.c_void_p(bufs[1].data_ptr()),
                                    ctypes.c_void_p(scratch.data_ptr()), ctypes.c_void_p(status.data_ptr()),
                                    ctypes.byref(out), ctypes.byref(fused), None)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return bufs[out.value][:plane // 2].clone(), fused.value, int(status.item())


def main():
    assert torch.cuda.is_available(), "vgg01_times needs a CUDA device"
    lib = _lib.load()
    res = {"card": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "crops_per_call": N, "calls_per_step": STEP_CROPS // N}
    net = mb.TrackingNet(2, appear_skippool=True, score_arch="branch_cls", dropblock=0)
    net.load_state_dict(synthetic_state_dict("C", seed=1))
    net.cuda().eval()
    wts = net.prepared()
    g = torch.Generator(device="cuda").manual_seed(0)
    crops = torch.randn(N, 3, HW, HW, device="cuda", generator=g)
    feats = {k: torch.empty(N // L, 3, 512, L, device="cuda") for k, _ in PATHS}
    nbytes = lib.mmmot_appearance_workspace(N, HW, HW)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    a = [ctypes.c_void_p(t.data_ptr()) for t in (crops, ws)]

    def call(name):
        rc = lib.mmmot_appearance_fwd(wts.ptr, a[0], N, HW, HW, L, ctypes.c_void_p(feats[name].data_ptr()), a[1], nbytes, None)
        assert rc == 0, rc

    clock = ClockSampler()
    step_ms = {k: [] for k, _ in PATHS}
    tags = {k: [] for k, _ in PATHS}
    assert lib.mmmot_status_reset(a[1], None) == 0
    for name, dbg in PATHS:                       # warm-up of both paths
        assert lib.mmmot_set_debug(dbg) == 0
        for _ in range(2):
            call(name)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for name, dbg in PATHS:
            assert lib.mmmot_set_debug(dbg) == 0
            reps = 6
            clock.on.set()
            e0.record()
            for _ in range(reps):
                call(name)
            e1.record()
            torch.cuda.synchronize()
            clock.on.clear()
            step_ms[name].append(e0.elapsed_time(e1) / reps * (STEP_CROPS / N))
            lib.mmmot_timing_collect_tags(None, None, None, None)
            lib.mmmot_timing_enable(1)
            call(name)
            lib.mmmot_timing_enable(0)
            k = lib.mmmot_timing_tag_count()
            tms, tfl, tby = (ctypes.c_double * k)(), (ctypes.c_double * k)(), (ctypes.c_double * k)()
            cnt = (ctypes.c_long * k)()
            assert lib.mmmot_timing_collect_tags(tms, tfl, tby, cnt) == 0
            tags[name].append({lib.mmmot_timing_tag_name(t).decode(): (tms[t], tfl[t], tby[t]) for t in range(k) if cnt[t]})
    assert lib.mmmot_set_debug(0) == 0
    assert lib.mmmot_status_check(a[1], None) == 0
    clock.close()
    scale = STEP_CROPS / N
    for name, _ in PATHS:
        names = sorted({t for d in tags[name] for t in d if t.startswith("vgg.")})
        rows = {}
        for t in names:
            ms = statistics.median(d[t][0] for d in tags[name] if t in d) * scale
            fl, by = tags[name][0][t][1] * scale, tags[name][0][t][2] * scale
            rows[t] = {"ms_per_step": round(ms, 2), "tflops": round(fl / (ms * 1e9), 1) if fl else None,
                       "tb_per_s": round(by / (ms * 1e9), 2) if by else None}
        res[name] = {"appearance_ms_per_step": [round(v, 1) for v in step_ms[name]],
                     "appearance_ms_per_step_median": round(statistics.median(step_ms[name]), 1), "tags": rows}
    f_ms = res["fused"]["tags"].get("vgg.conv1", {}).get("ms_per_step")
    t_tags = res["two_launch"]["tags"]
    t_ms = t_tags.get("vgg.conv0", {}).get("ms_per_step", 0) + t_tags.get("vgg.conv1", {}).get("ms_per_step", 0)
    res["block_ms_per_step"] = {"fused": f_ms, "two_launch_conv0_plus_conv1": round(t_ms, 2),
                                "ratio": round(f_ms / t_ms, 3) if f_ms and t_ms else None}
    res["sm_clock_median_mhz"] = statistics.median(clock.samples) if clock.samples else None
    res["features_byte_equal"] = bool(torch.equal(feats["fused"].view(torch.int32), feats["two_launch"].view(torch.int32)))
    outs = {}
    for name, dbg in PATHS:
        assert lib.mmmot_set_debug(dbg) == 0
        outs[name] = block_outputs(lib, wts, crops, 1024)
    assert lib.mmmot_set_debug(0) == 0
    res["block_fused_flags"] = [outs[k][1] for k, _ in PATHS]
    res["block_status"] = [outs[k][2] for k, _ in PATHS]
    res["pooled_byte_equal"] = bool(torch.equal(outs["fused"][0], outs["two_launch"][0]))
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
