#!/usr/bin/env python
"""Masked camera blur at scale: what leaving the person out of the background blur costs, on device-resident frames.

    python tools/blur_mode_bench.py [--rounds 30] [--warmup 10] [--runs 3] [--formats yuyv,nv12] [--cases ...]
                                    [--profile] [--lib PATH]

Meet full (segm_full_v679), 1280x720, no background image (every frame blends its own blurred camera frame), YUYV or
NV12 (packed) frames on the device.  Cases:
  src25_plain, src25_masked   one context with 64 sources, one frame per source per call, k = 25: plain / masked mode;
  src61_plain, src61_masked   the same at k = 61 (the row / column launch class);
  src25_half                  k = 25, every second source masked;
  plain25_plain, plain25_masked   8 plain contexts (streams) x 32-frame calls, k = 25.
Throughput: CUDA events around `rounds` rounds after `warmup`; frames/s = frames composited / time, `runs` times per case.
--profile: a separate torch.profiler run per case gives the device time per call of k_post_tma (in masked cases it
includes the mask-only launch) and of the Gaussian kernels, and the launches per call.
--lib: another build of the library (for example the parent commit's) runs the plain cases, which are all it has.  Prints
one JSON line per (case, format), with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.mask_refine_bench import BATCH, STREAMS, Bufs, bind_other, one_round, sync_all, timed  # noqa: E402
from tools.source_effects_bench import S, W, H, gpu_info  # noqa: E402

CASES = {"src25_plain": ("src", 25, "plain"), "src25_masked": ("src", 25, "masked"), "src61_plain": ("src", 61, "plain"),
         "src61_masked": ("src", 61, "masked"), "src25_half": ("src", 25, "half"),
         "plain25_plain": ("plain", 25, "plain"), "plain25_masked": ("plain", 25, "masked")}
KERNELS = ("k_post_tma", "k_gauss_fused", "k_gauss_rows", "k_gauss_cols", "k_gauss_stage_bgr", "k_gauss_slot_yuv",
           "k_mgauss_fused", "k_mgauss_rows", "k_mgauss_cols")


def make_ctxs(lib, kind, k, mode):
    from backscrub_b200 import api
    from tests.conftest import model_path
    model = model_path("meet_full")
    if kind == "src":
        g = api.MaskGen(lib, model, W, H, max_batch=S)
        g.set_bgblur(k)
        g.set_sources(S)
        if mode == "masked":
            g.set_blur_mode("masked")
        elif mode == "half":
            for s in range(0, S, 2):
                g.set_source_blur_mode(s, "masked")
        return [g]
    gs = []
    for _ in range(STREAMS):
        g = api.MaskGen(lib, model, W, H, max_batch=BATCH)
        g.set_bgblur(k)
        if mode == "masked":
            g.set_blur_mode("masked")
        gs.append(g)
    return gs


def profile_case(torch, kind, gs, fmt, bufs):
    from torch.profiler import ProfilerActivity, profile
    rounds = 8
    sync_all(gs)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            one_round(kind, gs, fmt, bufs)
        sync_all(gs)
    calls = rounds * len(gs)
    sums = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        tot = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        for k in KERNELS:
            if k + "<" in ev.key or k + "(" in ev.key or ev.key.endswith(k):
                sums[k] += tot
    return {"us_per_call": {k: round(v / calls, 1) for k, v in sums.items() if v}, "launches_per_call": gs[0].launches_per_call}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--lib", default=None, help="library of another build (default: the package's); runs the plain cases")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("blur_mode_bench needs a CUDA device")
    import backscrub_b200 as bs
    from backscrub_b200 import _binding
    lib = bind_other(_binding, os.path.abspath(args.lib)) if args.lib else bs.lib()
    info = gpu_info(0)
    cases = [c for c in args.cases.split(",") if not args.lib or c.endswith("_plain")]
    for fmt in args.formats.split(","):
        for case in cases:
            kind, k, mode = CASES[case]
            gs = make_ctxs(lib, kind, k, mode)
            bufs = [Bufs(torch, fmt, S, W, H)] if kind == "src" else [Bufs(torch, fmt, BATCH, W, H) for _ in gs]
            for _ in range(args.warmup):
                one_round(kind, gs, fmt, bufs)
            sync_all(gs)
            res = {"case": case, "format": fmt, "lib": args.lib or "package"}
            if args.profile:
                res.update(profile_case(torch, kind, gs, fmt, bufs))
            else:
                rates = [timed(torch, kind, gs, fmt, bufs, args.rounds) for _ in range(args.runs)]
                res.update({"frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1)})
            res.update(info)
            print(json.dumps(res), flush=True)
            for g in gs:
                g.close()


if __name__ == "__main__":
    main()
