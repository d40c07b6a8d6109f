#!/usr/bin/env python
"""Per-source output size at scale: the call tail (flip -> resize -> YUYV / NV12) of Meet 1280x720 calls.

    python tools/source_output_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--lib PATH] [--workloads a,b,c,d,e,f]
                                        [--formats yuyv,nv12] [--profile-calls 10]

Meet full (segm_full_v679), 1280x720, camera frames resident on the device (YUYV, or NV12 packed), the context image.
Workloads (a-e: one context with 64 sources, one call of one frame per source):
  a  no resize, no tail;
  b  context size 640x360 (bsb_set_output);
  c  every source its own 640x360 (bsb_set_source_output);
  d  a quarter each at 1280x720, 960x540, 640x360 and 320x180 (own sizes);
  e  every source mirrored with the post kernel's TMA path off (post_tma=0), so the flip runs in the tail;
  f  one plain context, 32-frame calls (bench.py's), with bsb_set_output(flip_h=1, 640x360).
With --lib (the library of another build, e.g. the parent of bsb_set_source_output) the workloads that build can run
(a, b, e, f) are run on it.  Output buffers hold 1280x720 frames in every workload (same strides).
Throughput: CUDA events around `rounds` calls after `warmup`; frames/s = frames * rounds / time, `runs` times.
Tail time: a separate torch.profiler run of --profile-calls calls, summing per call the kernels of the tail: k_tail for
this build, k_flip_u8c3[_frames] + k_resize_u8c3 + k_rgb_to_yuyv + k_yuyv_to_nv12 for older builds.
Prints one JSON line per (workload, format), with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.source_effects_bench import S, W, H, bind_older, frames, gpu_info  # noqa: E402

TAIL = ("k_tail", "k_flip_u8c3", "k_resize_u8c3", "k_rgb_to_yuyv", "k_yuyv_to_nv12")
PLAIN_BATCH = 32
MIXED = [(1280, 720), (960, 540), (640, 360), (320, 180)]


def make_ctx(lib, wl):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=PLAIN_BATCH if wl == "f" else S)
    g.set_background(synth.background()[::-1].copy())
    if wl == "b":
        g.set_output(out_size=(640, 360))
    if wl == "f":
        g.set_output(flip_h=True, out_size=(640, 360))
        return g
    g.set_sources(S)
    for s in range(S):
        if wl == "c":
            g.set_source_output(s, (640, 360))
        elif wl == "d":
            g.set_source_output(s, MIXED[s * len(MIXED) // S])
        elif wl == "e":
            g.set_source_flip(s, flip_h=True)
    return g


def run_calls(g, wl, fmt, bufs, n):
    d_in, d_out, d_vid, d_mask = (b.data_ptr() for b in bufs)
    ost, vst = W * H * 3, W * H * 3 // 2 if fmt == "nv12" else W * H * 2
    for _ in range(n):
        if wl == "f":
            if fmt == "nv12":
                g.composite_nv12_device(PLAIN_BATCH, d_in, d_out, d_vid, d_mask)
            else:
                g.composite_yuyv_device(PLAIN_BATCH, d_in, d_out, d_vid, d_mask)
            continue
        ids = list(range(S))
        if fmt == "nv12":
            g.composite_sources_nv12_device(S, ids, d_in, d_out, d_vid, d_mask, out_stride=ost, nv12_stride=vst)
        else:
            g.composite_sources_yuyv_device(S, ids, d_in, d_out, d_vid, d_mask, out_stride=ost, yuyv_stride=vst)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--lib", default=None, help="library of another build: workloads a, b, e and f")
    ap.add_argument("--workloads", default="a,b,c,d,e,f")
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--profile-calls", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("source_output_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bind_older(args.lib) if args.lib else bs.lib()
    wls = [w for w in args.workloads.split(",") if not (args.lib and w in "cd")]
    info = gpu_info(0)
    dev = "cuda:0"
    for fmt in args.formats.split(","):
        host = frames(fmt)
        d_in = torch.from_numpy(host).to(dev)
        d_out = torch.empty(S * W * H * 3, dtype=torch.uint8, device=dev)
        d_vid = torch.empty(S * (W * H * 3 // 2 if fmt == "nv12" else W * H * 2), dtype=torch.uint8, device=dev)
        d_mask = torch.empty((S, H, W), dtype=torch.uint8, device=dev)
        bufs = (d_in, d_out, d_vid, d_mask)
        for wl in wls:
            lib.bsb_set_tuning(b"post_tma", 0 if wl == "e" else 1)
            g = make_ctx(lib, wl)
            nfr = PLAIN_BATCH if wl == "f" else S
            stream = torch.cuda.ExternalStream(g.stream)
            run_calls(g, wl, fmt, bufs, args.warmup)
            g.synchronize()
            launches = g.launches_per_call
            rates = []
            for _ in range(args.runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run_calls(g, wl, fmt, bufs, args.rounds)
                e1.record(stream)
                e1.synchronize()
                rates.append(nfr * args.rounds / (e0.elapsed_time(e1) / 1e3))
            res = {"workload": wl, "format": fmt, "lib": args.lib or "package", "frames_per_call": nfr,
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "launches_per_call": launches, **info}
            if args.profile_calls:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run_calls(g, wl, fmt, bufs, args.profile_calls)
                    g.synchronize()
                per = {}
                for ev in prof.key_averages():
                    tot = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    if any(tag in ev.key for tag in TAIL):
                        per[ev.key.split("(")[0][-40:]] = round(tot / args.profile_calls, 1)
                res["tail_us_per_call"] = per
                res["tail_us_total"] = round(sum(per.values()), 1)
            print(json.dumps(res), flush=True)
            g.close()
    lib.bsb_set_tuning(b"post_tma", 1)


if __name__ == "__main__":
    main()
