#!/usr/bin/env python
"""The filter switch at scale: one Meet context with 64 sources, one call of one frame per source.

    python tools/source_filter_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--lib PATH] [--mixes none,half,all]
                                        [--formats yuyv,nv12] [--profile-dir DIR]

Meet full (segm_full_v679), 1280x720, 64 sources in one context with the context image, camera frames resident on the
device (YUYV, or NV12 packed).  Filter mixes:
  none  every source filtered on (the composite);
  half  every other source switched off (bsb_set_source_filter(s, 0)): its camera frame passes through;
  all   every source switched off.
With --lib (the library of another build, e.g. the parent of bsb_set_filter), only the "none" mix runs, which that build
runs too: calls without a filtered-off frame should not have changed.
Throughput: CUDA events around `rounds` calls after `warmup`; frames/s = 64 * rounds / time, `runs` times per mix.
With --profile-dir, a separate torch.profiler run per mix gives the time per call of k_post_tma.
post_bytes_per_call: the post kernel's DRAM-side bytes per call from the shapes: the outputs (BGR composite, video, mask)
are written for every frame; a filtered-on frame reads its background tile and the cached background video tile, and its
camera tile where a tile can contain a person (counted here for every tile: an upper bound); a filtered-off frame reads
only its camera frame (and the small mask patches, not counted).
Prints one JSON line per (mix, format), with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.source_effects_bench import S, W, H, bind_older, frames, gpu_info  # noqa: E402

TAGS = ("k_post_tma",)


def off_sources(mix):
    return [s for s in range(S) if mix == "all" or (mix == "half" and s % 2)]


def make_ctx(lib, mix):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=S)
    g.set_background(synth.background()[::-1].copy())
    g.set_sources(S)
    for s in off_sources(mix):
        g.set_source_filter(s, False)
    return g


def post_bytes(mix, fmt):
    npx = W * H
    video = npx * 3 // 2 if fmt == "nv12" else npx * 2
    n_off = len(off_sources(mix))
    writes = S * (npx * 3 + video + npx)
    reads = (S - n_off) * (npx * 3 + video + video) + n_off * video
    return {"reads_upper": reads, "writes": writes, "total_upper": reads + writes}


def run_calls(g, fmt, d_in, d_out, d_vid, d_mask, n):
    ids = list(range(S))
    for _ in range(n):
        if fmt == "nv12":
            g.composite_sources_nv12_device(S, ids, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr())
        else:
            g.composite_sources_yuyv_device(S, ids, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--lib", default=None, help="library of another build: the none mix only")
    ap.add_argument("--mixes", default="none,half,all")
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--profile-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("source_filter_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bind_older(args.lib) if args.lib else bs.lib()
    mixes = ["none"] if args.lib else args.mixes.split(",")
    info = gpu_info(0)
    dev = "cuda:0"
    for fmt in args.formats.split(","):
        host = frames(fmt)
        d_in = torch.from_numpy(host).to(dev)
        d_out = torch.empty((S, H, W, 3), dtype=torch.uint8, device=dev)
        d_vid = torch.empty(S * (W * H * 3 // 2 if fmt == "nv12" else W * H * 2), dtype=torch.uint8, device=dev)
        d_mask = torch.empty((S, H, W), dtype=torch.uint8, device=dev)
        for mix in mixes:
            g = make_ctx(lib, mix)
            stream = torch.cuda.ExternalStream(g.stream)
            run_calls(g, fmt, d_in, d_out, d_vid, d_mask, args.warmup)
            g.synchronize()
            native, launches = g.yuyv_native, g.launches_per_call
            rates = []
            for _ in range(args.runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run_calls(g, fmt, d_in, d_out, d_vid, d_mask, args.rounds)
                e1.record(stream)
                e1.synchronize()
                rates.append(S * args.rounds / (e0.elapsed_time(e1) / 1e3))
            res = {"mix": mix, "format": fmt, "lib": args.lib or "package", "sources": S, "filtered_off": len(off_sources(mix)),
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "native": native, "launches_per_call": launches, "post_bytes_per_call": post_bytes(mix, fmt), **info}
            if args.profile_dir:
                from torch.profiler import ProfilerActivity, profile
                os.makedirs(args.profile_dir, exist_ok=True)
                calls = 10
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run_calls(g, fmt, d_in, d_out, d_vid, d_mask, calls)
                    g.synchronize()
                per = {}
                for ev in prof.key_averages():
                    name = ev.key
                    tot = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    if any(tag in name for tag in TAGS):
                        per[name.split("(")[0][-60:]] = round(tot / calls, 1)
                res["us_per_call"] = per
                prof.export_chrome_trace(os.path.join(args.profile_dir, f"filter_trace_{mix}_{fmt}{'_lib' if args.lib else ''}.json"))
            print(json.dumps(res), flush=True)
            g.close()


if __name__ == "__main__":
    main()
