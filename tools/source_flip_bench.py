#!/usr/bin/env python
"""Per-source mirroring at scale: one Meet context with 64 sources, one call of one frame per source.

    python tools/source_flip_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--lib PATH] [--mixes none,half,all]
                                      [--formats yuyv,nv12] [--profile-dir DIR]

Meet full (segm_full_v679), 1280x720, 64 sources in one context with the context image, camera frames resident on the
device (YUYV, or NV12 packed).  Flip mixes:
  none  no source flipped;
  half  every other source mirrored (horizontal flip);
  all   every source mirrored.
With --lib (the library of another build, e.g. the parent of bsb_set_source_flip), the "none" and "all" mixes are set up
the way that build can run them; "all" is the context flip bsb_set_output(1, 0), which there takes the stand-alone tail
(post -> flip -> YUYV [-> NV12]).
Throughput: CUDA events around `rounds` calls after `warmup`; frames/s = 64 * rounds / time, `runs` times per mix.
With --profile-dir, a separate torch.profiler run per mix gives the time per call of k_post_tma and the tail kernels.
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

TAGS = ("k_post_tma", "k_flip_u8c3", "k_rgb_to_yuyv", "k_yuyv_to_nv12")


def make_ctx(lib, mix, context_flip):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=S)
    g.set_background(synth.background()[::-1].copy())
    if context_flip:
        if mix == "all":
            g.set_output(flip_h=True)
        elif mix != "none":
            raise SystemExit("--lib runs the none and all mixes only")
    g.set_sources(S)
    if not context_flip:
        for s in range(S):
            if mix == "all" or (mix == "half" and s % 2):
                g.set_source_flip(s, flip_h=True)
    return g


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
    ap.add_argument("--lib", default=None, help="library of another build: the none mix, and the all mix as a context flip")
    ap.add_argument("--mixes", default="none,half,all")
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--profile-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("source_flip_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bind_older(args.lib) if args.lib else bs.lib()
    mixes = [m for m in args.mixes.split(",") if m != "half"] if args.lib else args.mixes.split(",")
    info = gpu_info(0)
    dev = "cuda:0"
    for fmt in args.formats.split(","):
        host = frames(fmt)
        d_in = torch.from_numpy(host).to(dev)
        d_out = torch.empty((S, H, W, 3), dtype=torch.uint8, device=dev)
        d_vid = torch.empty(S * (W * H * 3 // 2 if fmt == "nv12" else W * H * 2), dtype=torch.uint8, device=dev)
        d_mask = torch.empty((S, H, W), dtype=torch.uint8, device=dev)
        for mix in mixes:
            g = make_ctx(lib, mix, bool(args.lib))
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
            res = {"mix": mix, "format": fmt, "context_flip": bool(args.lib), "lib": args.lib or "package", "sources": S,
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "native": native, "launches_per_call": launches, **info}
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
                prof.export_chrome_trace(os.path.join(args.profile_dir, f"flip_trace_{mix}_{fmt}{'_ctx' if args.lib else ''}.json"))
            print(json.dumps(res), flush=True)
            g.close()


if __name__ == "__main__":
    main()
