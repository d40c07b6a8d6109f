#!/usr/bin/env python
"""Per-source animated backgrounds at scale: one Meet context with 64 sources, one call of one frame per source.

    python tools/source_ring_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--ring 8] [--lib PATH]
                                      [--modes stills,rings,rings_blur,reset] [--formats yuyv,nv12] [--profile]

Meet full (segm_full_v679), 1280x720, 64 sources in one context, camera frames resident on the device (YUYV, or NV12
packed).  Modes:
  stills      every source blends its own still (bsb_set_source_background once);
  rings       every source plays its own ring of --ring images (each source's ring different), advance 1;
  rings_blur  the same with every source at its own strength k = 25;
  reset       what a caller without source rings must do: before every call, each source's still is replaced by
              bsb_set_source_background from a host frame (a ring of --ring host images, cycled).
With --lib (the library of another build, e.g. the parent of bsb_set_source_background_ring), only the stills and
reset modes run.  Throughput: CUDA events around `rounds` calls after `warmup`; frames/s = 64 * rounds / time, `runs`
times per mode (reset: the host clock around the same calls, since its set calls synchronise the stream).  With
--profile, a separate torch.profiler run per mode gives k_post_tma's time per call.  Bank bytes: the device memory of
the background bank (BGR, YUYV, NV12 per slot) and of the unblurred images kept for re-blurring.  Prints one JSON line
per (mode, format), with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.source_effects_bench import bind_older, frames, gpu_info   # noqa: E402

W, H, S, MAX_BATCH = 1280, 720, 64, 64


def ring_images(s, count):
    """source s's decoded images: the bundled background rolled and tinted per source and per image"""
    from tests import synth
    bg = synth.background()
    return np.stack([np.roll(bg, 37 * s + 113 * i, axis=1) ^ np.uint8((11 * s + 29 * i) & 0xFF) for i in range(count)])


def bank_bytes(mode, ring):
    """the bank: [max_batch] camera-blur | [1] context | [S] source slots | [pool] ring images, each BGR + YUYV + NV12;
    plus the unblurred images: [S] stills and [pool] ring images"""
    npix = W * H
    pool = S * ring if mode in ("rings", "rings_blur") else 0
    return (MAX_BATCH + 1 + S + pool) * (npix * 3 + npix * 2 + npix * 3 // 2) + (S + pool) * npix * 3


def make_ctx(lib, mode, ring):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=MAX_BATCH)
    g.set_background(synth.background()[::-1].copy())
    g.set_sources(S)
    for s in range(S):
        imgs = ring_images(s, ring)
        if mode in ("rings", "rings_blur"):
            g.set_source_background_ring(s, imgs, 1)
            if mode == "rings_blur":
                g.set_source_effect(s, "default", 25)
        else:
            g.set_source_background(s, imgs[0])
    return g


def run_calls(g, fmt, bufs, n, reset=None):
    d_in, d_out, d_vid, d_mask = bufs
    ids = list(range(S))
    for i in range(n):
        if reset is not None:
            for s in range(S):
                g.set_source_background(s, reset[s][i % len(reset[s])])
        if fmt == "nv12":
            g.composite_sources_nv12_device(S, ids, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr())
        else:
            g.composite_sources_yuyv_device(S, ids, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--ring", type=int, default=8)
    ap.add_argument("--lib", default=None, help="library to bind (default: the package's)")
    ap.add_argument("--modes", default="stills,rings,rings_blur,reset")
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("source_ring_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bind_older(args.lib) if args.lib else bs.lib()
    modes = args.modes.split(",")
    if args.lib:
        modes = [m for m in modes if m in ("stills", "reset")]
    info = gpu_info(0)
    dev = "cuda:0"
    reset_imgs = None
    for fmt in args.formats.split(","):
        d_in = torch.from_numpy(frames(fmt)).to(dev)
        bufs = (d_in, torch.empty((S, H, W, 3), dtype=torch.uint8, device=dev),
                torch.empty(S * (W * H * 3 // 2 if fmt == "nv12" else W * H * 2), dtype=torch.uint8, device=dev),
                torch.empty((S, H, W), dtype=torch.uint8, device=dev))
        for mode in modes:
            g = make_ctx(lib, mode, args.ring)
            reset = None
            if mode == "reset":
                if reset_imgs is None:
                    reset_imgs = [ring_images(s, args.ring) for s in range(S)]
                reset = reset_imgs
            stream = torch.cuda.ExternalStream(g.stream)
            run_calls(g, fmt, bufs, args.warmup, reset)
            g.synchronize()
            native = g.yuyv_native
            rates = []
            for _ in range(args.runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(stream)
                run_calls(g, fmt, bufs, args.rounds, reset)
                e1.record(stream)
                e1.synchronize()
                dt = time.perf_counter() - t0 if reset is not None else e0.elapsed_time(e1) / 1e3
                rates.append(S * args.rounds / dt)
            res = {"mode": mode, "format": fmt, "lib": args.lib or "package", "sources": S, "ring": args.ring,
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "native": native, "bank_bytes": bank_bytes(mode, args.ring), **info}
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                calls = 10
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run_calls(g, fmt, bufs, calls, reset)
                    g.synchronize()
                per = {}
                for ev in prof.key_averages():
                    tot = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    if "k_post_tma" in ev.key:
                        per[ev.key.split("(")[0][-60:]] = round(tot / calls, 1)
                res["k_post_tma_us_per_call"] = per
            print(json.dumps(res), flush=True)
            g.close()


if __name__ == "__main__":
    main()
