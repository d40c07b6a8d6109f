#!/usr/bin/env python
"""Mask edge refinement at scale: what refining every frame's mask costs, on device-resident camera frames.

    python tools/mask_refine_bench.py [--rounds 30] [--warmup 10] [--runs 3] [--formats yuyv,nv12] [--cases ...]
                                      [--profile] [--lib PATH]

Meet full (segm_full_v679), 1280x720, the context image as background, YUYV or NV12 (packed) frames on the device.
Cases:
  src_off, src_on, src_half   one context with 64 sources, one frame per source per call: refinement off, every source
                              at sigma 12, or every second source at sigma 12 and the others off;
  plain_off, plain_on         8 plain contexts (streams) x 32-frame calls, one call per stream per round, off / sigma 12;
  mlkit_off, mlkit_on         MLKit (256x256) at 640x480, 8 streams x 32 frames, off / sigma 12.
Throughput: CUDA events around `rounds` rounds after `warmup`; frames/s = frames composited / time, `runs` times per case.
--profile: a separate torch.profiler run per case gives k_post_tma's device time per call and the launches per call.
--lib: another build of the library (for example the parent commit's) runs the "off" cases, which are all it has.  Prints
one JSON line per (case, format), with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.source_effects_bench import S, W, H, frames, gpu_info  # noqa: E402

STREAMS, BATCH, SIGMA = 8, 32, 12
CASES = {"src_off": ("src", "off"), "src_on": ("src", "on"), "src_half": ("src", "half"),
         "plain_off": ("plain", "off"), "plain_on": ("plain", "on"), "mlkit_off": ("mlkit", "off"), "mlkit_on": ("mlkit", "on")}
KERNELS = ("k_post_tma", "k_post_fast")


def geometry(kind):
    return (640, 480) if kind == "mlkit" else (W, H)


def make_ctxs(lib, kind, k):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    bg = synth.background()[::-1].copy()
    w, h = geometry(kind)
    model = model_path("mlkit" if kind == "mlkit" else "meet_full")
    if kind == "src":
        g = api.MaskGen(lib, model, w, h, max_batch=S)
        g.set_background(bg)
        g.set_sources(S)
        if k == "on":
            g.set_mask_refine(SIGMA)
        elif k == "half":
            for s in range(0, S, 2):
                g.set_source_mask_refine(s, SIGMA)
        return [g]
    gs = []
    for _ in range(STREAMS):
        g = api.MaskGen(lib, model, w, h, max_batch=BATCH)
        g.set_background(bg)
        if k == "on":
            g.set_mask_refine(SIGMA)
        gs.append(g)
    return gs


def camera_frames(fmt, w, h, n):
    if (w, h) == (W, H):
        host = frames(fmt)
    else:
        from tests import synth
        yuyv = [synth.yuyv_frame(w, h, t=t) for t in range(4)]
        host = np.stack(yuyv if fmt == "yuyv" else [np.concatenate([y[..., 0], y[0::2, :, 1]], axis=0) for y in yuyv])
    reps = (n + len(host) - 1) // len(host)
    return np.concatenate([host] * reps)[:n].copy()


class Bufs:
    def __init__(self, torch, fmt, n, w, h):
        dev = "cuda:0"
        self.d_in = torch.from_numpy(camera_frames(fmt, w, h, n)).to(dev)
        self.d_out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
        self.d_vid = torch.empty(n * (w * h * 3 // 2 if fmt == "nv12" else w * h * 2), dtype=torch.uint8, device=dev)
        self.d_mask = torch.empty((n, h, w), dtype=torch.uint8, device=dev)


def one_round(kind, gs, fmt, bufs):
    """one call per context; returns the frames it composited"""
    if kind == "src":
        b = bufs[0]
        ptrs = (b.d_in.data_ptr(), b.d_out.data_ptr(), b.d_vid.data_ptr(), b.d_mask.data_ptr())
        ids = list(range(S))
        if fmt == "nv12":
            gs[0].composite_sources_nv12_device(S, ids, *ptrs)
        else:
            gs[0].composite_sources_yuyv_device(S, ids, *ptrs)
        return S
    for g, b in zip(gs, bufs):
        p = (b.d_in.data_ptr(), b.d_out.data_ptr(), b.d_vid.data_ptr(), b.d_mask.data_ptr())
        if fmt == "nv12":
            g.composite_nv12_device(BATCH, *p)
        else:
            g.composite_yuyv_device(BATCH, *p)
    return BATCH * len(gs)


def sync_all(gs):
    for g in gs:
        g.synchronize()


def timed(torch, kind, gs, fmt, bufs, rounds):
    streams = [torch.cuda.ExternalStream(g.stream) for g in gs]
    sync_all(gs)
    e0 = torch.cuda.Event(enable_timing=True)
    e0.record(streams[0])
    for s in streams[1:]:
        s.wait_event(e0)
    n = sum(one_round(kind, gs, fmt, bufs) for _ in range(rounds))
    ends = []
    for s in streams:
        e = torch.cuda.Event(enable_timing=True)
        e.record(s)
        ends.append(e)
    for e in ends:
        e.synchronize()
    return n / (max(e0.elapsed_time(e) for e in ends) / 1e3)


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
            if k in ev.key:
                sums[k] += tot
    return {"us_per_call": {k: round(v / calls, 1) for k, v in sums.items()}, "launches_per_call": gs[0].launches_per_call}


def bind_other(_binding, path):
    """bind another build, which may predate some symbols of the binding (e.g. the parent of this feature): a missing
    symbol binds to a stub that fails when called, and the "off" cases never call it"""
    import ctypes

    class Lenient(ctypes.CDLL):
        def __getattr__(self, name):
            try:
                return super().__getattr__(name)
            except AttributeError:
                if name.startswith("__"):
                    raise
                def missing(*_a):
                    raise RuntimeError(f"{path} has no {name}")
                setattr(self, name, missing)
                return missing

    real = _binding.C.CDLL
    _binding.C.CDLL = Lenient
    try:
        return _binding.bind(path)
    finally:
        _binding.C.CDLL = real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--lib", default=None, help="library of another build (default: the package's); runs the off cases")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mask_refine_bench needs a CUDA device")
    import backscrub_b200 as bs
    from backscrub_b200 import _binding
    lib = bind_other(_binding, os.path.abspath(args.lib)) if args.lib else bs.lib()
    info = gpu_info(0)
    cases = [c for c in args.cases.split(",") if not args.lib or c.endswith("_off")]
    for fmt in args.formats.split(","):
        for case in cases:
            kind, k = CASES[case]
            w, h = geometry(kind)
            gs = make_ctxs(lib, kind, k)
            bufs = [Bufs(torch, fmt, S, w, h)] if kind == "src" else [Bufs(torch, fmt, BATCH, w, h) for _ in gs]
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
