#!/usr/bin/env python
"""Framing at scale: what cropping every frame's output costs, on device-resident camera frames.

    python tools/framing_bench.py [--rounds 30] [--warmup 10] [--runs 3] [--formats yuyv,nv12] [--cases ...] [--profile]

Meet full (segm_full_v679), 1280x720, the context image as background, YUYV or NV12 (packed) frames on the device.
Cases:
  src_off            one context with 64 sources, one frame per source per call, framing off (the unframed kernels);
  src_auto           the same with every source in AUTO (1280x720 output);
  src_auto_360       every source in AUTO with a 640x360 output;
  src_half           half the sources RECT (a 640x360 crop, a copy), half off (whole frames through the cropping tail);
  plain_off, plain_auto  8 plain contexts (streams) x 32-frame calls, one call per stream per round, off / AUTO.
Throughput: CUDA events around `rounds` rounds after `warmup`; frames/s = frames composited / time, `runs` times per case.
Sources cases time the context's stream; plain cases enqueue the 8 streams in turn and time from an event before the
first to the end of all.  --profile: a separate torch.profiler run per case gives the device time per call of k_framing
and k_tail, and the launches per call.  Prints one JSON line per (case, format), with the GPU name and power limit read
in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.source_effects_bench import S, W, H, frames, gpu_info  # noqa: E402

STREAMS, BATCH = 8, 32
CASES = {"src_off": ("src", "off"), "src_auto": ("src", "auto"), "src_auto_360": ("src", "auto_360"), "src_half": ("src", "half"),
         "plain_off": ("plain", "off"), "plain_auto": ("plain", "auto")}
KERNELS = ("k_framing", "k_tail")


def make_ctxs(lib, kind, k):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    bg = synth.background()[::-1].copy()
    if kind == "src":
        g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=S)
        g.set_background(bg)
        g.set_sources(S)
        if k == "auto_360":
            g.set_output(out_size=(640, 360))
        if k.startswith("auto"):
            g.set_framing("auto")
        elif k == "half":
            for s in range(0, S, 2):
                g.set_source_framing(s, "rect", (320 + s, 180, 640, 360))
        return [g]
    gs = []
    for _ in range(STREAMS):
        g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=BATCH)
        g.set_background(bg)
        if k == "auto":
            g.set_framing("auto")
        gs.append(g)
    return gs


class Bufs:
    def __init__(self, torch, fmt, n):
        dev = "cuda:0"
        host = frames(fmt)
        reps = (n + S - 1) // S
        self.d_in = torch.from_numpy(np.concatenate([host] * reps)[:n].copy()).to(dev)
        self.d_out = torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev)
        self.d_vid = torch.empty(n * (W * H * 3 // 2 if fmt == "nv12" else W * H * 2), dtype=torch.uint8, device=dev)
        self.d_mask = torch.empty((n, H, W), dtype=torch.uint8, device=dev)


def one_round(kind, gs, fmt, bufs):
    """one call per context; returns the frames it composited"""
    ptrs = (bufs[0].d_in.data_ptr(), bufs[0].d_out.data_ptr(), bufs[0].d_vid.data_ptr(), bufs[0].d_mask.data_ptr())
    if kind == "src":
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("framing_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bs.lib()
    info = gpu_info(0)
    cases = args.cases.split(",")
    for fmt in args.formats.split(","):
        for case in cases:
            kind, k = CASES[case]
            gs = make_ctxs(lib, kind, k)
            bufs = [Bufs(torch, fmt, S)] if kind == "src" else [Bufs(torch, fmt, BATCH) for _ in gs]
            for _ in range(args.warmup):
                one_round(kind, gs, fmt, bufs)
            sync_all(gs)
            res = {"case": case, "format": fmt}
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
