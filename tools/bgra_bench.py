#!/usr/bin/env python
"""The transparent BGRA output against the composite, on device-resident camera YUYV frames.

    python tools/bgra_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--setups plain,sources] [--modes ...] [--profile-dir DIR]

Meet full (segm_full_v679), 1280x720, the context image as background.  Setups:
  plain    8 plain contexts, one stream each, 32 frames per call (calls of the 8 contexts interleaved);
  sources  one context with 64 sources, one frame per source per call.
Modes (the outputs of each call):
  yuyv        YUYV + mask, BGR format (the composite);
  bgra        BGRA + mask (no background is read);
  bgra_yuyv   BGRA + YUYV + mask;
  bgra_tail   BGRA + mask with a 640x360 horizontally flipped output (k_tail flips and resizes the staged BGRA).
Throughput: CUDA events around `rounds` rounds after `warmup`; frames/s = frames per round * rounds / time, `runs` times.
With --profile-dir, a separate torch.profiler run gives the time per call of k_post_tma and k_tail.
post_bytes_per_call: DRAM-side bytes per call of the post kernel and the tail from the shapes: the camera tile is read for
every tile in BGRA modes (an upper bound for the composite, which reads it only where a tile can contain a person);
background BGR and cached YUYV tiles are read by calls that blend; outputs are written once; the tail reads the staged
BGRA once (an upper bound when it down-scales).  Prints one JSON line per (setup, mode), with the GPU name and power
limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.source_effects_bench import gpu_info  # noqa: E402

W, H = 1280, 720
STREAMS, BATCH, SOURCES = 8, 32, 64
TAIL = (640, 360)
MODES = ("yuyv", "bgra", "bgra_yuyv", "bgra_tail")
TAGS = ("k_post_tma", "k_tail")


def post_bytes(mode, n):
    npx = W * H
    cam, bg, vid, mask, bgra = npx * 2, npx * 3, npx * 2, npx, npx * 4
    if mode == "yuyv":
        reads, writes = cam + bg + vid, vid + mask
    elif mode == "bgra":
        reads, writes = cam, bgra + mask
    elif mode == "bgra_yuyv":
        reads, writes = cam + bg + vid, bgra + vid + mask
    else:
        reads, writes = cam + bgra, bgra + mask + TAIL[0] * TAIL[1] * 4
    return {"reads": n * reads, "writes": n * writes, "total": n * (reads + writes)}


def make_ctx(lib, setup, mode):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    mb = SOURCES if setup == "sources" else BATCH
    g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=mb)
    g.set_background(synth.background())
    if setup == "sources":
        g.set_sources(SOURCES)
    if mode != "yuyv":
        g.set_out_format("bgra")
    if mode == "bgra_tail":
        g.set_output(True, False, TAIL)
    return g


class Setup:
    def __init__(self, torch, lib, setup, mode):
        from tests import synth
        self.torch, self.setup, self.mode = torch, setup, mode
        n_ctx = 1 if setup == "sources" else STREAMS
        self.n = SOURCES if setup == "sources" else BATCH
        self.ctxs = [make_ctx(lib, setup, mode) for _ in range(n_ctx)]
        dev = "cuda:0"
        host = np.stack([synth.yuyv_frame(W, H, t=0, stream=s) for s in range(self.n)])
        ow, oh = TAIL if mode == "bgra_tail" else (W, H)
        self.bufs = []
        for _ in self.ctxs:
            d_in = torch.from_numpy(host).to(dev)
            d_out = torch.empty((self.n, oh, ow, 4), dtype=torch.uint8, device=dev) if mode != "yuyv" else None
            d_vid = torch.empty((self.n, oh, ow, 2), dtype=torch.uint8, device=dev) if mode in ("yuyv", "bgra_yuyv") else None
            d_mask = torch.empty((self.n, H, W), dtype=torch.uint8, device=dev)
            self.bufs.append((d_in, d_out, d_vid, d_mask))
        self.streams = [torch.cuda.ExternalStream(g.stream) for g in self.ctxs]

    def round(self):
        ids = list(range(self.n))
        for g, (d_in, d_out, d_vid, d_mask) in zip(self.ctxs, self.bufs):
            o = d_out.data_ptr() if d_out is not None else 0
            v = d_vid.data_ptr() if d_vid is not None else 0
            if self.setup == "sources":
                g.composite_sources_yuyv_device(self.n, ids, d_in.data_ptr(), o, v, d_mask.data_ptr())
            else:
                g.composite_yuyv_device(self.n, d_in.data_ptr(), o, v, d_mask.data_ptr())

    def sync(self):
        for g in self.ctxs:
            g.synchronize()

    def close(self):
        for g in self.ctxs:
            g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--setups", default="plain,sources")
    ap.add_argument("--modes", default=",".join(MODES))
    ap.add_argument("--profile-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bgra_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bs.lib()
    info = gpu_info(0)
    for setup in args.setups.split(","):
        for mode in args.modes.split(","):
            st = Setup(torch, lib, setup, mode)
            for _ in range(args.warmup):
                st.round()
            st.sync()
            frames = st.n * len(st.ctxs)
            rates = []
            for _ in range(args.runs):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.rounds):
                    st.round()
                # the default stream's end event waits for every context's stream
                for s in st.streams:
                    ev = torch.cuda.Event()
                    ev.record(s)
                    torch.cuda.current_stream().wait_event(ev)
                e1.record()
                e1.synchronize()
                rates.append(frames * args.rounds / (e0.elapsed_time(e1) / 1e3))
            res = {"setup": setup, "mode": mode, "frames_per_call": st.n, "contexts": len(st.ctxs),
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "native": st.ctxs[0].yuyv_native, "launches_per_call": st.ctxs[0].launches_per_call,
                   "post_bytes_per_call": post_bytes(mode, st.n), **info}
            if args.profile_dir:
                from torch.profiler import ProfilerActivity, profile
                os.makedirs(args.profile_dir, exist_ok=True)
                rounds = 10
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(rounds):
                        st.round()
                    st.sync()
                per = {}
                for ev in prof.key_averages():
                    tot = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    for tag in TAGS:
                        if tag in ev.key:
                            per[tag] = round(per.get(tag, 0.0) + tot / (rounds * len(st.ctxs)), 1)
                res["us_per_call"] = per
                prof.export_chrome_trace(os.path.join(args.profile_dir, f"bgra_trace_{setup}_{mode}.json"))
            print(json.dumps(res), flush=True)
            st.close()


if __name__ == "__main__":
    main()
