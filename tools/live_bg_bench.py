#!/usr/bin/env python
"""Live backgrounds against still and host-set backgrounds, on device-resident camera frames.

    python tools/live_bg_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--cams yuyv,nv12] [--configs ...] [--bgblur 0]
                                  [--profile-dir DIR] [--lib PATH]

Meet full (segm_full_v679), 1280x720.  Configurations:
  still        one context, 64 sources, each with its own still (set once);
  live_nv12    the same, each source with a live 1920x1080 NV12 surface, a new surface every call
               (bsb_set_source_live_background before every call; two surfaces per source alternate);
  live_bgr     the same with live 1280x720 BGR images;
  host_set     the same backgrounds as live_bgr, set by bsb_set_source_background from host memory before every call;
  plain_live   8 plain contexts, 32 frames per call, frame b a live 1920x1080 NV12 surface of its own (frame_stride one
               surface), calls of the 8 contexts interleaved;
  plain_still  the same 8 x 32 with the context's still.
Throughput: CUDA events around `rounds` rounds after `warmup`; frames/s = frames per round * rounds / time, `runs` times.
With --profile-dir, a separate torch.profiler run gives the time per call of k_live_bg and k_post_tma.
live_bytes_per_call: the bytes k_live_bg moves per call from the shapes (live pixels read once, the slot's BGR and its
YUYV / NV12 written; plain slots have no cache).  --lib runs another build of the library.  Prints one JSON line per
(camera format, configuration), with the GPU name and power limit read in the same run."""
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
LIVE_NV12, LIVE_BGR = (1920, 1080), (1280, 720)
CONFIGS = ("still", "live_nv12", "live_bgr", "host_set", "plain_live", "plain_still")
TAGS = ("k_live_bg", "k_post_tma")


def live_bytes(config, cam, n):
    """bytes k_live_bg reads and writes per call of n frames"""
    npx = W * H
    cache = 0 if config.startswith("plain") else (npx * 3 // 2 if cam == "nv12" else npx * 2)
    if config in ("live_nv12", "plain_live"):
        reads = LIVE_NV12[0] * LIVE_NV12[1] * 3 // 2
    elif config == "live_bgr":
        reads = LIVE_BGR[0] * LIVE_BGR[1] * 3
    else:
        return {"reads": 0, "writes": 0, "total": 0}
    writes = npx * 3 + cache
    return {"reads": n * reads, "writes": n * writes, "total": n * (reads + writes)}


def nv12_surface(w, h, seed):
    from tests import synth
    yv = synth.yuyv_frame(w, h, t=seed, stream=3)
    return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)


def bgr_image(w, h, seed):
    import cv2
    from tests import synth
    return np.ascontiguousarray(np.roll(cv2.resize(synth.background(), (w, h)), 41 * seed, axis=1))


class Setup:
    def __init__(self, torch, lib, cam, config, bgblur):
        from backscrub_b200 import api
        from tests import synth
        from tests.conftest import model_path
        self.torch, self.cam, self.config = torch, cam, config
        dev = "cuda:0"
        plain = config.startswith("plain")
        n_ctx = STREAMS if plain else 1
        self.n = BATCH if plain else SOURCES
        self.ctxs = []
        for _ in range(n_ctx):
            g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=self.n)
            g.set_background(synth.background())
            g.set_bgblur(bgblur)
            if not plain:
                g.set_sources(SOURCES)
            self.ctxs.append(g)
        self.i = 0
        self.live = []                                        # device surfaces: [2][n] per source, or one block per context
        if config == "still":
            for s in range(SOURCES):
                self.ctxs[0].set_source_background(s, bgr_image(*LIVE_BGR, s))
        elif config in ("live_nv12", "live_bgr"):
            size = LIVE_NV12 if config == "live_nv12" else LIVE_BGR
            make = nv12_surface if config == "live_nv12" else bgr_image
            base = [make(*size, j) for j in range(4)]
            self.live = [[torch.from_numpy(base[(2 * k + s) % 4].reshape(-1).copy()).to(dev) for s in range(SOURCES)] for k in range(2)]
        elif config == "host_set":
            self.host = [[bgr_image(*LIVE_BGR, (2 * k + s) % 4) for s in range(SOURCES)] for k in range(2)]
        elif config == "plain_live":
            surf = np.stack([nv12_surface(*LIVE_NV12, j) for j in range(4)])
            fb = surf[0].size
            for g in self.ctxs:
                d = torch.from_numpy(np.concatenate([surf[b % 4].reshape(-1) for b in range(self.n)])).to(dev)
                g.set_live_background(d, "nv12", LIVE_NV12, frame_stride=fb)
                self.live.append(d)
        if cam == "nv12":
            host = np.stack([nv12_surface(W, H, s) for s in range(self.n)])
        else:
            host = np.stack([synth.yuyv_frame(W, H, t=0, stream=s) for s in range(self.n)])
        self.bufs = []
        for _ in self.ctxs:
            d_in = torch.from_numpy(host).to(dev)
            vb = W * H * 3 // 2 if cam == "nv12" else W * H * 2
            d_vid = torch.empty(self.n * vb, dtype=torch.uint8, device=dev)
            d_mask = torch.empty((self.n, H, W), dtype=torch.uint8, device=dev)
            self.bufs.append((d_in, d_vid, d_mask))
        self.streams = [torch.cuda.ExternalStream(g.stream) for g in self.ctxs]

    def round(self):
        ids = list(range(self.n))
        k = self.i & 1
        self.i += 1
        for g, (d_in, d_vid, d_mask) in zip(self.ctxs, self.bufs):
            if self.config in ("live_nv12", "live_bgr"):
                fmt, size = ("nv12", LIVE_NV12) if self.config == "live_nv12" else ("bgr", LIVE_BGR)
                for s in ids:
                    g.set_source_live_background(s, self.live[k][s], fmt, size)
            elif self.config == "host_set":
                for s in ids:
                    g.set_source_background(s, self.host[k][s])
            args = (self.n,) if self.config.startswith("plain") else (self.n, ids)
            if self.cam == "nv12":
                f = g.composite_nv12_device if self.config.startswith("plain") else g.composite_sources_nv12_device
            else:
                f = g.composite_yuyv_device if self.config.startswith("plain") else g.composite_sources_yuyv_device
            f(*args, d_in.data_ptr(), 0, d_vid.data_ptr(), d_mask.data_ptr())

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
    ap.add_argument("--cams", default="yuyv,nv12")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--bgblur", type=int, default=0)
    ap.add_argument("--profile-dir", default=None)
    ap.add_argument("--lib", default=None, help="another build of libbackscrub_b200.so")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("live_bg_bench needs a CUDA device")
    import backscrub_b200 as bs
    from backscrub_b200 import _binding
    lib = _binding.bind(os.path.abspath(args.lib)) if args.lib else bs.lib()
    info = gpu_info(0)
    for cam in args.cams.split(","):
        for config in args.configs.split(","):
            st = Setup(torch, lib, cam, config, args.bgblur)
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
            res = {"cam": cam, "config": config, "frames_per_call": st.n, "contexts": len(st.ctxs), "bgblur": args.bgblur,
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "launches_per_call": st.ctxs[0].launches_per_call, "live_bytes_per_call": live_bytes(config, cam, st.n), **info}
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
                if "k_live_bg" in per and per["k_live_bg"] > 0:
                    res["k_live_bg_GB_per_s"] = round(res["live_bytes_per_call"]["total"] / (per["k_live_bg"] * 1e3), 1)
            print(json.dumps(res), flush=True)
            st.close()


if __name__ == "__main__":
    main()
