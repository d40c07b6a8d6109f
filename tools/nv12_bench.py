#!/usr/bin/env python
"""YUYV against NV12 camera frames through the fused path: frames/s, the post kernel's time and bytes, and a sources line.

    python tools/nv12_bench.py [--steps 10] [--warmup 3] [--runs 3] [--profile-calls 20] [--sources 64]

Meet full (segm_full_v679), 1280x720, bench.py's default shape: 8 streams (one context each) x 32 frames per call, 20
calls per stream per step.  The camera frames of each format sit on the device in a ring of 32-frame batches larger than
2x the 50 MB L2, made from the same tests.synth frames (the NV12 frames carry the Y plane and the even rows' UV pairs of
the YUYV frames).
  * yuyv: composite_yuyv_device, YUYV in -> YUYV + mask out
  * nv12: composite_nv12_device, NV12 in -> NV12 + mask out
Runs alternate between the formats, `--runs` of each; frames/s = frames / (CUDA-event time of `steps` steps).
Post kernel: a separate torch.profiler run of `--profile-calls` calls per format on one context; the k_post_tma time per
call, and bytes/s on the algorithmic bytes of the stage: camera frame read (2 or 1.5 B/px), video written (2 or 1.5 B/px)
and mask written (1 B/px) — the background and the small mask are L2-resident and not counted.
Sources: one context with set_sources(S), calls of S frames (one per camera), each format.
Prints one JSON line with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.sources_bench import gpu_info  # noqa: E402

MODEL = "segm_full_v679.tflite"
W, H = 1280, 720
STREAMS, BATCH, CALLS = 8, 32, 20
L2_BYTES = 50 << 20
FMT_BYTES = {"yuyv": 2.0, "nv12": 1.5}


def rings(torch, dev):
    """device rings of 32-frame batches per format, each > 2x L2"""
    from tests import synth
    yv = np.stack([synth.yuyv_frame(W, H, t=t) for t in range(BATCH)])
    nv = np.concatenate([yv[..., 0], yv[:, 0::2, :, 1]], axis=1)          # [B, H*3/2, W]
    out = {}
    for name, base in (("yuyv", yv), ("nv12", nv)):
        nb = -(-2 * L2_BYTES // base.nbytes) + 1
        out[name] = [torch.from_numpy(np.roll(base, 2 * k, axis=-1 if name == "nv12" else -2).copy()).to(dev) for k in range(nb)]
    return out


class Ctx:
    def __init__(self, bs, torch, dev, model, bg, n, sources=0):
        self.g = bs.bs_maskgen_new(model, 2, W, H, device=dev, max_batch=n)
        d = f"cuda:{dev}"
        self.g.set_background(bg)
        if sources:
            self.g.set_sources(sources)
        self.n = n
        self.stream = torch.cuda.ExternalStream(self.g.stream, device=dev)
        self.mask = torch.empty((n, H, W), dtype=torch.uint8, device=d)
        self.vid = torch.empty(n * W * H * 2, dtype=torch.uint8, device=d)

    def call(self, fmt, frames, ids=None):
        if ids is not None and fmt == "nv12":
            self.g.composite_sources_nv12_device(self.n, ids, frames.data_ptr(), 0, self.vid.data_ptr(), self.mask.data_ptr())
        elif ids is not None:
            self.g.composite_sources_yuyv_device(self.n, ids, frames.data_ptr(), 0, self.vid.data_ptr(), self.mask.data_ptr())
        elif fmt == "nv12":
            self.g.composite_nv12_device(self.n, frames.data_ptr(), 0, self.vid.data_ptr(), self.mask.data_ptr())
        else:
            self.g.composite_yuyv_device(self.n, frames.data_ptr(), 0, self.vid.data_ptr(), self.mask.data_ptr())


def timed(torch, ctxs, fmt, ring, steps, warmup, ids=None, calls=CALLS):
    def step(k):
        for c in range(calls):
            for s, x in enumerate(ctxs):
                x.call(fmt, ring[(k * calls + c + s) % len(ring)], ids)

    for k in range(warmup):
        step(k)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e0.record(ctxs[0].stream)
    for x in ctxs[1:]:
        x.stream.wait_event(e0)
    for k in range(steps):
        step(warmup + k)
    ends = []
    for x in ctxs:
        e = torch.cuda.Event(enable_timing=True)
        e.record(x.stream)
        ends.append(e)
    torch.cuda.synchronize()
    ms = max(e0.elapsed_time(e) for e in ends)
    return len(ctxs) * steps * calls * ctxs[0].n / (ms * 1e-3)


def post_profile(torch, ctx, fmt, ring, calls):
    from torch.profiler import ProfilerActivity, profile
    for k in range(3):
        ctx.call(fmt, ring[k % len(ring)])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(calls):
            ctx.call(fmt, ring[k % len(ring)])
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if e.key.startswith("void bsb::k_post_tma"))
    kinds = sorted({e.key.split("(")[0] for e in prof.key_averages() if "k_post_tma" in e.key})
    per_call_us = us / calls
    px = W * H * ctx.n
    alg_bytes = px * (2 * FMT_BYTES[fmt] + 1.0)
    return {"k_post_tma_us_per_call": round(per_call_us, 2), "kernels": kinds, "algorithmic_bytes_per_call": int(alg_bytes),
            "achieved_GBps": round(alg_bytes / (per_call_us * 1e-6) / 1e9, 1) if per_call_us else None,
            "yuyv_native": bool(ctx.g.yuyv_native)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--profile-calls", type=int, default=20)
    ap.add_argument("--sources", type=int, default=64)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch

    import backscrub_b200 as bs
    from tests import synth

    if bs.device_count() <= 0:
        raise SystemExit("nv12_bench needs a CUDA device")
    dev = args.device
    torch.cuda.set_device(dev)
    d = f"cuda:{dev}"
    model = os.path.join(ROOT, "models", MODEL)
    bg = synth.background()
    ring = rings(torch, d)
    ctxs = [Ctx(bs, torch, dev, model, bg, BATCH) for _ in range(STREAMS)]
    fps = {"yuyv": [], "nv12": []}
    for _ in range(args.runs):
        for fmt in ("yuyv", "nv12"):
            fps[fmt].append(timed(torch, ctxs, fmt, ring[fmt], args.steps, args.warmup))
    native = {f: None for f in fps}
    for fmt in fps:
        ctxs[0].call(fmt, ring[fmt][0])
        torch.cuda.synchronize()
        native[fmt] = bool(ctxs[0].g.yuyv_native)
    summary = {f: {"median_frames_per_s": round(float(np.median(v)), 1), "range": [round(min(v), 1), round(max(v), 1)],
                   "runs": [round(x, 1) for x in v], "read_in_place": native[f]} for f, v in fps.items()}
    prof = {f: post_profile(torch, ctxs[0], f, ring[f], args.profile_calls) for f in fps}
    for x in ctxs:
        x.g.close()

    S = args.sources
    from tools.sources_bench import camera_frames
    yv = camera_frames(S, 1)[0]                                                     # [S, H, W, 2]
    src_ring = {"yuyv": [torch.from_numpy(yv).to(d)],
                "nv12": [torch.from_numpy(np.concatenate([yv[..., 0], yv[:, 0::2, :, 1]], axis=1).copy()).to(d)]}
    sc = Ctx(bs, torch, dev, model, bg, S, sources=S)
    ids = list(range(S))
    src = {f: round(timed(torch, [sc], f, src_ring[f], args.steps, args.warmup, ids=ids, calls=5), 1) for f in ("yuyv", "nv12")}
    sc.g.close()
    out = {"tool": "nv12_bench", **gpu_info(dev), "model": MODEL, "frame": f"{W}x{H}", "streams": STREAMS, "frames_per_call": BATCH,
           "calls_per_stream_per_step": CALLS, "steps": args.steps, "outputs": "video (YUYV or NV12) + mask", "frames_per_s": summary,
           "nv12_over_yuyv": round(summary["nv12"]["median_frames_per_s"] / summary["yuyv"]["median_frames_per_s"], 4),
           "post_kernel": prof, "sources": {"cameras": S, "frames_per_call": S, "frames_per_s": src}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
