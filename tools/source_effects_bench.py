#!/usr/bin/env python
"""Per-source background effects at scale: one Meet context with 64 sources, one call of one frame per source.

    python tools/source_effects_bench.py [--rounds 40] [--warmup 5] [--runs 3] [--lib PATH] [--mixes own,mixed,blur]
                                         [--formats yuyv,nv12] [--context-blur] [--profile-dir DIR]

Meet full (segm_full_v679), 1280x720, 64 sources in one context, camera frames resident on the device (YUYV, or NV12
packed).  Effect mixes:
  own    every source blends its own image;
  mixed  a third camera blur at k = 25, a third their own image, a third the context image;
  blur   every source camera blur at k = 25.
--context-blur sets the blur mix up the way a context without per-source effects must: bsb_set_bgblur(25) and no
background at all (what the parent of bsb_set_source_effect can run; with --lib, the library of another build).
Throughput: CUDA events around `rounds` calls after `warmup`; frames/s = 64 * rounds / time, `runs` times per mix.
With --profile-dir, a separate torch.profiler run per mix gives the Gaussian's and k_post_tma's time per call.
Prints one JSON line per (mix, format), with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MODEL = "segm_full_v679.tflite"
W, H, S = 1280, 720, 64


def gpu_info(dev):
    import torch
    info = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", str(dev)],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(out[0])
        info["sm_max_mhz"] = float(out[1])
    except Exception:
        pass
    return info


class _Missing:
    """a symbol the bound library lacks: binding it is harmless, calling it fails with its name"""

    def __init__(self, path, name):
        self.path, self.name, self.argtypes, self.restype = path, name, None, None

    def __call__(self, *args):
        raise RuntimeError(f"{self.path} has no {self.name}")


def bind_older(path):
    """_binding.bind on the library of an earlier build, which may lack symbols added since (bsb_set_source_effect)"""
    import ctypes
    from backscrub_b200 import _binding
    lib = ctypes.CDLL(path)
    for name in _binding.SYMBOLS:
        if not hasattr(lib, name):
            setattr(lib, name, _Missing(path, name))
    orig = ctypes.CDLL
    ctypes.CDLL = lambda p, *a, **k: lib if p == path else orig(p, *a, **k)   # bind() opens the same, patched handle
    try:
        return _binding.bind(path)
    finally:
        ctypes.CDLL = orig


def frames(fmt):
    from tests import synth
    out = []
    for s in range(S):
        yv = synth.yuyv_frame(W, H, t=0, stream=s)
        out.append(np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0).reshape(-1) if fmt == "nv12" else yv.reshape(-1))
    return np.stack(out)


def make_ctx(lib, mix, context_blur):
    from backscrub_b200 import api
    from tests import synth
    from tests.conftest import model_path
    g = api.MaskGen(lib, model_path("meet_full"), W, H, max_batch=S)
    bg = synth.background()
    if context_blur:
        if mix != "blur":
            raise SystemExit("--context-blur runs the blur mix only")
        g.set_bgblur(25)
        g.set_sources(S)
        return g
    g.set_background(bg[::-1].copy())
    g.set_sources(S)
    for s in range(S):
        if mix == "own" or (mix == "mixed" and s % 3 == 1):
            g.set_source_background(s, np.roll(bg, 37 * s, axis=1))
        if mix == "blur" or (mix == "mixed" and s % 3 == 0):
            g.set_source_effect(s, "none", 25)
    return g


def run_calls(torch, g, fmt, d_in, d_out, d_vid, d_mask, n):
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
    ap.add_argument("--lib", default=None, help="library to bind (default: the package's)")
    ap.add_argument("--mixes", default="own,mixed,blur")
    ap.add_argument("--formats", default="yuyv,nv12")
    ap.add_argument("--context-blur", action="store_true")
    ap.add_argument("--profile-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("source_effects_bench needs a CUDA device")
    import backscrub_b200 as bs
    lib = bind_older(args.lib) if args.lib else bs.lib()
    info = gpu_info(0)
    dev = "cuda:0"
    for fmt in args.formats.split(","):
        host = frames(fmt)
        d_in = torch.from_numpy(host).to(dev)
        d_out = torch.empty((S, H, W, 3), dtype=torch.uint8, device=dev)
        d_vid = torch.empty(S * (W * H * 3 // 2 if fmt == "nv12" else W * H * 2), dtype=torch.uint8, device=dev)
        d_mask = torch.empty((S, H, W), dtype=torch.uint8, device=dev)
        for mix in args.mixes.split(","):
            g = make_ctx(lib, mix, args.context_blur)
            stream = torch.cuda.ExternalStream(g.stream)
            run_calls(torch, g, fmt, d_in, d_out, d_vid, d_mask, args.warmup)
            g.synchronize()
            native = g.yuyv_native
            rates = []
            for _ in range(args.runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                run_calls(torch, g, fmt, d_in, d_out, d_vid, d_mask, args.rounds)
                e1.record(stream)
                e1.synchronize()
                rates.append(S * args.rounds / (e0.elapsed_time(e1) / 1e3))
            res = {"mix": mix, "format": fmt, "context_blur": args.context_blur, "lib": args.lib or "package", "sources": S,
                   "frames_per_s": [round(r, 1) for r in rates], "median_frames_per_s": round(float(np.median(rates)), 1),
                   "native": native, **info}
            if args.profile_dir:
                from torch.profiler import ProfilerActivity, profile
                os.makedirs(args.profile_dir, exist_ok=True)
                calls = 10
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run_calls(torch, g, fmt, d_in, d_out, d_vid, d_mask, calls)
                    g.synchronize()
                per = {}
                for ev in prof.key_averages():
                    name = ev.key
                    tot = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    for tag in ("k_gauss", "k_post_tma", "k_yuyv_to_bgr", "k_nv12_to_bgr"):
                        if tag in name:
                            per[name.split("(")[0][-60:]] = round(tot / calls, 1)
                res["us_per_call"] = per
                prof.export_chrome_trace(os.path.join(args.profile_dir, f"trace_{mix}_{fmt}{'_ctx' if args.context_blur else ''}.json"))
            print(json.dumps(res), flush=True)
            g.close()


if __name__ == "__main__":
    main()
