#!/usr/bin/env python
"""SM time of the low-resolution chain kernel (k_chain, kernels_chain.cu) per Meet frame.

    python tools/chain_bench.py --out DIR [--calls 30] [--warmup 5] [--lib PATH]

One Meet full context (segm_full_v679, 1280x720 camera YUYV frames resident on the device) with max_batch = 2 x SMs.
For n = SMs and n = 2 x SMs frames per call: `warmup` calls, then `calls` calls captured with torch.profiler (CUDA
activities only), one capture per n, written to DIR/chain_bench_n<n>.pt.trace.json.  From each trace: the median,
min and max k_chain duration per call, and the chain's SM time per frame = median x SMs / n.

With one CTA per SM the 2 x SMs call takes about twice the SMs call; with two co-resident CTAs per SM it takes
clearly less.  With --lib (the library of another build, e.g. the parent of a chain change) that library is timed
instead of the package's, so two builds can be run alternately in one session.  Prints one JSON line, with the GPU name
and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MODEL = "segm_full_v679.tflite"
W, H = 1280, 720
DISTINCT_FRAMES = 8


def chain_durations_us(trace_path):
    """durations (us) of every k_chain kernel in a torch.profiler chrome trace, in start order"""
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    ks = [e for e in events if e.get("cat") == "kernel" and "k_chain<" in e.get("name", "")]
    return [float(e["dur"]) for e in sorted(ks, key=lambda e: e["ts"])], sorted({e["name"] for e in ks})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the profiler traces")
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--lib", default=None, help="library of another build (default: the package's)")
    args = ap.parse_args()
    if args.calls < 20:
        raise SystemExit("--calls must be >= 20")

    import torch
    from torch.profiler import ProfilerActivity, profile

    import backscrub_b200 as bs
    from backscrub_b200 import api
    from tests import synth
    from tools.source_effects_bench import bind_older
    from tools.sources_bench import gpu_info

    if bs.device_count() <= 0:
        raise SystemExit("chain_bench needs a CUDA device")
    dev = args.device
    torch.cuda.set_device(dev)
    os.makedirs(args.out, exist_ok=True)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    n_max = 2 * sms
    cuda = f"cuda:{dev}"
    base = np.stack([synth.yuyv_frame(W, H, t=t) for t in range(DISTINCT_FRAMES)])
    frames = torch.from_numpy(base).to(cuda).repeat((n_max + DISTINCT_FRAMES - 1) // DISTINCT_FRAMES, 1, 1, 1)[:n_max].contiguous()
    d_out = torch.empty((n_max, H, W, 3), dtype=torch.uint8, device=cuda)
    d_yuyv = torch.empty((n_max, H, W, 2), dtype=torch.uint8, device=cuda)
    d_mask = torch.empty((n_max, H, W), dtype=torch.uint8, device=cuda)
    lib = bind_older(args.lib) if args.lib else bs.lib()
    g = api.MaskGen(lib, os.path.join(ROOT, "models", MODEL), W, H, device=dev, max_batch=n_max)
    g.set_background(synth.background())

    def call(n):
        g.composite_yuyv_device(n, frames.data_ptr(), d_out.data_ptr(), d_yuyv.data_ptr(), d_mask.data_ptr())

    res = []
    for n in (sms, n_max):
        for _ in range(args.warmup):
            call(n)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                call(n)
            torch.cuda.synchronize()
        tag = "_" + os.path.splitext(os.path.basename(args.lib))[0] if args.lib else ""
        path = os.path.join(args.out, f"chain_bench{tag}_n{n}.pt.trace.json")
        prof.export_chrome_trace(path)
        durs, names = chain_durations_us(path)
        if len(durs) != args.calls:
            raise SystemExit(f"expected {args.calls} k_chain kernels in {path}, found {len(durs)}")
        med = float(np.median(durs))
        res.append({"frames_per_call": n, "calls": len(durs), "kernel": names,
                    "k_chain_us_median": round(med, 2), "k_chain_us_min": round(min(durs), 2), "k_chain_us_max": round(max(durs), 2),
                    "chain_sm_us_per_frame": round(med * sms / n, 3), "trace": os.path.basename(path)})
    g.close()
    out = {"tool": "chain_bench", "lib": args.lib or "package", **gpu_info(dev), "sms": sms, "model": MODEL, "frame": f"{W}x{H}",
           "input": "device-resident camera YUYV", "warmup_calls": args.warmup, "results": res,
           "ratio_2x_sms_over_sms_call": round(res[1]["k_chain_us_median"] / res[0]["k_chain_us_median"], 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
