#!/usr/bin/env python
"""Per-kernel time shares of one call.

    python tools/launch_shares.py --profile --out DIR [--frames 256 32] [--calls 20] [--warmup 5] [--model M]
    python tools/launch_shares.py TRACE.json [--list]      # a torch.profiler chrome trace written by --profile
    python tools/launch_shares.py NCU.csv [--list]         # an `ncu --metrics gpu__time_duration.sum --csv` launch list

--profile: one Meet context (1280x720 camera YUYV frames resident on the device, max_batch = the largest --frames).
For each n in --frames: `warmup` calls, then `calls` calls captured with torch.profiler (CUDA activities only),
written to DIR/launch_shares_<model>_n<n>.pt.trace.json.  From each trace: per kernel, its time per call (sum of its
launches, median over the calls), share of the summed kernel time of a call and launches per call; and the encoder
blocks ahead of k_chain (the launches after the last squeeze-excite pool launch before k_chain) as one group.  At a
batch where every kernel fills the GPU the durations approximate SM-time shares.  Prints the GPU name and power limit
read in the same run, and one JSON line per n."""
import argparse
import collections
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

W, H = 1280, 720
DISTINCT_FRAMES = 8
FIRST = "k_resize_roi_swap"          # first kernel of a call
SE = ("k_rowsum", "k_pool_fc")      # squeeze-excite pool launches (k_rowsum, k_rowsum_fc, k_pool_fc)


def base_name(n):
    return n.split("(")[0].replace("void ", "").replace("bsb::", "").strip()


def calls_from_trace(path):
    """[[(kernel, us), ...] per call] from a torch.profiler chrome trace, in start order"""
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    ks = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    return split_calls([(base_name(e["name"]), float(e["dur"])) for e in ks])


def calls_from_ncu(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    rows = []
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(row["Metric Value"].replace(",", "")); unit = row["Metric Unit"]
        if unit in ("nsecond", "ns"): v /= 1e3
        elif unit in ("msecond", "ms"): v *= 1e3
        elif unit not in ("usecond", "us"): v /= 1e3
        rows.append((base_name(row["Kernel Name"]), v))
    return split_calls(rows)[1:]          # the first call of an ncu list is cold


def split_calls(launches):
    starts = [i for i, (n, _) in enumerate(launches) if n.startswith(FIRST)]
    return [launches[a:b] for a, b in zip(starts, starts[1:] + [len(launches)])]


def encoder_group(call):
    """indices of the launches between the last SE pool launch before k_chain and k_chain"""
    chain = [i for i, (n, _) in enumerate(call) if n.startswith("k_chain")]
    if not chain:
        return []
    se = [i for i in range(chain[0]) if call[i][0].startswith(SE)]
    return list(range(se[-1] + 1, chain[0])) if se else []


def median(v):
    v = sorted(v); m = len(v) // 2
    return v[m] if len(v) % 2 else 0.5 * (v[m - 1] + v[m])


def summarize(calls, list_launches=False, label=""):
    shapes = collections.Counter(tuple(n for n, _ in c) for c in calls)
    seq, n_same = shapes.most_common(1)[0]
    calls = [c for c in calls if tuple(n for n, _ in c) == seq]     # every call of a graph replay has the same list
    tot = [sum(v for _, v in c) for c in calls]
    per = collections.defaultdict(list)
    for c in calls:
        agg = collections.defaultdict(float)
        for n, v in c: agg[n] += v
        for n, v in agg.items(): per[n].append(v)
    count = collections.Counter(seq)
    T = median(tot)
    grp = encoder_group(calls[0])
    g_us = median([sum(c[i][1] for i in grp) for c in calls]) if grp else 0.0
    print(f"{label}{len(seq)} launches per call, {len(calls)} calls; summed kernel time per call {T:.1f} us (median)")
    for n in sorted(per, key=lambda n: -median(per[n])):
        print(f"  {n[:60]:60s} x{count[n]:3d} {median(per[n]):9.1f} us {100 * median(per[n]) / T:5.1f}%")
    if grp:
        print(f"  encoder blocks ahead of k_chain: {len(grp)} launches, {g_us:.1f} us per call, {100 * g_us / T:.1f}%")
        for i in grp:
            print(f"    #{i:2d} {seq[i][:56]:56s} {median([c[i][1] for c in calls]):8.1f} us")
    if list_launches:
        for i, n in enumerate(seq):
            print(f"  {i:3d} {n[:60]:60s} {median([c[i][1] for c in calls]):8.1f} us")
    return {"launches_per_call": len(seq), "calls": len(calls), "kernel_us_per_call": round(T, 2),
            "kernels": {n: {"us": round(median(per[n]), 2), "share": round(median(per[n]) / T, 4), "launches": count[n]}
                        for n in sorted(per, key=lambda n: -median(per[n]))},
            "encoder_blocks": {"launches": [seq[i] for i in grp], "us": round(g_us, 2), "share": round(g_us / T, 4) if T else 0.0}}


def profile(args):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    import backscrub_b200 as bs
    from tests import synth
    from tools.sources_bench import gpu_info

    if bs.device_count() <= 0:
        raise SystemExit("launch_shares --profile needs a CUDA device")
    dev = args.device
    torch.cuda.set_device(dev)
    os.makedirs(args.out, exist_ok=True)
    info = gpu_info(dev)
    print(f"GPU {info['gpu']}, power limit {info['power_limit_w']} W")
    n_max = max(args.frames)
    cuda = f"cuda:{dev}"
    base = np.stack([synth.yuyv_frame(W, H, t=t) for t in range(DISTINCT_FRAMES)])
    frames = torch.from_numpy(base).to(cuda).repeat((n_max + DISTINCT_FRAMES - 1) // DISTINCT_FRAMES, 1, 1, 1)[:n_max].contiguous()
    d_out = torch.empty((n_max, H, W, 3), dtype=torch.uint8, device=cuda)
    d_yuyv = torch.empty((n_max, H, W, 2), dtype=torch.uint8, device=cuda)
    d_mask = torch.empty((n_max, H, W), dtype=torch.uint8, device=cuda)
    g = bs.bs_maskgen_new(os.path.join(ROOT, "models", args.model), 2, W, H, device=dev, max_batch=n_max)
    g.set_background(synth.background())
    stem = os.path.splitext(args.model)[0]
    for n in args.frames:
        for _ in range(args.warmup):
            g.composite_yuyv_device(n, frames.data_ptr(), d_out.data_ptr(), d_yuyv.data_ptr(), d_mask.data_ptr())
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                g.composite_yuyv_device(n, frames.data_ptr(), d_out.data_ptr(), d_yuyv.data_ptr(), d_mask.data_ptr())
            torch.cuda.synchronize()
        path = os.path.join(args.out, f"launch_shares_{stem}_n{n}.pt.trace.json")
        prof.export_chrome_trace(path)
        res = summarize(calls_from_trace(path), args.list, label=f"{args.model} {W}x{H}, {n} frames per call: ")
        print(json.dumps({"tool": "launch_shares", **info, "model": args.model, "frame": f"{W}x{H}", "frames_per_call": n,
                          "trace": os.path.basename(path), **res}))
    g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("path", nargs="?", help="a torch.profiler chrome trace (.json) or an ncu CSV launch list")
    ap.add_argument("--list", action="store_true", help="also print every launch of the call in order")
    ap.add_argument("--profile", action="store_true", help="profile a Meet context on the GPU")
    ap.add_argument("--out", help="directory for the profiler traces (--profile)")
    ap.add_argument("--frames", type=int, nargs="+", default=[256, 32])
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--model", default="segm_full_v679.tflite")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    if args.profile:
        if not args.out:
            raise SystemExit("--profile needs --out")
        profile(args)
    elif args.path:
        calls = calls_from_trace(args.path) if args.path.endswith(".json") else calls_from_ncu(args.path)
        summarize(calls, args.list)
    else:
        ap.error("give a trace / CSV path or --profile")


if __name__ == "__main__":
    main()
