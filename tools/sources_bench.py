#!/usr/bin/env python
"""Many live cameras on one GPU: S plain contexts (one per camera, batch-1 calls) against one sources context (one frame
of each camera per call).

    python tools/sources_bench.py [--sources 8,32,128] [--rounds 30] [--warmup 5]

Meet full (segm_full_v679), 1280x720, camera YUYV frames resident on the device.  Every camera has its own frames, in a
ring of R frames per camera with S * R frames > 2x the 50 MB L2, and its own still background.  One round = one frame of
every camera:
  (a) plain:   S contexts, each on its own CUDA stream, each doing one batch-1 bsb_composite_yuyv_device call per round
               (what serving S cameras takes without the sources calls);
  (b) sources: one context with bsb_set_sources(S) doing calls of min(S, 64) frames, one frame per camera.
Throughput: CUDA events around `rounds` rounds after `warmup` rounds; composited frames/s = S * rounds / time.
Per-call time: a second pass with an event pair around every call; the median over the calls, in ms.  Prints one JSON
line, with the GPU name and power limit read in the same run."""
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
W, H = 1280, 720
L2_BYTES = 50 << 20
MAX_CALL = 64


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


def camera_frames(S, R):
    """[R, S, H, W, 2]: frame t of camera s (a moving person, shifted by an even number of pixels per camera)"""
    from tests import synth
    base = [synth.yuyv_frame(W, H, t=t) for t in range(R)]
    out = np.empty((R, S, H, W, 2), np.uint8)
    for t in range(R):
        for s in range(S):
            out[t, s] = np.roll(base[t], 2 * s, axis=1)
    return out


def median_call_ms(torch, launch, streams, n_rounds):
    """event pair around every call of n_rounds rounds; launch(r, k) issues call k of round r on streams[k]"""
    pairs = []
    for r in range(n_rounds):
        for k, st in enumerate(streams):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            launch(r, k)
            e1.record(st)
            pairs.append((e0, e1))
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in pairs]))


def timed_rounds(torch, launch_round, streams, warmup, rounds):
    for r in range(warmup):
        launch_round(r)
    torch.cuda.synchronize()
    ev0 = torch.cuda.Event(enable_timing=True)
    ev0.record(streams[0])
    for st in streams[1:]:
        st.wait_event(ev0)
    for r in range(rounds):
        launch_round(warmup + r)
    ends = []
    for st in streams:
        e = torch.cuda.Event(enable_timing=True)
        e.record(st)
        ends.append(e)
    torch.cuda.synchronize()
    return max(ev0.elapsed_time(e) for e in ends)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sources", default="8,32,128")
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--latency-rounds", type=int, default=10)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

    import torch

    import backscrub_b200 as bs
    from tests import synth

    if bs.device_count() <= 0:
        raise SystemExit("sources_bench needs a CUDA device")
    dev = args.device
    torch.cuda.set_device(dev)
    model = os.path.join(ROOT, "models", MODEL)
    counts = [int(x) for x in args.sources.split(",")]
    s_max = max(counts)
    fr_bytes = W * H * 2
    R = max(2, -(-2 * L2_BYTES // (min(counts) * fr_bytes)))          # ring frames per camera: > 2x L2 at the smallest S
    frames = torch.from_numpy(camera_frames(s_max, R)).to(f"cuda:{dev}")
    d_out = torch.empty((s_max, H, W, 3), dtype=torch.uint8, device=f"cuda:{dev}")
    d_yuyv = torch.empty((s_max, H, W, 2), dtype=torch.uint8, device=f"cuda:{dev}")
    d_mask = torch.empty((s_max, H, W), dtype=torch.uint8, device=f"cuda:{dev}")
    bg = synth.background()
    bgs = [np.roll(bg, 8 * s, axis=1) for s in range(s_max)]

    # (a) one plain context per camera
    plain = []
    for s in range(s_max):
        c = bs.bs_maskgen_new(model, 2, W, H, device=dev, max_batch=1)
        c.set_background(bgs[s])
        plain.append(c)
    plain_streams = [torch.cuda.ExternalStream(c.stream, device=dev) for c in plain]

    res = []
    for S in counts:
        def plain_call(r, s):
            t = r % R
            plain[s].composite_yuyv_device(1, frames[t, s].data_ptr(), d_out[s].data_ptr(), d_yuyv[s].data_ptr(), d_mask[s].data_ptr())

        def plain_round(r):
            for s in range(S):
                plain_call(r, s)

        ms_a = timed_rounds(torch, plain_round, plain_streams[:S], args.warmup, args.rounds)
        call_a = median_call_ms(torch, plain_call, plain_streams[:S], args.latency_rounds)

        # (b) one sources context, calls of min(S, 64) frames
        B = min(S, MAX_CALL)
        g = bs.bs_maskgen_new(model, 2, W, H, device=dev, max_batch=B)
        g.set_background(bg)
        g.set_sources(S)
        for s in range(S):
            g.set_source_background(s, bgs[s])
        gs = torch.cuda.ExternalStream(g.stream, device=dev)
        ids = [list(range(k, k + B)) for k in range(0, S, B)]

        def src_call(r, k):
            t, k0 = r % R, ids[k][0]
            g.composite_sources_yuyv_device(B, ids[k], frames[t, k0].data_ptr(), d_out[k0].data_ptr(), d_yuyv[k0].data_ptr(), d_mask[k0].data_ptr())

        def src_round(r):
            for k in range(len(ids)):
                src_call(r, k)

        ms_b = timed_rounds(torch, src_round, [gs], args.warmup, args.rounds)
        call_b = median_call_ms(torch, lambda r, k: src_call(r, k % len(ids)), [gs] * len(ids), args.latency_rounds)
        native = g.yuyv_native
        g.close()
        res.append({
            "sources": S,
            "plain": {"contexts": S, "frames_per_call": 1, "calls_per_round": S,
                      "frames_per_s": round(S * args.rounds / (ms_a * 1e-3), 1), "call_ms_median": round(call_a, 4)},
            "sources_call": {"contexts": 1, "frames_per_call": B, "calls_per_round": len(ids), "yuyv_native": native,
                             "frames_per_s": round(S * args.rounds / (ms_b * 1e-3), 1), "call_ms_median": round(call_b, 4)},
            "speedup": round(ms_a / ms_b, 3),
        })
    for c in plain:
        c.close()
    out = {"tool": "sources_bench", **gpu_info(dev), "model": MODEL, "frame": f"{W}x{H}", "input": "device-resident camera YUYV",
           "ring_frames_per_camera": R, "rounds": args.rounds, "warmup_rounds": args.warmup, "results": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
