"""Contexts that run at once (include/backscrub_b200.h: contexts are independent, one per stream or GPU).

bench.py drives eight contexts per GPU, each on its own CUDA stream, from eight host threads, and bsb_calcmask_* runs its
context on a worker thread of its own.  What contexts do share is process-wide: the launcher switches of bsb_set_tuning,
the per-device caches built on first use (ensure_dyn_smem's attributes, the encoder carveouts, the Gaussian tap
tables), the process-wide launch total, and the SMs their kernels run on.

The harness gives every host thread a fixed, seeded schedule of steps (create a context, set an option, make a call,
close it) over its own stream of tests/synth frames, and runs the schedules twice in one fresh interpreter:
  * the concurrent pass starts every thread behind one threading.Barrier;
  * the solo pass runs the same schedules one thread at a time on fresh contexts.
Every output of every call (composite or BGRA frame, YUYV or NV12, mask), the launches_per_call after every call and
bsb_last_error after every step must be bit-identical between the passes.  A fixed sample of the frames of the
contexts on the exact path (Meet, MLKit) is compared with oracle/pyoracle as well, so a solo run cannot hide an error
by repeating it.  Every library call counts itself in flight on the host under a lock, and the concurrent pass must
have had two calls in flight at once; ctypes.CDLL releases the GIL around every foreign call, so the threads do enter
the library together.

The harness runs in a fresh interpreter so that the churn thread's first context is the first context of the process:
the Gaussian tap tables are built inside context creation, so that first creation builds them while the other threads
create their contexts and capture their first graphs (the other threads start when its creation starts).  No code in
that interpreter calls bsb_set_tuning, so the launcher switches hold the defaults of struct Tuning in kernels.h.

`-m "not gpu"`: the kernel-logic emulator at small sizes.  It runs kernels eagerly, without graphs, so it checks the
host side: the planner, the caches, the launch counters and the error strings.
`-m gpu`: the sm_90a library on the H100 with the thread mix of bench.py and the front end.  It asserts that calls
overlapped on the host, not that kernels of different contexts were co-resident on the SMs.

Run one tier by hand: python -m tests.test_concurrent_contexts emu|gpu"""

import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from backscrub_b200 import api  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from tests import synth  # noqa: E402
from tests.conftest import model_path  # noqa: E402
from tests.test_source_filter import camera_bgr, nv12_frame, yuyv_to_nv12  # noqa: E402


def _tuning_defaults():
    """the shipped values of the launcher switches, read from struct Tuning in kernels.h"""
    with open(os.path.join(ROOT, "backscrub_b200", "csrc", "kernels.h")) as f:
        src = f.read()
    body = src[src.index("struct Tuning {"):]
    body = body[:body.index("};")]
    return {k: int(v) for k, v in re.findall(r"int (\w+) = (-?\d+);", body)}


TUNING = _tuning_defaults()
# the host-buffer YUYV thread: two full chunks of the copy / compute overlap and a short last one
HOST_FRAMES = 2 * TUNING["e2e_chunk"] + 3


def _digest(a):
    return hashlib.blake2b(np.ascontiguousarray(a).tobytes(), digest_size=16).hexdigest()


def _frames(fmt, W, H, ts, stream):
    if fmt == "yuyv":
        return np.stack([synth.yuyv_frame(W, H, t=t, stream=stream) for t in ts])
    if fmt == "nv12":
        return np.stack([nv12_frame(W, H, t=t, stream=stream) for t in ts])
    return np.stack([synth.frame(W, H, t=t, stream=stream) for t in ts])


# ---------------------------------------------------------------------------------------------------------------------
# memory the "device" entry points read and write: CUDA memory on the GPU, host memory on the emulator
# ---------------------------------------------------------------------------------------------------------------------
class HostMem:
    def put(self, a):
        return np.ascontiguousarray(a)

    def empty(self, nbytes):
        return np.zeros(nbytes, np.uint8)

    def ptr(self, a):
        return a.ctypes.data

    def get(self, a, nbytes, off=0):
        return a.reshape(-1)[off:off + nbytes].copy()


class CudaMem:
    def __init__(self):
        import torch
        self.torch = torch

    def put(self, a):
        t = self.torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to("cuda")
        self.torch.cuda.synchronize()
        return t

    def empty(self, nbytes):
        # no fill kernel: it would run on torch's stream, unordered with the context's non-blocking stream.  Only the
        # bytes a call writes are ever read back.
        return self.torch.empty(nbytes, dtype=self.torch.uint8, device="cuda")

    def ptr(self, a):
        return a.data_ptr()

    def get(self, a, nbytes, off=0):
        return a[off:off + nbytes].cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# calls in flight
# ---------------------------------------------------------------------------------------------------------------------
class InFlight:
    def __init__(self):
        self.lock = threading.Lock()
        self.now = self.peak = self.calls = 0

    def __enter__(self):
        with self.lock:
            self.now += 1
            self.calls += 1
            self.peak = max(self.peak, self.now)

    def __exit__(self, *exc):
        with self.lock:
            self.now -= 1


# ---------------------------------------------------------------------------------------------------------------------
# schedules
# ---------------------------------------------------------------------------------------------------------------------
class Sched:
    """one thread's steps: (kind, op, args), kind one of create / set / call / close.  `oracle` lists the frames checked
    against the oracle: (step index, frame of the call, oracle stream, frame of the stream); `streams` the oracle streams
    by name: model, size, format and camera frames, and for plain streams the background and blur, for sources streams
    the source id and mask interval"""

    def __init__(self, name):
        self.name = name
        self.steps = []
        self.oracle = []
        self.streams = {}
        self.wait_for = None         # name of an event to wait for before the first step (concurrent pass only)
        self.signals = None          # name of an event set just before the first step

    def add(self, kind, op, **args):
        self.steps.append((kind, op, args))
        return len(self.steps) - 1


def plain_schedule(name, lib_key, W, H, *, stream, calls, n, fmt, entry, bg=True, bgblur=0, out_fmt="bgr",
                   flags=0, oracle_frames=(), max_batch=None):
    """one plain context: `calls` calls of n frames of `fmt` through `entry` ("device" or "host"), the smoother state
    carried across them; oracle_frames: frame indices of the stream compared with the oracle"""
    s = Sched(name)
    back = synth.background() if bg else None
    s.add("create", "create", key=lib_key, W=W, H=H, max_batch=max_batch or n, flags=flags)
    if back is not None:
        s.add("set", "set_background", bg=back)
    if bgblur:
        s.add("set", "set_bgblur", k=bgblur)
    if out_fmt != "bgr":
        s.add("set", "set_out_format", fmt=out_fmt)
    all_frames = _frames(fmt, W, H, range(calls * n), stream)
    for c in range(calls):
        i = s.add("call", "plain", fmt=fmt, entry=entry, frames=all_frames[c * n:(c + 1) * n])
        for t in oracle_frames:
            if c * n <= t < (c + 1) * n:
                s.oracle.append((i, t - c * n, name, t))
    s.add("close", "close")
    if oracle_frames:
        s.streams[name] = dict(key=lib_key, W=W, H=H, bg=back, k=bgblur, fmt=fmt, frames=all_frames, plain=True)
    return s


def sources_schedule(name, lib_key, W, H, *, stream, n_sources, calls, seed, blur, own_size, oracle_sources):
    """one sources context of NV12 device calls, every call one frame of every source in a seeded order, context mask
    interval 2.  Source 0: camera blur `blur` with no background; 1: a background ring; 2: flip H; 3: its own output
    size; n_sources - 2 and n_sources - 1: framing AUTO; the rest follow the context.  The oracle checks the masks of
    oracle_sources: a segmented frame's mask is the oracle stream's, given only that source's segmented frames; a held
    frame's is its source's latest segmented mask."""
    rng = np.random.default_rng(seed)
    s = Sched(name)
    bg = synth.background()
    s.add("create", "create", key=lib_key, W=W, H=H, max_batch=n_sources, flags=0)
    s.add("set", "set_background", bg=bg)
    s.add("set", "set_sources", n=n_sources)
    s.add("set", "set_mask_interval", k=2)
    s.add("set", "set_source_effect", source=0, background="none", bgblur=blur)
    ring = np.stack([np.roll(bg, 40 * r, axis=1) for r in range(3)])
    s.add("set", "set_source_background_ring", source=1, frames=ring)
    s.add("set", "set_source_flip", source=2, flip_h=True)
    s.add("set", "set_source_output", source=3, size=own_size)
    for src in (n_sources - 2, n_sources - 1):
        s.add("set", "set_source_framing", source=src, mode="auto")
    per_source = {src: _frames("nv12", W, H, range(calls), 100 * stream + src) for src in range(n_sources)}
    for c in range(calls):
        ids = [int(v) for v in rng.permutation(n_sources)]
        frames = np.stack([per_source[src][c] for src in ids])
        i = s.add("call", "sources_nv12", ids=ids, frames=frames)
        for b, src in enumerate(ids):
            if src in oracle_sources:
                s.oracle.append((i, b, f"{name}/{src}", c))
    for src in oracle_sources:
        s.streams[f"{name}/{src}"] = dict(key=lib_key, W=W, H=H, fmt="nv12", frames=per_source[src], plain=False,
                                         source=src, interval=2)
    s.add("close", "close")
    return s


def churn_schedule(name, lib_key, W, H, *, stream, rounds, out_size, blurs):
    """`rounds` times: create a context, make a call, change the blur, the output and the framing (new graphs), make
    another call, close the context.  The first call of every round is compared with the oracle."""
    s = Sched(name)
    bg = synth.background()
    for r in range(rounds):
        s.add("create", "create", key=lib_key, W=W, H=H, max_batch=2, flags=0)
        s.add("set", "set_background", bg=bg)
        f = _frames("yuyv", W, H, range(4 * r, 4 * r + 4), stream)
        i = s.add("call", "plain", fmt="yuyv", entry="device", frames=f[:2])
        s.oracle += [(i, 0, f"{name}/{r}", 0), (i, 1, f"{name}/{r}", 1)]
        s.streams[f"{name}/{r}"] = dict(key=lib_key, W=W, H=H, bg=bg, k=0, fmt="yuyv", frames=f[:2], plain=True)
        s.add("set", "set_bgblur", k=blurs[r])
        s.add("set", "set_output", flip_h=bool(r & 1), flip_v=False, size=out_size)
        s.add("set", "set_framing", mode="auto")
        s.add("call", "plain", fmt="yuyv", entry="device", frames=f[2:])
        s.add("close", "close")
    return s


def errors_schedule(name, lib_key, W, H, *, stream, rounds):
    """a context whose calls succeed, between calls the library refuses on the host: an even blur strength, a null
    frame buffer, a source id of a context without sources.  Each refusal must leave this thread's own message."""
    s = Sched(name)
    s.add("create", "create", key=lib_key, W=W, H=H, max_batch=2, flags=0)
    s.add("set", "set_background", bg=synth.background())
    f = _frames("bgr", W, H, range(2 * rounds), stream)
    for r in range(rounds):
        i = s.add("call", "plain", fmt="bgr", entry="device", frames=f[2 * r:2 * r + 2])
        if r == 0:
            s.oracle += [(i, 0, name, 0), (i, 1, name, 1)]
        s.add("set", "refuse", what="even_blur")
        s.add("call", "refuse", what="null_frames")
        s.add("set", "refuse", what="bad_source")
    s.streams[name] = dict(key=lib_key, W=W, H=H, bg=synth.background(), k=0, fmt="bgr", frames=f[:2], plain=True)
    s.add("close", "close")
    return s


REFUSALS = {"even_blur": "strength value must be odd", "null_frames": "invalid frame", "bad_source": "no sources"}


def calcmask_schedule(name, lib_key, W, H, *, stream, n):
    """the bsb_calcmask_* worker: one frame at a time, each mask awaited by its mask_serial before the next frame"""
    s = Sched(name)
    s.add("create", "calcmask_new", key=lib_key, W=W, H=H)
    for t, fr in enumerate(_frames("bgr", W, H, range(n), stream)):
        s.add("call", "calcmask_frame", frame=fr, serial=t + 1)
    s.add("close", "calcmask_delete")
    return s


# ---------------------------------------------------------------------------------------------------------------------
# running a schedule
# ---------------------------------------------------------------------------------------------------------------------
class Runner:
    """runs one schedule on one thread and records what every step gave"""

    def __init__(self, lib, mem, sched, inflight, events, dev_inputs):
        self.lib, self.mem, self.s, self.fl, self.events = lib, mem, sched, inflight, events
        self.dev_inputs = dev_inputs     # step index -> the step's frames in "device" memory (uploaded once, read only)
        self.g = self.cm = None
        self.bufs = {}
        self.rec = []                    # (step, what, digest or value)
        self.keep = {}                   # (step, frame) -> {output: array}, the frames the oracle checks
        self.error = None

    def buf(self, tag, nbytes):
        b = self.bufs.get(tag)
        if b is None or len(b) < nbytes:
            b = self.bufs[tag] = self.mem.empty(nbytes)
        return b

    def run(self):
        try:
            if self.s.wait_for:
                self.events[self.s.wait_for].wait()
            for i, (kind, op, args) in enumerate(self.s.steps):
                if self.s.signals and i == 0:
                    self.events[self.s.signals].set()
                getattr(self, "op_" + op)(i, **args)
                self.rec.append((i, "last_error", self.lib.bsb_last_error().decode()))
        except BaseException as e:           # reported by the main thread
            self.error = f"{self.s.name}: {type(e).__name__}: {e}"
            for ev in self.events.values():
                ev.set()
            if self.g is not None:
                self.g.close()

    # -- steps
    def op_create(self, i, key, W, H, max_batch, flags):
        with self.fl:
            self.g = api.MaskGen(self.lib, model_path(key), W, H, max_batch=max_batch, flags=flags)

    def op_close(self, i):
        with self.fl:
            self.g.close()
        self.g = None

    def op_set_background(self, i, bg):
        with self.fl:
            self.g.set_background(bg)

    def op_set_bgblur(self, i, k):
        with self.fl:
            self.g.set_bgblur(k)

    def op_set_out_format(self, i, fmt):
        with self.fl:
            self.g.set_out_format(fmt)

    def op_set_output(self, i, flip_h, flip_v, size):
        with self.fl:
            self.g.set_output(flip_h, flip_v, size)

    def op_set_framing(self, i, mode):
        with self.fl:
            self.g.set_framing(mode)

    def op_set_sources(self, i, n):
        with self.fl:
            self.g.set_sources(n)

    def op_set_mask_interval(self, i, k):
        with self.fl:
            self.g.set_mask_interval(k)

    def op_set_source_effect(self, i, source, background, bgblur):
        with self.fl:
            self.g.set_source_effect(source, background, bgblur)

    def op_set_source_background_ring(self, i, source, frames):
        with self.fl:
            self.g.set_source_background_ring(source, frames)

    def op_set_source_flip(self, i, source, flip_h):
        with self.fl:
            self.g.set_source_flip(source, flip_h=flip_h)

    def op_set_source_output(self, i, source, size):
        with self.fl:
            self.g.set_source_output(source, size)

    def op_set_source_framing(self, i, source, mode):
        with self.fl:
            self.g.set_source_framing(source, mode)

    def op_refuse(self, i, what):
        L, h = self.lib, self.g._h
        with self.fl:
            if what == "even_blur":
                ok = L.bsb_set_bgblur(h, 4)
            elif what == "null_frames":
                ok = L.bsb_composite_yuyv_device(h, 1, None, None, 0, None, 0, None, 0, 1)
            else:
                ok = L.bsb_set_source_flip(h, 7, 1)
            msg = L.bsb_last_error().decode()
        assert not ok, f"{what} was accepted"
        assert REFUSALS[what] in msg, f"{what}: this thread's last error is {msg!r}"

    def _record(self, i, b, outs):
        for what, a in outs.items():
            self.rec.append((i, f"{what}[{b}]", _digest(a)))
        if any(st == i and fb == b for st, fb, _, _ in self.s.oracle):
            self.keep[(i, b)] = outs

    def op_plain(self, i, fmt, entry, frames):
        g, m = self.g, self.mem
        n, W, H = frames.shape[0], g.width, g.height
        ow, oh, oc = g.out_width, g.out_height, g.out_channels
        vbytes = ow * oh * 3 // 2 if fmt == "nv12" else ow * oh * 2
        obytes = ow * oh * oc
        if entry == "host":
            out = np.empty((n, oh, ow, oc), np.uint8)
            vid = np.empty((n, oh, ow, 2), np.uint8)
            mask = np.empty((n, H, W), np.uint8)
            with self.fl:
                g.composite_yuyv_into(frames, out, vid, mask)
            outs = [dict(out=out[b], video=vid[b], mask=mask[b]) for b in range(n)]
        else:
            d_in = self.dev_inputs[i]
            d_out, d_vid, d_mask = self.buf("out", n * obytes), self.buf("video", n * vbytes), self.buf("mask", n * W * H)
            p = (m.ptr(d_out), m.ptr(d_vid), m.ptr(d_mask))
            with self.fl:
                if fmt == "yuyv":
                    g.composite_yuyv_device(n, m.ptr(d_in), *p, sync=True)
                elif fmt == "nv12":
                    g.composite_nv12_device(n, m.ptr(d_in), *p, sync=True)
                else:
                    g.composite_device(n, m.ptr(d_in), *p, sync=True)
            out, vid, mask = m.get(d_out, n * obytes), m.get(d_vid, n * vbytes), m.get(d_mask, n * W * H)
            outs = [dict(out=out[b * obytes:(b + 1) * obytes], video=vid[b * vbytes:(b + 1) * vbytes],
                         mask=mask[b * W * H:(b + 1) * W * H]) for b in range(n)]
        for b in range(n):
            self._record(i, b, outs[b])
        with self.fl:
            self.rec.append((i, "launches_per_call", g.launches_per_call))

    def op_sources_nv12(self, i, ids, frames):
        g, m = self.g, self.mem
        n, W, H = len(ids), g.width, g.height
        opx = g._sources_out_px()
        d_in = self.dev_inputs[i]
        d_out, d_vid, d_mask = self.buf("out", n * opx * 3), self.buf("video", n * opx * 3 // 2), self.buf("mask", n * W * H)
        with self.fl:
            g.composite_sources_nv12_device(n, ids, m.ptr(d_in), m.ptr(d_out), m.ptr(d_vid), m.ptr(d_mask), sync=True)
        for b, src in enumerate(ids):
            w, h = g.source_output_size(src)
            self._record(i, b, dict(out=m.get(d_out, w * h * 3, b * opx * 3), video=m.get(d_vid, w * h * 3 // 2, b * opx * 3 // 2),
                                    mask=m.get(d_mask, W * H, b * W * H)))
        with self.fl:
            self.rec.append((i, "launches_per_call", g.launches_per_call))

    def op_calcmask_new(self, i, key, W, H):
        with self.fl:
            self.cm = self.lib.bsb_calcmask_new(model_path(key).encode(), 2, W, H, 0)
        assert self.cm, self.lib.bsb_last_error()
        self.W, self.H = W, H

    def op_calcmask_frame(self, i, frame, serial):
        L, cm = self.lib, self.cm
        out = np.empty((self.H, self.W), np.uint8)
        with self.fl:
            assert L.bsb_calcmask_set_input_frame(cm, frame.ctypes.data_as(C.c_void_p), self.W * 3) == 1
        t0 = time.time()
        while True:
            with self.fl:
                got = L.bsb_calcmask_mask_serial(cm)
            assert got >= 0, "the worker failed to process a frame"
            if got >= serial:
                break
            assert time.time() - t0 < 300, "no mask for frame %d" % serial
            time.sleep(0.002)
        assert got == serial, (got, serial)
        with self.fl:
            assert L.bsb_calcmask_get_output_mask(cm, out.ctypes.data_as(C.c_void_p), self.W) == 1
        self._record(i, 0, dict(mask=out))

    def op_calcmask_delete(self, i):
        with self.fl:
            self.lib.bsb_calcmask_delete(self.cm)
        self.cm = None


def _upload(mem, scheds):
    """every device-call step's frames in device memory, uploaded once and shared by both passes"""
    ups = {}
    for s in scheds:
        ups[s.name] = {i: mem.put(a["frames"]) for i, (k, op, a) in enumerate(s.steps)
                       if op in ("sources_nv12",) or (op == "plain" and a["entry"] == "device")}
    return ups


def run_pass(lib, mem, scheds, ups, concurrent):
    fl = InFlight()
    events = {"churn_started": threading.Event()}
    runners = [Runner(lib, mem, s, fl, events, ups[s.name]) for s in scheds]
    t0 = time.time()
    if concurrent:
        barrier = threading.Barrier(len(runners))

        def go(r):
            barrier.wait()
            r.run()
        ths = [threading.Thread(target=go, args=(r,), name=r.s.name) for r in runners]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
    else:
        events["churn_started"].set()
        for r in runners:                    # each on a thread of its own: fresh thread-local error text, as above
            t = threading.Thread(target=r.run, name=r.s.name)
            t.start()
            t.join()
    errors = [r.error for r in runners if r.error]
    assert not errors, "\n".join(errors)
    return runners, fl, time.time() - t0


def _compare(conc, solo):
    for a, b in zip(conc, solo):
        name = a.s.name
        assert len(a.rec) == len(b.rec), f"{name}: {len(a.rec)} records concurrently, {len(b.rec)} alone"
        for x, y in zip(a.rec, b.rec):
            assert x == y, f"{name}: step {x[0]} {a.s.steps[x[0]][1]}: {x[1]} differs: {x[2]!r} concurrently, {y[2]!r} alone"


def _error_isolation(runners, errors_thread):
    for r in runners:
        if r.s.name == errors_thread or r.s.name.startswith("calcmask"):
            continue
        seen = {v for _, w, v in r.rec if w == "last_error"}
        assert seen == {""}, f"{r.s.name}: bsb_last_error changed to {sorted(seen - {''})} in a thread whose calls all succeeded"


def _oracle_check(runners):
    """the kept frames against oracle/pyoracle streams"""
    checked = 0
    for r in runners:
        s = r.s
        for name, st in s.streams.items():
            want = {}
            o = po.MaskGen(model_path(st["key"]), st["W"], st["H"])
            ts = sorted(t for _, _, n_, t in s.oracle if n_ == name)
            if st["plain"]:
                for t in range(max(ts) + 1):
                    bgr = camera_bgr(st["frames"][t], st["fmt"])
                    ro, ry, rm = o.composite_ex(bgr, st["bg"], bgblur=st["k"])
                    want[t] = dict(out=ro, video=yuyv_to_nv12(ry) if st["fmt"] == "nv12" else ry, mask=rm)
            else:
                last = None
                for t in range(max(ts) + 1):
                    if t == 0 or (t + st["source"]) % st["interval"] == 0:
                        last = o.process(camera_bgr(st["frames"][t], st["fmt"]))
                    want[t] = dict(mask=last)
            o.close()
            for i, b, n_, t in s.oracle:
                if n_ != name:
                    continue
                got = r.keep[(i, b)]
                for what, ref in want[t].items():
                    assert np.array_equal(got[what].reshape(-1), ref.reshape(-1)), f"{name}: frame {t}: {what} differs from the oracle"
                    checked += 1
    return checked


def _calcmask_reference(lib, runners):
    """each calcmask mask against a plain context's bs_maskgen_process of the same frames, run alone"""
    checked = 0
    for r in runners:
        if not r.s.name.startswith("calcmask"):
            continue
        key, W, H = (r.s.steps[0][2][k] for k in ("key", "W", "H"))
        g = api.MaskGen(lib, model_path(key), W, H)
        for i, (kind, op, a) in enumerate(r.s.steps):
            if op == "calcmask_frame":
                want = _digest(g.process(a["frame"]))
                got = [v for st, w, v in r.rec if st == i and w == "mask[0]"]
                assert got == [want], f"{r.s.name}: mask of frame {a['serial']} differs from a solo context's"
                checked += 1
        g.close()
    return checked


def releases_the_gil(lib):
    return isinstance(lib, C.CDLL) and not isinstance(lib, C.PyDLL) and not (lib._func_flags_ & C._FUNCFLAG_PYTHONAPI)


def harness(lib, mem, scheds, errors_thread):
    assert releases_the_gil(lib), "the library is not loaded with ctypes.CDLL: its calls hold the GIL, so no two threads " \
                                  "are ever inside it at once and this harness proves nothing"
    ups = _upload(mem, scheds)
    conc, fl_c, dt_c = run_pass(lib, mem, scheds, ups, concurrent=True)
    solo, fl_s, dt_s = run_pass(lib, mem, scheds, ups, concurrent=False)
    _compare(conc, solo)
    _error_isolation(conc, errors_thread)
    n_oracle = _oracle_check(conc)
    n_cm = _calcmask_reference(lib, solo)
    assert fl_c.peak >= 2, f"the concurrent pass never had two library calls in flight ({fl_c.calls} calls)"
    return dict(threads=len(scheds), calls=fl_c.calls, peak_in_flight=fl_c.peak, concurrent_s=round(dt_c, 2),
                solo_s=round(dt_s, 2), oracle_checks=n_oracle, calcmask_checks=n_cm,
                records=sum(len(r.rec) for r in conc))


# ---------------------------------------------------------------------------------------------------------------------
# the two thread mixes
# ---------------------------------------------------------------------------------------------------------------------
def emu_schedules():
    churn = churn_schedule("churn", "mlkit", 64, 48, stream=5, rounds=3, out_size=(48, 36), blurs=(5, 9, 3))
    scheds = [
        plain_schedule("meet_lite", "meet_lite", 96, 64, stream=1, calls=3, n=3, fmt="yuyv", entry="device",
                       oracle_frames=(0, 4, 8)),
        plain_schedule("mlkit", "mlkit", 64, 48, stream=2, calls=2, n=2, fmt="nv12", entry="device", bgblur=7,
                       oracle_frames=(1, 2)),
        sources_schedule("sources", "mlkit", 64, 48, stream=3, n_sources=4, calls=3, seed=3, blur=5, own_size=(32, 24),
                         oracle_sources=(0, 3)),
        churn,
        errors_schedule("errors", "mlkit", 64, 48, stream=7, rounds=2),
    ]
    return _order(scheds)


def gpu_schedules():
    churn = churn_schedule("churn", "mlkit", 640, 480, stream=6, rounds=3, out_size=(480, 360), blurs=(25, 5, 45))
    scheds = [
        plain_schedule("meet_device_yuyv", "meet_full", 1280, 720, stream=1, calls=4, n=32, fmt="yuyv", entry="device",
                       oracle_frames=(0, 3, 6)),
        plain_schedule("meet_host_yuyv", "meet_full", 1280, 720, stream=2, calls=2, n=HOST_FRAMES, fmt="yuyv", entry="host",
                       oracle_frames=(1, 5)),
        sources_schedule("mlkit_sources", "mlkit", 640, 480, stream=3, n_sources=8, calls=4, seed=3, blur=25,
                         own_size=(320, 240), oracle_sources=(0, 3, 5)),
        plain_schedule("deeplab", "deeplab", 640, 480, stream=4, calls=3, n=4, fmt="bgr", entry="device"),
        plain_schedule("bodypix_blur45_bgra", "bodypix", 640, 480, stream=5, calls=3, n=4, fmt="bgr", entry="device",
                       bg=False, bgblur=45, out_fmt="bgra"),
        churn,
        errors_schedule("errors", "mlkit", 640, 480, stream=7, rounds=6),
        calcmask_schedule("calcmask", "mlkit", 640, 480, stream=8, n=6),
    ]
    return _order(scheds)


def _order(scheds):
    """the churn thread creates the process's first context; the others start as that creation starts"""
    for s in scheds:
        if s.name == "churn":
            s.signals = "churn_started"
        else:
            s.wait_for = "churn_started"
    return scheds


def main(tier):
    if tier == "gpu":
        import backscrub_b200 as bs
        lib, mem, scheds = bs.lib(), CudaMem(), gpu_schedules()
    else:
        from tests.emu.emu_lib import emu
        lib, mem, scheds = emu(), HostMem(), emu_schedules()
    stats = harness(lib, mem, scheds, "errors")
    print("RESULT " + json.dumps(stats), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
def test_launcher_switch_defaults():
    """the schedules assume the shipped switches: they are read from kernels.h, and nothing in the harness's interpreter
    sets them"""
    assert {"e2e_chunk", "dec_par", "post_tma", "pool_merge", "cnn_chain"} <= set(TUNING)
    chunk = TUNING["e2e_chunk"]
    assert chunk > 0 and HOST_FRAMES >= 2 * chunk and HOST_FRAMES % chunk, "the host-buffer thread must run chunked"
    assert (HOST_FRAMES + chunk - 1) // chunk <= 16, "more chunks than a host-buffer call overlaps"


def test_bindings_release_the_gil():
    from tests.emu.emu_lib import emu
    assert releases_the_gil(emu())
    assert not releases_the_gil(C.PyDLL(None))


def test_schedules_are_fixed():
    """the same seeds give the same steps and frames, so both passes run one schedule"""
    a, b = emu_schedules(), emu_schedules()
    for x, y in zip(a, b):
        assert [(k, op) for k, op, _ in x.steps] == [(k, op) for k, op, _ in y.steps]
        for (_, _, ax), (_, _, ay) in zip(x.steps, y.steps):
            for key in ax:
                va, vb = ax[key], ay[key]
                assert np.array_equal(va, vb) if isinstance(va, np.ndarray) else va == vb
    streams = [s.steps[i][2]["frames"] for s in a for i in range(len(s.steps)) if "frames" in s.steps[i][2]]
    assert len({_digest(f) for f in streams}) == len(streams), "two calls share frames"


def _run_tier(tier, timeout):
    env = dict(os.environ)
    p = subprocess.run([sys.executable, "-m", "tests.test_concurrent_contexts", tier], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    tail = (p.stdout + p.stderr)[-6000:]
    assert p.returncode == 0, f"the {tier} harness failed (exit {p.returncode}):\n{tail}"
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
    assert line, tail
    stats = json.loads(line[-1][len("RESULT "):])
    print(f"{tier}: {stats['calls']} calls, at most {stats['peak_in_flight']} in flight, concurrent pass "
          f"{stats['concurrent_s']} s, solo pass {stats['solo_s']} s, {stats['oracle_checks']} oracle checks")
    return stats


def test_emu_contexts_at_once():
    stats = _run_tier("emu", 600)
    assert stats["peak_in_flight"] >= 2 and stats["oracle_checks"] > 0


@pytest.mark.gpu
def test_gpu_contexts_at_once():
    stats = _run_tier("gpu", 900)
    assert stats["peak_in_flight"] >= 2 and stats["oracle_checks"] > 0 and stats["calcmask_checks"] == 6


if __name__ == "__main__":
    main(sys.argv[1])
