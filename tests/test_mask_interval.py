"""Mask interval (bsb_set_mask_interval, bsb_set_source_mask_interval): segment every k-th frame of a camera and composite
the frames between with its latest mask, as the reference's main loop composites every camera frame with whatever mask
its AI thread made last (app/deepseg.cc:627-661).

A segmented frame must equal an oracle stream that is given only that camera's segmented frames.  A held frame's mask
must equal the mask of the camera's latest segmented frame, and its composite and video output must equal the mask-feed
references of tests/test_feed_post.py applied to that oracle stream's smoother state.

`-m "not gpu"`: the kernel-logic emulator build against the oracle.
`-m gpu`: the sm_90a library against library contexts at interval 1 given only the segmented frames, and the same
mask-feed references for the held frames."""

import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_feed_post import geo, oracle_mask, ref_mask, ref_outputs
from tests.test_source_filter import _frames, _plain_call, camera_bgr, passthrough, yuyv_to_nv12

H_, V_ = 1, 2


def _same(got, want, what, tag):
    assert np.array_equal(np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)), f"{what} differs {tag}"


def _bg_at(bg, W, H):
    return bg if bg.shape[:2] == (H, W) else po.resize_linear_u8(bg, W, H)


class Cam:
    """one camera: its oracle stream, given only its segmented frames, and the references of its held frames"""

    def __init__(self, key, W, H, bg=None, k=0, flip=0, size=None, active=True):
        self.key, self.W, self.H = key, W, H
        self.o = po.MaskGen(model_path(key), W, H)
        self.bg, self.k, self.flip, self.size, self.active = bg, k, flip, size, active
        self.frames = 0                                  # frames delivered since the start / the last reset
        self.ofinal = self.mask = None

    def reset(self):
        self.o.close()
        self.o = po.MaskGen(model_path(self.key), self.W, self.H)
        self.frames = 0
        self.ofinal = self.mask = None

    def segmented(self, bgr, nv12):
        ro, ry, rm = self.o.composite_ex(bgr, self.bg, bgblur=self.k, flip_h=bool(self.flip & H_), flip_v=bool(self.flip & V_),
                                         out_size=self.size)
        self.ofinal, self.mask = self.o.ofinal, rm
        if not self.active:
            ro, rv = passthrough(bgr, self.flip, self.size, nv12=nv12)
        else:
            rv = yuyv_to_nv12(ry) if nv12 else ry
        return ro, rv, rm, self.ofinal

    def held(self, bgr, nv12):
        m = oracle_mask(geo(self.key, self.W, self.H), self.ofinal)
        _same(m, self.mask, "mask-feed reference", "of the latest segmented frame")
        if not self.active:
            ro, rv = passthrough(bgr, self.flip, self.size, nv12=nv12)
        else:
            bg = _bg_at(self.bg, self.W, self.H) if self.bg is not None else bgr
            if self.k:
                bg = po.gaussian_blur(bg, self.k)
            ro, rv = ref_outputs(m, bgr, bg, self.flip, self.size, nv12=nv12)
        return ro, rv, m, self.ofinal


def _check(g, got, want, b, tag):
    out, vid, mask = got
    ro, rv, rm, rf = want
    _same(g.stage_u8(2, b), rf, "smoother state", tag)
    _same(mask[b], rm, "mask", tag)
    _same(out[b], ro, "composite", tag)
    _same(vid[b], rv, "video output", tag)


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("fmt", ["bgr", "yuyv", "nv12"])
def test_plain_cadence(emu_lib, fmt, k):
    """one stream cut into calls of 5 + 4 + 3 frames, so the cadence crosses call boundaries (YUYV and NV12 on the device
    entry points, which read camera frames in place)"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=5)
    g.set_background(bg)
    g.set_mask_interval(k)
    cam = Cam(key, W, H, bg)
    c = 0
    for n in (5, 4, 3):
        frames = _frames(fmt, W, H, range(c, c + n))
        got = _plain_call(g, fmt, frames, device=fmt != "bgr")
        for b in range(n):
            bgr = camera_bgr(frames[b], fmt)
            want = cam.segmented(bgr, fmt == "nv12") if (c + b) % k == 0 else cam.held(bgr, fmt == "nv12")
            _check(g, got, want, b, (fmt, k, c + b))
        c += n
    g.close()


def test_plain_output_settings_and_interval_change(emu_lib):
    """held frames go through the context's flip and resize, blur and filter switch like any frame; a new interval applies
    from the next frame without resetting the count, and bsb_reset_state starts the count over"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    g.set_background(bg)
    g.set_bgblur(7)
    g.set_output(True, False, (240, 180))
    cam = Cam(key, W, H, bg, k=7, flip=H_, size=(240, 180))
    c, t = 0, 0
    for k, n, active, reset in ((2, 3, True, False), (3, 4, False, False), (3, 2, True, False), (4, 3, True, True),
                                (4, 4, True, False)):
        if reset:
            g.reset_state()
            cam.reset()
            c = 0
        g.set_mask_interval(k)
        g.set_filter(active)
        cam.active = active
        frames = _frames("bgr", W, H, range(t, t + n))
        got = g.composite(frames)
        for b in range(n):
            want = cam.segmented(frames[b], False) if (c + b) % k == 0 else cam.held(frames[b], False)
            _check(g, got, want, b, (k, active, c + b))
        c, t = c + n, t + n
    g.close()


class Sources:
    """six sources: 0 follows (the context image), 1 own interval 1 and flip H, 2 own interval 3 and camera blur 9, 3 follows
    with its own size, 4 own interval 4 with its filter off, 5 own interval 2 with its own image at strength 5"""

    def __init__(self, lib, fmt, key="meet_lite", W=320, H=240, ctx_k=2):
        self.fmt, self.W, self.H = fmt, W, H
        bg = synth.background()
        own = np.roll(bg, 90, axis=1)
        g = self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=6)
        g.set_background(bg)
        g.set_sources(6)
        g.set_mask_interval(ctx_k)
        self.ctx_k = ctx_k
        self.own_k = {0: None, 1: 1, 2: 3, 3: None, 4: 4, 5: 2}
        for s, k in self.own_k.items():
            g.set_source_mask_interval(s, k)
        g.set_source_flip(1, flip_h=True)
        g.set_source_effect(2, "none", 9)
        size3 = (160, 120)
        g.set_source_output(3, size3)
        g.set_source_filter(4, False)
        g.set_source_background(5, own)
        g.set_source_effect(5, "default", 5)
        self.cams = [Cam(key, W, H, bg), Cam(key, W, H, bg, flip=H_), Cam(key, W, H, None, k=9), Cam(key, W, H, bg, size=size3),
                     Cam(key, W, H, bg, active=False), Cam(key, W, H, own, k=5)]
        self.t = [0] * 6

    def k(self, s):
        return self.ctx_k if self.own_k[s] is None else self.own_k[s]

    def set_ctx(self, k):
        self.g.set_mask_interval(k)
        self.ctx_k = k

    def set_own(self, s, k):
        self.g.set_source_mask_interval(s, k)
        self.own_k[s] = k

    def reset(self, s):
        self.g.reset_source(s)
        self.cams[s].reset()

    def _run(self, ids, frames):
        g, n = self.g, len(ids)
        if self.fmt == "bgr":
            out, vid, mask = g.composite_sources(frames, ids)
            return [out[b] for b in range(n)], [vid[b] for b in range(n)], mask
        buf = np.ascontiguousarray(frames)
        opx = g._sources_out_px()
        out = np.zeros(n * opx * 3, np.uint8)
        vid = np.zeros(n * opx * 3 // 2, np.uint8)
        mask = np.empty((n, self.H, self.W), np.uint8)
        g.composite_sources_nv12_device(n, ids, buf.ctypes.data, out.ctypes.data, vid.ctypes.data, mask.ctypes.data, sync=True)
        outs, vids = [], []
        for b, s in enumerate(ids):
            w, h = g.source_output_size(s)
            outs.append(out[b * opx * 3: b * opx * 3 + w * h * 3])
            vids.append(vid[b * opx * 3 // 2: b * opx * 3 // 2 + w * h * 3 // 2])
        return outs, vids, mask

    def call(self, ids):
        frames = np.stack([_frames(self.fmt, self.W, self.H, [self.t[s]], stream=s)[0] for s in ids])
        outs, vids, mask = self._run(ids, frames)
        nseg = 0
        for b, s in enumerate(ids):
            cam = self.cams[s]
            f = cam.frames
            seg = f == 0 or (f + s) % self.k(s) == 0
            bgr = camera_bgr(frames[b], self.fmt)
            want = cam.segmented(bgr, self.fmt == "nv12") if seg else cam.held(bgr, self.fmt == "nv12")
            tag = (self.fmt, ids, b, s, f, self.k(s), seg)
            _check(self.g, (outs, vids, mask), want, b, tag)
            cam.frames += 1
            self.t[s] += 1
            nseg += seg
        return nseg


@pytest.mark.parametrize("fmt", ["bgr", "nv12"])
def test_sources_cadence(emu_lib, fmt):
    """subsets of the sources in shuffled order per call, with own and following intervals, a context interval change, a
    source switched to follow, and bsb_reset_source mid-stream (after which that source's next frame is segmented)"""
    d = Sources(emu_lib, fmt)
    rng = np.random.default_rng(3)
    for i in range(9):
        if i == 4:
            d.reset(2)
            d.reset(4)
        if i == 5:
            d.set_ctx(3)
        if i == 6:
            d.set_own(1, None)
        ids = [int(s) for s in rng.permutation(6)[: int(rng.integers(3, 7))]]
        if i in (4, 5):
            ids = sorted(set(ids) | {2, 4})
        d.call(ids)
    d.g.close()


def test_interval_one_is_the_default(emu_lib):
    """interval 1 set explicitly (context and every source) gives the bytes and the launch count of a context that never
    touched the setters"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    gs = []
    for explicit in (False, True):
        g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
        g.set_background(bg)
        g.set_sources(3)
        if explicit:
            g.set_mask_interval(1)
            for s in range(3):
                g.set_source_mask_interval(s, 1 if s else None)
        gs.append(g)
    for i in range(3):
        fr = _frames("yuyv", W, H, range(4 * i, 4 * i + 4))
        got = [_plain_call(g, "yuyv", fr, device=True) for g in gs]
        for a, b, what in zip(*got, ("composite", "video", "mask")):
            _same(a, b, what, ("plain", i))
        assert gs[0].launches_per_call == gs[1].launches_per_call
        fr = np.stack([synth.frame(W, H, t=i, stream=s) for s in range(3)])
        got = [g.composite_sources(fr, [2, 0, 1]) for g in gs]
        for a, b, what in zip(*got, ("composite", "video", "mask")):
            _same(a, b, what, ("sources", i))
        assert gs[0].launches_per_call == gs[1].launches_per_call
    for g in gs:
        g.close()


def test_call_without_segmented_frames(emu_lib):
    """a call whose frames are all held launches no pre-processing and no CNN: exactly the launches of a call fed its
    logits (conversion, decision and post), and it is still exact"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    g.set_background(bg)
    g.set_mask_interval(4)
    cam = Cam(key, W, H, bg)
    fr = _frames("yuyv", W, H, range(4))
    got = _plain_call(g, "yuyv", fr[:1], device=True)
    _check(g, got, cam.segmented(camera_bgr(fr[0], "yuyv"), False), 0, "segmented")
    full = g.launches_per_call
    got = _plain_call(g, "yuyv", fr[1:], device=True)
    held = g.launches_per_call
    for b in range(3):
        _check(g, got, cam.held(camera_bgr(fr[1 + b], "yuyv"), False), b, ("held", b))
    twin = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    twin.set_background(bg)
    twin.feed(1, np.zeros((3, *twin.feed_shape(1)), np.float32))
    _plain_call(twin, "yuyv", fr[1:], device=True)
    assert held == twin.launches_per_call < full, (held, twin.launches_per_call, full)
    twin.close()
    g.close()


def test_sources_call_without_segmented_frames(emu_lib):
    """sources at interval 2 whose frames are all held: their states are copied, nothing is segmented"""
    key, W, H = "meet_lite", 320, 240
    d = Sources(emu_lib, "bgr", ctx_k=2)
    for s in range(6):
        d.set_own(s, 2)
    d.call([0, 2, 4])                    # first frames: segmented
    assert d.call([2, 4, 0]) == 0        # frame 1 of even sources: (1 + s) % 2 == 1, held
    d.g.close()


def test_split_host_call(emu_lib):
    """a host-buffer YUYV call of 32 frames runs in chunks of 16 (e2e_chunk); at k = 3 the cadence runs across the chunks:
    the same bytes as one device call of the same frames on a twin context"""
    key, W, H, n = "meet_lite", 320, 240, 32
    bg = synth.background()
    gs = []
    for _ in range(2):
        g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
        g.set_background(bg)
        g.set_mask_interval(3)
        gs.append(g)
    for i in range(2):
        fr = _frames("yuyv", W, H, range(n * i, n * i + n))
        host = gs[0].composite_yuyv(fr)
        dev = _plain_call(gs[1], "yuyv", fr, device=True)
        for a, b, what in zip(host, dev, ("composite", "video", "mask")):
            _same(a, b, what, i)
    for g in gs:
        g.close()


def test_errors_and_fed_calls(emu_lib):
    key, W, H = "meet_lite", 320, 240
    L = emu_lib
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    for v in (0, 257, -2, -1):
        assert L.bsb_set_mask_interval(g._h, v) == 0 and b"interval" in L.bsb_last_error(), v
    assert L.bsb_set_source_mask_interval(g._h, 0, 2) == 0 and b"set_sources" in L.bsb_last_error()
    g.set_sources(3)
    for s, v, msg in ((3, 2, b"out of range"), (-1, 2, b"out of range"), (0, 0, b"interval"), (1, 257, b"interval"),
                      (2, -2, b"interval")):
        assert L.bsb_set_source_mask_interval(g._h, s, v) == 0, (s, v)
        assert msg in L.bsb_last_error(), (s, v, L.bsb_last_error())
    for v in (1, 256):
        assert L.bsb_set_mask_interval(g._h, v) == 1
        assert L.bsb_set_source_mask_interval(g._h, 2, v) == 1
    # fed calls ignore the interval and leave the count as it was
    g.set_mask_interval(2)
    fr = _frames("bgr", W, H, range(4))
    g.composite(fr[:1])                                  # plain frame 0: segmented
    state0 = g.stage_u8(2, 0)
    oh, ow, _ = g.feed_shape(2)
    g.feed(2, np.full((2, oh, ow), 255, np.uint8))
    g.composite(fr[1:3])                                 # fed: the counts do not move
    _same(g.stage_u8(2, 1), np.full((oh, ow), 255, np.uint8), "fed mask", "")
    g.composite(fr[1:3])                                 # plain frames 1 (held) and 2 (segmented)
    _same(g.stage_u8(2, 0), state0, "held state after a fed call", "")
    assert not np.array_equal(g.stage_u8(2, 1), state0)
    g.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    if bs.device_count() <= 0:
        pytest.skip("needs a CUDA device")
    return bs.lib()


@pytest.fixture
def tuning(gpu_lib):
    changed = []

    def set_(name, value, default):
        gpu_lib.bsb_set_tuning(name.encode(), value)
        changed.append((name, default))
    yield set_
    for name, default in changed:
        gpu_lib.bsb_set_tuning(name.encode(), default)


def _dev_frames(fmt, W, H, ts, streams):
    import torch
    if fmt == "yuyv":
        host = np.stack([synth.yuyv_frame(W, H, t=t, stream=s) for t, s in zip(ts, streams)])
    else:
        from tests.test_source_filter import nv12_frame
        host = np.stack([nv12_frame(W, H, t=t, stream=s) for t, s in zip(ts, streams)])
    return host, torch.from_numpy(host).cuda()


class GpuRun:
    """one context under test with a mask interval, and a twin at interval 1 that is given only the segmented frames"""

    def __init__(self, lib, key, W, H, fmt, n, sources=0, flips=()):
        import torch
        self.torch, self.key, self.W, self.H, self.fmt = torch, key, W, H, fmt
        self.bg = synth.background()
        self.gs = []
        for _ in range(2):
            g = api.MaskGen(lib, model_path(key), W, H, max_batch=n)
            g.set_background(self.bg)
            if sources:
                g.set_sources(sources)
                for s in flips:
                    g.set_source_flip(s, flip_h=True)
            self.gs.append(g)
        self.g, self.ref = self.gs
        self.flips = set(flips)
        self.ofinal = {}                                 # camera -> smoother state after its latest segmented frame
        self.bgw = _bg_at(self.bg, W, H)
        self.geo = geo(key, W, H)

    def close(self):
        for g in self.gs:
            g.close()

    def _call(self, g, host, ids):
        torch, n = self.torch, host.shape[0]
        W, H = self.W, self.H
        d_in = torch.from_numpy(np.ascontiguousarray(host)).cuda()
        out = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")
        vid = torch.empty((n, H * 3 // 2, W) if self.fmt == "nv12" else (n, H, W, 2), dtype=torch.uint8, device="cuda")
        mask = torch.empty((n, H, W), dtype=torch.uint8, device="cuda")
        args = (d_in.data_ptr(), out.data_ptr(), vid.data_ptr(), mask.data_ptr())
        if ids is None:
            (g.composite_nv12_device if self.fmt == "nv12" else g.composite_yuyv_device)(n, *args, sync=True)
        else:
            (g.composite_sources_nv12_device if self.fmt == "nv12" else g.composite_sources_yuyv_device)(n, ids, *args, sync=True)
        states = np.stack([g.stage_u8(2, b) for b in range(n)])
        return out.cpu().numpy(), vid.cpu().numpy(), mask.cpu().numpy(), states

    def step(self, host, ids, seg):
        """one call of the context under test; frames with seg[b] also go to the twin, as one call of just those frames"""
        got = self._call(self.g, host, ids)
        sel = [b for b in range(len(seg)) if seg[b]]
        want = {}
        if sel:
            r = self._call(self.ref, host[sel], None if ids is None else [ids[b] for b in sel])
            for i, b in enumerate(sel):
                want[b] = tuple(x[i] for x in r)
        nv12 = self.fmt == "nv12"
        for b in range(len(seg)):
            cam = 0 if ids is None else ids[b]
            flip = H_ if cam in self.flips else 0
            tag = (self.key, self.fmt, ids is not None, b, cam, bool(seg[b]))
            if seg[b]:
                ro, rv, rm, rf = want[b]
                self.ofinal[cam] = rf
            else:
                rf = self.ofinal[cam]
                rm = ref_mask(self.geo, rf)
                ro, rv = ref_outputs(rm, camera_bgr(host[b], self.fmt), self.bgw, flip, nv12=nv12)
            _same(got[3][b], rf, "smoother state", tag)
            _same(got[2][b], rm, "mask", tag)
            _same(got[0][b], ro, "composite", tag)
            _same(got[1][b], rv, "video output", tag)
        return len(sel)


def _plain_gpu(lib, key, W, H, fmt, k, n=32, calls=3):
    r = GpuRun(lib, key, W, H, fmt, n)
    r.g.set_mask_interval(k)
    c = 0
    for i in range(calls):
        host = _frames(fmt, W, H, range(c, c + n))
        r.step(host, None, [(c + b) % k == 0 for b in range(n)])
        c += n
    r.close()


def _sources_gpu(lib, key, W, H, fmt, own, ctx_k=2, n_src=64, calls=6, seed=0):
    r = GpuRun(lib, key, W, H, fmt, n_src, sources=n_src, flips=range(0, n_src, 5))
    r.g.set_mask_interval(ctx_k)
    ks = {}
    for s in range(n_src):
        if own:
            k = (1, 2, 4, 8)[s % 4]
            r.g.set_source_mask_interval(s, k)
            ks[s] = k
        else:
            ks[s] = ctx_k
    rng = np.random.default_rng(seed)
    counts = [0] * n_src
    for i in range(calls):
        ids = [int(s) for s in rng.permutation(n_src)]
        if i % 2:
            ids = ids[: n_src - 7]
        host = np.stack([_frames(fmt, W, H, [counts[s]], stream=s)[0] for s in ids])
        seg = [counts[s] == 0 or (counts[s] + s) % ks[s] == 0 for s in ids]
        r.step(host, ids, seg)
        for s in ids:
            counts[s] += 1
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("fmt", ["yuyv", "nv12"])
def test_gpu_meet_sources(gpu_lib, tuning, fmt, tile):
    """Meet 1280x720, 64 sources at context interval 2 and with own intervals 1 / 2 / 4 / 8, over 6 calls, both post tile
    widths"""
    tuning("post_tile", tile, 0)
    _sources_gpu(gpu_lib, "meet_full", 1280, 720, fmt, own=False)
    _sources_gpu(gpu_lib, "meet_full", 1280, 720, fmt, own=True, seed=1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("fmt", ["yuyv", "nv12"])
def test_gpu_meet_plain(gpu_lib, fmt, k):
    _plain_gpu(gpu_lib, "meet_full", 1280, 720, fmt, k)


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("deeplab", 640, 480), ("bodypix", 640, 480)])
def test_gpu_other_models(gpu_lib, key, W, H):
    """DeepLab (the decision with the final resize folded in) and BodyPix (tensor-core 1x1 convolutions), plain and
    sources"""
    _plain_gpu(gpu_lib, key, W, H, "yuyv", 3, n=8, calls=2)
    _sources_gpu(gpu_lib, key, W, H, "nv12", own=True, n_src=8, calls=4)


@pytest.mark.gpu
def test_gpu_sequential_decision(gpu_lib, tuning):
    """dec_par = 0 (the one-thread-per-pixel decision kernels walk the call frames) gives the same bytes"""
    tuning("dec_par", 0, 1)
    _plain_gpu(gpu_lib, "meet_full", 1280, 720, "yuyv", 3, n=16, calls=2)
    _plain_gpu(gpu_lib, "deeplab", 640, 480, "yuyv", 2, n=6, calls=2)


@pytest.mark.gpu
def test_gpu_graph_replay(gpu_lib):
    """once a periodic cadence has gone round once, further calls capture nothing: the launches issued by a call are the
    graph's one replay, not a capture"""
    import torch
    key, W, H, n, k = "meet_full", 1280, 720, 32, 3
    g = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=n)
    g.set_background(synth.background())
    g.set_mask_interval(k)
    d_in = torch.from_numpy(_frames("yuyv", W, H, range(n))).cuda()
    out = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda")
    for _ in range(k):
        g.composite_yuyv_device(n, d_in.data_ptr(), out.data_ptr(), sync=True)
    l0 = gpu_lib.bsb_total_launches()
    for _ in range(2 * k):
        g.composite_yuyv_device(n, d_in.data_ptr(), out.data_ptr(), sync=True)
    assert gpu_lib.bsb_total_launches() == l0
    g.close()
    ids = list(range(64))
    d64 = torch.from_numpy(np.stack([synth.yuyv_frame(W, H, t=0, stream=s) for s in ids])).cuda()
    out64 = torch.empty((64, H, W, 3), dtype=torch.uint8, device="cuda")
    g = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=64)
    g.set_background(synth.background())
    g.set_sources(64)
    g.set_mask_interval(2)
    for _ in range(3):
        g.composite_sources_yuyv_device(64, ids, d64.data_ptr(), out64.data_ptr(), sync=True)
    l0 = gpu_lib.bsb_total_launches()
    for _ in range(4):
        g.composite_sources_yuyv_device(64, ids, d64.data_ptr(), out64.data_ptr(), sync=True)
    assert gpu_lib.bsb_total_launches() == l0
    g.close()
