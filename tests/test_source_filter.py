"""The filter switch (bsb_set_filter, bsb_set_source_filter; the reference's `s` key, app/deepseg.cc:624,639-664,782-784).

A frame whose filter is off gives the camera frame as BGR, then its flip, its resize and the YUYV / NV12 conversion
(app/deepseg.cc:662-681 with filterActive == false).  Its mask is byte for byte the mask of the same call with the filter
on, and its smoother advances as with the filter on (:634 feeds every frame).  Switching one frame off changes no other
frame's bytes.

`-m "not gpu"`: the kernel-logic emulator build (the fallback post kernels) against the oracle: the filter-on oracle
stream gives every mask and every filtered-on composite, and the oracle's flip, resize and YUYV restate the pass-through.
`-m gpu`: the sm_90a library (k_post_tma's pass-through tiles) against plain batch-1 contexts with the filter on, and the
same oracle pass-through."""

import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path

H_, V_ = 1, 2


def _code(flip):
    return bool(flip & H_), bool(flip & V_)


def nv12_frame(W, H, t=0, stream=0):
    """camera NV12 frame [H*3/2, W]: the Y plane of synth.yuyv_frame and the UV pairs of its even rows"""
    yv = synth.yuyv_frame(W, H, t=t, stream=stream)
    return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)


def nv12_to_bgr(nv12):
    """NV12 ingest: the oracle's YUYV ingest of (Y, the UV pair of the pixel's 2x2 block)"""
    H, W = nv12.shape[0] * 2 // 3, nv12.shape[1]
    yuyv = np.empty((H, W, 2), np.uint8)
    yuyv[..., 0] = nv12[:H]
    yuyv[..., 1] = np.repeat(nv12[H:], 2, axis=0)
    return po.yuyv_to_bgr(yuyv)


def yuyv_to_nv12(yuyv):
    """NV12 output: Y bytes, and bytes 1 / 3 of each YUYV pair averaged over a row pair with truncation"""
    H, W = yuyv.shape[:2]
    rows = yuyv.reshape(H, W * 2).astype(np.uint16)
    uv = ((rows[0::2, 1::2] + rows[1::2, 1::2]) >> 1).astype(np.uint8)
    return np.concatenate([yuyv[..., 0], uv], axis=0)


def camera_bgr(frame, fmt):
    """the camera frame as the fused path reads it: BGR as given, YUYV / NV12 converted"""
    if fmt == "yuyv":
        return po.yuyv_to_bgr(frame)
    if fmt == "nv12":
        return nv12_to_bgr(frame)
    return frame


def passthrough(bgr, flip=0, out_size=None, nv12=False):
    """app/deepseg.cc:662-681 with filterActive == false: cv::flip, cv::resize to the virtual-camera size, then
    convert_rgb_to_yuyv (and the NV12 derived from it) — the oracle's own functions, in the reference's order"""
    img = bgr
    if flip:
        fh, fv = _code(flip)
        img = po.flip(img, fh, fv)
    H, W = img.shape[:2]
    if out_size and tuple(out_size) != (W, H):
        img = po.resize_linear_u8(img, out_size[0], out_size[1])
    yuyv = po.convert_rgb_to_yuyv(img)
    return img, (yuyv_to_nv12(yuyv) if nv12 else yuyv)


def _same(got, want, what, tag):
    assert np.array_equal(np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)), f"{what} differs {tag}"


class _Stream:
    """one oracle stream of one camera (always filtered on: it gives the mask and the filtered-on composite) and what a
    frame of it must give for a filter switch"""

    def __init__(self, key, W, H, bg=None, k=0):
        self.o = po.MaskGen(model_path(key), W, H)
        self.bg, self.k = bg, k

    def expect(self, frame, fmt, active, flip=0, out_size=None, bg=None):
        bgr = camera_bgr(frame, fmt)
        fh, fv = _code(flip)
        ro, ry, rm = self.o.composite_ex(bgr, self.bg if bg is None else bg, bgblur=self.k, flip_h=fh, flip_v=fv, out_size=out_size)
        if active:
            return ro, (yuyv_to_nv12(ry) if fmt == "nv12" else ry), rm, self.o.ofinal
        po_, pv = passthrough(bgr, flip, out_size, nv12=fmt == "nv12")
        return po_, pv, rm, self.o.ofinal


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def _addr(a):
    return a.ctypes.data if a is not None else 0


def _plain_call(g, fmt, frames, device=False):
    """one plain call of frames in `fmt` on host buffers (or the device entry points, which on the emulator take host
    memory) -> (out, video, mask)"""
    n, H, W = frames.shape[0], g.height, g.width
    ow, oh = g.out_width, g.out_height
    if fmt == "bgr":
        return g.composite(frames)
    if not device:
        return g.composite_yuyv(frames) if fmt == "yuyv" else g.composite_nv12(frames)
    buf = np.ascontiguousarray(frames)
    out = np.empty((n, oh, ow, 3), np.uint8)
    mask = np.empty((n, H, W), np.uint8)
    if fmt == "yuyv":
        vid = np.empty((n, oh, ow, 2), np.uint8)
        g.composite_yuyv_device(n, _addr(buf), _addr(out), _addr(vid), _addr(mask), sync=True)
    else:
        vid = np.empty((n, oh * 3 // 2, ow), np.uint8)
        g.composite_nv12_device(n, _addr(buf), _addr(out), _addr(vid), _addr(mask), sync=True)
    return out, vid, mask


def _frames(fmt, W, H, ts, stream=0):
    if fmt == "yuyv":
        return np.stack([synth.yuyv_frame(W, H, t=t, stream=stream) for t in ts])
    if fmt == "nv12":
        return np.stack([nv12_frame(W, H, t=t, stream=stream) for t in ts])
    return np.stack([synth.frame(W, H, t=t, stream=stream) for t in ts])


def _check_plain(g, got, want, b, tag):
    out, vid, mask = got
    ro, rv, rm, rf = want
    _same(g.stage_u8(2, b), rf, "smoother state", tag)
    _same(mask[b], rm, "mask", tag)
    _same(out[b], ro, "composite", tag)
    _same(vid[b], rv, "video output", tag)


@pytest.mark.parametrize("fmt,device", [("bgr", False), ("yuyv", False), ("yuyv", True), ("nv12", False), ("nv12", True)],
                         ids=["bgr", "yuyv_host", "yuyv_device", "nv12_host", "nv12_device"])
def test_plain_filter_off(emu_lib, fmt, device):
    """a plain context with the filter off, then with a context flip, an output size, and an odd output height (flip
    before resize): the camera frame passes through; masks and smoother states are those of the filter-on stream"""
    key, W, H, n = "meet_lite", 320, 240, 2
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
    g.set_background(bg)
    g.set_filter(False)
    s = _Stream(key, W, H, bg)
    odd = (160, 120) if fmt == "nv12" else (240, 179)      # NV12 output sizes are even
    t = 0
    for flip, size in ((0, None), (H_ | V_, None), (H_, (240, 180)), (V_, odd)):
        g.set_output(*_code(flip), out_size=size)
        frames = _frames(fmt, W, H, range(t, t + n))
        got = _plain_call(g, fmt, frames, device)
        for b in range(n):
            _check_plain(g, got, s.expect(frames[b], fmt, False, flip, size), b, (fmt, device, flip, size, t + b))
        t += n
    g.close()


def test_plain_toggle_sequence(emu_lib):
    """on, off, off, on over one stream: every frame equals the oracle stream toggled the same way, and the frames after
    switching back on equal an always-on stream (the smoother never stopped)"""
    key, W, H, n = "meet_lite", 320, 240, 2
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
    g.set_background(bg)
    s = _Stream(key, W, H, bg)
    t = 0
    for active in (True, False, False, True):
        g.set_filter(active)
        frames = _frames("bgr", W, H, range(t, t + n))
        got = g.composite(frames)
        for b in range(n):
            _check_plain(g, got, s.expect(frames[b], "bgr", active), b, (active, t + b))
        t += n
    g.close()


def _gauss_launches(lib, k):
    img = synth.frame(64, 48)
    l0 = lib.bsb_total_launches()
    api.gaussian_blur(lib, img, k)
    return lib.bsb_total_launches() - l0


@pytest.mark.parametrize("fmt", ["bgr", "yuyv"])
def test_plain_camera_blur_off(emu_lib, fmt):
    """camera-blur mode (no background, bgblur 9): with the filter off the call launches no Gaussian, and its output is
    the camera frame"""
    key, W, H, n = "meet_lite", 320, 240, 2
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
    g.set_bgblur(9)
    s = _Stream(key, W, H, None, 9)
    frames = _frames(fmt, W, H, range(n))
    got = _plain_call(g, fmt, frames)
    on = g.launches_per_call
    for b in range(n):
        _check_plain(g, got, s.expect(frames[b], fmt, True), b, ("on", b))
    g.set_filter(False)
    frames = _frames(fmt, W, H, range(n, 2 * n))
    got = _plain_call(g, fmt, frames)
    assert on - g.launches_per_call == _gauss_launches(emu_lib, 9), (on, g.launches_per_call)
    for b in range(n):
        _check_plain(g, got, s.expect(frames[b], fmt, False), b, ("off", b))
    g.close()


def test_plain_ring_keeps_moving(emu_lib):
    """a ring background at advance 1: after filter-off frames the ring image blended on re-enable is the one an
    always-on stream blends (the cursor moved by n * advance for every call)"""
    key, W, H = "meet_lite", 320, 240
    base = synth.background()
    ring = np.stack([np.roll(base, 41 * i, axis=1) for i in range(3)])
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    g.set_background_ring(ring, advance=1)
    s = _Stream(key, W, H)
    cursor, t = 0, 0
    for active, n in ((True, 2), (False, 2), (False, 1), (True, 2), (True, 1)):
        g.set_filter(active)
        frames = _frames("bgr", W, H, range(t, t + n))
        got = g.composite(frames)
        for b in range(n):
            want = s.expect(frames[b], "bgr", active, bg=ring[(cursor + b) % 3])
            _check_plain(g, got, want, b, (active, t + b))
        cursor, t = (cursor + n) % 3, t + n
    g.close()


class _Sources:
    """five sources on the emulator: 0 the context image (follows everything), 1 its own image (flip H, own size), 2 camera
    blur 9 (no image), 3 the context image at strength 5 (flip H|V), 4 a ring of three images at advance 1 (own size)"""

    def __init__(self, lib, key="meet_lite", W=320, H=240):
        self.lib, self.key, self.W, self.H = lib, key, W, H
        bg = synth.background()
        self.ctx_bg = bg[::-1].copy()
        own = np.roll(bg, 90, axis=1)
        self.ring = np.stack([np.roll(bg, 53 * i, axis=0) for i in range(3)])
        g = self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=4)
        g.set_background(self.ctx_bg)
        g.set_sources(5)
        g.set_source_background(1, own)
        g.set_source_effect(2, "none", 9)
        g.set_source_effect(3, "default", 5)
        g.set_source_background_ring(4, self.ring, advance=1)
        self.flip = {0: 0, 1: H_, 2: 0, 3: H_ | V_, 4: 0}
        g.set_source_flip(1, flip_h=True)
        g.set_source_flip(3, flip_h=True, flip_v=True)
        self.size = {s: None for s in range(5)}
        for s, size in ((1, (240, 180)), (4, (160, 120))):
            g.set_source_output(s, size)
            self.size[s] = size
        self.streams = [_Stream(key, W, H, b, k) for b, k in ((self.ctx_bg, 0), (own, 0), (None, 9), (self.ctx_bg, 5), (None, 0))]
        self.filters = {s: None for s in range(5)}
        self.ctx = True
        self.cursor = 0
        self.t = [0] * 5

    def set_filter(self, active):
        self.g.set_filter(active)
        self.ctx = active

    def set_source(self, s, active):
        self.g.set_source_filter(s, active)
        self.filters[s] = active

    def active(self, s):
        return self.ctx if self.filters[s] is None else self.filters[s]

    def call(self, ids):
        fr = np.stack([synth.frame(self.W, self.H, t=self.t[s], stream=s) for s in ids])
        out, yuyv, mask = self.g.composite_sources(fr, ids)
        for b, s in enumerate(ids):
            bg = self.ring[self.cursor] if s == 4 else None
            want = self.streams[s].expect(fr[b], "bgr", self.active(s), self.flip[s], self.size[s], bg=bg)
            tag = (ids, b, s, self.t[s], self.active(s))
            _same(mask[b], want[2], "mask", tag)
            _same(out[b], want[0], "composite", tag)
            _same(yuyv[b], want[1], "YUYV", tag)
            self.t[s] += 1
        if 4 in ids:
            self.cursor = (self.cursor + 1) % 3
        return self.g.launches_per_call


def test_sources_mixed_switches(emu_lib):
    """follow / off / on mixed with the per-source effects, flips, own sizes and a ring, over calls of varying ids and
    per-call toggles; the context switch reaches only the sources that follow it"""
    d = _Sources(emu_lib)
    d.call([0, 1, 2, 3])
    d.set_source(1, False)
    d.set_source(3, True)
    d.call([3, 1, 4, 0])
    d.set_filter(False)                                 # 0, 2 and 4 follow; 3 stays on, 1 stays off
    d.call([0, 1, 2, 3])
    d.call([4, 2])
    d.set_source(2, True)
    d.set_source(1, None)                               # follows the context: off
    d.call([1, 2, 4, 3])
    d.set_filter(True)
    d.set_source(0, False)
    d.call([2, 0, 4])
    d.set_source(0, None)
    d.set_source(2, None)
    d.set_source(3, None)
    d.call([0, 1, 2, 3])
    d.g.close()


def test_sources_camera_blur_off_costs_no_gaussian(emu_lib):
    """a camera-blur source switched off adds no Gaussian to the call: the call with it off issues the Gaussian's
    launches fewer than with it on"""
    d = _Sources(emu_lib)
    on = d.call([2, 0])
    d.set_source(2, False)
    off = d.call([2, 0])
    assert on - off == _gauss_launches(emu_lib, 9), (on, off)
    d.set_source(2, None)
    assert d.call([2, 0]) == on
    d.g.close()


def test_fed_masks(emu_lib):
    """bsb_test_feed(BSB_FEED_MASK): with all-255 masks the filtered-off frames still show the camera and the others the
    background; with mixed masks the mask output is identical whatever the switch"""
    key, W, H = "meet_lite", 320, 240
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    bg = synth.background()
    g.set_background(bg)
    g.set_sources(4)
    oh, ow, _ = g.feed_shape(2)
    fr = np.stack([synth.frame(W, H, t=0, stream=s) for s in range(4)])
    ids = [0, 1, 2, 3]
    g.set_source_filter(1, False)
    g.set_source_filter(3, False)
    g.feed(2, np.full((4, oh, ow), 255, np.uint8))
    out, yuyv, mask = g.composite_sources(fr, ids)
    bgw = po.resize_linear_u8(bg, W, H)
    for b in range(4):
        want = fr[b] if b in (1, 3) else bgw
        _same(out[b], want, "composite", ("all-255", b))
        _same(yuyv[b], po.convert_rgb_to_yuyv(want), "YUYV", ("all-255", b))
        assert (mask[b] == 255).all(), b
    rng = np.random.default_rng(5)
    masks = rng.integers(0, 256, (4, oh, ow), dtype=np.uint8)
    masks[:, : oh // 2] = 0
    got = []
    for off in (False, True):
        for s in range(4):
            g.set_source_filter(s, not off)
        g.feed(2, masks)
        got.append(g.composite_sources(fr, ids))
    _same(got[0][2], got[1][2], "mask", "mixed masks")
    for b in range(4):
        _same(got[1][0][b], fr[b], "composite", ("mixed, off", b))
    g.close()


def test_filter_errors_and_reset(emu_lib):
    key, W, H = "meet_lite", 320, 240
    L = emu_lib
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    for v in (2, -1, 7):
        assert L.bsb_set_filter(g._h, v) == 0 and b"filter" in L.bsb_last_error(), v
    assert L.bsb_set_source_filter(g._h, 0, 0) == 0 and b"set_sources" in L.bsb_last_error()
    g.set_sources(3)
    for s, v, msg in ((3, 0, b"out of range"), (-1, 1, b"out of range"), (0, 2, b"filter"), (1, -2, b"filter")):
        assert L.bsb_set_source_filter(g._h, s, v) == 0, (s, v)
        assert msg in L.bsb_last_error(), (s, v, L.bsb_last_error())
    with pytest.raises(api.BackscrubError, match="bsb_set_source_filter"):
        g.set_source_filter(5, False)
    # still usable, still on everywhere; set_sources resets every source to follow the context
    bg = synth.background()
    g.set_background(bg)
    g.set_source_filter(0, False)
    g.set_source_filter(1, False)
    g.set_sources(3)
    o = [_Stream(key, W, H, bg) for _ in range(2)]
    fr = np.stack([synth.frame(W, H, t=0, stream=s) for s in (0, 1)])
    out, yuyv, mask = g.composite_sources(fr, [0, 1])
    for b in range(2):
        ro, ry, rm, _ = o[b].expect(fr[b], "bgr", True)
        _same(out[b], ro, "composite", b)
        _same(yuyv[b], ry, "YUYV", b)
        _same(mask[b], rm, "mask", b)
    g.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


@pytest.fixture
def post_tile():
    """k_post_tma's tile width for the contexts of one test (set before they are created), restored afterwards"""
    import backscrub_b200 as bs
    yield lambda tw: bs.set_tuning("post_tile", tw)
    bs.set_tuning("post_tile", 0)


def _pitched(frames, pitch, uv_offset, stride):
    n, H3, W = frames.shape
    H = H3 * 2 // 3
    buf = np.full(n * stride, 0x5A, np.uint8)
    for b, f in enumerate(frames):
        base = b * stride
        for y in range(H):
            buf[base + y * pitch: base + y * pitch + W] = f[y]
        for r in range(H // 2):
            buf[base + uv_offset + r * pitch: base + uv_offset + r * pitch + W] = f[H + r]
    return buf


# source s: (background, strength) — the context image, its own image, camera blur 25 (no image), the context image at 7
EFFECTS = [("ctx", 0), ("own", 0), ("none", 25), ("ctx", 7)]
FLIPS8 = [None, 0, H_, H_ | V_, V_, None, H_, 0]
# filter switches of the eight sources (None: follow the context); source 6 is a camera-blur source switched off
FILTERS8 = [None, False, True, False, None, False, False, True]
CALLS8 = ([0, 1, 2, 3, 4, 5, 6, 7], [7, 5, 3, 1], [6, 0, 4, 2, 1])


class _Dev:
    """a sources context fed by one of the three entry points (device YUYV, device NV12 with a layout, host BGR), and per
    source a plain batch-1 context set up as that source with the filter on: it gives every mask and every filtered-on
    frame; a filtered-off frame must be the oracle's pass-through of the camera frame"""

    def __init__(self, lib, key, W, H, n_sources, fmt="yuyv", layout=None, flips=None, filters=None, want_mask=True):
        import torch
        self.torch, self.lib, self.key, self.W, self.H, self.fmt = torch, lib, key, W, H, fmt
        self.want_mask = want_mask
        bg = synth.background()
        self.ctx_bg = bg[::-1].copy()
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=n_sources)
        self.g.set_background(self.ctx_bg)
        self.g.set_sources(n_sources)
        self.fx = {}
        for s in range(n_sources):
            kind, k = EFFECTS[s % len(EFFECTS)]
            if kind == "own":
                self.fx[s] = (np.roll(bg, 37 * s, axis=1), k)
                self.g.set_source_background(s, self.fx[s][0])
            elif kind == "none":
                self.fx[s] = (None, k)
                self.g.set_source_effect(s, "none", k)
            else:
                self.fx[s] = (self.ctx_bg, k)
                self.g.set_source_effect(s, "default", k)
        self.flips = {s: (flips[s % len(flips)] if flips else None) for s in range(n_sources)}
        for s, code in self.flips.items():
            if code is not None:
                self.g.set_source_flip(s, flip_h=bool(code & H_), flip_v=bool(code & V_))
        self.filters = {s: None for s in range(n_sources)}
        if filters:
            for s in range(n_sources):
                self.set_source(s, filters[s % len(filters)])
        self.ctx = True
        self.ref = {}
        self.t = [0] * n_sources
        dev = "cuda:0"
        self.fn = W * H * 3 // 2
        self.pitch, self.uv, self.stride = layout if layout else (W, W * H, self.fn)
        mb = n_sources
        if fmt == "nv12":
            self.d_in = torch.empty(mb * self.stride, dtype=torch.uint8, device=dev)
            self.d_vid = torch.empty(mb * self.fn, dtype=torch.uint8, device=dev)
        elif fmt == "yuyv":
            self.d_in = torch.empty((mb, H, W, 2), dtype=torch.uint8, device=dev)
            self.d_vid = torch.empty((mb, H, W, 2), dtype=torch.uint8, device=dev)
        if fmt != "bgr":
            self.d_out = torch.empty((mb, H, W, 3), dtype=torch.uint8, device=dev)
            self.d_mask = torch.empty((mb, H, W), dtype=torch.uint8, device=dev)

    def set_filter(self, active):
        self.g.set_filter(active)
        self.ctx = active

    def set_source(self, s, active):
        self.g.set_source_filter(s, active)
        self.filters[s] = active

    def active(self, s):
        return self.ctx if self.filters[s] is None else self.filters[s]

    def code(self, s):
        return self.flips[s] or 0

    def plain(self, s):
        bg, k = self.fx[s]
        if s not in self.ref:
            c = api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1)
            if bg is not None:
                c.set_background(bg)
            if k:
                c.set_bgblur(k)
            if self.code(s):
                c.set_output(*_code(self.code(s)))
            bufs = None
            if self.fmt != "bgr":
                cam = self.stride if self.fmt == "nv12" else self.W * self.H * 2
                vid = self.fn if self.fmt == "nv12" else self.W * self.H * 2
                bufs = [self.torch.empty(n, dtype=self.torch.uint8, device="cuda:0") for n in (cam, self.W * self.H * 3, vid, self.W * self.H)]
            self.ref[s] = (c, bufs)
        return self.ref[s]

    def frame(self, s, t):
        if self.fmt == "nv12":
            return nv12_frame(self.W, self.H, t, s)
        if self.fmt == "yuyv":
            return synth.yuyv_frame(self.W, self.H, t=t, stream=s)
        return synth.frame(self.W, self.H, t=t, stream=s)

    def load(self, ids):
        host = np.stack([self.frame(s, self.t[s]) for s in ids])
        if self.fmt == "nv12":
            buf = _pitched(host, self.pitch, self.uv, self.stride)
            self.d_in[:buf.size].copy_(self.torch.from_numpy(buf))
        elif self.fmt == "yuyv":
            self.d_in[:len(ids)].copy_(self.torch.from_numpy(host))
        self.host = host

    def run(self, ids):
        n = len(ids)
        m = self.d_mask.data_ptr() if self.fmt != "bgr" and self.want_mask else 0
        if self.fmt == "nv12":
            self.g.composite_sources_nv12_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(), m,
                                                 sync=True, pitch=self.pitch, uv_offset=self.uv, in_stride=self.stride)
        elif self.fmt == "yuyv":
            self.g.composite_sources_yuyv_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(), m, sync=True)
        else:
            self._res = self.g.composite_sources(self.host, ids, want_mask=self.want_mask)

    def results(self, n):
        if self.fmt == "bgr":
            return self._res
        vid = self.d_vid[:n * self.fn].cpu().numpy().reshape(n, -1) if self.fmt == "nv12" else self.d_vid[:n].cpu().numpy()
        return self.d_out[:n].cpu().numpy(), vid, (self.d_mask[:n].cpu().numpy() if self.want_mask else None)

    def check(self, ids, got, sample=None):
        out, vid, mask = got
        for b, s in enumerate(ids):
            if sample is not None and s not in sample:
                self.t[s] += 1
                continue
            c, bufs = self.plain(s)
            fr = self.frame(s, self.t[s])
            if self.fmt == "bgr":
                r_out, r_vid, r_mask = c.composite(fr)
            else:
                r_in, r_out, r_vid, r_mask = bufs
                r_in[:fr.size].copy_(self.torch.from_numpy(fr.reshape(-1)))
                if self.fmt == "nv12":
                    c.composite_nv12_device(1, r_in.data_ptr(), r_out.data_ptr(), r_vid.data_ptr(), r_mask.data_ptr(), sync=True)
                else:
                    c.composite_yuyv_device(1, r_in.data_ptr(), r_out.data_ptr(), r_vid.data_ptr(), r_mask.data_ptr(), sync=True)
                r_out, r_vid, r_mask = r_out.cpu().numpy(), r_vid.cpu().numpy(), r_mask.cpu().numpy()
            if not self.active(s):
                r_out, r_vid = passthrough(camera_bgr(fr, self.fmt), self.code(s), nv12=self.fmt == "nv12")
            tag = (self.fmt, ids, b, s, self.t[s], self.active(s), self.code(s))
            if mask is not None:
                _same(mask[b], r_mask, "mask", tag)
            _same(out[b], r_out, "composite", tag)
            _same(vid[b], r_vid, "video output", tag)
            self.t[s] += 1

    def step(self, ids, sample=None):
        self.load(ids)
        self.run(ids)
        self.check(ids, self.results(len(ids)), sample=sample)
        return self.g.launches_per_call

    def close(self):
        self.g.close()
        for c, _ in self.ref.values():
            c.close()


GEOMETRIES = [(1280, 720, 0), (1296, 720, 64), (1296, 720, 128)]
FORMATS = ["yuyv", "nv12", "nv12_pitched", "bgr"]


def _layout(fmt, H):
    return (1536, 1536 * (H + 16), 1536 * (H + 16) + 1536 * H // 2) if fmt == "nv12_pitched" else None


@pytest.mark.gpu
@pytest.mark.parametrize("geo", GEOMETRIES, ids=["1280x720", "1296x720_tw64", "1296x720_tw128"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_gpu_meet_720p_filters(gpu_lib, post_tile, geo, fmt):
    """Meet full, 8 sources with mixed filters, flips and effects: k_post_tma passes the filtered-off frames through
    (mirrored in place where flipped), and a call with filtered-off frames issues as many launches as the same call with
    none (fewer only when a camera-blur frame is off and no other frame needs its Gaussian class).  1296x720 has ragged
    right and bottom tiles."""
    W, H, tw = geo
    post_tile(tw)
    d = _Dev(gpu_lib, "meet_full", W, H, 8, fmt="nv12" if fmt.startswith("nv12") else fmt, layout=_layout(fmt, H), flips=FLIPS8)
    base = {}
    for ids in CALLS8:
        base[tuple(ids)] = d.step(ids)
    for s in range(8):
        d.set_source(s, FILTERS8[s])
    for ids in CALLS8:
        n = d.step(ids)
        if fmt != "bgr":
            assert d.g.yuyv_native, ids
        blur_on = any(EFFECTS[s % 4][0] == "none" and d.active(s) for s in ids)
        blur_off = any(EFFECTS[s % 4][0] == "none" and not d.active(s) for s in ids)
        if blur_off and not blur_on:
            assert n <= base[tuple(ids)], (ids, n, base[tuple(ids)])
        else:
            assert n == base[tuple(ids)], (ids, n, base[tuple(ids)])
    d.set_filter(False)                                 # sources 0 and 4 follow
    d.step(CALLS8[0])
    assert d.g.launches_per_call == base[tuple(CALLS8[0])]
    d.set_filter(True)
    d.step(CALLS8[2])
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuyv", "nv12", "bgr"])
def test_gpu_without_mask_output(gpu_lib, fmt):
    """no mask output: filtered-off frames load no mask patch and are pure camera -> BGR / YUYV / NV12 copies"""
    d = _Dev(gpu_lib, "meet_full", 1280, 720, 4, fmt=fmt, flips=[H_, 0, V_, None], filters=[False, None, False, True], want_mask=False)
    d.step([0, 1, 2, 3])
    d.set_filter(False)
    d.step([3, 1, 0, 2])
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuyv", "nv12", "bgr"])
def test_gpu_fallback_kernels(gpu_lib, fmt):
    """post_tma=0: k_post_fast passes the frames through itself (the flips run in the tail); same bytes"""
    import backscrub_b200 as bs
    bs.set_tuning("post_tma", 0)
    try:
        d = _Dev(gpu_lib, "meet_full", 1280, 720, 8, fmt=fmt, flips=FLIPS8, filters=FILTERS8)
        for ids in CALLS8:
            d.step(ids)
            assert not d.g.yuyv_native, ids
        d.close()
    finally:
        bs.set_tuning("post_tma", 1)


@pytest.mark.gpu
def test_gpu_graph_replayed_for_new_filters(gpu_lib):
    """sources: once the 'some off' and the 'none off' graphs exist, any change of the switches replays one of them (a
    call whose camera-blur frames are all off has no Gaussian class, and so a graph of its own); plain: toggling replays
    once both states have been captured"""
    d = _Dev(gpu_lib, "meet_full", 1280, 720, 4, flips=[H_, 0, V_, None])
    ids = [0, 1, 2, 3]
    d.step(ids)                                         # none off: captured

    def call(filters, replays):
        for s, v in enumerate(filters):
            d.set_source(s, v)
        d.load(ids)
        l0 = gpu_lib.bsb_total_launches()
        d.run(ids)
        assert (gpu_lib.bsb_total_launches() == l0) == replays, (filters, replays)
        d.check(ids, d.results(4))

    call([False, None, None, None], False)            # the first call with a frame off captures its graph
    call([None, False, True, False], True)
    call([True, True, True, True], True)
    call([False, False, True, False], True)
    call([None, None, None, None], True)
    # source 2 blurs its camera frame: with it off as well the call has no Gaussian class, which is a graph of its own
    call([False, False, False, False], False)
    call([True, False, False, True], True)
    d.set_filter(False)
    call([None, None, True, None], True)
    d.close()

    import torch
    W, H = 1280, 720
    g = api.MaskGen(gpu_lib, model_path("meet_full"), W, H, max_batch=2)
    g.set_background(synth.background())
    s = _Stream("meet_full", W, H, synth.background())
    d_in = torch.empty((2, H, W, 2), dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty((2, H, W, 3), dtype=torch.uint8, device="cuda:0")
    d_vid = torch.empty((2, H, W, 2), dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((2, H, W), dtype=torch.uint8, device="cuda:0")
    t = 0
    for active, replays in ((True, False), (False, False), (True, True), (False, True), (False, True)):
        g.set_filter(active)
        frames = _frames("yuyv", W, H, range(t, t + 2))
        d_in.copy_(torch.from_numpy(frames))
        l0 = gpu_lib.bsb_total_launches()
        g.composite_yuyv_device(2, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr(), sync=True)
        assert (gpu_lib.bsb_total_launches() == l0) == replays, (active, replays)
        assert g.yuyv_native
        out, vid, mask = d_out.cpu().numpy(), d_vid.cpu().numpy(), d_mask.cpu().numpy()
        for b in range(2):
            ro, rv, rm, _ = s.expect(frames[b], "yuyv", active)
            tag = (active, t + b)
            _same(mask[b], rm, "mask", tag)
            _same(out[b], ro, "composite", tag)
            _same(vid[b], rv, "YUYV", tag)
        t += 2
    g.close()


@pytest.mark.gpu
def test_gpu_plain_camera_blur_off(gpu_lib):
    """plain camera-blur mode with the filter off: no Gaussian, the YUYV frames are read in place, the output is the
    camera frame and the mask the filter-on stream's"""
    import torch
    W, H = 1280, 720
    g = api.MaskGen(gpu_lib, model_path("meet_full"), W, H, max_batch=2)
    g.set_bgblur(25)
    s = _Stream("meet_full", W, H, None, 25)
    d_in = torch.empty((2, H, W, 2), dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty((2, H, W, 3), dtype=torch.uint8, device="cuda:0")
    d_vid = torch.empty((2, H, W, 2), dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((2, H, W), dtype=torch.uint8, device="cuda:0")
    launches = {}
    for t, active in enumerate((True, False, True)):
        g.set_filter(active)
        frames = _frames("yuyv", W, H, range(2 * t, 2 * t + 2))
        d_in.copy_(torch.from_numpy(frames))
        g.composite_yuyv_device(2, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr(), sync=True)
        launches[active] = g.launches_per_call
        assert g.yuyv_native == (not active)
        out, vid, mask = d_out.cpu().numpy(), d_vid.cpu().numpy(), d_mask.cpu().numpy()
        for b in range(2):
            ro, rv, rm, _ = s.expect(frames[b], "yuyv", active)
            _same(mask[b], rm, "mask", (active, b))
            _same(out[b], ro, "composite", (active, b))
            _same(vid[b], rv, "YUYV", (active, b))
    assert launches[False] < launches[True], launches
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("active", [False, True], ids=["all_off", "all_on"])
def test_gpu_64_sources(gpu_lib, active):
    d = _Dev(gpu_lib, "meet_lite", 640, 480, 64, flips=[None, 0, H_, H_ | V_, V_])
    d.set_filter(active)
    sample = {0, 1, 2, 3, 4, 17, 42, 62, 63}
    d.step(list(range(64)), sample=sample)
    d.step(list(range(63, -1, -1)), sample=sample)
    d.close()
