"""The transparent output format (bsb_set_out_format BSB_OUT_BGRA, MaskGen.set_out_format("bgra")).

In BGRA format the `out` buffer of every composite entry point holds, for frame b with camera frame C (as the fused path
reads it) and mask M (the W x H mask the same call writes):

    A0 = (C.B, C.G, C.R, 255 - M)        (alpha 255 when the frame's filter is off)
    out_b = cv::resize(cv::flip(A0))      with the flip code and output size the frame's composite gets

The video output and the mask are byte for byte those of a BGR-format call on the same frames: every test runs a twin
context that never leaves BGR format and compares them.

`-m "not gpu"`: the kernel-logic emulator build (k_post_fast / k_post and k_tail) against the oracle: po.MaskGen.composite_ex
for mask and video, numpy for the flip, po.resize_linear_u8 on 4 channels for the resize.
`-m gpu`: the sm_90a library (k_post_tma's BGRA instantiations, k_tail) on the H100."""

import ctypes

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


def expect_bgra(cam, mask, active=True, flip=0, out_size=None):
    """the definition: camera bytes with alpha 255 - mask (255 with the filter off), cv::flip, then cv::resize 8UC4"""
    H, W = mask.shape
    alpha = (255 - mask).astype(np.uint8) if active else np.full((H, W), 255, np.uint8)
    img = np.dstack([cam, alpha])
    if flip & H_:
        img = img[:, ::-1]
    if flip & V_:
        img = img[::-1]
    img = np.ascontiguousarray(img)
    if out_size and tuple(out_size) != (W, H):
        img = po.resize_linear_u8(img, out_size[0], out_size[1])
    return img


def passthrough(cam, flip=0, out_size=None):
    """the composite of a frame whose filter is off: the camera frame, cv::flip, cv::resize (the oracle's functions)"""
    img = cam
    if flip:
        img = po.flip(img, *_code(flip))
    H, W = img.shape[:2]
    if out_size and tuple(out_size) != (W, H):
        img = po.resize_linear_u8(img, out_size[0], out_size[1])
    return img


def _same(got, want, what, tag):
    got, want = np.asarray(got), np.asarray(want)
    assert got.size == want.size, f"{what} size {got.size} != {want.size} {tag}"
    assert np.array_equal(got.reshape(-1), want.reshape(-1)), f"{what} differs {tag}"


def _frames(fmt, W, H, ts, stream=0):
    if fmt == "yuyv":
        return np.stack([synth.yuyv_frame(W, H, t=t, stream=stream) for t in ts])
    if fmt == "nv12":
        return np.stack([nv12_frame(W, H, t=t, stream=stream) for t in ts])
    return np.stack([synth.frame(W, H, t=t, stream=stream) for t in ts])


def _addr(a):
    return a.ctypes.data if a is not None else 0


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def _plain_call(g, fmt, frames, device=False, video=True):
    """one plain call on host buffers (or the device entry points, which on the emulator take host memory) -> (out,
    video, mask); `out` has the context's format"""
    n, H, W = frames.shape[0], g.height, g.width
    ow, oh, oc = g.out_width, g.out_height, g.out_channels
    if not device:
        if fmt == "bgr":
            return g.composite(frames, want_yuyv=video)
        if fmt == "nv12":
            return g.composite_nv12(frames, want_nv12=video)
        out = np.empty((n, oh, ow, oc), np.uint8)
        vid = np.empty((n, oh, ow, 2), np.uint8) if video else None
        mask = np.empty((n, H, W), np.uint8)
        g.composite_yuyv_into(np.ascontiguousarray(frames), out, vid, mask)
        return out, vid, mask
    buf = np.ascontiguousarray(frames)
    out = np.empty((n, oh, ow, oc), np.uint8)
    mask = np.empty((n, H, W), np.uint8)
    vid = None
    if fmt == "bgr":
        vid = np.empty((n, oh, ow, 2), np.uint8) if video else None
        g.composite_device(n, _addr(buf), _addr(out), _addr(vid), _addr(mask), sync=True)
    elif fmt == "yuyv":
        vid = np.empty((n, oh, ow, 2), np.uint8) if video else None
        g.composite_yuyv_device(n, _addr(buf), _addr(out), _addr(vid), _addr(mask), sync=True)
    else:
        vid = np.empty((n, oh * 3 // 2, ow), np.uint8) if video else None
        g.composite_nv12_device(n, _addr(buf), _addr(out), _addr(vid), _addr(mask), sync=True)
    return out, vid, mask


class _Twins:
    """a BGRA-format context, a BGR-format twin set up the same way, and the oracle stream of the camera"""

    def __init__(self, lib, key="meet_lite", W=320, H=240, n=2, bg="image", k=0):
        self.W, self.H, self.n = W, H, n
        self.bg = synth.background() if bg == "image" else None
        self.ring = None
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=n)
        self.t = api.MaskGen(lib, model_path(key), W, H, max_batch=n)
        self.o = po.MaskGen(model_path(key), W, H)
        self.k = k
        for c in (self.g, self.t):
            if self.bg is not None:
                c.set_background(self.bg)
            if k:
                c.set_bgblur(k)
        self.g.set_out_format("bgra")
        self.flip, self.size, self.active = 0, None, True

    def set_output(self, flip, size):
        for c in (self.g, self.t):
            c.set_output(*_code(flip), out_size=size)
        self.flip, self.size = flip, size

    def set_filter(self, active):
        for c in (self.g, self.t):
            c.set_filter(active)
        self.active = active

    def step(self, fmt, frames, device=False, video=True, tag=()):
        got = _plain_call(self.g, fmt, frames, device, video)
        twin = _plain_call(self.t, fmt, frames, device, video)
        out, vid, mask = got
        for b in range(frames.shape[0]):
            cam = camera_bgr(frames[b], fmt)
            fh, fv = _code(self.flip)
            _, ry, rm = self.o.composite_ex(cam, self.bg, bgblur=self.k, flip_h=fh, flip_v=fv, out_size=self.size, want_yuyv=video)
            t = tag + (b,)
            _same(mask[b], rm, "mask", t)
            _same(twin[2][b], rm, "twin mask", t)
            if video and not self.active:
                ry = po.convert_rgb_to_yuyv(passthrough(cam, self.flip, self.size))
            if video:
                _same(vid[b], yuyv_to_nv12(ry) if fmt == "nv12" else ry, "video", t)
                _same(twin[1][b], vid[b], "twin video", t)
            _same(out[b], expect_bgra(cam, rm, self.active, self.flip, self.size), "bgra", t)
        return got, twin

    def close(self):
        self.g.close()
        self.t.close()


@pytest.mark.parametrize("fmt,device", [("bgr", False), ("bgr", True), ("yuyv", False), ("yuyv", True), ("nv12", False),
                                        ("nv12", True)],
                         ids=["bgr_host", "bgr_device", "yuyv_host", "yuyv_device", "nv12_host", "nv12_device"])
def test_plain_bgra(emu_lib, fmt, device):
    """plain calls, unflipped at W x H, then each flip, then 640x360, exactly half size (the 2x2 area case) and an odd size
    (no video there: YUYV and NV12 need even sizes); with and without a video output"""
    T = _Twins(emu_lib)
    t = 0
    for flip, size, video in ((0, None, True), (0, None, False), (H_, None, True), (V_, None, False), (H_ | V_, None, True),
                              (0, (640, 360), True), (H_, (160, 120), True), (V_, (161, 121), False)):
        T.set_output(flip, size)
        frames = _frames(fmt, T.W, T.H, range(t, t + T.n))
        T.step(fmt, frames, device, video, (fmt, device, flip, size, video, t))
        t += T.n
    T.close()


def test_plain_filter_off_alpha_255(emu_lib):
    """filter off: alpha 255 everywhere, the colour bytes still the camera's; the mask is still the filter-on mask"""
    T = _Twins(emu_lib)
    t = 0
    for active, flip, size in ((False, 0, None), (False, H_, (240, 180)), (True, 0, None)):
        T.set_filter(active)
        T.set_output(flip, size)
        frames = _frames("yuyv", T.W, T.H, range(t, t + T.n))
        (out, _, _), _ = T.step("yuyv", frames, tag=(active, flip, size))
        if not active:
            assert (out[..., 3] == 255).all()
        t += T.n
    T.close()


def _gauss_launches(lib, k):
    img = synth.frame(64, 48)
    l0 = lib.bsb_total_launches()
    api.gaussian_blur(lib, img, k)
    return lib.bsb_total_launches() - l0


@pytest.mark.parametrize("fmt", ["bgr", "yuyv"])
def test_camera_blur_bgra_only_has_no_gaussian(emu_lib, fmt):
    """camera-blur mode (no background, bgblur 9): a BGRA call with a video output blurs the camera frame for the video, a
    BGRA call without one launches no Gaussian"""
    T = _Twins(emu_lib, bg=None, k=9)
    frames = _frames(fmt, T.W, T.H, range(2))
    T.step(fmt, frames, video=True, tag=("video",))
    with_video = T.g.launches_per_call
    frames = _frames(fmt, T.W, T.H, range(2, 4))
    T.step(fmt, frames, video=False, tag=("bgra only",))
    assert with_video - T.g.launches_per_call == _gauss_launches(emu_lib, 9), (with_video, T.g.launches_per_call)
    T.close()


def test_ring_cursor_moves_without_blend(emu_lib):
    """a ring background at advance 1: BGRA-only calls blend nothing but move the cursor, so the BGR calls after them blend
    the ring images of a context that composited every frame"""
    key, W, H = "meet_lite", 320, 240
    base = synth.background()
    ring = np.stack([np.roll(base, 41 * i, axis=1) for i in range(3)])
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    t_ = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    for c in (g, t_):
        c.set_background_ring(ring, advance=1)
    t = 0
    for fmt_g, n in (("bgra", 2), ("bgra", 1), ("bgr", 2), ("bgra", 1), ("bgr", 1)):
        g.set_out_format(fmt_g)
        frames = _frames("bgr", W, H, range(t, t + n))
        go, gv, gm = g.composite(frames, want_yuyv=fmt_g == "bgr")
        to, tv, tm = t_.composite(frames)
        _same(gm, tm, "mask", (fmt_g, t))
        if fmt_g == "bgr":
            _same(go, to, "composite", (fmt_g, t))
            _same(gv, tv, "video", (fmt_g, t))
        else:
            for b in range(n):
                _same(go[b], expect_bgra(frames[b], tm[b]), "bgra", (t, b))
        t += n
    g.close()
    t_.close()


def test_format_toggles(emu_lib):
    """BGR -> BGRA -> BGR -> BGRA on one context: the BGR calls give the bytes of a context that never switched, the BGRA
    calls' video and mask too"""
    key, W, H, n = "meet_lite", 320, 240, 2
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
    t_ = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
    for c in (g, t_):
        c.set_background(bg)
        c.set_output(True, False, (240, 180))
    t = 0
    for fmt_g in ("bgr", "bgra", "bgr", "bgra"):
        g.set_out_format(fmt_g)
        frames = _frames("yuyv", W, H, range(t, t + n))
        go, gv, gm = g.composite_yuyv(frames)
        to, tv, tm = t_.composite_yuyv(frames)
        assert go.shape[-1] == (3 if fmt_g == "bgr" else 4)
        _same(gm, tm, "mask", (fmt_g, t))
        _same(gv, tv, "video", (fmt_g, t))
        if fmt_g == "bgr":
            _same(go, to, "composite", (fmt_g, t))
        else:
            for b in range(n):
                _same(go[b], expect_bgra(po.yuyv_to_bgr(frames[b]), tm[b], True, H_, (240, 180)), "bgra", (t, b))
        t += n
    g.close()
    t_.close()


class _SrcTwins:
    """five sources on the emulator, in a BGRA context and a BGR twin: 0 the context image (follows everything), 1 its own
    image (flip H, own size 240x180), 2 camera blur 9 (no image) with its filter off, 3 the context image at strength 5 (flip
    H|V, exactly half size), 4 camera blur 9 (flip V)"""

    def __init__(self, lib, key="meet_lite", W=320, H=240):
        self.W, self.H = W, H
        bg = synth.background()
        own = np.roll(bg, 90, axis=1)
        self.flip = {0: 0, 1: H_, 2: 0, 3: H_ | V_, 4: V_}
        self.size = {0: None, 1: (240, 180), 2: None, 3: (160, 120), 4: None}
        self.active = {0: True, 1: True, 2: False, 3: True, 4: True}
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=4)
        self.t = api.MaskGen(lib, model_path(key), W, H, max_batch=4)
        for c in (self.g, self.t):
            c.set_background(bg)
            c.set_sources(5)
            c.set_source_background(1, own)
            c.set_source_effect(2, "none", 9)
            c.set_source_effect(3, "default", 5)
            c.set_source_effect(4, "none", 9)
            for s in range(5):
                if self.flip[s]:
                    c.set_source_flip(s, *_code(self.flip[s]))
                if self.size[s]:
                    c.set_source_output(s, self.size[s])
            c.set_source_filter(2, False)
        self.g.set_out_format("bgra")

    def step(self, frames, ids, video=True, tag=()):
        go, gv, gm = self.g.composite_sources(frames, ids, want_yuyv=video)
        to, tv, tm = self.t.composite_sources(frames, ids)
        _same(gm, tm, "mask", tag)
        for b, s in enumerate(ids):
            if video:
                _same(gv[b], tv[b], "video", tag + (s,))
            _same(go[b], expect_bgra(frames[b], tm[b], self.active[s], self.flip[s], self.size[s]), "bgra", tag + (s,))

    def close(self):
        self.g.close()
        self.t.close()


def test_sources_bgra(emu_lib):
    """sources calls with own sizes, flips, a filtered-off source and every effect; with and without a video output, the
    latter with no Gaussian for the camera-blur sources"""
    S = _SrcTwins(emu_lib)
    t = 0
    for ids, video in (([0, 1, 2, 3], True), ([4, 3, 1, 0], False), ([2, 4], True), ([3, 4, 0], False)):
        frames = np.stack([synth.frame(S.W, S.H, t=t, stream=s) for s in ids])
        S.step(frames, ids, video, (tuple(ids), video))
        t += 1
    S.close()


def test_sources_camera_blur_bgra_only_has_no_gaussian(emu_lib):
    """a sources call whose camera-blur frames blend nothing launches exactly what the same call without those effects
    launches"""
    S = _SrcTwins(emu_lib)
    ids = [4, 3, 1, 0]
    frames = np.stack([synth.frame(S.W, S.H, t=0, stream=s) for s in ids])
    S.step(frames, ids, False, ("blur",))
    blur = S.g.launches_per_call
    S.g.set_source_effect(4, "default", -1)
    S.t.set_source_effect(4, "default", -1)
    S.step(frames, ids, False, ("ctx",))
    assert S.g.launches_per_call == blur
    S.close()


def test_refusals_leave_the_context_usable(emu_lib):
    """an unknown format, a host out_pitch of 3 bytes per pixel and an own-size frame that does not fit its out stride at 4
    bytes per pixel are refused before any launch; the context then runs as before"""
    L = emu_lib
    key, W, H = "meet_lite", 320, 240
    g = api.MaskGen(L, model_path(key), W, H, max_batch=2)
    g.set_background(synth.background())
    g.set_out_format("bgra")
    for bad in (-1, 2, 7):
        assert L.bsb_set_out_format(g._h, bad) == 0 and b"format" in L.bsb_last_error(), bad
    with pytest.raises(api.BackscrubError):
        g.set_out_format("rgba")
    assert g.out_channels == 4
    frames = _frames("bgr", W, H, range(2))
    out = np.empty((2, H, W, 4), np.uint8)
    l0 = L.bsb_total_launches()
    assert L.bsb_composite(g._h, 2, _addr(frames), W * 3, W * H * 3, _addr(out), W * 3, W * H * 4, None, 0, None, 0) == 0
    assert b"pitch" in L.bsb_last_error()
    assert L.bsb_total_launches() == l0
    g.set_sources(2)
    g.set_source_output(1, (240, 180))
    g.set_source_output(0, (160, 120))
    l0 = L.bsb_total_launches()
    # a 240x180 frame fits a stride of 240*180*3 bytes as BGR, not as BGRA
    out = np.empty(2 * 240 * 180 * 4, np.uint8)
    ids = (ctypes.c_int * 2)(0, 1)
    assert L.bsb_composite_sources(g._h, 2, ids, _addr(frames), W * 3, W * H * 3, _addr(out), 240 * 180 * 3, None, 0, None, 0) == 0
    assert b"stride" in L.bsb_last_error()
    assert L.bsb_total_launches() == l0
    # still usable, still BGRA: the masks are the oracle's (no call ran in between)
    o = po.MaskGen(model_path(key), W, H)
    go, _, gm = g.composite_sources(frames, [0, 1], want_yuyv=False)
    _, _, rm = o.composite_ex(frames[0], synth.background())
    _same(gm[0], rm, "mask", 0)
    for b, size in enumerate([(160, 120), (240, 180)]):
        _same(go[b], expect_bgra(frames[b], gm[b], True, 0, size), "bgra", b)
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
def tuning():
    """launcher switches for the contexts of one test, restored afterwards"""
    import backscrub_b200 as bs
    yield bs.set_tuning
    bs.set_tuning("post_tile", 0)
    bs.set_tuning("post_tma", 1)


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


class _GpuSrc:
    """a sources context in BGRA format and its BGR twin on the H100, fed from device YUYV / NV12 (tight or pitched) or
    host BGR frames; source s has flip flips[s % len], filter filters[s % len] and, where sizes is given, own size
    sizes[s % len].  The BGRA frames are checked against the definition from the call's camera frames and masks, the
    video and the masks against the twin."""

    def __init__(self, lib, key, W, H, n_sources, fmt, pitched=False, flips=(0,), filters=(True,), sizes=(None,), mb=8):
        import torch
        self.torch, self.lib, self.W, self.H, self.fmt, self.mb = torch, lib, W, H, fmt, mb
        self.flips = [flips[s % len(flips)] for s in range(n_sources)]
        self.filters = [filters[s % len(filters)] for s in range(n_sources)]
        self.sizes = [sizes[s % len(sizes)] for s in range(n_sources)]
        bg = synth.background()
        own = np.roll(bg, 77, axis=1)
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=mb)
        self.t = api.MaskGen(lib, model_path(key), W, H, max_batch=mb)
        for c in (self.g, self.t):
            c.set_background(bg)
            c.set_sources(n_sources)
            for s in range(n_sources):
                if s % 4 == 1:
                    c.set_source_background(s, own)
                if s % 4 == 2:
                    c.set_source_effect(s, "none", 25)
                if self.flips[s]:
                    c.set_source_flip(s, *_code(self.flips[s]))
                if not self.filters[s]:
                    c.set_source_filter(s, False)
                if self.sizes[s]:
                    c.set_source_output(s, self.sizes[s])
        self.g.set_out_format("bgra")
        dev = "cuda:0"
        if fmt == "nv12":
            self.pitch = W + 64 if pitched else W
            self.uv = self.pitch * H + (128 if pitched else 0)
            self.stride = self.uv + self.pitch * (H // 2) + (256 if pitched else 0)
        opx = max(w * h for w, h in ((sz or (W, H)) for sz in self.sizes))
        self.opx = opx
        self.d_out = torch.empty(mb * opx * 4, dtype=torch.uint8, device=dev)
        self.t_out = torch.empty(mb * opx * 3, dtype=torch.uint8, device=dev)
        vb = opx * 3 // 2 if fmt == "nv12" else opx * 2
        self.vb = vb
        self.d_vid = torch.empty(mb * vb, dtype=torch.uint8, device=dev)
        self.t_vid = torch.empty(mb * vb, dtype=torch.uint8, device=dev)
        self.d_mask = torch.empty((mb, H, W), dtype=torch.uint8, device=dev)
        self.t_mask = torch.empty((mb, H, W), dtype=torch.uint8, device=dev)

    def _run(self, c, ids, frames, out, vid, mask, oc):
        n = len(ids)
        if self.fmt == "bgr":
            o, v, m = c.composite_sources(frames, ids, want_yuyv=vid is not None)
            return o, v, m
        torch = self.torch
        if self.fmt == "yuyv":
            d_in = torch.from_numpy(np.ascontiguousarray(frames)).to("cuda:0")
            c.composite_sources_yuyv_device(n, ids, d_in.data_ptr(), out.data_ptr(), vid.data_ptr() if vid is not None else 0,
                                            mask.data_ptr(), sync=True, out_stride=self.opx * oc, yuyv_stride=self.vb)
        else:
            d_in = torch.from_numpy(_pitched(frames, self.pitch, self.uv, self.stride)).to("cuda:0")
            c.composite_sources_nv12_device(n, ids, d_in.data_ptr(), out.data_ptr(), vid.data_ptr() if vid is not None else 0,
                                            mask.data_ptr(), sync=True, pitch=self.pitch, uv_offset=self.uv, in_stride=self.stride,
                                            out_stride=self.opx * oc, nv12_stride=self.vb)
        ho = out.cpu().numpy()
        frames_out = []
        for b, s in enumerate(ids):
            w, h = self.sizes[s] or (self.W, self.H)
            frames_out.append(ho[b * self.opx * oc: b * self.opx * oc + w * h * oc])
        hv = vid.cpu().numpy() if vid is not None else None
        vids = [hv[b * self.vb: (b + 1) * self.vb] for b in range(n)] if hv is not None else None
        return frames_out, vids, mask[:n].cpu().numpy()

    def step(self, ids, t, video=True, tag=()):
        fmt = self.fmt
        if fmt == "bgr":
            frames = np.stack([synth.frame(self.W, self.H, t=t, stream=s) for s in ids])
        elif fmt == "yuyv":
            frames = np.stack([synth.yuyv_frame(self.W, self.H, t=t, stream=s) for s in ids])
        else:
            frames = np.stack([nv12_frame(self.W, self.H, t=t, stream=s) for s in ids])
        go, gv, gm = self._run(self.g, ids, frames, self.d_out, self.d_vid if video else None, self.d_mask, 4)
        to, tv, tm = self._run(self.t, ids, frames, self.t_out, self.t_vid, self.t_mask, 3)
        for b, s in enumerate(ids):
            tg = tag + (s,)
            _same(gm[b], tm[b], "mask", tg)
            if video:
                w, h = self.sizes[s] or (self.W, self.H)
                nb = w * h * 3 // 2 if fmt == "nv12" else w * h * 2
                _same(np.asarray(gv[b]).reshape(-1)[:nb], np.asarray(tv[b]).reshape(-1)[:nb], "video", tg)
            want = expect_bgra(camera_bgr(frames[b], fmt), tm[b], self.filters[s], self.flips[s], self.sizes[s])
            _same(go[b], want, "bgra", tg)
        return go

    def close(self):
        self.g.close()
        self.t.close()


GEOMETRIES = [(1280, 720, 0), (1296, 720, 64), (1296, 720, 128)]
FORMATS = ["yuyv", "nv12", "nv12_pitched", "bgr"]
FLIPS8 = [0, 0, H_, H_ | V_, V_, 0, H_, 0]
FILTERS8 = [True, False, True, False, True, True, False, True]
CALLS8 = ([0, 1, 2, 3, 4, 5, 6, 7], [7, 5, 3, 1], [6, 0, 4, 2, 1])


@pytest.mark.gpu
@pytest.mark.parametrize("geo", GEOMETRIES, ids=["1280x720", "1296x720_tw64", "1296x720_tw128"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_gpu_meet_720p_bgra(gpu_lib, tuning, geo, fmt):
    """Meet 720p sources at W x H, mirrored in place by k_post_tma, with filtered-off frames: BGRA with and without video"""
    W, H, tw = geo
    if tw:
        tuning("post_tile", tw)
    d = _GpuSrc(gpu_lib, "meet_full", W, H, 8, "nv12" if fmt.startswith("nv12") else fmt, pitched=fmt == "nv12_pitched",
                flips=FLIPS8, filters=FILTERS8)
    for i, ids in enumerate(CALLS8):
        d.step(ids, i, video=True, tag=(fmt, geo, "video", i))
        d.step(ids, 10 + i, video=False, tag=(fmt, geo, "bgra only", i))
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuyv", "nv12"])
def test_gpu_sources_own_sizes(gpu_lib, fmt):
    """sources with an own size (640x360) beside W x H frames, with flips and a filtered-off frame: k_tail flips and resizes
    the staged BGRA frames, and derives the video from the staged composites"""
    d = _GpuSrc(gpu_lib, "meet_full", 1280, 720, 4, fmt, flips=[0, H_, V_, H_ | V_], filters=[True, True, False, True],
                sizes=[None, (640, 360), (640, 360), None])
    for i, ids in enumerate(([0, 1, 2, 3], [3, 2], [1, 0])):
        d.step(ids, i, video=True, tag=(fmt, i))
        d.step(ids, 5 + i, video=False, tag=(fmt, "bgra only", i))
    d.close()


@pytest.mark.gpu
def test_gpu_4k(gpu_lib):
    """3840x2160 (128-wide tiles): plain YUYV device calls, BGRA with and without video, unflipped and mirrored"""
    import torch
    W, H, n = 3840, 2160, 2
    bg = synth.background()
    g = api.MaskGen(gpu_lib, model_path("meet_full"), W, H, max_batch=n)
    t_ = api.MaskGen(gpu_lib, model_path("meet_full"), W, H, max_batch=n)
    for c in (g, t_):
        c.set_background(bg)
    g.set_out_format("bgra")
    d_in = torch.empty((n, H, W, 2), dtype=torch.uint8, device="cuda:0")
    bufs = {c: (torch.empty((n, H, W, c.out_channels), dtype=torch.uint8, device="cuda:0"),
                torch.empty((n, H, W, 2), dtype=torch.uint8, device="cuda:0"),
                torch.empty((n, H, W), dtype=torch.uint8, device="cuda:0")) for c in (g, t_)}
    t = 0
    for flip, video in ((0, True), (0, False), (H_, True)):
        for c in (g, t_):
            c.set_output(*_code(flip))
        frames = _frames("yuyv", W, H, range(t, t + n))
        d_in.copy_(torch.from_numpy(frames))
        for c in (g, t_):
            o, v, m = bufs[c]
            c.composite_yuyv_device(n, d_in.data_ptr(), o.data_ptr(), v.data_ptr() if (video or c is t_) else 0, m.data_ptr(), sync=True)
        go, gv, gm = (x.cpu().numpy() for x in bufs[g])
        to, tv, tm = (x.cpu().numpy() for x in bufs[t_])
        _same(gm, tm, "mask", (flip, video))
        if video:
            _same(gv, tv, "video", (flip, video))
        for b in range(n):
            _same(go[b], expect_bgra(po.yuyv_to_bgr(frames[b]), tm[b], True, flip), "bgra", (flip, video, b))
        t += n
    g.close()
    t_.close()


@pytest.mark.gpu
def test_gpu_64_sources(gpu_lib):
    """64 sources in one call at a ragged width (1296: the last tile column is partial), mirrored in place"""
    d = _GpuSrc(gpu_lib, "meet_lite", 1296, 720, 64, "yuyv", flips=[0, H_, H_ | V_, V_], filters=[True, True, True, False], mb=64)
    d.step(list(range(64)), 0, video=False, tag=("bgra only",))
    d.step(list(range(63, -1, -1)), 1, video=True, tag=("video",))
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuyv", "bgr"])
def test_gpu_fallback_kernels_match_tma(gpu_lib, tuning, fmt):
    """post_tma = 0 (k_post_fast, and k_tail for the mirrored frames) gives k_post_tma's bytes"""
    outs = []
    for tma in (1, 0):
        tuning("post_tma", tma)
        d = _GpuSrc(gpu_lib, "meet_full", 1280, 720, 8, fmt, flips=FLIPS8, filters=FILTERS8)
        outs.append([np.concatenate([np.asarray(x).reshape(-1) for x in d.step(ids, i, video=bool(i % 2), tag=(fmt, tma, i))])
                     for i, ids in enumerate(CALLS8)])
        d.close()
    for a, b in zip(*outs):
        _same(a, b, "fallback bgra", fmt)


@pytest.mark.gpu
def test_gpu_toggle_replays(gpu_lib):
    """once both formats of a call have been captured, toggling replays: no launch is enqueued outside the graphs, and
    each format reports its own launch count"""
    import torch
    W, H, n = 1280, 720, 2
    g = api.MaskGen(gpu_lib, model_path("meet_full"), W, H, max_batch=n)
    g.set_bgblur(9)                     # camera blur: the BGRA-only call has no Gaussian
    d_in = torch.empty((n, H, W, 2), dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty((n, H, W, 4), dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((n, H, W), dtype=torch.uint8, device="cuda:0")
    counts = {}
    t = 0
    for fmt, replays in (("bgr", False), ("bgra", False), ("bgr", True), ("bgra", True), ("bgr", True)):
        g.set_out_format(fmt)
        frames = _frames("yuyv", W, H, range(t, t + n))
        d_in.copy_(torch.from_numpy(frames))
        l0 = gpu_lib.bsb_total_launches()
        g.composite_yuyv_device(n, d_in.data_ptr(), d_out.data_ptr(), 0, d_mask.data_ptr(), sync=True)
        assert (gpu_lib.bsb_total_launches() == l0) == replays, (fmt, replays)
        counts.setdefault(fmt, g.launches_per_call)
        assert g.launches_per_call == counts[fmt], fmt
        if fmt == "bgra":
            mask = d_mask.cpu().numpy()
            out = d_out.cpu().numpy()
            for b in range(n):
                _same(out[b], expect_bgra(po.yuyv_to_bgr(frames[b]), mask[b]), "bgra", (t, b))
        t += n
    # the BGR call blurs the camera frame, and converts it to BGR for the Gaussian; the BGRA call reads the YUYV in place
    assert counts["bgr"] - counts["bgra"] == _gauss_launches(gpu_lib, 9) + 1
    g.close()
