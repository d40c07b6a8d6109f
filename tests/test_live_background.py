"""Live backgrounds (bsb_set_live_background / bsb_set_source_live_background): each frame of a call blends a device image
the caller hands over (BGR or NV12, any size), resized and blurred inside the call.  Frame b with live background L must
give exactly the bytes of a plain batch-1 context set up the same way plus bsb_set_background(L) (an NV12 L converted
with the NV12 ingest first), fed the same stream.

`-m "not gpu"`: the kernel-logic emulator build (emulated device pointers are host buffers) on fed masks, against the
oracle.  `-m gpu`: the sm_90a library against plain batch-1 contexts."""

import numpy as np
import pytest

from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_feed_post import geo, random_masks, ref_mask, ref_outputs
from tests.test_nv12 import ref_nv12_to_bgr


def live_bgr(w, h, seed):
    """a decoded BGR frame of a live source: the bundled background resized, rolled and tinted per seed"""
    import cv2
    bg = cv2.resize(synth.background(), (w, h), interpolation=cv2.INTER_LINEAR)
    return np.ascontiguousarray(np.roll(bg, 37 * seed, axis=1) ^ np.uint8((29 * seed) & 0xFF))


def live_nv12(w, h, seed):
    """a decoded NV12 surface [h*3/2, w]: the Y plane and the even rows' UV pairs of a YUYV frame"""
    yv = synth.yuyv_frame(w, h, t=seed, stream=7)
    return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)


def padded_bgr(img, pitch):
    """one BGR image in a buffer of `pitch`-byte rows (padding 0xa5)"""
    h, w, _ = img.shape
    buf = np.full((h, pitch), 0xA5, np.uint8)
    buf[:, :w * 3] = img.reshape(h, w * 3)
    return buf


def padded_nv12(img, pitch, uv_offset):
    """one NV12 surface with a row pitch and a UV plane offset (padding 0x5a)"""
    h3, w = img.shape
    h = h3 * 2 // 3
    buf = np.full(uv_offset + pitch * (h // 2), 0x5A, np.uint8)
    for y in range(h):
        buf[y * pitch: y * pitch + w] = img[y]
    for r in range(h // 2):
        buf[uv_offset + r * pitch: uv_offset + r * pitch + w] = img[h + r]
    return buf


def as_bgr(fmt, img):
    """what bsb_set_background would be given for live image img"""
    return ref_nv12_to_bgr(img) if fmt == "nv12" else img


def expected_bg(fmt, img, W, H, k):
    bg = po.resize_linear_u8(as_bgr(fmt, img), W, H)
    return po.gaussian_blur(bg, k) if k else bg


class Live:
    """a live image held in a buffer of its own layout (pitch, UV offset); its address is the emulated device pointer"""

    def __init__(self, fmt, img, pitch=None, uv_offset=None):
        self.fmt, self.img = fmt, img
        if fmt == "nv12":
            h, w = img.shape[0] * 2 // 3, img.shape[1]
            self.pitch = w if pitch is None else pitch
            self.uv = self.pitch * h if uv_offset is None else uv_offset
            self.buf = padded_nv12(img, self.pitch, self.uv)
        else:
            h, w = img.shape[:2]
            self.pitch = w * 3 if pitch is None else pitch
            self.uv = 0
            self.buf = padded_bgr(img, self.pitch)
        self.size = (w, h)

    @property
    def ptr(self):
        return self.buf.ctypes.data

    def set_plain(self, g, stride=0):
        g.set_live_background(self.ptr, self.fmt, self.size, self.pitch, self.uv, stride)

    def set_source(self, g, s):
        g.set_source_live_background(s, self.ptr, self.fmt, self.size, self.pitch, self.uv)


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


KEY, W, H = "meet_lite", 320, 240

# (fmt, image, pitch, uv_offset): up, down, exact 2x down (INTER_AREA), same size, odd sizes, padded pitches, NV12
LIVE_CASES = {
    "up_bgr": ("bgr", lambda: live_bgr(401, 263, 1), None, None),
    "down_bgr": ("bgr", lambda: live_bgr(517, 389, 2), None, None),
    "area2x_bgr": ("bgr", lambda: live_bgr(2 * W, 2 * H, 3), None, None),
    "same_bgr": ("bgr", lambda: live_bgr(W, H, 4), None, None),
    "odd_pitched_bgr": ("bgr", lambda: live_bgr(161, 121, 5), 161 * 3 + 13, None),
    "nv12_pitched": ("nv12", lambda: live_nv12(480, 270, 6), 512, 512 * 270 + 64),
    "nv12_area2x": ("nv12", lambda: live_nv12(2 * W, 2 * H, 7), 2 * W + 32, None),
    "nv12_up": ("nv12", lambda: live_nv12(200, 150, 8), None, None),
}


@pytest.mark.parametrize("case", sorted(LIVE_CASES))
@pytest.mark.parametrize("k", [0, 7])
def test_emu_plain_live(emu_lib, case, k):
    """a plain call, one live image for every frame (frame_stride 0): the composite and YUYV equal the oracle's blend over
    the resized (and blurred) image, on fed masks; k > 0 on a context without a background is camera-blur mode, where the
    live image is blurred instead of the camera frame"""
    fmt, make, pitch, uv = LIVE_CASES[case]
    g = geo(KEY, W, H)
    c = api.MaskGen(emu_lib, model_path(KEY), W, H, max_batch=3)
    if k:
        c.set_bgblur(k)
    lv = Live(fmt, make(), pitch, uv)
    lv.set_plain(c)
    bg = expected_bg(fmt, lv.img, W, H, k)
    masks = random_masks(g, 3, 11)[:3]
    masks[0][:] = 255                                   # all background: the composite is the resized image itself
    frames = np.stack([synth.frame(W, H, t=t) for t in range(3)])
    c.feed(B.FEED_MASK, masks)
    out, vid, mask = c.composite(frames)
    for b in range(3):
        rm = ref_mask(g, masks[b])
        ro, rv = ref_outputs(rm, frames[b], bg)
        assert np.array_equal(mask[b], rm), (case, b)
        assert np.array_equal(out[b], ro), (case, b, int((out[b] != ro).sum()))
        assert np.array_equal(vid[b], rv), (case, b)
    c.close()


def test_emu_plain_per_frame_and_ring(emu_lib):
    """frame b blends live frame b (a frame stride of one padded frame), over a context ring that keeps moving while hidden;
    then frame_stride 0; then cleared, the ring resumes at the advanced cursor; YUYV and NV12 host calls"""
    g = geo(KEY, W, H)
    c = api.MaskGen(emu_lib, model_path(KEY), W, H, max_batch=4)
    raw = synth.background()
    ring = np.stack([np.roll(raw, 97 * i, axis=1) for i in range(3)])
    c.set_background_ring(ring, advance=1)
    ring_bg = [po.resize_linear_u8(r, W, H) for r in ring]
    lw, lh, pitch = 250, 170, 250 * 3 + 6
    imgs = [live_bgr(lw, lh, 20 + i) for i in range(4)]
    stride = pitch * lh + 10
    buf = np.full(4 * stride, 0x33, np.uint8)
    for i, im in enumerate(imgs):
        buf[i * stride: i * stride + pitch * lh] = padded_bgr(im, pitch).reshape(-1)
    bgs = [po.resize_linear_u8(im, W, H) for im in imgs]
    yuyv = [synth.yuyv_frame(W, H, t=t) for t in range(4)]
    nv12 = [np.concatenate([y[..., 0], y[0::2, :, 1]], axis=0) for y in yuyv]
    cam = {"yuyv": [po.yuyv_to_bgr(y) for y in yuyv], "nv12": [ref_nv12_to_bgr(f) for f in nv12]}

    def call(n, expect, fmt="yuyv"):
        masks = random_masks(g, n, 30 + n)[:n]
        c.feed(B.FEED_MASK, masks)
        if fmt == "yuyv":
            out = np.empty((n, H, W, 3), np.uint8)
            vid = np.empty((n, H, W, 2), np.uint8)
            mask = np.empty((n, H, W), np.uint8)
            c.composite_yuyv_into(np.stack(yuyv[:n]), out, vid, mask)
        else:
            out, vid, mask = c.composite_nv12(np.stack(nv12[:n]))
        for b in range(n):
            rm = ref_mask(g, masks[b])
            ro, rv = ref_outputs(rm, cam[fmt][b], expect(b), nv12=fmt == "nv12")
            assert np.array_equal(out[b], ro), (fmt, n, b)
            assert np.array_equal(vid[b].reshape(-1), rv.reshape(-1)), (fmt, n, b)

    c.set_live_background(buf.ctypes.data, "bgr", (lw, lh), pitch, None, stride)
    call(4, lambda b: bgs[b])
    call(2, lambda b: bgs[b], "nv12")
    c.set_live_background(buf.ctypes.data + stride, "bgr", (lw, lh), pitch, None, 0)
    call(3, lambda b: bgs[1])
    c.set_live_background(None)
    cursor = (4 + 2 + 3) % 3                            # the ring moved on under the live frames
    call(2, lambda b: ring_bg[(cursor + b) % 3])
    c.close()


class _SrcModel:
    """what each source of a sources context blends: its live image, own still or ring (with cursor), the context image,
    or (BG_NONE) its camera frame blurred; and the strength"""

    def __init__(self, n, ctx_bg, ctx_k):
        self.ctx_bg, self.ctx_k = ctx_bg, ctx_k
        self.live, self.ring, self.fx = {}, {}, {s: ("default", -1) for s in range(n)}

    def bg(self, s, frame):
        kind, k = self.fx[s]
        k = self.ctx_k if k < 0 else k
        if kind == "none":
            return po.gaussian_blur(frame, k) if k else _green()
        if s in self.live:
            lv = self.live[s]
            return expected_bg(lv.fmt, lv.img, W, H, k)
        if s in self.ring:
            imgs, _, cur = self.ring[s]
            img = po.resize_linear_u8(imgs[cur], W, H)
        else:
            img = po.resize_linear_u8(self.ctx_bg, W, H)
        return po.gaussian_blur(img, k) if k else img

    def moved(self, ids):
        for s in ids:
            if s in self.ring:
                r = self.ring[s]
                r[2] = (r[2] + r[1]) % len(r[0])


def _green():
    g = np.zeros((H, W, 3), np.uint8)
    g[..., 1] = 255
    return g


def _src_call(c, m, ids, t, filt=None):
    g = geo(KEY, W, H)
    n = len(ids)
    masks = random_masks(g, n, 50 + t)[:n]
    frames = np.stack([synth.frame(W, H, t=t + b, stream=s) for b, s in enumerate(ids)])
    c.feed(B.FEED_MASK, masks)
    out, vid, mask = c.composite_sources(frames, ids)
    for b, s in enumerate(ids):
        rm = ref_mask(g, masks[b])
        bg = frames[b] if filt and filt.get(s) == 0 else m.bg(s, frames[b])
        ro, rv = ref_outputs(rm, frames[b], bg)
        assert np.array_equal(mask[b], rm), (ids, b, s)
        assert np.array_equal(out[b], ro), (ids, b, s, int((out[b] != ro).sum()))
        assert np.array_equal(vid[b], rv), (ids, b, s)
    m.moved(ids)


def test_emu_sources_mixed(emu_lib):
    """one call mixing live BGR and NV12 frames (context strength, own strength 0 and 35), an own still, a ring at advance 1,
    the context image, BG_NONE with a live image set (ignored: its camera frame blurred) and a filter-off frame with a live
    image; the ring's cursor keeps moving while a live image hides it"""
    c = api.MaskGen(emu_lib, model_path(KEY), W, H, max_batch=8)
    ctx = synth.background()[::-1].copy()
    c.set_background(ctx)
    c.set_bgblur(7)
    c.set_sources(8)
    m = _SrcModel(8, ctx, 7)
    lives = {0: Live("bgr", live_bgr(640, 360, 40)), 1: Live("nv12", live_nv12(400, 226, 41), 416, 416 * 226 + 32),
             2: Live("bgr", live_bgr(2 * W, 2 * H, 42)), 6: Live("bgr", live_bgr(300, 200, 43)),
             7: Live("nv12", live_nv12(W, H, 44))}
    for s in (0, 1, 2, 6, 7):
        lives[s].set_source(c, s)
        m.live[s] = lives[s]
    c.set_source_effect(1, "default", 0)
    m.fx[1] = ("default", 0)
    c.set_source_effect(2, "default", 35)
    m.fx[2] = ("default", 35)
    c.set_source_background(3, live_bgr(200, 150, 45))
    m.ring[3] = [[live_bgr(200, 150, 45)], 0, 0]
    ring = [live_bgr(180, 120, 46 + i) for i in range(3)]
    c.set_source_background_ring(4, np.stack(ring), 1)
    m.ring[4] = [ring, 1, 0]
    c.set_source_effect(6, "none", 9)                   # its live image is ignored: its camera frame at 9
    m.fx[6] = ("none", 9)
    c.set_source_filter(7, 0)
    _src_call(c, m, [0, 1, 2, 3, 4, 5, 6, 7], 0, {7: 0})
    # s4's ring hidden by a live image for one call, then shown again at the advanced cursor
    hide = Live("bgr", live_bgr(333, 222, 47))
    hide.set_source(c, 4)
    m.live[4] = hide
    _src_call(c, m, [4, 0, 5], 10)
    _src_call(c, m, [2, 5], 20)
    c.set_source_live_background(4, None)
    del m.live[4]
    assert m.ring[4][2] == 2                            # moved while hidden
    _src_call(c, m, [4, 1, 6], 30)
    # a new pointer of an already seen size, every call
    for t in range(2):
        lv = Live("bgr", live_bgr(640, 360, 60 + t))
        lv.set_source(c, 0)
        m.live[0] = lv
        _src_call(c, m, [0, 3], 40 + t)
    c.reset_source(0)                                   # the smoother only: the live image stays
    _src_call(c, m, [0], 50)
    c.set_sources(8)                                    # clears every live image
    m = _SrcModel(8, ctx, 7)
    _src_call(c, m, [0, 1, 2], 60)
    c.close()


def test_emu_frames_that_blend_nothing(emu_lib):
    """filter-off frames and BGRA calls without a video output read no live image: such a call launches exactly what it
    launches without one (no k_live_bg), and its outputs are unchanged"""
    L = emu_lib
    c = api.MaskGen(emu_lib, model_path(KEY), W, H, max_batch=2)
    c.set_sources(2)
    lv = Live("bgr", live_bgr(400, 300, 70))
    frames = np.stack([synth.frame(W, H, t=t) for t in range(2)])

    def launches(fn):
        l0 = L.bsb_total_launches()
        fn()
        return L.bsb_total_launches() - l0

    def plain():
        return c.composite(frames)

    def sources():
        return c.composite_sources(frames, [0, 1])

    def bgra_mask_only():
        return c.composite(frames, want_yuyv=False)

    for filt in ("plain", "sources"):
        base = launches(plain if filt == "plain" else sources)
        lv.set_plain(c)
        lv.set_source(c, 0)
        lv.set_source(c, 1)
        assert launches(plain if filt == "plain" else sources) == base + 1       # k_live_bg
        if filt == "plain":
            c.set_filter(False)
        else:
            c.set_source_filter(0, 0)
            c.set_source_filter(1, 0)
        off = launches(plain if filt == "plain" else sources)
        c.set_live_background(None)
        c.set_source_live_background(0, None)
        c.set_source_live_background(1, None)
        assert launches(plain if filt == "plain" else sources) == off
        c.set_filter(True)
        c.set_source_filter(0, -1)
        c.set_source_filter(1, -1)
    c.set_out_format("bgra")
    base = launches(bgra_mask_only)
    lv.set_plain(c)
    assert launches(bgra_mask_only) == base
    c.close()


def test_emu_errors(emu_lib):
    """every refused call returns 0 with a message and leaves the live images as they were"""
    L = emu_lib
    g = geo(KEY, W, H)
    c = api.MaskGen(emu_lib, model_path(KEY), W, H, max_batch=2)
    lv = Live("bgr", live_bgr(300, 200, 80))
    nv = Live("nv12", live_nv12(300, 200, 81))
    h = c._h
    assert L.bsb_set_source_live_background(h, 0, lv.ptr, 0, 300, 200, 900, 0) == 0 and b"set_sources" in L.bsb_last_error()
    c.set_sources(2)
    lv.set_plain(c)
    lv.set_source(c, 0)
    bad = [
        (lambda: L.bsb_set_live_background(h, lv.ptr, 2, 300, 200, 900, 0, 0), b"format"),
        (lambda: L.bsb_set_live_background(h, lv.ptr, -1, 300, 200, 900, 0, 0), b"format"),
        (lambda: L.bsb_set_live_background(h, lv.ptr, 0, 0, 200, 900, 0, 0), b"size"),
        (lambda: L.bsb_set_live_background(h, lv.ptr, 0, 300, 16385, 900, 0, 0), b"size"),
        (lambda: L.bsb_set_live_background(h, lv.ptr, 0, 300, 200, 899, 0, 0), b"pitch"),
        (lambda: L.bsb_set_live_background(h, nv.ptr, 1, 301, 200, 302, 302 * 200, 0), b"even"),
        (lambda: L.bsb_set_live_background(h, nv.ptr, 1, 300, 201, 300, 300 * 201, 0), b"even"),
        (lambda: L.bsb_set_live_background(h, nv.ptr, 1, 300, 200, 299, 300 * 200, 0), b"pitch"),
        (lambda: L.bsb_set_live_background(h, nv.ptr, 1, 300, 200, 300, 300 * 200 - 1, 0), b"UV"),
        (lambda: L.bsb_set_live_background(h, lv.ptr, 0, 300, 200, 900, 0, 900 * 200 - 1), b"stride"),
        (lambda: L.bsb_set_live_background(h, nv.ptr, 1, 300, 200, 300, 300 * 200, 300 * 300 - 1), b"stride"),
        (lambda: L.bsb_set_source_live_background(h, 2, lv.ptr, 0, 300, 200, 900, 0), b"out of range"),
        (lambda: L.bsb_set_source_live_background(h, -1, lv.ptr, 0, 300, 200, 900, 0), b"out of range"),
        (lambda: L.bsb_set_source_live_background(h, 0, lv.ptr, 3, 300, 200, 900, 0), b"format"),
        (lambda: L.bsb_set_source_live_background(h, 0, nv.ptr, 1, 300, 200, 300, 10), b"UV"),
    ]
    bg = expected_bg("bgr", lv.img, W, H, 0)
    frames = np.stack([synth.frame(W, H, t=t) for t in range(2)])
    for i, (call, msg) in enumerate(bad):
        assert call() == 0, i
        assert msg in L.bsb_last_error(), (i, L.bsb_last_error())
    # a stride of exactly one frame is accepted
    assert L.bsb_set_live_background(h, lv.ptr, 0, 300, 200, 900, 0, 900 * 199 + 900) == 1
    assert L.bsb_set_live_background(h, lv.ptr, 0, 300, 200, 900, 0, 0) == 1
    with pytest.raises(api.BackscrubError, match="format"):
        c.set_live_background(lv.ptr, "yuyv", (300, 200))
    masks = random_masks(g, 2, 90)[:2]
    c.feed(B.FEED_MASK, masks)
    out, _, _ = c.composite(frames)
    c.feed(B.FEED_MASK, masks)
    sout, _, _ = c.composite_sources(frames, [0, 1])
    ctx_bg = _green()
    for b in range(2):
        rm = ref_mask(g, masks[b])
        assert np.array_equal(out[b], ref_outputs(rm, frames[b], bg)[0]), b
        assert np.array_equal(sout[b], ref_outputs(rm, frames[b], bg if b == 0 else ctx_bg)[0]), b
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


def _cam(fmt, W_, H_, t, s):
    if fmt == "nv12":
        yv = synth.yuyv_frame(W_, H_, t=t, stream=s)
        return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)
    if fmt == "yuyv":
        return synth.yuyv_frame(W_, H_, t=t, stream=s)
    return synth.frame(W_, H_, t=t, stream=s)


class _GpuSources:
    """a sources context fed device camera frames with device live images per source, and per source a plain batch-1
    context with bsb_set_background(L) and the source's strength, flip, size, filter and output format"""

    def __init__(self, lib, key, W_, H_, n, fmt, ctx_k=0, bgra=False):
        import torch
        self.torch, self.lib, self.key, self.W, self.H, self.fmt, self.bgra = torch, lib, key, W_, H_, fmt, bgra
        self.g = api.MaskGen(lib, model_path(key), W_, H_, max_batch=n)
        self.g.set_bgblur(ctx_k)
        if bgra:
            self.g.set_out_format("bgra")
        self.g.set_sources(n)
        self.ctx_k, self.n = ctx_k, n
        self.k, self.flip, self.size, self.filt, self.live = {}, {}, {}, {}, {}
        self.refs, self.t = {}, [0] * n

    def set_live(self, s, fmt, img):
        """the source's live image, uploaded to a fresh device buffer (a new pointer every time)"""
        torch = self.torch
        d = torch.from_numpy(img.reshape(-1).copy()).to("cuda:0")
        size = (img.shape[1], img.shape[0] * 2 // 3) if fmt == "nv12" else (img.shape[1], img.shape[0])
        self.g.set_source_live_background(s, d, fmt, size)
        self.live[s] = (fmt, img, d)

    def set_fx(self, s, k):
        self.g.set_source_effect(s, "default", k)
        self.k[s] = k

    def out_size(self, s):
        return self.size.get(s, (self.W, self.H))

    def ref(self, s):
        """the plain context of source s with its live image as a still background"""
        fmt, img, _ = self.live[s]
        want = (id(img), self.k.get(s, self.ctx_k), self.flip.get(s, 0), self.out_size(s), self.filt.get(s, 1))
        if s not in self.refs:
            c = api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1)
            if self.bgra:
                c.set_out_format("bgra")
            self.refs[s] = [c, None]
        r = self.refs[s]
        if r[1] != want:
            c = r[0]
            c.set_background(as_bgr(fmt, img))
            c.set_bgblur(want[1])
            c.set_output(bool(want[2] & 1), bool(want[2] & 2), want[3])
            c.set_filter(bool(want[4]))
            r[1] = want
        return r[0]

    def _buffers(self, n, opx):
        torch, dev = self.torch, "cuda:0"
        oc = 4 if self.bgra else 3
        vb = opx * 3 // 2 if self.fmt == "nv12" else opx * 2
        return (torch.empty(n * opx * oc, dtype=torch.uint8, device=dev), torch.empty(n * vb, dtype=torch.uint8, device=dev),
                torch.empty(n * self.W * self.H, dtype=torch.uint8, device=dev), oc, vb)

    def _run(self, c, ids, cams, opx):
        torch = self.torch
        n = len(cams)
        d_in = torch.from_numpy(np.stack(cams).reshape(-1).copy()).to("cuda:0")
        out, vid, mask, oc, vb = self._buffers(n, opx)
        args = (n, d_in.data_ptr(), out.data_ptr(), vid.data_ptr(), mask.data_ptr())
        if ids is None:
            if self.fmt == "nv12":
                c.composite_nv12_device(*args, sync=True)
            else:
                c.composite_yuyv_device(*args, sync=True)
        elif self.fmt == "nv12":
            c.composite_sources_nv12_device(n, ids, *args[1:], sync=True, out_stride=opx * oc, nv12_stride=vb)
        else:
            c.composite_sources_yuyv_device(n, ids, *args[1:], sync=True, out_stride=opx * oc, yuyv_stride=vb)
        return out.cpu().numpy(), vid.cpu().numpy(), mask.cpu().numpy(), oc, vb

    def step(self, ids, check=None):
        check = range(len(ids)) if check is None else check
        cams = [_cam(self.fmt, self.W, self.H, self.t[s], s) for s in ids]
        opx = max(w * h for w, h in (self.out_size(s) for s in range(self.n)))
        out, vid, mask, oc, vb = self._run(self.g, ids, cams, opx)
        npx = self.W * self.H
        for b in check:
            s = ids[b]
            w, h = self.out_size(s)
            ro, rv, rm, _, _ = self._run(self.ref(s), None, [cams[b]], w * h)
            vn = w * h * 3 // 2 if self.fmt == "nv12" else w * h * 2
            tag = (ids, b, s, self.t[s])
            assert np.array_equal(mask[b * npx:(b + 1) * npx], rm), ("mask", tag)
            assert np.array_equal(out[b * opx * oc: b * opx * oc + w * h * oc], ro), ("out", tag)
            assert np.array_equal(vid[b * vb: b * vb + vn], rv), ("video", tag)
        for b, s in enumerate(ids):
            if b not in check and s in self.refs:
                # the reference's smoother must see every frame of the stream
                w, h = self.out_size(s)
                self._run(self.ref(s), None, [cams[b]], w * h)
            self.t[s] += 1

    def close(self):
        self.g.close()
        for r in self.refs.values():
            r[0].close()


LIVE_SIZES = [("nv12", 1920, 1080), ("bgr", 640, 360), ("bgr", 2560, 1440)]


@pytest.mark.gpu
@pytest.mark.parametrize("key,W_,H_,fmt", [("meet_full", 1280, 720, "yuyv"), ("meet_full", 1280, 720, "nv12"),
                                           ("mlkit", 1280, 720, "nv12"), ("mlkit", 642, 482, "yuyv")])
@pytest.mark.parametrize("k", [0, 25, 35])
def test_gpu_sources_live_vs_plain(gpu_lib, key, W_, H_, fmt, k):
    """six sources with live images of three sizes (1920x1080 NV12, 640x360 BGR, 2560x1440 BGR: the exact 2x) at the
    context strength k, one at its own strength, one mirrored, one at its own output size, one filtered off; each frame
    against its plain context; new live pointers between calls"""
    d = _GpuSources(gpu_lib, key, W_, H_, 6, fmt, ctx_k=k)
    for s in range(6):
        lf, lw, lh = LIVE_SIZES[s % 3]
        d.set_live(s, lf, live_nv12(lw, lh, s) if lf == "nv12" else live_bgr(lw, lh, s))
    d.set_fx(1, 7 if k != 7 else 9)
    d.g.set_source_flip(2, True, False)
    d.flip[2] = 1
    own = ((W_ // 2 + 2) // 2 * 2, (H_ // 2 + 2) // 2 * 2)
    d.g.set_source_output(3, own)
    d.size[3] = own
    d.g.set_source_filter(4, 0)
    d.filt[4] = 0
    d.step([0, 1, 2, 3, 4, 5])
    d.step([5, 3, 1])
    for s in (0, 2):
        lf, lw, lh = LIVE_SIZES[s % 3]
        d.set_live(s, lf, live_nv12(lw, lh, 10 + s) if lf == "nv12" else live_bgr(lw, lh, 10 + s))
    d.step([2, 0, 4, 1])
    d.close()


@pytest.mark.gpu
def test_gpu_bgra_live(gpu_lib):
    """BGRA output format with a video output: the BGRA frames, video and masks equal the plain contexts'"""
    d = _GpuSources(gpu_lib, "meet_full", 1280, 720, 3, "nv12", ctx_k=25, bgra=True)
    for s in range(3):
        lf, lw, lh = LIVE_SIZES[s]
        d.set_live(s, lf, live_nv12(lw, lh, 20 + s) if lf == "nv12" else live_bgr(lw, lh, 20 + s))
    d.g.set_source_flip(1, False, True)
    d.flip[1] = 2
    d.step([0, 1, 2])
    d.step([2, 0])
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 25, 35])
def test_gpu_plain_live(gpu_lib, k):
    """a plain context, 4 frames per call, frame b its own 1920x1080 NV12 surface (frame stride one surface), then one image
    for every frame (stride 0), against a plain batch-1 context with bsb_set_background of each converted surface"""
    import torch
    W_, H_, n = 1280, 720, 4
    c = api.MaskGen(gpu_lib, model_path("meet_full"), W_, H_, max_batch=n)
    c.set_bgblur(k)
    r = api.MaskGen(gpu_lib, model_path("meet_full"), W_, H_, max_batch=1)
    r.set_bgblur(k)
    lw, lh = 1920, 1080
    surf = [live_nv12(lw, lh, 30 + i) for i in range(n)]
    d_surf = torch.from_numpy(np.stack(surf).reshape(-1).copy()).to("cuda:0")
    fb = lw * lh * 3 // 2
    t = 0
    for stride in (fb, 0):
        c.set_live_background(d_surf, "nv12", (lw, lh), frame_stride=stride)
        yv = [synth.yuyv_frame(W_, H_, t=t + b) for b in range(n)]
        d_in = torch.from_numpy(np.stack(yv).reshape(-1).copy()).to("cuda:0")
        out = torch.empty(n * W_ * H_ * 3, dtype=torch.uint8, device="cuda:0")
        vid = torch.empty(n * W_ * H_ * 2, dtype=torch.uint8, device="cuda:0")
        mask = torch.empty(n * W_ * H_, dtype=torch.uint8, device="cuda:0")
        c.composite_yuyv_device(n, d_in.data_ptr(), out.data_ptr(), vid.data_ptr(), mask.data_ptr(), sync=True)
        out, vid, mask = out.cpu().numpy(), vid.cpu().numpy(), mask.cpu().numpy()
        for b in range(n):
            r.set_background(ref_nv12_to_bgr(surf[b if stride else 0]))
            ro, rv, rm = r.composite_yuyv(yv[b][None])
            npx = W_ * H_
            assert np.array_equal(mask[b * npx:(b + 1) * npx], rm.reshape(-1)), (stride, b)
            assert np.array_equal(out[b * npx * 3:(b + 1) * npx * 3], ro.reshape(-1)), (stride, b)
            assert np.array_equal(vid[b * npx * 2:(b + 1) * npx * 2], rv.reshape(-1)), (stride, b)
        t += n
    c.close()
    r.close()


@pytest.mark.gpu
def test_gpu_replay_and_launches(gpu_lib):
    """after the first live call, calls with new pointers and sizes already seen replay the captured graph (no launch outside
    it); a call without live frames keeps the launches per call it had before any live image was set"""
    import torch
    W_, H_, n = 1280, 720, 8
    g = api.MaskGen(gpu_lib, model_path("meet_full"), W_, H_, max_batch=n)
    g.set_background(synth.background())
    g.set_bgblur(25)
    g.set_sources(n)
    ids = list(range(n))
    d_in = torch.from_numpy(np.stack([_cam("nv12", W_, H_, 0, s) for s in ids]).reshape(-1).copy()).to("cuda:0")
    out = torch.empty(n * W_ * H_ * 3, dtype=torch.uint8, device="cuda:0")
    vid = torch.empty(n * W_ * H_ * 3 // 2, dtype=torch.uint8, device="cuda:0")
    mask = torch.empty(n * W_ * H_, dtype=torch.uint8, device="cuda:0")

    def call():
        g.composite_sources_nv12_device(n, ids, d_in.data_ptr(), out.data_ptr(), vid.data_ptr(), mask.data_ptr(), sync=True)

    call()
    call()
    base = g.launches_per_call
    sizes = [(1920, 1080), (640, 360), (2560, 1440)]
    bufs = [torch.empty(w * h * 3 // 2, dtype=torch.uint8, device="cuda:0") for _ in range(2) for w, h in sizes]
    for s in ids:
        g.set_source_live_background(s, bufs[s % 3], "nv12", sizes[s % 3])
    call()
    assert g.launches_per_call == base + 2                # k_live_bg and the fused Gaussian of the live frames
    for i in range(4):
        for s in ids:
            j = (s + i) % 3
            g.set_source_live_background(s, bufs[3 + j] if i % 2 else bufs[j], "nv12", sizes[j])
        l0 = gpu_lib.bsb_total_launches()
        call()
        assert gpu_lib.bsb_total_launches() == l0, i
    for s in ids:
        g.set_source_live_background(s, None)
    call()
    assert g.launches_per_call == base
    g.close()


@pytest.mark.gpu
def test_gpu_64_sources_live(gpu_lib):
    """64 sources, Meet 1280x720 NV12, each with its own 1920x1080 NV12 surface that changes every call; a sample of frames
    checked against plain contexts"""
    d = _GpuSources(gpu_lib, "meet_full", 1280, 720, 64, "nv12", ctx_k=25)
    ids = list(range(64))
    for call in range(3):
        for s in ids:
            d.set_live(s, "nv12", live_nv12(1920, 1080, 100 * call + s) if s in (0, 17, 63) else live_nv12(1920, 1080, call))
        d.step(ids, check=[0, 17, 63] if call != 1 else [17])
    d.close()
