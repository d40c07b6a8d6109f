"""Framing (bsb_set_framing): each frame's output is cv::resize(cv::flip(C[crop])) of its W x H composite C, with the crop
a fixed rectangle (RECT) or the auto-framing state of its camera (AUTO, backscrub_b200/csrc/framing.h).

References: `Ref` restates framing.h in numpy; the outputs are checked against cv2 applied to the composite an unframed
twin context makes of the same feed (fed masks, or the same camera stream: the CNN is batch-invariant).

`-m "not gpu"`: the shared tap arithmetic against the tables build_resize_tab made before it, the kernel-logic emulator
build of k_framing and the cropping k_tail, the C ABI's symbols and refusals.  `-m gpu`: the sm_90a library."""

import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_nv12 import ref_yuyv_to_nv12

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OFF, RECT, AUTO = 0, 1, 2
MODES = {OFF: "off", RECT: "rect", AUTO: "auto"}


# ---------------------------------------------------------------------------------------------------- numpy restatement
def _cdiv(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def _clamp(v, lo, hi):
    return lo if v < lo else (hi if v > hi else v)


class Geo:
    def __init__(self, g):
        self.W, self.H = g.width, g.height
        self.roi, self.out = list(g.roidim), list(g.out_roidim)


def person_box(geo, ofinal):
    ox, oy, sw, sh = geo.out
    m = ofinal[oy:oy + sh, ox:ox + sw] < 128
    ys, xs = np.nonzero(m)
    if not len(ys):
        return 0, 0, 0, 0, 0
    return len(ys), int(xs.min()), int(ys.min()), int(xs.max()), int(ys.max())


def target(geo, box, prm, ow, oh):
    W, H = geo.W, geo.H
    rx, ry, rw, rh = geo.roi
    sw, sh = geo.out[2:]
    max_zoom, margin, _ = prm
    cnt, j0, i0, j1, i1 = box
    x, y, w, h = 0, 0, W, H
    if cnt >= max(1, sw * sh // 1000):
        x0, x1 = rx + j0 * rw // sw, rx + ((j1 + 1) * rw + sw - 1) // sw
        y0, y1 = ry + i0 * rh // sh, ry + ((i1 + 1) * rh + sh - 1) // sh
        bh = y1 - y0
        h = _clamp(bh * (100 + 2 * margin) // 100, H * 100 // max_zoom, H)
        w = (2 * h * ow + oh) // (2 * oh)
        if w > W:
            w, h = W, _clamp((2 * W * oh + ow) // (2 * ow), 1, H)
        w = max(w, 1)
        x = _clamp((x0 + x1 - w + 2 * W) // 2 - W, 0, W - w)
        y = _clamp(y0 - margin * bh // 100, 0, H - h)
    return [16 * x, 16 * y, 16 * w, 16 * h]


def step(s, t, speed, jump):
    if jump:
        return list(t)
    out = []
    for sk, tk in zip(s, t):
        d = tk - sk
        out.append(sk + _cdiv(d * speed + (128 if d >= 0 else -128), 256))
    return out


def crop_of(s, W, H):
    w, h = _clamp((s[2] + 8) >> 4, 1, W), _clamp((s[3] + 8) >> 4, 1, H)
    return (_clamp((s[0] + 8) >> 4, 0, W - w), _clamp((s[1] + 8) >> 4, 0, H - h), w, h)


class Ref:
    """the framing of one context: a state per camera (None = the plain stream), modes and rectangles"""

    def __init__(self, geo, prm=(300, 10, 32)):
        self.geo, self.prm = geo, prm
        self.state, self.jump = {}, {}
        self.mode, self.rect = OFF, None
        self.src = {}

    def eff(self, cam):
        m = self.src.get(cam)
        return (self.mode, self.rect) if m is None else m

    def frame(self, cam, ofinal, ow, oh):
        mode, rect = self.eff(cam)
        if mode == AUTO:
            t = target(self.geo, person_box(self.geo, ofinal), self.prm, ow, oh)
            self.state[cam] = step(self.state.get(cam, [0] * 4), t, self.prm[2], self.jump.get(cam, True))
            c = crop_of(self.state[cam], self.geo.W, self.geo.H)
        else:
            c = tuple(rect) if mode == RECT else (0, 0, self.geo.W, self.geo.H)
        self.jump[cam] = mode != AUTO
        return c

    def reset(self, cam):
        self.jump[cam] = True


def framed_ref(C_, crop, flip, size):
    """cv::resize(cv::flip(C[crop]), size) (app/deepseg.cc:667-679 on the crop)"""
    x, y, w, h = crop
    img = np.ascontiguousarray(C_[y:y + h, x:x + w])
    if flip:
        img = cv2.flip(img, {1: 1, 2: 0, 3: -1}[flip])
    if (w, h) == tuple(size):
        return img
    return cv2.resize(img, tuple(size), interpolation=cv2.INTER_LINEAR)


def video_ref(out, nv12):
    y = po.convert_rgb_to_yuyv(out[..., :3])
    return ref_yuyv_to_nv12(y) if nv12 else y


# ---------------------------------------------------------------------------------------------------- masks
def box_mask(oh, ow, x0, y0, x1, y1, bg=0xFF, fg=0x00):
    m = np.full((oh, ow), bg, np.uint8)
    m[y0:y1, x0:x1] = fg
    return m


def mask_cases(oh, ow, seed):
    """empty, below the speckle threshold, the whole mask, a person at each edge and corner, a tiny one, random"""
    rng = np.random.default_rng(seed)
    cases = [np.full((oh, ow), 0xE0, np.uint8), box_mask(oh, ow, 5, 5, 6, 6), np.zeros((oh, ow), np.uint8)]
    bw, bh = ow // 4, oh // 3
    for x0, y0 in ((0, 0), (ow - bw, 0), (0, oh - bh), (ow - bw, oh - bh), (ow // 2 - bw // 2, 0), (0, oh // 2 - bh // 2),
                   (ow - bw, oh // 2), (ow // 2, oh - bh)):
        cases.append(box_mask(oh, ow, x0, y0, x0 + bw, y0 + bh, bg=0xE3, fg=0x1C))
    cases.append(box_mask(oh, ow, ow // 2, oh // 2, ow // 2 + 3, oh // 2 + 4))       # tiny: the zoom limit holds
    states = np.array([0x00, 0x03, 0x1C, 0x1F, 0xE0, 0xE3, 0xFC, 0xFF], np.uint8)
    for _ in range(3):
        m = np.full((oh, ow), 0xFF, np.uint8)
        x0, y0 = rng.integers(0, ow - 8), rng.integers(0, oh - 8)
        x1, y1 = rng.integers(x0 + 4, ow + 1), rng.integers(y0 + 4, oh + 1)
        m[y0:y1, x0:x1] = states[rng.integers(0, 8, (y1 - y0, x1 - x0))]
        cases.append(m)
    return cases


# ---------------------------------------------------------------------------------------------------- fed checks
class Twin:
    """a framed context and an unframed twin (no flip, W x H) fed the same masks and frames"""

    def __init__(self, lib, key, W, H, mb, fmt="bgr", bgra=False, flip=0, size=None, n_sources=0):
        self.W, self.H, self.fmt, self.bgra = W, H, fmt, bgra
        self.f = api.MaskGen(lib, model_path(key), W, H, max_batch=mb)
        self.u = api.MaskGen(lib, model_path(key), W, H, max_batch=mb)
        for g in (self.f, self.u):
            g.set_background(synth.background())
            if bgra:
                g.set_out_format("bgra")
            if n_sources:
                g.set_sources(n_sources)
        if flip or size:
            self.f.set_output(flip & 1, flip >> 1, size)
        self.flip, self.size = flip, size or (W, H)
        self.src_flip, self.src_size = {}, {}
        self.geo = Geo(self.f)
        self.oh, self.ow = self.f.feed_shape(B.FEED_MASK)[:2]
        self.ref = Ref(self.geo)
        self.t = 0
        self.crops = set()

    def close(self):
        self.f.close()
        self.u.close()

    def frames(self, n):
        W, H = self.W, self.H
        yuyv = np.stack([synth.yuyv_frame(W, H, t=self.t + b, stream=b) for b in range(n)])
        self.t += n
        if self.fmt == "bgr":
            return np.stack([po.yuyv_to_bgr(y) for y in yuyv])
        if self.fmt == "nv12":
            return np.stack([np.concatenate([y[..., 0], y[0::2, :, 1]], axis=0) for y in yuyv])
        return yuyv

    def run(self, g, fr, masks, ids):
        g.feed(B.FEED_MASK, masks)
        if ids is not None:
            return g.composite_sources(fr, ids)
        if self.fmt == "bgr":
            return g.composite(fr)
        if self.fmt == "nv12":
            return g.composite_nv12(fr)
        n = len(fr)
        ow, oh = g.out_width, g.out_height
        out = np.empty((n, oh, ow, g.out_channels), np.uint8)
        vid = np.empty((n, oh, ow, 2), np.uint8) if not self.bgra else None
        mask = np.empty((n, self.H, self.W), np.uint8)
        g.composite_yuyv_into(fr, out, vid, mask)
        return out, vid, mask

    def call(self, masks, ids=None, check_out=True):
        n = len(masks)
        fr = self.frames(n)
        fo, fv, fm = self.run(self.f, fr, masks, ids)
        uo, _, um = self.run(self.u, fr, masks, ids)
        assert np.array_equal(fm, um), "the mask output is not cropped"
        for b in range(n):
            cam = None if ids is None else ids[b]
            flip = self.flip if cam is None or cam not in self.src_flip else self.src_flip[cam]
            size = self.size if cam is None or cam not in self.src_size else self.src_size[cam]
            want = self.ref.frame(cam, masks[b], *size)
            got = self.f.framing(b)
            assert got == want, (b, cam, got, want)
            self.crops.add(got)
            if not check_out:
                continue
            ro = framed_ref(uo[b], got, flip, size)
            assert np.array_equal(fo[b].reshape(ro.shape), ro), ("out", b, cam, got, flip, size)
            if fv is not None and not self.bgra:
                rv = video_ref(ro, self.fmt == "nv12")
                assert np.array_equal(np.asarray(fv[b]).reshape(-1), rv.reshape(-1)), ("video", b, cam, got)

    def set_framing(self, mode, rect=None):
        self.f.set_framing(MODES[mode], rect)
        self.ref.mode, self.ref.rect = mode, rect

    def set_auto(self, *prm):
        self.f.set_framing_auto(*prm)
        self.ref.prm = prm

    def set_source(self, s, mode=None, rect=None, flip=None, size=None):
        self.f.set_source_framing(s, None if mode is None else MODES[mode], rect)
        self.ref.src[s] = None if mode is None else (mode, rect)
        if flip is not None:
            self.f.set_source_flip(s, bool(flip & 1), bool(flip & 2))
            self.src_flip[s] = flip
        if size is not None:
            self.f.set_source_output(s, size)
            self.src_size[s] = size


def _auto_stream(lib, key, W, H, fmt, speeds, mb=4):
    t = Twin(lib, key, W, H, mb, fmt=fmt, flip=1, size=(W // 2 + 2, H // 2))
    cases = mask_cases(t.oh, t.ow, 1)
    t.set_framing(AUTO)
    i = 0
    for sp in speeds:
        t.set_auto(250, 15, sp)
        for n in (3, 1, mb):
            t.call([cases[(i + k) % len(cases)] for k in range(n)])
            i += n
        if sp == speeds[0]:
            t.f.reset_state()
            t.ref.reset(None)
    assert len(t.crops) > 8, t.crops            # the crop moves
    t.close()


def _rect_and_full(lib, key, W, H, fmt, bgra=False):
    t = Twin(lib, key, W, H, 2, fmt=fmt, bgra=bgra, flip=3, size=(W // 2, H // 2))
    cases = mask_cases(t.oh, t.ow, 2)
    # an exact 2x crop (INTER_AREA), an odd crop, a crop of the output size (a copy)
    for rect in ((0, 0, W, H), (3, 5, W - 7, H - 9), (W // 4, H // 4, W // 2, H // 2), (1, 2, W // 2 - 1, H // 2 + 1)):
        t.set_framing(RECT, rect)
        t.call(cases[:2])
    t.set_framing(OFF)
    t.call(cases[2:4])
    t.close()


def _sources(lib, key, W, H, fmt, bgra=False):
    t = Twin(lib, key, W, H, 6, fmt=fmt, bgra=bgra, n_sources=6)
    cases = mask_cases(t.oh, t.ow, 3)
    t.set_framing(AUTO)
    t.set_auto(300, 10, 37)
    t.set_source(1, RECT, (2, 4, W // 2 + 1, H // 2 - 3), flip=1)
    t.set_source(2, OFF, flip=2)
    t.set_source(3, AUTO, size=(W // 2, H // 2 + 2), flip=3)
    t.set_source(4, None, size=(W - 2, H + 4))
    i = 0
    for ids in ([0, 1, 2, 3, 4, 5], [3, 5, 0], [2, 4], [5, 4, 3, 2, 1, 0]):
        t.call([cases[(i + k) % len(cases)] for k in range(len(ids))], ids)
        i += len(ids)
    t.f.reset_source(3)
    t.ref.reset(3)
    t.set_source(2, AUTO)
    t.call([cases[(i + k) % len(cases)] for k in range(4)], [2, 3, 0, 1])
    t.close()


# ---------------------------------------------------------------------------------------------------- CPU


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


TAPS_CC = r"""
#include <cstdio>
#include <cmath>
#include <algorithm>
#include "resize_taps.h"
// build_resize_tab's per-index arithmetic before resize_taps.h existed
int main() {
  long bad = 0;
  for (int s = 1; s <= 1024; ++s)
    for (int d = 1; d <= 1024; ++d) {
      const double sc = 1.0 / ((double)d / s), sc2 = bsb::resize_scale(s, d);
      if (sc != sc2) ++bad;
      for (int i = 0; i < d; ++i) {
        float fx = (float)((i + 0.5) * sc - 0.5);
        int sx = (int)std::floor(fx);
        fx -= (float)sx;
        int y0 = std::min(std::max(sx, 0), s - 1), y1 = std::min(std::max(sx + 1, 0), s - 1);
        const int yw0 = (short)std::lrintf((1.f - fx) * 2048.f), yw1 = (short)std::lrintf(fx * 2048.f);
        if (sx < 0) { fx = 0; sx = 0; }
        if (sx >= s - 1) { fx = 0; sx = s - 1; }
        const int xw0 = (short)std::lrintf((1.f - fx) * 2048.f), xw1 = (short)std::lrintf(fx * 2048.f);
        int a, b, c, e;
        bsb::resize_tap_x(i, sc2, s, &a, &b, &c);
        if (a != sx || b != xw0 || c != xw1) ++bad;
        bsb::resize_tap_y(i, sc2, s, &a, &e, &b, &c);
        if (a != y0 || e != y1 || b != yw0 || c != yw1) ++bad;
      }
    }
  std::printf("%ld\n", bad);
  return 0;
}
"""


def test_taps_equal_the_old_tables(tmp_path):
    """every (source, destination) size pair 1..1024 in both directions: the exact-2x and equal-size pairs included"""
    src = tmp_path / "taps.cc"
    src.write_text(TAPS_CC)
    exe = tmp_path / "taps"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DBSB_EMU", "-ffp-contract=off", "-fno-fast-math",
                           "-I", os.path.join(ROOT, "tests", "emu"), "-I", os.path.join(ROOT, "backscrub_b200", "csrc"),
                           "-o", str(exe), str(src)])
    assert subprocess.check_output([str(exe)]).strip() == b"0"


def test_symbols_and_refusals(emu_lib):
    for name in ("bsb_set_framing", "bsb_set_framing_auto", "bsb_set_source_framing", "bsb_get_framing"):
        assert hasattr(emu_lib, name)
    W, H = 160, 120
    g = api.MaskGen(emu_lib, model_path("meet_lite"), W, H, max_batch=2)
    L, h = emu_lib, g._h
    assert not L.bsb_set_framing(h, 3, 0, 0, 1, 1)
    assert not L.bsb_set_framing(h, -1, 0, 0, 1, 1)
    for r in ((-1, 0, 10, 10), (0, -1, 10, 10), (0, 0, 0, 10), (0, 0, 10, 0), (1, 0, W, H), (0, 1, W, H)):
        assert not L.bsb_set_framing(h, RECT, *r), r
    assert L.bsb_set_framing(h, RECT, 0, 0, W, H)
    assert L.bsb_set_framing(h, OFF, -5, -5, 0, 0)      # the rectangle is read for RECT only
    for prm in ((99, 10, 32), (1001, 10, 32), (300, -1, 32), (300, 101, 32), (300, 10, 0), (300, 10, 257)):
        assert not L.bsb_set_framing_auto(h, *prm), prm
    assert L.bsb_set_framing_auto(h, 100, 0, 256) and L.bsb_set_framing_auto(h, 1000, 100, 1)
    assert not L.bsb_set_source_framing(h, 0, AUTO, 0, 0, 0, 0)      # no sources yet
    r = (C.c_int * 4)()
    assert not L.bsb_get_framing(h, 0, r)                              # no call yet
    g.set_sources(2)
    assert not L.bsb_set_source_framing(h, 2, AUTO, 0, 0, 0, 0)
    assert not L.bsb_set_source_framing(h, 0, -2, 0, 0, 0, 0)
    assert not L.bsb_set_source_framing(h, 0, RECT, 0, 0, W + 1, H)
    assert L.bsb_set_source_framing(h, 0, -1, 0, 0, 0, 0)
    with pytest.raises(api.BackscrubError):
        g.set_framing("zoom")
    # a refused rectangle leaves the context as it was: the next call is not framed
    g.feed(B.FEED_MASK, np.zeros((1,) + g.feed_shape(B.FEED_MASK)[:2], np.uint8))
    g.composite(synth.frame(W, H, t=0))
    assert g.framing(0) == (0, 0, W, H)
    assert not L.bsb_get_framing(h, 1, r)
    g.close()


def test_unframed_launches_unchanged(emu_lib):
    W, H = 160, 120
    a = api.MaskGen(emu_lib, model_path("meet_lite"), W, H, max_batch=2)
    b = api.MaskGen(emu_lib, model_path("meet_lite"), W, H, max_batch=2)
    b.set_framing("rect", (0, 0, W, H))
    b.set_framing("off")
    fr = np.stack([synth.frame(W, H, t=t) for t in range(2)])
    ra, rb = a.composite(fr), b.composite(fr)
    assert a.launches_per_call == b.launches_per_call
    for x, y in zip(ra, rb):
        assert np.array_equal(x, y)
    b.set_framing("auto")
    b.composite(fr)
    assert b.launches_per_call == a.launches_per_call + 2      # k_framing and k_tail
    a.close()
    b.close()


@pytest.mark.parametrize("fmt", ["bgr", "yuyv"])
def test_emu_auto_plain(emu_lib, fmt):
    _auto_stream(emu_lib, "meet_lite", 160, 120, fmt, (1, 37, 256))


@pytest.mark.parametrize("bgra", [False, True])
def test_emu_rect_and_full(emu_lib, bgra):
    _rect_and_full(emu_lib, "meet_lite", 160, 120, "bgr", bgra)


def test_emu_sources(emu_lib):
    _sources(emu_lib, "meet_lite", 160, 120, "bgr")


# ---------------------------------------------------------------------------------------------------- H100


@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["bgr", "yuyv", "nv12"])
def test_gpu_auto_plain(gpu_lib, fmt):
    _auto_stream(gpu_lib, "meet_full", 1280, 720, fmt, (1, 37, 256), mb=8)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,bgra", [("bgr", False), ("yuyv", True), ("nv12", False)])
def test_gpu_rect_and_full(gpu_lib, fmt, bgra):
    _rect_and_full(gpu_lib, "meet_full", 1280, 720, fmt, bgra)


@pytest.mark.gpu
@pytest.mark.parametrize("bgra", [False, True])
def test_gpu_sources(gpu_lib, bgra):
    _sources(gpu_lib, "meet_full", 640, 360, "bgr", bgra)


def _stage2(g, n):
    oh, ow = g.feed_shape(B.FEED_MASK)[:2]
    out = []
    for b in range(n):
        a = np.empty(oh * ow, np.uint8)
        assert g._lib.bsb_get_stage_u8(g._h, 2, b, a.ctypes.data_as(C.POINTER(C.c_uint8)), a.size) > 0
        out.append(a.reshape(oh, ow))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("interval", [1, 2])
def test_gpu_real_frames(gpu_lib, interval):
    """CNN on: graph replay equals eager (flags 2), the crops restated from stage 2, a framed context against its unframed
    twin, with a mask interval and the filter switched off mid-stream"""
    W, H, n = 1280, 720, 4
    ctx = {k: api.MaskGen(gpu_lib, model_path("meet_full"), W, H, max_batch=n, flags=f)
           for k, f in (("graph", 0), ("eager", 2), ("plain", 0))}
    for k, g in ctx.items():
        g.set_background(synth.background())
        g.set_mask_interval(interval)
        if k != "plain":
            g.set_output(True, False, (640, 360))
            g.set_framing("auto")
            g.set_framing_auto(250, 12, 64)
    ref = Ref(Geo(ctx["graph"]), (250, 12, 64))
    ref.mode = AUTO
    for call in range(6):
        if call == 3:
            for g in ctx.values():
                g.set_filter(False)
        fr = np.stack([synth.frame(W, H, t=call * n + b) for b in range(n)])
        res = {k: g.composite(fr) for k, g in ctx.items()}
        for x, y in zip(res["graph"], res["eager"]):
            assert np.array_equal(x, y), call
        masks = _stage2(ctx["plain"], n)
        for b in range(n):
            c = ref.frame(None, masks[b], 640, 360)
            assert ctx["graph"].framing(b) == c and ctx["eager"].framing(b) == c, (call, b)
            assert np.array_equal(res["graph"][0][b], framed_ref(res["plain"][0][b], c, 1, (640, 360))), (call, b)
            assert np.array_equal(res["graph"][2][b], res["plain"][2][b])
    for g in ctx.values():
        g.close()
