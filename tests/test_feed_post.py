"""The decision and post stages on constructed inputs (bsb_test_feed), not only on what the CNN makes of a frame.

A smooth synthetic person gives smooth masks: nearly every post-stage tile is plainly background or person, the mixed
tiles have their edge well inside the patch of the small mask, and the logits never come near a tie, an overflow or the
0.65 threshold.  Here the library is fed chosen smoother outputs (FEED_MASK) and chosen logits (FEED_LOGITS), and every
output is compared bit for bit with references that do not depend on the kernels:

  * mask feeds: cv2 (the reference's cv::resize + cv::blur of lib/libbackscrub.cc:366-374) and the oracle's alpha_blend,
    convert_rgb_to_yuyv, flip and resize; the NV12 output by its definition (tests/test_nv12.py);
  * logit feeds: the oracle's decision + smoother (or_maskgen_post_from_output), one oracle context per stream, the
    DeepLab logits first resized by the oracle's RESIZE_BILINEAR.

Fixtures and what each one puts under pressure:
  UNIFORM        every reachable smoother state and its neighbours: the all-255 / all-0 tile shortcuts of k_post_tma.
  PROBES         one odd pixel on a lattice one wider than the largest patch, shifted until every small-mask pixel of
                 the ROI was probed: a patch extent one row or column short on any side, for TW = 64 and 128, copies a
                 background / person tile that should have been blended (test_probes_catch_each_short_patch shows
                 they do, on a model of the classifier).
  STEPS          a half-plane at every row and column offset: the edge on every patch boundary.
  RANDOM         random bytes and random smoother states: mixed tiles everywhere, masks with no symmetry.
  geometries     720p (TW 64), 4k BodyPix (TW 128), MLKit 640x480, portrait 720x1280 (roi_x > 0: the `inside` test at
                 an ROI edge off the tile grid), 336x250 (ragged tiles, store_clipped of mirrored frames), 324x250
                 (k_post_fast), 128x72 (area2x2: k_post), post_tile forced both ways, post_tma = 0.
  logits         Meet's softmax at ties, one ulp apart, exp overflow / underflow (inf/inf and 0/0 are NaN, and NaN
                 means background), +-inf, NaN, subnormals; MLKit / BodyPix at 0.65f and its neighbours; DeepLab's argmax
                 at ties with class 15, at or below its -10000 start, with NaN classes and with ties that only appear
                 after the folded 33 -> 257 resize.
Subnormal logits: the numeric contract flushes denormals (a CNN output never is one), so the reference sees them as zero.
"""
import math

import cv2
import numpy as np
import pytest

from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_nv12 import ref_yuyv_to_nv12

STATES = [0x00, 0x03, 0x1C, 0x1F, 0xE0, 0xE3, 0xFC, 0xFF]        # the bytes (v & 0xE0) | (s >> 3) can reach from 0
PF_H = 32                                                          # rows of a post-stage tile


# ---------------------------------------------------------------------------------------------------- references
class Geo:
    """frame and mask geometry of a model at W x H (lib/libbackscrub.cc:234-246, from the oracle)"""

    def __init__(self, key, W, H):
        g = po.MaskGen(model_path(key), W, H)
        self.key, self.W, self.H = key, W, H
        self.roi, self.out = g.roidim, g.out_roidim
        self.oh, self.ow = g.out_hwc[:2]
        g.close()


_GEOS = {}


def geo(key, W, H):
    if (key, W, H) not in _GEOS:
        _GEOS[(key, W, H)] = Geo(key, W, H)
    return _GEOS[(key, W, H)]


def ref_mask(g, ofinal):
    """lib/libbackscrub.cc:366-374 with cv2: 255 outside roidim, inside cv::blur(cv::resize(ofinal[out_roidim]), 5x5)"""
    rx, ry, rw, rh = g.roi
    ox, oy, ow, oh = g.out
    m = np.full((g.H, g.W), 255, np.uint8)
    up = cv2.resize(np.ascontiguousarray(ofinal[oy:oy + oh, ox:ox + ow]), (rw, rh), interpolation=cv2.INTER_LINEAR)
    m[ry:ry + rh, rx:rx + rw] = cv2.blur(up, (5, 5), borderType=cv2.BORDER_REFLECT_101)
    return m


def oracle_mask(g, ofinal):
    """the same mask from the oracle's primitives (oracle_pipeline.c upsample_and_blur)"""
    rx, ry, rw, rh = g.roi
    ox, oy, ow, oh = g.out
    m = np.full((g.H, g.W), 255, np.uint8)
    m[ry:ry + rh, rx:rx + rw] = po.box_blur5(po.resize_linear_u8(ofinal[oy:oy + oh, ox:ox + ow], rw, rh))
    return m


def ref_outputs(mask, frame, bg, flip=0, out_size=None, nv12=False, video=True):
    """app/deepseg.cc:661-681: blend, flip, resize to the virtual-camera size, YUYV (NV12 by its definition)"""
    out = po.alpha_blend(bg, frame, mask)
    if flip:
        out = po.flip(out, flip & 1, (flip >> 1) & 1)
    if out_size and out_size != (out.shape[1], out.shape[0]):
        out = po.resize_linear_u8(out, *out_size)
    if not video:
        return out, None
    video = po.convert_rgb_to_yuyv(out)
    return out, ref_yuyv_to_nv12(video) if nv12 else video


def daz(x):
    """the numeric contract's denormals-are-zero: a subnormal logit reads as a zero of its sign"""
    x = np.asarray(x, np.float32)
    return np.where(np.abs(x) < np.finfo(np.float32).tiny, np.copysign(np.float32(0), x), x).astype(np.float32)


def deeplab_resize_opts():
    from tools import tflite_graph
    gr = tflite_graph.load(model_path("deeplab"))
    o = [op for op in gr.ops if op.kind == "RESIZE_BILINEAR"][-1].opts
    return bool(o["align_corners"]), bool(o["half_pixel"])


class OracleStream:
    """one stream's decision + smoother + mask on the oracle"""

    def __init__(self, key, W, H):
        self.key, self.g = key, po.MaskGen(model_path(key), W, H)
        self.up = None
        if key == "deeplab":
            self.up = (self.g.out_hwc[0], self.g.out_hwc[1], *deeplab_resize_opts())

    def step(self, logits):
        x = daz(logits)
        if self.up:
            oh, ow, ac, hp = self.up
            x = po.resize_bilinear(x, oh, ow, align_corners=ac, half_pixel=hp)
        mask = self.g.post_from_output(x)
        return mask, self.g.ofinal.copy()


# ---------------------------------------------------------------------------------------------------- k_post_tma's patch tables
def resize_tab(sw, sh, dw, dh):
    """build_resize_tab (engine.cu): the source column of each destination column, the two source rows of each row"""
    sx, sy = 1.0 / (dw / sw), 1.0 / (dh / sh)
    xofs, y0, y1 = [], [], []
    for dx in range(dw):
        s = math.floor(float(np.float32((dx + 0.5) * sx - 0.5)))
        xofs.append(0 if s < 0 else (sw - 1 if s >= sw - 1 else s))
    for dy in range(dh):
        s = math.floor(float(np.float32((dy + 0.5) * sy - 0.5)))
        y0.append(min(max(s, 0), sh - 1))
        y1.append(min(max(s + 1, 0), sh - 1))
    return xofs, y0, y1


def _span(lo, ln, n, first, last, plus, lmax):
    hi = lo + ln - 1
    i0 = 0 if lo < 0 else min(lo, n - 1)
    i1 = n - 1 if hi >= n else max(hi, 0)
    a0, a1 = first[i0], min(last[i1] + plus, lmax)
    return a0, a1 - a0 + 1


def tile_patches(g, tw):
    """[(ty0, tx0, rmin, nrows, cmin, ncols)] of every tile that meets the ROI: the rows / columns of out_roidim the
    tile's halo (+-2, reflect-101) reads through the resize, as engine.cu's tables give them to k_post_tma"""
    rx, ry, rw, rh = g.roi
    sw, sh = g.out[2], g.out[3]
    xofs, y0, y1 = resize_tab(sw, sh, rw, rh)
    res = []
    for ty0 in range(0, g.H, PF_H):
        for tx0 in range(0, g.W, tw):
            if not (tx0 < rx + rw and tx0 + tw > rx and ty0 < ry + rh and ty0 + PF_H > ry):
                continue
            r = _span(ty0 - ry - 2, PF_H + 4, rh, y0, y1, 0, 1 << 30)
            c = _span(tx0 - rx - 2, tw + 4, rw, xofs, xofs, 1, sw - 1)
            res.append((ty0, tx0, r[0], r[1], c[0], c[1]))
    return res


SIDES = ("top", "bottom", "left", "right")


def shrink(p, side):
    ty0, tx0, r0, nr, c0, nc = p
    if side == "top":
        return ty0, tx0, r0 + 1, nr - 1, c0, nc
    if side == "bottom":
        return ty0, tx0, r0, nr - 1, c0, nc
    if side == "left":
        return ty0, tx0, r0, nr, c0 + 1, nc - 1
    return ty0, tx0, r0, nr, c0, nc - 1


def classify(g, tw, patches, odd):
    """k_post_tma's tile kinds (kernels_post.cu, warp 0) for one frame: 0 background (every examined byte 255), 1 person
    (every byte 0 and the tile inside the ROI), 2 mixed.  The kernel examines rows [rmin, rmin + nrows) and the 32-bit
    words of the 16-byte aligned box from its start to column cmin + ncols; `odd` is (hi, lo): where the small mask is
    not 255 / not 0 (bytes outside the mask read as 0, as TMA fills them)."""
    ox, oy = g.out[0], g.out[1]
    rx, ry, rw, rh = g.roi
    P = np.array(patches).T
    ty0, tx0, r0, nr, c0, nc = P
    coff = (ox + c0) & 15
    b0 = ox + c0 - coff
    b1 = b0 + ((coff + nc + 3) >> 2) * 4
    y0, y1 = oy + r0, oy + r0 + nr

    def count(ind):                                      # odd bytes inside each tile's examined box (summed-area table)
        S = np.zeros((ind.shape[0] + 1, ind.shape[1] + 1 + 64), np.int64)
        S[1:, 1:ind.shape[1] + 1] = ind.cumsum(0).cumsum(1)
        S[:, ind.shape[1] + 1:] = S[:, ind.shape[1]:ind.shape[1] + 1]
        return S[y1, b1] - S[y0, b1] - S[y1, b0] + S[y0, b0]
    not_hi = (count(odd[0]) > 0) | (b1 > g.ow)
    not_lo = count(odd[1]) > 0
    inside = (tx0 >= rx) & (np.minimum(tx0 + tw, g.W) <= rx + rw) & (ty0 >= ry) & (np.minimum(ty0 + PF_H, g.H) <= ry + rh)
    return np.where(~not_hi, 0, np.where(~not_lo & inside, 1, 2))


def tile_truth(g, tw, patches, mask):
    """what each tile's mask really is: 0 all 255, 1 all 0, 2 neither"""
    H2, W2 = -(-g.H // PF_H) * PF_H, -(-g.W // tw) * tw
    hi = np.zeros((H2, W2), bool)
    lo = np.zeros((H2, W2), bool)
    hi[:g.H, :g.W] = mask != 255
    lo[:g.H, :g.W] = mask != 0
    hi = hi.reshape(H2 // PF_H, PF_H, W2 // tw, tw).any(axis=(1, 3))
    lo = lo.reshape(H2 // PF_H, PF_H, W2 // tw, tw).any(axis=(1, 3))
    ty, tx = np.array([p[0] // PF_H for p in patches]), np.array([p[1] // tw for p in patches])
    return np.where(~hi[ty, tx], 0, np.where(~lo[ty, tx], 1, 2))


# ---------------------------------------------------------------------------------------------------- mask fixtures
def uniform(g):
    vals = sorted(set([0, 255, 1, 254] + STATES))
    return np.stack([np.full((g.oh, g.ow), v, np.uint8) for v in vals])


PROBES = [(255, 0), (255, 0xE0), (255, 0xFC), (255, 254), (0, 255), (0, 3)]    # (base, probe value)


def probe_spacing(g, tw):
    """one more than the largest patch of k_post_tma's tiles of width tw, in rows and in columns"""
    ext = tile_patches(g, tw)
    return max(p[3] for p in ext) + 1, max(p[5] for p in ext) + 1


def probes(g, base, v, spacing):
    """single-pixel probes of value v on a `base` mask, on a lattice `spacing` (rows, columns) apart, shifted from frame
    to frame until every pixel of out_roidim has been probed once"""
    ox, oy, ow, oh = g.out
    sy, sx = spacing
    frames = []
    for dy in range(min(sy, oh)):
        for dx in range(min(sx, ow)):
            m = np.full((g.oh, g.ow), base, np.uint8)
            m[oy + dy:oy + oh:sy, ox + dx:ox + ow:sx] = v
            frames.append(m)
    return np.stack(frames)


def steps(g):
    """a person half-plane (0) under a background one (255) at every row offset of out_roidim, then a person left part
    at every column offset"""
    ox, oy, ow, oh = g.out
    res = []
    for k in range(oh + 1):
        m = np.full((g.oh, g.ow), 255, np.uint8)
        m[:oy + k] = 0
        res.append(m)
    for k in range(ow + 1):
        m = np.full((g.oh, g.ow), 255, np.uint8)
        m[:, :ox + k] = 0
        res.append(m)
    return np.stack(res)


def random_masks(g, n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, (n, g.oh, g.ow), dtype=np.uint8)
    b = np.array(STATES, np.uint8)[rng.integers(0, 8, (n, g.oh, g.ow))]
    return np.concatenate([a, b])


# ---------------------------------------------------------------------------------------------------- CPU: references, fault models
CPU_GEOS = [("meet_full", 1280, 720), ("bodypix", 3840, 2160), ("mlkit", 640, 480), ("meet_full", 720, 1280), ("meet_lite", 336, 250),
            ("meet_lite", 324, 250), ("meet_full", 128, 72)]


@pytest.mark.parametrize("key,W,H", CPU_GEOS)
def test_cv2_reference_agrees_with_oracle(key, W, H):
    g = geo(key, W, H)
    sp = probe_spacing(g, 64)
    masks = np.concatenate([uniform(g), random_masks(g, 4, 1), steps(g)[::7], probes(g, 255, 0, sp)[::11], probes(g, 0, 3, sp)[::13]])
    for m in masks:
        assert np.array_equal(ref_mask(g, m), oracle_mask(g, m))


# tile width -> a geometry whose k_post_tma runs at that width by frame size
FAULT_GEOS = {64: [("meet_full", 1280, 720)], 128: [("bodypix", 3840, 2160)]}


@pytest.mark.parametrize("tw", [64, 128])
def test_probes_catch_each_short_patch(tw):
    """Non-vacuity of the probe fixtures: on a model of k_post_tma's classifier fed the engine's patch tables, the true
    tables never call a tile uniform whose reference mask is not, and each of the four one-short patches (a row or a
    column missing on one side) does so on at least one tile of the probe fixtures."""
    caught = {s: 0 for s in SIDES}
    for key, W, H in FAULT_GEOS[tw]:
        g = geo(key, W, H)
        true = tile_patches(g, tw)
        faulty = {s: [shrink(p, s) for p in true] for s in SIDES}
        for base, v in PROBES[::3]:
            for m in probes(g, base, v, probe_spacing(g, tw)):
                truth = tile_truth(g, tw, true, ref_mask(g, m))
                odd = (m != 255, m != 0)
                wrong = lambda kinds: int(((kinds != 2) & (kinds != truth)).sum())
                assert wrong(classify(g, tw, true, odd)) == 0, (key, W, H, base, v)
                for s in SIDES:
                    caught[s] += wrong(classify(g, tw, faulty[s], odd))
    assert all(caught.values()), caught


# ---------------------------------------------------------------------------------------------------- running fed calls
class Post:
    """One context fed mask batches: every output of every frame checked against ref_outputs.

    fmt: bgr / yuyv / nv12 host calls (the post kernel reads YUYV and NV12 frames in place where it can); bg: still (an
    image), ring (three images, advancing one per frame) or camblur (no image, the camera frame blurred)."""

    def __init__(self, lib, key, W, H, max_batch=32, bg="still", flip=0, out_size=None):
        self.g = geo(key, W, H)
        self.c = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch)
        self.mb, self.bg_kind, self.flip, self.out_size = max_batch, bg, flip, out_size
        self.blurred = {}
        raw = synth.background()
        if bg == "still":
            self.c.set_background(raw)
            self.bgs = [po.resize_linear_u8(raw, W, H)]
        elif bg == "ring":
            ring = np.stack([np.roll(raw, 97 * i, axis=1) for i in range(3)])
            self.c.set_background_ring(ring, advance=1)
            self.bgs = [po.resize_linear_u8(r, W, H) for r in ring]
            self.cursor = 0
        else:
            self.c.set_bgblur(7)
        if flip or out_size:
            self.c.set_output(flip & 1, (flip >> 1) & 1, out_size)
        self.yuyv = [synth.yuyv_frame(W, H, t=t) for t in range(2)]
        self.bgr = {"bgr": [synth.frame(W, H, t=t) for t in range(2)], "yuyv": [po.yuyv_to_bgr(y) for y in self.yuyv]}
        self.nv12 = [np.concatenate([y[..., 0], y[0::2, :, 1]], axis=0) for y in self.yuyv]
        self.bgr["nv12"] = [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in self.nv12]

    def close(self):
        self.c.close()

    def call(self, masks, fmt="bgr", want=(True, True, True)):
        n = len(masks)
        self.c.feed(B.FEED_MASK, masks)
        W, H = self.g.W, self.g.H
        ow, oh = self.c.out_width, self.c.out_height
        if fmt == "bgr":
            return self.c.composite(np.stack([self.bgr["bgr"][b % 2] for b in range(n)]), *want)
        if fmt == "yuyv":
            out = np.empty((n, oh, ow, 3), np.uint8) if want[0] else None
            vid = np.empty((n, oh, ow, 2), np.uint8) if want[1] else None
            mask = np.empty((n, H, W), np.uint8) if want[2] else None
            self.c.composite_yuyv_into(np.stack([self.yuyv[b % 2] for b in range(n)]), out, vid, mask)
            return out, vid, mask
        return self.c.composite_nv12(np.stack([self.nv12[b % 2] for b in range(n)]), *want)

    def background(self, b, fmt):
        if self.bg_kind == "camblur":
            if (fmt, b % 2) not in self.blurred:
                self.blurred[(fmt, b % 2)] = po.gaussian_blur(self.bgr[fmt][b % 2], 7)
            return self.blurred[(fmt, b % 2)]
        if self.bg_kind == "ring":
            return self.bgs[(self.cursor + b) % 3]
        return self.bgs[0]

    def check(self, masks, fmt="bgr", want=(True, True, True), tag=""):
        for i in range(0, len(masks), self.mb):
            chunk = masks[i:i + self.mb]
            out, vid, mask = self.call(chunk, fmt, want)
            for b, m in enumerate(chunk):
                rm = ref_mask(self.g, m)
                ro, rv = ref_outputs(rm, self.bgr[fmt][b % 2], self.background(b, fmt), self.flip, self.out_size, fmt == "nv12", want[1])
                where = (tag, fmt, want, i + b)
                if mask is not None:
                    assert np.array_equal(mask[b], rm), ("mask", where, int((mask[b] != rm).sum()))
                if out is not None:
                    assert np.array_equal(out[b], ro), ("composite", where, int((out[b] != ro).sum()))
                if vid is not None:
                    assert np.array_equal(vid[b].reshape(-1), rv.reshape(-1)), ("video", where)
            if self.bg_kind == "ring":
                self.cursor = (self.cursor + len(chunk)) % 3


def logits_cases(key, hwc, n, seed):
    """n frames of logits [n, h, w, c] whose pixels take the model's edge cases (and ordinary values between them)"""
    rng = np.random.default_rng(seed)
    h, w, c = hwc
    f32 = np.float32
    inf, nan, sub = f32(np.inf), f32(np.nan), f32(1e-40)
    if key.startswith("meet"):
        x = rng.normal(0, 3, 10).astype(f32)
        up = np.nextafter(x, f32(np.inf))
        cases = [(0, 0), (89, 89), (-104, -104), (x[0], x[0]), (x[1], x[1])]
        cases += [(a, b) for a, b in zip(x, up)] + [(b, a) for a, b in zip(x, up)]
        cases += [(89, 90), (100, 95), (88.7, 88.8), (88.72283935546875, 88.72284698486328), (-104, -110), (-200, -150), (-87.3, -87.4),
                  (100, -200), (-200, 100), (89, -104), (-104, 89)]
        cases += [(inf, 0), (0, inf), (-inf, 0), (0, -inf), (inf, inf), (-inf, -inf), (inf, -inf), (-inf, inf), (nan, 0), (0, nan), (nan, nan)]
        cases += [(sub, 0), (0, sub), (-sub, sub), (sub, -sub), (sub, f32(2e-40)), (f32(1.2e-38), 0), (0, f32(1.2e-38))]
        table = np.array(cases, f32)
    elif key == "deeplab":
        rows = []
        base = lambda: rng.normal(0, 2, 21).astype(f32)
        for lo in (0, 3, 14):
            r = base(); r[15] = r[lo] = f32(9)
            rows.append(r)                                   # tie with a lower class: the lower one wins (background)
        for hi in (16, 20):
            r = base(); r[15] = r[hi] = f32(9)
            rows.append(r)                                   # tie with a higher class: class 15 wins (person)
        rows.append(np.full(21, -10000, f32))
        r = np.full(21, -20000, f32); r[15] = -10000; rows.append(r)
        r = np.full(21, -20000, f32); r[15] = np.nextafter(f32(-10000), f32(0)); rows.append(r)
        r = np.full(21, -10001, f32); r[7] = -10000; rows.append(r)
        r = base(); r[15] = nan; rows.append(r)
        r = base(); r[:15] = nan; r[15] = -50; rows.append(r)
        r = base(); r[3] = nan; r[15] = 20; rows.append(r)
        r = np.full(21, nan, f32); rows.append(r)
        r = np.full(21, -inf, f32); r[15] = -1e30; rows.append(r)
        r = base(); r[15] = inf; rows.append(r)
        r = np.zeros(21, f32); r[15] = sub; rows.append(r)
        r = np.zeros(21, f32); r[2] = -sub; rows.append(r)
        for _ in range(8):
            rows.append(base())
        table = np.stack(rows)
        x = table[rng.integers(0, len(table), (n, h, w))]
        # exact ties after the resize: class 14 alternates 0 / 2 along the columns (rows) of some frames while class 15
        # holds 1, so every interpolated point halfway between two nodes ties (the dyadic weights keep it exact)
        for f in range(n):
            if f % 3 == 1:
                x[f, :, :, :] = f32(-5)
                x[f, :, :, 15] = 1
                if f % 2:
                    x[f, :, :, 14] = (np.arange(w) % 2 * 2)[None, :]
                else:
                    x[f, :, :, 14] = (np.arange(h) % 2 * 2)[:, None]
                x[f, :, :, 16] = np.where((np.arange(h)[:, None] + np.arange(w)[None, :]) % 2, 1, -3)
        return np.ascontiguousarray(x, f32)
    else:
        t = f32(0.65)
        vals = [t, np.nextafter(t, f32(1)), np.nextafter(t, f32(0)), inf, -inf, nan, sub, -sub, f32(0), f32(1), f32(-1)]
        vals += list(rng.uniform(0.6, 0.7, 8).astype(f32))
        table = np.array(vals, f32)[:, None]
    x = table[rng.integers(0, len(table), (n, h, w))]
    return np.ascontiguousarray(x.reshape(n, h, w, c), f32)


def check_logits(lib, key, W, H, n, calls=3, sources=False, seed=0):
    """`calls` consecutive fed calls of n frames (plain, or sources calls of n permuted sources), the smoother carrying
    from call to call: masks and smoother outputs against one oracle stream per camera"""
    c = api.MaskGen(lib, model_path(key), W, H, max_batch=n)
    hwc = c.feed_shape(B.FEED_LOGITS)
    refs = {}
    try:
        if sources:
            c.set_sources(n)
        for k in range(calls):
            x = logits_cases(key, hwc, n, seed + k)
            ids = list(np.random.default_rng(seed + k).permutation(n)) if sources else [0] * n
            c.feed(B.FEED_LOGITS, x)
            frames = np.stack([synth.frame(W, H, t=b) for b in range(n)])
            if sources:
                _, _, mask = c.composite_sources(frames, ids, want_out=False, want_yuyv=False)
            else:
                _, _, mask = c.composite(frames, want_out=False, want_yuyv=False)
            for b in range(n):
                s = int(ids[b])
                if s not in refs:
                    refs[s] = OracleStream(key, W, H)
                rm, rof = refs[s].step(x[b])
                assert np.array_equal(mask[b], rm), (key, k, b, s, int((mask[b] != rm).sum()))
                assert np.array_equal(c.stage_u8(2, b), rof), (key, k, b, s)
    finally:
        c.close()
        for r in refs.values():
            r.g.close()


# ---------------------------------------------------------------------------------------------------- CPU: the emulator
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


@pytest.mark.parametrize("key,W,H", [("meet_lite", 96, 64), ("meet_full", 128, 72), ("meet_lite", 98, 60)])
def test_emu_mask_feed(emu_lib, key, W, H):
    """k_post_fast / k_post (area2x2) and k_tail on every mask fixture of a small geometry"""
    g = geo(key, W, H)
    p = Post(emu_lib, key, W, H, max_batch=16)
    sp = (7, 7)                                      # k_post_fast / k_post: no patch classification
    masks = np.concatenate([uniform(g)[::2], steps(g)[::11], random_masks(g, 1, 5)] + [probes(g, b, v, sp)[::41] for b, v in PROBES])
    p.check(masks, "bgr", tag="emu")
    p.check(masks[:6], "yuyv", want=(False, True, True))
    p.close()
    t = Post(emu_lib, key, W, H, max_batch=4, bg="camblur", flip=3, out_size=(W // 2 * 2 + 18, H + 6))
    t.check(random_masks(g, 2, 7), "bgr", tag="emu tail")
    t.close()


@pytest.mark.parametrize("key", ["meet_lite", "mlkit", "bodypix"])
@pytest.mark.parametrize("par", [0, 1])
def test_emu_logits_feed(emu_lib, key, par):
    """k_decision_iir / k_decision_par (plain) and k_decision_sources on every logit fixture, the state carried over three
    calls"""
    assert emu_lib.bsb_set_tuning(b"dec_par", par)
    try:
        check_logits(emu_lib, key, 96, 64, n=5)
        check_logits(emu_lib, key, 96, 64, n=4, sources=True, seed=10)
    finally:
        emu_lib.bsb_set_tuning(b"dec_par", 1)


@pytest.mark.parametrize("par", [0, 1])
def test_emu_logits_feed_deeplab(emu_lib, par):
    """k_decision_up_iir / k_decision_up_par / k_decision_up_sources: the argmax after the folded 33 -> 257 resize"""
    assert emu_lib.bsb_set_tuning(b"dec_par", par)
    try:
        check_logits(emu_lib, "deeplab", 96, 64, n=3, calls=2)
        check_logits(emu_lib, "deeplab", 96, 64, n=3, calls=2, sources=True, seed=20)
    finally:
        emu_lib.bsb_set_tuning(b"dec_par", 1)


def test_emu_feed_errors_and_state(emu_lib):
    """misuse is refused and leaves the context usable; a mask feed leaves the smoother state alone, a logit feed advances
    it; the feed is consumed by one call"""
    key, W, H = "meet_lite", 96, 64
    c = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    g = geo(key, W, H)
    hwc = c.feed_shape(B.FEED_LOGITS)
    assert c.feed_shape(B.FEED_MASK) == (g.oh, g.ow, 1)
    fr = np.stack([synth.frame(W, H, t=t) for t in range(2)])
    with pytest.raises(api.BackscrubError, match="feed size"):
        c.feed(B.FEED_MASK, np.zeros((2, g.oh, g.ow + 1), np.uint8))
    with pytest.raises(api.BackscrubError, match="unknown feed stage"):
        c.feed(3, np.zeros((2, g.oh, g.ow), np.uint8))
    with pytest.raises(api.BackscrubError, match="unknown feed stage"):
        c.feed_shape(0)
    with pytest.raises(api.BackscrubError, match="n_frames"):
        c.feed(B.FEED_MASK, np.zeros((5, g.oh, g.ow), np.uint8))
    c.feed(B.FEED_MASK, np.zeros((3, g.oh, g.ow), np.uint8))
    with pytest.raises(api.BackscrubError, match="differs from the armed feed"):
        c.composite(fr)
    assert emu_lib.bsb_set_tuning(b"e2e_chunk", 1)
    try:
        c.feed(B.FEED_MASK, np.zeros((2, g.oh, g.ow), np.uint8))
        with pytest.raises(api.BackscrubError, match="split into chunks"):
            c.composite_yuyv(np.stack([synth.yuyv_frame(W, H, t=t) for t in range(2)]))
    finally:
        emu_lib.bsb_set_tuning(b"e2e_chunk", 16)
    # the refused calls consumed their feeds: a plain call runs the CNN again
    _, _, m_real = c.composite(fr)
    ref = po.MaskGen(model_path(key), W, H)
    assert np.array_equal(m_real[1], [ref.process(f) for f in fr][1])
    ref.close()
    # state: A = logits L0, mask M, logits L1; B = logits L0, logits L1
    x0, x1 = logits_cases(key, hwc, 2, 1), logits_cases(key, hwc, 2, 2)
    m = random_masks(g, 1, 3)
    res = []
    for with_mask in (True, False):
        c.reset_state()
        c.feed(B.FEED_LOGITS, x0)
        c.composite(fr)
        if with_mask:
            c.feed(B.FEED_MASK, m)
            _, _, mm = c.composite(fr)
            assert np.array_equal(mm[1], ref_mask(g, m[1]))
            assert np.array_equal(c.stage_u8(2, 1), m[1])
        c.feed(B.FEED_LOGITS, x1)
        _, _, ml = c.composite(fr)
        res.append((ml, c.stage_u8(2, 1)))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    c.close()


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    # host YUYV calls of 32 frames run as one launch (a fed call is never split into chunks)
    L.bsb_set_tuning(b"e2e_chunk", 0)
    yield L
    L.bsb_set_tuning(b"e2e_chunk", 16)


@pytest.fixture
def tuning(gpu_lib):
    """process-wide switches for one test, restored afterwards"""
    saved = []

    def set_(name, value, default):
        assert gpu_lib.bsb_set_tuning(name.encode(), value)
        saved.append((name, default))
    yield set_
    for name, default in saved:
        gpu_lib.bsb_set_tuning(name.encode(), default)


def all_fixtures(g, sp, n_random=16, probe_kinds=PROBES):
    """every mask fixture; the probe lattice `sp` apart.  The probes of 0 into 255 and of 255 into 0 sweep every pixel, the
    other probe values every seventh lattice position"""
    fx = {"uniform": uniform(g), "steps": steps(g), "random": random_masks(g, n_random, 11)}
    for b, v in probe_kinds:
        fx[f"probe_{b}_{v}"] = probes(g, b, v, sp)[::1 if v in (0, 255) else 7]
    return fx


# (key, W, H, post_tile, post_tma)
GPU_GEOS = [("meet_full", 1280, 720, 0, 1), ("bodypix", 3840, 2160, 0, 1), ("mlkit", 640, 480, 0, 1), ("meet_full", 720, 1280, 0, 1),
            ("meet_lite", 336, 250, 0, 1), ("meet_lite", 324, 250, 0, 1), ("meet_full", 128, 72, 0, 1), ("meet_full", 1280, 720, 128, 1),
            ("bodypix", 3840, 2160, 64, 1), ("meet_full", 1280, 720, 0, 0)]
GPU_IDS = ["meet720p_tw64", "bodypix4k_tw128", "mlkit640x480", "portrait720x1280", "lite336x250_ragged", "lite324x250_fast",
           "full128x72_area", "meet720p_tw128", "bodypix4k_tw64", "meet720p_no_tma"]


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H,tile,tma", GPU_GEOS, ids=GPU_IDS)
def test_gpu_mask_fixtures(gpu_lib, tuning, key, W, H, tile, tma):
    """every mask fixture, BGR frames, a still background; every output on all but the probe sweeps (composite and mask:
    what the tile classification decides).  Where k_post_tma runs, the probe lattice is one wider than its patches;
    elsewhere (W % 16 != 0, area2x2, post_tma = 0) 9 pixels.  The forced tile widths repeat the full probe sweeps only."""
    tuning("post_tile", tile, 0)
    tuning("post_tma", tma, 1)
    g = geo(key, W, H)
    tw = tile or (128 if W >= 2560 else 64)
    tma_ok = tma and W % 16 == 0 and not (g.out[2] == 2 * g.roi[2] and g.out[3] == 2 * g.roi[3])
    sp = probe_spacing(g, tw) if tma_ok else (9, 9)
    p = Post(gpu_lib, key, W, H)
    fx = all_fixtures(g, sp, n_random=4 if W * H > 4_000_000 else 16, probe_kinds=PROBES if not tile else [PROBES[0], PROBES[4]])
    for name, masks in fx.items():
        if tile and not name.startswith("probe"):
            continue
        p.check(masks, "bgr", want=(True, False, True) if name.startswith("probe") else (True, True, True), tag=name)
    p.close()


# formats x output subsets x backgrounds on the fixtures that mix tile kinds most
@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("meet_full", 1280, 720), ("meet_full", 720, 1280), ("meet_lite", 336, 250), ("meet_lite", 324, 250)])
@pytest.mark.parametrize("bg", ["still", "ring", "camblur"])
def test_gpu_formats_outputs_backgrounds(gpu_lib, key, W, H, bg):
    g = geo(key, W, H)
    p = Post(gpu_lib, key, W, H, bg=bg)
    sp = probe_spacing(g, 64)
    masks = np.concatenate([random_masks(g, 8, 3), steps(g)[::9], probes(g, 255, 0, sp)[::17], probes(g, 0, 255, sp)[::19]])
    for fmt in ("bgr", "yuyv", "nv12"):
        for want in [(True, True, True), (True, False, False), (False, True, False), (False, False, True), (False, True, True)]:
            p.check(masks[:32] if want != (True, True, True) else masks, fmt, want, tag=bg)
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("meet_full", 1280, 720), ("meet_lite", 336, 250)])
@pytest.mark.parametrize("fmt", ["bgr", "nv12"])
def test_gpu_plain_tail(gpu_lib, key, W, H, fmt):
    """a context flip and resize: k_tail after the post kernel"""
    g = geo(key, W, H)
    p = Post(gpu_lib, key, W, H, flip=1, out_size=(W // 4 * 2 + 2, H // 4 * 2 + 2))      # even: NV12 output
    p.check(np.concatenate([random_masks(g, 4, 9), probes(g, 255, 0, probe_spacing(g, 64))[::23]]), fmt, tag="tail")
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("meet_full", 1280, 720), ("meet_lite", 336, 250), ("meet_full", 720, 1280)])
@pytest.mark.parametrize("resized", [False, True])
def test_gpu_sources_mirrored(gpu_lib, key, W, H, resized):
    """sources calls with flips 0..3 mirrored in place by k_post_tma (336x250: ragged tiles stored clipped at negative box
    coordinates), one source blurring its camera frame; `resized`: one more source with its own output size sends the call
    through k_tail.  The masks have no symmetry, so a wrongly mirrored row shows."""
    g = geo(key, W, H)
    n = 6 if resized else 5
    c = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=n)
    raw = synth.background()
    c.set_background(raw)
    still = po.resize_linear_u8(raw, W, H)
    c.set_sources(n)
    flips = [0, 1, 2, 3, 1, 3]
    for s in range(n):
        c.set_source_flip(s, bool(flips[s] & 1), bool(flips[s] & 2))
    c.set_source_effect(4, "none", 9)
    own = (W // 2 + 4, H // 2 + 2)
    if resized:
        c.set_source_output(5, own)
    masks = np.concatenate([random_masks(g, 6, 4), probes(g, 255, 0, probe_spacing(g, 64))[::29], steps(g)[::31]])
    for k in range(0, len(masks) - n + 1, n):
        ids = list(np.random.default_rng(k).permutation(n))
        frames = np.stack([synth.frame(W, H, t=k + b) for b in range(n)])
        chunk = masks[k:k + n]
        c.feed(B.FEED_MASK, chunk)
        out, vid, mask = c.composite_sources(frames, ids)
        for b, s in enumerate(ids):
            rm = ref_mask(g, chunk[b])
            bg = po.gaussian_blur(frames[b], 9) if s == 4 else still
            ro, rv = ref_outputs(rm, frames[b], bg, flips[s], own if (resized and s == 5) else None)
            assert np.array_equal(mask[b], rm), ("mask", k, b, s)
            assert np.array_equal(out[b], ro), ("composite", k, b, s, int((np.asarray(out[b]) != ro).sum()))
            assert np.array_equal(np.asarray(vid[b]).reshape(-1), rv.reshape(-1)), ("video", k, b, s)
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["meet_full", "mlkit", "bodypix", "deeplab"])
@pytest.mark.parametrize("par", [0, 1])
def test_gpu_logits(gpu_lib, tuning, key, par):
    """every logit fixture of the model through plain calls (the frame-parallel window and the per-pixel loop) and
    sources calls, three calls in a row"""
    tuning("dec_par", par, 1)
    n = 8 if key == "deeplab" else 32
    check_logits(gpu_lib, key, 320, 240, n=n)
    check_logits(gpu_lib, key, 320, 240, n=min(n, 8), sources=True, seed=30)
