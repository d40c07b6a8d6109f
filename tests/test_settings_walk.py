"""The fused call's settings together: a seeded walk of setters and calls on one context, every frame of every call
against one reference model of the context (`Ref`), built from the references the feature tests use.

Each feature (NV12, per-source effects, flips, output sizes, rings, the filter switch, BGRA output, live backgrounds, the
mask interval, framing) is tested against its own reference with the other settings mostly at their defaults.  They all
meet in the per-call tables Engine::run builds (the source table, the framing, live and segment tables) and, on the GPU,
in the key that selects a captured graph.  Here they meet in any order: `walk(seed, steps)` draws setters and calls from
the public API, about one step in ten refused, and `Ref` predicts the refusal or every output byte.

  `-m "not gpu"`: the pair coverage of the walk (no library), and the walk on the kernel-logic emulator build.
  `-m gpu`: the same walk on a context that captures graphs and on a BSB_FLAG_NO_GRAPH twin given the same setters; every
  call graph vs eager and both vs `Ref`, with the graph cache overflowing and replays that launch nothing.

A walk is: drawn steps (random setters and calls, a new context every EPISODE steps), a sweep (one call per compound
pair of call kind x input format x out format and background kind x blur class), toggle blocks (one call repeated under
two values of a setting the graph key may or may not carry, so a missing key field replays a graph of the other value),
and on the GPU a tail of more distinct call signatures than the graph cache holds.

Masks: each camera cycles through FRAMES_PER_CAM frames per input format; the oracle's logits of each are computed once
and every camera's smoother is stepped from them (the CNN is stateless), so the CPU cost of a CNN frame is an oracle
smoother step.  About a third of the calls feed smoother outputs (FEED_MASK) from test_feed_post's fixtures instead.
On a failure the message gives the seed, the step, what differed and the steps so far as a script; `walk_prefix(seed, k)`
replays a walk up to step k."""

import itertools
from types import SimpleNamespace

import numpy as np
import pytest

from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_bgra_output import expect_bgra, nv12_to_bgr
from tests.test_feed_post import geo, probe_spacing, probes, random_masks, ref_mask, steps as step_masks
from tests.test_framing import AUTO, MODES, OFF, RECT, Ref as FramingRef, framed_ref, video_ref
from tests.test_live_background import expected_bg, live_bgr, live_nv12, padded_bgr, padded_nv12

KEY, W, H = "meet_lite", 336, 250        # W % 16 == 0, W % 64 != 0, H % 32 != 0: ragged k_post_tma tiles both ways
MB, N_SRC_CHOICES = 4, (3, 4)
OUT_STEP, VIDEO_STEP = 400 * 300 * 4, 400 * 300 * 2          # bytes per frame of the device outputs: the largest size
FRAMES_PER_CAM = 4
CHUNK = 2                                # e2e_chunk inside the walk: a host YUYV plain call of 4 frames runs as 2 chunks
PLAIN = -1                               # the plain stream's camera id
FMTS = ("bgr", "yuyv", "nv12")

CTX_SIZES = [None, (W, H), (240, 180), (400, 300), (240, 171)]        # equal, smaller, larger, odd height
OWN_SIZES = [None, (160, 120), (352, 264), (200, 151), (W, H)]
RECTS = [(3, 5, W - 7, H - 9), (W // 4, H // 4, W // 2, H // 2), (1, 2, W // 2 - 1, H // 2 + 1), (0, 0, W, H)]
BAD_RECTS = [(0, 0, W + 1, H), (-1, 0, 10, 10), (5, 5, 0, 10)]
# live images: (fmt, w, h, pitch, uv_offset); up, down, exact 2x (INTER_AREA), padded pitches, NV12 surfaces
LIVES = [("bgr", 401, 263, None, None), ("bgr", 2 * W, 2 * H, None, None), ("bgr", 161, 121, 161 * 3 + 13, None),
         ("nv12", 480, 270, 512, 512 * 270 + 64), ("nv12", 200, 150, None, None)]
GREEN = np.zeros((H, W, 3), np.uint8)
GREEN[..., 1] = 255


def blur_class(k):
    return "off" if k == 0 else ("small" if k <= 31 else "large")


# ---------------------------------------------------------------------------------------------------------------------
# images named by their parameters, so that a step is a printable line of Python
# ---------------------------------------------------------------------------------------------------------------------
def still(seed, w, h):
    return live_bgr(w, h, seed)


def ring(seed, count, w, h):
    return np.stack([live_bgr(w, h, seed + i) for i in range(count)])


class LiveBuf:
    """a live background of `count` images `stride` bytes apart (stride 0: one image) in the layout of LIVES[which]"""

    def __init__(self, which, seed, per_frame):
        fmt, w, h, pitch, uv = LIVES[which]
        self.fmt, self.size, self.per_frame = fmt, (w, h), per_frame
        count = MB if per_frame else 1
        if fmt == "nv12":
            self.imgs = [live_nv12(w, h, seed + i) for i in range(count)]
            self.pitch = w if pitch is None else pitch
            self.uv = self.pitch * h if uv is None else uv
            bufs = [padded_nv12(im, self.pitch, self.uv) for im in self.imgs]
        else:
            self.imgs = [live_bgr(w, h, seed + i) for i in range(count)]
            self.pitch, self.uv = (w * 3 if pitch is None else pitch), 0
            bufs = [padded_bgr(im, self.pitch).reshape(-1) for im in self.imgs]
        one = bufs[0].size
        self.stride = one + 96 if per_frame else 0
        self.host = np.full(max(1, count) * (one + 96), 0x3C, np.uint8)
        for i, b in enumerate(bufs):
            self.host[i * (one + 96): i * (one + 96) + one] = b

    def image(self, b):
        return self.imgs[b if self.per_frame else 0]


# ---------------------------------------------------------------------------------------------------------------------
# camera frames and their logits
# ---------------------------------------------------------------------------------------------------------------------
class Cameras:
    """FRAMES_PER_CAM frames per camera and input format, the BGR the fused path reads of each, and the oracle's logits"""

    def __init__(self):
        self.g = geo(KEY, W, H)
        self._frames, self._logits = {}, {}
        self._cnn = None
        sp = probe_spacing(self.g, 64)
        self.feeds = np.concatenate([random_masks(self.g, 8, 5), step_masks(self.g)[::13], probes(self.g, 255, 0, sp)[::17],
                                     probes(self.g, 0, 255, sp)[::19]])

    def frame(self, cam, i, fmt):
        key = (cam, i, fmt)
        if key not in self._frames:
            yv = synth.yuyv_frame(W, H, t=3 * i, stream=cam + 1)
            if fmt == "yuyv":
                raw, bgr = yv, po.yuyv_to_bgr(yv)
            elif fmt == "nv12":
                raw = np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)
                bgr = nv12_to_bgr(raw)
            else:
                raw = bgr = np.ascontiguousarray(po.yuyv_to_bgr(yv)[:, ::-1])      # another picture than the YUYV one
            self._frames[key] = (raw, bgr)
        return self._frames[key]

    def logits(self, cam, i, fmt):
        key = (cam, i, fmt)
        if key not in self._logits:
            if self._cnn is None:
                self._cnn = po.MaskGen(model_path(KEY), W, H)
            self._cnn.process(self.frame(cam, i, fmt)[1])
            self._logits[key] = self._cnn.output_f32
        return self._logits[key]


# ---------------------------------------------------------------------------------------------------------------------
# the reference model of one context
# ---------------------------------------------------------------------------------------------------------------------
class Refused(Exception):
    pass


def _need(cond, msg):
    if not cond:
        raise Refused(msg)


class Src:
    def __init__(self):
        self.fx, self.k, self.flip, self.size, self.filter, self.interval = "default", -1, -1, None, -1, -1
        self.own = None            # [images, advance, cursor]
        self.live = None


class Ref:
    """The host-visible state of one context (include/backscrub_b200.h, DESIGN.md section 4): the settings, each source's
    settings with their follow values, and per camera (PLAIN, each source) the smoother, the frame counter, the framing
    state and the ring cursor.  Setters validate and apply; `call` returns every frame's expected outputs and advances the
    state, or raises Refused with the message the library gives.  With compute=False only the state and the frame tags
    are tracked (no oracle work): what the coverage test reads."""

    def __init__(self, cams, compute=True):
        self.cams, self.compute = cams, compute
        self.bg = None                   # None, or [images, advance, cursor] (a still image: one image at advance 0)
        self.k, self.flip, self.size, self.filter, self.interval, self.bgra = 0, 0, None, True, 1, False
        self.live = None
        self.srcs = []
        self.fr = FramingRef(SimpleNamespace(W=W, H=H, roi=list(cams.g.roi), out=list(cams.g.out)))
        self.plain_frames = 0
        self.smoother, self.frames = {}, {}
        self.reset_cam(PLAIN)

    # -- state helpers
    def reset_cam(self, cam):
        if self.compute:
            old = self.smoother.pop(cam, None)
            if old is not None:
                old.close()
            self.smoother[cam] = po.MaskGen(model_path(KEY), W, H)
        self.frames[cam] = 0
        self.fr.reset(cam if cam != PLAIN else None)

    def snapshot(self):
        """the comparable state (refused steps must leave it as it was)"""
        def r(x):
            return None if x is None else (id(x[0]), x[1], x[2])
        srcs = tuple((s.fx, s.k, s.flip, s.size, s.filter, s.interval, r(s.own), id(s.live)) for s in self.srcs)
        return (r(self.bg), self.k, self.flip, self.size, self.filter, self.interval, self.bgra, id(self.live), srcs,
                self.plain_frames, tuple(sorted(self.frames.items())), self.fr.mode, self.fr.rect, self.fr.prm,
                tuple(sorted(((k, tuple(v)) for k, v in self.fr.state.items()), key=str)), tuple(sorted(self.fr.jump.items(), key=str)),
                tuple(sorted(self.fr.src.items(), key=str)))

    def _src(self, s):
        _need(self.srcs, "no sources: call bsb_set_sources first")
        _need(0 <= s < len(self.srcs), "source id out of range")
        return self.srcs[s]

    def out_size(self, cam):
        if cam != PLAIN and self.srcs[cam].size is not None:
            return self.srcs[cam].size
        return self.size or (W, H)

    def new_context(self):
        for sm in self.smoother.values():
            sm.close()
        self.__init__(self.cams, self.compute)

    # -- context setters
    def set_background(self, img):
        self.bg = [img[None], 0, 0]

    def set_background_ring(self, imgs, advance):
        self.bg = [imgs, advance, 0]

    def set_background_cursor(self, i):
        _need(0 <= i < (len(self.bg[0]) if self.bg else 1), "background index out of range")     # green counts as one image
        if self.bg:
            self.bg[2] = i

    def set_bgblur(self, k):
        _need(k == 0 or (k % 2 == 1 and 1 <= k <= 255), "strength value must be odd")
        self.k = k

    def set_output(self, flip, size):
        self.flip, self.size = flip, size

    def set_filter(self, active):
        self.filter = active

    def set_mask_interval(self, k):
        _need(1 <= k <= 256, "mask interval out of range")
        self.interval = k

    def set_framing(self, mode, rect):
        if mode == RECT:
            x, y, w, h = rect
            _need(x >= 0 and y >= 0 and w >= 1 and h >= 1 and x + w <= W and y + h <= H, "framing rectangle must lie inside")
        self.fr.mode, self.fr.rect = mode, rect

    def set_framing_auto(self, zoom, margin, speed):
        _need(100 <= zoom <= 1000, "max_zoom_pct out of range")
        _need(0 <= margin <= 100, "margin_pct out of range")
        _need(1 <= speed <= 256, "speed out of range")
        self.fr.prm = (zoom, margin, speed)

    def set_out_format(self, fmt):
        self.bgra = fmt == "bgra"

    def set_live_background(self, lv):
        self.live = lv

    def reset_state(self):
        self.plain_frames = 0
        self.reset_cam(PLAIN)

    # -- sources setters
    def set_sources(self, n):
        for s in range(len(self.srcs)):
            self.fr.src.pop(s, None)
            self.fr.state.pop(s, None)
        self.srcs = [Src() for _ in range(n)]
        for s in range(n):
            self.reset_cam(s)

    def reset_source(self, s):
        self._src(s)
        self.reset_cam(s)

    def set_source_background(self, s, img):
        self._src(s).own = None if img is None else [img[None], 0, 0]

    def set_source_background_ring(self, s, imgs, advance):
        self._src(s).own = [imgs, advance, 0]

    def set_source_background_cursor(self, s, i):
        src = self._src(s)
        _need(src.own is not None, "the source has no background of its own")
        _need(0 <= i < len(src.own[0]), "background index out of range")
        src.own[2] = i

    def set_source_effect(self, s, fx, k):
        src = self._src(s)
        _need(k == -1 or k == 0 or (k % 2 == 1 and 1 <= k <= 255), "source strength must be")
        src.fx, src.k = fx, k

    def set_source_flip(self, s, flip):
        self._src(s).flip = flip

    def set_source_output(self, s, size):
        self._src(s).size = size

    def set_source_filter(self, s, active):
        self._src(s).filter = active

    def set_source_mask_interval(self, s, k):
        src = self._src(s)
        _need(k == -1 or 1 <= k <= 256, "source mask interval out of range")
        src.interval = k

    def set_source_framing(self, s, mode, rect):
        self._src(s)
        if mode == RECT:
            x, y, w, h = rect
            _need(x >= 0 and y >= 0 and w >= 1 and h >= 1 and x + w <= W and y + h <= H, "framing rectangle must lie inside")
        if mode is None:
            self.fr.src.pop(s, None)
        else:
            self.fr.src[s] = (mode, rect)

    def set_source_live_background(self, s, lv):
        self._src(s).live = lv

    # -- a call
    def _background(self, cam, b, bgr):
        """(kind, strength, image or None when not computing) of frame b from camera cam"""
        if cam == PLAIN:
            k = self.k
            if self.live is not None:
                return "live", k, self.compute and expected_bg(self.live.fmt, self.live.image(b), W, H, k)
            if self.bg is not None:
                imgs, adv, cur = self.bg
                img = imgs[(cur + b * adv) % len(imgs)]
                return ("ring" if len(imgs) > 1 else "still"), k, self.compute and _blur(po.resize_linear_u8(img, W, H), k)
            return ("camblur", k, self.compute and po.gaussian_blur(bgr, k)) if k else ("none", 0, GREEN)
        src = self.srcs[cam]
        k = self.k if src.k < 0 else src.k
        if src.fx == "none":
            return ("camblur", k, self.compute and po.gaussian_blur(bgr, k)) if k else ("none", 0, GREEN)
        if src.live is not None:
            return "live", k, self.compute and expected_bg(src.live.fmt, src.live.image(0), W, H, k)
        if src.own is not None:
            imgs, _, cur = src.own
            return ("ring" if len(imgs) > 1 else "still"), k, self.compute and _blur(po.resize_linear_u8(imgs[cur], W, H), k)
        if self.bg is not None:
            return "still", k, self.compute and _blur(po.resize_linear_u8(self.bg[0][0], W, H), k)
        return ("camblur", k, self.compute and po.gaussian_blur(bgr, k)) if k else ("none", 0, GREEN)

    def call(self, c):
        """c: a Call step.  Returns [per frame: dict(tags, and with compute: out, video, mask, ofinal, crop)]"""
        n, ids, want = c.n, c.ids, c.want
        sources = ids is not None
        _need(1 <= n <= MB, "n_frames out of range")
        if c.fmt == "yuyv" and not c.dev and not sources and n >= 2 * CHUNK and c.feed is not None:
            raise Refused("split into chunks")
        cams = list(ids) if sources else [PLAIN] * n
        video = want[1]
        if sources:
            _need(self.srcs, "no sources: call bsb_set_sources first")
            if c.fmt == "nv12" and video:
                _need(not (self.out_size(PLAIN)[0] & 1 or self.out_size(PLAIN)[1] & 1), "NV12 output needs an even output width")
            _need(self.bg is None or len(self.bg[0]) == 1, "sources calls need a still context background")
            for b, s in enumerate(ids):
                _need(0 <= s < len(self.srcs), "source id out of range")
                _need(s not in ids[:b], "source ids must be distinct")
            for s in ids:
                w, h = self.out_size(s)
                if video and c.fmt == "nv12" and self.srcs[s].size is not None:
                    _need(not (w & 1 or h & 1), "NV12 output needs an even output width")
        elif c.fmt == "nv12" and video:
            w, h = self.out_size(PLAIN)
            _need(not (w & 1 or h & 1), "NV12 output needs an even output width")
        res = []
        fed = c.feed is not None
        for b, cam in enumerate(cams):
            raw_i = c.frames[b]
            bgr = self.cams.frame(cam, raw_i, c.fmt)[1] if self.compute else None
            if sources:
                src = self.srcs[cam]
                active = self.filter if src.filter < 0 else bool(src.filter)
                flip = self.flip if src.flip < 0 else src.flip
                k_i = self.interval if src.interval < 0 else src.interval
                f = self.frames[cam]
                seg = f == 0 or (f + cam) % k_i == 0
            else:
                active, flip = self.filter, self.flip
                seg = (self.plain_frames + b) % self.interval == 0
            seg = seg or fed
            size = self.out_size(cam)
            kind, k, bg = self._background(cam, b, bgr)
            fmode = self.fr.eff(None if cam == PLAIN else cam)[0]
            tags = dict(kind="sources" if sources else "plain", fmt=c.fmt, out="bgra" if self.bgra else "bgr", bg=kind, blur=blur_class(k),
                        flip=flip != 0, resized=tuple(size) != (W, H), filter_off=not active, held=not seg, framing=MODES[fmode],
                        fed=fed)
            r = dict(tags=tags)
            if self.compute:
                if fed:
                    ofinal = self.cams.feeds[c.feed[b] % len(self.cams.feeds)]
                elif seg:
                    sm = self.smoother[cam]
                    sm.post_from_output(self.cams.logits(cam, raw_i, c.fmt))
                    ofinal = sm.ofinal
                else:
                    ofinal = self.smoother[cam].ofinal
                mask = ref_mask(self.cams.g, ofinal)
                crop = self.fr.frame(None if cam == PLAIN else cam, ofinal, *size)
                comp = po.alpha_blend(bg, bgr, mask) if active else bgr
                out_bgr = framed_ref(comp, crop, flip, size)
                out = framed_ref(expect_bgra(bgr, mask, active), crop, flip, size) if self.bgra else out_bgr
                r.update(out=out, video=video and video_ref(out_bgr, c.fmt == "nv12"), mask=mask, ofinal=ofinal, crop=crop)
            else:
                self.fr.jump[None if cam == PLAIN else cam] = fmode != AUTO
            res.append(r)
        # after an enqueued call: cursors move, frame counters count (fed calls count nothing)
        if sources:
            for s in ids:
                own = self.srcs[s].own
                if own is not None:
                    own[2] = (own[2] + own[1]) % len(own[0])
                if not fed:
                    self.frames[s] += 1
        else:
            if self.bg is not None:
                self.bg[2] = (self.bg[2] + n * self.bg[1]) % len(self.bg[0])
            if not fed:
                self.plain_frames += n
        return res


def _blur(img, k):
    return po.gaussian_blur(img, k) if k else img


# ---------------------------------------------------------------------------------------------------------------------
# the walk
# ---------------------------------------------------------------------------------------------------------------------
class Set:
    """a setter step: MaskGen method `op` with arguments; image arguments are named by their maker and parameters"""

    def __init__(self, op, *args):
        self.op, self.args = op, args

    def __repr__(self):
        return f"Set({self.op!r}{''.join(', ' + repr(a) for a in self.args)})"


class Call:
    """a call step: plain (ids None) or sources, an input format, host or device entry point, the outputs wanted (out,
    video, mask), the frame of each camera's pool, and the fed masks (indices into Cameras.feeds) or None"""

    def __init__(self, fmt, dev, want, frames, ids=None, feed=None, expect=None):
        self.fmt, self.dev, self.want, self.frames, self.ids, self.feed = fmt, dev, tuple(want), list(frames), ids, feed
        self.n = len(self.frames)
        self.expect = expect        # on a graph context: "replay" (of the graph the step `expect` steps back captured) or "capture"

    def __repr__(self):
        return (f"Call({self.fmt!r}, dev={self.dev}, want={self.want}, frames={self.frames}, ids={self.ids}, "
                f"feed={self.feed}, expect={self.expect!r})")

    def signature(self):
        return ("sources" if self.ids is not None else "plain", self.fmt, self.dev, self.want, self.n)


# argument makers (named in the printed steps)
IMG = ("still", "ring", "live")


def _materialize(a):
    if isinstance(a, tuple) and a and a[0] in IMG:
        if a[0] == "still":
            return still(*a[1:])
        if a[0] == "ring":
            return ring(*a[1:])
        return LiveBuf(*a[1:])
    return a


WANTS = [w for w in itertools.product((True, False), repeat=3) if any(w)]
STRENGTHS = [0, 0, 0, 3, 7, 15, 31, 33, 45]
EPISODE = 50                             # steps per context


def walk(seed, n_steps, toggles=0, tail=0):
    """the steps of walk `seed`: n_steps drawn steps, then `toggles` toggle blocks (toggle_block), then `tail` calls that
    cycle through call signatures with no setter (more distinct graph keys than the graph cache holds)"""
    rng = np.random.default_rng(seed)
    out = []
    n_src = 0
    pick = lambda seq: seq[int(rng.integers(len(seq)))]

    def src_id():
        return int(rng.integers(n_src + 1)) if rng.random() < 0.06 else int(rng.integers(n_src))     # sometimes out of range

    def call():
        sources = rng.random() < 0.5
        fmt = pick(FMTS)
        dev = (fmt != "bgr") if sources else bool(rng.random() < 0.5)      # sources: BGR on host buffers, YUYV / NV12 on the device
        n = int(rng.integers(1, MB + 1))
        if sources:
            n = min(n, n_src)
            ids = [int(s) for s in rng.permutation(n_src)[:n]]
            if rng.random() < 0.03:
                ids[-1] = ids[0] if n > 1 else n_src       # refused: a repeated or out-of-range id
        else:
            ids = None
        feed = [int(i) for i in rng.integers(0, 10_000, n)] if rng.random() < 0.33 else None
        frames = [int(i) for i in rng.integers(0, FRAMES_PER_CAM, n)]
        return Call(fmt, dev, pick(WANTS), frames, ids, feed)

    ctx_setters = {
        "set_background": 3, "set_background_ring": 3, "set_background_cursor": 1, "set_bgblur": 4, "set_output": 4,
        "set_filter": 4, "set_mask_interval": 3, "set_framing": 5, "set_framing_auto": 1, "set_out_format": 2,
        "set_live_background": 3, "reset_state": 1}
    src_setters = {
        "set_sources": 1, "reset_source": 1, "set_source_background": 2, "set_source_background_ring": 2,
        "set_source_background_cursor": 1, "set_source_effect": 3, "set_source_flip": 2, "set_source_output": 2,
        "set_source_filter": 3, "set_source_mask_interval": 2, "set_source_framing": 2, "set_source_live_background": 2}
    names = list(ctx_setters) + list(src_setters)
    weights = np.array([ctx_setters.get(k, 0) + src_setters.get(k, 0) for k in names], float)
    weights /= weights.sum()
    no_bg = False
    while len(out) < n_steps:
        if len(out) % EPISODE == 0:
            # a new context: the plain background cannot be cleared, so some episodes never set one
            out.append(Set("new_context"))
            n_src, no_bg = pick(N_SRC_CHOICES), bool(rng.random() < 0.5)
            out.append(Set("set_sources", n_src))
            continue
        if rng.random() < 0.55:
            out.append(call())
            continue
        op = names[int(rng.choice(len(names), p=weights))]
        if len(out) % 7 == 0:
            op = pick(["set_out_format", "set_filter", "set_framing", "set_bgblur", "set_live_background", "set_background_ring"])
        if no_bg and op in ("set_background", "set_background_ring"):
            op = "set_bgblur"
        if op == "set_live_background" and rng.random() < 0.5:
            out.append(Set(op, None))                       # the context image or ring shows again
            continue
        bad = rng.random() < 0.08
        seed_img = int(rng.integers(1, 1000))
        if op == "set_background":
            out.append(Set(op, ("still", seed_img, pick([200, 336, 500]), pick([150, 250, 321]))))
        elif op == "set_background_ring":
            count = pick([1, 3])
            out.append(Set(op, ("ring", seed_img, count, 180, 120), int(rng.integers(0, 3))))
        elif op == "set_background_cursor":
            out.append(Set(op, int(rng.integers(0, 4 if bad else 3))))
        elif op == "set_bgblur":
            out.append(Set(op, pick([2, 8]) if bad else pick(STRENGTHS)))
        elif op == "set_output":
            out.append(Set(op, pick([0, 0, 0, 1, 2, 3]), pick(CTX_SIZES)))
        elif op == "set_filter":
            out.append(Set(op, bool(rng.random() < 0.5)))
        elif op == "set_mask_interval":
            out.append(Set(op, pick([0, 257]) if bad else pick([1, 1, 2, 3])))
        elif op == "set_framing":
            mode = pick([OFF, RECT, RECT, AUTO])
            out.append(Set(op, RECT if bad else mode, pick(BAD_RECTS) if bad else (pick(RECTS) if mode == RECT else None)))
        elif op == "set_framing_auto":
            out.append(Set(op, 99 if bad else pick([150, 300, 1000]), pick([0, 10, 40]), pick([1, 37, 256])))
        elif op == "set_out_format":
            out.append(Set(op, pick(["bgr", "bgra"])))
        elif op == "set_live_background":
            out.append(Set(op, None if rng.random() < 0.3 else ("live", int(rng.integers(len(LIVES))), seed_img, bool(rng.random() < 0.5))))
        elif op == "reset_state":
            out.append(Set(op))
        elif op == "set_sources":
            n_src = pick(N_SRC_CHOICES)
            out.append(Set(op, n_src))
        elif op == "reset_source":
            out.append(Set(op, src_id()))
        elif op == "set_source_background":
            out.append(Set(op, src_id(), None if rng.random() < 0.3 else ("still", seed_img, 250, 170)))
        elif op == "set_source_background_ring":
            out.append(Set(op, src_id(), ("ring", seed_img, pick([1, 3]), 170, 130), int(rng.integers(0, 3))))
        elif op == "set_source_background_cursor":
            out.append(Set(op, src_id(), int(rng.integers(0, 3))))
        elif op == "set_source_effect":
            out.append(Set(op, src_id(), pick(["default", "default", "none"]), 4 if bad else pick([-1, -1] + STRENGTHS)))
        elif op == "set_source_flip":
            out.append(Set(op, src_id(), int(rng.integers(-1, 4))))
        elif op == "set_source_output":
            out.append(Set(op, src_id(), pick(OWN_SIZES)))
        elif op == "set_source_filter":
            out.append(Set(op, src_id(), int(rng.integers(-1, 2))))
        elif op == "set_source_mask_interval":
            out.append(Set(op, src_id(), 0 if bad else pick([-1, 1, 2, 3])))
        elif op == "set_source_framing":
            mode = pick([None, OFF, RECT, AUTO])
            out.append(Set(op, src_id(), RECT if bad else mode, pick(BAD_RECTS) if bad else (pick(RECTS) if mode == RECT else None)))
        elif op == "set_source_live_background":
            out.append(Set(op, src_id(), None if rng.random() < 0.3 else ("live", int(rng.integers(len(LIVES))), seed_img, False)))
    trng = np.random.default_rng([seed, 1])             # the drawn steps do not depend on `toggles` or `tail`
    out += sweep(np.random.default_rng([seed, 2]))
    n_src = SWEEP_SOURCES
    for i in range(toggles):
        out += toggle_block(trng, TOGGLES[i % len(TOGGLES)], n_src)
    if tail:
        # every plain signature, CNN frames: more distinct graph keys than the cache's 64
        out += [Set("set_mask_interval", 1), Set("set_output", 0, None)]    # every tail call segments, none is refused
        sigs = [(fmt, dev, want, n) for n in range(1, MB + 1) for fmt in FMTS for dev in (True, False) for want in WANTS[:4]]
        order = trng.permutation(len(sigs))
        first = None
        for i in range(tail // 2):
            fmt, dev, want, n = sigs[order[i % len(sigs)]]
            c = Call(fmt, dev, want, [int(x) for x in trng.integers(0, FRAMES_PER_CAM, n)])
            split = fmt == "yuyv" and not dev and n >= 2 * CHUNK
            # the second replays the first, unless it is split into chunks: two graphs, and the cache may overflow between them
            out += [c, Call(fmt, dev, want, c.frames, expect=None if split else 1)]
            first = first or c
        # the cache overflowed and dropped every graph since: the first signature of the tail is captured again
        out.append(Call(first.fmt, first.dev, first.want, first.frames, expect="capture"))
    return out


SWEEP_SOURCES = 4


def sweep(rng):
    """one call for each (call kind, input format, out format) x (background kind, blur class) on a new context, every
    other setting drawn at random: the compound pairs a random walk of this length reaches only in part.  Plain calls
    without an image come before the first set_background (a context image cannot be cleared), sources calls before the
    plain ring (a ring of several images refuses sources calls)."""
    pick = lambda seq: seq[int(rng.integers(len(seq)))]
    n_src = SWEEP_SOURCES
    out = [Set("new_context"), Set("set_sources", n_src)]
    blurs = {"off": [0], "small": [3, 7, 15, 31], "large": [33, 45]}
    combos = []
    for kind, bgs in (("plain", ("camblur", "none", "live")), ("sources", BGS), ("plain", ("still", "ring"))):
        for bg in bgs:
            for blur in BLURS:
                if not possible(bg=bg, blur=blur):
                    continue
                combos += [(kind, fmt, o, bg, blur) for fmt in FMTS for o in ("bgr", "bgra")]
    seed_img = 500
    for kind, fmt, o, bg, blur in combos:
        seed_img += 1
        k = pick(blurs[blur])
        s = int(rng.integers(n_src))
        out += [Set("set_out_format", o), Set("set_output", pick([0, 0, 1, 2, 3]), pick([None, (240, 180), (400, 300)])),
                Set("set_filter", bool(rng.random() < 0.7)), Set("set_mask_interval", pick([1, 1, 2, 3]))]
        mode = pick([OFF, RECT, AUTO])
        out.append(Set("set_framing", mode, pick(RECTS) if mode == RECT else None))
        live = ("live", int(rng.integers(len(LIVES))), seed_img, bool(rng.random() < 0.5))
        if kind == "plain":
            out.append(Set("set_bgblur", k))
            out.append(Set("set_live_background", live if bg == "live" else None))
            if bg == "still":
                out.append(Set("set_background", ("still", seed_img, 230, 170)))
            elif bg == "ring":
                out.append(Set("set_background_ring", ("ring", seed_img, 3, 180, 120), int(rng.integers(1, 3))))
            n, ids = int(rng.integers(1, MB + 1)), None
        else:
            fx = "none" if bg in ("camblur", "none") else "default"
            out += [Set("set_source_effect", s, fx, k), Set("set_source_live_background", s, live[:3] + (False,) if bg == "live" else None)]
            if bg == "still":
                out.append(Set("set_source_background", s, ("still", seed_img, 230, 170)))
            elif bg == "ring":
                out.append(Set("set_source_background_ring", s, ("ring", seed_img, 3, 170, 130), int(rng.integers(1, 3))))
            elif bg == "live":
                out.append(Set("set_source_background", s, None))
            n = int(rng.integers(1, n_src + 1))
            ids = [s] + [int(x) for x in rng.permutation([i for i in range(n_src) if i != s])[:n - 1]]
        dev = (fmt != "bgr") if ids is not None else bool(rng.random() < 0.5)
        feed = [int(i) for i in rng.integers(0, 10_000, n)] if rng.random() < 0.4 else None
        out.append(Call(fmt, dev, pick(WANTS), [int(x) for x in rng.integers(0, FRAMES_PER_CAM, n)], ids, feed))
    return out


# Toggle blocks: call X runs under value a of one setting, then b, then a, then b, with nothing else in between.  A setting
# that is table data replays X's graph; one the graph key carries selects another graph.  Either way each call must give
# Ref's bytes, so a key field that is missing shows as a replayed graph of the other value.  (setter, a, b); "S" stands
# for a source of the call, "LIVE" for a live image.  The third call replays the first's graph unless b's first use grows
# a buffer (graphs are dropped then: live backgrounds, framing's staging); the fourth always replays the second's.
TOGGLES = [("set_filter", (True,), (False,)), ("set_out_format", ("bgr",), ("bgra",)), ("set_live_background", (None,), ("LIVE",)),
           ("set_framing", (OFF, None), (RECT, RECTS[1])), ("set_framing", (OFF, None), (AUTO, None)), ("set_mask_interval", (1,), (2,)),
           ("set_source_filter", ("S", 1), ("S", 0)), ("set_source_flip", ("S", 0), ("S", 3)),
           ("set_source_framing", ("S", OFF, None), ("S", RECT, RECTS[2])), ("set_source_mask_interval", ("S", 1), ("S", 2)),
           ("set_source_live_background", ("S", None), ("S", "LIVE")), ("set_source_output", ("S", None), ("S", OWN_SIZES[1]))]
GROWS = {"set_live_background", "set_source_live_background", "set_framing", "set_source_framing", "set_out_format", "set_source_output"}


def toggle_block(rng, toggle, n_src):
    op, a, b = toggle
    sources = op.startswith("set_source")
    s = int(rng.integers(n_src))
    seed_img = int(rng.integers(1, 1000))
    sub = lambda v: tuple(s if x == "S" else (("live", int(rng.integers(len(LIVES))), seed_img, False) if x == "LIVE" else x)
                          for x in v)
    a, b = sub(a), sub(b)
    # a context where every setting of the toggle shows: a still background, the filter on, BGR, unframed, every frame
    # segmented, no live image; the source following the context; then a graph drop, so the cache holds this block only
    out = [Set("set_background", ("still", seed_img, 200, 150)), Set("set_output", 0, None), Set("set_filter", True),
           Set("set_out_format", "bgr"),
           Set("set_framing", OFF, None), Set("set_mask_interval", 1), Set("set_live_background", None)]
    if sources:
        out += [Set("set_source_filter", s, -1), Set("set_source_flip", s, -1), Set("set_source_framing", s, None, None),
                Set("set_source_mask_interval", s, -1), Set("set_source_live_background", s, None),
                Set("set_source_effect", s, "default", -1), Set("set_source_background", s, None), Set("set_source_output", s, None)]
    out.append(Set("set_framing_auto", 300, 10, 32))
    frames = [int(i) for i in rng.integers(0, FRAMES_PER_CAM, MB)]
    if sources:
        n = min(MB, n_src)
        ids = [s] + [int(x) for x in rng.permutation([i for i in range(n_src) if i != s])[:n - 1]]
        x = dict(fmt="yuyv", dev=True, want=(True, True, True), frames=frames[:n], ids=ids)
    else:
        x = dict(fmt=("bgr", "yuyv", "nv12")[int(rng.integers(3))], dev=True, want=(True, True, True), frames=frames)
    for k, v in enumerate((a, b, a, b)):
        out.append(Set(op, *v))
        expect = 4 if k == 3 or (k == 2 and op not in GROWS) else None
        out.append(Call(**x, expect=expect))
    return out


def walk_prefix(seed, k, n_steps=None, tail=0):
    """the first k steps of walk(seed, ...): a failing step and what led to it"""
    return walk(seed, n_steps or DEFAULT_STEPS, tail)[:k]



def script(steps):
    return "\n".join(f"{i:4d}  {s!r}" for i, s in enumerate(steps))


DEFAULT_STEPS, WALK_SEED = 800, 8            # the default walk: every pair covered (test_walk_covers_every_pair)


# ---------------------------------------------------------------------------------------------------------------------
# running a walk on a library
# ---------------------------------------------------------------------------------------------------------------------
class HostMem:
    """the emulator's device memory: host buffers"""

    def __init__(self):
        self.bufs = {}

    def buf(self, key, nbytes):
        k = (key, nbytes)
        if k not in self.bufs:
            self.bufs[k] = np.zeros(nbytes, np.uint8)
        return self.bufs[k]

    def put(self, key, arr):
        b = self.buf(key, arr.nbytes)
        b[:] = arr.reshape(-1)
        return b

    @staticmethod
    def ptr(b):
        return b.ctypes.data

    @staticmethod
    def get(b):
        return b.copy()

    def hold(self, arr):
        return arr


class CudaMem(HostMem):
    """device buffers (torch), one per role and size, so a repeated call signature meets the same pointers"""

    def __init__(self):
        import torch
        self.torch = torch
        super().__init__()

    def buf(self, key, nbytes):
        k = (key, nbytes)
        if k not in self.bufs:
            self.bufs[k] = self.torch.zeros(nbytes, dtype=self.torch.uint8, device="cuda")
        return self.bufs[k]

    def put(self, key, arr):
        b = self.buf(key, arr.nbytes)
        b.copy_(self.torch.from_numpy(np.ascontiguousarray(arr).reshape(-1)))
        return b

    @staticmethod
    def ptr(b):
        return b.data_ptr()

    @staticmethod
    def get(b):
        return b.cpu().numpy()

    def hold(self, arr):
        return self.torch.from_numpy(arr).cuda()


class Runner:
    """one library context driven by the walk's steps"""

    def __init__(self, lib, mem, name, flags=0):
        self.lib, self.mem, self.name, self.flags = lib, mem, name, flags
        self.g = api.MaskGen(lib, model_path(KEY), W, H, max_batch=MB, flags=flags)
        self.held = {}

    def close(self):
        self.g.close()

    def setter(self, st):
        args = [_materialize(a) for a in st.args]
        if st.op == "new_context":
            self.g.close()
            self.g = api.MaskGen(self.lib, model_path(KEY), W, H, max_batch=MB, flags=self.flags)
            self.held = {}
            return None
        g = self.g
        if st.op == "set_output":
            return g.set_output(bool(args[0] & 1), bool(args[0] & 2), args[1])
        if st.op == "set_framing":
            return g.set_framing(MODES[args[0]], args[1])
        if st.op == "set_source_framing":
            return g.set_source_framing(args[0], None if args[1] is None else MODES[args[1]], args[2])
        if st.op == "set_source_flip":
            return g.set_source_flip(args[0], *((None, None) if args[1] < 0 else (bool(args[1] & 1), bool(args[1] & 2))))
        if st.op == "set_source_filter":
            return g.set_source_filter(args[0], None if args[1] < 0 else bool(args[1]))
        if st.op == "set_source_mask_interval":
            return g.set_source_mask_interval(args[0], None if args[1] < 0 else args[1])
        if st.op == "set_live_background":
            lv = args[0]
            if lv is None:
                return g.set_live_background(None)
            d = self.mem.hold(lv.host)
            self.held[None] = d
            return g.set_live_background(d if hasattr(d, "data_ptr") else d.ctypes.data, lv.fmt, lv.size, lv.pitch, lv.uv, lv.stride)
        if st.op == "set_source_live_background":
            s, lv = args
            if lv is None:
                return g.set_source_live_background(s, None)
            d = self.mem.hold(lv.host)
            self.held[s] = d
            return g.set_source_live_background(s, d if hasattr(d, "data_ptr") else d.ctypes.data, lv.fmt, lv.size, lv.pitch, lv.uv)
        return getattr(g, st.op)(*args)

    def call(self, c, cams):
        """-> per frame (out, video, mask, ofinal or None) as flat arrays"""
        g, n, m = self.g, c.n, self.mem
        raws = np.stack([cams.frame(PLAIN if c.ids is None else c.ids[b], c.frames[b], c.fmt)[0] for b in range(n)])
        if c.feed is not None:
            g.feed(B.FEED_MASK, cams.feeds[[i % len(cams.feeds) for i in c.feed]])
        wo, wv, wm = c.want
        oc, nv12 = g.out_channels, c.fmt == "nv12"
        sizes = [(g.out_width, g.out_height)] * n
        if c.ids is not None and g._n_sources:
            sizes = [g._src_out.get(s, (g.out_width, g.out_height)) for s in c.ids]
        vbytes = (lambda w, h: w * h * 3 // 2) if nv12 else (lambda w, h: w * h * 2)
        if not c.dev:
            if c.ids is not None:
                out, vid, mask = g.composite_sources(raws, c.ids, wo, wv, wm)
            elif c.fmt == "bgr":
                out, vid, mask = g.composite(raws, wo, wv, wm)
            elif c.fmt == "nv12":
                out, vid, mask = g.composite_nv12(raws, wo, wv, wm)
            else:
                ow, oh = g.out_width, g.out_height
                out = np.empty((n, oh, ow, oc), np.uint8) if wo else None
                vid = np.empty((n, oh, ow, 2), np.uint8) if wv else None
                mask = np.empty((n, H, W), np.uint8) if wm else None
                g.composite_yuyv_into(raws, out, vid, mask)
            per = lambda a, b: None if a is None else np.asarray(a[b]).reshape(-1)
            res = [(per(out, b), per(vid, b), per(mask, b)) for b in range(n)]
        else:
            # one buffer per role and frame count, frames OUT_STEP / VIDEO_STEP bytes apart whatever the format and sizes:
            # a BGR and a BGRA call, or calls before and after a size change, meet the same pointers and strides
            ostep, vstep = OUT_STEP, VIDEO_STEP
            d_in = m.put((self.name, "in", c.fmt, n), raws)
            d_out = m.buf((self.name, "out", n), n * ostep) if wo else None
            d_vid = m.buf((self.name, "vid", n), n * vstep) if wv else None
            d_mask = m.buf((self.name, "mask", n), n * W * H) if wm else None
            p = lambda b: m.ptr(b) if b is not None else None
            L, h = g._lib, g._h
            if c.ids is not None:
                fn = g.composite_sources_nv12_device if nv12 else g.composite_sources_yuyv_device
                kw = dict(out_stride=ostep, **({"nv12_stride": vstep} if nv12 else {"yuyv_stride": vstep}))
                fn(n, c.ids, p(d_in) or 0, p(d_out) or 0, p(d_vid) or 0, p(d_mask) or 0, sync=True, **kw)
            else:
                if c.fmt == "bgr":
                    ok = L.bsb_composite_device(h, n, p(d_in), W * H * 3, p(d_out), ostep, p(d_vid), vstep, p(d_mask), W * H, 1)
                elif c.fmt == "yuyv":
                    ok = L.bsb_composite_yuyv_device(h, n, p(d_in), p(d_out), ostep, p(d_vid), vstep, p(d_mask), W * H, 1)
                else:
                    ok = L.bsb_composite_nv12_device(h, n, p(d_in), W, W * H, W * H * 3 // 2, p(d_out), ostep, p(d_vid), vstep,
                                                     p(d_mask), W * H, 1)
                if not ok:
                    g._fail("composite device")
            o = m.get(d_out) if wo else None
            v = m.get(d_vid) if wv else None
            k = m.get(d_mask) if wm else None
            res = []
            for b, (w, h) in enumerate(sizes):
                res.append((None if o is None else o[b * ostep: b * ostep + w * h * oc],
                            None if v is None else v[b * vstep: b * vstep + vbytes(w, h)],
                            None if k is None else k[b * W * H: (b + 1) * W * H]))
        split = c.ids is None and not c.dev and c.fmt == "yuyv" and n >= 2 * CHUNK
        return [r + ((None if split else g.stage_u8(2, b).reshape(-1)),) for b, r in enumerate(res)]


def _fail(seed, i, steps, what):
    return f"walk seed {seed}, step {i}: {what}\nsteps so far:\n{script(steps[:i + 1])}"


def _compare(seed, i, steps, name, got, want):
    for b, (g, w) in enumerate(zip(got, want)):
        for what, x, ref in (("out", g[0], w["out"]), ("video", g[1], w["video"]), ("mask", g[2], w["mask"]),
                             ("ofinal", g[3], w["ofinal"])):
            if x is None:
                continue
            ref = np.asarray(ref).reshape(-1)
            if x.size != ref.size or not np.array_equal(x, ref):
                diff = int((x != ref).sum()) if x.size == ref.size else f"size {x.size} != {ref.size}"
                raise AssertionError(_fail(seed, i, steps, f"{name}: {what} of frame {b} differs ({diff} bytes), tags {w['tags']}"))


def run_walk(seed, steps, runners, cams, hook=None):
    """every step on every runner; refusals against Ref's, outputs against Ref's.  hook(i, step, ref, want) after each
    step, want None for a refused step.  Returns the per-frame tags."""
    ref = Ref(cams)
    tags = []
    for i, st in enumerate(steps):
        before = ref.snapshot()
        err = None
        try:
            want = ref.call(st) if isinstance(st, Call) else getattr(ref, st.op)(*[_materialize(a) for a in st.args])
        except Refused as e:
            err = str(e)
        got = []
        for r in runners:
            try:
                got.append(r.call(st, cams) if isinstance(st, Call) else r.setter(st))
                if err is not None:
                    raise AssertionError(_fail(seed, i, steps, f"{r.name}: accepted, the reference refuses it ({err})"))
            except api.BackscrubError as e:
                if err is None:
                    raise AssertionError(_fail(seed, i, steps, f"{r.name}: refused ({e}), the reference accepts it"))
                assert err in str(e), _fail(seed, i, steps, f"{r.name}: refused with {e!s}, expected '{err}'")
        if err is not None:
            assert ref.snapshot() == before, _fail(seed, i, steps, "the reference changed on a refused step")
            want = None
        elif isinstance(st, Call):
            for r, gv in zip(runners, got):
                _compare(seed, i, steps, r.name, gv, want)
            tags.extend(w["tags"] for w in want)
        else:
            want = True
        if hook:
            hook(i, st, ref, want)
    return tags


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
BGS, BLURS = ("still", "ring", "live", "camblur", "none"), ("off", "small", "large")
CALLS = [(k, f, o) for k in ("plain", "sources") for f in FMTS for o in ("bgr", "bgra")]
DIMS = ("call", "background", "flip", "resized", "filter_off", "held", "framing", "fed")


def possible(**t):
    """False for a combination no frame can have"""
    if t.get("held") and t.get("fed"):
        return False                                   # a fed call holds no frame
    bg, blur = t.get("background", (t.get("bg"), t.get("blur")))
    return not ((bg == "camblur" and blur == "off") or (bg == "none" and blur in ("small", "large")))


def dim_values():
    """every value of each dimension the walk must reach: call = (kind, input format, out format), background = (kind,
    blur class)"""
    return {"call": CALLS, "background": [(b, c) for b in BGS for c in BLURS if possible(bg=b, blur=c)],
            "flip": [False, True], "resized": [False, True], "filter_off": [False, True], "held": [False, True],
            "framing": ["off", "rect", "auto"], "fed": [False, True]}


def missing_pairs(tags):
    vals = dim_values()
    seen = {(a, b): set() for a, b in itertools.combinations(DIMS, 2)}
    for t in tags:
        t = dict(t, call=(t["kind"], t["fmt"], t["out"]), background=(t["bg"], t["blur"]))
        for a, b in seen:
            seen[(a, b)].add((t[a], t[b]))
    return [(a, va, b, vb) for (a, b), s in seen.items() for va in vals[a] for vb in vals[b]
            if possible(**{a: va, b: vb}) and (va, vb) not in s]


def tag_walk(steps):
    """(frame tags, refused steps) of a walk from the reference alone (no library, no oracle)"""
    ref = Ref(Cameras(), compute=False)
    tags, refused = [], 0
    for st in steps:
        try:
            if isinstance(st, Call):
                tags.extend(r["tags"] for r in ref.call(st))
            else:
                getattr(ref, st.op)(*[_materialize(a) for a in st.args])
        except Refused:
            refused += 1
    return tags, refused


def test_walk_covers_every_pair():
    """the default walk reaches every pair of values of every two dimensions, and refuses one step in twenty or more"""
    steps = walk(WALK_SEED, DEFAULT_STEPS)
    tags, refused = tag_walk(steps)
    miss = missing_pairs(tags)
    assert not miss, f"{len(miss)} pairs never reached, e.g. {miss[:10]}"
    assert refused >= DEFAULT_STEPS // 20, refused


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    L = emu()
    assert L.bsb_set_tuning(b"e2e_chunk", CHUNK)
    yield L
    L.bsb_set_tuning(b"e2e_chunk", 16)


@pytest.fixture(scope="module")
def cams():
    return Cameras()


def test_emu_walk(emu_lib, cams):
    steps = walk(WALK_SEED, DEFAULT_STEPS, len(TOGGLES))
    r = Runner(emu_lib, HostMem(), "emu")
    try:
        run_walk(WALK_SEED, steps, [r], cams)
    finally:
        r.close()


@pytest.mark.slow
@pytest.mark.parametrize("seed", [1])
def test_emu_walk_more_seeds(emu_lib, cams, seed):
    steps = walk(seed, DEFAULT_STEPS)
    r = Runner(emu_lib, HostMem(), "emu")
    try:
        run_walk(seed, steps, [r], cams)
    finally:
        r.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    assert L.bsb_set_tuning(b"e2e_chunk", CHUNK)
    yield L
    L.bsb_set_tuning(b"e2e_chunk", 16)


@pytest.fixture
def tuning(gpu_lib):
    saved = []

    def set_(name, value, default):
        assert gpu_lib.bsb_set_tuning(name.encode(), value)
        saved.append((name, default))
    yield set_
    for name, default in reversed(saved):
        gpu_lib.bsb_set_tuning(name.encode(), default)


# setters after which the library may hold no graph: the ones that always drop the captured graphs (set_bgblur, set_output,
# set_framing_auto, set_sources) and the ones that do when the ring pool changes (a new background or ring of another
# count or advance, a source's ring); a new context starts without graphs
DROPPING = {"new_context", "set_bgblur", "set_output", "set_framing_auto", "set_sources", "set_background", "set_background_ring",
            "set_source_background", "set_source_background_ring"}


def gpu_walk(lib, cams, seed, n_steps, toggles, tail):
    """The walk on a context that captures graphs and on an eager twin (BSB_FLAG_NO_GRAPH) given the same steps.  Every
    call of the graph context is counted in launches (bsb_total_launches): a call marked `expect=k` repeats the call k
    steps back with the same held frames, so it replays that graph and launches nothing; the call marked "capture" comes
    after more distinct graph keys than the cache holds, so its graph was dropped and it launches its kernels again.
    Host-side counts: distinct call signatures between setters that may drop graphs (at least as many graph keys), and
    how many of those setters ran."""
    mem = CudaMem()
    graph, eager = Runner(lib, mem, "graph"), Runner(lib, mem, "eager", flags=B.FLAG_NO_GRAPH)
    steps = walk(seed, n_steps, toggles, tail)
    stats = dict(max_signatures=0, dropping_setters=0, replays=0, recaptures=0)
    keys, held, launches = set(), {}, [0]
    graph_call = graph.call

    def counted(c, cams_):
        l0 = lib.bsb_total_launches()
        try:
            return graph_call(c, cams_)
        finally:
            launches[0] = lib.bsb_total_launches() - l0
    graph.call = counted

    def hook(i, st, ref, want):
        if isinstance(st, Set):
            if want is not None and st.op in DROPPING:
                stats["max_signatures"] = max(stats["max_signatures"], len(keys))
                keys.clear()
                stats["dropping_setters"] += 1
            return
        if want is None or st.feed is not None:            # refused, or fed (eager, never captured)
            return
        held[i] = tuple(w["tags"]["held"] for w in want)
        keys.add((st.signature(), tuple(st.ids or ()), held[i]))
        if st.expect == "capture":
            assert launches[0] > 0, _fail(seed, i, steps, "the graph cache kept a graph past 64 distinct keys")
            stats["recaptures"] += 1
        elif st.expect is not None and held.get(i - st.expect) == held[i]:
            assert launches[0] == 0, _fail(seed, i, steps, f"a repeated call launched {launches[0]} kernels")
            stats["replays"] += 1

    try:
        run_walk(seed, steps, [graph, eager], cams, hook)
    finally:
        graph.close()
        eager.close()
    stats["max_signatures"] = max(stats["max_signatures"], len(keys))
    return stats


GPU_TOGGLES = 3 * len(TOGGLES)
GPU_TAIL = 140                                   # 70 distinct plain call signatures, each twice


@pytest.mark.gpu
@pytest.mark.parametrize("tile,tma,seed", [(0, 1, WALK_SEED), (128, 1, 1), (0, 0, 2)], ids=["default", "tile128", "no_tma"])
def test_gpu_walk(gpu_lib, tuning, cams, tile, tma, seed, capsys):
    """graph vs eager vs Ref on every call; the cache overflows; repeated calls replay.  post_tile 128 and post_tma 0 take
    the walk through the other k_post_tma instantiations and the fallback post kernels."""
    tuning("post_tile", tile, 0)
    tuning("post_tma", tma, 1)
    stats = gpu_walk(gpu_lib, cams, seed, DEFAULT_STEPS, GPU_TOGGLES, GPU_TAIL)
    with capsys.disabled():
        print(f"\nsettings walk seed {seed} post_tile {tile} post_tma {tma}: {stats}")
    assert stats["max_signatures"] > 64 and stats["recaptures"] == 1, stats
    assert stats["replays"] >= GPU_TAIL // 2 + GPU_TOGGLES // 2, stats
