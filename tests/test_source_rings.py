"""Per-source animated backgrounds (bsb_set_source_background_ring / _cursor): each camera of a sources context plays its
own device-resident background ring.  Frame b of a sources call, from source s with its own ring, must give exactly the
bytes a plain batch-1 context gives for that camera's stream, set up with bsb_set_background_ring(same frames, same
advance), bsb_set_bgblur(k_s) and bsb_set_output(flip_s, size_s), with the same cursor moves.

`-m "not gpu"`: the kernel-logic emulator build vs the oracle.  `-m gpu`: the sm_90a library vs plain batch-1 contexts."""

import numpy as np
import pytest

from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_feed_post import geo, random_masks, ref_mask, ref_outputs


def _ring(count, seed, size=None):
    """count distinct decoded images (the bundled background rolled and tinted per image), optionally resized"""
    import cv2
    bg = synth.background()
    if size:
        bg = cv2.resize(bg, size, interpolation=cv2.INTER_LINEAR)
    return np.stack([np.roll(bg, 29 * seed + 53 * i, axis=1) ^ np.uint8((7 * seed + 31 * i) & 0xFF) for i in range(count)])


class _Model:
    """the test's own model of a sources context: context image / strength, and per source its effect, ring and cursor"""

    def __init__(self, n, ctx_bg=None, ctx_k=0):
        self.ctx_bg, self.ctx_k = ctx_bg, ctx_k
        self.ring = {}                                     # s -> [images, advance, cursor]
        self.version = {}                                  # s -> how many times its background was set
        self.fx = {s: ("default", -1) for s in range(n)}

    def setup(self, s):
        """(background image or None, strength) of the plain context that source s must equal for its next frame"""
        kind, k = self.fx[s]
        k = self.ctx_k if k < 0 else k
        if kind == "none":
            return None, k
        if s in self.ring:
            imgs, _, cur = self.ring[s]
            return imgs[cur], k
        return self.ctx_bg, k

    def moved(self, ids):
        """after a call that was enqueued: every ring of a source in it moves on, blended or not"""
        for s in ids:
            if s in self.ring:
                r = self.ring[s]
                r[2] = (r[2] + r[1]) % len(r[0])

    # the context and the model, changed together
    def set_ring(self, g, s, imgs, advance):
        g.set_source_background_ring(s, imgs, advance)
        self.ring[s] = [list(imgs), advance, 0]
        self.version[s] = self.version.get(s, 0) + 1

    def set_still(self, g, s, img):
        g.set_source_background(s, img)
        if img is None:
            self.ring.pop(s, None)
        else:
            self.ring[s] = [[img], 0, 0]
        self.version[s] = self.version.get(s, 0) + 1

    def set_cursor(self, g, s, i):
        g.set_source_background_cursor(s, i)
        self.ring[s][2] = i

    def set_fx(self, g, s, kind="default", k=-1):
        g.set_source_effect(s, kind, k)
        self.fx[s] = (kind, k)


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


class _Oracles:
    """one oracle stream per source (and one for the context's plain calls)"""

    def __init__(self, key, W, H, n):
        self.W, self.H = W, H
        self.o = [po.MaskGen(model_path(key), W, H) for _ in range(n)]
        self.t = [0] * n
        self.plain_o, self.plain_t = po.MaskGen(model_path(key), W, H), 0

    def _ref(self, o, frame, bg, k):
        if bg is None and not k:
            # a plain context without a background blends plain green (app/deepseg.cc:603); the oracle's "no image" is
            # the camera frame itself
            bg = np.zeros((self.H, self.W, 3), np.uint8)
            bg[..., 1] = 255
        return o.composite_ex(frame, bg, bgblur=k)

    def call(self, g, ids, m):
        fr = np.stack([synth.frame(self.W, self.H, t=self.t[s], stream=s) for s in ids])
        out, yuyv, mask = g.composite_sources(fr, ids)
        for b, s in enumerate(ids):
            bg, k = m.setup(s)
            ro, ry, rm = self._ref(self.o[s], fr[b], bg, k)
            tag = (ids, b, s, self.t[s], m.fx[s], k, m.ring[s][2] if s in m.ring else None)
            assert np.array_equal(mask[b], rm), f"mask differs {tag}"
            assert np.array_equal(out[b], ro), f"composite differs {tag}"
            assert np.array_equal(yuyv[b], ry), f"YUYV differs {tag}"
            self.t[s] += 1
        m.moved(ids)

    def plain(self, g, m):
        """a plain call on the same context: the context image at the context's strength, its own smoother state"""
        fr = synth.frame(self.W, self.H, t=self.plain_t, stream=99)
        out, yuyv, mask = g.composite(fr)
        ro, ry, rm = self._ref(self.plain_o, fr, m.ctx_bg, m.ctx_k)
        assert np.array_equal(mask, rm) and np.array_equal(out, ro) and np.array_equal(yuyv, ry), ("plain", self.plain_t)
        self.plain_t += 1


def test_cursors(emu_lib):
    """s0 its own ring of 3 at advance 1, s1 its own ring of 2 at advance 0 paced by the caller, s2 its own still, s3
    the context still; calls of varying subsets and orders, calls without s0 (its cursor stays), s0 wrapping"""
    key, W, H = "meet_lite", 320, 240
    m = _Model(4, ctx_bg=synth.background()[::-1].copy())
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    g.set_background(m.ctx_bg)
    g.set_sources(4)
    m.set_ring(g, 0, _ring(3, 0), 1)
    m.set_ring(g, 1, _ring(2, 1), 0)
    m.set_still(g, 2, _ring(1, 2)[0])
    o = _Oracles(key, W, H, 4)
    o.call(g, [0, 1, 2, 3], m)
    o.call(g, [3, 1], m)                             # no frame of s0: its cursor stays at 1
    m.set_cursor(g, 1, 1)
    o.call(g, [2, 0, 1], m)
    o.call(g, [1, 3], m)
    m.set_cursor(g, 1, 0)
    o.call(g, [0, 1], m)                             # s0 wraps: 2 -> 0
    o.call(g, [0, 2, 3], m)
    assert m.ring[0][2] == 1
    g.reset_source(0)                                # the smoother state only: the cursor stays
    o.o[0] = po.MaskGen(model_path(key), W, H)
    o.call(g, [0], m)
    g.close()


def test_strengths_and_replacement(emu_lib):
    """context strength 7; rings that follow it, that have their own strength 0 and 25.  Then a new context strength, a
    source without an image for a few calls and back (its ring resumes at the advanced cursor), a same-count replacement,
    a different-count replacement, a still replacing a ring and a cleared background; plain calls in between"""
    key, W, H = "meet_lite", 320, 240
    m = _Model(4, ctx_bg=synth.background()[:, ::-1].copy(), ctx_k=7)
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    g.set_background(m.ctx_bg)
    g.set_bgblur(7)
    g.set_sources(4)
    m.set_ring(g, 0, _ring(3, 10), 1)                # follows the context's strength
    m.set_ring(g, 1, _ring(2, 11), 1)
    m.set_fx(g, 1, "default", 0)
    m.set_ring(g, 2, _ring(4, 12), 1)
    m.set_fx(g, 2, "default", 25)
    o = _Oracles(key, W, H, 4)
    o.call(g, [0, 1, 2, 3], m)
    o.plain(g, m)
    g.set_bgblur(11)                                 # s0's ring is re-blurred, s1 and s2 keep theirs
    m.ctx_k = 11
    o.call(g, [2, 1, 0], m)
    m.set_fx(g, 0, "none", 25)                       # s0: its camera frame blurred; its ring keeps playing
    o.call(g, [0, 3], m)
    o.call(g, [1, 0], m)
    m.set_fx(g, 0)
    o.call(g, [0, 2], m)
    o.plain(g, m)
    m.set_ring(g, 2, _ring(4, 20), 1)                # same count: in place, the cursor back at 0
    o.call(g, [2, 0, 1, 3], m)
    m.set_ring(g, 1, _ring(5, 21), 2)                # another count: the pool is reallocated, s0 and s2 survive it
    o.call(g, [1, 2, 0], m)
    m.set_still(g, 0, _ring(1, 22)[0])               # a still replaces a ring
    o.call(g, [0, 1, 2], m)
    m.set_still(g, 2, None)                          # cleared: the context image at s2's own 25
    o.call(g, [2, 1, 0, 3], m)
    o.plain(g, m)
    g.close()


def _ring_raw(L, g, s, frames, count=None, bw=None, bh=None, pitch=None, stride=None, advance=1):
    n, h, w, _ = frames.shape
    return L.bsb_set_source_background_ring(g._h, s, frames.ctypes.data, n if count is None else count, w if bw is None else bw,
                                            h if bh is None else bh, w * 3 if pitch is None else pitch,
                                            h * w * 3 if stride is None else stride, advance)


def test_errors(emu_lib):
    """every refused ring, cursor and call leaves the context usable and every background and cursor as it was.  s0 plays
    a ring at 2W x 2H (the INTER_AREA 2x2 resize), s1 a ring at a size that takes the generic resize"""
    key, W, H = "meet_lite", 320, 240
    L = emu_lib
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    frames = _ring(3, 5, (2 * W, 2 * H))
    assert _ring_raw(L, g, 0, frames) == 0 and b"set_sources" in L.bsb_last_error()
    assert L.bsb_set_source_background_cursor(g._h, 0, 0) == 0 and b"set_sources" in L.bsb_last_error()
    m = _Model(3, ctx_bg=synth.background())
    g.set_background(m.ctx_bg)
    g.set_sources(3)
    m.set_ring(g, 0, frames, 1)
    m.set_ring(g, 1, _ring(2, 6, (250, 170)), 0)
    o = _Oracles(key, W, H, 3)
    o.call(g, [0, 1, 2], m)
    n, h, w, _ = frames.shape
    bad = [
        (lambda: _ring_raw(L, g, 3, frames), b"out of range"),
        (lambda: _ring_raw(L, g, -1, frames), b"out of range"),
        (lambda: _ring_raw(L, g, 0, frames, count=0), b"count"),
        (lambda: _ring_raw(L, g, 0, frames, bw=0), b"invalid background"),
        (lambda: _ring_raw(L, g, 0, frames, bh=0), b"invalid background"),
        (lambda: _ring_raw(L, g, 0, frames, pitch=w * 3 - 1), b"invalid background"),
        (lambda: _ring_raw(L, g, 0, frames, stride=(h - 1) * w * 3 + w * 3 - 1), b"stride"),
        (lambda: _ring_raw(L, g, 0, frames, advance=-1), b"advance"),
        (lambda: L.bsb_set_source_background_ring(g._h, 0, None, 3, w, h, w * 3, h * w * 3, 1), b"invalid background"),
        (lambda: L.bsb_set_source_background_cursor(g._h, 0, 3), b"out of range"),
        (lambda: L.bsb_set_source_background_cursor(g._h, 0, -1), b"out of range"),
        (lambda: L.bsb_set_source_background_cursor(g._h, 1, 2), b"out of range"),
        (lambda: L.bsb_set_source_background_cursor(g._h, 2, 0), b"no background of its own"),
        (lambda: L.bsb_set_source_background_cursor(g._h, 3, 0), b"out of range"),
    ]
    for i, (call, msg) in enumerate(bad):
        assert call() == 0, i
        assert msg in L.bsb_last_error(), (i, L.bsb_last_error())
        o.call(g, [0, 1] if i % 2 else [1, 0, 2], m)
    with pytest.raises(api.BackscrubError, match="distinct"):
        g.composite_sources(np.stack([synth.frame(W, H)] * 2), [0, 0])
    with pytest.raises(api.BackscrubError, match="n_frames"):
        g.composite_sources(np.stack([synth.frame(W, H)] * 4), [0, 1, 2, 0])
    o.call(g, [0, 2], m)                             # the refused calls moved no cursor
    # a stride of exactly one image is enough, and count 1 needs none
    one = np.ascontiguousarray(frames[:1])
    assert _ring_raw(L, g, 2, one, stride=0, advance=0) == 1
    m.ring[2] = [[one[0]], 0, 0]
    o.call(g, [2, 0], m)
    g.close()


def test_post_stage_on_fed_masks(emu_lib):
    """the post stage alone (bsb_test_feed FEED_MASK) over many sources calls mixing rings of 5 at advance 2 (one at its
    own strength 7), a still and camera blur: slot and cursor arithmetic against the oracle's blend"""
    key, W, H = "meet_lite", 320, 240
    gm = geo(key, W, H)
    c = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    c.set_background(synth.background())
    c.set_sources(5)
    rings = {0: _ring(5, 30), 3: _ring(5, 31)}
    c.set_source_background_ring(0, rings[0], 2)
    c.set_source_background_ring(3, rings[3], 2)
    c.set_source_effect(3, "default", 7)
    still = _ring(1, 32)[0]
    c.set_source_background(1, still)
    c.set_source_effect(2, "none", 9)
    resized = {s: [po.resize_linear_u8(r, W, H) for r in rings[s]] for s in rings}
    ctx = po.resize_linear_u8(synth.background(), W, H)
    cur = {0: 0, 3: 0}
    masks = random_masks(gm, 40, 5)
    rng = np.random.default_rng(5)
    k = 0
    while k + 4 <= len(masks):
        n = int(rng.integers(1, 5))
        ids = [int(s) for s in rng.permutation(5)[:n]]
        frames = np.stack([synth.frame(W, H, t=k + b, stream=s) for b, s in enumerate(ids)])
        chunk = masks[k:k + n]
        c.feed(B.FEED_MASK, chunk)
        out, vid, mask = c.composite_sources(frames, ids)
        for b, s in enumerate(ids):
            rm = ref_mask(gm, chunk[b])
            bg = {0: lambda: resized[0][cur[0]], 1: lambda: po.resize_linear_u8(still, W, H),
                  2: lambda: po.gaussian_blur(frames[b], 9), 3: lambda: po.gaussian_blur(resized[3][cur[3]], 7),
                  4: lambda: ctx}[s]()
            ro, rv = ref_outputs(rm, frames[b], bg)
            tag = (k, ids, b, s, cur.get(s))
            assert np.array_equal(mask[b], rm), ("mask", tag)
            assert np.array_equal(out[b], ro), ("composite", tag)
            assert np.array_equal(vid[b], rv), ("video", tag)
        for s in ids:
            if s in cur:
                cur[s] = (cur[s] + 2) % 5
        k += n
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100


@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


def _nv12_frame(W, H, t, s):
    yv = synth.yuyv_frame(W, H, t=t, stream=s)
    return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)


class _Dev:
    """a sources context fed device camera frames (YUYV or NV12) or host BGR frames, and one plain batch-1 context per
    source set up as the contract says: the source's ring (or still, or the context image, or none), its strength, its
    flip and output size, paced by the same cursor moves"""

    def __init__(self, lib, key, W, H, n_sources, max_batch, ctx_k, fmt):
        import torch
        self.torch, self.lib, self.key, self.W, self.H, self.fmt = torch, lib, key, W, H, fmt
        self.m = _Model(n_sources, ctx_bg=synth.background()[::-1].copy(), ctx_k=ctx_k)
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch)
        self.g.set_background(self.m.ctx_bg)
        self.g.set_bgblur(ctx_k)
        self.g.set_sources(n_sources)
        self.flip, self.size = {}, {}
        self.ref = {}
        self.t = [0] * n_sources
        self.npx = W * H
        self.fn = W * H * 3 // 2 if fmt == "nv12" else W * H * 2       # camera frame bytes
        self.opx = W * H                                               # largest output frame, grown by set_size
        self.max_batch = max_batch

    def set_cursor(self, s, i):
        """the source's cursor and its plain context's, moved together"""
        self.m.set_cursor(self.g, s, i)
        if s in self.ref:
            self.ref[s][0].set_background_cursor(i)

    def set_flip(self, s, flip):
        self.g.set_source_flip(s, bool(flip & 1), bool(flip & 2))
        self.flip[s] = flip

    def set_size(self, s, size):
        self.g.set_source_output(s, size)
        self.size[s] = size
        self.opx = max(self.opx, size[0] * size[1])

    def out_size(self, s):
        return self.size.get(s, (self.W, self.H))

    def plain(self, s):
        """the plain context of source s, (re)configured to the rule: a new background of the source is set on the same
        context (its smoother state carries on), with the source's cursor"""
        m = self.m
        kind, _ = m.fx[s]
        want = None if kind == "none" else (("ring", m.version[s]) if s in m.ring else ("ctx",))
        if s not in self.ref:
            self.ref[s] = [api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1), None, None, None]
        r = self.ref[s]
        c = r[0]
        if r[1] != want:
            assert want is not None, "a reference context cannot drop its background"
            if want[0] == "ring":
                imgs, adv, cur = m.ring[s]
                c.set_background_ring(np.stack(imgs), adv)
                if cur:
                    c.set_background_cursor(cur)
            else:
                c.set_background(m.ctx_bg)
            r[1] = want
        out = (self.flip.get(s, 0), self.out_size(s))
        if r[3] != out:
            c.set_output(bool(out[0] & 1), bool(out[0] & 2), out[1])
            r[3] = out
        k = m.setup(s)[1]
        if r[2] != k:
            r[0].set_bgblur(k)
            r[2] = k
        return r[0]

    def frame(self, s, t):
        if self.fmt == "nv12":
            return _nv12_frame(self.W, self.H, t, s)
        if self.fmt == "yuyv":
            return synth.yuyv_frame(self.W, self.H, t=t, stream=s)
        return synth.frame(self.W, self.H, t=t, stream=s)

    def alloc(self):
        torch, dev, B_ = self.torch, "cuda:0", self.max_batch
        self.d_in = torch.empty(B_ * self.fn, dtype=torch.uint8, device=dev)
        self.d_out = torch.empty(B_ * self.opx * 3, dtype=torch.uint8, device=dev)
        self.vb = self.opx * 3 // 2 if self.fmt == "nv12" else self.opx * 2
        self.d_vid = torch.empty(B_ * self.vb, dtype=torch.uint8, device=dev)
        self.d_mask = torch.empty(B_ * self.npx, dtype=torch.uint8, device=dev)

    def load(self, ids):
        host = np.stack([self.frame(s, self.t[s]) for s in ids])
        if self.fmt != "bgr":
            self.d_in[:host.size].copy_(self.torch.from_numpy(host.reshape(-1)))
        return host

    def run(self, ids, host, sync=True):
        n, g = len(ids), self.g
        if self.fmt == "bgr":
            out, vid, mask = g.composite_sources(host, ids)
            self.host_res = (out, vid, mask)
            return
        args = (n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(), self.d_mask.data_ptr())
        if self.fmt == "nv12":
            g.composite_sources_nv12_device(*args, sync=sync, out_stride=self.opx * 3, nv12_stride=self.vb)
        else:
            g.composite_sources_yuyv_device(*args, sync=sync, out_stride=self.opx * 3, yuyv_stride=self.vb)

    def results(self, ids):
        """per frame: (composite, video, mask) bytes at the frame's own size"""
        res = []
        if self.fmt == "bgr":
            out, vid, mask = self.host_res
            for b in range(len(ids)):
                res.append((np.asarray(out[b]).reshape(-1), np.asarray(vid[b]).reshape(-1), mask[b].reshape(-1)))
            return res
        out, vid, mask = self.d_out.cpu().numpy(), self.d_vid.cpu().numpy(), self.d_mask.cpu().numpy()
        for b, s in enumerate(ids):
            w, h = self.out_size(s)
            vn = w * h * 3 // 2 if self.fmt == "nv12" else w * h * 2
            res.append((out[b * self.opx * 3: b * self.opx * 3 + w * h * 3], vid[b * self.vb: b * self.vb + vn],
                        mask[b * self.npx: (b + 1) * self.npx]))
        return res

    def expect(self, s, t):
        """the plain context's bytes for frame t of source s (one call: its ring moves on as the source's does)"""
        c = self.plain(s)
        fr = self.frame(s, t)
        if self.fmt == "bgr":
            out, vid, mask = c.composite(fr[None])
            return out.reshape(-1), vid.reshape(-1), mask.reshape(-1)
        torch, dev = self.torch, "cuda:0"
        w, h = self.out_size(s)
        r_in = torch.from_numpy(fr.reshape(-1).copy()).to(dev)
        r_out = torch.empty(w * h * 3, dtype=torch.uint8, device=dev)
        r_vid = torch.empty(w * h * 3 // 2 if self.fmt == "nv12" else w * h * 2, dtype=torch.uint8, device=dev)
        r_mask = torch.empty(self.npx, dtype=torch.uint8, device=dev)
        if self.fmt == "nv12":
            c.composite_nv12_device(1, r_in.data_ptr(), r_out.data_ptr(), r_vid.data_ptr(), r_mask.data_ptr(), sync=True)
        else:
            c.composite_yuyv_device(1, r_in.data_ptr(), r_out.data_ptr(), r_vid.data_ptr(), r_mask.data_ptr(), sync=True)
        return r_out.cpu().numpy(), r_vid.cpu().numpy(), r_mask.cpu().numpy()

    def check(self, ids, res):
        for b, s in enumerate(ids):
            ro, rv, rm = self.expect(s, self.t[s])
            got = res[b]
            tag = (ids, b, s, self.t[s], self.m.fx[s], self.m.ring[s][2] if s in self.m.ring else None)
            assert np.array_equal(got[2], rm), f"mask differs {tag}"
            assert np.array_equal(got[0], ro), f"composite differs {tag}"
            assert np.array_equal(got[1], rv), f"video output differs {tag}"
            self.t[s] += 1
        self.m.moved(ids)

    def step(self, ids):
        host = self.load(ids)
        self.run(ids, host)
        self.check(ids, self.results(ids))

    def close(self):
        self.g.close()
        for r in self.ref.values():
            r[0].close()


def _mixed(d, own_size=None, flip_src=None):
    """s0 ring of 3 at advance 1, s1 ring of 4 at advance 1 at its own strength 25, s2 ring of 2 at advance 0 (paced by
    the caller), s3 its own still, s4 the context image, s5 its camera frame blurred at 25"""
    m, g = d.m, d.g
    m.set_ring(g, 0, _ring(3, 40), 1)
    m.set_ring(g, 1, _ring(4, 41), 1)
    m.set_fx(g, 1, "default", 25)
    m.set_ring(g, 2, _ring(2, 42), 0)
    m.set_still(g, 3, _ring(1, 43)[0])
    m.set_fx(g, 5, "none", 25)
    if flip_src is not None:
        d.set_flip(flip_src, 1)
    if own_size is not None:
        d.set_size(*own_size)


MIXED_CALLS = ([0, 1, 2, 3, 4, 5], [5, 3, 1], [2, 0, 4], [1, 0], [4, 3, 2, 1, 0], [0, 5, 1, 2], [1, 0, 3])


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("meet_full", 1280, 720), ("mlkit", 640, 480)])
@pytest.mark.parametrize("fmt", ["yuyv", "nv12", "bgr"])
def test_gpu_mixed_rings(gpu_lib, key, W, H, fmt):
    """rings at advance 1 and 0, an own still, the context image and camera blur in each call, until every ring has
    wrapped; source 4 mirrored (k_post_tma writes it in place), then source 3 at its own size too (the call through k_tail)"""
    d = _Dev(gpu_lib, key, W, H, 6, 6, 7, fmt)
    _mixed(d, flip_src=4)
    d.alloc()
    for i, ids in enumerate(MIXED_CALLS):
        if i == 3:
            d.set_cursor(2, 1)
        d.step(ids)
        if fmt != "bgr" and key == "meet_full":
            assert d.g.yuyv_native, ids              # the pool is read through the TMA post kernel's tensor map
    d.set_size(3, (W // 2 + 2, H // 2 + 2))
    d.alloc()
    for ids in MIXED_CALLS[:4]:
        d.step(ids)
    d.close()


@pytest.mark.gpu
def test_gpu_ring_set_between_replays(gpu_lib):
    """a new ring between replayed calls grows the pool and drops the graphs; a same-count replacement between
    asynchronous calls takes effect in stream order"""
    W, H = 1280, 720
    d = _Dev(gpu_lib, "meet_lite", W, H, 4, 4, 0, "yuyv")
    _m = d.m
    _m.set_ring(d.g, 0, _ring(3, 50), 1)
    d.alloc()
    ids = [0, 1, 2, 3]
    d.step(ids)
    d.step(ids)                                     # replayed
    _m.set_ring(d.g, 2, _ring(5, 51), 1)            # the pool grows: new bank, graphs dropped
    d.step(ids)
    d.step(ids)
    # asynchronous calls around a same-count replacement of s0 (in place), each from and into its own device buffers
    torch = d.torch
    bufs = []
    for j in range(4):
        host = np.stack([d.frame(s, d.t[s] + j) for s in ids])
        bufs.append((torch.from_numpy(host.reshape(-1).copy()).cuda(),
                     [torch.empty_like(d.d_out), torch.empty_like(d.d_vid), torch.empty_like(d.d_mask)]))
    torch.cuda.synchronize()
    new = _ring(3, 52)
    for j, (d_in, o) in enumerate(bufs):
        if j == 2:
            d.g.set_source_background_ring(0, new, 1)
        d.g.composite_sources_yuyv_device(4, ids, d_in.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), sync=False,
                                          out_stride=d.opx * 3, yuyv_stride=d.vb)
    d.g.synchronize()
    for j, (_, o) in enumerate(bufs):
        if j == 2:
            _m.ring[0] = [list(new), 1, 0]
            _m.version[0] += 1
        out, vid, mask = (x.cpu().numpy() for x in o)
        res = [(out[b * d.opx * 3:(b + 1) * d.opx * 3], vid[b * d.vb:(b + 1) * d.vb], mask[b * d.npx:(b + 1) * d.npx]) for b in range(4)]
        d.check(ids, res)
    d.close()


@pytest.mark.gpu
def test_gpu_allocation_refused(gpu_lib):
    """a ring whose bank would need ~1.3 TB (150000 images of 2x2 at 1280x720) is refused at once; the context, its rings
    and the next call are unchanged"""
    W, H = 1280, 720
    L = gpu_lib
    d = _Dev(gpu_lib, "meet_lite", W, H, 3, 3, 7, "yuyv")
    d.m.set_ring(d.g, 0, _ring(3, 60), 1)
    d.m.set_ring(d.g, 1, _ring(2, 61), 1)
    d.alloc()
    d.step([0, 1, 2])
    tiny = np.random.default_rng(0).integers(0, 256, (150000, 2, 2, 3), dtype=np.uint8)
    for s in (1, 2):
        assert _ring_raw(L, d.g, s, tiny) == 0, s
        assert b"allocate" in L.bsb_last_error(), L.bsb_last_error()
        d.step([2, 1, 0])
    d.close()


@pytest.mark.gpu
def test_gpu_16_sources_rings_of_4(gpu_lib):
    """16 sources, max_batch 16, each with its own ring of 4 at advance 1, over two wraps"""
    d = _Dev(gpu_lib, "meet_lite", 640, 480, 16, 16, 7, "yuyv")
    for s in range(16):
        d.m.set_ring(d.g, s, _ring(4, 70 + s), 1)
    d.alloc()
    rng = np.random.default_rng(16)
    for _ in range(8):
        d.step([int(s) for s in rng.permutation(16)])
    assert all(d.m.ring[s][2] == 0 for s in range(16))
    d.close()
