"""Per-source output size (bsb_set_source_output): each camera of a sources context picks its own virtual-camera geometry.
Frame b of a sources call, from source s, must give exactly the bytes a plain context gives for that camera's stream when
set up the same way plus bsb_set_output(flip_h_s, flip_v_s, out_w_s, out_h_s): composite, YUYV / NV12 and mask (W x H).

`-m "not gpu"`: the kernel-logic emulator build (the fallback post kernel and k_tail) vs the oracle.
`-m gpu`: the sm_90a library vs plain batch-1 contexts, and k_tail once against the oracle itself (the plain contexts run
the same tail, so only that check can catch an error both share).

161 x 121 from 320 x 240 is a size where flipping after the resize gives other bytes than flipping before it (the
fixed-point tables are not mirror-symmetric; 10 bytes differ horizontally, 80 vertically on synth frame 3 of stream 1), so
the per-tap mirroring of k_tail is checked where it matters."""

import ctypes as C

import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_nv12 import nv12_frame, ref_nv12_to_bgr, ref_yuyv_to_nv12
from tests.test_source_flip import FLIPS8, H_, V_, _code, _Dev, _set_flip

ORDER_SENSITIVE = (161, 121)


def _addr(a):
    return a.ctypes.data if a is not None else 0


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def test_flip_order_matters_at_the_named_size():
    """the oracle confirms that ORDER_SENSITIVE tells the two orders apart, in both directions"""
    img = synth.frame(320, 240, t=3, stream=1)
    w, h = ORDER_SENSITIVE
    for fh, fv in ((1, 0), (0, 1)):
        before = po.resize_linear_u8(po.flip(img, fh, fv), w, h)
        after = po.flip(po.resize_linear_u8(img, w, h), fh, fv)
        assert not np.array_equal(before, after), (fh, fv)


class _Streams:
    """one oracle stream per source; source s blends bgs[s] (None: its camera frame blurred at ks[s])"""

    def __init__(self, key, W, H, n, bgs, ks):
        self.W, self.H = W, H
        self.o = [po.MaskGen(model_path(key), W, H) for _ in range(n)]
        self.t = [0] * n
        self.bgs, self.ks = bgs, ks
        self.flips = {s: None for s in range(n)}
        self.sizes = {s: None for s in range(n)}
        self.ctx_flip, self.ctx_size = 0, (W, H)

    def size(self, s):
        return self.sizes[s] or self.ctx_size

    def ref(self, s, fr):
        code = self.ctx_flip if self.flips[s] is None else self.flips[s]
        fh, fv = _code(code)
        r = self.o[s].composite_ex(fr, self.bgs[s], bgblur=self.ks[s], flip_h=fh, flip_v=fv, out_size=self.size(s))
        self.t[s] += 1
        return r

    def call(self, g, ids, want_yuyv=True):
        """host BGR sources call"""
        fr = np.stack([synth.frame(self.W, self.H, t=self.t[s], stream=s) for s in ids])
        out, yuyv, mask = g.composite_sources(fr, ids, want_yuyv=want_yuyv)
        sizes = [self.size(s) for s in ids]
        if len(set(sizes)) == 1:
            assert isinstance(out, np.ndarray) and out.shape == (len(ids), sizes[0][1], sizes[0][0], 3)
        else:
            assert isinstance(out, list)
        for b, s in enumerate(ids):
            assert g.source_output_size(s) == self.size(s)
            ro, ry, rm = self.ref(s, fr[b])
            tag = (ids, b, s, self.t[s] - 1, self.size(s))
            assert np.array_equal(mask[b], rm), f"mask differs {tag}"
            assert np.array_equal(out[b], ro), f"composite differs {tag}"
            if want_yuyv:
                assert np.array_equal(yuyv[b], ry), f"YUYV differs {tag}"

    def call_yuyv_device(self, g, ids):
        """device YUYV sources call on the emulator (host memory stands in for device memory); flat pair layout"""
        n = len(ids)
        cam = np.stack([synth.yuyv_frame(self.W, self.H, t=self.t[s], stream=s) for s in ids])
        px = max(w * h for w, h in (self.size(s) for s in ids))
        out, vid = np.zeros(n * px * 3, np.uint8), np.zeros(n * px * 2, np.uint8)
        mask = np.empty((n, self.H, self.W), np.uint8)
        g.composite_sources_yuyv_device(n, ids, _addr(cam), _addr(out), _addr(vid), _addr(mask), sync=True,
                                        out_stride=px * 3, yuyv_stride=px * 2)
        for b, s in enumerate(ids):
            w, h = self.size(s)
            ro, ry, rm = self.ref(s, po.yuyv_to_bgr(cam[b]))
            pairs = w * h // 2
            tag = (ids, b, s, (w, h))
            assert np.array_equal(mask[b], rm), f"mask differs {tag}"
            assert np.array_equal(out[b * px * 3: b * px * 3 + w * h * 3], ro.reshape(-1)), f"composite differs {tag}"
            assert np.array_equal(vid[b * px * 2: b * px * 2 + pairs * 4], ry.reshape(-1)[:pairs * 4]), f"YUYV differs {tag}"


def _emu_setup(lib):
    """five sources of meet_lite 320x240: 0 follows the context; 1 240x180 with its own image; 2 160x120 (the exact 2x
    INTER_AREA path), camera blur 9, mirrored H; 3 400x300 (up-scale), the context image at strength 5, H | V; 4 an own
    320x240, mirrored V"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    ctx_bg = bg[::-1].copy()
    own = np.roll(bg, 90, axis=1)
    g = api.MaskGen(lib, model_path(key), W, H, max_batch=5)
    g.set_background(ctx_bg)
    g.set_sources(5)
    g.set_source_background(1, own)
    g.set_source_effect(2, "none", 9)
    g.set_source_effect(3, "default", 5)
    o = _Streams(key, W, H, 5, [ctx_bg, own, None, ctx_bg, ctx_bg], [0, 0, 9, 5, 0])
    for s, code in ((1, 0), (2, H_), (3, H_ | V_), (4, V_)):
        _set_flip(g, o.flips, s, code)
    for s, size in ((1, (240, 180)), (2, (160, 120)), (3, (400, 300)), (4, (320, 240))):
        g.set_source_output(s, size)
        o.sizes[s] = size
    return g, o


def test_sizes_follow_and_own(emu_lib):
    g, o = _emu_setup(emu_lib)
    for ids in ([0, 1, 2, 3, 4], [3, 1], [4, 2, 0], [0, 4]):
        o.call(g, ids)
    # a context size (and flip) that the following source picks up; the own 320x240 is then resized against it
    g.set_output(flip_h=True, out_size=(200, 150))
    o.ctx_flip, o.ctx_size = H_, (200, 150)
    for ids in ([0, 1, 2, 3, 4], [4, 0]):
        o.call(g, ids)
    # source 1 back to following; source 2 at a size where the flip order matters, with an odd width (composite only on
    # the host buffers, YUYV through the device entry's flat pixel pairs)
    g.set_source_output(1)
    o.sizes[1] = None
    g.set_source_output(2, ORDER_SENSITIVE)
    o.sizes[2] = ORDER_SENSITIVE
    _set_flip(g, o.flips, 3, V_)
    g.set_source_output(3, ORDER_SENSITIVE)
    o.sizes[3] = ORDER_SENSITIVE
    o.call(g, [1, 2, 3, 0], want_yuyv=False)
    o.call_yuyv_device(g, [2, 4, 3, 1])
    g.close()


def test_sources_nv12_sizes(emu_lib):
    """device NV12 call with mixed even sizes: k_tail writes the NV12 directly"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    g.set_background(bg)
    g.set_sources(3)
    sizes = {0: (W, H), 1: (240, 180), 2: (160, 120)}
    g.set_source_output(1, sizes[1])
    g.set_source_output(2, sizes[2])
    g.set_source_flip(2, flip_h=True)
    o = [po.MaskGen(model_path(key), W, H) for _ in range(3)]
    t = [0, 0, 0]
    for ids in ([0, 1, 2], [2, 1]):
        n = len(ids)
        frames = np.stack([nv12_frame(W, H, t=t[s], stream=s) for s in ids])
        px = max(sizes[s][0] * sizes[s][1] for s in ids)
        out, nv = np.zeros(n * px * 3, np.uint8), np.zeros(n * px * 3 // 2, np.uint8)
        mask = np.empty((n, H, W), np.uint8)
        g.composite_sources_nv12_device(n, ids, _addr(frames), _addr(out), _addr(nv), _addr(mask), sync=True, out_stride=px * 3,
                                        nv12_stride=px * 3 // 2)
        for b, s in enumerate(ids):
            w, h = sizes[s]
            ro, ry, rm = o[s].composite_ex(ref_nv12_to_bgr(frames[b]), bg, flip_h=s == 2, out_size=(w, h))
            assert np.array_equal(mask[b], rm), (ids, b)
            assert np.array_equal(out[b * px * 3: b * px * 3 + w * h * 3], ro.reshape(-1)), (ids, b)
            assert np.array_equal(nv[b * px * 3 // 2: b * px * 3 // 2 + w * h * 3 // 2], ref_yuyv_to_nv12(ry).reshape(-1)), (ids, b)
            t[s] += 1
    g.close()


ODD_SIZES = [(161, 121), (161, 120), (160, 121)]


def test_nv12_calls_without_video_output_at_odd_sizes(emu_lib):
    """NV12 camera frames in, only the composite and mask out: odd output sizes are allowed (no NV12 is written), and the
    tail writes every pixel of them — a plain context at odd context sizes, then sources at odd own sizes"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    g.set_background(bg)
    o = po.MaskGen(model_path(key), W, H)
    t = 0
    for size in ODD_SIZES:
        g.set_output(flip_v=True, out_size=size)
        frames = np.stack([nv12_frame(W, H, t=t + b) for b in range(2)])
        out, nv, mask = g.composite_nv12(frames, want_nv12=False)
        assert nv is None
        for b in range(2):
            ro, _, rm = o.composite_ex(ref_nv12_to_bgr(frames[b]), bg, flip_v=True, out_size=size)
            assert np.array_equal(mask[b], rm), (size, b)
            assert np.array_equal(out[b], ro), (size, b)
        t += 2
    g.close()

    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    g.set_background(bg)
    g.set_sources(3)
    for s, size in enumerate(ODD_SIZES):
        g.set_source_output(s, size)
    g.set_source_flip(0, flip_h=True)
    o = [po.MaskGen(model_path(key), W, H) for _ in range(3)]
    ts = [0, 0, 0]
    for ids in ([0, 1, 2], [2, 0]):
        n = len(ids)
        frames = np.stack([nv12_frame(W, H, t=ts[s], stream=s) for s in ids])
        px = max(ODD_SIZES[s][0] * ODD_SIZES[s][1] for s in ids)
        out, mask = np.zeros(n * px * 3, np.uint8), np.empty((n, H, W), np.uint8)
        g.composite_sources_nv12_device(n, ids, _addr(frames), _addr(out), 0, _addr(mask), sync=True, out_stride=px * 3)
        for b, s in enumerate(ids):
            w, h = ODD_SIZES[s]
            ro, _, rm = o[s].composite_ex(ref_nv12_to_bgr(frames[b]), bg, flip_h=s == 0, out_size=(w, h))
            assert np.array_equal(mask[b], rm), (ids, b)
            assert np.array_equal(out[b * px * 3: b * px * 3 + w * h * 3], ro.reshape(-1)), (ids, b)
            ts[s] += 1
    g.close()


def test_source_output_errors_and_reset(emu_lib):
    key, W, H = "meet_lite", 320, 240
    L = emu_lib
    g = api.MaskGen(L, model_path(key), W, H, max_batch=2)
    assert L.bsb_set_source_output(g._h, 0, 160, 120) == 0 and b"set_sources" in L.bsb_last_error()
    assert L.bsb_source_output_size(g._h, 0, None, None) == 0 and b"set_sources" in L.bsb_last_error()
    g.set_sources(3)
    bad = [(3, 160, 120, b"out of range"), (-1, 160, 120, b"out of range"), (0, 0, 120, b"size"), (0, 160, -1, b"size"),
           (0, 16385, 120, b"size"), (1, 160, 16385, b"size")]
    for s, w, h, msg in bad:
        assert L.bsb_set_source_output(g._h, s, w, h) == 0, (s, w, h)
        assert msg in L.bsb_last_error(), (s, w, h, L.bsb_last_error())
    with pytest.raises(api.BackscrubError, match="bsb_set_source_output"):
        g.set_source_output(5, (160, 120))
    w, h = C.c_int(), C.c_int()
    assert L.bsb_source_output_size(g._h, 3, C.byref(w), C.byref(h)) == 0 and b"out of range" in L.bsb_last_error()
    # sources moving between more distinct sizes than there are sources: every source's current size stays right
    for r in range(6):
        for s in range(3):
            size = (100 + 2 * ((r + s) % 5), 80)
            g.set_source_output(s, size)
            assert g.source_output_size(s) == size
    # call-time rules: a stride too small for a frame's own size, an NV12 output of odd own size, a host YUYV output of odd
    # own width; nothing is launched
    bg = synth.background()
    g.set_background(bg)
    g.set_source_output(0, (400, 300))
    g.set_source_output(1, (161, 120))
    n = 2
    fr = np.stack([synth.yuyv_frame(W, H, t=0, stream=s) for s in range(n)])
    out, vid, mask = np.zeros(n * 400 * 300 * 3, np.uint8), np.zeros(n * 400 * 300 * 2, np.uint8), np.empty((n, H, W), np.uint8)
    l0 = L.bsb_total_launches()
    ids = (C.c_int * 1)(0)
    assert L.bsb_composite_sources_yuyv_device(g._h, 1, ids, _addr(fr), _addr(out), W * H * 3, None, 0, None, 0, 1) == 0
    assert b"output stride" in L.bsb_last_error()
    assert L.bsb_composite_sources_yuyv_device(g._h, 1, ids, _addr(fr), None, 0, _addr(vid), W * H * 2, None, 0, 1) == 0
    assert b"video stride" in L.bsb_last_error()
    nv = np.stack([nv12_frame(W, H, t=0, stream=s) for s in range(n)])
    ids1 = (C.c_int * 1)(1)
    assert L.bsb_composite_sources_nv12_device(g._h, 1, ids1, _addr(nv), W, W * H, W * H * 3 // 2, None, 0, _addr(vid), 400 * 300 * 2,
                                                None, 0, 1) == 0
    assert b"even output width" in L.bsb_last_error()
    bgr = np.stack([synth.frame(W, H, t=0, stream=s) for s in range(n)])
    assert L.bsb_composite_sources(g._h, 1, ids1, _addr(bgr), W * 3, W * H * 3, None, 0, _addr(vid), 400 * 300 * 2, None, 0) == 0
    assert b"even width" in L.bsb_last_error()
    # an id out of range beside a frame of its own size: the id is reported, nothing is read past the source tables
    for bad_id in (1 << 28, -1, 3):
        ids2 = (C.c_int * 2)(1, bad_id)
        assert L.bsb_composite_sources(g._h, 2, ids2, _addr(bgr), W * 3, W * H * 3, _addr(out), 400 * 300 * 3, None, 0, None, 0) == 0
        assert b"source id out of range" in L.bsb_last_error(), bad_id
        assert L.bsb_composite_sources_yuyv_device(g._h, 2, ids2, _addr(fr), _addr(out), 400 * 300 * 3, None, 0, None, 0, 1) == 0
        assert b"source id out of range" in L.bsb_last_error(), bad_id
    assert L.bsb_total_launches() == l0
    # still usable; set_sources resets every source to follow the context
    g.set_sources(3)
    assert g.source_output_size(0) == (W, H) and g.source_output_size(1) == (W, H)
    o = [po.MaskGen(model_path(key), W, H) for _ in range(2)]
    out, yuyv, mask = g.composite_sources(bgr, [0, 1])
    for b in range(2):
        ro, ry, rm = o[b].composite(bgr[b], bg)
        assert np.array_equal(out[b], ro) and np.array_equal(yuyv[b], ry) and np.array_equal(mask[b], rm), b
    g.close()


def test_tail_is_one_launch(emu_lib):
    """a call with a tail (own sizes, a context resize, or a flip the post kernel does not write in place) issues exactly
    one launch more than the same call without one"""
    key, W, H = "meet_lite", 320, 240
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    g.set_background(synth.background())
    g.set_sources(3)
    fr = np.stack([synth.frame(W, H, t=0, stream=s) for s in range(3)])
    g.composite(fr)
    plain = g.launches_per_call
    g.composite_sources(fr, [0, 1, 2])
    base = g.launches_per_call
    g.set_source_output(1, (240, 180))
    g.composite_sources(fr, [0, 1, 2])
    assert g.launches_per_call == base + 1
    g.set_source_output(2, (160, 120))
    g.set_source_flip(0, flip_h=True)
    g.composite_sources(fr, [0, 1, 2])
    assert g.launches_per_call == base + 1
    g.set_source_output(1)
    g.set_source_output(2)
    g.composite_sources(fr, [0, 1, 2])                # the emulator's post kernel is not k_post_tma: the flip is in the tail
    assert g.launches_per_call == base + 1
    g.set_source_flip(0)
    g.composite_sources(fr, [0, 1, 2])
    assert g.launches_per_call == base
    g.set_output(out_size=(200, 150))                 # plain call with a context resize
    g.composite(fr)
    assert g.launches_per_call == plain + 1
    g.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100


@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


class _SizedDev(_Dev):
    """_Dev with a size per source: the sources context's buffers hold the largest size, frame b packed at its own; the
    plain reference context of source s runs bsb_set_output(flip_s, size_s)"""

    def __init__(self, lib, key, W, H, n_sources, sizes, fmt="yuyv", layout=None, flips=None, min_px=0):
        super().__init__(lib, key, W, H, n_sources, fmt=fmt, layout=layout, flips=flips)
        self.sizes = {s: None for s in range(n_sources)}
        for s in range(n_sources):
            self.set_size(s, sizes[s % len(sizes)])
        self.alloc(min_px)

    def set_size(self, s, size):
        self.g.set_source_output(s, size)
        self.sizes[s] = size

    def size(self, s):
        return self.sizes[s] or (self.W, self.H)

    def alloc(self, min_px=0):
        """output buffers for the largest size any source has (at least min_px pixels per frame)"""
        self.px = max([min_px] + [w * h for w, h in (self.size(s) for s in self.sizes)])
        mb, dev = len(self.sizes), "cuda:0"
        if self.fmt != "bgr":
            self.d_out = self.torch.zeros(mb * self.px * 3, dtype=self.torch.uint8, device=dev)
            vb = self.px * 3 // 2 if self.fmt == "nv12" else self.px * 2
            self.d_vid = self.torch.zeros(mb * vb, dtype=self.torch.uint8, device=dev)

    def plain(self, s):
        bg, k = self.fx[s]
        ow, oh = self.size(s)
        if s not in self.ref:
            c = api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1)
            if bg is not None:
                c.set_background(bg)
            if k:
                c.set_bgblur(k)
            self.ref[s] = [c, None, None, None]
        r = self.ref[s]
        if r[3] != (ow, oh) and self.fmt != "bgr":
            cam = self.stride if self.fmt == "nv12" else self.W * self.H * 2
            vid = ow * oh * 3 // 2 if self.fmt == "nv12" else ow * oh * 2
            r[1] = [self.torch.empty(m, dtype=self.torch.uint8, device="cuda:0") for m in (cam, ow * oh * 3, vid, self.W * self.H)]
        if (r[2], r[3]) != (self.code(s), (ow, oh)):
            fh, fv = _code(self.code(s))
            r[0].set_output(fh, fv, (ow, oh))
            r[2], r[3] = self.code(s), (ow, oh)
        return r[0], r[1]

    def results(self, n, ids=None):
        if self.fmt == "bgr":
            return self._res
        out, vid = self.d_out.cpu().numpy(), self.d_vid.cpu().numpy()
        vb = self.px * 3 // 2 if self.fmt == "nv12" else self.px * 2
        outs, vids = [], []
        for b, s in enumerate(self._ids):
            w, h = self.size(s)
            outs.append(out[b * self.px * 3: b * self.px * 3 + w * h * 3])
            vids.append(vid[b * vb: b * vb + (w * h * 3 // 2 if self.fmt == "nv12" else w * h * 2)])
        return outs, vids, self.d_mask[:n].cpu().numpy()

    def run(self, ids):
        """explicit strides: the buffers' own, so calls with other sizes within them keep the same arguments"""
        self._ids = list(ids)
        n = len(ids)
        if self.fmt == "bgr":
            self._res = self.g.composite_sources(self.host, ids)
        elif self.fmt == "nv12":
            self.g.composite_sources_nv12_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(), self.d_mask.data_ptr(),
                                                 sync=True, pitch=self.pitch, uv_offset=self.uv, in_stride=self.stride,
                                                 out_stride=self.px * 3, nv12_stride=self.px * 3 // 2)
        else:
            self.g.composite_sources_yuyv_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(),
                                                 self.d_mask.data_ptr(), sync=True, out_stride=self.px * 3, yuyv_stride=self.px * 2)


@pytest.mark.gpu
def test_gpu_tail_against_oracle(gpu_lib):
    """k_tail on sm_90a against the CPU oracle itself (the other GPU tests compare sources with plain contexts, which
    share the tail): meet_lite 320x240, own sizes down / exact 2x / up / odd (the flip order matters at 161x121) with
    flips, through host BGR and device NV12 (NV12 output, and composite only at the odd size)"""
    import torch
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    sizes = {0: (240, 180), 1: (160, 120), 2: (400, 300), 3: ORDER_SENSITIVE}
    codes = {0: H_ | V_, 1: V_, 2: H_, 3: H_ | V_}
    g = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=4)
    g.set_background(bg)
    g.set_sources(4)
    for s in range(4):
        g.set_source_output(s, sizes[s])
        fh, fv = _code(codes[s])
        g.set_source_flip(s, flip_h=fh, flip_v=fv)
    o = [po.MaskGen(model_path(key), W, H) for _ in range(4)]
    t = [0] * 4

    def ref(s, fr):
        fh, fv = _code(codes[s])
        r = o[s].composite_ex(fr, bg, flip_h=fh, flip_v=fv, out_size=sizes[s])
        t[s] += 1
        return r

    ids = [3, 0, 1, 2]                                   # host BGR, composite only (161 is odd)
    fr = np.stack([synth.frame(W, H, t=t[s], stream=s) for s in ids])
    out, _, mask = g.composite_sources(fr, ids, want_yuyv=False)
    for b, s in enumerate(ids):
        ro, _, rm = ref(s, fr[b])
        assert np.array_equal(mask[b], rm) and np.array_equal(out[b], ro), (ids, b, s)
    ids = [0, 1, 2]                                      # device NV12 in and out, even sizes
    n, px = 3, 400 * 300
    frames = np.stack([nv12_frame(W, H, t=t[s], stream=s) for s in ids])
    d_in = torch.from_numpy(frames).cuda()
    d_out = torch.zeros(n * px * 3, dtype=torch.uint8, device="cuda:0")
    d_nv = torch.zeros(n * px * 3 // 2, dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((n, H, W), dtype=torch.uint8, device="cuda:0")
    g.composite_sources_nv12_device(n, ids, d_in.data_ptr(), d_out.data_ptr(), d_nv.data_ptr(), d_mask.data_ptr(), sync=True,
                                    out_stride=px * 3, nv12_stride=px * 3 // 2)
    out, nv, mask = d_out.cpu().numpy(), d_nv.cpu().numpy(), d_mask.cpu().numpy()
    for b, s in enumerate(ids):
        w, h = sizes[s]
        ro, ry, rm = ref(s, ref_nv12_to_bgr(frames[b]))
        assert np.array_equal(mask[b], rm), (b, s)
        assert np.array_equal(out[b * px * 3: b * px * 3 + w * h * 3], ro.reshape(-1)), (b, s)
        assert np.array_equal(nv[b * px * 3 // 2: b * px * 3 // 2 + w * h * 3 // 2], ref_yuyv_to_nv12(ry).reshape(-1)), (b, s)
    g.close()


SIZES8 = [None, (640, 360), (1920, 1080), (1280, 720), (960, 540), (320, 180), (1296, 728), (642, 362)]


@pytest.mark.gpu
@pytest.mark.parametrize("tile", [0, 64, 128])
@pytest.mark.parametrize("fmt", ["yuyv", "nv12", "nv12_pitched", "bgr"])
def test_gpu_meet_720p_sizes(gpu_lib, post_tile, fmt, tile):
    """Meet full 1280x720, 8 sources with their own sizes (follow, down, up, own W x H, exact 2x, odd multiples), mixed
    flips and effects, every entry point; then the context size changes under the following source"""
    post_tile(tile)
    W, H = 1280, 720
    layout = (1536, 1536 * (H + 16), 1536 * (H + 16) + 1536 * H // 2) if fmt == "nv12_pitched" else None
    d = _SizedDev(gpu_lib, "meet_full", W, H, 8, SIZES8, fmt="nv12" if fmt.startswith("nv12") else fmt, layout=layout, flips=FLIPS8)
    for ids in ([0, 1, 2, 3, 4, 5, 6, 7], [7, 5, 3, 1], [6, 0, 4, 2, 1], [3, 0]):
        d.step(ids)
    d.set_size(2, None)                               # back to following; the largest size falls
    d.step([2, 1, 0])
    d.close()


@pytest.fixture
def post_tile():
    import backscrub_b200 as bs
    yield lambda tw: bs.set_tuning("post_tile", tw)
    bs.set_tuning("post_tile", 0)


@pytest.mark.gpu
def test_gpu_graph_replayed_for_new_sizes(gpu_lib):
    """same buffers and n: new sizes within the largest replay the captured graph (which frame has which size is table
    data); a size past the largest captures again; every call is right"""
    d = _SizedDev(gpu_lib, "meet_full", 1280, 720, 4, [(640, 360), None, (960, 540), (320, 180)], flips=[H_, 0, V_, None],
                  min_px=1920 * 1080)
    ids = [0, 1, 2, 3]
    d.step(ids)

    def call(sizes, replays):
        for s, size in enumerate(sizes):
            d.set_size(s, size)
        d.load(ids)
        l0 = gpu_lib.bsb_total_launches()
        d.run(ids)
        assert (gpu_lib.bsb_total_launches() == l0) == replays, (sizes, replays)
        d.check(ids, d.results(4))

    call([(320, 180), (640, 360), None, (960, 540)], True)
    call([(1280, 720), (642, 362), (320, 180), (640, 360)], True)
    call([(1920, 1080), None, (640, 360), (320, 180)], False)       # grows past the largest (1280x720): a new capture
    call([(640, 360), (1920, 1080), (1296, 728), None], True)
    d.close()


@pytest.mark.gpu
def test_gpu_64_sources_sized(gpu_lib):
    d = _SizedDev(gpu_lib, "meet_lite", 640, 480, 64, [None, (320, 240), (960, 720), (640, 480), (480, 360), (322, 242)],
                  flips=[None, 0, H_, H_ | V_, V_])
    d.set_ctx_flip(H_)
    sample = {0, 1, 2, 3, 4, 5, 17, 42, 62, 63}
    d.step(list(range(64)), sample=sample)
    d.step(list(range(63, -1, -1)), sample=sample)
    d.close()
