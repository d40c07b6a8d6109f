"""Per-source background effects (bsb_set_source_effect): each camera of a sources context picks its own blur strength,
or no background image.  Frame b of a sources call, from source s, must give exactly the bytes a plain context gives for
that camera's stream when set up with s's background (its own image, else the context image, else none) and
bsb_set_bgblur(k), k = s's effective strength.

`-m "not gpu"`: the kernel-logic emulator build vs the oracle.  `-m gpu`: the sm_90a library vs plain batch-1 contexts."""

import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path


def _frame(W, H, src, t):
    return synth.frame(W, H, t=t, stream=src)


class _Effects:
    """the test's own model of the context: context image / strength, own images and effects per source"""

    def __init__(self, n, ctx_bg=None, ctx_k=0):
        self.ctx_bg, self.ctx_k = ctx_bg, ctx_k
        self.own = {}
        self.fx = {s: ("default", -1) for s in range(n)}

    def setup(self, s):
        """(background image or None, strength) of the plain context that source s must equal"""
        kind, k = self.fx[s]
        k = self.ctx_k if k < 0 else k
        if kind == "none":
            return None, k
        if s in self.own:
            return self.own[s], k
        return self.ctx_bg, k


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator


# ---------------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")


def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


class _Oracles:
    def __init__(self, key, W, H, n):
        self.W, self.H = W, H
        self.o = [po.MaskGen(model_path(key), W, H) for _ in range(n)]
        self.t = [0] * n

    def call(self, g, ids, m):
        fr = np.stack([_frame(self.W, self.H, s, self.t[s]) for s in ids])
        out, yuyv, mask = g.composite_sources(fr, ids)
        for b, s in enumerate(ids):
            bg, k = m.setup(s)
            if bg is None and not k:
                # a plain context without a background blends plain green (app/deepseg.cc:603); the oracle's "no image"
                # means the camera frame itself
                bg = np.zeros((self.H, self.W, 3), np.uint8)
                bg[..., 1] = 255
            ro, ry, rm = self.o[s].composite_ex(fr[b], bg, bgblur=k)
            tag = (ids, b, s, self.t[s], m.fx[s], k)
            assert np.array_equal(mask[b], rm), f"mask differs {tag}"
            assert np.array_equal(out[b], ro), f"composite differs {tag}"
            assert np.array_equal(yuyv[b], ry), f"YUYV differs {tag}"
            self.t[s] += 1


def _set_fx(g, m, s, kind="default", k=-1):
    g.set_source_effect(s, kind, k)
    m.fx[s] = (kind, k)


def test_four_combinations_and_follow_ups(emu_lib):
    """camera blur 25 / own image sharp / context image at the context's 7 / green, over calls of varying subsets and
    orders; then a new context strength, a new context image, a cleared own image and a reset to the defaults"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    m = _Effects(4, ctx_bg=bg[::-1].copy(), ctx_k=7)
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=4)
    g.set_background(m.ctx_bg)
    g.set_bgblur(7)
    g.set_sources(4)
    m.own[1] = np.roll(bg, 90, axis=1)
    g.set_source_background(1, m.own[1])
    _set_fx(g, m, 0, "none", 25)
    _set_fx(g, m, 1, "default", 0)
    _set_fx(g, m, 3, "none", 0)
    o = _Oracles(key, W, H, 4)
    for ids in ([0, 1, 2, 3], [3, 1], [2, 0], [1, 3, 0, 2]):
        o.call(g, ids, m)
    g.set_bgblur(11)                                   # source 2 follows
    m.ctx_k = 11
    o.call(g, [2, 0, 1], m)
    m.ctx_bg = bg[:, ::-1].copy()
    g.set_background(m.ctx_bg)
    o.call(g, [2, 3], m)
    g.set_source_background(1, None)                  # source 1: the context image, sharp (its own strength 0)
    del m.own[1]
    o.call(g, [1, 2], m)
    _set_fx(g, m, 0)                                  # back to the defaults: the context image at 11
    o.call(g, [0, 1, 2, 3], m)
    g.close()


def test_strength_classes_in_one_call(emu_lib):
    """strengths 1, 3, 31, 33 and 255 in one call: both Gaussian launch classes, camera blur and still images"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    ks = [1, 3, 31, 33, 255]
    m = _Effects(10, ctx_bg=bg[::-1].copy(), ctx_k=0)
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=5)
    g.set_background(m.ctx_bg)
    g.set_sources(10)
    for i, k in enumerate(ks):
        _set_fx(g, m, i, "none", k)                   # camera blur at k
        if i % 2:
            m.own[5 + i] = np.roll(bg, 40 * i, axis=0)
            g.set_source_background(5 + i, m.own[5 + i])
        _set_fx(g, m, 5 + i, "default", k)            # own image or the context image at k
    o = _Oracles(key, W, H, 10)
    o.call(g, [0, 1, 2, 3, 4], m)
    o.call(g, [9, 8, 7, 6, 5], m)
    o.call(g, [4, 5, 0, 9, 2], m)
    g.close()


def test_effect_errors_and_resets(emu_lib):
    key, W, H = "meet_lite", 320, 240
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    L = emu_lib
    assert L.bsb_set_source_effect(g._h, 0, 0, -1) == 0 and b"set_sources" in L.bsb_last_error()
    g.set_sources(3)
    bad = [(3, 0, -1, b"out of range"), (-1, 0, -1, b"out of range"), (0, 2, -1, b"unknown source background"),
           (0, -1, -1, b"unknown source background"), (0, 0, 2, b"strength"), (0, 0, 256, b"strength"), (0, 0, 257, b"strength"),
           (0, 1, -2, b"strength")]
    for s, kind, k, msg in bad:
        assert L.bsb_set_source_effect(g._h, s, kind, k) == 0, (s, kind, k)
        assert msg in L.bsb_last_error(), (s, kind, k, L.bsb_last_error())
    with pytest.raises(api.BackscrubError, match="unknown background"):
        g.set_source_effect(0, "blur")
    # still usable; set_sources resets every effect to (default, -1)
    bg = synth.background()
    g.set_background(bg)
    g.set_source_effect(0, "none", 0)
    g.set_source_effect(1, "none", 9)
    g.set_sources(3)
    o = [po.MaskGen(model_path(key), W, H) for _ in range(2)]
    frames = np.stack([_frame(W, H, s, 0) for s in (0, 1)])
    out, yuyv, mask = g.composite_sources(frames, [0, 1])
    for b in range(2):
        ro, ry, rm = o[b].composite(frames[b], bg)
        assert np.array_equal(out[b], ro) and np.array_equal(yuyv[b], ry) and np.array_equal(mask[b], rm), b
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


def _nv12_frame(W, H, t, s):
    yv = synth.yuyv_frame(W, H, t=t, stream=s)
    return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)


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


class _Dev:
    """device camera frames (YUYV, or NV12 with a layout) of each source, and one plain batch-1 context per source set up
    by the rule as the reference"""

    def __init__(self, lib, key, W, H, n_sources, max_batch, ctx_k, fx, own, fmt="yuyv", layout=None):
        import torch
        self.torch, self.lib, self.key, self.W, self.H, self.fmt = torch, lib, key, W, H, fmt
        bg = synth.background()
        self.m = _Effects(n_sources, ctx_bg=bg[::-1].copy(), ctx_k=ctx_k)
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch)
        self.g.set_background(self.m.ctx_bg)
        self.g.set_bgblur(ctx_k)
        self.g.set_sources(n_sources)
        for s in own:
            self.m.own[s] = np.roll(bg, 37 * s, axis=1)
            self.g.set_source_background(s, self.m.own[s])
        for s, (kind, k) in fx.items():
            _set_fx(self.g, self.m, s, kind, k)
        self.ref = {}
        self.t = [0] * n_sources
        dev = "cuda:0"
        self.fn = W * H * 3 // 2
        self.pitch, self.uv, self.stride = layout if layout else (W, W * H, self.fn)
        if fmt == "nv12":
            self.d_in = torch.empty(max_batch * self.stride, dtype=torch.uint8, device=dev)
            self.d_vid = torch.empty(max_batch * self.fn, dtype=torch.uint8, device=dev)
        else:
            self.d_in = torch.empty((max_batch, H, W, 2), dtype=torch.uint8, device=dev)
            self.d_vid = torch.empty((max_batch, H, W, 2), dtype=torch.uint8, device=dev)
        self.d_out = torch.empty((max_batch, H, W, 3), dtype=torch.uint8, device=dev)
        self.d_mask = torch.empty((max_batch, H, W), dtype=torch.uint8, device=dev)

    def plain(self, s):
        """the reference context of source s, (re)configured to the rule"""
        bg, k = self.m.setup(s)
        if s not in self.ref:
            c = api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1)
            if bg is not None:
                c.set_background(bg)
            vid = self.fn if self.fmt == "nv12" else self.W * self.H * 2
            cam = self.stride if self.fmt == "nv12" else self.W * self.H * 2
            bufs = [self.torch.empty(n, dtype=self.torch.uint8, device="cuda:0") for n in (cam, self.W * self.H * 3, vid, self.W * self.H)]
            self.ref[s] = [c, bufs, bg is None, None]
        r = self.ref[s]
        assert r[2] == (bg is None), "a reference context cannot drop its background"
        if r[3] != k:
            r[0].set_bgblur(k)
            r[3] = k
        return r[0], r[1]

    def frame(self, s, t):
        return _nv12_frame(self.W, self.H, t, s) if self.fmt == "nv12" else synth.yuyv_frame(self.W, self.H, t=t, stream=s)

    def load(self, ids):
        host = np.stack([self.frame(s, self.t[s]) for s in ids])
        if self.fmt == "nv12":
            buf = _pitched(host, self.pitch, self.uv, self.stride)
            self.d_in[:buf.size].copy_(self.torch.from_numpy(buf))
        else:
            self.d_in[:len(ids)].copy_(self.torch.from_numpy(host))
        return host

    def run(self, ids, sync=True):
        n = len(ids)
        if self.fmt == "nv12":
            self.g.composite_sources_nv12_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(), self.d_mask.data_ptr(),
                                                 sync=sync, pitch=self.pitch, uv_offset=self.uv, in_stride=self.stride)
        else:
            self.g.composite_sources_yuyv_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(),
                                                 self.d_mask.data_ptr(), sync=sync)

    def results(self, n):
        vid = self.d_vid.cpu().numpy().reshape(-1)[:n * self.fn].reshape(n, -1) if self.fmt == "nv12" else self.d_vid[:n].cpu().numpy()
        return self.d_out[:n].cpu().numpy(), vid, self.d_mask[:n].cpu().numpy()

    def check(self, ids, got, sample=None):
        out, vid, mask = got
        for b, s in enumerate(ids):
            if sample is not None and s not in sample:
                self.t[s] += 1
                continue
            c, (r_in, r_out, r_vid, r_mask) = self.plain(s)
            fr = self.frame(s, self.t[s])
            r_in[:fr.size].copy_(self.torch.from_numpy(fr.reshape(-1)))
            if self.fmt == "nv12":
                c.composite_nv12_device(1, r_in.data_ptr(), r_out.data_ptr(), r_vid.data_ptr(), r_mask.data_ptr(), sync=True)
            else:
                c.composite_yuyv_device(1, r_in.data_ptr(), r_out.data_ptr(), r_vid.data_ptr(), r_mask.data_ptr(), sync=True)
            tag = (ids, b, s, self.t[s], self.m.fx[s])
            assert np.array_equal(mask[b].reshape(-1), r_mask.cpu().numpy()), f"mask differs {tag}"
            assert np.array_equal(out[b].reshape(-1), r_out.cpu().numpy()), f"composite differs {tag}"
            assert np.array_equal(vid[b].reshape(-1), r_vid.cpu().numpy()), f"video output differs {tag}"
            self.t[s] += 1

    def all_blur(self, ids):
        """every frame of the call blurs its camera frame: the call converts its frames to BGR (not read in place)"""
        return all(self.m.setup(s)[0] is None and self.m.setup(s)[1] > 0 for s in ids)

    def step(self, ids, sample=None):
        self.load(ids)
        self.run(ids)
        self.check(ids, self.results(len(ids)), sample=sample)

    def close(self):
        self.g.close()
        for r in self.ref.values():
            r[0].close()


# camera blur 25 (unrolled fused) / own image sharp / context image at the context's 7 / green / camera blur 9 (fused
# loops) / own image at the context's 7 / camera blur 45 (rows + columns) / context image at 13
MIXED = {0: ("none", 25), 1: ("default", 0), 3: ("none", 0), 4: ("none", 9), 6: ("none", 45), 7: ("default", 13)}
MIXED_OWN = (1, 5)
MIXED_CALLS = ([0, 1, 2, 3, 4, 5, 6, 7], [7, 5, 3, 1], [6], [6, 0, 4, 1, 7], [3, 2, 1, 0, 4, 5, 6, 7], [5, 4])


@pytest.mark.gpu


def test_gpu_meet_720p_mixed_effects_yuyv(gpu_lib):
    """Meet full 1280x720, 8 sources, YUYV device entry: every mixed call reads the camera YUYV in place (a call whose
    every frame blurs its camera frame converts them to BGR)"""
    d = _Dev(gpu_lib, "meet_full", 1280, 720, 8, 8, 7, MIXED, MIXED_OWN)
    for ids in MIXED_CALLS:
        d.step(ids)
        assert d.g.yuyv_native != d.all_blur(ids), ids
    d.close()


@pytest.mark.gpu


@pytest.mark.parametrize("layout", ["packed", "pitched"])


def test_gpu_meet_720p_mixed_effects_nv12(gpu_lib, layout):
    """the same through the NV12 device entry, packed and with a decoder-pitched layout"""
    W, H = 1280, 720
    lay = None if layout == "packed" else (1536, 1536 * 736, 1536 * 736 + 1536 * H // 2)
    d = _Dev(gpu_lib, "meet_full", W, H, 8, 8, 7, MIXED, MIXED_OWN, fmt="nv12", layout=lay)
    for ids in MIXED_CALLS[:4]:
        d.step(ids)
        assert d.g.yuyv_native != d.all_blur(ids), ids
    d.close()


@pytest.mark.gpu


def test_gpu_nv12_layout_without_tma_mixed_effects(gpu_lib):
    """NV12 sources calls on a row pitch that is not a multiple of 16: the post kernel cannot read the frames in place, so
    they are converted to BGR and the camera-blur slots must carry the YUYV that call's post kernel copies.  Sources 1 and
    2 follow the context's strength 25 with no image (the context-wide camera blur of a sources call)."""
    W, H, pitch = 1280, 720, 1288
    lay = (pitch, pitch * H, pitch * H + pitch * H // 2)
    fx = {0: ("none", 9), 1: ("none", -1), 2: ("none", -1), 3: ("default", 0)}
    d = _Dev(gpu_lib, "meet_lite", W, H, 4, 4, 25, fx, (3,), fmt="nv12", layout=lay)
    for ids in ([0, 1, 2, 3], [2, 1], [3, 0, 1]):
        d.step(ids)
        assert not d.g.yuyv_native, ids
    d.close()


@pytest.mark.gpu


def test_gpu_graph_replayed_for_new_strengths(gpu_lib):
    """same buffers and n: a strength moving 7 -> 25 -> 9 within the fused class issues no launches; 25 -> 45 (the
    row / column class) captures a new graph; every call is right"""
    d = _Dev(gpu_lib, "meet_lite", 640, 480, 3, 3, 0, {0: ("none", 7), 1: ("none", 3)}, (2,))
    ids = [0, 1, 2]
    d.step(ids)
    for k in (25, 9):
        _set_fx(d.g, d.m, 0, "none", k)
        d.load(ids)
        l0 = gpu_lib.bsb_total_launches()
        d.run(ids)
        assert gpu_lib.bsb_total_launches() == l0, k
        d.check(ids, d.results(3))
    _set_fx(d.g, d.m, 0, "none", 25)
    d.step(ids)
    _set_fx(d.g, d.m, 0, "none", 45)
    d.load(ids)
    l0 = gpu_lib.bsb_total_launches()
    d.run(ids)
    assert gpu_lib.bsb_total_launches() > l0
    d.check(ids, d.results(3))
    d.close()


@pytest.mark.gpu


def test_gpu_bgr_fallback_mixed_effects(gpu_lib):
    """width 1288: no TMA path, the camera frames are converted to BGR first; mixed effects are still right"""
    d = _Dev(gpu_lib, "meet_lite", 1288, 720, 8, 8, 7, MIXED, MIXED_OWN)
    for ids in MIXED_CALLS[:3]:
        d.step(ids)
        assert not d.g.yuyv_native
    d.close()


@pytest.mark.gpu


def test_gpu_64_sources_mixed(gpu_lib):
    fx = {}
    for s in range(64):
        fx[s] = [("none", 25), ("default", -1), ("none", 0), ("default", 33), ("none", 5)][s % 5]
    d = _Dev(gpu_lib, "meet_lite", 640, 480, 64, 64, 7, fx, range(0, 64, 3))
    sample = {0, 1, 2, 3, 4, 17, 42, 62, 63}
    d.step(list(range(64)), sample=sample)
    d.step(list(range(63, -1, -1)), sample=sample)
    d.close()


@pytest.mark.gpu


def test_gpu_host_bgr_entry_matches_device_path(gpu_lib):
    """bsb_composite_sources (host BGR frames) == the YUYV device entry on the same frames, mixed effects"""
    key, W, H = "mlkit", 640, 480
    d = _Dev(gpu_lib, key, W, H, 8, 8, 7, MIXED, MIXED_OWN)
    h = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=8)
    h.set_background(d.m.ctx_bg)
    h.set_bgblur(7)
    h.set_sources(8)
    for s, b in d.m.own.items():
        h.set_source_background(s, b)
    for s, (kind, k) in MIXED.items():
        h.set_source_effect(s, kind, k)
    for ids in MIXED_CALLS[:4]:
        yin = d.load(ids)
        d.run(ids)
        dev = d.results(len(ids))
        bgr = np.stack([api.convert_yuyv_to_bgr(gpu_lib, y) for y in yin])
        host = h.composite_sources(bgr, ids)
        for a, b, what in zip(dev, host, ("composite", "YUYV", "mask")):
            assert np.array_equal(a, b), (ids, what)
    h.close()
    d.close()
