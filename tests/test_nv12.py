"""NV12 camera frames in, NV12 composites out (bsb_composite_nv12*, bsb_composite_sources_nv12_device,
bsb_convert_nv12_to_bgr).

The two definitions (include/backscrub_b200.h) are restated here on top of the oracle: NV12 ingest is the oracle's YUYV
ingest of the YUYV frame built from the Y plane and each pixel's 2x2-block UV pair (pinned against cv2 below), and the NV12
output is the truncating vertical pair average of the oracle's YUYV output.  So the reference result of an NV12 frame is
ref_yuyv_to_nv12(oracle YUYV output of ref_nv12_to_bgr(frame)).

`-m "not gpu"`: the oracle against cv2, and the kernel-logic emulator build against the oracle (device pointers are host
memory there, so the device entries take numpy buffers).  `-m gpu`: the sm_90a library on an H100."""
import ctypes as C

import cv2
import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path

FLAG_EXACT = 16


# ---------------------------------------------------------------------------------------------------------------------
# frames and the reference functions
# ---------------------------------------------------------------------------------------------------------------------
def nv12_frame(W, H, t=0, stream=0):
    """camera NV12 frame [H*3/2, W]: the Y plane of synth.yuyv_frame and the UV pairs of its even rows"""
    yv = synth.yuyv_frame(W, H, t=t, stream=stream)
    return np.concatenate([yv[..., 0], yv[0::2, :, 1]], axis=0)


def ref_nv12_to_bgr(nv12):
    """NV12 ingest: the oracle's YUYV ingest of (Y, the UV pair of the pixel's 2x2 block)"""
    H, W = nv12.shape[0] * 2 // 3, nv12.shape[1]
    yuyv = np.empty((H, W, 2), np.uint8)
    yuyv[..., 0] = nv12[:H]
    yuyv[..., 1] = np.repeat(nv12[H:], 2, axis=0)
    return po.yuyv_to_bgr(yuyv)


def ref_yuyv_to_nv12(yuyv):
    """NV12 output: Y bytes, and bytes 1 / 3 of each YUYV pair averaged over a row pair with truncation"""
    H, W = yuyv.shape[:2]
    rows = yuyv.reshape(H, W * 2).astype(np.uint16)
    uv = ((rows[0::2, 1::2] + rows[1::2, 1::2]) >> 1).astype(np.uint8)
    return np.concatenate([yuyv[..., 0], uv], axis=0)


def pitched(frames, pitch, uv_offset, stride):
    """n tightly packed NV12 frames -> one buffer with the given row pitch / UV plane offset / frame stride (padding 0x5a)"""
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


def _addr(a):
    return a.ctypes.data if a is not None else 0


class _Oracle:
    """one oracle stream per camera: the NV12 reference result of each frame"""

    def __init__(self, key, W, H):
        self.o = po.MaskGen(model_path(key), W, H)

    def step(self, nv12, bg, **kw):
        out, yuyv, mask = self.o.composite_ex(ref_nv12_to_bgr(nv12), bg, **kw)
        return out, ref_yuyv_to_nv12(yuyv), mask, self.o.ofinal


# ---------------------------------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(2, 2), (64, 48), (642, 480)])
def test_nv12_ingest_is_cv2(W, H):
    rng = np.random.default_rng(W * 1000 + H)
    nv12 = rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
    codes = np.array([0, 16, 235, 240, 255], np.uint8)
    nv12.flat[: min(nv12.size, 40)] = np.resize(codes, min(nv12.size, 40))
    nv12[H:].flat[:10] = np.resize(codes[::-1], 10)
    assert np.array_equal(ref_nv12_to_bgr(nv12), cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12))


def test_nv12_output_definition():
    rng = np.random.default_rng(7)
    H, W = 6, 8
    yuyv = rng.integers(0, 256, (H, W, 2), dtype=np.uint8)
    want = np.empty((H * 3 // 2, W), np.uint8)
    for y in range(H):
        for x in range(W):
            want[y, x] = yuyv[y, x, 0]
    for r in range(H // 2):
        for j in range(W // 2):
            for k, byte in enumerate((1, 3)):
                a = int(yuyv[2 * r].reshape(-1)[4 * j + byte]); b = int(yuyv[2 * r + 1].reshape(-1)[4 * j + byte])
                want[H + r, 2 * j + k] = (a + b) >> 1
    assert np.array_equal(ref_yuyv_to_nv12(yuyv), want)


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def test_emu_convert_nv12_to_bgr(emu_lib):
    for W, H in ((2, 2), (64, 48), (322, 240)):
        nv12 = np.random.default_rng(W).integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
        assert np.array_equal(api.convert_nv12_to_bgr(emu_lib, nv12), ref_nv12_to_bgr(nv12)), (W, H)


def _check(g, b, got, want):
    out, nv, mask = got
    ro, rn, rm, rf = want
    assert np.array_equal(g.stage_u8(2, b), rf), f"smoother state differs (frame {b})"
    if mask is not None:
        assert np.array_equal(mask[b], rm), f"mask differs (frame {b})"
    if out is not None:
        assert np.array_equal(out[b], ro), f"composite differs (frame {b})"
    if nv is not None:
        assert np.array_equal(nv[b], rn), f"NV12 differs (frame {b})"


@pytest.mark.parametrize("key", ["meet_lite", "mlkit"])
def test_emu_composite_nv12_matches_oracle(emu_lib, key):
    W, H = 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    g.set_background(bg)
    o = _Oracle(key, W, H)
    for call in range(2):
        frames = np.stack([nv12_frame(W, H, t=2 * call + b) for b in range(2)])
        got = g.composite_nv12(frames)
        for b in range(2):
            _check(g, b, got, o.step(frames[b], bg))
    g.close()


@pytest.mark.parametrize("mode", ["flip_resize", "camera_blur", "pitched"])
def test_emu_composite_nv12_options(emu_lib, mode):
    key, W, H, n = "meet_lite", 320, 240, 2
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=n)
    o = _Oracle(key, W, H)
    kw = {}
    if mode == "flip_resize":
        g.set_background(bg)
        g.set_output(flip_h=True, out_size=(160, 120))
        kw = dict(flip_h=True, out_size=(160, 120))
    elif mode == "camera_blur":
        g.set_bgblur(7)
        bg, kw = None, dict(bgblur=7)
    else:
        g.set_background(bg)
    ow, oh = g.out_width, g.out_height
    for call in range(2):
        frames = np.stack([nv12_frame(W, H, t=2 * call + b) for b in range(n)])
        if mode == "pitched":
            pitch, uv = W + 64, (W + 64) * (H + 8)
            stride = uv + pitch * (H // 2) + 32
            buf = pitched(frames, pitch, uv, stride)
        else:
            pitch, uv, stride = W, W * H, W * H * 3 // 2
            buf = np.ascontiguousarray(frames).reshape(-1)
        out = np.empty((n, oh, ow, 3), np.uint8)
        nv = np.empty((n, oh * 3 // 2, ow), np.uint8)
        mask = np.empty((n, H, W), np.uint8)
        g.composite_nv12_device(n, _addr(buf), _addr(out), _addr(nv), _addr(mask), sync=True, pitch=pitch, uv_offset=uv, in_stride=stride)
        for b in range(n):
            _check(g, b, (out, nv, mask), o.step(frames[b], bg, **kw))
    g.close()


def test_emu_sources_nv12(emu_lib):
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    g.set_background(bg[::-1].copy())
    g.set_sources(3)
    g.set_source_background(1, bg)
    bg_of = {0: bg[::-1].copy(), 1: bg, 2: bg[::-1].copy()}
    o = [_Oracle(key, W, H) for _ in range(3)]
    t = [0, 0, 0]
    for ids in ([0, 1, 2], [2, 0], [1]):
        n = len(ids)
        frames = np.stack([nv12_frame(W, H, t=t[s], stream=s) for s in ids])
        out = np.empty((n, H, W, 3), np.uint8)
        nv = np.empty((n, H * 3 // 2, W), np.uint8)
        mask = np.empty((n, H, W), np.uint8)
        g.composite_sources_nv12_device(n, ids, _addr(frames), _addr(out), _addr(nv), _addr(mask), sync=True)
        for b, s in enumerate(ids):
            _check(g, b, (out, nv, mask), o[s].step(frames[b], bg_of[s]))
            t[s] += 1
    g.close()


def test_emu_nv12_errors(emu_lib):
    key, W, H = "meet_lite", 320, 240
    lib = emu_lib
    g = api.MaskGen(lib, model_path(key), W, H, max_batch=2)
    fr = np.stack([nv12_frame(W, H, t=b) for b in range(2)])
    out = np.empty((2, H, W, 3), np.uint8); nv = np.empty((2, H * 3 // 2, W), np.uint8); mask = np.empty((2, H, W), np.uint8)

    def call(n=1, p=W, uv=W * H, st=W * H * 3 // 2, frames=fr, nv_out=nv):
        return lib.bsb_composite_nv12_device(g._h, n, _addr(frames) or None, p, uv, st, _addr(out), W * H * 3, _addr(nv_out) or None,
                                             W * H * 3 // 2, _addr(mask), W * H, 1)

    bad = [dict(p=W - 2), dict(uv=W * H - 16), dict(st=W * H * 3 // 2 - 1), dict(n=0), dict(n=3)]
    for kw in bad:
        assert call(**kw) == 0, kw
        assert lib.bsb_last_error().decode(), kw
    assert lib.bsb_composite_nv12_device(g._h, 1, None, W, W * H, W * H * 3 // 2, None, 0, None, 0, _addr(mask), W * H, 1) == 0
    assert lib.bsb_composite_sources_nv12_device(g._h, 1, (C.c_int * 1)(0), _addr(fr), W, W * H, W * H * 3 // 2, None, 0, None, 0,
                                                 _addr(mask), W * H, 1) == 0
    assert b"set_sources" in lib.bsb_last_error()
    g.set_sources(2)
    assert lib.bsb_composite_sources_nv12_device(g._h, 2, (C.c_int * 2)(1, 1), _addr(fr), W, W * H, W * H * 3 // 2, None, 0, None, 0,
                                                 _addr(mask), W * H, 1) == 0
    assert b"distinct" in lib.bsb_last_error()
    g.set_output(out_size=(162, 121))
    assert call(nv_out=nv) == 0 and b"even" in lib.bsb_last_error()
    g.set_output()
    # still usable: the first valid call is the stream's first frame
    assert call() == 1
    ro, rn, rm, _ = _Oracle(key, W, H).step(fr[0], np.dstack([np.zeros((H, W), np.uint8), np.full((H, W), 255, np.uint8),
                                                              np.zeros((H, W), np.uint8)]))
    assert np.array_equal(mask[0], rm) and np.array_equal(out[0], ro) and np.array_equal(nv[0], rn)
    g.close()
    odd = api.MaskGen(lib, model_path(key), W, H + 1, max_batch=1)
    fo = np.zeros(W * (H + 1) * 2, np.uint8)
    assert lib.bsb_composite_nv12_device(odd._h, 1, _addr(fo), W, W * (H + 1), W * (H + 1) * 3 // 2 + W, None, 0, None, 0, None, 0, 1) == 0
    assert b"even" in lib.bsb_last_error()
    odd.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


class _GpuPair:
    """an NV12 context and a BGR context of the same configuration: the NV12 call must give the BGR call's composite and
    mask on ref_nv12_to_bgr(frames), and the NV12 of its YUYV"""

    def __init__(self, lib, key, W, H, n, flags=0, bgblur=0, output=None, bg=True):
        import torch
        self.torch, self.lib, self.W, self.H, self.n = torch, lib, W, H, n
        self.bg = synth.background() if bg else None
        self.g = [api.MaskGen(lib, model_path(key), W, H, max_batch=n, flags=flags) for _ in range(2)]
        for g in self.g:
            if bg:
                g.set_background(self.bg)
            if bgblur:
                g.set_bgblur(bgblur)
            if output:
                g.set_output(**output)
        self.ow, self.oh = self.g[0].out_width, self.g[0].out_height
        dev = "cuda:0"
        u8 = torch.uint8
        self.d_bgr = torch.empty((n, H, W, 3), dtype=u8, device=dev)
        self.d_out = [torch.empty((n, self.oh, self.ow, 3), dtype=u8, device=dev) for _ in range(2)]
        self.d_nv = torch.empty((n, self.oh * 3 // 2, self.ow), dtype=u8, device=dev)
        self.d_yuyv = torch.empty((n, self.oh, self.ow, 2), dtype=u8, device=dev)
        self.d_mask = [torch.empty((n, H, W), dtype=u8, device=dev) for _ in range(2)]

    def run(self, frames, pitch=None, uv_offset=None, want=("out", "nv12", "mask")):
        torch = self.torch
        n, W, H = len(frames), self.W, self.H
        if pitch is None:
            pitch, uv_offset, stride = W, W * H, W * H * 3 // 2
            host = np.ascontiguousarray(frames).reshape(-1)
        else:
            stride = uv_offset + pitch * (H // 2)
            host = pitched(frames, pitch, uv_offset, stride)
        d_in = torch.from_numpy(host).to("cuda:0")
        self.g[0].composite_nv12_device(n, d_in.data_ptr(), self.d_out[0].data_ptr() if "out" in want else 0,
                                        self.d_nv.data_ptr() if "nv12" in want else 0, self.d_mask[0].data_ptr() if "mask" in want else 0,
                                        sync=True, pitch=pitch, uv_offset=uv_offset, in_stride=stride)
        native = self.g[0].yuyv_native
        bgr = np.stack([ref_nv12_to_bgr(f) for f in frames])
        self.d_bgr[:n].copy_(torch.from_numpy(bgr))
        self.g[1].composite_device(n, self.d_bgr.data_ptr(), self.d_out[1].data_ptr(), self.d_yuyv.data_ptr(), self.d_mask[1].data_ptr(),
                                   sync=True)
        ref_out, ref_mask = self.d_out[1][:n].cpu().numpy(), self.d_mask[1][:n].cpu().numpy()
        ref_yuyv = self.d_yuyv[:n].cpu().numpy()
        if "out" in want:
            assert np.array_equal(self.d_out[0][:n].cpu().numpy(), ref_out), "composite differs from the BGR call"
        if "mask" in want:
            assert np.array_equal(self.d_mask[0][:n].cpu().numpy(), ref_mask), "mask differs from the BGR call"
        if "nv12" in want:
            nv = self.d_nv[:n].cpu().numpy()
            for b in range(n):
                assert np.array_equal(nv[b], ref_yuyv_to_nv12(ref_yuyv[b])), f"NV12 differs from the YUYV output (frame {b})"
        return native, ref_out, ref_yuyv, ref_mask

    def close(self):
        for g in self.g:
            g.close()


def _oracle_frames(key, W, H, frames, got, bg, count, flags_kw=None):
    """the first `count` frames of a fresh stream against the oracle"""
    o = _Oracle(key, W, H)
    out, yuyv, mask = got
    for b in range(count):
        ro, rn, rm, _ = o.step(frames[b], bg, **(flags_kw or {}))
        assert np.array_equal(mask[b], rm), f"mask differs from the oracle (frame {b})"
        assert np.array_equal(out[b], ro), f"composite differs from the oracle (frame {b})"
        assert np.array_equal(ref_yuyv_to_nv12(yuyv[b]), rn), f"NV12 differs from the oracle (frame {b})"


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["packed", "nvdec_pitched"])
def test_gpu_meet_720p_nv12_native(gpu_lib, layout):
    """Meet full 1280x720, 32 frames per call, NV12 read and written by the TMA post kernel; pitched like a hardware
    decoder surface (pitch 1536, UV plane at 1536 x 736)"""
    W, H, n = 1280, 720, 32
    p = _GpuPair(gpu_lib, "meet_full", W, H, n)
    frames = np.stack([nv12_frame(W, H, t=t) for t in range(n)])
    kw = dict(pitch=1536, uv_offset=1536 * 736) if layout == "nvdec_pitched" else {}
    native, out, yuyv, mask = p.run(frames, **kw)
    assert native, "the NV12 call should read the camera frames in place"
    _oracle_frames("meet_full", W, H, frames, (out, yuyv, mask), p.bg, 3)
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H,n,flags", [("meet_full", 1296, 712, 4, 0), ("bodypix", 3840, 2160, 2, FLAG_EXACT)])
def test_gpu_ragged_and_large(gpu_lib, key, W, H, n, flags):
    p = _GpuPair(gpu_lib, key, W, H, n, flags=flags)
    frames = np.stack([nv12_frame(W, H, t=t) for t in range(n)])
    native, out, yuyv, mask = p.run(frames)
    assert native
    _oracle_frames(key, W, H, frames, (out, yuyv, mask), p.bg, 1)
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("want", [("nv12",), ("mask",), ("out",), ("out", "nv12", "mask")])
def test_gpu_output_subsets(gpu_lib, want):
    W, H, n = 1280, 720, 4
    p = _GpuPair(gpu_lib, "meet_lite", W, H, n)
    native, *_ = p.run(np.stack([nv12_frame(W, H, t=t) for t in range(n)]), want=want)
    assert native
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["post_tma_off", "flip_resize", "camera_blur", "width_not_16"])
def test_gpu_fallbacks(gpu_lib, mode):
    key, W, H, n = "meet_lite", 1280, 720, 3
    kw = {}
    if mode == "post_tma_off":
        gpu_lib.bsb_set_tuning(b"post_tma", 0)
    elif mode == "flip_resize":
        kw = dict(output=dict(flip_h=True, out_size=(960, 540)))
    elif mode == "camera_blur":
        kw = dict(bg=False, bgblur=7)
    else:
        W = 1288
    try:
        p = _GpuPair(gpu_lib, key, W, H, n, **kw)
        frames = np.stack([nv12_frame(W, H, t=t) for t in range(n)])
        native, out, yuyv, mask = p.run(frames)
    finally:
        gpu_lib.bsb_set_tuning(b"post_tma", 1)
    if mode == "flip_resize":
        assert native, "flip / resize keep the NV12 read in place; only the NV12 output is derived after the tail"
    else:
        assert not native, "the BGR frame must be materialised here"
    ex = {"flip_resize": dict(flip_h=True, out_size=(960, 540)), "camera_blur": dict(bgblur=7)}.get(mode, {})
    _oracle_frames(key, W, H, frames, (out, yuyv, mask), p.bg, 2, ex)
    p.close()


@pytest.mark.gpu
def test_gpu_graphs_yuyv_and_nv12_on_same_buffers(gpu_lib):
    """a YUYV call and an NV12 call on the same device pointers never replay each other's graph; a repeated NV12 call
    replays its own (no new launches issued, same launches per call)"""
    import torch
    key, W, H, n = "meet_lite", 1280, 720, 2
    bg = synth.background()
    g = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=n)
    g.set_background(bg)
    o = _Oracle(key, W, H)
    d_in = torch.empty(n * W * H * 2, dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda:0")
    d_vid = torch.empty(n * W * H * 2, dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((n, H, W), dtype=torch.uint8, device="cuda:0")
    t = 0
    lpc = None
    for it in range(4):
        if it % 2 == 0:
            fr = np.stack([nv12_frame(W, H, t=t + b) for b in range(n)])
            d_in[: fr.size].copy_(torch.from_numpy(fr.reshape(-1)))
            l0 = gpu_lib.bsb_total_launches()
            g.composite_nv12_device(n, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr(), sync=True)
            if it == 2:
                assert gpu_lib.bsb_total_launches() == l0, "the repeated NV12 call should replay its graph"
                assert g.launches_per_call == lpc
            lpc = g.launches_per_call
            out, nv, mask = d_out.cpu().numpy(), d_vid[: n * W * H * 3 // 2].cpu().numpy().reshape(n, -1, W), d_mask.cpu().numpy()
            for b in range(n):
                ro, rn, rm, _ = o.step(fr[b], bg)
                assert np.array_equal(mask[b], rm) and np.array_equal(out[b], ro) and np.array_equal(nv[b], rn), (it, b)
        else:
            # the same stream continues as YUYV frames (the YUYV of the NV12 frames' BGR: same pixels for the oracle)
            yv = np.stack([synth.yuyv_frame(W, H, t=t + b) for b in range(n)])
            d_in.copy_(torch.from_numpy(yv.reshape(-1)))
            g.composite_yuyv_device(n, d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr(), sync=True)
            out, y2, mask = d_out.cpu().numpy(), d_vid.cpu().numpy().reshape(n, H, W, 2), d_mask.cpu().numpy()
            for b in range(n):
                ro, ry, rm = o.o.composite_ex(po.yuyv_to_bgr(yv[b]), bg)
                assert np.array_equal(mask[b], rm) and np.array_equal(out[b], ro) and np.array_equal(y2[b], ry), (it, b)
        t += n
    g.close()


@pytest.mark.gpu
def test_gpu_64_sources_nv12_match_plain_contexts(gpu_lib):
    import torch
    key, W, H, S = "meet_lite", 640, 480, 64
    bg = synth.background()
    g = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=S)
    g.set_background(bg[::-1].copy())
    g.set_sources(S)
    own = {s: np.roll(bg, 37 * s, axis=1) for s in range(0, S, 3)}
    for s, b in own.items():
        g.set_source_background(s, b)
    fn = W * H * 3 // 2
    d_in = torch.empty(S * fn, dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty((S, H, W, 3), dtype=torch.uint8, device="cuda:0")
    d_nv = torch.empty(S * fn, dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((S, H, W), dtype=torch.uint8, device="cuda:0")
    sample = (0, 1, 17, 42, 62, 63)
    ref = {}
    for s in sample:
        c = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=1)
        c.set_background(own.get(s, bg[::-1].copy()))
        ref[s] = (c, [torch.empty(k, dtype=torch.uint8, device="cuda:0") for k in (fn, W * H * 3, fn, W * H)])
    for t, ids in enumerate((list(range(S)), list(range(S - 1, -1, -1)))):
        fr = np.stack([nv12_frame(W, H, t=t, stream=s) for s in ids])
        d_in.copy_(torch.from_numpy(fr.reshape(-1)))
        g.composite_sources_nv12_device(S, ids, d_in.data_ptr(), d_out.data_ptr(), d_nv.data_ptr(), d_mask.data_ptr(), sync=True)
        assert g.yuyv_native
        out, nv, mask = d_out.cpu().numpy(), d_nv.cpu().numpy().reshape(S, -1), d_mask.cpu().numpy()
        for b, s in enumerate(ids):
            if s not in ref:
                continue
            c, (ri, ro, rn, rm) = ref[s]
            ri.copy_(torch.from_numpy(fr[b].reshape(-1)))
            c.composite_nv12_device(1, ri.data_ptr(), ro.data_ptr(), rn.data_ptr(), rm.data_ptr(), sync=True)
            assert np.array_equal(mask[b].reshape(-1), rm.cpu().numpy()), (t, s)
            assert np.array_equal(out[b].reshape(-1), ro.cpu().numpy()), (t, s)
            assert np.array_equal(nv[b], rn.cpu().numpy()), (t, s)
    for c, _ in ref.values():
        c.close()
    g.close()


@pytest.mark.gpu
def test_gpu_host_entry_matches_device_entry(gpu_lib):
    import torch
    key, W, H, n = "mlkit", 640, 480, 3
    bg = synth.background()
    gs = [api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=n) for _ in range(2)]
    for g in gs:
        g.set_background(bg)
    fn = W * H * 3 // 2
    d_in = torch.empty(n * fn, dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda:0")
    d_nv = torch.empty(n * fn, dtype=torch.uint8, device="cuda:0")
    d_mask = torch.empty((n, H, W), dtype=torch.uint8, device="cuda:0")
    for call in range(2):
        fr = np.stack([nv12_frame(W, H, t=call * n + b) for b in range(n)])
        host = gs[0].composite_nv12(fr)
        d_in.copy_(torch.from_numpy(fr.reshape(-1)))
        gs[1].composite_nv12_device(n, d_in.data_ptr(), d_out.data_ptr(), d_nv.data_ptr(), d_mask.data_ptr(), sync=True)
        dev = (d_out.cpu().numpy(), d_nv.cpu().numpy().reshape(n, -1, W), d_mask.cpu().numpy())
        for a, b, what in zip(host, dev, ("composite", "NV12", "mask")):
            assert np.array_equal(a, b), (call, what)
    for g in gs:
        g.close()
