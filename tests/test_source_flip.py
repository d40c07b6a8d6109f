"""Per-source mirroring (bsb_set_source_flip): each camera of a sources context picks its own cv::flip.  Frame b of a
sources call, from source s, must give exactly the bytes a plain context gives for that camera's stream when set up the
same way (background, effect, output size) plus bsb_set_output(flip_h_s, flip_v_s): composite, YUYV / NV12 and mask.

`-m "not gpu"`: the kernel-logic emulator build (the fallback post kernel and the per-frame flip tail) vs the oracle.
`-m gpu`: the sm_90a library (k_post_tma mirroring in place, and the tail) vs plain batch-1 contexts."""

import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path

H_, V_ = 1, 2


def _code(flip):
    """(flip_h, flip_v) of a flip code"""
    return bool(flip & H_), bool(flip & V_)


def _set_flip(g, flips, s, code):
    """code None = follow the context, else 0..3"""
    if code is None:
        g.set_source_flip(s)
    else:
        g.set_source_flip(s, flip_h=bool(code & H_), flip_v=bool(code & V_))
    flips[s] = code


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


class _Oracles:
    """one oracle stream per source; source s blends `bgs[s]` (None: its camera frame blurred at ks[s])"""

    def __init__(self, key, W, H, n, bgs, ks, out_size=None):
        self.W, self.H, self.out_size = W, H, out_size
        self.o = [po.MaskGen(model_path(key), W, H) for _ in range(n)]
        self.t = [0] * n
        self.bgs, self.ks = bgs, ks

    def call(self, g, ids, flips, ctx_flip):
        fr = np.stack([synth.frame(self.W, self.H, t=self.t[s], stream=s) for s in ids])
        out, yuyv, mask = g.composite_sources(fr, ids)
        for b, s in enumerate(ids):
            code = ctx_flip if flips[s] is None else flips[s]
            fh, fv = _code(code)
            ro, ry, rm = self.o[s].composite_ex(fr[b], self.bgs[s], bgblur=self.ks[s], flip_h=fh, flip_v=fv, out_size=self.out_size)
            tag = (ids, b, s, self.t[s], code)
            assert np.array_equal(mask[b], rm), f"mask differs {tag}"
            assert np.array_equal(out[b], ro), f"composite differs {tag}"
            assert np.array_equal(yuyv[b], ry), f"YUYV differs {tag}"
            self.t[s] += 1


def _emu_setup(lib, out_size=None):
    """four sources: the context image (follows the context flip), its own image (never flipped), camera blur 9 (H), the
    context image at strength 5 (H | V)"""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    ctx_bg = bg[::-1].copy()
    own = np.roll(bg, 90, axis=1)
    g = api.MaskGen(lib, model_path(key), W, H, max_batch=4)
    g.set_background(ctx_bg)
    if out_size:
        g.set_output(out_size=out_size)
    g.set_sources(4)
    g.set_source_background(1, own)
    g.set_source_effect(2, "none", 9)
    g.set_source_effect(3, "default", 5)
    flips = {0: None}
    for s, code in ((1, 0), (2, H_), (3, H_ | V_)):
        _set_flip(g, flips, s, code)
    o = _Oracles(key, W, H, 4, [ctx_bg, own, None, ctx_bg], [0, 0, 9, 5], out_size)
    return g, o, flips


def _emu_calls(g, o, flips, out_size=None):
    ctx = 0
    for ids in ([0, 1, 2, 3], [3, 1], [2, 0], [1, 3, 0, 2]):
        o.call(g, ids, flips, ctx)
    ctx = V_                                            # source 0 follows the new context flip; the others keep theirs
    g.set_output(flip_v=True, out_size=out_size)
    for ids in ([0, 1, 2, 3], [0], [3, 2, 1]):
        o.call(g, ids, flips, ctx)
    _set_flip(g, flips, 1, None)                        # source 1 follows the context too, source 3 stops mirroring
    _set_flip(g, flips, 3, 0)
    for ids in ([1, 3, 0], [2, 1, 3, 0]):
        o.call(g, ids, flips, ctx)
    _set_flip(g, flips, 2, 0)                           # no frame of the call flipped
    _set_flip(g, flips, 0, 0)
    _set_flip(g, flips, 1, 0)
    o.call(g, [0, 1, 2, 3], flips, ctx)


def test_flips_follow_and_own(emu_lib):
    """flips -1 / 0 / H / H|V, then the context flip changed to V, over calls of varying subsets and orders"""
    g, o, flips = _emu_setup(emu_lib)
    _emu_calls(g, o, flips)
    g.close()


def test_flips_before_resize(emu_lib):
    """the same with a context output size: the per-frame flip is followed by the resize"""
    g, o, flips = _emu_setup(emu_lib, out_size=(240, 180))
    _emu_calls(g, o, flips, out_size=(240, 180))
    g.close()


def test_flip_errors_and_reset(emu_lib):
    key, W, H = "meet_lite", 320, 240
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    L = emu_lib
    assert L.bsb_set_source_flip(g._h, 0, 1) == 0 and b"set_sources" in L.bsb_last_error()
    g.set_sources(3)
    bad = [(3, 0, b"out of range"), (-1, 1, b"out of range"), (0, 4, b"flip"), (0, -2, b"flip"), (1, 7, b"flip")]
    for s, code, msg in bad:
        assert L.bsb_set_source_flip(g._h, s, code) == 0, (s, code)
        assert msg in L.bsb_last_error(), (s, code, L.bsb_last_error())
    with pytest.raises(api.BackscrubError, match="bsb_set_source_flip"):
        g.set_source_flip(5, flip_h=True)
    # still usable; set_sources resets every source to follow the context (no flip here)
    bg = synth.background()
    g.set_background(bg)
    g.set_source_flip(0, flip_h=True)
    g.set_source_flip(1, flip_v=True)
    g.set_sources(3)
    o = [po.MaskGen(model_path(key), W, H) for _ in range(2)]
    frames = np.stack([synth.frame(W, H, t=0, stream=s) for s in (0, 1)])
    out, yuyv, mask = g.composite_sources(frames, [0, 1])
    for b in range(2):
        ro, ry, rm = o[b].composite(frames[b], bg)
        assert np.array_equal(out[b], ro) and np.array_equal(yuyv[b], ry) and np.array_equal(mask[b], rm), b
    g.close()


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
# flip codes of the eight sources (None: follow the context)
FLIPS8 = [None, 0, H_, H_ | V_, V_, None, H_, 0]
CALLS8 = ([0, 1, 2, 3, 4, 5, 6, 7], [7, 5, 3, 1], [6, 0, 4, 2, 1])


class _Dev:
    """a sources context fed by one of the three entry points (device YUYV, device NV12 with a layout, host BGR), and one
    plain batch-1 context per source set up as that source, which mirrors through the stand-alone tail"""

    def __init__(self, lib, key, W, H, n_sources, fmt="yuyv", layout=None, out_size=None, flips=None):
        import torch
        self.torch, self.lib, self.key, self.W, self.H, self.fmt = torch, lib, key, W, H, fmt
        self.out_size = out_size
        self.ow, self.oh = out_size if out_size else (W, H)
        bg = synth.background()
        self.ctx_bg = bg[::-1].copy()
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=n_sources)
        self.g.set_background(self.ctx_bg)
        if out_size:
            self.g.set_output(out_size=out_size)
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
        self.flips = {s: None for s in range(n_sources)}
        for s in range(n_sources):
            if flips and flips[s % len(flips)] is not None:
                _set_flip(self.g, self.flips, s, flips[s % len(flips)])
        self.ctx_flip = 0
        self.ref = {}
        self.t = [0] * n_sources
        dev = "cuda:0"
        self.fn = W * H * 3 // 2
        self.ofn = self.ow * self.oh * 3 // 2
        self.pitch, self.uv, self.stride = layout if layout else (W, W * H, self.fn)
        mb = n_sources
        if fmt == "nv12":
            self.d_in = torch.empty(mb * self.stride, dtype=torch.uint8, device=dev)
            self.d_vid = torch.empty(mb * self.ofn, dtype=torch.uint8, device=dev)
        elif fmt == "yuyv":
            self.d_in = torch.empty((mb, H, W, 2), dtype=torch.uint8, device=dev)
            self.d_vid = torch.empty((mb, self.oh, self.ow, 2), dtype=torch.uint8, device=dev)
        if fmt != "bgr":
            self.d_out = torch.empty((mb, self.oh, self.ow, 3), dtype=torch.uint8, device=dev)
            self.d_mask = torch.empty((mb, H, W), dtype=torch.uint8, device=dev)
        self.host = None

    def set_ctx_flip(self, code):
        fh, fv = _code(code)
        self.g.set_output(fh, fv, self.out_size)
        self.ctx_flip = code

    def code(self, s):
        return self.ctx_flip if self.flips[s] is None else self.flips[s]

    def plain(self, s):
        """the reference context of source s, with its current flip"""
        bg, k = self.fx[s]
        if s not in self.ref:
            c = api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1)
            if bg is not None:
                c.set_background(bg)
            if k:
                c.set_bgblur(k)
            bufs = None
            if self.fmt != "bgr":
                cam = self.stride if self.fmt == "nv12" else self.W * self.H * 2
                vid = self.ofn if self.fmt == "nv12" else self.ow * self.oh * 2
                bufs = [self.torch.empty(n, dtype=self.torch.uint8, device="cuda:0") for n in (cam, self.ow * self.oh * 3, vid, self.W * self.H)]
            self.ref[s] = [c, bufs, None]
        r = self.ref[s]
        if r[2] != self.code(s):
            fh, fv = _code(self.code(s))
            r[0].set_output(fh, fv, self.out_size)
            r[2] = self.code(s)
        return r[0], r[1]

    def frame(self, s, t):
        if self.fmt == "nv12":
            return _nv12_frame(self.W, self.H, t, s)
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
        if self.fmt == "nv12":
            self.g.composite_sources_nv12_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(), self.d_mask.data_ptr(),
                                                 sync=True, pitch=self.pitch, uv_offset=self.uv, in_stride=self.stride)
        elif self.fmt == "yuyv":
            self.g.composite_sources_yuyv_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_vid.data_ptr(),
                                                 self.d_mask.data_ptr(), sync=True)
        else:
            self._res = self.g.composite_sources(self.host, ids)

    def results(self, n):
        if self.fmt == "bgr":
            return self._res
        vid = self.d_vid.cpu().numpy().reshape(-1)[:n * self.ofn].reshape(n, -1) if self.fmt == "nv12" else self.d_vid[:n].cpu().numpy()
        return self.d_out[:n].cpu().numpy(), vid, self.d_mask[:n].cpu().numpy()

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
            tag = (self.fmt, ids, b, s, self.t[s], self.code(s))
            assert np.array_equal(mask[b].reshape(-1), r_mask.reshape(-1)), f"mask differs {tag}"
            assert np.array_equal(out[b].reshape(-1), r_out.reshape(-1)), f"composite differs {tag}"
            assert np.array_equal(vid[b].reshape(-1), r_vid.reshape(-1)), f"video output differs {tag}"
            self.t[s] += 1

    def step(self, ids, sample=None):
        self.load(ids)
        self.run(ids)
        self.check(ids, self.results(len(ids)), sample=sample)

    def close(self):
        self.g.close()
        for r in self.ref.values():
            r[0].close()


@pytest.fixture
def post_tile():
    """k_post_tma's tile width for the contexts of one test (set before they are created), restored afterwards"""
    import backscrub_b200 as bs
    yield lambda tw: bs.set_tuning("post_tile", tw)
    bs.set_tuning("post_tile", 0)


GEOMETRIES = [(1280, 720, 0), (1296, 720, 64), (1296, 720, 128)]
FORMATS = ["yuyv", "nv12", "nv12_pitched", "bgr"]


@pytest.mark.gpu
@pytest.mark.parametrize("geo", GEOMETRIES, ids=["1280x720", "1296x720_tw64", "1296x720_tw128"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_gpu_meet_720p_flips_in_place(gpu_lib, post_tile, geo, fmt):
    """Meet full, 8 sources with mixed flips and effects (context image, own image, camera blur 25, context image at 7):
    every call mixes flipped and unflipped frames and background, person and mixed tiles; k_post_tma mirrors in place, so
    a flipped call issues as many launches as the same call unflipped.  1296x720 has ragged right and bottom tiles."""
    W, H, tw = geo
    post_tile(tw)
    layout = (1536, 1536 * (H + 16), 1536 * (H + 16) + 1536 * H // 2) if fmt == "nv12_pitched" else None
    d = _Dev(gpu_lib, "meet_full", W, H, 8, fmt="nv12" if fmt.startswith("nv12") else fmt, layout=layout, flips=FLIPS8)
    # every call unflipped first: its launch count without a tail
    saved = dict(d.flips)
    for s in range(8):
        _set_flip(d.g, d.flips, s, 0)
    base = {}
    for ids in CALLS8:
        d.step(ids)
        base[tuple(ids)] = d.g.launches_per_call
    for s, code in saved.items():
        _set_flip(d.g, d.flips, s, code)
    for ids in CALLS8:
        d.step(ids)
        if fmt != "bgr":
            assert d.g.yuyv_native, ids
        assert d.g.launches_per_call == base[tuple(ids)], (ids, d.g.launches_per_call, base[tuple(ids)])
    d.set_ctx_flip(H_ | V_)                           # sources 0 and 5 follow
    d.step(CALLS8[0])
    assert d.g.launches_per_call == base[tuple(CALLS8[0])]
    d.set_ctx_flip(V_)
    d.step(CALLS8[2])
    assert d.g.launches_per_call == base[tuple(CALLS8[2])]
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuyv", "nv12"])
def test_gpu_flips_through_tail_without_tma(gpu_lib, fmt):
    """post_tma=0: the post kernel cannot mirror, so the per-frame flip runs in the tail; same bytes as the plain contexts"""
    import backscrub_b200 as bs
    bs.set_tuning("post_tma", 0)
    try:
        d = _Dev(gpu_lib, "meet_full", 1280, 720, 8, fmt=fmt, flips=FLIPS8)
        for ids in CALLS8:
            d.step(ids)
            assert not d.g.yuyv_native, ids
        d.close()
    finally:
        bs.set_tuning("post_tma", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuyv", "nv12"])
def test_gpu_flips_before_resize(gpu_lib, fmt):
    """a context output size: post -> stage -> per-frame flip -> resize -> YUYV (-> NV12)"""
    d = _Dev(gpu_lib, "meet_lite", 1280, 720, 4, fmt=fmt, out_size=(640, 360), flips=[None, H_, V_, 0])
    for ids in ([0, 1, 2, 3], [3, 1], [2, 0, 1]):
        d.step(ids)
    d.set_ctx_flip(H_)
    d.step([0, 1, 2, 3])
    d.close()


@pytest.mark.gpu
def test_gpu_graph_replayed_for_new_flips(gpu_lib):
    """same buffers and n: a call with flipped frames and one without are two graphs (the latter runs the post kernel as
    a plain call does); once both are captured, any new flips replay one of them, and every call is right"""
    d = _Dev(gpu_lib, "meet_full", 1280, 720, 4, flips=[H_, 0, V_, None])
    ids = [0, 1, 2, 3]
    d.step(ids)

    def call(codes, replays):
        for s, code in enumerate(codes):
            _set_flip(d.g, d.flips, s, code)
        d.load(ids)
        l0 = gpu_lib.bsb_total_launches()
        d.run(ids)
        assert (gpu_lib.bsb_total_launches() == l0) == replays, (codes, replays)
        d.check(ids, d.results(4))

    call([H_ | V_, H_, 0, V_], True)
    call([H_, H_, H_, H_], True)
    call([0, 0, 0, 0], False)                         # the first call without flipped frames captures its graph
    call([V_, 0, 0, 0], True)
    call([0, 0, 0, 0], True)
    call([None, None, None, None], True)              # following the context, which is not flipped
    d.set_ctx_flip(H_)                                # drops the graphs: a new capture, then replays again
    d.step(ids)
    call([None, 0, H_ | V_, None], True)
    d.close()


@pytest.mark.gpu
def test_gpu_64_sources_flipped(gpu_lib):
    d = _Dev(gpu_lib, "meet_lite", 640, 480, 64, flips=[None, 0, H_, H_ | V_, V_])
    d.set_ctx_flip(H_)
    sample = {0, 1, 2, 3, 4, 17, 42, 62, 63}
    d.step(list(range(64)), sample=sample)
    d.step(list(range(63, -1, -1)), sample=sample)
    d.close()
