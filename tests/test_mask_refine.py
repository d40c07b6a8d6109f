"""Mask edge refinement (include/backscrub_b200.h, bsb_set_mask_refine): the mask of a refined frame is the joint bilateral
upsample of its small mask guided by its own camera luma.

`ref_refine` restates the definition in numpy (the header and DESIGN.md §4 state it in words), and every refined output
of the library is compared with it byte for byte on fed small masks (bsb_test_feed), and on the small masks the library
itself held (stage 2) where the CNN runs.  The composite, video, BGRA and tail outputs follow from the refined mask by the
references the other post-stage tests use.  The quality tests check on a constructed scene with a known matte that the
refined mask is closer to the truth than the unrefined one, on the restatement and on the library's bytes.
"""
import cv2
import numpy as np
import pytest

import backscrub_b200 as bs
from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path
from tests.test_bgra_output import expect_bgra
from tests.test_feed_post import geo, ref_mask, ref_outputs


# ---------------------------------------------------------------------------------------------------- the definition
def refine_weights(sigma):
    """R_sigma[d] = max(1, floor(256 exp(-d^2 / (2 sigma^2)) + 0.5)), in double"""
    d = np.arange(256, dtype=np.float64)
    return np.maximum(1, np.floor(256.0 * np.exp(-d * d / (2.0 * sigma * sigma)) + 0.5)).astype(np.int64)


def refine_taps(n_roi, n_small):
    """per ROI index: the 4 small indices (clamped; their weight is 0 outside 0..n_small-1) and spatial weights"""
    scale = 1.0 / (n_roi / n_small)                          # cv::resize's source step, as OpenCV computes it
    f = ((np.arange(n_roi) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    a = np.rint((f - s) * np.float32(2048)).astype(np.int64)
    s = s.astype(np.int64)
    w = np.stack([np.maximum(0, 1024 - a), 3072 - a, 1024 + a, np.maximum(0, a - 1024)], 1)
    idx = s[:, None] - 1 + np.arange(4)[None]
    w = np.where((idx >= 0) & (idx < n_small), w, 0)
    return np.clip(idx, 0, n_small - 1), w


def luma(bgr):
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return (4899 * r + 9617 * g + 1868 * b + 8192) >> 14


def ref_refine(g, ofinal, frame, sigma):
    """the W x H mask of a frame refined at strength sigma (0: the unrefined mask, ref_mask); frame: BGR as composited"""
    if sigma == 0:
        return ref_mask(g, ofinal)
    rx, ry, rw, rh = g.roi
    ox, oy, sw, sh = g.out
    s = ofinal[oy:oy + sh, ox:ox + sw].astype(np.int64)
    L = luma(frame)
    gx = rx + ((2 * np.arange(sw) + 1) * rw) // (2 * sw)
    gy = ry + ((2 * np.arange(sh) + 1) * rh) // (2 * sh)
    G = L[np.ix_(gy, gx)]
    R = refine_weights(sigma)
    xi, xw = refine_taps(rw, sw)
    yi, yw = refine_taps(rh, sh)
    Lp = L[ry:ry + rh, rx:rx + rw]
    num = np.zeros((rh, rw), np.int64)
    den = np.zeros((rh, rw), np.int64)
    for i in range(4):
        for j in range(4):
            sp = (yw[:, i][:, None] * xw[:, j][None, :]) >> 12
            ii, jj = yi[:, i][:, None], xi[:, j][None, :]
            w = sp * R[np.abs(Lp - G[ii, jj])]
            assert w.max() < 1 << 20
            num += w * s[ii, jj]
            den += w
    assert den.min() >= 1024 and den.max() < 1 << 24 and num.max() < 1 << 32
    m = np.full((g.H, g.W), 255, np.uint8)
    m[ry:ry + rh, rx:rx + rw] = ((num + (den >> 1)) // den).astype(np.uint8)
    return m


# ---------------------------------------------------------------------------------------------------- fixtures
def small_masks(g, n, seed):
    """hard small masks (0 / 255, as the smoother makes them): blobs with single-pixel islands and holes, a half-plane
    edge on a tile border, and a few frames of random bytes"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        m = np.full((g.oh, g.ow), 255, np.uint8)
        ox, oy, sw, sh = g.out
        if k % 4 == 3:
            m[:] = rng.integers(0, 256, m.shape, dtype=np.uint8)
        elif k % 4 == 2:
            col = ox + int(round((32 * (k // 4 + 1) - g.roi[0]) * sw / g.roi[2]))
            m[:, :min(max(col, 0), g.ow)] = 0
        else:
            yy, xx = np.mgrid[0:g.oh, 0:g.ow]
            cx, cy = ox + sw * rng.uniform(0.3, 0.7), oy + sh * rng.uniform(0.4, 0.8)
            m[((xx - cx) / (0.25 * sw)) ** 2 + ((yy - cy) / (0.4 * sh)) ** 2 < 1] = 0
            pts = rng.integers(0, [g.oh, g.ow], (6, 2))
            m[pts[:, 0], pts[:, 1]] = 255 - m[pts[:, 0], pts[:, 1]]
        out.append(m)
    return np.stack(out)


def camera(W, H, t):
    """a camera frame with edges the small masks do not share"""
    f = synth.frame(W, H, t=t).astype(np.int16)
    f[:, : W // 3] //= 2
    return np.clip(f, 0, 255).astype(np.uint8)


def frames_of(W, H, n, fmt):
    """n camera frames in wire format, and the BGR the composite reads (the fused path's conversion)"""
    yuyv = [synth.yuyv_frame(W, H, t=t) for t in range(n)]
    if fmt == "bgr":
        bgr = [camera(W, H, t) for t in range(n)]
        return np.stack(bgr), bgr
    if fmt == "yuyv":
        return np.stack(yuyv), [po.yuyv_to_bgr(y) for y in yuyv]
    nv12 = [np.concatenate([y[..., 0], y[0::2, :, 1]], axis=0) for y in yuyv]
    return np.stack(nv12), [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in nv12]


def run_fed(c, masks, fmt, frames, want=(True, True, True)):
    c.feed(B.FEED_MASK, masks)
    if fmt == "bgr":
        return c.composite(frames, *want)
    if fmt == "yuyv":
        n, H, W = frames.shape[0], c.height, c.width
        out = np.empty((n, c.out_height, c.out_width, c.out_channels), np.uint8) if want[0] else None
        vid = np.empty((n, c.out_height, c.out_width, 2), np.uint8) if want[1] else None
        mask = np.empty((n, H, W), np.uint8) if want[2] else None
        c.composite_yuyv_into(frames, out, vid, mask)
        return out, vid, mask
    return c.composite_nv12(frames, *want)


def check_call(g, c, masks, sigmas, fmt, frames, bgrs, bg, flip=0, out_size=None, bgra=False, active=True, want=(True, True, True), tag=""):
    out, vid, mask = run_fed(c, masks, fmt, frames, want)
    for b in range(len(masks)):
        rm = ref_refine(g, masks[b], bgrs[b], sigmas[b])
        where = (tag, fmt, b, sigmas[b])
        if mask is not None:
            assert np.array_equal(mask[b], rm), ("mask", where, int((mask[b] != rm).sum()))
        w = rm if active else np.zeros_like(rm)
        ro, rv = ref_outputs(w, bgrs[b], bg, flip, out_size, fmt == "nv12", video=vid is not None)
        if out is not None:
            exp = expect_bgra(bgrs[b], rm, active, flip, out_size) if bgra else ro
            assert np.array_equal(out[b], exp), ("out", where, int((out[b] != exp).sum()))
        if vid is not None:
            assert np.array_equal(vid[b].reshape(-1), rv.reshape(-1)), ("video", where)
    return out, vid, mask


def context(lib, key, W, H, max_batch=8):
    c = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch)
    raw = synth.background()
    c.set_background(raw)
    return c, po.resize_linear_u8(raw, W, H)


# ---------------------------------------------------------------------------------------------------- CPU: definition
def test_restatement_uniform_and_bounds():
    """a small mask uniform over a pixel's taps gives exactly that value; the uint32 bounds hold at every strength"""
    g = geo("meet_lite", 320, 176)
    rng = np.random.default_rng(1)
    frame = rng.integers(0, 256, (g.H, g.W, 3), dtype=np.uint8)
    for v in (0, 1, 77, 254, 255):
        for sigma in (1, 12, 255):
            m = ref_refine(g, np.full((g.oh, g.ow), v, np.uint8), frame, sigma)
            rx, ry, rw, rh = g.roi
            assert (m[ry:ry + rh, rx:rx + rw] == v).all() and (m[:, :rx] == 255).all()


@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def test_emu_weights_and_refusals(emu_lib):
    for sigma in range(1, 256):
        assert np.array_equal(api.mask_refine_weights(emu_lib, sigma), refine_weights(sigma)), sigma
    for bad in (0, -1, 256):
        with pytest.raises(bs.BackscrubError):
            api.mask_refine_weights(emu_lib, bad)
    assert not emu_lib.bsb_mask_refine_weights(8, None)
    c, _ = context(emu_lib, "meet_lite", 160, 128, 2)
    try:
        for bad in (-1, 256, 1000):
            with pytest.raises(bs.BackscrubError, match="strength"):
                c.set_mask_refine(bad)
        with pytest.raises(bs.BackscrubError, match="no sources"):
            c.set_source_mask_refine(0, 8)
        c.set_sources(3)
        for s, v in ((3, 8), (-1, 8), (0, -2), (0, 256)):
            with pytest.raises(bs.BackscrubError):
                c.set_source_mask_refine(s, v)
        c.set_mask_refine(0)
        c.set_mask_refine(255)
        c.set_source_mask_refine(2, None)
    finally:
        c.close()


def test_emu_refused_where_no_kernel_takes_it(emu_lib):
    """a frame width that is not a multiple of 16 runs the generic post kernel, which does not refine: the call is
    refused, and the same call unrefined runs"""
    W, H = 324, 176
    g = geo("meet_lite", W, H)
    c, bg = context(emu_lib, "meet_lite", W, H, 2)
    try:
        masks = small_masks(g, 2, 3)
        frames, bgrs = frames_of(W, H, 2, "bgr")
        c.set_mask_refine(8)
        c.feed(B.FEED_MASK, masks)
        with pytest.raises(bs.BackscrubError, match="refinement"):
            c.composite(frames)
        c.set_mask_refine(0)
        check_call(g, c, masks, [0, 0], "bgr", frames, bgrs, bg)
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------- CPU: the emulator
@pytest.mark.parametrize("fmt", ["bgr", "yuyv", "nv12"])
@pytest.mark.parametrize("key,W,H", [("meet_lite", 320, 176), ("meet_lite", 160, 128)])
def test_emu_plain(emu_lib, key, W, H, fmt):
    """plain calls at every strength class, off in between; letterboxed ROIs both ways (roi_x > 0, out_x > 0)"""
    g = geo(key, W, H)
    c, bg = context(emu_lib, key, W, H, 4)
    try:
        frames, bgrs = frames_of(W, H, 4, fmt)
        for k, sigma in enumerate((1, 8, 0, 30, 255)):
            c.set_mask_refine(sigma)
            check_call(g, c, small_masks(g, 4, 10 + k), [sigma] * 4, fmt, frames, bgrs, bg, tag=key)
    finally:
        c.close()


def test_emu_outputs(emu_lib):
    """flip + resize tail, BGRA with and without video, the filter off (the refined mask is still stored), a mask-only
    call, and a chunked host-buffer YUYV call"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    c, bg = context(emu_lib, key, W, H, 4)
    try:
        c.set_mask_refine(12)
        s4 = [12] * 4
        for fmt in ("bgr", "nv12"):
            frames, bgrs = frames_of(W, H, 4, fmt)
            c.set_output(True, True, (W // 2, H // 2))
            check_call(g, c, small_masks(g, 4, 20), s4, fmt, frames, bgrs, bg, flip=3, out_size=(W // 2, H // 2), tag="tail")
            c.set_output(False, False, None)
            c.set_out_format("bgra")
            check_call(g, c, small_masks(g, 4, 21), s4, fmt, frames, bgrs, bg, bgra=True, tag="bgra")
            check_call(g, c, small_masks(g, 4, 22), s4, fmt, frames, bgrs, bg, bgra=True, want=(True, False, True), tag="bgra only")
            c.set_out_format("bgr")
            c.set_filter(False)
            check_call(g, c, small_masks(g, 4, 23), s4, fmt, frames, bgrs, bg, active=False, tag="filter off")
            c.set_filter(True)
            check_call(g, c, small_masks(g, 4, 24), s4, fmt, frames, bgrs, bg, want=(False, False, True), tag="mask only")
    finally:
        c.close()


def test_emu_sources(emu_lib):
    """six sources, own and following strengths, sigma 0 in the same call; bsb_reset_source keeps a source's strength,
    bsb_set_sources resets every one to follow the context"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    c, bg = context(emu_lib, key, W, H, 6)
    try:
        c.set_sources(6)
        frames, bgrs = frames_of(W, H, 6, "bgr")
        ids = [4, 0, 5, 2, 1, 3]
        own = {0: 1, 1: 0, 2: 30, 3: 255}
        for s, v in own.items():
            c.set_source_mask_refine(s, v)

        def call(ctx_sigma, expect, seed):
            c.set_mask_refine(ctx_sigma)
            masks = small_masks(g, 6, seed)
            c.feed(B.FEED_MASK, masks)
            out, _, mask = c.composite_sources(frames, ids, want_yuyv=False)
            for b, s in enumerate(ids):
                rm = ref_refine(g, masks[b], bgrs[b], expect[s])
                assert np.array_equal(mask[b], rm), (s, expect[s], int((mask[b] != rm).sum()))
                assert np.array_equal(out[b], ref_outputs(rm, bgrs[b], bg, video=False)[0]), s

        call(8, {**own, 4: 8, 5: 8}, 30)
        call(0, {**own, 4: 0, 5: 0}, 31)                       # the followers follow later changes
        c.reset_source(2)
        call(12, {**own, 4: 12, 5: 12}, 32)
        c.set_source_mask_refine(3, None)
        call(12, {**own, 3: 12, 4: 12, 5: 12}, 33)
        c.set_sources(6)
        call(0, {s: 0 for s in range(6)}, 34)
        call(30, {s: 30 for s in range(6)}, 35)
    finally:
        c.close()


def test_emu_off_is_untouched(emu_lib):
    """strength 0 everywhere: the bytes and launch counts of a context that never heard of refinement"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    a, bg = context(emu_lib, key, W, H, 4)
    b, _ = context(emu_lib, key, W, H, 4)
    try:
        b.set_mask_refine(9)
        b.set_mask_refine(0)
        frames, bgrs = frames_of(W, H, 4, "bgr")
        masks = small_masks(g, 4, 40)
        ra = run_fed(a, masks, "bgr", frames)
        rb = run_fed(b, masks, "bgr", frames)
        for x, y in zip(ra, rb):
            assert np.array_equal(x, y)
        assert a.launches_per_call == b.launches_per_call
        assert np.array_equal(ra[2][0], ref_mask(g, masks[0]))
    finally:
        a.close()
        b.close()


def test_emu_held_frames_and_mask_api(emu_lib):
    """with the CNN: at mask interval 2 a held frame refines the held small mask against its own camera frame; the
    mask-only API (bs_maskgen_process) never refines"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    c, bg = context(emu_lib, key, W, H, 4)
    try:
        c.set_mask_interval(2)
        c.set_mask_refine(10)
        frames = np.stack([camera(W, H, t) for t in range(4)])
        _, _, mask = c.composite(frames, want_out=False, want_yuyv=False)
        small = [c.stage_u8(2, b) for b in range(4)]
        assert np.array_equal(small[0], small[1]) and np.array_equal(small[2], small[3])
        for b in range(4):
            assert np.array_equal(mask[b], ref_refine(g, small[b], frames[b], 10)), b
        m = c.process(frames[0])
        assert np.array_equal(m, ref_mask(g, c.stage_u8(2, 0)))
    finally:
        c.close()


def test_emu_chunked_host_call(emu_lib):
    """a host YUYV call of 4 frames at e2e_chunk 2 runs as two chunks of the overlapped schedule: its refined outputs equal
    the same call in one piece, whose masks are the restatement on the small masks it held"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    frames, bgrs = frames_of(W, H, 4, "yuyv")
    res = []
    for chunk in (16, 2):
        c, _ = context(emu_lib, key, W, H, 4)
        assert emu_lib.bsb_set_tuning(b"e2e_chunk", chunk)
        try:
            c.set_mask_refine(10)
            out = np.empty((4, H, W, 3), np.uint8)
            mask = np.empty((4, H, W), np.uint8)
            c.composite_yuyv_into(frames, out, None, mask)
            res.append((out, mask))
            if chunk == 16:
                for b in range(4):
                    assert np.array_equal(mask[b], ref_refine(g, c.stage_u8(2, b), bgrs[b], 10)), b
        finally:
            emu_lib.bsb_set_tuning(b"e2e_chunk", 16)
            c.close()
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])


# ---------------------------------------------------------------------------------------------------- quality
def scene(W=1280, H=720, person=165, seed=0):
    """a constructed camera frame with a known matte: a textured person (a head on shoulders, a wavy outline, a thin
    strand of hair) over a darker graded background, camera noise sigma 6.  Returns (BGR frame, truth 0 person / 255)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    cx = W / 2 + 18 * np.sin(yy / 37.0)
    body = (np.abs(xx - cx) < W * 0.22 + 0.25 * np.maximum(yy - H * 0.55, 0)) & (yy > H * 0.55)
    head = ((xx - cx) / (W * 0.11)) ** 2 + ((yy - H * 0.38) / (H * 0.2)) ** 2 < 1
    hair = (np.abs(xx - (cx + W * 0.1 + 0.3 * (H * 0.38 - yy))) < 1.5) & (yy > H * 0.12) & (yy < H * 0.38)
    inside = body | head | hair
    lum = np.where(inside, person + 12 * np.sin(xx / 5.0) * np.sin(yy / 7.0), 60 + 40 * xx / W)
    lum = lum + rng.normal(0, 6, (H, W))
    frame = np.clip(np.stack([lum * 0.9, lum, lum * 1.05], -1), 0, 255).astype(np.uint8)
    return frame, np.where(inside, 0, 255).astype(np.uint8)


def scene_small(truth, sw=256, sh=144):
    """the fed small mask: the area-downsampled truth, thresholded"""
    return np.where(cv2.resize(truth, (sw, sh), interpolation=cv2.INTER_AREA) < 128, 0, 255).astype(np.uint8)


def edge_error(m, truth, band=12):
    near = cv2.dilate((truth == 0).astype(np.uint8), np.ones((2 * band + 1, 2 * band + 1), np.uint8)) != \
        cv2.erode((truth == 0).astype(np.uint8), np.ones((2 * band + 1, 2 * band + 1), np.uint8))
    return float(np.abs(m.astype(np.int64) - truth)[near].mean())


@pytest.mark.parametrize("person,sigma,factor", [(165, 12, 0.2), (100, 8, 1.0)])
def test_quality_restatement(person, sigma, factor):
    """high contrast: the edge error at sigma 12 is at most a fifth of the unrefined mask's; low contrast (person luma
    ~100): sigma 8 is no worse than the unrefined mask"""
    g = geo("meet_full", 1280, 720)
    frame, truth = scene(person=person)
    small = scene_small(truth)
    before = edge_error(ref_mask(g, small), truth)
    after = edge_error(ref_refine(g, small, frame, sigma), truth)
    assert after <= factor * before, (person, sigma, after, before)


def test_quality_large_sigma_degrades():
    """sigma 255 weighs every tap alike: a tent upsample of the hard small mask, worse than the blurred one (the header
    says so)"""
    g = geo("meet_full", 1280, 720)
    frame, truth = scene()
    small = scene_small(truth)
    assert edge_error(ref_refine(g, small, frame, 255), truth) > edge_error(ref_mask(g, small), truth)


def test_emu_quality_library(emu_lib):
    """the library's bytes on the constructed 1280x720 scene (Meet, fed 256x144 mask) equal the restatement"""
    g = geo("meet_full", 1280, 720)
    frame, truth = scene(seed=1)
    small = scene_small(truth)
    c, bg = context(emu_lib, "meet_full", 1280, 720, 1)
    try:
        c.set_mask_refine(12)
        c.feed(B.FEED_MASK, small[None])
        _, _, mask = c.composite(frame[None], want_out=False, want_yuyv=False)
        rm = ref_refine(g, small, frame, 12)
        assert np.array_equal(mask[0], rm), int((mask[0] != rm).sum())
        assert edge_error(mask[0], truth) <= 0.2 * edge_error(ref_mask(g, small), truth)
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------- GPU
def gpu_lib():
    if bs.device_count() <= 0:
        pytest.skip("needs a CUDA device")
    return bs.lib()


def _device_call(c, fmt, frames, n, ids=None):
    """device-resident YUYV / NV12 frames through the device entry points; returns (out BGR, video, mask) on the host"""
    import torch
    W, H = c.width, c.height
    # fixed buffers per context, format and batch: a call replays its captured graph
    bufs = c.__dict__.setdefault("_refine_bufs", {})
    if (fmt, n) not in bufs:
        bufs[(fmt, n)] = (torch.empty(frames.shape, dtype=torch.uint8, device="cuda"),
                          torch.empty((n, H, W, 3), dtype=torch.uint8, device="cuda"),
                          torch.empty((n, H * W * 2 if fmt == "yuyv" else H * W * 3 // 2), dtype=torch.uint8, device="cuda"),
                          torch.empty((n, H, W), dtype=torch.uint8, device="cuda"))
    d_in, d_out, d_vid, d_mask = bufs[(fmt, n)]
    d_in.copy_(torch.from_numpy(np.ascontiguousarray(frames)))
    args = (d_in.data_ptr(), d_out.data_ptr(), d_vid.data_ptr(), d_mask.data_ptr())
    if ids is None:
        fn = c.composite_yuyv_device if fmt == "yuyv" else c.composite_nv12_device
        fn(n, *args, sync=True)
    else:
        fn = c.composite_sources_yuyv_device if fmt == "yuyv" else c.composite_sources_nv12_device
        fn(n, ids, *args, sync=True)
    return d_out.cpu().numpy(), d_vid.cpu().numpy(), d_mask.cpu().numpy()


def _check_device(g, c, bg, fmt, n, sigmas, seed, ids=None, tag=""):
    frames, bgrs = frames_of(g.W, g.H, n, fmt)
    masks = small_masks(g, n, seed)
    c.feed(B.FEED_MASK, masks)
    out, vid, mask = _device_call(c, fmt, frames, n, ids)
    for b in range(n):
        rm = ref_refine(g, masks[b], bgrs[b], sigmas[b])
        assert np.array_equal(mask[b], rm), (tag, fmt, b, sigmas[b], int((mask[b] != rm).sum()))
        ro, rv = ref_outputs(rm, bgrs[b], bg, nv12=fmt == "nv12")
        assert np.array_equal(out[b], ro), (tag, fmt, b)
        assert np.array_equal(vid[b].reshape(-1), rv.reshape(-1)), (tag, fmt, b)
    return mask


@pytest.mark.gpu
@pytest.mark.parametrize("tuning", [("post_tile", 64), ("post_tile", 128), ("post_tma", 0)])
def test_gpu_meet_720p(tuning):
    """Meet 1280x720, device YUYV / NV12: 64 sources with mixed strengths and a plain 32-frame call, for both post tile
    widths and k_post_fast; every byte against the restatement"""
    lib = gpu_lib()
    key, W, H = "meet_full", 1280, 720
    g = geo(key, W, H)
    assert lib.bsb_set_tuning(tuning[0].encode(), tuning[1])
    try:
        c, bg = context(lib, key, W, H, 64)
        try:
            for fmt in ("yuyv", "nv12"):
                c.set_mask_refine(12)
                _check_device(g, c, bg, fmt, 32, [12] * 32, 50, tag=str(tuning))
            c.set_sources(64)
            rng = np.random.default_rng(5)
            own = rng.choice([-1, 0, 1, 8, 30, 255], 64)
            for s, v in enumerate(own):
                c.set_source_mask_refine(s, None if v < 0 else int(v))
            c.set_mask_refine(16)
            ids = list(rng.permutation(64))
            sig = [16 if own[s] < 0 else int(own[s]) for s in ids]
            for fmt in ("yuyv", "nv12") if tuning == ("post_tile", 64) else ("yuyv",):
                _check_device(g, c, bg, fmt, 64, sig, 51, ids=ids, tag=str(tuning))
        finally:
            c.close()
    finally:
        lib.bsb_set_tuning(tuning[0].encode(), {"post_tile": 0, "post_tma": 1}[tuning[0]])


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("mlkit", 640, 480), ("deeplab", 1280, 720)])
def test_gpu_geometries(key, W, H):
    """MLKit's ~1.9x up-scale and DeepLab's letterboxed 720p ROI, plain and flipped sources calls, TMA against k_post_fast"""
    lib = gpu_lib()
    g = geo(key, W, H)
    c, bg = context(lib, key, W, H, 8)
    try:
        c.set_mask_refine(8)
        for fmt in ("yuyv", "nv12"):
            a = _check_device(g, c, bg, fmt, 8, [8] * 8, 60, tag=key)
            assert lib.bsb_set_tuning(b"post_tma", 0)
            try:
                b = _check_device(g, c, bg, fmt, 8, [8] * 8, 60, tag=key + " fast")
            finally:
                lib.bsb_set_tuning(b"post_tma", 1)
            assert np.array_equal(a, b)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("interval", [1, 2])
def test_gpu_camera_stream(interval):
    """the CNN on synthetic camera frames (graph replay), mask interval 1 and 2: every mask is the restatement on the
    small mask the call held (stage 2) and the frame's own camera bytes; changing the strength replays (no new launch
    count, one graph for every strength)"""
    lib = gpu_lib()
    key, W, H = "meet_full", 1280, 720
    g = geo(key, W, H)
    c, bg = context(lib, key, W, H, 8)
    try:
        c.set_mask_interval(interval)
        n = 8
        frames, bgrs = frames_of(W, H, n, "yuyv")
        launches = {}
        for sigma in (0, 12, 30, 12, 0, 8):
            c.set_mask_refine(sigma)
            out, vid, mask = _device_call(c, "yuyv", frames, n)
            for b in range(n):
                rm = ref_refine(g, c.stage_u8(2, b), bgrs[b], sigma)
                assert np.array_equal(mask[b], rm), (interval, sigma, b, int((mask[b] != rm).sum()))
            launches.setdefault(sigma != 0, set()).add(c.launches_per_call)
        # the refined graph runs the same launches as the unrefined one
        assert launches[True] == launches[False] and len(launches[True]) == 1, launches
        # once both graphs exist, strengths change by table data: the calls replay and capture nothing (no launch counted)
        t1 = lib.bsb_total_launches()
        for sigma in (5, 6, 0, 7, 255, 0):
            c.set_mask_refine(sigma)
            _device_call(c, "yuyv", frames, n)
        assert lib.bsb_total_launches() == t1, "a strength change recaptured a graph"
    finally:
        c.close()
