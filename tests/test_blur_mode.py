"""Masked camera blur (include/backscrub_b200.h, bsb_set_blur_mode): a camera-blur frame in masked mode blends the
Gaussian of its camera frame weighted by its own mask, normalised by the Gaussian of the mask, so the person's colours
stay out of the blurred background.

`ref_masked_blur` restates the definition in int64 numpy and asserts its bounds; every masked output of the library is
compared with it byte for byte: the stand-alone stage on arbitrary masks, and calls on fed small masks (bsb_test_feed) or
on the CNN's own, where M is the call's own mask output.  The quality tests check on a constructed scene that the halo
around the person shrinks, on the restatement and on the library's bytes.
"""
import math

import cv2
import numpy as np
import pytest

import backscrub_b200 as bs
from backscrub_b200 import _binding as B
from backscrub_b200 import api
from oracle import pyoracle as po
from tests.conftest import model_path
from tests.test_bgra_output import expect_bgra
from tests.test_feed_post import geo, ref_outputs
from tests.test_mask_refine import camera, frames_of, ref_refine, run_fed, small_masks


# ---------------------------------------------------------------------------------------------------- the definition
def gauss_taps(k):
    """OpenCV's 8.8 fixed-point taps of GaussianBlur(Size(k, k), 0) (bsb_gaussian_taps)"""
    small = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
             7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125],
             9: [x / 256 for x in (4, 13, 30, 51, 60, 51, 30, 13, 4)]}
    n2 = k // 2
    if k <= 9:
        v = small[k]
    else:
        sigma = k * 0.15 + 0.35
        s2 = -0.125 / (sigma * sigma)
        v = [math.exp((x * x) * s2) for x in range(1 - k, 0, 2)]
        mul = 1.0 / (sum(v) * 2 + 1)
        v = [a * mul for a in v] + [mul]
    q = [0] * k
    err, acc = 0.0, 0
    for i in range(n2):
        adj = v[i] * 256 + err
        qi = int(round(adj))
        err = adj - qi
        q[i] = q[k - 1 - i] = qi
        acc += qi
    q[n2] = 256 - 2 * acc
    return np.array(q, np.int64)


def reflect101(i, n):
    if n == 1:
        return np.zeros_like(i)
    i = i.copy()
    while ((i < 0) | (i >= n)).any():
        i = np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i))
    return i


def _conv_rows(a, q):
    r = len(q) // 2
    W = a.shape[1]
    out = np.zeros(a.shape, np.int64)
    for j, w in enumerate(q):
        out += w * a[:, reflect101(np.arange(W) + j - r, W)]
    return out


def _conv_rows_f64(a, q):
    """_conv_rows by cv::sepFilter2D in float64: every product and partial sum is an integer below 2^53, so exact"""
    out = cv2.sepFilter2D(a.astype(np.float64), cv2.CV_64F, q.astype(np.float64), np.ones(1), borderType=cv2.BORDER_REFLECT_101)
    return out.astype(np.int64)


def ref_masked_blur(C, M, k, fast=True):
    """B of include/backscrub_b200.h (bsb_set_blur_mode): C H x W x 3, M H x W, both uint8.  fast: the separable sums by
    cv::sepFilter2D in float64 (frames larger than k; test_restatement_fast_path pins it to the numpy sums)"""
    q = gauss_taps(k)
    conv = _conv_rows_f64 if fast and min(C.shape[:2]) > k else _conv_rows
    Ci, Mi = C.astype(np.int64), M.astype(np.int64)
    h = conv(Mi[..., None] * Ci, q)
    g = conv(Mi, q)
    assert h.max() < 1 << 24 and g.max() < 1 << 16
    N = conv(np.ascontiguousarray(h.swapaxes(0, 1)), q).swapaxes(0, 1)
    D = conv(np.ascontiguousarray(g.T), q).T
    assert D.max() < 1 << 24 and (N + (D >> 1)[..., None]).max() < 1 << 32
    Dc = D[..., None]
    return np.where(Dc > 0, (N + (Dc >> 1)) // np.maximum(Dc, 1), Ci).astype(np.uint8)


KS = (1, 3, 25, 31, 33, 61, 255)


def test_restatement_properties():
    """a uniform mask v > 0 gives cv::GaussianBlur; k = 1 and M = 0 give C; the bounds hold at the worst case"""
    rng = np.random.default_rng(0)
    C = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    for k in KS:
        plain = po.gaussian_blur(C, k)
        for v in (1, 77, 255):
            assert np.array_equal(ref_masked_blur(C, np.full(C.shape[:2], v, np.uint8), k), plain), (k, v)
        assert np.array_equal(ref_masked_blur(C, np.zeros(C.shape[:2], np.uint8), k), C), k
    assert np.array_equal(ref_masked_blur(C, rng.integers(0, 256, C.shape[:2], dtype=np.uint8), 1), C)
    ref_masked_blur(np.full((300, 300, 3), 255, np.uint8), np.full((300, 300), 255, np.uint8), 255)


def test_restatement_fast_path():
    rng = np.random.default_rng(3)
    C = rng.integers(0, 256, (300, 280, 3), dtype=np.uint8)
    M = rng.integers(0, 256, (300, 280), dtype=np.uint8)
    M[50:120, 40:200] = 0
    for k in (3, 25, 61, 255):
        assert np.array_equal(ref_masked_blur(C, M, k), ref_masked_blur(C, M, k, fast=False)), k


# ---------------------------------------------------------------------------------------------------- emulator: the stage
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def random_mask(H, W, rng):
    """random bytes with zero patches (D = 0 inside them at small k) and a 255 band"""
    m = rng.integers(0, 256, (H, W), dtype=np.uint8)
    m[H // 4: H // 2, W // 5: W // 2] = 0
    m[:, -max(1, W // 8):] = 255
    m[rng.integers(0, H, 20), rng.integers(0, W, 20)] = 0
    return m


@pytest.mark.parametrize("W,H", [(97, 61), (130, 33), (5, 4)])
def test_emu_stage(emu_lib, W, H):
    """bsb_masked_gaussian_blur, both launch classes, at sizes that are no tile multiple and at a frame smaller than r"""
    rng = np.random.default_rng(W)
    C = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    M = random_mask(H, W, rng)
    for k in (1, 3, 7, 25, 31, 33, 61, 255) if W > 5 else (3, 61):
        assert np.array_equal(api.gaussian_taps(emu_lib, k), gauss_taps(k)), k
        got = api.masked_gaussian_blur(emu_lib, C, M, k)
        exp = ref_masked_blur(C, M, k)
        assert np.array_equal(got, exp), (W, H, k, int((got != exp).sum()))


def test_emu_stage_refusals(emu_lib):
    C = np.zeros((8, 8, 3), np.uint8)
    for k in (0, 2, 257, -1):
        with pytest.raises(bs.BackscrubError, match="strength"):
            api.masked_gaussian_blur(emu_lib, C, np.zeros((8, 8), np.uint8), k)
    assert not emu_lib.bsb_masked_gaussian_blur(0, None, None, None, 8, 8, 3)


# ---------------------------------------------------------------------------------------------------- emulator: calls
def blur_context(lib, key, W, H, k, max_batch=4, mode="masked"):
    """a context in camera-blur mode: no background image, strength k"""
    c = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch)
    c.set_bgblur(k)
    if mode is not None:
        c.set_blur_mode(mode)
    return c


def check_call(c, masks, fmt, frames, bgrs, k, flip=0, out_size=None, bgra=False, want=(True, True, True), refine=0, g=None, tag=""):
    """one fed call; M is the call's own mask output, which must also equal the (refined) restatement"""
    out, vid, mask = run_fed(c, masks, fmt, frames, want)
    for b in range(len(masks)):
        if g is not None:
            rm = ref_refine(g, masks[b], bgrs[b], refine)
            assert np.array_equal(mask[b], rm), (tag, b, "mask")
        bg = ref_masked_blur(bgrs[b], mask[b], k)
        ro, rv = ref_outputs(mask[b], bgrs[b], bg, flip, out_size, fmt == "nv12", video=vid is not None)
        if out is not None:
            exp = expect_bgra(bgrs[b], mask[b], True, flip, out_size) if bgra else ro
            assert np.array_equal(out[b], exp), (tag, fmt, k, b, "out", int((out[b] != exp).sum()))
        if vid is not None:
            assert np.array_equal(vid[b].reshape(-1), rv.reshape(-1)), (tag, fmt, k, b, "video")
    return out, vid, mask


@pytest.mark.parametrize("fmt", ["bgr", "yuyv", "nv12"])
def test_emu_plain(emu_lib, fmt):
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    frames, bgrs = frames_of(W, H, 3, fmt)
    for i, k in enumerate((7, 25, 33, 61)):
        c = blur_context(emu_lib, key, W, H, k, 3)
        try:
            check_call(c, small_masks(g, 3, 100 + i), fmt, frames, bgrs, k, g=g, tag="plain")
        finally:
            c.close()


def test_emu_outputs(emu_lib):
    """flip + resize tail, BGRA with video, refinement at sigma 12"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    c = blur_context(emu_lib, key, W, H, 25)
    try:
        for fmt in ("bgr", "nv12"):
            frames, bgrs = frames_of(W, H, 4, fmt)
            c.set_output(True, True, (W // 2, H // 2))
            check_call(c, small_masks(g, 4, 120), fmt, frames, bgrs, 25, flip=3, out_size=(W // 2, H // 2), g=g, tag="tail")
            c.set_output(False, False, None)
            c.set_out_format("bgra")
            # BGRA with video: the video is the composite over the masked blur
            check_call(c, small_masks(g, 4, 121), fmt, frames, bgrs, 25, bgra=True, g=g, tag="bgra")
            c.set_out_format("bgr")
            c.set_mask_refine(12)
            check_call(c, small_masks(g, 4, 122), fmt, frames, bgrs, 25, refine=12, g=g, tag="refined")
            c.set_mask_refine(0)
    finally:
        c.close()


def test_emu_held_frames(emu_lib):
    """with the CNN at mask interval 2: the held frames' masks weigh their blur"""
    key, W, H = "meet_lite", 320, 176
    c = blur_context(emu_lib, key, W, H, 33)
    try:
        c.set_mask_interval(2)
        frames = np.stack([camera(W, H, t) for t in range(4)])
        out, vid, mask = c.composite(frames)
        for b in range(4):
            ro, rv = ref_outputs(mask[b], frames[b], ref_masked_blur(frames[b], mask[b], 33))
            assert np.array_equal(out[b], ro) and np.array_equal(vid[b], rv), b
    finally:
        c.close()


def test_emu_chunked_host_call(emu_lib):
    """a host YUYV call at e2e_chunk 2 equals the same call in one piece, which equals the restatement"""
    key, W, H = "meet_lite", 320, 176
    frames, bgrs = frames_of(W, H, 4, "yuyv")
    res = []
    for chunk in (16, 2):
        c = blur_context(emu_lib, key, W, H, 25)
        assert emu_lib.bsb_set_tuning(b"e2e_chunk", chunk)
        try:
            out = np.empty((4, H, W, 3), np.uint8)
            mask = np.empty((4, H, W), np.uint8)
            c.composite_yuyv_into(frames, out, None, mask)
            res.append((out, mask))
        finally:
            emu_lib.bsb_set_tuning(b"e2e_chunk", 16)
            c.close()
    for b in range(4):
        assert np.array_equal(res[0][0][b], ref_outputs(res[0][1][b], bgrs[b], ref_masked_blur(bgrs[b], res[0][1][b], 25), video=False)[0])
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])


def test_emu_sources(emu_lib):
    """six sources: own, following and plain modes, strengths of both classes, an own image, no background, the
    context's strength; each frame against a batch-1 plain context set up the same way; refusals change nothing"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    c = blur_context(emu_lib, key, W, H, 25, 6, mode=None)
    try:
        with pytest.raises(bs.BackscrubError, match="no sources"):
            c.set_source_blur_mode(0, "masked")
        c.set_sources(6)
        own_img = po.resize_linear_u8(np.full((40, 60, 3), (30, 60, 200), np.uint8), W, H)
        c.set_source_background(1, np.full((40, 60, 3), (30, 60, 200), np.uint8))
        c.set_source_effect(2, "none", 61)
        c.set_source_effect(3, "none", 7)
        c.set_source_effect(4, "none", 0)
        # (source, mode): 0 follows (k 25), 1 own image, 2 masked k 61, 3 plain k 7, 4 green, 5 masked k 25
        c.set_source_blur_mode(2, "masked")
        c.set_source_blur_mode(3, "plain")
        c.set_source_blur_mode(5, "masked")
        for s, v in ((6, "masked"), (-1, "plain"), (0, "sideways")):
            with pytest.raises(bs.BackscrubError):
                c.set_source_blur_mode(s, v)
        with pytest.raises(bs.BackscrubError, match="blur mode"):
            c.set_blur_mode("sideways")
        frames, bgrs = frames_of(W, H, 6, "bgr")
        ids = [3, 0, 5, 2, 1, 4]

        def call(ctx_mode, seed):
            c.set_blur_mode(ctx_mode)
            masks = small_masks(g, 6, seed)
            c.feed(B.FEED_MASK, masks)
            out, vid, mask = c.composite_sources(frames, ids)
            for b, s in enumerate(ids):
                k = {0: 25, 2: 61, 3: 7, 5: 25}.get(s)
                masked = {0: ctx_mode == "masked", 2: True, 3: False, 5: True}.get(s)
                if k is None:
                    bg = own_img if s == 1 else np.broadcast_to(np.array([0, 255, 0], np.uint8), bgrs[b].shape)
                elif masked:
                    bg = ref_masked_blur(bgrs[b], mask[b], k)
                else:
                    bg = po.gaussian_blur(bgrs[b], k)
                ro, rv = ref_outputs(mask[b], bgrs[b], bg)
                assert np.array_equal(out[b], ro), (ctx_mode, s, int((out[b] != ro).sum()))
                assert np.array_equal(vid[b], rv), (ctx_mode, s)
            return masks, out, mask

        call("masked", 130)
        masks, out, mask = call("plain", 131)
        # a batch-1 plain context set up as source 2
        one = blur_context(emu_lib, key, W, H, 61, 1)
        try:
            o1, _, m1 = run_fed(one, masks[3:4], "bgr", frames[3:4])
            assert np.array_equal(o1[0], out[3]) and np.array_equal(m1[0], mask[3])
        finally:
            one.close()
        c.reset_source(2)                                           # keeps the source's mode
        call("plain", 132)
        c.set_sources(6)                                            # every source follows again
        c.set_blur_mode("masked")
        masks = small_masks(g, 6, 133)
        c.feed(B.FEED_MASK, masks)
        out, _, mask = c.composite_sources(frames, ids, want_yuyv=False)
        for b in range(6):
            assert np.array_equal(out[b], ref_outputs(mask[b], bgrs[b], ref_masked_blur(bgrs[b], mask[b], 25), video=False)[0]), b
    finally:
        c.close()


def test_emu_untouched(emu_lib):
    """an explicit PLAIN equals the default; MASKED with a background image, the filter off, or a BGRA-only call equals
    PLAIN: same bytes, same launches"""
    key, W, H = "meet_lite", 320, 176
    g = geo(key, W, H)
    frames, _ = frames_of(W, H, 3, "bgr")
    masks = small_masks(g, 3, 140)

    def run(setup, mode, want=(True, True, True)):
        c = blur_context(emu_lib, key, W, H, 25, 3, mode=mode)
        try:
            setup(c)
            r = run_fed(c, masks, "bgr", frames, want)
            return r, c.launches_per_call
        finally:
            c.close()

    def same(a, b):
        assert a[1] == b[1], (a[1], b[1])
        for x, y in zip(a[0], b[0]):
            assert (x is None and y is None) or np.array_equal(x, y)

    nothing = lambda c: None
    same(run(nothing, None), run(nothing, "plain"))
    masked = run(nothing, "masked")
    assert masked[1] > run(nothing, "plain")[1]                  # the mask-only post launch
    image = lambda c: c.set_background(np.full((30, 40, 3), 90, np.uint8))
    same(run(image, "plain"), run(image, "masked"))
    off = lambda c: c.set_filter(False)
    same(run(off, "plain"), run(off, "masked"))
    bgra = lambda c: c.set_out_format("bgra")
    same(run(bgra, "plain", (True, False, True)), run(bgra, "masked", (True, False, True)))
    img = np.full((20, 30, 3), 40, np.uint8)                     # the emulator's device memory is host memory
    live = lambda c: c.set_live_background(img.ctypes.data, size=(30, 20))
    same(run(live, "plain"), run(live, "masked"))


# ---------------------------------------------------------------------------------------------------- quality
def plate_scene(W=1280, H=720, seed=0):
    """a textured person (head on shoulders, wavy outline) over a graded, noisy background plate, camera noise sigma 6:
    (frame, plate, truth 0 person / 255)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    cx = W / 2 + 18 * np.sin(yy / 37.0)
    body = (np.abs(xx - cx) < W * 0.22 + 0.25 * np.maximum(yy - H * 0.55, 0)) & (yy > H * 0.55)
    head = ((xx - cx) / (W * 0.11)) ** 2 + ((yy - H * 0.38) / (H * 0.2)) ** 2 < 1
    inside = body | head
    person = 170 + 25 * np.sin(xx / 5.0) * np.sin(yy / 7.0) + rng.normal(0, 6, (H, W))
    lum = 60 + 40 * xx / W + 20 * yy / H + rng.normal(0, 6, (H, W))
    plate = np.clip(np.stack([lum * 0.9, lum, lum * 1.05], -1), 0, 255).astype(np.uint8)
    pers = np.clip(np.stack([person * 0.7, person * 0.85, person * 1.1], -1), 0, 255).astype(np.uint8)
    frame = np.where(inside[..., None], pers, plate)
    return frame, plate, np.where(inside, 0, 255).astype(np.uint8)


def scene_mask(truth):
    """Meet's 256x144 mask of the truth, resized and 5x5 blurred (an approximation of the library's mask)"""
    small = np.where(cv2.resize(truth, (256, 144), interpolation=cv2.INTER_AREA) < 128, 0, 255).astype(np.uint8)
    return cv2.blur(cv2.resize(small, (truth.shape[1], truth.shape[0]), interpolation=cv2.INTER_LINEAR), (5, 5)), small


def halo_error(comp, M, plate, truth, k):
    """|composite - blend(GaussianBlur(plate))| over background pixels (M = 255) within r of the person: mean, p99"""
    ideal = po.alpha_blend(po.gaussian_blur(plate, k), plate, M)
    r = k // 2
    near = cv2.dilate((truth == 0).astype(np.uint8), np.ones((2 * r + 1, 2 * r + 1), np.uint8)).astype(bool) & (M == 255)
    e = np.abs(comp.astype(np.int64) - ideal).max(-1)[near]
    return float(e.mean()), float(np.percentile(e, 99))


@pytest.mark.parametrize("k", [25, 61])
def test_quality_restatement(k):
    frame, plate, truth = plate_scene()
    M, _ = scene_mask(truth)
    plain = halo_error(po.alpha_blend(po.gaussian_blur(frame, k), frame, M), M, plate, truth, k)
    masked = halo_error(po.alpha_blend(ref_masked_blur(frame, M, k), frame, M), M, plate, truth, k)
    assert masked[0] <= 0.5 * plain[0] and masked[1] <= 0.5 * plain[1], (k, plain, masked)


@pytest.mark.parametrize("k", [25, 61])
def test_emu_quality_library(emu_lib, k):
    """the library's bytes on the scene (Meet 1280x720, fed 256x144 mask) equal the restatement, and halve the halo"""
    frame, plate, truth = plate_scene(seed=1)
    _, small = scene_mask(truth)
    c = blur_context(emu_lib, "meet_full", 1280, 720, k, 1)
    try:
        c.feed(B.FEED_MASK, small[None])
        out, _, mask = c.composite(frame[None], want_yuyv=False)
        M = mask[0]
        assert np.array_equal(out[0], po.alpha_blend(ref_masked_blur(frame, M, k), frame, M))
        plain = halo_error(po.alpha_blend(po.gaussian_blur(frame, k), frame, M), M, plate, truth, k)
        masked = halo_error(out[0], M, plate, truth, k)
        assert masked[0] <= 0.5 * plain[0] and masked[1] <= 0.5 * plain[1], (k, plain, masked)
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
    bufs = c.__dict__.setdefault("_blur_bufs", {})
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


def _check(out, vid, mask, bgrs, ks, fmt, tag, step=1):
    """frames 0, step, 2 step, .. and the last against the restatement (the emulator tests check every frame); ks[b] < 0:
    frame b blurs plain at -ks[b]"""
    for b in sorted(set(range(0, len(bgrs), step)) | {len(bgrs) - 1}):
        bg = ref_masked_blur(bgrs[b], mask[b], ks[b]) if ks[b] > 0 else po.gaussian_blur(bgrs[b], -ks[b])
        ro, rv = ref_outputs(mask[b], bgrs[b], bg, nv12=fmt == "nv12")
        assert np.array_equal(out[b], ro), (tag, fmt, b, ks[b], int((out[b] != ro).sum()))
        assert np.array_equal(vid[b].reshape(-1), rv.reshape(-1)), (tag, fmt, b)


@pytest.mark.gpu
@pytest.mark.parametrize("tuning", [("post_tile", 64), ("post_tile", 128), ("post_tma", 0)])
def test_gpu_meet_720p(tuning):
    """Meet 1280x720, device YUYV / NV12: 32-frame plain calls and a 64-source call with plain and masked frames at
    k = 25 and 61; every byte against the restatement on the call's own masks"""
    lib = gpu_lib()
    key, W, H = "meet_full", 1280, 720
    g = geo(key, W, H)
    assert lib.bsb_set_tuning(tuning[0].encode(), tuning[1])
    try:
        c = blur_context(lib, key, W, H, 25, 64)
        try:
            for k in (25, 61):
                c.set_bgblur(k)
                for fmt in ("yuyv", "nv12"):
                    frames, bgrs = frames_of(W, H, 32, fmt)
                    c.feed(B.FEED_MASK, small_masks(g, 32, k))
                    out, vid, mask = _device_call(c, fmt, frames, 32)
                    _check(out, vid, mask, bgrs, [k] * 32, fmt, str(tuning), step=4)
            c.set_bgblur(25)
            c.set_sources(64)
            rng = np.random.default_rng(7)
            ks = {}
            for s in range(64):
                k = int(rng.choice([25, 61]))
                c.set_source_effect(s, "none", k)
                mode = rng.choice(["masked", "plain", None])
                c.set_source_blur_mode(s, None if mode is None else str(mode))
                ks[s] = -k if mode == "plain" else k
            c.set_blur_mode("masked")
            ids = [int(i) for i in rng.permutation(64)]
            for fmt in ("yuyv", "nv12") if tuning == ("post_tile", 64) else ("yuyv",):
                frames, bgrs = frames_of(W, H, 64, fmt)
                c.feed(B.FEED_MASK, small_masks(g, 64, 9))
                out, vid, mask = _device_call(c, fmt, frames, 64, ids)
                _check(out, vid, mask, bgrs, [ks[s] for s in ids], fmt, str(tuning), step=3)
        finally:
            c.close()
    finally:
        lib.bsb_set_tuning(tuning[0].encode(), {"post_tile": 0, "post_tma": 1}[tuning[0]])


@pytest.mark.gpu
def test_gpu_camera_stream_and_replay():
    """the CNN on camera frames (graph replay): masked outputs against the restatement on the call's own masks; once both
    graphs exist (the first masked call allocates its staging, which drops the captured graphs once), toggling the mode
    captures nothing"""
    lib = gpu_lib()
    key, W, H = "meet_full", 1280, 720
    c = blur_context(lib, key, W, H, 25, 8, mode="plain")
    try:
        frames, bgrs = frames_of(W, H, 8, "yuyv")
        for mode in ("plain", "masked", "plain"):
            c.set_blur_mode(mode)
            out, vid, mask = _device_call(c, "yuyv", frames, 8)
            _check(out, vid, mask, bgrs, [25 if mode == "masked" else -25] * 8, "yuyv", mode)
        t1 = lib.bsb_total_launches()
        for mode in ("plain", "masked", "plain", "masked"):
            c.set_blur_mode(mode)
            _device_call(c, "yuyv", frames, 8)
        assert lib.bsb_total_launches() == t1, "a mode change recaptured a graph"
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("mlkit", 640, 480), ("deeplab", 1280, 720)])
def test_gpu_geometries(key, W, H):
    """MLKit 640x480 and DeepLab's letterboxed 720p ROI (M = 255 at the borders), fed masks"""
    lib = gpu_lib()
    g = geo(key, W, H)
    c = blur_context(lib, key, W, H, 25, 8)
    try:
        for k, fmt in ((25, "yuyv"), (61, "nv12")):
            c.set_bgblur(k)
            frames, bgrs = frames_of(W, H, 8, fmt)
            c.feed(B.FEED_MASK, small_masks(g, 8, k))
            out, vid, mask = _device_call(c, fmt, frames, 8)
            _check(out, vid, mask, bgrs, [k] * 8, fmt, key)
    finally:
        c.close()
