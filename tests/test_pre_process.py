"""The pre-processing stages on constructed camera frames: ROI geometry, ROI resize + letterbox + BGR->RGB swap
(k_resize_roi_swap for BGR, YUYV and NV12 frames), the bilateral filter and the input-tensor normalisation
(k_bilateral_norm), and the fused stem that reads the filtered bytes (k_stem_u8 / k_stem_u8_x2).

Every stage is compared with a reference that does not use the kernels:
- geometry: a numpy float32 restatement of lib/libbackscrub.cc:234-246 (plus the documented out_roidim scaling of
  models whose output grid is not the input grid), against bsb_geometry and the oracle;
- stage_u8(0): cv2.resize (INTER_LINEAR) of the ROI crop pasted into zeros and swapped to RGB, cross-checked with the
  oracle's resize; camera frames are converted with cv2.cvtColor first;
- stage_u8(1): the oracle's bilateral filter bit for bit, and a float64 evaluation of the same definition;
- the input tensor: float32(float64(r) * scale + offset), which is exact and so equals fmaf;
- the stem output: the oracle's conv2d on the reference input tensor, bit for bit.

Frames are uniform random bytes, extreme / out-of-gamut codes, constants, single-pixel impulse lattices and, at the 1:1
geometries, bilateral probes covering every colour-LUT index.  Each call carries three distinct frames and every frame
is checked, so a per-frame offset or stride error cannot hide.

`-m "not gpu"`: the geometry sweep, and the pixel fixtures of Meet lite and MLKit on the kernel-logic emulator.
`-m gpu`: every model x geometry x format x layout on the H100, and one call of 2 x SMs + 3 frames."""
import ctypes as C
import math

import cv2
import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests.conftest import model_path

KEEP_TENSORS = 1
MODEL_HW = {"meet_full": (256, 144), "meet_lite": (160, 96), "mlkit": (256, 256), "deeplab": (257, 257), "bodypix": (257, 257)}
OUT_HW = {"meet_full": (256, 144), "meet_lite": (160, 96), "mlkit": (256, 256), "deeplab": (257, 257), "bodypix": (33, 33)}
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# geometry reference
# ---------------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    """C integer division (truncation toward zero)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def ref_geometry(key, W, H):
    """lib/libbackscrub.cc:234-246 in float32 arithmetic with truncating conversions: (roidim, in_roidim, out_roidim) as
    x, y, w, h, or None where an extent is not positive (the context refuses the size)"""
    mw, mh = MODEL_HW[key]
    ow, oh = OUT_HW[key]
    ratio = F32(mh) / F32(mw)
    frameratio = F32(H) / F32(W)
    if frameratio < ratio:
        roi = [int((F32(W) - F32(H) / ratio) / F32(2)), 0, int(F32(H) / ratio), H]
        inr = [0, 0, mw, mh]
    else:
        roi = [0, 0, W, H]
        inr = [int((F32(mw) - F32(mh) / frameratio) / F32(2)), 0, int(F32(mh) / frameratio), mh]
    if (ow, oh) == (mw, mh):
        outr = list(inr)
    else:       # BodyPix: the in-model rectangle scaled by out / in (integer arithmetic)
        outr = [_cdiv(inr[0] * ow, mw), _cdiv(inr[1] * oh, mh), _cdiv(inr[2] * ow, mw), _cdiv(inr[3] * oh, mh)]
    if min(roi[2], roi[3], inr[2], inr[3], outr[2], outr[3]) <= 0:
        return None
    return roi, inr, outr


def _accepted(key, W, H):
    return ref_geometry(key, W, H) is not None


def _last_accepted(key, fixed, axis, lo=1, hi=16384):
    """largest size along `axis` (0 = width, 1 = height) accepted with the other side `fixed`; acceptance falls
    monotonically along the axis.  Returns hi when every size is accepted, lo - 1 when none is."""
    size = (lambda v: (v, fixed)) if axis == 0 else (lambda v: (fixed, v))
    if _accepted(key, *size(hi)):
        return hi
    if not _accepted(key, *size(lo)):
        return lo - 1
    a, b = lo, hi                   # accepted at a, refused at b
    while b - a > 1:
        m = (a + b) // 2
        a, b = (m, b) if _accepted(key, *size(m)) else (a, m)
    return a


def _geometry_class(key, W, H):
    """what the geometry of a size depends on beyond its scale: the branch taken and every truncation"""
    geo = ref_geometry(key, W, H)
    if geo is None:
        return None
    (rx, ry, rw, rh), inr, outr = geo
    return rx, ry, W - rw, H - rh, tuple(inr), tuple(outr)


def sweep_sizes(key):
    """the sizes of the geometry sweep of one model.  Every exact-aspect multiple up to 4096 and its +-1 neighbours in W
    and in H is evaluated by the restatement; contexts are made for all of them up to 64 multiples of the reduced
    aspect, and above that for the smallest and the largest size of each distinct geometry class (_geometry_class),
    so every outcome the restatement gives on that range meets the engine and the oracle."""
    mw, mh = MODEL_HW[key]
    g = math.gcd(mw, mh)
    a, b = mw // g, mh // g
    exact, first_of, last_of = set(), {}, {}
    for k in range(1, 4096 // max(a, b) + 1):
        for W, H in ((k * a, k * b), (k * a + 1, k * b), (k * a - 1, k * b), (k * a, k * b + 1), (k * a, k * b - 1)):
            if W < 1 or H < 1:
                continue
            if k <= 64:
                exact.add((W, H))
            c = _geometry_class(key, W, H)
            first_of.setdefault(c, (W, H))
            last_of[c] = (W, H)
    exact |= set(first_of.values()) | set(last_of.values())
    base = {(k * mw, k * mh) for k in range(1, 4096 // max(mw, mh) + 1)}    # multiples of the model input up to 4k
    base |= {(k * mw // 2, k * mh // 2) for k in (1, 3, 5, 7, 9, 15)}
    sizes = set(exact)
    for W, H in base:
        sizes |= {(W, H), (W + 1, H), (W - 1, H), (W, H + 1), (W, H - 1)}
    for i in range(1, 13):                                             # powers of two
        for j in range(max(0, i - 5), min(12, i + 5) + 1):
            sizes.add((1 << i, 1 << j))
    sizes |= {(160, 120), (320, 240), (352, 288), (640, 360), (640, 480), (800, 600), (960, 540), (1024, 768),
              (1280, 720), (1280, 800), (1280, 960), (1280, 1024), (1600, 1200), (1920, 1080), (1920, 1200),
              (2560, 1440), (3840, 2160), (4096, 2160), (720, 1280), (1080, 1920), (480, 640)}
    # smallest accepted / largest refused along each axis, and both sides of the transition
    for fixed in (1, 2, 3, 5, 9, 16, 144, 480):
        for axis in (0, 1):
            last = _last_accepted(key, fixed, axis)
            for v in (last - 1, last, last + 1, last + 2):
                if 1 <= v <= 16384:
                    sizes.add((v, fixed) if axis == 0 else (fixed, v))
        sizes |= {(16384, fixed), (fixed, 16384)}
    return sorted((W, H) for W, H in sizes if 1 <= W <= 16384 and 1 <= H <= 16384 and W * H <= 4096 * 4096)


# ---------------------------------------------------------------------------------------------------------------------
# resize / bilateral / tensor references
# ---------------------------------------------------------------------------------------------------------------------
def ref_in_u8(bgr, geo, mw, mh):
    """the model-sized RGB image: the ROI crop resized (cv2 INTER_LINEAR, OpenCV's own area shortcut at exact 2x) to the
    in-model rectangle, pasted into zeros and swapped BGR -> RGB"""
    (rx, ry, rw, rh), (ix, iy, iw, ih), _ = geo
    crop = np.ascontiguousarray(bgr[ry:ry + rh, rx:rx + rw])
    r = cv2.resize(crop, (iw, ih), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(r, po.resize_linear_u8(crop, iw, ih)), "cv2 and the oracle's resize disagree"
    out = np.zeros((mh, mw, 3), np.uint8)
    out[iy:iy + ih, ix:ix + iw] = r[..., ::-1]
    return out


def _bilateral_luts():
    """the library's float32 weights: colour LUT (float)exp(i^2 * -0.5/100^2), 13 space taps (float)exp(r^2 * -0.5/100^2)
    with r = sqrt(i^2 + j^2), i^2 + j^2 <= 4 in raster order"""
    gc = gs = -0.5 / (100.0 * 100.0)
    cw = np.array([F32(math.exp(float(i) * i * gc)) for i in range(768)], np.float32)
    taps, sw = [], []
    for i in range(-2, 3):
        for j in range(-2, 3):
            r = math.sqrt(float(i) * i + float(j) * j)
            if r > 2:
                continue
            taps.append((i, j))
            sw.append(F32(math.exp(r * r * gs)))
    return cw, np.array(sw, np.float32), taps


CW, SW, TAPS = _bilateral_luts()

# Half-integer margin of the float64 bilateral check.  The kernel rounds each weight w = sw * cw to float32 (relative
# error <= u = 2^-24), accumulates wsum and the three channel sums over 13 taps with one rounding per fmaf (all terms
# are >= 0, so each sum carries a relative error <= 14u: 13 accumulation roundings and the weight's), then rounds
# 1 / wsum (u) and s * (1 / wsum) (u).  The quotient is off by at most (14 + 14 + 2)u ~ 1.8e-6 relative, <= 4.6e-4
# absolute for q <= 255.  Wherever q is more than 1e-3 from a half-integer, the byte must therefore be round(q).
BILATERAL_MARGIN = 1e-3


def bilateral_q(img):
    """float64 quotient of cv::bilateralFilter(d=5, sigma 100/100) on an RGB u8 image with the library's float32 weights:
    sum_k w_k v_k / sum_k w_k, BORDER_REFLECT_101, the sums in float64"""
    h, w, _ = img.shape
    p = np.pad(img.astype(np.int64), ((2, 2), (2, 2), (0, 0)), mode="reflect")    # numpy's "reflect" is REFLECT_101
    c = img.astype(np.int64)
    num = np.zeros((h, w, 3))
    den = np.zeros((h, w))
    cw64, sw64 = CW.astype(np.float64), SW.astype(np.float64)
    for k, (i, j) in enumerate(TAPS):
        v = p[2 + i:2 + i + h, 2 + j:2 + j + w]
        wk = sw64[k] * cw64[np.abs(v - c).sum(-1)]        # a product of two float32 values is exact in float64
        den += wk
        num += v * wk[..., None]
    return num / den[..., None]


def check_bilateral(got, rgb, what):
    oracle = po.bilateral_d5(rgb)
    assert np.array_equal(got, oracle), f"{what}: bilateral output differs from the oracle " + _first_diff(got, oracle)
    q = bilateral_q(rgb)
    frac = q - np.floor(q)
    sure = np.abs(frac - 0.5) > BILATERAL_MARGIN
    want = np.floor(q + 0.5)
    g = got.astype(np.float64)
    assert np.array_equal(g[sure], want[sure]), f"{what}: bilateral byte is not round(q) " + _first_diff(np.where(sure, g, want), want)
    assert np.all((g == np.floor(q)) | (g == np.ceil(q))), f"{what}: bilateral byte not adjacent to q"


def ref_tensor(filt, key):
    scale, offset = (F32(1 / 127.5), F32(-1.0)) if key == "deeplab" else (F32(1 / 255.0), F32(0.0))
    return (filt.astype(np.float64) * np.float64(scale) + np.float64(offset)).astype(np.float32)


def _first_diff(a, b):
    d = np.argwhere(a != b)
    if not d.size:
        return ""
    idx = tuple(d[0])
    return f"(first at {idx}: got {a[idx]}, want {b[idx]}; {len(d)} elements differ)"


class Stem:
    """the model's first convolution (the stem the fused k_stem_u8 path computes) and the tensor the KEEP_TENSORS
    context holds for it"""
    ACT_OPS = {"HARD_SWISH": po.hard_swish, "RELU": po.relu, "RELU6": lambda x: po.relu(x, 3)}

    def __init__(self, key):
        from tools import tflite_graph
        gr = tflite_graph.load(model_path(key))
        op = next(o for o in gr.ops if o.kind == "CONV_2D" and o.inputs[0] == gr.inputs[0])
        self.input = gr.inputs[0]
        self.w, self.b = gr.const_f32(op.inputs[1]), gr.const_f32(op.inputs[2])
        self.stride, self.act = (op.opts["stride_h"], op.opts["stride_w"]), po.ACT[op.opts["act"]]
        self.out = op.outputs[0]
        # an activation op right after the conv is folded into the stem's epilogue: compare its output then
        nxt = [o for o in gr.ops if self.out in o.inputs]
        self.post = (nxt[0].outputs[0], self.ACT_OPS[nxt[0].kind]) if len(nxt) == 1 and nxt[0].kind in self.ACT_OPS else None

    def ref(self, x):
        return po.conv2d(x, self.w, self.b, stride=self.stride, padding=po.PAD_SAME, act=self.act)

    def check(self, g, frame, x, what):
        ref = self.ref(x)
        got = g.tensor(self.out, ref.size, frame)
        if got is None and self.post is not None:
            ref = self.post[1](ref)
            got = g.tensor(self.post[0], ref.size, frame)
        assert got is not None, f"{what}: stem output is not materialised in a KEEP_TENSORS context"
        assert np.array_equal(got.view(np.uint32), ref.ravel().view(np.uint32)), \
            f"{what}: stem output differs from conv2d on the input tensor " + _first_diff(got, ref.ravel())


# ---------------------------------------------------------------------------------------------------------------------
# frames
# ---------------------------------------------------------------------------------------------------------------------
FORMATS = ("bgr", "bgr_pitched", "yuyv_host", "yuyv_dev", "nv12_host", "nv12_dev")
CODES = np.array([0, 1, 15, 16, 17, 127, 128, 129, 235, 236, 239, 240, 241, 254, 255], np.uint8)   # Y / UV range edges, out of gamut


def wire_shape(fmt, W, H):
    return (H, W, 3) if fmt.startswith("bgr") else (H, W, 2) if fmt.startswith("yuyv") else (H * 3 // 2, W)


def to_bgr(fmt, raw):
    if fmt.startswith("yuyv"):
        return cv2.cvtColor(raw, cv2.COLOR_YUV2BGR_YUYV)
    if fmt.startswith("nv12"):
        return cv2.cvtColor(raw, cv2.COLOR_YUV2BGR_NV12)
    return raw


def probe_frame(W, H, part, parts, bg):
    """bilateral probes: isolated pixels 5 apart on a constant background, the colour distance |db|+|dg|+|dr| of probe
    and background running over this frame's share of 0..765; the border rows / columns carry random bytes"""
    rng = np.random.default_rng(1000 + part)
    f = np.full((H, W, 3), bg, np.uint8)
    ds = list(range(part, 766, parts))
    pos = [(y, x) for y in range(2, H - 2, 5) for x in range(2, W - 2, 5)]
    assert len(pos) >= len(ds), (W, H, len(pos), len(ds))
    for (y, x), d in zip(pos, ds):
        split = [min(d, 255), min(max(d - 255, 0), 255), max(d - 510, 0)]
        ch = rng.permutation(3)
        for c, s in zip(ch, split):
            f[y, x, c] = s if bg == 0 else 255 - s
    f[[0, 1, H - 2, H - 1]] = rng.integers(0, 256, (4, W, 3), dtype=np.uint8)
    f[:, [0, 1, W - 2, W - 1]] = rng.integers(0, 256, (H, 4, 3), dtype=np.uint8)
    return f


def make_raw(kind, fmt, W, H, seed, geo=None):
    """one camera frame in the wire format of `fmt`"""
    rng = np.random.default_rng(seed)
    shape = wire_shape(fmt, W, H)
    if kind == "random":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "codes":
        return CODES[rng.integers(0, CODES.size, shape)]
    if kind == "constant":
        return np.full(shape, int(rng.integers(0, 256)), np.uint8)
    if kind == "impulse":
        # single-pixel impulses on a lattice wider than the 2x2 tap footprint of a destination pixel, shifted by the seed
        (_, _, rw, rh), (_, _, iw, ih), _ = geo
        sp = max(5, 2 * math.ceil(max(rw / iw, rh / ih)) + 3)
        oy, ox = seed % sp, (seed // sp) % sp
        r = np.zeros(shape, np.uint8)
        if fmt.startswith("bgr"):
            sub = r[oy::sp, ox::sp, seed % 3]
        elif fmt.startswith("yuyv"):
            r[..., 0], r[..., 1] = 16, 128                   # black
            r[oy::sp, (ox | 1)::sp, 1] = rng.integers(0, 256, r[oy::sp, (ox | 1)::sp, 1].shape)    # a V byte
            sub = r[oy::sp, ox::sp, 0]
        else:
            r[:H], r[H:] = 16, 128
            uv = r[H:][oy // 2::sp, ox::sp]
            uv[...] = rng.integers(0, 256, uv.shape)          # a U or V byte
            sub = r[:H][oy::sp, ox::sp]
        sub[...] = rng.integers(128, 256, sub.shape)
        return r
    if kind.startswith("probe"):
        part, parts, bg = (int(v) for v in kind.split(":")[1:])
        return probe_frame(W, H, part, parts, bg)
    raise ValueError(kind)


def _addr(a):
    return a.ctypes.data


class Buffers:
    """device buffers: torch tensors on the H100, numpy arrays on the emulator (whose device pointers are host memory)"""

    def __init__(self, gpu):
        self.gpu, self.keep = gpu, []

    def dev(self, arr):
        if self.gpu:
            import torch
            t = torch.from_numpy(np.ascontiguousarray(arr).reshape(-1)).to("cuda:0")
            self.keep.append(t)
            return t.data_ptr()
        a = np.ascontiguousarray(arr).reshape(-1).copy()
        self.keep.append(a)
        return _addr(a)

    def empty(self, nbytes):
        return self.dev(np.zeros(nbytes, np.uint8))


def nv12_pitched(frames, pitch, uv_offset, stride):
    n, H3, W = frames.shape
    H = H3 * 2 // 3
    buf = np.full(n * stride, 0x5A, np.uint8)
    for b, f in enumerate(frames):
        img = buf[b * stride:(b + 1) * stride]
        img[:pitch * H].reshape(H, pitch)[:, :W] = f[:H]
        img[uv_offset:uv_offset + pitch * (H // 2)].reshape(H // 2, pitch)[:, :W] = f[H:]
    return buf


def run_call(lib, g, fmt, raw, bufs, ids=None):
    """one composite call of the frames `raw` (wire format of `fmt`); only the mask is written out"""
    n = raw.shape[0]
    W, H = g.width, g.height
    if ids is not None:
        assert fmt == "bgr"
        g.composite_sources(raw, ids, want_out=False, want_yuyv=False)
    elif fmt == "bgr":
        g.composite(raw, want_out=False, want_yuyv=False)
    elif fmt == "bgr_pitched":
        pitch = W * 3 + 13
        stride = pitch * H + 29
        buf = np.full(n * stride, 0xA5, np.uint8)
        for b in range(n):
            buf[b * stride:b * stride + pitch * H].reshape(H, pitch)[:, :W * 3] = raw[b].reshape(H, W * 3)
        mask = np.empty((n, H, W), np.uint8)
        if not lib.bsb_composite(g._h, n, _addr(buf), pitch, stride, None, 0, 0, None, 0, _addr(mask), W * H):
            raise api.BackscrubError(lib.bsb_last_error().decode())
    elif fmt == "yuyv_host":
        g.composite_yuyv_into(np.ascontiguousarray(raw), mask=np.empty((n, H, W), np.uint8))
    elif fmt == "yuyv_dev":
        g.composite_yuyv_device(n, bufs.dev(raw), d_mask=bufs.empty(n * W * H), sync=True)
    elif fmt == "nv12_host":
        g.composite_nv12(raw, want_out=False, want_nv12=False)
    elif fmt == "nv12_dev":
        # pitched like a decoder surface: row pitch > W, the UV plane past pitch * H, frames further apart than they need
        pitch = W + 24
        uv = pitch * (H + 6)
        stride = uv + pitch * (H // 2) + 40
        g.composite_nv12_device(n, bufs.dev(nv12_pitched(raw, pitch, uv, stride)), d_mask=bufs.empty(n * W * H), sync=True,
                                pitch=pitch, uv_offset=uv, in_stride=stride)
    else:
        raise ValueError(fmt)


# ---------------------------------------------------------------------------------------------------------------------
# the check of one call
# ---------------------------------------------------------------------------------------------------------------------
class Context:
    """One context and the checks of its calls.  `stem_x2` selects the stem kernel: the switch is read when a call is
    enqueued (on the GPU: when its graph is captured), so it stays set for the context's whole life and close() puts
    the default back."""

    def __init__(self, lib, key, W, H, n, keep=True, gpu=False, stem_x2=None):
        self.lib, self.key, self.W, self.H, self.keep = lib, key, W, H, keep
        self.mw, self.mh = MODEL_HW[key]
        self.geo = ref_geometry(key, W, H)
        assert self.geo is not None, (key, W, H)
        self.stem_x2 = stem_x2
        if stem_x2 is not None:
            lib.bsb_set_tuning(b"stem_x2", int(stem_x2))
        self.g = None
        try:
            self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=n, flags=KEEP_TENSORS if keep else 0)
            assert (self.g.roidim, self.g.in_roidim, self.g.out_roidim) == tuple(self.geo), (key, W, H)
        except BaseException:
            self.close()
            raise
        self.stem = Stem(key) if keep else None
        self.bufs = Buffers(gpu)

    def run(self, fmt, raws, ids=None, tag=""):
        raws = np.ascontiguousarray(np.stack(raws))
        run_call(self.lib, self.g, fmt, raws, self.bufs, ids)
        self.bufs.keep.clear()
        _, (ix, iy, iw, ih), _ = self.geo
        for b in range(raws.shape[0]):
            what = f"{self.key} {self.W}x{self.H} {fmt}{tag} frame {b}"
            bgr = to_bgr(fmt, raws[b])
            want = ref_in_u8(bgr, self.geo, self.mw, self.mh)
            got = self.g.stage_u8(0, b)
            pad = np.ones((self.mh, self.mw), bool)
            pad[iy:iy + ih, ix:ix + iw] = False
            assert not got[pad].any(), f"{what}: the letterbox of the resized input is not zero " + _first_diff(got * pad[..., None], want)
            assert np.array_equal(got, want), f"{what}: resized input differs from cv2 " + _first_diff(got, want)
            filt = self.g.stage_u8(1, b)
            check_bilateral(filt, want, what)
            if self.keep:
                x = ref_tensor(filt, self.key)
                t = self.g.tensor(self.stem.input, x.size, b)
                assert t is not None and np.array_equal(t.view(np.uint32), x.ravel().view(np.uint32)), \
                    f"{what}: input tensor differs from r * scale + offset " + _first_diff(t, x.ravel())
                self.stem.check(self.g, b, x, what)

    def _restore_tuning(self):
        if self.stem_x2 is not None:
            self.lib.bsb_set_tuning(b"stem_x2", 1)

    def close(self):
        if self.g is not None:
            self.g.close()
        self._restore_tuning()


def geometries(key):
    """the pixel-fixture geometries of one model: name -> (W, H)"""
    mw, mh = MODEL_HW[key]
    geo = {"one_to_one": (mw, mh), "area_2x": (2 * mw, 2 * mh)}
    geo.update({"meet_full": {"upscale": (128, 72), "downscale": (640, 480), "equal_aspect": (1920, 1080)},
                "meet_lite": {"upscale": (17, 9), "downscale": (640, 480), "equal_aspect": (80, 48)},
                "mlkit": {"upscale": (2, 2), "downscale": (1280, 720)},
                "deeplab": {"upscale": (128, 72), "downscale": (640, 480)},
                "bodypix": {"upscale": (17, 9), "downscale": (1280, 720)}}[key])
    geo["odd_crop"] = {"meet_full": (1296, 712), "mlkit": (642, 480)}.get(key) or odd_crop(key)
    geo["odd_letterbox"] = (480, 642) if ref_geometry(key, 480, 642)[1][2] % 2 else odd_letterbox(key)
    geo["wide"] = (16384, 2)
    geo["tall"] = (2, _last_accepted(key, 2, 1) // 2 * 2)
    return geo


def odd_crop(key):
    """a landscape frame (even W and H) whose crop has an odd x and, where the model's aspect allows it with an even
    height, an odd width (Meet full 1296x712: 15 / 1265; a square model crops H columns: MLKit 642x480, x 81)"""
    for want_odd_w in (True, False):
        for H in (480, 712, 360):
            for W in range(H + 2, H * 3, 2):
                geo = ref_geometry(key, W, H)
                if geo and geo[0][0] % 2 and (geo[0][2] % 2 or not want_odd_w):
                    return W, H
    raise AssertionError(key)


def odd_letterbox(key):
    """a portrait frame (even W and H) whose letterbox has an odd width (MLKit 480x642: 191 at x 32)"""
    for W in (480, 360, 720):
        for H in range(W + 2, W * 2, 2):
            geo = ref_geometry(key, W, H)
            if geo and geo[1][2] % 2 and geo[1][2] < MODEL_HW[key][0]:
                return W, H
    raise AssertionError(key)


def kinds_for(name, fmt, call):
    """three distinct frames per call; the 1:1 BGR calls carry bilateral probes"""
    if name == "one_to_one" and fmt.startswith("bgr"):
        return ["probe:%d:3:%d" % (call % 3, 255 * (call & 1)), "random", "probe:%d:3:%d" % ((call + 1) % 3, 255 * (1 - (call & 1)))]
    rest = ["codes", "impulse", "constant"]
    return ["random", rest[call % 3], rest[(call + 1) % 3]]


def run_geometry(lib, key, name, W, H, fmts, gpu, n=3, keep=True, calls=1):
    ctx = Context(lib, key, W, H, n, keep=keep, gpu=gpu)
    try:
        for fmt in fmts:
            if (W % 2 or H % 2) and not fmt.startswith("bgr"):
                continue
            for call in range(calls):
                kinds = kinds_for(name, fmt, call)
                raws = [make_raw(k, fmt, W, H, seed=97 * call + 13 * b + 1, geo=ctx.geo) for b, k in enumerate(kinds)]
                if n > 3:
                    raws += [make_raw("random", fmt, W, H, seed=5000 + b) for b in range(n - 3)]
                ctx.run(fmt, raws, tag=f" call {call}")
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------
# references and helpers on their own
# ---------------------------------------------------------------------------------------------------------------------
def test_geometry_restatement_examples():
    """the cases the fixtures are chosen for"""
    assert ref_geometry("mlkit", 642, 480)[0] == [81, 0, 480, 480]
    assert ref_geometry("mlkit", 480, 642)[1] == [32, 0, 191, 256]
    assert ref_geometry("meet_full", 1296, 712)[0] == [15, 0, 1265, 712]
    assert ref_geometry("meet_full", 1920, 1080)[1] == [0, 0, 256, 144]
    # 96 / 0.6f rounds to 160 (0.6f is below 0.6): Meet lite at 80x48 takes the letterbox branch with the full width
    assert ref_geometry("meet_lite", 80, 48)[1] == [0, 0, 160, 96]
    assert ref_geometry("bodypix", 480, 642)[2] == [4, 0, 24, 33]
    assert ref_geometry("mlkit", 1, 257) is None and ref_geometry("mlkit", 1, 256) is not None


def test_bilateral_float64_reference_agrees_with_cv2():
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (37, 41, 3), dtype=np.uint8)
    q = bilateral_q(img)
    ref = cv2.bilateralFilter(img, 5, 100, 100)
    assert np.abs(ref.astype(np.float64) - q).max() < 1.0 + 1e-9


def test_probe_frames_cover_every_lut_index():
    for W, H in ((160, 96), (256, 256), (257, 257)):
        seen = set()
        for part in range(3):
            for bg in (0, 255):
                f = probe_frame(W, H, part, 3, bg)
                inner = f[2:H - 2, 2:W - 2].astype(int)
                seen |= set(np.abs(inner - bg).sum(-1).ravel().tolist())
        assert seen == set(range(766)), (W, H)


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


@pytest.mark.parametrize("key", list(MODEL_HW))
def test_emu_geometry_sweep(emu_lib, key):
    """bsb_geometry and the oracle's geometry equal the restatement; a size is refused exactly where an extent is not
    positive; an accepted ROI lies inside the frame and the model input"""
    mw, mh = MODEL_HW[key]
    sizes = sweep_sizes(key)
    assert len(sizes) > 250, len(sizes)
    refused = 0
    for W, H in sizes:
        geo = ref_geometry(key, W, H)
        if geo is None:
            refused += 1
            with pytest.raises(api.BackscrubError, match="degenerate ROI"):
                api.MaskGen(emu_lib, model_path(key), W, H, max_batch=1)
            continue
        g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=1)
        got = (g.roidim, g.in_roidim, g.out_roidim)
        g.close()
        assert got == geo, (key, W, H, got, geo)
        o = po.MaskGen(model_path(key), W, H)
        assert (o.roidim, o.in_roidim, o.out_roidim) == geo, (key, W, H)
        o.close()
        (rx, ry, rw, rh), (ix, iy, iw, ih), (ox, oy, ow_, oh_) = geo
        assert 0 <= rx and rx + rw <= W and 0 <= ry and ry + rh <= H, (key, W, H, geo)
        assert 0 <= ix and ix + iw <= mw and 0 <= iy and iy + ih <= mh, (key, W, H, geo)
        assert 0 <= ox and ox + ow_ <= OUT_HW[key][0] and 0 <= oy and oy + oh_ <= OUT_HW[key][1], (key, W, H, geo)
    assert refused > 0, key


# Meet lite and MLKit on the emulator: every geometry class once, each format at least once, three frames per call
EMU_CASES = [
    ("meet_lite", "one_to_one", ("bgr", "yuyv_dev")),
    ("meet_lite", "area_2x", ("nv12_dev",)),
    ("meet_lite", "upscale", ("bgr_pitched",)),
    ("meet_lite", "equal_aspect", ("yuyv_host",)),
    ("meet_lite", "odd_crop", ("nv12_host", "yuyv_host")),
    ("meet_lite", "odd_letterbox", ("yuyv_dev",)),
    ("meet_lite", "downscale", ("nv12_dev",)),
    ("meet_lite", "wide", ("bgr",)),
    ("mlkit", "one_to_one", ("bgr_pitched",)),
    ("mlkit", "area_2x", ("yuyv_host",)),
    ("mlkit", "odd_crop", ("nv12_dev", "yuyv_dev")),
    ("mlkit", "odd_letterbox", ("bgr",)),
    ("mlkit", "upscale", ("yuyv_dev",)),
    ("mlkit", "tall", ("bgr",)),
]


@pytest.mark.parametrize("key,name,fmts", EMU_CASES, ids=[f"{k}-{n}" for k, n, _ in EMU_CASES])
def test_emu_pre_process(emu_lib, key, name, fmts):
    W, H = geometries(key)[name]
    run_geometry(emu_lib, key, name, W, H, fmts, gpu=False)


@pytest.mark.parametrize("key", ["meet_lite", "mlkit"])
def test_emu_stem_x2_off(emu_lib, key):
    """the one-pixel stem kernel k_stem_u8 (stem_x2 off for the context's whole life) on the same checks; the other
    emulator cases run k_stem_u8_x2, the default for the even stem output widths of Meet and MLKit"""
    mw, mh = MODEL_HW[key]
    ctx = Context(emu_lib, key, 2 * mw, 2 * mh, 3, stem_x2=0)
    try:
        ctx.run("bgr", [make_raw("random", "bgr", 2 * mw, 2 * mh, seed=s) for s in range(3)])
    finally:
        ctx.close()


def test_emu_sources_non_consecutive_ids(emu_lib):
    key = "meet_lite"
    W, H = odd_crop(key)
    ctx = Context(emu_lib, key, W, H, 3)
    try:
        ctx.g.set_sources(8)
        ctx.run("bgr", [make_raw(k, "bgr", W, H, seed=s, geo=ctx.geo) for s, k in enumerate(("impulse", "random", "codes"))],
                ids=[6, 1, 4], tag=" sources")
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


GPU_CASES = [(k, n) for k in MODEL_HW for n in ("one_to_one", "area_2x", "upscale", "downscale", "odd_crop", "odd_letterbox", "wide",
                                                "tall")] + [("meet_full", "equal_aspect"), ("meet_lite", "equal_aspect")]


@pytest.mark.gpu
@pytest.mark.parametrize("key,name", GPU_CASES, ids=[f"{k}-{n}" for k, n in GPU_CASES])
def test_gpu_pre_process(gpu_lib, key, name):
    """every format and layout, two calls each (the second replays the captured graph on new frames)"""
    W, H = geometries(key)[name]
    run_geometry(gpu_lib, key, name, W, H, FORMATS, gpu=True, calls=2)


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(MODEL_HW))
@pytest.mark.parametrize("stem_x2", [0, 1])
def test_gpu_stem(gpu_lib, key, stem_x2):
    """both stem kernels.  DeepLab's and BodyPix's stem output is 129 wide (odd), so they run the one-pixel kernel
    under either setting; Meet and MLKit run k_stem_u8 with stem_x2 off and k_stem_u8_x2 with it on"""
    mw, mh = MODEL_HW[key]
    for W, H in ((mw, mh), (2 * mw, 2 * mh), odd_crop(key)):
        ctx = Context(gpu_lib, key, W, H, 3, gpu=True, stem_x2=stem_x2)
        try:
            ctx.run("bgr", [make_raw(k, "bgr", W, H, seed=s, geo=ctx.geo) for s, k in enumerate(("random", "codes", "impulse"))])
        finally:
            ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [True, False])
def test_gpu_sources_non_consecutive_ids(gpu_lib, keep):
    key = "mlkit"
    W, H = odd_crop(key)
    ctx = Context(gpu_lib, key, W, H, 4, keep=keep, gpu=True)
    try:
        ctx.g.set_sources(9)
        ctx.run("bgr", [make_raw(k, "bgr", W, H, seed=s, geo=ctx.geo) for s, k in enumerate(("impulse", "random", "codes", "random"))],
                ids=[7, 2, 8, 0], tag=" sources")
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["deeplab", "bodypix"])
def test_gpu_large_batch_257(gpu_lib, key):
    """2 x SMs + 3 frames at 257x257 1:1 in one call: the grids end in partial blocks, every frame is checked"""
    import torch
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 3
    run_geometry(gpu_lib, key, "one_to_one", 257, 257, ("bgr",), gpu=True, n=n, keep=(key == "deeplab"))
