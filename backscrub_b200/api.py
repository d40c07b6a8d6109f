"""Host-side mirror of the reference's interface for the per-frame path.

Names follow the reference: `bs_maskgen_new / bs_maskgen_process / bs_maskgen_delete /
bs_tensorflow_version` (lib/libbackscrub.h:13-39), `alpha_blend`, `convert_rgb_to_yuyv`
(app/deepseg.cc:87-134), `load_background / grab_background` (app/background.h:14-23);
numpy arrays stand in for cv::Mat.  Everything computes on the GPU through the C ABI
(include/backscrub_b200.h); there is no CPU path.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _binding as B


class BackscrubError(RuntimeError):
    pass


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class MaskGen:
    """One mask-generation context == one video stream (holds the temporal IIR state).

    `lib` is the bound shared library (the product library by default)."""

    def __init__(self, lib, modelname: str, width: int, height: int, *, threads: int = 2, device: int = 0,
                 max_batch: int = 1, flags: int = 0, ondebug=None, onprep=None, oninfer=None, onmask=None):
        self._lib = lib
        self._msgs = []
        self._user_debug = ondebug

        def _dbg(_ctx, msg):
            text = msg.decode("utf-8", "replace")
            self._msgs.append(text)
            if self._user_debug:
                self._user_debug(text)

        mk = lambda f: B.STAGE_CB(lambda _c: f()) if f else C.cast(None, B.STAGE_CB)
        self._cbs = (B.DEBUG_CB(_dbg), mk(onprep), mk(oninfer), mk(onmask))  # keep alive
        self._h = lib.bsb_maskgen_new_ex(modelname.encode(), width, height, device, max_batch, flags, *self._cbs, None)
        if not self._h:
            raise BackscrubError("".join(self._msgs).strip() or lib.bsb_last_error().decode())
        self.width, self.height, self.max_batch, self.device = width, height, max_batch, device
        self.out_width, self.out_height = width, height
        self.out_channels = 3                        # bytes per pixel of the `out` frames: 3 (BGR), 4 (BGRA, set_out_format)
        self._n_sources, self._src_out = 0, {}       # sources with their own output size: source -> (w, h)
        r, i, o = (C.c_int * 4)(), (C.c_int * 4)(), (C.c_int * 4)()
        ih, oh = (C.c_int * 3)(), (C.c_int * 3)()
        lib.bsb_geometry(self._h, r, i, o, ih, oh)
        self.roidim, self.in_roidim, self.out_roidim = list(r), list(i), list(o)
        self.in_hwc, self.out_hwc = list(ih), list(oh)

    # -- lifecycle
    def close(self):
        if getattr(self, "_h", None):
            self._lib.bsb_maskgen_delete(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def _fail(self, what):
        raise BackscrubError(f"{what}: {self._lib.bsb_last_error().decode()}")

    # -- the reference's calls
    def process(self, frame: np.ndarray) -> np.ndarray:
        """bs_maskgen_process: BGR u8 H x W x 3 -> mask u8 H x W (255 = background)."""
        frame = np.ascontiguousarray(frame, np.uint8)
        if frame.shape != (self.height, self.width, 3):
            raise BackscrubError(f"frame shape {frame.shape} != {(self.height, self.width, 3)}")
        mp, pitch = B.u8p(), C.c_size_t()
        if not self._lib.bsb_maskgen_process(self._h, _ptr(frame), self.width * 3, C.byref(mp), C.byref(pitch)):
            self._fail("bs_maskgen_process")
        return np.ctypeslib.as_array(mp, shape=(self.height, pitch.value))[:, : self.width].copy()

    def set_background(self, bg_raw: np.ndarray):
        bg_raw = np.ascontiguousarray(bg_raw, np.uint8)
        if not self._lib.bsb_set_background(self._h, _ptr(bg_raw), bg_raw.shape[1], bg_raw.shape[0], bg_raw.shape[1] * 3):
            self._fail("bsb_set_background")

    def set_background_ring(self, frames: np.ndarray, advance: int = 1):
        """Animated background: frames [count, bh, bw, 3] -> device-resident ring (app/background.cc video branch)."""
        frames = np.ascontiguousarray(frames, np.uint8)
        c, bh, bw, _ = frames.shape
        if not self._lib.bsb_set_background_ring(self._h, _ptr(frames), c, bw, bh, bw * 3, bh * bw * 3, int(advance)):
            self._fail("bsb_set_background_ring")

    def set_background_cursor(self, index: int):
        if not self._lib.bsb_set_background_cursor(self._h, int(index)):
            self._fail("bsb_set_background_cursor")

    def set_bgblur(self, ksize: int):
        """`-p bgblur:k` (app/deepseg.cc:657-658); 0 = off."""
        if not self._lib.bsb_set_bgblur(self._h, int(ksize)):
            self._fail("bsb_set_bgblur")

    def set_output(self, flip_h=False, flip_v=False, out_size=None):
        """cv::flip + cv::resize to the virtual-camera size (app/deepseg.cc:667-679); out_size = (w, h)."""
        ow, oh = out_size if out_size else (0, 0)
        if not self._lib.bsb_set_output(self._h, int(bool(flip_h)), int(bool(flip_v)), int(ow), int(oh)):
            self._fail("bsb_set_output")
        w, h = C.c_int(), C.c_int()
        self._lib.bsb_output_size(self._h, C.byref(w), C.byref(h))
        self.out_width, self.out_height = w.value, h.value

    def set_filter(self, active: bool):
        """the filter switch (the `s` key, app/deepseg.cc:624,639-664): False passes the camera frame through, flipped,
        resized and converted as usual; the mask is still computed and written and the smoother still advances."""
        if not self._lib.bsb_set_filter(self._h, int(bool(active))):
            self._fail("bsb_set_filter")

    def set_mask_interval(self, k: int):
        """segment every k-th frame (1..256, default 1); the frames between are composited with their camera's latest mask
        (include/backscrub_b200.h, bsb_set_mask_interval)"""
        if not self._lib.bsb_set_mask_interval(self._h, int(k)):
            self._fail("bsb_set_mask_interval")

    def set_mask_refine(self, sigma: int):
        """mask edge refinement strength 0..255 (0 = off, the default): each frame's mask is upsampled guided by its own
        camera frame (include/backscrub_b200.h, bsb_set_mask_refine)"""
        if not self._lib.bsb_set_mask_refine(self._h, int(sigma)):
            self._fail("bsb_set_mask_refine")

    _BLUR_MODE = {"plain": 0, "masked": 1}

    def set_blur_mode(self, mode: str):
        """camera blur mode: "plain" (the default) blurs the whole camera frame, "masked" leaves the person out of the
        background blur (include/backscrub_b200.h, bsb_set_blur_mode)"""
        if not self._lib.bsb_set_blur_mode(self._h, self._BLUR_MODE.get(mode, -2)):
            self._fail("bsb_set_blur_mode")

    _FRAMING = {"off": 0, "rect": 1, "auto": 2}

    def _framing_args(self, what, mode, rect):
        if mode not in self._FRAMING:
            raise BackscrubError(f"{what}: unknown framing mode {mode!r} (\"off\", \"rect\" or \"auto\")")
        x, y, w, h = rect if rect is not None else (0, 0, 0, 0)
        return self._FRAMING[mode], int(x), int(y), int(w), int(h)

    def set_framing(self, mode: str = "off", rect=None):
        """framing of every frame's output (include/backscrub_b200.h, bsb_set_framing): "off" (the whole frame), "rect"
        (the crop rect = (x, y, w, h) of the camera frame) or "auto" (a crop that follows the person the mask finds)"""
        if not self._lib.bsb_set_framing(self._h, *self._framing_args("bsb_set_framing", mode, rect)):
            self._fail("bsb_set_framing")

    def set_framing_auto(self, max_zoom_pct: int = 300, margin_pct: int = 10, speed: int = 32):
        """auto-framing parameters: zoom limit 100..1000 %, headroom and side margin 0..100 % of the person's height,
        speed 1..256 (1/256 of the remaining distance per frame; 256 jumps)"""
        if not self._lib.bsb_set_framing_auto(self._h, int(max_zoom_pct), int(margin_pct), int(speed)):
            self._fail("bsb_set_framing_auto")

    def set_source_framing(self, source: int, mode=None, rect=None):
        """framing of one source: None = follow set_framing, including later changes; otherwise as set_framing"""
        args = (-1, 0, 0, 0, 0) if mode is None else self._framing_args("bsb_set_source_framing", mode, rect)
        if not self._lib.bsb_set_source_framing(self._h, int(source), *args):
            self._fail("bsb_set_source_framing")

    def framing(self, frame: int = 0):
        """the crop (x, y, w, h) frame `frame` of the last call showed; the whole frame when that call was not framed"""
        r = (C.c_int * 4)()
        if not self._lib.bsb_get_framing(self._h, int(frame), r):
            self._fail("bsb_get_framing")
        return tuple(r)

    def set_out_format(self, fmt: str):
        """format of the `out` frames of every composite call: "bgr" (the composite, the default) or "bgra" (the camera with
        alpha 255 - mask, straight alpha, flipped and resized like the composite; the video output and the mask are
        unchanged).  The wrappers then allocate out as [n, oh, ow, 4], and sources strides count 4 bytes per pixel."""
        code = {"bgr": 0, "bgra": 1}.get(fmt, -1) if isinstance(fmt, str) else -1
        if code < 0:
            raise BackscrubError(f"unknown output format {fmt!r} (\"bgr\" or \"bgra\")")
        if not self._lib.bsb_set_out_format(self._h, code):
            self._fail("bsb_set_out_format")
        self.out_channels = 3 + code

    @staticmethod
    def _live_args(frames, fmt, size, pitch, uv_offset):
        """(pointer, format code, w, h, pitch, uv_offset) of a live background: an int device pointer or a CUDA tensor"""
        code = {"bgr": 0, "nv12": 1}.get(fmt, -1) if isinstance(fmt, str) else -1
        if code < 0:
            raise BackscrubError(f"unknown live background format {fmt!r} (\"bgr\" or \"nv12\")")
        if frames is None:
            return None, code, 0, 0, 0, 0
        ptr = frames.data_ptr() if hasattr(frames, "data_ptr") else int(frames)
        w, h = size
        p = (w * 3 if code == 0 else w) if pitch is None else pitch
        uv = (p * h if code == 1 else 0) if uv_offset is None else uv_offset
        return ptr, code, int(w), int(h), int(p), int(uv)

    def set_live_background(self, frames, fmt="bgr", size=None, pitch=None, uv_offset=None, frame_stride=0):
        """Live background of plain calls: a device image (int pointer, or a CUDA torch.Tensor's data_ptr()) that every later
        plain call resizes to W x H, blurs at the context's strength and blends, inside the call.  fmt "bgr" (rows `pitch`
        bytes apart, default w*3) or "nv12" (pitch default w, UV plane at `uv_offset`, default pitch*h); size = (w, h).
        Frame b of a call blends frames + b*frame_stride (0: one image for every frame).  None clears.  The memory must stay
        valid and unchanged until the calls that read it have completed on bsb_stream; a tensor is kept referenced here
        until it is replaced."""
        ptr, code, w, h, p, uv = self._live_args(frames, fmt, size, pitch, uv_offset)
        if not self._lib.bsb_set_live_background(self._h, ptr, code, w, h, p, uv, int(frame_stride)):
            self._fail("bsb_set_live_background")
        self._live_refs = getattr(self, "_live_refs", {})
        self._live_refs[None] = frames

    def set_source_live_background(self, source: int, frame, fmt="bgr", size=None, pitch=None, uv_offset=None):
        """Live background of one source of a sources context (set_live_background's image rules): every later sources call
        carrying a frame of `source` blends it, at the source's strength, where the source's background is "default".
        None clears."""
        ptr, code, w, h, p, uv = self._live_args(frame, fmt, size, pitch, uv_offset)
        if not self._lib.bsb_set_source_live_background(self._h, int(source), ptr, code, w, h, p, uv):
            self._fail("bsb_set_source_live_background")
        self._live_refs = getattr(self, "_live_refs", {})
        self._live_refs[int(source)] = frame

    def background(self) -> np.ndarray:
        out = np.empty((self.height, self.width, 3), np.uint8)
        if not self._lib.bsb_get_background(self._h, _ptr(out), self.width * 3):
            self._fail("bsb_get_background")
        return out

    def composite(self, frames: np.ndarray, want_out=True, want_yuyv=True, want_mask=True):
        """Fused path on HOST buffers: frames [n, H, W, 3] (or [H, W, 3]) -> (out, yuyv, mask)."""
        single = frames.ndim == 3
        frames = np.ascontiguousarray(frames[None] if single else frames, np.uint8)
        n = frames.shape[0]
        if frames.shape[1:] != (self.height, self.width, 3):
            raise BackscrubError(f"frame shape {frames.shape[1:]} != {(self.height, self.width, 3)}")
        fb, npx = self.height * self.width * 3, self.height * self.width
        ow, oh = self.out_width, self.out_height
        oc = self.out_channels
        out = np.empty((n, oh, ow, oc), np.uint8) if want_out else None
        yuyv = np.empty((n, oh, ow, 2), np.uint8) if want_yuyv else None
        mask = np.empty((n, self.height, self.width), np.uint8) if want_mask else None
        ok = self._lib.bsb_composite(self._h, n, _ptr(frames), self.width * 3, fb,
                                     _ptr(out) if want_out else None, ow * oc, ow * oh * oc,
                                     _ptr(yuyv) if want_yuyv else None, ow * oh * 2,
                                     _ptr(mask) if want_mask else None, npx)
        if not ok:
            self._fail("bsb_composite")
        pick = (lambda a: a[0] if single and a is not None else a)
        return pick(out), pick(yuyv), pick(mask)

    def composite_into(self, frames: np.ndarray, out=None, yuyv=None, mask=None):
        """bsb_composite into caller-provided (e.g. pinned) host arrays; frames [n, H, W, 3]."""
        n = frames.shape[0]
        fb, npx = self.height * self.width * 3, self.height * self.width
        ow, opx = self.out_width, self.out_width * self.out_height
        ok = self._lib.bsb_composite(self._h, n, _ptr(frames), self.width * 3, fb,
                                     _ptr(out) if out is not None else None, ow * self.out_channels, opx * self.out_channels,
                                     _ptr(yuyv) if yuyv is not None else None, opx * 2,
                                     _ptr(mask) if mask is not None else None, npx)
        if not ok:
            self._fail("bsb_composite")

    def composite_yuyv_into(self, yuyv_frames: np.ndarray, out=None, yuyv=None, mask=None):
        """bsb_composite_yuyv: camera YUYV frames [n, H, W, 2] in, results into caller-provided host arrays."""
        n = yuyv_frames.shape[0]
        npx, opx = self.height * self.width, self.out_width * self.out_height
        ok = self._lib.bsb_composite_yuyv(self._h, n, _ptr(yuyv_frames), npx * 2,
                                          _ptr(out) if out is not None else None, opx * self.out_channels,
                                          _ptr(yuyv) if yuyv is not None else None, opx * 2,
                                          _ptr(mask) if mask is not None else None, npx)
        if not ok:
            self._fail("bsb_composite_yuyv")

    def composite_yuyv(self, yuyv_frames: np.ndarray):
        yuyv_frames = np.ascontiguousarray(yuyv_frames, np.uint8)
        n = yuyv_frames.shape[0]
        out = np.empty((n, self.out_height, self.out_width, self.out_channels), np.uint8)
        yuyv = np.empty((n, self.out_height, self.out_width, 2), np.uint8)
        mask = np.empty((n, self.height, self.width), np.uint8)
        self.composite_yuyv_into(yuyv_frames, out, yuyv, mask)
        return out, yuyv, mask

    def decode_mjpg(self, jpeg: bytes) -> np.ndarray:
        """one MJPG camera frame -> BGR, decoded on the GPU (NVJPG); what composite_mjpg feeds the pipeline"""
        buf = np.frombuffer(jpeg, np.uint8)
        out = np.empty((self.height, self.width, 3), np.uint8)
        if not self._lib.bsb_decode_mjpg(self._h, _ptr(buf), buf.size, _ptr(out)):
            self._fail("bsb_decode_mjpg")
        return out

    def composite_mjpg(self, jpegs):
        """MJPG camera ingest (app/deepseg.cc:548-553): a list of JPEG byte strings -> (out, yuyv, mask)"""
        bufs = [np.frombuffer(j, np.uint8) for j in jpegs]
        n = len(bufs)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        sizes = (C.c_size_t * n)(*[b.size for b in bufs])
        out = np.empty((n, self.out_height, self.out_width, self.out_channels), np.uint8)
        yuyv = np.empty((n, self.out_height, self.out_width, 2), np.uint8)
        mask = np.empty((n, self.height, self.width), np.uint8)
        opx = self.out_width * self.out_height
        if not self._lib.bsb_composite_mjpg(self._h, n, ptrs, sizes, _ptr(out), opx * self.out_channels, _ptr(yuyv), opx * 2, _ptr(mask), self.height * self.width):
            self._fail("bsb_composite_mjpg")
        return out, yuyv, mask

    def composite_device(self, n, d_frames, d_out=0, d_yuyv=0, d_mask=0, sync=False):
        """Fused path on DEVICE pointers (ints, e.g. torch.Tensor.data_ptr()); tightly packed frames."""
        fb, npx, opx = self.height * self.width * 3, self.height * self.width, self.out_width * self.out_height
        if not self._lib.bsb_composite_device(self._h, n, d_frames, fb, d_out or None, opx * self.out_channels, d_yuyv or None, opx * 2,
                                              d_mask or None, npx, int(sync)):
            self._fail("bsb_composite_device")

    def composite_yuyv_device(self, n, d_yuyv_in, d_out=0, d_yuyv=0, d_mask=0, sync=False):
        """Fused path from DEVICE-resident camera YUYV frames (tightly packed)."""
        npx, opx = self.height * self.width, self.out_width * self.out_height
        if not self._lib.bsb_composite_yuyv_device(self._h, n, d_yuyv_in, d_out or None, opx * self.out_channels, d_yuyv or None, opx * 2,
                                                   d_mask or None, npx, int(sync)):
            self._fail("bsb_composite_yuyv_device")

    # -- NV12 camera frames in, NV12 composites out (definitions in include/backscrub_b200.h)
    def _nv12_layout(self, pitch, uv_offset, in_stride):
        pitch = self.width if pitch is None else int(pitch)
        uv_offset = pitch * self.height if uv_offset is None else int(uv_offset)
        in_stride = uv_offset + pitch * (self.height // 2) if in_stride is None else int(in_stride)
        return pitch, uv_offset, in_stride

    def composite_nv12(self, frames: np.ndarray, want_out=True, want_nv12=True, want_mask=True):
        """HOST buffers: tightly packed NV12 frames [n, H*3/2, W] -> (out [n, oh, ow, 3], nv12 [n, oh*3/2, ow], mask)."""
        frames = np.ascontiguousarray(frames, np.uint8)
        n = frames.shape[0]
        if frames.shape[1:] != (self.height * 3 // 2, self.width):
            raise BackscrubError(f"frame shape {frames.shape[1:]} != {(self.height * 3 // 2, self.width)}")
        npx = self.height * self.width
        ow, oh = self.out_width, self.out_height
        oc = self.out_channels
        out = np.empty((n, oh, ow, oc), np.uint8) if want_out else None
        nv12 = np.empty((n, oh * 3 // 2, ow), np.uint8) if want_nv12 else None
        mask = np.empty((n, self.height, self.width), np.uint8) if want_mask else None
        ok = self._lib.bsb_composite_nv12(self._h, n, _ptr(frames), npx * 3 // 2,
                                          _ptr(out) if want_out else None, ow * oh * oc,
                                          _ptr(nv12) if want_nv12 else None, ow * oh * 3 // 2,
                                          _ptr(mask) if want_mask else None, npx)
        if not ok:
            self._fail("bsb_composite_nv12")
        return out, nv12, mask

    def composite_nv12_device(self, n, d_nv12, d_out=0, d_nv12_out=0, d_mask=0, sync=False, pitch=None, uv_offset=None, in_stride=None):
        """DEVICE-resident camera NV12 frames (row pitch, UV plane offset and frame stride default to tight packing) ->
        BGR / tightly packed NV12 / mask on the device; asynchronous unless `sync`."""
        p, uv, st = self._nv12_layout(pitch, uv_offset, in_stride)
        npx, opx = self.height * self.width, self.out_width * self.out_height
        if not self._lib.bsb_composite_nv12_device(self._h, n, d_nv12, p, uv, st, d_out or None, opx * self.out_channels, d_nv12_out or None, opx * 3 // 2,
                                                   d_mask or None, npx, int(sync)):
            self._fail("bsb_composite_nv12_device")

    # -- independent sources: one frame from each of several cameras per call
    @staticmethod
    def _ids(ids):
        ids = [int(i) for i in ids]
        return len(ids), (C.c_int * max(1, len(ids)))(*ids)

    def set_sources(self, n_sources: int):
        """n_sources zeroed smoother states + per-source background slots (again: everything reset)."""
        if not self._lib.bsb_set_sources(self._h, int(n_sources)):
            self._fail("bsb_set_sources")
        self._n_sources, self._src_out = int(n_sources), {}

    def reset_source(self, source: int):
        """start `source` over as a new camera (its smoother state is zeroed)"""
        if not self._lib.bsb_reset_source(self._h, int(source)):
            self._fail("bsb_reset_source")

    def set_source_background(self, source: int, bg_raw=None):
        """background of one source (resized like set_background); None = blend the context background again."""
        if bg_raw is None:
            ok = self._lib.bsb_set_source_background(self._h, int(source), None, 0, 0, 0)
        else:
            bg_raw = np.ascontiguousarray(bg_raw, np.uint8)
            ok = self._lib.bsb_set_source_background(self._h, int(source), _ptr(bg_raw), bg_raw.shape[1], bg_raw.shape[0], bg_raw.shape[1] * 3)
        if not ok:
            self._fail("bsb_set_source_background")

    def set_source_background_ring(self, source: int, frames: np.ndarray, advance: int = 1):
        """Animated background of one source: frames [count, bh, bw, 3] -> the source's device-resident ring (resized like
        set_background_ring, blurred at the source's strength).  Each sources call carrying a frame of the source blends
        ring image `cursor`, then moves the cursor on by `advance`; advance 0 leaves pacing to
        set_source_background_cursor.  set_source_background(source, None) clears it."""
        frames = np.ascontiguousarray(frames, np.uint8)
        c, bh, bw, _ = frames.shape
        if not self._lib.bsb_set_source_background_ring(self._h, int(source), _ptr(frames), c, bw, bh, bw * 3, bh * bw * 3, int(advance)):
            self._fail("bsb_set_source_background_ring")

    def set_source_background_cursor(self, source: int, index: int):
        """the ring image the next call carrying a frame of `source` blends (host bookkeeping only)"""
        if not self._lib.bsb_set_source_background_cursor(self._h, int(source), int(index)):
            self._fail("bsb_set_source_background_cursor")

    def set_source_effect(self, source: int, background: str = "default", bgblur: int = -1):
        """background effect of one source: background "default" (its own image, else the context's) or "none" (no
        image: the blurred camera frame when the strength is > 0, else green); bgblur -1 = follow set_bgblur, 0 = off,
        odd 1..255."""
        kinds = {"default": 0, "none": 1}
        if background not in kinds:
            raise BackscrubError(f"bsb_set_source_effect: unknown background {background!r} (\"default\" or \"none\")")
        if not self._lib.bsb_set_source_effect(self._h, int(source), kinds[background], int(bgblur)):
            self._fail("bsb_set_source_effect")

    def set_source_flip(self, source: int, flip_h=None, flip_v=None):
        """mirroring of one source's composite and video output (cv::flip, app/deepseg.cc:667-673; the mask is never
        flipped): flip_h / flip_v both None = follow set_output's flips, including later changes; otherwise the source's
        own setting (a None beside a bool counts as False)."""
        flip = -1 if flip_h is None and flip_v is None else (1 if flip_h else 0) | (2 if flip_v else 0)
        if not self._lib.bsb_set_source_flip(self._h, int(source), flip):
            self._fail("bsb_set_source_flip")

    def set_source_filter(self, source: int, active=None):
        """filter switch of one source: None = follow set_filter, including later changes; otherwise the source's own
        (False: its camera frame passes through; its mask and smoother are unaffected)."""
        v = -1 if active is None else int(bool(active))
        if not self._lib.bsb_set_source_filter(self._h, int(source), v):
            self._fail("bsb_set_source_filter")

    def set_source_mask_interval(self, source: int, k=None):
        """mask interval of one source: None = follow set_mask_interval, including later changes; otherwise 1..256"""
        if not self._lib.bsb_set_source_mask_interval(self._h, int(source), -1 if k is None else int(k)):
            self._fail("bsb_set_source_mask_interval")

    def set_source_mask_refine(self, source: int, sigma=None):
        """mask refinement strength of one source: None = follow set_mask_refine, including later changes; otherwise 0..255"""
        if not self._lib.bsb_set_source_mask_refine(self._h, int(source), -1 if sigma is None else int(sigma)):
            self._fail("bsb_set_source_mask_refine")

    def set_source_blur_mode(self, source: int, mode=None):
        """camera blur mode of one source: None = follow set_blur_mode, including later changes; otherwise "plain" or
        "masked"
        """
        v = -1 if mode is None else self._BLUR_MODE.get(mode, -2)
        if not self._lib.bsb_set_source_blur_mode(self._h, int(source), v):
            self._fail("bsb_set_source_blur_mode")

    def set_source_output(self, source: int, out_size=None):
        """virtual-camera size of one source (cv::resize after the flip, app/deepseg.cc:677-679): out_size = (w, h), or
        None to follow set_output's size, including later changes.  The mask stays W x H."""
        ow, oh = out_size if out_size else (0, 0)
        if not self._lib.bsb_set_source_output(self._h, int(source), int(ow), int(oh)):
            self._fail("bsb_set_source_output")
        if out_size:
            self._src_out[int(source)] = (int(ow), int(oh))
        else:
            self._src_out.pop(int(source), None)

    def source_output_size(self, source: int):
        """(w, h) of one source's composites: its own size, or the context's"""
        w, h = C.c_int(), C.c_int()
        if not self._lib.bsb_source_output_size(self._h, int(source), C.byref(w), C.byref(h)):
            self._fail("bsb_source_output_size")
        return w.value, h.value

    def _sources_out_px(self):
        """pixels of the largest effective output size among the sources (the context's when no source has its own)"""
        sizes = list(self._src_out.values())
        if len(sizes) < self._n_sources or not sizes:
            sizes.append((self.out_width, self.out_height))
        return max(w * h for w, h in sizes)

    def composite_sources(self, frames: np.ndarray, ids, want_out=True, want_yuyv=True, want_mask=True):
        """HOST buffers: frames [n, H, W, 3], frame b the next frame of source ids[b] (distinct ids) -> (out, yuyv, mask).
        out / yuyv are stacked arrays when every frame of the call has one output size, else lists of per-frame arrays."""
        frames = np.ascontiguousarray(frames, np.uint8)
        n, tab = self._ids(ids)
        if frames.shape != (n, self.height, self.width, 3):
            raise BackscrubError(f"frames shape {frames.shape} != {(n, self.height, self.width, 3)}")
        fb, npx = self.height * self.width * 3, self.height * self.width
        sizes = [self._src_out.get(int(s), (self.out_width, self.out_height)) for s in ids]
        opx = max(w * h for w, h in sizes) if sizes else self.out_width * self.out_height
        oc = self.out_channels
        out = np.empty(n * opx * oc, np.uint8) if want_out else None
        yuyv = np.empty(n * opx * 2, np.uint8) if want_yuyv else None
        mask = np.empty((n, self.height, self.width), np.uint8) if want_mask else None
        ok = self._lib.bsb_composite_sources(self._h, n, tab, _ptr(frames), self.width * 3, fb,
                                             _ptr(out) if want_out else None, opx * oc,
                                             _ptr(yuyv) if want_yuyv else None, opx * 2,
                                             _ptr(mask) if want_mask else None, npx)
        if not ok:
            self._fail("bsb_composite_sources")

        def shape(buf, ch):
            if buf is None:
                return None
            if len(set(sizes)) == 1:
                ow, oh = sizes[0]
                return buf.reshape(n, oh, ow, ch)
            return [buf[b * opx * ch: b * opx * ch + w * h * ch].reshape(h, w, ch) for b, (w, h) in enumerate(sizes)]
        return shape(out, oc), shape(yuyv, 2), mask

    def composite_sources_yuyv_device(self, n, ids, d_yuyv_in, d_out=0, d_yuyv=0, d_mask=0, sync=False, out_stride=None, yuyv_stride=None):
        """DEVICE-resident camera YUYV frames (tightly packed), frame b of source ids[b]; asynchronous unless `sync`.  Frame b's
        outputs are packed at its own size, out_stride / yuyv_stride bytes apart (default: the largest size of the sources)."""
        m, tab = self._ids(ids)
        if m != n:
            raise BackscrubError(f"{m} source ids for {n} frames")
        npx, opx = self.height * self.width, self._sources_out_px()
        ost = opx * self.out_channels if out_stride is None else int(out_stride)
        vst = opx * 2 if yuyv_stride is None else int(yuyv_stride)
        if not self._lib.bsb_composite_sources_yuyv_device(self._h, n, tab, d_yuyv_in, d_out or None, ost, d_yuyv or None, vst,
                                                           d_mask or None, npx, int(sync)):
            self._fail("bsb_composite_sources_yuyv_device")

    def composite_sources_nv12_device(self, n, ids, d_nv12, d_out=0, d_nv12_out=0, d_mask=0, sync=False, pitch=None, uv_offset=None,
                                      in_stride=None, out_stride=None, nv12_stride=None):
        """DEVICE-resident camera NV12 frames (layout as composite_nv12_device), frame b of source ids[b]; output strides as
        composite_sources_yuyv_device."""
        m, tab = self._ids(ids)
        if m != n:
            raise BackscrubError(f"{m} source ids for {n} frames")
        p, uv, st = self._nv12_layout(pitch, uv_offset, in_stride)
        npx, opx = self.height * self.width, self._sources_out_px()
        ost = opx * self.out_channels if out_stride is None else int(out_stride)
        vst = opx * 3 // 2 if nv12_stride is None else int(nv12_stride)
        if not self._lib.bsb_composite_sources_nv12_device(self._h, n, tab, d_nv12, p, uv, st, d_out or None, ost, d_nv12_out or None,
                                                           vst, d_mask or None, npx, int(sync)):
            self._fail("bsb_composite_sources_nv12_device")

    def synchronize(self):
        if not self._lib.bsb_synchronize(self._h):
            self._fail("bsb_synchronize")

    @property
    def stream(self) -> int:
        return self._lib.bsb_stream(self._h) or 0

    # -- introspection
    def infer(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, np.float32)
        n = 1 if x.ndim == 3 else x.shape[0]
        out = np.empty((n, *self.out_hwc), np.float32)
        if not self._lib.bsb_infer(self._h, n, _ptr(x), _ptr(out)):
            self._fail("bsb_infer")
        return out[0] if x.ndim == 3 else out

    def tensor(self, index: int, count: int, frame: int = 0):
        buf = np.empty(count, np.float32)
        n = self._lib.bsb_get_tensor_frame(self._h, index, frame, _ptr(buf), count)
        if n < 0:
            self._fail("bsb_get_tensor_frame")
        return buf[:n] if n else None

    def tc_steps(self) -> list:
        """the 1x1 convolutions planned for the tensor cores: dicts of op, in, out, residual (-1: none), K, N, act1..3"""
        n = self._lib.bsb_tc_steps(self._h, None, 0)
        rows = (C.c_int * max(1, 9 * n))()
        if n < 0 or self._lib.bsb_tc_steps(self._h, rows, n) != n:
            self._fail("bsb_tc_steps")
        keys = ("op", "in", "out", "residual", "K", "N", "act1", "act2", "act3")
        return [dict(zip(keys, rows[9 * i:9 * i + 9])) for i in range(n)]

    def stage_u8(self, which: int, frame: int = 0) -> np.ndarray:
        shape = self.in_hwc if which in (0, 1) else self.out_hwc[:2]
        buf = np.empty(int(np.prod(shape)), np.uint8)
        n = self._lib.bsb_get_stage_u8(self._h, which, frame, _ptr(buf), buf.size)
        if n < 0:
            self._fail("bsb_get_stage_u8")
        return buf.reshape(shape)

    def feed_shape(self, stage: int):
        """(h, w, c) of one frame of the tensor a feed of `stage` (_binding.FEED_LOGITS / FEED_MASK) replaces"""
        hwc = (C.c_int * 3)()
        if self._lib.bsb_test_feed_shape(self._h, int(stage), hwc) < 0:
            self._fail("bsb_test_feed_shape")
        return tuple(hwc)

    def feed(self, stage: int, array: np.ndarray):
        """Test entry point (bsb_test_feed): the next composite call takes `array` as the tensor of `stage` instead of
        computing it — FEED_LOGITS: float32 [n, h, w, c] logits the decision reads; FEED_MASK: uint8 [n, oh, ow] smoother
        output.  That call must have n frames."""
        dt = np.float32 if stage == B.FEED_LOGITS else np.uint8
        a = np.ascontiguousarray(array, dt)
        if not self._lib.bsb_test_feed(self._h, int(stage), int(a.shape[0]), _ptr(a), a.nbytes):
            self._fail("bsb_test_feed")

    def reset_state(self):
        if not self._lib.bsb_reset_state(self._h):
            self._fail("bsb_reset_state")

    def time_stage(self, stage: int, n_frames: int, iters: int) -> float:
        """ms per run of one stage (0 pre, 1 cnn, 2 decision, 3 post, 4 all) on device-resident buffers."""
        ms = self._lib.bsb_time_stage(self._h, stage, n_frames, iters)
        if ms < 0:
            self._fail("bsb_time_stage")
        return ms

    @property
    def uses_tensor_cores(self) -> bool:
        return bool(self._lib.bsb_uses_tensor_cores(self._h))

    @property
    def yuyv_native(self) -> bool:
        """the last call read the camera frames in their wire format (YUYV or NV12) in place (no BGR frame was materialised)"""
        return bool(self._lib.bsb_yuyv_native(self._h))

    @property
    def launches_per_call(self) -> int:
        return self._lib.bsb_launches_per_call(self._h, 1)

    @property
    def flops(self) -> float:
        return self._lib.bsb_model_flops(self._h)


def alpha_blend(lib, srca, srcb, mask, device=0):
    """app/deepseg.cc:108-134 (srca weight = mask, srcb weight = 255 - mask)."""
    srca, srcb, mask = (np.ascontiguousarray(a, np.uint8) for a in (srca, srcb, mask))
    out = np.empty_like(srca)
    if not lib.bsb_alpha_blend(device, _ptr(srca), _ptr(srcb), _ptr(mask), _ptr(out), mask.size):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def convert_rgb_to_yuyv(lib, rgb, device=0):
    """app/deepseg.cc:87-106."""
    rgb = np.ascontiguousarray(rgb, np.uint8)
    h, w, _ = rgb.shape
    out = np.empty((h, w, 2), np.uint8)
    if not lib.bsb_convert_rgb_to_yuyv(device, _ptr(rgb), _ptr(out), w, h):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def gaussian_blur(lib, src, ksize, device=0):
    """cv::GaussianBlur(src, Size(k,k), 0) 8UC3 (app/deepseg.cc:657-658)."""
    src = np.ascontiguousarray(src, np.uint8)
    out = np.empty_like(src)
    if not lib.bsb_gaussian_blur(device, _ptr(src), _ptr(out), src.shape[1], src.shape[0], int(ksize)):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def masked_gaussian_blur(lib, src, mask, ksize, device=0):
    """the masked camera blur of bsb_set_blur_mode: src 8UC3 blurred with every tap weighted by mask 8UC1
    (bsb_masked_gaussian_blur)"""
    src = np.ascontiguousarray(src, np.uint8)
    mask = np.ascontiguousarray(mask, np.uint8)
    if mask.shape != src.shape[:2]:
        raise ValueError("mask must be H x W of src")
    out = np.empty_like(src)
    if not lib.bsb_masked_gaussian_blur(device, _ptr(src), _ptr(mask), _ptr(out), src.shape[1], src.shape[0], int(ksize)):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def gaussian_taps(lib, ksize):
    q = (C.c_int * 255)()
    if not lib.bsb_gaussian_taps(int(ksize), q):
        raise BackscrubError(lib.bsb_last_error().decode())
    return np.array(q[:ksize], np.int64)


def mask_refine_weights(lib, sigma):
    """the range weights R_sigma[d], d = 0..255, of mask refinement strength sigma 1..255 (bsb_mask_refine_weights)"""
    w = (C.c_int * 256)()
    if not lib.bsb_mask_refine_weights(int(sigma), w):
        raise BackscrubError(lib.bsb_last_error().decode())
    return np.array(w[:], np.int64)


def flip(lib, src, flip_h, flip_v, device=0):
    """cv::flip (app/deepseg.cc:667-673)."""
    src = np.ascontiguousarray(src, np.uint8)
    out = np.empty_like(src)
    if not lib.bsb_flip(device, _ptr(src), _ptr(out), src.shape[1], src.shape[0], int(bool(flip_h)), int(bool(flip_v))):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def resize_u8c3(lib, src, dw, dh, device=0):
    """cv::resize(src, Size(dw, dh)) — what grab_background does (app/background.cc:178-194)."""
    src = np.ascontiguousarray(src, np.uint8)
    out = np.empty((dh, dw, 3), np.uint8)
    if not lib.bsb_resize_u8c3(device, _ptr(src), src.shape[1], src.shape[0], _ptr(out), dw, dh):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def pointwise(lib, A, W, bias=None, act=0, use_tc=False, device=0, variant=None, *, rows=None, a_off=0, ld_a=None,
              residual=None, res_off=0, ld_res=None, act2=0, act3=0, out=None, out_off=0, ld_out=None):
    """1x1 convolution stage: act3(act2(act(A [M, K] x W [N, K]^T + bias)) + residual) on the GPU.

    Plain call: A is [M, K] and a new [M, N] array is returned.  With `ld_a`, A is a flat buffer and the operand is its
    `rows` x K sub-matrix at element offset `a_off` with row pitch `ld_a`; the residual (flat, `res_off`, `ld_res`) and
    the output (`out`, flat, `out_off`, `ld_out`) are described the same way.  `out` is updated in place and returned:
    every element outside the written sub-matrix keeps its value."""
    W = np.ascontiguousarray(W, np.float32)
    N, K = W.shape
    b = np.ascontiguousarray(bias, np.float32) if bias is not None else None
    v = int(use_tc) if variant is None else int(variant)
    A = np.ascontiguousarray(A, np.float32)
    if ld_a is None:
        if rows is not None or a_off or A.ndim != 2 or A.shape[1] != K:
            raise ValueError("without ld_a, A is a plain [M, K] array: rows and a_off describe a flat buffer given with ld_a")
        rows = A.shape[0]
    elif rows is None or A.ndim != 1:
        raise ValueError("with ld_a, A is a flat buffer and rows (the M of the sub-matrix) is required")
    if out is None and (ld_out is not None or out_off):
        raise ValueError("ld_out and out_off describe a caller's out buffer")
    if residual is None and (ld_res is not None or res_off):
        raise ValueError("ld_res and res_off describe a residual buffer")
    if ld_a is None and residual is None and out is None and act2 == 0 and act3 == 0:
        M = A.shape[0]
        res = np.empty((M, N), np.float32)
        if not lib.bsb_pointwise(device, v, M, K, N, _ptr(A), _ptr(W), _ptr(b) if b is not None else None, act, _ptr(res)):
            raise BackscrubError(lib.bsb_last_error().decode())
        return res
    ld_a = K if ld_a is None else ld_a
    M = int(rows)
    a = np.ascontiguousarray(A, np.float32).reshape(-1)
    if out is None:
        out, ld_out = np.zeros(M * N, np.float32), N
    if out.dtype != np.float32 or not out.flags.c_contiguous:
        raise ValueError("out must be a contiguous float32 array")
    ld_out = N if ld_out is None else ld_out
    r = None
    if residual is not None:
        r = np.ascontiguousarray(residual, np.float32).reshape(-1)
        ld_res = N if ld_res is None else ld_res
    flat = out.reshape(-1)
    if not lib.bsb_pointwise_ex(device, v, M, K, N, _ptr(a), a.size, a_off, ld_a, _ptr(W), _ptr(b) if b is not None else None,
                                _ptr(r) if r is not None else None, r.size if r is not None else 0, res_off, ld_res or 0,
                                act, act2, act3, _ptr(flat), flat.size, out_off, ld_out):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def convert_yuyv_to_bgr(lib, yuyv, device=0):
    """cv::cvtColor(COLOR_YUV2BGR_YUYV) — the camera-frame ingest conversion."""
    yuyv = np.ascontiguousarray(yuyv, np.uint8)
    h, w, _ = yuyv.shape
    out = np.empty((h, w, 3), np.uint8)
    if not lib.bsb_convert_yuyv_to_bgr(device, _ptr(yuyv), _ptr(out), w, h):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out


def convert_nv12_to_bgr(lib, nv12, device=0):
    """cv::cvtColor(COLOR_YUV2BGR_NV12): tightly packed NV12 [H*3/2, W] -> BGR [H, W, 3]."""
    nv12 = np.ascontiguousarray(nv12, np.uint8)
    h, w = nv12.shape[0] * 2 // 3, nv12.shape[1]
    out = np.empty((h, w, 3), np.uint8)
    if not lib.bsb_convert_nv12_to_bgr(device, _ptr(nv12), _ptr(out), w, h):
        raise BackscrubError(lib.bsb_last_error().decode())
    return out
