"""backscrub_b200 — H100-native (sm_90a) implementation of backscrub's per-frame hot path.

The Python layer is a thin mirror of the reference's interface over the C ABI in
include/backscrub_b200.h.  All computation happens in `libbackscrub_b200.so` (hand-written
CUDA); importing the compute entry points without that library raises — there is no CPU
fallback.
"""
from __future__ import annotations

import os

from . import _binding, api
from .api import BackscrubError

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbackscrub_b200.so")
_LIB = None


def lib():
    """The product shared library (raises ImportError if it has not been built)."""
    global _LIB
    if _LIB is None:
        _LIB = _binding.bind(LIB_PATH)
    return _LIB


def bs_tensorflow_version() -> str:
    """lib/libbackscrub.h:13 — names the inference runtime."""
    return lib().bsb_version().decode()


def device_count() -> int:
    return lib().bsb_device_count()


def _require_gpu():
    if device_count() <= 0:
        raise BackscrubError("no CUDA device available: backscrub_b200 has no CPU path")


def bs_maskgen_new(modelname, threads, width, height, ondebug=None, onprep=None, oninfer=None, onmask=None, **gpu):
    """lib/libbackscrub.h:16-34.  Extra keyword arguments: device, max_batch, flags."""
    _require_gpu()
    return api.MaskGen(lib(), modelname, width, height, threads=threads, ondebug=ondebug, onprep=onprep,
                       oninfer=oninfer, onmask=onmask, **gpu)


def bs_maskgen_process(ctx, frame):
    """lib/libbackscrub.h:39 — returns the mask (the reference fills a cv::Mat&)."""
    return ctx.process(frame)


def bs_maskgen_delete(ctx):
    """lib/libbackscrub.h:37"""
    if ctx is not None:
        ctx.close()


def alpha_blend(srca, srcb, mask, device=0):
    _require_gpu()
    return api.alpha_blend(lib(), srca, srcb, mask, device)


def convert_rgb_to_yuyv(rgb, device=0):
    _require_gpu()
    return api.convert_rgb_to_yuyv(lib(), rgb, device)


def grab_background(raw, width, height, device=0):
    """app/background.cc:178-194: the per-frame cv::resize of the decoded background."""
    _require_gpu()
    return api.resize_u8c3(lib(), raw, width, height, device)


FLAG_KEEP_TENSORS = _binding.FLAG_KEEP_TENSORS
FLAG_NO_GRAPH = _binding.FLAG_NO_GRAPH
FLAG_TENSOR_CORES = _binding.FLAG_TENSOR_CORES
FLAG_EXACT = _binding.FLAG_EXACT


def set_tuning(name: str, value: int) -> None:
    """Process-wide launcher switch (include/backscrub_b200.h: bsb_set_tuning); selects between bit-identical kernels."""
    if not lib().bsb_set_tuning(name.encode(), int(value)):
        raise BackscrubError(lib().bsb_last_error().decode())


def masked_gaussian_blur(src, mask, ksize: int, device: int = 0):
    """The masked camera blur of bsb_set_blur_mode (include/backscrub_b200.h: bsb_masked_gaussian_blur): src 8UC3 blurred
    with every tap weighted by mask 8UC1 and normalised by the blurred mask."""
    return api.masked_gaussian_blur(lib(), src, mask, ksize, device)


def mask_refine_weights(sigma: int):
    """The range weights R_sigma[d], d = 0..255, of mask refinement strength sigma 1..255 (include/backscrub_b200.h:
    bsb_mask_refine_weights), as an int64 array."""
    return api.mask_refine_weights(lib(), sigma)
