"""ctypes binding of the C ABI in include/backscrub_b200.h.

The product package binds `backscrub_b200/libbackscrub_b200.so` (nvcc, sm_90a) and
nothing else: there is no CPU fallback, and a missing / unloadable library raises.
"""
from __future__ import annotations

import ctypes as C
import os

u8p = C.POINTER(C.c_uint8)
f32p = C.POINTER(C.c_float)
i32p = C.POINTER(C.c_int)
DEBUG_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_char_p)
STAGE_CB = C.CFUNCTYPE(None, C.c_void_p)
BG_READ_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_void_p), i32p, i32p, C.POINTER(C.c_size_t))
BG_REWIND_CB = C.CFUNCTYPE(C.c_int, C.c_void_p)

FEED_LOGITS, FEED_MASK = 1, 2
FLAG_KEEP_TENSORS, FLAG_NO_GRAPH, FLAG_TENSOR_CORES, FLAG_FUSE_BLOCKS, FLAG_EXACT = 1, 2, 4, 8, 16

# every symbol include/backscrub_b200.h declares (tests check the .so exports all of them)
SYMBOLS = [
    "bsb_version", "bsb_last_error", "bsb_device_count", "bsb_maskgen_new", "bsb_maskgen_new_ex",
    "bsb_maskgen_delete", "bsb_maskgen_process", "bsb_set_background", "bsb_get_background",
    "bsb_set_background_ring", "bsb_set_background_cursor", "bsb_set_bgblur", "bsb_set_output", "bsb_output_size",
    "bsb_gaussian_blur", "bsb_gaussian_taps", "bsb_flip",
    "bsb_composite", "bsb_composite_device", "bsb_composite_yuyv", "bsb_composite_yuyv_device", "bsb_composite_mjpg", "bsb_decode_mjpg", "bsb_convert_yuyv_to_bgr", "bsb_synchronize", "bsb_stream", "bsb_alpha_blend",
    "bsb_convert_rgb_to_yuyv", "bsb_resize_u8c3", "bsb_pointwise", "bsb_pointwise_ex", "bsb_time_pointwise", "bsb_geometry", "bsb_infer", "bsb_get_tensor", "bsb_get_tensor_frame", "bsb_tc_steps",
    "bsb_get_stage_u8", "bsb_reset_state", "bsb_time_stage", "bsb_launches_per_call", "bsb_total_launches", "bsb_model_flops", "bsb_set_tuning", "bsb_frame_size", "bsb_yuyv_native", "bsb_uses_tensor_cores",
    "bsb_calcmask_new", "bsb_calcmask_delete", "bsb_calcmask_set_input_frame", "bsb_calcmask_get_output_mask", "bsb_calcmask_timings",
    "bsb_calcmask_frames_done", "bsb_calcmask_mask_serial",
    "bsb_background_new_still", "bsb_background_new_video", "bsb_background_delete", "bsb_background_grab", "bsb_background_grab_into",
    "bsb_background_thumbnail", "bsb_background_frame", "bsb_background_running",
    "bsb_set_sources", "bsb_reset_source", "bsb_set_source_background", "bsb_composite_sources", "bsb_composite_sources_yuyv_device",
    "bsb_composite_nv12", "bsb_composite_nv12_device", "bsb_composite_sources_nv12_device", "bsb_convert_nv12_to_bgr",
    "bsb_set_source_effect", "bsb_set_source_flip", "bsb_set_source_output", "bsb_source_output_size",
    "bsb_set_source_background_ring", "bsb_set_source_background_cursor",
    "bsb_set_filter", "bsb_set_source_filter", "bsb_set_out_format",
    "bsb_set_live_background", "bsb_set_source_live_background",
    "bsb_set_mask_interval", "bsb_set_source_mask_interval",
    "bsb_set_framing", "bsb_set_framing_auto", "bsb_set_source_framing", "bsb_get_framing",
    "bsb_test_feed_shape", "bsb_test_feed",
]


def bind(path: str) -> C.CDLL:
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  backscrub_b200 has no CPU fallback.")
    L = C.CDLL(path)
    L.bsb_version.restype = C.c_char_p
    L.bsb_last_error.restype = C.c_char_p
    L.bsb_device_count.restype = C.c_int
    L.bsb_maskgen_new.restype = C.c_void_p
    L.bsb_maskgen_new.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t, C.c_size_t, DEBUG_CB, STAGE_CB, STAGE_CB, STAGE_CB, C.c_void_p]
    L.bsb_maskgen_new_ex.restype = C.c_void_p
    L.bsb_maskgen_new_ex.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_uint, DEBUG_CB, STAGE_CB, STAGE_CB, STAGE_CB, C.c_void_p]
    L.bsb_maskgen_delete.argtypes = [C.c_void_p]
    L.bsb_maskgen_delete.restype = None
    L.bsb_maskgen_process.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(u8p), C.POINTER(C.c_size_t)]
    L.bsb_set_background.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_size_t]
    L.bsb_get_background.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.bsb_set_background_ring.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_int]
    L.bsb_set_background_cursor.argtypes = [C.c_void_p, C.c_int]
    L.bsb_set_bgblur.argtypes = [C.c_void_p, C.c_int]
    L.bsb_set_output.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.bsb_output_size.argtypes = [C.c_void_p, i32p, i32p]
    L.bsb_gaussian_blur.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.bsb_gaussian_taps.argtypes = [C.c_int, i32p]
    L.bsb_flip.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.bsb_composite.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t,
                                C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.bsb_composite_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                       C.c_void_p, C.c_size_t, C.c_int]
    L.bsb_composite_yuyv.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.bsb_composite_yuyv_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    L.bsb_composite_mjpg.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                     C.c_void_p, C.c_size_t]
    L.bsb_decode_mjpg.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.bsb_convert_yuyv_to_bgr.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.bsb_synchronize.argtypes = [C.c_void_p]
    L.bsb_stream.restype = C.c_void_p
    L.bsb_stream.argtypes = [C.c_void_p]
    L.bsb_alpha_blend.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.bsb_convert_rgb_to_yuyv.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.bsb_resize_u8c3.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.bsb_pointwise.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.bsb_pointwise_ex.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long, C.c_long, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_long, C.c_int,
                                   C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long, C.c_long, C.c_int]
    L.bsb_time_pointwise.restype = C.c_double
    L.bsb_time_pointwise.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L.bsb_geometry.argtypes = [C.c_void_p, i32p, i32p, i32p, i32p, i32p]
    L.bsb_infer.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.bsb_get_tensor.restype = C.c_long
    L.bsb_get_tensor.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_long]
    L.bsb_get_tensor_frame.restype = C.c_long
    L.bsb_get_tensor_frame.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_long]
    L.bsb_tc_steps.argtypes = [C.c_void_p, i32p, C.c_int]
    L.bsb_get_stage_u8.restype = C.c_long
    L.bsb_get_stage_u8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_long]
    L.bsb_reset_state.argtypes = [C.c_void_p]
    L.bsb_launches_per_call.argtypes = [C.c_void_p, C.c_int]
    L.bsb_total_launches.restype = C.c_long
    L.bsb_time_stage.restype = C.c_double
    L.bsb_time_stage.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.bsb_model_flops.restype = C.c_double
    L.bsb_model_flops.argtypes = [C.c_void_p]
    L.bsb_set_tuning.argtypes = [C.c_char_p, C.c_int]
    L.bsb_frame_size.argtypes = [C.c_void_p, i32p, i32p]
    L.bsb_yuyv_native.argtypes = [C.c_void_p]
    L.bsb_uses_tensor_cores.argtypes = [C.c_void_p]
    L.bsb_calcmask_new.restype = C.c_void_p
    L.bsb_calcmask_new.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    L.bsb_calcmask_delete.restype = None
    L.bsb_calcmask_delete.argtypes = [C.c_void_p]
    L.bsb_calcmask_set_input_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.bsb_calcmask_get_output_mask.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.bsb_calcmask_timings.argtypes = [C.c_void_p, C.POINTER(C.c_long)]
    L.bsb_calcmask_frames_done.restype = C.c_long
    L.bsb_calcmask_frames_done.argtypes = [C.c_void_p]
    L.bsb_calcmask_mask_serial.restype = C.c_long
    L.bsb_calcmask_mask_serial.argtypes = [C.c_void_p]
    L.bsb_background_new_still.restype = C.c_void_p
    L.bsb_background_new_still.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.c_int]
    L.bsb_background_new_video.restype = C.c_void_p
    L.bsb_background_new_video.argtypes = [C.c_int, C.c_double, C.c_int, BG_READ_CB, BG_REWIND_CB, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_size_t, C.c_int]
    L.bsb_background_delete.restype = None
    L.bsb_background_delete.argtypes = [C.c_void_p]
    L.bsb_background_grab.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    L.bsb_background_grab_into.argtypes = [C.c_void_p, C.c_void_p]
    L.bsb_background_thumbnail.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, i32p, i32p]
    L.bsb_background_frame.argtypes = [C.c_void_p]
    L.bsb_background_running.argtypes = [C.c_void_p]
    L.bsb_set_sources.argtypes = [C.c_void_p, C.c_int]
    L.bsb_reset_source.argtypes = [C.c_void_p, C.c_int]
    L.bsb_set_source_background.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_size_t]
    L.bsb_set_source_background_ring.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_int]
    L.bsb_set_source_background_cursor.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.bsb_set_source_effect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.bsb_set_source_flip.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.bsb_set_filter.argtypes = [C.c_void_p, C.c_int]
    L.bsb_set_out_format.argtypes = [C.c_void_p, C.c_int]
    L.bsb_set_live_background.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t]
    L.bsb_set_source_live_background.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t]
    L.bsb_set_source_filter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.bsb_set_mask_interval.argtypes = [C.c_void_p, C.c_int]
    L.bsb_set_source_mask_interval.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.bsb_set_framing.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L.bsb_set_framing_auto.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.bsb_set_source_framing.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L.bsb_get_framing.argtypes = [C.c_void_p, C.c_int, i32p]
    L.bsb_set_source_output.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.bsb_source_output_size.argtypes = [C.c_void_p, C.c_int, i32p, i32p]
    L.bsb_composite_sources.argtypes = [C.c_void_p, C.c_int, i32p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t,
                                        C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.bsb_composite_sources_yuyv_device.argtypes = [C.c_void_p, C.c_int, i32p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                    C.c_void_p, C.c_size_t, C.c_int]
    L.bsb_composite_nv12.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                     C.c_void_p, C.c_size_t]
    L.bsb_composite_nv12_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    L.bsb_composite_sources_nv12_device.argtypes = [C.c_void_p, C.c_int, i32p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p,
                                                    C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    L.bsb_test_feed_shape.restype = C.c_long
    L.bsb_test_feed_shape.argtypes = [C.c_void_p, C.c_int, i32p]
    L.bsb_test_feed.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    L.bsb_convert_nv12_to_bgr.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    return L
