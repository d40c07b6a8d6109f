/* include/backscrub_b200.h — C ABI of the H100-native (sm_90a) backscrub hot path.
 *
 * This is the drop-in boundary for the reference's per-frame path.  The reference exposes
 * a C++ API (std::string, cv::Mat&) — lib/libbackscrub.h:13-39 — plus two free functions
 * compiled into the app (app/deepseg.cc:87-134) and the background provider
 * (app/background.h:14-23).  Everything below is plain C (pointers + sizes, no C++ or
 * torch types); include/libbackscrub.h and include/background.h are the header-only
 * cv::Mat shims that map the reference's signatures onto it, and INTEGRATION.md shows
 * the binding a maintainer adds.
 *
 * Conventions (same as the reference, SURVEY.md §8b):
 *   - frames are 8-bit 3-channel, in the channel order the camera delivers (BGR in
 *     backscrub), row pitch given in bytes; W x H fixed at bsb_maskgen_new;
 *   - masks are 8-bit 1-channel W x H, 255 = background, 0 = person;
 *   - errors: NULL / negative return + message via the ondebug callback (or stderr) and
 *     bsb_last_error(); no exceptions cross the boundary;
 *   - one context is used by one thread at a time; contexts are independent (one per
 *     stream / GPU) and may be used from several threads at once.  What they share:
 *       - the bsb_set_tuning switches: process-wide, set before contexts are created,
 *         and never changed while any call is in flight;
 *       - per-device caches built on first use under mutexes: the kernels' shared-memory
 *         attributes, the encoder carveouts, the Gaussian tap tables;
 *       - the process-wide launch total, bsb_total_launches (bsb_launches_per_call counts
 *         the launches of the calling thread only);
 *     the error string is per thread.  tests/test_concurrent_contexts.py runs contexts,
 *     the bsb_calcmask_* worker and refused calls from several threads at once, in a
 *     process whose first context builds the caches, and checks every output,
 *     launches_per_call and each thread's error string against the same calls made one
 *     thread at a time.  It keeps the switches at their defaults throughout.
 *   - There is NO CPU fallback: every entry point that computes requires a CUDA device
 *     and fails loudly without one.
 */
#ifndef BACKSCRUB_B200_H
#define BACKSCRUB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BSB_API __attribute__((visibility("default")))

typedef struct bsb_ctx bsb_ctx;

/* Optional callbacks, as in lib/libbackscrub.h:21-33.  onprep / oninfer / onmask fire in
 * this order, once per bsb_maskgen_process() call, on the calling thread, after the GPU
 * work of that stage has been *enqueued and completed* (the call synchronises the stage
 * boundary only when the callback is non-NULL). */
typedef void (*bsb_debug_cb)(void* caller_ctx, const char* msg);
typedef void (*bsb_stage_cb)(void* caller_ctx);

/* flags for bsb_maskgen_new_ex */
enum {
  BSB_FLAG_KEEP_TENSORS = 1,  /* keep every intermediate activation (tests / debugging) */
  BSB_FLAG_NO_GRAPH = 2,      /* launch kernels eagerly instead of one CUDA graph per batch */
  BSB_FLAG_TENSOR_CORES = 4,  /* wgmma 3xTF32 1x1 convs for ANY model (default only for the GEMM-dominated DeepLab / BodyPix graphs) */
  BSB_FLAG_FUSE_BLOCKS = 8,   /* round-1 experiment: one-kernel inverted-residual blocks (bit-exact; superseded by the chain kernel) */
  BSB_FLAG_EXACT = 16         /* fp32 FFMA 1x1 convs everywhere: every activation bit-identical to the CPU oracle (no tensor cores) */
};

/* replaces bs_tensorflow_version() (lib/libbackscrub.h:13, lib/libbackscrub.cc:150):
 * a static string naming the inference runtime. */
BSB_API const char* bsb_version(void);

/* Thread-local text of the last error raised by any entry point ("" if none). */
BSB_API const char* bsb_last_error(void);

/* Number of CUDA devices visible (0 => nothing below can run). */
BSB_API int bsb_device_count(void);

/* replaces bs_maskgen_new (lib/libbackscrub.h:16-34, lib/libbackscrub.cc:161-259).
 * Model family is chosen by file-name substring (body-pix / deeplab / segm_ / selfie),
 * lib/libbackscrub.cc:116-130.  `threads` is accepted and ignored (advisory in the
 * reference too).  Returns NULL after reporting through ondebug. */
BSB_API bsb_ctx* bsb_maskgen_new(const char* modelname, size_t threads, size_t width, size_t height,
                                 bsb_debug_cb ondebug, bsb_stage_cb onprep, bsb_stage_cb oninfer,
                                 bsb_stage_cb onmask, void* caller_ctx);

/* Same, with the GPU-side knobs: CUDA device ordinal, maximum frames per launch
 * (consecutive frames of ONE stream, the IIR advancing in order — or, through the sources
 * calls below, one frame each of up to max_batch independent cameras), flags above. */
BSB_API bsb_ctx* bsb_maskgen_new_ex(const char* modelname, size_t width, size_t height, int device,
                                    int max_batch, unsigned flags, bsb_debug_cb ondebug, bsb_stage_cb onprep,
                                    bsb_stage_cb oninfer, bsb_stage_cb onmask, void* caller_ctx);

/* replaces bs_maskgen_delete (lib/libbackscrub.h:37, lib/libbackscrub.cc:261-277); NULL-safe. */
BSB_API void bsb_maskgen_delete(bsb_ctx* ctx);

/* replaces bs_maskgen_process (lib/libbackscrub.h:39, lib/libbackscrub.cc:279-376).
 * frame: host pointer, W x H x 3, `frame_pitch` bytes per row (never written).
 * *mask / *mask_pitch receive a pointer to context-owned HOST storage holding the W x H
 * mask — valid until the next process call on this context (the reference returns a
 * cv::Mat header aliasing ctx.mask the same way, lib/libbackscrub.cc:374).
 * Returns 1 on success, 0 on error (the reference returns bool). */
BSB_API int bsb_maskgen_process(bsb_ctx* ctx, const uint8_t* frame, size_t frame_pitch,
                                const uint8_t** mask, size_t* mask_pitch);

/* ---- background provider (app/background.h:14-23, app/background.cc:178-194) ----
 * Decoding stays on the host (cv::VideoCapture / imread in the shim); the library takes
 * the decoded raw frame and performs grab_background's cv::resize(raw -> W x H) on the
 * GPU.  Call again whenever the decoded frame changes (video backgrounds). */
BSB_API int bsb_set_background(bsb_ctx* ctx, const uint8_t* bg_raw, int bg_w, int bg_h, size_t bg_pitch);
/* the resized background (what grab_background hands back), copied to host.  Until a background is set it is
 * plain green, like `bg` in app/deepseg.cc:603. */
BSB_API int bsb_get_background(bsb_ctx* ctx, uint8_t* out, size_t out_pitch);
/* Animated background (the video branch of app/background.cc:126-176 decodes; :178-194 resizes): `count` decoded
 * images, `frame_stride` bytes apart, are resized into a device-resident ring.  Batch frame b of a composite call
 * blends ring image (cursor + b*advance) % count, and the cursor then moves on by n_frames*advance.  advance 0
 * leaves pacing to the caller (bsb_set_background_cursor), as the reference paces by wall clock. */
BSB_API int bsb_set_background_ring(bsb_ctx* ctx, const uint8_t* frames, int count, int bg_w, int bg_h, size_t bg_pitch,
                                    size_t frame_stride, int advance);
BSB_API int bsb_set_background_cursor(bsb_ctx* ctx, int index);

/* ---- per-frame options of the reference's main loop around alpha_blend (app/deepseg.cc:649-679) ----
 * `-p bgblur:k` (:415-434, :657-658): cv::GaussianBlur(bg, bg, Size(k,k), 0) on the background — the grabbed
 * one, or, when no background was set, a copy of the camera frame (:652-654).  k odd in 1..255 ("strength value
 * must be odd"), 0 = off.  OpenCV's bit-exact 8-bit path. */
BSB_API int bsb_set_bgblur(bsb_ctx* ctx, int ksize);
/* `-H`/`-V` cv::flip of the composited frame (:667-673) and cv::resize to the virtual-camera geometry when it
 * differs from the capture geometry (:677-679); both before the YUYV conversion.  out_w/out_h <= 0 = frame size.
 * After this call `out` buffers are out_w x out_h x 3 (x 4 in the BGRA output format, bsb_set_out_format) and `out_yuyv`
 * out_w x out_h x 2; the mask stays W x H.
 * The flips and the size are the default of every source of a sources call (bsb_set_source_flip, bsb_set_source_output). */
BSB_API int bsb_set_output(bsb_ctx* ctx, int flip_h, int flip_v, int out_w, int out_h);
BSB_API int bsb_output_size(bsb_ctx* ctx, int* out_w, int* out_h);
/* The filter switch (app/deepseg.cc:624,639-664,782-784: the `s` key).  active: 1 = composite (the default), 0 = pass the
 * camera frame through: the composite is the camera frame (as BGR; YUYV / NV12 frames converted as the fused path converts
 * them), then the flip, the resize and the YUYV / NV12 conversion of bsb_set_output.  The mask is still computed and
 * written, byte for byte as with the filter on, and the smoother still advances (:634 feeds every frame), so switching
 * back on continues a stream that never stopped.  No background is read or blurred for such a frame; a background ring's
 * cursor still moves.  Every composite entry point honours it (plain calls, and sources calls through the sources that
 * follow the context, bsb_set_source_filter); bsb_maskgen_process and the bsb_calcmask_* front end produce masks only.
 * Host state only: the switch is part of the captured call, so once both states of a call have run, toggling replays.
 * active outside 0..1 returns 0 with a bsb_last_error() message and leaves the context as it was. */
BSB_API int bsb_set_filter(bsb_ctx* ctx, int active);
/* Output format of the `out` buffers of every composite entry point (bsb_composite, _device, _yuyv, _yuyv_device, _mjpg,
 * _nv12, _nv12_device and the three bsb_composite_sources*).  BSB_OUT_BGR (the default): the BGR composite.  BSB_OUT_BGRA:
 * the person on a transparent background, straight (not premultiplied) alpha, for compositors that take BGRA.  Frame b,
 * with C its camera frame as the fused path reads it (BGR as given, YUYV / NV12 converted exactly as for the composite) and
 * M the W x H mask the same call writes (255 = background, outside the ROI included):
 *   A0[y][x] = (C.B, C.G, C.R, 255 - M[y][x])   (its filter off, bsb_set_filter / bsb_set_source_filter: alpha 255)
 *   out_b    = cv::resize(cv::flip(A0), INTER_LINEAR) with the flip and output size the frame's composite gets (the
 *              context's, or its source's own), in the reference's order; OpenCV resizes 8UC4 channel by channel with
 *              the tables of the 3-channel composite, so the colour bytes are those of a filter-off composite.
 * Rows are out_w*4 bytes: packed on the device entry points and in the sources strides (a frame of its own size must fit
 * its out stride at 4 bytes per pixel), out_pitch >= out_w*4 for bsb_composite.  The video output (YUYV / NV12) and the
 * mask are byte for byte those of a BGR-format call; the smoother, rings and cursors behave as in one.  A call without a
 * video output blends nothing: it reads and blurs no background (camera blur included) while ring cursors still move.
 * Host state only, like bsb_set_filter: once both formats of a call have run, toggling replays; the host-buffer staging
 * grows to 4 bytes per pixel on the first BGRA call that needs it.  A format outside 0..1 returns 0 with a
 * bsb_last_error() message and changes nothing. */
enum { BSB_OUT_BGR = 0, BSB_OUT_BGRA = 1 };
BSB_API int bsb_set_out_format(bsb_ctx* ctx, int format);
/* Mask interval.  The reference composites every camera frame with whatever mask its AI thread made last
 * (app/deepseg.cc:627-661, `ai.get_output_mask(mask)`), so a 60 fps camera is routinely composited with masks made at a
 * lower rate.  These setters make that trade explicit: fewer frames pay for pre-processing and the CNN, and no output
 * frame is dropped.
 *   Segmented frame: pre-processing, the CNN, the decision and one smoother step, exactly as at interval 1.
 *   Held frame: none of those.  Its small mask (ofinal) is the smoother state its camera holds now, i.e. the state after
 *     the camera's latest segmented frame; upsampling, blur, blend, flip, resize, BGRA, YUYV / NV12 and the mask output
 *     then proceed as usual.  So without mask refinement (strength 0, bsb_set_mask_refine) its W x H mask is byte for byte
 *     that of the latest segmented frame, and its composite is that mask applied to the new camera frame; a refined held
 *     frame refines the held small mask against its own camera frame.
 *   Plain calls: the context counts the frames of its plain calls from 0 (at creation and after bsb_reset_state); frame c
 *     is segmented iff c % k == 0.  The cadence runs across calls and across the chunks of a split host-buffer call; held
 *     frames before a call's first segmented frame hold the state the previous call left.
 *   Sources calls: source s counts the frames it delivers from 0 (at bsb_set_sources and bsb_reset_source(s)); its frame f
 *     is segmented iff f == 0 || (f + s) % k_s == 0, k_s its effective interval.  The id as the phase staggers sources with
 *     consecutive ids (64 sources at k = 2 segment 32 frames per call), and a new or reset camera never composites with an
 *     empty mask.
 *   A new interval applies from the next frame; no counter is reset.  Frames with their filter off follow the cadence
 *   like any other (segmentation still runs).  Backgrounds, flips, sizes and formats are per call frame as before, and
 *   ring cursors move as before.  Fed calls (bsb_test_feed) ignore the interval and leave the counters unchanged.  A call
 *   with stage callbacks fires each once, also when no frame of it is segmented.  The library's own mask-only users
 *   (bs_maskgen_process, the bsb_calcmask_* front end) never set an interval and so segment every frame.
 *   Introspection: bsb_get_tensor_frame and stages 0 / 1 of bsb_get_stage_u8 index the call's i-th segmented frame;
 *   stage 2 (ofinal) and the mask index the call frame.
 *   Host state only: which frames are segmented reaches the device as table data with the call, so a periodic cadence
 *   replays at most k captured graphs per buffer set (one per CNN batch size it produces).
 * interval: 1..256, default 1 (every frame).  Out of range returns 0 with a bsb_last_error() message and changes nothing. */
BSB_API int bsb_set_mask_interval(bsb_ctx* ctx, int interval);
/* One source's interval: -1 follows bsb_set_mask_interval (including later changes), else 1..256.  bsb_set_sources resets
 * every source to -1; bsb_reset_source keeps it.  No bsb_set_sources yet, a source id out of range or an interval out of
 * range returns 0 with a bsb_last_error() message and changes nothing. */
BSB_API int bsb_set_source_mask_interval(bsb_ctx* ctx, int source, int interval);
/* Framing: each frame's output shows a crop of its camera frame, a fixed rectangle (a digital pan / zoom onto a
 * whiteboard, one seat of a room camera) or one that keeps the person the mask finds centred and sized (auto-framing).
 * C is the frame's W x H composite (BGR; the BGRA frame in the BGRA output format; the camera frame when its filter is off)
 * and crop_b = (x, y, w, h) lies in the unflipped camera frame.  Frame b's output is
 *   out_b = cv::resize(cv::flip(C[crop_b]), (ow_b, oh_b), INTER_LINEAR)
 * with the frame's own flip and output size (bsb_set_output, or the source's); the YUYV / NV12 output is derived from
 * out_b as always, and the mask stays W x H, unflipped and uncropped.  A crop of the output size is a copy and an exact 2x
 * crop the INTER_AREA mean, as OpenCV does; the crop (0, 0, W, H) gives the bytes of an unframed call.
 *   BSB_FRAMING_OFF: the whole frame (the default).
 *   BSB_FRAMING_RECT: crop_b = (x, y, w, h), inside the frame with w, h >= 1 (else refused); the aspect is not forced.
 *     Host bookkeeping only: a new rectangle every call replays the captured call.
 *   BSB_FRAMING_AUTO: crop_b follows one state per camera (the plain stream, each source), stepped once per call frame,
 *     in frame order, on that frame's small mask (bsb_get_stage_u8 stage 2): the box of its person pixels (ofinal < 128
 *     inside the output ROI; fewer than max(1, w*h/1000) of them: the whole frame) mapped to the frame through the ROI,
 *     widened to the frame's output aspect with margin_pct of the box height as headroom and on each side, at most
 *     max_zoom_pct zoom, shifted into the frame, then smoothed by `speed` (bsb_set_framing_auto).  A camera without a state
 *     (its first AUTO frame, after bsb_reset_state / bsb_reset_source / bsb_set_sources, or after a frame not in AUTO)
 *     jumps to its target.  DESIGN.md §4 states the formula.
 * Interactions: held frames (bsb_set_mask_interval) step the state on the small mask they are composited with; frames
 * with the filter off are framed like any other; fed calls (bsb_test_feed, both stages) step the state; ring cursors,
 * live backgrounds and callbacks are unchanged; a split host-buffer call carries the state across its chunks in stream
 * order; bs_maskgen_process and the bsb_calcmask_* front end never frame.  A call without a framed frame runs exactly the
 * kernels it ran before framing existed.
 * mode: BSB_FRAMING_*; x, y, w, h are read for BSB_FRAMING_RECT only.  An unknown mode or a rectangle outside the frame
 * returns 0 with a bsb_last_error() message and changes nothing. */
enum { BSB_FRAMING_OFF = 0, BSB_FRAMING_RECT = 1, BSB_FRAMING_AUTO = 2 };
BSB_API int bsb_set_framing(bsb_ctx* ctx, int mode, int x, int y, int w, int h);
/* Auto-framing parameters of the context (every camera): max_zoom_pct 100..1000 (the crop is at least H*100/max_zoom_pct
 * rows high; default 300), margin_pct 0..100 (default 10), speed 1..256 (the share of the remaining distance, in 1/256,
 * the crop moves per frame; 256 jumps; default 32).  Out of range returns 0 with a bsb_last_error() message and changes
 * nothing.  Captured calls are dropped (the parameters are kernel arguments). */
BSB_API int bsb_set_framing_auto(bsb_ctx* ctx, int max_zoom_pct, int margin_pct, int speed);
/* One source's framing: mode -1 follows bsb_set_framing (its rectangle included, and later changes), else the source's
 * own mode and rectangle.  bsb_set_sources resets every source to -1; bsb_reset_source keeps it.  Host bookkeeping only:
 * it reaches the device in the call's framing table.  No bsb_set_sources yet, a source id out of range, an unknown mode
 * or a rectangle outside the frame returns 0 with a bsb_last_error() message and changes nothing. */
BSB_API int bsb_set_source_framing(bsb_ctx* ctx, int source, int mode, int x, int y, int w, int h);
/* The crop (x, y, w, h) frame `frame` of the last call used (frames of a split host-buffer call by their index in the
 * caller's call); (0, 0, W, H) when that call was not framed.  Synchronises the context's stream.  A frame outside the
 * last call returns 0 with a bsb_last_error() message. */
BSB_API int bsb_get_framing(bsb_ctx* ctx, int frame, int rect[4]);
/* Mask edge refinement: the full-size mask of a refined frame follows the edges of its own camera frame instead of the
 * blocky, ~10-pixel-wide edge of blur(resize(small mask)) (lib/libbackscrub.cc:366-371): a joint bilateral upsample of the
 * small mask guided by the camera luma (Kopf et al., SIGGRAPH 2007), which keeps hair and shoulders and stops the
 * background bleeding around them.  It matters most where the matte is magnified or shown: BGRA output, auto-framing,
 * held frames.  Strength sigma 0..255; 0 is off, the bytes of the unrefined mask.
 * For a frame with sigma > 0, every pixel p = (x, y) inside roidim gets M'(p) below (outside it the mask stays 255).  s is
 * the sw x sh out_roidim region of the small mask (ofinal, bsb_get_stage_u8 stage 2), L the camera luma as the composite
 * reads the frame (BGR as given, YUYV / NV12 after the fused path's conversion): L = (4899 R + 9617 G + 1868 B + 8192) >> 14.
 *   taps: fx = (float)((x - roi_x + 0.5) * scale - 0.5) (cv::resize's source position, scale = sw / roi_w as OpenCV
 *     computes it, unclamped), s = floor(fx), a = lrintf((fx - s) * 2048); columns s-1 .. s+2 with spatial weights
 *     max(0, 1024 - a), 3072 - a, 1024 + a, max(0, a - 1024) (a tent of radius 1.5 small pixels); rows alike.  A tap
 *     outside 0..sw-1 / 0..sh-1 has weight 0.
 *   guide(i, j) = L at (roi_x + ((2j + 1) roi_w) / (2 sw), roi_y + ((2i + 1) roi_h) / (2 sh)) (integer division): the
 *     frame pixel nearest the centre of small pixel (i, j).
 *   R[d] = max(1, floor(256 exp(-d^2 / (2 sigma^2)) + 0.5)), d = |L(p) - guide(i, j)| (bsb_mask_refine_weights).
 *   w = ((wx * wy) >> 12) * R[d] per tap;  M'(p) = (sum w * s[i][j] + (sum w >> 1)) / sum w  (uint32; sum w >= 1024).
 * A small mask that is uniform over a pixel's taps gives exactly that value.  Guidance: sigma ~ 8..16 (about the camera's
 * noise plus a margin) separates person from background where their luma differs; sigma near 255 weighs every tap alike
 * and degrades toward a plain tent upsample of the hard small mask, which is blockier than the default blur; where
 * person and background have the same luma the refinement cannot find the edge.
 * The refined mask is the mask: the stored W x H mask, the blend weight, BGRA alpha (255 - M').  Flip, resize, framing's
 * crop and YUYV / NV12 follow from the composite as before; the mask is never flipped.  A frame with its filter off still
 * stores its refined mask.  Held frames refine the held small mask against their own camera frame.  Unchanged: AUTO
 * framing (it reads the small mask), bsb_get_stage_u8, rings, live backgrounds and the smoothers; fed calls
 * (bsb_test_feed) refine like any call; bs_maskgen_process and the bsb_calcmask_* front end never refine.
 * Host state only: each frame's strength reaches the device in a table with the call, so changing sigma replays the
 * captured call (a call with some refined frame replays one of at most two graphs per buffer set).  A call with no refined
 * frame runs exactly the kernels it ran before refinement existed.  A refined call needs the TMA or fast post kernel (frame
 * width a multiple of 16, a small mask that is up-scaled to the ROI); otherwise the call returns 0 with a bsb_last_error()
 * message.
 * sigma: 0..255, default 0.  Out of range returns 0 with a bsb_last_error() message and changes nothing. */
BSB_API int bsb_set_mask_refine(bsb_ctx* ctx, int sigma);
/* One source's strength: -1 follows bsb_set_mask_refine (including later changes), else 0..255.  bsb_set_sources resets
 * every source to -1; bsb_reset_source keeps it.  No bsb_set_sources yet, a source id out of range or a strength out of
 * range returns 0 with a bsb_last_error() message and changes nothing. */
BSB_API int bsb_set_source_mask_refine(bsb_ctx* ctx, int source, int sigma);
/* The range weights R_sigma[d], d = 0..255, of strength sigma 1..255 into w[256] (host only).  Out of range or a null w
 * returns 0 with a bsb_last_error() message. */
BSB_API int bsb_mask_refine_weights(int sigma, int* w);
/* Camera blur mode.  A camera-blur frame is one whose background is its own blurred camera frame: in a plain call, no
 * context image or ring, no live background, bgblur k > 0, the filter on, and a call that blends (a composite or video
 * output); in a sources call, a frame whose effect blurs its camera frame (bsb_set_source_effect without an image).
 * BSB_BLUR_PLAIN (the default) blurs the whole camera frame, person included, as the reference does
 * (app/deepseg.cc:652-658); the person's colours are then smeared into the background around them, a halo about k/2
 * pixels wide around the outline.  BSB_BLUR_MASKED leaves the person out of the background blur: for such a frame, with C
 * its camera frame as the composite reads it (BGR; YUYV / NV12 after the fused path's conversion), M its W x H mask
 * exactly as the call writes it (refined, held, 255 outside roidim), q the 8.8 taps of bsb_gaussian_taps(k), r = k >> 1
 * and rho the BORDER_REFLECT_101 index,
 *   h_c(x,y) = sum_j q[j] M(rho(x+j-r),y) C_c(rho(x+j-r),y)      (< 2^24)
 *   g(x,y)   = sum_j q[j] M(rho(x+j-r),y)                         (< 2^16)
 *   N_c(x,y) = sum_i q[i] h_c(x,rho(y+i-r))                       (< 2^32)
 *   D(x,y)   = sum_i q[i] g(x,rho(y+i-r))                         (< 2^24)
 *   B_c(x,y) = D > 0 ? (N_c + (D >> 1)) / D : C_c(x,y)            (uint32)
 * B takes the place of GaussianBlur(C); the blend with the same M, flip, resize, framing, YUYV / NV12, BGRA and the
 * camera-blur slots' cached YUYV / NV12 follow as before.  A mask uniform at any v > 0 gives GaussianBlur(C) byte for byte;
 * k = 1 gives C; D = 0 only where M = 0 at the pixel, whose background then has no weight in the blend.
 * The mode changes nothing for frames that blend an image (the context image or ring, a source image or ring, a live
 * background), filter-off frames, calls that blend nothing (BGRA or mask only), bs_maskgen_process and bsb_calcmask_*.
 * Host state only: each frame's mode reaches the device in a table with the call, so once both kinds of a call have run,
 * changing the mode replays a captured call (the context's first masked call allocates the mask staging, and the row /
 * column class's 16 bytes per pixel of row sums, which drops the captured calls once).  A call with no masked camera-blur frame runs exactly the kernels it runs in
 * plain mode; one with some runs the post kernel once more, mask only, and the masked Gaussian (see README for its cost).
 * mode: BSB_BLUR_PLAIN or BSB_BLUR_MASKED.  Out of range returns 0 with a bsb_last_error() message and changes nothing. */
enum { BSB_BLUR_PLAIN = 0, BSB_BLUR_MASKED = 1 };
BSB_API int bsb_set_blur_mode(bsb_ctx* ctx, int mode);
/* One source's mode: -1 follows bsb_set_blur_mode (including later changes), else BSB_BLUR_PLAIN or BSB_BLUR_MASKED.
 * bsb_set_sources resets every source to -1; bsb_reset_source keeps it.  No bsb_set_sources yet, a source id out of range
 * or a mode out of range returns 0 with a bsb_last_error() message and changes nothing. */
BSB_API int bsb_set_source_blur_mode(bsb_ctx* ctx, int source, int mode);
/* Live backgrounds (the reference's `-b` takes any OpenCV source and blends its newest frame every loop iteration,
 * app/deepseg.cc:522-524,648-661): device images the caller already holds (decoded video surfaces, screen captures, a
 * second camera) are resized, blurred and blended inside the call, with no host copy and no launch outside it.
 * BSB_LIVE_BGR: bg_w x bg_h x 3 rows `pitch` bytes apart.  BSB_LIVE_NV12: a Y plane of bg_h rows `pitch` bytes apart and the
 * interleaved UV plane at byte `uv_offset` (the pitched surfaces of a hardware decoder need no copy); uv_offset is ignored
 * for BGR.
 *   Exactness: frame b of a call with live background L gives exactly the composite, video output (YUYV / NV12), mask and
 *   BGRA output of a plain batch-1 context set up the same way (bgblur, output, filter and format settings) plus
 *   bsb_set_background(L), fed the same stream one frame per call; for an NV12 L, bsb_set_background of
 *   bsb_convert_nv12_to_bgr(L).  That is cv::resize INTER_LINEAR of L to W x H (the exact 2x down-scale takes OpenCV's
 *   INTER_AREA mean), then the Gaussian at the frame's strength, then alpha_blend.
 *   Precedence: in plain calls a live background wins over the context image or ring, and a camera-blur context blurs the
 *   live frame instead of the camera frame.  In sources calls, for a source at BSB_SOURCE_BG_DEFAULT: its live background,
 *   else its own image or ring, else the context background; at BSB_SOURCE_BG_NONE the live background is ignored, as its
 *   own image is.  The strength is the source's effective one; bsb_set_live_background applies to plain calls only.
 *   A ring cursor keeps moving while a live background hides the ring.  A frame that blends nothing (its filter off, or a
 *   BGRA call without a video output) reads no live background.
 *   Host bookkeeping only: no device work and no synchronisation, so the pointers may change every call; they reach the
 *   device with the call's tables, and a captured call replays for new pointers, sizes already seen and strengths within
 *   the Gaussian classes it was captured with.  A size not seen before has its resize tables built once (kept per distinct
 *   size; reusing the tables of a size no live background uses any more waits for the context's stream).
 *   Caller contract: device memory of the context's device, in place when the call's work runs on the context stream
 *   (bsb_stream) and unchanged until that work completes; read by every later call until replaced or cleared, the
 *   host-buffer entry points included.
 * A violated rule returns 0 with a bsb_last_error() message and leaves the context as it was: fmt outside 0..1, bg_w or bg_h
 * outside 1..16384, BGR pitch < bg_w*3, NV12 with an odd bg_w or bg_h, pitch < bg_w or uv_offset < pitch*bg_h. */
enum { BSB_LIVE_BGR = 0, BSB_LIVE_NV12 = 1 };
/* plain calls: frame b of every later plain composite call blends live frame b (d_frames + b*frame_stride; frame_stride 0 =
 * one image for every frame of the call; a nonzero frame_stride smaller than one frame is refused).  d_frames NULL clears. */
BSB_API int bsb_set_live_background(bsb_ctx* ctx, const uint8_t* d_frames, int fmt, int bg_w, int bg_h,
                                    size_t pitch, size_t uv_offset, size_t frame_stride);
/* sources calls: the frame of `source` in every later sources call blends this image.  d_frame NULL clears.  No
 * bsb_set_sources yet or a source id out of range is refused.  bsb_set_sources clears every source's live background;
 * bsb_reset_source keeps it. */
BSB_API int bsb_set_source_live_background(bsb_ctx* ctx, int source, const uint8_t* d_frame, int fmt, int bg_w, int bg_h,
                                           size_t pitch, size_t uv_offset);

/* ---- fused per-frame path: one CUDA-graph launch per call ---------------------------
 * mask generation (bs_maskgen_process) + alpha_blend(bg, frame, mask)
 * (app/deepseg.cc:108-134, :661) + convert_rgb_to_yuyv (app/deepseg.cc:87-106, :681).
 * HOST buffers; n_frames consecutive frames of the stream (1 <= n <= max_batch), laid out
 * `frame_stride` bytes apart.  Any of out / out_yuyv / out_mask may be NULL. */
BSB_API int bsb_composite(bsb_ctx* ctx, int n_frames, const uint8_t* frames, size_t frame_pitch, size_t frame_stride,
                          uint8_t* out, size_t out_pitch, size_t out_stride,
                          uint8_t* out_yuyv, size_t yuyv_stride, uint8_t* out_mask, size_t mask_stride);

/* Same with DEVICE pointers (frames already resident in HBM; tightly packed W*3 / W*2 / W
 * rows).  Asynchronous on the context's stream unless `sync` is non-zero. */
BSB_API int bsb_composite_device(bsb_ctx* ctx, int n_frames, const uint8_t* d_frames, size_t frame_stride,
                                 uint8_t* d_out, size_t out_stride, uint8_t* d_yuyv, size_t yuyv_stride,
                                 uint8_t* d_mask, size_t mask_stride, int sync);
/* Camera-format ingest: the same fused call fed with YUYV frames (W*2 bytes per row, tightly packed) — the
 * YUYV -> BGR conversion cv::VideoCapture performs for the reference (CAP_PROP_CONVERT_RGB,
 * app/deepseg.cc:553; cv::COLOR_YUV2BGR_YUYV) runs on the GPU ahead of the pipeline.  HOST buffers. */
BSB_API int bsb_composite_yuyv(bsb_ctx* ctx, int n_frames, const uint8_t* yuyv_frames, size_t in_stride,
                               uint8_t* out, size_t out_stride, uint8_t* out_yuyv, size_t yuyv_stride,
                               uint8_t* out_mask, size_t mask_stride);
/* MJPG camera ingest (app/deepseg.cc:548-553: the capture is opened with FOURCC MJPG and cv::VideoCapture decodes each
 * JPEG to BGR): `n_frames` JPEG images (pointer + size each, HOST memory) are decoded on the GPU by NVJPG (libnvjpeg,
 * loaded at run time; a library decoder for a wire format either side of the path, like FFmpeg is for the reference)
 * straight into the context's BGR frame buffer, then the fused call runs as in bsb_composite.  Decoded pixels may differ
 * from libjpeg's by a few LSB (different IDCT / chroma up-sampling), so bsb_decode_mjpg returns the frame the pipeline saw.
 * Returns 0 with an error message if libnvjpeg is not available. */
BSB_API int bsb_composite_mjpg(bsb_ctx* ctx, int n_frames, const uint8_t* const* jpegs, const size_t* jpeg_sizes,
                               uint8_t* out, size_t out_stride, uint8_t* out_yuyv, size_t yuyv_stride, uint8_t* out_mask, size_t mask_stride);
/* the decode step alone: one JPEG -> W x H x 3 BGR (tightly packed HOST buffer) */
BSB_API int bsb_decode_mjpg(bsb_ctx* ctx, const uint8_t* jpeg, size_t jpeg_size, uint8_t* bgr_out);
/* DEVICE pointers, asynchronous unless `sync`. */
BSB_API int bsb_composite_yuyv_device(bsb_ctx* ctx, int n_frames, const uint8_t* d_yuyv_frames,
                                      uint8_t* d_out, size_t out_stride, uint8_t* d_yuyv, size_t yuyv_stride,
                                      uint8_t* d_mask, size_t mask_stride, int sync);

/* ---- NV12 camera frames in, NV12 composites out ------------------------------------------
 * NV12 (8-bit 4:2:0, what hardware video decoders produce and encoders take): a Y plane of H rows, then an interleaved UV
 * plane of H/2 rows of W/2 (U, V) byte pairs.  Frames have an even width and height.
 * Ingest is cv::cvtColor(COLOR_YUV2BGR_NV12), which equals COLOR_YUV2BGR_YUYV on the YUYV frame built from the same Y
 * plane and, for each pixel, the UV pair of its 2x2 block: the arithmetic of the YUYV ingest.
 * Output is derived from the YUYV output (convert_rgb_to_yuyv, app/deepseg.cc:87-106) of the out_w x out_h composite
 * (both even), by byte position:
 *   Y[y][x]          = the Y byte of pixel x in row y of the YUYV output,
 *   UV[r][2j]        = (yuyv[2r][4j+1] + yuyv[2r+1][4j+1]) >> 1,
 *   UV[r][2j+1]      = (yuyv[2r][4j+3] + yuyv[2r+1][4j+3]) >> 1   (yuyv[row][byte]),
 * the reference's truncating pair average applied vertically.  The reference's "RGB2YUV" runs on BGR data, so its
 * channel names are swapped; keeping byte positions gives a consumer the colours of the YUYV output.
 * DEVICE pointers.  Input: row pitch `in_pitch` >= W, the UV plane at byte `uv_offset` >= in_pitch*H of each frame (the
 * pitched surfaces of a hardware decoder need no copy), `in_stride` bytes per frame.  The NV12 output is tightly packed
 * (W-byte rows, UV plane at byte out_w*out_h), `nv12_stride` bytes per frame.  Any of d_out / d_nv12_out / d_mask may be
 * NULL.  Asynchronous on the context's stream unless `sync`.  A violated rule (odd W or H, odd out_w / out_h with an NV12
 * output, in_pitch < W, uv_offset < in_pitch*H, a frame larger than in_stride, NULL frames, n_frames out of range)
 * returns 0 with a bsb_last_error() message and leaves the context usable. */
BSB_API int bsb_composite_nv12_device(bsb_ctx* ctx, int n_frames, const uint8_t* d_nv12, size_t in_pitch, size_t uv_offset, size_t in_stride,
                                      uint8_t* d_out, size_t out_stride, uint8_t* d_nv12_out, size_t nv12_stride,
                                      uint8_t* d_mask, size_t mask_stride, int sync);
/* HOST buffers, tightly packed NV12 frames (W-byte rows, UV plane at W*H), `in_stride` bytes per frame; one serial
 * copy in -> graph -> copy out. */
BSB_API int bsb_composite_nv12(bsb_ctx* ctx, int n_frames, const uint8_t* nv12, size_t in_stride, uint8_t* out, size_t out_stride,
                               uint8_t* nv12_out, size_t nv12_stride, uint8_t* out_mask, size_t mask_stride);

/* ---- independent sources: one frame from each of several cameras in one launch ----------
 * A "source" is one camera stream with its own temporal smoother state (what one
 * bs_maskgen_new context holds in the reference, lib/libbackscrub.cc:161-259).  A sources call
 * composites frame b as the next frame of source source_ids[b]; source_ids is a HOST array of
 * n_frames ids, all distinct, each in [0, n_sources), 1 <= n_frames <= max_batch.  Frame b blends,
 * in this order: the source's own background (bsb_set_source_background); else the context
 * background (bsb_set_background, or the green default), blurred when bgblur is on; else, with
 * bgblur on and no background of either kind, its own blurred camera frame (app/deepseg.cc:652-658).
 * That is the default effect of every source; bsb_set_source_effect changes it per source.
 * bsb_set_output's size and flips apply to every source without its own
 * (bsb_set_source_output, bsb_set_source_flip); callbacks do not fire; the context
 * background must not be a ring of more than one image.  Plain calls never touch the per-source
 * states and sources calls never touch the plain smoother state, so both can be mixed on one
 * context.  A violated rule returns 0 with a bsb_last_error() message and leaves the context usable. */
/* Allocates n_sources zeroed smoother states and the per-source background bank (n_sources may
 * exceed max_batch).  Calling it again reallocates and zeroes everything. */
BSB_API int bsb_set_sources(bsb_ctx* ctx, int n_sources);
/* Zeroes one source's smoother state: the source starts over as a new camera. */
BSB_API int bsb_reset_source(bsb_ctx* ctx, int source);
/* bsb_set_background for one source: cv::resize(raw -> W x H) on the GPU (app/background.cc:178-194) into
 * the source's slot, blurred once if bgblur is on.  bg_raw NULL clears the slot, or the source's ring (the source blends
 * the context background again).  The ring of one image at advance 0 (bsb_set_source_background_ring).  Video
 * backgrounds: bsb_set_source_background_ring. */
BSB_API int bsb_set_source_background(bsb_ctx* ctx, int source, const uint8_t* bg_raw, int bg_w, int bg_h, size_t bg_pitch);
/* Animated background of one source: bsb_set_background_ring for one camera of a sources context.  `count` decoded images,
 * `frame_stride` bytes apart, are resized to W x H on the GPU (app/background.cc:178-194), blurred at the source's
 * effective strength, and kept on the device with their YUYV / NV12.  The source's cursor starts at 0.  Each sources call
 * that carries a frame of the source blends ring image cursor, then moves the cursor on by `advance` (mod count).
 * advance 0 leaves pacing to the caller (bsb_set_source_background_cursor), as the reference paces by wall clock.
 * Frame b of a sources call, from source s with its own ring, gives exactly the composite, YUYV / NV12 output and mask of a
 * plain batch-1 context set up with bsb_set_background_ring(same frames, same advance), bsb_set_bgblur(k_s) and
 * bsb_set_output(flip_s, size_s), with the same cursor moves.  The rules:
 *   - the cursor moves only for a call that carries a frame of the source and is enqueued; a refused call moves none;
 *   - the cursor keeps moving while the ring is not blended (BSB_SOURCE_BG_NONE, camera blur), as a video keeps playing;
 *     back to BSB_SOURCE_BG_DEFAULT, the source resumes at the advanced cursor;
 *   - the ring follows the source's effective strength: bsb_set_source_effect with a new strength re-blurs it, and
 *     bsb_set_bgblur re-blurs every ring whose source follows the context (one Gaussian per image);
 *   - bsb_set_source_background(s, img) is the ring of one image at advance 0 (kept in the source's own bank slot);
 *     bsb_set_source_background(s, NULL) clears a ring of any count;
 *   - a ring replaced by one of the same count rewrites its images in place, in stream order (no reallocation, the
 *     captured graphs are kept): the way to stream decoded frames into a fixed ring.  Any other change of the ring pool (a
 *     new ring, another count, a cleared ring) allocates the new bank before freeing the old one, copies the other rings
 *     over, synchronises the context's stream and drops the captured graphs;
 *   - bsb_reset_source leaves the cursor; bsb_set_sources frees every ring.
 * Device memory: W*H*6.5 bytes per image (BGR, YUYV and NV12 of the blurred image) plus W*H*3 (the unblurred image kept
 * for re-blurring).  No bsb_set_sources yet, a source id out of range, NULL frames, count < 1, bg_w / bg_h <= 0,
 * bg_pitch < bg_w*3, a frame_stride too small for count > 1, advance < 0 or a refused device allocation return 0 with a
 * bsb_last_error() message and leave the context and every source's background and cursor as they were. */
BSB_API int bsb_set_source_background_ring(bsb_ctx* ctx, int source, const uint8_t* frames, int count, int bg_w, int bg_h,
                                           size_t bg_pitch, size_t frame_stride, int advance);
/* Host bookkeeping only (no device work, no synchronisation), so it may be called per frame: the index reaches the device
 * with the call's source table.  index in 0..count-1 of the source's own background; a source without an image of its
 * own, an index out of range, a source id out of range or no bsb_set_sources yet return 0 with a bsb_last_error() message. */
BSB_API int bsb_set_source_background_cursor(bsb_ctx* ctx, int source, int index);
/* Background effect of one source.  Frame b of a sources call, from source s, gives exactly the bytes a plain
 * context gives for that camera's stream when set up with the background s would blend (its own image, else the
 * context image, else none) and bsb_set_bgblur(k), k = s's effective strength.
 * background: BSB_SOURCE_BG_DEFAULT = the source's own image if set, else the context background (the rule above);
 *             BSB_SOURCE_BG_NONE    = no image at all, as a reference run without -b: the blurred camera frame when
 *                                     the strength is > 0, else plain green (the source's own image is kept,
 *                                     unused, until DEFAULT again).
 * bgblur:     -1 = follow the context (bsb_set_bgblur, including later changes), 0 = off, odd 1..255.
 * bsb_set_sources resets every source to (DEFAULT, -1).  The camera-blur mode of plain calls stays per context.  An unknown background, an even / out-of-range strength, a source id out of range or no
 * bsb_set_sources yet return 0 with a bsb_last_error() message.
 * Cost: bsb_set_background and bsb_set_bgblur refresh the background of every source except one with its own image (or
 * ring) at a fixed strength, and bsb_set_background leaves own images that follow the context's strength too: a Gaussian
 * for each such source image with a strength > 0, every image of a ring (nothing is cached by strength). */
enum { BSB_SOURCE_BG_DEFAULT = 0, BSB_SOURCE_BG_NONE = 1 };
BSB_API int bsb_set_source_effect(bsb_ctx* ctx, int source, int background, int bgblur);
/* Mirroring of one source (cv::flip, app/deepseg.cc:667-673, toggled at run time by the `h` / `v` keys, :785-790).
 * flip: -1 = follow bsb_set_output's flips, including later changes; 0..3 = the source's own, a mask of BSB_FLIP_H
 * (horizontal) and BSB_FLIP_V (vertical).  Frame b of a sources call, from source s, gives exactly the composite, YUYV /
 * NV12 output and mask of a plain context set up the same way plus bsb_set_output(flip_h_s, flip_v_s, out_w, out_h).
 * The mask is never flipped.  bsb_set_sources resets every source to -1.  Host bookkeeping only (no device work, no
 * synchronisation), so it may be called per frame; the flips reach the device with the call's source table.  Without a
 * resize in the call, where the TMA post kernel takes the geometry, it writes the mirrored frames in place; otherwise one
 * tail kernel flips, resizes and converts the staged frames.  A flip outside -1..3, a source id out of range or no
 * bsb_set_sources yet return 0 with a bsb_last_error() message. */
enum { BSB_FLIP_H = 1, BSB_FLIP_V = 2 };
BSB_API int bsb_set_source_flip(bsb_ctx* ctx, int source, int flip);
/* Filter switch of one source (app/deepseg.cc:624,639-664, toggled at run time by the `s` key, :782-784).
 * active: -1 = follow bsb_set_filter, including later changes; 0 = off; 1 = on.  Frame b of a sources call, from source s,
 * gives exactly the composite, YUYV / NV12 output and mask of a plain context set up the same way plus
 * bsb_set_filter(active_s): with the filter off, the camera frame flipped, resized and converted, the mask still written
 * and the source's smoother still advanced.  Switching one source changes no other frame's bytes.  A frame with its
 * filter off blends nothing, so a camera-blur source that is off costs no Gaussian.  bsb_set_sources resets every source
 * to -1.  Host bookkeeping only (no device work, no synchronisation), so it may be called per frame; which frames are off
 * reaches the device with the call's source table, and a call with some frame off replays one of at most two graphs per
 * buffer set.  active outside -1..1, a source id out of range or no bsb_set_sources yet return 0 with a bsb_last_error()
 * message and leave the context as it was. */
BSB_API int bsb_set_source_filter(bsb_ctx* ctx, int source, int active);
/* Virtual-camera size of one source (cv::resize after the flip, before the YUYV / NV12 conversion, app/deepseg.cc:667-681).
 * out_w <= 0 and out_h <= 0: follow bsb_set_output's size, including later changes; otherwise both in 1..16384.
 * Frame b of a sources call, from source s, gives exactly the composite, YUYV / NV12 output and mask of a plain context
 * set up the same way plus bsb_set_output(flip_h_s, flip_v_s, out_w_s, out_h_s).  The mask stays W x H.
 * Output layout of a sources call: frame b's composite is tightly packed at its own size (rows out_w_b*3 bytes) at
 * out + b*out_stride, its YUYV / NV12 tightly packed at video + b*video_stride; the strides must hold the largest frame of
 * the call.  A call refuses, before any launch, a frame of its own size whose bytes do not fit its stride, an NV12 output
 * for a frame of odd own width or height, and (host buffers) a YUYV output for a frame of odd own width.
 * bsb_set_sources resets every source to follow.  No bsb_set_sources yet, a source id out of range or a size out of range
 * or half given return 0 with a bsb_last_error() message.  Each distinct size keeps one set of resize tables on the
 * device; replacing tables a queued call may read waits for the context's stream, and the host-buffer staging grows to
 * the largest size (dropping the captured graphs) when a size exceeds it. */
BSB_API int bsb_set_source_output(bsb_ctx* ctx, int source, int out_w, int out_h);
/* the effective size of one source (its own, or the context's) */
BSB_API int bsb_source_output_size(bsb_ctx* ctx, int source, int* out_w, int* out_h);
/* HOST buffers, BGR frames, laid out as in bsb_composite (out rows tightly packed, `out_stride` bytes
 * per frame).  Any of out / out_yuyv / out_mask may be NULL. */
BSB_API int bsb_composite_sources(bsb_ctx* ctx, int n_frames, const int* source_ids, const uint8_t* frames, size_t frame_pitch,
                                  size_t frame_stride, uint8_t* out, size_t out_stride, uint8_t* out_yuyv, size_t yuyv_stride,
                                  uint8_t* out_mask, size_t mask_stride);
/* DEVICE pointers, camera YUYV frames, laid out as in bsb_composite_yuyv_device; asynchronous unless
 * `sync`.  The id table is copied before the call returns, so it may be reused at once. */
BSB_API int bsb_composite_sources_yuyv_device(bsb_ctx* ctx, int n_frames, const int* source_ids, const uint8_t* d_yuyv_frames,
                                              uint8_t* d_out, size_t out_stride, uint8_t* d_yuyv, size_t yuyv_stride,
                                              uint8_t* d_mask, size_t mask_stride, int sync);
/* DEVICE pointers, camera NV12 frames and NV12 output, laid out as in bsb_composite_nv12_device. */
BSB_API int bsb_composite_sources_nv12_device(bsb_ctx* ctx, int n_frames, const int* source_ids, const uint8_t* d_nv12, size_t in_pitch,
                                              size_t uv_offset, size_t in_stride, uint8_t* d_out, size_t out_stride,
                                              uint8_t* d_nv12_out, size_t nv12_stride, uint8_t* d_mask, size_t mask_stride, int sync);
/* ---- asynchronous mask front-end: the reference's CalcMask (app/deepseg.cc:159-286) ----
 * A worker thread owns the mask-generation context.  set_input_frame clones the frame and wakes the worker (a
 * frame that arrives while the worker is busy replaces the pending one: latest frame wins); get_output_mask copies
 * the newest finished mask ONCE (returns 1) and otherwise leaves `out` untouched and returns 0, so the caller keeps
 * blending with its previous mask exactly like `ai.get_output_mask(mask)` in app/deepseg.cc:641; -1 after a
 * processing error (the reference exits the process there).  timings: waitns, prepns, tfltns, maskns, loopns
 * (app/deepseg.cc:233-237, printed by `-d`). */
typedef struct bsb_calcmask bsb_calcmask;
BSB_API bsb_calcmask* bsb_calcmask_new(const char* modelname, size_t threads, size_t width, size_t height, int device);
BSB_API void bsb_calcmask_delete(bsb_calcmask* cm);
BSB_API int bsb_calcmask_set_input_frame(bsb_calcmask* cm, const uint8_t* frame, size_t frame_pitch);
BSB_API int bsb_calcmask_get_output_mask(bsb_calcmask* cm, uint8_t* out, size_t out_pitch);
BSB_API int bsb_calcmask_timings(bsb_calcmask* cm, long ns[5]);
/* frames the worker has finished; the 1-based index (count of set_input_frame calls) of the frame behind the newest mask */
BSB_API long bsb_calcmask_frames_done(bsb_calcmask* cm);
BSB_API long bsb_calcmask_mask_serial(bsb_calcmask* cm);

/* ---- background provider object: the reference's background_t (app/background.cc:13-202) ----
 * still image: the decoded image is kept; grab returns it resized and frame number 1.
 * video: a reader thread pulls decoded frames through `read` (1 = a frame, 0 = end of stream; the pixels must stay
 * valid until the next call), publishes the latest one under a mutex, counts frames, paces itself to `fps`
 * (all sources play in real time, app/background.cc:84-92) and at end of stream calls `rewind` (1 = repositioned
 * at frame 0) and starts over with frame number 0, or stops when the source cannot rewind (:93-102).
 * `first`: the frame load_background() decoded while probing (may be NULL); start_frame: 0 after a successful
 * rewind of the probe reads, else 2 (:146-149).  grab: cv::resize(latest -> width x height) on the GPU, returns the
 * frame number (1 for stills, may wrap to 0), -1 on error (app/background.cc:178-194).  grab_into: the same resize
 * straight into a context's device-resident background (no host round trip).  thumbnail: 160-pixel-wide copy of the
 * latest frame, refreshed by the reader when debug > 1 (:65-78); returns 0 and the size (0 x 0 if none yet). */
typedef struct bsb_background bsb_background;
typedef int (*bsb_bg_read_cb)(void* user, const uint8_t** data, int* width, int* height, size_t* pitch);
typedef int (*bsb_bg_rewind_cb)(void* user);
BSB_API bsb_background* bsb_background_new_still(int device, const uint8_t* raw, int width, int height, size_t pitch, int debug);
BSB_API bsb_background* bsb_background_new_video(int device, double fps, int start_frame, bsb_bg_read_cb read, bsb_bg_rewind_cb rewind,
                                                 void* user, const uint8_t* first, int width, int height, size_t pitch, int debug);
BSB_API void bsb_background_delete(bsb_background* bg);
BSB_API int bsb_background_grab(bsb_background* bg, int width, int height, uint8_t* out, size_t out_pitch);
BSB_API int bsb_background_grab_into(bsb_background* bg, bsb_ctx* ctx);
BSB_API int bsb_background_thumbnail(bsb_background* bg, uint8_t* out, size_t capacity, int* width, int* height);
BSB_API int bsb_background_frame(bsb_background* bg);
BSB_API int bsb_background_running(bsb_background* bg);

BSB_API int bsb_synchronize(bsb_ctx* ctx);
/* the context's cudaStream_t (for event timing on the launching stream) */
BSB_API void* bsb_stream(bsb_ctx* ctx);

/* ---- stand-alone stages (stage-level parity; HOST buffers, tightly packed) -----------
 * app/deepseg.cc:108-134 */
BSB_API int bsb_alpha_blend(int device, const uint8_t* srca, const uint8_t* srcb, const uint8_t* mask,
                            uint8_t* out, size_t npix);
/* app/deepseg.cc:87-106 */
BSB_API int bsb_convert_rgb_to_yuyv(int device, const uint8_t* rgb, uint8_t* yuyv, int width, int height);
/* cv::cvtColor(COLOR_YUV2BGR_YUYV) (camera ingest, app/deepseg.cc:553,725) */
BSB_API int bsb_convert_yuyv_to_bgr(int device, const uint8_t* yuyv, uint8_t* bgr, int width, int height);
/* cv::cvtColor(COLOR_YUV2BGR_NV12), tightly packed NV12 (width, height even) */
BSB_API int bsb_convert_nv12_to_bgr(int device, const uint8_t* nv12, uint8_t* bgr, int width, int height);
/* cv::GaussianBlur(src, dst, Size(k,k), 0) 8UC3 (app/deepseg.cc:657-658) and its 8.8 fixed-point taps (host only) */
BSB_API int bsb_gaussian_blur(int device, const uint8_t* src, uint8_t* dst, int width, int height, int ksize);
BSB_API int bsb_gaussian_taps(int ksize, int* taps);
/* The masked camera blur B of bsb_set_blur_mode: src 8UC3, mask 8UC1 (any bytes), both width x height */
BSB_API int bsb_masked_gaussian_blur(int device, const uint8_t* src, const uint8_t* mask, uint8_t* dst, int width, int height, int ksize);
/* cv::flip(src, dst, code) 8UC3 (app/deepseg.cc:667-673) */
BSB_API int bsb_flip(int device, const uint8_t* src, uint8_t* dst, int width, int height, int flip_h, int flip_v);
/* cv::resize(src, dst, Size(dw, dh)) 8UC3 (app/background.cc:178-194) */
BSB_API int bsb_resize_u8c3(int device, const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh);

/* 1x1 convolution stage on HOST buffers: out[M][N] = act(A[M][K] * W[N][K]^T + bias).  variant 0: exact FFMA
 * kernels, chosen by shape (k-ascending fmaf, bit-identical to the oracle); 1: wgmma 3xTF32 tensor-core kernel
 * (needs K % 4 == 0); 2 / 3: force the classic / the register-tiled exact FFMA kernel (same bits as 0).
 * act is a TFLite fused-activation code (0 none, 1 relu, 3 relu6). */
BSB_API int bsb_pointwise(int device, int variant, int M, int K, int N, const float* A, const float* W,
                          const float* bias, int act, float* out);
/* The same stage the way the engine calls it: operands that are sub-matrices of larger buffers and the full epilogue
 *   out[m][n] = act3(act2(act1(sum_k A[m][k] W[n][k] + bias[n])) + residual[m][n])
 * A[m][k] is a[a_off + m * ld_a + k] (ld_a >= K), residual[m][n] is res[res_off + m * ld_res + n] (optional) and
 * out[m][n] is out[out_off + m * ld_out + n] (ld_out >= N).  Each buffer is copied whole to the device (a_len /
 * res_len / out_len floats, `out` included, so whatever lies outside the written elements comes back unchanged).
 * A must start on a 16-byte boundary (a_off % 4 == 0); the exact FFMA kernels also need out_off % 4 == 0.  The
 * tensor-core kernel refuses a shape or alignment it cannot take; then the call returns 0 and says why. */
BSB_API int bsb_pointwise_ex(int device, int variant, int M, int K, int N, const float* a, long a_len, long a_off, int ld_a,
                             const float* W, const float* bias, const float* res, long res_len, long res_off, int ld_res,
                             int act1, int act2, int act3, float* out, long out_len, long out_off, int ld_out);
/* ms per launch of the pointwise kernel `variant` (0, 2, 3, ...: exact FFMA kernels; 1: the tensor-core kernel selected by the
 * "tc_variant" tuning switch) on an M x K x N problem (CUDA events, zero data) */
BSB_API double bsb_time_pointwise(int device, int variant, int M, int K, int N, int iters);

/* ---- introspection (tests, bench) -------------------------------------------------- */
/* geometry: roidim / in_roidim / out_roidim as x,y,w,h (lib/libbackscrub.cc:234-246);
 * model input / output dims as h,w,c */
/* frame size the context was created for */
BSB_API int bsb_frame_size(bsb_ctx* ctx, int* width, int* height);
BSB_API int bsb_geometry(bsb_ctx* ctx, int roidim[4], int in_roidim[4], int out_roidim[4], int in_hwc[3], int out_hwc[3]);
/* run only the CNN on a caller-provided fp32 NHWC input batch (host), output to host */
BSB_API int bsb_infer(bsb_ctx* ctx, int n_frames, const float* input, float* output);
/* copy an intermediate activation (frame 0) to host; needs BSB_FLAG_KEEP_TENSORS.
 * Returns the element count, 0 if the tensor was folded away, -1 on error. */
BSB_API long bsb_get_tensor(bsb_ctx* ctx, int tensor_index, float* out, long capacity);
/* the same for frame `frame` of the last batch (with a mask interval: its frame-th segmented frame) */
BSB_API long bsb_get_tensor_frame(bsb_ctx* ctx, int tensor_index, int frame, float* out, long capacity);
/* the 1x1 convolutions planned for the tensor cores, 9 ints per step into rows (at most `capacity` steps): TFLite op
 * index, input, output and residual tensor (-1: none), K, N, act1, act2, act3 of the step's epilogue
 * out = act3(act2(act1(in * W^T + bias)) + residual).  Returns the number of such steps, -1 on error. */
BSB_API int bsb_tc_steps(bsb_ctx* ctx, int* rows, int capacity);
/* stage buffers of the last call, frame `frame`: which = 0 model-sized RGB u8 (after resize +
 * BGR2RGB), 1 bilateral-filtered u8, 2 ofinal (IIR state after that frame).  With a mask interval (bsb_set_mask_interval)
 * stages 0 and 1 index the call's segmented frames (the frame-th of them), stage 2 the call frame. */
BSB_API long bsb_get_stage_u8(bsb_ctx* ctx, int which, int frame, uint8_t* out, long capacity);
/* Test entry point: feed chosen values to the decision or the post stage of the next composite call, so that their
 * kernels can be checked on constructed inputs (ties, overflows, thresholds, single-pixel masks) rather than on what the
 * CNN makes of a frame.
 *   BSB_FEED_LOGITS: float32 values of the tensor the decision stage reads, [n][h][w][c] packed (DeepLab: the low-
 *                    resolution tensor of the resize the decision kernel folds in); pre-processing and the CNN are skipped.
 *                    The smoother states advance as in a real call.
 *   BSB_FEED_MASK:   the smoother output (`ofinal`) bytes, [n][oh][ow] packed; the decision is skipped too, and neither
 *                    the plain nor any source's smoother state changes.
 * bsb_test_feed copies `bytes` bytes (n_frames times the stage's frame size) and arms them for the next composite call on
 * the context, of any kind (plain, YUYV, NV12, device or host buffers, sources), which must have n_frames frames.  That
 * call runs eagerly (the captured CUDA graphs are neither used nor changed) and is synchronous; the YUYV / NV12 -> BGR
 * conversion and everything from the post stage on run as in any call.  The next composite call consumes the feed
 * whatever its outcome.  A wrong size, an unknown stage, a call of another frame count or a host call that would be
 * split into chunks (e2e_chunk) returns 0 with a bsb_last_error() message and leaves the context usable.
 * bsb_test_feed_shape: h, w, c of one frame of a stage's tensor into hwc; returns its bytes, -1 for an unknown stage. */
enum { BSB_FEED_LOGITS = 1, BSB_FEED_MASK = 2 };
BSB_API long bsb_test_feed_shape(bsb_ctx* ctx, int stage, int hwc[3]);
BSB_API int bsb_test_feed(bsb_ctx* ctx, int stage, int n_frames, const void* data, size_t bytes);
/* reset the temporal IIR state to zero (start of a new stream) */
BSB_API int bsb_reset_state(bsb_ctx* ctx);
/* kernel launches per n-frame call (graph nodes) and launches issued so far by this process */
BSB_API int bsb_launches_per_call(bsb_ctx* ctx, int n_frames);
BSB_API long bsb_total_launches(void);
/* Average device time (ms, CUDA events on the context's stream) of one stage of the per-call
 * kernel sequence, run `iters` times back to back on the context-owned device buffers:
 * stage 0 = pre-proc (resize+bilateral+normalise), 1 = CNN, 2 = decision+IIR,
 * 3 = post (mask upsample + blur + blend + YUYV), 4 = whole call.  Returns < 0 on error.
 * Measurement aid for bench.py's roofline block; it advances the IIR state. */
BSB_API double bsb_time_stage(bsb_ctx* ctx, int stage, int n_frames, int iters);
/* 1 if the last fused call read the camera frames in their wire format (YUYV or NV12) in place (pre-processing and post
 * kernels convert per tap / per tile), 0 if a BGR frame was materialised first (k_yuyv_to_bgr / k_nv12_to_bgr) or the
 * input was BGR */
BSB_API int bsb_yuyv_native(bsb_ctx* ctx);
/* 1 if at least one 1x1 conv of this context runs on the tensor cores */
BSB_API int bsb_uses_tensor_cores(bsb_ctx* ctx);
/* algorithmic FLOPs of one CNN frame (2*MAC) */
BSB_API double bsb_model_flops(bsb_ctx* ctx);
/* Process-wide measurement switches of the kernel launchers (A/B runs in bench.py / tools/): they select between
 * bit-identical kernel variants / schedules and never change results.  Names (defaults in csrc/kernels.h, struct Tuning):
 * planner fusions "cnn_chain", "pool_merge", "up_pw", "up_staged", "head", "pw_dws2", "stem_pw", "stem_x2", "dec_up", "sub_batch_mb";
 * kernel variants "pw_variant", "dw_px", "dw_plane", "dw_plane_cs", "epi_static", "dec_par", "tc_variant", "tc_min_k", "tc_mask_hi";
 * post stage "post_tma", "post_tile" (0 = by frame size), "post_l1"; host-buffer calls "e2e_chunk" (frames per
 * overlapped chunk of bsb_composite_yuyv, 0 = serial).  Set them before creating contexts (plans and captured CUDA graphs
 * keep the variant they were built with).  Returns 1, or 0 for an unknown name. */
BSB_API int bsb_set_tuning(const char* name, int value);

#ifdef __cplusplus
}
#endif
#endif
