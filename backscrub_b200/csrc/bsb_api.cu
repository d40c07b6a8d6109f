// backscrub_b200/csrc/bsb_api.cu — extern "C" entry points declared in include/backscrub_b200.h.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/backscrub_b200.h"
#include "engine.h"

#ifndef BSB_EMU
#include <dlfcn.h>
#include <nvjpeg.h>       // types only: the library is dlopen()ed so the product links against cudart alone
#include <mutex>
#endif

using bsb::Engine;

struct bsb_ctx {
  Engine* eng = nullptr;
  bsb::Callbacks cb;
  void* jpeg_state = nullptr;      // nvjpegJpegState_t of this context (MJPG ingest), created on first use
  // copy / compute overlap inside one host-buffer call (bsb_composite_yuyv): two copy streams and per-chunk events
  static constexpr int kMaxChunks = 16;
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_in[kMaxChunks] = {}, ev_done[kMaxChunks] = {};
  bool pipe_ready = false;
};

namespace {

thread_local std::string g_last_error;

// lib/libbackscrub.cc:72-83 (_dbg): message to the ondebug callback, else stderr
void report(const bsb::Callbacks* cb, const std::string& msg) {
  g_last_error = msg;
  std::string line = msg;
  if (line.empty() || line.back() != '\n') line += "\n";
  if (cb && cb->ondebug) cb->ondebug(cb->caller_ctx, line.c_str());
  else std::fputs(line.c_str(), stderr);
}

bool check_ctx(bsb_ctx* ctx) {
  if (!ctx || !ctx->eng) { g_last_error = "null context"; return false; }
  return true;
}

#define API_CUDA(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) { report(cbp, std::string("error: CUDA: ") + cudaGetErrorString(_e) + " at " #expr); return 0; } \
  } while (0)

}  // namespace

// ---- NVJPG (MJPG camera ingest) --------------------------------------------------------------------------
#ifndef BSB_EMU
namespace {
struct NvJpegApi {
  void* lib = nullptr;
  nvjpegHandle_t handle = nullptr;
  nvjpegStatus_t (*create)(nvjpegHandle_t*) = nullptr;
  nvjpegStatus_t (*state_create)(nvjpegHandle_t, nvjpegJpegState_t*) = nullptr;
  nvjpegStatus_t (*state_destroy)(nvjpegJpegState_t) = nullptr;
  nvjpegStatus_t (*info)(nvjpegHandle_t, const unsigned char*, size_t, int*, nvjpegChromaSubsampling_t*, int*, int*) = nullptr;
  nvjpegStatus_t (*decode)(nvjpegHandle_t, nvjpegJpegState_t, const unsigned char*, size_t, nvjpegOutputFormat_t, nvjpegImage_t*, cudaStream_t) = nullptr;
  bool ok = false;
};
NvJpegApi& nvjpeg_api() {
  static NvJpegApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    for (const char* name : {"libnvjpeg.so.12", "libnvjpeg.so"}) { api.lib = dlopen(name, RTLD_NOW | RTLD_LOCAL); if (api.lib) break; }
    if (!api.lib) return;
    api.create = reinterpret_cast<decltype(api.create)>(dlsym(api.lib, "nvjpegCreateSimple"));
    api.state_create = reinterpret_cast<decltype(api.state_create)>(dlsym(api.lib, "nvjpegJpegStateCreate"));
    api.state_destroy = reinterpret_cast<decltype(api.state_destroy)>(dlsym(api.lib, "nvjpegJpegStateDestroy"));
    api.info = reinterpret_cast<decltype(api.info)>(dlsym(api.lib, "nvjpegGetImageInfo"));
    api.decode = reinterpret_cast<decltype(api.decode)>(dlsym(api.lib, "nvjpegDecode"));
    if (!api.create || !api.state_create || !api.state_destroy || !api.info || !api.decode) return;
    api.ok = api.create(&api.handle) == NVJPEG_STATUS_SUCCESS;
  });
  return api;
}
// decode one JPEG into `d_bgr` (W x H x 3 device buffer) on the context's stream; "" on success
std::string jpeg_decode(bsb_ctx* ctx, const uint8_t* jpeg, size_t size, uint8_t* d_bgr) {
  NvJpegApi& api = nvjpeg_api();
  if (!api.ok) return "libnvjpeg is not available (MJPG ingest needs the CUDA toolkit's NVJPG library)";
  Engine* e = ctx->eng;
  if (!ctx->jpeg_state) {
    nvjpegJpegState_t st = nullptr;
    if (api.state_create(api.handle, &st) != NVJPEG_STATUS_SUCCESS) return "nvjpegJpegStateCreate failed";
    ctx->jpeg_state = st;
  }
  int ncomp = 0, ws[NVJPEG_MAX_COMPONENT] = {0}, hs[NVJPEG_MAX_COMPONENT] = {0};
  nvjpegChromaSubsampling_t sub;
  if (!jpeg || api.info(api.handle, jpeg, size, &ncomp, &sub, ws, hs) != NVJPEG_STATUS_SUCCESS) return "not a decodable JPEG image";
  if (ws[0] != e->W() || hs[0] != e->H()) return "JPEG frame size differs from the context's frame size";
  nvjpegImage_t img{};
  img.channel[0] = d_bgr; img.pitch[0] = (size_t)e->W() * 3;
  if (api.decode(api.handle, static_cast<nvjpegJpegState_t>(ctx->jpeg_state), jpeg, size, NVJPEG_OUTPUT_BGRI, &img, e->stream()) != NVJPEG_STATUS_SUCCESS)
    return "nvjpegDecode failed";
  return "";
}
}  // namespace
static void bsb_jpeg_release(bsb_ctx* ctx) {
  if (ctx->jpeg_state && nvjpeg_api().ok) nvjpeg_api().state_destroy(static_cast<nvjpegJpegState_t>(ctx->jpeg_state));
  ctx->jpeg_state = nullptr;
}
#else
static void bsb_jpeg_release(bsb_ctx*) {}
#endif

// ---- composite calls ---------------------------------------------------------------------------------------
namespace {
const char* const kProcessErr = "failed to process video frame: ";

// n frames of `rows` rows of `row` bytes, `sstride` bytes apart with rows `spitch` apart, to frames `dstride` apart with
// rows `dpitch` apart: one copy when both sides are tightly packed, else one per frame
cudaError_t copy_frames(uint8_t* dst, size_t dpitch, size_t dstride, const uint8_t* src, size_t spitch, size_t sstride, size_t row,
                        size_t rows, int n, cudaMemcpyKind kind, cudaStream_t s) {
  const size_t fb = row * rows;
  if (dpitch == row && spitch == row && dstride == fb && sstride == fb) return cudaMemcpyAsync(dst, src, fb * n, kind, s);
  for (int b = 0; b < n; ++b) {
    const cudaError_t e = cudaMemcpy2DAsync(dst + b * dstride, dpitch, src + b * sstride, spitch, row, rows, kind, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// frames [b0, b0 + n) of a call
bsb::Call frames_of(bsb::Call c, int b0, int n) {
  auto at = [b0](auto* p, size_t stride) { return p ? p + (size_t)b0 * stride : p; };
  c.n = n; c.in = at(c.in, c.stride); c.out = at(c.out, c.out_stride); c.video = at(c.video, c.video_stride); c.mask = at(c.mask, c.mask_stride);
  c.frame0 += b0;
  return c;
}

// the requested outputs of call `d` (on the context staging: packed, `orow`-byte BGR rows, `orows` rows, `vbytes`-byte
// video frames) back into the host buffers of call `h` (BGR rows `out_pitch` bytes apart, the video and mask frames packed)
cudaError_t copy_out(const bsb::Call& h, size_t out_pitch, const bsb::Call& d, size_t orow, size_t orows, size_t vbytes, cudaStream_t s) {
  const cudaMemcpyKind k = cudaMemcpyDeviceToHost;
  cudaError_t r = cudaSuccess;
  if (h.out) r = copy_frames(h.out, out_pitch, h.out_stride, d.out, orow, d.out_stride, orow, orows, h.n, k, s);
  if (h.video && r == cudaSuccess) r = copy_frames(h.video, vbytes, h.video_stride, d.video, vbytes, d.video_stride, vbytes, 1, h.n, k, s);
  if (h.mask && r == cudaSuccess) r = copy_frames(h.mask, d.mask_stride, h.mask_stride, d.mask, d.mask_stride, d.mask_stride, d.mask_stride, 1, h.n, k, s);
  return r;
}

// a sources call some of whose frames have their own output size (bsb_set_source_output): each frame's composite (or
// BGRA frame) and video output back at its own size, packed
cudaError_t copy_out_sized(const bsb::Call& h, const bsb::Call& d, const Engine* e, bool nv12, cudaStream_t s) {
  const cudaMemcpyKind k = cudaMemcpyDeviceToHost;
  for (int b = 0; b < h.n; ++b) {
    int w = 0, hh = 0;
    e->source_output_size(h.ids[b], &w, &hh);
    const size_t px = (size_t)w * hh;
    cudaError_t r = cudaSuccess;
    if (h.out) r = cudaMemcpyAsync(h.out + b * h.out_stride, d.out + b * d.out_stride, px * e->out_bpp(), k, s);
    if (h.video && r == cudaSuccess) r = cudaMemcpyAsync(h.video + b * h.video_stride, d.video + b * d.video_stride, nv12 ? px * 3 / 2 : px * 2, k, s);
    if (h.mask && r == cudaSuccess) r = cudaMemcpyAsync(h.mask + b * h.mask_stride, d.mask + b * d.mask_stride, d.mask_stride, k, s);
    if (r != cudaSuccess) return r;
  }
  return cudaSuccess;
}

// A feed armed by bsb_test_feed is consumed by the next composite call, also when that call is refused before it runs
struct FeedConsumed {
  Engine* e;
  ~FeedConsumed() { if (e->feed_armed()) e->disarm_feed(); }
};

// Every host-buffer composite call.  `h` describes the caller's host buffers: every row is packed except BGR input rows
// (h.pitch bytes apart) and, where given, output rows (*out_pitch bytes apart).  The frames are copied into the context
// staging (MJPG: `jpegs` decoded there instead), the call runs on it, and each requested output is copied back before
// the return.  `what` prefixes the engine's error.
int host_call(bsb_ctx* ctx, const bsb::Call& h, const char* what, const size_t* out_pitch = nullptr,
              const uint8_t* const* jpegs = nullptr, const size_t* jpeg_sizes = nullptr) {
  if (!check_ctx(ctx)) return 0;
  const bsb::Callbacks* cbp = &ctx->cb;
  Engine* e = ctx->eng;
  const FeedConsumed consumed{e};
  const bool bgr = h.fmt == bsb::IN_BGR, nv12 = h.fmt == bsb::IN_NV12;
  const size_t bpp = (size_t)e->out_bpp();            // bytes per `out` pixel: 3 (BGR), 4 (BGRA)
  const size_t W = e->W(), H = e->H(), orow = (size_t)e->out_w() * bpp, cpx = (size_t)e->out_w() * e->out_h();
  // sources calls: the staging holds frames of the largest size any source has; `sized`: some frame's size is its own
  bool sized = false;
  size_t opix = cpx;
  if (h.ids && e->n_sources()) {
    opix = std::max(opix, (size_t)e->sources_out_px_max());
    for (int b = 0; b < h.n && b < e->max_batch(); ++b) {
      int w = 0, hh = 0;
      if (!e->source_output_size(h.ids[b], &w, &hh)) continue;     // the engine reports the id
      if (w == e->out_w() && hh == e->out_h()) continue;
      sized = true;
      if (h.video && !nv12 && (w & 1)) { report(cbp, "error: YUYV output needs an even width"); return 0; }
    }
  }
  const size_t pitch = bgr ? W * 3 : nv12 ? W : W * 2, fbytes = nv12 ? W * H * 3 / 2 : pitch * H;   // of the staged frames
  const size_t opitch = out_pitch ? *out_pitch : orow;
  if (h.n < 1 || h.n > e->max_batch()) { report(cbp, "error: n_frames out of range (1..max_batch)"); return 0; }
  if (jpegs ? !jpeg_sizes : (!h.in || (bgr ? h.pitch < pitch : h.stride < fbytes))) { report(cbp, "error: invalid frame"); return 0; }
  if (nv12 && ((W | H) & 1)) { report(cbp, "error: NV12 needs an even frame width and height"); return 0; }
  if (h.out && opitch < orow) { report(cbp, "error: invalid output pitch"); return 0; }
  if (h.video && !nv12 && (e->out_w() & 1)) { report(cbp, "error: YUYV output needs an even width"); return 0; }
  API_CUDA(cudaSetDevice(e->device()));
  std::string err;
  if (sized && !e->check_source_outputs(h, &err)) { report(cbp, std::string("error: ") + what + err); return 0; }
  uint8_t* stage = bgr ? e->d_frames() : e->d_yuyv_in();
  bsb::Call d = h;                                   // the same call on the context staging
  d.in = stage; d.pitch = pitch; d.uv = nv12 ? W * H : 0; d.stride = fbytes;
  d.out = h.out ? (bpp == 3 ? e->d_out() : e->out_staging(&err)) : nullptr; d.out_stride = opix * bpp;
  if (h.out && !d.out) { report(cbp, "error: " + err); return 0; }
  d.video = nullptr; d.video_stride = nv12 ? opix * 3 / 2 : opix * 2;
  if (h.video && !(d.video = nv12 ? e->nv12_staging(&err) : e->d_yuyv())) { report(cbp, "error: " + err); return 0; }
  d.mask = h.mask ? e->d_mask() : nullptr; d.mask_stride = W * H;
  // YUYV calls of two chunks or more run chunked: the H2D copy of chunk c+1, the graph of chunk c and the D2H copy of
  // chunk c-1 overlap on three streams (the temporal smoother's state simply carries from chunk to chunk on the compute
  // stream).  A single-stream caller no longer pays copy + compute + copy back to back (app/deepseg.cc does exactly
  // that: cap.read -> CalcMask -> write); results are identical, only the schedule changes.
  const int chunk = bsb::tuning().e2e_chunk;
  const bool piped = h.fmt == bsb::IN_YUYV && chunk > 0 && h.n >= 2 * chunk && (h.n + chunk - 1) / chunk <= bsb_ctx::kMaxChunks;
  if (piped && e->feed_armed()) {
    report(cbp, std::string("error: ") + what + "a fed call runs as one launch, and this call would be split into chunks (e2e_chunk)");
    return 0;
  }
  if (piped && !ctx->pipe_ready) {
    API_CUDA(cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
    API_CUDA(cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < bsb_ctx::kMaxChunks; ++i) {
      API_CUDA(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
      API_CUDA(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming));
    }
    ctx->pipe_ready = true;
  }
  cudaStream_t s = e->stream(), s_in = piped ? ctx->s_in : s, s_out = piped ? ctx->s_out : s;
  const int step = piped ? chunk : h.n, nchunks = (h.n + step - 1) / step;
  for (int c = 0; c < nchunks; ++c) {
    const int b0 = c * step, nb = std::min(step, h.n - b0);
#ifndef BSB_EMU
    for (int b = b0; jpegs && b < b0 + nb; ++b) {
      const std::string derr = jpeg_decode(ctx, jpegs[b], jpeg_sizes[b], stage + (size_t)b * fbytes);
      if (!derr.empty()) { report(cbp, "error: " + derr); return 0; }
    }
#endif
    if (!jpegs)
      API_CUDA(copy_frames(stage + (size_t)b0 * fbytes, pitch, fbytes, h.in + (size_t)b0 * h.stride, bgr ? h.pitch : pitch, h.stride, pitch,
                           fbytes / pitch, nb, cudaMemcpyHostToDevice, s_in));
    if (piped) API_CUDA(cudaEventRecord(ctx->ev_in[c], s_in));
  }
  for (int c = 0; c < nchunks; ++c) {
    const int b0 = c * step, nb = std::min(step, h.n - b0);
    if (piped) API_CUDA(cudaStreamWaitEvent(s, ctx->ev_in[c], 0));
    const bsb::Call dc = frames_of(d, b0, nb);
    if (!e->run(dc, &err)) {
      if (piped) { cudaStreamSynchronize(s_in); cudaStreamSynchronize(s); cudaStreamSynchronize(s_out); }
      report(cbp, std::string("error: ") + what + err); return 0;
    }
    if (piped) { API_CUDA(cudaEventRecord(ctx->ev_done[c], s)); API_CUDA(cudaStreamWaitEvent(s_out, ctx->ev_done[c], 0)); }
    if (sized) API_CUDA(copy_out_sized(h, dc, e, nv12, s_out));
    else API_CUDA(copy_out(frames_of(h, b0, nb), opitch, dc, orow, e->out_h(), nv12 ? cpx * 3 / 2 : cpx * 2, s_out));
  }
  if (piped) API_CUDA(cudaStreamSynchronize(s_out));
  API_CUDA(cudaStreamSynchronize(s));
  API_CUDA(cudaGetLastError());
  return 1;
}

// Every device-pointer composite call.  The C ABI's device BGR frames have packed rows, its YUYV frames are packed.
int device_call(bsb_ctx* ctx, bsb::Call c, int sync) {
  if (!check_ctx(ctx)) return 0;
  const bsb::Callbacks* cbp = &ctx->cb;
  Engine* e = ctx->eng;
  const FeedConsumed consumed{e};
  if (c.fmt == bsb::IN_BGR) c.pitch = (size_t)e->W() * 3;
  if (c.fmt == bsb::IN_YUYV) { c.pitch = (size_t)e->W() * 2; c.stride = c.pitch * e->H(); }
  // the engine checks an NV12 call's frames and output with their layout
  if (c.fmt != bsb::IN_NV12 && !c.in) { report(cbp, "error: invalid frame"); return 0; }
  if (c.fmt != bsb::IN_NV12 && c.video && (e->out_w() & 1)) { report(cbp, "error: YUYV output needs an even width"); return 0; }
  std::string err;
  if (!e->run(c, &err)) { report(cbp, "error: " + err); return 0; }
  if (sync) { API_CUDA(cudaStreamSynchronize(e->stream())); API_CUDA(cudaGetLastError()); }
  return 1;
}

// sources entry points refuse a null id table first (a Call without ids is a plain call)
bool null_ids(bsb_ctx* ctx, const int* ids) {
  if (ids || !check_ctx(ctx)) return false;
  const FeedConsumed consumed{ctx->eng};
  report(&ctx->cb, "error: null source id table");
  return true;
}
}  // namespace

extern "C" {

const char* bsb_version(void) { return "backscrub-b200 0.1 (sm_90a CUDA; TFLite schema v3 graph runtime)"; }

const char* bsb_last_error(void) { return g_last_error.c_str(); }

int bsb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

bsb_ctx* bsb_maskgen_new_ex(const char* modelname, size_t width, size_t height, int device, int max_batch, unsigned flags,
                            bsb_debug_cb ondebug, bsb_stage_cb onprep, bsb_stage_cb oninfer, bsb_stage_cb onmask, void* caller_ctx) {
  bsb::Callbacks cb;
  cb.ondebug = ondebug; cb.onprep = onprep; cb.oninfer = oninfer; cb.onmask = onmask; cb.caller_ctx = caller_ctx;
  if (!modelname) { report(&cb, "error: null model name"); return nullptr; }
  std::string err;
  Engine* e = Engine::create(modelname, (int)width, (int)height, device, max_batch, flags, cb, &err);
  if (!e) { report(&cb, "error: " + err); return nullptr; }
  bsb_ctx* c = new bsb_ctx();
  c->eng = e; c->cb = cb;
  g_last_error.clear();
  return c;
}

bsb_ctx* bsb_maskgen_new(const char* modelname, size_t threads, size_t width, size_t height, bsb_debug_cb ondebug,
                         bsb_stage_cb onprep, bsb_stage_cb oninfer, bsb_stage_cb onmask, void* caller_ctx) {
  (void)threads;  // advisory in the reference as well (SetNumThreads after AllocateTensors, lib/libbackscrub.cc:217,224)
  return bsb_maskgen_new_ex(modelname, width, height, 0, 1, 0, ondebug, onprep, oninfer, onmask, caller_ctx);
}

void bsb_maskgen_delete(bsb_ctx* ctx) {
  if (!ctx) return;
  bsb_jpeg_release(ctx);
  if (ctx->pipe_ready && ctx->eng && cudaSetDevice(ctx->eng->device()) == cudaSuccess) {
    for (int i = 0; i < bsb_ctx::kMaxChunks; ++i) { if (ctx->ev_in[i]) cudaEventDestroy(ctx->ev_in[i]); if (ctx->ev_done[i]) cudaEventDestroy(ctx->ev_done[i]); }
    if (ctx->s_in) cudaStreamDestroy(ctx->s_in);
    if (ctx->s_out) cudaStreamDestroy(ctx->s_out);
  }
  delete ctx->eng;
  delete ctx;
}

int bsb_maskgen_process(bsb_ctx* ctx, const uint8_t* frame, size_t frame_pitch, const uint8_t** mask, size_t* mask_pitch) {
  if (!check_ctx(ctx)) return 0;
  Engine* e = ctx->eng;
  const size_t npix = (size_t)e->W() * e->H();
  bsb::Call c{1, bsb::IN_BGR, frame, frame_pitch, 0, npix * 3, nullptr, nullptr, 0, nullptr, 0, e->h_mask(), npix, true};
  c.mask_only_api = true;                      // the drop-in mask API is never refined
  if (!host_call(ctx, c, "failed to interpret video frame: ")) return 0;
  if (mask) *mask = e->h_mask();
  if (mask_pitch) *mask_pitch = (size_t)e->W();
  return 1;
}

int bsb_set_background(bsb_ctx* ctx, const uint8_t* bg_raw, int bg_w, int bg_h, size_t bg_pitch) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_background(bg_raw, bg_w, bg_h, bg_pitch, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_background_ring(bsb_ctx* ctx, const uint8_t* frames, int count, int bg_w, int bg_h, size_t bg_pitch, size_t frame_stride, int advance) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_background_ring(frames, count, bg_w, bg_h, bg_pitch, frame_stride, advance, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_background_cursor(bsb_ctx* ctx, int index) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_background_cursor(index, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_bgblur(bsb_ctx* ctx, int ksize) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_bgblur(ksize, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_output(bsb_ctx* ctx, int flip_h, int flip_v, int out_w, int out_h) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_output(flip_h != 0, flip_v != 0, out_w, out_h, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_filter(bsb_ctx* ctx, int active) {
  if (!check_ctx(ctx)) return 0;
  if (active != 0 && active != 1) { report(&ctx->cb, "error: filter must be 0 (off) or 1 (on)"); return 0; }
  ctx->eng->set_filter(active != 0);
  return 1;
}

int bsb_set_mask_interval(bsb_ctx* ctx, int interval) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_mask_interval(interval, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_mask_interval(bsb_ctx* ctx, int source, int interval) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_mask_interval(source, interval, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_framing(bsb_ctx* ctx, int mode, int x, int y, int w, int h) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_framing(mode, x, y, w, h, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_framing_auto(bsb_ctx* ctx, int max_zoom_pct, int margin_pct, int speed) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_framing_auto(max_zoom_pct, margin_pct, speed, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_framing(bsb_ctx* ctx, int source, int mode, int x, int y, int w, int h) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_framing(source, mode, x, y, w, h, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_mask_refine(bsb_ctx* ctx, int sigma) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_mask_refine(sigma, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_mask_refine(bsb_ctx* ctx, int source, int sigma) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_mask_refine(source, sigma, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_blur_mode(bsb_ctx* ctx, int mode) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_blur_mode(mode, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_blur_mode(bsb_ctx* ctx, int source, int mode) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_blur_mode(source, mode, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_get_framing(bsb_ctx* ctx, int frame, int rect[4]) {
  if (!check_ctx(ctx)) return 0;
  if (!rect) { report(&ctx->cb, "error: rect is null"); return 0; }
  std::string err;
  if (!ctx->eng->get_framing(frame, rect, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_out_format(bsb_ctx* ctx, int format) {
  if (!check_ctx(ctx)) return 0;
  if (format != BSB_OUT_BGR && format != BSB_OUT_BGRA) { report(&ctx->cb, "error: output format must be BSB_OUT_BGR (0) or BSB_OUT_BGRA (1)"); return 0; }
  ctx->eng->set_out_bgra(format == BSB_OUT_BGRA);
  return 1;
}

int bsb_set_live_background(bsb_ctx* ctx, const uint8_t* d_frames, int fmt, int bg_w, int bg_h, size_t pitch, size_t uv_offset,
                            size_t frame_stride) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_live_background(d_frames, fmt, bg_w, bg_h, pitch, uv_offset, frame_stride, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_live_background(bsb_ctx* ctx, int source, const uint8_t* d_frame, int fmt, int bg_w, int bg_h, size_t pitch,
                                   size_t uv_offset) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_live_background(source, d_frame, fmt, bg_w, bg_h, pitch, uv_offset, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_output_size(bsb_ctx* ctx, int* out_w, int* out_h) {
  if (!check_ctx(ctx)) return 0;
  if (out_w) *out_w = ctx->eng->out_w();
  if (out_h) *out_h = ctx->eng->out_h();
  return 1;
}

int bsb_get_background(bsb_ctx* ctx, uint8_t* out, size_t out_pitch) {
  if (!check_ctx(ctx)) return 0;
  const bsb::Callbacks* cbp = &ctx->cb;
  Engine* e = ctx->eng;
  if (!out || out_pitch < (size_t)e->W() * 3) { report(cbp, "error: invalid output buffer"); return 0; }
  API_CUDA(cudaSetDevice(e->device()));
  API_CUDA(cudaStreamSynchronize(e->stream()));
  const size_t row = (size_t)e->W() * 3;
  for (int y = 0; y < e->H(); ++y) API_CUDA(cudaMemcpy(out + (size_t)y * out_pitch, e->d_bg() + (size_t)y * row, row, cudaMemcpyDeviceToHost));
  return 1;
}

int bsb_composite(bsb_ctx* ctx, int n_frames, const uint8_t* frames, size_t frame_pitch, size_t frame_stride,
                  uint8_t* out, size_t out_pitch, size_t out_stride, uint8_t* out_yuyv, size_t yuyv_stride,
                  uint8_t* out_mask, size_t mask_stride) {
  return host_call(ctx, {n_frames, bsb::IN_BGR, frames, frame_pitch, 0, frame_stride, nullptr, out, out_stride, out_yuyv, yuyv_stride, out_mask,
                         mask_stride}, kProcessErr, &out_pitch);
}

int bsb_composite_device(bsb_ctx* ctx, int n_frames, const uint8_t* d_frames, size_t frame_stride, uint8_t* d_out, size_t out_stride,
                         uint8_t* d_yuyv, size_t yuyv_stride, uint8_t* d_mask, size_t mask_stride, int sync) {
  return device_call(ctx, {n_frames, bsb::IN_BGR, d_frames, 0, 0, frame_stride, nullptr, d_out, out_stride, d_yuyv, yuyv_stride, d_mask, mask_stride},
                     sync);
}

int bsb_composite_yuyv(bsb_ctx* ctx, int n_frames, const uint8_t* yuyv_frames, size_t in_stride, uint8_t* out, size_t out_stride,
                       uint8_t* out_yuyv, size_t yuyv_stride, uint8_t* out_mask, size_t mask_stride) {
  return host_call(ctx, {n_frames, bsb::IN_YUYV, yuyv_frames, 0, 0, in_stride, nullptr, out, out_stride, out_yuyv, yuyv_stride, out_mask, mask_stride},
                   kProcessErr);
}

int bsb_decode_mjpg(bsb_ctx* ctx, const uint8_t* jpeg, size_t jpeg_size, uint8_t* bgr_out) {
  if (!check_ctx(ctx)) return 0;
  const bsb::Callbacks* cbp = &ctx->cb;
#ifdef BSB_EMU
  (void)jpeg; (void)jpeg_size; (void)bgr_out;
  report(cbp, "error: MJPG ingest needs a GPU (NVJPG)"); return 0;
#else
  Engine* e = ctx->eng;
  if (!bgr_out) { report(cbp, "error: null buffer"); return 0; }
  API_CUDA(cudaSetDevice(e->device()));
  const std::string err = jpeg_decode(ctx, jpeg, jpeg_size, e->d_frames());
  if (!err.empty()) { report(cbp, "error: " + err); return 0; }
  API_CUDA(cudaMemcpyAsync(bgr_out, e->d_frames(), (size_t)e->W() * e->H() * 3, cudaMemcpyDeviceToHost, e->stream()));
  API_CUDA(cudaStreamSynchronize(e->stream()));
  return 1;
#endif
}

int bsb_composite_mjpg(bsb_ctx* ctx, int n_frames, const uint8_t* const* jpegs, const size_t* jpeg_sizes, uint8_t* out, size_t out_stride,
                       uint8_t* out_yuyv, size_t yuyv_stride, uint8_t* out_mask, size_t mask_stride) {
#ifdef BSB_EMU
  if (!check_ctx(ctx)) return 0;
  (void)n_frames; (void)jpegs; (void)jpeg_sizes; (void)out; (void)out_stride; (void)out_yuyv; (void)yuyv_stride; (void)out_mask; (void)mask_stride;
  report(&ctx->cb, "error: MJPG ingest needs a GPU (NVJPG)"); return 0;
#else
  return host_call(ctx, {n_frames, bsb::IN_BGR, nullptr, 0, 0, 0, nullptr, out, out_stride, out_yuyv, yuyv_stride, out_mask, mask_stride},
                   kProcessErr, nullptr, jpegs, jpeg_sizes);
#endif
}

int bsb_composite_yuyv_device(bsb_ctx* ctx, int n_frames, const uint8_t* d_yuyv_frames, uint8_t* d_out, size_t out_stride,
                              uint8_t* d_yuyv, size_t yuyv_stride, uint8_t* d_mask, size_t mask_stride, int sync) {
  return device_call(ctx, {n_frames, bsb::IN_YUYV, d_yuyv_frames, 0, 0, 0, nullptr, d_out, out_stride, d_yuyv, yuyv_stride, d_mask, mask_stride},
                     sync);
}

// ---- NV12 camera frames in, NV12 composites out ------------------------------------
int bsb_composite_nv12(bsb_ctx* ctx, int n_frames, const uint8_t* nv12, size_t in_stride, uint8_t* out, size_t out_stride,
                       uint8_t* nv12_out, size_t nv12_stride, uint8_t* out_mask, size_t mask_stride) {
  return host_call(ctx, {n_frames, bsb::IN_NV12, nv12, 0, 0, in_stride, nullptr, out, out_stride, nv12_out, nv12_stride, out_mask, mask_stride},
                   kProcessErr);
}

int bsb_composite_nv12_device(bsb_ctx* ctx, int n_frames, const uint8_t* d_nv12, size_t in_pitch, size_t uv_offset, size_t in_stride,
                              uint8_t* d_out, size_t out_stride, uint8_t* d_nv12_out, size_t nv12_stride, uint8_t* d_mask, size_t mask_stride,
                              int sync) {
  return device_call(ctx, {n_frames, bsb::IN_NV12, d_nv12, in_pitch, uv_offset, in_stride, nullptr, d_out, out_stride, d_nv12_out, nv12_stride,
                           d_mask, mask_stride}, sync);
}

// ---- independent sources ---------------------------------------------------------
int bsb_set_sources(bsb_ctx* ctx, int n_sources) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_sources(n_sources, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_reset_source(bsb_ctx* ctx, int source) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->reset_source(source, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_background(bsb_ctx* ctx, int source, const uint8_t* bg_raw, int w, int h, size_t pitch) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_background(source, bg_raw, w, h, pitch, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_background_ring(bsb_ctx* ctx, int source, const uint8_t* frames, int count, int bg_w, int bg_h, size_t bg_pitch,
                                   size_t frame_stride, int advance) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!frames) { report(&ctx->cb, "error: invalid background (null frames; bsb_set_source_background(NULL) clears a source's background)"); return 0; }
  if (!ctx->eng->set_source_ring(source, frames, count, bg_w, bg_h, bg_pitch, frame_stride, advance, &err)) {
    report(&ctx->cb, "error: " + err);
    return 0;
  }
  return 1;
}

int bsb_set_source_background_cursor(bsb_ctx* ctx, int source, int index) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_cursor(source, index, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_effect(bsb_ctx* ctx, int source, int background, int bgblur) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_effect(source, background, bgblur, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_flip(bsb_ctx* ctx, int source, int flip) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_flip(source, flip, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_filter(bsb_ctx* ctx, int source, int active) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_filter(source, active, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_set_source_output(bsb_ctx* ctx, int source, int out_w, int out_h) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->set_source_output(source, out_w, out_h, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_source_output_size(bsb_ctx* ctx, int source, int* out_w, int* out_h) {
  if (!check_ctx(ctx)) return 0;
  int w = 0, h = 0;
  if (!ctx->eng->n_sources()) { report(&ctx->cb, "error: no sources: call bsb_set_sources first"); return 0; }
  if (!ctx->eng->source_output_size(source, &w, &h)) { report(&ctx->cb, "error: source id out of range"); return 0; }
  if (out_w) *out_w = w;
  if (out_h) *out_h = h;
  return 1;
}

int bsb_composite_sources(bsb_ctx* ctx, int n, const int* source_ids, const uint8_t* frames, size_t frame_pitch, size_t frame_stride,
                          uint8_t* out, size_t out_stride, uint8_t* out_yuyv, size_t yuyv_stride, uint8_t* out_mask, size_t mask_stride) {
  if (null_ids(ctx, source_ids)) return 0;
  return host_call(ctx, {n, bsb::IN_BGR, frames, frame_pitch, 0, frame_stride, source_ids, out, out_stride, out_yuyv, yuyv_stride, out_mask, mask_stride},
                   "");
}

int bsb_composite_sources_yuyv_device(bsb_ctx* ctx, int n, const int* source_ids, const uint8_t* d_yuyv_frames, uint8_t* d_out, size_t out_stride,
                                      uint8_t* d_yuyv, size_t yuyv_stride, uint8_t* d_mask, size_t mask_stride, int sync) {
  if (null_ids(ctx, source_ids)) return 0;
  return device_call(ctx, {n, bsb::IN_YUYV, d_yuyv_frames, 0, 0, 0, source_ids, d_out, out_stride, d_yuyv, yuyv_stride, d_mask, mask_stride}, sync);
}

int bsb_composite_sources_nv12_device(bsb_ctx* ctx, int n_frames, const int* source_ids, const uint8_t* d_nv12, size_t in_pitch,
                                      size_t uv_offset, size_t in_stride, uint8_t* d_out, size_t out_stride, uint8_t* d_nv12_out,
                                      size_t nv12_stride, uint8_t* d_mask, size_t mask_stride, int sync) {
  if (null_ids(ctx, source_ids)) return 0;
  return device_call(ctx, {n_frames, bsb::IN_NV12, d_nv12, in_pitch, uv_offset, in_stride, source_ids, d_out, out_stride, d_nv12_out, nv12_stride,
                           d_mask, mask_stride}, sync);
}

int bsb_synchronize(bsb_ctx* ctx) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->sync(&err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

void* bsb_stream(bsb_ctx* ctx) { return check_ctx(ctx) ? (void*)ctx->eng->stream() : nullptr; }

// ---- stand-alone stages -------------------------------------------------------
namespace {
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  bool alloc(size_t n) { return cudaMalloc(&p, n ? n : 1) == cudaSuccess; }
  uint8_t* u8() const { return static_cast<uint8_t*>(p); }
};
bool stage_begin(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { g_last_error = "no CUDA device available (this library has no CPU path)"; return false; }
  if (device < 0 || device >= n || cudaSetDevice(device) != cudaSuccess) { g_last_error = "invalid CUDA device"; return false; }
  return true;
}
// the helpers run on the legacy default stream; a device-wide synchronise would break another thread's graph capture
bool stage_end() {
  cudaError_t e = cudaStreamSynchronize(0);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { g_last_error = std::string("CUDA error: ") + cudaGetErrorString(e); return false; }
  return true;
}
}  // namespace

int bsb_alpha_blend(int device, const uint8_t* srca, const uint8_t* srcb, const uint8_t* mask, uint8_t* out, size_t npix) {
  if (!srca || !srcb || !mask || !out) { g_last_error = "null buffer"; return 0; }
  if (!stage_begin(device)) return 0;
  DevBuf a, b, m, o;
  if (!a.alloc(npix * 3) || !b.alloc(npix * 3) || !m.alloc(npix) || !o.alloc(npix * 3)) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, srca, npix * 3, cudaMemcpyHostToDevice); cudaMemcpy(b.p, srcb, npix * 3, cudaMemcpyHostToDevice);
  cudaMemcpy(m.p, mask, npix, cudaMemcpyHostToDevice);
  if (npix) bsb::launch_alpha_blend(nullptr, a.u8(), b.u8(), m.u8(), o.u8(), npix);
  if (!stage_end()) return 0;
  cudaMemcpy(out, o.p, npix * 3, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_convert_rgb_to_yuyv(int device, const uint8_t* rgb, uint8_t* yuyv, int width, int height) {
  if (!rgb || !yuyv || width < 0 || height < 0) { g_last_error = "invalid argument"; return 0; }
  const size_t npix = (size_t)width * height;
  if (npix & 1) { g_last_error = "YUYV needs an even number of pixels"; return 0; }
  if (!stage_begin(device)) return 0;
  DevBuf a, o;
  if (!a.alloc(npix * 3) || !o.alloc(npix * 2)) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, rgb, npix * 3, cudaMemcpyHostToDevice);
  if (npix) bsb::launch_rgb_to_yuyv(nullptr, a.u8(), o.u8(), npix);
  if (!stage_end()) return 0;
  cudaMemcpy(yuyv, o.p, npix * 2, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_convert_yuyv_to_bgr(int device, const uint8_t* yuyv, uint8_t* bgr, int width, int height) {
  if (!yuyv || !bgr || width < 0 || height < 0) { g_last_error = "invalid argument"; return 0; }
  const size_t npix = (size_t)width * height;
  if (npix & 1) { g_last_error = "YUYV needs an even number of pixels"; return 0; }
  if (!stage_begin(device)) return 0;
  DevBuf a, o;
  if (!a.alloc(npix * 2) || !o.alloc(npix * 3)) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, yuyv, npix * 2, cudaMemcpyHostToDevice);
  if (npix) bsb::launch_yuyv_to_bgr(nullptr, a.u8(), o.u8(), npix);
  if (!stage_end()) return 0;
  cudaMemcpy(bgr, o.p, npix * 3, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_convert_nv12_to_bgr(int device, const uint8_t* nv12, uint8_t* bgr, int width, int height) {
  if (!nv12 || !bgr || width < 0 || height < 0) { g_last_error = "invalid argument"; return 0; }
  if ((width | height) & 1) { g_last_error = "NV12 needs an even width and height"; return 0; }
  const size_t npix = (size_t)width * height;
  if (!stage_begin(device)) return 0;
  DevBuf a, o;
  if (!a.alloc(npix * 3 / 2) || !o.alloc(npix * 3)) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, nv12, npix * 3 / 2, cudaMemcpyHostToDevice);
  if (npix) bsb::launch_nv12_to_bgr(nullptr, 1, a.u8(), (size_t)width, npix, npix * 3 / 2, o.u8(), width, height);
  if (!stage_end()) return 0;
  cudaMemcpy(bgr, o.p, npix * 3, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_gaussian_taps(int ksize, int* taps) {
  bsb::GaussTaps t{};
  if (!taps || !bsb::gauss_taps(ksize, &t)) { g_last_error = "strength value must be odd (1..255)"; return 0; }
  for (int i = 0; i < ksize; ++i) taps[i] = t.q[i];
  return 1;
}

int bsb_mask_refine_weights(int sigma, int* w) {
  if (!w || !bsb::refine_weights(sigma, w)) { g_last_error = "mask refinement strength must be 1..255 (and w non-null)"; return 0; }
  return 1;
}

int bsb_gaussian_blur(int device, const uint8_t* src, uint8_t* dst, int width, int height, int ksize) {
  bsb::GaussTaps t{};
  if (!src || !dst || width <= 0 || height <= 0) { g_last_error = "invalid argument"; return 0; }
  if (!bsb::gauss_taps(ksize, &t)) { g_last_error = "strength value must be odd (1..255)"; return 0; }
  if (!stage_begin(device)) return 0;
  const size_t nb = (size_t)width * height * 3;
  DevBuf a, o, tmp;
  if (!a.alloc(nb) || !o.alloc(nb) || !tmp.alloc(nb * 2)) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, src, nb, cudaMemcpyHostToDevice);
  if (!bsb::launch_gauss_blur(nullptr, 1, a.u8(), (size_t)width * 3, nb, static_cast<uint16_t*>(tmp.p), o.u8(), (size_t)width * 3, nb, width,
                              height, t)) {
    g_last_error = "could not allocate the Gaussian tap tables";
    return 0;
  }
  if (!stage_end()) return 0;
  cudaMemcpy(dst, o.p, nb, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_masked_gaussian_blur(int device, const uint8_t* src, const uint8_t* mask, uint8_t* dst, int width, int height, int ksize) {
  if (!src || !mask || !dst || width <= 0 || height <= 0) { g_last_error = "invalid argument"; return 0; }
  if (ksize < 1 || !(ksize & 1) || ksize > 255) { g_last_error = "strength value must be odd (1..255)"; return 0; }
  if (!stage_begin(device)) return 0;
  const size_t npix = (size_t)width * height, nb = npix * 3;
  DevBuf a, m, o, tmp;
  if (!a.alloc(nb) || !m.alloc(npix) || !o.alloc(nb) || !tmp.alloc(npix * sizeof(uint4))) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, src, nb, cudaMemcpyHostToDevice);
  cudaMemcpy(m.p, mask, npix, cudaMemcpyHostToDevice);
  if (!bsb::launch_masked_gauss(nullptr, 1, a.u8(), (size_t)width * 3, nb, m.u8(), npix, nullptr, ksize, (unsigned)bsb::gauss_class(ksize),
                                static_cast<uint4*>(tmp.p), o.u8(), (size_t)width * 3, nb, width, height)) {
    g_last_error = "could not allocate the Gaussian tap tables";
    return 0;
  }
  if (!stage_end()) return 0;
  cudaMemcpy(dst, o.p, nb, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_flip(int device, const uint8_t* src, uint8_t* dst, int width, int height, int flip_h, int flip_v) {
  if (!src || !dst || width <= 0 || height <= 0) { g_last_error = "invalid argument"; return 0; }
  if (!stage_begin(device)) return 0;
  const size_t nb = (size_t)width * height * 3;
  DevBuf a, o;
  if (!a.alloc(nb) || !o.alloc(nb)) { g_last_error = "cudaMalloc failed"; return 0; }
  cudaMemcpy(a.p, src, nb, cudaMemcpyHostToDevice);
  bsb::launch_flip_u8c3(nullptr, 1, a.u8(), nb, o.u8(), nb, width, height, flip_h != 0, flip_v != 0);
  if (!stage_end()) return 0;
  cudaMemcpy(dst, o.p, nb, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_resize_u8c3(int device, const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh) {
  if (!src || !dst || sw <= 0 || sh <= 0 || dw <= 0 || dh <= 0) { g_last_error = "invalid argument"; return 0; }
  if (!stage_begin(device)) return 0;
  const bsb::HostResizeTab h = bsb::build_resize_tab(sw, sh, dw, dh);
  DevBuf a, o, t0, t1, t2, t3, t4;
  const size_t sb = (size_t)sw * sh * 3, db = (size_t)dw * dh * 3;
  if (!a.alloc(sb) || !o.alloc(db) || !t0.alloc(dw * 4) || !t1.alloc(dw * 4) || !t2.alloc(dh * 4) || !t3.alloc(dh * 4) || !t4.alloc(dh * 4)) {
    g_last_error = "cudaMalloc failed"; return 0;
  }
  cudaMemcpy(a.p, src, sb, cudaMemcpyHostToDevice);
  cudaMemcpy(t0.p, h.xofs.data(), (size_t)dw * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(t1.p, h.xw.data(), (size_t)dw * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(t2.p, h.yofs0.data(), (size_t)dh * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(t3.p, h.yofs1.data(), (size_t)dh * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(t4.p, h.yw.data(), (size_t)dh * 4, cudaMemcpyHostToDevice);
  bsb::ResizeTab tab{(const int*)t0.p, (const short*)t1.p, (const int*)t2.p, (const int*)t3.p, (const short*)t4.p, nullptr};
  bsb::launch_resize_u8c3(nullptr, a.u8(), sw, sh, (size_t)sw * 3, o.u8(), dw, dh, (size_t)dw * 3, tab, h.area2x2);
  if (!stage_end()) return 0;
  cudaMemcpy(dst, o.p, db, cudaMemcpyDeviceToHost);
  return 1;
}

int bsb_pointwise(int device, int variant, int M, int K, int N, const float* A, const float* W, const float* bias, int act, float* out) {
  if (M <= 0 || K <= 0 || N <= 0) { g_last_error = "invalid argument"; return 0; }
  return bsb_pointwise_ex(device, variant, M, K, N, A, (long)M * K, 0, K, W, bias, nullptr, 0, 0, 0, act, 0, 0, out, (long)M * N, 0, N);
}

int bsb_pointwise_ex(int device, int variant, int M, int K, int N, const float* A, long a_len, long a_off, int ld_a,
                     const float* W, const float* bias, const float* res, long res_len, long res_off, int ld_res,
                     int act1, int act2, int act3, float* out, long out_len, long out_off, int ld_out) {
  if (!A || !W || !out || M <= 0 || K <= 0 || N <= 0) { g_last_error = "invalid argument"; return 0; }
  // every element the kernel may touch lies inside its buffer
  auto spans = [](long len, long off, int ld, int rows, int cols) { return off >= 0 && ld >= cols && off + (long)(rows - 1) * ld + cols <= len; };
  if (!spans(a_len, a_off, ld_a, M, K) || !spans(out_len, out_off, ld_out, M, N) || (res && !spans(res_len, res_off, ld_res, M, N))) {
    g_last_error = "sub-matrix outside its buffer"; return 0;
  }
  const bool use_tc = variant == 1;
  if (!use_tc && (a_off % 4 || out_off % 4)) { g_last_error = "the exact kernels need A and out on 16-byte boundaries"; return 0; }
  if (!stage_begin(device)) return 0;
  DevBuf dA, dW, dW2, dB, dO, dR;
  if (!dA.alloc((size_t)a_len * 4) || !dO.alloc((size_t)out_len * 4) || (bias && !dB.alloc((size_t)N * 4)) || (res && !dR.alloc((size_t)res_len * 4))) {
    g_last_error = "cudaMalloc failed"; return 0;
  }
  cudaMemcpy(dA.p, A, (size_t)a_len * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dO.p, out, (size_t)out_len * 4, cudaMemcpyHostToDevice);
  if (bias) cudaMemcpy(dB.p, bias, (size_t)N * 4, cudaMemcpyHostToDevice);
  if (res) cudaMemcpy(dR.p, res, (size_t)res_len * 4, cudaMemcpyHostToDevice);
  const float* dAm = (const float*)dA.p + a_off;
  float* dOm = (float*)dO.p + out_off;
  bsb::Epilogue e; e.bias = bias ? (const float*)dB.p : nullptr; e.act1 = act1; e.act2 = act2; e.act3 = act3;
  if (res) { e.residual = (const float*)dR.p + res_off; e.ld_res = ld_res; }
  if (use_tc) {
    const int kpad = (K + 31) / 32 * 32;
    if (const char* why = bsb::pointwise_tc_refusal(K, dAm, ld_a, kpad, dOm, ld_out, e)) {
      g_last_error = std::string("the tensor-core kernel refuses this call: ") + why; return 0;
    }
    const int bn = bsb::pointwise_tc_tile_n(N);
    if (bn <= 0) { g_last_error = "shape not supported by the tensor-core kernel"; return 0; }
    const int npad = (N + bn - 1) / bn * bn;
    std::vector<float> hi((size_t)npad * kpad, 0.f), lo((size_t)npad * kpad, 0.f);
    for (int n = 0; n < N; ++n) for (int k = 0; k < K; ++k) {
      const float v = W[(size_t)n * K + k];
      uint32_t bits; std::memcpy(&bits, &v, 4); bits &= 0xffffe000u;
      float h; std::memcpy(&h, &bits, 4);
      hi[(size_t)n * kpad + k] = h; lo[(size_t)n * kpad + k] = v - h;
    }
    if (!dW.alloc(hi.size() * 4) || !dW2.alloc(lo.size() * 4)) { g_last_error = "cudaMalloc failed"; return 0; }
    cudaMemcpy(dW.p, hi.data(), hi.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dW2.p, lo.data(), lo.size() * 4, cudaMemcpyHostToDevice);
    if (!bsb::launch_pointwise_tc(nullptr, M, K, N, dAm, ld_a, (const float*)dW.p, (const float*)dW2.p, kpad, npad, dOm, ld_out, e)) {
      g_last_error = "tensor-core launch rejected the shape or alignment"; return 0;
    }
  } else {
    const int n4 = (N + 3) / 4 * 4;
    std::vector<float> wt((size_t)K * n4, 0.f);
    for (int n = 0; n < N; ++n) for (int k = 0; k < K; ++k) wt[(size_t)k * n4 + n] = W[(size_t)n * K + k];
    if (!dW.alloc(wt.size() * 4)) { g_last_error = "cudaMalloc failed"; return 0; }
    cudaMemcpy(dW.p, wt.data(), wt.size() * 4, cudaMemcpyHostToDevice);
    const int saved = bsb::pointwise_variant();
    bsb::set_pointwise_variant(variant);
    bsb::launch_pointwise(nullptr, M, K, N, dAm, ld_a, (const float*)dW.p, n4, dOm, ld_out, e, nullptr, 1, nullptr, 0);
    bsb::set_pointwise_variant(saved);
  }
  if (!stage_end()) return 0;
  cudaMemcpy(out, dO.p, (size_t)out_len * 4, cudaMemcpyDeviceToHost);
  return 1;
}

double bsb_time_pointwise(int device, int variant, int M, int K, int N, int iters) {
  if (M <= 0 || K <= 0 || N <= 0 || iters < 1) { g_last_error = "invalid argument"; return -1.0; }
  if (!stage_begin(device)) return -1.0;
  const int n4 = (N + 3) / 4 * 4;
  const bool use_tc = variant == 1;
  const int bn = use_tc ? bsb::pointwise_tc_tile_n(N) : 0;
  if (use_tc && (bn <= 0 || K % 4)) { g_last_error = "shape not supported by the tensor-core kernel"; return -1.0; }
  const int kpad = (K + 31) / 32 * 32, npad = use_tc ? (N + bn - 1) / bn * bn : 0;
  DevBuf dA, dW, dW2, dB, dO;
  const size_t wbytes = use_tc ? (size_t)npad * kpad * 4 : (size_t)K * n4 * 4;
  if (!dA.alloc((size_t)M * K * 4) || !dO.alloc((size_t)M * N * 4) || !dW.alloc(wbytes) || !dW2.alloc(wbytes) || !dB.alloc((size_t)N * 4)) { g_last_error = "cudaMalloc failed"; return -1.0; }
  cudaMemset(dA.p, 0, (size_t)M * K * 4); cudaMemset(dW.p, 0, wbytes); cudaMemset(dW2.p, 0, wbytes); cudaMemset(dB.p, 0, (size_t)N * 4);
  bsb::Epilogue e; e.bias = (const float*)dB.p; e.act1 = 3;
  const int saved = bsb::pointwise_variant();
  if (!use_tc) bsb::set_pointwise_variant(variant);
  bool ok = true;
  auto once = [&]() {
    if (use_tc) ok = ok && bsb::launch_pointwise_tc(nullptr, M, K, N, (const float*)dA.p, K, (const float*)dW.p, (const float*)dW2.p, kpad, npad, (float*)dO.p, N, e);
    else bsb::launch_pointwise(nullptr, M, K, N, (const float*)dA.p, K, (const float*)dW.p, n4, (float*)dO.p, N, e, nullptr, 1, nullptr, 0);
  };
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 2; ++i) once();
  cudaEventRecord(e0, nullptr);
  for (int i = 0; i < iters; ++i) once();
  cudaEventRecord(e1, nullptr);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  bsb::set_pointwise_variant(saved);
  if (!ok) { g_last_error = "tensor-core launch rejected the shape"; return -1.0; }
  if (!stage_end()) return -1.0;
  return (double)ms / iters;
}

// ---- introspection ----------------------------------------------------------------
int bsb_frame_size(bsb_ctx* ctx, int* width, int* height) {
  if (!check_ctx(ctx)) return 0;
  if (width) *width = ctx->eng->W();
  if (height) *height = ctx->eng->H();
  return 1;
}

int bsb_geometry(bsb_ctx* ctx, int roidim[4], int in_roidim[4], int out_roidim[4], int in_hwc[3], int out_hwc[3]) {
  if (!check_ctx(ctx)) return 0;
  Engine* e = ctx->eng;
  if (roidim) std::memcpy(roidim, e->roidim(), 16);
  if (in_roidim) std::memcpy(in_roidim, e->in_roidim(), 16);
  if (out_roidim) std::memcpy(out_roidim, e->out_roidim(), 16);
  if (in_hwc) e->in_hwc(in_hwc);
  if (out_hwc) e->out_hwc(out_hwc);
  return 1;
}

int bsb_infer(bsb_ctx* ctx, int n_frames, const float* input, float* output) {
  if (!check_ctx(ctx)) return 0;
  if (!input || !output) { report(&ctx->cb, "error: null buffer"); return 0; }
  std::string err;
  if (!ctx->eng->infer(n_frames, input, output, &err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

long bsb_get_tensor(bsb_ctx* ctx, int tensor_index, float* out, long capacity) {
  return bsb_get_tensor_frame(ctx, tensor_index, 0, out, capacity);
}

long bsb_get_tensor_frame(bsb_ctx* ctx, int tensor_index, int frame, float* out, long capacity) {
  if (!check_ctx(ctx)) return -1;
  std::string err;
  long n = ctx->eng->get_tensor(tensor_index, frame, out, capacity, &err);
  if (n < 0) report(&ctx->cb, "error: " + err);
  return n;
}

int bsb_tc_steps(bsb_ctx* ctx, int* rows, int capacity) {
  if (!check_ctx(ctx)) return -1;
  return ctx->eng->tc_steps(rows, capacity);
}

long bsb_get_stage_u8(bsb_ctx* ctx, int which, int frame, uint8_t* out, long capacity) {
  if (!check_ctx(ctx)) return -1;
  std::string err;
  long n = ctx->eng->get_stage_u8(which, frame, out, capacity, &err);
  if (n < 0) report(&ctx->cb, "error: " + err);
  return n;
}

long bsb_test_feed_shape(bsb_ctx* ctx, int stage, int hwc[3]) {
  if (!check_ctx(ctx)) return -1;
  int h = 0, w = 0, c = 0;
  if (!ctx->eng->feed_shape(stage, &h, &w, &c)) { report(&ctx->cb, "error: unknown feed stage"); return -1; }
  if (hwc) { hwc[0] = h; hwc[1] = w; hwc[2] = c; }
  return (long)h * w * c * (stage == BSB_FEED_LOGITS ? (long)sizeof(float) : 1L);
}

int bsb_test_feed(bsb_ctx* ctx, int stage, int n_frames, const void* data, size_t bytes) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->arm_feed(stage, n_frames, data, bytes, &err)) { report(&ctx->cb, "error: bsb_test_feed: " + err); return 0; }
  return 1;
}

int bsb_reset_state(bsb_ctx* ctx) {
  if (!check_ctx(ctx)) return 0;
  std::string err;
  if (!ctx->eng->reset_state(&err)) { report(&ctx->cb, "error: " + err); return 0; }
  return 1;
}

int bsb_launches_per_call(bsb_ctx* ctx, int n_frames) {
  (void)n_frames;
  return check_ctx(ctx) ? ctx->eng->launches_per_call() : 0;
}

double bsb_time_stage(bsb_ctx* ctx, int stage, int n_frames, int iters) {
  if (!check_ctx(ctx)) return -1.0;
  std::string err;
  double ms = ctx->eng->time_stage(stage, n_frames, iters, &err);
  if (ms < 0) report(&ctx->cb, "error: " + err);
  return ms;
}

long bsb_total_launches(void) { return bsb::launch_count(); }

double bsb_model_flops(bsb_ctx* ctx) { return check_ctx(ctx) ? ctx->eng->flops() : 0.0; }

int bsb_uses_tensor_cores(bsb_ctx* ctx) { return check_ctx(ctx) && ctx->eng->uses_tensor_cores() ? 1 : 0; }

int bsb_yuyv_native(bsb_ctx* ctx) { return check_ctx(ctx) && ctx->eng->last_native() ? 1 : 0; }

int bsb_set_tuning(const char* name, int value) {
  if (!name) { g_last_error = "null tuning name"; return 0; }
  bsb::Tuning& t = bsb::tuning();
  const std::string n(name);
  if (n == "pw_variant") t.pw_variant = value;
  else if (n == "dw_plane") t.dw_plane = value;
  else if (n == "dec_up") t.dec_up = value;
  else if (n == "dec_par") t.dec_par = value;
  else if (n == "stem_x2") t.stem_x2 = value;
  else if (n == "pw_dws2") t.pw_dws2 = value;
  else if (n == "dw_plane_cs") t.dw_plane_cs = value;
  else if (n == "up_staged") t.up_staged = value;
  else if (n == "e2e_chunk") t.e2e_chunk = value;
  else if (n == "epi_static") t.epi_static = value;
  else if (n == "dw_px") t.dw_px = value;
  else if (n == "post_tma") t.post_tma = value;
  else if (n == "cnn_chain") t.cnn_chain = value;
  else if (n == "pool_merge") t.pool_merge = value;
  else if (n == "stem_pw") t.stem_pw = value;
  else if (n == "up_pw") t.up_pw = value;
  else if (n == "head") t.head = value;
  else if (n == "tc_variant") t.tc_variant = value;
  else if (n == "tc_mask_hi") t.tc_mask_hi = value;
  else if (n == "tc_min_k") t.tc_min_k = value;
  else if (n == "post_tile") t.post_tile = value;
  else if (n == "sub_batch_mb") t.sub_batch_mb = value;
  else if (n == "post_l1") t.post_l1 = value;
  else { g_last_error = "unknown tuning switch '" + n + "'"; return 0; }
  return 1;
}

}  // extern "C"
