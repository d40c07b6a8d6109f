// backscrub_b200/csrc/kernels_img.cu — integer image stages of the hot path (sm_90a).
//
// Replaces the OpenCV calls of lib/libbackscrub.cc:285-302 (ROI resize, BGR2RGB,
// bilateralFilter, convertTo), :314-361 (decision + IIR), :366-371 (mask upsample + 5x5
// blur) and app/deepseg.cc:108-134 (alpha_blend), :87-106 (convert_rgb_to_yuyv),
// app/background.cc:178-194 (background resize).  All integer arithmetic is OpenCV's
// fixed-point arithmetic restated (see oracle/oracle_img.c for the formulas and their
// cv2 pins); results are bit-exact against the oracle.
#include "kernels.h"
#include "post_math.h"
#include "resize_taps.h"

#include <cmath>
#include <map>
#include <mutex>
#include <vector>

namespace bsb {

void count_launch();

// cv::resize INTER_LINEAR 8-bit, one output sample: horizontal taps at scale 2^11, vertical
// descale ((b0*(H0>>4))>>16) + ((b1*(H1>>4))>>16) + 2) >> 2.
BSB_D int lin_h(const uint8_t* row, int sx, int sx1, int cn, int c, int a0, int a1) {
  return (int)row[sx * cn + c] * a0 + (int)row[sx1 * cn + c] * a1;
}
BSB_D uint8_t lin_v(int h0, int h1, int b0, int b1) {
  return bsb_sat_u8((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2);
}

// background of batch frame b: one static image (bg_stride 0), one image per frame, or a ring of
// bg_count images entered at the device-side cursor (animated backgrounds, app/background.cc:126-176), or the image a
// per-frame table names (independent sources)
BSB_D size_t bg_frame_offset(const PostArgs& a, int b) {
  if (a.bg_index) b = __ldg(a.bg_index + b);
  else if (a.bg_cursor) b = (int)(((unsigned)__ldg(a.bg_cursor) + (unsigned)b * (unsigned)a.bg_advance) % (unsigned)a.bg_count);
  return (size_t)b * a.bg_stride;
}

// ---------------------------------------------------------------------------
// ROI crop -> resize -> BGR2RGB into the zero-padded model-sized image.
// One thread = one destination pixel (3 channels).
// ---------------------------------------------------------------------------
// FMT (InFmt): IN_BGR frames; IN_YUYV: camera YUYV frames (W*2-byte rows); IN_NV12: camera NV12 frames (Y rows `pitch`
// bytes apart, the UV plane at byte `uv_off` of the frame).  Every tap of a camera frame is first converted the way
// cv::cvtColor(COLOR_YUV2BGR_YUYV / _NV12) would have (cv::VideoCapture's conversion, app/deepseg.cc:553), so the result
// equals converting the whole frame first — without materialising the BGR frame.
// GATHER (calls with held frames, bsb_set_mask_interval): output frame b is camera frame gather[b] of the call.
template <int FMT, bool GATHER>
__global__ void __launch_bounds__(256) k_resize_roi_swap(int B, const uint8_t* frames, size_t frame_stride, size_t pitch,
                                                         int roi_x, int roi_y, int roi_w, int roi_h, ResizeTab t,
                                                         uint8_t* in_u8, int mw, int mh, int in_x, int in_y, int in_w, int in_h,
                                                         bool area2x2, size_t uv_off, const int* gather) {
  const long total = (long)B * in_w * in_h;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int dx = (int)(idx % in_w), dy = (int)((idx / in_w) % in_h), b = (int)(idx / ((long)in_w * in_h));
  const int fb = GATHER ? __ldg(gather + b) : b;
  uint8_t px[3];
  if (FMT == IN_NV12) {
    const uint8_t* img = frames + (size_t)fb * frame_stride;
    int p00[3], p01[3], p10[3], p11[3];
    if (area2x2) {
      const int y0 = roi_y + 2 * dy, x0 = roi_x + 2 * dx;
      nv12_px_to_bgr(img, pitch, uv_off, x0, y0, p00); nv12_px_to_bgr(img, pitch, uv_off, x0 + 1, y0, p01);
      nv12_px_to_bgr(img, pitch, uv_off, x0, y0 + 1, p10); nv12_px_to_bgr(img, pitch, uv_off, x0 + 1, y0 + 1, p11);
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = (uint8_t)((p00[c] + p01[c] + p10[c] + p11[c] + 2) >> 2);
    } else {
      const int sx = __ldg(t.xofs + dx), sx1 = min(sx + 1, roi_w - 1);
      const int a0 = __ldg(t.xw + 2 * dx), a1 = __ldg(t.xw + 2 * dx + 1);
      const int b0 = __ldg(t.yw + 2 * dy), b1 = __ldg(t.yw + 2 * dy + 1);
      const int y0 = roi_y + __ldg(t.yofs0 + dy), y1 = roi_y + __ldg(t.yofs1 + dy);
      nv12_px_to_bgr(img, pitch, uv_off, roi_x + sx, y0, p00); nv12_px_to_bgr(img, pitch, uv_off, roi_x + sx1, y0, p01);
      nv12_px_to_bgr(img, pitch, uv_off, roi_x + sx, y1, p10); nv12_px_to_bgr(img, pitch, uv_off, roi_x + sx1, y1, p11);
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = lin_v(p00[c] * a0 + p01[c] * a1, p10[c] * a0 + p11[c] * a1, b0, b1);
    }
  } else if (FMT == IN_YUYV) {
    const uint8_t* img = frames + (size_t)fb * frame_stride;
    if (area2x2) {
      int p00[3], p01[3], p10[3], p11[3];
      const uint8_t* s0 = img + (size_t)(roi_y + 2 * dy) * pitch;
      const uint8_t* s1 = s0 + pitch;
      yuyv_px_to_bgr(s0, roi_x + 2 * dx, p00); yuyv_px_to_bgr(s0, roi_x + 2 * dx + 1, p01);
      yuyv_px_to_bgr(s1, roi_x + 2 * dx, p10); yuyv_px_to_bgr(s1, roi_x + 2 * dx + 1, p11);
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = (uint8_t)((p00[c] + p01[c] + p10[c] + p11[c] + 2) >> 2);
    } else {
      const int sx = __ldg(t.xofs + dx), sx1 = min(sx + 1, roi_w - 1);
      const int a0 = __ldg(t.xw + 2 * dx), a1 = __ldg(t.xw + 2 * dx + 1);
      const int b0 = __ldg(t.yw + 2 * dy), b1 = __ldg(t.yw + 2 * dy + 1);
      const uint8_t* r0 = img + (size_t)(roi_y + __ldg(t.yofs0 + dy)) * pitch;
      const uint8_t* r1 = img + (size_t)(roi_y + __ldg(t.yofs1 + dy)) * pitch;
      int p00[3], p01[3], p10[3], p11[3];
      yuyv_px_to_bgr(r0, roi_x + sx, p00); yuyv_px_to_bgr(r0, roi_x + sx1, p01);
      yuyv_px_to_bgr(r1, roi_x + sx, p10); yuyv_px_to_bgr(r1, roi_x + sx1, p11);
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = lin_v(p00[c] * a0 + p01[c] * a1, p10[c] * a0 + p11[c] * a1, b0, b1);
    }
  } else {
    const uint8_t* roi = frames + (size_t)fb * frame_stride + (size_t)roi_y * pitch + (size_t)roi_x * 3;
    if (area2x2) {
      const uint8_t* s0 = roi + (size_t)(2 * dy) * pitch + (size_t)(2 * dx) * 3;
      const uint8_t* s1 = s0 + pitch;
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = (uint8_t)((s0[c] + s0[3 + c] + s1[c] + s1[3 + c] + 2) >> 2);
    } else {
      const int sx = __ldg(t.xofs + dx), sx1 = min(sx + 1, roi_w - 1);
      const int a0 = __ldg(t.xw + 2 * dx), a1 = __ldg(t.xw + 2 * dx + 1);
      const int b0 = __ldg(t.yw + 2 * dy), b1 = __ldg(t.yw + 2 * dy + 1);
      const uint8_t* r0 = roi + (size_t)__ldg(t.yofs0 + dy) * pitch;
      const uint8_t* r1 = roi + (size_t)__ldg(t.yofs1 + dy) * pitch;
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = lin_v(lin_h(r0, sx, sx1, 3, c, a0, a1), lin_h(r1, sx, sx1, 3, c, a0, a1), b0, b1);
    }
  }
  uint8_t* d = in_u8 + ((size_t)b * mh * mw + (size_t)(in_y + dy) * mw + (in_x + dx)) * 3;
  d[0] = px[2]; d[1] = px[1]; d[2] = px[0];   // BGR -> RGB
}

void launch_resize_roi_swap(cudaStream_t s, int B, const uint8_t* frames, size_t frame_stride, size_t frame_pitch,
                            int roi_x, int roi_y, int roi_w, int roi_h, ResizeTab tab,
                            uint8_t* in_u8, int mw, int mh, int in_x, int in_y, int in_w, int in_h, bool area2x2, int in_fmt,
                            size_t uv_off, const int* gather) {
  const long total = (long)B * in_w * in_h;
  const dim3 grid((unsigned)((total + 255) / 256));
  auto k = k_resize_roi_swap<IN_BGR, false>;
  if (in_fmt == IN_NV12) k = gather ? k_resize_roi_swap<IN_NV12, true> : k_resize_roi_swap<IN_NV12, false>;
  else if (in_fmt == IN_YUYV) k = gather ? k_resize_roi_swap<IN_YUYV, true> : k_resize_roi_swap<IN_YUYV, false>;
  else if (gather) k = k_resize_roi_swap<IN_BGR, true>;
  BSB_LAUNCH(k, grid, dim3(256), 0, s, B, frames, frame_stride, frame_pitch, roi_x, roi_y, roi_w, roi_h, tab, in_u8, mw, mh, in_x, in_y,
             in_w, in_h, area2x2, uv_off, gather);
  count_launch();
}

// ---------------------------------------------------------------------------
// cv::bilateralFilter(d=5, sigma 100/100) + convertTo(CV_32F, scale, offset).
// 13 taps (i^2+j^2 <= 4) in raster order, weights = space_w[k] * color_w[|db|+|dg|+|dr|],
// per-tap fmaf accumulation, cvRound(sum * (1/wsum)), BORDER_REFLECT_101.
// One thread = one pixel.
// ---------------------------------------------------------------------------
// One block = a 32 x 8 pixel tile: the tile plus its 2-pixel REFLECT_101 border is staged once in shared memory as
// packed words (b | g << 8 | r << 16), so each tap costs one LDS instead of three byte loads and two reflections.
constexpr int BF_TW = 32, BF_TH = 8, BF_SW = BF_TW + 4, BF_SH = BF_TH + 4;

__global__ void __launch_bounds__(256) k_bilateral_norm(int B, const uint8_t* in_u8, int mw, int mh,
                                                        const float* color_w, const float* space_w,
                                                        float scale, float offset, float* out_f32, uint8_t* out_u8) {
  __shared__ float cw[768];
  __shared__ unsigned tile[BF_SH * BF_SW];
  __shared__ float sw[16];
  (void)B;
  const int tid = threadIdx.x;
  const int x0 = blockIdx.x * BF_TW, y0 = blockIdx.y * BF_TH, b = blockIdx.z;
  const uint8_t* img = in_u8 + (size_t)b * mh * mw * 3;
  for (int i = tid; i < 768; i += 256) cw[i] = __ldg(color_w + i);
  if (tid < 13) sw[tid] = __ldg(space_w + tid);
  for (int i = tid; i < BF_SH * BF_SW; i += 256) {
    const int ty = i / BF_SW, tx = i - ty * BF_SW;
    const uint8_t* p = img + ((size_t)bsb_reflect101(y0 + ty - 2, mh) * mw + bsb_reflect101(x0 + tx - 2, mw)) * 3;
    tile[i] = (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16);
  }
  __syncthreads();
  const int lx = tid & (BF_TW - 1), ly = tid >> 5;
  const int x = x0 + lx, y = y0 + ly;
  if (x >= mw || y >= mh) return;
  const unsigned* t0 = tile + (ly + 2) * BF_SW + lx + 2;
  const unsigned cc = t0[0];
  const int c0 = (int)(cc & 255u), c1 = (int)((cc >> 8) & 255u), c2 = (int)(cc >> 16);
  float wsum = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f;
  int k = 0;
#pragma unroll
  for (int i = -2; i <= 2; ++i) {
#pragma unroll
    for (int j = -2; j <= 2; ++j) {
      if (i * i + j * j > 4) continue;
      const unsigned v = t0[i * BF_SW + j];
      const int v0 = (int)(v & 255u), v1 = (int)((v >> 8) & 255u), v2 = (int)(v >> 16);
      const float w = sw[k] * cw[abs(v0 - c0) + abs(v1 - c1) + abs(v2 - c2)];
      ++k;
      wsum = wsum + w;
      s0 = fmaf((float)v0, w, s0);
      s1 = fmaf((float)v1, w, s1);
      s2 = fmaf((float)v2, w, s2);
    }
  }
  const size_t idx = ((size_t)b * mh + y) * mw + x;
  const float inv = bsb_div(1.f, wsum);
  const int r0 = bsb_sat_u8(__float2int_rn(s0 * inv)), r1 = bsb_sat_u8(__float2int_rn(s1 * inv)), r2 = bsb_sat_u8(__float2int_rn(s2 * inv));
  if (out_f32) {
    float* o = out_f32 + idx * 3;
    o[0] = fmaf((float)r0, scale, offset);
    o[1] = fmaf((float)r1, scale, offset);
    o[2] = fmaf((float)r2, scale, offset);
  }
  if (out_u8) { uint8_t* u = out_u8 + idx * 3; u[0] = (uint8_t)r0; u[1] = (uint8_t)r1; u[2] = (uint8_t)r2; }
}

void launch_bilateral_norm(cudaStream_t s, int B, const uint8_t* in_u8, int mw, int mh,
                           const float* color_w, const float* space_w, float scale, float offset,
                           float* out_f32, uint8_t* out_u8_dbg) {
  BSB_LAUNCH(k_bilateral_norm, dim3((unsigned)ceil_div(mw, BF_TW), (unsigned)ceil_div(mh, BF_TH), (unsigned)B), dim3(256), 0, s, B, in_u8, mw, mh,
             color_w, space_w, scale, offset, out_f32, out_u8_dbg);
  count_launch();
}

// ---------------------------------------------------------------------------
// Decision + temporal IIR, lib/libbackscrub.cc:314-361.  One thread = one model-output
// pixel, looping over the B consecutive frames of the batch so the 3-tap state
// out = (val & 0xE0) | (out >> 3) advances in frame order.
// ---------------------------------------------------------------------------
BSB_D unsigned decide(int model_type, const float* t) {
  if (model_type == MODEL_DEEPLAB) {
    float maxval = -10000.f; int maxpos = 0;
    for (int i = 0; i < 21; ++i) { const float v = __ldg(t + i); if (v > maxval) { maxval = v; maxpos = i; } }
    return (maxpos == 15) ? 0u : 1u;
  }
  if (model_type == MODEL_MEET) {
    const float e0 = bsb_expf(__ldg(t)), e1 = bsb_expf(__ldg(t + 1));
    const float p0 = bsb_div(e0, e0 + e1), p1 = bsb_div(e1, e0 + e1);
    return (p0 < p1) ? 0u : 1u;
  }
  // `tmp[n] > 0.65` compares float with the double literal; equivalent to > 0.65f
  // (0.65 lies strictly between two adjacent floats) — SURVEY.md Appendix A
  return (__ldg(t) > 0.65f) ? 0u : 1u;
}

// The per-frame decisions of a pixel are independent (computed 8 at a time so their loads
// overlap); only the 3-tap state update is sequential, and it is pure ALU on a bit mask.
// GATHER (calls with held frames, bsb_set_mask_interval): out_f holds the B segmented frames of the call's nf frames;
// call frame b advances the state on segmented frame cidx[b], or holds it (cidx[b] < 0), and stores it either way.
template <bool GATHER>
__global__ void __launch_bounds__(128) k_decision_iir(int model_type, int B, const float* out_f, int npix, int oc,
                                                      uint8_t* state, uint8_t* ofinal, int ow, int opitch, int oframe, int nf,
                                                      const int* cidx) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= npix) return;
  const int opos = (n / ow) * opitch + (n % ow);      // row-padded position inside one frame of ofinal
  unsigned st = state[n];
  if (GATHER) {
    for (int b = 0; b < nf; ++b) {
      const int j = __ldg(cidx + b);
      if (j >= 0) st = (decide(model_type, out_f + ((size_t)j * npix + n) * oc) ? 0xE0u : 0u) | (st >> 3);
      ofinal[(size_t)b * oframe + opos] = (uint8_t)st;
    }
  } else {
    for (int b0 = 0; b0 < B; b0 += 8) {
      unsigned bits = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (b0 + j < B) bits |= decide(model_type, out_f + ((size_t)(b0 + j) * npix + n) * oc) << j;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (b0 + j < B) {
          const unsigned val = ((bits >> j) & 1u) ? 255u : 0u;
          st = (val & 0xE0u) | (st >> 3);
          ofinal[(size_t)(b0 + j) * oframe + opos] = (uint8_t)st;
        }
    }
  }
  state[n] = (uint8_t)st;
}

// Frame-parallel form of the same stage.  The 3-tap state is a finite window: unrolling
//   st_b = (val_b & 0xE0) | (st_{b-1} >> 3)
// gives st_b = E0*d_b | 1C*d_{b-1} | 03*d_{b-2} for b >= 2, st_1 = E0*d_1 | 1C*d_0 | (s >> 6), st_0 = E0*d_0 | (s >> 3)
// (s = the state the previous call left, any byte; d = 1 where val = 255), so nothing but the three latest decisions
// is carried from frame to frame.  k_decision_iir walks the B frames of a pixel in ONE thread — 36 864 threads for the
// Meet output however large the batch is, a small fraction of the GPU's thread slots.  Here a block owns 32 pixels x all B frames: its eight warps take the frames round-robin,
// park the decisions in shared memory ([B][32] bytes) and, after one barrier, each thread assembles the state bytes of
// its frames from three of them.  The block that owns a pixel is the only one that touches its state byte: read before
// the barrier, written (by the owner of frame B-1) after it.
constexpr int DEC_PX = 32, DEC_WARPS = 8;

// the state after decision j of d ([B][32], this thread's column tx), entered with state s_in
BSB_D unsigned decision_window(const uint8_t* d, int tx, int j, unsigned s_in) {
  unsigned st = d[j * DEC_PX + tx] ? 0xE0u : 0u;
  if (j >= 1) st |= d[(j - 1) * DEC_PX + tx] ? 0x1Cu : 0u; else st |= s_in >> 3;
  if (j >= 2) st |= d[(j - 2) * DEC_PX + tx] ? 0x03u : 0u; else if (j == 1) st |= s_in >> 6;
  return st;
}

BSB_D void decision_window_store(const uint8_t* d, int tx, int ty, int B, unsigned s_in, uint8_t* state_px, uint8_t* ofinal_px, int oframe) {
  for (int b = ty; b < B; b += DEC_WARPS) {
    const unsigned st = decision_window(d, tx, b, s_in);
    ofinal_px[(size_t)b * oframe] = (uint8_t)st;
    if (b == B - 1) *state_px = (uint8_t)st;
  }
}

// Calls with held frames: d holds the decisions of the call's segmented frames only, and call frame b of nf stores the
// state after its latest segmented frame lat[b] (s_in when none precedes it).  The last call frame's latest segmented
// frame is the last one, so its state is the new state byte (s_in again when no frame is segmented).
BSB_D void decision_window_store_held(const uint8_t* d, int tx, int ty, int nf, const int* lat, unsigned s_in, uint8_t* state_px,
                                      uint8_t* ofinal_px, int oframe) {
  for (int b = ty; b < nf; b += DEC_WARPS) {
    const int j = __ldg(lat + b);
    const unsigned st = j < 0 ? s_in : decision_window(d, tx, j, s_in);
    ofinal_px[(size_t)b * oframe] = (uint8_t)st;
    if (b == nf - 1) *state_px = (uint8_t)st;
  }
}

template <bool GATHER>
__global__ void __launch_bounds__(DEC_PX * DEC_WARPS) k_decision_par(int model_type, int B, const float* out_f, int npix, int oc,
                                                                     uint8_t* state, uint8_t* ofinal, int ow, int opitch, int oframe,
                                                                     int nf, const int* lat) {
  BSB_DYN_SMEM(smem_raw);
  uint8_t* d = reinterpret_cast<uint8_t*>(smem_raw);               // [B][32] decisions
  const int tx = threadIdx.x % DEC_PX, ty = threadIdx.x / DEC_PX;
  const int n = blockIdx.x * DEC_PX + tx;
  const bool valid = n < npix;
  // held-frame calls park the entry state behind the decisions (row B), so it is not live across the decision loop
  const unsigned s_in = (!GATHER && valid) ? state[n] : 0u;
  if (valid) {
    if (GATHER && ty == 0) d[B * DEC_PX + tx] = state[n];
#pragma unroll 4
    for (int b = ty; b < B; b += DEC_WARPS) d[b * DEC_PX + tx] = (uint8_t)decide(model_type, out_f + ((size_t)b * npix + n) * oc);
  }
  __syncthreads();
  if (!valid) return;
  if (GATHER) decision_window_store_held(d, tx, ty, nf, lat, d[B * DEC_PX + tx], state + n, ofinal + (n / ow) * opitch + (n % ow), oframe);
  else decision_window_store(d, tx, ty, B, s_in, state + n, ofinal + (n / ow) * opitch + (n % ow), oframe);
}

void launch_decision_iir(cudaStream_t s, int model_type, int B, const float* model_out, int oh, int ow, int oc,
                         uint8_t* state, uint8_t* ofinal, int opitch, const SegRows& seg) {
  const int npix = oh * ow;
  const bool held = seg.cidx != nullptr;
  const size_t smem = (size_t)(B + (held ? 1 : 0)) * DEC_PX;
  if (tuning().dec_par && smem <= 48 * 1024) {
    auto k = held ? k_decision_par<true> : k_decision_par<false>;
    BSB_LAUNCH(k, dim3((unsigned)ceil_div(npix, DEC_PX)), dim3(DEC_PX * DEC_WARPS), smem, s, model_type, B, model_out,
               npix, oc, state, ofinal, ow, opitch, oh * opitch, seg.n, seg.lat);
    count_launch();
    return;
  }
  auto k = held ? k_decision_iir<true> : k_decision_iir<false>;
  BSB_LAUNCH(k, dim3((unsigned)ceil_div(npix, 128)), dim3(128), 0, s, model_type, B, model_out, npix, oc, state, ofinal,
             ow, opitch, oh * opitch, seg.n, seg.cidx);
  count_launch();
}

// DeepLab: RESIZE_BILINEAR (33x33x21 -> 257x257x21) + argmax + IIR in one pass.  One thread = one output pixel; the four
// neighbours and weights are those of k_resize_bilinear, the value of class i is formed with the same expression
// (-fmad=false: every product and sum rounds separately), the argmax scans the classes in order with a strict >.
struct UpTap { int o00, o10, o01, o11; float dy, dx, wy0, wx0; };

BSB_D UpTap up_tap(int y, int x, int ih, int iw, int ld, float hs, float ws, bool half_pixel) {
  float fy, fx; int y0, y1, x0, x1;
  bsb_resize_interp((float)y, hs, half_pixel, ih, &fy, &y0, &y1);
  bsb_resize_interp((float)x, ws, half_pixel, iw, &fx, &x0, &x1);
  UpTap t;
  t.dy = fy - (float)y0; t.dx = fx - (float)x0;
  t.wy0 = 1.f - t.dy; t.wx0 = 1.f - t.dx;
  t.o00 = (y0 * iw + x0) * ld; t.o10 = (y1 * iw + x0) * ld; t.o01 = (y0 * iw + x1) * ld; t.o11 = (y1 * iw + x1) * ld;
  return t;
}

// the decision of one output pixel of one frame (`f`: that frame's 33x33x21 tensor): 1 = background (argmax != person)
BSB_D unsigned up_decide(const float* f, const UpTap& t) {
  float maxval = -10000.f; int maxpos = 0;
#pragma unroll 7
  for (int i = 0; i < 21; ++i) {
    const float a = __ldg(f + t.o00 + i) * t.wy0 * t.wx0;
    const float bb = __ldg(f + t.o10 + i) * t.dy * t.wx0;
    const float d = __ldg(f + t.o01 + i) * t.wy0 * t.dx;
    const float e = __ldg(f + t.o11 + i) * t.dy * t.dx;
    const float v = ((a + bb) + d) + e;
    if (v > maxval) { maxval = v; maxpos = i; }
  }
  return (maxpos == 15) ? 0u : 1u;
}

template <bool GATHER>
__global__ void __launch_bounds__(128) k_decision_up_iir(int B, const float* low, int ih, int iw, int ld, float hs, float ws, bool half_pixel,
                                                         int oh, int ow, uint8_t* state, uint8_t* ofinal, int opitch, int oframe, int nf,
                                                         const int* cidx) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= oh * ow) return;
  const int y = n / ow, x = n - y * ow;
  const UpTap t = up_tap(y, x, ih, iw, ld, hs, ws, half_pixel);
  const int opos = y * opitch + x;
  unsigned st = state[n];
  if (GATHER) {                                       // as k_decision_iir<true>
    for (int b = 0; b < nf; ++b) {
      const int j = __ldg(cidx + b);
      if (j >= 0) st = (up_decide(low + (size_t)j * ih * iw * ld, t) ? 0xE0u : 0u) | (st >> 3);
      ofinal[(size_t)b * oframe + opos] = (uint8_t)st;
    }
  } else {
    for (int b = 0; b < B; ++b) {
      const unsigned val = up_decide(low + (size_t)b * ih * iw * ld, t) ? 255u : 0u;
      st = (val & 0xE0u) | (st >> 3);
      ofinal[(size_t)b * oframe + opos] = (uint8_t)st;
    }
  }
  state[n] = (uint8_t)st;
}

// frame-parallel form (see k_decision_par): a block = 32 output pixels x all B frames
template <bool GATHER>
__global__ void __launch_bounds__(DEC_PX * DEC_WARPS) k_decision_up_par(int B, const float* low, int ih, int iw, int ld, float hs, float ws, bool half_pixel,
                                                                        int oh, int ow, uint8_t* state, uint8_t* ofinal, int opitch, int oframe,
                                                                        int nf, const int* lat) {
  BSB_DYN_SMEM(smem_raw);
  uint8_t* d = reinterpret_cast<uint8_t*>(smem_raw);
  const int tx = threadIdx.x % DEC_PX, ty = threadIdx.x / DEC_PX;
  const int n = blockIdx.x * DEC_PX + tx;
  const bool valid = n < oh * ow;
  const unsigned s_in = (!GATHER && valid) ? state[n] : 0u;       // held-frame calls: row B, as in k_decision_par
  const int y = valid ? n / ow : 0, x = valid ? n - y * ow : 0;
  if (valid) {
    if (GATHER && ty == 0) d[B * DEC_PX + tx] = state[n];
    const UpTap t = up_tap(y, x, ih, iw, ld, hs, ws, half_pixel);
    for (int b = ty; b < B; b += DEC_WARPS) d[b * DEC_PX + tx] = (uint8_t)up_decide(low + (size_t)b * ih * iw * ld, t);
  }
  __syncthreads();
  if (!valid) return;
  if (GATHER) decision_window_store_held(d, tx, ty, nf, lat, d[B * DEC_PX + tx], state + n, ofinal + y * opitch + x, oframe);
  else decision_window_store(d, tx, ty, B, s_in, state + n, ofinal + y * opitch + x, oframe);
}

void launch_decision_up_iir(cudaStream_t s, int B, const float* low, int ih, int iw, int ld, bool align_corners, bool half_pixel,
                            int oh, int ow, uint8_t* state, uint8_t* ofinal, int opitch, const SegRows& seg) {
  float hs = (float)ih / (float)oh, ws = (float)iw / (float)ow;
  if (align_corners && oh > 1) hs = (float)(ih - 1) / (float)(oh - 1);
  if (align_corners && ow > 1) ws = (float)(iw - 1) / (float)(ow - 1);
  const bool held = seg.cidx != nullptr;
  const size_t smem = (size_t)(B + (held ? 1 : 0)) * DEC_PX;
  if (tuning().dec_par && smem <= 48 * 1024) {
    auto k = held ? k_decision_up_par<true> : k_decision_up_par<false>;
    BSB_LAUNCH(k, dim3((unsigned)ceil_div(oh * ow, DEC_PX)), dim3(DEC_PX * DEC_WARPS), smem, s, B, low, ih, iw, ld, hs, ws,
               half_pixel, oh, ow, state, ofinal, opitch, oh * opitch, seg.n, seg.lat);
    count_launch();
    return;
  }
  auto k = held ? k_decision_up_iir<true> : k_decision_up_iir<false>;
  BSB_LAUNCH(k, dim3((unsigned)ceil_div(oh * ow, 128)), dim3(128), 0, s, B, low, ih, iw, ld, hs, ws, half_pixel, oh, ow, state,
             ofinal, opitch, oh * opitch, seg.n, seg.cidx);
  count_launch();
}

// ---------------------------------------------------------------------------
// Independent sources (one frame per source and call): frame b advances the state of source src[b] by exactly one IIR
// step, st = (d ? 0xE0 : 0) | (state >> 3).  Ids are distinct within a call, so no two frames share a state byte and
// every (pixel, frame) is independent: one thread each, blockIdx.y = frame, threads along pixels (coalesced state,
// ofinal and model-output loads).
// ---------------------------------------------------------------------------
constexpr int DEC_SRC_T = 128;

// GATHER (calls with held frames): the grid still covers the call's frames; frame b is segmented frame cidx[b] of out_f,
// or, at cidx[b] < 0, held: its ofinal is its source's state as it stands (no frame of the launch writes that state, the
// ids being distinct).
template <bool GATHER>
__global__ void __launch_bounds__(DEC_SRC_T) k_decision_sources(int model_type, const float* out_f, int npix, int oc, uint8_t* states,
                                                                const int* src, uint8_t* ofinal, int ow, int opitch, int oframe,
                                                                const int* cidx) {
  const int n = blockIdx.x * DEC_SRC_T + threadIdx.x, b = blockIdx.y;
  if (n >= npix) return;
  uint8_t* sp = states + (size_t)__ldg(src + b) * npix + n;
  const int j = GATHER ? __ldg(cidx + b) : b;
  if (GATHER && j < 0) { ofinal[(size_t)b * oframe + (n / ow) * opitch + (n % ow)] = *sp; return; }
  const unsigned st = (decide(model_type, out_f + ((size_t)j * npix + n) * oc) ? 0xE0u : 0u) | ((unsigned)*sp >> 3);
  ofinal[(size_t)b * oframe + (n / ow) * opitch + (n % ow)] = (uint8_t)st;
  *sp = (uint8_t)st;
}

template <bool GATHER>
__global__ void __launch_bounds__(DEC_SRC_T) k_decision_up_sources(const float* low, int ih, int iw, int ld, float hs, float ws, bool half_pixel,
                                                                   int oh, int ow, uint8_t* states, const int* src, uint8_t* ofinal, int opitch,
                                                                   int oframe, const int* cidx) {
  const int n = blockIdx.x * DEC_SRC_T + threadIdx.x, b = blockIdx.y;
  if (n >= oh * ow) return;
  const int y = n / ow, x = n - y * ow;
  uint8_t* sp = states + (size_t)__ldg(src + b) * oh * ow + n;
  const int j = GATHER ? __ldg(cidx + b) : b;
  if (GATHER && j < 0) { ofinal[(size_t)b * oframe + y * opitch + x] = *sp; return; }
  const unsigned d = up_decide(low + (size_t)j * ih * iw * ld, up_tap(y, x, ih, iw, ld, hs, ws, half_pixel));
  const unsigned st = (d ? 0xE0u : 0u) | ((unsigned)*sp >> 3);
  ofinal[(size_t)b * oframe + y * opitch + x] = (uint8_t)st;
  *sp = (uint8_t)st;
}

void launch_decision_sources(cudaStream_t s, int model_type, int B, const float* model_out, int oh, int ow, int oc,
                             uint8_t* states, const int* src, uint8_t* ofinal, int opitch, const int* cidx) {
  const int npix = oh * ow;
  auto k = cidx ? k_decision_sources<true> : k_decision_sources<false>;
  BSB_LAUNCH(k, dim3((unsigned)ceil_div(npix, DEC_SRC_T), (unsigned)B), dim3(DEC_SRC_T), 0, s, model_type, model_out, npix, oc,
             states, src, ofinal, ow, opitch, oh * opitch, cidx);
  count_launch();
}

void launch_decision_up_sources(cudaStream_t s, int B, const float* low, int ih, int iw, int ld, bool align_corners, bool half_pixel,
                                int oh, int ow, uint8_t* states, const int* src, uint8_t* ofinal, int opitch, const int* cidx) {
  float hs = (float)ih / (float)oh, ws = (float)iw / (float)ow;
  if (align_corners && oh > 1) hs = (float)(ih - 1) / (float)(oh - 1);
  if (align_corners && ow > 1) ws = (float)(iw - 1) / (float)(ow - 1);
  auto k = cidx ? k_decision_up_sources<true> : k_decision_up_sources<false>;
  BSB_LAUNCH(k, dim3((unsigned)ceil_div(oh * ow, DEC_SRC_T), (unsigned)B), dim3(DEC_SRC_T), 0, s, low, ih, iw, ld, hs, ws,
             half_pixel, oh, ow, states, src, ofinal, opitch, oh * opitch, cidx);
  count_launch();
}

// ---------------------------------------------------------------------------
// Fused post stage: mask upsample (cv::resize 8UC1) + cv::blur 5x5 (REFLECT_101 inside the
// ROI) + alpha_blend + optional RGB->YUYV + optional mask store.
//
// Block = 256 threads = one 128 x 32 pixel tile; thread = 16 consecutive pixels of one row
// (48 B per 3-channel array: three 16-byte vector accesses).  Shared memory holds the
// upsampled tile with a 2-pixel halo (u8) and its vertical 5-sums (u16); box sums are
// integer, so the separable evaluation is exact.
// ---------------------------------------------------------------------------
constexpr int PT_W = 128, PT_H = 32, PT_PX = 16;
constexpr int PT_UW = PT_W + 4, PT_UH = PT_H + 4, PT_US = PT_UW + 4;   // smem row stride (bytes)

struct Px16 { uint4 v[3]; };

BSB_D void load48(const uint8_t* p, bool fast, Px16& r) {
  if (fast) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    r.v[0] = __ldg(q); r.v[1] = __ldg(q + 1); r.v[2] = __ldg(q + 2);
  } else {
    uint8_t* d = reinterpret_cast<uint8_t*>(&r);
    for (int i = 0; i < 48; ++i) d[i] = p[i];
  }
}

// PASS: the launch has a filter table (PostArgs::pass), BGRA a transparent output (PostArgs::bgra), as k_post_fast
template <bool PASS, bool BGRA = false>
__global__ void __launch_bounds__(256) k_post(PostArgs a) {
  __shared__ __align__(16) uint8_t Us[PT_UH * PT_US];
  __shared__ __align__(16) unsigned short Vs[PT_H * PT_UW];
  const int b = blockIdx.z;
  const int tx0 = blockIdx.x * PT_W, ty0 = blockIdx.y * PT_H;
  const int tid = threadIdx.x;
  const bool pass = PASS && __ldg(a.pass + b) != 0;
  const bool hits_roi = (!pass || a.mask) && tx0 < a.roi_x + a.roi_w && tx0 + PT_W > a.roi_x && ty0 < a.roi_y + a.roi_h && ty0 + PT_H > a.roi_y;

  if (hits_roi) {
    // ---- A: upsampled mask tile with halo, reflect-101 at the ROI border ----
    const uint8_t* src = a.ofinal + (size_t)b * a.opitch * a.oh + (size_t)a.out_y * a.opitch + a.out_x;
    for (int i = tid; i < PT_UH * PT_UW; i += 256) {
      const int uy = i / PT_UW, ux = i % PT_UW;
      const int gy = bsb_reflect101(ty0 - a.roi_y - 2 + uy, a.roi_h);
      const int gx = bsb_reflect101(tx0 - a.roi_x - 2 + ux, a.roi_w);
      if (a.area2x2) {      // exact 2x down-scale: cv::resize takes its INTER_AREA 2x2 mean ((a + b + c + d + 2) >> 2)
        const uint8_t* s0 = src + (size_t)(2 * gy) * a.opitch + 2 * gx;
        const uint8_t* s1 = s0 + a.opitch;
        Us[uy * PT_US + ux] = (uint8_t)(((int)s0[0] + s0[1] + s1[0] + s1[1] + 2) >> 2);
        continue;
      }
      const int sx = __ldg(a.tab.xofs + gx), sx1 = min(sx + 1, a.out_w - 1);
      const int a0 = __ldg(a.tab.xw + 2 * gx), a1 = __ldg(a.tab.xw + 2 * gx + 1);
      const int b0 = __ldg(a.tab.yw + 2 * gy), b1 = __ldg(a.tab.yw + 2 * gy + 1);
      const uint8_t* r0 = src + (size_t)__ldg(a.tab.yofs0 + gy) * a.opitch;
      const uint8_t* r1 = src + (size_t)__ldg(a.tab.yofs1 + gy) * a.opitch;
      Us[uy * PT_US + ux] = lin_v(lin_h(r0, sx, sx1, 1, 0, a0, a1), lin_h(r1, sx, sx1, 1, 0, a0, a1), b0, b1);
    }
    __syncthreads();
    // ---- B: vertical 5-sums ----
    for (int i = tid; i < PT_H * PT_UW; i += 256) {
      const int y = i / PT_UW, x = i % PT_UW;
      const uint8_t* u = Us + y * PT_US + x;
      Vs[i] = (unsigned short)(u[0] + u[PT_US] + u[2 * PT_US] + u[3 * PT_US] + u[4 * PT_US]);
    }
    __syncthreads();
  }

  const int lx = (tid % (PT_W / PT_PX)) * PT_PX, ly = tid / (PT_W / PT_PX);
  const int x0 = tx0 + lx, y = ty0 + ly;
  if (y >= a.H || x0 >= a.W) return;
  const int npx = min(PT_PX, a.W - x0);

  // ---- C: horizontal 5-sums -> mask ----
  uint8_t m[PT_PX];
  const bool row_in = hits_roi && y >= a.roi_y && y < a.roi_y + a.roi_h;
#pragma unroll
  for (int i = 0; i < PT_PX; ++i) {
    const int x = x0 + i;
    unsigned mv = 255u;
    if (row_in && x >= a.roi_x && x < a.roi_x + a.roi_w) {
      const unsigned short* v = Vs + ly * PT_UW + lx + i;
      mv = bsb_box25((unsigned)v[0] + v[1] + v[2] + v[3] + v[4]);
    }
    m[i] = (uint8_t)mv;
  }

  // ---- D: blend (+ YUYV, + mask) ----
  const size_t fo = (size_t)b * a.frame_stride + (size_t)y * a.frame_pitch + (size_t)x0 * 3;
  const bool full = npx == PT_PX;
  Px16 f, g, o;
  // (a transparent output without a composite or video output blends nothing: no background is read)
  if (pass || (BGRA && !a.out && !a.yuyv)) {
    // filter off: the camera frame alone, blended at weight 0
    const bool fast_in = full && (reinterpret_cast<uintptr_t>(a.frames + fo) & 15) == 0;
    if (full) load48(a.frames + fo, fast_in, f);
    else {
      uint8_t* fd = reinterpret_cast<uint8_t*>(&f);
      for (int i = 0; i < npx * 3; ++i) fd[i] = a.frames[fo + i];
    }
    g = f;
  } else {
    const size_t bo = bg_frame_offset(a, b) + (size_t)y * a.bg_pitch + (size_t)x0 * 3;
    const bool fast_in = full && ((reinterpret_cast<uintptr_t>(a.frames + fo) | reinterpret_cast<uintptr_t>(a.bg + bo)) & 15) == 0;
    if (full) { load48(a.frames + fo, fast_in, f); load48(a.bg + bo, fast_in, g); }
    else {
      uint8_t* fd = reinterpret_cast<uint8_t*>(&f); uint8_t* gd = reinterpret_cast<uint8_t*>(&g);
      for (int i = 0; i < npx * 3; ++i) { fd[i] = a.frames[fo + i]; gd[i] = a.bg[bo + i]; }
    }
  }
  const uint8_t* fb = reinterpret_cast<const uint8_t*>(&f);
  const uint8_t* gb = reinterpret_cast<const uint8_t*>(&g);
  uint8_t* ob = reinterpret_cast<uint8_t*>(&o);
  if (BGRA) {
    uint8_t* bp = a.bgra + (size_t)b * a.bgra_stride + (size_t)y * a.bgra_pitch + (size_t)x0 * 4;
    for (int i = 0; i < npx; ++i) {
      bp[4 * i] = fb[3 * i]; bp[4 * i + 1] = fb[3 * i + 1]; bp[4 * i + 2] = fb[3 * i + 2];
      bp[4 * i + 3] = (uint8_t)(pass ? 255u : 255u - m[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < PT_PX; ++i) {
    const unsigned aw = blend_weight(pass, m[i]), bw = 255u - aw;
#pragma unroll
    for (int c = 0; c < 3; ++c) ob[3 * i + c] = (uint8_t)bsb_div255((unsigned)gb[3 * i + c] * aw + (unsigned)fb[3 * i + c] * bw);
  }
  if (a.out) {
    uint8_t* op = a.out + (size_t)b * a.out_stride + (size_t)y * a.out_pitch + (size_t)x0 * 3;
    if (full && (reinterpret_cast<uintptr_t>(op) & 15) == 0) {
      uint4* q = reinterpret_cast<uint4*>(op); q[0] = o.v[0]; q[1] = o.v[1]; q[2] = o.v[2];
    } else for (int i = 0; i < npx * 3; ++i) op[i] = ob[i];
  }
  if (a.mask) {
    uint8_t* mp = a.mask + (size_t)b * a.mask_stride + (size_t)y * a.W + x0;
    if (full && (reinterpret_cast<uintptr_t>(mp) & 15) == 0) *reinterpret_cast<uint4*>(mp) = *reinterpret_cast<const uint4*>(m);
    else for (int i = 0; i < npx; ++i) mp[i] = m[i];
  }
  if (a.yuyv) {
    // pairs are taken over the flattened image (app/deepseg.cc:97-104); W even => pairs never straddle rows
    __align__(16) uint8_t yy[PT_PX * 2];
#pragma unroll
    for (int i = 0; i < PT_PX; i += 2) {
      int Y0, U0, V0, Y1, U1, V1;
      rgb2yuv(ob[3 * i], ob[3 * i + 1], ob[3 * i + 2], Y0, U0, V0);
      rgb2yuv(ob[3 * i + 3], ob[3 * i + 4], ob[3 * i + 5], Y1, U1, V1);
      yy[2 * i] = (uint8_t)Y0; yy[2 * i + 1] = (uint8_t)((V0 + V1) / 2);
      yy[2 * i + 2] = (uint8_t)Y1; yy[2 * i + 3] = (uint8_t)((U0 + U1) / 2);
    }
    uint8_t* yp = a.yuyv + (size_t)b * a.yuyv_stride + ((size_t)y * a.W + x0) * 2;
    if (full && (reinterpret_cast<uintptr_t>(yp) & 15) == 0) {
      uint4* q = reinterpret_cast<uint4*>(yp); const uint4* sv = reinterpret_cast<const uint4*>(yy); q[0] = sv[0]; q[1] = sv[1];
    } else for (int i = 0; i < (npx & ~1) * 2; ++i) yp[i] = yy[i];
  }
}

// ---------------------------------------------------------------------------
// Fast path of the same fused stage (W % 16 == 0, tight 16-byte aligned rows).
// The kernel is bound by integer instruction issue, not by HBM, so it is organised to
// minimise instructions per pixel:
//   A0  column / row interpolation parameters of the tile -> shared memory (once)
//   A1  horizontal pass of cv::resize for the few source rows the tile touches (Hs, >>4)
//   A2  vertical pass -> upsampled mask tile with halo (Us, u16)
//   B   vertical 5-sums on packed u16x2 lanes with a sliding window (Vs)
//   C   horizontal 5-sums on packed lanes -> mask = (S + 12) / 25 as a multiply-shift
//   D   alpha blend with two channels per 32-bit IMAD (16-bit lanes share the pixel's
//       mask) and one via DP4A, division by 255 on packed lanes, RGB->YUV with DP2A,
//       16-byte streaming loads / stores.
// ---------------------------------------------------------------------------

// PASS: the launch has a filter table (PostArgs::pass); without one the kernel is compiled without the pass-through.
// BGRA: the launch writes the transparent output (PostArgs::bgra); without OUT and YUYV it reads no background.
// REFINE: the launch has a refinement table (PostArgs::refine).  A mixed tile of a refined frame loads the patch its
// refinement reaches, puts it with the guide lumas into Hs and the frame's range row into Us, and computes each thread's
// mask from the camera bytes after they are loaded (refine_mask16, staged through Vs); A1 / A2 / B do not run.
template <bool OUT, bool YUYV, bool PASS, bool BGRA = false, bool REFINE = false>
__global__ void __launch_bounds__(256, 4) k_post_fast(PostArgs a) {
  __shared__ __align__(16) unsigned short Hs[PF_RMAX * PF_US];
  __shared__ __align__(16) unsigned short Us[PF_UH * PF_US];
  __shared__ __align__(16) unsigned short Vs[PF_H * PF_US];
  __shared__ __align__(16) uint4 rows[PF_UH];     // r0, r1, b0 << 16, b1 << 16
  __shared__ __align__(16) uint8_t Ps[PF_RMAX * PF_PS];   // source patch of the small mask
  const int b = blockIdx.z;
  const int tx0 = blockIdx.x * PF_W, ty0 = blockIdx.y * PF_H;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // a frame whose filter is off reads no background, and computes its mask only when the call stores it
  const bool pass = PASS && __ldg(a.pass + b) != 0;
  const bool hits_roi = (!pass || a.mask) && tx0 < a.roi_x + a.roi_w && tx0 + PF_W > a.roi_x && ty0 < a.roi_y + a.roi_h && ty0 + PF_H > a.roi_y;
  int tile_const = -1;                       // 255 / 0 when the whole mask tile is known to be constant
  const int sig = REFINE ? __ldg(a.refine + b) : 0;
  int rmin = 0, cmin = 0;                    // the patch's first small row / column
  {
    // pull this thread's 48 bytes of camera frame into L2 while the mask tile is being built
    const int px0 = tx0 + (tid & 7) * PF_PX, py = ty0 + (tid >> 3);
    if ((OUT || YUYV || BGRA) && py < a.H && px0 < a.W) prefetch_l2(a.frames + (size_t)b * a.frame_stride + (size_t)py * a.frame_pitch + (size_t)px0 * 3);
  }

  if (hits_roi) {
    // yofs0/yofs1/xofs are monotonic, so the source patch this tile touches follows from the smallest /
    // largest (reflected) destination coordinates of the tile — no reduction needed.
    const int gy_lo = ty0 - a.roi_y - 2, gy_hi = gy_lo + PF_UH - 1;
    const int gy_min = gy_lo < 0 ? 0 : min(gy_lo, a.roi_h - 1);
    const int gy_max = gy_hi >= a.roi_h ? a.roi_h - 1 : max(gy_hi, 0);
    const int gx_lo = tx0 - a.roi_x - 2, gx_hi = gx_lo + PF_UW - 1;
    const int gx_min = gx_lo < 0 ? 0 : min(gx_lo, a.roi_w - 1);
    const int gx_max = gx_hi >= a.roi_w ? a.roi_w - 1 : max(gx_hi, 0);
    rmin = __ldg(a.tab.yofs0 + gy_min);
    int nrows = __ldg(a.tab.yofs1 + gy_max) - rmin + 1;
    cmin = (int)(__ldg(&a.tab.xcol[gx_min].x) & 0xffffu);
    int ncols = (int)(__ldg(&a.tab.xcol[gx_max].x) >> 16) - cmin + 1;
    if (REFINE && sig) {
      // a refined frame: the small rows / columns taps s - 1 .. s + 2 of the tile's ROI pixels reach
      const int ylo = max(ty0, a.roi_y) - a.roi_y, yhi = min(ty0 + PF_H, a.roi_y + a.roi_h) - 1 - a.roi_y;
      const int xlo = max(tx0, a.roi_x) - a.roi_x, xhi = min(tx0 + PF_W, a.roi_x + a.roi_w) - 1 - a.roi_x;
      rmin = max((int)(__ldg(a.refine_y + ylo) & 0xffffu) - 2, 0);
      nrows = min((int)(__ldg(a.refine_y + yhi) & 0xffffu) + 1, a.out_h - 1) - rmin + 1;
      cmin = max((int)(__ldg(a.refine_x + xlo) & 0xffffu) - 2, 0);
      ncols = min((int)(__ldg(a.refine_x + xhi) & 0xffffu) + 1, a.out_w - 1) - cmin + 1;
    }
    // ---- P: source patch of the small mask -> shared memory (coalesced); row parameters for A2.
    //      If every source pixel of the patch is 255 (or 0) the upsampled + blurred tile is 255 (or 0)
    //      whatever the interpolation weights are (their sums are 2048 +- 1), so A1/A2/B are skipped. ----
    unsigned p_and = 255u, p_or = 0u;
    {
      const uint8_t* src = a.ofinal + (size_t)b * a.opitch * a.oh + (size_t)(a.out_y + rmin) * a.opitch + a.out_x + cmin;
      for (int r = warp; r < nrows; r += 8)
        for (int c = lane; c < ncols; c += 32) {
          const unsigned v = src[(size_t)r * a.opitch + c];
          Ps[r * PF_PS + c] = (uint8_t)v;
          p_and &= v; p_or |= v;
        }
      if (tid >= 192 && tid < 192 + PF_UH) {
        const int uy = tid - 192;
        int gy = gy_lo + uy;
        gy = gy < 0 ? -gy : gy; gy = gy >= a.roi_h ? 2 * a.roi_h - 2 - gy : gy;     // reflect-101 (single fold)
        gy = min(max(gy, 0), a.roi_h - 1);
        rows[uy] = make_uint4((unsigned)__ldg(a.tab.yofs0 + gy), (unsigned)__ldg(a.tab.yofs1 + gy),
                              (unsigned)(int)__ldg(a.tab.yw + 2 * gy) << 16, (unsigned)(int)__ldg(a.tab.yw + 2 * gy + 1) << 16);
      }
    }
    const int all_hi = __syncthreads_and(p_and == 255u);
    const int all_lo = all_hi ? 0 : __syncthreads_and(p_or == 0u);
    tile_const = all_hi ? 255 : (all_lo ? 0 : -1);
    if (REFINE && sig && tile_const < 0) {
      // ---- R: the refinement patch (mask | guide luma << 8) -> Hs, the frame's range row -> Us ----
      const uint8_t* fr = a.frames + (size_t)b * a.frame_stride;
      refine_patch(a, Ps, PF_PS, rmin, nrows, cmin, ncols, Hs, PF_US, tid, 256, [&](int x, int yy, int* bgr) {
        const uint8_t* p = fr + (size_t)yy * a.frame_pitch + (size_t)x * 3;
        bgr[0] = p[0]; bgr[1] = p[1]; bgr[2] = p[2];
      });
      Us[tid] = __ldg(a.refine_w + (size_t)(sig - 1) * 256 + tid);
      __syncthreads();
    } else if (tile_const < 0) {
    // ---- A1: horizontal pass of cv::resize on the patch rows: Hs = (s[sx]*a0 + s[sx1]*a1) >> 4.
    //      A thread owns a column (parameters in registers) and walks every second patch row. ----
    {
      const int phase = tid >> 7;
      for (int ux = tid & 127; ux < PF_UW; ux += 128) {
        int gx = gx_lo + ux;
        gx = gx < 0 ? -gx : gx; gx = gx >= a.roi_w ? 2 * a.roi_w - 2 - gx : gx;
        gx = min(max(gx, 0), a.roi_w - 1);
        const uint2 xc = __ldg(a.tab.xcol + gx);
        const int sx = (int)(xc.x & 0xffffu) - cmin, sx1 = (int)(xc.x >> 16) - cmin;
        const int a0 = (int)(short)(xc.y & 0xffffu), a1 = (int)(short)(xc.y >> 16);
        const uint8_t* pr = Ps + phase * PF_PS;
        unsigned short* hp = Hs + phase * PF_US + ux;
        for (int r = phase; r < nrows; r += 2) {
          *hp = (unsigned short)(((int)pr[sx] * a0 + (int)pr[sx1] * a1) >> 4);
          pr += 2 * PF_PS; hp += 2 * PF_US;
        }
      }
    }
    __syncthreads();
    // ---- A2: vertical pass -> upsampled tile.  ((b*h) >> 16) is one IMAD.HI with b pre-shifted by 16.
    //      A warp takes a row; each lane produces columns lane, lane+32, ... ----
    for (int uy = warp; uy < PF_UH; uy += 8) {
      const uint4 rp = rows[uy];
      const unsigned short* h0 = Hs + ((int)rp.x - rmin) * PF_US + lane;
      const unsigned short* h1 = Hs + ((int)rp.y - rmin) * PF_US + lane;
      unsigned short* up = Us + uy * PF_US + lane;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        up[32 * k] = (unsigned short)((__umulhi(rp.z, (unsigned)h0[32 * k]) + __umulhi(rp.w, (unsigned)h1[32 * k]) + 2u) >> 2);
      if (lane < PF_UW - 128)
        up[128] = (unsigned short)((__umulhi(rp.z, (unsigned)h0[128]) + __umulhi(rp.w, (unsigned)h1[128]) + 2u) >> 2);
    }
    __syncthreads();
    // ---- B: vertical 5-sums, two columns per 32-bit word, sliding window over 8 rows ----
    for (int it = tid; it < (PF_UW / 2) * 4; it += 256) {
      const int pair = it % (PF_UW / 2), seg = it / (PF_UW / 2);
      const unsigned* up = reinterpret_cast<const unsigned*>(Us + (seg * 8) * PF_US) + pair;
      unsigned* vp = reinterpret_cast<unsigned*>(Vs + (seg * 8) * PF_US) + pair;
      unsigned u[12];
#pragma unroll
      for (int k = 0; k < 12; ++k) u[k] = up[k * (PF_US / 2)];
      unsigned v = u[0] + u[1] + u[2] + u[3] + u[4];
      vp[0] = v;
#pragma unroll
      for (int k = 1; k < 8; ++k) { v = v + u[k + 4] - u[k - 1]; vp[k * (PF_US / 2)] = v; }
    }
    __syncthreads();
    }
  }

  const int lx = (tid & 7) * PF_PX, ly = tid >> 3;
  const int x0 = tx0 + lx, y = ty0 + ly;
  if (y >= a.H || x0 >= a.W) return;

  // ---- issue the streaming loads early ----
  unsigned f[12], g[12];
  const bool refined = REFINE && sig && hits_roi && tile_const < 0;    // the refined mask reads the camera bytes
  if (OUT || YUYV || BGRA || refined) {
    const uint8_t* fp = a.frames + (size_t)b * a.frame_stride + (size_t)y * a.frame_pitch + (size_t)x0 * 3;
    const uint8_t* gp = a.bg + bg_frame_offset(a, b) + (size_t)y * a.bg_pitch + (size_t)x0 * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const uint4 t = a.frame_l1 ? __ldg(reinterpret_cast<const uint4*>(fp + 16 * k)) : ldg_stream(fp + 16 * k);
      f[4 * k] = t.x; f[4 * k + 1] = t.y; f[4 * k + 2] = t.z; f[4 * k + 3] = t.w;
      const uint4 s = (pass || !(OUT || YUYV)) ? t : __ldg(reinterpret_cast<const uint4*>(gp + 16 * k));
      g[4 * k] = s.x; g[4 * k + 1] = s.y; g[4 * k + 2] = s.z; g[4 * k + 3] = s.w;
    }
  }

  // ---- C: horizontal 5-sums on packed lanes -> 16 mask values ----
  unsigned m[PF_PX];
  const bool row_in = hits_roi && y >= a.roi_y && y < a.roi_y + a.roi_h;
  if (refined) refine_mask16(a, row_in, x0, y, f, Hs, PF_US, rmin, cmin, Us, reinterpret_cast<uint8_t*>(Vs) + ly * PF_W + lx, m);
  else post_mask16(a, row_in, tile_const, x0, Vs + ly * PF_US + lx, m);

  if (a.mask) {
    uint4 mv;
    mv.x = m[0] | (m[1] << 8) | (m[2] << 16) | (m[3] << 24);
    mv.y = m[4] | (m[5] << 8) | (m[6] << 16) | (m[7] << 24);
    mv.z = m[8] | (m[9] << 8) | (m[10] << 16) | (m[11] << 24);
    mv.w = m[12] | (m[13] << 8) | (m[14] << 16) | (m[15] << 24);
    stg_stream(a.mask + (size_t)b * a.mask_stride + (size_t)y * a.W + x0, mv);
  }
  if (BGRA) {
    // (m becomes the blend weights here, as below for a filtered-off frame: the mask is stored already)
#pragma unroll
    for (int i = 0; i < PF_PX; ++i) m[i] = blend_weight(pass, m[i]);
    uint8_t* bp = a.bgra + (size_t)b * a.bgra_stride + (size_t)y * a.bgra_pitch + (size_t)x0 * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) stg_stream(bp + 16 * k, bgra4(f + 3 * k, m + 4 * k, false));
  }
  if (!(OUT || YUYV)) return;
  if (pass) {
#pragma unroll
    for (int i = 0; i < PF_PX; ++i) m[i] = blend_weight(true, m[i]);
  }

  // ---- D: blend (+ RGB->YUV) ----
  unsigned o[12], yy[8];
  post_blend16<OUT, YUYV>(f, g, m, o, yy);
  if (OUT) {
    uint8_t* op = a.out + (size_t)b * a.out_stride + (size_t)y * a.out_pitch + (size_t)x0 * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) stg_stream(op + 16 * k, make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]));
  }
  if (YUYV) {
    uint8_t* yp = a.yuyv + (size_t)b * a.yuyv_stride + ((size_t)y * a.W + x0) * 2;
    stg_stream(yp, make_uint4(yy[0], yy[1], yy[2], yy[3]));
    stg_stream(yp + 16, make_uint4(yy[4], yy[5], yy[6], yy[7]));
  }
}

static bool post_fast_ok(const PostArgs& a) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (a.W % 16 != 0 || a.area2x2) return false;
  if (!al16(a.frames) || !al16(a.bg) || a.frame_pitch % 16 || a.frame_stride % 16 || a.bg_pitch % 16 || a.bg_stride % 16) return false;
  if (a.out && (!al16(a.out) || a.out_pitch % 16 || a.out_stride % 16)) return false;
  if (a.yuyv && (!al16(a.yuyv) || a.yuyv_stride % 16)) return false;
  if (a.mask && (!al16(a.mask) || a.mask_stride % 16)) return false;
  if (a.bgra && (!al16(a.bgra) || a.bgra_pitch % 16 || a.bgra_stride % 16)) return false;
  if (a.ow > 32000 || a.oh > 32000 || a.roi_w < 8 || a.roi_h < 8) return false;
  // source rows touched by one 36-row tile must fit the Hs buffer: ceil(36 * scale) + 2
  const double scale_y = (double)a.out_h / (double)a.roi_h;
  if ((int)(PF_UH * scale_y) + 3 > PF_RMAX) return false;
  const double scale_x = (double)a.out_w / (double)a.roi_w;
  if ((int)(PF_UW * scale_x) + 4 > PF_PS || a.tab.xcol == nullptr) return false;
  // a refined tile's patch: taps s - 1 .. s + 2 of its 32 rows / 128 columns, in Ps and (u16, PF_US apart) in Hs
  if (a.refine && ((int)((PF_H - 1) * scale_y) + 6 > PF_RMAX || (int)((PF_W - 1) * scale_x) + 6 > PF_US || !a.refine_x)) return false;
  return true;
}

bool launch_post_tma(cudaStream_t s, const PostArgs& a);   // kernels_post.cu

template <bool PASS, bool BGRA = false, bool REFINE = false>
static void launch_post_fast(cudaStream_t s, dim3 grid, const PostArgs& a) {
  if (a.yuyv && a.out) { auto k = k_post_fast<true, true, PASS, BGRA, REFINE>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else if (a.yuyv) { auto k = k_post_fast<false, true, PASS, BGRA, REFINE>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else if (a.out) { auto k = k_post_fast<true, false, PASS, BGRA, REFINE>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else { auto k = k_post_fast<false, false, PASS, BGRA, REFINE>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
}
template <bool REFINE>
static void launch_post_fast_r(cudaStream_t s, dim3 grid, const PostArgs& a) {
  if (a.bgra) { if (a.pass) launch_post_fast<true, true, REFINE>(s, grid, a); else launch_post_fast<false, true, REFINE>(s, grid, a); }
  else if (a.pass) launch_post_fast<true, false, REFINE>(s, grid, a);
  else launch_post_fast<false, false, REFINE>(s, grid, a);
}

bool launch_post(cudaStream_t s, const PostArgs& a_in) {
  if (launch_post_tma(s, a_in)) return true;
  // only k_post_tma writes mirrored frames: a flip table it could not take is an error, never unmirrored output
  if (a_in.flip) return false;
  PostArgs a = a_in;
  a.frame_l1 = tuning().post_l1;                 // measurement switch: frame loads allocate in L1
  if (post_fast_ok(a)) {
    dim3 grid((unsigned)ceil_div(a.W, PF_W), (unsigned)ceil_div(a.H, PF_H), (unsigned)a.B);
    if (a.refine) launch_post_fast_r<true>(s, grid, a);
    else launch_post_fast_r<false>(s, grid, a);
    count_launch();
    return true;
  }
  // refined frames are taken by k_post_tma and k_post_fast only: a refinement table neither can take is an error
  if (a.refine) return false;
  dim3 grid((unsigned)ceil_div(a.W, PT_W), (unsigned)ceil_div(a.H, PT_H), (unsigned)a.B);
  if (a.bgra) {
    if (a.pass) { auto k = k_post<true, true>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
    else { auto k = k_post<false, true>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  } else if (a.pass) { auto k = k_post<true>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else { auto k = k_post<false>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  count_launch();
  return true;
}

// ---------------------------------------------------------------------------
// cv::resize(src -> dst) 8UC3 (background provider).  One thread = one dst pixel.
// ---------------------------------------------------------------------------
// One output pixel (dx, dy) of cv::resize 8UC3 of the sw x sh image `src` (rows spitch bytes apart): the exact 2x
// INTER_AREA mean (a+b+c+d+2)>>2 when area2x2, else INTER_LINEAR through the tables.  flip (bit 0 horizontally, bit 1
// vertically) mirrors the image before the resize (app/deepseg.cc:667-679): each tap's source coordinate is mirrored and
// its weight kept, which is not the same as mirroring the resized image (the fixed-point tables need not be symmetric).
// CN channels (3, or 4 for the BGRA output): OpenCV resizes channel by channel with the same tables.
template <int CN = 3>
BSB_D void resize_px(const uint8_t* src, int sw, int sh, size_t spitch, const ResizeTab& t, bool area2x2, int flip, int dx, int dy,
                     uint8_t* d) {
  if (area2x2) {
    int x0 = 2 * dx, x1 = 2 * dx + 1, y0 = 2 * dy, y1 = 2 * dy + 1;
    if (flip & 1) { x0 = sw - 1 - x0; x1 = sw - 1 - x1; }
    if (flip & 2) { y0 = sh - 1 - y0; y1 = sh - 1 - y1; }
    const uint8_t* s0 = src + (size_t)y0 * spitch;
    const uint8_t* s1 = src + (size_t)y1 * spitch;
#pragma unroll
    for (int c = 0; c < CN; ++c) d[c] = (uint8_t)((s0[CN * x0 + c] + s0[CN * x1 + c] + s1[CN * x0 + c] + s1[CN * x1 + c] + 2) >> 2);
    return;
  }
  int sx = __ldg(t.xofs + dx), sx1 = min(sx + 1, sw - 1);
  int y0 = __ldg(t.yofs0 + dy), y1 = __ldg(t.yofs1 + dy);
  if (flip & 1) { sx = sw - 1 - sx; sx1 = sw - 1 - sx1; }
  if (flip & 2) { y0 = sh - 1 - y0; y1 = sh - 1 - y1; }
  const int a0 = __ldg(t.xw + 2 * dx), a1 = __ldg(t.xw + 2 * dx + 1);
  const int b0 = __ldg(t.yw + 2 * dy), b1 = __ldg(t.yw + 2 * dy + 1);
  const uint8_t* r0 = src + (size_t)y0 * spitch;
  const uint8_t* r1 = src + (size_t)y1 * spitch;
#pragma unroll
  for (int c = 0; c < CN; ++c) d[c] = lin_v(lin_h(r0, sx, sx1, CN, c, a0, a1), lin_h(r1, sx, sx1, CN, c, a0, a1), b0, b1);
}

__global__ void __launch_bounds__(256) k_resize_u8c3(const uint8_t* src, int sw, int sh, size_t spitch,
                                                     uint8_t* dst, int dw, int dh, size_t dpitch, ResizeTab t, bool area2x2,
                                                     size_t sstride, size_t dstride) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)dw * dh) return;
  src += (size_t)blockIdx.y * sstride; dst += (size_t)blockIdx.y * dstride;
  const int dx = (int)(idx % dw), dy = (int)(idx / dw);
  resize_px(src, sw, sh, spitch, t, area2x2, 0, dx, dy, dst + (size_t)dy * dpitch + (size_t)dx * 3);
}

void launch_resize_u8c3(cudaStream_t s, const uint8_t* src, int sw, int sh, size_t spitch,
                        uint8_t* dst, int dw, int dh, size_t dpitch, ResizeTab tab, bool area2x2,
                        int n, size_t sstride, size_t dstride) {
  const long total = (long)dw * dh;
  BSB_LAUNCH(k_resize_u8c3, dim3((unsigned)((total + 255) / 256), (unsigned)n), dim3(256), 0, s, src, sw, sh, spitch, dst, dw, dh, dpitch, tab, area2x2,
             sstride, dstride);
  count_launch();
}

// ---------------------------------------------------------------------------
// Live backgrounds: the caller's device image of each frame resized to W x H (app/background.cc:178-194) inside the call.
// One thread = one 2x2 output block of one frame (frames along blockIdx.y), so the block's two YUYV words and its NV12
// come from registers.  NV12 images are never converted as a whole: each tap is converted where resize_px reads it
// (cv::cvtColor(COLOR_YUV2BGR_NV12) then cv::resize, as the pre-processing reads NV12 camera frames).
// ---------------------------------------------------------------------------
// output pixel (dx, dy) of live image d
BSB_D void live_px(const LiveDesc& d, int dx, int dy, uint8_t* o) {
  if (d.fmt == LIVE_BGR) { resize_px(d.p, d.w, d.h, d.pitch, d.tab, d.area2x2 != 0, 0, dx, dy, o); return; }
  int p00[3], p01[3], p10[3], p11[3];
  if (d.area2x2) {
    const int x0 = 2 * dx, y0 = 2 * dy;
    nv12_px_to_bgr(d.p, d.pitch, d.uv, x0, y0, p00); nv12_px_to_bgr(d.p, d.pitch, d.uv, x0 + 1, y0, p01);
    nv12_px_to_bgr(d.p, d.pitch, d.uv, x0, y0 + 1, p10); nv12_px_to_bgr(d.p, d.pitch, d.uv, x0 + 1, y0 + 1, p11);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)((p00[c] + p01[c] + p10[c] + p11[c] + 2) >> 2);
    return;
  }
  const int sx = __ldg(d.tab.xofs + dx), sx1 = min(sx + 1, d.w - 1);
  const int y0 = __ldg(d.tab.yofs0 + dy), y1 = __ldg(d.tab.yofs1 + dy);
  const int a0 = __ldg(d.tab.xw + 2 * dx), a1 = __ldg(d.tab.xw + 2 * dx + 1);
  const int b0 = __ldg(d.tab.yw + 2 * dy), b1 = __ldg(d.tab.yw + 2 * dy + 1);
  nv12_px_to_bgr(d.p, d.pitch, d.uv, sx, y0, p00); nv12_px_to_bgr(d.p, d.pitch, d.uv, sx1, y0, p01);
  nv12_px_to_bgr(d.p, d.pitch, d.uv, sx, y1, p10); nv12_px_to_bgr(d.p, d.pitch, d.uv, sx1, y1, p11);
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = lin_v(p00[c] * a0 + p01[c] * a1, p10[c] * a0 + p11[c] * a1, b0, b1);
}

__global__ void __launch_bounds__(256) k_live_bg(const LiveDesc* descs, uint8_t* slot, uint8_t* stage, uint8_t* yuyv, uint8_t* nv12,
                                                 int W, int H) {
  const int b = blockIdx.y;
  const LiveDesc d = descs[b];
  if (!d.p) return;
  const int hw = (W + 1) / 2;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)hw * ((H + 1) / 2)) return;
  const int x = (int)(i % hw) * 2, y = (int)(i / hw) * 2;
  const bool xr = x + 1 < W, yr = y + 1 < H;             // the block's right column / lower row exist
  uint8_t px[12];                                         // (x, y) (x+1, y) | (x, y+1) (x+1, y+1)
  live_px(d, x, y, px);
  if (xr) live_px(d, x + 1, y, px + 3);
  if (yr) {
    live_px(d, x, y + 1, px + 6);
    if (xr) live_px(d, x + 1, y + 1, px + 9);
  }
  const size_t npix = (size_t)W * H;
  uint8_t* o = (d.blur ? stage : slot) + (size_t)b * npix * 3 + ((size_t)y * W + x) * 3;
  const int nb = xr ? 6 : 3;
  for (int k = 0; k < nb; ++k) o[k] = px[k];
  if (yr) for (int k = 0; k < nb; ++k) o[(size_t)W * 3 + k] = px[6 + k];
  if (d.blur) return;
  if (nv12) {                                             // W and H even
    uint8_t* f = nv12 + (size_t)b * (npix * 3 / 2);
    nv12_block(yuyv_pair_word(px), yuyv_pair_word(px + 6), f + (size_t)y * W + x, W, f + npix + (size_t)(y / 2) * W + x);
  } else if (yuyv) {                                      // W even: the pixel pairs of convert_rgb_to_yuyv are row pairs
    unsigned* f = reinterpret_cast<unsigned*>(yuyv + (size_t)b * npix * 2);
    f[((size_t)y * W + x) / 2] = yuyv_pair_word(px);
    if (yr) f[((size_t)(y + 1) * W + x) / 2] = yuyv_pair_word(px + 6);
  }
}

void launch_live_bg(cudaStream_t s, int n, const LiveDesc* descs, uint8_t* slot, uint8_t* stage, uint8_t* yuyv, uint8_t* nv12, int W, int H) {
  const long blocks = ((long)((W + 1) / 2) * ((H + 1) / 2) + 255) / 256;
  BSB_LAUNCH(k_live_bg, dim3((unsigned)blocks, (unsigned)n), dim3(256), 0, s, descs, slot, stage, yuyv, nv12, W, H);
  count_launch();
}

// ---------------------------------------------------------------------------
// YUYV -> BGR ingest (cv::cvtColor COLOR_YUV2BGR_YUYV, BT.601 limited range, 20-bit fixed point).
// One thread = 8 pixels: one 16-byte load, 24 bytes out.
// ---------------------------------------------------------------------------
BSB_D void yuv2bgr_px(int y, int ruv, int guv, int buv, uint8_t* o) {
  const int yy = max(y - 16, 0) * 1220542;
  o[0] = bsb_sat_u8((yy + buv) >> 20); o[1] = bsb_sat_u8((yy + guv) >> 20); o[2] = bsb_sat_u8((yy + ruv) >> 20);
}

__global__ void __launch_bounds__(256) k_yuyv_to_bgr(const uint8_t* yuyv, uint8_t* bgr, size_t ngroups, size_t npix, int vec_ok) {
  const size_t gidx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gidx >= ngroups) return;          // (only in the last, partial block: full blocks reach the barrier below together)
  const size_t p0 = gidx * 8;
  const int n = (npix - p0) < 8 ? (int)(npix - p0) : 8;
  unsigned w[4] = {0u, 0u, 0u, 0u};     // 8 pixels = 4 words of Y0 U Y1 V
  if (n == 8) {
    const uint4 t = __ldg(reinterpret_cast<const uint4*>(yuyv + 2 * p0));
    w[0] = t.x; w[1] = t.y; w[2] = t.z; w[3] = t.w;
  } else {
    for (int i = 0; i < 2 * n; ++i) w[i >> 2] |= (unsigned)yuyv[2 * p0 + i] << (8 * (i & 3));
  }
  unsigned o[6];                              // 24 output bytes, assembled in registers
  yuyv8_to_bgr24(w, o);
  // full blocks: stage the 24-byte groups in shared memory and write 16-byte vectors (a warp then writes 768
  // contiguous bytes in 1.5 passes instead of three 8-byte-strided passes that each touch every sector)
  __shared__ __align__(16) uint2 stage[256 * 3];
  const size_t blk_p0 = (size_t)blockIdx.x * blockDim.x * 8;
  const bool full_block = blk_p0 + (size_t)blockDim.x * 8 <= npix && blockDim.x == 256 && vec_ok;
  if (full_block) {
    uint2* q = stage + threadIdx.x * 3;
    q[0] = make_uint2(o[0], o[1]); q[1] = make_uint2(o[2], o[3]); q[2] = make_uint2(o[4], o[5]);
    __syncthreads();
    uint4* dst = reinterpret_cast<uint4*>(bgr + 3 * blk_p0);
    const uint4* src = reinterpret_cast<const uint4*>(stage);
    dst[threadIdx.x] = src[threadIdx.x];
    if (threadIdx.x < 128) dst[256 + threadIdx.x] = src[256 + threadIdx.x];
    return;
  }
  uint8_t* d = bgr + 3 * p0;
  if (n == 8 && (reinterpret_cast<uintptr_t>(d) & 7) == 0) {
    uint2* q = reinterpret_cast<uint2*>(d);
    q[0] = make_uint2(o[0], o[1]); q[1] = make_uint2(o[2], o[3]); q[2] = make_uint2(o[4], o[5]);
  } else {
    for (int i = 0; i < 3 * n; ++i) d[i] = (uint8_t)(o[i >> 2] >> (8 * (i & 3)));
  }
}

void launch_yuyv_to_bgr(cudaStream_t s, const uint8_t* yuyv, uint8_t* bgr, size_t npix_total) {
  const size_t ngroups = (npix_total + 7) / 8;
  const int vec_ok = (reinterpret_cast<uintptr_t>(bgr) & 15) == 0 ? 1 : 0;
  BSB_LAUNCH(k_yuyv_to_bgr, dim3((unsigned)((ngroups + 255) / 256)), dim3(256), 0, s, yuyv, bgr, ngroups, npix_total, vec_ok);
  count_launch();
}

// ---------------------------------------------------------------------------
// Stand-alone alpha_blend / convert_rgb_to_yuyv (stage-level parity through the C-ABI).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_alpha_blend(const uint8_t* a, const uint8_t* b, const uint8_t* mask, uint8_t* out, size_t npix) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const unsigned aw = mask[p], bw = 255u - aw;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[3 * p + c] = (uint8_t)bsb_div255((unsigned)a[3 * p + c] * aw + (unsigned)b[3 * p + c] * bw);
}

void launch_alpha_blend(cudaStream_t s, const uint8_t* a, const uint8_t* b, const uint8_t* mask, uint8_t* out, size_t npix) {
  BSB_LAUNCH(k_alpha_blend, dim3((unsigned)((npix + 255) / 256)), dim3(256), 0, s, a, b, mask, out, npix);
  count_launch();
}

__global__ void __launch_bounds__(256) k_rgb_to_yuyv(const uint8_t* rgb, uint8_t* yuyv, size_t npairs, size_t rgb_stride, size_t yuyv_stride) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  rgb += (size_t)blockIdx.y * rgb_stride; yuyv += (size_t)blockIdx.y * yuyv_stride;
  const unsigned w = yuyv_pair_word(rgb + 6 * p);
  uint8_t* d = yuyv + 4 * p;
  d[0] = (uint8_t)w; d[1] = (uint8_t)(w >> 8); d[2] = (uint8_t)(w >> 16); d[3] = (uint8_t)(w >> 24);
}

void launch_rgb_to_yuyv(cudaStream_t s, const uint8_t* rgb, uint8_t* yuyv, size_t npix, int n, size_t rgb_stride, size_t yuyv_stride) {
  const size_t npairs = npix / 2;
  BSB_LAUNCH(k_rgb_to_yuyv, dim3((unsigned)((npairs + 255) / 256), (unsigned)n), dim3(256), 0, s, rgb, yuyv, npairs, rgb_stride, yuyv_stride);
  count_launch();
}

// ---------------------------------------------------------------------------
// NV12 <-> the project's YUYV / BGR (definitions in include/backscrub_b200.h).  Used where the post stage cannot read or
// write NV12 itself; one thread = a 2x2 pixel block (one UV pair), n frames along blockIdx.y.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_nv12_to_bgr(const uint8_t* nv12, size_t pitch, size_t uv_off, size_t in_stride, uint8_t* bgr,
                                                     int W, int H) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = W / 2;
  if (idx >= (long)hw * (H / 2)) return;
  const int x = (int)(idx % hw) * 2, y = (int)(idx / hw) * 2;
  const uint8_t* img = nv12 + (size_t)blockIdx.y * in_stride;
  const uint8_t* uv = img + uv_off + (size_t)(y >> 1) * pitch + x;
  const int u = uv[0], v = uv[1];
  uint8_t* d = bgr + (size_t)blockIdx.y * ((size_t)W * H * 3) + ((size_t)y * W + x) * 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const uint8_t* yr = img + (size_t)(y + r) * pitch + x;
    int p0[3], p1[3];
    yuv_px_to_bgr(yr[0], u, v, p0); yuv_px_to_bgr(yr[1], u, v, p1);
    uint8_t* o = d + (size_t)r * W * 3;
    o[0] = (uint8_t)p0[0]; o[1] = (uint8_t)p0[1]; o[2] = (uint8_t)p0[2]; o[3] = (uint8_t)p1[0]; o[4] = (uint8_t)p1[1]; o[5] = (uint8_t)p1[2];
  }
}

void launch_nv12_to_bgr(cudaStream_t s, int n, const uint8_t* nv12, size_t pitch, size_t uv_off, size_t in_stride, uint8_t* bgr, int W, int H) {
  const long blocks = ((long)(W / 2) * (H / 2) + 255) / 256;
  BSB_LAUNCH(k_nv12_to_bgr, dim3((unsigned)blocks, (unsigned)n), dim3(256), 0, s, nv12, pitch, uv_off, in_stride, bgr, W, H);
  count_launch();
}

// Y bytes copied; the UV pair of a 2x2 block is the truncating average of the two rows' (byte 1, byte 3) of the YUYV pair
__global__ void __launch_bounds__(256) k_yuyv_to_nv12(const uint8_t* yuyv, size_t yuyv_stride, uint8_t* nv12, size_t nv12_stride, int W, int H) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = W / 2;
  if (idx >= (long)hw * (H / 2)) return;
  const int j = (int)(idx % hw), r = (int)(idx / hw);
  const uint8_t* s0 = yuyv + (size_t)blockIdx.y * yuyv_stride + ((size_t)(2 * r) * W + 2 * j) * 2;
  const uint8_t* s1 = s0 + (size_t)W * 2;
  uint8_t* y0 = nv12 + (size_t)blockIdx.y * nv12_stride + (size_t)(2 * r) * W + 2 * j;
  uint8_t* y1 = y0 + W;
  y0[0] = s0[0]; y0[1] = s0[2]; y1[0] = s1[0]; y1[1] = s1[2];
  uint8_t* uv = nv12 + (size_t)blockIdx.y * nv12_stride + (size_t)W * H + (size_t)r * W + 2 * j;
  uv[0] = (uint8_t)((s0[1] + s1[1]) >> 1);
  uv[1] = (uint8_t)((s0[3] + s1[3]) >> 1);
}

void launch_yuyv_to_nv12(cudaStream_t s, int n, const uint8_t* yuyv, size_t yuyv_stride, uint8_t* nv12, size_t nv12_stride, int W, int H) {
  const long blocks = ((long)(W / 2) * (H / 2) + 255) / 256;
  BSB_LAUNCH(k_yuyv_to_nv12, dim3((unsigned)blocks, (unsigned)n), dim3(256), 0, s, yuyv, yuyv_stride, nv12, nv12_stride, W, H);
  count_launch();
}

// ---------------------------------------------------------------------------
// The call's tail (app/deepseg.cc:667-681): flip -> resize -> YUYV / NV12 of the staged composites, frames along
// blockIdx.y.  YUYV: one thread = one flat pixel pair of the packed output (convert_rgb_to_yuyv walks total(), so with an
// odd width a pair spans a row end; a last odd pixel has no pair).  NV12: one thread = one 2x2 block, whose two YUYV
// words give its Y bytes and UV pair directly.
// ---------------------------------------------------------------------------
// pixel (x, y) of frame geometry g: the mirrored copy when g is the staged size, else the mirrored resize (CN channels)
template <int CN = 3>
BSB_D void tail_px(const uint8_t* src, int W, int H, const TailGeo& g, int flip, int x, int y, uint8_t* d) {
  if (g.ow == W && g.oh == H) {
    const uint8_t* s = src + ((size_t)((flip & 2) ? H - 1 - y : y) * W + ((flip & 1) ? W - 1 - x : x)) * CN;
#pragma unroll
    for (int c = 0; c < CN; ++c) d[c] = s[c];
  } else {
    resize_px<CN>(src, W, H, (size_t)W * CN, g.tab, g.area2x2 != 0, flip, x, y, d);
  }
}

// pixel (x, y) of a framed frame: crop cr = (x, y, w, h) of the staged W-wide frame, mirrored within the crop, then
// resized to ow x oh as resize_px does (a crop of the output size is a copy, an exact 2x crop the INTER_AREA mean); the
// taps come from resize_taps.h, on the fly (sx_scale / sy_scale: resize_scale of the crop to the output)
template <int CN = 3>
BSB_D void crop_px(const uint8_t* src, int W, const int4& cr, int ow, int oh, double sx_scale, double sy_scale, int flip, int x, int y,
                   uint8_t* d) {
  const size_t sp = (size_t)W * CN;
  src += (size_t)cr.y * sp + (size_t)cr.x * CN;
  if (cr.z == ow && cr.w == oh) {
    const uint8_t* s = src + (size_t)((flip & 2) ? cr.w - 1 - y : y) * sp + (size_t)((flip & 1) ? cr.z - 1 - x : x) * CN;
#pragma unroll
    for (int c = 0; c < CN; ++c) d[c] = s[c];
    return;
  }
  if (cr.z == 2 * ow && cr.w == 2 * oh) {
    int x0 = 2 * x, x1 = 2 * x + 1, y0 = 2 * y, y1 = 2 * y + 1;
    if (flip & 1) { x0 = cr.z - 1 - x0; x1 = cr.z - 1 - x1; }
    if (flip & 2) { y0 = cr.w - 1 - y0; y1 = cr.w - 1 - y1; }
    const uint8_t* s0 = src + (size_t)y0 * sp;
    const uint8_t* s1 = src + (size_t)y1 * sp;
#pragma unroll
    for (int c = 0; c < CN; ++c) d[c] = (uint8_t)((s0[CN * x0 + c] + s0[CN * x1 + c] + s1[CN * x0 + c] + s1[CN * x1 + c] + 2) >> 2);
    return;
  }
  int sx, a0, a1, y0, y1, b0, b1;
  resize_tap_x(x, sx_scale, cr.z, &sx, &a0, &a1);
  resize_tap_y(y, sy_scale, cr.w, &y0, &y1, &b0, &b1);
  int sx1 = min(sx + 1, cr.z - 1);
  if (flip & 1) { sx = cr.z - 1 - sx; sx1 = cr.z - 1 - sx1; }
  if (flip & 2) { y0 = cr.w - 1 - y0; y1 = cr.w - 1 - y1; }
  const uint8_t* r0 = src + (size_t)y0 * sp;
  const uint8_t* r1 = src + (size_t)y1 * sp;
#pragma unroll
  for (int c = 0; c < CN; ++c) d[c] = lin_v(lin_h(r0, sx, sx1, CN, c, a0, a1), lin_h(r1, sx, sx1, CN, c, a0, a1), b0, b1);
}

// the frame's crop and its resize steps (framed calls)
struct TailCrop { int4 cr; double sx, sy; };

template <int CN = 3, bool CROP = false>
BSB_D void tail_pick(const uint8_t* src, int W, int H, const TailGeo& g, const TailCrop& k, int flip, int x, int y, uint8_t* d) {
  if (CROP) crop_px<CN>(src, W, k.cr, g.ow, g.oh, k.sx, k.sy, flip, x, y, d);
  else tail_px<CN>(src, W, H, g, flip, x, y, d);
}

// BGRA: TailArgs::bgra, the output is the transparent BGRA (from src4; the BGR composite is read for the video only).
// CROP: TailArgs::crop, a framed call (a separate instantiation: the unframed tails compile as before)
template <bool BGRA, bool CROP = false>
__global__ void __launch_bounds__(256) k_tail(TailArgs a) {
  const int b = blockIdx.y;
  const TailGeo g = a.slot ? a.geos[__ldg(a.slot + b)] : a.geo;
  TailCrop k{};
  if (CROP) {
    const FrameCrop& c = a.crop[__ldg(a.crop_idx + b)];
    k.cr = make_int4(c.x, c.y, c.w, c.h); k.sx = c.sx; k.sy = c.sy;
  }
  const int fl = a.flips ? __ldg(a.flips + b) : a.flip;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long npx = (long)g.ow * g.oh;
  const uint8_t* src = a.src + (size_t)b * a.src_stride;
  uint8_t* out = a.out ? a.out + (size_t)b * a.out_stride : nullptr;
  uint8_t* vid = a.video ? a.video + (size_t)b * a.video_stride : nullptr;
  const uint8_t* src4 = BGRA ? a.src4 + (size_t)b * a.src4_stride : nullptr;
  if (a.nv12) {
    if (i >= npx / 4) return;
    const int hw = g.ow / 2, x = (int)(i % hw) * 2, y = (int)(i / hw) * 2;
    uint8_t px[12];                                   // (x, y) (x+1, y) | (x, y+1) (x+1, y+1)
    if (!BGRA || vid) {
      tail_pick<3, CROP>(src, a.W, a.H, g, k, fl, x, y, px);
      tail_pick<3, CROP>(src, a.W, a.H, g, k, fl, x + 1, y, px + 3);
      tail_pick<3, CROP>(src, a.W, a.H, g, k, fl, x, y + 1, px + 6);
      tail_pick<3, CROP>(src, a.W, a.H, g, k, fl, x + 1, y + 1, px + 9);
    }
    if (BGRA && out) {
      uint8_t* o = out + ((size_t)y * g.ow + x) * 4;
      tail_pick<4, CROP>(src4, a.W, a.H, g, k, fl, x, y, o);
      tail_pick<4, CROP>(src4, a.W, a.H, g, k, fl, x + 1, y, o + 4);
      tail_pick<4, CROP>(src4, a.W, a.H, g, k, fl, x, y + 1, o + (size_t)g.ow * 4);
      tail_pick<4, CROP>(src4, a.W, a.H, g, k, fl, x + 1, y + 1, o + (size_t)g.ow * 4 + 4);
    } else if (out) {
      uint8_t* o = out + ((size_t)y * g.ow + x) * 3;
#pragma unroll
      for (int k = 0; k < 6; ++k) { o[k] = px[k]; o[(size_t)g.ow * 3 + k] = px[6 + k]; }
    }
    if (vid) nv12_block(yuyv_pair_word(px), yuyv_pair_word(px + 6), vid + (size_t)y * g.ow + x, g.ow, vid + npx + (size_t)(y / 2) * g.ow + x);
    return;
  }
  const long p = 2 * i;
  if (p >= npx) return;
  const bool pair = p + 1 < npx;
  uint8_t px[6];
  if (!BGRA || vid) {
    tail_pick<3, CROP>(src, a.W, a.H, g, k, fl, (int)(p % g.ow), (int)(p / g.ow), px);
    if (pair) tail_pick<3, CROP>(src, a.W, a.H, g, k, fl, (int)((p + 1) % g.ow), (int)((p + 1) / g.ow), px + 3);
  }
  if (BGRA && out) {
    tail_pick<4, CROP>(src4, a.W, a.H, g, k, fl, (int)(p % g.ow), (int)(p / g.ow), out + 4 * p);
    if (pair) tail_pick<4, CROP>(src4, a.W, a.H, g, k, fl, (int)((p + 1) % g.ow), (int)((p + 1) / g.ow), out + 4 * p + 4);
  } else if (out) {
    uint8_t* o = out + 3 * p;
    o[0] = px[0]; o[1] = px[1]; o[2] = px[2];
    if (pair) { o[3] = px[3]; o[4] = px[4]; o[5] = px[5]; }
  }
  if (vid && pair) {
    const unsigned w = yuyv_pair_word(px);
    uint8_t* v = vid + 4 * i;
    if ((reinterpret_cast<uintptr_t>(v) & 3) == 0) {
      *reinterpret_cast<unsigned*>(v) = w;
    } else {
      v[0] = (uint8_t)w; v[1] = (uint8_t)(w >> 8); v[2] = (uint8_t)(w >> 16); v[3] = (uint8_t)(w >> 24);
    }
  }
}

void launch_tail(cudaStream_t s, const TailArgs& a, long max_px) {
  const long threads = (max_px + 1) / 2;
  const dim3 grid((unsigned)((threads + 255) / 256), (unsigned)a.n);
  if (a.crop) {
    if (a.bgra) { auto k = k_tail<true, true>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
    else { auto k = k_tail<false, true>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  } else if (a.bgra) { auto k = k_tail<true>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else { auto k = k_tail<false>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  count_launch();
}

// ---------------------------------------------------------------------------
// Framing (framing.h): one CTA = one frame's small mask; warps walk rows, lanes columns (coalesced), then a warp and a
// block reduction of the person count and box.  Plain calls step the context's one state in frame order, so the CTA
// that arrives last (as k_rowsum_fc's tail does) walks the frames' boxes; sources frames step distinct states at once.
// ---------------------------------------------------------------------------
// the crop record of one frame: the crop and the resize steps from it to the frame's output size
BSB_D void framing_put(FrameCrop* o, const int* c, int ow, int oh) {
  o->x = c[0]; o->y = c[1]; o->w = c[2]; o->h = c[3];
  o->sx = resize_scale(c[2], ow); o->sy = resize_scale(c[3], oh);
}

__global__ void __launch_bounds__(256) k_framing(FramingArgs a) {
  const int b = blockIdx.x, mb = a.mb;
  const int mode = __ldg(a.tab + b), ci = __ldg(a.tab + 9 * mb + b);
  const int ow = __ldg(a.tab + 3 * mb + b), oh = __ldg(a.tab + 4 * mb + b);
  if (mode != FRAMING_AUTO) {
    if (threadIdx.x == 0) {
      int c[4];
      for (int k = 0; k < 4; ++k) c[k] = __ldg(a.tab + (5 + k) * mb + b);
      framing_put(a.crop + ci, c, ow, oh);
    }
    return;
  }
  const int sw = a.g.sw, sh = a.g.sh, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint8_t* m = a.ofinal + ((size_t)b * a.oh + a.oy) * a.opitch + a.ox;
  int v[5] = {0, 1 << 30, 1 << 30, -1, -1};          // count, j0, i0, j1, i1
  for (int i = warp; i < sh; i += 8)
    for (int j = lane; j < sw; j += 32)
      if (m[(size_t)i * a.opitch + j] < 128) {
        ++v[0]; v[1] = min(v[1], j); v[2] = min(v[2], i); v[3] = max(v[3], j); v[4] = max(v[4], i);
      }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
    v[1] = min(v[1], __shfl_xor_sync(0xffffffffu, v[1], o)); v[2] = min(v[2], __shfl_xor_sync(0xffffffffu, v[2], o));
    v[3] = max(v[3], __shfl_xor_sync(0xffffffffu, v[3], o)); v[4] = max(v[4], __shfl_xor_sync(0xffffffffu, v[4], o));
  }
  __shared__ int part[8][5];
  __shared__ int last;
  if (lane == 0)
    for (int k = 0; k < 5; ++k) part[warp][k] = v[k];
  __syncthreads();
  int t[4];
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) {
      v[0] += part[w][0];
      v[1] = min(v[1], part[w][1]); v[2] = min(v[2], part[w][2]); v[3] = max(v[3], part[w][3]); v[4] = max(v[4], part[w][4]);
    }
    framing_target(FramingBox{v[0], v[1], v[2], v[3], v[4]}, a.g, a.p, ow, oh, t);
    if (!a.plain) {
      int c[4];
      int* st = a.state + 4 * __ldg(a.tab + 2 * mb + b);
      framing_step(st, t, a.p.speed, __ldg(a.tab + mb + b) != 0);
      framing_crop(st, a.g.W, a.g.H, c);
      framing_put(a.crop + ci, c, ow, oh);
    } else {
      // the targets need no state, so every CTA makes its own; the CTA that arrives last steps them in frame order
      for (int k = 0; k < 4; ++k) a.targets[4 * b + k] = t[k];
      __threadfence();
      last = atomicAdd(a.counter, 1u) == (unsigned)a.n - 1;
    }
  }
  if (!a.plain) return;
  __syncthreads();
  if (!last) return;
  __shared__ int tg[4 * 256];
  __threadfence();
  int st[4];
  for (int k = 0; k < 4; ++k) st[k] = a.state[k];
  for (int f0 = 0; f0 < a.n; f0 += 256) {               // the targets of 256 frames at a time, loaded in parallel
    const int nf = min(256, a.n - f0);
    __syncthreads();
    for (int k = threadIdx.x; k < 4 * nf; k += blockDim.x) tg[k] = __ldcg(a.targets + 4 * f0 + k);
    __syncthreads();
    if (threadIdx.x == 0)
      for (int f = f0; f < f0 + nf; ++f) {
        int c[4];
        framing_step(st, tg + 4 * (f - f0), a.p.speed, __ldg(a.tab + mb + f) != 0);
        framing_crop(st, a.g.W, a.g.H, c);
        framing_put(a.crop + __ldg(a.tab + 9 * mb + f), c, __ldg(a.tab + 3 * mb + f), __ldg(a.tab + 4 * mb + f));
      }
  }
  if (threadIdx.x) return;
  for (int k = 0; k < 4; ++k) a.state[k] = st[k];
  *a.counter = 0;                                    // the next launch starts from 0 (stream order)
}

void launch_framing(cudaStream_t s, const FramingArgs& a) {
  BSB_LAUNCH(k_framing, dim3((unsigned)a.n), dim3(256), 0, s, a);
  count_launch();
}

// ---------------------------------------------------------------------------
// Mask edge refinement: the range weights (include/backscrub_b200.h, bsb_mask_refine_weights)
// ---------------------------------------------------------------------------
bool refine_weights(int sigma, int* w) {
  if (sigma < 1 || sigma > 255) return false;
  for (int d = 0; d < 256; ++d) {
    const int v = (int)std::floor(256.0 * std::exp(-(double)d * d / (2.0 * sigma * sigma)) + 0.5);
    w[d] = v < 1 ? 1 : v;
  }
  return true;
}

const unsigned short* refine_tables() {
  static std::mutex mu;
  static std::map<int, unsigned short*> tabs;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  auto it = tabs.find(dev);
  if (it != tabs.end()) return it->second;
  std::vector<unsigned short> h((size_t)255 * 256);
  int w[256];
  for (int sg = 1; sg <= 255; ++sg) {
    refine_weights(sg, w);
    for (int d = 0; d < 256; ++d) h[(size_t)(sg - 1) * 256 + d] = (unsigned short)w[d];
  }
  unsigned short* d = nullptr;
  if (cudaMalloc((void**)&d, h.size() * sizeof(unsigned short)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.data(), h.size() * sizeof(unsigned short), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  tabs[dev] = d;
  return d;
}

}  // namespace bsb
