// backscrub_b200/csrc/kernels_nn.cu — fp32 CNN kernels for sm_90a (CUDA cores).
//
// These replace the XNNPACK/TFLite CPU kernels behind Interpreter::Invoke()
// (lib/libbackscrub.cc:307; op semantics: reference tensorflow/lite/kernels/internal/
// reference/{conv,depthwiseconv_float,pooling,resize_bilinear,hard_swish,logistic,
// fully_connected}.h and lib/transpose_conv_bias.cc).  Every output element accumulates
// its products with fmaf in the reference loop order (ky, kx, cin), so results are
// bit-identical to the CPU oracle; parallelism comes from pixels x channels x frames.
#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>

#include "kernels.h"

namespace bsb {

static std::atomic<long> g_launches{0};
long launch_count() { return g_launches.load(); }
static thread_local long t_launches = 0;
long thread_launch_count() { return t_launches; }
void count_launch() { g_launches.fetch_add(1); ++t_launches; }

Tuning& tuning() { static Tuning t; return t; }

bool ensure_dyn_smem(const void* func, size_t bytes) {
#ifdef BSB_EMU
  (void)func; (void)bytes;
  return true;
#else
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> configured;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  std::lock_guard<std::mutex> lock(mu);
  const auto key = std::make_pair(dev, func);
  auto it = configured.find(key);
  if (it == configured.end()) {
    // without the opt-in attribute a block gets 48 KB of shared memory in all: the kernel's static share plus the dynamic
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, func) != cudaSuccess) { cudaGetLastError(); return false; }
    it = configured.emplace(key, 48 * 1024 - std::min<size_t>(fa.sharedSizeBytes, 48 * 1024)).first;
  }
  size_t& have = it->second;
  if (bytes <= have) return true;
  if (cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) { cudaGetLastError(); return false; }
  have = bytes;
  return true;
#endif
}

int device_sms() {
#ifdef BSB_EMU
  return 132;
#else
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
    cudaGetLastError();
    return 132;
  }
  return n;
#endif
}

struct EpiDev {
  const float* bias; const float* residual; int ld_res; int act1, act2, act3;
};
static inline EpiDev to_dev(const Epilogue& e) { return EpiDev{e.bias, e.residual, e.ld_res, e.act1, e.act2, e.act3}; }

BSB_D float epilogue(float total, int ch, size_t pix, const EpiDev& e) {
  float v = total + (e.bias ? __ldg(e.bias + ch) : 0.f);
  v = bsb_act(v, e.act1);
  v = bsb_act(v, e.act2);
  if (e.residual) v = bsb_act(v + __ldg(e.residual + pix * (size_t)e.ld_res + ch), e.act3);
  return v;
}

// Compile-time epilogue.  The generic one above costs ~25 instructions per value (a bias load from global memory at the
// very end of the kernel, two activation switches, a residual test), a large share of the 16 -> 16 1x1 conv of the Meet
// graph.  MODE < 0: that generic path.
// MODE >= 0: value = act(acc + bias) with act = MODE & 7 fixed at compile time and the bias preloaded by the caller
// (before its main loop); MODE & 8: + residual, no activation after it.  Same operations in the same order as the generic
// path for these combinations (a missing bias is + 0.f there and here), so the bits are unchanged.
template <int MODE>
BSB_D float epilogue_m(float total, float bias, int ch, size_t pix, const EpiDev& e) {
  if (MODE < 0) return epilogue(total, ch, pix, e);
  float v = bsb_act(total + bias, MODE & 7);
  if (MODE & 8) v = v + __ldg(e.residual + pix * (size_t)e.ld_res + ch);
  return v;
}
template <int MODE>
BSB_D float4 epilogue_bias4(const EpiDev& e, int ch0, int N) {
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  if (MODE >= 0 && e.bias) {
    if (ch0 + 3 < N) { b.x = __ldg(e.bias + ch0); b.y = __ldg(e.bias + ch0 + 1); b.z = __ldg(e.bias + ch0 + 2); b.w = __ldg(e.bias + ch0 + 3); }
    else { if (ch0 < N) b.x = __ldg(e.bias + ch0); if (ch0 + 1 < N) b.y = __ldg(e.bias + ch0 + 1); if (ch0 + 2 < N) b.z = __ldg(e.bias + ch0 + 2); }
  }
  return b;
}
// the combinations the five bundled graphs use outside the chain kernel; anything else runs the generic path
static int epi_mode(const Epilogue& e) {
  if (!tuning().epi_static) return -1;
  int act;
  if (e.act1 == ACT_NONE) act = e.act2; else if (e.act2 == ACT_NONE) act = e.act1; else return -1;
  int mode;
  if (!e.residual) mode = act; else if (e.act3 == ACT_NONE) mode = 8 | act; else return -1;
  return (mode == 0 || mode == 1 || mode == 3 || mode == 4 || mode == 8 || mode == 11) ? mode : -1;
}
template <int M> struct EpiTag { static constexpr int value = M; };
template <class F> static void epi_dispatch(int mode, F&& f) {
  switch (mode) {
    case 0: f(EpiTag<0>{}); break;
    case 1: f(EpiTag<1>{}); break;
    case 3: f(EpiTag<3>{}); break;
    case 4: f(EpiTag<4>{}); break;
    case 8: f(EpiTag<8>{}); break;
    case 11: f(EpiTag<11>{}); break;
    default: f(EpiTag<-1>{}); break;
  }
}

// four adjacent channels of one row, as a real call: keeps the 32/64-output epilogue of the register-tiled
// kernel from being unrolled into tens of thousands of instructions
BSB_D_NOINLINE float4 epilogue4(float4 v, int ch, size_t pix, const EpiDev& e) {
  return make_float4(epilogue(v.x, ch, pix, e), epilogue(v.y, ch + 1, pix, e), epilogue(v.z, ch + 2, pix, e), epilogue(v.w, ch + 3, pix, e));
}
BSB_D_NOINLINE float epilogue1(float v, int ch, size_t pix, const EpiDev& e) { return epilogue(v, ch, pix, e); }

// ---------------------------------------------------------------------------
// Dense KxK conv, small Cin (stem).  One thread = one output pixel x 4 output channels.
// Weights [kh][kw][ic][oc4] staged in shared memory (broadcast reads).
// ---------------------------------------------------------------------------
struct ConvArgs {
  const float* in; const float* w; float* out;
  int B, ih, iw, ic, ld_in, oc, oc4, kh, kw, sh, sw, dh, dw, pt, pl, oh, ow, ld_out;
  EpiDev e;
};

__global__ void __launch_bounds__(256) k_conv_direct(ConvArgs a) {
  BSB_DYN_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);
  const int wcount = a.kh * a.kw * a.ic * a.oc4;
  for (int i = threadIdx.x; i < wcount; i += blockDim.x) ws[i] = __ldg(a.w + i);
  __syncthreads();
  const int groups = a.oc4 / 4;
  const long total = (long)a.B * a.oh * a.ow * groups;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % groups);
  const long pix = idx / groups;
  const int ox = (int)(pix % a.ow);
  const int oy = (int)((pix / a.ow) % a.oh);
  const int b = (int)(pix / ((long)a.ow * a.oh));
  const float* inb = a.in + (size_t)b * a.ih * a.iw * a.ld_in;
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
  const int iy0 = oy * a.sh - a.pt, ix0 = ox * a.sw - a.pl;
  for (int fy = 0; fy < a.kh; ++fy) {
    const int iy = iy0 + a.dh * fy;
    if (iy < 0 || iy >= a.ih) continue;
    for (int fx = 0; fx < a.kw; ++fx) {
      const int ix = ix0 + a.dw * fx;
      if (ix < 0 || ix >= a.iw) continue;
      const float* ip = inb + ((size_t)iy * a.iw + ix) * a.ld_in;
      const float* wp = ws + ((fy * a.kw + fx) * a.ic) * a.oc4 + g * 4;
      for (int c = 0; c < a.ic; ++c) {
        const float v = __ldg(ip + c);
        const float4 w4 = *reinterpret_cast<const float4*>(wp + c * a.oc4);
        acc0 = fmaf(v, w4.x, acc0); acc1 = fmaf(v, w4.y, acc1);
        acc2 = fmaf(v, w4.z, acc2); acc3 = fmaf(v, w4.w, acc3);
      }
    }
  }
  float* op = a.out + (size_t)pix * a.ld_out;
  const float accs[4] = {acc0, acc1, acc2, acc3};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ch = g * 4 + j;
    if (ch < a.oc) op[ch] = epilogue(accs[j], ch, (size_t)pix, a.e);
  }
}

void launch_conv_direct(cudaStream_t s, int B, const float* in, int ih, int iw, int ic, int ld_in,
                        const float* w_t, int oc, int kh, int kw, int stride_h, int stride_w,
                        int dil_h, int dil_w, int pad_t, int pad_l,
                        float* out, int oh, int ow, int ld_out, const Epilogue& e) {
  ConvArgs a{in, w_t, out, B, ih, iw, ic, ld_in, oc, (oc + 3) / 4 * 4, kh, kw, stride_h, stride_w, dil_h, dil_w,
             pad_t, pad_l, oh, ow, ld_out, to_dev(e)};
  const long total = (long)B * oh * ow * (a.oc4 / 4);
  const size_t smem = sizeof(float) * (size_t)kh * kw * ic * a.oc4;
  // the planner admits up to 96 KB of weights (engine.cu); above 48 KB the kernel needs the opt-in attribute
  ensure_dyn_smem(reinterpret_cast<const void*>(k_conv_direct), smem);
  BSB_LAUNCH(k_conv_direct, dim3((unsigned)((total + 255) / 256)), dim3(256), smem, s, a);
  count_launch();
}

// ---------------------------------------------------------------------------
// Stem conv on the u8 image: one thread = one output pixel x all 16 output channels.
// Each tap value is fmaf((float)u8, scale, offset) — exactly what convertTo stores — and the
// accumulation order is the reference's (fy, fx, c).
// ---------------------------------------------------------------------------
struct StemArgs {
  const uint8_t* in; const float* w; float* out;
  int B, ih, iw, kh, kw, sh, sw, pt, pl, oh, ow, ld_out;
  float scale, offset;
  EpiDev e;
  // optional fused 1x1 conv 16 -> 16 on the stem's output (the thread already holds the pixel's 16 channels):
  // out2[p][n] = act(sum_k out[p][k] * w2[k][n] + bias2), k ascending — the same chain the stand-alone kernel computes
  const float* w2; float* out2; int ld_out2; EpiDev e2;
};

template <int MODE>
__global__ void __launch_bounds__(128) k_stem_u8(StemArgs a) {
  BSB_DYN_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);     // [kh][kw][3][16] | [16][16] second stage | [16] bias
  const int wcount = a.kh * a.kw * 3 * 16;
  for (int i = threadIdx.x; i < wcount; i += blockDim.x) ws[i] = __ldg(a.w + i);
  if (a.w2) for (int i = threadIdx.x; i < 256; i += blockDim.x) ws[wcount + i] = __ldg(a.w2 + i);
  float* bs = ws + wcount + 256;
  if (MODE >= 0 && threadIdx.x < 16) bs[threadIdx.x] = a.e.bias ? __ldg(a.e.bias + threadIdx.x) : 0.f;
  __syncthreads();
  const long total = (long)a.B * a.oh * a.ow;
  const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = pix < total;
  float acc[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) acc[o] = 0.f;
  if (valid) {
    const int ox = (int)(pix % a.ow), oy = (int)((pix / a.ow) % a.oh), b = (int)(pix / ((long)a.ow * a.oh));
    const uint8_t* inb = a.in + (size_t)b * a.ih * a.iw * 3;
    const int iy0 = oy * a.sh - a.pt, ix0 = ox * a.sw - a.pl;
    for (int fy = 0; fy < a.kh; ++fy) {
      const int iy = iy0 + fy;
      if (iy < 0 || iy >= a.ih) continue;
      for (int fx = 0; fx < a.kw; ++fx) {
        const int ix = ix0 + fx;
        if (ix < 0 || ix >= a.iw) continue;
        const uint8_t* ip = inb + ((size_t)iy * a.iw + ix) * 3;
        const float* wp = ws + (fy * a.kw + fx) * 48;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float v = fmaf((float)ip[c], a.scale, a.offset);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 w4 = *reinterpret_cast<const float4*>(wp + c * 16 + q * 4);
            acc[4 * q] = fmaf(v, w4.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, w4.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(v, w4.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, w4.w, acc[4 * q + 3]);
          }
        }
      }
    }
  }
  float4 r[4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
    r[q] = valid ? make_float4(epilogue_m<MODE>(acc[4 * q], MODE >= 0 ? bs[4 * q] : 0.f, 4 * q, (size_t)pix, a.e),
                               epilogue_m<MODE>(acc[4 * q + 1], MODE >= 0 ? bs[4 * q + 1] : 0.f, 4 * q + 1, (size_t)pix, a.e),
                               epilogue_m<MODE>(acc[4 * q + 2], MODE >= 0 ? bs[4 * q + 2] : 0.f, 4 * q + 2, (size_t)pix, a.e),
                               epilogue_m<MODE>(acc[4 * q + 3], MODE >= 0 ? bs[4 * q + 3] : 0.f, 4 * q + 3, (size_t)pix, a.e))
                 : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 r2[4];
  if (a.w2) {
    // second stage: 16 x 16 weights [k][n] behind the stem weights in shared memory
    const float* w2s = ws + wcount;
    float acc2[16];
#pragma unroll
    for (int n = 0; n < 16; ++n) acc2[n] = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float xk = k % 4 == 0 ? r[k / 4].x : (k % 4 == 1 ? r[k / 4].y : (k % 4 == 2 ? r[k / 4].z : r[k / 4].w));
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 w4 = *reinterpret_cast<const float4*>(w2s + k * 16 + q * 4);
        acc2[4 * q] = fmaf(xk, w4.x, acc2[4 * q]); acc2[4 * q + 1] = fmaf(xk, w4.y, acc2[4 * q + 1]);
        acc2[4 * q + 2] = fmaf(xk, w4.z, acc2[4 * q + 2]); acc2[4 * q + 3] = fmaf(xk, w4.w, acc2[4 * q + 3]);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
      r2[q] = valid ? make_float4(epilogue(acc2[4 * q], 4 * q, (size_t)pix, a.e2), epilogue(acc2[4 * q + 1], 4 * q + 1, (size_t)pix, a.e2),
                                  epilogue(acc2[4 * q + 2], 4 * q + 2, (size_t)pix, a.e2), epilogue(acc2[4 * q + 3], 4 * q + 3, (size_t)pix, a.e2))
                    : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (a.ld_out == 16 && (!a.w2 || a.ld_out2 == 16)) {
    // packed output: a thread's 16 channels are 64 contiguous bytes, so four strided float4 stores per thread would
    // touch every sector four times; transpose through shared memory and let the block write 8 KB contiguously
    __shared__ float4 stage[4 * 129];
#pragma unroll
    for (int q = 0; q < 4; ++q) stage[q * 129 + threadIdx.x] = r[q];
    __syncthreads();
    const long blk0 = (long)blockIdx.x * blockDim.x;
    float4* dst = reinterpret_cast<float4*>(a.out + (size_t)blk0 * 16);
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int j = it * 128 + threadIdx.x;                   // float4 index inside the block's output: pixel j / 4, quad j % 4
      if (blk0 + (j >> 2) < total) dst[j] = stage[(j & 3) * 129 + (j >> 2)];
    }
    if (a.w2) {
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 4; ++q) stage[q * 129 + threadIdx.x] = r2[q];
      __syncthreads();
      float4* dst2 = reinterpret_cast<float4*>(a.out2 + (size_t)blk0 * 16);
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int j = it * 128 + threadIdx.x;
        if (blk0 + (j >> 2) < total) dst2[j] = stage[(j & 3) * 129 + (j >> 2)];
      }
    }
    return;
  }
  if (!valid) return;
  float* op = a.out + (size_t)pix * a.ld_out;
#pragma unroll
  for (int q = 0; q < 4; ++q) *reinterpret_cast<float4*>(op + 4 * q) = r[q];
  if (a.w2) {
    float* op2 = a.out2 + (size_t)pix * a.ld_out2;
#pragma unroll
    for (int q = 0; q < 4; ++q) *reinterpret_cast<float4*>(op2 + 4 * q) = r2[q];
  }
}

// Two horizontally adjacent output pixels per thread (3x3, stride 2, even output width, packed 16-channel output — the
// stems of the Meet / MLKit graphs).  The one-pixel kernel above issues 108 LDS.128 of weights and 27 byte loads behind
// bounds tests per 432 fmaf; here the weight vectors are shared by the two pixels (108 LDS.128 per 864 fmaf), the 3 x 5
// input window (one shared column) is fetched up front with predicated loads, all in flight together, and out-of-image
// taps enter as +0 instead of being skipped: fmaf(+0, w, acc) leaves an accumulator that started at +0 unchanged bit
// for bit, so each output still sees exactly the oracle's (fy, fx, c) chain.
template <int MODE>
__global__ void __launch_bounds__(128) k_stem_u8_x2(StemArgs a) {
  __shared__ __align__(16) float ws[27 * 16];           // [3][3][3][16]
  __shared__ __align__(16) float bs[16];
  __shared__ float4 stage[8 * 129];
  for (int i = threadIdx.x; i < 27 * 16; i += blockDim.x) ws[i] = __ldg(a.w + i);
  if (threadIdx.x < 16) bs[threadIdx.x] = a.e.bias ? __ldg(a.e.bias + threadIdx.x) : 0.f;
  __syncthreads();
  const long total = (long)a.B * a.oh * a.ow;           // even: ow is even
  const long blk0 = (long)blockIdx.x * 256;
  const long pix = blk0 + 2 * threadIdx.x;              // this thread's pixels: pix, pix + 1 (same row)
  const bool valid = pix < total;
  float acc[2][16];
#pragma unroll
  for (int o = 0; o < 16; ++o) { acc[0][o] = 0.f; acc[1][o] = 0.f; }
  if (valid) {
    const int ox = (int)(pix % a.ow), oy = (int)((pix / a.ow) % a.oh), b = (int)(pix / ((long)a.ow * a.oh));
    const uint8_t* inb = a.in + (size_t)b * a.ih * a.iw * 3;
    const int iy0 = oy * 2 - a.pt, ix0 = ox * 2 - a.pl;
    float v[3][5][3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = iy0 + r;
      const bool vy = iy >= 0 && iy < a.ih;
#pragma unroll
      for (int c5 = 0; c5 < 5; ++c5) {
        const int ix = ix0 + c5;
        const bool ok = vy && ix >= 0 && ix < a.iw;
        const uint8_t* ip = inb + ((size_t)(ok ? iy : 0) * a.iw + (ok ? ix : 0)) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[r][c5][c] = ok ? fmaf((float)ip[c], a.scale, a.offset) : 0.f;
      }
    }
#pragma unroll
    for (int fy = 0; fy < 3; ++fy)
#pragma unroll
      for (int fx = 0; fx < 3; ++fx)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float* wp = ws + ((fy * 3 + fx) * 3 + c) * 16;
          const float v0 = v[fy][fx][c], v1 = v[fy][fx + 2][c];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 w4 = *reinterpret_cast<const float4*>(wp + q * 4);
            acc[0][4 * q] = fmaf(v0, w4.x, acc[0][4 * q]); acc[0][4 * q + 1] = fmaf(v0, w4.y, acc[0][4 * q + 1]);
            acc[0][4 * q + 2] = fmaf(v0, w4.z, acc[0][4 * q + 2]); acc[0][4 * q + 3] = fmaf(v0, w4.w, acc[0][4 * q + 3]);
            acc[1][4 * q] = fmaf(v1, w4.x, acc[1][4 * q]); acc[1][4 * q + 1] = fmaf(v1, w4.y, acc[1][4 * q + 1]);
            acc[1][4 * q + 2] = fmaf(v1, w4.z, acc[1][4 * q + 2]); acc[1][4 * q + 3] = fmaf(v1, w4.w, acc[1][4 * q + 3]);
          }
        }
  }
  // the block's 256 pixels x 16 channels are 16 KB of contiguous output: transpose through shared memory so that a warp
  // writes 512 contiguous bytes per store instruction
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q)
      stage[(p * 4 + q) * 129 + threadIdx.x] =
          valid ? make_float4(epilogue_m<MODE>(acc[p][4 * q], MODE >= 0 ? bs[4 * q] : 0.f, 4 * q, (size_t)(pix + p), a.e),
                              epilogue_m<MODE>(acc[p][4 * q + 1], MODE >= 0 ? bs[4 * q + 1] : 0.f, 4 * q + 1, (size_t)(pix + p), a.e),
                              epilogue_m<MODE>(acc[p][4 * q + 2], MODE >= 0 ? bs[4 * q + 2] : 0.f, 4 * q + 2, (size_t)(pix + p), a.e),
                              epilogue_m<MODE>(acc[p][4 * q + 3], MODE >= 0 ? bs[4 * q + 3] : 0.f, 4 * q + 3, (size_t)(pix + p), a.e))
                : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  float4* dst = reinterpret_cast<float4*>(a.out + (size_t)blk0 * 16);
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int j = it * 128 + threadIdx.x;                 // float4 index inside the block's output: thread j / 8, its k-th vector j % 8
    if (blk0 + (j >> 2) < total) dst[j] = stage[(j & 7) * 129 + (j >> 3)];
  }
}

void launch_stem_u8(cudaStream_t s, int B, const uint8_t* in_u8, int ih, int iw, float scale, float offset,
                    const float* w_t, int kh, int kw, int stride_h, int stride_w, int pad_t, int pad_l,
                    float* out, int oh, int ow, int ld_out, const Epilogue& e,
                    const float* w2_kn, float* out2, int ld_out2, const Epilogue* e2) {
  StemArgs a{in_u8, w_t, out, B, ih, iw, kh, kw, stride_h, stride_w, pad_t, pad_l, oh, ow, ld_out, scale, offset, to_dev(e),
             w2_kn, out2, ld_out2, e2 ? to_dev(*e2) : EpiDev{nullptr, nullptr, 0, 0, 0, 0}};
  const long total = (long)B * oh * ow;
  if (tuning().stem_x2 && !w2_kn && kh == 3 && kw == 3 && stride_h == 2 && stride_w == 2 && (ow & 1) == 0 && ld_out == 16 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    epi_dispatch(epi_mode(e), [&](auto tag) {
      auto k = k_stem_u8_x2<decltype(tag)::value>;
      BSB_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(128), 0, s, a);
    });
    count_launch();
    return;
  }
  epi_dispatch(epi_mode(e), [&](auto tag) {
    auto k = k_stem_u8<decltype(tag)::value>;
    BSB_LAUNCH(k, dim3((unsigned)((total + 127) / 128)), dim3(128), sizeof(float) * ((size_t)kh * kw * 48 + 256 + 16), s, a);
  });
  count_launch();
}

// ---------------------------------------------------------------------------
// Pointwise (1x1) conv / fully connected as a shared-memory tiled FFMA GEMM.
//   out[m][n] = epilogue( sum_k A'[m][k] * W[k][n] ),  A' = A (* scale[frame][k]) (+ add[m][k])
// 256 threads; thread tile TM rows x 4 cols; K consumed in ascending chunks of 16 so each
// accumulator sees its products in k order (bit-exact vs the oracle).
// ---------------------------------------------------------------------------
struct PWArgs {
  const float* A; const float* w; float* out; const float* in_scale; const float* in_add;
  int M, K, N, n4, ld_a, ld_out, rows_per_frame, ld_add;
  EpiDev e;
};

template <int BN, int TM, int MODE>
__global__ void __launch_bounds__(256) k_pointwise(PWArgs a) {
  constexpr int BK = 16;
  constexpr int CT = BN / 4;          // column threads
  constexpr int RT = 256 / CT;        // row threads
  constexpr int BM = RT * TM;
  constexpr int LDS_A = BM + 2;       // 4*(BM+2) % 32 == 8: conflict-free transposed stores
  __shared__ float As[BK * LDS_A];
  __shared__ __align__(16) float Ws[BK * BN];
  const int tid = threadIdx.x;
  const int tx = tid % CT, ty = tid / CT;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  float acc[TM][4];
#pragma unroll
  for (int i = 0; i < TM; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
  const float4 bias4 = epilogue_bias4<MODE>(a.e, n0 + tx * 4, a.N);
  // frame of a row (for the per-frame operand scale) without a division per element: the tile starts in frame f0 and,
  // when a frame has at least BM rows, crosses at most one frame boundary
  const int f0 = a.in_scale ? m0 / a.rows_per_frame : 0;
  const int fnext = (f0 + 1) * a.rows_per_frame;
  const bool two_frames = a.rows_per_frame >= BM;

  for (int k0 = 0; k0 < a.K; k0 += BK) {
    // ---- stage A tile (BM x BK) transposed into As[k][m] ----
    for (int q = tid; q < BM * (BK / 4); q += 256) {
      const int m = q / (BK / 4), kq = (q % (BK / 4)) * 4;
      const int gm = m0 + m, gk = k0 + kq;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (gm < a.M) {
        const float* ap = a.A + (size_t)gm * a.ld_a + gk;
        if (gk + 3 < a.K && (a.ld_a & 3) == 0) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(ap));
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (gk + j < a.K) v[j] = __ldg(ap + j);
        }
        if (a.in_scale) {
          const int fr = two_frames ? f0 + (gm >= fnext ? 1 : 0) : gm / a.rows_per_frame;
          const float* sp = a.in_scale + (size_t)fr * a.K + gk;
#pragma unroll
          for (int j = 0; j < 4; ++j) if (gk + j < a.K) v[j] = v[j] * __ldg(sp + j);
        }
        if (a.in_add) {
          const float* dp = a.in_add + (size_t)gm * a.ld_add + gk;
#pragma unroll
          for (int j = 0; j < 4; ++j) if (gk + j < a.K) v[j] = v[j] + __ldg(dp + j);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) As[(kq + j) * LDS_A + m] = v[j];
    }
    // ---- stage W tile (BK x BN) ----
    for (int q = tid; q < BK * (BN / 4); q += 256) {
      const int k = q / (BN / 4), nq = (q % (BN / 4)) * 4;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + k < a.K && n0 + nq < a.n4) t = __ldg(reinterpret_cast<const float4*>(a.w + (size_t)(k0 + k) * a.n4 + n0 + nq));
      *reinterpret_cast<float4*>(&Ws[k * BN + nq]) = t;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 w4 = *reinterpret_cast<const float4*>(&Ws[k * BN + tx * 4]);
#pragma unroll
      for (int i = 0; i < TM; ++i) {
        const float av = As[k * LDS_A + ty + RT * i];
        acc[i][0] = fmaf(av, w4.x, acc[i][0]);
        acc[i][1] = fmaf(av, w4.y, acc[i][1]);
        acc[i][2] = fmaf(av, w4.z, acc[i][2]);
        acc[i][3] = fmaf(av, w4.w, acc[i][3]);
      }
    }
    __syncthreads();
  }
  // ---- epilogue ----
  const bool vec_o = (a.ld_out & 3) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 15) == 0;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int gm = m0 + ty + RT * i;
    if (gm >= a.M) continue;
    float* op = a.out + (size_t)gm * a.ld_out;
    const int ch0 = n0 + tx * 4;
    const float bj[4] = {bias4.x, bias4.y, bias4.z, bias4.w};
    if (vec_o && ch0 + 3 < a.N) {      // one 16-byte store per row segment instead of four strided scalar stores
      *reinterpret_cast<float4*>(op + ch0) = make_float4(epilogue_m<MODE>(acc[i][0], bj[0], ch0, (size_t)gm, a.e), epilogue_m<MODE>(acc[i][1], bj[1], ch0 + 1, (size_t)gm, a.e),
                                                         epilogue_m<MODE>(acc[i][2], bj[2], ch0 + 2, (size_t)gm, a.e), epilogue_m<MODE>(acc[i][3], bj[3], ch0 + 3, (size_t)gm, a.e));
      continue;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ch = ch0 + j;
      if (ch < a.N) op[ch] = epilogue_m<MODE>(acc[i][j], bj[j], ch, (size_t)gm, a.e);
    }
  }
}

// Register-tiled variant for the GEMM-heavy layers (DeepLab / BodyPix, K and N in the hundreds):
// block tile 128 x (16*TN), thread tile 8 rows x TN columns (TN = 4 or 8), BK = 16, shared memory double
// buffered with the next chunk prefetched into registers while the current one is consumed.  Per k step a
// thread issues 2 + TN/4 LDS.128 for 8*TN FFMAs, so the kernel is FFMA-issue bound rather than LDS bound.
// Every accumulator still sees its products in ascending k (bit-exact vs the oracle).
template <int TN>
__global__ void __launch_bounds__(256, TN == 8 ? 2 : 3) k_pointwise_tile(PWArgs a) {
  constexpr int BM = 128, BN = 16 * TN, BK = 16, LDA = BM + 4, WV = TN / 4;
  __shared__ __align__(16) float As[2][BK * LDA];
  __shared__ __align__(16) float Ws[2][BK * BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  float4 ra[2], rw[WV];
  const bool vec_a = (a.ld_a & 3) == 0;

  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = tid + 256 * i, m = q >> 2, kq = (q & 3) * 4;
      const int gm = m0 + m, gk = k0 + kq;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (gm < a.M) {
        const float* ap = a.A + (size_t)gm * a.ld_a + gk;
        if (gk + 3 < a.K && vec_a) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(ap));
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (gk + j < a.K) v[j] = __ldg(ap + j);
        }
        if (a.in_scale) {
          const float* sp = a.in_scale + (size_t)(gm / a.rows_per_frame) * a.K + gk;
#pragma unroll
          for (int j = 0; j < 4; ++j) if (gk + j < a.K) v[j] = v[j] * __ldg(sp + j);
        }
        if (a.in_add) {
          const float* dp = a.in_add + (size_t)gm * a.ld_add + gk;
#pragma unroll
          for (int j = 0; j < 4; ++j) if (gk + j < a.K) v[j] = v[j] + __ldg(dp + j);
        }
      }
      ra[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
#pragma unroll
    for (int i = 0; i < WV; ++i) {
      const int q = tid + 256 * i, k = q / (BN / 4), nq = (q % (BN / 4)) * 4;
      rw[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + k < a.K && n0 + nq < a.n4) rw[i] = __ldg(reinterpret_cast<const float4*>(a.w + (size_t)(k0 + k) * a.n4 + n0 + nq));
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = tid + 256 * i, m = q >> 2, kq = (q & 3) * 4;
      float* d = &As[buf][kq * LDA + m];
      d[0] = ra[i].x; d[LDA] = ra[i].y; d[2 * LDA] = ra[i].z; d[3 * LDA] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < WV; ++i) {
      const int q = tid + 256 * i, k = q / (BN / 4), nq = (q % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Ws[buf][k * BN + nq]) = rw[i];
    }
  };

  gload(0);
  sstore(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < a.K; k0 += BK) {
    const bool more = k0 + BK < a.K;
    if (more) gload(k0 + BK);
    const float* as = &As[buf][ty * 8];
    const float* ws = &Ws[buf][tx * 4];
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(as + k * LDA);
      const float4 a1 = *reinterpret_cast<const float4*>(as + k * LDA + 4);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int h = 0; h < WV; ++h) {
        const float4 w4 = *reinterpret_cast<const float4*>(ws + k * BN + 64 * h);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][4 * h] = fmaf(av[i], w4.x, acc[i][4 * h]);
          acc[i][4 * h + 1] = fmaf(av[i], w4.y, acc[i][4 * h + 1]);
          acc[i][4 * h + 2] = fmaf(av[i], w4.z, acc[i][4 * h + 2]);
          acc[i][4 * h + 3] = fmaf(av[i], w4.w, acc[i][4 * h + 3]);
        }
      }
    }
    if (more) sstore(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
  // ---- epilogue ----
  const bool vec_o = (a.ld_out & 3) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 15) == 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + ty * 8 + i;
    if (gm >= a.M) continue;
    float* op = a.out + (size_t)gm * a.ld_out;
#pragma unroll
    for (int h = 0; h < WV; ++h) {
      const int ch = n0 + tx * 4 + 64 * h;
      if (ch + 3 < a.N && vec_o) {
        *reinterpret_cast<float4*>(op + ch) = epilogue4(make_float4(acc[i][4 * h], acc[i][4 * h + 1], acc[i][4 * h + 2], acc[i][4 * h + 3]), ch, (size_t)gm, a.e);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (ch + j < a.N) op[ch + j] = epilogue1(acc[i][4 * h + j], ch + j, (size_t)gm, a.e);
      }
    }
  }
}

// Row-streaming variant for small K x N (the high-resolution MobileNet layers, K, N <= 64):
// the whole weight matrix sits in shared memory; a thread owns 4 output channels of one
// pixel and walks K in ascending order (float4 loads of the pixel row are shared by the
// CT threads of that pixel through the L1 broadcast path).  Memory-bound by design.
template <int MODE>
__global__ void __launch_bounds__(256) k_pointwise_rows(PWArgs a, int ct) {
  BSB_DYN_SMEM(smem_raw);
  float* Ws = reinterpret_cast<float*>(smem_raw);            // [K][n4]
  for (int i = threadIdx.x * 4; i < a.K * a.n4; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(Ws + i) = __ldg(reinterpret_cast<const float4*>(a.w + i));
  __syncthreads();
  const int rows_per_block = 256 / ct;
  const int tx = threadIdx.x % ct, tr = threadIdx.x / ct;
  if (tr >= rows_per_block) return;
  const int n0 = tx * 4;
  const float4 bias4 = epilogue_bias4<MODE>(a.e, n0, a.N);
  for (long gm = (long)blockIdx.x * rows_per_block + tr; gm < a.M; gm += (long)gridDim.x * rows_per_block) {
    const float* ap = a.A + (size_t)gm * a.ld_a;
    const float* sp = a.in_scale ? a.in_scale + (size_t)((unsigned)gm / (unsigned)a.rows_per_frame) * a.K : nullptr;
    const float* dp = a.in_add ? a.in_add + (size_t)gm * a.ld_add : nullptr;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    for (int k = 0; k < a.K; k += 4) {
      float4 v = __ldg(reinterpret_cast<const float4*>(ap + k));
      if (sp) { const float4 sc = __ldg(reinterpret_cast<const float4*>(sp + k)); v.x = v.x * sc.x; v.y = v.y * sc.y; v.z = v.z * sc.z; v.w = v.w * sc.w; }
      if (dp) { const float4 ad = __ldg(reinterpret_cast<const float4*>(dp + k)); v.x = v.x + ad.x; v.y = v.y + ad.y; v.z = v.z + ad.z; v.w = v.w + ad.w; }
      const float av[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 w4 = *reinterpret_cast<const float4*>(Ws + (k + j) * a.n4 + n0);
        acc0 = fmaf(av[j], w4.x, acc0); acc1 = fmaf(av[j], w4.y, acc1);
        acc2 = fmaf(av[j], w4.z, acc2); acc3 = fmaf(av[j], w4.w, acc3);
      }
    }
    float* op = a.out + (size_t)gm * a.ld_out + n0;
    const float r0 = epilogue_m<MODE>(acc0, bias4.x, n0, (size_t)gm, a.e);
    if (n0 + 3 < a.N && (a.ld_out & 3) == 0) {
      *reinterpret_cast<float4*>(op) = make_float4(r0, epilogue_m<MODE>(acc1, bias4.y, n0 + 1, (size_t)gm, a.e), epilogue_m<MODE>(acc2, bias4.z, n0 + 2, (size_t)gm, a.e),
                                                   epilogue_m<MODE>(acc3, bias4.w, n0 + 3, (size_t)gm, a.e));
    } else {
      op[0] = r0;
      if (n0 + 1 < a.N) op[1] = epilogue_m<MODE>(acc1, bias4.y, n0 + 1, (size_t)gm, a.e);
      if (n0 + 2 < a.N) op[2] = epilogue_m<MODE>(acc2, bias4.z, n0 + 2, (size_t)gm, a.e);
      if (n0 + 3 < a.N) op[3] = epilogue_m<MODE>(acc3, bias4.w, n0 + 3, (size_t)gm, a.e);
    }
  }
}

// kernel selection override for A/B measurements: 0 = heuristics, 2 = never the register-tiled kernel, 3 = always
// (set through bsb_pointwise's `variant` argument or bsb_set_tuning("pw_variant", v); results are bit-identical
// whichever kernel runs)
void set_pointwise_variant(int v) { tuning().pw_variant = v; }
int pointwise_variant() { return tuning().pw_variant; }

void launch_pointwise(cudaStream_t s, int M, int K, int N, const float* A, int ld_a,
                      const float* w_kn, int n4, float* out, int ld_out, const Epilogue& e,
                      const float* in_scale, int rows_per_frame, const float* in_add, int ld_add) {
  PWArgs a{A, w_kn, out, in_scale, in_add, M, K, N, n4, ld_a, ld_out, rows_per_frame > 0 ? rows_per_frame : 1, ld_add, to_dev(e)};
  const int variant = pointwise_variant();
  const long sms = device_sms();
  // GEMM-heavy layers: register-tiled kernel (128-row tiles need enough rows to fill the SMs)
  if (variant == 3 || variant == 4 || variant == 8 || (variant == 0 && ((K >= 128 && N >= 32) || (K >= 192 && N >= 16)) && (long)ceil_div(M, 128) * ceil_div(N, 64) >= sms)) {
    // 8x8 register tiles (128 columns) unless padding N to 128 wastes a whole 64-column tile
    const int pad64 = (N + 63) / 64 * 64, pad128 = (N + 127) / 128 * 128;
    const bool wide = variant == 8 || (variant != 4 && pad128 - N < 64 && (long)ceil_div(M, 128) * (pad128 / 128) >= sms);
    if (wide) {
      auto k = k_pointwise_tile<8>; BSB_LAUNCH(k, dim3((unsigned)ceil_div(M, 128), (unsigned)(pad128 / 128)), dim3(256), 0, s, a);
    } else {
      auto k = k_pointwise_tile<4>; BSB_LAUNCH(k, dim3((unsigned)ceil_div(M, 128), (unsigned)(pad64 / 64)), dim3(256), 0, s, a);
    }
    count_launch();
    return;
  }
  const bool rows_ok = K % 4 == 0 && ld_a % 4 == 0 && (!in_add || ld_add % 4 == 0) && n4 <= 64 && K * n4 <= 4096;
  // the row-streaming kernel for very narrow outputs (<= 8 channels), 20..28 output channels, and K <= 8; the classic
  // tiles elsewhere (e.g. 16 -> 16, 64 -> 64)
  const bool rows_wins = n4 <= 8 || (n4 >= 20 && n4 <= 28) || K <= 8;
  if (rows_ok && (variant == 5 || (variant < 16 && M >= 4096 && rows_wins))) {
    const int ct = n4 / 4, rows_per_block = 256 / ct;
    long blocks = ((long)M + rows_per_block - 1) / rows_per_block;
    if (blocks > sms * 16) blocks = sms * 16;               // grid-stride: a few waves over the SMs
    epi_dispatch(epi_mode(e), [&](auto tag) {
      auto k = k_pointwise_rows<decltype(tag)::value>;
      BSB_LAUNCH(k, dim3((unsigned)blocks), dim3(256), sizeof(float) * (size_t)K * n4, s, a, ct);
    });
    count_launch();
    return;
  }
  // choose the N tile that wastes the fewest columns; ties go to the wider tile
  const int pad16 = (N + 15) / 16 * 16, pad32 = (N + 31) / 32 * 32, pad64 = (N + 63) / 64 * 64;
  int bn = 64;
  if (pad32 < pad64) bn = 32;
  if (pad16 < (bn == 64 ? pad64 : pad32)) bn = 16;
  if (variant >= 16) bn = variant;                           // A/B measurements: force the classic kernel's N tile (16 / 32 / 64)
  // small problems: one row per thread (TM = 1) gives 4x more blocks to spread over the SMs
  const int rt = 256 / (bn / 4);
  const bool small = (long)ceil_div(M, rt * 4) * ceil_div(N, bn) < 2 * sms;
  const int bm = small ? rt : rt * 4;
  dim3 grid((unsigned)ceil_div(M, bm), (unsigned)ceil_div(N, bn));
  epi_dispatch(epi_mode(e), [&](auto tag) {
    constexpr int MD = decltype(tag)::value;
    if (bn == 64) { if (small) { auto k = k_pointwise<64, 1, MD>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); } else { auto k = k_pointwise<64, 4, MD>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); } }
    else if (bn == 32) { if (small) { auto k = k_pointwise<32, 1, MD>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); } else { auto k = k_pointwise<32, 4, MD>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); } }
    else { if (small) { auto k = k_pointwise<16, 1, MD>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); } else { auto k = k_pointwise<16, 4, MD>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); } }
  });
  count_launch();
}

// ---------------------------------------------------------------------------
// Depthwise KxK.  One thread = one output pixel x 4 channels (float4 over C).
// ---------------------------------------------------------------------------
struct DWArgs {
  const float* in; const float* w; float* out;
  int B, ih, iw, c, ld_in, kh, kw, sh, sw, dh, dw, pt, pl, oh, ow, ld_out;
  EpiDev e;
};

template <int VEC>
__global__ void __launch_bounds__(256) k_depthwise(DWArgs a) {
  const int groups = (a.c + VEC - 1) / VEC;
  const long total = (long)a.B * a.oh * a.ow * groups;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c0 = (int)(idx % groups) * VEC;
  const long pix = idx / groups;
  const int ox = (int)(pix % a.ow);
  const int oy = (int)((pix / a.ow) % a.oh);
  const int b = (int)(pix / ((long)a.ow * a.oh));
  const float* inb = a.in + (size_t)b * a.ih * a.iw * a.ld_in;
  float acc[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
  const int iy0 = oy * a.sh - a.pt, ix0 = ox * a.sw - a.pl;
  for (int fy = 0; fy < a.kh; ++fy) {
    const int iy = iy0 + a.dh * fy;
    if (iy < 0 || iy >= a.ih) continue;
    for (int fx = 0; fx < a.kw; ++fx) {
      const int ix = ix0 + a.dw * fx;
      if (ix < 0 || ix >= a.iw) continue;
      const float* ip = inb + ((size_t)iy * a.iw + ix) * a.ld_in + c0;
      const float* wp = a.w + (size_t)(fy * a.kw + fx) * a.c + c0;
      if (VEC == 4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(ip));
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(wp));
        acc[0] = fmaf(v.x, w4.x, acc[0]); acc[1 % VEC] = fmaf(v.y, w4.y, acc[1 % VEC]);
        acc[2 % VEC] = fmaf(v.z, w4.z, acc[2 % VEC]); acc[3 % VEC] = fmaf(v.w, w4.w, acc[3 % VEC]);
      } else {
        acc[0] = fmaf(__ldg(ip), __ldg(wp), acc[0]);
      }
    }
  }
  float* op = a.out + (size_t)pix * a.ld_out + c0;
  if (VEC == 4) {   // (the launcher picks VEC = 4 only when c, ld_in and ld_out are multiples of 4)
    *reinterpret_cast<float4*>(op) = make_float4(epilogue(acc[0], c0, (size_t)pix, a.e), epilogue(acc[1 % VEC], c0 + 1, (size_t)pix, a.e),
                                                 epilogue(acc[2 % VEC], c0 + 2, (size_t)pix, a.e), epilogue(acc[3 % VEC], c0 + 3, (size_t)pix, a.e));
    return;
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) op[j] = epilogue(acc[j], c0 + j, (size_t)pix, a.e);
}

// Strip variant (dilation 1, C % 4 == 0): a thread produces 4 consecutive output pixels x 4
// channels, so each input row segment is loaded once and reused by the overlapping windows
// (3x3 s1: 18 float4 loads for 4 outputs instead of 36).  Per output the taps are still
// accumulated in (fy, fx) order and out-of-image taps are skipped, exactly like the oracle.
BSB_D void fma4(float4& acc, const float4& v, const float4& w) {
  acc.x = fmaf(v.x, w.x, acc.x); acc.y = fmaf(v.y, w.y, acc.y); acc.z = fmaf(v.z, w.z, acc.z); acc.w = fmaf(v.w, w.w, acc.w);
}

// One output pixel x 4 channels per thread, like k_depthwise<4>, for the layers too small for the strip kernel to fill the
// GPU — but the KS loads of a kernel row are issued together (and all the rows are unrolled), where the generic kernel
// waits for each tap's load before it even computes the next address (taps behind `continue`s): on these small,
// latency-bound layers memory-level parallelism per thread is what counts.  Same (fy, fx) accumulation order; out-of-image
// taps are skipped.
template <int KS, int MODE>
__global__ void __launch_bounds__(256) k_depthwise_px(DWArgs a) {
  const int groups = a.c / 4;
  const long total = (long)a.B * a.oh * a.ow * groups;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c0 = (int)(idx % groups) * 4;
  const long pix = idx / groups;
  const int ox = (int)(pix % a.ow);
  const int oy = (int)((pix / a.ow) % a.oh);
  const int b = (int)(pix / ((long)a.ow * a.oh));
  const float* inb = a.in + (size_t)b * a.ih * a.iw * a.ld_in + c0;
  const int iy0 = oy * a.sh - a.pt, ix0 = ox * a.sw - a.pl;
  const float4 bias4 = epilogue_bias4<MODE>(a.e, c0, a.c);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int fy = 0; fy < KS; ++fy) {
    const int iy = iy0 + a.dh * fy;
    const bool vy = iy >= 0 && iy < a.ih;
    const float* rowp = inb + (size_t)(vy ? iy : 0) * a.iw * a.ld_in;
    float4 v[KS], w[KS];
    bool ok[KS];
#pragma unroll
    for (int fx = 0; fx < KS; ++fx) {
      const int ix = ix0 + a.dw * fx;
      ok[fx] = vy && ix >= 0 && ix < a.iw;
      v[fx] = ok[fx] ? __ldg(reinterpret_cast<const float4*>(rowp + (size_t)ix * a.ld_in)) : make_float4(0.f, 0.f, 0.f, 0.f);
      w[fx] = __ldg(reinterpret_cast<const float4*>(a.w + (size_t)(fy * KS + fx) * a.c + c0));
    }
#pragma unroll
    for (int fx = 0; fx < KS; ++fx)
      if (ok[fx]) fma4(acc, v[fx], w[fx]);
  }
  float* op = a.out + (size_t)pix * a.ld_out + c0;
  *reinterpret_cast<float4*>(op) = make_float4(epilogue_m<MODE>(acc.x, bias4.x, c0, (size_t)pix, a.e), epilogue_m<MODE>(acc.y, bias4.y, c0 + 1, (size_t)pix, a.e),
                                               epilogue_m<MODE>(acc.z, bias4.z, c0 + 2, (size_t)pix, a.e), epilogue_m<MODE>(acc.w, bias4.w, c0 + 3, (size_t)pix, a.e));
}


template <int KS, int S, int D, int MODE>   // D = dilation (DeepLab / BodyPix atrous layers): taps sit D pixels apart
__global__ void __launch_bounds__(128) k_depthwise_strip(DWArgs a) {
  constexpr int CNT = 3 * S + (KS - 1) * D + 1;
  const int groups = a.c / 4, strips = (a.ow + 3) / 4;
  const long total = (long)a.B * a.oh * strips * groups;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c0 = (int)(idx % groups) * 4;
  long t = idx / groups;
  const int ox0 = (int)(t % strips) * 4; t /= strips;
  const int oy = (int)(t % a.oh);
  const int b = (int)(t / a.oh);
  const float* inb = a.in + (size_t)b * a.ih * a.iw * a.ld_in + c0;
  const float4 bias4 = epilogue_bias4<MODE>(a.e, c0, a.c);
  float4 acc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int ix0 = ox0 * S - a.pl;
#pragma unroll
  for (int fy = 0; fy < KS; ++fy) {
    const int iy = oy * S - a.pt + fy * D;
    if (iy < 0 || iy >= a.ih) continue;
    const float* rowp = inb + (size_t)iy * a.iw * a.ld_in;
    float4 v[CNT];
#pragma unroll
    for (int cidx = 0; cidx < CNT; ++cidx) {
      const int ix = ix0 + cidx;
      v[cidx] = (ix >= 0 && ix < a.iw) ? __ldg(reinterpret_cast<const float4*>(rowp + (size_t)ix * a.ld_in)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float4 wr[KS];
#pragma unroll
    for (int fx = 0; fx < KS; ++fx) wr[fx] = __ldg(reinterpret_cast<const float4*>(a.w + (size_t)(fy * KS + fx) * a.c + c0));
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int fx = 0; fx < KS; ++fx) {
        const int ix = ix0 + j * S + fx * D;
        if (ix >= 0 && ix < a.iw) fma4(acc[j], v[j * S + fx * D], wr[fx]);
      }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ox = ox0 + j;
    if (ox >= a.ow) break;
    const size_t pix = ((size_t)b * a.oh + oy) * a.ow + ox;
    float* op = a.out + pix * a.ld_out + c0;
    *reinterpret_cast<float4*>(op) = make_float4(epilogue_m<MODE>(acc[j].x, bias4.x, c0, pix, a.e), epilogue_m<MODE>(acc[j].y, bias4.y, c0 + 1, pix, a.e),
                                                 epilogue_m<MODE>(acc[j].z, bias4.z, c0 + 2, pix, a.e), epilogue_m<MODE>(acc[j].w, bias4.w, c0 + 3, pix, a.e));
  }
}

// Whole-plane variant for the 33x33 atrous layers of DeepLab / BodyPix (stride 1, 3x3, any dilation): one block owns
// 16 channels of one frame, stages that 33x33x16 slice in shared memory once (every input byte is read from L2/HBM
// exactly once, where the strip kernel re-reads each pixel up to nine times through L2) and produces all its outputs
// from there.  A thread owns 4 channels of FOUR vertically adjacent output pixels: the nine weight vectors sit in
// registers, the four accumulation chains are independent (the first version — one pixel per thread, 180 instructions per
// output with a 9-deep dependent LDS -> FFMA chain — was latency-bound).
// Tap order and the skipping of out-of-image taps are those of the oracle.
constexpr int DWP_R = 4;     // (channels per block: template parameter DWP_CS, 16 or 8 — 70 KB or 35 KB of shared memory for a 33x33 plane)
// RELU6_ONLY: the epilogue is bias + RELU6 and nothing else (every atrous layer of DeepLab and BodyPix): the four bias
// values of the thread's channels are loaded once and the activation is a compile-time constant, where the generic
// epilogue re-loads the bias and walks two activation switches and a residual test per value.
template <bool RELU6_ONLY, int DWP_CS>
__global__ void __launch_bounds__(256) k_depthwise_plane(DWArgs a) {
  constexpr int QN = DWP_CS / 4;                               // float4 quads per pixel of the slice
  BSB_DYN_SMEM(smem_raw);
  float* plane = reinterpret_cast<float*>(smem_raw);           // [ih*iw][16]
  float* ws = plane + (size_t)a.ih * a.iw * DWP_CS;             // [9][16]
  const int c0 = blockIdx.x * DWP_CS, b = blockIdx.y;
  const int hw = a.ih * a.iw;
  const float* inb = a.in + (size_t)b * hw * a.ld_in + c0;
  // asynchronous 16-byte copies straight into shared memory (LDGSTS): all ~17 copies of a thread are in flight together.
  // The first version went through registers one load at a time and ran at the latency of a single outstanding load per
  // thread.
  for (int i = threadIdx.x; i < hw * (DWP_CS / 4); i += blockDim.x) {
    const int p = i / QN, q = i % QN;
#if defined(BSB_EMU)
    *reinterpret_cast<float4*>(plane + p * DWP_CS + 4 * q) = __ldg(reinterpret_cast<const float4*>(inb + (size_t)p * a.ld_in + 4 * q));
#else
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((unsigned)__cvta_generic_to_shared(plane + p * DWP_CS + 4 * q)),
                 "l"(inb + (size_t)p * a.ld_in + 4 * q) : "memory");
#endif
  }
  for (int i = threadIdx.x; i < 9 * DWP_CS; i += blockDim.x) ws[i] = __ldg(a.w + (size_t)(i / DWP_CS) * a.c + c0 + (i % DWP_CS));
#if !defined(BSB_EMU)
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
  __syncthreads();
  const int q = threadIdx.x % QN, ch = c0 + 4 * q;
  float4 w[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) w[t] = *reinterpret_cast<const float4*>(ws + t * DWP_CS + 4 * q);
  float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (RELU6_ONLY && a.e.bias) bias4 = make_float4(__ldg(a.e.bias + ch), __ldg(a.e.bias + ch + 1), __ldg(a.e.bias + ch + 2), __ldg(a.e.bias + ch + 3));
  const int row_groups = (a.oh + DWP_R - 1) / DWP_R;
  for (int p = threadIdx.x / QN; p < row_groups * a.ow; p += blockDim.x / QN) {
    const int rg = p / a.ow, ox = p - rg * a.ow, oy0 = rg * DWP_R;
    float4 acc[DWP_R];
#pragma unroll
    for (int j = 0; j < DWP_R; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    int ixs[3]; bool vx[3];
#pragma unroll
    for (int fx = 0; fx < 3; ++fx) { ixs[fx] = ox - a.pl + a.dw * fx; vx[fx] = ixs[fx] >= 0 && ixs[fx] < a.iw; }
#pragma unroll
    for (int fy = 0; fy < 3; ++fy) {
#pragma unroll
      for (int j = 0; j < DWP_R; ++j) {
        const int iy = oy0 + j - a.pt + a.dh * fy;
        if (iy < 0 || iy >= a.ih) continue;                  // (rows past the image: their outputs are never stored)
        const float* rowp = plane + (size_t)iy * a.iw * DWP_CS + 4 * q;
#pragma unroll
        for (int fx = 0; fx < 3; ++fx)
          if (vx[fx]) fma4(acc[j], *reinterpret_cast<const float4*>(rowp + ixs[fx] * DWP_CS), w[fy * 3 + fx]);
      }
    }
#pragma unroll
    for (int j = 0; j < DWP_R; ++j) {
      const int oy = oy0 + j;
      if (oy >= a.oh) break;
      const size_t pix = (size_t)b * a.oh * a.ow + (size_t)oy * a.ow + ox;
      float4 r;
      if (RELU6_ONLY) {
        r = make_float4(bsb_act(acc[j].x + bias4.x, ACT_RELU6), bsb_act(acc[j].y + bias4.y, ACT_RELU6), bsb_act(acc[j].z + bias4.z, ACT_RELU6),
                        bsb_act(acc[j].w + bias4.w, ACT_RELU6));
      } else {
        r = make_float4(epilogue(acc[j].x, ch, pix, a.e), epilogue(acc[j].y, ch + 1, pix, a.e), epilogue(acc[j].z, ch + 2, pix, a.e),
                        epilogue(acc[j].w, ch + 3, pix, a.e));
      }
      *reinterpret_cast<float4*>(a.out + pix * a.ld_out + ch) = r;
    }
  }
}

void launch_depthwise(cudaStream_t s, int B, const float* in, int ih, int iw, int c, int ld_in,
                      const float* w, int kh, int kw, int stride_h, int stride_w, int dil_h, int dil_w,
                      int pad_t, int pad_l, float* out, int oh, int ow, int ld_out, const Epilogue& e) {
  DWArgs a{in, w, out, B, ih, iw, c, ld_in, kh, kw, stride_h, stride_w, dil_h, dil_w, pad_t, pad_l, oh, ow, ld_out, to_dev(e)};
  const bool vec = (c % 4 == 0) && (ld_in % 4 == 0) && (ld_out % 4 == 0);
  const int cs = tuning().dw_plane_cs == 8 ? 8 : 16;
  const size_t plane_smem = ((size_t)ih * iw + 9) * cs * sizeof(float);
  if (tuning().dw_plane && (dil_h > 1 || dil_w > 1) && (c % cs == 0) && (ld_in % 4 == 0) && (ld_out % 4 == 0) && kh == 3 && kw == 3 &&
      stride_h == 1 && stride_w == 1 && oh == ih && ow == iw && plane_smem <= 100 * 1024 &&
      ensure_dyn_smem(reinterpret_cast<const void*>(k_depthwise_plane<true, 16>), plane_smem) &&
      ensure_dyn_smem(reinterpret_cast<const void*>(k_depthwise_plane<false, 16>), plane_smem) &&
      ensure_dyn_smem(reinterpret_cast<const void*>(k_depthwise_plane<true, 8>), plane_smem) &&
      ensure_dyn_smem(reinterpret_cast<const void*>(k_depthwise_plane<false, 8>), plane_smem)) {
    const bool relu6_only = !e.residual && ((e.act1 == ACT_RELU6 && e.act2 == ACT_NONE) || (e.act1 == ACT_NONE && e.act2 == ACT_RELU6));
    const dim3 pgrid((unsigned)(c / cs), (unsigned)B);
    // (local names keep "k_depthwise_plane" in the emulator's launch trace)
    if (cs == 16) {
      if (relu6_only) { auto k_depthwise_plane_r16 = k_depthwise_plane<true, 16>; BSB_LAUNCH(k_depthwise_plane_r16, pgrid, dim3(256), plane_smem, s, a); }
      else { auto k_depthwise_plane_g16 = k_depthwise_plane<false, 16>; BSB_LAUNCH(k_depthwise_plane_g16, pgrid, dim3(256), plane_smem, s, a); }
    } else {
      if (relu6_only) { auto k_depthwise_plane_r8 = k_depthwise_plane<true, 8>; BSB_LAUNCH(k_depthwise_plane_r8, pgrid, dim3(256), plane_smem, s, a); }
      else { auto k_depthwise_plane_g8 = k_depthwise_plane<false, 8>; BSB_LAUNCH(k_depthwise_plane_g8, pgrid, dim3(256), plane_smem, s, a); }
    }
    count_launch();
    return;
  }
  const bool atrous = dil_h == dil_w && (dil_h == 2 || dil_h == 4) && kh == 3 && kw == 3 && stride_h == 1 && stride_w == 1;
  if (vec && ((dil_h == 1 && dil_w == 1) || atrous) && kh == kw && stride_h == stride_w && (kh == 3 || kh == 5) && (stride_h == 1 || stride_h == 2)) {
    const long nthreads = (long)B * oh * ((ow + 3) / 4) * (c / 4);
    if (nthreads >= device_sms() * 1024L) {   // enough strips to fill the GPU; small layers keep one pixel per thread
    const dim3 grid((unsigned)((nthreads + 127) / 128)), block(128);
    epi_dispatch(epi_mode(e), [&](auto tag) {
      constexpr int MD = decltype(tag)::value;
      if (atrous && dil_h == 2) { auto k = k_depthwise_strip<3, 1, 2, MD>; BSB_LAUNCH(k, grid, block, 0, s, a); }
      else if (atrous) { auto k = k_depthwise_strip<3, 1, 4, MD>; BSB_LAUNCH(k, grid, block, 0, s, a); }
      else if (kh == 3 && stride_h == 1) { auto k = k_depthwise_strip<3, 1, 1, MD>; BSB_LAUNCH(k, grid, block, 0, s, a); }
      else if (kh == 3) { auto k = k_depthwise_strip<3, 2, 1, MD>; BSB_LAUNCH(k, grid, block, 0, s, a); }
      else if (stride_h == 1) { auto k = k_depthwise_strip<5, 1, 1, MD>; BSB_LAUNCH(k, grid, block, 0, s, a); }
      else { auto k = k_depthwise_strip<5, 2, 1, MD>; BSB_LAUNCH(k, grid, block, 0, s, a); }
    });
    count_launch();
    return;
    }
  }
  const long total = (long)B * oh * ow * (vec ? c / 4 : c);
  if (vec && kh == kw && (kh == 3 || kh == 5) && tuning().dw_px) {
    epi_dispatch(epi_mode(e), [&](auto tag) {
      constexpr int MD = decltype(tag)::value;
      if (kh == 3) { auto k = k_depthwise_px<3, MD>; BSB_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, a); }
      else { auto k = k_depthwise_px<5, MD>; BSB_LAUNCH(k, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, a); }
    });
    count_launch();
    return;
  }
  if (vec) BSB_LAUNCH(k_depthwise<4>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, a);
  else BSB_LAUNCH(k_depthwise<1>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, a);
  count_launch();
}

// ---------------------------------------------------------------------------
// Global average pool + SE fully-connected chain.  Summation order (shared with the
// oracle): each row left to right, then the row sums top to bottom; total / (float)(H*W).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rowsum(int B, const float* inA, int cA, int ldA, const float* inB, int cB, int ldB,
                                                int h, int w, float* rowsum) {
  const int C = cA + cB;
  const long total = (long)B * h * C;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = (int)(idx % C);
  const long row = idx / C;                       // b * h + y
  const float* p; int ld;
  if (ch < cA) { p = inA + (size_t)row * w * ldA + ch; ld = ldA; }
  else { p = inB + (size_t)row * w * ldB + (ch - cA); ld = ldB; }
  float r = 0.f;
  int x = 0;
  for (; x + 8 <= w; x += 8) {                    // loads first (independent), adds in x order
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __ldg(p + (size_t)(x + j) * ld);
#pragma unroll
    for (int j = 0; j < 8; ++j) r = r + v[j];
  }
  for (; x < w; ++x) r = r + __ldg(p + (size_t)x * ld);
  rowsum[idx] = r;
}

struct FcDev { const float* w; const float* bias; int K, N, n4, act1, act2; };

// One block per frame.  Each FC weight matrix ([K][n4], <= 64 KB) is first pulled into shared memory by
// all 256 threads with every load in flight at once (one L2 round trip instead of K dependent ones);
// the dot products then run out of shared memory with k ascending.
BSB_D void stage_weights(float* ws, const float* w, int count) {
  for (int i = threadIdx.x * 4; i < count; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(ws + i) = __ldg(reinterpret_cast<const float4*>(w + i));
}

// frame b: column sums of the row sums (y ascending), / count, activation, then the FC chain — one 256-thread block
BSB_D void pool_fc_frame(const float* rowsum, int b, int h, int C, float count, int pool_act, float* pooled_out,
                         int n_fc, const FcDev& f0, const FcDev& f1, float* out, int ld_out, float* ws, float* v0, float* v1, bool coherent) {
  if (n_fc > 0) stage_weights(ws, f0.w, f0.K * f0.n4);          // overlaps with the pooling reads below
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    const float* p = rowsum + (size_t)b * h * C + ch;
    float t = 0.f;
    int y = 0;
    for (; y + 8 <= h; y += 8) {
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = coherent ? __ldcg(p + (size_t)(y + j) * C) : __ldg(p + (size_t)(y + j) * C);
#pragma unroll
      for (int j = 0; j < 8; ++j) t = t + r[j];
    }
    for (; y < h; ++y) t = t + (coherent ? __ldcg(p + (size_t)y * C) : __ldg(p + (size_t)y * C));
    const float a = bsb_act(bsb_div(t, count), pool_act);
    v0[ch] = a;
    if (pooled_out) pooled_out[(size_t)b * C + ch] = a;
    if (n_fc == 0) out[(size_t)b * ld_out + ch] = a;
  }
  if (n_fc == 0) return;
  __syncthreads();
  for (int n = threadIdx.x; n < f0.N; n += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < f0.K; ++k) acc = fmaf(v0[k], ws[k * f0.n4 + n], acc);
    const float r = bsb_act(bsb_act(acc + (f0.bias ? __ldg(f0.bias + n) : 0.f), f0.act1), f0.act2);
    if (n_fc == 1) out[(size_t)b * ld_out + n] = r; else v1[n] = r;
  }
  if (n_fc == 1) return;
  __syncthreads();
  stage_weights(ws, f1.w, f1.K * f1.n4);
  __syncthreads();
  for (int n = threadIdx.x; n < f1.N; n += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < f1.K; ++k) acc = fmaf(v1[k], ws[k * f1.n4 + n], acc);
    out[(size_t)b * ld_out + n] = bsb_act(bsb_act(acc + (f1.bias ? __ldg(f1.bias + n) : 0.f), f1.act1), f1.act2);
  }
}

__global__ void __launch_bounds__(256) k_pool_fc(const float* rowsum, int h, int C, float count, int pool_act, float* pooled_out,
                                                 int n_fc, FcDev f0, FcDev f1, float* out, int ld_out) {
  BSB_DYN_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);
  __shared__ float v0[512];
  __shared__ float v1[512];
  pool_fc_frame(rowsum, blockIdx.x, h, C, count, pool_act, pooled_out, n_fc, f0, f1, out, ld_out, ws, v0, v1, false);
}

// Row sums and the per-frame tail in ONE launch: grid (blocks per frame, B).  Every block writes its share of
// rowsum[b][y][c]; the block that finishes last for a frame (a per-frame arrival counter, reset for the next launch)
// runs the column sums + FC chain for that frame.  Which block is last only decides WHO does the tail — the sums are
// taken in the fixed (row, then column) order from the complete rowsum array, so results do not depend on timing.
__global__ void __launch_bounds__(256) k_rowsum_fc(const float* inA, int cA, int ldA, const float* inB, int cB, int ldB, int h, int w,
                                                   float* rowsum, unsigned* counters, float count, int pool_act,
                                                   int n_fc, FcDev f0, FcDev f1, float* out, int ld_out) {
  BSB_DYN_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);
  __shared__ float v0[512];
  __shared__ float v1[512];
  __shared__ int is_last;
  const int C = cA + cB, b = blockIdx.y;
  const int per_frame = h * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_frame; i += gridDim.x * blockDim.x) {
    const int ch = i % C, y = i / C;
    const size_t row = (size_t)b * h + y;
    const float* p; int ld;
    if (ch < cA) { p = inA + row * w * ldA + ch; ld = ldA; }
    else { p = inB + row * w * ldB + (ch - cA); ld = ldB; }
    float r = 0.f;
    int x = 0;
    for (; x + 8 <= w; x += 8) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __ldg(p + (size_t)(x + j) * ld);
#pragma unroll
      for (int j = 0; j < 8; ++j) r = r + v[j];
    }
    for (; x < w; ++x) r = r + __ldg(p + (size_t)x * ld);
    rowsum[(size_t)b * per_frame + i] = r;
  }
  __threadfence();                                   // this block's row sums are visible device-wide ...
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(counters + b, 1u);   // ... before its arrival is
    is_last = prev == gridDim.x - 1;
    if (is_last) counters[b] = 0u;                   // ready for the next launch (stream order)
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  pool_fc_frame(rowsum, b, h, C, count, pool_act, nullptr, n_fc, f0, f1, out, ld_out, ws, v0, v1, true);
}

void launch_pool_fc(cudaStream_t s, int B, const float* inA, int cA, int ldA, const float* inB, int cB, int ldB,
                    int h, int w, float* rowsum_scratch, int pool_act, float* pooled_out,
                    int n_fc, const FcLayer* fc, float* out, int ld_out, unsigned* counters) {
  const int C = cA + cB;
  FcDev f[2] = {{nullptr, nullptr, 0, 0, 0, 0, 0}, {nullptr, nullptr, 0, 0, 0, 0, 0}};
  for (int i = 0; i < n_fc && i < 2; ++i) f[i] = FcDev{fc[i].w, fc[i].bias, fc[i].K, fc[i].N, fc[i].n4, fc[i].act1, fc[i].act2};
  size_t wbytes = 16;
  for (int i = 0; i < n_fc && i < 2; ++i) wbytes = std::max(wbytes, sizeof(float) * (size_t)f[i].K * f[i].n4);
  if (counters && !pooled_out && wbytes <= 48 * 1024 && tuning().pool_merge) {
    // one launch: enough blocks per frame to spread the row sums, the last one per frame does the tail
    const int per_frame = h * C;
    int bpf = std::min(ceil_div(per_frame, 256), std::max(1, (device_sms() * 8) / std::max(B, 1)));
    ensure_dyn_smem(reinterpret_cast<const void*>(k_rowsum_fc), wbytes);
    BSB_LAUNCH(k_rowsum_fc, dim3((unsigned)bpf, (unsigned)B), dim3(256), wbytes, s, inA, cA, ldA, inB, cB, ldB, h, w, rowsum_scratch, counters,
               (float)(h * w), pool_act, n_fc, f[0], f[1], out, ld_out);
    count_launch();
    return;
  }
  const long total = (long)B * h * C;
  BSB_LAUNCH(k_rowsum, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, B, inA, cA, ldA, inB, cB, ldB, h, w, rowsum_scratch);
  count_launch();
  ensure_dyn_smem(reinterpret_cast<const void*>(k_pool_fc), wbytes);
  BSB_LAUNCH(k_pool_fc, dim3((unsigned)B), dim3(256), wbytes, s, rowsum_scratch, h, C, (float)(h * w), pool_act, pooled_out, n_fc, f[0], f[1], out, ld_out);
  count_launch();
}

// ---------------------------------------------------------------------------
// Fused low-resolution inverted-residual block (see kernels.h).  Shared memory (floats):
//   xs [P][cin] | es [P][32] (one 32-channel slice of the expanded tensor) | ds [P][cexp] | rs [h][cexp] | fw [fcw]
// `fw` holds, one after another, the two SE weight matrices and the projection weights; when the whole
// layout would not fit it overlaps xs|es, which are dead by then (the residual is re-read from global).
// ---------------------------------------------------------------------------
struct MbDev {
  MbBlockArgs a; FcDev f0, f1;
  int off_es, off_ds, off_rs, off_fw;
};

__global__ void __launch_bounds__(512) k_mb_block(MbDev m) {
  BSB_DYN_SMEM(smem_raw);
  float* sm = reinterpret_cast<float*>(smem_raw);
  const MbBlockArgs& a = m.a;
  float* xs = sm; float* es = sm + m.off_es; float* ds = sm + m.off_ds; float* rs = sm + m.off_rs; float* fw = sm + m.off_fw;
  __shared__ float v0[128];
  __shared__ float v1[128];
  __shared__ float sv[128];
  __shared__ float w1s[64 * 32];
  const int tid = threadIdx.x, T = blockDim.x;
  const int P = a.h * a.w;
  const int b = blockIdx.x;
  const float* xg = a.x + (size_t)b * P * a.ld_x;
  // ---- x -> shared ----
  for (int i = tid; i < P * (a.cin / 4); i += T) {
    const int p = i / (a.cin / 4), q = i % (a.cin / 4);
    *reinterpret_cast<float4*>(xs + p * a.cin + 4 * q) = __ldg(reinterpret_cast<const float4*>(xg + (size_t)p * a.ld_x + 4 * q));
  }
  // ---- expand + depthwise, 32 channels at a time ----
  for (int c0 = 0; c0 < a.cexp; c0 += 32) {
    const int cw = min(32, a.cexp - c0);
    __syncthreads();                                   // xs ready / previous slice fully consumed
    for (int i = tid; i < a.cin * 32; i += T) {
      const int kk = i >> 5, j = i & 31;
      w1s[i] = j < cw ? __ldg(a.w1 + (size_t)kk * a.n4_1 + c0 + j) : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < P * 32; i += T) {
      const int p = i >> 5, j = i & 31;
      if (j >= cw) continue;
      float acc = 0.f;
      const float* xp = xs + p * a.cin;
      for (int kk = 0; kk < a.cin; ++kk) acc = fmaf(xp[kk], w1s[kk * 32 + j], acc);
      float v = acc + (a.b1 ? __ldg(a.b1 + c0 + j) : 0.f);
      es[i] = bsb_act(bsb_act(v, a.a1a), a.a1b);
    }
    __syncthreads();
    for (int i = tid; i < P * 32; i += T) {
      const int p = i >> 5, j = i & 31;
      if (j >= cw) continue;
      const int oy = p / a.w, ox = p - oy * a.w;
      float acc = 0.f;
      for (int fy = 0; fy < a.k; ++fy) {
        const int iy = oy - a.pt + fy;
        if (iy < 0 || iy >= a.h) continue;
        for (int fx = 0; fx < a.k; ++fx) {
          const int ix = ox - a.pl + fx;
          if (ix < 0 || ix >= a.w) continue;
          acc = fmaf(es[(iy * a.w + ix) * 32 + j], __ldg(a.wd + (size_t)(fy * a.k + fx) * a.cexp + c0 + j), acc);
        }
      }
      float v = acc + (a.bd ? __ldg(a.bd + c0 + j) : 0.f);
      ds[p * a.cexp + c0 + j] = bsb_act(bsb_act(v, a.ada), a.adb);
    }
  }
  __syncthreads();
  // ---- squeeze: row sums (x ascending), then rows (y ascending), / (h*w) ----
  for (int i = tid; i < a.h * a.cexp; i += T) {
    const int y = i / a.cexp, c = i - y * a.cexp;
    const float* dp = ds + (size_t)(y * a.w) * a.cexp + c;
    float r = 0.f;
    for (int x = 0; x < a.w; ++x) r = r + dp[x * a.cexp];
    rs[i] = r;
  }
  __syncthreads();                                     // also: xs / es are dead from here on
  for (int i = tid * 4; i < m.f0.K * m.f0.n4; i += T * 4) *reinterpret_cast<float4*>(fw + i) = __ldg(reinterpret_cast<const float4*>(m.f0.w + i));
  if (tid < a.cexp) {
    float t = 0.f;
    for (int y = 0; y < a.h; ++y) t = t + rs[y * a.cexp + tid];
    v0[tid] = bsb_act(bsb_div(t, (float)(a.h * a.w)), a.pool_act);
  }
  __syncthreads();
  if (tid < m.f0.N) {
    float acc = 0.f;
    for (int kk = 0; kk < m.f0.K; ++kk) acc = fmaf(v0[kk], fw[kk * m.f0.n4 + tid], acc);
    v1[tid] = bsb_act(bsb_act(acc + (m.f0.bias ? __ldg(m.f0.bias + tid) : 0.f), m.f0.act1), m.f0.act2);
  }
  __syncthreads();
  for (int i = tid * 4; i < m.f1.K * m.f1.n4; i += T * 4) *reinterpret_cast<float4*>(fw + i) = __ldg(reinterpret_cast<const float4*>(m.f1.w + i));
  __syncthreads();
  if (tid < m.f1.N) {
    float acc = 0.f;
    for (int kk = 0; kk < m.f1.K; ++kk) acc = fmaf(v1[kk], fw[kk * m.f1.n4 + tid], acc);
    sv[tid] = bsb_act(bsb_act(acc + (m.f1.bias ? __ldg(m.f1.bias + tid) : 0.f), m.f1.act1), m.f1.act2);
  }
  __syncthreads();
  // ---- excite + project (+ residual) ----
  for (int i = tid * 4; i < a.cexp * a.n4_2; i += T * 4) *reinterpret_cast<float4*>(fw + i) = __ldg(reinterpret_cast<const float4*>(a.w2 + i));
  __syncthreads();
  float* yg = a.y + (size_t)b * P * a.ld_y;
  const int cw2 = a.n4_2;                              // threads per pixel (output channels padded to 4)
  for (int i = tid; i < P * cw2; i += T) {
    const int p = i / cw2, n = i - p * cw2;
    if (n >= a.cout) continue;
    const float* dp = ds + (size_t)p * a.cexp;
    float acc = 0.f;
    for (int kk = 0; kk < a.cexp; ++kk) acc = fmaf(dp[kk] * sv[kk], fw[kk * a.n4_2 + n], acc);
    float v = acc + (a.b2 ? __ldg(a.b2 + n) : 0.f);
    v = bsb_act(bsb_act(v, a.a2a), a.a2b);
    if (a.residual) v = bsb_act(v + __ldg(xg + (size_t)p * a.ld_x + n), a.a3);
    yg[(size_t)p * a.ld_y + n] = v;
  }
}

static void mb_layout(int h, int w, int cin, int cexp, int fc_max, int* off_es, int* off_ds, int* off_rs, int* off_fw, size_t* total) {
  const int P = h * w;
  *off_es = P * cin; *off_ds = *off_es + P * 32; *off_rs = *off_ds + P * cexp;
  const int end = *off_rs + h * cexp;
  if ((size_t)(end + fc_max) * 4 <= 200 * 1024) { *off_fw = end; *total = (size_t)(end + fc_max) * 4; }
  else { *off_fw = 0; *total = (size_t)end * 4; if (fc_max > *off_ds) *total = 0; }      // overlap xs|es (dead by then)
}

size_t mb_block_smem_bytes(int h, int w, int cin, int cexp, int cout, int fc_max_floats) {
  if (h * w > 256 || cin > 64 || cexp > 128 || cout > 64 || cin % 4 || cexp % 4) return 0;
  int a, b, c, d; size_t total;
  mb_layout(h, w, cin, cexp, fc_max_floats, &a, &b, &c, &d, &total);
  return total <= 200 * 1024 ? total : 0;
}

void launch_mb_block(cudaStream_t s, int B, const MbBlockArgs& a) {
  MbDev m; m.a = a;
  m.f0 = FcDev{a.f0.w, a.f0.bias, a.f0.K, a.f0.N, a.f0.n4, a.f0.act1, a.f0.act2};
  m.f1 = FcDev{a.f1.w, a.f1.bias, a.f1.K, a.f1.N, a.f1.n4, a.f1.act1, a.f1.act2};
  const int fc_max = std::max(std::max(a.f0.K * a.f0.n4, a.f1.K * a.f1.n4), a.cexp * a.n4_2);
  size_t total;
  mb_layout(a.h, a.w, a.cin, a.cexp, fc_max, &m.off_es, &m.off_ds, &m.off_rs, &m.off_fw, &total);
  ensure_dyn_smem(reinterpret_cast<const void*>(k_mb_block), total);
  BSB_LAUNCH(k_mb_block, dim3((unsigned)B), dim3(512), total, s, m);
  count_launch();
}

// ---------------------------------------------------------------------------
// RESIZE_BILINEAR, float, NHWC.  One thread = one output pixel x 4 channels.
// ---------------------------------------------------------------------------
#define interp bsb_resize_interp

template <int VEC>
__global__ void __launch_bounds__(256) k_resize_bilinear(const float* in, int B, int ih, int iw, int c, int ld_in,
                                                         float* out, int oh, int ow, int ld_out,
                                                         float hs, float ws, bool half_pixel) {
  const int groups = (c + VEC - 1) / VEC;
  const long total = (long)B * oh * ow * groups;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c0 = (int)(idx % groups) * VEC;
  const long pix = idx / groups;
  const int x = (int)(pix % ow), y = (int)((pix / ow) % oh), b = (int)(pix / ((long)ow * oh));
  float fy, fx; int y0, y1, x0, x1;
  interp((float)y, hs, half_pixel, ih, &fy, &y0, &y1);
  interp((float)x, ws, half_pixel, iw, &fx, &x0, &x1);
  const float dy = fy - (float)y0, dx = fx - (float)x0;
  const float wy0 = 1.f - dy, wx0 = 1.f - dx;
  const float* inb = in + (size_t)b * ih * iw * ld_in + c0;
  const float* p00 = inb + ((size_t)y0 * iw + x0) * ld_in;
  const float* p10 = inb + ((size_t)y1 * iw + x0) * ld_in;
  const float* p01 = inb + ((size_t)y0 * iw + x1) * ld_in;
  const float* p11 = inb + ((size_t)y1 * iw + x1) * ld_in;
  float* op = out + (size_t)pix * ld_out + c0;
  if (VEC == 4 && ((c | ld_in | ld_out) & 3) == 0 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
    // channel counts that are multiples of 4 (all but DeepLab's 21-class head): 16-byte loads and one 16-byte store
    const float4 v00 = __ldg(reinterpret_cast<const float4*>(p00)), v10 = __ldg(reinterpret_cast<const float4*>(p10));
    const float4 v01 = __ldg(reinterpret_cast<const float4*>(p01)), v11 = __ldg(reinterpret_cast<const float4*>(p11));
    float4 r;
    r.x = ((v00.x * wy0 * wx0 + v10.x * dy * wx0) + v01.x * wy0 * dx) + v11.x * dy * dx;
    r.y = ((v00.y * wy0 * wx0 + v10.y * dy * wx0) + v01.y * wy0 * dx) + v11.y * dy * dx;
    r.z = ((v00.z * wy0 * wx0 + v10.z * dy * wx0) + v01.z * wy0 * dx) + v11.z * dy * dx;
    r.w = ((v00.w * wy0 * wx0 + v10.w * dy * wx0) + v01.w * wy0 * dx) + v11.w * dy * dx;
    *reinterpret_cast<float4*>(op) = r;
    return;
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    if (c0 + j >= c) break;
    const float a = __ldg(p00 + j) * wy0 * wx0;
    const float bb = __ldg(p10 + j) * dy * wx0;
    const float d = __ldg(p01 + j) * wy0 * dx;
    const float e = __ldg(p11 + j) * dy * dx;
    op[j] = ((a + bb) + d) + e;
  }
}

// RESIZE_BILINEAR fused into the 1x1 conv that consumes it: one thread = one output pixel and ALL its output channels
// (N <= 24); the interpolated input value (the exact expression of k_resize_bilinear above) is formed per channel in
// registers and fed straight into the k-ascending fmaf chains, so the up-sampled tensor is never written or re-read.
struct UpPwArgs {
  const float* in; const float* w; float* out;
  int B, ih, iw, K, ld_in, oh, ow, N, n4, ld_out;
  float hs, ws; bool half_pixel;
  EpiDev e;
};

template <int NQ, int MODE>     // output channel quads per thread; a pixel is shared by n4 / (4 * NQ) threads
__global__ void __launch_bounds__(128) k_upsample_pw(UpPwArgs a, int groups) {
  BSB_DYN_SMEM(smem_raw);
  float* Ws = reinterpret_cast<float*>(smem_raw);            // [K][n4]
  for (int i = threadIdx.x * 4; i < a.K * a.n4; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(Ws + i) = __ldg(reinterpret_cast<const float4*>(a.w + i));
  __syncthreads();
  const long total = (long)a.B * a.oh * a.ow * groups;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int grp = (int)(idx % groups);
  const long pix = idx / groups;
  const int nbase = grp * NQ * 4;
  const int x = (int)(pix % a.ow), y = (int)((pix / a.ow) % a.oh), b = (int)(pix / ((long)a.ow * a.oh));
  float fy, fx; int y0, y1, x0, x1;
  interp((float)y, a.hs, a.half_pixel, a.ih, &fy, &y0, &y1);
  interp((float)x, a.ws, a.half_pixel, a.iw, &fx, &x0, &x1);
  const float dy = fy - (float)y0, dx = fx - (float)x0;
  const float wy0 = 1.f - dy, wx0 = 1.f - dx;
  const float* inb = a.in + (size_t)b * a.ih * a.iw * a.ld_in;
  const float* p00 = inb + ((size_t)y0 * a.iw + x0) * a.ld_in;
  const float* p10 = inb + ((size_t)y1 * a.iw + x0) * a.ld_in;
  const float* p01 = inb + ((size_t)y0 * a.iw + x1) * a.ld_in;
  const float* p11 = inb + ((size_t)y1 * a.iw + x1) * a.ld_in;
  float acc[NQ * 4];
#pragma unroll
  for (int n = 0; n < NQ * 4; ++n) acc[n] = 0.f;
  float4 bias4[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) bias4[q] = epilogue_bias4<MODE>(a.e, nbase + 4 * q, a.N);
  // (unrolled so that the 16 loads of four k steps are in flight together: with one step at a time the 128-deep layer
  //  waits for them)
#pragma unroll 4
  for (int k = 0; k < a.K; k += 4) {
    const float4 v00 = __ldg(reinterpret_cast<const float4*>(p00 + k)), v10 = __ldg(reinterpret_cast<const float4*>(p10 + k));
    const float4 v01 = __ldg(reinterpret_cast<const float4*>(p01 + k)), v11 = __ldg(reinterpret_cast<const float4*>(p11 + k));
    float r[4];
    r[0] = ((v00.x * wy0 * wx0 + v10.x * dy * wx0) + v01.x * wy0 * dx) + v11.x * dy * dx;
    r[1] = ((v00.y * wy0 * wx0 + v10.y * dy * wx0) + v01.y * wy0 * dx) + v11.y * dy * dx;
    r[2] = ((v00.z * wy0 * wx0 + v10.z * dy * wx0) + v01.z * wy0 * dx) + v11.z * dy * dx;
    r[3] = ((v00.w * wy0 * wx0 + v10.w * dy * wx0) + v01.w * wy0 * dx) + v11.w * dy * dx;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* wr = Ws + (size_t)(k + j) * a.n4 + nbase;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const float4 w4 = *reinterpret_cast<const float4*>(wr + 4 * q);
        acc[4 * q] = fmaf(r[j], w4.x, acc[4 * q]); acc[4 * q + 1] = fmaf(r[j], w4.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(r[j], w4.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(r[j], w4.w, acc[4 * q + 3]);
      }
    }
  }
  float* op = a.out + (size_t)pix * a.ld_out;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const int n0 = nbase + 4 * q;
    const float bj[4] = {bias4[q].x, bias4[q].y, bias4[q].z, bias4[q].w};
    if (n0 + 3 < a.N) {
      *reinterpret_cast<float4*>(op + n0) = make_float4(epilogue_m<MODE>(acc[4 * q], bj[0], n0, (size_t)pix, a.e), epilogue_m<MODE>(acc[4 * q + 1], bj[1], n0 + 1, (size_t)pix, a.e),
                                                        epilogue_m<MODE>(acc[4 * q + 2], bj[2], n0 + 2, (size_t)pix, a.e), epilogue_m<MODE>(acc[4 * q + 3], bj[3], n0 + 3, (size_t)pix, a.e));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (n0 + j < a.N) op[n0 + j] = epilogue_m<MODE>(acc[4 * q + j], bj[j], n0 + j, (size_t)pix, a.e);
    }
  }
}

// Staged form for pixels that are shared by several threads (groups > 1: few output quads per thread so that small
// layers still fill the GPU): the kernel above recomputes the interpolated operand — 4 loads and 44 flops per 4 input
// channels — in every one of the pixel's threads, 6 times over for the 128 -> 24 layer of the Meet decoder, where it was
// 2/3 of the instructions.
// Here a block owns PB = 128 / groups pixels: its threads first build the interpolated rows once ([PB][K + 4] floats in
// shared memory; thread (pixel, g) takes the float4 chunks g, g + groups, ...), then run the k-ascending fmaf chains from
// there.  The interpolated value is formed by the same expression, so the bits are those of the unstaged kernel.
template <int NQ, int MODE>
__global__ void __launch_bounds__(128) k_upsample_pw_staged(UpPwArgs a, int groups) {
  BSB_DYN_SMEM(smem_raw);
  float* Ws = reinterpret_cast<float*>(smem_raw);            // [K][n4]
  float* As = Ws + (size_t)a.K * a.n4;                        // [PB][K + 4]
  const int lda = a.K + 4;
  for (int i = threadIdx.x * 4; i < a.K * a.n4; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(Ws + i) = __ldg(reinterpret_cast<const float4*>(a.w + i));
  const int PB = 128 / groups;
  const int lp = threadIdx.x / groups, grp = threadIdx.x - lp * groups;
  const long pix = (long)blockIdx.x * PB + lp;
  const bool valid = lp < PB && pix < (long)a.B * a.oh * a.ow;
  if (valid) {
    const int x = (int)(pix % a.ow), y = (int)((pix / a.ow) % a.oh), b = (int)(pix / ((long)a.ow * a.oh));
    float fy, fx; int y0, y1, x0, x1;
    interp((float)y, a.hs, a.half_pixel, a.ih, &fy, &y0, &y1);
    interp((float)x, a.ws, a.half_pixel, a.iw, &fx, &x0, &x1);
    const float dy = fy - (float)y0, dx = fx - (float)x0;
    const float wy0 = 1.f - dy, wx0 = 1.f - dx;
    const float* inb = a.in + (size_t)b * a.ih * a.iw * a.ld_in;
    const float* p00 = inb + ((size_t)y0 * a.iw + x0) * a.ld_in;
    const float* p10 = inb + ((size_t)y1 * a.iw + x0) * a.ld_in;
    const float* p01 = inb + ((size_t)y0 * a.iw + x1) * a.ld_in;
    const float* p11 = inb + ((size_t)y1 * a.iw + x1) * a.ld_in;
    float* arow = As + (size_t)lp * lda;
#pragma unroll 2
    for (int k = 4 * grp; k < a.K; k += 4 * groups) {
      const float4 v00 = __ldg(reinterpret_cast<const float4*>(p00 + k)), v10 = __ldg(reinterpret_cast<const float4*>(p10 + k));
      const float4 v01 = __ldg(reinterpret_cast<const float4*>(p01 + k)), v11 = __ldg(reinterpret_cast<const float4*>(p11 + k));
      float4 r;
      r.x = ((v00.x * wy0 * wx0 + v10.x * dy * wx0) + v01.x * wy0 * dx) + v11.x * dy * dx;
      r.y = ((v00.y * wy0 * wx0 + v10.y * dy * wx0) + v01.y * wy0 * dx) + v11.y * dy * dx;
      r.z = ((v00.z * wy0 * wx0 + v10.z * dy * wx0) + v01.z * wy0 * dx) + v11.z * dy * dx;
      r.w = ((v00.w * wy0 * wx0 + v10.w * dy * wx0) + v01.w * wy0 * dx) + v11.w * dy * dx;
      *reinterpret_cast<float4*>(arow + k) = r;
    }
  }
  __syncthreads();
  if (!valid) return;
  const int nbase = grp * NQ * 4;
  float acc[NQ * 4];
#pragma unroll
  for (int n = 0; n < NQ * 4; ++n) acc[n] = 0.f;
  float4 bias4[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) bias4[q] = epilogue_bias4<MODE>(a.e, nbase + 4 * q, a.N);
  const float* arow = As + (size_t)lp * lda;
#pragma unroll 4
  for (int k = 0; k < a.K; k += 4) {
    const float4 r4 = *reinterpret_cast<const float4*>(arow + k);
    const float r[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* wr = Ws + (size_t)(k + j) * a.n4 + nbase;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const float4 w4 = *reinterpret_cast<const float4*>(wr + 4 * q);
        acc[4 * q] = fmaf(r[j], w4.x, acc[4 * q]); acc[4 * q + 1] = fmaf(r[j], w4.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(r[j], w4.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(r[j], w4.w, acc[4 * q + 3]);
      }
    }
  }
  float* op = a.out + (size_t)pix * a.ld_out;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const int n0 = nbase + 4 * q;
    const float bj[4] = {bias4[q].x, bias4[q].y, bias4[q].z, bias4[q].w};
    if (n0 + 3 < a.N) {
      *reinterpret_cast<float4*>(op + n0) = make_float4(epilogue_m<MODE>(acc[4 * q], bj[0], n0, (size_t)pix, a.e), epilogue_m<MODE>(acc[4 * q + 1], bj[1], n0 + 1, (size_t)pix, a.e),
                                                        epilogue_m<MODE>(acc[4 * q + 2], bj[2], n0 + 2, (size_t)pix, a.e), epilogue_m<MODE>(acc[4 * q + 3], bj[3], n0 + 3, (size_t)pix, a.e));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (n0 + j < a.N) op[n0 + j] = epilogue_m<MODE>(acc[4 * q + j], bj[j], n0 + j, (size_t)pix, a.e);
    }
  }
}

bool upsample_pw_supported(int K, int N, int n4, int ld_in, int ld_out) {
  return K % 4 == 0 && ld_in % 4 == 0 && ld_out % 4 == 0 && n4 % 4 == 0 && n4 >= 4 && n4 <= 24 && N <= n4 && (size_t)K * n4 * 4 <= 48 * 1024;
}

void launch_upsample_pw(cudaStream_t s, int B, const float* in, int ih, int iw, int K, int ld_in, bool align_corners, bool half_pixel,
                        const float* w_kn, int n4, int N, float* out, int oh, int ow, int ld_out, const Epilogue& e) {
  float hs = (float)ih / (float)oh, ws = (float)iw / (float)ow;
  if (align_corners && oh > 1) hs = (float)(ih - 1) / (float)(oh - 1);
  if (align_corners && ow > 1) ws = (float)(iw - 1) / (float)(ow - 1);
  UpPwArgs a{in, w_kn, out, B, ih, iw, K, ld_in, oh, ow, N, n4, ld_out, hs, ws, half_pixel, to_dev(e)};
  const long pixels = (long)B * oh * ow;
  const size_t smem = sizeof(float) * (size_t)K * n4;
  const int quads = n4 / 4;
  // a pixel's output quads are split over threads until the grid fills the GPU a few times over (the interpolation is
  // recomputed per thread; it is cheap next to the K x 4 fmaf chains)
  int nq = quads;
  while (nq > 1 && (nq % 2 == 0 || nq % 3 == 0) && pixels * (quads / nq) < device_sms() * 2048L) nq = (nq % 2 == 0) ? nq / 2 : nq / 3;
  const int groups = quads / nq;
  const dim3 grid((unsigned)((pixels * groups + 127) / 128)), block(128);
  // (the five graphs only ever put a plain bias behind this op: one specialised instance per NQ, generic otherwise)
  const bool plain = epi_mode(e) == 0;
  const size_t smem_staged = smem + sizeof(float) * (size_t)(128 / groups) * (K + 4);
  if (tuning().up_staged && groups > 1 && nq <= 3 && smem_staged <= 48 * 1024) {
    const int PB = 128 / groups;
    const dim3 sgrid((unsigned)((pixels + PB - 1) / PB));
    switch (nq) {
      case 1: if (plain) { auto k = k_upsample_pw_staged<1, 0>; BSB_LAUNCH(k, sgrid, block, smem_staged, s, a, groups); } else { auto k = k_upsample_pw_staged<1, -1>; BSB_LAUNCH(k, sgrid, block, smem_staged, s, a, groups); } break;
      case 2: if (plain) { auto k = k_upsample_pw_staged<2, 0>; BSB_LAUNCH(k, sgrid, block, smem_staged, s, a, groups); } else { auto k = k_upsample_pw_staged<2, -1>; BSB_LAUNCH(k, sgrid, block, smem_staged, s, a, groups); } break;
      default: if (plain) { auto k = k_upsample_pw_staged<3, 0>; BSB_LAUNCH(k, sgrid, block, smem_staged, s, a, groups); } else { auto k = k_upsample_pw_staged<3, -1>; BSB_LAUNCH(k, sgrid, block, smem_staged, s, a, groups); } break;
    }
    count_launch();
    return;
  }
  switch (nq) {
    case 1: if (plain) { auto k = k_upsample_pw<1, 0>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } else { auto k = k_upsample_pw<1, -1>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } break;
    case 2: if (plain) { auto k = k_upsample_pw<2, 0>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } else { auto k = k_upsample_pw<2, -1>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } break;
    case 3: if (plain) { auto k = k_upsample_pw<3, 0>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } else { auto k = k_upsample_pw<3, -1>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } break;
    case 4: if (plain) { auto k = k_upsample_pw<4, 0>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } else { auto k = k_upsample_pw<4, -1>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } break;
    case 5: if (plain) { auto k = k_upsample_pw<5, 0>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } else { auto k = k_upsample_pw<5, -1>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } break;
    default: if (plain) { auto k = k_upsample_pw<6, 0>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } else { auto k = k_upsample_pw<6, -1>; BSB_LAUNCH(k, grid, block, smem, s, a, groups); } break;
  }
  count_launch();
}

void launch_resize_bilinear(cudaStream_t s, int B, const float* in, int ih, int iw, int c, int ld_in,
                            float* out, int oh, int ow, int ld_out, bool align_corners, bool half_pixel) {
  float hs = (float)ih / (float)oh, ws = (float)iw / (float)ow;
  if (align_corners && oh > 1) hs = (float)(ih - 1) / (float)(oh - 1);
  if (align_corners && ow > 1) ws = (float)(iw - 1) / (float)(ow - 1);
  const long total = (long)B * oh * ow * ((c + 3) / 4);
  BSB_LAUNCH(k_resize_bilinear<4>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s,
             in, B, ih, iw, c, ld_in, out, oh, ow, ld_out, hs, ws, half_pixel);
  count_launch();
}

// ---------------------------------------------------------------------------
// Decoder stage of the MobileNetV3-style graphs in one kernel (C = 16 or 24 channels):
//     t = act_p( (x * sv + add) . Wp + bp )            1x1 conv with the squeeze-excite scale / skip add on its operand
//     u = act_r( t + act_d( dw3x3(t) + bd ) )          depthwise 3x3 (stride 1) + residual of its own input
//     out = u                                          ... or, for the last stage,
//     out = act_t( tconv2x2( u ) + bt )                Convolution2DTransposeBias k2 s2 (lib/transpose_conv_bias.cc:37-114)
// One CTA = a 32 x 8 pixel tile: phase A computes t for the tile and its 1-pixel ring into shared memory (a pixel and all
// its C channels per thread: the k-ascending fmaf chains of the stand-alone 1x1 kernel); phase B = one thread per pixel:
// 9 taps x C from shared memory in (fy, fx) order skipping out-of-image taps, residual, then the 2x2 x oc transposed
// conv straight from registers.  t and u never touch global memory.
// ---------------------------------------------------------------------------
struct HeadArgs {
  const float* x; int ld_x; const float* sv; const float* add; int ld_add;     // sv: [B][C] or null; add: same shape as x or null
  const float* wp; const float* bp; int actp1, actp2;                             // [C][n4 = C]
  const float* wd; const float* bd; int actd1, actd2, actr;                       // [3][3][C]
  const float* wt; const float* bt; int oc, actt;                                 // OHWI [oc][2][2][C]; null -> no transposed conv
  float* out; int ld_out;                                                          // [B][h][w][ld_out] or [B][2h][2w][oc]
  int B, h, w, pt, pl;
};
constexpr int HD_TW = 32, HD_TH = 8, HD_SW = HD_TW + 2, HD_SH = HD_TH + 2;

// FAST: no activation on the 1x1, bias + RELU6 on the depthwise, plain residual add, no activation on the transposed
// conv — what the three decoder stages of the Meet / MLKit graphs are — fixed at compile time; anything else takes the
// run-time switches.  A pixel's channels sit C + 4 floats apart in shared memory: with a stride of C (64 / 96 bytes) the
// 16-byte accesses of neighbouring lanes fell on two / four bank groups (4-way conflicts on every tap load and store).
// CFG 1: Meet (1x1 none, depthwise RELU6, transposed conv none); CFG 2: MLKit (RELU, RELU, LOGISTIC); CFG 0: run time.
template <int CFG> struct HeadCfg { static constexpr int P = CFG == 1 ? ACT_NONE : ACT_RELU, D = CFG == 1 ? ACT_RELU6 : ACT_RELU, T = CFG == 1 ? ACT_NONE : ACT_LOGISTIC; };
template <int C, int CFG>
__global__ void __launch_bounds__(256) k_head(HeadArgs a) {
  constexpr bool FAST = CFG != 0;
  using HC = HeadCfg<CFG>;
  constexpr int CP = C + 4;
  __shared__ __align__(16) float ts[HD_SH * HD_SW * CP];
  __shared__ __align__(16) float wps[C * C];
  __shared__ __align__(16) float wds[9 * C];
  __shared__ __align__(16) float wts[2 * 4 * C];
  __shared__ __align__(16) float bps[C], bds[C], bts[4];
  const int tid = threadIdx.x;
  const int x0 = blockIdx.x * HD_TW, y0 = blockIdx.y * HD_TH, b = blockIdx.z;
  for (int i = tid; i < C * C; i += 256) wps[i] = __ldg(a.wp + i);
  for (int i = tid; i < 9 * C; i += 256) wds[i] = __ldg(a.wd + i);
  if (a.wt) for (int i = tid; i < a.oc * 4 * C; i += 256) wts[i] = __ldg(a.wt + i);
  if (tid < C) { bps[tid] = a.bp ? __ldg(a.bp + tid) : 0.f; bds[tid] = a.bd ? __ldg(a.bd + tid) : 0.f; }
  if (tid < 4) bts[tid] = (a.wt && tid < a.oc) ? __ldg(a.bt + tid) : 0.f;
  __syncthreads();
  const float* xb = a.x + (size_t)b * a.h * a.w * a.ld_x;
  const float* ab = a.add ? a.add + (size_t)b * a.h * a.w * a.ld_add : nullptr;
  const float* svb = a.sv ? a.sv + (size_t)b * C : nullptr;
  // ---- A: t on the (TH + 2) x (TW + 2) ring-extended tile ----
  for (int i = tid; i < HD_SH * HD_SW; i += 256) {
    const int sy = i / HD_SW, sx = i - sy * HD_SW;
    const int gy = y0 + sy - 1, gx = x0 + sx - 1;
    if (gy < 0 || gy >= a.h || gx < 0 || gx >= a.w) continue;          // never read: phase B skips out-of-image taps
    const size_t pix = (size_t)gy * a.w + gx;
    float4 xv[C / 4];
#pragma unroll
    for (int k = 0; k < C / 4; ++k) xv[k] = __ldg(reinterpret_cast<const float4*>(xb + pix * a.ld_x + 4 * k));
    if (svb) {
#pragma unroll
      for (int k = 0; k < C / 4; ++k) {
        const float4 sc = __ldg(reinterpret_cast<const float4*>(svb + 4 * k));
        xv[k].x = xv[k].x * sc.x; xv[k].y = xv[k].y * sc.y; xv[k].z = xv[k].z * sc.z; xv[k].w = xv[k].w * sc.w;
      }
    }
    if (ab) {
#pragma unroll
      for (int k = 0; k < C / 4; ++k) {
        const float4 ad = __ldg(reinterpret_cast<const float4*>(ab + pix * a.ld_add + 4 * k));
        xv[k].x = xv[k].x + ad.x; xv[k].y = xv[k].y + ad.y; xv[k].z = xv[k].z + ad.z; xv[k].w = xv[k].w + ad.w;
      }
    }
    float acc[C];
#pragma unroll
    for (int n = 0; n < C; ++n) acc[n] = 0.f;
#pragma unroll
    for (int k = 0; k < C / 4; ++k) {
      const float vv[4] = {xv[k].x, xv[k].y, xv[k].z, xv[k].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < C / 4; ++q) {
          const float4 w4 = *reinterpret_cast<const float4*>(wps + (4 * k + j) * C + 4 * q);
          acc[4 * q] = fmaf(vv[j], w4.x, acc[4 * q]); acc[4 * q + 1] = fmaf(vv[j], w4.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(vv[j], w4.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(vv[j], w4.w, acc[4 * q + 3]);
        }
    }
    float* tp = ts + (size_t)i * CP;
#pragma unroll
    for (int q = 0; q < C / 4; ++q) {
      float r[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = acc[4 * q + j] + bps[4 * q + j];
        r[j] = FAST ? bsb_act(v, HC::P) : bsb_act(bsb_act(v, a.actp1), a.actp2);
      }
      *reinterpret_cast<float4*>(tp + 4 * q) = make_float4(r[0], r[1], r[2], r[3]);
    }
  }
  __syncthreads();
  // ---- B: depthwise 3x3 + residual (+ transposed conv) ----
  const int lx = tid & (HD_TW - 1), ly = tid >> 5;
  const int gx = x0 + lx, gy = y0 + ly;
  if (gx >= a.w || gy >= a.h) return;
  float u[C];
#pragma unroll
  for (int c = 0; c < C; ++c) u[c] = 0.f;
#pragma unroll
  for (int fy = 0; fy < 3; ++fy) {
    const int iy = gy - a.pt + fy;
    if (iy < 0 || iy >= a.h) continue;
#pragma unroll
    for (int fx = 0; fx < 3; ++fx) {
      const int ix = gx - a.pl + fx;
      if (ix < 0 || ix >= a.w) continue;
      const float* tp = ts + (size_t)((iy - y0 + 1) * HD_SW + (ix - x0 + 1)) * CP;
      const float* wp = wds + (fy * 3 + fx) * C;
#pragma unroll
      for (int q = 0; q < C / 4; ++q) {
        const float4 t4 = *reinterpret_cast<const float4*>(tp + 4 * q), w4 = *reinterpret_cast<const float4*>(wp + 4 * q);
        u[4 * q] = fmaf(t4.x, w4.x, u[4 * q]); u[4 * q + 1] = fmaf(t4.y, w4.y, u[4 * q + 1]);
        u[4 * q + 2] = fmaf(t4.z, w4.z, u[4 * q + 2]); u[4 * q + 3] = fmaf(t4.w, w4.w, u[4 * q + 3]);
      }
    }
  }
  {
    const float* tc = ts + (size_t)((ly + 1) * HD_SW + lx + 1) * CP;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float v = u[c] + bds[c];
      const float d = FAST ? bsb_act(v, HC::D) : bsb_act(bsb_act(v, a.actd1), a.actd2);
      u[c] = FAST ? d + tc[c] : bsb_act(d + tc[c], a.actr);    // ADD(t, act(dw(t))): the planner folded it as residual of the depthwise step
    }
  }
  if (!a.wt) {
    float* op = a.out + (((size_t)b * a.h + gy) * a.w + gx) * a.ld_out;
#pragma unroll
    for (int c = 0; c < C; c += 4) *reinterpret_cast<float4*>(op + c) = make_float4(u[c], u[c + 1], u[c + 2], u[c + 3]);
    return;
  }
  const int oh = 2 * a.h, ow = 2 * a.w;
#pragma unroll
  for (int fy = 0; fy < 2; ++fy) {
    float r[2][2];
#pragma unroll
    for (int fx = 0; fx < 2; ++fx)
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        r[fx][o] = 0.f;
        if (o >= a.oc) continue;
        const float* wq = wts + ((o * 2 + fy) * 2 + fx) * C;
        float acc = bts[o];
#pragma unroll
        for (int c = 0; c < C; ++c) acc = fmaf(u[c], wq[c], acc);
        r[fx][o] = FAST ? bsb_act(acc, HC::T) : bsb_act(acc, a.actt);
      }
    float* op = a.out + (((size_t)b * oh + 2 * gy + fy) * ow + 2 * gx) * a.oc;
    if (a.oc == 2) *reinterpret_cast<float4*>(op) = make_float4(r[0][0], r[0][1], r[1][0], r[1][1]);
    else *reinterpret_cast<float2*>(op) = make_float2(r[0][0], r[1][0]);
  }
}

// ---------------------------------------------------------------------------
// Encoder entry of the MobileNetV3-style graphs in one kernel (16 channels):
//     t   = act_p( x . Wp + bp )                       1x1 conv on the stem's output (72x128 / 128x128 pixels)
//     out = act_d( dw3x3 stride 2 (t) + bd )           depthwise 3x3, stride 2
// The 1x1's output — the largest activation of the graph — is never written or re-read: one CTA = a 16 x 8 tile of the
// depthwise OUTPUT; phase A computes t on the 33 x 17 input pixels the tile needs into shared memory (a pixel and its 16
// channels per thread, k-ascending fmaf chains, as the stand-alone 1x1 kernel), phase B = a thread per output pixel and
// 8 channels: 9 taps in (fy, fx) order from shared memory, out-of-image taps skipped.  (Pixels shared by neighbouring
// tiles — one row and one column in 17 x 33 — are computed twice; each value is still the one chain of the oracle.)
// ---------------------------------------------------------------------------
struct PwDwArgs {
  const float* x; int ld_x; const float* wp; const float* bp; int actp;     // [16][16]
  const float* wd; const float* bd; int actd;                                 // [3][3][16]
  float* out; int ld_out;
  int B, ih, iw, oh, ow, pt, pl;
};
constexpr int PD_TW = 16, PD_TH = 8, PD_SW = 2 * PD_TW + 1, PD_SH = 2 * PD_TH + 1, PD_C = 16, PD_CP = PD_C + 4;

template <int ACTP, int ACTD>     // -1: run-time activation code
__global__ void __launch_bounds__(256) k_pw_dws2(PwDwArgs a) {
  __shared__ __align__(16) float ts[PD_SH * PD_SW * PD_CP];
  __shared__ __align__(16) float wps[PD_C * PD_C];
  __shared__ __align__(16) float wds[9 * PD_C];
  __shared__ __align__(16) float bps[PD_C], bds[PD_C];
  const int tid = threadIdx.x;
  const int ox0 = blockIdx.x * PD_TW, oy0 = blockIdx.y * PD_TH, b = blockIdx.z;
  const int ix0 = ox0 * 2 - a.pl, iy0 = oy0 * 2 - a.pt;         // input pixel of the tile's shared-memory origin
  for (int i = tid; i < PD_C * PD_C; i += 256) wps[i] = __ldg(a.wp + i);
  for (int i = tid; i < 9 * PD_C; i += 256) wds[i] = __ldg(a.wd + i);
  if (tid < PD_C) { bps[tid] = a.bp ? __ldg(a.bp + tid) : 0.f; bds[tid] = a.bd ? __ldg(a.bd + tid) : 0.f; }
  __syncthreads();
  const float* xb = a.x + (size_t)b * a.ih * a.iw * a.ld_x;
  // ---- A: t on the (2 TH + 1) x (2 TW + 1) input window ----
  for (int i = tid; i < PD_SH * PD_SW; i += 256) {
    const int sy = i / PD_SW, sx = i - sy * PD_SW;
    const int gy = iy0 + sy, gx = ix0 + sx;
    if (gy < 0 || gy >= a.ih || gx < 0 || gx >= a.iw) continue;          // never read: phase B skips out-of-image taps
    const float* xp = xb + ((size_t)gy * a.iw + gx) * a.ld_x;
    float4 xv[PD_C / 4];
#pragma unroll
    for (int k = 0; k < PD_C / 4; ++k) xv[k] = __ldg(reinterpret_cast<const float4*>(xp + 4 * k));
    float acc[PD_C];
#pragma unroll
    for (int n = 0; n < PD_C; ++n) acc[n] = 0.f;
#pragma unroll
    for (int k = 0; k < PD_C / 4; ++k) {
      const float vv[4] = {xv[k].x, xv[k].y, xv[k].z, xv[k].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < PD_C / 4; ++q) {
          const float4 w4 = *reinterpret_cast<const float4*>(wps + (4 * k + j) * PD_C + 4 * q);
          acc[4 * q] = fmaf(vv[j], w4.x, acc[4 * q]); acc[4 * q + 1] = fmaf(vv[j], w4.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(vv[j], w4.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(vv[j], w4.w, acc[4 * q + 3]);
        }
    }
    float* tp = ts + (size_t)i * PD_CP;
#pragma unroll
    for (int q = 0; q < PD_C / 4; ++q) {
      float r[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) r[j] = bsb_act(acc[4 * q + j] + bps[4 * q + j], ACTP >= 0 ? ACTP : a.actp);
      *reinterpret_cast<float4*>(tp + 4 * q) = make_float4(r[0], r[1], r[2], r[3]);
    }
  }
  __syncthreads();
  // ---- B: depthwise 3x3 stride 2: thread = output pixel x 8 channels ----
  const int half = tid & 1, lp = tid >> 1;
  const int lx = lp % PD_TW, ly = lp / PD_TW;
  const int ox = ox0 + lx, oy = oy0 + ly;
  if (ox >= a.ow || oy >= a.oh) return;
  const int c0 = half * 8;
  float4 u0 = make_float4(0.f, 0.f, 0.f, 0.f), u1 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int fy = 0; fy < 3; ++fy) {
    const int iy = oy * 2 - a.pt + fy;
    if (iy < 0 || iy >= a.ih) continue;
#pragma unroll
    for (int fx = 0; fx < 3; ++fx) {
      const int ix = ox * 2 - a.pl + fx;
      if (ix < 0 || ix >= a.iw) continue;
      const float* tp = ts + (size_t)((2 * ly + fy) * PD_SW + (2 * lx + fx)) * PD_CP + c0;
      const float* wp = wds + (fy * 3 + fx) * PD_C + c0;
      const float4 t0 = *reinterpret_cast<const float4*>(tp), t1 = *reinterpret_cast<const float4*>(tp + 4);
      const float4 w0 = *reinterpret_cast<const float4*>(wp), w1 = *reinterpret_cast<const float4*>(wp + 4);
      u0.x = fmaf(t0.x, w0.x, u0.x); u0.y = fmaf(t0.y, w0.y, u0.y); u0.z = fmaf(t0.z, w0.z, u0.z); u0.w = fmaf(t0.w, w0.w, u0.w);
      u1.x = fmaf(t1.x, w1.x, u1.x); u1.y = fmaf(t1.y, w1.y, u1.y); u1.z = fmaf(t1.z, w1.z, u1.z); u1.w = fmaf(t1.w, w1.w, u1.w);
    }
  }
  const int ad = ACTD >= 0 ? ACTD : a.actd;
  float* op = a.out + (((size_t)b * a.oh + oy) * a.ow + ox) * a.ld_out + c0;
  *reinterpret_cast<float4*>(op) = make_float4(bsb_act(u0.x + bds[c0], ad), bsb_act(u0.y + bds[c0 + 1], ad), bsb_act(u0.z + bds[c0 + 2], ad), bsb_act(u0.w + bds[c0 + 3], ad));
  *reinterpret_cast<float4*>(op + 4) = make_float4(bsb_act(u1.x + bds[c0 + 4], ad), bsb_act(u1.y + bds[c0 + 5], ad), bsb_act(u1.z + bds[c0 + 6], ad), bsb_act(u1.w + bds[c0 + 7], ad));
}

bool pw_dws2_supported(int K, int N, int ld_x, int ld_out) { return K == PD_C && N == PD_C && ld_x % 4 == 0 && ld_out % 4 == 0; }

void launch_pw_dws2(cudaStream_t s, const float* x, int ld_x, const float* wp, const float* bp, int actp, const float* wd, const float* bd, int actd,
                    float* out, int ld_out, int B, int ih, int iw, int oh, int ow, int pt, int pl) {
  PwDwArgs a{x, ld_x, wp, bp, actp, wd, bd, actd, out, ld_out, B, ih, iw, oh, ow, pt, pl};
  const dim3 grid((unsigned)ceil_div(ow, PD_TW), (unsigned)ceil_div(oh, PD_TH), (unsigned)B);
  if (actp == ACT_RELU6 && actd == ACT_RELU6) { auto k = k_pw_dws2<ACT_RELU6, ACT_RELU6>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else if (actp == ACT_RELU && actd == ACT_RELU) { auto k = k_pw_dws2<ACT_RELU, ACT_RELU>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  else { auto k = k_pw_dws2<-1, -1>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  count_launch();
}

bool head_supported(int C, int ld_x, int ld_add, int ld_out, int oc, bool tconv) {
  if (C != 16 && C != 24) return false;
  if (ld_x % 4 || ld_add % 4) return false;
  if (tconv) return oc >= 1 && oc <= 2;
  return ld_out % 4 == 0;
}

void launch_head(cudaStream_t s, int C, const float* x, int ld_x, const float* sv, const float* add, int ld_add,
                 const float* wp, const float* bp, int actp1, int actp2, const float* wd, const float* bd, int actd1, int actd2, int actr,
                 const float* wt, const float* bt, int oc, int actt, float* out, int ld_out, int B, int h, int w, int pt, int pl) {
  HeadArgs a{x, ld_x, sv, add, ld_add, wp, bp, actp1, actp2, wd, bd, actd1, actd2, actr, wt, bt, oc, actt, out, ld_out, B, h, w, pt, pl};
  const dim3 grid((unsigned)ceil_div(w, HD_TW), (unsigned)ceil_div(h, HD_TH), (unsigned)B);
  auto one = [](int a1, int a2, int want) { return (a1 == ACT_NONE && a2 == want) || (a1 == want && a2 == ACT_NONE); };
  int cfg = 0;
  if (actr == ACT_NONE && one(actp1, actp2, ACT_NONE) && one(actd1, actd2, ACT_RELU6) && (!wt || actt == ACT_NONE)) cfg = 1;
  else if (actr == ACT_NONE && one(actp1, actp2, ACT_RELU) && one(actd1, actd2, ACT_RELU) && (!wt || actt == ACT_LOGISTIC)) cfg = 2;
  if (C == 16) {
    if (cfg == 1) { auto k = k_head<16, 1>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
    else if (cfg == 2) { auto k = k_head<16, 2>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
    else { auto k = k_head<16, 0>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  } else {
    if (cfg == 1) { auto k = k_head<24, 1>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
    else if (cfg == 2) { auto k = k_head<24, 2>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
    else { auto k = k_head<24, 0>; BSB_LAUNCH(k, grid, dim3(256), 0, s, a); }
  }
  count_launch();
}

// ---------------------------------------------------------------------------
// The two inverted-residual blocks between the encoder entry and the chain of the Meet / MLKit graphs, one kernel each
// (kernels.h, EncBlocksArgs).  One CTA = a 4 x 16 tile of the block's output; everything it needs from the block's
// input window is recomputed in shared memory, so the expanded tensors (t29 .. t44, 72 / 88 channels) never reach
// global memory.  Pixels shared with neighbouring tiles are computed twice; each value is still the one chain of the
// stand-alone kernels (1x1: fmaf over k ascending from +0, operand scaled first, bias last, then the activation, then
// the residual; depthwise: taps in (fy, fx) order, out-of-image taps skipped, bias last).
//   A (k_enc_block_s2): window (2 TH + 1) x (2 TW + 1) of the input; t25 on the window (written to global only for
//     the pixels this tile owns, so each t25 pixel has one writer), then the 72 expanded channels in slices of 24:
//     expand -> stride-2 depthwise -> project, the project's accumulators persisting across the slices.
//   B (k_enc_block_res): window (TH + 2) x (TW + 2) of t36; expand all 88 channels -> depthwise -> project + t36
//     (from the window centre) = t48, then t52 = hswish(t48 . W5 + b5) from the tile's t48 in shared memory.
// Thread maps: the lanes of a warp take consecutive pixels and one channel group, so every weight read is a broadcast;
// the pixel-major buffers read by pixel have an odd stride and the depthwise results are stored channel-major [c][64],
// so those reads are free of bank conflicts.  Projects: thread = tile pixel (tid % 64) x 6 of the 24 output channels.
// ---------------------------------------------------------------------------
constexpr int EB_TH = 4, EB_TW = 16, EB_NP = EB_TH * EB_TW;
constexpr int EB_C0 = 16, EB_E1 = 72, EB_C1 = 24, EB_E2 = 88, EB_C2 = 96;
constexpr int eb_r4(int x) { return (x + 3) / 4 * 4; }
// A: shared memory in floats (every region starts on 16 bytes)
constexpr int EA_WH = 2 * EB_TH + 1, EA_WW = 2 * EB_TW + 1, EA_WP = EA_WH * EA_WW, EA_S = 24, EA_Q = 12;
constexpr int EA_P25 = EB_C0 + 1, EA_PE = EA_S + 4;                       // pixel strides of t25 (odd), of the slice
constexpr int EA_W0 = 0, EA_B0 = EA_W0 + EB_C0 * EB_C0, EA_SV = EA_B0 + EB_C0, EA_W1 = EA_SV + EB_C0, EA_B1 = EA_W1 + EB_C0 * EB_E1,
              EA_WD = EA_B1 + EB_E1, EA_BD = EA_WD + 9 * EB_E1, EA_W2 = EA_BD + EB_E1, EA_B2 = EA_W2 + EB_E1 * EB_C1,
              EA_T25 = EA_B2 + EB_C1, EA_E = EA_T25 + eb_r4(EA_WP * EA_P25), EA_D = EA_E + EA_WP * EA_PE, EA_END = EA_D + EA_S * EB_NP;
// B
constexpr int EB_WH = EB_TH + 2, EB_WW = EB_TW + 2, EB_WP = EB_WH * EB_WW, EB_Q = 8;
constexpr int EB_PX = EB_C1 + 1, EB_PE = EB_E2 + 4;                       // pixel strides of t36 (odd), of the expanded tensor
constexpr int EB_W3 = 0, EB_B3 = EB_W3 + EB_C1 * EB_E2, EB_WD = EB_B3 + EB_E2, EB_BD = EB_WD + 9 * EB_E2, EB_W4 = EB_BD + EB_E2,
              EB_B4 = EB_W4 + EB_E2 * EB_C1, EB_W5 = EB_B4 + EB_C1, EB_B5 = EB_W5 + EB_C1 * EB_C2, EB_X = EB_B5 + EB_C2,
              EB_E = EB_X + eb_r4(EB_WP * EB_PX), EB_D = EB_E + EB_WP * EB_PE, EB_END = EB_D + EB_E2 * EB_NP;
constexpr size_t EA_SMEM = sizeof(float) * EA_END, EB_SMEM = sizeof(float) * EB_END;
static_assert(EA_W1 % 4 == 0 && EA_WD % 4 == 0 && EA_W2 % 4 == 0 && EA_E % 4 == 0 && EA_D % 4 == 0, "16-byte rows");
static_assert(EB_WD % 4 == 0 && EB_W4 % 4 == 0 && EB_W5 % 4 == 0 && EB_E % 4 == 0 && EB_D % 4 == 0, "16-byte rows");
static_assert(EB_C1 * EB_NP <= EB_WP * EB_PE, "t48 of the tile reuses the expanded tensor's buffer");

BSB_D void eb_copy(float* dst, const float* src, int n) {            // n % 4 == 0, src 16-byte aligned
  for (int i = threadIdx.x * 4; i < n; i += 256 * 4) *reinterpret_cast<float4*>(dst + i) = __ldg(reinterpret_cast<const float4*>(src + i));
}
BSB_D void eb_bias(float* dst, const float* src, int n) {
  for (int i = threadIdx.x; i < n; i += 256) dst[i] = src ? __ldg(src + i) : 0.f;
}
BSB_D void fma4s(float4& acc, float v, const float4& w) {
  acc.x = fmaf(v, w.x, acc.x); acc.y = fmaf(v, w.y, acc.y); acc.z = fmaf(v, w.z, acc.z); acc.w = fmaf(v, w.w, acc.w);
}
template <int ACT> BSB_D float4 bias_act4(const float4& u, const float* b) {
  return make_float4(bsb_act(u.x + b[0], ACT), bsb_act(u.y + b[1], ACT), bsb_act(u.z + b[2], ACT), bsb_act(u.w + b[3], ACT));
}
// act(x . W + b) for N consecutive columns of W ([K][ldw] in shared memory) from x (K values in shared memory)
template <int K, int N, int ACT>
BSB_D void eb_expand(const float* x, const float* w, int ldw, const float* b, float* out) {
  float4 u[N / 4];
#pragma unroll
  for (int q = 0; q < N / 4; ++q) u[q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float v = x[k];
#pragma unroll
    for (int q = 0; q < N / 4; ++q) fma4s(u[q], v, *reinterpret_cast<const float4*>(w + k * ldw + 4 * q));
  }
#pragma unroll
  for (int q = 0; q < N / 4; ++q) *reinterpret_cast<float4*>(out + 4 * q) = bias_act4<ACT>(u[q], b + 4 * q);
}
// depthwise result of 4 channels of one tile pixel into the channel-major buffer d[c][EB_NP]
template <int ACT> BSB_D void eb_store_dw(float* d, int pp, const float4& u, const float* b) {
  const float4 r = bias_act4<ACT>(u, b);
  d[pp] = r.x; d[EB_NP + pp] = r.y; d[2 * EB_NP + pp] = r.z; d[3 * EB_NP + pp] = r.w;
}
// acc[j] += d[k][p] * w[k][j], k ascending, for 6 output channels (w: row stride EB_C1, 8-byte aligned)
template <int K> BSB_D void eb_project6(const float* d, int p, const float* w, float* acc) {
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float v = d[k * EB_NP + p];
    const float2 w0 = *reinterpret_cast<const float2*>(w + k * EB_C1), w1 = *reinterpret_cast<const float2*>(w + k * EB_C1 + 2),
                 w2 = *reinterpret_cast<const float2*>(w + k * EB_C1 + 4);
    acc[0] = fmaf(v, w0.x, acc[0]); acc[1] = fmaf(v, w0.y, acc[1]); acc[2] = fmaf(v, w1.x, acc[2]);
    acc[3] = fmaf(v, w1.y, acc[3]); acc[4] = fmaf(v, w2.x, acc[4]); acc[5] = fmaf(v, w2.y, acc[5]);
  }
}

template <int ACT>
__global__ void __launch_bounds__(256, 2) k_enc_block_s2(EncBlocksArgs a) {
  BSB_DYN_SMEM(smem_raw);
  float* sm = reinterpret_cast<float*>(smem_raw);
  float* s25 = sm + EA_T25; float* se = sm + EA_E; float* sd = sm + EA_D;
  const int tid = threadIdx.x;
  const int ox0 = blockIdx.x * EB_TW, oy0 = blockIdx.y * EB_TH, b = blockIdx.z;
  const int ix0 = 2 * ox0 - a.pl_a, iy0 = 2 * oy0 - a.pt_a;          // input pixel of the window's origin
  eb_copy(sm + EA_W0, a.w[0], EB_C0 * EB_C0); eb_copy(sm + EA_W1, a.w[1], EB_C0 * EB_E1);
  eb_copy(sm + EA_WD, a.wd[0], 9 * EB_E1); eb_copy(sm + EA_W2, a.w[2], EB_E1 * EB_C1);
  eb_bias(sm + EA_B0, a.b[0], EB_C0); eb_bias(sm + EA_B1, a.b[1], EB_E1); eb_bias(sm + EA_BD, a.bd[0], EB_E1); eb_bias(sm + EA_B2, a.b[2], EB_C1);
  if (tid < EB_C0) sm[EA_SV + tid] = __ldg(a.sv + (size_t)b * EB_C0 + tid);
  __syncthreads();
  // ---- t25 on the window.  This tile writes the t25 rows [2 TH by, 2 TH (by + 1)) and columns [2 TW bx, 2 TW (bx + 1))
  // (the last tile row / column: up to the image edge); with SAME padding (pt, pl <= 1, oh = ceil(ih / 2)) they lie in
  // its window ----
  const int r0 = 2 * oy0, r1 = blockIdx.y + 1 == gridDim.y ? a.ih : 2 * (oy0 + EB_TH);
  const int q0 = 2 * ox0, q1 = blockIdx.x + 1 == gridDim.x ? a.iw : 2 * (ox0 + EB_TW);
  const float* xb = a.x + (size_t)b * a.ih * a.iw * a.ld_x;
  float* t25b = a.t25 + (size_t)b * a.ih * a.iw * a.ld25;
  for (int i = tid; i < EA_WP; i += 256) {
    const int sy = i / EA_WW, sx = i - sy * EA_WW;
    const int gy = iy0 + sy, gx = ix0 + sx;
    if (gy < 0 || gy >= a.ih || gx < 0 || gx >= a.iw) continue;          // never read: the depthwise skips out-of-image taps
    const size_t pix = (size_t)gy * a.iw + gx;
    float xv[EB_C0];
#pragma unroll
    for (int k = 0; k < EB_C0 / 4; ++k) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(xb + pix * a.ld_x + 4 * k));
      xv[4 * k] = t.x * sm[EA_SV + 4 * k]; xv[4 * k + 1] = t.y * sm[EA_SV + 4 * k + 1];
      xv[4 * k + 2] = t.z * sm[EA_SV + 4 * k + 2]; xv[4 * k + 3] = t.w * sm[EA_SV + 4 * k + 3];
    }
    float4 acc[EB_C0 / 4];
#pragma unroll
    for (int q = 0; q < EB_C0 / 4; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < EB_C0; ++k)
#pragma unroll
      for (int q = 0; q < EB_C0 / 4; ++q) fma4s(acc[q], xv[k], *reinterpret_cast<const float4*>(sm + EA_W0 + k * EB_C0 + 4 * q));
    const bool own = gy >= r0 && gy < r1 && gx >= q0 && gx < q1;
    float* tp = s25 + i * EA_P25;
#pragma unroll
    for (int q = 0; q < EB_C0 / 4; ++q) {
      const float4 r = bias_act4<ACT_NONE>(acc[q], sm + EA_B0 + 4 * q);
      tp[4 * q] = r.x; tp[4 * q + 1] = r.y; tp[4 * q + 2] = r.z; tp[4 * q + 3] = r.w;
      if (own) *reinterpret_cast<float4*>(t25b + pix * a.ld25 + 4 * q) = r;
    }
  }
  __syncthreads();
  const int g = tid / EB_NP, p = tid % EB_NP;                         // project: tile pixel p, output channels 6g .. 6g + 5
  const int py = oy0 + p / EB_TW, px = ox0 + p % EB_TW;
  const bool p_ok = py < a.oh && px < a.ow;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int s0 = 0; s0 < EB_E1; s0 += EA_S) {
    // ---- expand: channels s0 .. s0 + 23 on the window, 12 per item ----
    for (int it = tid; it < EA_WP * (EA_S / EA_Q); it += 256) {
      const int q = it / EA_WP, i = it - q * EA_WP;
      const int sy = i / EA_WW, sx = i - sy * EA_WW;
      const int gy = iy0 + sy, gx = ix0 + sx;
      if (gy < 0 || gy >= a.ih || gx < 0 || gx >= a.iw) continue;
      eb_expand<EB_C0, EA_Q, ACT>(s25 + i * EA_P25, sm + EA_W1 + s0 + EA_Q * q, EB_E1, sm + EA_B1 + s0 + EA_Q * q, se + i * EA_PE + EA_Q * q);
    }
    __syncthreads();
    // ---- depthwise 3x3 stride 2 on the tile, 4 channels per item ----
    for (int it = tid; it < EB_NP * (EA_S / 4); it += 256) {
      const int q = it / EB_NP, pp = it - q * EB_NP;
      const int ly = pp / EB_TW, lx = pp % EB_TW;
      const int oy = oy0 + ly, ox = ox0 + lx;
      if (oy >= a.oh || ox >= a.ow) continue;
      float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int fy = 0; fy < 3; ++fy) {
        const int iy = 2 * oy - a.pt_a + fy;
        if (iy < 0 || iy >= a.ih) continue;
#pragma unroll
        for (int fx = 0; fx < 3; ++fx) {
          const int ix = 2 * ox - a.pl_a + fx;
          if (ix < 0 || ix >= a.iw) continue;
          fma4(u, *reinterpret_cast<const float4*>(se + ((2 * ly + fy) * EA_WW + 2 * lx + fx) * EA_PE + 4 * q),
               *reinterpret_cast<const float4*>(sm + EA_WD + (fy * 3 + fx) * EB_E1 + s0 + 4 * q));
        }
      }
      eb_store_dw<ACT>(sd + 4 * q * EB_NP, pp, u, sm + EA_BD + s0 + 4 * q);
    }
    __syncthreads();
    // ---- project: k ascending across the slices (the next slice's expand only writes the window buffer; the barrier
    // after it orders this read of sd before the next depthwise) ----
    if (p_ok) eb_project6<EA_S>(sd, p, sm + EA_W2 + s0 * EB_C1 + 6 * g, acc);
  }
  if (!p_ok) return;
  float* op = a.t36 + (((size_t)b * a.oh + py) * a.ow + px) * a.ld36 + 6 * g;
#pragma unroll
  for (int j = 0; j < 6; j += 2)
    *reinterpret_cast<float2*>(op + j) = make_float2(acc[j] + sm[EA_B2 + 6 * g + j], acc[j + 1] + sm[EA_B2 + 6 * g + j + 1]);
}

template <int ACT>
__global__ void __launch_bounds__(256, 2) k_enc_block_res(EncBlocksArgs a) {
  BSB_DYN_SMEM(smem_raw);
  float* sm = reinterpret_cast<float*>(smem_raw);
  float* sx = sm + EB_X; float* se = sm + EB_E; float* sd = sm + EB_D;
  float* s48 = se;                                                   // the tile's t48 [24][64], once the expanded tensor is consumed
  const int tid = threadIdx.x;
  const int h = a.oh, w = a.ow;
  const int ox0 = blockIdx.x * EB_TW, oy0 = blockIdx.y * EB_TH, b = blockIdx.z;
  const int ix0 = ox0 - 1, iy0 = oy0 - 1;                            // SAME 3x3: one pixel of halo
  eb_copy(sm + EB_W3, a.w[3], EB_C1 * EB_E2); eb_copy(sm + EB_WD, a.wd[1], 9 * EB_E2);
  eb_copy(sm + EB_W4, a.w[4], EB_E2 * EB_C1); eb_copy(sm + EB_W5, a.w[5], EB_C1 * EB_C2);
  eb_bias(sm + EB_B3, a.b[3], EB_E2); eb_bias(sm + EB_BD, a.bd[1], EB_E2); eb_bias(sm + EB_B4, a.b[4], EB_C1); eb_bias(sm + EB_B5, a.b[5], EB_C2);
  const float* xb = a.t36 + (size_t)b * h * w * a.ld36;
  for (int it = tid; it < EB_WP * (EB_C1 / 4); it += 256) {
    const int i = it / (EB_C1 / 4), q = it - i * (EB_C1 / 4);
    const int gy = iy0 + i / EB_WW, gx = ix0 + i % EB_WW;
    if (gy < 0 || gy >= h || gx < 0 || gx >= w) continue;
    const float4 v = __ldg(reinterpret_cast<const float4*>(xb + ((size_t)gy * w + gx) * a.ld36 + 4 * q));
    float* xp = sx + i * EB_PX + 4 * q;
    xp[0] = v.x; xp[1] = v.y; xp[2] = v.z; xp[3] = v.w;
  }
  __syncthreads();
  // ---- expand 24 -> 88 on the window, 8 channels per item ----
  for (int it = tid; it < EB_WP * (EB_E2 / EB_Q); it += 256) {
    const int q = it / EB_WP, i = it - q * EB_WP;
    const int gy = iy0 + i / EB_WW, gx = ix0 + i % EB_WW;
    if (gy < 0 || gy >= h || gx < 0 || gx >= w) continue;
    eb_expand<EB_C1, EB_Q, ACT>(sx + i * EB_PX, sm + EB_W3 + EB_Q * q, EB_E2, sm + EB_B3 + EB_Q * q, se + i * EB_PE + EB_Q * q);
  }
  __syncthreads();
  // ---- depthwise 3x3 stride 1 on the tile, 4 channels per item ----
  for (int it = tid; it < EB_NP * (EB_E2 / 4); it += 256) {
    const int q = it / EB_NP, pp = it - q * EB_NP;
    const int ly = pp / EB_TW, lx = pp % EB_TW;
    const int oy = oy0 + ly, ox = ox0 + lx;
    if (oy >= h || ox >= w) continue;
    float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int fy = 0; fy < 3; ++fy) {
      const int iy = oy - 1 + fy;
      if (iy < 0 || iy >= h) continue;
#pragma unroll
      for (int fx = 0; fx < 3; ++fx) {
        const int ix = ox - 1 + fx;
        if (ix < 0 || ix >= w) continue;
        fma4(u, *reinterpret_cast<const float4*>(se + ((ly + fy) * EB_WW + lx + fx) * EB_PE + 4 * q),
             *reinterpret_cast<const float4*>(sm + EB_WD + (fy * 3 + fx) * EB_E2 + 4 * q));
      }
    }
    eb_store_dw<ACT>(sd + 4 * q * EB_NP, pp, u, sm + EB_BD + 4 * q);
  }
  __syncthreads();
  // ---- project 88 -> 24 + t36 = t48 ----
  const int g = tid / EB_NP, p = tid % EB_NP;
  const int ly = p / EB_TW, lx = p % EB_TW;
  const int py = oy0 + ly, px = ox0 + lx;
  const bool p_ok = py < h && px < w;
  const size_t pix = ((size_t)b * h + py) * w + px;
  if (p_ok) {
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    eb_project6<EB_E2>(sd, p, sm + EB_W4 + 6 * g, acc);
    const float* res = sx + ((ly + 1) * EB_WW + lx + 1) * EB_PX + 6 * g;
    float r[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      r[j] = (acc[j] + sm[EB_B4 + 6 * g + j]) + res[j];
      s48[(6 * g + j) * EB_NP + p] = r[j];
    }
    float* op = a.t48 + pix * a.ld48 + 6 * g;
#pragma unroll
    for (int j = 0; j < 6; j += 2) *reinterpret_cast<float2*>(op + j) = make_float2(r[j], r[j + 1]);
  }
  __syncthreads();
  // ---- t52 = hswish(t48 . W5 + b5): channels 24g .. 24g + 23 ----
  if (!p_ok) return;
  float4 u[6];
#pragma unroll
  for (int q = 0; q < 6; ++q) u[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* wp = sm + EB_W5 + 24 * g;
#pragma unroll 4
  for (int k = 0; k < EB_C1; ++k) {
    const float v = s48[k * EB_NP + p];
#pragma unroll
    for (int q = 0; q < 6; ++q) fma4s(u[q], v, *reinterpret_cast<const float4*>(wp + k * EB_C2 + 4 * q));
  }
  float* op = a.t52 + pix * a.ld52 + 24 * g;
#pragma unroll
  for (int q = 0; q < 6; ++q) *reinterpret_cast<float4*>(op + 4 * q) = bias_act4<ACT_HARD_SWISH>(u[q], sm + EB_B5 + 24 * g + 4 * q);
}

bool enc_blocks_supported(int device, int c_in, int c_25, int c_e1, int c_36, int c_e2, int c_52, int ld_x, int ld25, int ld36, int ld48, int ld52) {
  if (c_in != EB_C0 || c_25 != EB_C0 || c_e1 != EB_E1 || c_36 != EB_C1 || c_e2 != EB_E2 || c_52 != EB_C2) return false;
  if (ld_x % 4 || ld25 % 4 || ld36 % 4 || ld48 % 4 || ld52 % 4) return false;
#ifdef BSB_EMU
  (void)device;
#else
  int optin = 0;
  if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) { cudaGetLastError(); return false; }
  if ((size_t)optin < std::max(EA_SMEM, EB_SMEM)) return false;
#endif
  return true;
}

// dynamic shared memory and, for two co-resident CTAs, the whole unified L1 / shared array as shared memory
static void enc_prepare(const void* k, size_t smem) {
  ensure_dyn_smem(k, smem);
#ifndef BSB_EMU
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, bool> done;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return; }
  std::lock_guard<std::mutex> lock(mu);
  if (done[std::make_pair(dev, k)]) return;
  if (cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess) cudaGetLastError();
  done[std::make_pair(dev, k)] = true;
#endif
}

template <int ACT>
static void launch_enc_blocks_t(cudaStream_t s, dim3 grid, const EncBlocksArgs& a, bool block_b) {
  if (!block_b) {
    auto k = k_enc_block_s2<ACT>;
    enc_prepare(reinterpret_cast<const void*>(k), EA_SMEM);
    BSB_LAUNCH(k, grid, dim3(256), EA_SMEM, s, a);
  } else {
    auto k = k_enc_block_res<ACT>;
    enc_prepare(reinterpret_cast<const void*>(k), EB_SMEM);
    BSB_LAUNCH(k, grid, dim3(256), EB_SMEM, s, a);
  }
}

void launch_enc_blocks(cudaStream_t s, int B, const EncBlocksArgs& a, bool block_b) {
  const dim3 grid((unsigned)ceil_div(a.ow, EB_TW), (unsigned)ceil_div(a.oh, EB_TH), (unsigned)B);
  if (a.act == ACT_RELU) launch_enc_blocks_t<ACT_RELU>(s, grid, a, block_b);
  else launch_enc_blocks_t<ACT_RELU6>(s, grid, a, block_b);
  count_launch();
}

// ---------------------------------------------------------------------------
// Convolution2DTransposeBias, k = 2x2, stride 2, SAME (even output): no overlap, so
// out[2y+fy][2x+fx][o] = bias[o] + sum_ic in[y][x][ic] * w[o][fy][fx][ic], ic ascending
// (the order in which lib/transpose_conv_bias.cc:80-108 scatters into one output).
// One thread = one output pixel; weights in shared memory.
// ---------------------------------------------------------------------------
// One thread = one INPUT pixel: its ic values are loaded once (float4) and produce the 2x2 x oc
// outputs it alone determines.
__global__ void __launch_bounds__(128) k_tconv2x2(const float* in, int B, int ih, int iw, int ic, int ld_in,
                                                  const float* w, const float* bias, int oc,
                                                  float* out, int oh, int ow, int ld_out, int act2) {
  BSB_DYN_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);    // [oc][2][2][ic]
  for (int i = threadIdx.x; i < oc * 4 * ic; i += blockDim.x) ws[i] = __ldg(w + i);
  __syncthreads();
  const long total = (long)B * ih * iw;
  const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const int ix = (int)(pix % iw), iy = (int)((pix / iw) % ih), b = (int)(pix / ((long)iw * ih));
  const float* ip = in + (size_t)pix * ld_in;
  const bool vec = (ic % 4 == 0) && (ld_in % 4 == 0);
  if (vec && ic == 16 && oc <= 2 && ld_out == oc && (ow & 1) == 0) {
    // the MLKit / Meet heads: 16 inputs held in registers, each output row (2 pixels x oc) leaves as one vector store
    float v[16];
#pragma unroll
    for (int c = 0; c < 16; c += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(ip + c));
      v[c] = t.x; v[c + 1] = t.y; v[c + 2] = t.z; v[c + 3] = t.w;
    }
#pragma unroll
    for (int fy = 0; fy < 2; ++fy) {
      float r[2][2];                      // [fx][o]
#pragma unroll
      for (int fx = 0; fx < 2; ++fx)
#pragma unroll
        for (int o = 0; o < 2; ++o) {
          r[fx][o] = 0.f;
          if (o >= oc) continue;
          const float* wp = ws + ((o * 2 + fy) * 2 + fx) * 16;
          float acc = __ldg(bias + o);
#pragma unroll
          for (int c = 0; c < 16; ++c) acc = fmaf(v[c], wp[c], acc);
          r[fx][o] = bsb_act(acc, act2);
        }
      float* op = out + (((size_t)b * oh + 2 * iy + fy) * ow + 2 * ix) * oc;
      if (oc == 2) *reinterpret_cast<float4*>(op) = make_float4(r[0][0], r[0][1], r[1][0], r[1][1]);
      else *reinterpret_cast<float2*>(op) = make_float2(r[0][0], r[1][0]);
    }
    return;
  }
  for (int fy = 0; fy < 2; ++fy)
    for (int fx = 0; fx < 2; ++fx) {
      float* op = out + (((size_t)b * oh + 2 * iy + fy) * ow + 2 * ix + fx) * ld_out;
      for (int o = 0; o < oc; ++o) {
        const float* wp = ws + ((o * 2 + fy) * 2 + fx) * ic;
        float acc = __ldg(bias + o);
        if (vec) {
          for (int c = 0; c < ic; c += 4) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(ip + c));
            acc = fmaf(v.x, wp[c], acc); acc = fmaf(v.y, wp[c + 1], acc); acc = fmaf(v.z, wp[c + 2], acc); acc = fmaf(v.w, wp[c + 3], acc);
          }
        } else {
          for (int c = 0; c < ic; ++c) acc = fmaf(__ldg(ip + c), wp[c], acc);
        }
        op[o] = bsb_act(acc, act2);
      }
    }
}

void launch_tconv2x2(cudaStream_t s, int B, const float* in, int ih, int iw, int ic, int ld_in,
                     const float* w, const float* bias, int oc, float* out, int oh, int ow, int ld_out, int act2) {
  const long total = (long)B * ih * iw;
  BSB_LAUNCH(k_tconv2x2, dim3((unsigned)((total + 127) / 128)), dim3(128), sizeof(float) * (size_t)oc * 4 * ic, s,
             in, B, ih, iw, ic, ld_in, w, bias, oc, out, oh, ow, ld_out, act2);
  count_launch();
}

// ---------------------------------------------------------------------------
// Element-wise (only what the planner could not fold into a producer/consumer).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_eltwise(int mode, long rows, int hw, int c, const float* a, int ld_a,
                                                 const float* b, int ld_b, const float* scale,
                                                 float* out, int ld_out, int act) {
  const long total = rows * c;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = (int)(idx % c);
  const long row = idx / c;
  const float av = __ldg(a + (size_t)row * ld_a + ch);
  float v;
  switch (mode) {
    case 0: v = av; break;
    case 1: v = av + __ldg(b + (size_t)row * ld_b + ch); break;
    case 2: v = av * __ldg(b + (size_t)row * ld_b + ch); break;
    case 3: v = av * __ldg(scale + (size_t)(row / hw) * c + ch); break;
    default: v = av * __ldg(scale + (size_t)(row / hw) * c + ch); v = v + __ldg(b + (size_t)row * ld_b + ch); break;
  }
  out[(size_t)row * ld_out + ch] = bsb_act(v, act);
}

void launch_eltwise(cudaStream_t s, int mode, int B, int hw, int c, const float* a, int ld_a,
                    const float* b, int ld_b, const float* scale, float* out, int ld_out, int act) {
  const long rows = (long)B * hw;
  const long total = rows * c;
  BSB_LAUNCH(k_eltwise, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, mode, rows, hw, c, a, ld_a, b, ld_b, scale, out, ld_out, act);
  count_launch();
}

__global__ void __launch_bounds__(256) k_copy_channels(long rows, int c, const float* in, int ld_in, float* out, int ld_out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * c) return;
  const int ch = (int)(idx % c);
  const long row = idx / c;
  out[(size_t)row * ld_out + ch] = __ldg(in + (size_t)row * ld_in + ch);
}

void launch_copy_channels(cudaStream_t s, int rows, int c, const float* in, int ld_in, float* out, int ld_out) {
  const long total = (long)rows * c;
  BSB_LAUNCH(k_copy_channels, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, (long)rows, c, in, ld_in, out, ld_out);
  count_launch();
}

}  // namespace bsb
