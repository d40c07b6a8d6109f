// backscrub_b200/csrc/kernels_app.cu — the optional per-frame stages of the reference's main loop
// that sit either side of alpha_blend (app/deepseg.cc:649-679):
//   * `-p bgblur:k`  cv::GaussianBlur(bg, bg, Size(k,k), 0)            (:657-658)
//   * `-H` / `-V`    cv::flip(raw, raw, 1 / 0 / -1)                     (:667-673)
//   * virtual-camera geometry  cv::resize(raw, raw, vidGeo)             (:677-679) — k_resize_u8c3 (kernels_img.cu)
// Integer arithmetic is OpenCV's bit-exact 8-bit path restated (oracle/oracle_img.c pins it on cv2).
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "post_math.h"

namespace bsb {

void count_launch();

// ---------------------------------------------------------------------------
// Gaussian blur, 8UC3, BORDER_REFLECT_101, OpenCV fixed point: taps q (8.8, sum 256);
//   rows: h = sum_j q[j]*src[x+j-r]   (<= 255*256, 16 bit)     cols: (sum_j q[j]*h[y+j-r] + 32768) >> 16
// Both sums are exact integers, so tap order is free.
//
// Every kernel blurs frame b with strength ks[b] when given a per-frame strength table (sources calls; 0 = the frame is
// not blurred), else every frame with k_all.  Strengths 3..31 run the fused tile kernel, 1 and 33..255 the row /
// column pair (the two launch classes); a CTA whose frame belongs to the other class, or has strength 0, exits at
// once.  The taps of every odd strength are pre-computed once per device (GaussTables), so a captured launch stays
// valid whatever strengths its frames get.  The kernels read BGR frames; a sources call whose post kernel reads the
// camera YUYV / NV12 in place first converts only its camera-blur frames (k_gauss_stage_bgr): converting each pixel
// once there is cheaper than converting every pixel of every overlapping halo patch inside the Gaussian.
// ---------------------------------------------------------------------------
constexpr int GF_TW = 64, GF_TH = 32, GF_MAXR = 15, GF_RM = GF_TH + 2 * GF_MAXR, GF_PW = 100, GF_HR = 66;
constexpr int GF_NW = 9, GF_NV = 16, GF_NK = GF_MAXR;    // fused strengths 3, 5, .., 31

struct GaussFast { int k, nw, nv; unsigned hq[4][GF_NW]; unsigned cw[GF_NV]; };
struct GaussTables { GaussFast fast[GF_NK]; GaussTaps taps[128]; };   // fast[(k - 3) / 2], taps[(k - 1) / 2]

// The camera frames of a sources call's camera-blur frames (ks[b] != 0) as tightly packed BGR, for the Gaussian:
// cv::cvtColor(COLOR_YUV2BGR_YUYV / _NV12), the arithmetic of yuyv_px_to_bgr / nv12_px_to_bgr.  One thread = one pixel
// pair (W even).
__global__ void __launch_bounds__(256) k_gauss_stage_bgr(GaussSrc src, uint8_t* bgr, int W, int H, const int* ks) {
  const int b = blockIdx.y;
  if (!ks[b]) return;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = W / 2;
  if (idx >= (long)hw * H) return;
  const int x = (int)(idx % hw) * 2, y = (int)(idx / hw);
  const uint8_t* img = src.p + (size_t)b * src.stride;
  int p0[3], p1[3];
  if (src.fmt == IN_YUYV) {
    const uint8_t* q = img + (size_t)y * src.pitch + (size_t)x * 2;
    yuv_px_to_bgr(q[0], q[1], q[3], p0); yuv_px_to_bgr(q[2], q[1], q[3], p1);
  } else {
    const uint8_t* yr = img + (size_t)y * src.pitch + x;
    const uint8_t* uv = img + src.uv + (size_t)(y >> 1) * src.pitch + x;
    yuv_px_to_bgr(yr[0], uv[0], uv[1], p0); yuv_px_to_bgr(yr[1], uv[0], uv[1], p1);
  }
  uint8_t* o = bgr + (size_t)b * ((size_t)W * H * 3) + ((size_t)y * W + x) * 3;
  o[0] = (uint8_t)p0[0]; o[1] = (uint8_t)p0[1]; o[2] = (uint8_t)p0[2]; o[3] = (uint8_t)p1[0]; o[4] = (uint8_t)p1[1]; o[5] = (uint8_t)p1[2];
}

// Row pass: one block = 256 pixels of one row; the reflected source span is staged in shared
// memory once, every thread then produces three byte lanes.
constexpr int GAUSS_TW = 256;

__global__ void __launch_bounds__(256) k_gauss_rows(const uint8_t* src, size_t pitch, size_t frame_stride, uint16_t* tmp, int W, int H,
                                                    const GaussTables* T, int k_all, const int* ks) {
  __shared__ uint8_t s[(GAUSS_TW + 2 * 127) * 3 + 2];
  __shared__ uint16_t q[256];
  const int x0 = blockIdx.x * GAUSS_TW, y = blockIdx.y, b = blockIdx.z;
  const int k = ks ? ks[b] : k_all;
  if (gauss_class(k) != GAUSS_SEPARABLE) return;
  const int r = k >> 1;
  const int tw = min(GAUSS_TW, W - x0);
  const uint8_t* row = src + (size_t)b * frame_stride + (size_t)y * pitch;
  for (int j = threadIdx.x; j < k; j += blockDim.x) q[j] = T->taps[(k - 1) >> 1].q[j];
  const int span = tw + 2 * r;
  for (int i = threadIdx.x; i < span; i += blockDim.x) {
    const int sx = bsb_reflect101(x0 + i - r, W);
    s[3 * i] = row[3 * sx]; s[3 * i + 1] = row[3 * sx + 1]; s[3 * i + 2] = row[3 * sx + 2];
  }
  __syncthreads();
  uint16_t* d = tmp + ((size_t)b * H + y) * (size_t)W * 3 + (size_t)x0 * 3;
  for (int l = threadIdx.x; l < tw * 3; l += blockDim.x) {
    unsigned acc = 0;
    for (int j = 0; j < k; ++j) acc += (unsigned)q[j] * s[l + 3 * j];
    d[l] = (uint16_t)acc;
  }
}

// Column pass: one block = 128 byte lanes x 32 rows; the (32 + 2r) reflected rows of 16-bit row sums
// are staged in dynamic shared memory (sized by the launcher for the largest strength of the call's class).
constexpr int GAUSS_CL = 128, GAUSS_CH = 32;

__global__ void __launch_bounds__(256) k_gauss_cols(const uint16_t* tmp, uint8_t* dst, size_t pitch, size_t frame_stride,
                                                    int W, int H, const GaussTables* T, int k_all, const int* ks) {
  BSB_DYN_SMEM(smem_raw);
  __shared__ uint16_t q[256];
  uint16_t* sm = reinterpret_cast<uint16_t*>(smem_raw);
  const int b = blockIdx.z;
  const int k = ks ? ks[b] : k_all;
  if (gauss_class(k) != GAUSS_SEPARABLE) return;
  const int r = k >> 1, lanes = W * 3;
  const int l0 = blockIdx.x * GAUSS_CL, y0 = blockIdx.y * GAUSS_CH;
  const int nl = min(GAUSS_CL, lanes - l0), nr = min(GAUSS_CH, H - y0);
  const uint16_t* t = tmp + (size_t)b * H * lanes;
  for (int j = threadIdx.x; j < k; j += blockDim.x) q[j] = T->taps[(k - 1) >> 1].q[j];
  const int rows = nr + 2 * r;
  for (int i = threadIdx.x; i < rows * GAUSS_CL; i += blockDim.x) {
    const int rr = i / GAUSS_CL, l = i % GAUSS_CL;
    if (l < nl) sm[i] = t[(size_t)bsb_reflect101(y0 + rr - r, H) * lanes + l0 + l];
  }
  __syncthreads();
  const int l = threadIdx.x % GAUSS_CL;
  if (l >= nl) return;
  for (int yy = threadIdx.x / GAUSS_CL; yy < nr; yy += 256 / GAUSS_CL) {
    unsigned acc = 32768u;
    for (int j = 0; j < k; ++j) acc += (unsigned)q[j] * sm[(yy + j) * GAUSS_CL + l];
    dst[(size_t)b * frame_stride + (size_t)(y0 + yy) * pitch + l0 + l] = (uint8_t)(acc >> 16);
  }
}

// ---------------------------------------------------------------------------
// Fused tile kernel for 3 <= k <= 31 (the default strength is 25): one block = 64 x 32 output pixels.
//   A  the reflected (32+2r) x (64+2r) source patch is staged de-interleaved (one byte plane per channel),
//   B  row sums with DP4A: a thread owns 4 adjacent outputs of one plane row; it reads aligned 32-bit words
//      and the taps come pre-shifted per output (hq[i][g], byte b = q[4g+b-i]) so no byte realignment is needed;
//      the 16-bit sums are stored transposed (row index fastest) so that
//   C  column sums run on DP2A: a thread owns two vertically adjacent outputs and reads (row, row+1) pairs as
//      words; cw[g] packs the tap pairs of both outputs (low half: q[2g],q[2g+1]; high half: q[2g-1],q[2g]),
//   D  the re-interleaved tile goes out in 16-byte stores.
// All sums are exact integers (<= 255*256*256 < 2^24), so the regrouping is bit-neutral.
// ---------------------------------------------------------------------------

// B and C.  NWC / NVC > 0: tap-word counts fixed at compile time (the default strength 25 -> 7 / 13), so the
// dot-product chains are straight-line code; 0: run-time loops for the other strengths.
template <int NWC, int NVC>
BSB_D void gauss_fused_bc(uint8_t* P, uint16_t* Ht, const GaussFast& g, int rows, int tid) {
  const int warp = tid >> 5, lane = tid & 31;
  // ---- B: row sums (DP4A), stored transposed ----
  const int nw = NWC > 0 ? NWC : g.nw, nv = NVC > 0 ? NVC : g.nv;
  for (int cm = warp; cm < 3 * (GF_TW / 4); cm += 8) {          // one (plane, 4-pixel group) per warp, lanes walk the rows
    const int c = cm / (GF_TW / 4), m = cm % (GF_TW / 4);
    for (int row = lane; row < rows; row += 32) {
      const unsigned* pw = reinterpret_cast<const unsigned*>(P + (c * GF_RM + row) * GF_PW + 4 * m);
      unsigned a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      if constexpr (NWC > 0) {
#pragma unroll
        for (int q = 0; q < NWC; ++q) {
          const unsigned w = pw[q];
          a0 = __dp4a(w, g.hq[0][q], a0); a1 = __dp4a(w, g.hq[1][q], a1);
          a2 = __dp4a(w, g.hq[2][q], a2); a3 = __dp4a(w, g.hq[3][q], a3);
        }
      } else {
#pragma unroll 1
        for (int q = 0; q < nw; ++q) {
          const unsigned w = pw[q];
          a0 = __dp4a(w, g.hq[0][q], a0); a1 = __dp4a(w, g.hq[1][q], a1);
          a2 = __dp4a(w, g.hq[2][q], a2); a3 = __dp4a(w, g.hq[3][q], a3);
        }
      }
      uint16_t* hp = Ht + (c * GF_TW + 4 * m) * GF_HR + row;
      hp[0] = (uint16_t)a0; hp[GF_HR] = (uint16_t)a1; hp[2 * GF_HR] = (uint16_t)a2; hp[3 * GF_HR] = (uint16_t)a3;
    }
  }
  __syncthreads();

  // ---- C: column sums (DP2A), re-interleaved into the output tile ----
  uint8_t* O = P;                                               // [GF_TH][GF_TW * 3]
  for (int it = tid; it < 3 * (GF_TH / 2) * GF_TW; it += 256) {
    const int x = it % GF_TW, yp = (it / GF_TW) % (GF_TH / 2), c = it / (GF_TW * (GF_TH / 2));
    const unsigned* hw = reinterpret_cast<const unsigned*>(Ht + (c * GF_TW + x) * GF_HR + 2 * yp);
    unsigned a0 = 32768u, a1 = 32768u;
    if constexpr (NVC > 0) {
#pragma unroll
      for (int q = 0; q < NVC; ++q) {
        const unsigned w = hw[q];
        a0 = __dp2a_lo(w, g.cw[q], a0); a1 = __dp2a_hi(w, g.cw[q], a1);
      }
    } else {
#pragma unroll 1
      for (int q = 0; q < nv; ++q) {
        const unsigned w = hw[q];
        a0 = __dp2a_lo(w, g.cw[q], a0); a1 = __dp2a_hi(w, g.cw[q], a1);
      }
    }
    O[(2 * yp) * (GF_TW * 3) + x * 3 + c] = (uint8_t)(a0 >> 16);
    O[(2 * yp + 1) * (GF_TW * 3) + x * 3 + c] = (uint8_t)(a1 >> 16);
  }
}

// yuyv / nv12 (may be null; W even, NV12 also H even): [n] W*H*2 / W*H*3/2-byte frames that receive the blurred frame's
// YUYV / NV12, written from the output tile in stage D
__global__ void __launch_bounds__(256) k_gauss_fused(const uint8_t* src, size_t spitch, size_t sstride, uint8_t* dst, size_t dpitch,
                                                     size_t dstride, int W, int H, const GaussTables* T, GaussFast g25, int k_all,
                                                     const int* ks, int vec_ok, uint8_t* yuyv, uint8_t* nv12) {
  __shared__ __align__(16) uint8_t P[3 * GF_RM * GF_PW];      // planes; reused as the interleaved output tile in C/D
  __shared__ __align__(16) uint16_t Ht[3 * GF_TW * GF_HR];
  __shared__ GaussFast g;
  const int tid = threadIdx.x;
  const int x0 = blockIdx.x * GF_TW, y0 = blockIdx.y * GF_TH, b = blockIdx.z;
  const int k = ks ? ks[b] : k_all;
  if (gauss_class(k) != GAUSS_FUSED) return;
  if (k != 25 && tid < (int)(sizeof(GaussFast) / 4))            // the 25-tap body takes g25
    reinterpret_cast<unsigned*>(&g)[tid] = reinterpret_cast<const unsigned*>(&T->fast[(k - 3) >> 1])[tid];
  const int r = k >> 1;
  const int tw = min(GF_TW, W - x0), th = min(GF_TH, H - y0);
  const int rows = GF_TH + 2 * r, cols = GF_TW + 2 * r;
  const uint8_t* frame = src + (size_t)b * sstride;
  const int warp = tid >> 5, lane = tid & 31;

  // ---- A: stage + de-interleave (loads of three column groups and two rows are issued before any store: the
  //      patch comes from L2/HBM and the loop is latency bound unless several requests per thread are in flight)
  const bool interior = x0 - r >= 0 && x0 + GF_TW + r <= W && y0 - r >= 0 && y0 + GF_TH + r <= H;
  if (interior) {
    const uint8_t* base = frame + (size_t)(y0 - r) * spitch + (size_t)(x0 - r) * 3;
#pragma unroll 2
    for (int row = warp; row < rows; row += 8) {
      const uint8_t* srow = base + (size_t)row * spitch;
      uint8_t v[3][3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int col = lane + 32 * j;
        if (col < cols) { const uint8_t* sp = srow + col * 3; v[j][0] = sp[0]; v[j][1] = sp[1]; v[j][2] = sp[2]; }
      }
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int col = lane + 32 * j;
        if (col < cols) { uint8_t* pp = P + row * GF_PW + col; pp[0] = v[j][0]; pp[GF_RM * GF_PW] = v[j][1]; pp[2 * GF_RM * GF_PW] = v[j][2]; }
      }
    }
  } else {
    for (int row = warp; row < rows; row += 8) {
      const uint8_t* srow = frame + (size_t)bsb_reflect101(y0 + row - r, H) * spitch;
      for (int col = lane; col < cols; col += 32) {
        const uint8_t* sp = srow + (size_t)bsb_reflect101(x0 + col - r, W) * 3;
        uint8_t* pp = P + row * GF_PW + col;
        pp[0] = sp[0]; pp[GF_RM * GF_PW] = sp[1]; pp[2 * GF_RM * GF_PW] = sp[2];
      }
    }
  }
  __syncthreads();

  // ---- B, C: the unrolled 25-tap specialisation (its tap words are kernel parameters: operands of the dot products,
  //      no loads), or the run-time loops ----
  if (k == 25) gauss_fused_bc<7, 13>(P, Ht, g25, rows, tid);
  else gauss_fused_bc<0, 0>(P, Ht, g, rows, tid);
  __syncthreads();

  // ---- D: write out, and the tile's YUYV / NV12 from the same shared tile ----
  const uint8_t* O = P;
  uint8_t* out = dst + (size_t)b * dstride + (size_t)y0 * dpitch + (size_t)x0 * 3;
  if (vec_ok && tw == GF_TW) {
    for (int i = tid; i < th * (GF_TW * 3 / 16); i += 256) {
      const int row = i / (GF_TW * 3 / 16), v = i % (GF_TW * 3 / 16);
      *reinterpret_cast<uint4*>(out + (size_t)row * dpitch + 16 * v) = *reinterpret_cast<const uint4*>(O + row * (GF_TW * 3) + 16 * v);
    }
  } else {
    for (int i = tid; i < th * tw * 3; i += 256) {
      const int row = i / (tw * 3), l = i - row * (tw * 3);
      out[(size_t)row * dpitch + l] = O[row * (GF_TW * 3) + l];
    }
  }
  const int np = tw / 2;                                        // pixel pairs per tile row (x0 and W are even)
  const size_t npix = (size_t)W * H;
  if (nv12) {                                                   // tile rows start even, th is even (H even)
    uint8_t* f = nv12 + (size_t)b * (npix * 3 / 2);
    for (int i = tid; i < (th / 2) * np; i += 256) {
      const int rp = i / np, j = i - rp * np;
      const unsigned w0 = yuyv_pair_word(O + (2 * rp) * (GF_TW * 3) + 6 * j), w1 = yuyv_pair_word(O + (2 * rp + 1) * (GF_TW * 3) + 6 * j);
      const int y = y0 + 2 * rp, x = x0 + 2 * j;
      nv12_block(w0, w1, f + (size_t)y * W + x, W, f + npix + (size_t)(y >> 1) * W + x);
    }
  } else if (yuyv) {
    unsigned* f = reinterpret_cast<unsigned*>(yuyv + (size_t)b * npix * 2);
    for (int i = tid; i < th * np; i += 256) {
      const int row = i / np, j = i - row * np;
      f[((size_t)(y0 + row) * W + x0) / 2 + j] = yuyv_pair_word(O + row * (GF_TW * 3) + 6 * j);
    }
  }
}

// The same YUYV / NV12 for the frames of the row / column class (ks[b] in it), from the blurred BGR frames.  One
// thread = one pixel pair of two rows.
__global__ void __launch_bounds__(256) k_gauss_slot_yuv(const uint8_t* bgr, size_t bstride, uint8_t* yuyv, uint8_t* nv12, int W, int H,
                                                        const int* ks) {
  const int b = blockIdx.y;
  if (gauss_class(ks[b]) != GAUSS_SEPARABLE) return;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = W / 2;
  if (idx >= (long)hw * ((H + 1) / 2)) return;
  const int j = (int)(idx % hw), rp = (int)(idx / hw);
  const size_t npix = (size_t)W * H;
  const uint8_t* s0 = bgr + (size_t)b * bstride + ((size_t)(2 * rp) * W + 2 * j) * 3;
  const unsigned w0 = yuyv_pair_word(s0);
  if (nv12) {                                                   // H even (NV12 calls)
    const unsigned w1 = yuyv_pair_word(s0 + (size_t)W * 3);
    uint8_t* f = nv12 + (size_t)b * (npix * 3 / 2);
    nv12_block(w0, w1, f + (size_t)(2 * rp) * W + 2 * j, W, f + npix + (size_t)rp * W + 2 * j);
  } else if (yuyv) {
    unsigned* f = reinterpret_cast<unsigned*>(yuyv + (size_t)b * npix * 2);
    f[((size_t)(2 * rp) * W) / 2 + j] = w0;
    if (2 * rp + 1 < H) f[((size_t)(2 * rp + 1) * W) / 2 + j] = yuyv_pair_word(s0 + (size_t)W * 3);
  }
}

static bool gauss_fast_params(const GaussTaps& t, GaussFast* f) {
  if (t.k < 3 || t.k > 2 * GF_MAXR + 1) return false;
  f->k = t.k; f->nw = (t.k + 3 + 3) / 4; f->nv = (t.k + 1 + 1) / 2;
  auto q = [&](int j) -> unsigned { return (j >= 0 && j < t.k) ? (unsigned)t.q[j] : 0u; };
  for (int i = 0; i < 4; ++i)
    for (int w = 0; w < GF_NW; ++w) {
      unsigned v = 0;
      for (int b = 0; b < 4; ++b) v |= q(4 * w + b - i) << (8 * b);
      f->hq[i][w] = v;
    }
  for (int w = 0; w < GF_NV; ++w) f->cw[w] = q(2 * w) | (q(2 * w + 1) << 8) | (q(2 * w - 1) << 16) | (q(2 * w) << 24);
  return true;
}

// the taps of every odd strength on the CURRENT device, built from gauss_taps on first use (one per device, under a
// mutex like ensure_dyn_smem; contexts call it before they capture a graph)
static const GaussTables* gauss_tables() {
  static std::mutex mu;
  static std::map<int, GaussTables*> tabs;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  auto it = tabs.find(dev);
  if (it != tabs.end()) return it->second;
  std::vector<GaussTables> h(1);
  GaussTables& t = h[0];
  std::memset(&t, 0, sizeof(t));
  for (int k = 1; k <= 255; k += 2) {
    gauss_taps(k, &t.taps[(k - 1) >> 1]);
    if (gauss_class(k) == GAUSS_FUSED) gauss_fast_params(t.taps[(k - 1) >> 1], &t.fast[(k - 3) >> 1]);
  }
  GaussTables* d = nullptr;
  if (cudaMalloc((void**)&d, sizeof(GaussTables)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, &t, sizeof(GaussTables), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  tabs[dev] = d;
  return d;
}

bool gauss_tables_ready() { return gauss_tables() != nullptr; }

size_t gauss_cols_smem(int k) { return (size_t)(GAUSS_CH + 2 * (k >> 1)) * GAUSS_CL * sizeof(uint16_t); }

// classes: GAUSS_FUSED and / or GAUSS_SEPARABLE launches; ks null: every frame at k_all
static bool launch_gauss_classes(cudaStream_t s, int n, const uint8_t* src, size_t spitch, size_t sstride, const int* ks, int k_all,
                                 unsigned classes, uint16_t* tmp, uint8_t* dst, size_t dpitch, size_t dstride, int W, int H,
                                 uint8_t* yuyv = nullptr, uint8_t* nv12 = nullptr) {
  const GaussTables* T = gauss_tables();
  if (!T) return false;
  static const GaussFast g25 = [] { GaussTaps t{}; GaussFast f{}; gauss_taps(25, &t); gauss_fast_params(t, &f); return f; }();
  if (classes & GAUSS_FUSED) {
    const int vec_ok = (reinterpret_cast<uintptr_t>(dst) % 16 == 0 && dpitch % 16 == 0 && dstride % 16 == 0) ? 1 : 0;
    const dim3 grid((unsigned)ceil_div(W, GF_TW), (unsigned)ceil_div(H, GF_TH), (unsigned)n);
    BSB_LAUNCH(k_gauss_fused, grid, dim3(256), 0, s, src, spitch, sstride, dst, dpitch, dstride, W, H, T, g25, k_all, ks, vec_ok, yuyv,
               nv12);
    count_launch();
  }
  if (classes & GAUSS_SEPARABLE) {
    BSB_LAUNCH(k_gauss_rows, dim3((unsigned)ceil_div(W, GAUSS_TW), (unsigned)H, (unsigned)n), dim3(256), 0, s, src, spitch, sstride, tmp, W, H,
               T, k_all, ks);
    count_launch();
    // a table call may replay with any strength of the class: room for k = 255
    const size_t smem = gauss_cols_smem(ks ? 255 : k_all);
    ensure_dyn_smem(reinterpret_cast<const void*>(k_gauss_cols), smem);
    BSB_LAUNCH(k_gauss_cols, dim3((unsigned)ceil_div(W * 3, GAUSS_CL), (unsigned)ceil_div(H, GAUSS_CH), (unsigned)n), dim3(256), smem, s,
               tmp, dst, dpitch, dstride, W, H, T, k_all, ks);
    count_launch();
  }
  return true;
}

bool launch_gauss_blur(cudaStream_t s, int n, const uint8_t* src, size_t spitch, size_t sstride, uint16_t* tmp,
                       uint8_t* dst, size_t dpitch, size_t dstride, int W, int H, const GaussTaps& g) {
  return launch_gauss_classes(s, n, src, spitch, sstride, nullptr, g.k, (unsigned)gauss_class(g.k), tmp, dst, dpitch, dstride, W, H);
}

bool launch_gauss_frames(cudaStream_t s, int n, const GaussSrc& cam, const int* ks, unsigned classes, uint8_t* frames, uint16_t* tmp,
                         uint8_t* dst, uint8_t* dst_yuyv, uint8_t* dst_nv12, int W, int H) {
  const size_t fbytes = (size_t)W * H * 3;
  if (cam.p) {
    const long blocks = ((long)(W / 2) * H + 255) / 256;
    BSB_LAUNCH(k_gauss_stage_bgr, dim3((unsigned)blocks, (unsigned)n), dim3(256), 0, s, cam, frames, W, H, ks);
    count_launch();
  }
  if (!launch_gauss_classes(s, n, frames, (size_t)W * 3, fbytes, ks, 0, classes, tmp, dst, (size_t)W * 3, fbytes, W, H, dst_yuyv, dst_nv12))
    return false;
  if ((classes & GAUSS_SEPARABLE) && (dst_yuyv || dst_nv12)) {
    const long blocks = ((long)(W / 2) * ((H + 1) / 2) + 255) / 256;
    BSB_LAUNCH(k_gauss_slot_yuv, dim3((unsigned)blocks, (unsigned)n), dim3(256), 0, s, dst, fbytes, dst_yuyv, dst_nv12, W, H, ks);
    count_launch();
  }
  return true;
}

// OpenCV getGaussianKernelBitExact + getGaussianKernelFixedPoint_ED for sigma = 0 (8 fractional bits).
bool gauss_taps(int k, GaussTaps* out) {
  if (k < 1 || !(k & 1) || k > 255) return false;
  static const double small[5][9] = {
      {1.0}, {0.25, 0.5, 0.25}, {0.0625, 0.25, 0.375, 0.25, 0.0625},
      {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125},
      {4.0 / 256, 13.0 / 256, 30.0 / 256, 51.0 / 256, 60.0 / 256, 51.0 / 256, 30.0 / 256, 13.0 / 256, 4.0 / 256}};
  double v[255];
  const int n2 = k / 2;
  if (k <= 9) {
    for (int i = 0; i < k; ++i) v[i] = small[n2][i];
  } else {
    const double sigma = std::fma((double)k, 0.15, 0.35), scale2x = -0.125 / (sigma * sigma);
    double sum = 0.0;
    for (int i = 0, x = 1 - k; i < n2; ++i, x += 2) { v[i] = std::exp((double)(x * x) * scale2x); sum += v[i]; }
    const double mul = 1.0 / (sum * 2.0 + 1.0);
    for (int i = 0; i < n2; ++i) v[i] *= mul;
    v[n2] = mul;
  }
  double err = 0.0;
  int acc = 0;
  for (int i = 0; i < n2; ++i) {
    const double adj = v[i] * 256.0 + err;
    const int q = (int)std::nearbyint(adj);
    err = adj - (double)q;
    out->q[i] = out->q[k - 1 - i] = (uint16_t)q;
    acc += q;
  }
  out->q[n2] = (uint16_t)(256 - 2 * acc);
  out->k = k;
  return true;
}

// ---------------------------------------------------------------------------
// cv::flip for n packed W x H x 3 frames.  One thread = one destination pixel.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_flip_u8c3(const uint8_t* src, size_t sstride, uint8_t* dst, size_t dstride, int W, int H,
                                                   int flip_h, int flip_v) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (size_t)W * H) return;
  const int x = (int)(p % W), y = (int)(p / W);
  const uint8_t* sp = src + (size_t)blockIdx.y * sstride + ((size_t)(flip_v ? H - 1 - y : y) * W + (flip_h ? W - 1 - x : x)) * 3;
  uint8_t* dp = dst + (size_t)blockIdx.y * dstride + 3 * p;
  dp[0] = sp[0]; dp[1] = sp[1]; dp[2] = sp[2];
}

void launch_flip_u8c3(cudaStream_t s, int n, const uint8_t* src, size_t sstride, uint8_t* dst, size_t dstride, int W, int H, bool flip_h, bool flip_v) {
  const size_t npix = (size_t)W * H;
  BSB_LAUNCH(k_flip_u8c3, dim3((unsigned)((npix + 255) / 256), (unsigned)n), dim3(256), 0, s, src, sstride, dst, dstride, W, H,
             flip_h ? 1 : 0, flip_v ? 1 : 0);
  count_launch();
}

__global__ void k_advance_cursor(int* cursor, int step, int count) { *cursor = (int)(((unsigned)*cursor + (unsigned)step) % (unsigned)count); }

void launch_advance_cursor(cudaStream_t s, int* cursor, int step, int count) {
  BSB_LAUNCH(k_advance_cursor, dim3(1), dim3(1), 0, s, cursor, step, count);
  count_launch();
}

}  // namespace bsb
