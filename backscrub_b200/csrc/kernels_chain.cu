// backscrub_b200/csrc/kernels_chain.cu — the low-resolution middle of the MobileNetV3-style graphs in ONE kernel.
//
// The Meet / MLKit graphs spend 20+ operators (and, unfused, 30 kernel launches) on tensors of 9x16 / 16x16 pixels:
// depthwise 5x5, squeeze-excite (global pool -> FC -> FC -> sigmoid -> channel scale), 1x1 project / expand
// (reference kernels: depthwiseconv_float.h:25-96, pooling.h:26-79, fully_connected.h:27-61, conv.h:25-99; delegated to
// XNNPACK by the reference, xnnpack_delegate.cc:1840-2497).  None of those launches can fill the GPU, and the SE
// reductions serialise them.  Here one CTA owns one frame and keeps every activation of the chain in shared memory
// (see kernels.h: X / D / E); the batch x streams dimension provides the parallelism.  For the Meet geometries the
// expanded tensor goes through E 16 channels at a time, which brings the CTA under half an SM's shared memory and
// registers: two frames share an SM and cover each other's barrier and L2 waits.  MLKit (16x16) cannot fit two at any
// slice width and keeps 32-channel slices, one frame per SM.
//
// Arithmetic contract: identical to the stand-alone kernels (kernels_nn.cu) and therefore to the oracle —
// every output accumulates fmaf in ascending k / (fy, fx) order, the pool sums each row left to right and then the
// rows top to bottom, the SE scale multiplies the operand (one rounding) before the fmaf.
#include <algorithm>
#include <mutex>

#include "kernels.h"

namespace bsb {

void count_launch();

#ifdef BSB_EMU
// the kernel-logic emulator build only (tests/emu, set by the tests through ctypes): nonzero runs every geometry on the
// runtime-shape instantiations (Meet lite reaches the two-per-SM one anyway; no bundled graph reaches the one-per-SM one)
extern "C" {
int bsb_emu_chain_runtime_shape = 0;
}
static bool chain_fixed_shape() { return !bsb_emu_chain_runtime_shape; }
#else
constexpr bool chain_fixed_shape() { return true; }
#endif

namespace {

constexpr int CH_T = 512;            // threads per CTA of the one-frame-per-SM instantiation
constexpr int CH_T2 = 384;           // threads per CTA of the two-frames-per-SM instantiation
constexpr int CH_XLD = 32;           // X row stride (floats): block inputs / outputs have <= 32 channels
constexpr int CH_DLD = 128;          // D row stride: expanded tensors have <= 128 channels

constexpr int CH_PAD = 2;            // zero halo of the E slice (covers 3x3 and 5x5 stride-1 windows)
// pixel row stride of the haloed E grid.  With 16-channel slices a warp reads two pixel rows at once (one per
// half-warp); an odd stride puts them 16 banks apart.  With 32-channel slices a warp reads one pixel, any stride is free.
BSB_HD int chain_estride(int w, int eld) { return eld < 32 ? (w + 2 * CH_PAD) | 1 : w + 2 * CH_PAD; }
struct ChainLayout { int off_x, off_d, off_e, e_floats, off_w1, off_wd, off_vec, total; };   // float offsets
// eld: E slice width (16 or 32 channels)
BSB_HD ChainLayout chain_layout(int h, int w, int eld) {
  // the fixed-size pieces first: their addresses are compile-time constants in the kernel and cost no registers
  ChainLayout L;
  const int P = h * w;
  L.off_vec = 0;                                  // v0 | v1 | sv
  L.off_wd = L.off_vec + 3 * 128;                 // depthwise taps of one slice [k*k <= 25][eld]
  L.off_w1 = L.off_wd + 25 * eld;                 // expand weights of one slice [cin <= 32][eld]
  L.off_x = L.off_w1 + 32 * eld;
  L.off_d = L.off_x + P * CH_XLD;
  L.off_e = L.off_d + P * CH_DLD;                 // zero-haloed E slice; PW / FC weight staging and the pool row sums alias it
  int e_floats = (h + 2 * CH_PAD) * chain_estride(w, eld) * eld;
  if (e_floats < 4096) e_floats = 4096;           // PW staging: K * n4 <= 4096 (Engine::detect_chain)
  if (e_floats < h * CH_DLD) e_floats = h * CH_DLD;
  L.e_floats = e_floats;
  L.total = L.off_e + e_floats;
  return L;
}

BSB_D float chain_act2(float v, int a1, int a2) { return bsb_act(bsb_act(v, a1), a2); }

// dst[p][n] = act(sum_k A[p][k] (* sv[k]) * Ws[k][n] + bias) (+ residual), R rows x 4 columns per thread, k ascending.
// A: shared [P][lda]; Ws: shared [K][n4] (zero padded); dst: shared, row p at dst + drow(p) * ldd (may be the residual
// source: each element is read and then written by the same thread).  pw > 0: dst is the zero-haloed E slice
// (row p = pixel (p / pw, p % pw) of a (h + 4) x (pw + 4) grid of row stride es).  ACT2 >= 0 fixes the second
// activation at compile time (the first one must then be ACT_NONE); ACT2 < 0 is the generic path.
template <int R, int ACT2>
BSB_D void chain_gemm_t(const float* A, int lda, int K, const float* sv, const float* Ws, int n4, int N, const float* bias,
                        int a1, int a2, bool residual, int a3, float* dst, int ldd, int P, int pw, int es) {
  const int cg = n4 / 4, rg = (P + R - 1) / R;
  for (int t = threadIdx.x; t < cg * rg; t += blockDim.x) {
    const int tx = t % cg, ty = t / cg;
    const int n0 = tx * 4, p0 = ty * R;
    float acc[R][4];
#pragma unroll
    for (int i = 0; i < R; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    const float* ar[R];
#pragma unroll
    for (int i = 0; i < R; ++i) ar[i] = A + (size_t)min(p0 + i, P - 1) * lda;
    for (int k = 0; k < K; k += 4) {
      float4 av[R];
#pragma unroll
      for (int i = 0; i < R; ++i) av[i] = *reinterpret_cast<const float4*>(ar[i] + k);
      if (sv) {
        const float4 sc = *reinterpret_cast<const float4*>(sv + k);
#pragma unroll
        for (int i = 0; i < R; ++i) { av[i].x = av[i].x * sc.x; av[i].y = av[i].y * sc.y; av[i].z = av[i].z * sc.z; av[i].w = av[i].w * sc.w; }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 w4 = *reinterpret_cast<const float4*>(Ws + (size_t)(k + j) * n4 + n0);
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const float a = j == 0 ? av[i].x : (j == 1 ? av[i].y : (j == 2 ? av[i].z : av[i].w));
          acc[i][0] = fmaf(a, w4.x, acc[i][0]); acc[i][1] = fmaf(a, w4.y, acc[i][1]);
          acc[i][2] = fmaf(a, w4.z, acc[i][2]); acc[i][3] = fmaf(a, w4.w, acc[i][3]);
        }
      }
    }
    float bv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) bv[j] = (bias && n0 + j < N) ? __ldg(bias + n0 + j) : 0.f;
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int p = p0 + i;
      if (p >= P) break;
      const int drow = pw > 0 ? ((p / pw + CH_PAD) * es + (p % pw) + CH_PAD) : p;
      float* dp = dst + (size_t)drow * ldd + n0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (n0 + j >= N) break;
        float v = acc[i][j] + bv[j];
        v = ACT2 >= 0 ? bsb_act(v, ACT2) : chain_act2(v, a1, a2);
        if (residual) v = bsb_act(v + dp[j], a3);
        dp[j] = v;
      }
    }
  }
}

template <int R>
BSB_D void chain_gemm(const float* A, int lda, int K, const float* sv, const float* Ws, int n4, int N, const float* bias,
                      int a1, int a2, bool residual, int a3, float* dst, int ldd, int P, int pw, int es) {
  // the activation combinations of the MobileNetV3-style graphs get their own instantiation (no per-element switch)
  if (a1 == ACT_NONE && a2 == ACT_NONE) chain_gemm_t<R, ACT_NONE>(A, lda, K, sv, Ws, n4, N, bias, a1, a2, residual, a3, dst, ldd, P, pw, es);
  else if (a1 == ACT_NONE && a2 == ACT_HARD_SWISH) chain_gemm_t<R, ACT_HARD_SWISH>(A, lda, K, sv, Ws, n4, N, bias, a1, a2, residual, a3, dst, ldd, P, pw, es);
  else if (a1 == ACT_NONE && a2 == ACT_RELU6) chain_gemm_t<R, ACT_RELU6>(A, lda, K, sv, Ws, n4, N, bias, a1, a2, residual, a3, dst, ldd, P, pw, es);
  else if (a1 == ACT_NONE && a2 == ACT_RELU) chain_gemm_t<R, ACT_RELU>(A, lda, K, sv, Ws, n4, N, bias, a1, a2, residual, a3, dst, ldd, P, pw, es);
  else chain_gemm_t<R, -1>(A, lda, K, sv, Ws, n4, N, bias, a1, a2, residual, a3, dst, ldd, P, pw, es);
}

// global [K][n4] -> shared, all loads in flight
BSB_D void chain_stage(float* ws, const float* w, int count) {
  for (int i = threadIdx.x * 4; i < count; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(ws + i) = __ldg(reinterpret_cast<const float4*>(w + i));
}

// one fully-connected layer of the SE path: out[n] = act(sum_k in[k] * w[k][n] + bias), k ascending.  The weights are
// pulled into shared memory (`stage`, `cap` floats) by the whole CTA in chunks of rows — one coalesced L2 round trip per
// chunk instead of K dependent ones — and the running sums stay in registers across chunks.
BSB_D void chain_fc(const float* in, const FcLayer& f, float* out, float* stage, int cap) {
  const int rows_per_chunk = max(1, cap / f.n4);
  const int n = threadIdx.x;
  float acc = 0.f;
  for (int k0 = 0; k0 < f.K; k0 += rows_per_chunk) {
    const int rows = min(rows_per_chunk, f.K - k0);
    __syncthreads();                                              // the previous chunk (or the caller's use of `stage`) is consumed
    chain_stage(stage, f.w + (size_t)k0 * f.n4, rows * f.n4);
    __syncthreads();
    if (n < f.N) for (int k = 0; k < rows; ++k) acc = fmaf(in[k0 + k], stage[k * f.n4 + n], acc);
  }
  if (n < f.N) out[n] = chain_act2(acc + (f.bias ? __ldg(f.bias + n) : 0.f), f.act1, f.act2);
}

// depthwise KS x KS, stride 1, SAME, of one ELD-channel slice: E (zero-haloed (h+4) x (w+4) grid of [ELD], row stride
// chain_estride) -> D[:, c0 : c0 + cw].  A lane keeps its channel, so its KS*KS taps live in registers; a thread produces
// 4 consecutive pixels of a row from KS x (KS + 3) loads.  With 16-channel slices the two half-warps take the same strip
// of two consecutive rows (an odd row stride apart: no bank conflict).  Out-of-image taps read the halo's zeros:
// fmaf(+0, w, acc) leaves acc unchanged bit for bit (an accumulator that starts at +0 can never become -0 by adding
// zeros), so skipping them as the oracle does gives the same bits.
template <int KS, int ACT2, int ELD>
BSB_D void chain_dw_slice_t(const float* E, const float* wds, const ChainOp& op, int c0, int cw, int h, int w, int es, float* D) {
  constexpr int ROWS = 32 / ELD;                  // output rows per warp
  const int j = threadIdx.x % ELD, half = (threadIdx.x & 31) / ELD;
  if (j >= cw) return;
  float wr[KS * KS];
#pragma unroll
  for (int t = 0; t < KS * KS; ++t) wr[t] = wds[t * ELD + j];
  const float bias = op.bd ? __ldg(op.bd + c0 + j) : 0.f;
  const int ew = w + 2 * CH_PAD, strips = (w + 3) / 4, row_groups = (h + ROWS - 1) / ROWS;
  const bool full = (w & 3) == 0;                 // every strip has 4 pixels and its KS + 3 columns lie inside the haloed grid
  for (int sidx = threadIdx.x >> 5; sidx < row_groups * strips; sidx += blockDim.x >> 5) {
    const int ry = sidx / strips, oy = ry * ROWS + half, ox0 = (sidx - ry * strips) * 4;
    if (oy >= h) continue;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    // window origin in the haloed grid: (oy - pt + CH_PAD, ox0 - pl + CH_PAD); pt, pl <= CH_PAD
    const float* e0 = E + ((size_t)(oy - op.pt + CH_PAD) * es + (ox0 - op.pl + CH_PAD)) * ELD + j;
#pragma unroll
    for (int fy = 0; fy < KS; ++fy) {
      float v[KS + 3];
      if (full) {
#pragma unroll
        for (int c = 0; c < KS + 3; ++c) v[c] = e0[((size_t)fy * es + c) * ELD];
      } else {
#pragma unroll
        for (int c = 0; c < KS + 3; ++c) v[c] = (ox0 - op.pl + CH_PAD + c < ew) ? e0[((size_t)fy * es + c) * ELD] : 0.f;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int fx = 0; fx < KS; ++fx) acc[q] = fmaf(v[q + fx], wr[fy * KS + fx], acc[q]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (ox0 + q < w) {
        const float r = acc[q] + bias;
        D[(size_t)(oy * w + ox0 + q) * CH_DLD + c0 + j] = ACT2 >= 0 ? bsb_act(r, ACT2) : chain_act2(r, op.dact1, op.dact2);
      }
  }
}

template <int KS, int ELD>
BSB_D void chain_dw_slice(const float* E, const float* wds, const ChainOp& op, int c0, int cw, int h, int w, int es, float* D) {
  if (op.dact1 == ACT_NONE && op.dact2 == ACT_HARD_SWISH) chain_dw_slice_t<KS, ACT_HARD_SWISH, ELD>(E, wds, op, c0, cw, h, w, es, D);
  else if (op.dact1 == ACT_NONE && op.dact2 == ACT_RELU6) chain_dw_slice_t<KS, ACT_RELU6, ELD>(E, wds, op, c0, cw, h, w, es, D);
  else if (op.dact1 == ACT_NONE && op.dact2 == ACT_RELU) chain_dw_slice_t<KS, ACT_RELU, ELD>(E, wds, op, c0, cw, h, w, es, D);
  else chain_dw_slice_t<KS, -1, ELD>(E, wds, op, c0, cw, h, w, es, D);
}

// CH_DWG: depthwise KS x KS, stride op.s, SAME, from the global tensor op.gin into D[p][c]; taps from shared `wsm`
// ([KS*KS][C]).  A thread computes 4 channels of one pixel; each window row's KS input loads are issued together before
// its fmafs.  Out-of-image taps load +0 instead of being skipped: the accumulator starts at +0 and can never become -0
// (fmaf rounds an exact zero sum to +0), so fmaf(+0, w, acc) leaves it unchanged bit for bit and every output keeps
// the oracle's fmaf chain over the in-image taps in (fy, fx) order.
template <int KS>
BSB_D void chain_dwg(const ChainOp& op, const float* wsm, float* D, int b, int P, int w) {
  const float* gin = op.gin + (size_t)b * op.gin_frame;
  const int C = op.cin, groups = C / 4, ld = op.gin_ld, ih = op.ih, iw = op.iw, st = op.s;
  for (int i = threadIdx.x; i < P * groups; i += blockDim.x) {
    const int p = i / groups, c0 = (i - p * groups) * 4;
    const int oy = p / w, ox = p - oy * w;
    const int iy0 = oy * st - op.pt, ix0 = ox * st - op.pl;
    const int g0 = (iy0 * iw + ix0) * ld + c0;      // element offset of the window origin (may lie outside the image)
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int fy = 0; fy < KS; ++fy) {                // one row's loads in flight at a time: more do not fit 80 registers
      const bool row_in = (unsigned)(iy0 + fy) < (unsigned)ih;
      float4 v[KS];
#pragma unroll
      for (int fx = 0; fx < KS; ++fx)
        v[fx] = row_in && (unsigned)(ix0 + fx) < (unsigned)iw ? __ldg(reinterpret_cast<const float4*>(gin + g0 + (fy * iw + fx) * ld))
                                                               : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int fx = 0; fx < KS; ++fx) {
        const float4 wv = *reinterpret_cast<const float4*>(wsm + (fy * KS + fx) * C + c0);
        acc.x = fmaf(v[fx].x, wv.x, acc.x); acc.y = fmaf(v[fx].y, wv.y, acc.y);
        acc.z = fmaf(v[fx].z, wv.z, acc.z); acc.w = fmaf(v[fx].w, wv.w, acc.w);
      }
    }
    const float4 bv = op.bd ? __ldg(reinterpret_cast<const float4*>(op.bd + c0)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float* d = D + (size_t)p * CH_DLD + c0;
    d[0] = chain_act2(acc.x + bv.x, op.dact1, op.dact2);
    d[1] = chain_act2(acc.y + bv.y, op.dact1, op.dact2);
    d[2] = chain_act2(acc.z + bv.z, op.dact1, op.dact2);
    d[3] = chain_act2(acc.w + bv.w, op.dact1, op.dact2);
  }
}

}  // namespace

// The op descriptors are copied into shared memory, one op ahead: the loops then read their fields (k, strides, channel
// counts, weight pointers) from a uniform shared address instead of from global memory behind every barrier.
constexpr int CH_OP_WORDS = (int)(sizeof(ChainOp) / sizeof(int));
static_assert(sizeof(ChainOp) % sizeof(int) == 0 && CH_OP_WORDS <= CH_T2, "one thread per ChainOp word");
constexpr size_t CH_OP_SMEM = 2 * sizeof(ChainOp);   // static shared memory of k_chain: the double-buffered descriptor

BSB_D void chain_fetch_op(int* dst, const ChainOp* src) {
  if ((int)threadIdx.x < CH_OP_WORDS) dst[threadIdx.x] = __ldg(reinterpret_cast<const int*>(src) + threadIdx.x);
}

// R: rows per thread tile of the GEMMs; ELD: E slice width; NT, MIN_CTAS: threads per CTA and CTAs per SM.
// HC x WC: the geometry fixed at compile time (pixel counts, strides, strip and tile counts become constants, index
// divisions by them become multiplies and shifts); HC = WC = 0 takes h, w and es = chain_estride(w, ELD) at run time
// (read from the constant bank, they cost no register).
template <int R, int ELD, int NT, int MIN_CTAS, int HC, int WC>
__global__ void __launch_bounds__(NT, MIN_CTAS) k_chain(const ChainOp* ops, int n_ops, int h_rt, int w_rt, int es_rt) {
  // expand GEMM into a 16-column slice: (P / 2) x 4 thread tiles (Meet: 288 of the 384 threads)
  constexpr int RE = ELD == 16 ? 2 : R;
  const int h = HC ? HC : h_rt, w = WC ? WC : w_rt, es = HC ? chain_estride(WC, ELD) : es_rt;
  BSB_DYN_SMEM(smem_raw);
  __shared__ __align__(16) int op_sm[2][CH_OP_WORDS];
  float* sm = reinterpret_cast<float*>(smem_raw);
  const int P = h * w;
  const ChainLayout L = chain_layout(h, w, ELD);
  float* X = sm + L.off_x; float* D = sm + L.off_d; float* E = sm + L.off_e;
  float* w1s = sm + L.off_w1; float* wds = sm + L.off_wd;
  float* v0 = sm + L.off_vec; float* v1 = v0 + 128; float* sv = v1 + 128;
  const int tid = threadIdx.x, T = NT;                  // launched with NT threads
  const int b = blockIdx.x;

  chain_fetch_op(op_sm[0], ops);
  for (int oi = 0; oi < n_ops; ++oi) {
    __syncthreads();                                      // the previous op's results (and op_sm[oi & 1]) are complete
    if (oi + 1 < n_ops) chain_fetch_op(op_sm[(oi + 1) & 1], ops + oi + 1);   // its buffer was last read by op oi - 1
    const ChainOp& op = *reinterpret_cast<const ChainOp*>(op_sm[oi & 1]);
    switch (op.type) {
      case CH_DWG: {
        // depthwise k x k, stride s, SAME padding, straight from the global input tensor into D[p][c].  The taps
        // (k * k * C <= 25 * 128 floats, Engine::detect_chain) are staged in E, which is free here.
        chain_stage(E, op.wd, op.k * op.k * op.cin);
        __syncthreads();
        if (op.k == 5) chain_dwg<5>(op, E, D, b, P, w);
        else chain_dwg<3>(op, E, D, b, P, w);
        break;
      }
      case CH_EXPAND_DW: {
        // X [P][cin] -> expand 1x1 (+act) -> depthwise k x k stride 1 (+act) -> D [P][cout], one ELD-channel slice at a
        // time (E was used as scratch by the ops in between: its zero halo is rebuilt first)
        {
          const int eh = h + 2 * CH_PAD;
          for (int i = tid; i < eh * es * (ELD / 4); i += T) {
            const int cell = i / (ELD / 4), ey = cell / es, ex = cell - ey * es;
            if (ey < CH_PAD || ey >= h + CH_PAD || ex < CH_PAD || ex >= w + CH_PAD)
              *reinterpret_cast<float4*>(E + (size_t)cell * ELD + 4 * (i % (ELD / 4))) = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
        for (int c0 = 0; c0 < op.cout; c0 += ELD) {
          const int cw = min(ELD, op.cout - c0);
          if (c0) __syncthreads();                        // the previous slice's E / w1s / wds are fully consumed
          for (int i = tid; i < op.cin * ELD; i += T) {
            const int kk = i / ELD, j = i % ELD;
            w1s[i] = j < cw ? __ldg(op.w + (size_t)kk * op.n4 + c0 + j) : 0.f;
          }
          for (int i = tid; i < op.k * op.k * ELD; i += T) {
            const int tp = i / ELD, j = i % ELD;
            wds[i] = j < cw ? __ldg(op.wd + (size_t)tp * op.cout + c0 + j) : 0.f;
          }
          __syncthreads();
          chain_gemm<RE>(X, CH_XLD, op.cin, nullptr, w1s, ELD, cw, op.b ? op.b + c0 : nullptr, op.act1, op.act2, false, 0, E, ELD, P, w, es);
          __syncthreads();
          if (op.k == 5) chain_dw_slice<5, ELD>(E, wds, op, c0, cw, h, w, es, D);
          else chain_dw_slice<3, ELD>(E, wds, op, c0, cw, h, w, es, D);
        }
        break;
      }
      case CH_SE: {
        // global average pool: row sums (x ascending) -> E (aliased as rs[h][C]), then rows (y ascending), / (h*w)
        const float* src = op.src ? D : X;
        const int ld = op.src ? CH_DLD : CH_XLD, C = op.cin;
        float* rs = E;
        for (int i = tid; i < h * C; i += T) {
          const int y = i / C, c = i - y * C;
          const float* sp = src + (size_t)(y * w) * ld + c;
          float r = 0.f;
          for (int x = 0; x < w; ++x) r = r + sp[(size_t)x * ld];
          rs[i] = r;
        }
        __syncthreads();
        for (int c = tid; c < C; c += T) {
          float t = 0.f;
          for (int y = 0; y < h; ++y) t = t + rs[y * C + c];
          v0[c] = bsb_act(bsb_div(t, (float)(h * w)), op.pool_act);
        }
        __syncthreads();
        if (op.n_fc == 1) chain_fc(v0, op.f0, sv, E, L.e_floats);
        else {
          chain_fc(v0, op.f0, v1, E, L.e_floats);
          chain_fc(v1, op.f1, sv, E, L.e_floats);
        }
        break;
      }
      case CH_PW: {
        const float* A = op.src ? D : X;
        const int lda = op.src ? CH_DLD : CH_XLD;
        float* dst = op.dst ? D : X;
        const int ldd = op.dst ? CH_DLD : CH_XLD;
        float* Ws = E;                                    // [K][n4] staging (E is dead outside EXPAND_DW)
        chain_stage(Ws, op.w, op.cin * op.n4);
        __syncthreads();
        chain_gemm<R>(A, lda, op.cin, op.use_scale ? sv : nullptr, Ws, op.n4, op.cout, op.b, op.act1, op.act2, op.residual != 0, op.act3, dst, ldd, P, 0, 0);
        break;
      }
      case CH_SCALE_STORE: {
        float* go = op.gout + (size_t)b * op.gout_frame;
        const int C = op.cin, groups = C / 4;
        for (int i = tid; i < P * groups; i += T) {
          const int p = i / groups, c0 = (i - p * groups) * 4;
          const float* d = D + (size_t)p * CH_DLD + c0;
          *reinterpret_cast<float4*>(go + (size_t)p * op.gout_ld + c0) =
              make_float4(bsb_act(d[0] * sv[c0], op.act1), bsb_act(d[1] * sv[c0 + 1], op.act1), bsb_act(d[2] * sv[c0 + 2], op.act1),
                          bsb_act(d[3] * sv[c0 + 3], op.act1));
        }
        break;
      }
      default: break;
    }
  }
}

namespace {

// Which instantiation runs a chain over h x w pixels.  The 384-thread one (GEMM tiles of 3 rows: (P / 3) x 8 = 384 tiles
// for Meet's 9x16) uses 16-channel E slices so that two CTAs fit on one SM; it is chosen when the geometry allows that on
// the current device (Meet full 9x16: 114 816 B, Meet lite 6x10).  Everything else (MLKit's 16x16: 512 threads, 4-row
// tiles, 219 KiB) runs one CTA per SM with 32-channel slices.
struct ChainConfig { bool two_per_sm; size_t smem; };

ChainConfig chain_config(int h, int w) {
  const int P = h * w;
  if (P % 3 == 0 && (P / 3) * 8 <= CH_T2) {
    const size_t bytes = (size_t)chain_layout(h, w, 16).total * sizeof(float);
    int per_sm = 228 * 1024, reserved = 1024;     // H100
#ifndef BSB_EMU
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev) != cudaSuccess) {
      cudaGetLastError();
      per_sm = 0;
    }
#endif
    if (2 * (bytes + CH_OP_SMEM + (size_t)reserved) <= (size_t)per_sm) return {true, bytes};
  }
  return {false, (size_t)chain_layout(h, w, 32).total * sizeof(float)};
}

}  // namespace

size_t chain_smem_bytes(int h, int w) {
  const int P = h * w;
  if (P < 1 || P > 256 || h > 64) return 0;
  const size_t bytes = chain_config(h, w).smem;
  return bytes <= 226 * 1024 ? bytes : 0;
}

namespace {

// two 384-thread CTAs per SM, 16-channel E slices
template <int HC, int WC>
void launch_chain_two(cudaStream_t s, int B, int h, int w, size_t smem, const ChainOp* d_ops, int n_ops) {
  auto k = k_chain<3, 16, CH_T2, 2, HC, WC>;
  ensure_dyn_smem(reinterpret_cast<const void*>(k), smem);
#ifndef BSB_EMU
  // the whole unified L1 / shared array as shared memory: room for the two CTAs (set once per device and instantiation)
  static std::once_flag carveout[64];
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && dev < 64)
    std::call_once(carveout[dev], [&] {
      if (cudaFuncSetAttribute(reinterpret_cast<const void*>(k), cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess)
        cudaGetLastError();
    });
#endif
  BSB_LAUNCH(k, dim3((unsigned)B), dim3(CH_T2), smem, s, d_ops, n_ops, h, w, chain_estride(w, 16));
}

// one 512-thread CTA per SM, 32-channel E slices
template <int HC, int WC>
void launch_chain_one(cudaStream_t s, int B, int h, int w, size_t smem, const ChainOp* d_ops, int n_ops) {
  auto k = k_chain<4, 32, CH_T, 1, HC, WC>;
  ensure_dyn_smem(reinterpret_cast<const void*>(k), smem);
  BSB_LAUNCH(k, dim3((unsigned)B), dim3(CH_T), smem, s, d_ops, n_ops, h, w, chain_estride(w, 32));
}

}  // namespace

// Meet full (9x16) and MLKit (16x16) run instantiations with the shape fixed at compile time; any other shape
// chain_smem_bytes accepts, Meet lite's 6x10 among them, runs the runtime-shape one of its configuration (a 6x10
// instantiation needs one register more than the 80 that two CTAs per SM allow, and would spill).
void launch_chain(cudaStream_t s, int B, int h, int w, const ChainOp* d_ops, int n_ops) {
  const ChainConfig cfg = chain_config(h, w);
  if (cfg.two_per_sm) {
    if (chain_fixed_shape() && h == 9 && w == 16) launch_chain_two<9, 16>(s, B, h, w, cfg.smem, d_ops, n_ops);
    else launch_chain_two<0, 0>(s, B, h, w, cfg.smem, d_ops, n_ops);
  } else {
    if (chain_fixed_shape() && h == 16 && w == 16) launch_chain_one<16, 16>(s, B, h, w, cfg.smem, d_ops, n_ops);
    else launch_chain_one<0, 0>(s, B, h, w, cfg.smem, d_ops, n_ops);
  }
  count_launch();
}

}  // namespace bsb
