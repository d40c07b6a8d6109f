// backscrub_b200/csrc/kernels_tc.cu — tensor-core pointwise (1x1) convolution for sm_90a.
//
// The 1x1 convs are the only dense GEMMs on the path (out[M][N] = A[M][K] * W[N][K]^T, M = frames*H*W).
// This kernel runs them on Hopper's warpgroup tensor cores: wgmma.mma_async m64nNk8 .tf32, fp32 accumulators in
// registers, operands in 128-byte-swizzled shared memory.  Single-pass TF32 breaks the mask-parity bar (SURVEY.md
// Appendix D), so every product is the 3xTF32 split
//     a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo,   x_hi = tf32(x) (truncation), x_lo = x - x_hi,
// three MMAs per K step into the same accumulator (the dropped a_lo*w_lo term is ~2^-22 relative).
// It is NOT bit-identical to the FFMA path / the oracle (different summation order); it is selected only
// with BSB_FLAG_TENSOR_CORES and is validated on output tolerance + decision agreement, and per call against float64
// (tests/test_tc_float64.py: exact dyadic fixtures and a derived error bound).
//
// A 128-row output tile is computed by two consumer warpgroups, 64 rows each (wgmma's M is 64 per warpgroup).
// Shared-memory operand layout (K-major, SWIZZLE_128B): one K chunk = 32 fp32 = one 128-byte row per
// M/N index; 8 rows form a 1024-byte swizzle atom in which the 16-byte column c of row r is stored at
// column c ^ (r & 7).  Descriptor: start >> 4, LBO = 1, SBO = 1024 >> 4, layout 1 (128-byte swizzle).
#include <algorithm>

#include "kernels.h"

namespace bsb {

void count_launch();

const char* pointwise_tc_refusal(int K, const float* A, int ld_a, int kpad, const float* out, int ld_out, const Epilogue& e) {
  if (K % 4 != 0 || ld_a % 4 != 0) return "K and ld_a must be multiples of 4";
  if (kpad % 32 != 0 || kpad < K) return "the padded weight depth kpad must be a multiple of 32 and at least K";
  // both kernels read A in 16-byte pieces (cp.async / TMA)
  if (reinterpret_cast<uintptr_t>(A) & 15) return "A must start on a 16-byte boundary";
  // tc_store writes out and reads the residual as float2 whenever both pitches are even
  const bool vec = (ld_out & 1) == 0 && (!e.residual || (e.ld_res & 1) == 0);
  if (vec && ((reinterpret_cast<uintptr_t>(out) & 7) || (reinterpret_cast<uintptr_t>(e.residual) & 7)))
    return "with even ld_out and ld_res, out and the residual must start on 8-byte boundaries";
  return nullptr;
}

#ifndef BSB_EMU

struct EpiDevTc { const float* bias; const float* residual; int ld_res; int act1, act2, act3; };

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the 128 threads of one warpgroup (named barriers 1 and 2: barrier 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" :: "r"(1 + wg) : "memory"); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

// D[64 x BN] (+)= A[64 x 8] * B[BN x 8]^T, both operands K-major tf32 in shared memory; acc = 0 overwrites D.
// Accumulator fragment of thread t of the warpgroup: d[i] is row 16*(t/32) + (t%32)/4 + 8*((i/2)%2),
// column 8*(i/4) + 2*(t%4) + i%2.
template <int BN> __device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(da), "l"(db), "r"(acc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(da), "l"(db), "r"(acc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(acc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<80>(float (&d)[40], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
               : "l"(da), "l"(db), "r"(acc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<96>(float (&d)[48], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
               : "l"(da), "l"(db), "r"(acc) : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(da), "l"(db), "r"(acc) : "memory");
}
// K-major SWIZZLE_128B shared-memory matrix descriptor (wgmma descriptor bit layout)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fffu);          // start address, bits [0,14)
  d |= (uint64_t)1u << 16;                           // leading byte offset (unused for swizzled K-major), bits [16,30)
  d |= (uint64_t)(1024u >> 4) << 32;                 // stride byte offset between 8-row groups, bits [32,46)
  d |= (uint64_t)1u << 62;                           // layout type SWIZZLE_128B, bits [62,64)
  return d;
}

__device__ __forceinline__ uint32_t swz(int row, int c16) {       // byte offset of 16-byte column c16 of row `row`
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((c16 ^ (row & 7)) << 4));
}

__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

// One K chunk (32) of a warpgroup's 64 x BN tile: 12 wgmma (a_lo*w_hi, a*w_lo, a*w_hi for 4 K steps; small terms first).
// a / a_lo / b_hi / b_lo: shared addresses of the operand tiles.  first: the chunk opens the accumulation.
template <int BN>
__device__ __forceinline__ void mma_chunk(float (&acc)[BN / 2], uint32_t a, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, bool first) {
  const uint64_t dA = make_desc(a), dA_lo = make_desc(a_lo), dB_hi = make_desc(b_hi), dB_lo = make_desc(b_lo);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {                      // K step = 8 tf32 = 32 bytes -> +2 in the (>>4) address field
    const uint64_t adv = (uint64_t)(ks * 2);
    wgmma_tf32<BN>(acc, dA_lo + adv, dB_hi + adv, (first && ks == 0) ? 0u : 1u);
    wgmma_tf32<BN>(acc, dA + adv, dB_lo + adv, 1u);
    wgmma_tf32<BN>(acc, dA + adv, dB_hi + adv, 1u);
  }
}

}  // namespace tc

// generic per-element epilogue (activation chains the fast path in tc_store does not cover); not inlined, so the fully
// unrolled store loop of every tile width carries only the fast path
__device__ __noinline__ float tc_epilogue(float total, int ch, size_t pix, const EpiDevTc e) {
  float v = total + (e.bias ? __ldg(e.bias + ch) : 0.f);
  v = bsb_act(v, e.act1);
  v = bsb_act(v, e.act2);
  if (e.residual) v = bsb_act(v + __ldg(e.residual + pix * (size_t)e.ld_res + ch), e.act3);
  return v;
}

// Accumulators of one warpgroup's 64 x BN tile (rows row0.., columns n0..) -> bias / activations / residual -> global.
// t: thread index in the warpgroup.  Each thread owns pairs of adjacent columns: 8-byte stores.
template <int BN>
__device__ __forceinline__ void tc_store(const float (&acc)[BN / 2], float* out, int ld_out, int M, int N, int row0, int n0,
                                         const EpiDevTc& e, int t) {
  // the activations of the GEMM-heavy graphs (none / relu / relu6 after the bias, then an optional residual add) become
  // two clamps with +-inf bounds; anything else takes the generic per-element path
  const bool simple = e.act2 == ACT_NONE && e.act3 == ACT_NONE && (e.act1 == ACT_NONE || e.act1 == ACT_RELU || e.act1 == ACT_RELU6);
  const float lo_b = e.act1 == ACT_NONE ? -INFINITY : 0.f, hi_b = e.act1 == ACT_RELU6 ? 6.f : INFINITY;
  const bool vec = (ld_out & 1) == 0 && (!e.residual || (e.ld_res & 1) == 0);
  const int r0 = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int ch = n0 + 8 * j + 2 * (t & 3);
    if (ch >= N) continue;
    const float b0 = e.bias ? __ldg(e.bias + ch) : 0.f;
    const float b1 = (e.bias && ch + 1 < N) ? __ldg(e.bias + ch + 1) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gm = r0 + 8 * h;
      if (gm >= M) continue;
      const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      float* op = out + (size_t)gm * ld_out + ch;
      if (simple && vec && ch + 1 < N) {
        float2 r = make_float2(fminf(fmaxf(v0 + b0, lo_b), hi_b), fminf(fmaxf(v1 + b1, lo_b), hi_b));
        if (e.residual) {
          const float2 q = __ldg(reinterpret_cast<const float2*>(e.residual + (size_t)gm * e.ld_res + ch));
          r.x += q.x; r.y += q.y;
        }
        *reinterpret_cast<float2*>(op) = r;
      } else {
        op[0] = tc_epilogue(v0, ch, (size_t)gm, e);
        if (ch + 1 < N) op[1] = tc_epilogue(v1, ch + 1, (size_t)gm, e);
      }
    }
  }
}

struct TcArgs {
  const float* A; const float* w_hi; const float* w_lo; float* out;
  int M, K, N, ld_a, ld_out, kpad;             // w_*: [npad][kpad], zero padded; kpad % 32 == 0, npad % BN == 0
  EpiDevTc e;
};

// One CTA = one 128 x BN output tile (BN <= 128).  256 threads = two warpgroups, 64 rows each.  Three shared-memory
// stages fed by cp.async (16-byte copies land directly at their swizzled position, two K chunks in flight ahead of the
// tensor core); per chunk the threads split the A tile in place into hi / lo, then each warpgroup issues its twelve
// wgmma and waits for them before the stage can be refilled.
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;                      // src-size 0 => 16 bytes of zeros
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

template <int BN>
__global__ void __launch_bounds__(256, 1) k_pointwise_tc(TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  constexpr int NS = 3;
  constexpr int A_BYTES = 128 * 128;            // 128 rows x 32 fp32
  constexpr int B_BYTES = BN * 128;
  constexpr int STAGE = 2 * A_BYTES + 2 * B_BYTES;
  uint8_t* base = smem_dyn;                      // 1024-byte aligned by declaration (SWIZZLE_128B atoms need it)

  const int tid = threadIdx.x, wg = tid >> 7;
  const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BN;
  const int nchunks = a.kpad / 32;
  const uint32_t sbase = tc::smem_u32(base);

  auto issue_loads = [&](int c) {           // global -> shared for K chunk c (A raw, W hi, W lo)
    const uint32_t st = sbase + (uint32_t)((c % NS) * STAGE);
    const int k0 = c * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = tid + 256 * i, row = q >> 3, c16 = q & 7;
      const int gm = m0 + row, gk = k0 + c16 * 4;
      const bool ok = gm < a.M && gk < a.K;
      cp_async16(st + tc::swz(row, c16), ok ? (const void*)(a.A + (size_t)gm * a.ld_a + gk) : (const void*)a.A, ok);
    }
    for (int q = tid; q < BN * 8; q += 256) {
      const int row = q >> 3, c16 = q & 7;
      const size_t g = (size_t)(n0 + row) * a.kpad + k0 + c16 * 4;
      const uint32_t off = tc::swz(row, c16);
      cp_async16(st + 2 * A_BYTES + off, a.w_hi + g, true);
      cp_async16(st + 2 * A_BYTES + B_BYTES + off, a.w_lo + g, true);
    }
  };

  // prologue: two chunks in flight
  issue_loads(0); cp_async_commit();
  if (nchunks > 1) issue_loads(1);
  cp_async_commit();

  float acc[BN / 2] = {};
  for (int c = 0; c < nchunks; ++c) {
    const int s = c % NS;
    // refill the stage that chunk c+2 will use (last read by the MMAs of chunk c-1, which both warpgroups have waited for)
    if (c + 2 < nchunks) issue_loads(c + 2);
    cp_async_commit();
    cp_async_wait<2>();                      // this thread's copies of chunk c have landed (it splits exactly those)
    uint8_t* sA_hi = base + s * STAGE;
    uint8_t* sA_lo = sA_hi + A_BYTES;
    // split the A tile in place: hi = tf32-representable part, lo = a - hi (exact)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int q = tid + 256 * i;
      const uint32_t off = tc::swz(q >> 3, q & 7);
      const float4 v = *reinterpret_cast<const float4*>(sA_hi + off);
      const float4 hi = make_float4(tc::tf32_trunc(v.x), tc::tf32_trunc(v.y), tc::tf32_trunc(v.z), tc::tf32_trunc(v.w));
      *reinterpret_cast<float4*>(sA_hi + off) = hi;
      *reinterpret_cast<float4*>(sA_lo + off) = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
    }
    tc::fence_proxy_async();                 // generic-proxy smem writes (cp.async + split) -> async proxy (tensor core)
    __syncthreads();
    const uint32_t st = sbase + (uint32_t)(s * STAGE);
    tc::wg_fence();
    tc::mma_chunk<BN>(acc, st + wg * 8192, st + A_BYTES + wg * 8192, st + 2 * A_BYTES, st + 2 * A_BYTES + B_BYTES, c == 0);
    tc::wg_commit();
    tc::wg_wait<0>();
    __syncthreads();                         // both warpgroups are done with stage s before it is refilled
  }
  tc_store<BN>(acc, a.out, a.ld_out, a.M, a.N, m0 + 64 * wg, n0, a.e, tid & 127);
}

template <int BN>
static bool launch_tc_bn(cudaStream_t s, const TcArgs& a, int npad) {
  const size_t smem = 3 * (2 * 128 * 128 + 2 * BN * 128);
  if (!ensure_dyn_smem(reinterpret_cast<const void*>(k_pointwise_tc<BN>), smem)) return false;
  dim3 grid((unsigned)ceil_div(a.M, 128), (unsigned)(npad / BN));
  k_pointwise_tc<BN><<<grid, 256, smem, s>>>(a);
  return true;
}


// ---------------------------------------------------------------------------------------------------------
// Warp-specialised, persistent, TMA-fed version (the default tensor-core kernel).  384 threads:
//
//   warpgroup 0      TMA producer (one thread): per K chunk of 32 floats one bulk tensor copy each for the raw A tile
//                    (128 rows, fp32 as stored by the producing layer), W_hi and W_lo (BN rows) into 128-byte-swizzled
//                    stages, completion on the stage's `full` mbarrier
//   warpgroups 1-2   consumers, 64 rows of the tile each: split a_lo = a - tf32_trunc(a) for their rows into the stage's
//                    A_lo tile (the tensor core truncates the raw fp32 operand to tf32 itself, so the "hi" part of A needs
//                    no pass of its own unless tc_mask_hi asks for it), issue the 12 wgmma of the chunk, and release the
//                    stage of the previous chunk (`empty` mbarrier) once its wgmma group has completed; after a tile's
//                    last chunk the epilogue runs from the accumulator registers while the producer fills the next stages
// CTAs are persistent (grid = #SMs) and walk the (M tile, N tile) list with a static stride.
// ---------------------------------------------------------------------------------------------------------
}  // namespace bsb
#include <cuda.h>
namespace bsb {

namespace tc {
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               :: "r"(dst), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
}  // namespace tc

struct TcMaps { CUtensorMap a, whi, wlo; };
struct Tc2Args { float* out; int M, K, N, ld_out, tiles_m, tiles_n, nchunks, mask_hi; EpiDevTc e; };

template <int BN>
struct Tc2Cfg {
  static constexpr int A_BYTES = 128 * 128;                       // 128 rows x 32 fp32
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE = 2 * A_BYTES + 2 * B_BYTES;        // A raw | A lo | W hi | W lo
  static constexpr int NS = (STAGE * 4 <= 220 * 1024) ? 4 : 3;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM = NS * STAGE + BAR_BYTES + 1024;      // + slack to align the stages to 1024 bytes
};

template <int BN>
__global__ void __launch_bounds__(384, 1) k_pointwise_tc2(const __grid_constant__ TcMaps tm, const Tc2Args a) {
  using C = Tc2Cfg<BN>;
  extern __shared__ uint8_t smem_tc2[];
  const uint32_t raw_base = tc::smem_u32(smem_tc2);
  const uint32_t sbase = (raw_base + 1023u) & ~1023u;             // SWIZZLE_128B atoms need 1024-byte alignment
  uint8_t* gen_base = smem_tc2 + (sbase - raw_base);
  uint64_t* bars = reinterpret_cast<uint64_t*>(gen_base + C::NS * C::STAGE);
  uint64_t* full = bars;                        // [NS] TMA bytes landed
  uint64_t* empty = bars + C::NS;               // [NS] both consumer warpgroups' wgmma that read the stage have completed

  const int tid = threadIdx.x, wg = tid >> 7;
  if (tid == 0) {
    for (int i = 0; i < C::NS; ++i) { tc::mbar_init(&full[i], 1); tc::mbar_init(&empty[i], 2); }
    tc::fence_barrier_init();
  }
  __syncthreads();
  const int ntiles = a.tiles_m * a.tiles_n;

  if (wg == 0) {
    // ===== TMA producer =====
    if (tid == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int m0 = (tile / a.tiles_n) * 128, n0 = (tile % a.tiles_n) * BN;
        for (int c = 0; c < a.nchunks; ++c, ++it) {
          const int s = it % C::NS;
          if (it >= C::NS) tc::mbar_wait(&empty[s], (uint32_t)((it / C::NS - 1) & 1));
          const uint32_t st = sbase + (uint32_t)(s * C::STAGE);
          tc::mbar_expect_tx(&full[s], (uint32_t)(C::A_BYTES + 2 * C::B_BYTES));
          tc::tma_load_2d(st, &tm.a, c * 32, m0, &full[s]);
          tc::tma_load_2d(st + 2 * C::A_BYTES, &tm.whi, c * 32, n0, &full[s]);
          tc::tma_load_2d(st + 2 * C::A_BYTES + C::B_BYTES, &tm.wlo, c * 32, n0, &full[s]);
        }
      }
    }
  } else {
    // ===== consumers =====
    const int cw = wg - 1, t = tid & 127;
    int it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int m0 = (tile / a.tiles_n) * 128, n0 = (tile % a.tiles_n) * BN;
      float acc[BN / 2] = {};
      for (int c = 0; c < a.nchunks; ++c, ++it) {
        const int s = it % C::NS;
        tc::mbar_wait(&full[s], (uint32_t)((it / C::NS) & 1));
        // A_lo = a - tf32_trunc(a) for this warpgroup's 64 rows (512 16-byte columns, 4 per thread)
        uint8_t* sA = gen_base + s * C::STAGE;
        uint8_t* sLo = sA + C::A_BYTES;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int q = t + 128 * i;
          const uint32_t off = tc::swz(64 * cw + (q >> 3), q & 7);
          const float4 v = *reinterpret_cast<const float4*>(sA + off);
          const float4 hi = make_float4(tc::tf32_trunc(v.x), tc::tf32_trunc(v.y), tc::tf32_trunc(v.z), tc::tf32_trunc(v.w));
          *reinterpret_cast<float4*>(sLo + off) = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
          if (a.mask_hi) *reinterpret_cast<float4*>(sA + off) = hi;   // do not rely on the tensor core truncating the raw operand
        }
        tc::fence_proxy_async();                 // generic-proxy writes of A_lo -> visible to the tensor core (async proxy)
        tc::wg_sync(cw);
        const uint32_t st = sbase + (uint32_t)(s * C::STAGE);
        tc::wg_fence();
        tc::mma_chunk<BN>(acc, st + cw * 8192, st + C::A_BYTES + cw * 8192, st + 2 * C::A_BYTES, st + 2 * C::A_BYTES + C::B_BYTES, c == 0);
        tc::wg_commit();
        tc::wg_wait<1>();                        // the previous chunk's wgmma have completed: its stage can be refilled
        if (c > 0 && t == 0) tc::mbar_arrive(&empty[(it - 1) % C::NS]);
      }
      tc::wg_wait<0>();
      if (t == 0) tc::mbar_arrive(&empty[(it - 1) % C::NS]);
      tc_store<BN>(acc, a.out, a.ld_out, a.M, a.N, m0 + 64 * cw, n0, a.e, t);
    }
  }
}

typedef CUresult (*TcEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TcEncodeFn tc_encode_fn() {
  static TcEncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); p = nullptr; }
    return reinterpret_cast<TcEncodeFn>(p);
  }();
  return fn;
}
// fp32 matrix [rows][cols], row pitch in floats; box = 32 floats x box_rows, 128-byte swizzle
static bool tc_make_map(CUtensorMap* m, const float* base, size_t rows, size_t cols, size_t pitch_floats, unsigned box_rows) {
  TcEncodeFn enc = tc_encode_fn();
  if (!enc || (reinterpret_cast<uintptr_t>(base) & 15) || (pitch_floats & 3)) return false;
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstr[1] = {pitch_floats * 4};
  const cuuint32_t box[2] = {32, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int BN>
static bool launch_tc2_bn(cudaStream_t s, int M, int K, int N, const float* A, int ld_a, const float* w_hi, const float* w_lo, int kpad, int npad,
                          float* out, int ld_out, const EpiDevTc& e) {
  TcMaps tm;
  if (!tc_make_map(&tm.a, A, (size_t)M, (size_t)K, (size_t)ld_a, 128)) return false;
  if (!tc_make_map(&tm.whi, w_hi, (size_t)npad, (size_t)kpad, (size_t)kpad, BN)) return false;
  if (!tc_make_map(&tm.wlo, w_lo, (size_t)npad, (size_t)kpad, (size_t)kpad, BN)) return false;
  Tc2Args a{out, M, K, N, ld_out, ceil_div(M, 128), npad / BN, kpad / 32, tuning().tc_mask_hi, e};
  if (!ensure_dyn_smem(reinterpret_cast<const void*>(k_pointwise_tc2<BN>), Tc2Cfg<BN>::SMEM)) return false;
  const int grid = std::min(device_sms(), a.tiles_m * a.tiles_n);
  k_pointwise_tc2<BN><<<grid, 384, Tc2Cfg<BN>::SMEM, s>>>(tm, a);
  return true;
}

int pointwise_tc_tile_n(int N) {       // tile width the launcher will use for this N (weights are padded to a multiple of it)
  if (N <= 16) return 16;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  if (N <= 96) return 96;
  if (N == 160 || N == 240 || N == 480) return 80;
  return 128;
}

bool launch_pointwise_tc(cudaStream_t s, int M, int K, int N, const float* A, int ld_a, const float* w_hi, const float* w_lo,
                         int kpad, int npad, float* out, int ld_out, const Epilogue& e) {
  if (pointwise_tc_refusal(K, A, ld_a, kpad, out, ld_out, e)) return false;
  const EpiDevTc ed{e.bias, e.residual, e.ld_res, e.act1, e.act2, e.act3};
  TcArgs a{A, w_hi, w_lo, out, M, K, N, ld_a, ld_out, kpad, ed};
  const int bn = pointwise_tc_tile_n(N);
  if (npad % bn != 0) return false;
  bool ok = false;
  if (tuning().tc_variant == 2) {
    switch (bn) {
      case 16: ok = launch_tc2_bn<16>(s, M, K, N, A, ld_a, w_hi, w_lo, kpad, npad, out, ld_out, ed); break;
      case 32: ok = launch_tc2_bn<32>(s, M, K, N, A, ld_a, w_hi, w_lo, kpad, npad, out, ld_out, ed); break;
      case 64: ok = launch_tc2_bn<64>(s, M, K, N, A, ld_a, w_hi, w_lo, kpad, npad, out, ld_out, ed); break;
      case 80: ok = launch_tc2_bn<80>(s, M, K, N, A, ld_a, w_hi, w_lo, kpad, npad, out, ld_out, ed); break;
      case 96: ok = launch_tc2_bn<96>(s, M, K, N, A, ld_a, w_hi, w_lo, kpad, npad, out, ld_out, ed); break;
      case 128: ok = launch_tc2_bn<128>(s, M, K, N, A, ld_a, w_hi, w_lo, kpad, npad, out, ld_out, ed); break;
      default: return false;
    }
    if (!ok) return false;
    count_launch();
    return true;
  }
  switch (bn) {
    case 16: ok = launch_tc_bn<16>(s, a, npad); break;
    case 32: ok = launch_tc_bn<32>(s, a, npad); break;
    case 64: ok = launch_tc_bn<64>(s, a, npad); break;
    case 80: ok = launch_tc_bn<80>(s, a, npad); break;
    case 96: ok = launch_tc_bn<96>(s, a, npad); break;
    case 128: ok = launch_tc_bn<128>(s, a, npad); break;
    default: return false;
  }
  if (!ok) return false;          // the caller falls back to the exact FFMA kernel
  count_launch();
  return true;
}

#else   // BSB_EMU: wgmma cannot be emulated; the emulator build never selects this path

int pointwise_tc_tile_n(int) { return 0; }
bool launch_pointwise_tc(cudaStream_t, int, int, int, const float*, int, const float*, const float*, int, int, float*, int, const Epilogue&) { return false; }

#endif

}  // namespace bsb
