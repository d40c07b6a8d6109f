// backscrub_b200/csrc/bsb_common.h — shared definitions for the CUDA hot path.
//
// Compiled by nvcc for sm_90a (the product).  With -DBSB_EMU the same sources are
// compiled by g++ against tests/emu/cuemu.h, a kernel-logic emulator used ONLY by the
// CPU-side unit tests; the product library never contains that build.
#pragma once

#include <cmath>
#include <cstddef>
#include <cstdint>

#ifdef BSB_EMU
#include "cuemu.h"
#else
#include <cuda_runtime.h>
#define BSB_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define BSB_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

#define BSB_HD __host__ __device__ __forceinline__
#define BSB_D __device__ __forceinline__
#ifdef BSB_EMU
#define BSB_D_NOINLINE __attribute__((noinline))
#else
#define BSB_D_NOINLINE __device__ __noinline__
#endif

namespace bsb {

// Activation / epilogue codes.  0..3 are TFLite's fused-activation enum
// (schema.fbs ActivationFunctionType :512), the rest are stand-alone unary ops that the
// planner folds into the producing kernel.
enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_RELU_N1_TO_1 = 2, ACT_RELU6 = 3, ACT_HARD_SWISH = 4, ACT_LOGISTIC = 5 };

enum ModelType : int { MODEL_UNKNOWN = 0, MODEL_BODYPIX = 1, MODEL_DEEPLAB = 2, MODEL_MEET = 3, MODEL_MLKIT = 4 };

// ---------------------------------------------------------------------------
// Numeric contract (identical, operation for operation, in oracle/oracle_nn.c):
//   * every multiply-accumulate is ONE fused fmaf in the reference loop order;
//   * no implicit contraction anywhere else (nvcc -fmad=false / g++ -ffp-contract=off);
//   * exp is the fixed polynomial bsb_expf below; divisions are IEEE (-prec-div=true);
//   * denormals flush to zero (-ftz=true), as TFLite's Invoke runs under FTZ/DAZ
//     (reference tensorflow/lite/interpreter.cc:226).
// ---------------------------------------------------------------------------

BSB_HD float bsb_bits_to_float(int i) {
#if defined(__CUDA_ARCH__)
  return __int_as_float(i);
#else
  union { int i; float f; } u; u.i = i; return u.f;
#endif
}

// IEEE-754 round-to-nearest division.  Spelled out because nvcc -ftz=true strength-reduces
// `x / constant` into `x * (1/constant)` even with -prec-div=true (seen in SASS as
// FMUL.FTZ by 0.16666667), which is not the correctly rounded quotient the oracle computes.
BSB_HD float bsb_div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// exp(x): Cody-Waite reduction by ln2 (2 constants), degree-5 Horner polynomial in fmaf
// form (Cephes expf coefficients), exact two-step power-of-two scaling.  Stands in for
// std::exp in reference logistic.h:30-57 and expf in lib/libbackscrub.cc:350-351.
BSB_HD float bsb_expf(float x) {
  if (x != x) return x;
  if (x > 88.7228394f) return bsb_bits_to_float(0x7f800000);
  if (x < -87.3365479f) return 0.0f;
  float n = rintf(x * 1.44269504088896341f);
  float r = fmaf(n, -0.693359375f, x);
  r = fmaf(n, 2.12194440e-4f, r);
  float p = 1.9875691500E-4f;
  p = fmaf(p, r, 1.3981999507E-3f);
  p = fmaf(p, r, 8.3334519073E-3f);
  p = fmaf(p, r, 4.1665795894E-2f);
  p = fmaf(p, r, 1.6666665459E-1f);
  p = fmaf(p, r, 5.0000001201E-1f);
  float r2 = r * r;
  float y = fmaf(p, r2, r);
  y = y + 1.0f;
  int ni = (int)n;
  int n1 = ni / 2, n2 = ni - n1;
  float s1 = bsb_bits_to_float((n1 + 127) << 23);
  float s2 = bsb_bits_to_float((n2 + 127) << 23);
  return (y * s1) * s2;
}

// reference logistic.h:30-57 (cut-offs included)
BSB_HD float bsb_logistic(float v) {
  if (v > 16.619047164916992188f) return 1.0f;
  if (v < -9.f) return bsb_expf(v);
  return bsb_div(1.f, 1.f + bsb_expf(-v));
}

// v / 6, correctly rounded (the bits of bsb_div(v, 6.f) under FTZ / DAZ), without the IEEE divide subroutine: the
// product by RN(1/6) is within one ulp of the quotient, its residual v - 6q is exact in one fmaf, and one correction
// step rounds to nearest.  The residual of a tiny v would be flushed, the product sends -0 to +0 and +-inf to NaN, so
// non-finite v and nonzero |v| < 2^-100 take the division; zero (hard-swish of x <= -3) stays on the fast path and
// copysignf restores its sign.  tests/test_chain_overhead.py compares every float32 bit pattern against the division,
// on the CPU under FTZ + DAZ and on the GPU against __fdiv_rn.
BSB_HD float bsb_div6(float v) {
  const float a = fabsf(v);
  if (!((a >= 0x1p-100f && a <= 0x1.fffffep127f) || v == 0.f)) return bsb_div(v, 6.f);
  const float q = v * 0x1.555556p-3f;             // RN(1/6)
  const float r = fmaf(-q, 6.f, v);
  return copysignf(fmaf(r, 0x1.555556p-3f, q), v);
}

// reference hard_swish.h:45-56: x * min(6, max(0, x + 3)) / 6
BSB_HD float bsb_hard_swish(float x) {
  float t = x + 3.f;
  t = t < 0.f ? 0.f : t;
  t = t > 6.f ? 6.f : t;
#if defined(__CUDA_ARCH__)
  return bsb_div6(x * t);
#else
  return bsb_div(x * t, 6.f);
#endif
}

BSB_HD float bsb_act(float x, int act) {
  switch (act) {
    case ACT_RELU: return x < 0.f ? 0.f : x;
    case ACT_RELU6: { float y = x < 0.f ? 0.f : x; return y > 6.f ? 6.f : y; }
    case ACT_RELU_N1_TO_1: { float y = x < -1.f ? -1.f : x; return y > 1.f ? 1.f : y; }
    case ACT_HARD_SWISH: return bsb_hard_swish(x);
    case ACT_LOGISTIC: return bsb_logistic(x);
    default: return x;
  }
}

// x / 255 for 0 <= x <= 255*255 without a division (tests/test_oracle_img.py proves the identity)
BSB_HD unsigned bsb_div255(unsigned x) { return (x + 1u + (x >> 8)) >> 8; }

// cvRound(S * (1.0/25)) for the 5x5 box sum S of u8 values == (S + 12) / 25
BSB_HD unsigned bsb_box25(unsigned s) { return (s + 12u) / 25u; }

BSB_HD int bsb_reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) { p = p < 0 ? -p : 2 * n - 2 - p; }
  return p;
}

BSB_HD unsigned char bsb_sat_u8(int v) { return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

}  // namespace bsb
