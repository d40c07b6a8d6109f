// backscrub_b200/csrc/post_math.h — per-thread arithmetic of the fused post stage (mask = (S + 12) / 25, alpha blend,
// RGB -> YUV, YUYV -> BGR), shared by k_post_fast (kernels_img.cu) and the TMA-staged k_post_tma (kernels_post.cu).
// Everything here is exact integer arithmetic restating OpenCV / app/deepseg.cc:87-134 (see oracle/oracle_img.c).
#pragma once
#include "kernels.h"

namespace bsb {

constexpr int PF_W = 128, PF_H = 32, PF_PX = 16;
constexpr int PF_UW = PF_W + 4, PF_UH = PF_H + 4, PF_US = 136, PF_RMAX = 40, PF_PS = 144;

BSB_D uint4 ldg_stream(const uint8_t* p) {
#if defined(BSB_EMU)
  return *reinterpret_cast<const uint4*>(p);
#else
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
#endif
}
BSB_D void prefetch_l2(const uint8_t* p) {
#if !defined(BSB_EMU)
  asm volatile("prefetch.global.L2 [%0];" :: "l"(p));
  asm volatile("prefetch.global.L2 [%0];" :: "l"(p + 32));
#else
  (void)p;
#endif
}
BSB_D void stg_stream(uint8_t* p, uint4 v) {
#if defined(BSB_EMU)
  *reinterpret_cast<uint4*>(p) = v;
#else
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#endif
}


// one pixel: pair channels (two 16-bit lanes) + single channel; returns T = (c0, c1, c2, x) bytes
template <int PAIR_SEL, int SINGLE_SEL, int T_SEL>
BSB_D unsigned blend_px(unsigned g_pair_w, unsigned f_pair_w, unsigned g_single_w, unsigned f_single_w, unsigned m) {
  const unsigned nm = 255u - m;
  const unsigned gp = __byte_perm(g_pair_w, 0u, PAIR_SEL), fp = __byte_perm(f_pair_w, 0u, PAIR_SEL);
  const unsigned x = gp * m + fp * nm;                                   // two lanes, each <= 65025
  const unsigned y = x + __byte_perm(x, 0u, 0x4341) + 0x00010001u;       // (x + 1 + (x >> 8)) per lane; result in bytes 1, 3
  const unsigned sw = __byte_perm(g_single_w, f_single_w, SINGLE_SEL);   // (g, f, g, f)
  const unsigned xs = __dp4a(sw, m | (nm << 8), 0u);                     // g*m + f*(255-m)
  const unsigned ys = xs + 1u + (xs >> 8);                               // result in byte 1
  return __byte_perm(y, ys, T_SEL);
}


// cv::cvtColor(COLOR_YUV2BGR_YUYV) on 8 pixels: w = 4 words of (Y0 U Y1 V) -> o = 24 bytes of BGR (6 words).
// BT.601 limited range, 20-bit fixed point (oracle_img.c:or_yuyv_to_bgr, pinned on cv2).
BSB_D void yuyv8_to_bgr24(const unsigned* w, unsigned* o) {
  // saturate with one VIMNMX.RELU per channel (min(v, 255) then max(.., 0)); the 24 bytes
  // are assembled with byte permutes (pixel = b | g << 8 | r << 16, then three words per four pixels)
  // All the constant terms are folded so that every channel is ONE multiply-add from the raw bytes:
  //   C (Y' - 16) + K (X - 128) + 2^19  ==  C max(Y, 16) + K X + (2^19 - 128 K - 16 C)      (exact in int32: |.| < 2^30)
  constexpr int CY = 1220542, KRV = 1673527, KGV = -852492, KGU = -409993, KBU = 2116026;
  constexpr int CR = (1 << 19) - 128 * KRV - 16 * CY, CG = (1 << 19) - 128 * (KGV + KGU) - 16 * CY, CB = (1 << 19) - 128 * KBU - 16 * CY;
  unsigned px[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int u = (int)__byte_perm(w[k], 0u, 0x4441), v = (int)(w[k] >> 24);
    const int ruv = KRV * v + CR, guv = KGV * v + (KGU * u + CG), buv = KBU * u + CB;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int yc = max((int)__byte_perm(w[k], 0u, h ? 0x4442 : 0x4440), 16);
      const unsigned bb = (unsigned)__vimin_s32_relu((CY * yc + buv) >> 20, 255), gg = (unsigned)__vimin_s32_relu((CY * yc + guv) >> 20, 255),
                     rr = (unsigned)__vimin_s32_relu((CY * yc + ruv) >> 20, 255);
      px[2 * k + h] = __byte_perm(__byte_perm(bb, gg, 0x0040), rr, 0x0410);      // b | g << 8 | r << 16
    }
  }
#pragma unroll
  for (int q = 0; q < 2; ++q) {        // four pixels (b0 g0 r0 | b1 g1 r1 | b2 g2 r2 | b3 g3 r3) -> three words
    const unsigned p0 = px[4 * q], p1 = px[4 * q + 1], p2 = px[4 * q + 2], p3 = px[4 * q + 3];
    o[3 * q] = __byte_perm(p0, p1, 0x4210);          // b0 g0 r0 b1
    o[3 * q + 1] = __byte_perm(p1, p2, 0x5421);      // g1 r1 b2 g2
    o[3 * q + 2] = __byte_perm(p2, p3, 0x6542);      // r2 b3 g3 r3
  }
}
BSB_D void rgb2yuv(int R, int G, int Bc, int& Y, int& U, int& V) {
  // cv::cvtColor(COLOR_RGB2YUV) 8-bit, 14-bit fixed point (oracle_img.c:or_rgb2yuv_u8)
  Y = (4899 * R + 9617 * G + 1868 * Bc + 8192) >> 14;
  U = ((Bc - Y) * 8061 + (128 << 14) + 8192) >> 14;
  V = ((R - Y) * 14369 + (128 << 14) + 8192) >> 14;
  Y = Y > 255 ? 255 : Y;
  U = U < 0 ? 0 : (U > 255 ? 255 : U);
  V = V < 0 ? 0 : (V > 255 ? 255 : V);
}
// convert_rgb_to_yuyv of one pixel pair (two 3-byte BGR pixels) as the word (Y0, V, Y1, U) (app/deepseg.cc:87-106)
BSB_D unsigned yuyv_pair_word(const uint8_t* p0, const uint8_t* p1) {
  int Y0, U0, V0, Y1, U1, V1;
  rgb2yuv(p0[0], p0[1], p0[2], Y0, U0, V0);
  rgb2yuv(p1[0], p1[1], p1[2], Y1, U1, V1);
  return (unsigned)Y0 | ((unsigned)((V0 + V1) / 2) << 8) | ((unsigned)Y1 << 16) | ((unsigned)((U0 + U1) / 2) << 24);
}
BSB_D unsigned yuyv_pair_word(const uint8_t* s) { return yuyv_pair_word(s, s + 3); }
// the NV12 of one 2x2 block from the YUYV words of its two rows (W bytes apart in the Y plane): Y copied, UV the
// truncating row-pair average (include/backscrub_b200.h)
BSB_D void nv12_block(unsigned w0, unsigned w1, uint8_t* y0, int W, uint8_t* uv) {
  y0[0] = (uint8_t)w0; y0[1] = (uint8_t)(w0 >> 16); y0[W] = (uint8_t)w1; y0[W + 1] = (uint8_t)(w1 >> 16);
  uv[0] = (uint8_t)((((w0 >> 8) & 255u) + ((w1 >> 8) & 255u)) >> 1);
  uv[1] = (uint8_t)(((w0 >> 24) + (w1 >> 24)) >> 1);
}

// one pixel from its Y byte and the U / V bytes it shares (the arithmetic of yuyv8_to_bgr24)
BSB_D void yuv_px_to_bgr(int y, int u8, int v8, int* bgr) {
  const int u = u8 - 128, v = v8 - 128;
  const int yy = max(y - 16, 0) * 1220542;
  bgr[0] = bsb_sat_u8((yy + (1 << 19) + 2116026 * u) >> 20);
  bgr[1] = bsb_sat_u8((yy + (1 << 19) - 852492 * v - 409993 * u) >> 20);
  bgr[2] = bsb_sat_u8((yy + (1 << 19) + 1673527 * v) >> 20);
}
// one pixel of a YUYV row: BGR of pixel x (the pair's U / V are shared)
BSB_D void yuyv_px_to_bgr(const uint8_t* row, int x, int* bgr) {
  const uint8_t* q = row + (size_t)(x & ~1) * 2;
  yuv_px_to_bgr((int)q[(x & 1) * 2], (int)q[1], (int)q[3], bgr);
}
// one pixel of an NV12 frame (Y plane rows `pitch` bytes apart, UV plane at byte `uv_off`): pixel (x, y) takes the UV pair
// of its 2x2 block.  cv::cvtColor(COLOR_YUV2BGR_NV12) equals COLOR_YUV2BGR_YUYV on the YUYV frame built that way.
BSB_D void nv12_px_to_bgr(const uint8_t* img, size_t pitch, size_t uv_off, int x, int y, int* bgr) {
  const uint8_t* q = img + uv_off + (size_t)(y >> 1) * pitch + (size_t)(x & ~1);
  yuv_px_to_bgr((int)img[(size_t)y * pitch + x], (int)q[0], (int)q[1], bgr);
}

// 16 mask values of one thread from the vertical 5-sums `vrow` (packed u16, the thread's first column), or from the
// tile constant; 255 outside the ROI.
BSB_D void post_mask16(const PostArgs& a, bool row_in, int tile_const, int x0, const unsigned short* vrow, unsigned* m) {
  if (row_in && tile_const >= 0) {
#pragma unroll
    for (int i = 0; i < PF_PX; ++i) m[i] = (unsigned)tile_const;
    if (x0 < a.roi_x || x0 + PF_PX > a.roi_x + a.roi_w) {
#pragma unroll
      for (int i = 0; i < PF_PX; ++i) if (x0 + i < a.roi_x || x0 + i >= a.roi_x + a.roi_w) m[i] = 255u;
    }
  } else if (row_in) {
    const uint4* vq = reinterpret_cast<const uint4*>(vrow);
    const uint4 q0 = vq[0], q1 = vq[1];
    const uint2 q2 = *reinterpret_cast<const uint2*>(vq + 2);
    const unsigned w[10] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y};
    unsigned c[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) c[k] = __byte_perm(w[k], w[k + 1], 0x5432);
#pragma unroll
    for (int k = 1; k <= 8; ++k) {
      const unsigned s = w[k - 1] + w[k] + w[k + 1] + c[k - 1] + c[k];
      m[2 * (k - 1)] = ((s & 0xffffu) * 5243u + 62916u) >> 17;          // (S + 12) / 25
      m[2 * (k - 1) + 1] = ((s >> 16) * 5243u + 62916u) >> 17;
    }
    if (x0 < a.roi_x || x0 + PF_PX > a.roi_x + a.roi_w) {
#pragma unroll
      for (int i = 0; i < PF_PX; ++i) if (x0 + i < a.roi_x || x0 + i >= a.roi_x + a.roi_w) m[i] = 255u;
    }
  } else {
#pragma unroll
    for (int i = 0; i < PF_PX; ++i) m[i] = 255u;
  }

}

// the blend weight of a pixel with mask m: m, or 0 when its frame's filter is off (PostArgs::pass), so that alpha_blend
// returns the camera byte exactly ((f * 255) / 255 == f) and post_blend16 takes its all-person path.  The stored mask
// is m either way.
BSB_D unsigned blend_weight(bool pass, unsigned m) { return pass ? 0u : m; }

// the transparent output (PostArgs::bgra) of 4 pixels from their blend weights w (blend_weight): the camera bytes f (3 words
// of BGR) with alpha 255 - w, i.e. 255 - mask (the person matte), or 255 when the frame's filter is off -> 4 BGRA words.
// rev: in reversed pixel order (a mirrored frame).
BSB_D uint4 bgra4(const unsigned* f, const unsigned* w, bool rev) {
  const unsigned A = f[0], B = f[1], C = f[2];                          // b0 g0 r0 b1 | g1 r1 b2 g2 | r2 b3 g3 r3
  const unsigned p0 = __byte_perm(A, 255u - w[0], 0x4210);
  const unsigned p1 = __byte_perm(__byte_perm(A, B, 0x0543), 255u - w[1], 0x4210);
  const unsigned p2 = __byte_perm(__byte_perm(B, C, 0x0432), 255u - w[2], 0x4210);
  const unsigned p3 = __byte_perm(C >> 8, 255u - w[3], 0x4210);
  return rev ? make_uint4(p3, p2, p1, p0) : make_uint4(p0, p1, p2, p3);
}

// 16 pixels: f / g = frame / background bytes (12 words each), m = masks; o = blended BGR (12 words), yy = YUYV (8 words)
template <bool OUT, bool YUYV>
BSB_D void post_blend16(const unsigned* f, const unsigned* g, const unsigned* m, unsigned* o, unsigned* yy) {
  // ---- D: blend, 4 pixels = 3 words at a time.  Most 16-pixel runs are entirely background
  //      (mask 255 -> out = bg) or entirely person (mask 0 -> out = frame): those skip the arithmetic. ----
  unsigned m_and = m[0], m_or = m[0];
#pragma unroll
  for (int i = 1; i < PF_PX; ++i) { m_and &= m[i]; m_or |= m[i]; }
  const bool all_bg = m_and == 255u, all_fg = m_or == 0u;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const unsigned fA = f[3 * q], fB = f[3 * q + 1], fC = f[3 * q + 2];
    const unsigned gA = g[3 * q], gB = g[3 * q + 1], gC = g[3 * q + 2];
    // T = (c0, c1, c2, -) per pixel
    unsigned T0, T1, T2, T3;
    if (all_bg || all_fg) {
      const unsigned sA = all_bg ? gA : fA, sB = all_bg ? gB : fB, sC = all_bg ? gC : fC;
      T0 = sA; T1 = __byte_perm(sA, sB, 0x0543); T2 = __byte_perm(sB, sC, 0x0432); T3 = sC >> 8;
      if (OUT) { o[3 * q] = sA; o[3 * q + 1] = sB; o[3 * q + 2] = sC; }
    } else {
      T0 = blend_px<0x4140, 0x6262, 0x0531>(gA, fA, gA, fA, m[4 * q]);          // A.b0 A.b1 | A.b2
      T1 = blend_px<0x4140, 0x7373, 0x0315>(gB, fB, gA, fA, m[4 * q + 1]);      // B.b0 B.b1 | A.b3 (c0)
      T2 = blend_px<0x4342, 0x4040, 0x0531>(gB, fB, gC, fC, m[4 * q + 2]);      // B.b2 B.b3 | C.b0
      T3 = blend_px<0x4241, 0x7373, 0x0531>(gC, fC, gC, fC, m[4 * q + 3]);      // C.b1 C.b2 | C.b3
      if (OUT) {
        o[3 * q] = __byte_perm(T0, T1, 0x4210);
        o[3 * q + 1] = __byte_perm(T1, T2, 0x5421);
        o[3 * q + 2] = __byte_perm(T2, T3, 0x6542);
      }
    }
    if (YUYV) {
      const unsigned T[4] = {T0, T1, T2, T3};
      unsigned Y[4], U[4]; int V[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const unsigned y14 = __dp2a_hi(1868u, T[j], __dp2a_lo(4899u | (9617u << 16), T[j], 8192u));
        Y[j] = y14 >> 14;
        U[j] = __dp2a_hi(8061u, T[j], 2105344u - 8061u * Y[j]) >> 14;
        V[j] = (int)__dp2a_lo(14369u, T[j], 2105344u - 14369u * Y[j]) >> 14;
        V[j] = __vimin_s32_relu(V[j], 255);
      }
      yy[2 * q] = Y[0] | ((unsigned)((V[0] + V[1]) >> 1) << 8) | (Y[1] << 16) | (((U[0] + U[1]) >> 1) << 24);
      yy[2 * q + 1] = Y[2] | ((unsigned)((V[2] + V[3]) >> 1) << 8) | (Y[3] << 16) | (((U[2] + U[3]) >> 1) << 24);
    }
  }
}

}  // namespace bsb
