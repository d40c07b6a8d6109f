// backscrub_b200/csrc/kernels_post.cu — TMA-staged variant of the fused post stage (sm_90a).
//
// Same stage as k_post_fast (kernels_img.cu): mask upsample (cv::resize 8UC1) + cv::blur 5x5 inside the ROI
// (lib/libbackscrub.cc:366-371), alpha_blend (app/deepseg.cc:108-134), convert_rgb_to_yuyv (:87-106), mask store —
// reorganised around the copy engine:
//   * every global access of the tile is a TMA bulk tensor copy (cp.async.bulk.tensor, SASS UTMALDG / UTMASTG)
//     between global memory and shared memory, issued by one thread: no per-thread address arithmetic, no
//     sector bookkeeping, image edges clipped by the tensor map;
//   * the source patch of the small mask arrives first; if it is uniformly 255 (background) or 0 (person) — exact
//     for any interpolation weights, see k_post_fast — the tile needs NO per-pixel arithmetic on the copy path:
//       background tile:  out <- background tile, YUYV <- cached YUYV of the background, mask <- 255
//                         (the camera frame is not even read),
//       person tile:      out <- frame tile (camera YUYV converted per thread when the frames are in wire format),
//       mixed tile:       the k_post_fast arithmetic on shared-memory operands;
//   * results are staged in shared memory and leave with TMA stores;
//   * a frame with a flip code (PostArgs::flip, sources calls) is written mirrored: each thread puts its 16 pixels,
//     reversed, into the mirrored slot of the staging tiles, and the stores go to the mirrored box;
//   * a frame whose filter is off (PostArgs::pass) loads no background: every tile loads the camera tile and takes the
//     person-tile path, and the mask patch is loaded and classified only when the call stores the mask;
//   * a launch with the transparent output (PostArgs::bgra) loads the camera tile of every tile, and background tiles
//     take the mixed-tile path (the blend of mask 255 is the background, bit for bit); each thread writes its 16 BGRA
//     pixels (camera bytes, alpha 255 - mask) with 16-byte stores straight from registers, mirrored in place for a
//     flipped frame.  Without a composite or video output it loads no background at all;
//   * a launch with a refinement table (PostArgs::refine) loads, for a refined frame, the patch of the small mask its
//     refinement reaches (geo_r_*); a mixed tile gathers the guide luma of every patch entry from the camera frame in its
//     wire format, takes the frame's range row into shared memory and computes each pixel's mask from the camera tile
//     (post_math.h refine_mask16) instead of the resize + blur passes.  Uniform tiles keep their copy path.
// Arithmetic is shared with k_post_fast through post_math.h, so both kernels produce the oracle's bits.
#include "kernels.h"
#include "post_math.h"

#include <type_traits>

#ifndef BSB_EMU
#include <cuda.h>   // CUtensorMap types only; cuTensorMapEncodeTiled is resolved at run time (no libcuda link)
#endif

namespace bsb {

void count_launch();

#ifndef BSB_EMU

namespace tma {
BSB_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
BSB_D void mbar_init(uint64_t* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory"); }
BSB_D void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
BSB_D void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
BSB_D bool mbar_try_wait(uint64_t* bar, unsigned parity) {
  unsigned ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
BSB_D void mbar_wait(uint64_t* bar, unsigned parity) { while (!mbar_try_wait(bar, parity)) {} }
BSB_D void load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
BSB_D void store_3d(const CUtensorMap* map, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               :: "l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
BSB_D void store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
BSB_D void store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
BSB_D void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
BSB_D void prefetch_map(const CUtensorMap* map) { asm volatile("prefetch.tensormap [%0];" :: "l"(map) : "memory"); }
}  // namespace tma

// 16 pixels in reversed order: BGR (12 words; four groups of 4 pixels = 3 words, each group's pixels reversed), YUYV
// (8 words of 2 pixels: word order reversed, Y0 / Y1 swapped; a pair's U / V are a symmetric average and stay), 16 Y
// bytes, 4 UV pairs (2-byte units)
BSB_D void rev_bgr16(const unsigned* s, unsigned* d) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const unsigned A = s[3 * (3 - q)], B = s[3 * (3 - q) + 1], C = s[3 * (3 - q) + 2];   // p0 p0 p0 p1 | p1 p1 p2 p2 | p2 p3 p3 p3
    d[3 * q] = __byte_perm(C, B, 0x6321);
    d[3 * q + 1] = __byte_perm(__byte_perm(B, C, 0x0043), A, 0x3710);
    d[3 * q + 2] = __byte_perm(A, B, 0x2105);
  }
}
BSB_D void rev_yuyv16(const unsigned* s, unsigned* d) {
#pragma unroll
  for (int j = 0; j < 8; ++j) d[j] = __byte_perm(s[7 - j], 0, 0x3012);
}
BSB_D uint4 rev_y16(uint4 v) {
  return make_uint4(__byte_perm(v.w, 0, 0x0123), __byte_perm(v.z, 0, 0x0123), __byte_perm(v.y, 0, 0x0123), __byte_perm(v.x, 0, 0x0123));
}
BSB_D uint2 rev_uv4(uint2 v) { return make_uint2(__byte_perm(v.y, 0, 0x1032), __byte_perm(v.x, 0, 0x1032)); }

// A staged tile of `rows` rows of RB bytes whose box starts at byte column gx / row gy of a frame with fb-byte rows
// (`pitch` apart) and fh rows, stored by every thread with 16-byte stores, clipped to the frame.  Mirrored boxes of ragged
// edge tiles start at negative coordinates, which the TMA store does not take; gx and fb are multiples of 16.
template <int NT, int RB>
BSB_D void store_clipped(const uint8_t* src, int rows, uint8_t* dst, size_t pitch, int gx, int gy, int fb, int fh, int tid) {
  constexpr int CPR = RB / 16;                       // 16-byte chunks per row
  for (int i = tid; i < rows * CPR; i += NT) {
    const int r = i / CPR, c = (i % CPR) * 16, x = gx + c, y = gy + r;
    if (x >= 0 && x < fb && y >= 0 && y < fh)
      *reinterpret_cast<uint4*>(dst + (size_t)y * pitch + x) = *reinterpret_cast<const uint4*>(src + r * RB + c);
  }
}

struct PostMaps { CUtensorMap frame, bg, bgy, out, yuyv, mask, ofinal; };
// NV12 calls: frame / bgy / yuyv are the Y planes of the camera frames, the background NV12 and the NV12 output; these are
// their UV planes
struct PostMapsNv12 : PostMaps { CUtensorMap frame_uv, bgy_uv, yuyv_uv; };
template <int FMT> using PostMapsOf = typename std::conditional<FMT == IN_NV12, PostMapsNv12, PostMaps>::type;
// has_yuyv / has_bgy: a video output / a cached background in the call's video format (YUYV, NV12 for NV12 calls)
struct PostTmaCfg { int has_out, has_yuyv, has_mask, has_bgy; };

// Tile geometry.  A CTA owns one TW x 32 tile (TW = 64 or 128), one thread per 16 pixels of a row.
//   * two 128-wide tiles per CTA (95 KB, two CTAs per SM) halve the warp count, which costs more than the amortised load
//     latency saves;
//   * the stage is a dependent chain per CTA (patch -> classify -> tiles -> arithmetic -> stores), so what hides latency
//     is the number of independent chains per SM: a 64-wide tile needs ~27 KB and 128 threads, eight CTAs per SM instead
//     of four with the same number of resident warps (tuning switch post_tile).
// The patch of the small mask a (TW + 4) x 36 halo tile can touch has <= PT_RMAX rows and <= PCOLS columns (up-scales
// >= ~1.75x).  A TMA box must START on a 16-byte boundary of global memory (an unaligned innermost coordinate raises
// "illegal instruction"), so the box begins at the patch's first column rounded down to 16 and is 16 columns wider.
constexpr int PT_RMAX = 24;
template <int TW> struct PtL {
  static constexpr int NT = TW * PF_H / PF_PX;                   // threads
  static constexpr int UW = TW + 4, US = TW + 8;                 // halo tile width, its row stride (u16 elements)
  static constexpr int PCOLS = TW == 128 ? 80 : 48, PW = PCOLS + 16;
  static constexpr int F_BYTES = TW * PF_H * 3, Y_BYTES = TW * PF_H * 2, M_BYTES = TW * PF_H;
  static constexpr int OFF_F = 0, OFF_B = F_BYTES, OFF_Y = 2 * F_BYTES, OFF_P = 2 * F_BYTES + Y_BYTES;
  static constexpr int OFF_HS = OFF_P + PT_RMAX * PW;            // Hs [PT_RMAX][US] u16, later Vs [PF_H][US] u16
  static constexpr int HV_BYTES = (PT_RMAX > PF_H ? PT_RMAX : PF_H) * US * 2;
  static constexpr int OFF_ROWS = OFF_HS + PT_RMAX * US * 2;     // [PF_UH] uint4 in the part of Vs that Hs does not use
  static constexpr int OFF_US = OFF_HS + HV_BYTES;               // Us [PF_UH][US] u16, later the mask staging tile
  static constexpr int OFF_BAR = OFF_US + PF_UH * US * 2;
  static constexpr int OFF_GEO = OFF_BAR + 32;                   // 12 ints of tile geometry / classification
  static constexpr int SMEM = OFF_GEO + 48;
  static constexpr int CTAS = TW == 128 ? 4 : 8;
  // NV12 calls: the camera tile (Y TW x 32 | UV TW x 16) in the frame tile's place, the background NV12 tile in the YUYV
  // tile's place, and the NV12 result tile staged over Hs / Vs (dead once the mask is computed)
  static constexpr int N_BYTES = TW * PF_H * 3 / 2, OFF_N = OFF_HS;
  static_assert(N_BYTES <= F_BYTES && N_BYTES <= Y_BYTES && N_BYTES <= HV_BYTES && OFF_N % 128 == 0, "NV12 staging");
  static_assert(PW % 16 == 0 && OFF_P % 128 == 0 && OFF_HS % 16 == 0 && OFF_US % 128 == 0 && OFF_ROWS % 16 == 0 && OFF_BAR % 8 == 0 &&
                (PF_H - PT_RMAX) * US * 2 >= PF_UH * 16 && PF_UH * US * 2 >= M_BYTES && US % 8 == 0 && NT % 64 == 0 && NT >= PF_UH &&
                (SMEM + 1024) * CTAS <= 228 * 1024, "smem layout");
};

// FMT: IN_BGR / IN_YUYV frames with YUYV video output, or IN_NV12 frames with NV12 video output.  FLIP: the launch has a
// flip table (sources calls); without one the kernel is compiled without the mirroring paths.  PASS: the launch has a
// filter table; without one the kernel is compiled without the pass-through paths.  BGRA: the launch writes the
// transparent output; without it the kernel is compiled without those paths.  REFINE: the launch has a refinement table;
// without one the kernel is compiled without the refinement.
template <int FMT, int TW, bool FLIP, bool PASS, bool BGRA, bool REFINE>
__global__ void __launch_bounds__(PtL<TW>::NT, PtL<TW>::CTAS) k_post_tma(const __grid_constant__ PostMapsOf<FMT> tm, const PostArgs a, const PostTmaCfg cfg) {
  using L = PtL<TW>;
  constexpr bool IN_YUYV = FMT == InFmt::IN_YUYV, NV12 = FMT == InFmt::IN_NV12;
  constexpr int NT = L::NT, UW = L::UW, US = L::US, PW = L::PW;
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned short* Hs = reinterpret_cast<unsigned short*>(smem + L::OFF_HS);
  unsigned short* Us = reinterpret_cast<unsigned short*>(smem + L::OFF_US);
  unsigned short* Vs = Hs;
  uint4* rows = reinterpret_cast<uint4*>(smem + L::OFF_ROWS);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);      // patch | background (+ its YUYV) | camera tile
  uint8_t* sF = smem + L::OFF_F;          // frame tile [32][3 TW] (BGR) or [32][2 TW] (YUYV); later the blended tile
  uint8_t* sB = smem + L::OFF_B;          // background tile [32][3 TW]
  uint8_t* sY = smem + L::OFF_Y;          // YUYV tile [32][2 TW]: cached background YUYV in, result out
  uint8_t* sM = smem + L::OFF_US;         // mask tile [32][TW] (reuses Us, dead by then)
  uint8_t* sP = smem + L::OFF_P;          // source patch of the small mask [PT_RMAX][PW]
  uint8_t* sN = smem + L::OFF_N;          // NV12 result tile: Y [32][TW] | UV [16][TW] (NV12 calls)
  uint64_t* barP = bars; uint64_t* barB = bars + 1; uint64_t* barF = bars + 2;

  const int b = blockIdx.z;
  const int ty0 = blockIdx.y * PF_H, tx0 = blockIdx.x * TW;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int* geo = reinterpret_cast<int*>(smem + L::OFF_GEO);                 // tile geometry, published by thread 0
  // geo[9]: the frame's flip code, with PASS its filter-off flag in bit 2, with REFINE its refinement strength from bit 8
  auto flip_code = [&]() -> int { return FLIP ? ((PASS || REFINE) ? (geo[9] & 3) : geo[9]) : 0; };
  // a transparent output alone blends nothing: no background tile is loaded or waited for
  const bool bgra_only = BGRA && !cfg.has_out && !cfg.has_yuyv;

  // ---- thread 0: geometry of the tile and ALL the loads, before anybody else does anything.  The geometry is uniform
  //      over the CTA: computing it once and publishing it through shared memory takes ~25 instructions off every other
  //      warp ----
  if (tid == 0) {
    tma::mbar_init(barP, 1); tma::mbar_init(barB, 1); tma::mbar_init(barF, 1);
    tma::fence_barrier_init();
    // a filtered-off frame needs the mask patch only for the mask output
    const bool pass = PASS && __ldg(a.pass + b) != 0;
    const int sig = REFINE ? __ldg(a.refine + b) : 0;
    const bool hit = (!pass || cfg.has_mask) && tx0 < a.roi_x + a.roi_w && tx0 + TW > a.roi_x && ty0 < a.roi_y + a.roi_h && ty0 + PF_H > a.roi_y;
    // the patch of the small mask this tile touches comes from two per-context tables (engine.cu): two independent
    // loads whose addresses need nothing but the block index, then the patch request — the head of the CTA's critical
    // path — goes out first ...
    int gy_lo = 0, gx_lo = 0, rmin = 0, nrows = 0, cmin = 0, ncols = 0, coff = 0;
    if (hit) {
      int2 gr = __ldg(a.geo_rows + blockIdx.y), gc = __ldg((TW == 64 ? a.geo_cols64 : a.geo_cols128) + blockIdx.x);
      if (REFINE) {
        // (both patches are requested at once: the strength selects without a dependent load)
        const int2 rr = __ldg(a.geo_r_rows + blockIdx.y), rc = __ldg((TW == 64 ? a.geo_r_cols64 : a.geo_r_cols128) + blockIdx.x);
        if (sig) { gr = rr; gc = rc; }
      }
      gy_lo = ty0 - a.roi_y - 2; gx_lo = tx0 - a.roi_x - 2;
      rmin = gr.x; nrows = gr.y; cmin = gc.x; ncols = gc.y;
      coff = (a.out_x + cmin) & 15;                     // the patch's first column inside the 16-byte aligned box
      tma::mbar_expect_tx(barP, PT_RMAX * PW);
      tma::load_3d(sP, &tm.ofinal, a.out_x + cmin - coff, a.out_y + rmin, b, barP);
    }
    // ... then the big tiles: the background tile (L2-resident for a still image) and its cached YUYV (a background
    // tile needs nothing else, a mixed tile has its second operand early) ...
    int bgi = 0;
    if (a.bg_index) bgi = __ldg(a.bg_index + b);
    else if (a.bg_cursor) bgi = (int)(((unsigned)__ldg(a.bg_cursor) + (unsigned)b * (unsigned)a.bg_advance) % (unsigned)a.bg_count);
    else if (a.bg_stride) bgi = b;
    if (FLIP) geo[9] = __ldg(a.flip + b);             // the frame's flip code, read by every thread after the first barrier
    if (PASS) geo[9] = (FLIP ? geo[9] : 0) | (pass ? 4 : 0);
    if (REFINE) geo[9] = ((FLIP || PASS) ? geo[9] : 0) | (sig << 8);
    if (!pass && !bgra_only) {                         // (a filtered-off frame arms no background barrier, nor waits on it)
      tma::mbar_expect_tx(barB, (unsigned)L::F_BYTES + (cfg.has_bgy ? (NV12 ? (unsigned)L::N_BYTES : (unsigned)L::Y_BYTES) : 0u));
      tma::load_3d(sB, &tm.bg, blockIdx.x * (TW * 3 / 4), ty0, bgi, barB);
      if constexpr (NV12) {
        if (cfg.has_bgy) {
          tma::load_3d(sY, &tm.bgy, blockIdx.x * (TW / 4), ty0, bgi, barB);
          tma::load_3d(sY + TW * PF_H, &tm.bgy_uv, blockIdx.x * (TW / 4), ty0 / 2, bgi, barB);
        }
      } else {
        if (cfg.has_bgy) tma::load_3d(sY, &tm.bgy, blockIdx.x * (TW / 2), ty0, bgi, barB);
      }
    }
    // ... and the camera tile when the tile can contain a person at all (every tile of a filtered-off frame): waiting for
    // the classification first would put a second memory round trip on the critical path of every person / mixed tile
    if (hit || pass || BGRA) {
      if constexpr (NV12) {
        tma::mbar_expect_tx(barF, (unsigned)L::N_BYTES);
        tma::load_3d(sF, &tm.frame, blockIdx.x * (TW / 4), ty0, b, barF);
        tma::load_3d(sF + TW * PF_H, &tm.frame_uv, blockIdx.x * (TW / 4), ty0 / 2, b, barF);   // ty0 is even (PF_H = 32)
      } else {
        tma::mbar_expect_tx(barF, IN_YUYV ? (unsigned)L::Y_BYTES : (unsigned)L::F_BYTES);
        tma::load_3d(sF, &tm.frame, blockIdx.x * (IN_YUYV ? TW / 2 : TW * 3 / 4), ty0, b, barF);
      }
    }
    const bool inside = tx0 >= a.roi_x && min(tx0 + TW, a.W) <= a.roi_x + a.roi_w && ty0 >= a.roi_y && min(ty0 + PF_H, a.H) <= a.roi_y + a.roi_h;
    *reinterpret_cast<int4*>(geo) = make_int4(hit ? 1 : 0, gy_lo, gx_lo, rmin);
    *reinterpret_cast<int4*>(geo + 4) = make_int4(nrows, cmin, ncols, coff);
    geo[8] = inside ? 1 : 0;
  }
  __syncthreads();
  const int4 g0 = *reinterpret_cast<const int4*>(geo), g1 = *reinterpret_cast<const int4*>(geo + 4);
  const bool hits_roi = g0.x != 0;
  const bool pz = PASS && (geo[9] & 4) != 0;            // the frame's filter is off
  const bool nobg = pz || bgra_only;                     // no background tile was loaded
  const int gy_lo = g0.y, gx_lo = g0.z, rmin = g0.w, nrows = g1.x, cmin = g1.y, ncols = g1.z, coff = g1.w;
  const int sig = REFINE ? (geo[9] >> 8) : 0;            // the frame's refinement strength
  unsigned short* Rs = reinterpret_cast<unsigned short*>(smem + L::OFF_US + L::M_BYTES);   // its range row (refined tiles)

  const int lx = (tid % (TW / PF_PX)) * PF_PX, ly = tid / (TW / PF_PX);
  const int y = ty0 + ly;

  int tile_const = -1, kind = 0;                         // background / person / mixed
  if (hits_roi) {
    if (warp == 0) {
      // warp 0 alone waits for the patch and classifies it: all-255 / all-0 test, one 32-bit word per lane, over the box
      // columns [0, coff + ncols) rounded up to words — a few columns more than the patch.  The classification only
      // selects the code path (the mixed path is always correct), so a conservative test costs nothing in exactness and
      // needs no per-byte masks.
      tma::mbar_wait(barP, 0);
      constexpr int WP2 = PW / 4 <= 16 ? 16 : 32;                      // words per patch row, rounded up to a power of two
      const int wpr = (coff + ncols + 3) >> 2;                         // words per row to look at (<= PW / 4)
      const int wc = lane % WP2;
      bool hi = true, lo = true;
      if (wc < wpr) {
        for (int r = lane / WP2; r < nrows; r += 32 / WP2) {
          const unsigned v = *reinterpret_cast<const unsigned*>(sP + r * PW + wc * 4);
          hi = hi && (v == 0xffffffffu);
          lo = lo && (v == 0u);
        }
      }
      const bool all_hi = __all_sync(0xffffffffu, hi), all_lo = __all_sync(0xffffffffu, lo);
      if (lane == 0) {
        const int tc = all_hi ? 255 : (all_lo ? 0 : -1);
        *reinterpret_cast<int2*>(geo + 10) = make_int2(tc, tc == 255 ? 0 : ((tc == 0 && geo[8]) ? 1 : 2));
      }
    } else if (tid - 32 < PF_UH) {                    // row parameters of the vertical resize pass (used by mixed tiles)
      const int uy = tid - 32;
      int gy = gy_lo + uy;
      gy = gy < 0 ? -gy : gy; gy = gy >= a.roi_h ? 2 * a.roi_h - 2 - gy : gy;     // reflect-101 (single fold)
      gy = min(max(gy, 0), a.roi_h - 1);
      rows[uy] = make_uint4((unsigned)__ldg(a.tab.yofs0 + gy), (unsigned)__ldg(a.tab.yofs1 + gy),
                            (unsigned)(int)__ldg(a.tab.yw + 2 * gy) << 16, (unsigned)(int)__ldg(a.tab.yw + 2 * gy + 1) << 16);
    }
    __syncthreads();
    const int2 tk = *reinterpret_cast<const int2*>(geo + 10);
    tile_const = tk.x; kind = tk.y;
  }

  const bool refined = REFINE && sig && kind == 2 && tile_const < 0;
  if (refined) {
    // ---- R: the refinement patch (mask | guide luma << 8, PCOLS apart) over Hs, the frame's range row after the mask
    //      staging tile.  The guide lumas are gathered from the camera frame in its wire format. ----
    auto px = [&](int x, int yy, int* bgr) {
      if constexpr (NV12) {
        nv12_px_to_bgr(a.nv12_in + (size_t)b * a.nv12_in_stride, a.nv12_in_pitch, a.nv12_in_uv, x, yy, bgr);
      } else if constexpr (IN_YUYV) {
        yuyv_px_to_bgr(a.yuyv_in + (size_t)b * a.yuyv_in_stride + (size_t)yy * a.W * 2, x, bgr);
      } else {
        const uint8_t* p = a.frames + (size_t)b * a.frame_stride + (size_t)yy * a.frame_pitch + (size_t)x * 3;
        bgr[0] = p[0]; bgr[1] = p[1]; bgr[2] = p[2];
      }
    };
    refine_patch(a, sP + coff, PW, rmin, nrows, cmin, ncols, Hs, L::PCOLS, tid, NT, px);
    const unsigned* rw = reinterpret_cast<const unsigned*>(a.refine_w + (size_t)(sig - 1) * 256);
    for (int i = tid; i < 128; i += NT) reinterpret_cast<unsigned*>(Rs)[i] = __ldg(rw + i);
    __syncthreads();
  } else if (kind == 2 && tile_const < 0) {
    // ---- A1: horizontal pass of cv::resize on the patch rows (see k_post_fast) ----
    {
      constexpr int HALF = NT / 2;
      const int phase = tid / HALF;
      for (int ux = tid % HALF; ux < UW; ux += HALF) {
        int gx = gx_lo + ux;
        gx = gx < 0 ? -gx : gx; gx = gx >= a.roi_w ? 2 * a.roi_w - 2 - gx : gx;
        gx = min(max(gx, 0), a.roi_w - 1);
        const uint2 xc = __ldg(a.tab.xcol + gx);
        const int sx = (int)(xc.x & 0xffffu) - cmin + coff, sx1 = (int)(xc.x >> 16) - cmin + coff;
        const int a0 = (int)(short)(xc.y & 0xffffu), a1 = (int)(short)(xc.y >> 16);
        const uint8_t* pr = sP + phase * PW;
        unsigned short* hp = Hs + phase * US + ux;
        for (int r = phase; r < nrows; r += 2) {
          *hp = (unsigned short)(((int)pr[sx] * a0 + (int)pr[sx1] * a1) >> 4);
          pr += 2 * PW; hp += 2 * US;
        }
      }
    }
    __syncthreads();
    // ---- A2: vertical pass -> upsampled tile ----
    for (int uy = warp; uy < PF_UH; uy += NT / 32) {
      const uint4 rp = rows[uy];
      const unsigned short* h0 = Hs + ((int)rp.x - rmin) * US + lane;
      const unsigned short* h1 = Hs + ((int)rp.y - rmin) * US + lane;
      unsigned short* up = Us + uy * US + lane;
#pragma unroll
      for (int k = 0; k < TW / 32; ++k)
        up[32 * k] = (unsigned short)((__umulhi(rp.z, (unsigned)h0[32 * k]) + __umulhi(rp.w, (unsigned)h1[32 * k]) + 2u) >> 2);
      if (lane < UW - TW)
        up[TW] = (unsigned short)((__umulhi(rp.z, (unsigned)h0[TW]) + __umulhi(rp.w, (unsigned)h1[TW]) + 2u) >> 2);
    }
    __syncthreads();
    // ---- B: vertical 5-sums, two columns per word, sliding window over 8 rows (Vs overwrites Hs and the row table) ----
    for (int it = tid; it < (UW / 2) * 4; it += NT) {
      const int pair = it % (UW / 2), seg = it / (UW / 2);
      const unsigned* up = reinterpret_cast<const unsigned*>(Us + (seg * 8) * US) + pair;
      unsigned* vp = reinterpret_cast<unsigned*>(Vs + (seg * 8) * US) + pair;
      unsigned u[12];
#pragma unroll
      for (int k = 0; k < 12; ++k) u[k] = up[k * (US / 2)];
      unsigned v = u[0] + u[1] + u[2] + u[3] + u[4];
      vp[0] = v;
#pragma unroll
      for (int k = 1; k < 8; ++k) { v = v + u[k + 4] - u[k - 1]; vp[k * (US / 2)] = v; }
    }
    __syncthreads();
  }

  const int x0 = tx0 + lx;
  uint4* mdst = reinterpret_cast<uint4*>(sM + ly * TW + lx);
  uint4* ydst = reinterpret_cast<uint4*>(sY + ly * (TW * 2) + lx * 2);
  const uint8_t* out_src = sB;

  // a background tile with a cached YUYV copy is moved by the copy engine alone: only thread 0 (which issues the stores)
  // waits for the background tiles, and for the (speculatively loaded, unused) camera tile after the stores are on their
  // way — shared memory must be quiet when the CTA exits.  A mirrored frame's background tile is reversed by the threads.
  // A filtered-off frame's tiles all take the person-tile path on the camera tile, which every one of them loaded.
  const bool bg_copy = !BGRA && kind == 0 && !pz && !(cfg.has_yuyv && !cfg.has_bgy);
  const bool engine_only = bg_copy && !(FLIP && flip_code());
  if (!engine_only && !nobg) tma::mbar_wait(barB, 0);
  if ((hits_roi && kind != 0) || pz || BGRA) tma::mbar_wait(barF, 0);
  if (!BGRA && kind == 0 && !pz) {
    // ---- background tile: out = background tile, YUYV = cached YUYV tile, mask = 255.  No per-pixel arithmetic ----
    if (cfg.has_mask) *mdst = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    const int fl = flip_code();
    if (fl) {
      // mirrored frame: every thread reads its chunk of the staged tiles (the YUYV converted from the background when
      // there is no cached copy), and after a barrier writes it reversed to the mirrored slot — in place, since every
      // slot is read before any is written
      const int mx = (fl & 1) ? TW - PF_PX - lx : lx, my = (fl & 2) ? PF_H - 1 - ly : ly;
      const int ur = tid / (TW / 8), uq = tid % (TW / 8);            // NV12 UV tile: 8 bytes (4 pairs) per thread
      const uint4* gq = reinterpret_cast<const uint4*>(sB + ly * (TW * 3) + lx * 3);
      const uint4 g0 = gq[0], g1 = gq[1], g2 = gq[2];
      unsigned gg[12] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w, g2.x, g2.y, g2.z, g2.w};
      unsigned yy[8];
      if (cfg.has_yuyv && !cfg.has_bgy) {
        unsigned m[PF_PX], o[12];
#pragma unroll
        for (int i = 0; i < PF_PX; ++i) m[i] = 255u;
        post_blend16<false, true>(gg, gg, m, o, yy);
      } else if (NV12) {
        const uint4 yq = *reinterpret_cast<const uint4*>(sY + ly * TW + lx);
        const uint2 cq = *reinterpret_cast<const uint2*>(sY + TW * PF_H + ur * TW + 8 * uq);
        yy[0] = yq.x; yy[1] = yq.y; yy[2] = yq.z; yy[3] = yq.w; yy[4] = cq.x; yy[5] = cq.y;
      } else {
        const uint4 y0 = ydst[0], y1 = ydst[1];
        yy[0] = y0.x; yy[1] = y0.y; yy[2] = y0.z; yy[3] = y0.w; yy[4] = y1.x; yy[5] = y1.y; yy[6] = y1.z; yy[7] = y1.w;
      }
      __syncthreads();
      if (cfg.has_out) {
        unsigned r[12];
        if (fl & 1) rev_bgr16(gg, r);
        else {
#pragma unroll
          for (int i = 0; i < 12; ++i) r[i] = gg[i];
        }
        uint4* bq = reinterpret_cast<uint4*>(sB + my * (TW * 3) + mx * 3);
        bq[0] = make_uint4(r[0], r[1], r[2], r[3]); bq[1] = make_uint4(r[4], r[5], r[6], r[7]); bq[2] = make_uint4(r[8], r[9], r[10], r[11]);
      }
      if (cfg.has_yuyv) {
        if (NV12 && cfg.has_bgy) {
          const uint4 yq = make_uint4(yy[0], yy[1], yy[2], yy[3]);
          const uint2 cq = make_uint2(yy[4], yy[5]);
          *reinterpret_cast<uint4*>(sY + my * TW + mx) = (fl & 1) ? rev_y16(yq) : yq;
          *reinterpret_cast<uint2*>(sY + TW * PF_H + ((fl & 2) ? PF_H / 2 - 1 - ur : ur) * TW + ((fl & 1) ? TW - 8 - 8 * uq : 8 * uq)) =
              (fl & 1) ? rev_uv4(cq) : cq;
        } else {
          unsigned r[8];
          if (fl & 1) rev_yuyv16(yy, r);
          else {
#pragma unroll
            for (int i = 0; i < 8; ++i) r[i] = yy[i];
          }
          uint4* yq = reinterpret_cast<uint4*>(sY + my * (TW * 2) + mx * 2);
          yq[0] = make_uint4(r[0], r[1], r[2], r[3]); yq[1] = make_uint4(r[4], r[5], r[6], r[7]);
        }
      }
    } else if (cfg.has_yuyv && !cfg.has_bgy) {
      const uint4* gq = reinterpret_cast<const uint4*>(sB + ly * (TW * 3) + lx * 3);
      const uint4 g0 = gq[0], g1 = gq[1], g2 = gq[2];
      const unsigned gg[12] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w, g2.x, g2.y, g2.z, g2.w};
      unsigned m[PF_PX], o[12], yy[8];
#pragma unroll
      for (int i = 0; i < PF_PX; ++i) m[i] = 255u;
      post_blend16<false, true>(gg, gg, m, o, yy);
      ydst[0] = make_uint4(yy[0], yy[1], yy[2], yy[3]); ydst[1] = make_uint4(yy[4], yy[5], yy[6], yy[7]);
    }
  } else {
    // (a filtered-off frame: the mask of any kind of tile, computed only when it is stored; outside the ROI it is 255)
    unsigned m[PF_PX];
    if (kind == 1) {
#pragma unroll
      for (int i = 0; i < PF_PX; ++i) m[i] = 0u;
    } else if (!pz || cfg.has_mask) {
      // (a refined tile's values are replaced below, once its camera bytes are known)
      const bool row_in = (!(PASS || BGRA) || hits_roi) && y >= a.roi_y && y < a.roi_y + a.roi_h;
      post_mask16(a, row_in, tile_const, x0, Vs + ly * US + lx, m);
    }
    unsigned f[12], gg[12];
    if (NV12) {
      // the thread's 16 Y bytes and the 8 UV pairs of its row pair -> 8 (Y0 U Y1 V) words, then the YUYV arithmetic
      const uint4 yq = *reinterpret_cast<const uint4*>(sF + ly * TW + lx);
      const uint4 cq = *reinterpret_cast<const uint4*>(sF + TW * PF_H + (ly >> 1) * TW + lx);
      const unsigned wa[4] = {__byte_perm(yq.x, cq.x, 0x5140), __byte_perm(yq.x, cq.x, 0x7362), __byte_perm(yq.y, cq.y, 0x5140),
                              __byte_perm(yq.y, cq.y, 0x7362)};
      const unsigned wb[4] = {__byte_perm(yq.z, cq.z, 0x5140), __byte_perm(yq.z, cq.z, 0x7362), __byte_perm(yq.w, cq.w, 0x5140),
                              __byte_perm(yq.w, cq.w, 0x7362)};
      yuyv8_to_bgr24(wa, f); yuyv8_to_bgr24(wb, f + 6);
    } else if (IN_YUYV) {
      const uint4* fq = reinterpret_cast<const uint4*>(sF + ly * (TW * 2) + lx * 2);
      const uint4 w0 = fq[0], w1 = fq[1];
      const unsigned wa[4] = {w0.x, w0.y, w0.z, w0.w}, wb[4] = {w1.x, w1.y, w1.z, w1.w};
      yuyv8_to_bgr24(wa, f); yuyv8_to_bgr24(wb, f + 6);
    } else {
      const uint4* fq = reinterpret_cast<const uint4*>(sF + ly * (TW * 3) + lx * 3);
      const uint4 f0 = fq[0], f1 = fq[1], f2 = fq[2];
      f[0] = f0.x; f[1] = f0.y; f[2] = f0.z; f[3] = f0.w; f[4] = f1.x; f[5] = f1.y; f[6] = f1.z; f[7] = f1.w;
      f[8] = f2.x; f[9] = f2.y; f[10] = f2.z; f[11] = f2.w;
    }
    if constexpr (REFINE) {
      if (refined) refine_mask16(a, y >= a.roi_y && y < a.roi_y + a.roi_h, x0, y, f, Hs, L::PCOLS, rmin, cmin, Rs, sM + ly * TW + lx, m);
    }
    if (BGRA) {
      // the transparent output, from the camera bytes before the blend overwrites the tile: straight to global memory,
      // at the mirrored position of a flipped frame (x0 and W are multiples of 16 pixels, so a run is wholly inside).
      // The mask is staged first, so that m can turn into the blend weights (alpha = 255 - weight).
      if (!pz || cfg.has_mask)
        *mdst = make_uint4(m[0] | (m[1] << 8) | (m[2] << 16) | (m[3] << 24), m[4] | (m[5] << 8) | (m[6] << 16) | (m[7] << 24),
                           m[8] | (m[9] << 8) | (m[10] << 16) | (m[11] << 24), m[12] | (m[13] << 8) | (m[14] << 16) | (m[15] << 24));
#pragma unroll
      for (int i = 0; i < PF_PX; ++i) m[i] = blend_weight(pz, m[i]);
      const int fl = flip_code();
      if (x0 < a.W && y < a.H) {
        uint8_t* bp = a.bgra + (size_t)b * a.bgra_stride + (size_t)((fl & 2) ? a.H - 1 - y : y) * a.bgra_pitch +
                      (size_t)((fl & 1) ? a.W - PF_PX - x0 : x0) * 4;
        // pixels 4k..4k+3, reversed into the mirrored quarter of the run when the frame is flipped horizontally
#pragma unroll
        for (int k = 0; k < 4; ++k) stg_stream(bp + 16 * ((fl & 1) ? 3 - k : k), bgra4(f + 3 * k, m + 4 * k, (fl & 1) != 0));
      }
    }
    if ((kind == 2 || (BGRA && kind == 0)) && !nobg) {
      const uint4* gq = reinterpret_cast<const uint4*>(sB + ly * (TW * 3) + lx * 3);
      const uint4 g0 = gq[0], g1 = gq[1], g2 = gq[2];
      gg[0] = g0.x; gg[1] = g0.y; gg[2] = g0.z; gg[3] = g0.w; gg[4] = g1.x; gg[5] = g1.y; gg[6] = g1.z; gg[7] = g1.w;
      gg[8] = g2.x; gg[9] = g2.y; gg[10] = g2.z; gg[11] = g2.w;
    } else {
#pragma unroll
      for (int i = 0; i < 12; ++i) gg[i] = f[i];
    }
    unsigned o[12], yy[8];
    unsigned w[PF_PX];
#pragma unroll
    for (int i = 0; i < PF_PX; ++i) w[i] = blend_weight(pz, m[i]);
    post_blend16<true, true>(f, gg, w, o, yy);
    // the YUYV camera tile is fully consumed before the (wider) BGR tile overwrites it, and a mirrored frame's camera tile
    // before any thread writes another's slot; the mask staging tile reuses Us, whose last readers (phase B) are behind a
    // barrier already
    const int fl = flip_code();
    if (IN_YUYV || NV12 || fl) __syncthreads();
    if (fl) {
      // mirrored frame: the thread's 16 pixels, reversed when horizontal, go to the mirrored slot
      const int mx = (fl & 1) ? TW - PF_PX - lx : lx, my = (fl & 2) ? PF_H - 1 - ly : ly;
      unsigned ro[12], ry[8];
      if (fl & 1) { rev_bgr16(o, ro); rev_yuyv16(yy, ry); }
      else {
#pragma unroll
        for (int i = 0; i < 12; ++i) ro[i] = o[i];
#pragma unroll
        for (int i = 0; i < 8; ++i) ry[i] = yy[i];
      }
      uint4* odst = reinterpret_cast<uint4*>(sF + my * (TW * 3) + mx * 3);
      odst[0] = make_uint4(ro[0], ro[1], ro[2], ro[3]); odst[1] = make_uint4(ro[4], ro[5], ro[6], ro[7]); odst[2] = make_uint4(ro[8], ro[9], ro[10], ro[11]);
      uint4* yq = reinterpret_cast<uint4*>(sY + my * (TW * 2) + mx * 2);
      yq[0] = make_uint4(ry[0], ry[1], ry[2], ry[3]); yq[1] = make_uint4(ry[4], ry[5], ry[6], ry[7]);
    } else {
      uint4* odst = reinterpret_cast<uint4*>(sF + ly * (TW * 3) + lx * 3);
      odst[0] = make_uint4(o[0], o[1], o[2], o[3]); odst[1] = make_uint4(o[4], o[5], o[6], o[7]); odst[2] = make_uint4(o[8], o[9], o[10], o[11]);
      ydst[0] = make_uint4(yy[0], yy[1], yy[2], yy[3]); ydst[1] = make_uint4(yy[4], yy[5], yy[6], yy[7]);
    }
    if (!BGRA && (!pz || cfg.has_mask))
      *mdst = make_uint4(m[0] | (m[1] << 8) | (m[2] << 16) | (m[3] << 24), m[4] | (m[5] << 8) | (m[6] << 16) | (m[7] << 24),
                         m[8] | (m[9] << 8) | (m[10] << 16) | (m[11] << 24), m[12] | (m[13] << 8) | (m[14] << 16) | (m[15] << 24));
    out_src = sF;
  }
  const uint8_t* nv_src = sY;          // NV12 calls: the tile the NV12 stores read (the cached background, else sN)
  if constexpr (NV12) {
    if (cfg.has_yuyv && !bg_copy) {
      // YUYV tile -> NV12: each thread takes 4 pairs of a row pair, copies the 8 + 8 Y bytes and averages the two rows'
      // U / V bytes with a per-byte truncating halving add (the NV12 output definition)
      __syncthreads();
      const int r = tid / (TW / 8), q = tid % (TW / 8);
      const uint4 a0 = *reinterpret_cast<const uint4*>(sY + (2 * r) * (TW * 2) + 16 * q);
      const uint4 a1 = *reinterpret_cast<const uint4*>(sY + (2 * r + 1) * (TW * 2) + 16 * q);
      *reinterpret_cast<uint2*>(sN + (2 * r) * TW + 8 * q) = make_uint2(__byte_perm(a0.x, a0.y, 0x6420), __byte_perm(a0.z, a0.w, 0x6420));
      *reinterpret_cast<uint2*>(sN + (2 * r + 1) * TW + 8 * q) = make_uint2(__byte_perm(a1.x, a1.y, 0x6420), __byte_perm(a1.z, a1.w, 0x6420));
      const unsigned h0 = __vhaddu4(a0.x, a1.x), h1 = __vhaddu4(a0.y, a1.y), h2 = __vhaddu4(a0.z, a1.z), h3 = __vhaddu4(a0.w, a1.w);
      *reinterpret_cast<uint2*>(sN + TW * PF_H + r * TW + 8 * q) = make_uint2(__byte_perm(h0, h1, 0x7531), __byte_perm(h2, h3, 0x7531));
      nv_src = sN;
    }
  }
  tma::fence_proxy_async();            // generic-proxy writes of the staging tiles -> visible to the TMA engine
  __syncthreads();
  // the tile's box, or for a mirrored frame the mirrored box (x = W - tx0 - TW, y = H - ty0 - 32, the UV plane's
  // H/2 - ty0/2 - 16).  x stays a multiple of 16 pixels (W % 16 == 0), so every box starts 16-byte aligned.  At ragged
  // edges the mirrored box starts at a negative coordinate: the threads store it, dropping exactly the rows / columns that
  // came from outside the frame.
  const int fl = flip_code();
  const int sx = (fl & 1) ? a.W - tx0 - TW : tx0, sy = (fl & 2) ? a.H - ty0 - PF_H : ty0;
  const bool clipped = FLIP && (sx < 0 || sy < 0);
  if (clipped) {
    if (cfg.has_out) store_clipped<NT, TW * 3>(out_src, PF_H, a.out + (size_t)b * a.out_stride, a.out_pitch, sx * 3, sy, a.W * 3, a.H, tid);
    if constexpr (NV12) {
      if (cfg.has_yuyv) {
        uint8_t* d = a.nv12 + (size_t)b * a.nv12_stride;
        store_clipped<NT, TW>(nv_src, PF_H, d, (size_t)a.W, sx, sy, a.W, a.H, tid);
        store_clipped<NT, TW>(nv_src + TW * PF_H, PF_H / 2, d + (size_t)a.W * a.H, (size_t)a.W, sx, sy / 2, a.W, a.H / 2, tid);
      }
    } else {
      if (cfg.has_yuyv) store_clipped<NT, TW * 2>(sY, PF_H, a.yuyv + (size_t)b * a.yuyv_stride, (size_t)a.W * 2, sx * 2, sy, a.W * 2, a.H, tid);
    }
  }
  if (tid == 0) {
    if (engine_only) tma::mbar_wait(barB, 0);
    if (!clipped) {
      if (cfg.has_out) tma::store_3d(&tm.out, out_src, sx / 4 * 3, sy, b);
      if constexpr (NV12) {
        if (cfg.has_yuyv) {
          tma::store_3d(&tm.yuyv, nv_src, sx / 4, sy, b);
          tma::store_3d(&tm.yuyv_uv, nv_src + TW * PF_H, sx / 4, sy / 2, b);
        }
      } else {
        if (cfg.has_yuyv) tma::store_3d(&tm.yuyv, sY, sx / 2, sy, b);
      }
    }
    if (cfg.has_mask) tma::store_3d(&tm.mask, sM, tx0, ty0, b);
    tma::store_commit();
    if (!BGRA && hits_roi && kind == 0 && !pz) tma::mbar_wait(barF, 0);
    tma::store_wait_read();            // shared memory may be handed to the next CTA only after the engine has read it
  }
}

// ---- host side: tensor maps --------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); p = nullptr; }
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// [n2][n1][row_bytes] bytes, row pitch / plane stride in bytes; box = box_bytes x box_rows x 1.  Elements are 32-bit
// words when `words` (row_bytes % 4 == 0), else bytes.
static bool make_map(CUtensorMap* m, const void* base, bool words, size_t row_bytes, size_t n1, size_t n2, size_t pitch, size_t stride,
                     unsigned box_bytes, unsigned box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) return false;
  const unsigned es = words ? 4u : 1u;
  const cuuint64_t gdim[3] = {row_bytes / es, n1, n2 ? n2 : 1};
  const cuuint64_t gstr[2] = {pitch, stride ? stride : pitch * n1};
  const cuuint32_t box[3] = {box_bytes / es, box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return enc(m, words ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static bool build_post_maps(const PostArgs& a, PostMaps* tm, int TW, PostMapsNv12* nv = nullptr) {
  const unsigned bw3 = (unsigned)TW * 3, bw2 = (unsigned)TW * 2, pw = TW == 128 ? (unsigned)PtL<128>::PW : (unsigned)PtL<64>::PW;
  const size_t W = (size_t)a.W, H = (size_t)a.H, B = (size_t)a.B;
  const size_t nbg = (a.bg_index || a.bg_cursor) ? (size_t)a.bg_count : (a.bg_stride ? B : 1);
  bool ok = true;
  if (a.yuyv_in) ok = ok && make_map(&tm->frame, a.yuyv_in, true, W * 2, H, B, W * 2, a.yuyv_in_stride, bw2, PF_H);
  else ok = ok && make_map(&tm->frame, a.frames, true, W * 3, H, B, a.frame_pitch, a.frame_stride, bw3, PF_H);
  ok = ok && make_map(&tm->bg, a.bg, true, W * 3, H, nbg, a.bg_pitch, a.bg_stride ? a.bg_stride : a.bg_pitch * H, bw3, PF_H);
  // unused maps still have to be valid descriptors: alias them to a live one
  if (a.bg_yuyv) ok = ok && make_map(&tm->bgy, a.bg_yuyv, true, W * 2, H, nbg, W * 2, W * 2 * H, bw2, PF_H); else tm->bgy = tm->bg;
  if (a.out) ok = ok && make_map(&tm->out, a.out, true, W * 3, H, B, a.out_pitch, a.out_stride, bw3, PF_H); else tm->out = tm->bg;
  if (a.yuyv) ok = ok && make_map(&tm->yuyv, a.yuyv, true, W * 2, H, B, W * 2, a.yuyv_stride, bw2, PF_H); else tm->yuyv = tm->bg;
  if (a.mask) ok = ok && make_map(&tm->mask, a.mask, false, W, H, B, W, a.mask_stride, (unsigned)TW, PF_H); else tm->mask = tm->bg;
  ok = ok && make_map(&tm->ofinal, a.ofinal, false, (size_t)a.ow, (size_t)a.oh, B, (size_t)a.opitch, (size_t)a.opitch * a.oh, pw, PT_RMAX);
  if (a.nv12_in) {
    // NV12 calls: Y planes (TW x 32 boxes) in the frame / bgy / yuyv maps, UV planes (TW x 16 boxes, H / 2 rows) beside them
    if (!nv) return false;
    const unsigned bw = (unsigned)TW;
    const size_t npix = W * H, nvb = npix * 3 / 2;
    ok = ok && make_map(&tm->frame, a.nv12_in, true, W, H, B, a.nv12_in_pitch, a.nv12_in_stride, bw, PF_H);
    ok = ok && make_map(&nv->frame_uv, a.nv12_in + a.nv12_in_uv, true, W, H / 2, B, a.nv12_in_pitch, a.nv12_in_stride, bw, PF_H / 2);
    if (a.bg_nv12) {
      ok = ok && make_map(&tm->bgy, a.bg_nv12, true, W, H, nbg, W, nvb, bw, PF_H);
      ok = ok && make_map(&nv->bgy_uv, a.bg_nv12 + npix, true, W, H / 2, nbg, W, nvb, bw, PF_H / 2);
    } else {
      nv->bgy_uv = tm->bg;
    }
    if (a.nv12) {
      ok = ok && make_map(&tm->yuyv, a.nv12, true, W, H, B, W, a.nv12_stride, bw, PF_H);
      ok = ok && make_map(&nv->yuyv_uv, a.nv12 + npix, true, W, H / 2, B, W, a.nv12_stride, bw, PF_H / 2);
    } else {
      nv->yuyv_uv = tm->bg;
    }
  }
  return ok;
}

// 64-wide tiles (eight CTAs per SM) hide more latency at 720p; at 3840x2160, where > 95 % of the tiles are pure copies,
// 128-wide tiles halve the per-CTA fixed cost
static int post_tile_width(const PostArgs& a) {
  const int t = tuning().post_tile;
  if (t == 64 || t == 128) return t;
  return a.W >= 2560 ? 128 : 64;
}

static bool post_tma_shape_ok(const PostArgs& a) {
  if (!tuning().post_tma || !encode_fn()) return false;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (a.B < 1 || a.W % 16 != 0 || a.area2x2 || a.tab.xcol == nullptr || a.geo_rows == nullptr) return false;
  if (a.nv12_in) {
    if (!al16(a.nv12_in) || a.nv12_in_pitch % 16 || a.nv12_in_uv % 16 || a.nv12_in_stride % 16 || (a.H & 1) || a.yuyv || a.bg_yuyv) return false;
    if (a.nv12 && (!al16(a.nv12) || a.nv12_stride % 16)) return false;
    if (a.bg_nv12 && !al16(a.bg_nv12)) return false;
  } else if (a.nv12 || a.bg_nv12) {
    return false;
  }
  if (a.yuyv_in) { if (!al16(a.yuyv_in) || a.yuyv_in_stride % 16) return false; }
  else if (!a.nv12_in && (!al16(a.frames) || a.frame_pitch % 16 || a.frame_stride % 16)) return false;
  if (!al16(a.bg) || a.bg_pitch % 16 || a.bg_stride % 16 || (a.bg_yuyv && !al16(a.bg_yuyv))) return false;
  if (a.out && (!al16(a.out) || a.out_pitch % 16 || a.out_stride % 16)) return false;
  if (a.yuyv && (!al16(a.yuyv) || a.yuyv_stride % 16)) return false;
  if (a.mask && (!al16(a.mask) || a.mask_stride % 16)) return false;
  if (a.bgra && (!al16(a.bgra) || a.bgra_pitch % 16 || a.bgra_stride % 16)) return false;
  if (!(a.out || a.yuyv || a.nv12 || a.mask || a.bgra) || !al16(a.ofinal) || a.opitch % 16) return false;
  if (a.ow > 32000 || a.oh > 32000 || a.roi_w < 8 || a.roi_h < 8) return false;
  const double scale_y = (double)a.out_h / (double)a.roi_h, scale_x = (double)a.out_w / (double)a.roi_w;
  const int tw = post_tile_width(a);
  const int pcols = tw == 128 ? PtL<128>::PCOLS : PtL<64>::PCOLS;
  if ((int)(PF_UH * scale_y) + 3 > PT_RMAX || (int)((tw + 4) * scale_x) + 4 > pcols) return false;
  // a refined tile's patch: taps s - 1 .. s + 2 of its 32 rows / tw columns
  if (a.refine && (!a.refine_w || !a.refine_x || !a.geo_r_rows || (int)((PF_H - 1) * scale_y) + 6 > PT_RMAX || (int)((tw - 1) * scale_x) + 6 > pcols))
    return false;
  return true;
}

bool post_tma_eligible(const PostArgs& a) {
  PostMapsNv12 tm;
  return post_tma_shape_ok(a) && build_post_maps(a, &tm, post_tile_width(a), &tm);
}

template <int FMT, int TW, bool FLIP, bool PASS, bool BGRA, bool REFINE>
static bool launch_post_tma_f(cudaStream_t s, const PostMapsOf<FMT>& tm, const PostArgs& a, const PostTmaCfg& cfg) {
  using L = PtL<TW>;
  if (!ensure_dyn_smem(reinterpret_cast<const void*>(k_post_tma<FMT, TW, FLIP, PASS, BGRA, REFINE>), L::SMEM)) return false;
  const dim3 grid((unsigned)ceil_div(a.W, TW), (unsigned)ceil_div(a.H, PF_H), (unsigned)a.B);
  k_post_tma<FMT, TW, FLIP, PASS, BGRA, REFINE><<<grid, L::NT, L::SMEM, s>>>(tm, a, cfg);
  return true;
}
template <int FMT, int TW, bool PASS, bool BGRA, bool REFINE>
static bool launch_post_tma_p(cudaStream_t s, const PostMapsOf<FMT>& tm, const PostArgs& a, const PostTmaCfg& cfg) {
  return a.flip ? launch_post_tma_f<FMT, TW, true, PASS, BGRA, REFINE>(s, tm, a, cfg) : launch_post_tma_f<FMT, TW, false, PASS, BGRA, REFINE>(s, tm, a, cfg);
}
template <int FMT, int TW, bool BGRA, bool REFINE>
static bool launch_post_tma_b(cudaStream_t s, const PostMapsOf<FMT>& tm, const PostArgs& a, const PostTmaCfg& cfg) {
  return a.pass ? launch_post_tma_p<FMT, TW, true, BGRA, REFINE>(s, tm, a, cfg) : launch_post_tma_p<FMT, TW, false, BGRA, REFINE>(s, tm, a, cfg);
}
template <int FMT, int TW, bool REFINE>
static bool launch_post_tma_r(cudaStream_t s, const PostMapsOf<FMT>& tm, const PostArgs& a, const PostTmaCfg& cfg) {
  return a.bgra ? launch_post_tma_b<FMT, TW, true, REFINE>(s, tm, a, cfg) : launch_post_tma_b<FMT, TW, false, REFINE>(s, tm, a, cfg);
}
template <int FMT, int TW>
static bool launch_post_tma_t(cudaStream_t s, const PostMapsOf<FMT>& tm, const PostArgs& a, const PostTmaCfg& cfg) {
  return a.refine ? launch_post_tma_r<FMT, TW, true>(s, tm, a, cfg) : launch_post_tma_r<FMT, TW, false>(s, tm, a, cfg);
}

bool launch_post_tma(cudaStream_t s, const PostArgs& a) {
  PostMapsNv12 tm;
  const int tw = post_tile_width(a);
  if (!post_tma_shape_ok(a) || !build_post_maps(a, &tm, tw, &tm)) return false;
  // (a launch with the transparent output blends its background tiles per thread: it copies no cached video tile)
  const PostTmaCfg cfg{a.out ? 1 : 0, (a.yuyv || a.nv12) ? 1 : 0, a.mask ? 1 : 0, ((a.bg_yuyv || a.bg_nv12) && !a.bgra) ? 1 : 0};
  const PostMaps& pm = tm;
  bool ok;
  if (a.nv12_in) ok = tw == 128 ? launch_post_tma_t<IN_NV12, 128>(s, tm, a, cfg) : launch_post_tma_t<IN_NV12, 64>(s, tm, a, cfg);
  else if (a.yuyv_in) ok = tw == 128 ? launch_post_tma_t<IN_YUYV, 128>(s, pm, a, cfg) : launch_post_tma_t<IN_YUYV, 64>(s, pm, a, cfg);
  else ok = tw == 128 ? launch_post_tma_t<IN_BGR, 128>(s, pm, a, cfg) : launch_post_tma_t<IN_BGR, 64>(s, pm, a, cfg);
  if (ok) count_launch();
  return ok;
}

#else   // BSB_EMU: TMA cannot be emulated; the emulator build always takes k_post_fast / k_post

bool post_tma_eligible(const PostArgs&) { return false; }
bool launch_post_tma(cudaStream_t, const PostArgs&) { return false; }

#endif

}  // namespace bsb
