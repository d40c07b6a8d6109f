// backscrub_b200/csrc/kernels.h — host-side launchers of the sm_90a kernels.
// All activations are fp32 NHWC with an explicit per-pixel channel stride (`ld`, in
// floats) so producers can write straight into a concatenated buffer; a batch of B
// frames is B consecutive images.
#pragma once
#include "bsb_common.h"
#include "framing.h"

namespace bsb {

// Epilogue shared by conv / pointwise / depthwise kernels, in graph order:
//   v = act1(total + bias)   (TFLite fused activation)
//   v = act2(v)              (following stand-alone unary op, folded by the planner)
//   v = act3(v + residual)   (following ADD, folded by the planner)
struct Epilogue {
  const float* bias = nullptr;
  int act1 = ACT_NONE, act2 = ACT_NONE, act3 = ACT_NONE;
  const float* residual = nullptr;  // same N/H/W/C as the output
  int ld_res = 0;
};

// ---- CNN ---------------------------------------------------------------------
// Dense KxK convolution, small Cin (the 3x3 s2 stems).  w_t: [kh][kw][ic][oc4] (oc padded to 4).
void launch_conv_direct(cudaStream_t s, int B, const float* in, int ih, int iw, int ic, int ld_in,
                        const float* w_t, int oc, int kh, int kw, int stride_h, int stride_w,
                        int dil_h, int dil_w, int pad_t, int pad_l,
                        float* out, int oh, int ow, int ld_out, const Epilogue& e);

// Stem variant that reads the bilateral-filtered u8 image directly and applies convertTo's
// fmaf(u8, scale, offset) on the fly (identical values, no fp32 input tensor round trip).  oc == 16, ic == 3.
void launch_stem_u8(cudaStream_t s, int B, const uint8_t* in_u8, int ih, int iw, float scale, float offset,
                    const float* w_t, int kh, int kw, int stride_h, int stride_w, int pad_t, int pad_l,
                    float* out, int oh, int ow, int ld_out, const Epilogue& e,
                    // optional fused 1x1 conv 16 -> 16 of the stem output (w2_kn: [16][16] k-major; no residual / scale)
                    const float* w2_kn = nullptr, float* out2 = nullptr, int ld_out2 = 0, const Epilogue* e2 = nullptr);

// 1x1 convolution / fully-connected as a GEMM: out[M][N] = A[M][K] * w_kn[K][N4] (+ epilogue).
// in_scale (optional): [B][K] per-frame channel scale applied to A on load (folded SE MUL);
// in_add (optional): tensor added after the scale (folded ADD), same layout as A.
void launch_pointwise(cudaStream_t s, int M, int K, int N, const float* A, int ld_a,
                      const float* w_kn, int n4, float* out, int ld_out, const Epilogue& e,
                      const float* in_scale, int rows_per_frame, const float* in_add, int ld_add);

void set_pointwise_variant(int v);   // 0 heuristics, 2 classic tiles, 3 register-tiled (A/B measurements; same bits)
int pointwise_variant();

// Tensor-core variant (wgmma.mma_async .tf32, 3xTF32 split, register accumulators) — kernels_tc.cu.
// w_hi / w_lo: [npad][kpad] zero-padded copies of W[N][K] split as w = hi + lo with hi tf32-representable;
// kpad % 32 == 0, npad % pointwise_tc_tile_n(N) == 0.  Returns false if the shape is not supported.
int pointwise_tc_tile_n(int N);
bool launch_pointwise_tc(cudaStream_t s, int M, int K, int N, const float* A, int ld_a, const float* w_hi, const float* w_lo,
                         int kpad, int npad, float* out, int ld_out, const Epilogue& e);
// Why launch_pointwise_tc would refuse these operands (pitches, alignment), or nullptr if it takes them.
const char* pointwise_tc_refusal(int K, const float* A, int ld_a, int kpad, const float* out, int ld_out, const Epilogue& e);

// Depthwise KxK (depth multiplier 1).  w: [kh][kw][C].
void launch_depthwise(cudaStream_t s, int B, const float* in, int ih, int iw, int c, int ld_in,
                      const float* w, int kh, int kw, int stride_h, int stride_w, int dil_h, int dil_w,
                      int pad_t, int pad_l, float* out, int oh, int ow, int ld_out, const Epilogue& e);

// Global average pool (+ optional squeeze-excite FC chain), two launches:
//   1. row sums: rowsum[b][y][c] = sum_x in[b][y][x][c]   (x ascending; many blocks)
//      — the input may be the channel concatenation of two tensors (inA | inB);
//   2. one block per frame: total = sum_y rowsum (y ascending), avg = total / (H*W), pool
//      activation, then up to two fully-connected layers (w: [K][N4], k ascending fmaf,
//      + bias, activations) — the SE "squeeze" path of MobileNetV3-style blocks.
struct FcLayer { const float* w = nullptr; const float* bias = nullptr; int K = 0, N = 0, n4 = 0, act1 = 0, act2 = 0; };
void launch_pool_fc(cudaStream_t s, int B, const float* inA, int cA, int ldA, const float* inB, int cB, int ldB,
                    int h, int w, float* rowsum_scratch, int pool_act, float* pooled_out /*may be null*/,
                    int n_fc, const FcLayer* fc, float* out, int ld_out,
                    unsigned* counters = nullptr /* [B] zeroed arrival counters: enables the one-launch variant */);

// Fused MobileNetV3 inverted-residual block at low resolution (<= 256 pixels per frame): 1x1 expand (+act) ->
// depthwise k x k stride 1 (+act) -> global pool -> FC -> FC (squeeze-excite) -> channel scale -> 1x1 project
// (+ residual).  One CTA per frame keeps every intermediate in shared memory; each stage accumulates in the
// same order as the stand-alone kernels, so results are bit-identical to running them one after another.
struct MbBlockArgs {
  const float* x; int ld_x; float* y; int ld_y;
  int h, w, cin, cexp, cout;
  const float* w1; const float* b1; int n4_1, a1a, a1b;                    // expand  [cin][n4_1]
  const float* wd; const float* bd; int k, pt, pl, ada, adb;               // depthwise [k][k][cexp]
  int pool_act; FcLayer f0, f1;                                            // SE
  const float* w2; const float* b2; int n4_2, a2a, a2b;                    // project [cexp][n4_2]
  int residual, a3;                                                        // y += x (cin == cout)
};
size_t mb_block_smem_bytes(int h, int w, int cin, int cexp, int cout, int fc_max_floats);   // 0 if it does not fit
void launch_mb_block(cudaStream_t s, int B, const MbBlockArgs& a);

// Low-resolution chain (the MobileNetV3 "middle" of the Meet / MLKit graphs: every tensor has P = h*w <= 256 pixels and
// <= 128 channels): ONE kernel, one CTA per frame, walks a list of ops with every activation resident in shared
// memory —  X [P][32] (the narrow block input / output), D [P][128] (the expanded tensor after its depthwise conv),
// E (one zero-haloed 16- or 32-channel slice of the expanded tensor: 16 where that fits two CTAs on an SM, i.e. Meet's
// 9x16 and 6x10; 32 for MLKit's 16x16).  Each op accumulates in the order of the stand-alone kernel it
// replaces (k ascending fmaf, taps in (fy, fx) order, pool rows-then-columns), so results are bit-identical.
enum ChainOpType : int {
  CH_DWG = 0,         // depthwise k x k (stride s) from a GLOBAL tensor [ih*iw][ld] into D            (block entry)
  CH_SE = 1,          // global average pool of D or X -> FC (-> FC) -> channel scale vector sv
  CH_PW = 2,          // 1x1 conv: src (D or X, optionally * sv) -> dst (X or D), optional in-place residual
  CH_EXPAND_DW = 3,   // X -> 1x1 expand (+act) -> depthwise k x k stride 1 (+act) -> D, one E slice at a time
  CH_SCALE_STORE = 4  // global out[p][c] = D[p][c] * sv[c]                                             (chain exit)
};
struct ChainOp {
  int type;
  int src, dst;                        // 0 = X, 1 = D
  int cin, cout;                       // channels of src / dst (PW: K / N; EXPAND_DW: cin -> cout; DWG / SE: C)
  // 1x1 conv / expand weights [K][n4]
  const float* w; const float* b; int n4, act1, act2;
  int use_scale, residual, act3;
  // depthwise [k][k][C]
  const float* wd; const float* bd; int k, s, pt, pl, dact1, dact2;
  // DWG input / SCALE_STORE output (per-frame stride in floats)
  const float* gin; int gin_ld, ih, iw; size_t gin_frame;
  float* gout; int gout_ld; size_t gout_frame;
  // SE
  int pool_act, n_fc; FcLayer f0, f1;
};
// shared memory needed for a chain over h x w pixels (0 if it cannot run)
size_t chain_smem_bytes(int h, int w);
// ops: DEVICE array of n_ops ChainOp
void launch_chain(cudaStream_t s, int B, int h, int w, const ChainOp* d_ops, int n_ops);

// RESIZE_BILINEAR (reference resize_bilinear.h:29-117 float path)
void launch_resize_bilinear(cudaStream_t s, int B, const float* in, int ih, int iw, int c, int ld_in,
                            float* out, int oh, int ow, int ld_out, bool align_corners, bool half_pixel);

// RESIZE_BILINEAR + the 1x1 conv that consumes it, fused (N <= 24 output channels; the up-sampled tensor is never
// materialised; same arithmetic per output as the two stand-alone kernels)
bool upsample_pw_supported(int K, int N, int n4, int ld_in, int ld_out);
void launch_upsample_pw(cudaStream_t s, int B, const float* in, int ih, int iw, int K, int ld_in, bool align_corners, bool half_pixel,
                        const float* w_kn, int n4, int N, float* out, int oh, int ow, int ld_out, const Epilogue& e);

// Decoder stage in one kernel: 1x1 conv (optional SE scale / skip add on its operand) -> depthwise 3x3 + residual of its
// own input -> optionally Convolution2DTransposeBias k2 s2.  C = 16 or 24.  Same arithmetic per output as the stand-alone kernels.
bool pw_dws2_supported(int K, int N, int ld_x, int ld_out);
void launch_pw_dws2(cudaStream_t s, const float* x, int ld_x, const float* wp, const float* bp, int actp, const float* wd, const float* bd, int actd,
                    float* out, int ld_out, int B, int ih, int iw, int oh, int ow, int pt, int pl);
bool head_supported(int C, int ld_x, int ld_add, int ld_out, int oc, bool tconv);
void launch_head(cudaStream_t s, int C, const float* x, int ld_x, const float* sv, const float* add, int ld_add,
                 const float* wp, const float* bp, int actp1, int actp2, const float* wd, const float* bd, int actd1, int actd2, int actr,
                 const float* wt, const float* bt, int oc, int actt, float* out, int ld_out, int B, int h, int w, int pt, int pl);

// The two MobileNetV3 inverted-residual blocks between the encoder entry and the chain (Meet / MLKit), as two kernels;
// the expanded tensors are never materialised.  Same arithmetic per output as the stand-alone kernels.
//   A: t25 = (x * sv) . W0 + b0;  t36 = act(dw3x3 s2 (act(t25 . W1 + b1)) + bd) . W2 + b2          (16 -> 72 -> 24)
//   B: t48 = act(dw3x3 (act(t36 . W3 + b3)) + bd) . W4 + b4 + t36;  t52 = hswish(t48 . W5 + b5)      (24 -> 88 -> 24 -> 96)
// act = RELU6 or RELU (the expand and the depthwise of both blocks); the weights are [K][N] with N a multiple of 4.
struct EncBlocksArgs {
  const float* x; int ld_x; const float* sv;                 // [B][ih][iw][ld_x] (16 channels), SE scale [B][16]
  const float* w[6]; const float* b[6];                       // 1x1 convs W0, W1, W2, W3, W4, W5 (b: null -> 0)
  const float* wd[2]; const float* bd[2];                     // depthwise [3][3][C] of block A, block B
  float* t25; int ld25; float* t36; int ld36; float* t48; int ld48; float* t52; int ld52;
  int ih, iw, oh, ow, pt_a, pl_a, act;                        // act: ACT_RELU6 or ACT_RELU
};
// the channel counts (16, 16, 72, 24, 88, 96) the kernels are compiled for, the strides, and the shared memory of this device
bool enc_blocks_supported(int device, int c_in, int c_25, int c_e1, int c_36, int c_e2, int c_52, int ld_x, int ld25, int ld36, int ld48, int ld52);
void launch_enc_blocks(cudaStream_t s, int B, const EncBlocksArgs& a, bool block_b);

// Convolution2DTransposeBias k2x2 s2 (lib/transpose_conv_bias.cc:37-114).  w: OHWI [oc][2][2][ic].
void launch_tconv2x2(cudaStream_t s, int B, const float* in, int ih, int iw, int ic, int ld_in,
                     const float* w, const float* bias, int oc, float* out, int oh, int ow, int ld_out, int act2);

// Element-wise: mode 0 unary act(a); 1 act(a + b); 2 act(a * b); 3 act(a * scale[b][c]) (channel broadcast);
// 4: act(a * scale[b][c] + b2) (MUL then ADD, two roundings).
void launch_eltwise(cudaStream_t s, int mode, int B, int hw, int c, const float* a, int ld_a,
                    const float* b, int ld_b, const float* scale, float* out, int ld_out, int act);

// Strided channel copy (CONCATENATION fallback): out[..., off:off+c] = in
void launch_copy_channels(cudaStream_t s, int rows, int c, const float* in, int ld_in, float* out, int ld_out);

// ---- image stages ---------------------------------------------------------------
struct ResizeTab {        // OpenCV INTER_LINEAR 8-bit tables (device pointers)
  const int* xofs;        // [dw] source column
  const short* xw;        // [dw][2] weights (scale 2^11)
  const int* yofs0;       // [dh] clamped row r0
  const int* yofs1;       // [dh] clamped row r1
  const short* yw;        // [dh][2]
  const uint2* xcol;      // [dw] packed {sx | sx1 << 16, a0 | a1 << 16} (sx1 = min(sx + 1, sw - 1))
};

// format of the frames a call reads: BGR, or a camera wire format read in place
enum InFmt : int { IN_BGR = 0, IN_YUYV = 1, IN_NV12 = 2 };

// lib/libbackscrub.cc:285-290: ROI crop -> cv::resize(INTER_LINEAR) -> BGR2RGB, into the
// zero-padded model-sized u8 image.  frames: B x (H x W x 3, stride bytes).
void launch_resize_roi_swap(cudaStream_t s, int B, const uint8_t* frames, size_t frame_stride, size_t frame_pitch,
                            int roi_x, int roi_y, int roi_w, int roi_h, ResizeTab tab,
                            uint8_t* in_u8, int mw, int mh, int in_x, int in_y, int in_w, int in_h, bool area2x2,
                            int in_fmt = IN_BGR,     // IN_YUYV: camera YUYV frames (pitch W*2); IN_NV12: camera NV12 frames
                            size_t uv_off = 0,       // (Y rows `frame_pitch` apart, UV plane at byte uv_off); converted per tap
                            const int* gather = nullptr);   // DEVICE [B]: output frame b is input frame gather[b] (null: b)

// lib/libbackscrub.cc:295-302: bilateralFilter(5,100,100) + convertTo(CV_32F, scale, offset)
void launch_bilateral_norm(cudaStream_t s, int B, const uint8_t* in_u8, int mw, int mh,
                           const float* color_w, const float* space_w, float scale, float offset,
                           float* out_f32, uint8_t* out_u8_dbg);

// Calls with held frames (bsb_set_mask_interval): DEVICE rows over the call's n frames, of which the B the CNN ran on are
// segmented.  gather[i]: the call frame of segmented frame i; cidx[b]: call frame b's index among the segmented frames, -1
// when it is held; lat[b] (plain calls): the index of the latest segmented frame at or before b, -1 when none.  A held
// frame's ofinal is its smoother's state after the latest segmented frame.  Null rows: every frame is segmented (n == B).
struct SegRows { int n = 0; const int* gather = nullptr; const int* cidx = nullptr; const int* lat = nullptr; };

// lib/libbackscrub.cc:314-361: decision + 3-tap bit-shift IIR over B consecutive frames.
// state: [oh*ow] persistent; ofinal: [B][oh][opitch] state after each frame (opitch >= ow: rows are padded to a
// multiple of 16 bytes so the post kernel can fetch patches of it with TMA).
void launch_decision_iir(cudaStream_t s, int model_type, int B, const float* model_out, int oh, int ow, int oc,
                         uint8_t* state, uint8_t* ofinal, int opitch, const SegRows& seg = SegRows{});
// DeepLab: the graph ends with RESIZE_BILINEAR 33x33x21 -> 257x257x21 and the decision is an argmax over the 21 classes of
// every output pixel.  This variant interpolates the 21 values of a pixel on the fly (the exact expression of the resize
// kernel) instead of writing and re-reading the 5.5 MB-per-frame tensor.
void launch_decision_up_iir(cudaStream_t s, int B, const float* low, int ih, int iw, int ld, bool align_corners, bool half_pixel,
                            int oh, int ow, uint8_t* state, uint8_t* ofinal, int opitch, const SegRows& seg = SegRows{});
// Independent sources: frame b of the batch belongs to source src[b] (DEVICE table [B], ids distinct within the call) and
// advances that source's state, states: [n_sources][oh*ow].  One step of the IIR per frame, every frame in parallel.
// cidx (SegRows::cidx, B = the call's frames): frame b reads segmented frame cidx[b] of model_out, or holds its state.
void launch_decision_sources(cudaStream_t s, int model_type, int B, const float* model_out, int oh, int ow, int oc,
                             uint8_t* states, const int* src, uint8_t* ofinal, int opitch, const int* cidx = nullptr);
// DeepLab form with the final 33 -> 257 resize folded in (as launch_decision_up_iir)
void launch_decision_up_sources(cudaStream_t s, int B, const float* low, int ih, int iw, int ld, bool align_corners, bool half_pixel,
                                int oh, int ow, uint8_t* states, const int* src, uint8_t* ofinal, int opitch, const int* cidx = nullptr);
// source coordinate / neighbours of RESIZE_BILINEAR (TF/lite/kernels/internal/reference/resize_bilinear.h:29-57)
BSB_D void bsb_resize_interp(float value, float scale, bool half_pixel, int in_size, float* scaled, int* lo, int* hi) {
  *scaled = half_pixel ? (value + 0.5f) * scale - 0.5f : value * scale;
  const float fl = floorf(*scaled);
  int l = (int)fl; if (l < 0) l = 0;
  int h = (int)ceilf(*scaled); if (h > in_size - 1) h = in_size - 1;
  *lo = l; *hi = h;
}

// lib/libbackscrub.cc:366-371 + app/deepseg.cc:108-134,87-106 fused:
// mask = blur5x5(resize(ofinal(out_roi) -> roi)) inside roidim, 255 outside;
// out = (bg*mask + frame*(255-mask))/255; optional YUYV of out; optional mask store.
struct PostArgs {
  int B, W, H;
  const uint8_t* frames; size_t frame_pitch, frame_stride;   // row pitch / per-frame stride (bytes)
  const uint8_t* bg; size_t bg_pitch, bg_stride;             // bg_stride 0 => one static background
  const int* bg_cursor; int bg_count, bg_advance;             // non-null: frame b blends ring image (*cursor + b*advance) % count
  const int* bg_index;                                         // non-null (DEVICE [B]): frame b blends image bg_index[b] of bg_count (wins over bg_cursor)
  const uint8_t* ofinal; int ow, oh, opitch;                  // [B][oh][opitch]
  int out_x, out_y, out_w, out_h;                              // out_roidim inside ofinal
  int roi_x, roi_y, roi_w, roi_h;                              // roidim inside the frame
  ResizeTab tab;                                               // out_roi -> roi upsample tables
  bool area2x2;
  uint8_t* out; size_t out_pitch, out_stride;                  // may be null
  uint8_t* yuyv; size_t yuyv_stride;                           // may be null (W*2 bytes per row)
  uint8_t* mask; size_t mask_stride;                           // may be null (W bytes per row)
  int frame_l1;                                                // frame loads allocate in L1 (measurement switch)
  // TMA path only (k_post_tma): the camera frames may stay in their wire format (YUYV, W*2 bytes per row, tightly
  // packed, `yuyv_in_stride` bytes per frame) and are converted per tile; `bg_yuyv` is the background (ring) already
  // converted to YUYV, same indexing as `bg` with W*2-byte rows, so all-background tiles are pure copies.
  const uint8_t* yuyv_in; size_t yuyv_in_stride;
  const uint8_t* bg_yuyv;
  // TMA path only, NV12 calls: camera NV12 frames read in place (Y rows `nv12_in_pitch` bytes apart, the UV plane at byte
  // `nv12_in_uv` of a frame, `nv12_in_stride` bytes per frame), the video output written as tightly packed NV12
  // (`nv12_stride` bytes per frame; yuyv is null), and the background (ring / bank) as NV12, W*H*3/2 bytes per image
  const uint8_t* nv12_in; size_t nv12_in_pitch, nv12_in_uv, nv12_in_stride;
  uint8_t* nv12; size_t nv12_stride;
  const uint8_t* bg_nv12;
  // per tile row / tile column: the patch of the small mask a (TW + 4) x 36 halo tile touches, {first, count}
  // (precomputed once per context from `tab`: the patch request is the head of every CTA's critical path)
  const int2* geo_rows; const int2* geo_cols64; const int2* geo_cols128;
  // TMA path only: non-null (DEVICE [B]): frame b's out / YUYV / NV12 are written mirrored by flip[b] (bit 0 horizontally,
  // bit 1 vertically; 0 = as is).  The mask is never mirrored.  launch_post refuses it where k_post_tma cannot run.
  const int* flip;
  // non-null (DEVICE [B]): frame b with pass[b] != 0 has its filter switched off (app/deepseg.cc:624,639-664): its
  // composite is the camera frame (blend weight 0) and no background is read; its mask is stored as for any frame.  Every
  // post kernel honours it; each compiles it into separate instantiations, so a call without it runs as before.
  const int* pass;
  // may be null: the transparent output, straight-alpha BGRA (rows `bgra_pitch` bytes apart, W*4 used): the camera pixel
  // with alpha 255 - mask, or 255 for a frame whose filter is off.  Written mirrored by `flip` like `out`.  Every post
  // kernel compiles it into separate instantiations; with neither `out` nor a video output the call reads no background.
  uint8_t* bgra; size_t bgra_pitch, bgra_stride;
};
// false (nothing launched) when a.flip is set and k_post_tma cannot take the arguments
bool launch_post(cudaStream_t s, const PostArgs& a);
// true if launch_post will take the TMA kernel for these arguments (the only one that can read a.yuyv_in / a.nv12_in)
bool post_tma_eligible(const PostArgs& a);

// app/background.cc:178-194: cv::resize(raw -> W x H), 3 channels
// n images (frame strides in bytes; n = 1 for the background provider)
void launch_resize_u8c3(cudaStream_t s, const uint8_t* src, int sw, int sh, size_t spitch,
                        uint8_t* dst, int dw, int dh, size_t dpitch, ResizeTab tab, bool area2x2,
                        int n = 1, size_t sstride = 0, size_t dstride = 0);

// Live backgrounds (include/backscrub_b200.h, bsb_set_live_background / bsb_set_source_live_background): frame b of a call
// blends a caller-owned device image, BGR or NV12 of any size, resized to W x H inside the call (app/background.cc:178-194
// on the newest frame of the `-b` source, app/deepseg.cc:648-650).
enum LiveFmt : int { LIVE_BGR = 0, LIVE_NV12 = 1 };
struct LiveDesc {
  const uint8_t* p;          // null: the frame has no live background (its CTAs exit at once)
  size_t pitch, uv;          // row pitch; NV12: the UV plane's byte offset
  int fmt, w, h;             // LiveFmt and size
  int blur;                  // non-zero: a Gaussian follows, so the frame goes to the staging, else to its slot
  int area2x2;               // exact 2x down (OpenCV's INTER_AREA case), else INTER_LINEAR through tab
  ResizeTab tab;             // w x h -> W x H (the tables of the live size, kept per distinct size)
};
// descs: DEVICE [n].  Frame b: cv::resize(INTER_LINEAR) of its live image to W x H (NV12 taps converted per source pixel as
// cv::cvtColor(COLOR_YUV2BGR_NV12) would) into slot + b*W*H*3 and, where given, the slot's YUYV (yuyv + b*W*H*2, W even)
// or NV12 (nv12 + b*W*H*3/2, W and H even); a frame with `blur` set goes to stage + b*W*H*3 instead (tightly packed BGR
// the Gaussian reads), without YUYV / NV12.
void launch_live_bg(cudaStream_t s, int n, const LiveDesc* descs, uint8_t* slot, uint8_t* stage, uint8_t* yuyv, uint8_t* nv12, int W, int H);

// app/deepseg.cc:657-658: cv::GaussianBlur(bg, bg, Size(k,k), 0), 8UC3 — OpenCV's 8.8 fixed-point taps (sum 256)
struct GaussTaps { int k; uint16_t q[255]; };
bool gauss_taps(int k, GaussTaps* out);           // false unless k is odd, 1..255
// n frames; tmp holds n*H*W*3 16-bit row sums.  False if the per-device tap tables could not be allocated.
bool launch_gauss_blur(cudaStream_t s, int n, const uint8_t* src, size_t spitch, size_t sstride, uint16_t* tmp,
                       uint8_t* dst, size_t dpitch, size_t dstride, int W, int H, const GaussTaps& g);
// Launch classes of the Gaussian: the fused tile kernel (strengths 3..31) or the row / column pair (1, 33..255); 0 = off
enum : unsigned { GAUSS_FUSED = 1, GAUSS_SEPARABLE = 2 };
BSB_HD int gauss_class(int k) { return k == 0 ? 0 : (k >= 3 && k <= 31) ? (int)GAUSS_FUSED : (int)GAUSS_SEPARABLE; }
// camera frames in their wire format: YUYV or NV12 (InFmt), `pitch` bytes per row, `stride` per frame, NV12's UV plane
// at byte `uv`
struct GaussSrc { const uint8_t* p; size_t pitch, stride, uv; int fmt; };
// the per-device tap tables every launch reads (built on first use); false if they could not be allocated
bool gauss_tables_ready();
// Sources calls: frame b blurred with strength ks[b] (DEVICE table [n]; 0 = not blurred) from the tightly packed BGR
// frame b of `frames` into frame b of dst (same layout); `classes` (GAUSS_FUSED | GAUSS_SEPARABLE) are the launch classes
// the call may need, so a captured launch replays for any strengths within them.  cam.p non-null: `frames` is first
// filled, for the blurred frames only, from the camera frames.  dst_yuyv / dst_nv12 (may be null): the blurred frames'
// YUYV / NV12 (W*H*2 / W*H*3/2 bytes per frame; W even, NV12 also H even).
bool launch_gauss_frames(cudaStream_t s, int n, const GaussSrc& cam, const int* ks, unsigned classes, uint8_t* frames, uint16_t* tmp,
                         uint8_t* dst, uint8_t* dst_yuyv, uint8_t* dst_nv12, int W, int H);
// app/deepseg.cc:667-673: cv::flip on n packed frames
void launch_flip_u8c3(cudaStream_t s, int n, const uint8_t* src, size_t sstride, uint8_t* dst, size_t dstride, int W, int H, bool flip_h, bool flip_v);
// app/deepseg.cc:667-681 in one launch, the tail of a call whose frames are mirrored or resized outside the post kernel:
// cv::flip, then cv::resize to the frame's virtual-camera geometry, then the YUYV (or NV12) conversion, from the staged
// W x H BGR composites (and the BGRA output from the staged BGRA frames, 8UC4).  The flip mirrors each tap's source coordinate and keeps the weights; ow == W and oh == H is a
// mirrored copy.  Bit-exact against the chain k_flip_u8c3 -> k_resize_u8c3 -> k_rgb_to_yuyv (-> k_yuyv_to_nv12).
struct TailGeo { int ow, oh; ResizeTab tab; int area2x2; };
// a framed frame's crop (x, y, w, h) and the resize steps (resize_scale) from it to the frame's output size
struct FrameCrop { int x, y, w, h; double sx, sy; };   // tab: INTER_LINEAR tables W x H -> ow x oh
struct TailArgs {
  int n, W, H;
  const uint8_t* src; size_t src_stride;   // staged composites, rows W*3 bytes
  uint8_t* out; size_t out_stride;         // may be null: BGR, tightly packed rows ow*3 bytes
  uint8_t* video; size_t video_stride;     // may be null: tightly packed YUYV (floor(ow*oh/2) flat pixel pairs), or NV12
  int nv12;                                //   (ow, oh even; Y plane, UV plane at byte ow*oh) when nv12 != 0
  TailGeo geo; int flip;                   // every frame's geometry and flip code (bit 0 horizontal, bit 1 vertical) ...
  const int* slot; const TailGeo* geos;    // ... unless set: frame b's geometry is geos[slot[b]] (DEVICE)
  const int* flips;                        // ... and its flip code flips[b] (DEVICE)
  // bgra != 0: `out` is BGRA (tightly packed rows ow*4 bytes), flipped and resized channel by channel from the staged
  // W x H BGRA frames `src4` (rows W*4 bytes); `src` is then read only for the video output
  const uint8_t* src4; size_t src4_stride; int bgra;
  // framed calls (bsb_set_framing; a separate k_tail instantiation): non-null (DEVICE) frame b shows crop
  // crop[crop_idx[b]] of its staged frame, flipped within the crop and resized to its geometry's ow x oh with taps
  // computed on the fly (resize_taps.h; a crop of the output size is a copy, an exact 2x crop the INTER_AREA mean).  The
  // geometry's tables are not read.
  const FrameCrop* crop; const int* crop_idx;
};
// max_px: the largest ow * oh a frame of the call can have (the grid covers it; smaller frames' extra CTAs exit)
void launch_tail(cudaStream_t s, const TailArgs& a, long max_px);

// Framing (framing.h): one CTA per frame reduces the frame's small mask (ofinal, inside out_roidim) to the person count
// and bounding box; AUTO frames then step their camera's state and write their crop, RECT / OFF frames copy the table's
// rectangle.  tab: DEVICE [FRAMING_ROWS][mb] rows mode | jump (the camera has no state yet) | state slot | ow | oh | x | y
// | w | h | crop index.  Sources calls: every frame steps state[slot] in parallel (distinct ids).  Plain calls (`plain`):
// every frame steps state[0] in frame order, in the CTA that arrives last (targets: [n][4] scratch, counter:
// 0 between launches).
enum { FRAMING_ROWS = 10 };
struct FramingArgs {
  int n;
  const uint8_t* ofinal; int oh, opitch, ox, oy;   // [n][oh][opitch], out_roidim's origin
  FramingGeo g; FramingParams p;
  const int* tab; int mb;
  int* state;                                       // [slots][4] 1/16-pixel states
  FrameCrop* crop;                                  // written at the crop index
  int* targets; unsigned* counter; int plain;
};
void launch_framing(cudaStream_t s, const FramingArgs& a);

// cv::cvtColor(COLOR_YUV2BGR_YUYV): camera YUYV frames -> BGR (what cv::VideoCapture does for the
// reference, app/deepseg.cc:553).  n frames of W x H, tightly packed.
void launch_yuyv_to_bgr(cudaStream_t s, const uint8_t* yuyv, uint8_t* bgr, size_t npix_total);

// stand-alone stage kernels (exported through the C-ABI for stage-level parity tests)
void launch_alpha_blend(cudaStream_t s, const uint8_t* a, const uint8_t* b, const uint8_t* mask, uint8_t* out, size_t npix);
// npix pixels per frame (even), n frames
void launch_rgb_to_yuyv(cudaStream_t s, const uint8_t* rgb, uint8_t* yuyv, size_t npix, int n = 1, size_t rgb_stride = 0, size_t yuyv_stride = 0);
// cv::cvtColor(COLOR_YUV2BGR_NV12): n camera NV12 frames (W, H even; Y rows `pitch` apart, UV plane at byte uv_off,
// `in_stride` bytes per frame) -> tightly packed BGR frames
void launch_nv12_to_bgr(cudaStream_t s, int n, const uint8_t* nv12, size_t pitch, size_t uv_off, size_t in_stride, uint8_t* bgr, int W, int H);
// the project's NV12 output from its YUYV output (include/backscrub_b200.h): n frames of W x H (even), tightly packed
// W*2-byte YUYV rows -> tightly packed NV12 (Y plane, UV plane at byte W*H)
void launch_yuyv_to_nv12(cudaStream_t s, int n, const uint8_t* yuyv, size_t yuyv_stride, uint8_t* nv12, size_t nv12_stride, int W, int H);
// *cursor = (*cursor + step) % count, after the frames of a call have been blended
void launch_advance_cursor(cudaStream_t s, int* cursor, int step, int count);

// number of kernel launches issued through the launchers above (bench gpu_launches); per calling thread
long launch_count();
long thread_launch_count();

// Opt a kernel into `bytes` of dynamic shared memory on the CURRENT device (cudaFuncSetAttribute is per device and
// per function; the largest request so far is remembered per (device, function) under a mutex, so contexts on several
// devices and the host threads of one process can share the launchers).  Returns false if the driver refuses.
bool ensure_dyn_smem(const void* func, size_t bytes);

// Streaming multiprocessors of the CURRENT device (grid sizing of the launchers).
int device_sms();

// Measurement switches of the launchers (bsb_set_tuning in the C ABI; tools/ and bench.py A/B runs).  They never change
// results, only which bit-identical kernel variant runs.  Defaults are the variants the project ships.
struct Tuning {
  int pw_variant = 0;      // launch_pointwise: 0 heuristics, 2 classic tiles, 3/4/8 register-tiled, 5 row-streaming, 16/32/64 classic N tile
  int dw_px = 1;           // small depthwise layers: row-batched loads (k_depthwise_px) instead of the generic tap loop
  int dec_up = 1;          // DeepLab: final 33 -> 257 resize folded into the argmax decision kernel
  int epi_static = 1;      // compile-time epilogues (bias preloaded, activation fixed) for the common combinations; 0 = the generic run-time epilogue everywhere
  int pw_dws2 = 1;         // 16 -> 16 1x1 conv + the stride-2 depthwise 3x3 that consumes it in one kernel (the 1x1's output is never materialised)
  int up_staged = 1;       // resize + 1x1: interpolated operand rows built once per pixel in shared memory when a pixel is shared by several threads
  int stem_x2 = 1;         // stem conv: two adjacent output pixels per thread (3x3 stride 2, even width), shared weight loads
  int e2e_chunk = 16;      // bsb_composite_yuyv (host buffers): frames per chunk of the copy / compute overlap (0 = one serial H2D -> graph -> D2H)
  int dec_par = 1;         // decision + temporal smoother: frames in parallel (a block = 32 pixels x all frames) instead of one thread per pixel
  int dw_plane = 1;        // whole-plane depthwise kernel for the 33x33 atrous layers
  int dw_plane_cs = 16;    // ... channels per block (16: 70 KB of shared memory per 33x33 plane, 3 blocks per SM; 8: 35 KB, 6 blocks)
  int post_tma = 1;        // TMA-staged post kernel where the geometry allows it
  int tc_variant = 2;      // tensor-core pointwise kernel: 2 = warp-specialised TMA-fed persistent kernel, 1 = the round-1 kernel
  int tc_min_k = 16;       // smallest input depth of a 1x1 conv that goes to the tensor cores (with BSB_FLAG_TENSOR_CORES)
  int tc_mask_hi = 0;      // tensor-core kernel: clear the low mantissa bits of A explicitly instead of relying on the hardware truncation
  int head = 1;            // decoder stages (1x1 -> depthwise 3x3 + residual [-> transposed conv]) in one kernel (k_head)
  int up_pw = 1;           // fuse RESIZE_BILINEAR into the 1x1 conv that consumes it
  int stem_pw = 0;         // run the 16 -> 16 1x1 conv that follows the stem inside the stem kernel (off by default)
  int pool_merge = 1;      // global pool + SE tail in one launch (last block per frame runs the tail)
  int cnn_chain = 1;       // one kernel for the low-resolution middle of the MobileNetV3-style graphs (kernels_chain.cu)
  int sub_batch_mb = 0;    // engine: wide-layer segments run in frame groups whose largest tensor is <= this many MB (0 = off)
  int post_tile = 0;       // k_post_tma: tile width (64: eight CTAs per SM, 128: four; 0 = by frame size: 128 from 2560 pixels wide)
  int post_l1 = 1;         // k_post_fast: frame loads allocate in L1
};
Tuning& tuning();

}  // namespace bsb
