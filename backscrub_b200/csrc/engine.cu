// backscrub_b200/csrc/engine.cu — planner + per-stream engine (see engine.h).
#include "engine.h"
#include "resize_taps.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace bsb {

#define CUDA_OK(expr)                                                                      \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      if (err) *err = std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #expr; \
      return false;                                                                        \
    }                                                                                      \
  } while (0)

// ---------------------------------------------------------------------------
// OpenCV INTER_LINEAR 8-bit tables (cv::resize; formulas pinned in oracle/oracle_img.c)
// ---------------------------------------------------------------------------
HostResizeTab build_resize_tab(int sw, int sh, int dw, int dh) {
  HostResizeTab t;
  t.sw = sw;
  t.area2x2 = (sw == dw * 2 && sh == dh * 2);
  const double scale_x = resize_scale(sw, dw), scale_y = resize_scale(sh, dh);
  t.xofs.resize(dw); t.xw.resize(2 * (size_t)dw);
  for (int dx = 0; dx < dw; ++dx) {
    int w0, w1;
    resize_tap_x(dx, scale_x, sw, &t.xofs[dx], &w0, &w1);
    t.xw[2 * dx] = (short)w0; t.xw[2 * dx + 1] = (short)w1;
  }
  t.yofs0.resize(dh); t.yofs1.resize(dh); t.yw.resize(2 * (size_t)dh);
  for (int dy = 0; dy < dh; ++dy) {
    int w0, w1;
    resize_tap_y(dy, scale_y, sh, &t.yofs0[dy], &t.yofs1[dy], &w0, &w1);
    t.yw[2 * dy] = (short)w0; t.yw[2 * dy + 1] = (short)w1;
  }
  return t;
}

bool upload_resize_tab(const HostResizeTab& h, DevResizeTab* d, std::string* err) {
  const size_t nx = h.xofs.size(), ny = h.yofs0.size();
  auto al = [](size_t n) { return (n + 15) / 16 * 16; };
  const size_t o_xofs = 0, o_y0 = o_xofs + al(nx * 4), o_y1 = o_y0 + al(ny * 4), o_xw = o_y1 + al(ny * 4), o_yw = o_xw + al(nx * 4);
  const size_t o_xcol = o_yw + al(ny * 4);
  const size_t total = o_xcol + al(nx * 8);
  std::vector<uint8_t> blob(total, 0);
  {
    std::vector<uint32_t> xc(2 * nx);
    for (size_t i = 0; i < nx; ++i) {
      const int sx = h.xofs[i], sx1 = std::min(sx + 1, h.sw - 1);
      xc[2 * i] = (uint32_t)sx | ((uint32_t)sx1 << 16);
      xc[2 * i + 1] = (uint32_t)(uint16_t)h.xw[2 * i] | ((uint32_t)(uint16_t)h.xw[2 * i + 1] << 16);
    }
    std::memcpy(blob.data() + o_xcol, xc.data(), nx * 8);
  }
  std::memcpy(blob.data() + o_xofs, h.xofs.data(), nx * 4);
  std::memcpy(blob.data() + o_y0, h.yofs0.data(), ny * 4);
  std::memcpy(blob.data() + o_y1, h.yofs1.data(), ny * 4);
  std::memcpy(blob.data() + o_xw, h.xw.data(), nx * 4);
  std::memcpy(blob.data() + o_yw, h.yw.data(), ny * 4);
  if (d->blob) { cudaFree(d->blob); d->blob = nullptr; }
  CUDA_OK(cudaMalloc(&d->blob, blob.size()));
  CUDA_OK(cudaMemcpy(d->blob, blob.data(), blob.size(), cudaMemcpyHostToDevice));
  uint8_t* b = static_cast<uint8_t*>(d->blob);
  d->tab.xofs = reinterpret_cast<const int*>(b + o_xofs);
  d->tab.yofs0 = reinterpret_cast<const int*>(b + o_y0);
  d->tab.yofs1 = reinterpret_cast<const int*>(b + o_y1);
  d->tab.xw = reinterpret_cast<const short*>(b + o_xw);
  d->tab.yw = reinterpret_cast<const short*>(b + o_yw);
  d->tab.xcol = reinterpret_cast<const uint2*>(b + o_xcol);
  d->area2x2 = h.area2x2;
  return true;
}

// TF SAME/VALID output size + leading pad (reference kernels/padding.h:23-82)
static void conv_geom(int in, int k, int stride, int dil, int padding, int* out, int* pad_before) {
  const int eff = (k - 1) * dil + 1;
  const int o = padding == 0 ? (in + stride - 1) / stride : (in + stride - eff) / stride;
  int total = (o - 1) * stride + eff - in;
  if (total < 0) total = 0;
  *out = o; *pad_before = total / 2;
}

static int unary_act(int kind) {
  switch (kind) {
    case OP_HARD_SWISH: return ACT_HARD_SWISH;
    case OP_RELU: return ACT_RELU;
    case OP_RELU6: return ACT_RELU6;
    case OP_LOGISTIC: return ACT_LOGISTIC;
    default: return -1;
  }
}

// ---------------------------------------------------------------------------
// Planner: TFLite op list -> fused steps + arena layout
// ---------------------------------------------------------------------------
bool Engine::plan(std::string* err) {
  const int nt = (int)g_.tensors.size(), nops = (int)g_.ops.size();
  // Tensor cores for the 1x1 convs (3xTF32 split, ~1e-6 relative to the exact fp32 chain — the tolerance the reference's
  // own XNNPACK-vs-builtin conv tests use): on by default for the GEMM-dominated graphs (DeepLab 93 %, BodyPix 95 % of
  // their FLOPs are 1x1 convs), on request for the others (BSB_FLAG_TENSOR_CORES), never with BSB_FLAG_EXACT.  When
  // every intermediate tensor is kept for bit-level comparison (BSB_FLAG_KEEP_TENSORS) they stay off unless
  // BSB_FLAG_TENSOR_CORES is passed too (then each tensor-core layer can be checked in place against its own inputs).
  tc_enabled_ = !(flags_ & 16u) && (!(flags_ & 1u) || (flags_ & 4u)) &&
                ((flags_ & 4u) || model_type_ == MODEL_DEEPLAB || model_type_ == MODEL_BODYPIX);
  std::vector<std::vector<int>> consumers(nt);
  std::vector<int> produced_at(nt, -1);
  for (int i = 0; i < nops; ++i) {
    const GOp& O = g_.ops[i];
    if (O.kind == OP_DEQUANTIZE) continue;
    for (int t : O.in) if (t >= 0 && !g_.tensors[t].is_const) consumers[t].push_back(i);
    if (O.out >= 0) produced_at[O.out] = i;
  }
  tinfo_.assign(nt, TensorInfo());
  for (int t = 0; t < nt; ++t) {
    const GTensor& T = g_.tensors[t];
    if (T.is_const || T.dtype != 0) continue;
    if (T.dim4(0) != 1) { *err = "tensor '" + T.name + "': batch dimension must be 1"; return false; }
    TensorInfo& I = tinfo_[t];
    I.h = T.dim4(1); I.w = T.dim4(2); I.c = T.dim4(3); I.ld = I.c;
    I.frame_elems = (size_t)I.h * I.w * I.ld;
  }
  auto is_pw = [&](const GOp& O) {
    if (O.kind != OP_CONV_2D || O.in.size() < 2 || O.in[1] < 0) return false;
    const GTensor& w = g_.tensors[O.in[1]];
    return w.shape.size() == 4 && w.shape[1] == 1 && w.shape[2] == 1 && O.stride_w == 1 && O.stride_h == 1;
  };
  auto add_blob = [&](const std::vector<float>& v) {
    size_t off = (wblob_h_.size() + 63) / 64 * 64;
    wblob_h_.resize(off + v.size(), 0.f);
    std::copy(v.begin(), v.end(), wblob_h_.begin() + off);
    return off;
  };
  struct Fold { int x, s, add; };
  std::map<int, Fold> prologue;      // tensor consumed by a PW conv -> (x, scale, add)
  std::map<int, std::pair<int, int>> concat_for_pool;
  std::map<int, int> producer_step;  // tensor -> index in steps_ of the step that writes it
  std::map<int, std::vector<int>> aliased_into;
  std::vector<int> concat_virtual;
  std::vector<char> done(nops, 0);

  auto fold_unary = [&](int i, Step& st) {  // fold a single-consumer unary op after op i
    const int t = st.out;
    if (consumers[t].size() != 1) return;
    const int j = consumers[t][0];
    const int a = unary_act(g_.ops[j].kind);
    if (a < 0 || done[j] || j <= i) return;
    st.act2 = a; done[j] = 1; st.out = g_.ops[j].out;
  };
  auto fold_add = [&](int i, Step& st) {    // fold a single-consumer residual ADD
    const int t = st.out;
    if (t == g_.output || consumers[t].size() != 1) return;
    const int j = consumers[t][0];
    const GOp& A = g_.ops[j];
    if (A.kind != OP_ADD || done[j] || j <= i || A.in.size() != 2) return;
    const int other = A.in[0] == t ? A.in[1] : A.in[0];
    if (other == t || g_.tensors[other].is_const) return;
    if (g_.tensors[other].count() != g_.tensors[t].count()) return;
    if (other != g_.input && !(produced_at[other] >= 0 && produced_at[other] < i)) return;
    if (prologue.count(other)) return;
    st.residual = other; st.act3 = A.act; done[j] = 1; st.out = A.out;
  };
  auto pack_pw_weights = [&](const GTensor& w, int N, int K, Step& st) {
    st.K = K; st.N = N; st.n4 = (N + 3) / 4 * 4;
    std::vector<float> wt((size_t)K * st.n4, 0.f);
    for (int n = 0; n < N; ++n) for (int k = 0; k < K; ++k) wt[(size_t)k * st.n4 + n] = w.f32[(size_t)n * K + k];
    st.w_off = add_blob(wt);
  };
  // 3xTF32 operand split for the tensor-core path: w = hi + lo, hi = w with the 13 low mantissa bits cleared
  auto pack_tc_weights = [&](const GTensor& w, int N, int K, Step& st) {
    const int bn = pointwise_tc_tile_n(N);
    if (bn <= 0) return;
    st.kpad = (K + 31) / 32 * 32; st.npad = (N + bn - 1) / bn * bn;
    std::vector<float> hi((size_t)st.npad * st.kpad, 0.f), lo((size_t)st.npad * st.kpad, 0.f);
    for (int n = 0; n < N; ++n) for (int k = 0; k < K; ++k) {
      const float v = w.f32[(size_t)n * K + k];
      uint32_t bits; std::memcpy(&bits, &v, 4); bits &= 0xffffe000u;
      float h; std::memcpy(&h, &bits, 4);
      hi[(size_t)n * st.kpad + k] = h; lo[(size_t)n * st.kpad + k] = v - h;
    }
    st.tc_hi_off = add_blob(hi); st.tc_lo_off = add_blob(lo); st.use_tc = true;
  };

  for (int i = 0; i < nops; ++i) {
    const GOp& O = g_.ops[i];
    if (done[i] || O.kind == OP_DEQUANTIZE) continue;
    Step st; st.op_index = i;
    auto need = [&](bool c, const char* what) { if (!c) { *err = std::string("unsupported model construct: ") + what; } return c; };
    switch (O.kind) {
      case OP_CONV_2D: {
        if (!need(O.in.size() >= 2 && O.in[1] >= 0 && g_.tensors[O.in[1]].is_const, "CONV_2D with non-constant weights")) return false;
        const GTensor& w = g_.tensors[O.in[1]];
        if (!need(w.shape.size() == 4 && w.f32.size() == w.count(), "CONV_2D weights that are not a rank-4 float tensor")) return false;
        if (!need(O.in.size() < 3 || O.in[2] < 0 || (int)g_.tensors[O.in[2]].f32.size() == w.shape[0], "CONV_2D bias size")) return false;
        if (!need(w.shape[3] == tinfo_[O.in[0]].c, "CONV_2D input depth")) return false;
        const int oc = w.shape[0], kh = w.shape[1], kw = w.shape[2], ic = w.shape[3];
        st.in = O.in[0]; st.out = O.out; st.act1 = O.act;
        if (O.in.size() > 2 && O.in[2] >= 0) { st.has_bias = true; st.b_off = add_blob(g_.tensors[O.in[2]].f32); }
        if (is_pw(O)) {
          st.kind = Step::PW;
          pack_pw_weights(w, oc, ic, st);
          auto it = prologue.find(st.in);
          if (it != prologue.end()) { st.in = it->second.x; st.scale = it->second.s; st.in_add = it->second.add; }
          // tensor cores (opt-in): plain GEMM-shaped layers with enough rows and depth to fill a 128 x N x 32 tile pipeline
          if (tc_enabled_ && st.scale < 0 && st.in_add < 0 && ic >= tuning().tc_min_k && ic % 4 == 0 && oc >= 8 &&
              tinfo_[st.in].h * tinfo_[st.in].w >= 1024 && tinfo_[st.in].ld % 4 == 0)
            pack_tc_weights(w, oc, ic, st);
        } else {
          st.kind = Step::CONV;
          st.kh = kh; st.kw = kw; st.sh = O.stride_h; st.sw = O.stride_w; st.dh = O.dil_h; st.dw = O.dil_w;
          st.K = ic; st.N = oc; st.n4 = (oc + 3) / 4 * 4;
          int o_h, o_w;
          conv_geom(tinfo_[st.in].h, kh, st.sh, st.dh, O.padding, &o_h, &st.pt);
          conv_geom(tinfo_[st.in].w, kw, st.sw, st.dw, O.padding, &o_w, &st.pl);
          if (!need(o_h == tinfo_[O.out].h && o_w == tinfo_[O.out].w, "CONV_2D output shape")) return false;
          if (!need((size_t)kh * kw * ic * st.n4 * 4 <= 96 * 1024, "dense KxK conv too large for the direct kernel")) return false;
          std::vector<float> wt((size_t)kh * kw * ic * st.n4, 0.f);   // [kh][kw][ic][oc4]
          for (int o = 0; o < oc; ++o) for (int y = 0; y < kh; ++y) for (int x = 0; x < kw; ++x) for (int c = 0; c < ic; ++c)
            wt[(((size_t)y * kw + x) * ic + c) * st.n4 + o] = w.f32[(((size_t)o * kh + y) * kw + x) * ic + c];
          st.w_off = add_blob(wt);
        }
        fold_unary(i, st); fold_add(i, st);
        break;
      }
      case OP_FULLY_CONNECTED: {
        if (!need(O.in.size() >= 2 && O.in[1] >= 0 && g_.tensors[O.in[1]].is_const, "FULLY_CONNECTED with non-constant weights")) return false;
        const GTensor& w = g_.tensors[O.in[1]];
        if (!need(w.shape.size() >= 2 && w.f32.size() == w.count(), "FULLY_CONNECTED weights that are not a float matrix")) return false;
        st.kind = Step::PW; st.in = O.in[0]; st.out = O.out; st.act1 = O.act;
        const int out_depth = w.shape[w.shape.size() - 2], in_depth = w.shape[w.shape.size() - 1];
        if (!need(tinfo_[st.in].c == in_depth, "FULLY_CONNECTED over flattened spatial dims")) return false;
        pack_pw_weights(w, out_depth, in_depth, st);
        if (O.in.size() > 2 && O.in[2] >= 0) { st.has_bias = true; st.b_off = add_blob(g_.tensors[O.in[2]].f32); }
        fold_unary(i, st);
        break;
      }
      case OP_DEPTHWISE_CONV_2D: {
        if (!need(O.depth_mult == 1, "depthwise multiplier != 1")) return false;
        if (!need(O.in.size() >= 2 && O.in[1] >= 0 && g_.tensors[O.in[1]].is_const, "DEPTHWISE_CONV_2D with non-constant weights")) return false;
        const GTensor& w = g_.tensors[O.in[1]];
        if (!need(w.shape.size() == 4 && w.f32.size() == w.count() && w.shape[3] == tinfo_[O.in[0]].c, "DEPTHWISE_CONV_2D weight shape")) return false;
        st.kind = Step::DW; st.in = O.in[0]; st.out = O.out; st.act1 = O.act;
        st.kh = w.shape[1]; st.kw = w.shape[2]; st.sh = O.stride_h; st.sw = O.stride_w; st.dh = O.dil_h; st.dw = O.dil_w;
        int o_h, o_w;
        conv_geom(tinfo_[st.in].h, st.kh, st.sh, st.dh, O.padding, &o_h, &st.pt);
        conv_geom(tinfo_[st.in].w, st.kw, st.sw, st.dw, O.padding, &o_w, &st.pl);
        if (!need(o_h == tinfo_[O.out].h && o_w == tinfo_[O.out].w, "DEPTHWISE_CONV_2D output shape")) return false;
        st.w_off = add_blob(w.f32);
        if (O.in.size() > 2 && O.in[2] >= 0) { st.has_bias = true; st.b_off = add_blob(g_.tensors[O.in[2]].f32); }
        fold_unary(i, st); fold_add(i, st);
        break;
      }
      case OP_AVERAGE_POOL_2D: {
        st.kind = Step::POOL; st.in = O.in[0]; st.out = O.out; st.act1 = O.act;
        int ph = tinfo_[st.in].h, pw = tinfo_[st.in].w, pc = tinfo_[st.in].c;
        if (!need(O.filter_h == ph && O.filter_w == pw && tinfo_[O.out].h == 1 && tinfo_[O.out].w == 1,
                  "AVERAGE_POOL_2D that is not global")) return false;
        if (!need(pc <= 512, "global pool over more than 512 channels")) return false;
        auto cp = concat_for_pool.find(st.in);
        if (cp != concat_for_pool.end()) { st.in = cp->second.first; st.in2 = cp->second.second; }
        rowsum_elems_ = std::max(rowsum_elems_, (size_t)ph * pc);
        // fold the squeeze-excite FC chain: pool -> {1x1 conv | FC} (+unary) [-> {1x1 conv | FC} (+unary)]
        int cur = st.out;
        while (st.n_fc < 2 && cur != g_.output && consumers[cur].size() == 1) {
          const int j = consumers[cur][0];
          const GOp& F = g_.ops[j];
          if (done[j] || j <= i || F.in.empty() || F.in[0] != cur || F.in.size() < 2 || !g_.tensors[F.in[1]].is_const) break;
          const GTensor& w = g_.tensors[F.in[1]];
          int K, N;
          if (is_pw(F)) { N = w.shape[0]; K = w.shape[3]; }
          else if (F.kind == OP_FULLY_CONNECTED) { N = w.shape[w.shape.size() - 2]; K = w.shape[w.shape.size() - 1]; }
          else break;
          // the FC weights are staged in shared memory by k_pool_fc: keep K x N4 inside the opt-in limit
          if (K != tinfo_[cur].c || K > 512 || N > 512 || (size_t)K * ((N + 3) / 4 * 4) * 4 > 192 * 1024 ||
              tinfo_[F.out].h != 1 || tinfo_[F.out].w != 1) break;
          Step tmp;
          pack_pw_weights(w, N, K, tmp);
          Step::Fc& fc = st.fc[st.n_fc++];
          fc.w_off = tmp.w_off; fc.K = K; fc.N = N; fc.n4 = tmp.n4; fc.act1 = F.act;
          if (F.in.size() > 2 && F.in[2] >= 0) { fc.has_bias = true; fc.b_off = add_blob(g_.tensors[F.in[2]].f32); }
          done[j] = 1; cur = F.out;
          if (consumers[cur].size() == 1) {
            const int u = consumers[cur][0];
            const int ua = unary_act(g_.ops[u].kind);
            if (ua >= 0 && !done[u] && u > j) { fc.act2 = ua; done[u] = 1; cur = g_.ops[u].out; }
          }
        }
        st.out = cur;
        break;
      }
      case OP_RESIZE_BILINEAR: {
        st.kind = Step::RESIZE; st.in = O.in[0]; st.out = O.out; st.align_corners = O.align_corners; st.half_pixel = O.half_pixel;
        if (!need(O.in.size() >= 2 && O.in[1] >= 0, "RESIZE_BILINEAR without a size tensor")) return false;
        const GTensor& sz = g_.tensors[O.in[1]];
        if (!need(sz.is_const && sz.i32.size() == 2 && sz.i32[0] == tinfo_[O.out].h && sz.i32[1] == tinfo_[O.out].w, "RESIZE_BILINEAR size")) return false;
        break;
      }
      case OP_CUSTOM: {
        if (!need(O.custom == "Convolution2DTransposeBias", "unknown custom op")) return false;
        if (!need(O.in.size() >= 3 && O.in[1] >= 0 && O.in[2] >= 0 && g_.tensors[O.in[1]].is_const && g_.tensors[O.in[2]].is_const,
                  "Convolution2DTransposeBias with non-constant weights / bias")) return false;
        const GTensor& w = g_.tensors[O.in[1]];
        if (!need(w.shape.size() == 4 && w.f32.size() == w.count() && w.shape[3] == tinfo_[O.in[0]].c &&
                  (int)g_.tensors[O.in[2]].f32.size() == w.shape[0], "Convolution2DTransposeBias weight shape")) return false;
        if (!need(w.shape[1] == 2 && w.shape[2] == 2 && O.stride_w == 2 && O.stride_h == 2 && O.tconv_same &&
                  tinfo_[O.out].h == 2 * tinfo_[O.in[0]].h && tinfo_[O.out].w == 2 * tinfo_[O.in[0]].w,
                  "Convolution2DTransposeBias other than k2 s2 SAME on even sizes")) return false;
        st.kind = Step::TCONV; st.in = O.in[0]; st.out = O.out; st.N = w.shape[0]; st.K = w.shape[3];
        st.w_off = add_blob(w.f32); st.has_bias = true; st.b_off = add_blob(g_.tensors[O.in[2]].f32);
        fold_unary(i, st);
        break;
      }
      case OP_MUL: {
        if (!need(O.in.size() == 2, "MUL arity")) return false;
        int x = O.in[0], s = O.in[1];
        if (g_.tensors[x].count() < g_.tensors[s].count()) std::swap(x, s);
        const bool bcast = g_.tensors[s].count() != g_.tensors[x].count();
        if (bcast && !need((int)g_.tensors[s].count() == tinfo_[x].c && !g_.tensors[s].is_const, "MUL broadcast other than per-channel")) return false;
        if (bcast && O.act == ACT_NONE && consumers[O.out].size() == 1 && O.out != g_.output) {
          const int j = consumers[O.out][0];
          const GOp& C = g_.ops[j];
          if (is_pw(C) && C.in[0] == O.out) { prologue[O.out] = Fold{x, s, -1}; done[i] = 1; continue; }
          if (C.kind == OP_ADD && C.act == ACT_NONE && C.in.size() == 2 && consumers[C.out].size() == 1 && C.out != g_.output) {
            const int other = C.in[0] == O.out ? C.in[1] : C.in[0];
            const GOp& P = g_.ops[consumers[C.out][0]];
            if (other != O.out && !g_.tensors[other].is_const && g_.tensors[other].count() == g_.tensors[x].count() &&
                is_pw(P) && P.in[0] == C.out && !prologue.count(other)) {
              prologue[C.out] = Fold{x, s, other}; done[i] = 1; done[j] = 1; continue;
            }
          }
        }
        st.kind = Step::ELT; st.in = x; st.out = O.out; st.act1 = O.act;
        if (bcast) { st.elt_mode = 3; st.scale = s; } else { st.elt_mode = 2; st.in2 = s; }
        break;
      }
      case OP_ADD: {
        if (!need(O.in.size() == 2 && g_.tensors[O.in[0]].count() == g_.tensors[O.in[1]].count(), "ADD with broadcasting")) return false;
        st.kind = Step::ELT; st.elt_mode = 1; st.in = O.in[0]; st.in2 = O.in[1]; st.out = O.out; st.act1 = O.act;
        break;
      }
      case OP_HARD_SWISH: case OP_RELU: case OP_RELU6: case OP_LOGISTIC:
        st.kind = Step::ELT; st.elt_mode = 0; st.in = O.in[0]; st.out = O.out; st.act1 = unary_act(O.kind);
        break;
      case OP_CONCATENATION: {
        const int rank = (int)g_.tensors[O.out].shape.size();
        const int axis = O.axis < 0 ? O.axis + rank : O.axis;
        if (!need(axis == rank - 1 && O.act == ACT_NONE, "CONCATENATION not on the channel axis")) return false;
        // (1) a concatenation that only feeds a global pool is never materialised: the pool's
        //     row-sum kernel reads both sources (pool(concat(a,b)) == concat(pool(a),pool(b)) exactly)
        if (O.in.size() == 2 && O.out != g_.output && consumers[O.out].size() == 1 &&
            g_.ops[consumers[O.out][0]].kind == OP_AVERAGE_POOL_2D && !prologue.count(O.in[0]) && !prologue.count(O.in[1])) {
          concat_for_pool[O.out] = std::make_pair(O.in[0], O.in[1]);
          continue;
        }
        // (2) otherwise producers write straight into the concatenated buffer when they can
        int off = 0;
        for (int t : O.in) {
          const bool can_alias = t != g_.input && consumers[t].size() == 1 && producer_step.count(t) && tinfo_[t].alias_parent < 0 &&
                                 off % 4 == 0 && tinfo_[O.out].c % 4 == 0 && !prologue.count(t);
          if (can_alias) {
            tinfo_[t].alias_parent = O.out; tinfo_[t].alias_off = off; tinfo_[t].ld = tinfo_[O.out].ld;
            tinfo_[t].frame_elems = tinfo_[O.out].frame_elems;
            aliased_into[O.out].push_back(t);
          } else {
            Step c; c.op_index = i; c.kind = Step::COPY; c.in = t; c.out = O.out; c.copy_off = off;
            steps_.push_back(c);
          }
          off += tinfo_[t].c;
        }
        if (aliased_into.count(O.out)) {   // a no-op marker step so the buffer counts as produced here
          bool any_copy = false;
          for (const Step& c : steps_) any_copy = any_copy || (c.kind == Step::COPY && c.out == O.out);
          if (!any_copy) concat_virtual.push_back(O.out);
        }
        continue;
      }
      default:
        *err = "unsupported TFLite operator code " + std::to_string(O.kind);
        return false;
    }
    producer_step[st.out] = (int)steps_.size();
    steps_.push_back(st);
  }

  // ---- fuse low-resolution inverted-residual blocks (expand -> depthwise -> SE -> project) into one kernel ----
  if ((flags_ & 8u) && !(flags_ & 1u)) {   // opt-in (BSB_FLAG_FUSE_BLOCKS); KEEP_TENSORS keeps every intermediate -> stand-alone kernels
    std::vector<int> readers(nt, 0);
    for (const Step& st : steps_) for (int t : {st.in, st.in2, st.scale, st.in_add, st.residual}) if (t >= 0) ++readers[t];
    std::vector<Step> fused;
    for (size_t i = 0; i < steps_.size(); ++i) {
      bool ok = i + 3 < steps_.size();
      if (ok) {
        const Step& e = steps_[i]; const Step& d = steps_[i + 1]; const Step& p = steps_[i + 2]; const Step& q = steps_[i + 3];
        ok = e.kind == Step::PW && !e.use_tc && e.scale < 0 && e.in_add < 0 && e.residual < 0 && e.out != g_.output &&
             d.kind == Step::DW && d.in == e.out && d.sh == 1 && d.sw == 1 && d.dh == 1 && d.dw == 1 && d.residual < 0 && d.kh == d.kw &&
             p.kind == Step::POOL && p.in == d.out && p.in2 < 0 && p.n_fc == 2 &&
             q.kind == Step::PW && !q.use_tc && q.in == d.out && q.scale == p.out && q.in_add < 0 && (q.residual < 0 || q.residual == e.in) &&
             readers[e.out] == 1 && readers[d.out] == 2 && readers[p.out] == 1 && p.out != g_.output && d.out != g_.output;
        if (ok) {
          const TensorInfo& X = tinfo_[e.in]; const TensorInfo& D = tinfo_[d.out];
          const int fc_max = std::max(std::max(p.fc[0].K * p.fc[0].n4, p.fc[1].K * p.fc[1].n4), q.K * q.n4);
          ok = X.h == D.h && X.w == D.w && p.fc[0].K == e.N && p.fc[1].N == e.N && p.fc[0].N <= 128 && e.N <= 128 &&
               (q.residual < 0 || X.c == q.N) && X.ld % 4 == 0 &&
               mb_block_smem_bytes(X.h, X.w, X.c, e.N, q.N, fc_max) > 0;
        }
      }
      if (!ok) { fused.push_back(steps_[i]); continue; }
      Step b; b.kind = Step::BLOCK; b.op_index = steps_[i].op_index; b.in = steps_[i].in; b.out = steps_[i + 3].out;
      b.residual = steps_[i + 3].residual; b.block = (int)blocks_.size();
      blocks_.push_back(FusedBlock{steps_[i], steps_[i + 1], steps_[i + 2], steps_[i + 3]});
      tinfo_[steps_[i].out].materialized = false; tinfo_[steps_[i + 1].out].materialized = false; tinfo_[steps_[i + 2].out].materialized = false;
      fused.push_back(b);
      i += 3;
    }
    steps_.swap(fused);
  }

  // ---- RESIZE_BILINEAR folded into the 1x1 conv that is its only reader ----
  if (tuning().up_pw) {
    for (size_t i = 0; i + 1 < steps_.size(); ++i) {
      const Step& r = steps_[i]; Step& q = steps_[i + 1];
      if (r.kind != Step::RESIZE || q.kind != Step::PW || q.in != r.out || q.scale >= 0 || q.in_add >= 0 || q.residual >= 0 || q.use_tc) continue;
      if (r.out == g_.output || consumers[r.out].size() != 1) continue;
      if (!upsample_pw_supported(q.K, q.N, q.n4, tinfo_[r.in].ld, tinfo_[q.out].ld)) continue;
      q.up_from = r.in; q.align_corners = r.align_corners; q.half_pixel = r.half_pixel;
      q.in = r.in;                                    // liveness: the conv now reads the low-resolution tensor
      tinfo_[r.out].materialized = false;
      steps_.erase(steps_.begin() + i);
    }
  }
  for (const Step& st : steps_) uses_tc_ = uses_tc_ || st.use_tc;
  // ---- the low-resolution middle of MobileNetV3-style graphs as one kernel ----
  if (tuning().cnn_chain && !(flags_ & (1u | 8u))) detect_chain();
  // ---- decoder stages (1x1 -> depthwise + residual [-> transposed conv]) as one kernel each ----
  if (tuning().head && !(flags_ & (1u | 8u))) detect_heads();
  // ---- encoder entry (16 -> 16 1x1 -> depthwise 3x3 stride 2) as one kernel ----
  if (tuning().pw_dws2 && !tuning().stem_pw && !(flags_ & (1u | 8u))) detect_pw_dws2();
  // ---- the two inverted-residual blocks between the encoder entry and the chain as two kernels ----
  if (!(flags_ & (1u | 8u))) detect_enc_blocks();
  find_segments();
  dec_up_step_ = -1;
  if (tuning().dec_up && model_type_ == MODEL_DEEPLAB && !(flags_ & 1u) && !steps_.empty()) {
    const Step& last = steps_.back();
    if (last.kind == Step::RESIZE && last.out == g_.output && tinfo_[last.out].c == 21 && tinfo_[last.in].c == 21) dec_up_step_ = (int)steps_.size() - 1;
  }

  // ---- liveness + arena (floats; every tensor is max_batch frames) ----
  const int ns = (int)steps_.size();
  auto root = [&](int t) { return tinfo_[t].alias_parent >= 0 ? tinfo_[t].alias_parent : t; };
  auto use = [&](int t, int s) { if (t >= 0) { const int r = root(t); tinfo_[r].last_use = std::max(tinfo_[r].last_use, s); } };
  tinfo_[g_.input].materialized = true; tinfo_[g_.input].first_def = -1;
  for (int s = 0; s < ns; ++s) {
    const Step& st = steps_[s];
    use(st.in, s); use(st.in2, s); use(st.scale, s); use(st.in_add, s); use(st.residual, s);
    for (int o : {st.out, st.out2}) {
      if (o < 0) continue;
      tinfo_[o].materialized = true;
      const int r = root(o);
      tinfo_[r].materialized = true;
      tinfo_[r].first_def = std::min(tinfo_[r].first_def, s);
      use(o, s);
    }
  }
  // a sub-batched segment runs its steps once per frame group: every tensor it touches must stay allocated from the
  // segment's first step to its last (a buffer recycled inside the segment would be overwritten by group g while group
  // g + 1 still has to read it)
  for (int s0 = 0; s0 < ns; ++s0) {
    if (s0 >= (int)seg_len_.size() || seg_len_[s0] <= 0) continue;
    const int s1 = s0 + seg_len_[s0] - 1;
    for (int s = s0; s <= s1; ++s) {
      const Step& st = steps_[s];
      for (int t : {st.in, st.in2, st.scale, st.in_add, st.residual, st.up_from, st.out, st.out2}) {
        if (t < 0) continue;
        const int r = root(t);
        tinfo_[r].last_use = std::max(tinfo_[r].last_use, s1);
        if (tinfo_[r].first_def > s0 && tinfo_[r].first_def <= s1) tinfo_[r].first_def = s0;
      }
    }
  }
  tinfo_[root(g_.output)].last_use = 1 << 30;
  tinfo_[g_.input].last_use = std::max(tinfo_[g_.input].last_use, 0);
  if (!tinfo_[g_.output].materialized) { *err = "graph output is never produced"; return false; }
  for (const Step& st : steps_)
    for (int t : {st.in, st.in2, st.scale, st.in_add, st.residual})
      if (t >= 0 && !tinfo_[t].materialized) { *err = "planner: step reads a tensor that was folded away"; return false; }

  struct Free { size_t off, size; };
  std::vector<Free> free_list;
  size_t top = 0;
  auto alloc = [&](size_t n) {
    n = (n + 63) / 64 * 64;
    for (size_t k = 0; k < free_list.size(); ++k)
      if (free_list[k].size >= n) {
        size_t off = free_list[k].off;
        free_list[k].off += n; free_list[k].size -= n;
        if (!free_list[k].size) free_list.erase(free_list.begin() + k);
        return off;
      }
    size_t off = top; top += n; return off;
  };
  auto release = [&](size_t off, size_t n) {
    n = (n + 63) / 64 * 64;
    free_list.push_back({off, n});
    std::sort(free_list.begin(), free_list.end(), [](const Free& a, const Free& b) { return a.off < b.off; });
    for (size_t k = 0; k + 1 < free_list.size();)
      if (free_list[k].off + free_list[k].size == free_list[k + 1].off) { free_list[k].size += free_list[k + 1].size; free_list.erase(free_list.begin() + k + 1); }
      else ++k;
  };
  const bool keep = (flags_ & 1u) != 0;
  std::vector<char> allocated(nt, 0);
  tinfo_[g_.input].offset = alloc(tinfo_[g_.input].frame_elems * max_batch_); allocated[g_.input] = 1;
  for (int s = 0; s < ns; ++s) {
    for (int t : {steps_[s].out, steps_[s].out2}) {
      if (t < 0) continue;
      const int o = root(t);
      if (!allocated[o]) { tinfo_[o].offset = alloc(tinfo_[o].frame_elems * max_batch_); allocated[o] = 1; }
    }
    if (keep) continue;
    for (int t = 0; t < nt; ++t)
      if (allocated[t] == 1 && tinfo_[t].alias_parent < 0 && tinfo_[t].materialized && tinfo_[t].last_use == s) {
        release(tinfo_[t].offset, tinfo_[t].frame_elems * max_batch_); allocated[t] = 2;
      }
  }
  arena_elems_ = top;

  {
    const Step& s0 = steps_[0];
    stem_u8_ok_ = s0.kind == Step::CONV && s0.in == g_.input && s0.K == 3 && s0.N == 16 && s0.dh == 1 && s0.dw == 1 &&
                  consumers[g_.input].size() == 1 && tinfo_[s0.out].ld % 4 == 0 && s0.residual < 0;
    stem_pw_ok_ = false;
    if (stem_u8_ok_ && steps_.size() > 1) {
      const Step& s1 = steps_[1];
      stem_pw_ok_ = s1.kind == Step::PW && s1.in == s0.out && s1.K == 16 && s1.N == 16 && s1.n4 == 16 && s1.scale < 0 && s1.in_add < 0 &&
                    s1.residual < 0 && !s1.use_tc && tinfo_[s1.out].ld % 4 == 0;
    }
  }
  // algorithmic FLOPs (2*MAC of conv / depthwise / fc / tconv), SURVEY.md Appendix A
  flops_ = 0;
  for (const GOp& O : g_.ops) {
    if (O.out < 0 || O.in.size() < 2) continue;
    const GTensor& out = g_.tensors[O.out]; const GTensor& w = g_.tensors[O.in[1]];
    if (O.kind == OP_CONV_2D) flops_ += 2.0 * out.count() * w.shape[1] * w.shape[2] * w.shape[3];
    else if (O.kind == OP_DEPTHWISE_CONV_2D) flops_ += 2.0 * out.count() * w.shape[1] * w.shape[2];
    else if (O.kind == OP_FULLY_CONNECTED) flops_ += 2.0 * out.count() * w.shape.back();
    else if (O.kind == OP_CUSTOM) flops_ += 2.0 * out.count() * w.shape[3];
  }
  return true;
}

void Engine::detect_heads() {
  auto reads = [&](const Step& r, int t) { return r.in == t || r.in2 == t || r.scale == t || r.in_add == t || r.residual == t; };
  for (size_t i = 0; i + 1 < steps_.size(); ++i) {
    const Step& P = steps_[i]; const Step& D = steps_[i + 1];
    if (P.kind != Step::PW || P.use_tc || P.up_from >= 0 || P.residual >= 0 || P.K != P.N || (P.N != 16 && P.N != 24) || P.n4 != P.N) continue;
    if (D.kind != Step::DW || D.in != P.out || D.residual != P.out || D.kh != 3 || D.kw != 3 || D.sh != 1 || D.sw != 1 || D.dh != 1 || D.dw != 1) continue;
    if (tinfo_[D.out].c != P.N || P.out == g_.output || D.out == g_.output) continue;
    bool only_d = true;                                         // t (the 1x1 output) must be private to the depthwise step
    for (size_t k = 0; k < steps_.size(); ++k) if (k != i + 1 && reads(steps_[k], P.out)) only_d = false;
    if (!only_d) continue;
    HeadPlan hp; hp.p = P; hp.d = D;
    if (i + 2 < steps_.size()) {
      const Step& T = steps_[i + 2];
      bool only_t = T.kind == Step::TCONV && T.in == D.out && T.K == P.N && T.N <= 2 && tinfo_[T.out].ld == T.N;
      for (size_t k = 0; k < steps_.size() && only_t; ++k) if (k != i + 2 && reads(steps_[k], D.out)) only_t = false;
      if (only_t) { hp.t = T; hp.has_t = true; }
    }
    const int ld_add = P.in_add >= 0 ? tinfo_[P.in_add].ld : 4;
    const int out_t = hp.has_t ? hp.t.out : D.out;
    if (!head_supported(P.N, tinfo_[P.in].ld, ld_add, tinfo_[out_t].ld, hp.has_t ? hp.t.N : 0, hp.has_t)) continue;
    Step h; h.kind = Step::HEAD; h.op_index = P.op_index; h.in = P.in; h.scale = P.scale; h.in_add = P.in_add; h.out = out_t;
    h.block = (int)heads_.size();
    heads_.push_back(hp);
    tinfo_[P.out].materialized = false;
    if (hp.has_t) tinfo_[D.out].materialized = false;
    const size_t n_erase = hp.has_t ? 3 : 2;
    steps_.erase(steps_.begin() + i, steps_.begin() + i + n_erase);
    steps_.insert(steps_.begin() + i, h);
  }
}

void Engine::detect_pw_dws2() {
  auto reads = [&](const Step& r, int t) { return r.in == t || r.in2 == t || r.scale == t || r.in_add == t || r.residual == t; };
  for (size_t i = 0; i + 1 < steps_.size(); ++i) {
    const Step& P = steps_[i]; const Step& D = steps_[i + 1];
    if (P.kind != Step::PW || P.use_tc || P.up_from >= 0 || P.residual >= 0 || P.scale >= 0 || P.in_add >= 0 || P.K != 16 || P.N != 16 || P.n4 != 16) continue;
    if (D.kind != Step::DW || D.in != P.out || D.residual >= 0 || D.kh != 3 || D.kw != 3 || D.sh != 2 || D.sw != 2 || D.dh != 1 || D.dw != 1) continue;
    if ((P.act1 != ACT_NONE && P.act2 != ACT_NONE) || (D.act1 != ACT_NONE && D.act2 != ACT_NONE)) continue;
    if (tinfo_[D.out].c != 16 || P.out == g_.output || D.out == g_.output) continue;
    bool only_d = true;                                         // the 1x1 output must be private to the depthwise step
    for (size_t k = 0; k < steps_.size(); ++k) if (k != i + 1 && reads(steps_[k], P.out)) only_d = false;
    if (!only_d || !pw_dws2_supported(P.K, P.N, tinfo_[P.in].ld, tinfo_[D.out].ld)) continue;
    HeadPlan hp; hp.p = P; hp.d = D; hp.s2 = true;
    Step h; h.kind = Step::HEAD; h.op_index = P.op_index; h.in = P.in; h.out = D.out;
    h.block = (int)heads_.size();
    heads_.push_back(hp);
    tinfo_[P.out].materialized = false;
    steps_.erase(steps_.begin() + i, steps_.begin() + i + 2);
    steps_.insert(steps_.begin() + i, h);
  }
}

// Find   PW(scaled, no act) -> PW(expand, act) -> DW 3x3 s2 (act) -> PW(project)                    = block A
//        -> PW(expand, act) -> DW 3x3 s1 (act) -> PW(project + residual of A's output) -> PW(hswish) = block B
// with act RELU6 or RELU throughout, the channel counts the kernels are compiled for, and the four expanded tensors
// read only inside the run; replace the eight steps by ENC_A (outputs: the project, and the scaled 1x1 as out2) and
// ENC_B (outputs: the hswish 1x1, and the residual sum as out2).  Same arithmetic per output element.
void Engine::detect_enc_blocks() {
  auto reads = [&](const Step& r, int t) { return r.in == t || r.in2 == t || r.scale == t || r.in_add == t || r.residual == t; };
  auto one = [](const Step& s, int want) { return (s.act1 == ACT_NONE && s.act2 == want) || (s.act1 == want && s.act2 == ACT_NONE); };
  auto pw = [&](const Step& s, int in, int act) {
    return s.kind == Step::PW && s.in == in && !s.use_tc && s.up_from < 0 && s.in_add < 0 && s.n4 == s.N && one(s, act);
  };
  auto dw3 = [&](const Step& s, int in, int stride, int act) {
    return s.kind == Step::DW && s.in == in && s.residual < 0 && s.kh == 3 && s.kw == 3 && s.sh == stride && s.sw == stride &&
           s.dh == 1 && s.dw == 1 && one(s, act) && tinfo_[s.out].c == tinfo_[in].c;
  };
  for (size_t i = 0; i + 8 <= steps_.size(); ++i) {
    const Step* s = &steps_[i];
    const int act = s[1].act1 != ACT_NONE ? s[1].act1 : s[1].act2;
    if (act != ACT_RELU6 && act != ACT_RELU) continue;
    if (!(pw(s[0], s[0].in, ACT_NONE) && s[0].scale >= 0 && s[0].residual < 0 &&
          pw(s[1], s[0].out, act) && s[1].scale < 0 && s[1].residual < 0 &&
          dw3(s[2], s[1].out, 2, act) &&
          pw(s[3], s[2].out, ACT_NONE) && s[3].scale < 0 && s[3].residual < 0 &&
          pw(s[4], s[3].out, act) && s[4].scale < 0 && s[4].residual < 0 &&
          dw3(s[5], s[4].out, 1, act) &&
          pw(s[6], s[5].out, ACT_NONE) && s[6].scale < 0 && s[6].residual == s[3].out && s[6].act3 == ACT_NONE &&
          pw(s[7], s[6].out, ACT_HARD_SWISH) && s[7].scale < 0 && s[7].residual < 0))
      continue;
    const TensorInfo& X = tinfo_[s[0].in]; const TensorInfo& T25 = tinfo_[s[0].out]; const TensorInfo& T36 = tinfo_[s[3].out];
    const TensorInfo& T48 = tinfo_[s[6].out]; const TensorInfo& T52 = tinfo_[s[7].out];
    // SAME padding of the stride-2 depthwise: its window of the 1x1 output covers every pixel a tile owns
    if (s[2].pt > 1 || s[2].pl > 1 || T36.h != (T25.h + 1) / 2 || T36.w != (T25.w + 1) / 2 || s[5].pt != 1 || s[5].pl != 1) continue;
    if (T25.h != X.h || T25.w != X.w || T48.h != T36.h || T48.w != T36.w || T52.h != T36.h || T52.w != T36.w) continue;
    if (!enc_blocks_supported(device_, X.c, s[0].N, s[1].N, s[3].N, s[4].N, s[7].N, X.ld, T25.ld, T36.ld, T48.ld, T52.ld) ||
        s[0].K != X.c || s[6].N != s[3].N)
      continue;
    // the expanded tensors are private to the run; the four outputs are materialised
    bool contained = true;
    for (int k : {1, 2, 4, 5}) {
      if (s[k].out == g_.output) contained = false;
      for (size_t r = 0; r < steps_.size() && contained; ++r)
        if ((r < i || r >= i + 8 || (int)(r - i) != k + 1) && reads(steps_[r], s[k].out)) contained = false;
    }
    if (!contained) continue;
    EncPlan ep; ep.act = act;
    for (int k = 0; k < 8; ++k) ep.s[k] = s[k];
    Step a; a.kind = Step::ENC_A; a.op_index = s[0].op_index; a.in = s[0].in; a.scale = s[0].scale; a.out = s[3].out; a.out2 = s[0].out;
    Step b; b.kind = Step::ENC_B; b.op_index = s[4].op_index; b.in = s[3].out; b.out = s[7].out; b.out2 = s[6].out;
    a.block = b.block = (int)encs_.size();
    encs_.push_back(ep);
    for (int k : {1, 2, 4, 5}) tinfo_[s[k].out].materialized = false;
    steps_.erase(steps_.begin() + i, steps_.begin() + i + 8);
    steps_.insert(steps_.begin() + i, {a, b});
    ++i;
  }
}

// Find   DW(strided, from a larger tensor) -> SE -> PW(scaled)  { -> PW(expand) -> DW -> SE -> PW(scaled [+ residual]) }*
//        -> PW -> SE(1 FC, of the narrow tensor) -> MUL(channel scale)
// on tensors of <= 256 pixels and <= 128 channels, with every intermediate read only inside the run, and replace it
// by one CHAIN step (kernels_chain.cu).  Same arithmetic per output element, so results do not change.
bool Engine::detect_chain() {
  const int ns = (int)steps_.size();
  auto px = [&](int t) { return tinfo_[t].h * tinfo_[t].w; };
  auto plain_pw = [&](const Step& s) {
    return s.kind == Step::PW && !s.use_tc && s.in_add < 0 && s.K % 4 == 0 && (size_t)s.K * s.n4 <= 4096 && s.K <= 128 && s.N <= 128;
  };
  auto se_ok = [&](const Step& s, int in, int n_fc, int C) {
    if (s.kind != Step::POOL || s.in != in || s.in2 >= 0 || s.n_fc != n_fc || C > 128) return false;
    for (int k = 0; k < n_fc; ++k) if (s.fc[k].K > 128 || s.fc[k].N > 128) return false;
    return s.fc[0].K == C;
  };
  for (int i = 0; i + 6 < ns; ++i) {
    const Step& d0 = steps_[i];
    if (d0.kind != Step::DW || d0.residual >= 0 || d0.dh != 1 || d0.dw != 1 || d0.kh != d0.kw || (d0.kh != 3 && d0.kh != 5) || d0.sh != d0.sw) continue;
    const TensorInfo& T0 = tinfo_[d0.out];
    const int h = T0.h, w = T0.w, P = h * w;
    if (P > 256 || px(d0.in) <= P || T0.c > 128 || T0.c % 4 || tinfo_[d0.in].ld % 4 || chain_smem_bytes(h, w) == 0) continue;
    std::vector<int> types;
    int j = i + 1, curD = d0.out, curX = -1;
    types.push_back(CH_DWG);
    // entry: SE of D, scaled project into X
    if (!(j + 1 < ns && se_ok(steps_[j], curD, 2, T0.c) && plain_pw(steps_[j + 1]) && steps_[j + 1].in == curD && steps_[j + 1].scale == steps_[j].out &&
          steps_[j + 1].residual < 0 && steps_[j + 1].N <= 32)) continue;
    types.push_back(CH_SE); types.push_back(CH_PW);
    curX = steps_[j + 1].out; j += 2;
    // inverted-residual blocks
    while (j + 3 < ns) {
      const Step& e = steps_[j]; const Step& dd = steps_[j + 1]; const Step& p = steps_[j + 2]; const Step& q = steps_[j + 3];
      const bool ok = plain_pw(e) && e.in == curX && e.scale < 0 && e.residual < 0 && e.K <= 32 &&
                      dd.kind == Step::DW && dd.in == e.out && dd.sh == 1 && dd.sw == 1 && dd.dh == 1 && dd.dw == 1 && dd.residual < 0 &&
                      dd.kh == dd.kw && (dd.kh == 3 || dd.kh == 5) && px(dd.out) == P &&
                      se_ok(p, dd.out, 2, e.N) && plain_pw(q) && q.in == dd.out && q.scale == p.out && q.N <= 32 &&
                      (q.residual < 0 || q.residual == curX);
      if (!ok) break;
      types.push_back(CH_EXPAND_DW); types.push_back(-1); types.push_back(CH_SE); types.push_back(CH_PW);
      curX = q.out; curD = dd.out; j += 4;
    }
    // exit: PW of X into D and SE (one FC) of X, in either graph order, then D * sv -> global
    if (!(j + 2 < ns)) continue;
    const bool pw_first = steps_[j].kind == Step::PW;
    const Step& t0 = steps_[pw_first ? j : j + 1]; const Step& t1 = steps_[pw_first ? j + 1 : j]; const Step& t2 = steps_[j + 2];
    if (!(plain_pw(t0) && t0.in == curX && t0.scale < 0 && t0.residual < 0 && t0.N % 4 == 0 &&
          se_ok(t1, curX, 1, tinfo_[curX].c) && t1.fc[0].N == t0.N &&
          t2.kind == Step::ELT && t2.elt_mode == 3 && t2.in == t0.out && t2.scale == t1.out && tinfo_[t2.out].ld % 4 == 0)) continue;
    if (pw_first) { types.push_back(CH_PW | 256); types.push_back(CH_SE | 256); } else { types.push_back(CH_SE | 256); types.push_back(CH_PW | 256); }
    types.push_back(CH_SCALE_STORE);
    const int jend = j + 2;
    // every tensor produced inside the run (except the last) must be read only inside it
    bool contained = true;
    for (int a = i; a < jend && contained; ++a) {
      const int t = steps_[a].out;
      for (int b = 0; b < ns && contained; ++b) {
        if (b >= i && b <= jend) continue;
        const Step& r = steps_[b];
        for (int u : {r.in, r.in2, r.scale, r.in_add, r.residual}) if (u == t) contained = false;
      }
      if (t == g_.output) contained = false;
    }
    if (!contained) continue;
    ChainPlan cp; cp.h = h; cp.w = w;
    cp.seq.assign(steps_.begin() + i, steps_.begin() + jend + 1);
    cp.types = types;
    for (int a = i; a < jend; ++a) tinfo_[steps_[a].out].materialized = false;
    Step c; c.kind = Step::CHAIN; c.op_index = d0.op_index; c.in = d0.in; c.out = steps_[jend].out; c.block = (int)chains_.size();
    chains_.push_back(cp);
    steps_.erase(steps_.begin() + i, steps_.begin() + jend + 1);
    steps_.insert(steps_.begin() + i, c);
    return true;                                   // one chain per graph
  }
  return false;
}

// ---------------------------------------------------------------------------
// create / destroy
// ---------------------------------------------------------------------------
Engine* Engine::create(const std::string& model_path, int width, int height, int device, int max_batch,
                       unsigned flags, const Callbacks& cb, std::string* err) {
  Engine* e = new Engine();
  e->cb_ = cb; e->W_ = width; e->H_ = height; e->device_ = device; e->max_batch_ = std::max(1, max_batch); e->flags_ = flags;
  auto fail = [&](const std::string& m) { *err = m; delete e; return (Engine*)nullptr; };
  if (width <= 0 || height <= 0 || width > 16384 || height > 16384) return fail("invalid frame size");
  if (!load_tflite(model_path, &e->g_, err)) { delete e; return nullptr; }
  // lib/libbackscrub.cc:194-200
  e->model_type_ = model_type_from_name(model_path);
  if (e->model_type_ == MODEL_UNKNOWN) return fail("unknown model type '" + model_path + "'.");
  // lib/libbackscrub.cc:132-148
  if (e->model_type_ == MODEL_DEEPLAB) { e->scaling_ = (float)(1 / 127.5); e->offset_ = -1.f; }
  else { e->scaling_ = (float)(1 / 255.0); e->offset_ = 0.f; }
  const GTensor& in = e->g_.tensors[e->g_.input]; const GTensor& out = e->g_.tensors[e->g_.output];
  // lib/libbackscrub.cc:85-112: float32, batch 1
  if (in.dtype != 0 || out.dtype != 0) return fail("error: input/output tensor is not float32 type");
  if (in.shape.size() != 4 || out.shape.size() != 4 || in.shape[0] != 1 || out.shape[0] != 1) return fail("error: input/output tensor is not single vector");
  e->mh_ = in.shape[1]; e->mw_ = in.shape[2];
  if (in.shape[3] != 3) return fail("model input must have 3 channels");
  e->oh_ = out.shape[1]; e->ow_ = out.shape[2]; e->oc_ = out.shape[3];
  const int need_oc = e->model_type_ == MODEL_DEEPLAB ? 21 : (e->model_type_ == MODEL_MEET ? 2 : 1);
  if (e->oc_ != need_oc) return fail("model output channel count does not match the model family");
  // lib/libbackscrub.cc:231-246 (float arithmetic, truncating conversion)
  const float ratio = (float)e->mh_ / (float)e->mw_, frameratio = (float)height / (float)width;
  if (frameratio < ratio) {
    e->roidim_[0] = (int)(((float)width - (float)height / ratio) / 2); e->roidim_[1] = 0;
    e->roidim_[2] = (int)((float)height / ratio); e->roidim_[3] = height;
    e->in_roidim_[0] = 0; e->in_roidim_[1] = 0; e->in_roidim_[2] = e->mw_; e->in_roidim_[3] = e->mh_;
  } else {
    e->roidim_[0] = 0; e->roidim_[1] = 0; e->roidim_[2] = width; e->roidim_[3] = height;
    e->in_roidim_[0] = (int)(((float)e->mw_ - (float)e->mh_ / frameratio) / 2); e->in_roidim_[1] = 0;
    e->in_roidim_[2] = (int)((float)e->mh_ / frameratio); e->in_roidim_[3] = e->mh_;
  }
  // documented deviation for models whose output grid differs from the input grid (body-pix):
  // the reference slices ofinal with in_roidim and throws; scale the rectangle by out/in.
  if (e->oh_ == e->mh_ && e->ow_ == e->mw_) std::memcpy(e->out_roidim_, e->in_roidim_, sizeof(e->in_roidim_));
  else {
    e->out_roidim_[0] = e->in_roidim_[0] * e->ow_ / e->mw_; e->out_roidim_[1] = e->in_roidim_[1] * e->oh_ / e->mh_;
    e->out_roidim_[2] = e->in_roidim_[2] * e->ow_ / e->mw_; e->out_roidim_[3] = e->in_roidim_[3] * e->oh_ / e->mh_;
  }
  for (int k = 2; k < 4; ++k)
    if (e->roidim_[k] <= 0 || e->in_roidim_[k] <= 0 || e->out_roidim_[k] <= 0) return fail("degenerate ROI for this frame size");
  if (e->roidim_[0] < 0 || e->roidim_[0] + e->roidim_[2] > width || e->in_roidim_[0] < 0 || e->in_roidim_[0] + e->in_roidim_[2] > e->mw_)
    return fail("ROI outside the frame");
  if (!e->plan(err)) { delete e; return nullptr; }
  if (!e->upload(err)) { delete e; return nullptr; }
  return e;
}

bool Engine::upload(std::string* err) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { *err = "no CUDA device available (this library has no CPU path)"; return false; }
  if (device_ < 0 || device_ >= ndev) { *err = "CUDA device ordinal out of range"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  const size_t B = (size_t)max_batch_;
  CUDA_OK(cudaMalloc((void**)&wblob_, std::max<size_t>(wblob_h_.size(), 64) * 4));
  CUDA_OK(cudaMemcpy(wblob_, wblob_h_.data(), wblob_h_.size() * 4, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMalloc((void**)&arena_, std::max<size_t>(arena_elems_, 64) * 4));
  CUDA_OK(cudaMemset(arena_, 0, std::max<size_t>(arena_elems_, 64) * 4));
  CUDA_OK(cudaMalloc((void**)&rowsum_, std::max<size_t>(rowsum_elems_ * B, 64) * 4));
  CUDA_OK(cudaMalloc((void**)&pool_counters_, B * sizeof(unsigned)));
  CUDA_OK(cudaMemset(pool_counters_, 0, B * sizeof(unsigned)));
  // chain op lists (device pointers into the weight blob / arena are final from here on)
  for (ChainPlan& cp : chains_) {
    std::vector<ChainOp> ops;
    const int ne = (int)cp.seq.size();
    auto fc_of = [&](const Step::Fc& f) {
      FcLayer l; l.w = wblob_ + f.w_off; l.bias = f.has_bias ? wblob_ + f.b_off : nullptr; l.K = f.K; l.N = f.N; l.n4 = f.n4; l.act1 = f.act1; l.act2 = f.act2;
      return l;
    };
    for (int k = 0; k < ne; ++k) {
      if (cp.types[k] < 0) continue;
      const int ty = cp.types[k] & 255;
      const bool tail = (cp.types[k] & 256) != 0;           // the exit pair works on the narrow tensor X
      const Step& st = cp.seq[k];
      ChainOp o{};
      o.type = ty;
      switch (ty) {
        case CH_DWG:
          o.cin = tinfo_[st.out].c; o.wd = wblob_ + st.w_off; o.bd = st.has_bias ? wblob_ + st.b_off : nullptr;
          o.k = st.kh; o.s = st.sh; o.pt = st.pt; o.pl = st.pl; o.dact1 = st.act1; o.dact2 = st.act2;
          o.gin = tptr(st.in); o.gin_ld = tinfo_[st.in].ld; o.ih = tinfo_[st.in].h; o.iw = tinfo_[st.in].w; o.gin_frame = tinfo_[st.in].frame_elems;
          break;
        case CH_SE:
          o.src = tail ? 0 : 1; o.cin = st.fc[0].K; o.pool_act = st.act1; o.n_fc = st.n_fc;
          o.f0 = fc_of(st.fc[0]); if (st.n_fc > 1) o.f1 = fc_of(st.fc[1]);
          break;
        case CH_PW: {
          o.src = tail ? 0 : 1; o.dst = tail ? 1 : 0; o.cin = st.K; o.cout = st.N; o.w = wblob_ + st.w_off; o.b = st.has_bias ? wblob_ + st.b_off : nullptr;
          o.n4 = st.n4; o.act1 = st.act1; o.act2 = st.act2; o.use_scale = st.scale >= 0 ? 1 : 0; o.residual = st.residual >= 0 ? 1 : 0; o.act3 = st.act3;
          break;
        }
        case CH_EXPAND_DW: {
          const Step& dd = cp.seq[k + 1];
          o.cin = st.K; o.cout = st.N; o.w = wblob_ + st.w_off; o.b = st.has_bias ? wblob_ + st.b_off : nullptr; o.n4 = st.n4; o.act1 = st.act1; o.act2 = st.act2;
          o.wd = wblob_ + dd.w_off; o.bd = dd.has_bias ? wblob_ + dd.b_off : nullptr; o.k = dd.kh; o.s = 1; o.pt = dd.pt; o.pl = dd.pl;
          o.dact1 = dd.act1; o.dact2 = dd.act2;
          break;
        }
        case CH_SCALE_STORE:
          o.cin = tinfo_[st.in].c; o.act1 = st.act1; o.gout = tptr(st.out); o.gout_ld = tinfo_[st.out].ld; o.gout_frame = tinfo_[st.out].frame_elems;
          break;
      }
      ops.push_back(o);
    }
    cp.n_ops = (int)ops.size();
    CUDA_OK(cudaMalloc((void**)&cp.d_ops, ops.size() * sizeof(ChainOp)));
    CUDA_OK(cudaMemcpy(cp.d_ops, ops.data(), ops.size() * sizeof(ChainOp), cudaMemcpyHostToDevice));
  }
  // bilateral LUTs (cv::bilateralFilter d=5, sigma 100/100; oracle_img.c:or_bilateral_d5_u8c3)
  {
    std::vector<float> lut(768 + 16, 0.f);
    const double gc = -0.5 / (100.0 * 100.0), gs = -0.5 / (100.0 * 100.0);
    for (int i = 0; i < 768; ++i) lut[i] = (float)std::exp((double)i * i * gc);
    int k = 0;
    for (int i = -2; i <= 2; ++i) for (int j = -2; j <= 2; ++j) {
      const double r = std::sqrt((double)i * i + (double)j * j);
      if (r > 2) continue;
      lut[768 + k++] = (float)std::exp(r * r * gs);
    }
    CUDA_OK(cudaMalloc((void**)&lut_, lut.size() * 4));
    CUDA_OK(cudaMemcpy(lut_, lut.data(), lut.size() * 4, cudaMemcpyHostToDevice));
  }
  const size_t in_px = (size_t)mh_ * mw_, out_px = (size_t)oh_ * ow_, fpx = (size_t)W_ * H_;
  CUDA_OK(cudaMalloc((void**)&in_u8_, B * in_px * 3));
  CUDA_OK(cudaMemset(in_u8_, 0, B * in_px * 3));      // zero padding outside in_roidim stays zero
  CUDA_OK(cudaMalloc((void**)&filt_u8_, B * in_px * 3));
  CUDA_OK(cudaMalloc((void**)&state_, out_px));
  CUDA_OK(cudaMemset(state_, 0, out_px));
  opitch_ = (ow_ + 15) / 16 * 16;
  CUDA_OK(cudaMalloc((void**)&ofinal_, B * (size_t)oh_ * opitch_));
  CUDA_OK(cudaMemset(ofinal_, 0, B * (size_t)oh_ * opitch_));
  CUDA_OK(cudaMalloc((void**)&d_frames_, B * fpx * 3));
  CUDA_OK(cudaMalloc((void**)&d_out_, B * fpx * 3));
  CUDA_OK(cudaMalloc((void**)&d_yuyv_, B * fpx * 2));
  CUDA_OK(cudaMalloc((void**)&d_mask_, B * fpx));
  CUDA_OK(cudaMalloc((void**)&d_yuyv_in_, B * fpx * 2));
  {
    // app/deepseg.cc:603: until a background is set the frame is blended over plain green
    std::vector<uint8_t> green(fpx * 3);
    for (size_t i = 0; i < fpx; ++i) { green[3 * i] = 0; green[3 * i + 1] = 255; green[3 * i + 2] = 0; }
    CUDA_OK(cudaMalloc((void**)&d_bg_, fpx * 3));
    CUDA_OK(cudaMemcpy(d_bg_, green.data(), fpx * 3, cudaMemcpyHostToDevice));
    bg_cap_ = fpx * 3;
    CUDA_OK(cudaMalloc((void**)&d_bg_cursor_, sizeof(int)));
    CUDA_OK(cudaMemset(d_bg_cursor_, 0, sizeof(int)));
    const std::vector<int> ones(B, 1);
    CUDA_OK(cudaMalloc((void**)&d_pass_all_, B * sizeof(int)));
    CUDA_OK(cudaMemcpy(d_pass_all_, ones.data(), B * sizeof(int), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMalloc((void**)&d_live_tab_, B * sizeof(LiveDesc)));
  }
  out_w_ = W_; out_h_ = H_;
  out_cap_ = B * fpx * 3; yuyv_cap_ = B * fpx * 2;
  CUDA_OK(cudaMallocHost((void**)&h_mask_, fpx));
  if (!upload_resize_tab(build_resize_tab(roidim_[2], roidim_[3], in_roidim_[2], in_roidim_[3]), &tab_in_, err)) return false;
  {
    const HostResizeTab up = build_resize_tab(out_roidim_[2], out_roidim_[3], roidim_[2], roidim_[3]);
    if (!upload_resize_tab(up, &tab_up_, err)) return false;
    // patch geometry of the post stage's tiles (k_post_tma): yofs / xofs are monotonic, so the extremes of a halo tile
    // give the rows / columns of the small mask it touches
    const int roi_x = roidim_[0], roi_y = roidim_[1], roi_w = roidim_[2], roi_h = roidim_[3], sw = out_roidim_[2];
    auto span = [&](int lo, int len, int n, const std::vector<int>& first, const std::vector<int>& last, int last_plus, int last_max) {
      const int hi = lo + len - 1;
      const int i0 = lo < 0 ? 0 : std::min(lo, n - 1), i1 = hi >= n ? n - 1 : std::max(hi, 0);
      const int a0 = first[i0], a1 = std::min(last[i1] + last_plus, last_max);
      return make_int2(a0, a1 - a0 + 1);
    };
    geo_nty_ = (H_ + 31) / 32; geo_ntx64_ = (W_ + 63) / 64;
    const int ntx128 = (W_ + 127) / 128;
    std::vector<int2> geo((size_t)geo_nty_ + geo_ntx64_ + ntx128);
    for (int ty = 0; ty < geo_nty_; ++ty) geo[ty] = span(ty * 32 - roi_y - 2, 36, roi_h, up.yofs0, up.yofs1, 0, 1 << 30);
    for (int tx = 0; tx < geo_ntx64_; ++tx) geo[geo_nty_ + tx] = span(tx * 64 - roi_x - 2, 68, roi_w, up.xofs, up.xofs, 1, sw - 1);
    for (int tx = 0; tx < ntx128; ++tx) geo[geo_nty_ + geo_ntx64_ + tx] = span(tx * 128 - roi_x - 2, 132, roi_w, up.xofs, up.xofs, 1, sw - 1);
    CUDA_OK(cudaMalloc((void**)&d_tile_geo_, geo.size() * sizeof(int2)));
    CUDA_OK(cudaMemcpy(d_tile_geo_, geo.data(), geo.size() * sizeof(int2), cudaMemcpyHostToDevice));
    // mask edge refinement: the unclamped cv::resize position of every ROI column / row, and the patch a tile's
    // refinement reaches (taps s - 1 .. s + 2 of its ROI pixels, clamped into the small mask)
    const int sh = out_roidim_[3];
    std::vector<unsigned> taps((size_t)roi_w + roi_h);
    const double scx = resize_scale(sw, roi_w), scy = resize_scale(sh, roi_h);
    for (int x = 0; x < roi_w; ++x) taps[x] = refine_tap(x, scx);
    for (int y = 0; y < roi_h; ++y) taps[(size_t)roi_w + y] = refine_tap(y, scy);
    auto rspan = [&](int lo, int len, int origin, int n_roi, const unsigned* t, int n) {
      const int a = std::max(lo - origin, 0), b = std::min(lo + len - 1 - origin, n_roi - 1);
      if (a > b) return make_int2(0, 1);        // no ROI pixel: the tile loads no patch
      const int r0 = std::max((int)(t[a] & 0xffffu) - 2, 0), r1 = std::min((int)(t[b] & 0xffffu) + 1, n - 1);
      return make_int2(r0, r1 - r0 + 1);
    };
    std::vector<int2> geo_r(geo.size());
    for (int ty = 0; ty < geo_nty_; ++ty) geo_r[ty] = rspan(ty * 32, 32, roi_y, roi_h, taps.data() + roi_w, sh);
    for (int tx = 0; tx < geo_ntx64_; ++tx) geo_r[geo_nty_ + tx] = rspan(tx * 64, 64, roi_x, roi_w, taps.data(), sw);
    for (int tx = 0; tx < ntx128; ++tx) geo_r[geo_nty_ + geo_ntx64_ + tx] = rspan(tx * 128, 128, roi_x, roi_w, taps.data(), sw);
    CUDA_OK(cudaMalloc((void**)&d_refine_taps_, taps.size() * sizeof(unsigned)));
    CUDA_OK(cudaMemcpy(d_refine_taps_, taps.data(), taps.size() * sizeof(unsigned), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMalloc((void**)&d_tile_geo_r_, geo_r.size() * sizeof(int2)));
    CUDA_OK(cudaMemcpy(d_tile_geo_r_, geo_r.data(), geo_r.size() * sizeof(int2), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMalloc((void**)&d_refine_, (size_t)max_batch_ * sizeof(int)));
  }
  if (!refresh_bg_yuyv(err)) return false;
  // the Gaussian's tap tables must exist before a launch is captured into a graph
  if (!gauss_tables_ready()) { *err = "could not allocate the Gaussian tap tables"; return false; }
  // wait for the copies and kernels above: they ran on the legacy default stream and on stream_.  Not a device-wide
  // synchronise: that is refused while another thread's context captures a graph, and it breaks that capture.
  CUDA_OK(cudaStreamSynchronize(0));
  CUDA_OK(cudaStreamSynchronize(stream_));
  return true;
}

Engine::~Engine() {
#ifndef BSB_EMU
  for (auto& kv : graphs_) cudaGraphExecDestroy(kv.second.exec);
#endif
  if (stream_) { cudaStreamSynchronize(stream_); }
  for (void* p : {(void*)wblob_, (void*)arena_, (void*)lut_, (void*)rowsum_, (void*)in_u8_, (void*)filt_u8_, (void*)state_, (void*)ofinal_,
                  (void*)d_frames_, (void*)d_out_, (void*)d_yuyv_, (void*)d_mask_, (void*)d_bg_, (void*)d_bg_raw_, (void*)d_yuyv_in_,
                  tab_in_.blob, tab_up_.blob, tab_bg_.blob, tab_out_.blob, (void*)d_bg_cursor_, (void*)d_bg_eff_, (void*)d_bg_frames_,
                  (void*)d_gauss_tmp_, (void*)d_stage_a_, (void*)d_bg_yuyv_, (void*)pool_counters_, (void*)d_tile_geo_,
                  (void*)d_bg_nv12_, (void*)d_nv12_})
    if (p) cudaFree(p);
  for (ChainPlan& cp : chains_) if (cp.d_ops) cudaFree(cp.d_ops);
  free_sources();
  for (void* p : {(void*)d_src_tab_, (void*)d_src_raw_, tab_src_.blob, (void*)d_pass_all_, (void*)d_live_tab_, (void*)d_live_stage_, (void*)d_seg_tab_,
                  (void*)d_frame_tab_, (void*)d_crop_, (void*)d_frame_box_, (void*)d_frame_counter_, (void*)d_frame_state_,
                  (void*)d_refine_, (void*)d_refine_taps_, (void*)d_tile_geo_r_, (void*)d_mblur_mask_, (void*)d_mgauss_tmp_})
    if (p) cudaFree(p);
  for (LiveSize& l : live_sizes_) if (l.tab.blob) cudaFree(l.tab.blob);
  if (h_mask_) cudaFreeHost(h_mask_);
  if (stream_) cudaStreamDestroy(stream_);
}

// ---------------------------------------------------------------------------
// enqueue: the per-call kernel sequence (captured into a CUDA graph by run())
// ---------------------------------------------------------------------------
void Engine::enqueue_pre(const Call& c, int m, const int* gather) {
  // camera YUYV / NV12 frames are read in place (each bilinear tap converted like cv::COLOR_YUV2BGR_YUYV / _NV12 would have)
  launch_resize_roi_swap(stream_, m, c.in, c.stride, c.pitch, roidim_[0], roidim_[1], roidim_[2], roidim_[3], tab_in_.tab,
                         in_u8_, mw_, mh_, in_roidim_[0], in_roidim_[1], in_roidim_[2], in_roidim_[3], tab_in_.area2x2, c.fmt, c.uv, gather);
  // with the fused stem the fp32 input tensor is only materialised for introspection (KEEP_TENSORS)
  float* f32 = (stem_u8_ok_ && !(flags_ & 1u)) ? nullptr : tptr(g_.input);
  launch_bilateral_norm(stream_, m, in_u8_, mw_, mh_, lut_, lut_ + 768, scaling_, offset_, f32, filt_u8_);
}

// Frames per pass of a sub-batched segment: the segment's largest tensor, in and out, should stay L2-resident
// (tuning().sub_batch_mb megabytes per tensor; 0 = off).
static int sub_batch_frames(size_t frame_bytes, int n) {
  const size_t budget = (size_t)tuning().sub_batch_mb << 20;
  if (!budget || !frame_bytes) return n;
  const size_t f = std::max<size_t>(1, budget / frame_bytes);
  return (int)std::min<size_t>(f, (size_t)n);
}

void Engine::enqueue_cnn(int n, bool from_u8) {
  bool first = true;
  bool skip_next = false;
  for (size_t si = 0; si < steps_.size(); ++si) {
    if (si < seg_len_.size() && seg_len_[si] > 0) {
      const int sub = sub_batch_frames(seg_frame_bytes_[si], n);
      if (sub < n) {
        const size_t end = si + (size_t)seg_len_[si];
        for (int f0 = 0; f0 < n; f0 += sub) {
          frame_off_ = f0;
          for (size_t k = si; k < end; ++k) run_step(k, std::min(sub, n - f0), from_u8, &first, &skip_next);
        }
        frame_off_ = 0;
        si = end - 1;
        continue;
      }
    }
    run_step(si, n, from_u8, &first, &skip_next);
  }
}

// Segments: maximal runs of plain per-frame steps (1x1 conv, depthwise, element-wise, copy, resize) that touch a tensor
// of more than 1 MB per frame.  Everything in such a run depends only on its own frame, so the run can be executed
// frame-group by frame-group.
void Engine::find_segments() {
  seg_len_.assign(steps_.size(), 0);
  seg_frame_bytes_.assign(steps_.size(), 0);
  if (tuning().sub_batch_mb <= 0) return;       // off: no segments, the arena recycles buffers step by step as before
  auto plain = [&](const Step& st) {
    return st.kind == Step::PW || st.kind == Step::DW || st.kind == Step::ELT || st.kind == Step::COPY || st.kind == Step::RESIZE;
  };
  auto fbytes = [&](const Step& st) {
    size_t m = 0;
    for (int t : {st.in, st.in2, st.in_add, st.residual, st.out, st.up_from})
      if (t >= 0) m = std::max(m, tinfo_[tinfo_[t].alias_parent >= 0 ? tinfo_[t].alias_parent : t].frame_elems * sizeof(float));
    return m;
  };
  for (size_t i = 0; i < steps_.size();) {
    if (!plain(steps_[i])) { ++i; continue; }
    size_t j = i, big = 0;
    while (j < steps_.size() && plain(steps_[j])) { big = std::max(big, fbytes(steps_[j])); ++j; }
    if (big > ((size_t)1 << 20) && j - i >= 2) { seg_len_[i] = (int)(j - i); seg_frame_bytes_[i] = big; }
    i = j;
  }
}

void Engine::run_step(size_t si, int n, bool from_u8, bool* first_p, bool* skip_next_p) {
  bool& first = *first_p;
  bool& skip_next = *skip_next_p;
  {
    const Step& st = steps_[si];
    if (skip_next) { skip_next = false; return; }        // the 1x1 conv that ran inside the stem kernel
    if (from_u8 && (int)si == dec_up_step_) return;      // pipeline call: the decision kernel interpolates on the fly
    const bool fused_stem = first && from_u8 && stem_u8_ok_;
    first = false;
    const TensorInfo& I = tinfo_[st.in];
    const TensorInfo& O = tinfo_[st.out];
    Epilogue e;
    e.bias = st.has_bias ? wblob_ + st.b_off : nullptr;
    e.act1 = st.act1; e.act2 = st.act2; e.act3 = st.act3;
    if (st.residual >= 0) { e.residual = tptr(st.residual); e.ld_res = tinfo_[st.residual].ld; }
    switch (st.kind) {
      case Step::CONV:
        if (fused_stem) {
          // the thread that produced a stem pixel holds its 16 channels: a following plain 16 -> 16 1x1 conv runs there too
          const Step* pw = (stem_pw_ok_ && tuning().stem_pw && si + 1 < steps_.size()) ? &steps_[si + 1] : nullptr;
          if (pw) {
            Epilogue e2;
            e2.bias = pw->has_bias ? wblob_ + pw->b_off : nullptr; e2.act1 = pw->act1; e2.act2 = pw->act2;
            launch_stem_u8(stream_, n, filt_u8_, I.h, I.w, scaling_, offset_, wblob_ + st.w_off, st.kh, st.kw, st.sh, st.sw, st.pt, st.pl,
                           tptr(st.out), O.h, O.w, O.ld, e, wblob_ + pw->w_off, tptr(pw->out), tinfo_[pw->out].ld, &e2);
            skip_next = true;
          } else {
            launch_stem_u8(stream_, n, filt_u8_, I.h, I.w, scaling_, offset_, wblob_ + st.w_off, st.kh, st.kw, st.sh, st.sw, st.pt, st.pl,
                           tptr(st.out), O.h, O.w, O.ld, e);
          }
          break;
        }
        launch_conv_direct(stream_, n, tptr(st.in), I.h, I.w, I.c, I.ld, wblob_ + st.w_off, st.N, st.kh, st.kw, st.sh, st.sw,
                           st.dh, st.dw, st.pt, st.pl, tptr(st.out), O.h, O.w, O.ld, e);
        break;
      case Step::PW:
        if (st.up_from >= 0) {
          const TensorInfo& S = tinfo_[st.up_from];
          launch_upsample_pw(stream_, n, tptr(st.up_from), S.h, S.w, st.K, S.ld, st.align_corners, st.half_pixel, wblob_ + st.w_off, st.n4, st.N,
                             tptr(st.out), O.h, O.w, O.ld, e);
          break;
        }
        if (st.use_tc && launch_pointwise_tc(stream_, n * I.h * I.w, st.K, st.N, tptr(st.in), I.ld, wblob_ + st.tc_hi_off, wblob_ + st.tc_lo_off,
                                             st.kpad, st.npad, tptr(st.out), O.ld, e))
          break;
        launch_pointwise(stream_, n * I.h * I.w, st.K, st.N, tptr(st.in), I.ld, wblob_ + st.w_off, st.n4, tptr(st.out), O.ld, e,
                         st.scale >= 0 ? tptr(st.scale) : nullptr, I.h * I.w,
                         st.in_add >= 0 ? tptr(st.in_add) : nullptr, st.in_add >= 0 ? tinfo_[st.in_add].ld : 0);
        break;
      case Step::DW:
        launch_depthwise(stream_, n, tptr(st.in), I.h, I.w, I.c, I.ld, wblob_ + st.w_off, st.kh, st.kw, st.sh, st.sw, st.dh, st.dw,
                         st.pt, st.pl, tptr(st.out), O.h, O.w, O.ld, e);
        break;
      case Step::POOL: {
        FcLayer fc[2];
        for (int k = 0; k < st.n_fc; ++k) {
          fc[k].w = wblob_ + st.fc[k].w_off; fc[k].bias = st.fc[k].has_bias ? wblob_ + st.fc[k].b_off : nullptr;
          fc[k].K = st.fc[k].K; fc[k].N = st.fc[k].N; fc[k].n4 = st.fc[k].n4; fc[k].act1 = st.fc[k].act1; fc[k].act2 = st.fc[k].act2;
        }
        const bool two = st.in2 >= 0;
        launch_pool_fc(stream_, n, tptr(st.in), I.c, I.ld, two ? tptr(st.in2) : nullptr, two ? tinfo_[st.in2].c : 0,
                       two ? tinfo_[st.in2].ld : 0, I.h, I.w, rowsum_, st.act1, nullptr, st.n_fc, fc, tptr(st.out), O.ld, pool_counters_);
        break;
      }
      case Step::RESIZE:
        launch_resize_bilinear(stream_, n, tptr(st.in), I.h, I.w, I.c, I.ld, tptr(st.out), O.h, O.w, O.ld, st.align_corners, st.half_pixel);
        break;
      case Step::TCONV:
        launch_tconv2x2(stream_, n, tptr(st.in), I.h, I.w, I.c, I.ld, wblob_ + st.w_off, wblob_ + st.b_off, st.N, tptr(st.out), O.h, O.w, O.ld, st.act2);
        break;
      case Step::ELT:
        launch_eltwise(stream_, st.elt_mode, n, I.h * I.w, I.c, tptr(st.in), I.ld, st.in2 >= 0 ? tptr(st.in2) : nullptr,
                       st.in2 >= 0 ? tinfo_[st.in2].ld : 0, st.scale >= 0 ? tptr(st.scale) : nullptr, tptr(st.out), O.ld, st.act1);
        break;
      case Step::BLOCK: {
        const FusedBlock& fb = blocks_[st.block];
        MbBlockArgs a{};
        a.x = tptr(st.in); a.ld_x = I.ld; a.y = tptr(st.out); a.ld_y = O.ld;
        a.h = I.h; a.w = I.w; a.cin = I.c; a.cexp = fb.expand.N; a.cout = fb.project.N;
        a.w1 = wblob_ + fb.expand.w_off; a.b1 = fb.expand.has_bias ? wblob_ + fb.expand.b_off : nullptr; a.n4_1 = fb.expand.n4;
        a.a1a = fb.expand.act1; a.a1b = fb.expand.act2;
        a.wd = wblob_ + fb.dw.w_off; a.bd = fb.dw.has_bias ? wblob_ + fb.dw.b_off : nullptr; a.k = fb.dw.kh; a.pt = fb.dw.pt; a.pl = fb.dw.pl;
        a.ada = fb.dw.act1; a.adb = fb.dw.act2;
        a.pool_act = fb.pool.act1;
        FcLayer* fl[2] = {&a.f0, &a.f1};
        for (int k = 0; k < 2; ++k) {
          fl[k]->w = wblob_ + fb.pool.fc[k].w_off; fl[k]->bias = fb.pool.fc[k].has_bias ? wblob_ + fb.pool.fc[k].b_off : nullptr;
          fl[k]->K = fb.pool.fc[k].K; fl[k]->N = fb.pool.fc[k].N; fl[k]->n4 = fb.pool.fc[k].n4; fl[k]->act1 = fb.pool.fc[k].act1; fl[k]->act2 = fb.pool.fc[k].act2;
        }
        a.w2 = wblob_ + fb.project.w_off; a.b2 = fb.project.has_bias ? wblob_ + fb.project.b_off : nullptr; a.n4_2 = fb.project.n4;
        a.a2a = fb.project.act1; a.a2b = fb.project.act2; a.residual = fb.project.residual >= 0 ? 1 : 0; a.a3 = fb.project.act3;
        launch_mb_block(stream_, n, a);
        break;
      }
      case Step::HEAD: {
        const HeadPlan& hp = heads_[st.block];
        const Step& P = hp.p; const Step& D = hp.d; const Step& T = hp.t;
        if (hp.s2) {
          launch_pw_dws2(stream_, tptr(P.in), I.ld, wblob_ + P.w_off, P.has_bias ? wblob_ + P.b_off : nullptr, P.act1 != ACT_NONE ? P.act1 : P.act2,
                         wblob_ + D.w_off, D.has_bias ? wblob_ + D.b_off : nullptr, D.act1 != ACT_NONE ? D.act1 : D.act2,
                         tptr(st.out), O.ld, n, I.h, I.w, O.h, O.w, D.pt, D.pl);
          break;
        }
        launch_head(stream_, P.N, tptr(P.in), I.ld, P.scale >= 0 ? tptr(P.scale) : nullptr, P.in_add >= 0 ? tptr(P.in_add) : nullptr,
                    P.in_add >= 0 ? tinfo_[P.in_add].ld : 0, wblob_ + P.w_off, P.has_bias ? wblob_ + P.b_off : nullptr, P.act1, P.act2,
                    wblob_ + D.w_off, D.has_bias ? wblob_ + D.b_off : nullptr, D.act1, D.act2, D.act3,
                    hp.has_t ? wblob_ + T.w_off : nullptr, hp.has_t ? wblob_ + T.b_off : nullptr, hp.has_t ? T.N : 0, hp.has_t ? T.act2 : 0,
                    tptr(st.out), O.ld, n, I.h, I.w, D.pt, D.pl);
        break;
      }
      case Step::ENC_A:
      case Step::ENC_B: {
        const EncPlan& ep = encs_[st.block];
        const Step* s = ep.s;
        EncBlocksArgs a{};
        a.x = tptr(s[0].in); a.ld_x = tinfo_[s[0].in].ld; a.sv = tptr(s[0].scale);
        for (int k = 0, pwk = 0; k < 8; ++k) {
          if (s[k].kind != Step::PW) continue;
          a.w[pwk] = wblob_ + s[k].w_off; a.b[pwk] = s[k].has_bias ? wblob_ + s[k].b_off : nullptr; ++pwk;
        }
        for (int d = 0; d < 2; ++d) { const Step& D = s[d ? 5 : 2]; a.wd[d] = wblob_ + D.w_off; a.bd[d] = D.has_bias ? wblob_ + D.b_off : nullptr; }
        a.t25 = tptr(s[0].out); a.ld25 = tinfo_[s[0].out].ld; a.t36 = tptr(s[3].out); a.ld36 = tinfo_[s[3].out].ld;
        a.t48 = tptr(s[6].out); a.ld48 = tinfo_[s[6].out].ld; a.t52 = tptr(s[7].out); a.ld52 = tinfo_[s[7].out].ld;
        a.ih = tinfo_[s[0].out].h; a.iw = tinfo_[s[0].out].w; a.oh = tinfo_[s[3].out].h; a.ow = tinfo_[s[3].out].w;
        a.pt_a = s[2].pt; a.pl_a = s[2].pl; a.act = ep.act;
        launch_enc_blocks(stream_, n, a, st.kind == Step::ENC_B);
        break;
      }
      case Step::CHAIN: {
        const ChainPlan& cp = chains_[st.block];
        launch_chain(stream_, n, cp.h, cp.w, cp.d_ops, cp.n_ops);
        break;
      }
      case Step::COPY:
        launch_copy_channels(stream_, n * I.h * I.w, I.c, tptr(st.in), I.ld, tptr(st.out) + st.copy_off, O.ld);
        break;
    }
  }
}

// sources: per-source states, looked up through the id table.  n call frames, m of them segmented (the CNN batch; m == n
// with null rows when none is held).  Sources calls launch over the n frames, plain calls over the m decisions.
void Engine::enqueue_decision(int n, bool sources, int m, const SegRows& seg) {
  if (dec_up_step_ >= 0) {
    const Step& st = steps_[dec_up_step_];
    const TensorInfo& I = tinfo_[st.in];
    if (sources)
      launch_decision_up_sources(stream_, n, tptr(st.in), I.h, I.w, I.ld, st.align_corners, st.half_pixel, oh_, ow_, src_state_, d_src_tab_,
                                 ofinal_, opitch_, seg.cidx);
    else
      launch_decision_up_iir(stream_, m, tptr(st.in), I.h, I.w, I.ld, st.align_corners, st.half_pixel, oh_, ow_, state_, ofinal_, opitch_, seg);
    return;
  }
  if (sources) launch_decision_sources(stream_, model_type_, n, tptr(g_.output), oh_, ow_, oc_, src_state_, d_src_tab_, ofinal_, opitch_, seg.cidx);
  else launch_decision_iir(stream_, model_type_, m, tptr(g_.output), oh_, ow_, oc_, state_, ofinal_, opitch_, seg);
}

// Mask interval: plain frame c (counted over the context's plain calls) is segmented iff c % k == 0; frame f of source s
// iff f == 0 || (f + s) % k_s == 0 (the id as the phase staggers sources with consecutive ids, and a new or reset camera
// always starts with a mask of its own).
int Engine::segment(const Call& c, std::vector<int>* rows) const {
  const int n = c.n;
  if (fed_ || (!c.ids && mask_interval_ == 1)) return n;
  rows->assign(3 * (size_t)max_batch_, -1);
  int m = 0;
  for (int b = 0; b < n; ++b) {
    bool seg;
    if (c.ids) {
      const int s = c.ids[b];
      seg = src_frames_[s] == 0 || (src_frames_[s] + s) % src_interval(s) == 0;
    } else {
      seg = (plain_frames_ + b) % mask_interval_ == 0;
    }
    if (seg) { (*rows)[m] = b; (*rows)[(size_t)max_batch_ + b] = m; ++m; }
    (*rows)[2 * (size_t)max_batch_ + b] = m - 1;
  }
  return m;
}

SegRows Engine::seg_rows(const Call& c, const Plan& p) const {
  if (p.m == c.n) return SegRows{};
  const size_t mb = (size_t)max_batch_;
  if (p.mode == CALL_PLAIN) return SegRows{c.n, d_seg_tab_, d_seg_tab_ + mb, d_seg_tab_ + 2 * mb};
  const int* t = d_src_tab_ + SRC_TAB_SEG * mb;
  return SegRows{c.n, t, t + mb, nullptr};
}

void Engine::count_frames(const Call& c) {
  if (fed_) return;
  if (!c.ids) { plain_frames_ += c.n; return; }
  for (int b = 0; b < c.n; ++b) ++src_frames_[c.ids[b]];
}

bool Engine::set_mask_interval(int k, std::string* err) {
  if (k < 1 || k > MASK_INTERVAL_MAX) { *err = "mask interval out of range (1..256)"; return false; }
  mask_interval_ = k;
  return true;
}

bool Engine::set_source_mask_interval(int source, int k, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (k != -1 && (k < 1 || k > MASK_INTERVAL_MAX)) { *err = "source mask interval out of range (-1, or 1..256)"; return false; }
  src_interval_[source] = k;
  return true;
}

bool Engine::framing_rows(const Call& c, std::vector<int>* rows) const {
  bool any = false;
  for (int b = 0; b < c.n && !any; ++b) any = frame_framing(c.ids ? c.ids[b] : -1).mode != FRAMING_OFF;
  if (!any) return false;
  const size_t mb = (size_t)max_batch_;
  rows->assign(FRAMING_ROWS * mb, 0);
  int* r = rows->data();
  const int full[4] = {0, 0, W_, H_};
  for (int b = 0; b < c.n; ++b) {
    const int id = c.ids ? c.ids[b] : -1;
    const Framing& f = frame_framing(id);
    int ow = out_w_, oh = out_h_;
    if (c.ids) source_output_size(id, &ow, &oh);
    r[b] = f.mode;
    r[mb + b] = c.ids ? src_jump_[id] : (b == 0 && plain_jump_);    // a plain call's later frames follow its first
    r[2 * mb + b] = c.ids ? id : 0;
    r[3 * mb + b] = ow; r[4 * mb + b] = oh;
    for (int k = 0; k < 4; ++k) r[(5 + k) * mb + b] = f.mode == FRAMING_RECT ? f.rect[k] : full[k];
    r[9 * mb + b] = c.ids ? b : c.frame0 + b;                        // a split host-buffer call's crops by caller frame
  }
  return true;
}

void Engine::count_framing(const Call& c, const Plan& p) {
  last_framed_ = p.framed;
  last_frames_ = c.ids ? c.n : c.frame0 + c.n;
  if (!c.ids) { plain_jump_ = framing_.mode != FRAMING_AUTO; return; }
  for (int b = 0; b < c.n; ++b) src_jump_[c.ids[b]] = frame_framing(c.ids[b]).mode != FRAMING_AUTO;
}

void Engine::enqueue_framing(const Call& c) {
  FramingArgs a{};
  a.n = c.n; a.ofinal = ofinal_; a.oh = oh_; a.opitch = opitch_; a.ox = out_roidim_[0]; a.oy = out_roidim_[1];
  a.g = FramingGeo{W_, H_, roidim_[0], roidim_[1], roidim_[2], roidim_[3], out_roidim_[2], out_roidim_[3]};
  a.p = framing_auto_;
  a.tab = d_frame_tab_; a.mb = max_batch_;
  a.state = c.ids ? d_src_frame_state_ : d_frame_state_;
  a.crop = d_crop_; a.targets = d_frame_box_; a.counter = d_frame_counter_; a.plain = c.ids ? 0 : 1;
  launch_framing(stream_, a);
}

namespace {
bool check_framing(int mode, int x, int y, int w, int h, int W, int H, bool follow, std::string* err) {
  if (mode < (follow ? -1 : FRAMING_OFF) || mode > FRAMING_AUTO) {
    *err = follow ? "source framing mode must be -1 (follow the context), BSB_FRAMING_OFF, BSB_FRAMING_RECT or BSB_FRAMING_AUTO"
                  : "framing mode must be BSB_FRAMING_OFF, BSB_FRAMING_RECT or BSB_FRAMING_AUTO";
    return false;
  }
  if (mode == FRAMING_RECT && (x < 0 || y < 0 || w < 1 || h < 1 || (long)x + w > W || (long)y + h > H)) {
    *err = "framing rectangle must lie inside the frame, with w and h >= 1";
    return false;
  }
  return true;
}
}  // namespace

bool Engine::set_mask_refine(int sigma, std::string* err) {
  if (sigma < 0 || sigma > 255) { *err = "mask refinement strength must be 0 (off) .. 255"; return false; }
  refine_ = sigma;
  return true;
}

bool Engine::set_source_mask_refine(int source, int sigma, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (sigma < -1 || sigma > 255) { *err = "source mask refinement strength must be -1 (follow the context) or 0 (off) .. 255"; return false; }
  src_refine_[source] = (short)sigma;
  return true;
}

bool Engine::set_blur_mode(int mode, std::string* err) {
  if (mode != BLUR_PLAIN && mode != BLUR_MASKED) { *err = "blur mode must be BSB_BLUR_PLAIN (0) or BSB_BLUR_MASKED (1)"; return false; }
  blur_mode_ = mode;
  return true;
}

bool Engine::set_source_blur_mode(int source, int mode, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (mode < -1 || mode > BLUR_MASKED) { *err = "source blur mode must be -1 (follow the context), BSB_BLUR_PLAIN (0) or BSB_BLUR_MASKED (1)"; return false; }
  src_blur_mode_[source] = (signed char)mode;
  return true;
}

bool Engine::set_framing(int mode, int x, int y, int w, int h, std::string* err) {
  if (!check_framing(mode, x, y, w, h, W_, H_, false, err)) return false;
  framing_ = Framing{mode, {x, y, w, h}};
  return true;
}

bool Engine::set_framing_auto(int max_zoom, int margin, int speed, std::string* err) {
  if (max_zoom < 100 || max_zoom > 1000) { *err = "framing max_zoom_pct out of range (100..1000)"; return false; }
  if (margin < 0 || margin > 100) { *err = "framing margin_pct out of range (0..100)"; return false; }
  if (speed < 1 || speed > 256) { *err = "framing speed out of range (1..256)"; return false; }
  // the parameters are kernel arguments of the captured calls
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  drop_graphs();
  framing_auto_ = FramingParams{max_zoom, margin, speed};
  return true;
}

bool Engine::set_source_framing(int source, int mode, int x, int y, int w, int h, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (!check_framing(mode, x, y, w, h, W_, H_, true, err)) return false;
  src_framing_[source] = Framing{mode, {x, y, w, h}};
  return true;
}

bool Engine::get_framing(int frame, int* rect, std::string* err) {
  if (frame < 0 || frame >= last_frames_) { *err = "frame out of range (0 .. the last call's n_frames - 1)"; return false; }
  if (!last_framed_) { rect[0] = 0; rect[1] = 0; rect[2] = W_; rect[3] = H_; return true; }
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  CUDA_OK(cudaMemcpy(rect, d_crop_ + frame, 4 * sizeof(int), cudaMemcpyDeviceToHost));
  return true;
}

// PostArgs of one call.  p.native: the post kernel reads the camera frames in place — YUYV, or NV12, which then also
// writes its video output as NV12; p.nv12_staged: the video output goes to d_yuyv_ as YUYV.
PostArgs Engine::post_args(const Call& c, const Plan& p) const {
  const size_t fbytes = (size_t)W_ * H_ * 3;
  const bool tail = call_tail(p);
  const bool nv12_in = p.native && c.fmt == IN_NV12;
  PostArgs a{};
  a.B = c.n; a.W = W_; a.H = H_;
  if (c.fmt == IN_BGR) { a.frames = c.in; a.frame_pitch = c.pitch; a.frame_stride = c.stride; }
  else { a.frames = d_frames_; a.frame_pitch = (size_t)W_ * 3; a.frame_stride = fbytes; }   // YUYV / NV12: the staging they are converted into
  if (nv12_in) {
    a.nv12_in = c.in; a.nv12_in_pitch = c.pitch; a.nv12_in_uv = c.uv; a.nv12_in_stride = c.stride;
  } else {
    a.yuyv_in = p.native ? c.in : nullptr; a.yuyv_in_stride = (size_t)W_ * H_ * 2;
  }
  a.bg = d_bg_; a.bg_pitch = (size_t)W_ * 3; a.bg_stride = 0;
  if (p.mode == CALL_PLAIN && p.live) {
    // the resized (and blurred) live images, written by enqueue_post into the per-frame background frames; no YUYV cache
    a.bg = d_bg_frames_; a.bg_stride = p.live == 2 ? fbytes : 0;
  } else if (has_bg_) {
    if (bgblur_k_) a.bg = d_bg_eff_;                       // blurred once, when the background / strength was set
    if (bg_count_ > 1) { a.bg_stride = fbytes; a.bg_cursor = d_bg_cursor_; a.bg_count = bg_count_; a.bg_advance = bg_advance_; }
  } else if (bgblur_k_ && blends(c, p) && !p.passed) {
    a.bg = d_bg_frames_; a.bg_stride = fbytes;            // the blurred camera frame itself (filled by enqueue_post)
  }
  if (bg_yuyv_valid_ && !(bgblur_k_ && !has_bg_) && !p.live) { a.bg_yuyv = d_bg_yuyv_; a.bg_nv12 = bg_nv12_valid_ ? d_bg_nv12_ : nullptr; }
  if (p.mode != CALL_PLAIN) {
    // sources: frame b blends bank slot bg_index[b]; the camera-blur slots' YUYV / NV12 are written by the call's
    // Gaussian, so every slot's cached copy is valid.  A call whose every frame is camera blur runs without them, as a
    // plain context in camera-blur mode does: each slot is read by one tile only, and converting the blurred BGR tile
    // the kernel loads anyway is cheaper than writing and re-reading a YUYV copy.
    a.bg = d_bank_; a.bg_stride = fbytes; a.bg_cursor = nullptr; a.bg_advance = 0;
    a.bg_index = d_src_tab_ + max_batch_; a.bg_count = bank_slots();
    a.bg_yuyv = (!p.all_blur && !(W_ & 1)) ? d_bank_yuyv_ : nullptr;
    a.bg_nv12 = p.all_blur ? nullptr : d_bank_nv12_;
  }
  // the cached background in the call's video format (NV12 where the kernel writes NV12, else YUYV)
  if (nv12_in) a.bg_yuyv = nullptr; else a.bg_nv12 = nullptr;
  a.ofinal = ofinal_; a.ow = ow_; a.oh = oh_; a.opitch = opitch_;
  a.out_x = out_roidim_[0]; a.out_y = out_roidim_[1]; a.out_w = out_roidim_[2]; a.out_h = out_roidim_[3];
  a.roi_x = roidim_[0]; a.roi_y = roidim_[1]; a.roi_w = roidim_[2]; a.roi_h = roidim_[3];
  a.tab = tab_up_.tab; a.area2x2 = tab_up_.area2x2;
  a.out_pitch = (size_t)W_ * 3;
  if (!tail) {
    a.out = p.bgra ? nullptr : c.out; a.out_stride = c.out_stride;
    if (p.bgra) { a.bgra = c.out; a.bgra_pitch = (size_t)W_ * 4; a.bgra_stride = c.out_stride; }
    uint8_t* video = p.nv12_staged ? d_yuyv_ : c.video;
    const size_t vstride = p.nv12_staged ? (size_t)W_ * H_ * 2 : c.video_stride;
    if (nv12_in) { a.nv12 = video; a.nv12_stride = vstride; }
    else { a.yuyv = video; a.yuyv_stride = vstride; }
    // sources calls with flipped frames and no tail: k_post_tma writes the frames of the table's flip row mirrored.
    // Without flipped frames no table is passed, and the post kernel runs as for a plain call.
    if (p.mode != CALL_PLAIN && p.flipped) a.flip = d_src_tab_ + 3 * (size_t)max_batch_;
  } else {
    // the tail reads the staged BGR composites for the video (and a BGR output), the staged BGRA frames for a BGRA output
    a.out = blends(c, p) ? d_stage_a_ : nullptr; a.out_stride = fbytes;
    a.yuyv = nullptr; a.yuyv_stride = 0;
    if (p.bgra) { a.bgra = d_stage_a_ + stage_bgra_off(c, p); a.bgra_pitch = (size_t)W_ * 4; a.bgra_stride = (size_t)W_ * H_ * 4; }
  }
  a.mask = c.mask; a.mask_stride = c.mask_stride;
  // frames whose filter is off (app/deepseg.cc:639-664): the post kernel passes their camera frame through.  A call without
  // any passes no table, and its post kernel runs as before.
  if (p.passed) a.pass = p.mode == CALL_PLAIN ? d_pass_all_ : d_src_tab_ + 5 * (size_t)max_batch_;
  a.geo_rows = d_tile_geo_; a.geo_cols64 = d_tile_geo_ + geo_nty_; a.geo_cols128 = d_tile_geo_ + geo_nty_ + geo_ntx64_;
  // refined frames: the strength table, written before the launch.  A call without one passes no table, and its post
  // kernel runs as before.
  if (p.refined) {
    a.refine = d_refine_; a.refine_w = refine_w_; a.refine_x = d_refine_taps_; a.refine_y = d_refine_taps_ + roidim_[2];
    a.geo_r_rows = d_tile_geo_r_; a.geo_r_cols64 = d_tile_geo_r_ + geo_nty_; a.geo_r_cols128 = d_tile_geo_r_ + geo_nty_ + geo_ntx64_;
  }
  return a;
}

bool Engine::enqueue_post(const Call& c, const Plan& p) {
  const int n = c.n;
  const size_t fbytes = (size_t)W_ * H_ * 3;
  const bool tail = call_tail(p);
  const bool want_rgb = c.out || c.video;
  const bool ring = p.mode == CALL_PLAIN && has_bg_ && bg_count_ > 1;
  const PostArgs a = post_args(c, p);
  // app/deepseg.cc:652-658: no background source => the background is the blurred camera frame itself (sources: frame b
  // at its own strength into the bank's camera-blur slot b, with the slot's YUYV / NV12; the camera frame is read in
  // its wire format when the post kernel reads it so)
  // Masked frames first get their masks M: the post kernel's own, from a mask-only launch into d_mblur_mask_
  if (p.mgclass) {
    PostArgs m = a;
    m.out = nullptr; m.yuyv = nullptr; m.nv12 = nullptr; m.bgra = nullptr; m.flip = nullptr;
    m.mask = d_mblur_mask_; m.mask_stride = mblur_mstride();
    if (!launch_post(stream_, m)) return false;
  }
  if (p.mode == CALL_SOURCES_CAMBLUR && blends(c, p)) {
    // the slots' cached video format is the one the post kernel copies: NV12 when it reads the NV12 frames in place, else
    // YUYV (also for an NV12 call that falls back to BGR frames)
    const bool nv12_in = p.native && c.fmt == IN_NV12;
    GaussSrc cam{};
    if (p.native) cam = GaussSrc{c.in, c.pitch, c.stride, c.uv, c.fmt};
    uint8_t* yv = (!p.all_blur && !nv12_in && !(W_ & 1)) ? d_bank_yuyv_ : nullptr;
    uint8_t* nv = (!p.all_blur && nv12_in) ? d_bank_nv12_ : nullptr;
    const size_t mb = (size_t)max_batch_;
    const MaskedFrames mf{d_src_tab_ + SRC_TAB_MASKED * mb, d_src_tab_ + 2 * mb, p.mgclass, d_mblur_mask_, mblur_mstride(), d_mgauss_tmp_};
    launch_gauss_frames(stream_, n, cam, d_src_tab_ + (p.mgclass ? SRC_TAB_PLAIN : 2) * mb, p.gclass, const_cast<uint8_t*>(a.frames), d_gauss_tmp_,
                        d_bank_, yv, nv, W_, H_, p.mgclass ? &mf : nullptr);
  } else if (p.mgclass) {
    launch_masked_gauss(stream_, n, a.frames, a.frame_pitch, a.frame_stride, d_mblur_mask_, mblur_mstride(), nullptr, bgblur_k_, p.mgclass,
                        d_mgauss_tmp_, d_bg_frames_, (size_t)W_ * 3, fbytes, W_, H_);
  } else if (p.mode == CALL_PLAIN && !has_bg_ && bgblur_k_ && blends(c, p) && !p.passed && !p.live)
    launch_gauss_blur(stream_, n, a.frames, a.frame_pitch, a.frame_stride, d_gauss_tmp_, d_bg_frames_, (size_t)W_ * 3, fbytes, W_, H_, taps_);
  if (p.live) enqueue_live(c, p);
  if (!launch_post(stream_, a)) return false;
  if (ring && bg_advance_) launch_advance_cursor(stream_, d_bg_cursor_, (int)(((long)n * bg_advance_) % bg_count_), bg_count_);
  if (!tail || !want_rgb) return true;
  // app/deepseg.cc:667-681: flip, then scale to the virtual-camera geometry, then YUYV (NV12 for NV12 calls).  Plain calls
  // by the context's flip and size; sources calls by frame, from the table's flip and geometry rows.
  TailArgs t{};
  t.n = n; t.W = W_; t.H = H_; t.src = d_stage_a_; t.src_stride = fbytes;
  t.out = c.out; t.out_stride = c.out_stride; t.video = c.video; t.video_stride = c.video_stride;
  if (p.bgra) { t.bgra = 1; t.src4 = d_stage_a_ + stage_bgra_off(c, p); t.src4_stride = (size_t)W_ * H_ * 4; }
  t.nv12 = c.fmt == IN_NV12 && c.video;     // 2x2 blocks only where an NV12 output (even sizes) is written
  long max_px = (long)out_w_ * out_h_;
  if (p.mode == CALL_PLAIN) {
    t.geo = ctx_geo(); t.flip = (flip_h_ ? 1 : 0) | (flip_v_ ? 2 : 0);
  } else {
    t.slot = d_src_tab_ + 4 * (size_t)max_batch_; t.geos = d_geo_; t.flips = d_src_tab_ + 3 * (size_t)max_batch_;
    max_px = sources_out_px_max();
  }
  if (p.framed) { t.crop = d_crop_; t.crop_idx = d_frame_tab_ + 9 * (size_t)max_batch_; }
  launch_tail(stream_, t, max_px);
  return true;
}

// Camera YUYV / NV12 input: the pre-processing kernel always reads the frames in place; the BGR frame is materialised
// (k_yuyv_to_bgr / k_nv12_to_bgr into d_frames_) only when the post stage cannot read the wire format itself — no TMA
// path for this geometry or layout, or the blur-my-background mode of plain calls, whose Gaussian runs on the BGR frame
// (a sources call's Gaussian reads the wire format itself).  Decided on the call's own outputs.
bool Engine::yuyv_native(const Call& c, Plan p) const {
  // a sources call whose every frame blurs its camera frame converts every frame to BGR for the Gaussian anyway, and the
  // post kernel reads BGR frames faster than it converts the wire format.  A plain call with the filter off has no
  // Gaussian.
  const bool camblur = p.mode == CALL_PLAIN ? (bgblur_k_ && !has_bg_ && !p.passed && blends(c, p) && !p.live) : p.all_blur;
  if (c.fmt == IN_BGR || camblur) return false;
  p.native = true; p.nv12_staged = false;
  return post_tma_eligible(post_args(c, p));
}

// Decided where the call is enqueued (eagerly, or on a graph miss: the GraphKey fixes everything these decisions read),
// so a replay costs no host work.
bool Engine::plan_launch(const Call& c, Plan* p, std::string* err) {
  // NV12 output: the post kernel writes it when it reads the NV12 frames in place and no tail follows (a sources call
  // mirrored in place included), k_tail when a tail follows; otherwise the YUYV output goes to the context staging and
  // k_yuyv_to_nv12 derives the NV12 from it (the definition)
  auto decide = [&] {
    p->native = yuyv_native(c, *p);
    p->nv12_staged = c.fmt == IN_NV12 && c.video && !p->native && !call_tail(*p);
  };
  // Sources calls with flipped frames (app/deepseg.cc:667-681 flips before the resize): when every frame is W x H, and
  // where k_post_tma takes the call, it writes them mirrored in place; otherwise the tail flips them.
  p->flip_tail = false;
  if (p->mode != CALL_PLAIN && p->flipped) {
    bool in_place = !p->resized && !p->framed && tuning().post_tma;
    if (in_place) {
      decide();
      in_place = post_tma_eligible(post_args(c, *p));
    }
    p->flip_tail = !in_place;
  }
  // set_output allocates the staging for a context flip / resize; grown once (dropping the graphs) on first other need
  // (BGRA calls: the BGRA frames, after the BGR composites when the call stages those too)
  const size_t stage_px = (size_t)max_batch_ * W_ * H_;
  const size_t stage_need = p->bgra ? stage_bgra_off(c, *p) + stage_px * 4 : stage_px * 3;
  if (call_tail(*p) && (c.out || c.video) && !ensure((void**)&d_stage_a_, &stage_a_cap_, stage_need, err))
    return false;
  decide();
  return true;
}

bool Engine::enqueue_all(const Call& c, const Plan& p) {
  const long l0 = thread_launch_count();
  const int n = c.n;
  if (c.fmt == IN_NV12 && !p.native) launch_nv12_to_bgr(stream_, n, c.in, c.pitch, c.uv, c.stride, d_frames_, W_, H_);
  if (c.fmt == IN_YUYV && !p.native) launch_yuyv_to_bgr(stream_, c.in, d_frames_, (size_t)n * W_ * H_);
  if (fed_) {
    enqueue_feed(*fed_);
    if (fed_->stage == FEED_LOGITS) enqueue_decision(n, p.mode != CALL_PLAIN, n, SegRows{});
  } else {
    // a call with held frames pre-processes and segments its m segmented frames only (none: no launch before the decision)
    const SegRows seg = seg_rows(c, p);
    if (p.m) enqueue_pre(c, p.m, seg.gather);
    if (c.callbacks && cb_.onprep) { cudaStreamSynchronize(stream_); cb_.onprep(cb_.caller_ctx); }
    if (p.m) enqueue_cnn(p.m, true);
    if (c.callbacks && cb_.oninfer) { cudaStreamSynchronize(stream_); cb_.oninfer(cb_.caller_ctx); }
    enqueue_decision(n, p.mode != CALL_PLAIN, p.m, seg);
    if (c.callbacks && cb_.onmask) { cudaStreamSynchronize(stream_); cb_.onmask(cb_.caller_ctx); }
  }
  if (p.framed) enqueue_framing(c);
  if (!enqueue_post(c, p)) return false;
  if (p.nv12_staged) launch_yuyv_to_nv12(stream_, n, d_yuyv_, (size_t)W_ * H_ * 2, c.video, c.video_stride, W_, H_);
  last_call_launches_ = (int)(thread_launch_count() - l0);
  return true;
}

bool Engine::feed_shape(int stage, int* h, int* w, int* c) const {
  if (stage == FEED_MASK) { *h = oh_; *w = ow_; *c = 1; return true; }
  if (stage != FEED_LOGITS) return false;
  const TensorInfo& I = tinfo_[dec_up_step_ >= 0 ? steps_[dec_up_step_].in : g_.output];
  *h = I.h; *w = I.w; *c = I.c;
  return true;
}

bool Engine::arm_feed(int stage, int n, const void* data, size_t bytes, std::string* err) {
  feed_ = Feed{};
  int h = 0, w = 0, ch = 0;
  if (!feed_shape(stage, &h, &w, &ch)) { *err = "unknown feed stage"; return false; }
  if (n < 1 || n > max_batch_) { *err = "n_frames out of range (1..max_batch)"; return false; }
  const size_t need = (size_t)n * h * w * ch * (stage == FEED_LOGITS ? sizeof(float) : 1);
  if (!data || bytes != need) { *err = "feed size differs from n_frames times the stage's frame size"; return false; }
  feed_.stage = stage; feed_.n = n;
  feed_.data.assign((const uint8_t*)data, (const uint8_t*)data + bytes);
  return true;
}

void Engine::enqueue_feed(const Feed& f) {
  const int n = f.n;
  if (f.stage == FEED_MASK) {
    cudaMemcpy2DAsync(ofinal_, opitch_, f.data.data(), ow_, ow_, (size_t)n * oh_, cudaMemcpyHostToDevice, stream_);
    return;
  }
  // the layout the decision kernels read: [n][h][w][ld] floats, the first c of each pixel's ld
  const int t = dec_up_step_ >= 0 ? steps_[dec_up_step_].in : g_.output;
  const TensorInfo& I = tinfo_[t];
  cudaMemcpy2DAsync(tptr(t), (size_t)I.ld * 4, f.data.data(), (size_t)I.c * 4, (size_t)I.c * 4, (size_t)n * I.h * I.w,
                    cudaMemcpyHostToDevice, stream_);
}

// A call with an armed feed: eager (the captured graphs are neither used nor changed), the feed consumed whatever the outcome
bool Engine::run_fed(const Call& c, std::string* err) {
  Feed f;
  std::swap(f, feed_);
  if (c.n != f.n) { *err = "the call's n_frames differs from the armed feed's"; return false; }
  fed_ = &f;
  const bool ok = run(c, err);
  fed_ = nullptr;
  if (ok) CUDA_OK(cudaStreamSynchronize(stream_));    // the feed's host copy is read by the queued copy
  return ok;
}

bool Engine::run(const Call& c, std::string* err) {
  if (feed_.stage != FEED_NONE) return run_fed(c, err);
  const int n = c.n;
  if (c.fmt == IN_NV12) {
    if ((W_ & 1) || (H_ & 1)) { *err = "NV12 needs an even frame width and height"; return false; }
    if (c.video && ((out_w_ & 1) || (out_h_ & 1))) { *err = "NV12 output needs an even output width and height"; return false; }
    if (!c.in) { *err = "invalid frame"; return false; }
    if (c.pitch < (size_t)W_) { *err = "NV12 row pitch is smaller than the frame width"; return false; }
    if (c.uv < c.pitch * H_) { *err = "NV12 UV plane offset lies inside the Y plane"; return false; }
    if (c.stride < c.uv + c.pitch * (size_t)(H_ / 2 - 1) + (size_t)W_) { *err = "NV12 frame does not fit in the frame stride"; return false; }
  }
  if (c.ids && !n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (n < 1 || n > max_batch_) { *err = "n_frames out of range (1..max_batch)"; return false; }
  Plan p;
  // a call without a composite or video output is the same whatever the filter switches say (the mask is unaffected)
  const bool want_rgb = c.out || c.video;
  p.passed = want_rgb && !c.ids && !filter_;
  p.bgra = bgra_ && c.out;
  // a call that blends nothing (BGRA and mask only) adds no Gaussian class for its camera-blur frames
  const bool blend = blends(c, p);
  std::vector<int> tab;
  // live backgrounds: a plain call's when it blends; a sources call's frames from their sources' (below)
  std::vector<LiveDesc> ltab;
  if (!c.ids && live_.p && blend && !p.passed) {
    p.live = live_.stride ? 2 : 1;
    p.live_gclass = (unsigned)gauss_class(bgblur_k_);
    ltab.resize(p.live == 2 ? (size_t)n : 1);
    for (size_t b = 0; b < ltab.size(); ++b) ltab[b] = live_desc(live_, live_.p + ((size_t)c.frame0 + b) * live_.stride, bgblur_k_ != 0);
  }
  // masked camera blur: a plain call whose background is its blurred camera frame, in the context's mode
  if (!c.ids && blur_mode_ == BLUR_MASKED && !has_bg_ && bgblur_k_ && blend && !p.passed && !p.live) p.mgclass = (unsigned)gauss_class(bgblur_k_);
  if (c.ids) {
    if (has_bg_ && bg_count_ > 1) { *err = "sources calls need a still context background (animate a source with bsb_set_source_background)"; return false; }
    // frame b: state of source ids[b]; background (source_bg) = the context slot, the source's slot, or its camera frame
    // blurred at the source's strength into camera-blur slot b; flip, geometry and filter switch = the source's own, else
    // the context's.  A frame whose filter is off blends nothing: it adds no Gaussian class and is no camera-blur frame.
    // A frame that blends its source's live background takes camera-blur slot b for it, blurred at the source's strength.
    tab.assign(SRC_TAB_ROWS * (size_t)max_batch_, 0);
    ltab.assign((size_t)n, LiveDesc{});
    int n_blur = 0;
    const int ctx_flip = (flip_h_ ? 1 : 0) | (flip_v_ ? 2 : 0);
    for (int b = 0; b < n; ++b) {
      const int id = c.ids[b];
      if (id < 0 || id >= n_sources_) { *err = "source id out of range"; return false; }
      for (int j = 0; j < b; ++j)
        if (c.ids[j] == id) { *err = "source ids must be distinct within one call"; return false; }
      tab[b] = id;
      int k = 0;
      size_t slot = 0;
      const bool off = want_rgb && (src_filter_[id] < 0 ? !filter_ : src_filter_[id] == 0);
      tab[5 * (size_t)max_batch_ + b] = off ? 1 : 0;
      p.passed = p.passed || off;
      const int from = source_bg(id, &k, &slot);
      const Live& lv = src_live_[id];
      if (lv.p && src_fx_[id].bg == SRC_BG_DEFAULT && !off && blend) {
        slot = b;
        tab[6 * (size_t)max_batch_ + b] = k;
        p.live_gclass |= (unsigned)gauss_class(k);
        p.live = 2;
        ltab[b] = live_desc(lv, lv.p, k != 0);
      } else {
        if (from == SRC_FROM_CAMBLUR) slot = b;
        if (from == SRC_FROM_CAMBLUR && !off && blend) {
          tab[2 * (size_t)max_batch_ + b] = k;
          ++n_blur;
          const int mode = src_blur_mode_[id] < 0 ? blur_mode_ : src_blur_mode_[id];
          if (mode == BLUR_MASKED) { tab[SRC_TAB_MASKED * (size_t)max_batch_ + b] = k; p.mgclass |= (unsigned)gauss_class(k); }
          else { tab[SRC_TAB_PLAIN * (size_t)max_batch_ + b] = k; p.gclass |= (unsigned)gauss_class(k); }
        }
      }
      tab[(size_t)max_batch_ + b] = (int)slot;
      const int fl = src_flip_[id] < 0 ? ctx_flip : src_flip_[id];
      tab[3 * (size_t)max_batch_ + b] = fl;
      p.flipped = p.flipped || fl != 0;
      const int sz = src_size_[id];
      tab[4 * (size_t)max_batch_ + b] = sz + 1;
      const int ow = sz < 0 ? out_w_ : own_sizes_[sz].w, oh = sz < 0 ? out_h_ : own_sizes_[sz].h;
      p.resized = p.resized || ow != W_ || oh != H_;
    }
    if (!check_source_outputs(c, err)) return false;
    p.mode = (p.gclass | p.mgclass) ? CALL_SOURCES_CAMBLUR : CALL_SOURCES;
    p.all_blur = n_blur == n;
  }
  if (c.fmt != IN_BGR && (W_ & 1)) { *err = "YUYV ingest needs an even width"; return false; }
  std::vector<int> ftab;
  p.framed = framing_rows(c, &ftab);
  // mask edge refinement: each frame's strength (the source's own, else the context's); the mask-only API never refines
  std::vector<int> rtab;
  if (!c.mask_only_api) {
    rtab.assign((size_t)n, 0);
    for (int b = 0; b < n; ++b) {
      rtab[b] = c.ids && src_refine_[c.ids[b]] >= 0 ? src_refine_[c.ids[b]] : refine_;
      p.refined = p.refined || rtab[b] != 0;
    }
  }
  std::vector<int> seg;
  p.m = segment(c, &seg);
  if (c.ids && p.m < n) std::copy(seg.begin(), seg.begin() + 2 * (size_t)max_batch_, tab.begin() + SRC_TAB_SEG * (size_t)max_batch_);
  CUDA_OK(cudaSetDevice(device_));
  if (p.framed) {
    const size_t mb = (size_t)max_batch_;
    if (!d_frame_tab_) {
      CUDA_OK(cudaMalloc((void**)&d_frame_tab_, FRAMING_ROWS * mb * sizeof(int)));
      CUDA_OK(cudaMalloc((void**)&d_crop_, mb * sizeof(FrameCrop)));
      CUDA_OK(cudaMalloc((void**)&d_frame_box_, 4 * mb * sizeof(int)));
      CUDA_OK(cudaMalloc((void**)&d_frame_counter_, sizeof(unsigned)));
      CUDA_OK(cudaMemsetAsync(d_frame_counter_, 0, sizeof(unsigned), stream_));
      CUDA_OK(cudaMalloc((void**)&d_frame_state_, 4 * sizeof(int)));
    }
    // outside the graph, before its launch, like the source table
    CUDA_OK(cudaMemcpyAsync(d_frame_tab_, ftab.data(), ftab.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
  }
  if (!c.ids && p.m < n) {
    // outside the graph, before its launch, like the source table
    if (!d_seg_tab_) CUDA_OK(cudaMalloc((void**)&d_seg_tab_, seg.size() * sizeof(int)));
    CUDA_OK(cudaMemcpyAsync(d_seg_tab_, seg.data(), seg.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
  }
  if (p.refined) {
    if (!refine_w_ && !(refine_w_ = refine_tables())) { *err = "could not allocate the mask refinement tables"; return false; }
    // outside the graph, before its launch, like the source table
    CUDA_OK(cudaMemcpyAsync(d_refine_, rtab.data(), rtab.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
  }
  if (p.mgclass) {
    // grown once (dropping the graphs), on the first call with masked frames that needs them
    if (!ensure((void**)&d_mblur_mask_, &mblur_mask_cap_, (size_t)max_batch_ * mblur_mstride(), err)) return false;
    if ((p.mgclass & GAUSS_SEPARABLE) && !ensure((void**)&d_mgauss_tmp_, &mgauss_tmp_cap_, (size_t)max_batch_ * W_ * H_ * sizeof(uint4), err))
      return false;
  }
  if (c.ids) {
    if (((p.gclass | p.live_gclass) & GAUSS_SEPARABLE) && !ensure_gauss_tmp(err)) return false;
    // outside the graph, before its launch: stream order keeps the previous launch's reads ahead of this write
    CUDA_OK(cudaMemcpyAsync(d_src_tab_, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, stream_));
  }
  if (p.live) {
    // grown once (dropping the graphs): a plain call's per-frame background frames, the Gaussian's staging
    const size_t fb = (size_t)max_batch_ * W_ * H_ * 3;
    if (!c.ids && !ensure((void**)&d_bg_frames_, &bg_frames_cap_, fb, err)) return false;
    if (p.live_gclass && !ensure((void**)&d_live_stage_, &live_stage_cap_, fb, err)) return false;
    CUDA_OK(cudaMemcpyAsync(d_live_tab_, ltab.data(), ltab.size() * sizeof(LiveDesc), cudaMemcpyHostToDevice, stream_));
  }
  const bool cbs = c.callbacks && (cb_.onprep || cb_.oninfer || cb_.onmask);
  bool eager = cbs || (flags_ & 2u) || fed_;
#ifdef BSB_EMU
  eager = true;
#endif
  static const char* kNoMirror = "the post kernel cannot write this call's mirrored frames";
  static const char* kNoRefine = "the post kernel cannot take this call's mask refinement (or mirrored frames) at this geometry";
  if (eager) {
    if (!plan_launch(c, &p, err)) return false;
    last_native_ = p.native;
    if (!enqueue_all(c, p)) { *err = p.refined ? kNoRefine : kNoMirror; return false; }
    CUDA_OK(cudaGetLastError());
    move_cursors(c);
    count_frames(c);
    count_framing(c, p);
    return true;
  }
#ifndef BSB_EMU
  const GraphKey key(c, p, c.ids ? sources_out_px_max() : 0);
  auto it = graphs_.find(key);
  if (it == graphs_.end()) {
    if (graphs_.size() >= 64) drop_graphs();
    if (!plan_launch(c, &p, err)) return false;
    last_native_ = p.native;
    cudaGraph_t graph = nullptr;
    CUDA_OK(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
    const bool enq = enqueue_all(c, p);
    // the capture is always closed, also when a launch inside it failed: a stream left in capture mode would
    // poison every later call on this context
    const cudaError_t ce = cudaStreamEndCapture(stream_, &graph);
    if (!enq) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      *err = p.refined ? kNoRefine : kNoMirror;
      return false;
    }
    if (ce != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      *err = std::string("CUDA graph capture failed: ") + cudaGetErrorString(ce);
      return false;
    }
    cudaGraphExec_t exec = nullptr;
    const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) { cudaGetLastError(); *err = std::string("cudaGraphInstantiate failed: ") + cudaGetErrorString(ie); return false; }
    it = graphs_.emplace(key, CapturedCall{exec, last_call_launches_, last_native_}).first;
  }
  last_call_launches_ = it->second.launches;
  last_native_ = it->second.native;
  CUDA_OK(cudaGraphLaunch(it->second.exec, stream_));
  move_cursors(c);
  count_frames(c);
  count_framing(c, p);
#endif
  return true;
}

// The live frames of a call (app/deepseg.cc:648-661 on a live `-b` source): resized into their background slots, or into
// the staging for the Gaussian that then writes the slots.  Plain calls: the per-frame background frames at the context's
// strength (one frame at frame_stride 0), without a YUYV cache; sources calls: camera-blur slot b of the bank at the
// source's strength, with the slot's YUYV / NV12 in the format the post kernel copies.
void Engine::enqueue_live(const Call& c, const Plan& p) {
  const size_t fbytes = (size_t)W_ * H_ * 3;
  if (p.mode == CALL_PLAIN) {
    const int n = p.live == 2 ? c.n : 1;
    launch_live_bg(stream_, n, d_live_tab_, d_bg_frames_, d_live_stage_, nullptr, nullptr, W_, H_);
    if (bgblur_k_)
      launch_gauss_blur(stream_, n, d_live_stage_, (size_t)W_ * 3, fbytes, d_gauss_tmp_, d_bg_frames_, (size_t)W_ * 3, fbytes, W_, H_, taps_);
    return;
  }
  const bool nv12_in = p.native && c.fmt == IN_NV12;
  uint8_t* yv = (!nv12_in && !(W_ & 1)) ? d_bank_yuyv_ : nullptr;
  uint8_t* nv = nv12_in ? d_bank_nv12_ : nullptr;
  launch_live_bg(stream_, c.n, d_live_tab_, d_bank_, d_live_stage_, yv, nv, W_, H_);
  if (p.live_gclass)
    launch_gauss_frames(stream_, c.n, GaussSrc{}, d_src_tab_ + 6 * (size_t)max_batch_, p.live_gclass, d_live_stage_, d_gauss_tmp_, d_bank_, yv, nv,
                        W_, H_);
}

LiveDesc Engine::live_desc(const Live& l, const uint8_t* p, bool blur) const {
  const DevResizeTab& t = live_sizes_[l.size].tab;
  LiveDesc d{};
  d.p = p; d.pitch = l.pitch; d.uv = l.uv; d.fmt = l.fmt; d.w = l.w; d.h = l.h;
  d.blur = blur ? 1 : 0; d.area2x2 = t.area2x2 ? 1 : 0; d.tab = t.tab;
  return d;
}

bool Engine::check_live(int fmt, int w, int h, size_t pitch, size_t uv, std::string* err) const {
  if (fmt != LIVE_BGR && fmt != LIVE_NV12) { *err = "live background format must be BSB_LIVE_BGR (0) or BSB_LIVE_NV12 (1)"; return false; }
  if (w < 1 || h < 1 || w > 16384 || h > 16384) { *err = "live background size out of range (1..16384)"; return false; }
  if (fmt == LIVE_BGR && pitch < (size_t)w * 3) { *err = "live background row pitch is smaller than bg_w*3"; return false; }
  if (fmt == LIVE_NV12) {
    if ((w & 1) || (h & 1)) { *err = "NV12 live background needs an even width and height"; return false; }
    if (pitch < (size_t)w) { *err = "NV12 live background row pitch is smaller than bg_w"; return false; }
    if (uv < pitch * (size_t)h) { *err = "NV12 live background UV plane offset lies inside the Y plane"; return false; }
  }
  return true;
}

// The resize tables of live size w x h: an entry of that size (its tables are kept while unused), else a free entry (a
// queued call may still read its old tables, so wait for the stream), else a new one
bool Engine::live_size_acquire(int w, int h, int* idx, std::string* err) {
  int i = -1;
  for (size_t j = 0; j < live_sizes_.size() && i < 0; ++j)
    if (live_sizes_[j].w == w && live_sizes_[j].h == h) i = (int)j;
  if (i < 0) {
    for (size_t j = 0; j < live_sizes_.size() && i < 0; ++j)
      if (!live_sizes_[j].refs) i = (int)j;
    CUDA_OK(cudaSetDevice(device_));
    if (i >= 0) CUDA_OK(cudaStreamSynchronize(stream_));
    else { i = (int)live_sizes_.size(); live_sizes_.emplace_back(); }
    LiveSize& l = live_sizes_[i];
    l.w = l.h = 0;                                   // until the new tables are in place
    if (!upload_resize_tab(build_resize_tab(w, h, W_, H_), &l.tab, err)) return false;
    l.w = w; l.h = h;
  }
  ++live_sizes_[i].refs;
  *idx = i;
  return true;
}

bool Engine::set_live_background(const uint8_t* p, int fmt, int w, int h, size_t pitch, size_t uv, size_t stride, std::string* err) {
  if (p) {
    if (!check_live(fmt, w, h, pitch, uv, err)) return false;
    const size_t frame = fmt == LIVE_BGR ? pitch * (size_t)(h - 1) + (size_t)w * 3 : uv + pitch * (size_t)(h / 2 - 1) + (size_t)w;
    if (stride && stride < frame) { *err = "live background frame stride is smaller than one frame"; return false; }
  }
  Live l{};
  if (p) {
    l = Live{p, fmt, w, h, pitch, fmt == LIVE_NV12 ? uv : 0, stride, -1};
    if (!live_size_acquire(w, h, &l.size, err)) return false;
  }
  live_size_release(live_.size);
  live_ = l;
  return true;
}

bool Engine::set_source_live_background(int source, const uint8_t* p, int fmt, int w, int h, size_t pitch, size_t uv, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (p && !check_live(fmt, w, h, pitch, uv, err)) return false;
  Live l{};
  if (p) {
    l = Live{p, fmt, w, h, pitch, fmt == LIVE_NV12 ? uv : 0, 0, -1};
    if (!live_size_acquire(w, h, &l.size, err)) return false;
  }
  live_size_release(src_live_[source].size);
  src_live_[source] = l;
  return true;
}

// after a sources call is enqueued: the ring of every source with a frame in it moves on, blended or not (a video keeps
// playing while a source shows no image or its blurred camera frame).  The next call's table carries the new slots.
void Engine::move_cursors(const Call& c) {
  if (!c.ids) return;
  for (int b = 0; b < c.n; ++b) {
    SrcRing& r = src_ring_[c.ids[b]];
    if (r.count > 1) r.cursor = (int)(((long)r.cursor + r.advance) % r.count);
  }
}

uint8_t* Engine::out_staging(std::string* err) {
  const long px = std::max({(long)out_w_ * out_h_, (long)W_ * H_, n_sources_ ? sources_out_px_max() : 0L});
  if (!ensure((void**)&d_out_, &out_cap_, (size_t)max_batch_ * px * out_bpp(), err)) return nullptr;
  return d_out_;
}

uint8_t* Engine::nv12_staging(std::string* err) {
  const long px = std::max((long)out_w_ * out_h_, n_sources_ ? sources_out_px_max() : 0L);
  if (!ensure((void**)&d_nv12_, &nv12_cap_, (size_t)max_batch_ * px * 3 / 2, err)) return nullptr;
  return d_nv12_;
}

bool Engine::infer(int n, const float* h_in, float* h_out, std::string* err) {
  if (n < 1 || n > max_batch_) { *err = "n_frames out of range (1..max_batch)"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  const TensorInfo& I = tinfo_[g_.input]; const TensorInfo& O = tinfo_[g_.output];
  CUDA_OK(cudaMemcpyAsync(tptr(g_.input), h_in, (size_t)n * I.frame_elems * 4, cudaMemcpyHostToDevice, stream_));
  enqueue_cnn(n, false);
  CUDA_OK(cudaMemcpyAsync(h_out, tptr(g_.output), (size_t)n * O.frame_elems * 4, cudaMemcpyDeviceToHost, stream_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  CUDA_OK(cudaGetLastError());
  return true;
}

void Engine::drop_graphs() {
#ifndef BSB_EMU
  for (auto& kv : graphs_) cudaGraphExecDestroy(kv.second.exec);
  graphs_.clear();
#endif
}

bool Engine::ensure(void** p, size_t* cap, size_t need, std::string* err) {
  if (need <= *cap && *p) return true;
  CUDA_OK(cudaStreamSynchronize(stream_));
  drop_graphs();                                  // captured launches hold the old pointer
  if (*p) cudaFree(*p);
  *p = nullptr; *cap = 0;
  CUDA_OK(cudaMalloc(p, need));
  *cap = need;
  return true;
}

bool Engine::set_background_ring(const uint8_t* frames, int count, int bw, int bh, size_t pitch, size_t frame_stride, int advance,
                                 std::string* err) {
  if (!frames || count < 1 || bw <= 0 || bh <= 0 || pitch < (size_t)bw * 3 || advance < 0 ||
      (count > 1 && frame_stride < pitch * (size_t)(bh - 1) + (size_t)bw * 3)) { *err = "invalid background"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  const size_t raw = (size_t)bw * bh * 3, fbytes = (size_t)W_ * H_ * 3;
  if (!ensure((void**)&d_bg_raw_, &bg_raw_cap_, raw * count, err)) return false;
  if (!ensure((void**)&d_bg_, &bg_cap_, fbytes * count, err)) return false;
  if (bw != bg_w_ || bh != bg_h_) {
    CUDA_OK(cudaStreamSynchronize(stream_));
    if (!upload_resize_tab(build_resize_tab(bw, bh, W_, H_), &tab_bg_, err)) return false;
    bg_w_ = bw; bg_h_ = bh;
  }
  if (count != bg_count_ || advance != bg_advance_ || !has_bg_) { CUDA_OK(cudaStreamSynchronize(stream_)); drop_graphs(); }
  for (int i = 0; i < count; ++i)
    CUDA_OK(cudaMemcpy2DAsync(d_bg_raw_ + (size_t)i * raw, (size_t)bw * 3, frames + (size_t)i * frame_stride, pitch, (size_t)bw * 3, (size_t)bh,
                              cudaMemcpyHostToDevice, stream_));
  // app/background.cc:178-194: cv::resize(raw, out, Size(width, height))
  launch_resize_u8c3(stream_, d_bg_raw_, bw, bh, (size_t)bw * 3, d_bg_, W_, H_, (size_t)W_ * 3, tab_bg_.tab, tab_bg_.area2x2, count, raw, fbytes);
  CUDA_OK(cudaMemsetAsync(d_bg_cursor_, 0, sizeof(int), stream_));
  bg_count_ = count; bg_advance_ = advance;
  has_bg_ = true;
  if (!refresh_bg_blur(err)) return false;
  if (!refresh_bg_yuyv(err)) return false;
  if (!refresh_bank_ctx(err)) return false;
  if (!refresh_bank_sources_after_ctx(false, err)) return false;
  CUDA_OK(cudaStreamSynchronize(stream_));
  CUDA_OK(cudaGetLastError());
  return true;
}

bool Engine::set_background_cursor(int index, std::string* err) {
  if (index < 0 || index >= bg_count_) { *err = "background index out of range"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaMemcpyAsync(d_bg_cursor_, &index, sizeof(int), cudaMemcpyHostToDevice, stream_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  return true;
}

// (re)compute the blurred copy of the background ring; per-frame work only in camera-blur mode
bool Engine::refresh_bg_blur(std::string* err) {
  if (!bgblur_k_) return true;
  const size_t fbytes = (size_t)W_ * H_ * 3;
  if (!ensure((void**)&d_gauss_tmp_, &gauss_tmp_cap_, (size_t)max_batch_ * fbytes * sizeof(uint16_t), err)) return false;
  if (!has_bg_) return ensure((void**)&d_bg_frames_, &bg_frames_cap_, (size_t)max_batch_ * fbytes, err);
  if (!ensure((void**)&d_bg_eff_, &bg_eff_cap_, fbytes * bg_count_, err)) return false;
  for (int i = 0; i < bg_count_; i += max_batch_) {
    const int n = std::min(max_batch_, bg_count_ - i);
    launch_gauss_blur(stream_, n, d_bg_ + (size_t)i * fbytes, (size_t)W_ * 3, fbytes, d_gauss_tmp_, d_bg_eff_ + (size_t)i * fbytes, (size_t)W_ * 3,
                      fbytes, W_, H_, taps_);
  }
  CUDA_OK(cudaGetLastError());
  return true;
}

// YUYV of the effective background (ring): what convert_rgb_to_yuyv (app/deepseg.cc:87-106) yields wherever the composite
// equals the background, so all-background tiles of the post stage are copies.  Recomputed when the background changes.
bool Engine::refresh_bg_yuyv(std::string* err) {
  bg_yuyv_valid_ = false;
  if (W_ & 1) return true;
  const size_t npix = (size_t)W_ * H_;
  if (!ensure((void**)&d_bg_yuyv_, &bg_yuyv_cap_, npix * 2 * (size_t)bg_count_, err)) return false;
  const uint8_t* src = (has_bg_ && bgblur_k_) ? d_bg_eff_ : d_bg_;
  launch_rgb_to_yuyv(stream_, src, d_bg_yuyv_, npix, bg_count_, npix * 3, npix * 2);
  CUDA_OK(cudaGetLastError());
  bg_yuyv_valid_ = true;
  // ... and its NV12 for NV12 calls
  bg_nv12_valid_ = false;
  if (H_ & 1) return true;
  if (!ensure((void**)&d_bg_nv12_, &bg_nv12_cap_, npix * 3 / 2 * (size_t)bg_count_, err)) return false;
  launch_yuyv_to_nv12(stream_, bg_count_, d_bg_yuyv_, npix * 2, d_bg_nv12_, npix * 3 / 2, W_, H_);
  CUDA_OK(cudaGetLastError());
  bg_nv12_valid_ = true;
  return true;
}

bool Engine::set_bgblur(int k, std::string* err) {
  GaussTaps t{};
  if (k != 0 && !gauss_taps(k, &t)) { *err = "strength value must be odd (1..255)"; return false; }   // app/deepseg.cc:423-426
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  drop_graphs();
  bgblur_k_ = k; taps_ = t;
  if (!refresh_bg_blur(err)) return false;
  if (!refresh_bg_yuyv(err)) return false;
  if (!refresh_bank_ctx(err)) return false;
  if (!refresh_bank_sources_after_ctx(true, err)) return false;
  CUDA_OK(cudaStreamSynchronize(stream_));
  return true;
}

bool Engine::set_output(bool flip_h, bool flip_v, int out_w, int out_h, std::string* err) {
  if (out_w <= 0) out_w = W_;
  if (out_h <= 0) out_h = H_;
  if (out_w > 16384 || out_h > 16384) { *err = "output size out of range"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  drop_graphs();
  const size_t B = (size_t)max_batch_, fbytes = (size_t)W_ * H_ * 3, obytes = (size_t)out_w * out_h * 3;
  const bool flip = flip_h || flip_v, resized = out_w != W_ || out_h != H_;
  if (flip || resized) { if (!ensure((void**)&d_stage_a_, &stage_a_cap_, B * fbytes, err)) return false; }
  if (resized) {
    if (!upload_resize_tab(build_resize_tab(W_, H_, out_w, out_h), &tab_out_, err)) return false;
    // host-buffer API staging must hold the larger of the two geometries
    if (!ensure((void**)&d_out_, &out_cap_, B * std::max(fbytes, obytes), err)) return false;
    if (!ensure((void**)&d_yuyv_, &yuyv_cap_, B * std::max(fbytes, obytes) / 3 * 2, err)) return false;
  }
  flip_h_ = flip_h; flip_v_ = flip_v; out_w_ = out_w; out_h_ = out_h;
  return !d_geo_ || upload_geo(0, ctx_geo(), err);
}

bool Engine::sync(std::string* err) {
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  CUDA_OK(cudaGetLastError());
  return true;
}

bool Engine::reset_state(std::string* err) {
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaMemsetAsync(state_, 0, (size_t)oh_ * ow_, stream_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  plain_frames_ = 0;
  plain_jump_ = true;
  return true;
}

// ---------------------------------------------------------------------------
// independent sources
// ---------------------------------------------------------------------------
void Engine::free_sources() {
  for (void* p : {(void*)src_state_, (void*)d_bank_, (void*)d_bank_yuyv_, (void*)d_bank_nv12_, (void*)d_src_bg_, (void*)d_pool_bg_, (void*)d_green_})
    if (p) cudaFree(p);
  src_state_ = nullptr; d_bank_ = nullptr; d_bank_yuyv_ = nullptr; d_bank_nv12_ = nullptr; d_src_bg_ = nullptr; d_pool_bg_ = nullptr; d_green_ = nullptr;
  n_sources_ = 0;
  pool_slots_ = 0;
  src_ring_.clear();
  src_fx_.clear();
  src_flip_.clear();
  src_filter_.clear();
  src_size_.clear();
  src_interval_.clear();
  src_refine_.clear();
  src_blur_mode_.clear();
  src_frames_.clear();
  src_framing_.clear();
  src_jump_.clear();
  if (d_src_frame_state_) cudaFree(d_src_frame_state_);
  d_src_frame_state_ = nullptr;
  for (const Live& l : src_live_) live_size_release(l.size);
  src_live_.clear();
  for (OwnSize& o : own_sizes_) if (o.tab.blob) cudaFree(o.tab.blob);
  own_sizes_.clear();
  if (d_geo_) cudaFree(d_geo_);
  d_geo_ = nullptr;
}

bool Engine::set_sources(int n_sources, std::string* err) {
  if (n_sources < 1 || n_sources > 65536) { *err = "n_sources out of range (1..65536)"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  drop_graphs();                                  // captured launches hold the old state / bank pointers
  free_sources();
  const size_t fbytes = (size_t)W_ * H_ * 3, npix = (size_t)W_ * H_, opx = (size_t)oh_ * ow_;
  const size_t slots = (size_t)max_batch_ + 1 + (size_t)n_sources;
  if (!d_src_tab_) {
    CUDA_OK(cudaMalloc((void**)&d_src_tab_, SRC_TAB_ROWS * (size_t)max_batch_ * sizeof(int)));
    CUDA_OK(cudaMemset(d_src_tab_, 0, SRC_TAB_ROWS * (size_t)max_batch_ * sizeof(int)));
  }
  CUDA_OK(cudaMalloc((void**)&src_state_, (size_t)n_sources * opx));
  CUDA_OK(cudaMemset(src_state_, 0, (size_t)n_sources * opx));
  CUDA_OK(cudaMalloc((void**)&d_bank_, slots * fbytes));
  CUDA_OK(cudaMemset(d_bank_, 0, slots * fbytes));
  if (!(W_ & 1)) {
    CUDA_OK(cudaMalloc((void**)&d_bank_yuyv_, slots * npix * 2));
    CUDA_OK(cudaMemset(d_bank_yuyv_, 0, slots * npix * 2));
    if (!(H_ & 1)) {
      CUDA_OK(cudaMalloc((void**)&d_bank_nv12_, slots * npix * 3 / 2));
      CUDA_OK(cudaMemset(d_bank_nv12_, 0, slots * npix * 3 / 2));
    }
  }
  CUDA_OK(cudaMalloc((void**)&d_src_bg_, (size_t)n_sources * fbytes));
  {
    std::vector<uint8_t> green(fbytes);
    for (size_t i = 0; i < npix; ++i) { green[3 * i] = 0; green[3 * i + 1] = 255; green[3 * i + 2] = 0; }
    CUDA_OK(cudaMalloc((void**)&d_green_, fbytes));
    CUDA_OK(cudaMemcpy(d_green_, green.data(), fbytes, cudaMemcpyHostToDevice));
  }
  n_sources_ = n_sources;
  src_ring_.assign((size_t)n_sources, SrcRing{});
  src_fx_.assign((size_t)n_sources, SrcEffect{});
  src_flip_.assign((size_t)n_sources, -1);
  src_filter_.assign((size_t)n_sources, -1);
  src_size_.assign((size_t)n_sources, -1);
  src_live_.assign((size_t)n_sources, Live{});
  src_interval_.assign((size_t)n_sources, -1);
  src_refine_.assign((size_t)n_sources, -1);
  src_blur_mode_.assign((size_t)n_sources, -1);
  src_frames_.assign((size_t)n_sources, 0);
  src_framing_.assign((size_t)n_sources, Framing{});
  src_jump_.assign((size_t)n_sources, 1);
  CUDA_OK(cudaMalloc((void**)&d_src_frame_state_, (size_t)n_sources * 4 * sizeof(int)));
  CUDA_OK(cudaMalloc((void**)&d_geo_, (1 + (size_t)n_sources) * sizeof(TailGeo)));
  if (!upload_geo(0, ctx_geo(), err)) return false;
  if (!refresh_bank_ctx(err)) return false;
  CUDA_OK(cudaStreamSynchronize(stream_));
  return true;
}

bool Engine::reset_source(int source, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  const size_t opx = (size_t)oh_ * ow_;
  CUDA_OK(cudaMemsetAsync(src_state_ + (size_t)source * opx, 0, opx, stream_));
  CUDA_OK(cudaStreamSynchronize(stream_));
  src_frames_[source] = 0;
  src_jump_[source] = 1;
  return true;
}

// bank slot of the context's effective background: the still background (blurred when bgblur is on), or plain green
bool Engine::refresh_bank_ctx(std::string* err) {
  if (!d_bank_ || bg_count_ > 1) return true;     // a ring of several images cannot serve sources calls (they reject it)
  const size_t fbytes = (size_t)W_ * H_ * 3, npix = (size_t)W_ * H_;
  uint8_t* slot = d_bank_ + (size_t)max_batch_ * fbytes;
  CUDA_OK(cudaMemcpyAsync(slot, (has_bg_ && bgblur_k_) ? d_bg_eff_ : d_bg_, fbytes, cudaMemcpyDeviceToDevice, stream_));
  if (d_bank_yuyv_) launch_rgb_to_yuyv(stream_, slot, d_bank_yuyv_ + (size_t)max_batch_ * npix * 2, npix);
  if (d_bank_nv12_)
    launch_yuyv_to_nv12(stream_, 1, d_bank_yuyv_ + (size_t)max_batch_ * npix * 2, 0, d_bank_nv12_ + (size_t)max_batch_ * npix * 3 / 2, 0, W_, H_);
  CUDA_OK(cudaGetLastError());
  return true;
}

int Engine::source_bg(int s, int* k, size_t* slot) const {
  const SrcEffect& f = src_fx_[s];
  const SrcRing& r = src_ring_[s];
  *k = f.k < 0 ? bgblur_k_ : f.k;
  int from;
  if (f.bg == SRC_BG_DEFAULT && r.count) from = SRC_FROM_SLOT;                                // its own image, blurred with k
  else if (f.bg == SRC_BG_DEFAULT && has_bg_) from = *k == bgblur_k_ ? SRC_FROM_CTX : SRC_FROM_SLOT;   // the context image at k
  else if (*k) from = SRC_FROM_CAMBLUR;                                                       // no image: its blurred camera frame
  else from = has_bg_ ? SRC_FROM_SLOT : SRC_FROM_CTX;    // green (the context slot is green while there is no context image)
  if (slot) {
    if (from == SRC_FROM_CTX) *slot = (size_t)max_batch_;
    else if (f.bg == SRC_BG_DEFAULT && r.count > 1) *slot = pool0() + r.base + (size_t)r.cursor;   // its ring's current image
    else *slot = (size_t)max_batch_ + 1 + (size_t)s;
  }
  return from;
}

// d_gauss_tmp_ (16-bit row sums of the row / column Gaussian) for max_batch frames
bool Engine::ensure_gauss_tmp(std::string* err) {
  return ensure((void**)&d_gauss_tmp_, &gauss_tmp_cap_, (size_t)max_batch_ * W_ * H_ * 3 * sizeof(uint16_t), err);
}

// bank slots of source s when its still background differs from the context slot: its own image (every image of its
// ring), the context image or green, blurred with the source's strength; then their YUYV / NV12.  A ring of more than
// one image fills its pool slots max_batch images at a time (the Gaussian's row sums hold max_batch frames).
bool Engine::refresh_bank_source(int s, std::string* err) {
  int k = 0;
  size_t slot_i = 0;
  if (source_bg(s, &k, &slot_i) != SRC_FROM_SLOT) return true;
  const SrcEffect& f = src_fx_[s];
  const SrcRing& r = src_ring_[s];
  const size_t fbytes = (size_t)W_ * H_ * 3, npix = (size_t)W_ * H_;
  const bool own = f.bg == SRC_BG_DEFAULT && r.count, pooled = own && r.count > 1;
  const int n = pooled ? r.count : 1;
  if (pooled) slot_i = pool0() + r.base;
  const uint8_t* src = !own ? (f.bg == SRC_BG_DEFAULT && has_bg_ ? d_bg_ : d_green_)
                            : pooled ? d_pool_bg_ + r.base * fbytes : d_src_bg_ + (size_t)s * fbytes;
  uint8_t* slot = d_bank_ + slot_i * fbytes;
  if (k) {
    GaussTaps t{};
    gauss_taps(k, &t);
    if (gauss_class(k) == GAUSS_SEPARABLE && !ensure_gauss_tmp(err)) return false;
    for (int i = 0; i < n; i += max_batch_)
      launch_gauss_blur(stream_, std::min(max_batch_, n - i), src + (size_t)i * fbytes, (size_t)W_ * 3, fbytes, d_gauss_tmp_, slot + (size_t)i * fbytes,
                        (size_t)W_ * 3, fbytes, W_, H_, t);
  } else {
    CUDA_OK(cudaMemcpyAsync(slot, src, (size_t)n * fbytes, cudaMemcpyDeviceToDevice, stream_));
  }
  if (d_bank_yuyv_) launch_rgb_to_yuyv(stream_, slot, d_bank_yuyv_ + slot_i * npix * 2, npix, n, fbytes, npix * 2);
  if (d_bank_nv12_)
    launch_yuyv_to_nv12(stream_, n, d_bank_yuyv_ + slot_i * npix * 2, npix * 2, d_bank_nv12_ + slot_i * npix * 3 / 2, npix * 3 / 2, W_, H_);
  CUDA_OK(cudaGetLastError());
  return true;
}

// after a new context background or strength: every source slot except an own image (still or ring) at a fixed strength
// depends on them (one Gaussian per such source image with a strength > 0); own images that follow the context's strength
// only when it changed
bool Engine::refresh_bank_sources_after_ctx(bool strength, std::string* err) {
  for (int s = 0; s < n_sources_; ++s) {
    const SrcEffect& f = src_fx_[s];
    if (f.bg == SRC_BG_DEFAULT && src_ring_[s].count && (f.k >= 0 || !strength)) continue;
    if (!refresh_bank_source(s, err)) return false;
  }
  return true;
}

bool Engine::set_source_effect(int source, int background, int bgblur, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (background != SRC_BG_DEFAULT && background != SRC_BG_NONE) {
    *err = "unknown source background (BSB_SOURCE_BG_DEFAULT or BSB_SOURCE_BG_NONE)"; return false;
  }
  if (bgblur < -1 || bgblur > 255 || (bgblur > 0 && !(bgblur & 1))) {
    *err = "source strength must be -1 (follow the context), 0 (off) or odd 1..255"; return false;
  }
  CUDA_OK(cudaSetDevice(device_));
  src_fx_[source] = SrcEffect{background, bgblur};
  if (!refresh_bank_source(source, err)) return false;
  CUDA_OK(cudaStreamSynchronize(stream_));
  CUDA_OK(cudaGetLastError());
  return true;
}

bool Engine::set_source_flip(int source, int flip, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (flip < -1 || flip > 3) { *err = "source flip must be -1 (follow the context) or 0..3 (BSB_FLIP_H | BSB_FLIP_V)"; return false; }
  src_flip_[source] = (signed char)flip;
  return true;
}

bool Engine::set_source_filter(int source, int active, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  if (active < -1 || active > 1) { *err = "source filter must be -1 (follow the context), 0 (off) or 1 (on)"; return false; }
  src_filter_[source] = (signed char)active;
  return true;
}

TailGeo Engine::ctx_geo() const {
  return TailGeo{out_w_, out_h_, tab_out_.tab, tab_out_.area2x2 ? 1 : 0};
}

// after a synchronisation, or into a slot no queued call reads
bool Engine::upload_geo(int slot, const TailGeo& g, std::string* err) {
  CUDA_OK(cudaMemcpy(d_geo_ + slot, &g, sizeof(TailGeo), cudaMemcpyHostToDevice));
  return true;
}

bool Engine::source_output_size(int s, int* out_w, int* out_h) const {
  if (s < 0 || s >= n_sources_) return false;
  const int i = src_size_[s];
  *out_w = i < 0 ? out_w_ : own_sizes_[i].w;
  *out_h = i < 0 ? out_h_ : own_sizes_[i].h;
  return true;
}

long Engine::sources_out_px_max() const {
  int own_refs = 0;
  long px = 0;
  for (const OwnSize& o : own_sizes_)
    if (o.refs) { own_refs += o.refs; px = std::max(px, (long)o.w * o.h); }
  if (own_refs < n_sources_) px = std::max(px, (long)out_w_ * out_h_);
  return px;
}

bool Engine::check_source_outputs(const Call& c, std::string* err) const {
  for (int b = 0; b < c.n; ++b) {
    const int id = c.ids[b];
    if (id < 0 || id >= n_sources_) continue;                   // run() reports the id
    const int i = src_size_[id];
    if (i < 0) continue;                                        // at the context size: checked as a plain call's frames
    const size_t w = (size_t)own_sizes_[i].w, h = (size_t)own_sizes_[i].h;
    if (c.out && w * h * (size_t)out_bpp() > c.out_stride) { *err = "a source's output frame does not fit in the output stride"; return false; }
    if (!c.video) continue;
    if (c.fmt == IN_NV12 && ((w & 1) || (h & 1))) { *err = "NV12 output needs an even output width and height"; return false; }
    if ((c.fmt == IN_NV12 ? w * h * 3 / 2 : w * h / 2 * 4) > c.video_stride) {
      *err = "a source's video frame does not fit in the video stride"; return false;
    }
  }
  return true;
}

bool Engine::set_source_output(int source, int out_w, int out_h, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  const bool follow = out_w <= 0 && out_h <= 0;
  if (!follow && (out_w < 1 || out_h < 1 || out_w > 16384 || out_h > 16384)) {
    *err = "source output size out of range (both <= 0 to follow the context, else 1..16384)"; return false;
  }
  CUDA_OK(cudaSetDevice(device_));
  // the old size is released first, so at most n_sources sizes are ever in use (d_geo_ has a slot for each)
  const int old = src_size_[source];
  if (old >= 0 && !follow && own_sizes_[old].w == out_w && own_sizes_[old].h == out_h) return true;
  if (old >= 0) --own_sizes_[old].refs;
  src_size_[source] = -1;
  int idx = -1;
  if (!follow) {
    for (size_t i = 0; i < own_sizes_.size() && idx < 0; ++i)
      if (own_sizes_[i].refs && own_sizes_[i].w == out_w && own_sizes_[i].h == out_h) idx = (int)i;
    if (idx < 0) {
      // a new size: a free slot (a queued call may still read its old tables, so wait for it) or a new one
      for (size_t i = 0; i < own_sizes_.size() && idx < 0; ++i)
        if (!own_sizes_[i].refs) idx = (int)i;
      if (idx >= 0) CUDA_OK(cudaStreamSynchronize(stream_));
      else { idx = (int)own_sizes_.size(); own_sizes_.emplace_back(); }
      OwnSize& o = own_sizes_[idx];
      o.w = out_w; o.h = out_h;
      TailGeo g{out_w, out_h, ResizeTab{}, 0};
      if (out_w != W_ || out_h != H_) {
        if (!upload_resize_tab(build_resize_tab(W_, H_, out_w, out_h), &o.tab, err)) return false;
        g.tab = o.tab.tab; g.area2x2 = o.tab.area2x2 ? 1 : 0;
      }
      if (!upload_geo(1 + idx, g, err)) return false;
    }
    ++own_sizes_[idx].refs;
  }
  src_size_[source] = idx;
  // host-buffer API staging holds max_batch frames of the largest size (grown: synchronises and drops the graphs)
  const size_t B = (size_t)max_batch_, px = (size_t)std::max(sources_out_px_max(), (long)W_ * H_);
  if (!ensure((void**)&d_out_, &out_cap_, B * px * 3, err)) return false;
  if (!ensure((void**)&d_yuyv_, &yuyv_cap_, B * px * 2, err)) return false;
  return true;
}

// Every new source background goes through here (a still is the ring of one image at advance 0).  Checked first, then
// each buffer the ring needs is allocated before anything is changed, so an error leaves every source as it was.
bool Engine::set_source_ring(int source, const uint8_t* frames, int count, int bw, int bh, size_t pitch, size_t frame_stride, int advance,
                             std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  SrcRing& r = src_ring_[source];
  if (!frames) {                                               // later calls blend the context background again
    CUDA_OK(cudaSetDevice(device_));
    if (r.count > 1 && !resize_pool(source, 0, err)) return false;
    r = SrcRing{};
    if (!refresh_bank_source(source, err)) return false;
    CUDA_OK(cudaStreamSynchronize(stream_));
    return true;
  }
  if (count < 1) { *err = "background count must be >= 1"; return false; }
  if (bw <= 0 || bh <= 0 || pitch < (size_t)bw * 3) { *err = "invalid background"; return false; }
  if (count > 1 && frame_stride < pitch * (size_t)(bh - 1) + (size_t)bw * 3) { *err = "background frame stride is smaller than one image"; return false; }
  if (advance < 0) { *err = "background advance must be >= 0"; return false; }
  CUDA_OK(cudaSetDevice(device_));
  // decoded images are staged and resized max_batch at a time
  const int chunk = std::min(count, max_batch_);
  const size_t raw = (size_t)bw * bh * 3, fbytes = (size_t)W_ * H_ * 3;
  if ((size_t)chunk * raw > src_raw_cap_) {
    CUDA_OK(cudaStreamSynchronize(stream_));
    if (d_src_raw_) cudaFree(d_src_raw_);
    d_src_raw_ = nullptr; src_raw_cap_ = 0;
    CUDA_OK(cudaMalloc((void**)&d_src_raw_, (size_t)chunk * raw));
    src_raw_cap_ = (size_t)chunk * raw;
  }
  if (bw != src_bg_w_ || bh != src_bg_h_) {
    CUDA_OK(cudaStreamSynchronize(stream_));
    src_bg_w_ = src_bg_h_ = 0;                                 // until the new tables are in place
    if (!upload_resize_tab(build_resize_tab(bw, bh, W_, H_), &tab_src_, err)) return false;
    src_bg_w_ = bw; src_bg_h_ = bh;
  }
  // a ring of the same count rewrites its slots in place, in stream order; any other change of the pool reallocates it
  if ((count > 1 || r.count > 1) && count != r.count && !resize_pool(source, count, err)) return false;
  uint8_t* dst = count > 1 ? d_pool_bg_ + r.base * fbytes : d_src_bg_ + (size_t)source * fbytes;
  for (int i = 0; i < count; i += chunk) {
    const int n = std::min(chunk, count - i);
    for (int j = 0; j < n; ++j)
      CUDA_OK(cudaMemcpy2DAsync(d_src_raw_ + (size_t)j * raw, (size_t)bw * 3, frames + (size_t)(i + j) * frame_stride, pitch, (size_t)bw * 3,
                                (size_t)bh, cudaMemcpyHostToDevice, stream_));
    // app/background.cc:178-194: cv::resize(raw, out, Size(width, height))
    launch_resize_u8c3(stream_, d_src_raw_, bw, bh, (size_t)bw * 3, dst + (size_t)i * fbytes, W_, H_, (size_t)W_ * 3, tab_src_.tab, tab_src_.area2x2,
                       n, raw, fbytes);
  }
  r.count = count; r.advance = advance; r.cursor = 0;
  if (!refresh_bank_source(source, err)) return false;
  CUDA_OK(cudaStreamSynchronize(stream_));
  CUDA_OK(cudaGetLastError());
  return true;
}

bool Engine::set_source_cursor(int source, int index, std::string* err) {
  if (!n_sources_) { *err = "no sources: call bsb_set_sources first"; return false; }
  if (source < 0 || source >= n_sources_) { *err = "source id out of range"; return false; }
  const SrcRing& r = src_ring_[source];
  if (!r.count) { *err = "the source has no background of its own"; return false; }
  if (index < 0 || index >= r.count) { *err = "background index out of range"; return false; }
  src_ring_[source].cursor = index;
  return true;
}

bool Engine::resize_pool(int s, int count, std::string* err) {
  const size_t fbytes = (size_t)W_ * H_ * 3, npix = (size_t)W_ * H_, fixed = pool0();
  std::vector<size_t> base((size_t)n_sources_, 0);
  size_t total = 0;
  for (int i = 0; i < n_sources_; ++i) {
    const int c = i == s ? count : src_ring_[i].count;
    if (c > 1) { base[i] = total; total += (size_t)c; }
  }
  const size_t slots = fixed + total;
  uint8_t* bank = nullptr, *yuyv = nullptr, *nv12 = nullptr, *pool = nullptr;
  cudaError_t e = cudaMalloc((void**)&bank, slots * fbytes);
  if (e == cudaSuccess && d_bank_yuyv_) e = cudaMalloc((void**)&yuyv, slots * npix * 2);
  if (e == cudaSuccess && d_bank_nv12_) e = cudaMalloc((void**)&nv12, slots * npix * 3 / 2);
  if (e == cudaSuccess && total) e = cudaMalloc((void**)&pool, total * fbytes);
  if (e != cudaSuccess) {
    for (void* p : {(void*)bank, (void*)yuyv, (void*)nv12, (void*)pool}) if (p) cudaFree(p);
    cudaGetLastError();
    *err = std::string("cannot allocate the background bank (") + std::to_string(slots) + " images): " + cudaGetErrorString(e);
    return false;
  }
  // in stream order, behind every queued call that reads the old bank
  auto copy = [&](uint8_t* dst, const uint8_t* src, size_t bytes, size_t to, size_t from, size_t n) {
    return cudaMemcpyAsync(dst + to * bytes, src + from * bytes, n * bytes, cudaMemcpyDeviceToDevice, stream_);
  };
  CUDA_OK(copy(bank, d_bank_, fbytes, 0, 0, fixed));
  if (yuyv) CUDA_OK(copy(yuyv, d_bank_yuyv_, npix * 2, 0, 0, fixed));
  if (nv12) CUDA_OK(copy(nv12, d_bank_nv12_, npix * 3 / 2, 0, 0, fixed));
  for (int i = 0; i < n_sources_; ++i) {
    const SrcRing& r = src_ring_[i];
    if (i == s || r.count < 2) continue;
    const size_t n = (size_t)r.count;
    CUDA_OK(copy(bank, d_bank_, fbytes, fixed + base[i], fixed + r.base, n));
    if (yuyv) CUDA_OK(copy(yuyv, d_bank_yuyv_, npix * 2, fixed + base[i], fixed + r.base, n));
    if (nv12) CUDA_OK(copy(nv12, d_bank_nv12_, npix * 3 / 2, fixed + base[i], fixed + r.base, n));
    CUDA_OK(copy(pool, d_pool_bg_, fbytes, base[i], r.base, n));
  }
  CUDA_OK(cudaStreamSynchronize(stream_));
  drop_graphs();                                  // captured launches hold the old bank's base and tensor maps
  for (void* p : {(void*)d_bank_, (void*)d_bank_yuyv_, (void*)d_bank_nv12_, (void*)d_pool_bg_}) if (p) cudaFree(p);
  d_bank_ = bank; d_bank_yuyv_ = yuyv; d_bank_nv12_ = nv12; d_pool_bg_ = pool;
  pool_slots_ = total;
  for (int i = 0; i < n_sources_; ++i) src_ring_[i].base = base[i];
  src_ring_[s].count = std::max(count, 0); src_ring_[s].cursor = 0;   // the layout's count; the caller fills the images
  return true;
}

double Engine::time_stage(int stage, int n, int iters, std::string* err) {
  if (n < 1 || n > max_batch_ || iters < 1 || stage < 0 || stage > 4) { *err = "bad arguments"; return -1.0; }
  if (cudaSetDevice(device_) != cudaSuccess) { *err = "cudaSetDevice failed"; return -1.0; }
  const size_t row = (size_t)W_ * 3, fbytes = row * H_, npix = (size_t)W_ * H_;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  // a plain call on the context buffers; the last call's input format decides which kernels are timed (camera YUYV read
  // in place, or BGR frames)
  const bool yuyv = last_native_;
  const Call c{n, yuyv ? IN_YUYV : IN_BGR, yuyv ? d_yuyv_in_ : d_frames_, yuyv ? (size_t)W_ * 2 : row, 0, yuyv ? npix * 2 : fbytes,
               nullptr, d_out_, fbytes, d_yuyv_, npix * 2, d_mask_, npix};
  Plan p;
  p.native = yuyv;
  auto once = [&]() {
    if (stage == 0 || stage == 4) enqueue_pre(c, n, nullptr);
    if (stage == 1 || stage == 4) enqueue_cnn(n, true);
    if (stage == 2 || stage == 4) enqueue_decision(n, false, n, SegRows{});
    if (stage == 3 || stage == 4) (void)enqueue_post(c, p);
  };
  once();                                   // warm-up (instruction cache, tables)
  cudaStreamSynchronize(stream_);
  cudaEventRecord(e0, stream_);
  for (int i = 0; i < iters; ++i) once();
  cudaEventRecord(e1, stream_);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (cudaGetLastError() != cudaSuccess) { *err = "CUDA error while timing"; return -1.0; }
  return (double)ms / iters;
}

long Engine::get_tensor(int t, int frame, float* out, long cap, std::string* err) {
  if (!(flags_ & 1u)) { *err = "bsb_get_tensor needs BSB_FLAG_KEEP_TENSORS"; return -1; }
  if (t < 0 || t >= (int)tinfo_.size()) { *err = "tensor index out of range"; return -1; }
  if (frame < 0 || frame >= max_batch_) { *err = "frame index out of range"; return -1; }
  const TensorInfo& I = tinfo_[t];
  if (!I.materialized) return 0;
  const long n = (long)I.h * I.w * I.c;
  if (cap < n) { *err = "output buffer too small"; return -1; }
  if (cudaSetDevice(device_) != cudaSuccess || cudaStreamSynchronize(stream_) != cudaSuccess) { *err = "CUDA error in get_tensor"; return -1; }
  const float* src = tptr(t) + (size_t)frame * I.frame_elems;
  const cudaError_t ce = cudaMemcpy2D(out, (size_t)I.c * 4, src, (size_t)I.ld * 4, (size_t)I.c * 4, (size_t)I.h * I.w, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) { *err = "CUDA memcpy failed"; return -1; }
  return n;
}

int Engine::tc_steps(int* rows, int cap) const {
  int n = 0;
  for (const Step& st : steps_) {
    if (st.kind != Step::PW || !st.use_tc || st.up_from >= 0) continue;
    if (rows && n < cap) {
      const int r[9] = {st.op_index, st.in, st.out, st.residual, st.K, st.N, st.act1, st.act2, st.act3};
      std::memcpy(rows + 9 * n, r, sizeof r);
    }
    ++n;
  }
  return n;
}

long Engine::get_stage_u8(int which, int frame, uint8_t* out, long cap, std::string* err) {
  if (frame < 0 || frame >= max_batch_) { *err = "frame index out of range"; return -1; }
  const uint8_t* src = nullptr; long n = 0;
  if (which == 0) { n = (long)mh_ * mw_ * 3; src = in_u8_ + (size_t)frame * n; }
  else if (which == 1) { n = (long)mh_ * mw_ * 3; src = filt_u8_ ? filt_u8_ + (size_t)frame * n : nullptr; }
  else if (which == 2) { n = (long)oh_ * ow_; src = ofinal_ + (size_t)frame * oh_ * opitch_; }
  if (!src) { *err = which == 1 ? "stage buffer needs BSB_FLAG_KEEP_TENSORS" : "unknown stage"; return -1; }
  if (cap < n) { *err = "output buffer too small"; return -1; }
  if (cudaSetDevice(device_) != cudaSuccess || cudaStreamSynchronize(stream_) != cudaSuccess) { *err = "CUDA error in get_stage_u8"; return -1; }
  const cudaError_t ce = which == 2 ? cudaMemcpy2D(out, (size_t)ow_, src, (size_t)opitch_, (size_t)ow_, (size_t)oh_, cudaMemcpyDeviceToHost)
                                    : cudaMemcpy(out, src, (size_t)n, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) { *err = "CUDA error in get_stage_u8"; return -1; }
  return n;
}

}  // namespace bsb
