// backscrub_b200/csrc/engine.h — per-stream context: model plan, HBM layout, CUDA graph.
//
// Host-side equivalent of backscrub_ctx_t + bs_maskgen_new/process
// (lib/libbackscrub.cc:28-54,161-376), re-designed for one GPU per process:
//   * the .tflite graph is planned once into a short list of fused kernel launches
//     (unary ops, residual ADDs, SE channel scales folded into producers/consumers),
//   * activations live in one liveness-packed arena sized for `max_batch` frames so a
//     whole batch stays L2-resident between layers,
//   * a whole call (pre-proc -> CNN -> decision/IIR -> mask upsample/blur/blend/YUYV) is
//     captured once per batch size into a CUDA graph and replayed with one launch.
#pragma once
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "kernels.h"
#include "tflite_model.h"

namespace bsb {

struct TensorInfo {
  int h = 1, w = 1, c = 1, ld = 1;
  size_t frame_elems = 0;     // h*w*ld floats per frame
  size_t offset = 0;          // float offset inside the arena
  int alias_parent = -1;      // >= 0: lives inside that tensor's buffer (in-place CONCATENATION)
  int alias_off = 0;          // channel offset inside the parent
  bool materialized = false;
  int first_def = 1 << 30, last_use = -1;
};

struct Step {
  enum Kind { CONV, PW, DW, POOL, RESIZE, TCONV, ELT, COPY, BLOCK, CHAIN, HEAD, ENC_A, ENC_B } kind = ELT;
  int block = -1;             // BLOCK: index into Engine::blocks_ (the four fused sub-steps); CHAIN: index into Engine::chains_;
                              // ENC_A / ENC_B: index into Engine::encs_
  int op_index = -1;
  int in = -1, in2 = -1, out = -1, scale = -1, in_add = -1, residual = -1;
  int out2 = -1;               // ENC_A / ENC_B: the block's second output (a decoder skip)
  size_t w_off = 0, b_off = 0; bool has_bias = false;
  int act1 = 0, act2 = 0, act3 = 0;
  int K = 0, N = 0, n4 = 0;
  int kh = 1, kw = 1, sh = 1, sw = 1, dh = 1, dw = 1, pt = 0, pl = 0;
  int elt_mode = 0;
  bool align_corners = false, half_pixel = false;
  int copy_off = 0;
  int up_from = -1;           // PW: >= 0 -> the input is RESIZE_BILINEAR(up_from), interpolated on the fly (k_upsample_pw)
  bool use_tc = false; size_t tc_hi_off = 0, tc_lo_off = 0; int kpad = 0, npad = 0;   // tensor-core pointwise
  // POOL: optional fused fully-connected chain (squeeze-excite) after the global average pool
  struct Fc { size_t w_off = 0, b_off = 0; bool has_bias = false; int K = 0, N = 0, n4 = 0, act1 = 0, act2 = 0; };
  int n_fc = 0;
  Fc fc[2];
  int launches() const { return 1; }
};

struct HostResizeTab {
  std::vector<int> xofs, yofs0, yofs1;
  std::vector<short> xw, yw;
  bool area2x2 = false;
  int sw = 0;
};
// OpenCV INTER_LINEAR 8-bit coefficient tables for sw x sh -> dw x dh
HostResizeTab build_resize_tab(int sw, int sh, int dw, int dh);

struct DevResizeTab { void* blob = nullptr; ResizeTab tab{}; bool area2x2 = false; };
// tables -> device memory of the current device (frees a previous blob)
bool upload_resize_tab(const HostResizeTab& h, DevResizeTab* d, std::string* err);

struct Callbacks {
  void (*ondebug)(void*, const char*) = nullptr;
  void (*onprep)(void*) = nullptr;
  void (*oninfer)(void*) = nullptr;
  void (*onmask)(void*) = nullptr;
  void* caller_ctx = nullptr;
};

// One fused call: n camera frames in, up to three outputs (any may be null).  Device memory, byte pitches and strides.
struct Call {
  int n = 0;
  InFmt fmt = IN_BGR;                // BGR, YUYV (tightly packed: pitch W*2, stride W*H*2) or NV12 (W and H even)
  const uint8_t* in = nullptr;
  size_t pitch = 0, uv = 0, stride = 0;   // row pitch, NV12's UV plane offset inside a frame (else 0), frame stride
  const int* ids = nullptr;          // HOST array: frame b belongs to source ids[b] (n distinct ids); null: a plain call
  uint8_t* out = nullptr; size_t out_stride = 0;       // BGR composite, out_w x out_h (sources: the frame's own), rows out_w*3 bytes;
                                                       // in the BGRA output format the transparent BGRA frames, rows out_w*4 bytes
  uint8_t* video = nullptr; size_t video_stride = 0;   // tightly packed YUYV, or NV12 when the input is NV12
  uint8_t* mask = nullptr; size_t mask_stride = 0;     // W x H
  bool callbacks = false;            // fire the stage callbacks (the call then runs eagerly, synchronised at each stage)
  int frame0 = 0;                    // frame 0's index in the caller's call (a chunk of a split call): plain live backgrounds
};

class Engine {
 public:
  static Engine* create(const std::string& model_path, int width, int height, int device, int max_batch,
                        unsigned flags, const Callbacks& cb, std::string* err);
  ~Engine();

  // Enqueues one call on the context's stream (a captured graph, replayed when the call matches one).  YUYV / NV12 frames
  // that have to be read as BGR are converted into the context staging d_frames().
  bool run(const Call& c, std::string* err);
  bool infer(int n, const float* h_in, float* h_out, std::string* err);
  bool set_background(const uint8_t* bg_raw, int bw, int bh, size_t pitch, std::string* err) {
    return set_background_ring(bg_raw, 1, bw, bh, pitch, 0, 0, err);
  }
  // animated background (app/background.cc:126-176 decodes, :178-194 resizes): `count` decoded images are
  // resized into a device ring; batch frame b of a call blends ring image (cursor + b*advance) % count and the
  // cursor then moves on by n*advance (advance 0: the caller moves it with set_background_cursor)
  bool set_background_ring(const uint8_t* frames, int count, int bw, int bh, size_t pitch, size_t frame_stride, int advance,
                           std::string* err);
  bool set_background_cursor(int index, std::string* err);
  // app/deepseg.cc:657-658 `-p bgblur:k`: Gaussian-blur the background (the grabbed one, else a copy of the
  // camera frame); k = 0 switches it off
  bool set_bgblur(int k, std::string* err);
  // app/deepseg.cc:667-679: cv::flip and cv::resize to the virtual-camera size before the YUYV conversion
  bool set_output(bool flip_h, bool flip_v, int out_w, int out_h, std::string* err);
  // app/deepseg.cc:624,639-664 (the `s` key): off, a call's composite is the camera frame, flipped, resized and converted as
  // usual; the mask is still computed and written and the smoother still advances.  Host state only: the switch is part of
  // the captured call, so toggling replays once both states have been captured.
  void set_filter(bool active) { filter_ = active; }
  bool filter() const { return filter_; }
  // Output format of the `out` buffers (include/backscrub_b200.h, bsb_set_out_format): BGR composites, or straight-alpha
  // BGRA frames (the camera with alpha 255 - mask, flipped and resized like the composite).  Host state only, like
  // set_filter: the format is part of the captured call.
  void set_out_bgra(bool bgra) { bgra_ = bgra; }
  bool out_bgra() const { return bgra_; }
  int out_bpp() const { return bgra_ ? 4 : 3; }
  // Live backgrounds (include/backscrub_b200.h): a caller-owned device image (LiveFmt, any size) that later calls resize
  // (and blur) inside the call.  Host bookkeeping only, except that a size not seen before has its resize tables built
  // once.  Plain calls: frame b blends p + b*stride (stride 0: one image for every frame); p null clears.
  bool set_live_background(const uint8_t* p, int fmt, int w, int h, size_t pitch, size_t uv, size_t stride, std::string* err);
  // sources calls: every frame of `source` blends this image (where the source's background is BSB_SOURCE_BG_DEFAULT)
  bool set_source_live_background(int source, const uint8_t* p, int fmt, int w, int h, size_t pitch, size_t uv, std::string* err);
  // device staging of max_batch `out` frames in the current format (host-buffer API), grown on demand; nullptr on error
  uint8_t* out_staging(std::string* err);
  // Mask interval (include/backscrub_b200.h, bsb_set_mask_interval): segment every k-th frame of a camera, composite the
  // frames between with its latest mask.  Host state only: which frames are segmented reaches the device as table data.
  enum { MASK_INTERVAL_MAX = 256 };
  bool set_mask_interval(int k, std::string* err);
  // one source's interval: -1 follows set_mask_interval, else 1..MASK_INTERVAL_MAX
  bool set_source_mask_interval(int source, int k, std::string* err);
  bool sync(std::string* err);
  bool reset_state(std::string* err);
  // Framing (include/backscrub_b200.h, bsb_set_framing): the output shows a crop of the camera frame, a fixed rectangle
  // (RECT) or one that follows the person the mask finds (AUTO, framing.h).  Host state only: the modes and rectangles
  // reach the device as table data with the call.
  bool set_framing(int mode, int x, int y, int w, int h, std::string* err);
  bool set_framing_auto(int max_zoom, int margin, int speed, std::string* err);
  // one source's framing: mode -1 follows set_framing (rectangle included), else its own
  bool set_source_framing(int source, int mode, int x, int y, int w, int h, std::string* err);
  // the crop (x, y, w, h) frame `frame` of the last call showed (synchronises)
  bool get_framing(int frame, int* rect, std::string* err);

  // Independent sources (camera streams) batched one frame each into a call.  set_sources allocates n zeroed smoother
  // states and the per-source background bank (again: everything reallocated and zeroed, graphs dropped).
  bool set_sources(int n_sources, std::string* err);
  bool reset_source(int source, std::string* err);
  // cv::resize(raw -> W x H) into the source's bank slot (+ bgblur, + its YUYV); bg_raw == nullptr clears the slot.  The
  // ring of one image at advance 0.
  bool set_source_background(int source, const uint8_t* bg_raw, int bw, int bh, size_t pitch, std::string* err) {
    return set_source_ring(source, bg_raw, 1, bw, bh, pitch, 0, 0, err);
  }
  // animated background of one source (app/background.cc:126-194): `count` decoded images resized into the bank (one: the
  // source's own slot; more: the ring pool), blurred at the source's strength; each call carrying a frame of the source
  // blends ring image `cursor`, then moves the cursor on by `advance`.  frames == nullptr clears the source's background.
  bool set_source_ring(int source, const uint8_t* frames, int count, int bw, int bh, size_t pitch, size_t frame_stride, int advance,
                       std::string* err);
  // host bookkeeping only: the cursor reaches the device with the next call's source table
  bool set_source_cursor(int source, int index, std::string* err);
  // background effect of one source (include/backscrub_b200.h): background SRC_BG_DEFAULT / SRC_BG_NONE, bgblur -1 (follow
  // the context), 0 or odd 1..255
  enum { SRC_BG_DEFAULT = 0, SRC_BG_NONE = 1 };
  bool set_source_effect(int source, int background, int bgblur, std::string* err);
  // mirroring of one source: -1 follows set_output's flips, 0..3 its own (bit 0 horizontal, bit 1 vertical).  Host
  // bookkeeping only: the flip reaches the device through the per-frame table of each call.
  bool set_source_flip(int source, int flip, std::string* err);
  // filter switch of one source: -1 follows set_filter, 0 off, 1 on.  Host bookkeeping only: which frames are filtered off
  // reaches the device through the per-frame table of each call.
  bool set_source_filter(int source, int active, std::string* err);
  // virtual-camera size of one source: out_w <= 0 and out_h <= 0 follow set_output's size, else both in 1..16384
  bool set_source_output(int source, int out_w, int out_h, std::string* err);
  // the effective size of source s (its own, or the context's); false when s is not a source
  bool source_output_size(int s, int* out_w, int* out_h) const;
  // the largest effective size (w * h) among the sources, which bounds every frame of a sources call
  long sources_out_px_max() const;
  // the frames of sources call c with an own size: each fits its output strides, and an NV12 output is even-sized
  bool check_source_outputs(const Call& c, std::string* err) const;
  // device staging of max_batch NV12 output frames (host-buffer API), grown on demand; nullptr on error
  uint8_t* nv12_staging(std::string* err);
  int n_sources() const { return n_sources_; }
  double time_stage(int stage, int n, int iters, std::string* err);

  // Test entry point (include/backscrub_b200.h, bsb_test_feed): the next call takes the tensor a stage reads from the
  // caller instead of computing it.  FEED_LOGITS: the fp32 tensor the decision reads, [n][h][w][c] packed (pre-processing
  // and the CNN are skipped); FEED_MASK: the smoother output ofinal, [n][oh][ow] bytes (the decision is skipped too, and
  // no smoother state changes).  The fed call runs eagerly and consumes the feed whatever its outcome.
  enum { FEED_NONE = 0, FEED_LOGITS = 1, FEED_MASK = 2 };
  // h, w, c of one frame of a stage's tensor; false for an unknown stage
  bool feed_shape(int stage, int* h, int* w, int* c) const;
  bool arm_feed(int stage, int n, const void* data, size_t bytes, std::string* err);
  bool feed_armed() const { return feed_.stage != FEED_NONE; }
  void disarm_feed() { feed_ = Feed{}; }

  // accessors
  int W() const { return W_; }
  int H() const { return H_; }
  int out_w() const { return out_w_; }
  int out_h() const { return out_h_; }
  int bgblur() const { return bgblur_k_; }
  int bg_count() const { return bg_count_; }
  int max_batch() const { return max_batch_; }
  int device() const { return device_; }
  cudaStream_t stream() const { return stream_; }
  const int* roidim() const { return roidim_; }
  const int* in_roidim() const { return in_roidim_; }
  const int* out_roidim() const { return out_roidim_; }
  void in_hwc(int* v) const { v[0] = mh_; v[1] = mw_; v[2] = 3; }
  void out_hwc(int* v) const { v[0] = oh_; v[1] = ow_; v[2] = oc_; }
  double flops() const { return flops_; }
  int launches_per_call() const {
    // counted while the last call was enqueued / captured (a replay restores its graph's count, so a sources call reports
    // whether its tail mirrors frames)
    if (last_call_launches_ > 0) return last_call_launches_;
    int n = 4;
    for (const Step& s : steps_) n += s.launches();
    if (bgblur_k_ && !has_bg_ && filter_ && !bgra_) n += 2;   // (a BGRA call without video blurs nothing)
    if (bg_count_ > 1 && bg_advance_) n += 1;
    if (flip_h_ || flip_v_ || out_w_ != W_ || out_h_ != H_) n += 1;   // k_tail
    return n;
  }
  long get_tensor(int t, int frame, float* out, long cap, std::string* err);
  // the steps that run the tensor-core 1x1 convolution: 9 ints each (op index, input, output and residual tensor, K, N,
  // act1, act2, act3) into rows (up to cap steps); returns how many there are
  int tc_steps(int* rows, int cap) const;
  long get_stage_u8(int which, int frame, uint8_t* out, long cap, std::string* err);

  // device staging owned by the context (host-buffer API)
  uint8_t* d_frames() const { return d_frames_; }
  uint8_t* d_out() const { return d_out_; }
  uint8_t* d_yuyv() const { return d_yuyv_; }
  uint8_t* d_mask() const { return d_mask_; }
  uint8_t* d_bg() const { return d_bg_; }          // resized, unblurred (what grab_background returns)
  uint8_t* d_yuyv_in() const { return d_yuyv_in_; }
  uint8_t* h_mask() const { return h_mask_; }
  bool has_background() const { return has_bg_; }
  bool last_native() const { return last_native_; }
  bool uses_tensor_cores() const { return uses_tc_; }

 private:
  Engine() = default;
  bool plan(std::string* err);
  bool upload(std::string* err);
  // What the engine derives from a Call and the context: the kind of call — plain (one stream, state_), sources, or
  // sources with at least one frame that blends its own blurred camera frame (a source with no image and a strength > 0)
  // — and how it is enqueued.
  enum CallMode { CALL_PLAIN = 0, CALL_SOURCES = 1, CALL_SOURCES_CAMBLUR = 2 };
  struct Plan {
    int mode = CALL_PLAIN;
    unsigned gclass = 0;             // sources: the Gaussian launch classes of the camera-blur frames (GAUSS_FUSED | GAUSS_SEPARABLE)
    bool all_blur = false;           // sources: every frame blurs its camera frame (the BGR frames are materialised)
    bool flipped = false;            // sources: some frame is mirrored (the table's flip row is not all 0)
    bool resized = false;            // sources: some frame's output size is not W x H (the table's geometry row)
    bool passed = false;             // some frame's filter is off (plain: the context's switch; sources: the table's filter
                                     // row is not all 0); only calls with a composite or video output have one
    bool flip_tail = false;          // ... and the tail mirrors them (k_tail): the call resizes or its post kernel is not k_post_tma
    bool native = false;             // the post stage reads the camera frames (YUYV or NV12) in place, no BGR frame is materialised
    bool nv12_staged = false;        // the NV12 output is converted from a YUYV output staged in d_yuyv_ (k_yuyv_to_nv12): an
                                     // NV12 call whose post kernel reads BGR frames, without a tail
    bool bgra = false;               // the call's `out` takes BGRA frames (the context's format, and the call has an out buffer)
    int live = 0;                    // frames that blend a live background: 0 none, 1 one image for every frame (a plain call
                                     // at frame_stride 0), 2 one per frame (the live table's descriptors say which)
    unsigned live_gclass = 0;        // the Gaussian launch classes of the blurred live frames
    int m = 0;                       // frames segmented (the CNN batch); m == n: every frame, the parent path with no table
    bool framed = false;             // some frame is framed (RECT or AUTO): k_framing runs and every frame goes through the
                                     // cropping tail from unflipped staging
  };
  // the call blends a composite: it has a video output, or a BGR composite output.  A call that does not reads no
  // background and blurs nothing.
  static bool blends(const Call& c, const Plan& p) { return c.video || (c.out && !p.bgra); }
  // where the tail's staged BGRA frames begin in d_stage_a_ (after the staged BGR composites when the call stages them)
  size_t stage_bgra_off(const Call& c, const Plan& p) const { return blends(c, p) ? (size_t)max_batch_ * W_ * H_ * 3 : 0; }
  // flip_tail, native and nv12_staged (and the tail's staging); false with *err when a buffer cannot be grown
  bool plan_launch(const Call& c, Plan* p, std::string* err);
  // pre-processing of the m segmented frames of c (gather: the device row of their call frames; null: all n, m == n)
  void enqueue_pre(const Call& c, int m, const int* gather);
  PostArgs post_args(const Call& c, const Plan& p) const;
  bool yuyv_native(const Call& c, Plan p) const;
  // the call ends with k_tail (post -> stage -> flip, resize, YUYV / NV12): plain calls with a context flip or resize;
  // sources calls with a frame not at W x H, or with mirrored frames the post kernel cannot mirror in place
  bool call_tail(const Plan& p) const {
    return p.framed || (p.mode == CALL_PLAIN ? (flip_h_ || flip_v_ || out_w_ != W_ || out_h_ != H_) : (p.resized || p.flip_tail));
  }
  // false (nothing more enqueued) only when the post kernel cannot write a call's mirrored frames
  bool enqueue_all(const Call& c, const Plan& p);
  struct Feed { int stage = FEED_NONE, n = 0; std::vector<uint8_t> data; };
  Feed feed_;                        // armed by arm_feed for the next call
  const Feed* fed_ = nullptr;        // the feed of the call being enqueued (run_fed), else null
  bool run_fed(const Call& c, std::string* err);
  // the fed tensor into the place the skipped stages write (ofinal_, or the tensor the decision reads)
  void enqueue_feed(const Feed& f);
  bool refresh_bg_yuyv(std::string* err);
  void enqueue_cnn(int n, bool from_u8);
  void enqueue_decision(int n, bool sources, int m, const SegRows& seg);
  // the segmented frames of call c (the cadence of set_mask_interval) into rows [gather | cidx | lat] of max_batch_ ints
  // each (SegRows); returns m.  A fed call segments every frame.
  int segment(const Call& c, std::vector<int>* rows) const;
  // the device segment rows of a call with held frames (p.m < c.n); null rows when every frame is segmented
  SegRows seg_rows(const Call& c, const Plan& p) const;
  // after a call is enqueued: the frame counters of the cadence move on (not for a fed call)
  void count_frames(const Call& c);
  // the framing rows of call c (FRAMING_ROWS x max_batch_, kernels.h) into *rows; true when some frame is framed
  bool framing_rows(const Call& c, std::vector<int>* rows) const;
  // after a call is enqueued (fed calls included): which cameras now hold a framing state
  void count_framing(const Call& c, const Plan& p);
  void enqueue_framing(const Call& c);
  bool enqueue_post(const Call& c, const Plan& p);
  void enqueue_live(const Call& c, const Plan& p);
  // base of tensor t for the frames [frame_off_, ...) of the batch (frame_off_ != 0 only inside a sub-batched segment)
  float* tptr(int t) const {
    const TensorInfo& I = tinfo_[t];
    if (I.alias_parent >= 0) {
      const TensorInfo& P = tinfo_[I.alias_parent];
      return arena_ + P.offset + (size_t)frame_off_ * P.frame_elems + I.alias_off;
    }
    return arena_ + I.offset + (size_t)frame_off_ * I.frame_elems;
  }
  void run_step(size_t si, int n, bool from_u8, bool* first, bool* skip_next);
  void find_segments();

  Graph g_;
  int model_type_ = 0;
  float scaling_ = 0.f, offset_ = 0.f;
  int W_ = 0, H_ = 0, device_ = 0, max_batch_ = 1;
  unsigned flags_ = 0;
  Callbacks cb_;
  int mh_ = 0, mw_ = 0, oh_ = 0, ow_ = 0, oc_ = 0;
  int roidim_[4] = {0, 0, 0, 0}, in_roidim_[4] = {0, 0, 0, 0}, out_roidim_[4] = {0, 0, 0, 0};
  double flops_ = 0;

  std::vector<TensorInfo> tinfo_;
  std::vector<Step> steps_;
  // Optional (tuning().sub_batch_mb, off by default): a run of per-frame steps whose tensors are too large for the L2 at
  // the full batch is executed a few frames at a time, so that each step finds its input where the previous one left it
  // instead of streaming it through HBM.  The smaller launches can cost more than the HBM traffic they save — kept as
  // a bit-exact, tested switch.  seg_len_[si] > 0: steps [si, si + seg_len_[si]) form a segment whose largest tensor has
  // seg_frame_bytes_[si] bytes per frame.
  std::vector<int> seg_len_;
  std::vector<size_t> seg_frame_bytes_;
  int frame_off_ = 0;
  struct FusedBlock { Step expand, dw, pool, project; };
  std::vector<FusedBlock> blocks_;
  // the low-resolution middle of the graph run by one kernel (kernels_chain.cu): the original steps in order, each
  // tagged with the chain op it became
  struct ChainPlan { int h = 0, w = 0; std::vector<Step> seq; std::vector<int> types; ChainOp* d_ops = nullptr; int n_ops = 0; };
  std::vector<ChainPlan> chains_;
  bool detect_chain();
  // decoder stage run by one kernel (k_head): 1x1 conv -> depthwise 3x3 + residual [-> transposed conv]
  struct HeadPlan { Step p, d, t; bool has_t = false; bool s2 = false; };   // s2: 1x1 + stride-2 depthwise (k_pw_dws2), else a decoder stage (k_head)
  std::vector<HeadPlan> heads_;
  void detect_heads();
  void detect_pw_dws2();
  // the two inverted-residual blocks between the encoder entry and the chain (kernels_nn.cu, k_enc_block_s2 / _res):
  // the eight original steps (scaled 1x1, expand, depthwise s2, project | expand, depthwise, project + residual, expand)
  struct EncPlan { Step s[8]; int act = 0; };
  std::vector<EncPlan> encs_;
  void detect_enc_blocks();
  std::vector<float> wblob_h_;
  size_t arena_elems_ = 0;
  bool tc_enabled_ = false, uses_tc_ = false;   // tensor-core 1x1 convs allowed / actually planned for at least one layer
  bool stem_u8_ok_ = false;          // step 0 is a 3->16 dense conv that is the only reader of the graph input
  int dec_up_step_ = -1;             // DeepLab: index of the final RESIZE_BILINEAR step the decision kernel performs itself (pipeline calls)
  bool stem_pw_ok_ = false;          // ... and step 1 is a plain 16 -> 16 1x1 conv of its output (runs inside the stem kernel)

  // device memory
  cudaStream_t stream_ = nullptr;
  float* wblob_ = nullptr;
  float* arena_ = nullptr;
  float* lut_ = nullptr;             // color_w[768] + space_w[16]
  float* rowsum_ = nullptr;          // scratch of the global-average-pool row sums
  size_t rowsum_elems_ = 0;
  unsigned* pool_counters_ = nullptr; // [B] arrival counters of the one-launch pool + SE kernel (zero between launches)
  uint8_t* in_u8_ = nullptr;         // [B][mh][mw][3] zero outside in_roidim
  uint8_t* filt_u8_ = nullptr;       // [B][mh][mw][3] (KEEP_TENSORS only)
  uint8_t* state_ = nullptr;         // [oh*ow] IIR state
  uint8_t* ofinal_ = nullptr;        // [B][oh][opitch_]
  int opitch_ = 0;                   // ofinal row pitch (ow rounded up to 16 bytes: TMA-addressable)
  uint8_t* d_frames_ = nullptr, *d_out_ = nullptr, *d_yuyv_ = nullptr, *d_mask_ = nullptr, *d_bg_ = nullptr, *d_bg_raw_ = nullptr, *d_yuyv_in_ = nullptr;
  size_t bg_raw_cap_ = 0;
  uint8_t* h_mask_ = nullptr;        // pinned host W*H
  bool has_bg_ = false;
  DevResizeTab tab_in_, tab_up_, tab_bg_, tab_out_;
  int bg_w_ = 0, bg_h_ = 0;

  // optional stages around the blend (app/deepseg.cc:649-679)
  bool ensure(void** p, size_t* cap, size_t need, std::string* err);   // grow-only device buffer; drops the graphs
  bool refresh_bg_blur(std::string* err);
  void drop_graphs();
  int bg_count_ = 1, bg_advance_ = 0;
  size_t bg_cap_ = 0;
  int* d_bg_cursor_ = nullptr;
  int bgblur_k_ = 0;
  GaussTaps taps_{};
  uint8_t* d_bg_eff_ = nullptr;      // blurred copy of the background ring
  uint8_t* d_bg_frames_ = nullptr;   // [B][H][W][3] blurred camera frames (bgblur without a background)
  uint16_t* d_gauss_tmp_ = nullptr;  // [B][H][W*3] row sums
  size_t bg_eff_cap_ = 0, bg_frames_cap_ = 0, gauss_tmp_cap_ = 0;
  bool flip_h_ = false, flip_v_ = false;
  int out_w_ = 0, out_h_ = 0;
  bool filter_ = true;
  bool bgra_ = false;                // set_out_bgra
  int* d_pass_all_ = nullptr;        // [max_batch] ones: the filter table of a plain call with the filter off
  uint8_t* d_stage_a_ = nullptr;     // [B][H][W][3] unflipped composites that k_tail reads, then [B][H][W][4] BGRA frames (BGRA calls)
  int2* d_tile_geo_ = nullptr;       // k_post_tma patch geometry per tile row | per 64-wide tile column | per 128-wide tile column
  int geo_nty_ = 0, geo_ntx64_ = 0;
  uint8_t* d_bg_yuyv_ = nullptr;     // YUYV of the effective background (ring): all-background tiles are copies
  size_t bg_yuyv_cap_ = 0;
  bool bg_yuyv_valid_ = false;
  uint8_t* d_bg_nv12_ = nullptr;     // ... and its NV12 (W*H*3/2 bytes per image; even W and H), for NV12 calls
  size_t bg_nv12_cap_ = 0;
  bool bg_nv12_valid_ = false;
  bool last_native_ = false;         // the last call read the camera frames (YUYV or NV12) in place (no BGR frame was materialised)
  uint8_t* d_nv12_ = nullptr;        // host-buffer API staging of the NV12 output
  size_t nv12_cap_ = 0;
  int last_call_launches_ = 0;
  size_t stage_a_cap_ = 0, out_cap_ = 0, yuyv_cap_ = 0;

  // ---- independent sources (calls with ids) ----
  int n_sources_ = 0;
  uint8_t* src_state_ = nullptr;     // [n_sources][oh*ow] smoother state per source
  // [9][max_batch]: source id of frame b | background-bank slot of frame b | camera-blur strength of frame b (0 = none) |
  // flip code of frame b (bit 0 horizontal, bit 1 vertical; the source's own, or the context's) | geometry slot of frame b
  // (d_geo_ index) | 1 when frame b's filter is off (the source's own switch, or the context's) | live-background strength
  // of frame b (0 = not blurred, or no live background) | the segment rows gather and cidx (calls with held frames, else
  // unused), written before each launch
  int* d_src_tab_ = nullptr;
  enum { SRC_TAB_ROWS = 9, SRC_TAB_SEG = 7 };
  // ---- mask interval ----
  int mask_interval_ = 1;
  long long plain_frames_ = 0;       // frames of plain calls since creation / reset_state: frame c is segmented iff c % k == 0
  std::vector<int> src_interval_;    // per source: -1 = mask_interval_, else its own
  std::vector<long long> src_frames_;   // per source: frames delivered since set_sources / reset_source
  int src_interval(int s) const { return src_interval_[s] < 0 ? mask_interval_ : src_interval_[s]; }
  int* d_seg_tab_ = nullptr;         // [3][max_batch] the segment rows of a plain call with held frames, written before its launch
  // ---- framing ----
  struct Framing { int mode = -1; int rect[4] = {0, 0, 0, 0}; };
  Framing framing_{0, {0, 0, 0, 0}};   // the context's (plain calls, and sources that follow it)
  FramingParams framing_auto_{300, 10, 32};
  std::vector<Framing> src_framing_;   // per source: mode -1 follows framing_
  const Framing& frame_framing(int id) const { return id < 0 || src_framing_[id].mode < 0 ? framing_ : src_framing_[id]; }
  // the camera has no framing state yet (new, reset, or its last frame was not AUTO): its next AUTO frame jumps
  bool plain_jump_ = true;
  std::vector<char> src_jump_;
  int* d_frame_tab_ = nullptr;       // [FRAMING_ROWS][max_batch] the framing rows of a framed call, written before its launch
  FrameCrop* d_crop_ = nullptr;      // [max_batch] the crop of each frame of the last framed call (the tail reads it)
  int* d_frame_box_ = nullptr;       // [max_batch][4] targets of a plain call (k_framing scratch)
  unsigned* d_frame_counter_ = nullptr;
  int* d_frame_state_ = nullptr;     // [4] the plain stream's state, 1/16 pixel
  int* d_src_frame_state_ = nullptr; // [n_sources][4] the sources' states
  bool last_framed_ = false;         // the last call was framed; last_frames_: its frame count (chunks included)
  int last_frames_ = 0;
  // ---- live backgrounds ----
  struct Live { const uint8_t* p = nullptr; int fmt = 0, w = 0, h = 0; size_t pitch = 0, uv = 0, stride = 0; int size = -1; };
  Live live_;                        // plain calls
  std::vector<Live> src_live_;       // per source
  // resize tables per distinct live size, shared by the plain and the source live backgrounds; an entry no live background
  // uses any more keeps its tables until a new size needs the entry
  struct LiveSize { int w = 0, h = 0, refs = 0; DevResizeTab tab; };
  std::vector<LiveSize> live_sizes_;
  bool check_live(int fmt, int w, int h, size_t pitch, size_t uv, std::string* err) const;
  bool live_size_acquire(int w, int h, int* idx, std::string* err);
  void live_size_release(int idx) { if (idx >= 0) --live_sizes_[idx].refs; }
  // the descriptor of live image l at p, blurred by a Gaussian that follows or not
  LiveDesc live_desc(const Live& l, const uint8_t* p, bool blur) const;
  LiveDesc* d_live_tab_ = nullptr;   // [max_batch] descriptors of a call's frames, written before each launch with live frames
  uint8_t* d_live_stage_ = nullptr;  // [max_batch][H][W][3] resized live images the Gaussian reads
  size_t live_stage_cap_ = 0;
  // Output geometries k_tail reads, [1 + n_sources]: slot 0 the context's (set_output), slot 1 + i own size i.  Each own
  // size is kept once, however many sources use it; a slot no source uses any more is reused by the next new size.
  TailGeo* d_geo_ = nullptr;
  struct OwnSize { int w = 0, h = 0, refs = 0; DevResizeTab tab; };
  std::vector<OwnSize> own_sizes_;
  std::vector<int> src_size_;        // per source: -1 = the context's size, else an index into own_sizes_
  TailGeo ctx_geo() const;
  bool upload_geo(int slot, const TailGeo& g, std::string* err);
  // background bank, one base + one stride for the post kernel: [max_batch] camera-blur slots | [1] the context's effective
  // background | [n_sources] source slots | [pool_slots_] the ring pool, the images of every source ring of more than one
  // image; d_bank_yuyv_ is its YUYV and d_bank_nv12_ its NV12 (the camera-blur slots' are written by the Gaussian of the
  // call, in the call's video format)
  uint8_t* d_bank_ = nullptr, *d_bank_yuyv_ = nullptr, *d_bank_nv12_ = nullptr;
  uint8_t* d_src_bg_ = nullptr;      // [n_sources] resized, unblurred source backgrounds (re-blurred when their strength changes)
  uint8_t* d_pool_bg_ = nullptr;     // [pool_slots_] the same for the ring pool
  size_t pool_slots_ = 0;
  uint8_t* d_green_ = nullptr;       // one plain green frame (the still background of a source without an image)
  uint8_t* d_src_raw_ = nullptr;     // staging of one decoded source background
  size_t src_raw_cap_ = 0;
  DevResizeTab tab_src_;
  int src_bg_w_ = 0, src_bg_h_ = 0;
  // own background of source s: count 0 none, 1 a still in its own slot, more a ring in the pool from bank slot
  // pool0() + base; it blends ring image `cursor`, and every call carrying a frame of s moves the cursor on by `advance`
  struct SrcRing { int count = 0, advance = 0, cursor = 0; size_t base = 0; };
  std::vector<SrcRing> src_ring_;
  size_t pool0() const { return (size_t)max_batch_ + 1 + (size_t)n_sources_; }
  // the pool with source s's ring replaced by one of `count` images (none when count <= 1); false with *err, and nothing
  // changed, when an allocation is refused
  bool resize_pool(int s, int count, std::string* err);
  void move_cursors(const Call& c);
  struct SrcEffect { int bg = SRC_BG_DEFAULT, k = -1; };
  std::vector<SrcEffect> src_fx_;
  std::vector<signed char> src_flip_;   // per source: -1 = the context's flips (flip_h_ / flip_v_), else 0..3
  std::vector<signed char> src_filter_; // per source: -1 = the context's switch (filter_), else 0 (off) or 1 (on)
  // Where source s's background comes from: the context slot, its own bank slot (its effective still background differs
  // from the context's) or the slot of its ring's current image, or its camera frame blurred at strength *k.  *slot: the
  // bank slot the source blends now (not set for camera blur, whose slot is the frame's)
  enum SrcBg { SRC_FROM_CTX = 0, SRC_FROM_SLOT = 1, SRC_FROM_CAMBLUR = 2 };
  int source_bg(int s, int* k, size_t* slot = nullptr) const;
  int bank_slots() const { return (int)(pool0() + pool_slots_); }
  bool refresh_bank_ctx(std::string* err);
  bool refresh_bank_source(int s, std::string* err);
  // every source slot that depends on the context background / strength (strength: the context's strength changed, so
  // own images that follow it are re-blurred too)
  bool refresh_bank_sources_after_ctx(bool strength, std::string* err);
  bool ensure_gauss_tmp(std::string* err);
  void free_sources();

  // Everything a captured launch sequence bakes into its kernel arguments: the call's buffers and layouts (the stride of
  // an absent output does not matter), and the plan's mode (a plain and a sources graph over the same buffers are
  // different graphs), Gaussian classes (strengths within them replay), all-blur, flipped and passed (which frames flip or
  // are filtered off is table data), resized and the largest output size of the sources, which the tail's grid covers
  // (which frame has which size is table data too), the output format, whether frames blend live backgrounds, with
  // the Gaussian classes they add (their images, sizes and strengths within the classes are the live table's data), and the
  // CNN batch of a call with held frames (which frames are segmented is the segment rows' data), and whether the call is
  // framed (modes, rectangles and crops are table data).  The rest of the plan is
  // decided from these.
  struct GraphKey {
    int n, fmt; const void* in; size_t pitch, uv, stride;
    const void* out; const void* video; const void* mask; size_t ostride, vstride, mstride;
    int mode; unsigned gclass; bool all_blur, flipped, resized, passed; long out_px_max; bool bgra; int live; unsigned live_gclass;
    bool framed;
    GraphKey(const Call& c, const Plan& p, long px_max)
        : n(c.n), fmt(c.fmt), in(c.in), pitch(c.pitch), uv(c.uv), stride(c.stride), out(c.out), video(c.video), mask(c.mask),
          ostride(c.out ? c.out_stride : 0), vstride(c.video ? c.video_stride : 0), mstride(c.mask ? c.mask_stride : 0),
          mode(p.mode), gclass(p.gclass), all_blur(p.all_blur), flipped(p.flipped), resized(p.resized), passed(p.passed),
          out_px_max(px_max), bgra(p.bgra), live(p.live), live_gclass(p.live_gclass), framed(p.framed), seg(p.m) {}
    int seg;                         // the CNN batch m (n: every frame segmented, the parent's launches)
    auto tie() const {
      return std::tie(n, fmt, in, pitch, uv, stride, out, video, mask, ostride, vstride, mstride, mode, gclass, all_blur, flipped, resized,
                      passed, out_px_max, bgra, live, live_gclass, framed, seg);
    }
    bool operator<(const GraphKey& r) const { return tie() < r.tie(); }
  };
#ifndef BSB_EMU
  // a replay restores the launch count and the native flag of its graph: toggling the filter switch alternates graphs
  struct CapturedCall { cudaGraphExec_t exec; int launches; bool native; };
  std::map<GraphKey, CapturedCall> graphs_;
#endif
};

}  // namespace bsb
