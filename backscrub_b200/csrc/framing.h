// backscrub_b200/csrc/framing.h — auto-framing (include/backscrub_b200.h, bsb_set_framing): the per-camera state step
// that k_framing runs on the device, compiled unchanged into the CPU tests.  DESIGN.md §4 states the formula once.
// Coordinates are frame pixels of the unflipped camera frame; the smoothed state is in 1/16 pixel.
#pragma once
#include "bsb_common.h"

namespace bsb {

enum { FRAMING_OFF = 0, FRAMING_RECT = 1, FRAMING_AUTO = 2 };

// the person pixels (ofinal < 128) of one frame's small mask inside out_roidim: their count and bounding box, columns
// j0..j1 and rows i0..i1 inclusive, relative to out_roidim's origin
struct FramingBox { int count, j0, i0, j1, i1; };
// the context's geometry: frame W x H, roidim (rx, ry, rw, rh) inside it, out_roidim's size sw x sh in the small mask
struct FramingGeo { int W, H, rx, ry, rw, rh, sw, sh; };
// bsb_set_framing_auto: max_zoom in percent (100..1000), margin in percent of the box height (0..100), speed 1..256
struct FramingParams { int max_zoom, margin, speed; };

BSB_HD int framing_clamp(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// target crop t = (x, y, w, h), 1/16 pixel, of a frame with output size ow x oh: the person's box widened to the output
// aspect with `margin` of headroom, or the whole frame when fewer than max(1, sw*sh/1000) pixels are person
BSB_HD void framing_target(const FramingBox& b, const FramingGeo& g, const FramingParams& p, int ow, int oh, int* t) {
  const int thresh = g.sw * g.sh / 1000 > 1 ? g.sw * g.sh / 1000 : 1;
  int x = 0, y = 0, w = g.W, h = g.H;
  if (b.count >= thresh) {
    const int x0 = g.rx + b.j0 * g.rw / g.sw, x1 = g.rx + ((b.j1 + 1) * g.rw + g.sw - 1) / g.sw;
    const int y0 = g.ry + b.i0 * g.rh / g.sh, y1 = g.ry + ((b.i1 + 1) * g.rh + g.sh - 1) / g.sh;
    const int bh = y1 - y0;
    h = framing_clamp(bh * (100 + 2 * p.margin) / 100, g.H * 100 / p.max_zoom, g.H);
    w = (2 * h * ow + oh) / (2 * oh);
    if (w > g.W) { w = g.W; h = framing_clamp((2 * g.W * oh + ow) / (2 * ow), 1, g.H); }
    if (w < 1) w = 1;
    x = framing_clamp((x0 + x1 - w + 2 * g.W) / 2 - g.W, 0, g.W - w);    // centred on the box (floor of the half)
    y = framing_clamp(y0 - p.margin * bh / 100, 0, g.H - h);             // headroom above the box
  }
  t[0] = 16 * x; t[1] = 16 * y; t[2] = 16 * w; t[3] = 16 * h;
}

// one step of state s towards target t: d = t - s; s += (d*speed +- 128) / 256 (C division, so speed 256 jumps); a
// camera without a state (jump) takes the target
BSB_HD void framing_step(int* s, const int* t, int speed, bool jump) {
  for (int k = 0; k < 4; ++k) {
    const int d = t[k] - s[k];
    s[k] = jump ? t[k] : s[k] + (d * speed + (d >= 0 ? 128 : -128)) / 256;
  }
}

// the crop (x, y, w, h) of state s: rounded to pixels and clamped into the W x H frame, w and h >= 1
BSB_HD void framing_crop(const int* s, int W, int H, int* c) {
  const int w = framing_clamp((s[2] + 8) >> 4, 1, W), h = framing_clamp((s[3] + 8) >> 4, 1, H);
  c[0] = framing_clamp((s[0] + 8) >> 4, 0, W - w);
  c[1] = framing_clamp((s[1] + 8) >> 4, 0, H - h);
  c[2] = w; c[3] = h;
}

}  // namespace bsb
