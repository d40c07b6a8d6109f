// backscrub_b200/csrc/resize_taps.h — OpenCV INTER_LINEAR 8-bit taps of cv::resize (formulas pinned in
// oracle/oracle_img.c), one output index at a time.  The host tables (build_resize_tab) and the framed tail, which
// computes the taps of each frame's crop on the fly, run this same arithmetic, so the two cannot drift.  Both sides
// compile without contraction (-fmad=false, -ffp-contract=off), so the double and float steps round alike.
#pragma once
#include "bsb_common.h"

namespace bsb {

// source step of sn -> dn, computed as OpenCV computes it (once per resize)
BSB_HD double resize_scale(int sn, int dn) { return 1.0 / ((double)dn / sn); }

// column dx: left tap *sx (the right one is min(sx + 1, sw - 1)), weights *w0 + *w1 = 2048, clamped at both edges
BSB_HD void resize_tap_x(int dx, double scale, int sw, int* sx, int* w0, int* w1) {
  float fx = (float)((dx + 0.5) * scale - 0.5);
  int s = (int)floorf(fx);
  fx -= (float)s;
  if (s < 0) { fx = 0; s = 0; }
  if (s >= sw - 1) { fx = 0; s = sw - 1; }
  *sx = s;
  *w0 = (int)lrintf((1.f - fx) * 2048.f);
  *w1 = (int)lrintf(fx * 2048.f);
}

// row dy: rows *y0, *y1 clamped into the image, weights unclamped (OpenCV's vertical pass)
BSB_HD void resize_tap_y(int dy, double scale, int sh, int* y0, int* y1, int* w0, int* w1) {
  float fy = (float)((dy + 0.5) * scale - 0.5);
  const int s = (int)floorf(fy);
  fy -= (float)s;
  *y0 = s < 0 ? 0 : (s > sh - 1 ? sh - 1 : s);
  *y1 = s + 1 < 0 ? 0 : (s + 1 > sh - 1 ? sh - 1 : s + 1);
  *w0 = (int)lrintf((1.f - fy) * 2048.f);
  *w1 = (int)lrintf(fy * 2048.f);
}

}  // namespace bsb
