// Arithmetic of the pose-axis drawing (utils/inference.py:199-244, draw_axis: three cv2.line calls of thickness 4 per
// face), shared by the CUDA kernel (kernels_draw.cuh) and by the host emulation the CPU tests run
// (tests/host_emul/draw_emul.cpp compiles this header with g++).
//
// The result must be OpenCV's, byte for byte.  cv2.line(img, p0, p1, color, 4) with the default LINE_8 and shift 0 is
// restated here from OpenCV 4.x's algorithm (imgproc/src/drawing.cpp: line, ThickLine, FillConvexPoly, Line2, Circle)
// and held to the cv2 binary (4.13.0) by tests/test_draw_emulation.py:
//   * the segment is first clipped (clipLine) to the canvas grown by the thickness on every side, the rectangle
//     [-4, w + 3] x [-4, h + 3]; a segment wholly outside draws nothing.  The clipped ends are integers again.
//   * the ends go to 16-bit fixed point (v << 16);  dx = (p0.x - p1.x) / 2^16, dy = (p1.y - p0.y) / 2^16 (double);
//     if dx^2 + dy^2 > DBL_EPSILON:  r = 2^17 / sqrt(dx^2 + dy^2),  dp = (cvRound(dy r), cvRound(dx r)),  and the
//     parallelogram p0 + dp, p0 - dp, p1 - dp, p1 + dp is filled by FillConvexPoly (shift 16):
//       - its four edges are drawn as 8-connected fixed-point lines (Line2), each clipped to the canvas (in 1/2^16 px);
//       - it is scanned row by row between its two vertex chains: an edge from vertex a to b is entered at row ty(a)
//         with x = x(a) and stepped by (2 (x(b) - x(a)) + n) / (2 n) per row, n = ty(b) - ty(a), ty(v) = (y(v) + 2^15)
//         >> 16; a row spans ((x_left + 2^15) >> 16) .. ((x_right + 2^15) >> 16), clipped.  The scan stops at the row
//         of the lowest vertex, which only the outline covers.
//   * a filled circle of radius (2^17 + 2^15) >> 16 = 2 (OpenCV's Bresenham Circle) at each clipped end.
// Every pixel of one call gets the one colour; only the set matters, not the order in which it is written.
//
// 64-bit range: an int32 end grown by 4 leaves int32, so the first clip works in int64 (as OpenCV's Point2l does); its
// intersection offsets are double, as in OpenCV.  After it every coordinate lies in [-4, max(w, h) + 3], so fixed point
// stays below 2^47 for any canvas below 2^31 pixels a side, the per-row step of a fill edge below 2^49 and the closed
// forms below (x at row y, point k of a line) below 2^48.  Those closed forms equal OpenCV's accumulated sums because
// every step is an exact integer addition.  Where OpenCV narrows an int64 pixel coordinate to int, narrow() does the same.
#pragma once
#include <stdint.h>
#include <math.h>
#include <float.h>

#if defined(__CUDACC__)
#define SYN_DR_HD __host__ __device__ __forceinline__
#else
#define SYN_DR_HD inline
#endif

namespace syn {
namespace dmath {

constexpr int kShift = 16;                       // XY_SHIFT
constexpr int64_t kOne = (int64_t)1 << kShift;   // XY_ONE
constexpr int64_t kHalf = kOne >> 1;
constexpr int kThickness = 4;                    // the only thickness draw_axis uses (and the only one restated)

#if defined(__CUDA_ARCH__)
SYN_DR_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
SYN_DR_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
SYN_DR_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
SYN_DR_HD double dsqrt(double a) { return __dsqrt_rn(a); }
SYN_DR_HD int cv_round(double v) { return __double2int_rn(v); }
#else
SYN_DR_HD double dmul(double a, double b) { return a * b; }
SYN_DR_HD double dadd(double a, double b) { return a + b; }
SYN_DR_HD double ddiv(double a, double b) { return a / b; }
SYN_DR_HD double dsqrt(double a) { return sqrt(a); }
SYN_DR_HD int cv_round(double v) { return (int)lrint(v); }      // cvRound: round half to even (cvtsd2si)
#endif

SYN_DR_HD int narrow(int64_t v) { return (int)(uint32_t)(uint64_t)v; }     // OpenCV's (int) of an int64, modulo 2^32

struct P64 { int64_t x, y; };

// ---- clipLine(Size2l, Point2l&, Point2l&) --------------------------------------------------------------------------------
// Cohen-Sutherland against [0, w) x [0, h) of the scaled canvas; the intersection offsets in double, truncated.
SYN_DR_HD bool clip_line(int64_t w, int64_t h, P64& p1, P64& p2) {
  const int64_t right = w - 1, bottom = h - 1;
  if (w <= 0 || h <= 0) return false;
  int64_t &x1 = p1.x, &y1 = p1.y, &x2 = p2.x, &y2 = p2.y;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    int64_t a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (int64_t)ddiv(dmul((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (int64_t)ddiv(dmul((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (int64_t)ddiv(dmul((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (int64_t)ddiv(dmul((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// ---- Line2: one 8-connected line between fixed-point points, as a point list -----------------------------------------
// The end point (rounded) is put first, then count points k = 0 .. count-1 stepping along the major axis.
struct Line8 {
  int count;                // 0: nothing (clipped away); the end point is not drawn either
  bool xmajor;
  int64_t bx, by, step;     // major-axis start (pixels) / minor-axis start (fixed point) and the minor step per point
  int ex, ey;               // the separately drawn end point
};

SYN_DR_HD Line8 line8_setup(P64 p1, P64 p2, int w, int h) {
  Line8 s;
  s.count = 0; s.xmajor = false; s.bx = s.by = s.step = 0; s.ex = s.ey = 0;
  if (!clip_line((int64_t)w << kShift, (int64_t)h << kShift, p1, p2)) return s;
  int64_t dx = p2.x - p1.x, dy = p2.y - p1.y;
  const int64_t j = dx < 0 ? -1 : 0, i = dy < 0 ? -1 : 0;
  const int64_t ax = (dx ^ j) - j, ay = (dy ^ i) - i;
  int64_t ecount;
  if (ax > ay) {                                           // swap the points if dx < 0 (j = -1)
    dy = (dy ^ j) - j;
    p1.x ^= p2.x & j; p2.x ^= p1.x & j; p1.x ^= p2.x & j;
    p1.y ^= p2.y & j; p2.y ^= p1.y & j; p1.y ^= p2.y & j;
    s.step = dy * kOne / (ax | 1);
    ecount = (p2.x - p1.x) >> kShift;
    s.xmajor = true;
  } else {
    dx = (dx ^ i) - i;
    p1.x ^= p2.x & i; p2.x ^= p1.x & i; p1.x ^= p2.x & i;
    p1.y ^= p2.y & i; p2.y ^= p1.y & i; p1.y ^= p2.y & i;
    s.step = dx * kOne / (ay | 1);
    ecount = (p2.y - p1.y) >> kShift;
  }
  p1.x += kHalf;
  p1.y += kHalf;
  s.ex = (int)((p2.x + kHalf) >> kShift);
  s.ey = (int)((p2.y + kHalf) >> kShift);
  if (s.xmajor) { s.bx = p1.x >> kShift; s.by = p1.y; }
  else { s.bx = p1.y >> kShift; s.by = p1.x; }
  s.count = (int)(ecount + 1);
  return s;
}

// point k of the loop (the closed form of `major++, minor += step`)
SYN_DR_HD void line8_point(const Line8& s, int k, int& x, int& y) {
  const int major = (int)(s.bx + k), minor = (int)((s.by + (int64_t)k * s.step) >> kShift);
  x = s.xmajor ? major : minor;
  y = s.xmajor ? minor : major;
}

// ---- FillConvexPoly of the four-corner polygon, row by row -------------------------------------------------------------
struct Fill {
  int row0, row1;           // rows to scan, clipped to the canvas; empty if row1 < row0
  int64_t vx[4];
  int ty[4];
  int imin;
};

SYN_DR_HD Fill fill_setup(const P64* v, int w, int h) {
  Fill f;
  f.row0 = 0; f.row1 = -1; f.imin = 0;
  int64_t xmin = v[0].x, xmax = v[0].x, ymin = v[0].y, ymax = v[0].y;
  for (int i = 0; i < 4; ++i) {
    if (v[i].y < ymin) { ymin = v[i].y; f.imin = i; }
    ymax = v[i].y > ymax ? v[i].y : ymax;
    xmax = v[i].x > xmax ? v[i].x : xmax;
    xmin = v[i].x < xmin ? v[i].x : xmin;
    f.vx[i] = v[i].x;
    f.ty[i] = narrow((v[i].y + kHalf) >> kShift);
  }
  xmin = (xmin + kHalf) >> kShift; xmax = (xmax + kHalf) >> kShift;
  ymin = (ymin + kHalf) >> kShift; ymax = (ymax + kHalf) >> kShift;
  if (narrow(xmax) < 0 || narrow(ymax) < 0 || narrow(xmin) >= w || narrow(ymin) >= h) return f;
  // rows ty(top) .. min(ty(bottom), h - 1); the row of the bottom vertex ends the scan before it is drawn
  int bottom = f.ty[0];
  for (int i = 1; i < 4; ++i) bottom = f.ty[i] > bottom ? f.ty[i] : bottom;
  const int last = narrow(ymax < h - 1 ? ymax : (int64_t)(h - 1));
  f.row0 = f.ty[f.imin] < 0 ? 0 : f.ty[f.imin];
  f.row1 = bottom <= last ? bottom - 1 : last;
  return f;
}

// x (fixed point) of the chain walking from the top vertex in direction di (+1 or +3 = -1 mod 4) at row y
SYN_DR_HD int64_t fill_chain_x(const Fill& f, int di, int y) {
  int i0 = f.imin, i1 = (f.imin + di) & 3;
  for (int k = 0; k < 3 && f.ty[i1] <= y; ++k) { i0 = i1; i1 = (i1 + di) & 3; }
  const int64_t n = (int64_t)f.ty[i1] - f.ty[i0];
  const int64_t dx = ((f.vx[i1] - f.vx[i0]) * 2 + n) / (2 * n);
  return f.vx[i0] + ((int64_t)y - f.ty[i0]) * dx;
}

// the pixels [xl, xr] of row y (row0 <= y <= row1); false if the row has none on the canvas
SYN_DR_HD bool fill_span(const Fill& f, int y, int w, int& xl, int& xr) {
  const int64_t a = fill_chain_x(f, 1, y), b = fill_chain_x(f, 3, y);
  const int64_t left = a > b ? b : a, right = a > b ? a : b;
  xl = narrow((left + kHalf) >> kShift);
  xr = narrow((right + kHalf) >> kShift);
  if (xr < 0 || xl >= w) return false;
  if (xl < 0) xl = 0;
  if (xr >= w) xr = w - 1;
  return xl <= xr;
}

// ---- Circle(img, center, radius, color, fill = 1) ------------------------------------------------------------------------
// hline(y, xl, xr) draws the pixels xl..xr of row y (nothing if xl > xr); every call is inside the canvas.
template <class HLine>
SYN_DR_HD void circle_fill(int cx, int cy, int radius, int w, int h, HLine hline) {
  int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
  const bool inside = cx >= radius && cx < w - radius && cy >= radius && cy < h - radius;
  while (dx >= dy) {
    const int y11 = cy - dy, y12 = cy + dy, y21 = cy - dx, y22 = cy + dx;
    int x11 = cx - dx, x12 = cx + dx, x21 = cx - dy, x22 = cx + dy;
    if (inside) {
      hline(y11, x11, x12); hline(y12, x11, x12);
      hline(y21, x21, x22); hline(y22, x21, x22);
    } else if (x11 < w && x12 >= 0 && y21 < h && y22 >= 0) {
      x11 = x11 > 0 ? x11 : 0;
      x12 = x12 < w - 1 ? x12 : w - 1;
      if ((unsigned)y11 < (unsigned)h) hline(y11, x11, x12);
      if ((unsigned)y12 < (unsigned)h) hline(y12, x11, x12);
      if (x21 < w && x22 >= 0) {
        x21 = x21 > 0 ? x21 : 0;
        x22 = x22 < w - 1 ? x22 : w - 1;
        if ((unsigned)y21 < (unsigned)h) hline(y21, x21, x22);
        if ((unsigned)y22 < (unsigned)h) hline(y22, x21, x22);
      }
    }
    dy++;
    err += plus;
    plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask;
    dx += mask;
    minus -= mask & 2;
  }
}

// ---- ThickLine: cv2.line(img, (x0, y0), (x1, y1), color, 4) --------------------------------------------------------------
struct ThickLine {
  bool live;                // false: the segment lies wholly outside the grown canvas, nothing is drawn
  bool poly;                // false: a zero-length line, only the two caps
  Fill fill;
  Line8 edge[4];            // the outline FillConvexPoly draws: (v3, v0), (v0, v1), (v1, v2), (v2, v3)
  int cx[2], cy[2], radius;
};

SYN_DR_HD ThickLine thick_line_setup(int x0, int y0, int x1, int y1, int w, int h) {
  ThickLine t;
  t.live = false;
  t.poly = false;
  t.fill.row0 = 0; t.fill.row1 = -1;
  for (int k = 0; k < 4; ++k) t.edge[k].count = 0;
  t.radius = 0;
  t.cx[0] = t.cx[1] = t.cy[0] = t.cy[1] = 0;
  // cv::line first clips the segment to the canvas grown by the thickness on every side (clipLine of the Rect
  // (-4, -4, w + 8, h + 8)); a segment wholly outside draws nothing, caps included
  P64 c0 = {(int64_t)x0 + kThickness, (int64_t)y0 + kThickness}, c1 = {(int64_t)x1 + kThickness, (int64_t)y1 + kThickness};
  if (!clip_line((int64_t)w + 2 * kThickness, (int64_t)h + 2 * kThickness, c0, c1)) return t;
  x0 = (int)c0.x - kThickness; y0 = (int)c0.y - kThickness;
  x1 = (int)c1.x - kThickness; y1 = (int)c1.y - kThickness;
  t.live = true;
  const P64 p0 = {(int64_t)x0 * kOne, (int64_t)y0 * kOne}, p1 = {(int64_t)x1 * kOne, (int64_t)y1 * kOne};
  const int64_t half_width = (int64_t)kThickness << (kShift - 1);           // thickness <<= XY_SHIFT - 1; even: no odd term
  const double inv_one = 1.0 / (double)kOne;
  const double dx = dmul((double)(p0.x - p1.x), inv_one), dy = dmul((double)(p1.y - p0.y), inv_one);
  double r = dadd(dmul(dx, dx), dmul(dy, dy));
  t.poly = fabs(r) > DBL_EPSILON;
  if (t.poly) {
    r = ddiv((double)half_width, dsqrt(r));
    const int64_t dpx = cv_round(dmul(dy, r)), dpy = cv_round(dmul(dx, r));
    const P64 v[4] = {{p0.x + dpx, p0.y + dpy}, {p0.x - dpx, p0.y - dpy}, {p1.x - dpx, p1.y - dpy}, {p1.x + dpx, p1.y + dpy}};
    for (int k = 0; k < 4; ++k) t.edge[k] = line8_setup(v[(k + 3) & 3], v[k], w, h);
    t.fill = fill_setup(v, w, h);
  }
  t.cx[0] = narrow((p0.x + kHalf) >> kShift); t.cy[0] = narrow((p0.y + kHalf) >> kShift);
  t.cx[1] = narrow((p1.x + kHalf) >> kShift); t.cy[1] = narrow((p1.y + kHalf) >> kShift);
  t.radius = (int)((half_width + kHalf) >> kShift);
  return t;
}

}  // namespace dmath
}  // namespace syn
