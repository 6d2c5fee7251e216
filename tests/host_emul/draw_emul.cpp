// Serial host emulation of the line-drawing kernel (synergynet_b200/csrc/kernels_draw.cuh): the segments of each image
// drawn one after the other from the same draw_math.h functions, as loops instead of threads.
// Build: g++ -O2 -ffp-contract=off -shared -fPIC (tests/test_draw_emulation.py does it).  -DSYN_DRAW_VARIANT=n builds
// a deliberately wrong variant for the negative controls of that test.
#include "../../synergynet_b200/csrc/draw_math.h"

using namespace syn::dmath;

namespace {

void put(unsigned char* img, int w, int x, int y, const unsigned char* bgr) {
  unsigned char* p = img + 3 * ((long long)y * w + x);
  p[0] = bgr[0]; p[1] = bgr[1]; p[2] = bgr[2];
}

void draw_one(unsigned char* img, int h, int w, const int32_t* s) {
  const unsigned char bgr[3] = {(unsigned char)(s[4] & 255), (unsigned char)((s[4] >> 8) & 255), (unsigned char)((s[4] >> 16) & 255)};
#if SYN_DRAW_VARIANT == 1
  // variant 1: the first cap centred one pixel right of the rounded end point
  const ThickLine t0 = thick_line_setup(s[0], s[1], s[2], s[3], w, h);
  ThickLine t = t0;
  t.cx[0] = t0.cx[0] + 1;
#elif SYN_DRAW_VARIANT == 2
  // variant 2: the polygon offset dp truncated instead of rounded (cvRound -> (int))
  ThickLine t = thick_line_setup(s[0], s[1], s[2], s[3], w, h);
  if (t.poly) {
    const P64 p0 = {(int64_t)s[0] * kOne, (int64_t)s[1] * kOne}, p1 = {(int64_t)s[2] * kOne, (int64_t)s[3] * kOne};
    const double dx = (double)(p0.x - p1.x) / kOne, dy = (double)(p1.y - p0.y) / kOne;
    const double r = (double)(kThickness << (kShift - 1)) / sqrt(dx * dx + dy * dy);
    const int64_t dpx = (int64_t)(dy * r), dpy = (int64_t)(dx * r);
    const P64 v[4] = {{p0.x + dpx, p0.y + dpy}, {p0.x - dpx, p0.y - dpy}, {p1.x - dpx, p1.y - dpy}, {p1.x + dpx, p1.y + dpy}};
    for (int k = 0; k < 4; ++k) t.edge[k] = line8_setup(v[(k + 3) & 3], v[k], w, h);
    t.fill = fill_setup(v, w, h);
  }
#else
  const ThickLine t = thick_line_setup(s[0], s[1], s[2], s[3], w, h);
#endif
  for (int e = 0; e < 4; ++e) {
    const Line8& l = t.edge[e];
    if (l.count > 0 && (unsigned)l.ex < (unsigned)w && (unsigned)l.ey < (unsigned)h) put(img, w, l.ex, l.ey, bgr);
    for (int k = 0; k < l.count; ++k) {
      int x, y;
      line8_point(l, k, x, y);
      if ((unsigned)x < (unsigned)w && (unsigned)y < (unsigned)h) put(img, w, x, y, bgr);
    }
  }
  for (int y = t.fill.row0; y <= t.fill.row1; ++y) {
    int xl, xr;
    if (fill_span(t.fill, y, w, xl, xr))
      for (int x = xl; x <= xr; ++x) put(img, w, x, y, bgr);
  }
  for (int c = 0; c < 2 && t.live; ++c)
    circle_fill(t.cx[c], t.cy[c], t.radius, w, h, [&](int y, int xl, int xr) {
      for (int x = xl; x <= xr; ++x) put(img, w, x, y, bgr);
    });
}

}  // namespace

extern "C" {

// segs (n,5) int32: x0, y0, x1, y1, colour b | g << 8 | r << 16, drawn in order onto one (h,w,3) image
void emul_draw_lines(unsigned char* img, int h, int w, const int32_t* segs, int n) {
  for (int i = 0; i < n; ++i) draw_one(img, h, w, segs + 5 * i);
}

// the same over a packed image list: image f is (heights[f], widths[f], 3) at byte offsets[f] of `data`, its segments
// seg_start[f] .. seg_start[f+1]-1
void emul_draw_images(unsigned char* data, int n_images, const int64_t* offsets, const int32_t* heights, const int32_t* widths,
                      const int32_t* seg_start, const int32_t* segs) {
  for (int f = 0; f < n_images; ++f)
    emul_draw_lines(data + offsets[f], heights[f], widths[f], segs + 5 * (int64_t)seg_start[f], seg_start[f + 1] - seg_start[f]);
}

}  // extern "C"
