// The pose axes of draw_axis (utils/inference.py:199-244) on the GPU: cv2.line(img, p0, p1, colour, 4) for many segments
// on many images in one launch (syn_draw_lines).  The geometry of one segment -- OpenCV's grown-canvas clip, its
// thick-line parallelogram with outline and scan fill, and the two round caps -- comes from draw_math.h, which the host
// emulation the CPU tests hold to cv2 compiles too.
//
// One CTA per image walks that image's segments in draw order.  Every pixel of one segment takes the one colour, so the
// CTA's threads write a segment's pixels in any order: warps take the fill rows (lanes along the row), threads the
// outline points and the caps.  A barrier separates consecutive segments, so where segments overlap the later one's
// bytes are the ones left, as in the reference's sequence of cv2.line calls.  Writes stay inside the image's own
// (h, w, 3) bytes: every coordinate is clipped to [0, w) x [0, h) before it is stored.
#pragma once
#include "common.cuh"
#include "draw_math.h"

namespace syn {

constexpr int kDrawThreads = 256;

__device__ __forceinline__ void draw_put(uint8_t* img, int w, int x, int y, uint8_t b, uint8_t g, uint8_t r) {
  uint8_t* p = img + 3 * ((long long)y * w + x);
  p[0] = b; p[1] = g; p[2] = r;
}

// frames (n,3) int64: byte offset, height, width of each image; seg_start (n+1); segs (S,5) int32: x0, y0, x1, y1 and the
// colour b | g << 8 | r << 16
__global__ void __launch_bounds__(kDrawThreads) draw_lines_kernel(uint8_t* images, const long long* frames, const int32_t* seg_start,
                                                                  const int32_t* segs) {
  const int f = blockIdx.x;
  uint8_t* img = images + frames[3 * f];
  const int h = (int)frames[3 * f + 1], w = (int)frames[3 * f + 2];
  const int s0 = seg_start[f], s1 = seg_start[f + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  for (int s = s0; s < s1; ++s) {
    const int32_t* q = segs + 5 * (long long)s;
    const uint32_t c = (uint32_t)q[4];
    const uint8_t cb = c & 255, cg = (c >> 8) & 255, cr = (c >> 16) & 255;
    const dmath::ThickLine t = dmath::thick_line_setup(q[0], q[1], q[2], q[3], w, h);
    if (t.live) {
      for (int y = t.fill.row0 + warp; y <= t.fill.row1; y += n_warps) {
        int xl, xr;
        if (dmath::fill_span(t.fill, y, w, xl, xr))
          for (int x = xl + lane; x <= xr; x += 32) draw_put(img, w, x, y, cb, cg, cr);
      }
      // outline: per edge its end point (item 0) and its count points; then the two caps
      int n_items = 2;
      for (int e = 0; e < 4; ++e) n_items += t.edge[e].count > 0 ? t.edge[e].count + 1 : 0;
      for (int i = threadIdx.x; i < n_items; i += blockDim.x) {
        int k = i, e = 0;
        while (e < 4 && k >= (t.edge[e].count > 0 ? t.edge[e].count + 1 : 0)) {
          k -= t.edge[e].count > 0 ? t.edge[e].count + 1 : 0;
          ++e;
        }
        if (e == 4) {
          dmath::circle_fill(t.cx[k], t.cy[k], t.radius, w, h, [&](int y, int xl, int xr) {
            for (int x = xl; x <= xr; ++x) draw_put(img, w, x, y, cb, cg, cr);
          });
          continue;
        }
        int x, y;
        if (k == 0) { x = t.edge[e].ex; y = t.edge[e].ey; }
        else dmath::line8_point(t.edge[e], k - 1, x, y);
        if ((unsigned)x < (unsigned)w && (unsigned)y < (unsigned)h) draw_put(img, w, x, y, cb, cg, cr);
      }
    }
    __syncthreads();
  }
}

}  // namespace syn
