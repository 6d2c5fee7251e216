// Arithmetic of the ROI crop + resize stage (cv2.resize on uint8 BGR crops), shared by the CUDA kernel
// (kernels_resize.cuh) and by the host emulation the CPU tests run (tests/host_emul/resize_emul.cpp compiles this header
// with g++).
//
// The result must be OpenCV's, bit for bit: the get_all_outputs goldens were recorded from crops cv2 made.  cv2.resize on
// CV_8UC3 with INTER_LINEAR / INTER_LANCZOS4 runs OpenCV's generic fixed-point path (imgproc/src/resize.cpp: resize(),
// interpolateLanczos4, HResizeLinear / HResizeLanczos4, VResizeLinear / VResizeLanczos4, resizeAreaFast_); the same bytes
// come out with IPP on or off.  What it does, per axis of a source of length n resized to m:
//   scale = 1 / ((double)m / n);  f = (float)((d + 0.5) * scale - 0.5);  s = floor(f);  f -= s (float)
//   linear, x axis only: s < 0 -> (s, f) = (0, 0); s >= n-1 -> (s, f) = (n-1, 0).  The y axis is not clamped.
//   coefficients (float): linear (1-f, f); Lanczos4 as interpolateLanczos4 below
//   fixed point: short = saturate(cvRound(c * 2048))                      (INTER_RESIZE_COEF_BITS = 11)
//   taps: source index s - (k/2 - 1) + j, j < k, clamped to [0, n-1] (replicate border)
//   horizontal: H = sum src * alpha (int);  vertical: Lanczos4 sat_u8((sum beta * H + 2^21) >> 22), linear the vector
//   formula of VResizeLinearVec_32s8u, sat_u8((((b0 * (H0 >> 4)) >> 16) + ((b1 * (H1 >> 4)) >> 16) + 2) >> 2)
//   INTER_LINEAR with the source exactly twice the destination on both axes is resizeAreaFast_: (a + b + c + d + 2) >> 2.
// int32 range (OpenCV sums in int as well): with P / N the sums of the positive / negative fixed-point taps of one
// output, H lies in [-255 N_alpha, 255 P_alpha] and sum beta * H within +-255 (P^2 + N^2) for the largest P, N.  For
// Lanczos4, P <= 2780 and N <= 732 (tests/test_resize_emulation.py scans 200 000 fractional positions; neighbouring
// positions move a tap by far less than one unit), so |sum + 2^21| <= 255 * (2780^2 + 732^2) + 2^21 ~ 2.110e9 < 2^31 - 1.
// Linear taps are non-negative and sum to 2048: far below.
// Crop semantics (crop_img, utils/inference.py:95-125): crop pixel (cy, cx) = img[y0 + cy, x0 + cx] inside the image, 0
// outside; the resampler clamps a tap to the crop's bounds first (border replication of the zero fill), then maps it.
#pragma once
#include <stdint.h>
#include <math.h>
#include <float.h>

#if defined(__CUDACC__)
#define SYN_RZ_HD __host__ __device__ __forceinline__
#else
#define SYN_RZ_HD inline
#endif

namespace syn {
namespace rsz {

enum { kInterLinear = 1, kInterLanczos4 = 4 };          // cv::INTER_LINEAR, cv::INTER_LANCZOS4

// ---- plan layout ----------------------------------------------------------------------------------------------------------
// One byte buffer for B ROIs resized to out_h x out_w with k taps (2 linear, 8 Lanczos4):
//   RoiHdr[B]  |  int32 xofs[B][out_w]  |  int32 yofs[B][out_h]  |  int16 xcoef[B][out_w][k]  |  int16 ycoef[B][out_h][k]
// xofs / yofs hold the first tap's crop index s - (k/2 - 1), unclamped.
struct RoiHdr {
  int32_t x0, y0, cw, ch;    // crop origin in the image (may be negative) and crop size
  int32_t area;              // 1: exact 2x shrink on both axes in linear mode (resizeAreaFast_); tables unused
  int32_t frame;             // image of the stack this ROI reads (syn_crop_resize_batch); 0 in a one-image plan
  int32_t pad[2];
};

struct PlanView {
  const RoiHdr* hdr;
  const int32_t *xofs, *yofs;
  const int16_t *xcoef, *ycoef;
};

SYN_RZ_HD int taps_of(int mode) { return mode == kInterLanczos4 ? 8 : 2; }

SYN_RZ_HD long long plan_bytes(int batch, int out_h, int out_w, int k) {
  return (long long)batch * ((long long)sizeof(RoiHdr) + (long long)(out_w + out_h) * (4 + 2 * k));
}

SYN_RZ_HD PlanView plan_view(const void* plan, int batch, int out_h, int out_w, int k) {
  const char* p = static_cast<const char*>(plan);
  PlanView v;
  v.hdr = reinterpret_cast<const RoiHdr*>(p);
  p += sizeof(RoiHdr) * (size_t)batch;
  v.xofs = reinterpret_cast<const int32_t*>(p);
  p += 4 * (size_t)batch * out_w;
  v.yofs = reinterpret_cast<const int32_t*>(p);
  p += 4 * (size_t)batch * out_h;
  v.xcoef = reinterpret_cast<const int16_t*>(p);
  p += 2 * (size_t)batch * out_w * k;
  v.ycoef = reinterpret_cast<const int16_t*>(p);
  return v;
}

// ---- plan builder (plain host functions: the Lanczos4 tables take libm's double sin / cos, as OpenCV does; CUDA's may
// differ in the last ulp and flip a tap that sits on a rounding boundary) --------------------------------------------------

// interpolateLanczos4 (resize.cpp): float accumulation of the float-rounded taps, then scaled by the float reciprocal
inline void lanczos4_coeffs(float x, float* c) {
  static const double s45 = 0.70710678118654752440;
  static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  if (x < FLT_EPSILON) {
    for (int i = 0; i < 8; ++i) c[i] = 0.f;
    c[3] = 1.f;
    return;
  }
  const float x3 = x + 3.0f;                             // `x+3` is float arithmetic in the C++ source
  const double y0 = -(double)x3 * 3.14159265358979323846 * 0.25, s0 = sin(y0), c0 = cos(y0);
  float sum = 0.f;
  for (int i = 0; i < 8; ++i) {
    const double y = -(double)(x3 - (float)i) * 3.14159265358979323846 * 0.25;
    c[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    sum += c[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) c[i] *= sum;
}

// saturate_cast<short>(float): cvRound (round half to even) then clamp
inline int16_t fix11(float c) {
  const float v = nearbyintf(c * 2048.f);
  return (int16_t)(v > 32767.f ? 32767 : (v < -32768.f ? -32768 : (int)v));
}

// One axis: n source pixels -> m outputs.  x_axis selects the linear mode's edge clamp (resize.cpp clamps xofs only).
inline void build_axis(int n, int m, int mode, bool x_axis, int32_t* ofs, int16_t* coef) {
  const int k = taps_of(mode);
  const double scale = 1.0 / ((double)m / n);
  for (int d = 0; d < m; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= (float)s;
    float c[8];
    if (mode == kInterLanczos4) {
      lanczos4_coeffs(f, c);
    } else {
      if (x_axis && s < 0) { f = 0.f; s = 0; }
      if (x_axis && s >= n - 1) { f = 0.f; s = n - 1; }
      c[0] = 1.f - f;
      c[1] = f;
    }
    ofs[d] = s - (k / 2 - 1);
    for (int j = 0; j < k; ++j) coef[(size_t)d * k + j] = fix11(c[j]);
  }
}

// resize(): INTER_LINEAR turns into the fast area path when both scales are exactly 2
inline bool exact_halving(int n_w, int n_h, int m_w, int m_h) {
  const double sx = 1.0 / ((double)m_w / n_w), sy = 1.0 / ((double)m_h / n_h);
  const int ix = (int)nearbyint(sx), iy = (int)nearbyint(sy);
  return fabs(sx - ix) < DBL_EPSILON && fabs(sy - iy) < DBL_EPSILON && ix == 2 && iy == 2;
}

// rois: (B,4) int32 x0, y0, x1, y1 already rounded; every ROI non-empty, sizes >= 1, mode linear / Lanczos4 (the caller
// validated them).  plan: plan_bytes(batch, out_h, out_w, taps_of(mode)) bytes.  frames: nullptr (one image), or the
// frame index of every ROI.
inline void build_plan(const int32_t* rois, int batch, int out_h, int out_w, int mode, void* plan, const int32_t* frames = nullptr) {
  const int k = taps_of(mode);
  const PlanView v = plan_view(plan, batch, out_h, out_w, k);
  RoiHdr* hdr = const_cast<RoiHdr*>(v.hdr);
  for (int b = 0; b < batch; ++b) {
    RoiHdr& h = hdr[b];
    h.x0 = rois[4 * b];
    h.y0 = rois[4 * b + 1];
    h.cw = rois[4 * b + 2] - rois[4 * b];
    h.ch = rois[4 * b + 3] - rois[4 * b + 1];
    h.area = (mode == kInterLinear && exact_halving(h.cw, h.ch, out_w, out_h)) ? 1 : 0;
    h.frame = frames ? frames[b] : 0;
    h.pad[0] = h.pad[1] = 0;
    build_axis(h.cw, out_w, mode, true, const_cast<int32_t*>(v.xofs) + (size_t)b * out_w, const_cast<int16_t*>(v.xcoef) + (size_t)b * out_w * k);
    build_axis(h.ch, out_h, mode, false, const_cast<int32_t*>(v.yofs) + (size_t)b * out_h, const_cast<int16_t*>(v.ycoef) + (size_t)b * out_h * k);
  }
}

// ---- per-pixel integer arithmetic ----------------------------------------------------------------------------------------
SYN_RZ_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
SYN_RZ_HD uint8_t sat_u8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// Crop pixel (cy, cx) of ROI h, channel 0..2 into px; zero outside the image (crop_img's fill).
SYN_RZ_HD void crop_pixel(const uint8_t* img, int height, int width, const RoiHdr& h, int cy, int cx, int* px) {
  const int iy = h.y0 + cy, ix = h.x0 + cx;
  if (iy < 0 || iy >= height || ix < 0 || ix >= width) {
    px[0] = px[1] = px[2] = 0;
    return;
  }
  const uint8_t* p = img + ((size_t)iy * width + ix) * 3;
  px[0] = p[0];
  px[1] = p[1];
  px[2] = p[2];
}

// Output pixel (oy, ox) of ROI b, three channels into out[0..2].  K = taps_of(mode).
template <int K>
SYN_RZ_HD void resize_pixel(const uint8_t* img, int height, int width, const PlanView& v, int b, int out_h, int out_w, int oy, int ox,
                            uint8_t* out) {
  const RoiHdr h = v.hdr[b];
  int px[3];
  if (K == 2 && h.area) {                              // resizeAreaFast_: 2x2 mean, (a+b+c+d+2) >> 2
    int acc[3] = {2, 2, 2};
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        crop_pixel(img, height, width, h, 2 * oy + dy, 2 * ox + dx, px);
        for (int c = 0; c < 3; ++c) acc[c] += px[c];
      }
    for (int c = 0; c < 3; ++c) out[c] = (uint8_t)(acc[c] >> 2);
    return;
  }
  const int sx0 = v.xofs[(size_t)b * out_w + ox], sy0 = v.yofs[(size_t)b * out_h + oy];
  const int16_t* ax = v.xcoef + ((size_t)b * out_w + ox) * K;
  const int16_t* by = v.ycoef + ((size_t)b * out_h + oy) * K;
  int acc[3] = {0, 0, 0};                              // int32 cannot overflow: see the bound in the header comment
  for (int j = 0; j < K; ++j) {
    const int cy = clampi(sy0 + j, 0, h.ch - 1);
    int H[3] = {0, 0, 0};
    for (int i = 0; i < K; ++i) {
      crop_pixel(img, height, width, h, cy, clampi(sx0 + i, 0, h.cw - 1), px);
      for (int c = 0; c < 3; ++c) H[c] += px[c] * (int)ax[i];
    }
    const int beta = by[j];
    for (int c = 0; c < 3; ++c) acc[c] += (K == 2) ? ((beta * (H[c] >> 4)) >> 16) : beta * H[c];
  }
  for (int c = 0; c < 3; ++c) out[c] = (K == 2) ? sat_u8((acc[c] + 2) >> 2) : sat_u8((acc[c] + (1 << 21)) >> 22);
}

}  // namespace rsz
}  // namespace syn
