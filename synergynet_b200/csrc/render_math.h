// Arithmetic of the Sim3DR path (SURVEY.md section 8 row f2), shared by the CUDA kernels (kernels_render.cuh) and by
// the host-side emulation the CPU tests run (tests/host_emul/render_emul.cpp compiles this header with g++).
//
// The reference is scalar C++ built for baseline x86-64: every float operation rounds once and none is contracted into
// an FMA (Sim3DR/setup.py passes no -march, so gcc has no FMA to contract to).  To return the same bits, every
// operation here is an explicit round-to-nearest intrinsic on the device (nvcc contracts a*b+c by default) and a
// plain operator on the host (build with -ffp-contract=off).  Operand order follows the reference expression by
// expression; the functions cite the lines they follow (paths relative to the reference root).
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define SYN_HD __host__ __device__ __forceinline__
#else
#define SYN_HD inline
#endif

namespace syn {
namespace rmath {

#if defined(__CUDA_ARCH__)
SYN_HD float mul(float a, float b) { return __fmul_rn(a, b); }
SYN_HD float add(float a, float b) { return __fadd_rn(a, b); }
SYN_HD float sub(float a, float b) { return __fsub_rn(a, b); }
SYN_HD float dvd(float a, float b) { return __fdiv_rn(a, b); }
SYN_HD float sqr(float a) { return __fsqrt_rn(a); }
SYN_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
SYN_HD float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
#else
SYN_HD float mul(float a, float b) { return a * b; }
SYN_HD float add(float a, float b) { return a + b; }
SYN_HD float sub(float a, float b) { return a - b; }
SYN_HD float dvd(float a, float b) { return a / b; }
SYN_HD float sqr(float a) { return sqrtf(a); }
SYN_HD double dmul(double a, double b) { return a * b; }
SYN_HD float fma_rn(float a, float b, float c) { return fmaf(a, b, c); }
#endif

// std::min / std::max as the reference calls them (NaN behaviour of the comparison form, not fminf/fmaxf)
SYN_HD float min_std(float a, float b) { return (b < a) ? b : a; }
SYN_HD float max_std(float a, float b) { return (a < b) ? b : a; }

// (int)v as the reference's x86-64 build computes it (cvttss2si): truncation inside [-2^31, 2^31), INT_MIN for
// everything else, NaN included.  C leaves the out-of-range conversion undefined and nvcc resolves it differently
// (cvt.rzi.s32.f32 saturates to INT_MAX, NaN -> 0), so the range is tested here rather than left to either compiler.
SYN_HD int to_int_x86(float v) {
  return (v >= -2147483648.0f && v < 2147483648.0f) ? (int)v : (int)0x80000000u;
}

// ---- barycentric coordinates -------------------------------------------------------------------------------------
// Sim3DR/lib/rasterize_kernel.cpp:26-51 (is_point_in_tri) and :53-80 (get_point_weight) evaluate the same
// expressions; one evaluation serves both.  v0 = p2 - p0, v1 = p1 - p0, v2 = p - p0.
struct Bary {
  float w0, w1, w2;   // weight[0] = 1 - u - v, weight[1] = v, weight[2] = u  (:77-79)
  bool inside;        // (u >= 0) && (v >= 0) && (u + v < 1)                   (:50)
};

SYN_HD Bary barycentric(float px, float py, float x0, float y0, float x1, float y1, float x2, float y2) {
  const float v0x = sub(x2, x0), v0y = sub(y2, y0);
  const float v1x = sub(x1, x0), v1y = sub(y1, y0);
  const float v2x = sub(px, x0), v2y = sub(py, y0);
  const float dot00 = add(mul(v0x, v0x), mul(v0y, v0y));
  const float dot01 = add(mul(v0x, v1x), mul(v0y, v1y));
  const float dot02 = add(mul(v0x, v2x), mul(v0y, v2y));
  const float dot11 = add(mul(v1x, v1x), mul(v1y, v1y));
  const float dot12 = add(mul(v1x, v2x), mul(v1y, v2y));
  const float den = sub(mul(dot00, dot11), mul(dot01, dot01));
  const float inv = (den == 0.0f) ? 0.0f : dvd(1.0f, den);
  const float u = mul(sub(mul(dot11, dot02), mul(dot01, dot12)), inv);
  const float v = mul(sub(mul(dot00, dot12), mul(dot01, dot02)), inv);
  Bary b;
  b.w0 = sub(sub(1.0f, u), v);
  b.w1 = v;
  b.w2 = u;
  b.inside = (u >= 0.0f) && (v >= 0.0f) && (add(u, v) < 1.0f);
  return b;
}

// weight[0] * a0 + weight[1] * a1 + weight[2] * a2, left to right (depth :239, colour :247)
SYN_HD float interp(const Bary& b, float a0, float a1, float a2) {
  return add(add(mul(b.w0, a0), mul(b.w1, a1)), mul(b.w2, a2));
}

// ---- one triangle, set up for the z-buffer pass -----------------------------------------------------------------------
struct TriSetup {
  float x0, y0, z0, x1, y1, z1, x2, y2, z2;
  int xmin, xmax, ymin, ymax;   // pixel bounding box, clamped to the image (:226-234); empty if xmax < xmin || ymax < ymin
};

// A maximum at or beyond 2^31 (or NaN) converts to INT_MIN, so the reference skips the triangle (its box is empty).
SYN_HD bool tri_setup(TriSetup& t, int w, int h) {
  t.xmin = to_int_x86(floorf(min_std(t.x0, min_std(t.x1, t.x2))));
  t.xmax = to_int_x86(ceilf(max_std(t.x0, max_std(t.x1, t.x2))));
  t.ymin = to_int_x86(floorf(min_std(t.y0, min_std(t.y1, t.y2))));
  t.ymax = to_int_x86(ceilf(max_std(t.y0, max_std(t.y1, t.y2))));
  if (t.xmin < 0) t.xmin = 0;
  if (t.xmax > w - 1) t.xmax = w - 1;
  if (t.ymin < 0) t.ymin = 0;
  if (t.ymax > h - 1) t.ymax = h - 1;
  return !(t.xmax < t.xmin || t.ymax < t.ymin);
}

// The serial loop keeps, per pixel, the triangle with the greatest interpolated depth and -- because its test is a
// strict `>` against the buffer (:241) -- the FIRST such triangle on ties; the buffer starts at -1e8 (Sim3DR.py:23).
// Packed as a 64-bit key whose maximum is that winner: high word = the depth's bits mapped to an order-preserving
// unsigned, low word = ~triangle index.  Key 0 = "nothing drawn" (every depth above -1e8 maps above 0x334143DF).
constexpr float kDepthInit = -1e8f;

SYN_HD uint32_t float_ordered(float f) {
  union { float f; uint32_t u; } c;
  c.f = f;
  return (c.u & 0x80000000u) ? ~c.u : (c.u | 0x80000000u);
}
SYN_HD float ordered_float(uint32_t o) {
  union { float f; uint32_t u; } c;
  c.u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
  return c.f;
}
// -0 and +0 are one depth: the serial `>` test sees them as a tie, which the lower triangle index wins
SYN_HD uint64_t depth_key(float depth, uint32_t tri) {
  return ((uint64_t)float_ordered(depth == 0.0f ? 0.0f : depth) << 32) | (uint64_t)(0xFFFFFFFFu - tri);
}
SYN_HD uint32_t key_tri(uint64_t key) { return 0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull); }
SYN_HD float key_depth(uint64_t key) { return ordered_float((uint32_t)(key >> 32)); }

// Candidate key of triangle `tri` at pixel (x, y); false = the pixel is outside, or its depth does not beat the initial buffer.
SYN_HD bool pixel_key(const TriSetup& t, uint32_t tri, int x, int y, uint64_t& key) {
  const Bary b = barycentric((float)x, (float)y, t.x0, t.y0, t.x1, t.y1, t.x2, t.y2);
  if (!b.inside) return false;
  const float d = interp(b, t.z0, t.z1, t.z2);
  if (!(d > kDepthInit)) return false;
  key = depth_key(d, tri);
  return true;
}

// (unsigned char)((1 - alpha) * image + alpha * 255 * p_color)  (:249-255): x86 truncates to int32 and keeps the low
// byte, so a value in [256, 2^31) wraps, a negative one wraps from below, and one at or beyond 2^31 (or NaN) gives 0
SYN_HD unsigned char blend_u8(unsigned char img, float alpha, float p_color) {
  const float v = add(mul(sub(1.0f, alpha), (float)(int)img), mul(mul(alpha, 255.0f), p_color));
  return (unsigned char)to_int_x86(v);
}

// ---- the overlay blend (utils/render.py:45, cv2.addWeighted(img, 1 - alpha, overlap, alpha, 0) on uint8) ----------------
// OpenCV 4.x evaluates every element, in its SIMD body and its scalar tail alike, as
//   saturate_cast<uchar>(fma(a, w_a, b * w_b))      w_a = (float)(1 - alpha) (the subtraction is Python's, in double),
//                                                   w_b = (float)alpha, the product b * w_b rounded once, gamma = 0
// so the fused multiply-add is written out here rather than left to the compiler's contraction: the unfused
// a * w_a + b * w_b gives other bytes (733 of the 65 536 (a, b) pairs at alpha = 0.1).  saturate_cast rounds half to
// even (cvRound) and clamps to [0, 255]; a value outside int's range converts to INT_MIN on x86 (cvtss2si / cvtps2dq),
// which the clamp then sends to 0 (to_int_x86) -- kept so that every finite alpha gives cv2's byte.
SYN_HD unsigned char add_weighted_u8(unsigned char a, unsigned char b, double alpha) {
  const float wa = (float)(1.0 - alpha), wb = (float)alpha;
  const int iv = to_int_x86(rintf(fma_rn((float)a, wa, mul((float)b, wb))));
  return (unsigned char)(iv < 0 ? 0 : (iv > 255 ? 255 : iv));
}

// ---- per-mesh pixel boxes of the frame-axis rasteriser ---------------------------------------------------------------------
// A mesh's box is the union of the clamped boxes tri_setup gives its drawable triangles: every pixel its depth pass can
// key lies inside, so its keys need only box-many slots.  Empty: x1 < x0 (then area 0).
struct PixBox { int x0, y0, x1, y1; };
SYN_HD PixBox pix_box_empty() { PixBox b; b.x0 = b.y0 = 0; b.x1 = b.y1 = -1; return b; }
SYN_HD void pix_box_add(PixBox& b, const TriSetup& t) {
  if (b.x1 < b.x0 || b.y1 < b.y0) { b.x0 = t.xmin; b.y0 = t.ymin; b.x1 = t.xmax; b.y1 = t.ymax; return; }
  if (t.xmin < b.x0) b.x0 = t.xmin;
  if (t.ymin < b.y0) b.y0 = t.ymin;
  if (t.xmax > b.x1) b.x1 = t.xmax;
  if (t.ymax > b.y1) b.y1 = t.ymax;
}
SYN_HD long long pix_box_area(const PixBox& b) {
  return (b.x1 < b.x0 || b.y1 < b.y0) ? 0ll : (long long)(b.x1 - b.x0 + 1) * (long long)(b.y1 - b.y0 + 1);
}
// slot of pixel (x, y) in the box's keys, row-major
SYN_HD long long pix_box_slot(const PixBox& b, int x, int y) { return (long long)(y - b.y0) * (b.x1 - b.x0 + 1) + (x - b.x0); }

// ---- normals (Sim3DR/lib/rasterize_kernel.cpp:158-213, _get_normal) ----------------------------------------------------
// un-normalised face normal (p1 - p0) x (p2 - p0)  (:173-186)
SYN_HD void tri_normal(const float* p0, const float* p1, const float* p2, float* n) {
  const float v1x = sub(p1[0], p0[0]), v1y = sub(p1[1], p0[1]), v1z = sub(p1[2], p0[2]);
  const float v2x = sub(p2[0], p0[0]), v2y = sub(p2[1], p0[1]), v2z = sub(p2[2], p0[2]);
  n[0] = sub(mul(v1y, v2z), mul(v1z, v2y));
  n[1] = sub(mul(v1z, v2x), mul(v1x, v2z));
  n[2] = sub(mul(v1x, v2y), mul(v1y, v2x));
}
// n / sqrt(nx^2 + ny^2 + nz^2); the reference has its zero guard commented out (:207), an isolated vertex is 0/0 = NaN
SYN_HD void normalize3(float* n) {
  const float det = sqr(add(add(mul(n[0], n[0]), mul(n[1], n[1])), mul(n[2], n[2])));
  n[0] = dvd(n[0], det);
  n[1] = dvd(n[1], det);
  n[2] = dvd(n[2], det);
}

// ---- lighting (Sim3DR/lighting.py:37-66, RenderPipeline.__call__, float32 numpy arithmetic) ---------------------------
struct LightCfg {          // lighting.py:24-32 after convert_type
  float intensity_ambient, intensity_directional, intensity_specular;
  float color_ambient[3], color_directional[3], light_pos[3], view_pos[3];
  int specular_exp;
};
// per-face statistics of norm_vertices (lighting.py:9-14): since subtraction, division by a positive number and
// doubling are monotonic, the extremes of every intermediate array are the images of the coordinate extremes
struct NormStats { float mn[3], mx[3]; };

// x ** n for the small integer exponent of the specular term.  numpy calls powf (an SVML variant on AVX-512 hosts,
// <= 1 ulp off the exact value and different from glibc's): there is no bit pattern to match, so this returns the
// correctly rounded result of the exact product (double arithmetic, one final rounding).
SYN_HD float powi(float x, int n) {
  double r = 1.0, b = (double)x;
  int e = n < 0 ? -n : n;
  while (e) {
    if (e & 1) r = dmul(r, b);
    b = dmul(b, b);
    e >>= 1;
  }
  return (float)(n < 0 ? 1.0 / r : r);
}
SYN_HD float clip01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

SYN_HD void vertex_light(const float* v, const float* nrm, const NormStats& s, const LightCfg& c, float* light) {
  // norm_vertices: v -= min; v /= max(v); v *= 2; v -= max(v, axis 0) / 2
  float gmax = sub(s.mx[0], s.mn[0]);
  gmax = fmaxf(gmax, sub(s.mx[1], s.mn[1]));
  gmax = fmaxf(gmax, sub(s.mx[2], s.mn[2]));
  float vn[3];
  for (int k = 0; k < 3; ++k) {
    const float top = mul(dvd(sub(s.mx[k], s.mn[k]), gmax), 2.0f);
    vn[k] = sub(mul(dvd(sub(v[k], s.mn[k]), gmax), 2.0f), dvd(top, 2.0f));
  }
  float l[3] = {0.0f, 0.0f, 0.0f};
  if (c.intensity_ambient > 0.0f)
    for (int k = 0; k < 3; ++k) l[k] = add(l[k], mul(c.intensity_ambient, c.color_ambient[k]));
  if (c.intensity_directional > 0.0f) {
    float d[3], dn;
    for (int k = 0; k < 3; ++k) d[k] = sub(c.light_pos[k], vn[k]);
    dn = sqr(add(add(mul(d[0], d[0]), mul(d[1], d[1])), mul(d[2], d[2])));
    for (int k = 0; k < 3; ++k) d[k] = dvd(d[k], dn);
    const float cosv = add(add(mul(nrm[0], d[0]), mul(nrm[1], d[1])), mul(nrm[2], d[2]));
    // numpy's clip propagates NaN (an isolated vertex has a NaN normal); fminf/fmaxf would not
    const float cc = (cosv != cosv) ? cosv : clip01(cosv);
    for (int k = 0; k < 3; ++k) l[k] = add(l[k], mul(c.intensity_directional, mul(c.color_directional[k], cc)));
    if (c.intensity_specular > 0.0f) {
      float e[3], en;
      for (int k = 0; k < 3; ++k) e[k] = sub(c.view_pos[k], vn[k]);
      en = sqr(add(add(mul(e[0], e[0]), mul(e[1], e[1])), mul(e[2], e[2])));
      float spe = 0.0f;
      const float two_cos = mul(2.0f, cosv);
      for (int k = 0; k < 3; ++k) {
        const float refl = sub(mul(two_cos, nrm[k]), d[k]);
        const float t = powi(mul(dvd(e[k], en), refl), c.specular_exp);
        spe = (k == 0) ? t : add(spe, t);
      }
      // np.where(cos != 0, clip(spe, 0, 1), 0), then clip again
      float sp = (cosv != 0.0f) ? ((spe != spe) ? spe : clip01(spe)) : 0.0f;
      sp = (sp != sp) ? sp : clip01(sp);
      for (int k = 0; k < 3; ++k) l[k] = add(l[k], mul(mul(c.intensity_specular, c.color_directional[k]), sp));
    }
  }
  for (int k = 0; k < 3; ++k) light[k] = (l[k] != l[k]) ? l[k] : clip01(l[k]);
}

// ---- NMS overlap test (FaceBoxes/utils/nms/cpu_nms.pyx:52-66, py_cpu_nms.py:20-33), float32 like both ---------------------
SYN_HD float box_area(float x1, float y1, float x2, float y2) { return mul(add(sub(x2, x1), 1.0f), add(sub(y2, y1), 1.0f)); }
SYN_HD float box_overlap(const float* a, float area_a, const float* b, float area_b) {
  const float xx1 = (a[0] >= b[0]) ? a[0] : b[0];
  const float yy1 = (a[1] >= b[1]) ? a[1] : b[1];
  const float xx2 = (a[2] <= b[2]) ? a[2] : b[2];
  const float yy2 = (a[3] <= b[3]) ? a[3] : b[3];
  const float ww = add(sub(xx2, xx1), 1.0f), hh = add(sub(yy2, yy1), 1.0f);
  const float w = (0.0f >= ww) ? 0.0f : ww, h = (0.0f >= hh) ? 0.0f : hh;
  const float inter = mul(w, h);
  return dvd(inter, sub(add(area_a, area_b), inter));
}

}  // namespace rmath
}  // namespace syn
