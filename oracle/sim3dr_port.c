/* TEST INFRASTRUCTURE ONLY -- CPU restatement (oracle) of the Sim3DR and NMS algorithms of the reference; nothing under
 * synergynet_b200/ may link or load this file (tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg do).
 *
 * Restates, in plain C and in this project's own words:
 *   port_get_normal   Sim3DR/lib/rasterize_kernel.cpp:158-213   (_get_normal)
 *   port_rasterize    Sim3DR/lib/rasterize_kernel.cpp:217-287   (_rasterize), helpers :26-80
 *   port_cpu_nms      FaceBoxes/utils/nms/cpu_nms.pyx:17-68      (cpu_nms; the .pyx does not build with Cython 3 / numpy 2)
 * Pinned: tests/test_oracle_render.py holds it bit-for-bit to oracle/_ref/libsim3dr_ref.so (the reference's own
 * rasterize_kernel.cpp compiled where it lies, oracle/Makefile) when that is present, and to the golden vectors
 * tests/golden/render_vectors.npz recorded from the reference's Cython module and py_cpu_nms.
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC (no FMA contraction: the reference is baseline x86-64 code). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float w[3]; int inside; } bary_t;

/* barycentric coordinates of (px,py) in triangle a,b,c -- :26-51 and :53-80 compute the same u, v */
static bary_t bary_of(float px, float py, const float* a, const float* b, const float* c) {
  const float e0[2] = {c[0] - a[0], c[1] - a[1]};   /* v0 = p2 - p0 */
  const float e1[2] = {b[0] - a[0], b[1] - a[1]};   /* v1 = p1 - p0 */
  const float e2[2] = {px - a[0], py - a[1]};       /* v2 = p  - p0 */
  const float d00 = e0[0] * e0[0] + e0[1] * e0[1];
  const float d01 = e0[0] * e1[0] + e0[1] * e1[1];
  const float d02 = e0[0] * e2[0] + e0[1] * e2[1];
  const float d11 = e1[0] * e1[0] + e1[1] * e1[1];
  const float d12 = e1[0] * e2[0] + e1[1] * e2[1];
  const float den = d00 * d11 - d01 * d01;
  const float inv = (den == 0) ? 0 : 1 / den;
  const float u = (d11 * d02 - d01 * d12) * inv;
  const float v = (d00 * d12 - d01 * d02) * inv;
  bary_t r;
  r.w[0] = 1 - u - v;
  r.w[1] = v;
  r.w[2] = u;
  r.inside = (u >= 0) && (v >= 0) && (u + v < 1);
  return r;
}

static float fmin_cmp(float a, float b) { return b < a ? b : a; }   /* std::min */
static float fmax_cmp(float a, float b) { return a < b ? b : a; }   /* std::max */

/* vertices (nver,3), triangles (ntri,3) int32; normal (nver,3) is overwritten */
void port_get_normal(float* normal, const float* vertices, const int32_t* triangles, int nver, int ntri) {
  memset(normal, 0, sizeof(float) * 3 * (size_t)nver);          /* np.zeros_like, Sim3DR.py:9 */
  for (int t = 0; t < ntri; ++t) {
    const float* p[3];
    for (int k = 0; k < 3; ++k) p[k] = vertices + 3 * (size_t)triangles[3 * t + k];
    float a[3], b[3], n[3];
    for (int k = 0; k < 3; ++k) { a[k] = p[1][k] - p[0][k]; b[k] = p[2][k] - p[0][k]; }
    n[0] = a[1] * b[2] - a[2] * b[1];
    n[1] = a[2] * b[0] - a[0] * b[2];
    n[2] = a[0] * b[1] - a[1] * b[0];
    /* the reference fills a triangle-normal array first and scatters it in a second loop over the same order:
     * the sums into each vertex associate identically when done in one loop */
    for (int k = 0; k < 3; ++k) {
      float* dst = normal + 3 * (size_t)triangles[3 * t + k];
      dst[0] += n[0]; dst[1] += n[1]; dst[2] += n[2];
    }
  }
  for (int v = 0; v < nver; ++v) {
    float* n = normal + 3 * (size_t)v;
    const float len = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    n[0] = n[0] / len; n[1] = n[1] / len; n[2] = n[2] / len;     /* no zero guard (:207 is commented out) */
  }
}

/* image (h,w,c) uint8 in place; depth (h,w) in place (caller initialises it, Sim3DR.py:23 uses -1e8) */
void port_rasterize(unsigned char* image, const float* vertices, const int32_t* triangles, const float* colors, float* depth,
                    int ntri, int h, int w, int c, float alpha, int reverse) {
  for (int t = 0; t < ntri; ++t) {
    const int32_t* id = triangles + 3 * (size_t)t;
    const float* a = vertices + 3 * (size_t)id[0];
    const float* b = vertices + 3 * (size_t)id[1];
    const float* q = vertices + 3 * (size_t)id[2];
    int x_lo = (int)floorf(fmin_cmp(a[0], fmin_cmp(b[0], q[0])));
    int x_hi = (int)ceilf(fmax_cmp(a[0], fmax_cmp(b[0], q[0])));
    int y_lo = (int)floorf(fmin_cmp(a[1], fmin_cmp(b[1], q[1])));
    int y_hi = (int)ceilf(fmax_cmp(a[1], fmax_cmp(b[1], q[1])));
    if (x_lo < 0) x_lo = 0;
    if (y_lo < 0) y_lo = 0;
    if (x_hi > w - 1) x_hi = w - 1;
    if (y_hi > h - 1) y_hi = h - 1;
    if (x_hi < x_lo || y_hi < y_lo) continue;
    for (int y = y_lo; y <= y_hi; ++y)
      for (int x = x_lo; x <= x_hi; ++x) {
        const bary_t r = bary_of((float)x, (float)y, a, b, q);
        if (!r.inside) continue;
        const float z = r.w[0] * a[2] + r.w[1] * b[2] + r.w[2] * q[2];
        if (!(z > depth[(size_t)y * w + x])) continue;
        unsigned char* px = image + ((size_t)(reverse ? h - 1 - y : y) * w + x) * c;
        for (int k = 0; k < c; ++k) {
          const float col = r.w[0] * colors[(size_t)c * id[0] + k] + r.w[1] * colors[(size_t)c * id[1] + k] +
                            r.w[2] * colors[(size_t)c * id[2] + k];
          px[k] = (unsigned char)((1 - alpha) * px[k] + alpha * 255 * col);
        }
        depth[(size_t)y * w + x] = z;
      }
  }
}

/* dets (n,5) float32, order (n) = indices by descending score (the caller's argsort, as :27); keep (n) out; returns count.
 * ge != 0: suppress when ovr >= thresh (cpu_nms.pyx:65, thresh a C double); ge == 0: py_cpu_nms.py:35 keeps ovr <= thresh
 * with a float32 comparison, so a NaN overlap suppresses there */
int port_nms(const float* dets, const int64_t* order, int n, double thresh, int ge, int64_t* keep) {
  unsigned char* dead = (unsigned char*)calloc((size_t)(n > 0 ? n : 1), 1);
  int cnt = 0;
  const float thr_f = (float)thresh;
  for (int a = 0; a < n; ++a) {
    const int64_t i = order[a];
    if (dead[i]) continue;
    keep[cnt++] = i;
    const float* bi = dets + 5 * i;
    const float area_i = (bi[2] - bi[0] + 1) * (bi[3] - bi[1] + 1);
    for (int q = a + 1; q < n; ++q) {
      const int64_t j = order[q];
      if (dead[j]) continue;
      const float* bj = dets + 5 * j;
      const float area_j = (bj[2] - bj[0] + 1) * (bj[3] - bj[1] + 1);
      const float xx1 = bi[0] >= bj[0] ? bi[0] : bj[0], yy1 = bi[1] >= bj[1] ? bi[1] : bj[1];
      const float xx2 = bi[2] <= bj[2] ? bi[2] : bj[2], yy2 = bi[3] <= bj[3] ? bi[3] : bj[3];
      const float ww = xx2 - xx1 + 1, hh = yy2 - yy1 + 1;
      const float iw = 0.0f >= ww ? 0.0f : ww, ih = 0.0f >= hh ? 0.0f : hh;
      const float inter = iw * ih;
      const float ovr = inter / (area_i + area_j - inter);
      if (ge ? ((double)ovr >= thresh) : !(ovr <= thr_f)) dead[j] = 1;
    }
  }
  free(dead);
  return cnt;
}
