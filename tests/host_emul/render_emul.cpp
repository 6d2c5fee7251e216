// Serial host emulation of the GPU render / NMS kernels (synergynet_b200/csrc/kernels_render.cuh): the same
// render_math.h functions, the same key-maximum and incidence-list algorithms, executed by loops instead of threads.
// Lets the CPU test-suite (no GPU in the build container) hold the arithmetic and the order-free reformulation to the
// oracle bit for bit; the -m gpu tests then only have to show that the CUDA launch code is wired the same way.
// Build: g++ -O2 -ffp-contract=off -shared -fPIC (tests/test_render_emulation.py does it).
#include "../../synergynet_b200/csrc/render_math.h"

#include <cstring>
#include <vector>

using namespace syn::rmath;

extern "C" {

void emul_normals(const float* v, int sv, int sc, int nver, const int32_t* tri, int ntri, const int32_t* inc_start,
                  const int32_t* inc_tri, float* out) {
  std::vector<float> tn(3 * (size_t)ntri);
  for (int i = 0; i < ntri; ++i) {
    float p[3][3];
    for (int k = 0; k < 3; ++k)
      for (int c = 0; c < 3; ++c) p[k][c] = v[(size_t)tri[3 * i + k] * sv + c * sc];
    tri_normal(p[0], p[1], p[2], &tn[3 * (size_t)i]);
  }
  for (int i = 0; i < nver; ++i) {
    float n[3] = {0.f, 0.f, 0.f};
    for (int e = inc_start[i]; e < inc_start[i + 1]; ++e)
      for (int c = 0; c < 3; ++c) n[c] = add(n[c], tn[3 * (size_t)inc_tri[e] + c]);
    normalize3(n);
    for (int c = 0; c < 3; ++c) out[3 * (size_t)i + c] = n[c];
  }
}

void emul_lighting(const float* v, int sv, int sc, int nver, const float* normals, const LightCfg* cfg, const float* texture, float* out) {
  uint32_t lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  for (int i = 0; i < nver; ++i)
    for (int c = 0; c < 3; ++c) {
      const uint32_t o = float_ordered(v[(size_t)i * sv + c * sc]);
      if (~o > lo[c]) lo[c] = ~o;
      if (o > hi[c]) hi[c] = o;
    }
  NormStats s;
  for (int c = 0; c < 3; ++c) { s.mn[c] = ordered_float(~lo[c]); s.mx[c] = ordered_float(hi[c]); }
  for (int i = 0; i < nver; ++i) {
    float p[3], l[3];
    for (int c = 0; c < 3; ++c) p[c] = v[(size_t)i * sv + c * sc];
    vertex_light(p, normals + 3 * (size_t)i, s, *cfg, l);
    for (int c = 0; c < 3; ++c) out[3 * (size_t)i + c] = texture ? mul(texture[3 * (size_t)i + c], l[c]) : l[c];
  }
}

// B meshes: v[b * sb + i * sv + c * sc]; colors (B,nver,ch); image in place; depth_out (B,h,w) or NULL.
// `shuffle` != 0 visits the triangles in a scrambled order: the result must not depend on it.
void emul_rasterize(unsigned char* image, int h, int w, int ch, const float* v, long long sb, int sv, int sc, int batch, int nver,
                    const int32_t* tri, int ntri, const float* colors, float alpha, int reverse, float* depth_out, int shuffle) {
  std::vector<uint64_t> keys((size_t)batch * h * w, 0);
  for (int b = 0; b < batch; ++b)
    for (int q = 0; q < ntri; ++q) {
      const int i = shuffle ? (int)(((long long)q * 7919 + 13) % ntri) : q;
      TriSetup t;
      const float* vb = v + (size_t)b * sb;
      const int i0 = tri[3 * i], i1 = tri[3 * i + 1], i2 = tri[3 * i + 2];
      t.x0 = vb[(size_t)i0 * sv]; t.y0 = vb[(size_t)i0 * sv + sc]; t.z0 = vb[(size_t)i0 * sv + 2 * sc];
      t.x1 = vb[(size_t)i1 * sv]; t.y1 = vb[(size_t)i1 * sv + sc]; t.z1 = vb[(size_t)i1 * sv + 2 * sc];
      t.x2 = vb[(size_t)i2 * sv]; t.y2 = vb[(size_t)i2 * sv + sc]; t.z2 = vb[(size_t)i2 * sv + 2 * sc];
      if (!tri_setup(t, w, h)) continue;
      for (int y = t.ymin; y <= t.ymax; ++y)
        for (int x = t.xmin; x <= t.xmax; ++x) {
          uint64_t key;
          if (pixel_key(t, (uint32_t)i, x, y, key)) {
            uint64_t& slot = keys[((size_t)b * h + y) * w + x];
            if (key > slot) slot = key;
          }
        }
    }
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      bool drawn = false;
      for (int b = batch - 1; b >= 0; --b) {
        const uint64_t key = keys[((size_t)b * h + y) * w + x];
        if (depth_out) depth_out[((size_t)b * h + y) * w + x] = key ? key_depth(key) : kDepthInit;
        if (!key || drawn) continue;
        drawn = true;
        const int i = (int)key_tri(key);
        const float* vb = v + (size_t)b * sb;
        const int id[3] = {tri[3 * i], tri[3 * i + 1], tri[3 * i + 2]};
        const Bary bw = barycentric((float)x, (float)y, vb[(size_t)id[0] * sv], vb[(size_t)id[0] * sv + sc], vb[(size_t)id[1] * sv],
                                    vb[(size_t)id[1] * sv + sc], vb[(size_t)id[2] * sv], vb[(size_t)id[2] * sv + sc]);
        const float* cb = colors + (size_t)b * nver * ch;
        unsigned char* dst = image + ((size_t)(reverse ? h - 1 - y : y) * w + x) * ch;
        for (int k = 0; k < ch; ++k)
          dst[k] = blend_u8(dst[k], alpha, interp(bw, cb[(size_t)id[0] * ch + k], cb[(size_t)id[1] * ch + k], cb[(size_t)id[2] * ch + k]));
      }
    }
}

// dets (n,5) in visiting order; the bit-matrix + scan formulation of the GPU kernels
int emul_nms(const float* dets, int n, double thresh, int ge, int32_t* keep) {
  const int words = (n + 63) / 64;
  std::vector<uint64_t> mask((size_t)n * words, 0), removed(words, 0);
  const float thr_f = (float)thresh;
  for (int i = 0; i < n; ++i) {
    const float* a = dets + 5 * (size_t)i;
    const float area_a = box_area(a[0], a[1], a[2], a[3]);
    for (int j = i + 1; j < n; ++j) {
      const float* b = dets + 5 * (size_t)j;
      const float ovr = box_overlap(a, area_a, b, box_area(b[0], b[1], b[2], b[3]));
      if (ge ? ((double)ovr >= thresh) : !(ovr <= thr_f)) mask[(size_t)i * words + j / 64] |= 1ull << (j % 64);
    }
  }
  // the scan of nms_scan_kernel: one 64-box block at a time -- resolve the block against its diagonal word, then OR the
  // rows of the survivors into the words to its right
  int cnt = 0;
  for (int blk = 0; blk < words; ++blk) {
    const int base = blk * 64, c = (n - base < 64) ? n - base : 64;
    uint64_t cur = removed[blk], keepbits = 0;
    for (int b = 0; b < c; ++b)
      if (!((cur >> b) & 1ull)) { keepbits |= 1ull << b; cur |= mask[(size_t)(base + b) * words + blk]; }
    for (int b = 0; b < c; ++b)
      if ((keepbits >> b) & 1ull) {
        keep[cnt++] = base + b;
        for (int q = blk + 1; q < words; ++q) removed[q] |= mask[(size_t)(base + b) * words + q];
      }
  }
  return cnt;
}

}  // extern "C"
