// Serial host emulation of the frame-axis render kernels (synergynet_b200/csrc/kernels_render.cuh): the overlay blend
// (add_weighted_u8_kernel), the per-mesh pixel boxes (mesh_box_kernel + mesh_box_scan_kernel) and the depth pass keyed
// inside them (raster_depth_kernel with boxes), from the same render_math.h functions, as loops instead of threads.
// Build: g++ -O2 -ffp-contract=off -shared -fPIC (tests/test_render_frames_emulation.py does it).
#include "../../synergynet_b200/csrc/render_math.h"

using namespace syn::rmath;

namespace {

// load_tri of the kernels: false for a triangle with a vertex index outside [0, nver) or an empty clamped box
bool tri_of(const float* v, long long sb, int sv, int sc, int nver, const int32_t* tri, int b, int i, int w, int h, TriSetup& t) {
  const int id[3] = {tri[3 * i], tri[3 * i + 1], tri[3 * i + 2]};
  for (int k = 0; k < 3; ++k)
    if ((unsigned)id[k] >= (unsigned)nver) return false;
  const float* vb = v + (size_t)b * sb;
  t.x0 = vb[(size_t)id[0] * sv]; t.y0 = vb[(size_t)id[0] * sv + sc]; t.z0 = vb[(size_t)id[0] * sv + 2 * sc];
  t.x1 = vb[(size_t)id[1] * sv]; t.y1 = vb[(size_t)id[1] * sv + sc]; t.z1 = vb[(size_t)id[1] * sv + 2 * sc];
  t.x2 = vb[(size_t)id[2] * sv]; t.y2 = vb[(size_t)id[2] * sv + sc]; t.z2 = vb[(size_t)id[2] * sv + 2 * sc];
  return tri_setup(t, w, h);
}

}  // namespace

extern "C" {

void emul_add_weighted(const unsigned char* a, const unsigned char* b, unsigned char* out, long long n, double alpha) {
  for (long long i = 0; i < n; ++i) out[i] = add_weighted_u8(a[i], b[i], alpha);
}

// boxes (M,4) x0, y0, x1, y1 and key_off (M+1), as syn_render_frames_plan writes them
void emul_frame_plan(const float* v, long long sb, int sv, int sc, int nmesh, int nver, const int32_t* tri, int ntri, int h, int w,
                     int32_t* boxes, long long* key_off) {
  long long off = 0;
  for (int b = 0; b < nmesh; ++b) {
    PixBox box = pix_box_empty();
    for (int i = 0; i < ntri; ++i) {
      TriSetup t;
      if (tri_of(v, sb, sv, sc, nver, tri, b, i, w, h, t)) pix_box_add(box, t);
    }
    boxes[4 * b] = box.x0; boxes[4 * b + 1] = box.y0; boxes[4 * b + 2] = box.x1; boxes[4 * b + 3] = box.y1;
    key_off[b] = off;
    off += pix_box_area(box);
  }
  key_off[nmesh] = off;
}

// The depth pass over every (mesh, triangle, pixel of its box): keys (key_off[M]) receive the key maxima in the box slots,
// full (M,h,w) the same maxima on the whole canvas.  Returns the number of keyed pixels outside their mesh's box (which
// are then not stored in `keys`).
long long emul_frame_keys(const float* v, long long sb, int sv, int sc, int nmesh, int nver, const int32_t* tri, int ntri, int h, int w,
                          const int32_t* boxes, const long long* key_off, uint64_t* keys, uint64_t* full) {
  long long outside = 0;
  for (int b = 0; b < nmesh; ++b) {
    PixBox box;
    box.x0 = boxes[4 * b]; box.y0 = boxes[4 * b + 1]; box.x1 = boxes[4 * b + 2]; box.y1 = boxes[4 * b + 3];
    for (int i = 0; i < ntri; ++i) {
      TriSetup t;
      if (!tri_of(v, sb, sv, sc, nver, tri, b, i, w, h, t)) continue;
      for (int y = t.ymin; y <= t.ymax; ++y)
        for (int x = t.xmin; x <= t.xmax; ++x) {
          uint64_t key;
          if (!pixel_key(t, (uint32_t)i, x, y, key)) continue;
          uint64_t& f = full[((size_t)b * h + y) * w + x];
          if (key > f) f = key;
          if (x < box.x0 || x > box.x1 || y < box.y0 || y > box.y1) { ++outside; continue; }
          uint64_t& s = keys[key_off[b] + pix_box_slot(box, x, y)];
          if (key > s) s = key;
        }
    }
  }
  return outside;
}

}  // extern "C"
