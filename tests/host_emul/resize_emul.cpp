// Serial host emulation of the crop + resize kernel (synergynet_b200/csrc/kernels_resize.cuh): the same resize_math.h
// per-pixel function over a plan the library's host planner built, executed by loops instead of threads.  Lets the CPU
// test-suite hold the arithmetic to live cv2.resize byte for byte; the -m gpu tests then only have to show that the CUDA
// launch code is wired the same way.
// Build: g++ -O2 -shared -fPIC (tests/test_resize_emulation.py does it).
#include "../../synergynet_b200/csrc/resize_math.h"

using namespace syn::rsz;

extern "C" {

// img (height,width,3) uint8; out[b*sb + oy*sy + ox*sx + c*sc]
void emul_crop_resize(const uint8_t* img, int height, int width, const void* plan, int batch, int out_h, int out_w, int mode,
                      uint8_t* out, long long sb, long long sy, long long sx, long long sc) {
  const int k = taps_of(mode);
  const PlanView v = plan_view(plan, batch, out_h, out_w, k);
  for (int b = 0; b < batch; ++b)
    for (int oy = 0; oy < out_h; ++oy)
      for (int ox = 0; ox < out_w; ++ox) {
        uint8_t px[3];
        if (k == 8) resize_pixel<8>(img, height, width, v, b, out_h, out_w, oy, ox, px);
        else resize_pixel<2>(img, height, width, v, b, out_h, out_w, oy, ox, px);
        for (int c = 0; c < 3; ++c) out[b * sb + oy * sy + ox * sx + c * sc] = px[c];
      }
}

// Sums of the positive and of the negative fixed-point Lanczos4 taps at fractional position f (the int32 range check).
void emul_lanczos4_tap_sums(float f, int* pos, int* neg) {
  float c[8];
  lanczos4_coeffs(f, c);
  *pos = *neg = 0;
  for (int i = 0; i < 8; ++i) {
    const int q = fix11(c[i]);
    if (q > 0) *pos += q;
    else *neg -= q;
  }
}

}  // extern "C"
