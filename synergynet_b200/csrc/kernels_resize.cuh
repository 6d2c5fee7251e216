// ROI crop + resize of uint8 BGR images on the GPU: crop_img followed by cv2.resize (synergy3DMM.py:186-188,
// model_building.py:285-287, singleImage.py:76-77; the detector's shrink, FaceBoxes/FaceBoxes.py:62-79), bit-exact with
// OpenCV.  The arithmetic and the plan layout are resize_math.h's; this file only maps threads onto output pixels.
//
// One thread per output pixel (all three channels), one grid z-slice per ROI: 8 x 8 source taps for Lanczos4, 2 x 2 for
// linear, read straight from the image (the taps of neighbouring threads overlap, so L1 serves most of them).  The work
// is small (16 Lanczos4 faces at 120 x 120 are ~44 M integer multiply-adds); the tables sit in the plan buffer the host
// built, so the device computes no transcendental function.
#pragma once
#include "common.cuh"
#include "resize_math.h"

namespace syn {

constexpr int kResizeBX = 32, kResizeBY = 8;

// out[b*sb + oy*sy + ox*sx + c*sc] (element strides): planar (B,3,h,w) crops or an interleaved (h,w,3) image.
// frames > 0 (syn_crop_resize_batch): img is a stack of `frames` images and ROI b reads the one its plan header names.
template <int K>
__global__ void __launch_bounds__(kResizeBX * kResizeBY) crop_resize_kernel(const uint8_t* __restrict__ img, int height, int width,
                                                                            const void* __restrict__ plan, int batch, int out_h,
                                                                            int out_w, uint8_t* __restrict__ out, long long sb,
                                                                            long long sy, long long sx, long long sc, int frames) {
  const int ox = blockIdx.x * kResizeBX + threadIdx.x, oy = blockIdx.y * kResizeBY + threadIdx.y, b = blockIdx.z;
  if (ox >= out_w || oy >= out_h) return;
  const rsz::PlanView v = rsz::plan_view(plan, batch, out_h, out_w, K);
  uint8_t px[3];
  if (frames > 0) img += (size_t)rsz::clampi(v.hdr[b].frame, 0, frames - 1) * height * width * 3;
  rsz::resize_pixel<K>(img, height, width, v, b, out_h, out_w, oy, ox, px);
  uint8_t* o = out + b * sb + oy * sy + ox * sx;
  o[0] = px[0];
  o[sc] = px[1];
  o[2 * sc] = px[2];
}

// The crops of a list of images of any sizes (syn_crop_resize_images): every ROI has its own source image and its own output
// size.  The plan is CropImagesRoi[B] followed by one one-ROI plan per ROI (resize_math.h's layout and tables, the bytes
// syn_crop_resize_plan_host makes for that ROI alone).
struct CropImagesRoi {
  long long src;           // byte offset of the ROI's image in the packed images (image i at sum_{j<i} 3 h_j w_j)
  int h, w;                // that image's size
  int out_h, out_w;        // this ROI's output size
  long long out;           // byte offset of its output: outputs packed back to back, 3 out_h out_w bytes each
  long long plan;          // byte offset of its one-ROI plan in the plan buffer
};

// grid.z = ROI, grid.x / .y cover the largest output; planar: (3,h,w) outputs (the backbone's crops), else (h,w,3) images
template <int K>
__global__ void __launch_bounds__(kResizeBX * kResizeBY) crop_resize_images_kernel(const uint8_t* __restrict__ images,
                                                                                   const void* __restrict__ plan,
                                                                                   uint8_t* __restrict__ out, int planar) {
  const CropImagesRoi r = static_cast<const CropImagesRoi*>(plan)[blockIdx.z];
  const int ox = blockIdx.x * kResizeBX + threadIdx.x, oy = blockIdx.y * kResizeBY + threadIdx.y;
  if (ox >= r.out_w || oy >= r.out_h) return;
  const rsz::PlanView v = rsz::plan_view(static_cast<const char*>(plan) + r.plan, 1, r.out_h, r.out_w, K);
  uint8_t px[3];
  rsz::resize_pixel<K>(images + r.src, r.h, r.w, v, 0, r.out_h, r.out_w, oy, ox, px);
  const long long plane = (long long)r.out_h * r.out_w, at = (long long)oy * r.out_w + ox;
  uint8_t* o = out + r.out + (planar ? at : 3 * at);
  const long long sc = planar ? plane : 1;
  o[0] = px[0];
  o[sc] = px[1];
  o[2 * sc] = px[2];
}

}  // namespace syn
