// CUDA-core piece of the GhostNet backbone that no other family has (reference backbone_nets/ghostnet_backbone.py:41-58):
// the squeeze-and-excite gate.  The depthwise convs, the ghost modules' cheap operation and concat run on dw_kernel
// (kernels_mbv1.cuh), the stem on mbv1_stem_kernel, every 1x1 conv, the SE FCs and the heads on tc_gemm_kernel, the
// pools on avgpool_kernel.
#pragma once
#include "common.cuh"

namespace syn {

// hard_sigmoid (:34-38) as the reference computes it in fp32: relu6(z + 3) / 6
__device__ __forceinline__ float hard_sigmoid(float z) { return fminf(fmaxf(z + 3.f, 0.f), 6.f) / 6.f; }

// x * hard_sigmoid(z) on NHWC maps (:57): x (B,P,C), z (B,C) the conv_expand output of the face, y (B,P,C), C a multiple
// of 4.  One warp per pixel, float4 over the channels; rowmax[pixel] = max_c |y| as fp32 bits (the next GEMM's row scale).
constexpr int kSeThreads = 256;
__global__ void __launch_bounds__(kSeThreads) se_apply_kernel(const float* __restrict__ x, const float* __restrict__ z,
                                                              float* __restrict__ y, unsigned* __restrict__ rowmax, int npix,
                                                              int P, int C) {
  const int pix = (int)((blockIdx.x * (size_t)kSeThreads + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (pix >= npix) return;                                     // warp-uniform
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)pix * C);
  const float4* zr = reinterpret_cast<const float4*>(z + (size_t)(pix / P) * C);
  float4* yr = reinterpret_cast<float4*>(y + (size_t)pix * C);
  float m = 0.f;
  for (int q = lane; q < C / 4; q += 32) {
    const float4 v = xr[q], g = zr[q];
    const float4 o = make_float4(v.x * hard_sigmoid(g.x), v.y * hard_sigmoid(g.y), v.z * hard_sigmoid(g.z), v.w * hard_sigmoid(g.w));
    yr[q] = o;
    m = fmaxf(m, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
  }
#pragma unroll
  for (int sh = 16; sh > 0; sh >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, sh));
  if (lane == 0) rowmax[pix] = __float_as_uint(m);
}

}  // namespace syn
