// CUDA-core pieces of the ResNet backbones (reference backbone_nets/resnet_backbone.py:227-249; BASELINE.json configs[4]
// is resnet50): the 7x7/s2 stem convolution (K = 147 is too thin for an MMA tile), the 3x3/s2 max-pool and the global
// average pool.  Every other convolution and the four Linear heads run on tc_gemm_kernel (kernels_gemm.cuh).
// Activations are NHWC fp32; every kernel also records max|x| per pixel row for the next GEMM's dynamic scaling.
#pragma once
#include "common.cuh"

namespace syn {

// conv1 7x7 stride 2 pad 3 (3 -> 64) + folded BN + ReLU: (B,3,120,120) NCHW -> (B,60,60,64) NHWC.
// One CTA per (face, output row): 7 input rows x 3 channels staged with the zero padding, weights [147][64] in smem,
// thread = (output pixel, 16-channel group).  The input is the fp32 crop or, when x_u8 is set, the raw uint8 crop,
// normalised while staging as (v - 127.5) / 128 -- exact in fp32, so both inputs give the same bits.  `border` zeroes the
// uint8 frame like normalize_u8_kernel (syn_set_center_crop).
constexpr int kRsStemThreads = 256;
__global__ void __launch_bounds__(kRsStemThreads) resnet_stem_kernel(const float* __restrict__ x, const uint8_t* __restrict__ x_u8,
                                                                      const float* __restrict__ Wkn, const float* __restrict__ bias,
                                                                      float* __restrict__ y, unsigned* __restrict__ rowmax, int batch,
                                                                      int border) {
  __shared__ float s_in[3][7][kImg + 6];
  __shared__ __align__(16) float s_w[147 * 64];
  __shared__ unsigned s_max[60];
  const int b = blockIdx.x / 60, oy = blockIdx.x % 60, tid = threadIdx.x;
  if (b >= batch) return;
  for (int i = tid; i < 147 * 64; i += kRsStemThreads) s_w[i] = Wkn[i];
  for (int i = tid; i < 3 * 7 * (kImg + 6); i += kRsStemThreads) {
    const int col = i % (kImg + 6), r = (i / (kImg + 6)) % 7, ci = i / (7 * (kImg + 6));
    const int iy = oy * 2 - 3 + r, ix = col - 3;
    float v = 0.f;
    if (iy >= 0 && iy < kImg && ix >= 0 && ix < kImg) {
      const size_t off = ((size_t)(b * 3 + ci) * kImg + iy) * kImg + ix;
      if (x_u8 != nullptr) {
        const bool out = iy < border || iy >= kImg - border || ix < border || ix >= kImg - border;
        v = ((float)(out ? 0 : x_u8[off]) - 127.5f) / 128.0f;
      } else {
        v = x[off];
      }
    }
    s_in[ci][r][col] = v;
  }
  if (tid < 60) s_max[tid] = 0u;
  __syncthreads();
  const int ox = tid >> 2, cg = tid & 3;
  if (ox < 60) {
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = bias[cg * 16 + j];
    for (int ci = 0; ci < 3; ++ci)
      for (int ky = 0; ky < 7; ++ky)
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const float v = s_in[ci][ky][ox * 2 + kx];
          const float4* w4 = reinterpret_cast<const float4*>(s_w + ((ci * 7 + ky) * 7 + kx) * 64 + cg * 16);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 w = w4[q];
            acc[4 * q] = fmaf(v, w.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, w.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(v, w.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, w.w, acc[4 * q + 3]);
          }
        }
    float m = 0.f;
    float* o = y + (((size_t)b * 60 + oy) * 60 + ox) * 64 + cg * 16;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 r = make_float4(fmaxf(acc[4 * q], 0.f), fmaxf(acc[4 * q + 1], 0.f), fmaxf(acc[4 * q + 2], 0.f), fmaxf(acc[4 * q + 3], 0.f));
      m = fmaxf(m, fmaxf(fmaxf(r.x, r.y), fmaxf(r.z, r.w)));
      reinterpret_cast<float4*>(o)[q] = r;
    }
    atomicMax(&s_max[ox], __float_as_uint(m));
  }
  __syncthreads();
  if (tid < 60) rowmax[((size_t)b * 60 + oy) * 60 + tid] = s_max[tid];
}

// MaxPool2d(3, stride 2, padding 1) on NHWC (values >= 0 after ReLU, so the implicit -inf padding never wins):
// one warp per output pixel, lane = channel pair (C = 64).
__global__ void maxpool3x3s2_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned* __restrict__ rowmax, int batch,
                                    int H, int HO, int C) {
  const int pix = blockIdx.x * blockDim.y + threadIdx.y;
  if (pix >= batch * HO * HO) return;
  const int b = pix / (HO * HO), r = pix - b * HO * HO, oy = r / HO, ox = r - oy * HO;
  float m = 0.f;
  for (int c = threadIdx.x; c < C; c += 32) {
    float v = -3.402823466e38f;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const int iy = oy * 2 - 1 + ky, ix = ox * 2 - 1 + kx;
        if (iy >= 0 && iy < H && ix >= 0 && ix < H) v = fmaxf(v, x[(((size_t)b * H + iy) * H + ix) * C + c]);
      }
    y[(size_t)pix * C + c] = v;
    m = fmaxf(m, fabsf(v));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x == 0) rowmax[pix] = __float_as_uint(m);
}

// AdaptiveAvgPool2d((1,1)) + flatten: (B, P pixels, C) -> (B, C); one CTA per face; also the row maximum of the result.
__global__ void __launch_bounds__(256) avgpool_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned* __restrict__ rowmax,
                                                      int P, int C) {
  __shared__ unsigned s_m;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) s_m = 0u;
  __syncthreads();
  float m = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += x[((size_t)b * P + p) * C + c];
    s /= (float)P;
    y[(size_t)b * C + c] = s;
    m = fmaxf(m, fabsf(s));
  }
  atomicMax(&s_m, __float_as_uint(m));
  __syncthreads();
  if (threadIdx.x == 0) rowmax[b] = s_m;
}

}  // namespace syn
