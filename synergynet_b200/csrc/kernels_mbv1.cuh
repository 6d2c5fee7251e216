// CUDA-core pieces of the MobileNetV1 backbones (reference backbone_nets/mobilenetv1_backbone.py:21-140, prelu=False):
// the 3x3/s2 stem convolution (K = 27 is too thin for an MMA tile) and the depthwise 3x3 convolutions of the 13
// DepthWiseBlocks.  GhostNet (ghost_host.inl) reuses the stem and runs its depthwise convs on the same kernel.  Every 1x1 convolution and the four Linear heads run on tc_gemm_kernel (kernels_gemm.cuh) in plain
// mode, the pool on avgpool_kernel (kernels_resnet.cuh).  Activations are NHWC fp32; both kernels here also record
// max|y| of every output pixel (fp32 bits), which is the row scale the next GEMM needs before its hi/lo split.
#pragma once
#include "common.cuh"

namespace syn {

// conv1 3x3 stride 2 pad 1 (3 -> C0, C0 a multiple of 8 up to 64) + folded BN + ReLU: (B,3,120,120) NCHW -> (B,60,60,C0).
// One CTA per (face, output row): 3 input rows x 3 channels staged with the zero padding, weights [27][C0] (k = (ci*3 +
// ky)*3 + kx, the OIHW order) in smem; thread = (output pixel, 8-channel group).  The input is the fp32 crop or the raw
// uint8 crop, normalised here as (v - 127.5) / 128 -- exact in fp32, so both inputs give the same bits.  `border` zeroes
// the uint8 frame like normalize_u8_kernel (syn_set_center_crop).
constexpr int kMbStemThreads = 256;
constexpr int kMbStemMaxC = 64;
__global__ void __launch_bounds__(kMbStemThreads) mbv1_stem_kernel(const float* __restrict__ x, const uint8_t* __restrict__ x_u8,
                                                                    const float* __restrict__ Wkn, const float* __restrict__ bias,
                                                                    float* __restrict__ y, unsigned* __restrict__ rowmax, int C0,
                                                                    int border) {
  __shared__ float s_in[3][3][kImg + 2];
  __shared__ __align__(16) float s_w[27 * kMbStemMaxC];
  __shared__ __align__(16) float s_b[kMbStemMaxC];
  __shared__ unsigned s_max[60];
  const int b = blockIdx.x / 60, oy = blockIdx.x % 60, tid = threadIdx.x;
  for (int i = tid; i < 27 * C0; i += kMbStemThreads) s_w[i] = Wkn[i];
  for (int i = tid; i < C0; i += kMbStemThreads) s_b[i] = bias[i];
  for (int i = tid; i < 3 * 3 * (kImg + 2); i += kMbStemThreads) {
    const int col = i % (kImg + 2), r = (i / (kImg + 2)) % 3, ci = i / (3 * (kImg + 2));
    const int iy = oy * 2 - 1 + r, ix = col - 1;
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
  const int groups = C0 >> 3;
  for (int it = tid; it < 60 * groups; it += kMbStemThreads) {
    const int ox = it / groups, cg = it - ox * groups;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float v = s_in[ci][ky][ox * 2 + kx];
          const float4* w4 = reinterpret_cast<const float4*>(s_w + ((ci * 3 + ky) * 3 + kx) * C0 + cg * 8);
          const float4 w0 = w4[0], w1 = w4[1];
          acc[0] = fmaf(v, w0.x, acc[0]); acc[1] = fmaf(v, w0.y, acc[1]); acc[2] = fmaf(v, w0.z, acc[2]); acc[3] = fmaf(v, w0.w, acc[3]);
          acc[4] = fmaf(v, w1.x, acc[4]); acc[5] = fmaf(v, w1.y, acc[5]); acc[6] = fmaf(v, w1.z, acc[6]); acc[7] = fmaf(v, w1.w, acc[7]);
        }
    float r[8], m = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      r[j] = fmaxf(acc[j] + s_b[cg * 8 + j], 0.f);
      m = fmaxf(m, r[j]);
    }
    float4* o = reinterpret_cast<float4*>(y + (((size_t)b * 60 + oy) * 60 + ox) * C0 + cg * 8);
    o[0] = make_float4(r[0], r[1], r[2], r[3]);
    o[1] = make_float4(r[4], r[5], r[6], r[7]);
    atomicMax(&s_max[ox], __float_as_uint(m));                 // values >= 0: the bit pattern orders like the value
  }
  __syncthreads();
  if (tid < 60) rowmax[((size_t)b * 60 + oy) * 60 + tid] = s_max[tid];
}

// Depthwise k x k (k = 3 or 5), pad k/2, stride 1 or 2 + folded BN on NHWC fp32 maps: (B,H,H,C) -> (B,HO,HO,C), C a
// multiple of 4.  CTA = (band of `rows` output rows, face).  The channels are walked in chunks of `cc` (a multiple of 4):
// the band's input rows plus the k/2-pixel halo, the chunk's k*k weight rows ([k*k][C], tap-major) and its bias are
// staged in smem with 16-byte cp.async copies (the zero padding comes from the zero-fill form of the copy), then thread
// = (output pixel, 4 channels) sums the taps in the fixed order ky, kx with fmaf, adds the bias and, when kRelu, applies
// the ReLU.  Each pixel's max over all chunks is collected in smem and written once as fp32 bits.
//   * MobileNetV1 (k = 3, kRelu, !kGhost): rowmax = max_c y, the ReLU output being >= 0.
//   * linear (!kRelu): the GhostNet conv_dw and shortcut depthwise convs; rowmax = max_c |y|.
//   * ghost (kGhost, k = 3, stride 1): GhostModule's cheap operation, its concat and the bottleneck's shortcut add in one
//     pass.  y is (B,H,H,2C) = [x + res_lo | dw(x) + b + res_hi] (res (B,H,H,2C) nullable; the host never passes it
//     with kRelu), rowmax = max |y| over both halves.
// smem: s_in [rin][W + k - 1][cc] | s_w [k*k][cc] | s_b [cc] | s_max [rows * HO], rin = (rows - 1) * stride + k.
constexpr int kDwThreads = 256;

__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

__host__ __device__ constexpr int dw_in_rows(int rows, int stride, int ks = 3) { return (rows - 1) * stride + ks; }
__host__ __device__ constexpr size_t dw_smem_bytes(int rows, int stride, int H, int HO, int cc, int ks = 3) {
  return ((size_t)dw_in_rows(rows, stride, ks) * (H + ks - 1) * cc + (size_t)(ks * ks + 1) * cc) * sizeof(float) +
         (size_t)rows * HO * sizeof(unsigned);
}
__device__ __forceinline__ float max_abs4(float4 v) { return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

template <int KS, bool kRelu, bool kGhost>
__global__ void __launch_bounds__(kDwThreads) dw_kernel(const float* __restrict__ x, const float* __restrict__ wkc,
                                                        const float* __restrict__ bias, const float* __restrict__ res,
                                                        float* __restrict__ y, unsigned* __restrict__ rowmax, int H, int HO,
                                                        int C, int stride, int rows, int cc) {
  static_assert(!kGhost || KS == 3, "the ghost module's cheap operation is a 3x3");
  constexpr int PAD = KS / 2;
  extern __shared__ __align__(16) float dw_smem[];
  const int W = H, WO = HO, Wp = W + 2 * PAD;
  const int rin = dw_in_rows(rows, stride, KS);
  float* s_in = dw_smem;
  float* s_w = s_in + (size_t)rin * Wp * cc;
  float* s_b = s_w + KS * KS * cc;
  unsigned* s_max = reinterpret_cast<unsigned*>(s_b + cc);
  const int b = blockIdx.y, oy0 = blockIdx.x * rows, tid = threadIdx.x;
  const int nrows = min(rows, HO - oy0), npix = nrows * WO;
  const int iy0 = oy0 * stride - PAD;
  for (int i = tid; i < npix; i += kDwThreads) s_max[i] = 0u;
  const float* xb = x + (size_t)b * H * W * C;
  for (int c0 = 0; c0 < C; c0 += cc) {
    const int cn = min(cc, C - c0), q4 = cn >> 2;
    const int nin = dw_in_rows(nrows, stride, KS);
    for (int i = tid; i < nin * Wp * q4; i += kDwThreads) {
      const int q = i % q4, pc = i / q4, col = pc % Wp, r = pc / Wp;
      const int iy = iy0 + r, ix = col - PAD;
      const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
      cp_async16(s_in + ((size_t)r * Wp + col) * cc + 4 * q, ok ? xb + ((size_t)iy * W + ix) * C + c0 + 4 * q : xb, ok);
    }
    for (int i = tid; i < (KS * KS + 1) * q4; i += kDwThreads) {   // the k*k weight rows, then the bias
      const int q = i % q4, t = i / q4;
      cp_async16((t < KS * KS ? s_w + t * cc : s_b) + 4 * q, (t < KS * KS ? wkc + (size_t)t * C : bias) + c0 + 4 * q, true);
    }
    cp_async_wait_all();
    __syncthreads();
    for (int i = tid; i < npix * q4; i += kDwThreads) {
      const int q = i % q4, p = i / q4, oyl = p / WO, ox = p - oyl * WO;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int ky = 0; ky < KS; ++ky)
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const float4 v = *reinterpret_cast<const float4*>(s_in + ((size_t)(oyl * stride + ky) * Wp + ox * stride + kx) * cc + 4 * q);
          const float4 w = *reinterpret_cast<const float4*>(s_w + (ky * KS + kx) * cc + 4 * q);
          acc.x = fmaf(v.x, w.x, acc.x); acc.y = fmaf(v.y, w.y, acc.y);
          acc.z = fmaf(v.z, w.z, acc.z); acc.w = fmaf(v.w, w.w, acc.w);
        }
      const float4 bb = *reinterpret_cast<const float4*>(s_b + 4 * q);
      float4 r;
      if constexpr (kRelu)
        r = make_float4(fmaxf(acc.x + bb.x, 0.f), fmaxf(acc.y + bb.y, 0.f), fmaxf(acc.z + bb.z, 0.f), fmaxf(acc.w + bb.w, 0.f));
      else
        r = add4(acc, bb);
      const size_t pix = ((size_t)b * HO + oy0 + oyl) * WO + ox;
      float m;
      if constexpr (kGhost) {                                  // stride 1: the centre tap is the input pixel itself
        float4 v = *reinterpret_cast<const float4*>(s_in + ((size_t)(oyl + PAD) * Wp + ox + PAD) * cc + 4 * q);
        if (res != nullptr) {
          v = add4(v, *reinterpret_cast<const float4*>(res + pix * 2 * C + c0 + 4 * q));
          r = add4(r, *reinterpret_cast<const float4*>(res + pix * 2 * C + C + c0 + 4 * q));
        }
        *reinterpret_cast<float4*>(y + pix * 2 * C + c0 + 4 * q) = v;
        *reinterpret_cast<float4*>(y + pix * 2 * C + C + c0 + 4 * q) = r;
        m = fmaxf(max_abs4(v), max_abs4(r));
      } else {
        *reinterpret_cast<float4*>(y + pix * C + c0 + 4 * q) = r;
        m = kRelu ? fmaxf(fmaxf(r.x, r.y), fmaxf(r.z, r.w)) : max_abs4(r);
      }
      atomicMax(&s_max[p], __float_as_uint(m));
    }
    __syncthreads();                                          // the next chunk overwrites the staged rows
  }
  for (int i = tid; i < npix; i += kDwThreads) rowmax[((size_t)b * HO + oy0) * WO + i] = s_max[i];
}

}  // namespace syn
