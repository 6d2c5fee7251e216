// Small CUDA-core kernels around the PointNet refinement heads and the training-forward losses
// (reference model_building.py:141-157, loss_definition.py:8-42, backbone_nets/pointnet_backbone.py:31-64).
#pragma once
#include "common.cuh"

namespace syn {

// conv6 input of MLP_for that is constant over the 68 points of a face (pointnet_backbone.py:42-58):
// [global max-pool features (1024) | avgpool (1280) | shape code (40) | expression code (10)], padded to `ld` floats.
// `gmax` holds the max-pooled conv5 outputs as fp32 bit patterns (atomicMax accumulators, values >= 0).
__global__ void pointnet_face_vector_kernel(const unsigned* __restrict__ gmax, const float* __restrict__ pool,
                                            const float* __restrict__ params, float* __restrict__ out, int batch, int ld) {
  const int b = blockIdx.x;
  if (b >= batch) return;
  float* o = out + (size_t)b * ld;
  for (int i = threadIdx.x; i < ld; i += blockDim.x) {
    float v = 0.f;
    if (i < 1024) v = __uint_as_float(gmax[(size_t)b * 1024 + i]);
    else if (i < 1024 + kLastCh) v = pool[(size_t)b * kLastCh + (i - 1024)];
    else if (i < 1024 + kLastCh + kNumAlpha) v = params[(size_t)b * kNumParams + 12 + (i - 1024 - kLastCh)];
    o[i] = v;
  }
}

// point_residual (B*68, 3) point-major -> (B,3,68) like the reference's Conv1d output, and the refined landmarks
// vertex_lmk + 0.05 * point_residual (model_building.py:150)
__global__ void pointnet_residual_kernel(const float* __restrict__ res_pm, int ld, const float* __restrict__ lmk,
                                         float* __restrict__ residual, float* __restrict__ refined, int batch, int pts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * 3 * pts) return;
  const int b = i / (3 * pts), r = i - b * 3 * pts, c = r / pts, pt = r - c * pts;
  const float v = res_pm[((size_t)b * pts + pt) * ld + c];
  if (residual != nullptr) residual[i] = v;
  if (refined != nullptr) refined[i] = lmk[i] + 0.05f * v;
}

__global__ void bits_to_float_kernel(const unsigned* __restrict__ src, float* __restrict__ dst, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __uint_as_float(src[i]);
}

// WingLoss (loss_definition.py:8-27): mean over the B*3*N coordinates whose d = |target - pred| passes `d < omega` or
// `d >= omega` (a NaN delta passes neither and is left out of the sums and the count, as the reference's masks do) of
//   omega * log(1 + d / eps)  if d < omega   else   d - C,   C = omega - omega * log(1 + omega / eps)
// with C evaluated in double and rounded to fp32 where it meets the fp32 delta, like the reference's Python float.
// One CTA; partial sums in double, fixed reduction order (deterministic).
__global__ void __launch_bounds__(1024) wing_loss_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                         size_t n, float omega, float epsilon, float* __restrict__ out) {
  __shared__ double part[1024];
  __shared__ unsigned long long cnt[1024];
  const double om = omega;
  const float C = (float)__dsub_rn(om, __dmul_rn(om, log(1.0 + om / (double)epsilon)));
  double s = 0.0;
  unsigned long long c = 0;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float d = fabsf(target[i] - pred[i]);
    if (d < omega) { s += (double)(omega * logf(1.0f + d / epsilon)); ++c; }
    else if (d >= omega) { s += (double)(d - C); ++c; }
  }
  part[threadIdx.x] = s;
  cnt[threadIdx.x] = c;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) { part[threadIdx.x] += part[threadIdx.x + o]; cnt[threadIdx.x] += cnt[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)(part[0] / (double)cnt[0]);
}

// ParamLoss (loss_definition.py:29-42), one value per sample:
//   mode 0 'normal':    sqrt( mean((in[:12]-tg[:12])^2) + mean((in[12:62]-tg[12:62])^2) )
//   mode 1 'only_3dmm': sqrt( mean((in[:50]-tg[12:62])^2) )
__global__ void param_loss_kernel(const float* __restrict__ in, const float* __restrict__ tg, int batch, int mode,
                                  float* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const float* x = in + (size_t)b * kNumParams;
  const float* t = tg + (size_t)b * kNumParams;
  if (mode == 0) {
    float s0 = 0.f, s1 = 0.f;
    for (int j = 0; j < 12; ++j) { const float d = x[j] - t[j]; s0 += d * d; }
    for (int j = 12; j < kNumParams; ++j) { const float d = x[j] - t[j]; s1 += d * d; }
    out[b] = sqrtf(s0 / 12.0f + s1 / 50.0f);
  } else {
    float s = 0.f;
    for (int j = 0; j < 50; ++j) { const float d = x[j] - t[12 + j]; s += d * d; }
    out[b] = sqrtf(s / 50.0f);
  }
}

}  // namespace syn
