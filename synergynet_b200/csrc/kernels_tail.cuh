// Tail of the backbone on tensor cores (wgmma): features[18] (1x1 conv 320 -> 1280 + BN + ReLU6) fused with the
// global average pool (reference backbone_nets/mobilenetv2_backbone.py:136,179-180), then the three
// Linear heads (:147-158,184-188).  The 1280-channel map (82 KB/face) is never written to HBM.
//
// tail_conv_pool_kernel: transposed GEMM  D[ch, px] = W[ch, :] . X[px, :]  so that accumulator rows are
// output channels and the 16 pixels of a face are 16 adjacent accumulator columns: pooling is a sum over
// four values per thread and two shuffles.  Weight-stationary: a CTA owns one 128-channel slice (its fp16 hi/lo
// weights, 160 KB, stay in smem) and walks over pixel tiles of 8 faces (128 px):
//   warps 0-7   producers: fp32 NHWC rows -> fp16 hi/lo canonical B tiles, 2-stage ring (K chunks of 64)
//   warps 8-15  two MMA warpgroups, 64 channels each (split-16x3: 3 passes x 4 K-steps per chunk, accumulators
//               in registers), then relu6(s*v + b) -> mean over 16 px -> pooled (B,1280)
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace syn {

constexpr int kTailK = 320, kTailN = 1280, kTailKC = 64, kTailChunks = kTailK / kTailKC;  // 5
constexpr int kTailFaces = 8, kTailPx = 16;
constexpr int kTailPlane = 128 * kTailKC * 2;                     // 16 KB: one plane of one K chunk
constexpr int kTailWBytes = kTailChunks * 2 * kTailPlane;         // 160 KB per 128-channel slice
constexpr int kTailXStage = 2 * kTailPlane;                       // 32 KB
constexpr int kTailSmem = kTailWBytes + 2 * kTailXStage + 1024;
constexpr int kTailThreads = 16 * 32;

struct TailArgs {
  const float* x;        // (B,4,4,320) NHWC
  const uint8_t* wimg;   // [10 slices][5 chunks][hi|lo][128 x 64] canonical (SBO 128, LBO 2048)
  const float* bias;     // 1280
  const float* oscale;   // 1280: 1 / (kActScale * weight scale)
  float* pooled;         // (B,1280)
  int batch;
  int ctas_per_slice;
  int* err;
  int* sat;              // sticky flag: an input value was clamped by the fp16 split (|x| > 937.5, +-Inf or NaN)
  int npass;             // 3 = split-fp16 x3, 1 = single fp16 pass
};

__global__ void __launch_bounds__(kTailThreads, 1) tail_conv_pool_kernel(const TailArgs p) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_w, bar_xfull[2], bar_xempty[2];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sW = smem;
  uint8_t* sX = smem + kTailWBytes;

  const int tid = threadIdx.x, warp = tid >> 5;
  const int slice = blockIdx.x / p.ctas_per_slice, pi = blockIdx.x % p.ctas_per_slice;
  const int ntiles = (p.batch + kTailFaces - 1) / kTailFaces;
  const int my_tiles = (ntiles > pi) ? (ntiles - 1 - pi) / p.ctas_per_slice + 1 : 0;

  if (tid == 0) {
    mbar_init(smem_u32(&bar_w), 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(smem_u32(&bar_xfull[i]), 256);
      mbar_init(smem_u32(&bar_xempty[i]), 256);          // every MMA thread, once its warpgroup's MMAs of the stage are done
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ------------------------------ producers -----------------------------------------------------
    const int row = tid & 127, half = tid >> 7;            // pixel row of the tile, which 4 of the 8 k-groups
    uint32_t g = 0;
    bool out_of_range = false;                             // the split below clamps a value: |x| > 937.5, +-Inf or NaN
    for (int i = 0; i < my_tiles; ++i) {
      const int tile = pi + i * p.ctas_per_slice;
      const int f0 = tile * kTailFaces;
      const int npx = min(kTailFaces, p.batch - f0) * kTailPx;
      const float* xrow = p.x + ((size_t)f0 * kTailPx + row) * kTailK;
      for (int kc = 0; kc < kTailChunks; ++kc, ++g) {
        const int s = g & 1;
        mbar_wait(smem_u32(&bar_xempty[s]), ((g >> 1) & 1) ^ 1, p.err);
        uint8_t* xh = sX + s * kTailXStage + (row >> 3) * 128 + (row & 7) * 16;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int kg = half * 4 + q;
          float4 a = make_float4(0.f, 0.f, 0.f, 0.f), e = a;
          if (row < npx) {
            a = *reinterpret_cast<const float4*>(xrow + kc * kTailKC + kg * 8);
            e = *reinterpret_cast<const float4*>(xrow + kc * kTailKC + kg * 8 + 4);
          }
          const float v[8] = {a.x, a.y, a.z, a.w, e.x, e.y, e.z, e.w};
#pragma unroll
          for (int j = 0; j < 8; ++j) out_of_range |= act_clamped(v[j]);
          uint32_t h[4], l[4];
          split2_f16(a.x * kActScale, a.y * kActScale, h[0], l[0]);
          split2_f16(a.z * kActScale, a.w * kActScale, h[1], l[1]);
          split2_f16(e.x * kActScale, e.y * kActScale, h[2], l[2]);
          split2_f16(e.z * kActScale, e.w * kActScale, h[3], l[3]);
          *reinterpret_cast<uint4*>(xh + kg * 2048) = make_uint4(h[0], h[1], h[2], h[3]);
          *reinterpret_cast<uint4*>(xh + kTailPlane + kg * 2048) = make_uint4(l[0], l[1], l[2], l[3]);
        }
        fence_proxy_async_smem();
        mbar_arrive(smem_u32(&bar_xfull[s]));
      }
    }
    if (out_of_range) *p.sat = 1;                           // sticky, cleared by syn_poll_saturation
  } else {
    // ------------------------------ MMA + pooling: warpgroup wg owns channels 64 wg .. 64 wg + 63 of the slice ----
    const int t = tid & 127, wg = (tid >> 7) - 2;
    if (warp == 8) {
      if (elect_one()) {
        mbar_expect_tx(smem_u32(&bar_w), kTailWBytes);
        bulk_g2s(smem_u32(sW), p.wimg + (size_t)slice * kTailWBytes, kTailWBytes, smem_u32(&bar_w));
      }
      __syncwarp();
    }
    mbar_wait(smem_u32(&bar_w), 0, p.err);
    float b[2], sc[2];
    int ch[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      ch[h] = slice * 128 + 64 * wg + acc_row(t, 2 * h);
      b[h] = p.bias[ch[h]];
      sc[h] = p.oscale[ch[h]];
    }
    const uint32_t d_hi = smem_desc_hi(128);
    const uint32_t w_lo = smem_desc_lo(smem_u32(sW) + wg * 1024, 2048), x_lo = smem_desc_lo(smem_u32(sX), 2048);
    float acc[64];
    uint32_t g = 0;
    for (int i = 0; i < my_tiles; ++i) {
      const int tile = pi + i * p.ctas_per_slice;
      const int f0 = tile * kTailFaces;
      const int nf = min(kTailFaces, p.batch - f0);
      for (int kc = 0; kc < kTailChunks; ++kc, ++g) {
        const int s = g & 1;
        mbar_wait(smem_u32(&bar_xfull[s]), (g >> 1) & 1, p.err);
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
          if (pass >= p.npass) break;
          const uint32_t a_off = kc * 2 * kTailPlane + (pass == 2 ? kTailPlane : 0);   // W: hi,hi,lo
          const uint32_t b_off = s * kTailXStage + (pass == 1 ? kTailPlane : 0);       // X: hi,lo,hi
#pragma unroll
          for (int ks = 0; ks < kTailKC / 16; ++ks)
            wgmma_f16<128>(acc, desc64(d_hi, w_lo + ((a_off + ks * 4096) >> 4)),
                           desc64(d_hi, x_lo + ((b_off + ks * 4096) >> 4)), (kc > 0 || pass > 0 || ks > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        mbar_arrive(smem_u32(&bar_xempty[s]));
      }
      // face f = accumulator columns 16f..16f+15 = values 8f..8f+7 of this thread (4 per row) and of the 3 other lanes
      // of its quad
#pragma unroll
      for (int f = 0; f < kTailFaces; ++f) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float s = 0.f;
#pragma unroll
          for (int jj = 0; jj < 2; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) s += relu6f(fmaf(acc[(2 * f + jj) * 4 + 2 * h + e], sc[h], b[h]));
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          if ((t & 3) == 0 && f < nf) p.pooled[(size_t)(f0 + f) * kTailN + ch[h]] = s * (1.0f / 16.0f);
        }
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------
// Heads: params[b, :62] = pooled[b, :1280] . Wh^T + bh   (classifier_ori | shape | exp concatenated).
// One CTA per 8 faces x half of the 62 outputs (grid.y = 2): each weight row is read once per 8 faces.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) heads_kernel(const float* __restrict__ pooled, const float* __restrict__ Wh,
                                                    const float* __restrict__ bh, float* __restrict__ params,
                                                    int batch) {
  constexpr int F = 8;
  __shared__ __align__(16) float s_pool[F][kLastCh];
  const int b0 = blockIdx.x * F, tid = threadIdx.x;
  const int nf = min(F, batch - b0);
  for (int i = tid; i < F * kLastCh / 4; i += 256) {
    const int f = i / (kLastCh / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (f < nf) v = reinterpret_cast<const float4*>(pooled + (size_t)b0 * kLastCh)[i];
    reinterpret_cast<float4*>(&s_pool[0][0])[i] = v;
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  const int j_lo = blockIdx.y * (kNumParams / 2), j_hi = j_lo + kNumParams / 2;
  for (int j = j_lo + warp; j < j_hi; j += 8) {
    const float* wr = Wh + (size_t)j * kLastCh;
    float acc[F];
#pragma unroll
    for (int f = 0; f < F; ++f) acc[f] = 0.f;
    for (int c = lane * 4; c < kLastCh; c += 128) {
      const float4 wv = *reinterpret_cast<const float4*>(wr + c);
#pragma unroll
      for (int f = 0; f < F; ++f) {
        const float4 pv = *reinterpret_cast<const float4*>(&s_pool[f][c]);
        acc[f] = fmaf(wv.x, pv.x, acc[f]); acc[f] = fmaf(wv.y, pv.y, acc[f]);
        acc[f] = fmaf(wv.z, pv.z, acc[f]); acc[f] = fmaf(wv.w, pv.w, acc[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < F; ++f) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[f] += __shfl_xor_sync(0xffffffffu, acc[f], o);
    }
    if (lane == 0) {
      const float bj = bh[j];
      for (int f = 0; f < nf; ++f) params[(size_t)(b0 + f) * kNumParams + j] = acc[f] + bj;
    }
  }
}

}  // namespace syn
