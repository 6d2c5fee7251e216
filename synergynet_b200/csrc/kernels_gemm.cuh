// General fp32-accurate GEMM / implicit-GEMM convolution on tensor cores (wgmma) for the layers outside the fused MobileNetV2
// blocks: the PointNet refinement heads MLP_for / MLP_rev (reference backbone_nets/pointnet_backbone.py:31-64,
// 90-106; Conv1d(k=1) + BatchNorm1d + ReLU over B x 68 points) and the ResNet-50 backbone variant
// (backbone_nets/resnet_backbone.py:227-249; 1x1 / 3x3 convolutions + BatchNorm2d + ReLU, NHWC here).
//
//   out[m, n] = act( sum_k A[m, k] * W[n, k] + bias[n] + addend[m / group, n] + residual[m, n] )
//
// Precision: the split-fp16 x3 scheme of kernels_tc.cuh, but with a DYNAMIC power-of-two scale per A row instead of
// the fixed kActScale: the producing layer's epilogue records max|x| of every row (`rowmax`, atomicMax on the fp32
// bit pattern), and the consumer scales row m by 2^e(m) so that its largest element lands in [2^13, 2^14) before
// the hi/lo split -- exact, undone by one multiply in the epilogue, and immune to the |x| < ~937 range limit of
// the fixed scale (ReLU outputs of these layers are unbounded).  The weights are scaled per output channel the same
// way, by 2^f(n) so that the channel's max |w| lands in [2^8, 2^9); the epilogue undoes both with 2^(g(n) - e(m)),
// g = -f.  Every finite row and channel is covered, subnormal ones included: e is in [-114, 162] and g in [-157, 119],
// so rows with e > 126 scale by two exact factors, and a row or channel outside the plain range (|e| > 100, g < -149)
// takes an epilogue that applies the combined exponent in two normal steps (gemm_wide_out).  A non-finite A value is
// the one input the split still clamps when the row maxima are right: it raises the sticky saturation flag (as does a
// value that the scale takes past 2^15, about twice the row maximum the kernel was given or more).
//
// Roles: 8 warps = two warpgroups, one code path.  Every thread is a producer (GEMM row tid % 128 x half tid / 128 of
// a chunk's k groups: gathers the fp32 row -- or, in conv mode, the k x k x C patch of an NHWC pixel -- splits it and
// stores the canonical K-major operand); warpgroup g then issues the wgmma of rows 64g..64g+63 (accumulators in
// registers) and runs their epilogue.  Thread 0 also launches the bulk copy of each pre-packed weight chunk once its
// ring slot is free.  K streams in chunks of 32 through a 4-stage ring (193 KB smem).
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace syn {

constexpr int kGmKC = 32;                                 // K chunk
constexpr int kGmStages = 4;                              // chunk ring: global-load latency of three chunks hidden
constexpr int kGmThreads = 256;                           // thread = (GEMM row, half of the chunk's k groups)
constexpr int kGmMaxNr = 256;
constexpr int kGmStageA = 128 * kGmKC * 2;                // 8 KB: one plane (hi or lo) of the A tile
constexpr int kGmStageB = kGmMaxNr * kGmKC * 2;           // 16 KB
constexpr int kGmStage = 2 * kGmStageA + 2 * kGmStageB;   // 48 KB
constexpr int kGmSmem = kGmStages * kGmStage + 1024;

enum { kActNone = 0, kActRelu6 = 1, kActRelu = 2 };

struct GemmArgs {
  const float* A;            // plain mode: [M][lda]; conv mode: NHWC activations (B, H, W, C)
  const uint8_t* Wimg;       // per n-range, per K chunk: [hi plane nr x kc][lo plane]  (pack_gemm_weights)
  const float* bias;         // [N] (BatchNorm folded), never null
  const int* oexp;           // [N]: g(n), the channel's weight scale is 2^-g(n)  (g in [-157, 119])
  const float* addend;       // nullable: [M / addend_group][N], broadcast over the rows of a group (PointNet conv6)
  const float* residual;     // nullable: [M][N], added before the activation (ResNet shortcut)
  float* out;                // nullable: [M][N]
  const unsigned* rowmax_in; // max|a| per source row as fp32 bits (conv mode: per input pixel)
  unsigned* rowmax_out;      // nullable: atomicMax of |out| per output row
  unsigned* colmax_out;      // nullable: max over the rows of a group per channel (PointNet max-pool; values >= 0)
  int addend_group, colmax_group;
  int M, K, N, Kp, nr, lda, act;
  // conv mode (ksize > 0): implicit GEMM over k = (ky * ksize + kx) * C + c
  int ksize, stride, pad, H, W, C, HO, WO;
  int* err;
  int* sat;                  // sticky saturation flag: a scaled A value reached 2^15 (NaN, +-Inf, ~2x above rowmax)
};

// exponent e such that max * 2^e lies in [2^13, 2^14) for every finite max > 0, subnormal included (e in [-114, 162]);
// max == 0 (all-zero row) or inf / nan -> 0
__device__ __forceinline__ int gemm_row_exp(unsigned maxbits) {
  const int be = (int)((maxbits >> 23) & 0xffu);
  if (be == 255 || maxbits == 0u) return 0;
  if (be == 0) return 13 - (31 - __clz(maxbits) - 149);   // subnormal: floor(log2 max) = (top set bit) - 149
  return 13 - (be - 127);
}
__device__ __forceinline__ float exp2i(int e) { return __uint_as_float((unsigned)(e + 127) << 23); }   // e in [-126, 127]
// 2^e for e in [-149, 127]: subnormal below -126
__device__ __forceinline__ float exp2i_sub(int e) {
  return e >= -126 ? __uint_as_float((unsigned)(e + 127) << 23) : __uint_as_float(1u << (e + 149));
}
__device__ __forceinline__ float4 scale4(float4 v, float s) { return make_float4(v.x * s, v.y * s, v.z * s, v.w * s); }
template <bool B> struct BoolTag { static constexpr bool value = B; };
constexpr int kGmPlainExp = 100;   // rows with |e| <= 100 against channels with g >= -149 take the plain epilogue
// acc * 2^c + bias with one rounding for any c the kernel meets ([-319, 233]): c = c1 + c2 with 2^c2 representable
// (subnormal included) and acc * 2^c1 exact -- c1 = 0 whenever c is in [-149, 127].  Beyond: c1 > 0 only when |result|
// exceeds 2^127 (acc * 2^c1 is exact or overflows to the right infinity); c1 < 0 only when |acc * 2^c| < 2^-114, where
// what acc * 2^c1 rounds away lies below 2^-298 of the result, and below c = -275 both are far under half of 2^-149.
__device__ __forceinline__ float gemm_wide_out(float acc, int c, float bias) {
  const int c2 = max(-149, min(127, c));
  const int c1 = max(-126, min(127, c - c2));
  return fmaf(acc * exp2i(c1), exp2i_sub(c2), bias);
}

__global__ void __launch_bounds__(kGmThreads, 1) tc_gemm_kernel(const GemmArgs p) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[kGmStages], bar_empty[kGmStages];
  __shared__ __align__(16) float s_bias[kGmMaxNr], s_osc[kGmMaxNr];       // epilogue constants of this n-range
  __shared__ int s_oexp[kGmMaxNr];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * 128;
  const int n0 = blockIdx.y * p.nr;
  bool chan_plain = true;                                     // 2^g exact in fp32 for every channel of the n-range
  for (int i = tid; i < p.nr; i += kGmThreads) {              // the packed arrays are padded to nranges * nr entries
    const int g = p.oexp[n0 + i];
    s_bias[i] = p.bias[n0 + i];
    s_oexp[i] = g;
    s_osc[i] = g >= -149 ? exp2i_sub(g) : 0.f;
    chan_plain = chan_plain && g >= -149;
  }
  const int nchunks = (p.Kp + kGmKC - 1) / kGmKC;
  const uint8_t* wimg = p.Wimg + (size_t)blockIdx.y * (size_t)p.nr * p.Kp * 4;

  if (tid == 0) {
    for (int i = 0; i < kGmStages; ++i) {
      mbar_init(smem_u32(&bar_full[i]), kGmThreads + 1);     // producer arrivals + the weight copy's expect_tx arrival
      mbar_init(smem_u32(&bar_empty[i]), kGmThreads);        // every thread, once its warpgroup's MMAs of the slot are done
    }
    fence_mbar_init();
  }
  const bool all_chan_plain = __syncthreads_and(chan_plain) != 0;
  auto stage_a = [&](int s, int plane) { return smem + s * kGmStage + plane * kGmStageA; };
  auto stage_b = [&](int s, int plane) { return smem + s * kGmStage + 2 * kGmStageA + plane * kGmStageB; };

  {
    // ------------------------------ producers + MMA ---------------------------------------------
    const int row = tid & 127, kh = tid >> 7, m = m0 + row;        // kh: which two of the chunk's four 8-element k groups
    const int wg = kh;                                              // warpgroup: MMA rows 64 wg .. 64 wg + 63
    const bool row_ok = m < p.M;
    int b = 0, oy = 0, ox = 0;
    unsigned mx = 0;
    if (p.ksize > 0) {
      if (row_ok) {
        b = m / (p.HO * p.WO);
        const int r = m - b * p.HO * p.WO;
        oy = r / p.WO; ox = r - oy * p.WO;
        for (int ky = 0; ky < p.ksize; ++ky)
          for (int kx = 0; kx < p.ksize; ++kx) {
            const int iy = oy * p.stride - p.pad + ky, ix = ox * p.stride - p.pad + kx;
            if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) mx = max(mx, p.rowmax_in[((size_t)b * p.H + iy) * p.W + ix]);
          }
      }
    } else if (row_ok) {
      mx = p.rowmax_in[m];
    }
    const int e_row = gemm_row_exp(mx);
    const float a_scale = exp2i(min(e_row, 126));
    const float a_scale2 = exp2i(max(e_row - 126, 0));              // max < 2^-113: 2^e = 2^(e - 126) * 2^126
    // max |hi| of the row's scaled values: below 2^15 for every finite value within the row maximum the kernel was
    // given (they scale to at most 2^14); a NaN or an Inf (clamped to 60000) or a value about twice that maximum or
    // more reaches it
    __half2 hmax = __float2half2_rn(0.f);
    const float* arow = p.A + (size_t)m * p.lda;
    const uint32_t lbo_b = (uint32_t)(p.nr >> 3) * 128;
    const uint32_t d_hi = smem_desc_hi(128);
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int c = 0; c < nchunks; ++c) {
      const int s = c % kGmStages, use = c / kGmStages;
      const int k0 = c * kGmKC;
      const int kc = min(kGmKC, p.Kp - k0);
      // gather first (the loads do not depend on the slot), then wait for the slot: the global latency overlaps the wait
      float4 va[2], ve[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int kg = kh * 2 + q, k = k0 + kg * 8;
        const float* src = nullptr;
        if (row_ok && kg * 8 < kc && k < p.K) {
          if (p.ksize > 0) {
            const int tap = k / p.C, cc = k - tap * p.C;
            const int ky = tap / p.ksize, kx = tap - ky * p.ksize;
            const int iy = oy * p.stride - p.pad + ky, ix = ox * p.stride - p.pad + kx;
            if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) src = p.A + (((size_t)b * p.H + iy) * p.W + ix) * p.C + cc;
          } else {
            src = arow + k;
          }
        }
        va[q] = make_float4(0.f, 0.f, 0.f, 0.f); ve[q] = va[q];
        if (src != nullptr) {                                 // K and C are multiples of 8, rows 16-byte aligned
          va[q] = __ldg(reinterpret_cast<const float4*>(src));
          ve[q] = __ldg(reinterpret_cast<const float4*>(src + 4));
        }
      }
      mbar_wait(smem_u32(&bar_empty[s]), (use & 1) ^ 1, p.err);
      if (tid == 0) {                                         // the weight chunk of this slot
        const uint32_t plane_bytes = (uint32_t)p.nr * kc * 2;
        const uint8_t* src = wimg + (size_t)p.nr * k0 * 4;    // chunks of this range are consecutive
        mbar_expect_tx(smem_u32(&bar_full[s]), 2 * plane_bytes);
        bulk_g2s(smem_u32(stage_b(s, 0)), src, plane_bytes, smem_u32(&bar_full[s]));
        bulk_g2s(smem_u32(stage_b(s, 1)), src + plane_bytes, plane_bytes, smem_u32(&bar_full[s]));
      }
      uint8_t* ah = stage_a(s, 0) + (row >> 3) * 128 + (row & 7) * 16;
      uint8_t* al = stage_a(s, 1) + (row >> 3) * 128 + (row & 7) * 16;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int kg = kh * 2 + q;
        if (kg * 8 < kc) {
          va[q] = scale4(va[q], a_scale2); ve[q] = scale4(ve[q], a_scale2);   // exact; 1 unless e > 126
          uint32_t h[4], l[4];
          split2_f16(va[q].x * a_scale, va[q].y * a_scale, h[0], l[0]);
          split2_f16(va[q].z * a_scale, va[q].w * a_scale, h[1], l[1]);
          split2_f16(ve[q].x * a_scale, ve[q].y * a_scale, h[2], l[2]);
          split2_f16(ve[q].z * a_scale, ve[q].w * a_scale, h[3], l[3]);
#pragma unroll
          for (int j = 0; j < 4; ++j) hmax = __hmax2(hmax, __habs2(*reinterpret_cast<const __half2*>(&h[j])));
          *reinterpret_cast<uint4*>(ah + kg * 2048) = make_uint4(h[0], h[1], h[2], h[3]);
          *reinterpret_cast<uint4*>(al + kg * 2048) = make_uint4(l[0], l[1], l[2], l[3]);
        }
      }
      fence_proxy_async_smem();
      mbar_arrive(smem_u32(&bar_full[s]));
      mbar_wait(smem_u32(&bar_full[s]), use & 1, p.err);     // the whole A chunk and the weight chunk landed
      const uint32_t a_lo = smem_desc_lo(smem_u32(stage_a(s, 0)) + wg * 1024, 2048);
      const uint32_t b_lo = smem_desc_lo(smem_u32(stage_b(s, 0)), lbo_b);
      wgmma_fence();
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {                 // hi*hi, hi*lo, lo*hi
        const uint32_t a_off = (pass == 2 ? kGmStageA : 0), b_off = (pass == 1 ? kGmStageB : 0);
        for (int ks = 0; ks < kc / 16; ++ks)
          wgmma_f16_rt(acc, p.nr, desc64(d_hi, a_lo + ((a_off + ks * 4096) >> 4)),
                       desc64(d_hi, b_lo + ((b_off + ks * 2 * lbo_b) >> 4)), (c > 0 || pass > 0 || ks > 0) ? 1u : 0u);
      }
      wgmma_commit();
      // retire the chunk's MMAs before the next chunk's (divergent) gather: no accumulator stays in flight there
      wgmma_wait<0>();
      mbar_arrive(smem_u32(&bar_empty[s]));                  // slot s may be refilled
    }
    if (__hge(__hmax(__low2half(hmax), __high2half(hmax)), __float2half(32768.f))) *p.sat = 1;   // sticky, cleared by syn_poll_saturation
    // ------------------------------ epilogue from the accumulators -------------------------------
    // thread t of the warpgroup holds rows r0 = acc_row(t, 0) and r0 + 8 of its 64, columns 8 j + 2 (t % 4) + {0, 1}
    const int t = tid & 127;
    const int ncols = min(p.nr, p.N - n0);
    const bool pair_vec = (p.N & 1) == 0;                      // rows of out / residual / addend are 8-byte aligned
    int mr[2];
    bool ok[2];
    float inv_a[2], rmax[2] = {0.f, 0.f};   // rmax: |out| of the row over this thread's columns
    int erow[2];
    bool wide[2];                            // the row takes gemm_wide_out
    const float *rrow[2], *arow2[2];
    float* orow[2];
    unsigned* crow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mr[h] = m0 + 64 * wg + acc_row(t, 2 * h);
      ok[h] = mr[h] < p.M;
      orow[h] = p.out ? p.out + (size_t)mr[h] * p.N + n0 : nullptr;
      rrow[h] = p.residual ? p.residual + (size_t)mr[h] * p.N + n0 : nullptr;
      arow2[h] = p.addend ? p.addend + (size_t)(mr[h] / p.addend_group) * p.N + n0 : nullptr;
      crow[h] = p.colmax_out ? p.colmax_out + (size_t)(mr[h] / p.colmax_group) * p.N + n0 : nullptr;
    }
    {
      // a row's dynamic scale was computed by its producer thread, which may sit in the other warpgroup
      __shared__ int s_erow[128];
      if (kh == 0) s_erow[row] = e_row;
      __syncthreads();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        erow[h] = s_erow[64 * wg + acc_row(t, 2 * h)];
        wide[h] = !all_chan_plain || erow[h] > kGmPlainExp || erow[h] < -kGmPlainExp;
        inv_a[h] = exp2i(wide[h] ? 0 : -erow[h]);
      }
    }
    // max-pool over the rows of a group (PointNet): the 16 rows of a warp almost always belong to one group (68 points
    // per face), so the warp reduces over its 8 row lanes first and issues ONE atomic per column instead of 16
    // (the shuffle sits outside the && chain: every lane of the warp must execute it)
    const int cgrp = __shfl_sync(0xffffffffu, p.colmax_out ? mr[0] / p.colmax_group : 0, 0);
    const bool warp_one_group = p.colmax_out != nullptr &&
        __all_sync(0xffffffffu, ok[0] && ok[1] && mr[0] / p.colmax_group == cgrp && mr[1] / p.colmax_group == cgrp);
    // the output loop, twice: as it runs in range, and for a warp holding a row that takes gemm_wide_out
    auto epilogue = [&](auto wide_tag) {
      constexpr bool kWide = decltype(wide_tag)::value;
#pragma unroll
      for (int i = 0; i < 128; i += 4) {
        const int col = acc_col(t, i);
        if (8 * (i >> 2) >= ncols) break;                        // warp-uniform: no column of this 8-column block is valid
        const bool cv = col < ncols;                             // lanes differ: everything below stays convergent
        float2 o[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float v0 = acc[i + 2 * h], v1 = acc[i + 2 * h + 1];
          const bool one = cv && ok[h], two = col + 1 < ncols;
          float x0 = 0.f, x1 = 0.f;
          if (kWide && wide[h]) {
            if (cv) x0 = gemm_wide_out(v0, s_oexp[col] - erow[h], s_bias[col]);
            if (two) x1 = gemm_wide_out(v1, s_oexp[col + 1] - erow[h], s_bias[col + 1]);
          } else {
            if (cv) x0 = fmaf(v0 * inv_a[h], s_osc[col], s_bias[col]);
            if (two) x1 = fmaf(v1 * inv_a[h], s_osc[col + 1], s_bias[col + 1]);
          }
          if (one) {
            if (arow2[h]) { x0 += arow2[h][col]; if (two) x1 += arow2[h][col + 1]; }
            if (rrow[h]) { x0 += rrow[h][col]; if (two) x1 += rrow[h][col + 1]; }
          }
          if (p.act == kActRelu6) { x0 = relu6f(x0); x1 = relu6f(x1); }
          else if (p.act == kActRelu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
          if (!two) x1 = 0.f;
          if (one) {
            rmax[h] = fmaxf(rmax[h], fmaxf(fabsf(x0), two ? fabsf(x1) : 0.f));
            if (orow[h]) {
              if (two && pair_vec) *reinterpret_cast<float2*>(orow[h] + col) = make_float2(x0, x1);
              else { orow[h][col] = x0; if (two) orow[h][col + 1] = x1; }
            }
          }
          o[h] = make_float2(x0, x1);
        }
        if (p.colmax_out != nullptr) {                           // o >= 0 (ReLU): the bit pattern orders like the value
          if (warp_one_group) {
            unsigned b0 = max(__float_as_uint(o[0].x), __float_as_uint(o[1].x));
            unsigned b1 = max(__float_as_uint(o[0].y), __float_as_uint(o[1].y));
#pragma unroll
            for (int sh = 4; sh < 32; sh <<= 1) {               // the 8 row lanes sharing this column pair
              b0 = max(b0, __shfl_xor_sync(0xffffffffu, b0, sh));
              b1 = max(b1, __shfl_xor_sync(0xffffffffu, b1, sh));
            }
            if ((t & 31) < 4 && cv) {
              atomicMax(crow[0] + col, b0);
              if (col + 1 < ncols) atomicMax(crow[0] + col + 1, b1);
            }
          } else {
#pragma unroll
            for (int h = 0; h < 2; ++h)
              if (ok[h] && cv) {
                atomicMax(crow[h] + col, __float_as_uint(o[h].x));
                if (col + 1 < ncols) atomicMax(crow[h] + col + 1, __float_as_uint(o[h].y));
              }
          }
        }
      }
    };
    if (__any_sync(0xffffffffu, wide[0] || wide[1])) {
      epilogue(BoolTag<true>{});
    } else {
      epilogue(BoolTag<false>{});
    }
    if (p.rowmax_out != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {                            // the 4 lanes of a row hold its column pairs
        rmax[h] = fmaxf(rmax[h], __shfl_xor_sync(0xffffffffu, rmax[h], 1));
        rmax[h] = fmaxf(rmax[h], __shfl_xor_sync(0xffffffffu, rmax[h], 2));
        if ((t & 3) == 0 && ok[h]) atomicMax(p.rowmax_out + mr[h], __float_as_uint(rmax[h]));
      }
    }
  }
}

// ---- small CUDA-core helpers of the same layer families ---------------------------------------------------------
// K < 8 first layer (PointNet conv1: 3 -> 64 on the landmark coordinates): out[m, n] = act(sum_k A[m,k] W[k,n] + b[n]).
// A is read through (row stride, element stride) so that the (B,3,68) landmark tensor is consumed in place:
// row m = (b, point) reads x[b, k, point].
__global__ void small_k_layer_kernel(const float* __restrict__ x, const float* __restrict__ Wkn, const float* __restrict__ bias,
                                     float* __restrict__ out, unsigned* __restrict__ rowmax_out, int M, int K, int N, int pts,
                                     int act) {
  const int m = blockIdx.x * blockDim.y + threadIdx.y;
  if (m >= M) return;
  const int b = m / pts, pt = m - b * pts;
  float a[8];
  for (int k = 0; k < K; ++k) a[k] = x[((size_t)b * K + k) * pts + pt];
  float rmax = 0.f;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float o = bias[n];
    for (int k = 0; k < K; ++k) o = fmaf(a[k], Wkn[k * N + n], o);
    if (act == kActRelu) o = fmaxf(o, 0.f);
    out[(size_t)m * N + n] = o;
    rmax = fmaxf(rmax, fabsf(o));
  }
  for (int o = 16; o > 0; o >>= 1) rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
  if (threadIdx.x == 0 && rowmax_out != nullptr) rowmax_out[m] = __float_as_uint(rmax);
}

// rowmax of an arbitrary [M][K] fp32 matrix (inputs that no GEMM epilogue produced)
__global__ void rowmax_kernel(const float* __restrict__ A, unsigned* __restrict__ rowmax, int M, int K, int lda) {
  const int m = blockIdx.x * blockDim.y + threadIdx.y;
  if (m >= M) return;
  float r = 0.f;
  for (int k = threadIdx.x; k < K; k += 32) r = fmaxf(r, fabsf(A[(size_t)m * lda + k]));
  for (int o = 16; o > 0; o >>= 1) r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, o));
  if (threadIdx.x == 0) rowmax[m] = __float_as_uint(r);
}

}  // namespace syn
