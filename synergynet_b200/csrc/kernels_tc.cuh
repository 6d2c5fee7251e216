// Tensor-core (wgmma) kernels of the SYN_ENGINE_TC_BF16X3 engine.
//
// Precision scheme ("split-16x3"): every fp32 operand x is split into hi = fp16(x) and
// lo = fp16(x - hi); a product a*b is evaluated as hi_a*hi_b + hi_a*lo_b + lo_a*hi_b with fp32
// accumulation (the lo*lo term, <= 2^-22 relative, is dropped).  Three f16 MMAs per
// algorithmic MAC keep each product within ~5e-7 of fp32.  A bf16 hi/lo split (8+8 mantissa bits)
// was measured first: 1.7e-4 on the 62 parameters with a calibrated checkpoint -- outside the 1e-4
// parity bar, like single-pass bf16/tf32/fp16 (SURVEY.md fact 6) -- so the split uses fp16
// (11+11 bits) with power-of-two pre-scaling: activations by kActScale, weights per output channel
// (max |w| in [256,512)), both undone exactly by one multiply in the epilogue.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace syn {

// -------------------------------------------------------------------------------------------------
// Pointwise (1x1) convolution on tensor cores:
//   out[M,N] = act(A[M,K] * W^T + bias) (+ residual),   A fp32 NHWC rows, W = [N][K] (K-major).
//
// CTA = 128 rows x one n-range of `nr` (<= 256, multiple of 16) output channels, 8 warps = 2 warpgroups.
//   every thread: producer of GEMM row tid % 128, half tid / 128 of a chunk's k groups
//       global fp32 A chunk -> fp16 hi/lo -> canonical smem tile (SBO = 128 B, LBO = 2 KB);
//       thread 0 also launches the bulk (TMA) copy of the pre-packed weight chunk
//   warpgroup g: wgmma on rows 64g..64g+63 (3 passes x kc/16 K-steps per chunk, accumulators in
//       registers), then the epilogue straight from its accumulators
// K is streamed in chunks of up to 64 through a 2-stage full/empty mbarrier ring; the weight copy of chunk c+1
// is in flight while chunk c is converted and multiplied.
//
// Weight image (built by syn_commit, see pack_tc_pointwise): for n-range j, K-chunk c:
//   [hi plane nr x kc][lo plane nr x kc], each plane canonical with SBO = 128, LBO = nr/8 * 128.
// -------------------------------------------------------------------------------------------------
constexpr int kTcKChunk = 64;
constexpr int kTcThreads = 256;
constexpr int kTcStageA = 128 * kTcKChunk * 2;       // bytes of one A plane (hi or lo)
constexpr int kTcMaxNr = 256;
constexpr int kTcStageB = kTcMaxNr * kTcKChunk * 2;  // bytes of one B plane
constexpr int kTcSmemBytes = 2 * (2 * kTcStageA + 2 * kTcStageB) + 1024;

struct TcPointwiseArgs {
  const float* A;
  const uint8_t* Wimg;     // packed fp16 hi/lo weight image of this layer
  const float* bias;
  const float* oscale;     // per output channel: 1 / (kActScale * weight scale)
  const float* residual;   // nullable
  float* out;
  int M, K, N;             // K, N: true sizes;
  int Kp;                  // K padded to a multiple of 16
  int nr;                  // channels per n-range (multiple of 16, <= 256)
  int relu6;
  int* err;
  int* sat;                // sticky flag: an A value was clamped by the fp16 split (|x| > 937.5, +-Inf or NaN)
};

__global__ void __launch_bounds__(kTcThreads, 1) tc_pointwise_kernel(const TcPointwiseArgs p) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_full[2], bar_empty[2];

  // keep the pointer in the shared address space (no integer round trip): a generic pointer here
  // turns every tile access into LD.E/ST.E instead of LDS/STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;
  const int m0 = blockIdx.x * 128;
  const int n0 = blockIdx.y * p.nr;
  const int nchunks = (p.Kp + kTcKChunk - 1) / kTcKChunk;
  // bytes of the weight image preceding this n-range: every range holds 2 planes of nr x Kp fp16
  const uint8_t* wimg = p.Wimg + (size_t)blockIdx.y * (size_t)p.nr * p.Kp * 4;

  if (tid == 0) {
    mbar_init(smem_u32(&bar_full[0]), kTcThreads + 1);   // producer arrivals + the weight copy's expect_tx arrival
    mbar_init(smem_u32(&bar_full[1]), kTcThreads + 1);
    mbar_init(smem_u32(&bar_empty[0]), kTcThreads);      // every thread, once its warpgroup's MMAs of the slot are done
    mbar_init(smem_u32(&bar_empty[1]), kTcThreads);
    fence_mbar_init();
  }
  __syncthreads();

  auto stage_a = [&](int s, int plane) { return smem + s * (2 * kTcStageA + 2 * kTcStageB) + plane * kTcStageA; };
  auto stage_b = [&](int s, int plane) {
    return smem + s * (2 * kTcStageA + 2 * kTcStageB) + 2 * kTcStageA + plane * kTcStageB;
  };

  const int row = t, kh = wg;                            // producer: GEMM row, which half of the chunk's k groups
  const bool row_ok = (m0 + row) < p.M;
  const float* arow = p.A + (size_t)(m0 + row) * p.K;
  const uint32_t lbo_b = (uint32_t)(p.nr >> 3) * 128;
  const uint32_t d_hi = smem_desc_hi(128);
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  bool out_of_range = false;                             // the split below clamps a value: |x| > 937.5, +-Inf or NaN
  for (int c = 0; c < nchunks; ++c) {
    const int s = c & 1, use = c >> 1;
    const int k0 = c * kTcKChunk;
    const int kc = min(kTcKChunk, p.Kp - k0);
    mbar_wait(smem_u32(&bar_empty[s]), (use & 1) ^ 1, p.err);
    if (tid == 0) {
      const uint32_t plane_bytes = (uint32_t)p.nr * kc * 2;
      const uint8_t* src = wimg + (size_t)p.nr * k0 * 4;     // chunks of this range are consecutive
      mbar_expect_tx(smem_u32(&bar_full[s]), 2 * plane_bytes);
      bulk_g2s(smem_u32(stage_b(s, 0)), src, plane_bytes, smem_u32(&bar_full[s]));
      bulk_g2s(smem_u32(stage_b(s, 1)), src + plane_bytes, plane_bytes, smem_u32(&bar_full[s]));
    }
    uint8_t* ah = stage_a(s, 0) + (row >> 3) * 128 + (row & 7) * 16;
    uint8_t* al = stage_a(s, 1) + (row >> 3) * 128 + (row & 7) * 16;
#pragma unroll 2
    for (int kg = kh; kg < kc / 8; kg += 2) {
      float v[8];
      const int k = k0 + kg * 8;
      if (row_ok && k < p.K) {       // K is a multiple of 8
        const float4 a = *reinterpret_cast<const float4*>(arow + k);
        const float4 b = *reinterpret_cast<const float4*>(arow + k + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) out_of_range |= act_clamped(v[j]);
      uint32_t h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split2_f16(v[2 * j] * kActScale, v[2 * j + 1] * kActScale, h[j], l[j]);
      *reinterpret_cast<uint4*>(ah + kg * 2048) = make_uint4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<uint4*>(al + kg * 2048) = make_uint4(l[0], l[1], l[2], l[3]);
    }
    fence_proxy_async_smem();
    mbar_arrive(smem_u32(&bar_full[s]));
    mbar_wait(smem_u32(&bar_full[s]), use & 1, p.err);     // both halves of the A chunk and the weight chunk landed
    // ---- MMAs of this warpgroup's 64 rows (rows 64 wg.. start 8 core-matrix rows = 1 KB into the A plane)
    const uint32_t a_lo = smem_desc_lo(smem_u32(stage_a(s, 0)) + wg * 1024, 2048);
    const uint32_t b_lo = smem_desc_lo(smem_u32(stage_b(s, 0)), lbo_b);
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {                 // hi*hi, hi*lo, lo*hi
      const uint32_t a_off = (pass == 2 ? kTcStageA : 0), b_off = (pass == 1 ? kTcStageB : 0);
      for (int ks = 0; ks < kc / 16; ++ks)
        wgmma_f16_rt(acc, p.nr, desc64(d_hi, a_lo + ((a_off + ks * 4096) >> 4)),
                     desc64(d_hi, b_lo + ((b_off + ks * 2 * lbo_b) >> 4)), (c > 0 || pass > 0 || ks > 0) ? 1u : 0u);
    }
    wgmma_commit();
    // retire the chunk's MMAs before the next chunk's (divergent) conversion: no accumulator may be in flight there
    wgmma_wait<0>();
    mbar_arrive(smem_u32(&bar_empty[s]));                  // slot s may be refilled
  }
  if (out_of_range) *p.sat = 1;                            // sticky, cleared by syn_poll_saturation
  // ------------------------------ epilogue from the accumulators ------------------------------------
  const int ncols = min(p.nr, p.N - n0);                   // valid channels of this range
#pragma unroll
  for (int i = 0; i < 128; i += 2) {
    const int col = acc_col(t, i);
    const int m = m0 + 64 * wg + acc_row(t, i);
    if (col >= ncols || m >= p.M) continue;                // N is a multiple of 8: pairs never straddle the end
    const float2 b = *reinterpret_cast<const float2*>(p.bias + n0 + col);
    const float2 sc = *reinterpret_cast<const float2*>(p.oscale + n0 + col);
    float2 o = make_float2(fmaf(acc[i], sc.x, b.x), fmaf(acc[i + 1], sc.y, b.y));
    if (p.relu6) { o.x = relu6f(o.x); o.y = relu6f(o.y); }
    if (p.residual) {
      const float2 r = *reinterpret_cast<const float2*>(p.residual + (size_t)m * p.N + n0 + col);
      o.x += r.x; o.y += r.y;
    }
    *reinterpret_cast<float2*>(p.out + (size_t)m * p.N + n0 + col) = o;
  }
}

}  // namespace syn
