// Stem 3x3/s2 conv (+BN+ReLU6) fused with block 1 (3x3 depthwise + BN + ReLU6 -> 1x1 project + BN),
// mobilenetv2_backbone.py:127 + features[1], as one kernel of its own: the crop (NCHW fp32, or uint8 normalised while
// staging) goes in, the 60x60x16 block-1 output comes out, and neither the stem output nor block 1's hidden tensor
// touches HBM.
//
// The arithmetic is that of the fused MBConv template (kernels_fused.cuh) with the 27-tap im2col of the stem as GEMM1's
// A operand:
//   prep   crop rows (NCHW) -> im2col (K = 27, padded to 32) -> fp16 hi/lo XA                         (CUDA)
//   GEMM1  D1 (64-row slabs x 32 hidden channels) = XA * W1^T                                         (tensor)
//   EPI1   Hs = relu6(s1 * D1 + b1) / 6 (one FFMA.SAT) into an fp32 window with a zero halo           (CUDA)
//   DW     A2 = split(relu6(dw3x3(6 Hs) + bdw))                                                       (CUDA)
//   GEMM2  D2 (64-row slabs x 16) = A2 * W3^T                                                         (tensor)
//   EPI2   y = s3 * D2 + b3                                                                           (CUDA)
// Block 1 has a single 32-channel hidden chunk, so inside one strip every phase waits on the one before it.  What the
// template overlaps across chunks, this kernel overlaps across strips: a CTA runs two independent strip PIPELINES, each
// with its own worker warpgroup(s), buffers and named barrier, and the two take the CTA's strips of the persistent
// tile order alternately.  One pipeline's depthwise pass and output stores then run while the other's im2col and MMAs
// do; no CTA-wide barrier is used after set-up.  A strip is 4 output rows (a 6-row hidden window, 360 GEMM1 rows,
// 240 GEMM2 rows): two pipelines' buffers then fit in shared memory because each pipeline's GEMM2 operand shares bytes
// with its GEMM1 operand and its staged crop rows share bytes with its hidden window (see StemCfg).
//
// Roles: warps 0-3 = pipeline 0, warps 4-7 = pipeline 1 (one warpgroup each), warp 8 = loader (the weight image once;
// for fp32 crops, each pipeline's next crop rows by bulk copy, one bar_in / bar_x pair per pipeline).  Nine warps
// leave 168 registers per thread, which the kernel fits without spills; two warpgroups per pipeline (17 warps, 96
// registers) spill.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"
#include "kernels_fused.cuh"

namespace syn {

struct StemCfg {
  static constexpr int CIN = 27, CIN_P = 32;               // im2col taps k = (ci*3 + ky)*3 + kx
  static constexpr int CHID = 32, NC = 32, NCHUNK = 1;
  static constexpr int COUT = 16, COUT_P = 16;
  static constexpr int W = 60, WO = 60, RO = 4, STRIPS = WO / RO;
  static constexpr int RWIN = RO + 2;                      // hidden window rows incl. the halo
  static constexpr int M1_MAX = RWIN * W, SLABS1 = ceil_div_c(M1_MAX, 64);
  static constexpr int M2 = RO * WO, SLABS2 = ceil_div_c(M2, 64);
  static constexpr int HS_COLS = W + 2, HS_STRIDE = NC + 4, DWS = NC + 4;
  // ---- weight image: the layout of FusedCfg with one chunk (pack_fused writes it) ----------------------
  static constexpr int B3_BYTES = round_up_c(2 * COUT_P * 4, 128);
  static constexpr int W1_PLANE = NC * CIN_P * 2, W3_PLANE = COUT_P * NC * 2;
  static constexpr int DW_ROWS = 12;
  static constexpr int CH_W1 = 0, CH_W3 = 2 * W1_PLANE, CH_DW = CH_W3 + 2 * W3_PLANE;
  static constexpr int CHUNK_BYTES = round_up_c(CH_DW + DW_ROWS * DWS * 4, 128);
  static constexpr int W_BYTES = B3_BYTES + CHUNK_BYTES;
  // ---- one pipeline's buffers ------------------------------------------------------------------------
  // XA: GEMM1's A operand, [hi plane | lo plane] of SLABS1 canonical 64-row slabs (SBO 128 B, LBO 1 KB).  A2, GEMM2's
  // A operand in the same layout, lives in the same bytes: every GEMM1 of the strip is retired before the depthwise
  // pass writes A2, and GEMM2 is retired before the next strip's prep writes XA.
  static constexpr int XA_TILE = 64 * CIN_P * 2, XA_PLANE = SLABS1 * XA_TILE;
  static constexpr int A2_TILE = 64 * NC * 2, A2_PLANE = SLABS2 * A2_TILE;
  static constexpr int IN_ROWS = 2 * RWIN + 1, IN_STRIDE = kImg;   // staged crop rows [3][IN_ROWS][120] fp32
  static constexpr int P_XA = 0;
  // The staged crop rows live in the bytes of the hidden window: a strip's rows are staged after the previous strip's
  // depthwise pass has read the window, and converted before its own EPI1 writes it.
  static constexpr int P_H = P_XA + 2 * XA_PLANE;
  static constexpr int P_IN = P_H;
  static constexpr int H_BYTES = RWIN * HS_COLS * HS_STRIDE * 4;
  static constexpr int PIPE_BYTES = round_up_c(P_H + H_BYTES, 1024);
  static_assert(3 * IN_ROWS * IN_STRIDE * 4 <= H_BYTES, "staged rows alias the hidden window");
  static constexpr int S_PIPE = round_up_c(W_BYTES, 1024);
  static constexpr int SMEM_BYTES = S_PIPE + 2 * PIPE_BYTES + 1024;   // + alignment slack
  static_assert(2 * A2_PLANE <= 2 * XA_PLANE, "A2 aliases XA");
  static_assert(WO % RO == 0, "strips must tile the output");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

struct StemArgs {
  const float* x;        // NCHW (B,3,120,120) fp32 crop, or null
  const uint8_t* x_u8;   // raw uint8 crop, normalised (v-127.5)/128 while staging; null for fp32 crops
  const uint8_t* wimg;   // packed weight image (StemCfg::W_BYTES)
  float* y;              // NHWC (B,60,60,16)
  int ntiles;            // batch * STRIPS
  int* err;              // sticky time-out flag of the bounded mbarrier waits (mapped pinned host memory)
  int* sat;              // sticky "a stem input was clamped to the fp16 range" flag (device memory)
  int border;            // uint8 only: CenterCrop margin, pixels of the frame read as 0 (utils/ddfa.py:162-243); 0 = off
  int npass;             // 3 = split-fp16 x3 (hi*hi + hi*lo + lo*hi); 1 = single fp16 pass
};

// Phase trace (debug builds only, -DSYN_FUSED_TRACE): clock64 stamps of CTA 0's second strip of each pipeline, in the
// block-1 rows of g_fused_trace: role = pipeline, row 63 = the strip, row 62 = the prep of its next strip.
#ifdef SYN_FUSED_TRACE
#define STEM_TRACE(row, ev)                                                                                   \
  do {                                                                                                        \
    if (trace_on) g_fused_trace[((1 * 2 + pl) * 64 + (row)) * 8 + (ev)] = clock64();                         \
  } while (0)
#else
#define STEM_TRACE(row, ev) do { } while (0)
#endif

constexpr int kStemB1Threads = 9 * 32;

__global__ void __launch_bounds__(kStemB1Threads, 1) stem_block1_kernel(const StemArgs p) {
  using C = StemCfg;
  using namespace tc;
  constexpr int PT = 128;                                // threads of a pipeline: one warpgroup
  constexpr int NWW = 8;                                 // worker warps of the CTA
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_w, bar_in[2], bar_x[2];

  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int ntiles = p.ntiles;
  const int step = 2 * (int)gridDim.x;                   // a pipeline's stride through the persistent tile order

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel's prologue may overlap this one's tail
  if (tid == 0) {
    mbar_init(smem_u32(&bar_w), 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(smem_u32(&bar_in[i]), 1);
      mbar_init(smem_u32(&bar_x[i]), PT);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const uint8_t* sW = smem + C::B3_BYTES;                // the one weight chunk
  const float* sB3 = reinterpret_cast<const float*>(smem);

  if (warp < NWW) {
    // =============================== strip pipelines ====================================================
    // pipeline of this warp, broadcast from lane 0 so that ptxas knows it is warp-uniform: the MMAs sit under branches
    // that depend on it
    const int pl = __shfl_sync(0xffffffffu, warp >> 2, 0);
    const int ptid = tid - pl * PT;
    uint8_t* pbase = smem + C::S_PIPE + pl * C::PIPE_BYTES;
    uint8_t* sXA = pbase + C::P_XA;
    uint8_t* sA2 = pbase + C::P_XA;                      // aliases XA (see StemCfg)
    float* sH = reinterpret_cast<float*>(pbase + C::P_H);
    float* sIn = reinterpret_cast<float*>(pbase + C::P_IN);
    const uint32_t bin = smem_u32(&bar_in[pl]), bx = smem_u32(&bar_x[pl]);
    auto pipe_bar = [&]() { group_bar_sync<PT>(pl); };

    mbar_wait_inl(smem_u32(&bar_w), 0, p.err);               // the weight image landed
    uint32_t n_in = 0;                                   // staged-row phases consumed
    const uint32_t d_hi = smem_desc_hi(128);
    constexpr uint32_t LBO_W1 = (C::NC / 8) * 128, LBO_W3 = (C::COUT_P / 8) * 128;
    const float* dwc = reinterpret_cast<const float*>(sW + C::CH_DW);

    // GEMM1 of one 64-row slab as one committed group (an empty group when the slab does not exist, so that every
    // strip commits the same sequence and each wait_group count is a compile-time constant)
    auto issue_g1 = [&](bool on, float* acc, int s1) {
      if (on) {
        const uint32_t a_lo = smem_desc_lo(smem_u32(sXA + s1 * C::XA_TILE), 1024);
        const uint32_t w_lo = smem_desc_lo(smem_u32(sW + C::CH_W1), LBO_W1);
        if (p.npass == 1) fused_mma_group<C::NC, C::CIN_P / 16, 1>(acc, d_hi, a_lo, C::XA_PLANE, 2048, w_lo, C::W1_PLANE, 2 * LBO_W1, false);
        else fused_mma_group<C::NC, C::CIN_P / 16, 3>(acc, d_hi, a_lo, C::XA_PLANE, 2048, w_lo, C::W1_PLANE, 2 * LBO_W1, false);
      } else {
        wgmma_fence();
        wgmma_commit();
      }
    };

#ifdef SYN_FUSED_TRACE
    int k_strip = 0;                                     // strips of this pipeline so far
#endif
    // ---- prep: stage the strip's crop rows and build its im2col operand XA -------------------------------------
    // Runs after GEMM2 of the previous strip is retired (XA and A2 share bytes) and before that strip's EPI2, so the
    // latency of the staging overlaps the output stores.
    auto prep = [&](int tile) {
      const int f0 = tile / C::STRIPS, sp = tile - f0 * C::STRIPS;
      const int iy0 = sp * C::RO - 1;
      const int rf = max(iy0, 0), rl = min(iy0 + C::RWIN - 1, C::W - 1);
      const int M1 = (rl - rf + 1) * C::W;
#ifdef SYN_FUSED_TRACE
      const bool trace_on = blockIdx.x == 0 && k_strip == 1 && ptid == 0;   // prep of the strip after the traced one
#endif
      STEM_TRACE(62, 0);
      // ---- the crop rows this strip needs, zero outside the image --------------------------------------
      const int iy_first = 2 * rf - 1, nin = 2 * (rl - rf + 1) + 1;
      if (p.x_u8 != nullptr) {              // uint8 crops: threads load, normalise and stage
        for (int i = ptid; i < 3 * nin * 30; i += PT) {
          const int c4 = i % 30, r = (i / 30) % nin, ci = i / (30 * nin);
          const int iy = iy_first + r;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (iy >= 0 && iy < kImg) {
            uchar4 u = *reinterpret_cast<const uchar4*>(p.x_u8 + ((size_t)(f0 * 3 + ci) * kImg + iy) * kImg + c4 * 4);
            if (p.border > 0) {                                   // zero frame of the reference loader, before normalisation
              const int col = c4 * 4;
              const bool row_out = iy < p.border || iy >= kImg - p.border;
              if (row_out || col < p.border || col >= kImg - p.border) u.x = 0;
              if (row_out || col + 1 < p.border || col + 1 >= kImg - p.border) u.y = 0;
              if (row_out || col + 2 < p.border || col + 2 >= kImg - p.border) u.z = 0;
              if (row_out || col + 3 < p.border || col + 3 >= kImg - p.border) u.w = 0;
            }
            v = make_float4(((float)u.x - 127.5f) / 128.0f, ((float)u.y - 127.5f) / 128.0f,
                            ((float)u.z - 127.5f) / 128.0f, ((float)u.w - 127.5f) / 128.0f);
          }
          *reinterpret_cast<float4*>(sIn + (ci * C::IN_ROWS + r) * C::IN_STRIDE + c4 * 4) = v;
        }
      } else {                              // fp32 crops: rows were bulk-copied by the loader one strip ahead
        mbar_wait_inl(bin, n_in & 1, p.err);
        ++n_in;
        for (int r = 0; r < nin; ++r) {     // rows outside the image are not copied: zero them (edge strips)
          const int iy = iy_first + r;
          if (iy < 0 || iy >= kImg)
            for (int i = ptid; i < 3 * 30; i += PT)
              *reinterpret_cast<float4*>(sIn + ((i / 30) * C::IN_ROWS + r) * C::IN_STRIDE + (i % 30) * 4) =
                  make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      STEM_TRACE(62, 1);
      pipe_bar();                           // rows staged; every GEMM2 of the previous strip is retired (A2 = XA)
      STEM_TRACE(62, 2);
      // ---- im2col of the 3x3 stride-2 pad-1 stem conv -> fp16 hi/lo XA ------------------------------------
      // A thread converts whole GEMM rows (all 32 K values, k = (ci*3+ky)*3+kx), so that the taps kx = 1, 2 of a
      // (ci, ky) pair -- crop columns 2xx, 2xx+1 -- come in one 8-byte load and kx = 0 (column 2xx-1; -1 is the zero
      // pad) in a 4-byte one: 18 loads per row, and a warp's loads cover 256 contiguous bytes without conflicts.  Rows
      // past M1 up to the slab end are zero.
      {
        const int rows = (M1 + 63) & ~63;
        for (int m = ptid; m < rows; m += PT) {
          float v[C::CIN_P];
#pragma unroll
          for (int k = 0; k < C::CIN_P; ++k) v[k] = 0.f;
          if (m < M1) {
            const int yl = m / C::W, xx = m - yl * C::W;
            const float* base = sIn + (2 * yl) * C::IN_STRIDE + 2 * xx;
#pragma unroll
            for (int q = 0; q < 9; ++q) {                               // q = ci*3 + ky
              const float* r = base + ((q / 3) * C::IN_ROWS + q % 3) * C::IN_STRIDE;
              const float2 t = *reinterpret_cast<const float2*>(r);
              v[3 * q] = xx > 0 ? r[-1] : 0.f;
              v[3 * q + 1] = t.x;
              v[3 * q + 2] = t.y;
            }
          }
          uint8_t* xa = sXA + (m >> 6) * C::XA_TILE + ((m & 63) >> 3) * 128 + (m & 7) * 16;
#pragma unroll
          for (int kg = 0; kg < C::CIN_P / 8; ++kg) {
            const float* w = v + 8 * kg;
            uint32_t h[4], l[4];
            bool out_of_range = false;                                  // |x| > 937.5, +-Inf or NaN
#pragma unroll
            for (int j = 0; j < 8; ++j) out_of_range |= act_clamped(w[j]);
            if (out_of_range) *p.sat = 1;                               // the clamp below changes a value: tell the host (sticky)
#pragma unroll
            for (int j = 0; j < 4; ++j) split2_f16(w[2 * j] * kActScale, w[2 * j + 1] * kActScale, h[j], l[j]);
            *reinterpret_cast<uint4*>(xa + kg * 1024) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4*>(xa + kg * 1024 + C::XA_PLANE) = make_uint4(l[0], l[1], l[2], l[3]);
          }
        }
      }
      STEM_TRACE(62, 3);
      fence_proxy_async_smem();                             // XA is read by wgmma after the next pipeline barrier
      STEM_TRACE(62, 4);
    };

    // Programmatic dependent launch: the set-up above does not depend on the previous kernel; its output (this
    // kernel's input) is first touched below, and this kernel's first global store comes later still.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int first = (int)blockIdx.x + pl * (int)gridDim.x;
    if (first < ntiles) prep(first);

    for (int tile = first; tile < ntiles; tile += step) {
      const int f0 = tile / C::STRIPS, sp = tile - f0 * C::STRIPS;
      const int oy0 = sp * C::RO;
      const int iy0 = oy0 - 1;
      const int rf = max(iy0, 0), rl = min(iy0 + C::RWIN - 1, C::W - 1);
      const int M1 = (rl - rf + 1) * C::W;
      const int slabs1 = (M1 + 63) >> 6;
#ifdef SYN_FUSED_TRACE
      const bool trace_on = blockIdx.x == 0 && k_strip == 1 && ptid == 0;
#endif
      STEM_TRACE(63, 0);
      // the accumulator row offsets of EPI1 / EPI2 are recomputed per strip: hoisted out of the strip loop they would
      // be held in (and spilled from) registers for the whole kernel
      int row = ptid & 127;
      asm volatile("" : "+r"(row));
      float acc1[2][C::NC / 2];                            // D1 double buffer: slab j + 1 is in flight under EPI1 of slab j
      float acc2[C::SLABS2][C::COUT_P / 2];
      pipe_bar();                                          // XA complete; the previous strip's depthwise reads are done
      // the halo columns and the window rows outside the image must read as zero (they may hold staged crop rows or a
      // previous strip)
      for (int i = ptid; i < C::RWIN * 2 * (C::NC / 4); i += PT) {
        const int r = i / (2 * (C::NC / 4)), side = (i / (C::NC / 4)) & 1, c4 = i % (C::NC / 4);
        *reinterpret_cast<float4*>(sH + (size_t)(r * C::HS_COLS + side * (C::HS_COLS - 1)) * C::HS_STRIDE + c4 * 4) =
            make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (iy0 < 0)
        for (int i = ptid; i < C::HS_COLS * (C::NC / 4); i += PT)
          *reinterpret_cast<float4*>(sH + (size_t)(i / (C::NC / 4)) * C::HS_STRIDE + (i % (C::NC / 4)) * 4) =
              make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy0 + C::RWIN - 1 > C::W - 1)
        for (int i = ptid; i < C::HS_COLS * (C::NC / 4); i += PT)
          *reinterpret_cast<float4*>(sH + (size_t)((C::RWIN - 1) * C::HS_COLS + i / (C::NC / 4)) * C::HS_STRIDE +
                                     (i % (C::NC / 4)) * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      STEM_TRACE(63, 1);
      // ---- GEMM1 + EPI1: relu6(s1*D1 + b1) / 6 -> hidden window, one 64-row slab at a time ---------------------
      issue_g1(true, acc1[0], 0);
      {
        // {b1 / 6, b1 / 6, s1, s1} per channel pair, s1 per channel: a thread's columns are the same in every slab and
        // both row halves, so its NC / 8 vectors are loaded once per strip
        const float* bs1 = dwc + 10 * C::DWS;
        float4 bs[C::NC / 8];
#pragma unroll
        for (int q = 0; q < C::NC / 8; ++q) bs[q] = *reinterpret_cast<const float4*>(bs1 + 2 * acc_col(row, 4 * q));
#pragma unroll
        for (int s1 = 0; s1 < C::SLABS1; ++s1) {
          if (s1 + 1 < C::SLABS1) issue_g1(s1 + 1 < slabs1, acc1[(s1 + 1) & 1], s1 + 1);
          if (s1 + 1 < C::SLABS1) wgmma_wait<1>();
          else wgmma_wait<0>();
          if (s1 >= slabs1) continue;
          const float* acc = acc1[s1 & 1];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = 64 * s1 + acc_row(row, 2 * h);
            if (m < M1) {
              const int yl = m / C::W, xx = m - yl * C::W;
              float* hrow = sH + (size_t)((rf - iy0 + yl) * C::HS_COLS + xx + 1) * C::HS_STRIDE;
#pragma unroll
              for (int q = 0; q < C::NC / 8; ++q) {
                const int i = 4 * q + 2 * h, j0 = acc_col(row, i);
                *reinterpret_cast<float2*>(hrow + j0) = make_float2(__saturatef(fmaf(acc[i], bs[q].z, bs[q].x)),
                                                                   __saturatef(fmaf(acc[i + 1], bs[q].w, bs[q].y)));
              }
            }
          }
        }
        wgmma_wait<0>();
      }
      STEM_TRACE(63, 2);
      pipe_bar();                                          // the hidden window is complete; every GEMM1 read of XA is done
      STEM_TRACE(63, 3);
      // ---- DW: 3x3 depthwise on the window -> A2 operand --------------------------------------------------------
      // Item = (8 hidden channels, two vertically adjacent output rows, 8 lanes along x): the two rows' 3x3 windows
      // share 2 of 4 input rows.  A thread keeps one channel octet for all its items, so its nine tap vectors and the
      // bias are loaded once per strip and stay in registers.  Hidden values are stored as relu6(h)/6 in [0,1] and the
      // bias row holds bdw/6, so the activation is a single saturate and the fp16 pre-scale becomes 6 * kActScale.
      // Each output sums from the bias, taps dx-outer, dy-inner, as the template's row-pair item does.
      {
        constexpr int NKG = C::NC / 8;
        constexpr int GX = 8;
        constexpr int XG = (C::WO + GX - 1) / GX;                        // x groups per output row
        constexpr int PER_KG = XG * (C::RO / 2);                         // row-pair items per channel octet
        constexpr int QPK = PT / 8 / NKG;                                // quarter-warps per channel octet
        static_assert(C::RO % 2 == 0 && PER_KG % QPK == 0, "row pairs split evenly over the quarter-warps");
        const int lx = tid & 7, kg = (ptid >> 3) % NKG, q0 = (ptid >> 3) / NKG;
        const float* wbase = dwc + kg * 8;
        float2 w[3][3][4], bias[4];                                      // [dx][dy][channel pair]
        {
          const float4 a = *reinterpret_cast<const float4*>(wbase + 9 * C::DWS);
          const float4 e = *reinterpret_cast<const float4*>(wbase + 9 * C::DWS + 4);
          bias[0] = make_float2(a.x, a.y); bias[1] = make_float2(a.z, a.w); bias[2] = make_float2(e.x, e.y); bias[3] = make_float2(e.z, e.w);
        }
#pragma unroll
        for (int dx = 0; dx < 3; ++dx)
#pragma unroll
          for (int dy = 0; dy < 3; ++dy) {
            const float4 a = *reinterpret_cast<const float4*>(wbase + (dy * 3 + dx) * C::DWS);
            const float4 e = *reinterpret_cast<const float4*>(wbase + (dy * 3 + dx) * C::DWS + 4);
            w[dx][dy][0] = make_float2(a.x, a.y); w[dx][dy][1] = make_float2(a.z, a.w);
            w[dx][dy][2] = make_float2(e.x, e.y); w[dx][dy][3] = make_float2(e.z, e.w);
          }
#pragma unroll 1
        for (int r2 = q0; r2 < PER_KG; r2 += QPK) {
          const int rp = r2 / XG, xg = r2 - rp * XG;
          const int ox = xg * GX + lx, oy = 2 * rp;
          if (ox >= C::WO) continue;
          const float* h0 = sH + (size_t)(oy * C::HS_COLS + ox) * C::HS_STRIDE + kg * 8;
          float2 acc0[4], acc1[4];                                       // channel pairs
#pragma unroll
          for (int j = 0; j < 4; ++j) acc0[j] = acc1[j] = bias[j];
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
#pragma unroll
            for (int wr = 0; wr < 4; ++wr) {
              const float* hp = h0 + (wr * C::HS_COLS + dx) * C::HS_STRIDE;
              const float4 a = *reinterpret_cast<const float4*>(hp);
              const float4 e = *reinterpret_cast<const float4*>(hp + 4);
              const float2 d[4] = {make_float2(a.x, a.y), make_float2(a.z, a.w), make_float2(e.x, e.y), make_float2(e.z, e.w)};
              if (wr < 3) {
#pragma unroll
                for (int j = 0; j < 4; ++j) acc0[j] = ffma2(d[j], w[dx][wr][j], acc0[j]);
              }
              if (wr >= 1) {
#pragma unroll
                for (int j = 0; j < 4; ++j) acc1[j] = ffma2(d[j], w[dx][wr - 1][j], acc1[j]);
              }
            }
          }
          constexpr float kOut = 6.0f * kActScale;                       // relu6(x) * kActScale = sat(x/6) * 384
#pragma unroll
          for (int ro = 0; ro < 2; ++ro) {
            const float2* acc = ro ? acc1 : acc0;
            const int m2 = (oy + ro) * C::WO + ox;
            uint32_t h[4], l[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
              split2_f16<false>(__saturatef(acc[j].x) * kOut, __saturatef(acc[j].y) * kOut, h[j], l[j]);
            uint8_t* dst = sA2 + (m2 >> 6) * C::A2_TILE + ((m2 & 63) >> 3) * 128 + kg * 1024 + (m2 & 7) * 16;
            *reinterpret_cast<uint4*>(dst) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4*>(dst + C::A2_PLANE) = make_uint4(l[0], l[1], l[2], l[3]);
          }
        }
      }
      STEM_TRACE(63, 4);
      fence_proxy_async_smem();
      mbar_arrive(bx);                                     // this thread's window reads are done: the next rows may land
      pipe_bar();                                          // A2 is complete
      {
        // ---- GEMM2: D2 = A2 * W3^T, one group per 64-row slab, retired at once
        const uint32_t w_lo = smem_desc_lo(smem_u32(sW + C::CH_W3), LBO_W3);
#pragma unroll
        for (int s2 = 0; s2 < C::SLABS2; ++s2) {
          const uint32_t a_lo = smem_desc_lo(smem_u32(sA2 + s2 * C::A2_TILE), 1024);
          if (p.npass == 1) fused_mma_group<C::COUT_P, C::NC / 16, 1>(acc2[s2], d_hi, a_lo, C::A2_PLANE, 2048, w_lo, C::W3_PLANE, 2 * LBO_W3, false);
          else fused_mma_group<C::COUT_P, C::NC / 16, 3>(acc2[s2], d_hi, a_lo, C::A2_PLANE, 2048, w_lo, C::W3_PLANE, 2 * LBO_W3, false);
        }
        wgmma_wait<0>();
      }
      STEM_TRACE(63, 5);
      if (tile + step < ntiles) prep(tile + step);
      STEM_TRACE(63, 6);
      // ---- EPI2: s3*D2 + b3 -> global NHWC (the strip's 180 pixels are contiguous) --------------------------------
      float* ybase = p.y + ((size_t)(f0 * C::WO + oy0) * C::WO) * C::COUT;
#pragma unroll
      for (int s2 = 0; s2 < C::SLABS2; ++s2) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int pix = 64 * s2 + acc_row(row, 2 * h);
          if (pix >= C::M2) continue;
          float* orow = ybase + (size_t)pix * C::COUT;
#pragma unroll
          for (int q = 0; q < C::COUT_P / 8; ++q) {
            const int i = 4 * q + 2 * h, j = acc_col(row, i);
            const float2 bb = *reinterpret_cast<const float2*>(sB3 + j);
            const float2 sc = *reinterpret_cast<const float2*>(sB3 + C::COUT_P + j);
            *reinterpret_cast<float2*>(orow + j) = make_float2(fmaf(acc2[s2][i], sc.x, bb.x), fmaf(acc2[s2][i + 1], sc.y, bb.y));
          }
        }
      }
      STEM_TRACE(63, 7);
#ifdef SYN_FUSED_TRACE
      ++k_strip;
#endif
    }
  } else if (warp == NWW) {
    // =============================== loader ==========================================================
    // The whole warp runs this control flow convergently and every batch of bulk copies sits under one elect.sync.
    if (elect_one()) {
      mbar_expect_tx(smem_u32(&bar_w), C::W_BYTES);
      bulk_g2s(smem_u32(smem), p.wimg, C::W_BYTES, smem_u32(&bar_w));
    }
    __syncwarp();
    if (p.x_u8 != nullptr) return;                       // uint8 crops are staged by the workers themselves
    // fp32 crops: bulk-copy (TMA) the crop rows of a pipeline's strip into its sIn, one strip ahead of its workers
    auto stage_rows = [&](int pl, int tile) {
      if (!elect_one()) return;
      const int f0 = tile / C::STRIPS, sp = tile - f0 * C::STRIPS;
      const int iy0 = sp * C::RO - 1;
      const int rf = max(iy0, 0), rl = min(iy0 + C::RWIN - 1, C::W - 1);
      const int iy_first = 2 * rf - 1, nin = 2 * (rl - rf + 1) + 1;
      const int r_lo = (iy_first < 0) ? -iy_first : 0;                     // first / last staged row inside the crop
      const int r_hi = min(nin - 1, kImg - 1 - iy_first);
      const uint32_t bytes = (uint32_t)(r_hi - r_lo + 1) * kImg * 4;          // contiguous in the crop and in sIn
      float* sIn = reinterpret_cast<float*>(smem + C::S_PIPE + pl * C::PIPE_BYTES + C::P_IN);
      mbar_expect_tx(smem_u32(&bar_in[pl]), 3 * bytes);
      for (int ci = 0; ci < 3; ++ci)
        bulk_g2s(smem_u32(sIn + (ci * C::IN_ROWS + r_lo) * C::IN_STRIDE),
                 p.x + ((size_t)(f0 * 3 + ci) * kImg + iy_first + r_lo) * kImg, bytes, smem_u32(&bar_in[pl]));
    };
    asm volatile("griddepcontrol.wait;" ::: "memory");   // the crop rows are the previous kernel's output
    const int first0 = (int)blockIdx.x, first1 = first0 + (int)gridDim.x;
    if (first0 < ntiles) stage_rows(0, first0);
    __syncwarp();
    if (first1 < ntiles) stage_rows(1, first1);
    __syncwarp();
    // strip k + 1 of a pipeline goes into its sIn once the depthwise pass of strip k has read the window (bar_x phase k);
    // pipeline 0 never has fewer strips than pipeline 1
    for (int k = 0; first0 + (k + 1) * step < ntiles; ++k) {
      for (int pl = 0; pl < 2; ++pl) {
        const int next = first0 + pl * (int)gridDim.x + (k + 1) * step;
        if (next >= ntiles) continue;
        mbar_wait_inl(smem_u32(&bar_x[pl]), k & 1, p.err);
        stage_rows(pl, next);
        __syncwarp();
      }
    }
  }
}

}  // namespace syn
