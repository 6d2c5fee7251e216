// Fused inverted-residual block on tensor cores (wgmma):  1x1 expand (+BN+ReLU6) -> 3x3 depthwise (+BN+ReLU6)
// -> 1x1 project (+BN)(+skip), reference backbone_nets/mobilenetv2_backbone.py:45-74, in ONE
// kernel, so the 6x-expanded hidden tensor (up to 1.38 MB per face) never touches HBM.  Blocks 2-17; the stem and
// block 1 run in a kernel of their own (kernels_stem.cuh).
//
// Work item (tile) = RO output rows of one face (large maps) or FACES whole faces (8x8 / 4x4 maps).
// Per tile the block input is converted once to fp16 hi/lo and stored in shared memory (XA); then, for
// each chunk of NC hidden channels:
//   GEMM1  D1 (64-row slabs x NC, registers) = XA * W1c^T (smem x smem)                        (tensor)
//   EPI1   Hs[pixel][NC] (fp32, smem, zero halo) = relu6(s1 * D1 + b1) / 6  (one FFMA.SAT)   (CUDA)
//   DW     A2[out pixel][NC] (fp16 hi/lo, smem)  = split(relu6(dw3x3(6 Hs) + bdw))          (CUDA)
//   GEMM2  D2 (64-row slabs x column pieces, registers) += A2 * W3c^T                       (tensor)
// and finally EPI2: out = s3 * D2 + b3 (+ x).  The worker warpgroups issue the MMAs themselves: a warpgroup
// owns a fixed set of (64-row slab, column piece) items of D2 for the whole tile, so the D2 accumulator stays
// in its registers across the chunks (a 128 x 320 fp32 accumulator would not: blocks 15 / 17 use 4-face tiles).
// CTAs are persistent (grid = #SMs).  Weights (fp16 hi/lo, split-16x3 scheme of kernels_tc.cuh) are either
// resident in shared memory for the whole kernel (early blocks) or streamed chunk by chunk through a 2-3-slot
// bulk-copy (TMA) ring (late blocks).
//
// Roles: warps 0..kFusedWorkerWarps-1 = workers (thread = GEMM row / pixel in the conversion, channel octets in EPI1 /
// DW, MMA operand slabs per warpgroup), warp kFusedWorkerWarps = weight loader (converged warp, bulk copies under
// elect.sync).  smem operand tiles use the canonical K-major no-swizzle layout of tc_common.cuh (SBO 128 B,
// LBO = rows/8 * 128 B).
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace syn {

// Worker warps of a fused CTA (whole warpgroups).  8 rather than 16: on an H100 a 1024-face step measured 5.13 ms
// against 5.76 ms with 16, whose 17-warp CTAs leave 96 registers per thread and spill.
constexpr int kFusedWorkerWarps = 8;
static_assert(kFusedWorkerWarps % 4 == 0, "worker warps form whole warpgroups");

__host__ __device__ constexpr int ceil_div_c(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ constexpr int round_up_c(int a, int b) { return ceil_div_c(a, b) * b; }

template <int CIN_, int CHID_, int NC_, int COUT_, int W_, int STRIDE_, int RO_, int FACES_, bool RES_, int WSTREAM_>
struct FusedCfg {
  static constexpr bool RES = RES_;
  static constexpr bool WSTREAM = WSTREAM_ > 0;  // weights streamed per chunk (ring of WSTREAM_ slots) instead of resident
  static constexpr int CIN = CIN_;               // channels of the NHWC input
  static constexpr int CIN_P = round_up_c(CIN_, 16);
  static constexpr int CHID = CHID_, NC = NC_, NCHUNK = CHID_ / NC_;
  static constexpr int COUT = COUT_, COUT_P = round_up_c(COUT_, 16);
  static constexpr int W = W_, STRIDE = STRIDE_, WO = (W_ - 1) / STRIDE_ + 1;
  static constexpr int RO = RO_, STRIPS = WO / RO_, FACES = FACES_;
  static constexpr int RWIN = (RO_ - 1) * STRIDE_ + 3;                   // window rows incl. halo
  static constexpr int ROWS_MAX = (RWIN < W_ ? RWIN : W_);               // valid input rows per face
  static constexpr int M1_MAX = FACES_ * ROWS_MAX * W_;
  static constexpr int MT1 = ceil_div_c(M1_MAX, 128);
  static constexpr int M2F = RO_ * WO;                                   // GEMM2 rows per face
  static constexpr int M2_MAX = FACES_ * M2F;
  static constexpr int MT2 = ceil_div_c(M2_MAX, 128);
  static constexpr int HS_COLS = W_ + 2;                                 // hidden window row incl. the halo columns
  static constexpr int HS_FACE = RWIN * HS_COLS, HS_PIX = FACES_ * HS_FACE, HS_STRIDE = NC_ + 4;
  static constexpr int DWS = NC_ + 4;     // floats between the tap rows of a chunk: mirrored lanes of the 2x2 depthwise read
                                          // taps kx and 2-kx, which must not lie a multiple of 128 bytes apart
  static constexpr int SLABS1 = ceil_div_c(M1_MAX, 64), SLABS2 = ceil_div_c(M2_MAX, 64);   // 64-row MMA slabs
  // ---- weight image: [b3 | s3] then NCHUNK x { W1c hi, W1c lo, W3c hi, W3c lo, DW rows } -----------
  static constexpr int B3_BYTES = round_up_c(2 * COUT_P * 4, 128);       // [2][COUT_P] fp32: b3, s3
  static constexpr int W1_PLANE = NC_ * CIN_P * 2;                       // bytes, one plane of one chunk
  static constexpr int W3_PLANE = COUT_P * NC_ * 2;
  static constexpr int DW_ROWS = 12;   // 9 taps, depthwise bias, expand bias b1 and output scale s1 (per channel,
                                       // rows 10-11 interleaved as {b1, b1, s1, s1} per channel pair)
  static constexpr int CH_W1 = 0, CH_W3 = 2 * W1_PLANE, CH_DW = CH_W3 + 2 * W3_PLANE;
  static constexpr int CHUNK_BYTES = round_up_c(CH_DW + DW_ROWS * DWS * 4, 128);
  static constexpr int W_BYTES = B3_BYTES + NCHUNK * CHUNK_BYTES;
  static constexpr int WSTAGES = WSTREAM_ > 0 ? WSTREAM_ : NCHUNK;       // chunk slots held in smem
  // ---- shared memory carve-up --------------------------------------------------------------------
  static constexpr int A2_PLANE = MT2 * 128 * NC_ * 2;
  // GEMM1's A operand: the block input as fp16 hi/lo, [hi plane | lo plane], each SLABS1 slabs of 64 rows x CIN_P
  // (canonical, SBO = 128, LBO = 1 KB)
  static constexpr int XA_TILE = 64 * CIN_P * 2, XA_PLANE = SLABS1 * XA_TILE;
  static constexpr int S_B3 = 0;
  static constexpr int S_WCH = S_B3 + B3_BYTES;
  static constexpr int S_XA = S_WCH + WSTAGES * CHUNK_BYTES;
  static constexpr int S_A2 = S_XA + 2 * XA_PLANE;
  static constexpr int S_H = S_A2 + 2 * A2_PLANE;
  static constexpr int S_TOTAL = S_H + HS_PIX * HS_STRIDE * 4;
  static constexpr int SMEM_BYTES = S_TOTAL + 1024;                      // + alignment slack
  static_assert(CHID_ % NC_ == 0 && NC_ % 16 == 0, "hidden chunking");
  static_assert(WO % RO_ == 0, "strips must tile the output");
  static_assert(FACES_ == 1 || RO_ == WO, "multi-face tiles hold whole faces");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
  static_assert(NC_ <= 256, "MMA N");
  static_assert(WSTREAM_ == 0 || (WSTREAM_ >= 2 && WSTREAM_ <= 4 && NCHUNK >= WSTREAM_), "weight ring");
};

struct FusedArgs {
  const float* x;        // NHWC (B,W,W,CIN)
  const uint8_t* wimg;   // packed weight image (FusedCfg::W_BYTES)
  float* y;              // NHWC (B,WO,WO,COUT)
  int batch;
  int split;             // two-face configs: face groups >= split hold ONE face (tail wave, see fused_tile_plan)
  int face_groups;       // number of face groups (tiles = face_groups * STRIPS)
  int* err;              // sticky time-out flag of the bounded mbarrier waits (mapped pinned host memory)
  int* sat;              // sticky "a block input was clamped to the fp16 range" flag (device memory)
  int npass;             // 3 = split-fp16 x3 (hi*hi + hi*lo + lo*hi); 1 = single fp16 pass (SYN_ENGINE_TC_FUSED_1PASS)
#ifdef SYN_FUSED_TRACE
  int trace_id;          // backbone block of this launch (1..17)
#endif
};

// Phase trace (debug builds only, -DSYN_FUSED_TRACE): clock64 stamps of CTA 0's second tile, one row of 8
// events per (block, role, chunk); read back with syn_debug_read_trace.  role 0 = worker thread 0 (role 1 is unused).
#ifdef SYN_FUSED_TRACE
__device__ long long g_fused_trace[18 * 2 * 64 * 8];
#define SYN_TRACE(role, chunk, ev)                                                                        \
  do {                                                                                                    \
    if (trace_on) g_fused_trace[((p.trace_id * 2 + (role)) * 64 + (chunk)) * 8 + (ev)] = clock64();      \
  } while (0)
#else
#define SYN_TRACE(role, chunk, ev) do { } while (0)
#endif

// Named barrier of a worker group with an IMMEDIATE id (a register id makes ptxas reserve all 16 hardware barriers).
template <int THREADS>
__device__ __forceinline__ void group_bar_sync(int grp) {
  switch (grp) {
    case 0: asm volatile("bar.sync 1, %0;" ::"n"(THREADS) : "memory"); break;
    case 1: asm volatile("bar.sync 2, %0;" ::"n"(THREADS) : "memory"); break;
    case 2: asm volatile("bar.sync 3, %0;" ::"n"(THREADS) : "memory"); break;
    default: asm volatile("bar.sync 4, %0;" ::"n"(THREADS) : "memory"); break;
  }
}

// D2 column pieces: the fewest (halving the width) that give every worker warpgroup at least one (slab, piece) item
__host__ __device__ constexpr int fused_d2_pieces(int cout_p, int slabs, int nwg) {
  int s = 1;
  while (slabs * s < nwg && (cout_p / (2 * s)) % 8 == 0) s *= 2;
  return s;
}

// The MMAs of one accumulator for one chunk as one committed group, in straight-line code: pass 0 = hi*hi, 1 = hi*lo
// (B's lo plane), 2 = lo*hi (A's lo plane); KSTEPS steps of K = 16 each.  The pass count is a template parameter and
// fence, MMAs and commit share one basic block: a branch or a join inside the group makes ptxas insert a
// warpgroup.arrive there and serialise every wgmma.mma_async of the kernel.
template <int N, int KSTEPS, int NPASS>
__device__ __forceinline__ void fused_mma_group(float* acc, uint32_t d_hi, uint32_t a_lo, uint32_t a_plane, uint32_t a_kstep,
                                                uint32_t b_lo, uint32_t b_plane, uint32_t b_kstep, bool acc_in) {
  tc::wgmma_fence();
#pragma unroll
  for (int pass = 0; pass < NPASS; ++pass)
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks)
      tc::wgmma_f16<N>(acc, tc::desc64(d_hi, a_lo + (((pass == 2 ? a_plane : 0) + ks * a_kstep) >> 4)),
                       tc::desc64(d_hi, b_lo + (((pass == 1 ? b_plane : 0) + ks * b_kstep) >> 4)),
                       (acc_in || pass > 0 || ks > 0) ? 1u : 0u);
  tc::wgmma_commit();
}

template <class C>
__global__ void __launch_bounds__((kFusedWorkerWarps + 1) * 32, 1) fused_mbconv_kernel(const FusedArgs p) {
  constexpr int NWW = kFusedWorkerWarps;
  constexpr int NWT = NWW * 32;          // worker threads
  constexpr int NWG = NWW / 4;           // worker warpgroups
  // EPI1 and the depthwise conv are separated by a barrier of all workers (every warpgroup's GEMM1 slabs hold all
  // NC channels of their rows), so the depthwise items are spread over all workers as one channel group
  constexpr int NKG_ = C::NC / 8;
  constexpr int NG = 1;
  constexpr int WPG = NWW / NG, TPG = WPG * 32;
  constexpr int KPG = NKG_ / NG;
  // GEMM2 / EPI2 items: (64-row slab, column piece of N2 channels); item i belongs to warpgroup i % NWG
  constexpr int NSPL = fused_d2_pieces(C::COUT_P, C::SLABS2, NWG);
  constexpr int N2 = C::COUT_P / NSPL;
  constexpr int IPW = ceil_div_c(C::SLABS2 * NSPL, NWG);               // items per warpgroup (at most)
  static_assert(N2 % 8 == 0 && N2 <= 256, "MMA N");
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_w, bar_wfull[4], bar_wempty[4];

  // keep the pointer in the shared address space (no integer round trip): a generic pointer here
  // turns every tile access into LD.E/ST.E instead of LDS/STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, warp = tid >> 5;
  // GEMM row of this worker in the conversion, and its warpgroup.  The warpgroup index is broadcast from lane 0 so that
  // ptxas knows it is warp-uniform: the MMAs sit under branches on it, and in a path ptxas must treat as divergent it
  // serialises every wgmma.mma_async.
  const int row = tid & 127, wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const int grp = warp / WPG;                  // channel group (workers only)
  const int gtid = tid - grp * TPG;
  const int ntiles = p.face_groups * C::STRIPS;
  // faces of a face group.  Two-face tiles (8x8 maps): 512 groups over 132 SMs would leave the last wave
  // 88 % full, so the host turns the groups of that wave into single-face groups (twice as many CTAs busy,
  // each done sooner); small batches become single-face groups altogether.
  auto group_faces = [&](int fg, int& f0, int& nfaces) {
    if constexpr (C::FACES == 2) {
      if (fg < p.split) { f0 = 2 * fg; nfaces = 2; }
      else { f0 = 2 * p.split + (fg - p.split); nfaces = 1; }
    } else {
      f0 = fg * C::FACES;
      nfaces = min(C::FACES, p.batch - f0);
    }
  };

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel's prologue may overlap this one's tail
  if (tid == 0) {
    mbar_init(smem_u32(&bar_w), 1);
    for (int i = 0; i < 4; ++i) {
      mbar_init(smem_u32(&bar_wfull[i]), 1);
      mbar_init(smem_u32(&bar_wempty[i]), NWT);
    }
    fence_mbar_init();
  }
  __syncthreads();

  uint8_t* sWch = smem + C::S_WCH;
  uint8_t* sXA = smem + C::S_XA;
  uint8_t* sA2 = smem + C::S_A2;
  float* sH = reinterpret_cast<float*>(smem + C::S_H);
  const float* sB3 = reinterpret_cast<const float*>(smem + C::S_B3);

  if (warp < NWW) {
    // =============================== workers ====================================================
    // zero the whole hidden window once: halo columns are never written afterwards
    for (int i = tid; i < C::HS_PIX * C::HS_STRIDE / 4; i += NWT)
      reinterpret_cast<float4*>(sH)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    mbar_wait(smem_u32(&bar_w), 0, p.err);                // b3/s3 (and, if resident, all chunks) landed
    uint32_t g = 0;                                       // chunk counter
    asm volatile("bar.sync 5, %0;" ::"n"(NWT) : "memory");
    const uint32_t d_hi = smem_desc_hi(128);
    constexpr uint32_t LBO_W1 = (C::NC / 8) * 128, LBO_W3 = (C::COUT_P / 8) * 128;

    // ---- MMA schedule.  A warpgroup keeps its tensor-core work in flight under its CUDA-core phases, and
    // wgmma.wait_group retires groups in issue order, so the issue order is the schedule:
    //   GEMM1 slab j of a chunk -> D1 buffer j & 1, issued before EPI1 of slab j - 1 (the next slab is always in
    //   flight during an epilogue); the first slab of chunk c + 1 -> buffer 0, issued before the depthwise pass of
    //   chunk c (after it when the weights stream through two slots: chunk c + 1 lands in the slot that GEMM2(c - 1)
    //   releases only at the end of chunk c - 1).  Every accumulator receives the same MMAs in the same order as
    //   a synchronous schedule.
    // Every warpgroup commits the same sequence of groups on every path -- a slab or D2 item it does not have is an
    // empty group -- so each wait_group count is a compile-time constant.  ptxas proves from these counts that no
    // register of a pending MMA is read; with a run-time count it cannot, and serialises every MMA.
    constexpr int SPW = ceil_div_c(C::SLABS1, NWG);       // GEMM1 slabs per warpgroup and chunk (at most)
    constexpr bool LATE_G1 = C::WSTREAM && C::WSTAGES == 2;
    auto issue_g1 = [&](bool on, float* acc, int s1, const uint8_t* wch) {
      if (on) {
        const uint32_t a_lo = smem_desc_lo(smem_u32(sXA + s1 * C::XA_TILE), 1024);
        const uint32_t w_lo = smem_desc_lo(smem_u32(wch + C::CH_W1), LBO_W1);
        if (p.npass == 1) fused_mma_group<C::NC, C::CIN_P / 16, 1>(acc, d_hi, a_lo, C::XA_PLANE, 2048, w_lo, C::W1_PLANE, 2 * LBO_W1, false);
        else fused_mma_group<C::NC, C::CIN_P / 16, 3>(acc, d_hi, a_lo, C::XA_PLANE, 2048, w_lo, C::W1_PLANE, 2 * LBO_W1, false);
      } else {
        wgmma_fence();
        wgmma_commit();
      }
    };

    // Geometry of a tile + "prep": convert its input into the GEMM1 A operand.  prep(next tile) runs
    // BEFORE the current tile's EPI2 (XA is free once the last GEMM1 of the tile is done), so the global-load
    // latency of the conversion overlaps the output stores.
    auto prep = [&](int tile) {
      const int fg = tile / C::STRIPS, sp = tile - fg * C::STRIPS;
      int f0, nfaces;
      group_faces(fg, f0, nfaces);
      const int iy0 = sp * C::RO * C::STRIDE - 1;
      const int rf = max(iy0, 0), rl = min(iy0 + C::RWIN - 1, C::W - 1);
      const int ppf = (rl - rf + 1) * C::W;
      const int M1 = nfaces * ppf;
      const int mt1 = (M1 + 127) >> 7;
#ifdef SYN_FUSED_TRACE
      const bool trace_on = blockIdx.x == 0 && tile == 2 * (int)gridDim.x && tid == 0;   // prep of the tile after the traced one
#endif
      SYN_TRACE(0, 62, 0);
      // ---- X tile -> fp16 hi/lo operand in smem ---------------------------------------------------
      // The conversion sits between the last depthwise and EPI2 of the current tile, so its global-load
      // latency is exposed once per batch of loads: all loads of a batch are issued unconditionally (from a
      // clamped, always valid address) before the first use, and masked afterwards -- a predicated load per
      // item would put a branch between the loads and serialise one DRAM latency per item.
      {
        constexpr int KG = C::CIN_P / 8;
        constexpr int NXG = NWT / 64;                                    // thread groups of 64 = one slab's rows
        constexpr int ITERS = (C::SLABS1 * KG + NXG - 1) / NXG;          // items per thread
        constexpr int PB = ITERS < 4 ? ITERS : 4;                        // items per batch of loads
        const int r64 = tid & 63, xg = tid >> 6;
        const int n_items = ((M1 + 63) >> 6) * KG;
        for (int e0 = xg; e0 < n_items; e0 += PB * NXG) {
          float v[PB][8];
          float4 qa[PB], qb[PB];
          bool ok[PB];
#pragma unroll
          for (int u = 0; u < PB; ++u) {
            const int e = min(e0 + u * NXG, n_items - 1);
            const int t = e / KG, kg = e - t * KG;
            const int m = t * 64 + r64;
            ok[u] = (e0 + u * NXG < n_items) && (m < M1) && (kg * 8 < C::CIN);
            const int mc = min(m, M1 - 1), kgc = min(kg, (C::CIN - 1) / 8);
            const int f = (C::FACES > 1) ? mc / ppf : 0;
            const int mr = mc - f * ppf;                    // pixel inside the face's valid rows
            const float* src = p.x + ((size_t)((f0 + f) * C::W + rf) * C::W + mr) * C::CIN + kgc * 8;
            qa[u] = __ldg(reinterpret_cast<const float4*>(src));
            qb[u] = __ldg(reinterpret_cast<const float4*>(src + 4));
          }
          if (e0 == xg) SYN_TRACE(0, 62, 5);
#pragma unroll
          for (int u = 0; u < PB; ++u) {
            v[u][0] = ok[u] ? qa[u].x : 0.f; v[u][1] = ok[u] ? qa[u].y : 0.f; v[u][2] = ok[u] ? qa[u].z : 0.f; v[u][3] = ok[u] ? qa[u].w : 0.f;
            v[u][4] = ok[u] ? qb[u].x : 0.f; v[u][5] = ok[u] ? qb[u].y : 0.f; v[u][6] = ok[u] ? qb[u].z : 0.f; v[u][7] = ok[u] ? qb[u].w : 0.f;
          }
#pragma unroll
          for (int u = 0; u < PB; ++u) {
            const int e = e0 + u * NXG;
            if (e < n_items) {
              const int t = e / KG, kg = e - t * KG;
              uint32_t h[4], l[4];
              bool out_of_range = false;                            // |x| > 937.5, +-Inf or NaN
#pragma unroll
              for (int j = 0; j < 8; ++j) out_of_range |= act_clamped(v[u][j]);
              if (out_of_range) *p.sat = 1;                         // the clamp below changes a value: tell the host (sticky)
#pragma unroll
              for (int j = 0; j < 4; ++j) split2_f16(v[u][2 * j] * kActScale, v[u][2 * j + 1] * kActScale, h[j], l[j]);
              // canonical K-major operand: row of this thread in slab t, 8 K values = one 16-byte core-matrix row
              uint8_t* xa = sXA + t * C::XA_TILE + (r64 >> 3) * 128 + kg * 1024 + (r64 & 7) * 16;
              *reinterpret_cast<uint4*>(xa) = make_uint4(h[0], h[1], h[2], h[3]);
              *reinterpret_cast<uint4*>(xa + C::XA_PLANE) = make_uint4(l[0], l[1], l[2], l[3]);
              if (e == xg) SYN_TRACE(0, 62, 6);
            }
          }
          if (e0 == xg) SYN_TRACE(0, 62, 7);
        }
      }
      SYN_TRACE(0, 62, 3);
      fence_proxy_async_smem();                             // XA is read by wgmma after the next worker barrier
      SYN_TRACE(0, 62, 4);

    };
    // L2 prefetch of a tile's input (one contiguous NHWC range) a whole tile ahead of its conversion: the
    // loads in prep() then hit L2 with warm TLB entries instead of paying ~2000 cycles per batch
    auto prefetch_x = [&](int tile) {
      if (tile >= ntiles) return;
      const int fg = tile / C::STRIPS, sp = tile - fg * C::STRIPS;
      int f0, nfaces;
      group_faces(fg, f0, nfaces);
      const int iy0 = sp * C::RO * C::STRIDE - 1;
      const int rf = max(iy0, 0), rl = min(iy0 + C::RWIN - 1, C::W - 1);
      const char* base = reinterpret_cast<const char*>(p.x + ((size_t)(f0 * C::W + rf) * C::W) * C::CIN);
      const int bytes = (C::FACES > 1 ? nfaces * C::W * C::W : (rl - rf + 1) * C::W) * C::CIN * 4;
      for (int o = tid * 128; o < bytes; o += NWT * 128)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(base + o));
    };
    // Programmatic dependent launch: everything above (barriers, the zeroed window, the weight image) does not
    // depend on the previous kernel; its output -- this kernel's input -- is first touched below, and this kernel's
    // first global store comes later still.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if ((int)blockIdx.x < ntiles) prep(blockIdx.x);
    prefetch_x(blockIdx.x + gridDim.x);

    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int fg = tile / C::STRIPS, sp = tile - fg * C::STRIPS;
      int f0, nfaces;
      group_faces(fg, f0, nfaces);
      const int oy0 = sp * C::RO;
      const int iy0 = oy0 * C::STRIDE - 1;
      const int rf = max(iy0, 0), rl = min(iy0 + C::RWIN - 1, C::W - 1);
      const int ppf = (rl - rf + 1) * C::W;               // valid input pixels per face
#ifdef SYN_FUSED_TRACE
      const bool trace_on = blockIdx.x == 0 && tile == (int)gridDim.x && tid == 0;
#endif
      SYN_TRACE(0, 63, 0);
      const int M1 = nfaces * ppf;
      const int mt1 = (M1 + 127) >> 7;
      const int M2 = nfaces * C::M2F;
      const int mt2 = (M2 + 127) >> 7;

      const int slabs1 = (M1 + 63) >> 6;
      float acc1[2][C::NC / 2];                            // D1 double buffer (see the MMA schedule above)
      float acc2[IPW][N2 / 2];                             // this warpgroup's D2 items, accumulated over the chunks
      // weight slot of chunk c (chunk counter gc); streamed slots are waited for by every worker: all of them read
      // the chunk's depthwise taps and EPI1 constants
      auto chunk_slot = [&](uint32_t gc, int c) -> const uint8_t* {
        const int slot = C::WSTREAM ? (int)(gc % C::WSTAGES) : c;
        if constexpr (C::WSTREAM) mbar_wait(smem_u32(&bar_wfull[slot]), (gc / C::WSTAGES) & 1, p.err);
        return sWch + slot * C::CHUNK_BYTES;
      };
      // ---- GEMM1 + EPI1 of chunk c, one 64-row slab of D1 at a time per warpgroup: relu6(s1*D1 + b1) / 6 -> hidden
      // window.  The first slab is in flight on entry.  The expand scale is one power of two per hidden channel, read
      // with the bias (rows 10-11 hold {b1, b1, s1, s1} per channel pair), so an element costs one FFMA.SAT.
      auto gemm1_epi1 = [&](int c, const uint8_t* wch) {
        const float* dwc = reinterpret_cast<const float*>(wch + C::CH_DW);
        const float* bs1 = dwc + 10 * C::DWS;
        // a thread's columns are the same in every slab and both row halves: its NC / 8 {b1 / 6, b1 / 6, s1, s1}
        // vectors are loaded once per chunk
        float4 bs[C::NC / 8];
#pragma unroll
        for (int q = 0; q < C::NC / 8; ++q) bs[q] = *reinterpret_cast<const float4*>(bs1 + 2 * acc_col(row, 4 * q));
#pragma unroll
        for (int j = 0; j < SPW; ++j) {
          const int s1 = wg + j * NWG;                                // warpgroup-uniform
          if (j + 1 < SPW) issue_g1(s1 + NWG < slabs1, acc1[(j + 1) & 1], s1 + NWG, wch);
          // retire slab j; slab j + 1 stays in flight
          if (j + 1 < SPW) wgmma_wait<1>();
          else wgmma_wait<0>();
          if (s1 >= slabs1) continue;
          const float* acc = acc1[j & 1];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = 64 * s1 + acc_row(row, 2 * h);
            if (m < M1) {
              const int f = (C::FACES > 1) ? m / ppf : 0;
              const int mr = m - f * ppf;
              const int yl = mr / C::W, xx = mr - yl * C::W;
              float* hrow = sH + (size_t)(f * C::HS_FACE + (rf - iy0 + yl) * C::HS_COLS + xx + 1) * C::HS_STRIDE;
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
        SYN_TRACE(0, c, 3);
      };
      {
        SYN_TRACE(0, 0, 0);
        const uint8_t* w0 = chunk_slot(g, 0);
        // XA of this tile is complete (and every depthwise read of the previous tile's window is done)
        group_bar_sync<TPG>(grp);
        SYN_TRACE(0, 0, 1);
        // ---- strip mode: window rows outside the image must read as zero (may hold a previous tile)
        if constexpr (C::STRIPS > 1) {
          constexpr int CQ = KPG * 2;                               // float4 per pixel
          if (iy0 < 0)
            for (int i = gtid; i < C::HS_COLS * CQ; i += TPG)
              *reinterpret_cast<float4*>(sH + (size_t)(i / CQ) * C::HS_STRIDE + grp * KPG * 8 + (i % CQ) * 4) =
                  make_float4(0.f, 0.f, 0.f, 0.f);
          if (iy0 + C::RWIN - 1 > C::W - 1)
            for (int i = gtid; i < C::HS_COLS * CQ; i += TPG)
              *reinterpret_cast<float4*>(sH + (size_t)((C::RWIN - 1) * C::HS_COLS + i / CQ) * C::HS_STRIDE +
                                         grp * KPG * 8 + (i % CQ) * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        issue_g1(wg < slabs1, acc1[0], wg, w0);
        gemm1_epi1(0, w0);
      }
      // Chunk c runs from its depthwise pass to EPI1 of chunk c + 1, so that no MMA is in flight across the loop's
      // back edge: ptxas would serialise every MMA otherwise.
      for (int c = 0; c < C::NCHUNK; ++c, ++g) {
        const int slot = C::WSTREAM ? (int)(g % C::WSTAGES) : c;
        const uint8_t* wch = sWch + slot * C::CHUNK_BYTES;
        const float* dwc = reinterpret_cast<const float*>(wch + C::CH_DW);
        // the hidden window of this chunk is complete, and no warpgroup reads A2 any more
        group_bar_sync<TPG>(grp);
        SYN_TRACE(0, c, 4);
        // the first GEMM1 slab of the next chunk runs under the depthwise pass (an empty group after the last chunk)
        const bool more = c + 1 < C::NCHUNK;
        const uint8_t* wn = wch;
        if constexpr (!LATE_G1) {
          if (more) wn = chunk_slot(g + 1, c + 1);
          issue_g1(more && wg < slabs1, acc1[0], wg, wn);
        }
        // ---- DW: 3x3 depthwise on the window -> A2 operand ----------------------------------------
        if constexpr (C::STRIDE == 1 && ((C::WO >= 15 && C::WO <= 30) || C::WO == 8)) {
          // Stride-1 30^2, 15^2 and 8^2 maps (on the 60^2 map of block 1 the units do not divide evenly between
          // the channel groups and the row-pair items below are faster): the window loads of the depthwise
          // conv are what the shared-memory pipe spends its time on, so an item is register-blocked over a 2 x 2 output patch
          // of ONE channel quad -- 16 window + 10 tap LDS.128 per 16 outputs instead of 24 + 20.
          // A unit of 16 threads = 8 lanes along x (column pairs) x the two quads of a channel octet.
          // Lanes 4-7 are MIRRORED: they walk the four window columns right to left, use the taps with kx
          // reversed and own the patch columns in the opposite order.  Neighbouring lanes are 2 pixels =
          // an even number of 16-byte bank groups apart, and the mirror image shifts lanes 4-7 onto the odd
          // groups: every window load (quarter-warp) and every 8-byte operand store (half-warp) is
          // bank-conflict free.
          // 8x8 maps: the 8 lanes are 4 column pairs x 2 row pairs; the second row pair lies 2 window rows = 4 bank
          // groups further and is the mirrored half.
          constexpr int XL = (C::WO >= 15) ? 8 : 4, YL = 8 / XL;           // lanes of a unit along x / along row pairs
          constexpr int CPR = (C::WO + 1) / 2, XG2 = (CPR + XL - 1) / XL, RP2 = (C::RO + 1) / 2;
          constexpr int RPU = (RP2 + YL - 1) / YL, UPK = RPU * XG2;        // units per (face, channel octet)
          const int l8 = tid & 7, qh = (tid >> 3) & 1;
          const int lx = l8 % XL, ly = l8 / XL;
          const bool mir = (l8 & 4) != 0;
          const int units = KPG * nfaces * UPK;
          for (int u = gtid >> 4; u < units; u += TPG / 16) {
            const int kgl = u / (nfaces * UPK), r1 = u - kgl * (nfaces * UPK);
            const int f = r1 / UPK, r2 = r1 - f * UPK;
            const int rpu = r2 / XG2, xg = r2 - rpu * XG2;
            const int kg = grp * KPG + kgl, j0 = kg * 8 + qh * 4;
            const int ox = 2 * (xg * XL + lx), oy = 2 * (rpu * YL + ly);
            if (ox >= C::WO || oy >= C::RO) continue;
            const bool two = (oy + 1 < C::RO);
            const float* wq = dwc + j0;
            float2 w[3][3][2];                                             // [ky][local kx][channel pair]
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
              for (int kl = 0; kl < 3; ++kl) {
                const float4 t4 = *reinterpret_cast<const float4*>(wq + (ky * 3 + (mir ? 2 - kl : kl)) * C::DWS);
                w[ky][kl][0] = make_float2(t4.x, t4.y); w[ky][kl][1] = make_float2(t4.z, t4.w);
              }
            float2 acc[2][2][2];                                           // [output row][local column][channel pair]
            {
              const float4 b4 = *reinterpret_cast<const float4*>(wq + 9 * C::DWS);
#pragma unroll
              for (int ro = 0; ro < 2; ++ro)
#pragma unroll
                for (int a = 0; a < 2; ++a) { acc[ro][a][0] = make_float2(b4.x, b4.y); acc[ro][a][1] = make_float2(b4.z, b4.w); }
            }
            // window columns ox-1 .. ox+2 are Hs columns ox .. ox+3; local column ic is Hs column ox+ic (ox+3-ic mirrored)
            const float* hb = sH + (size_t)(f * C::HS_FACE + oy * C::HS_COLS + ox + (mir ? 3 : 0)) * C::HS_STRIDE + j0;
            const int cstep = mir ? -C::HS_STRIDE : C::HS_STRIDE;
#pragma unroll
            for (int ic = 0; ic < 4; ++ic) {
              float2 d[4][2];
#pragma unroll
              for (int r = 0; r < 4; ++r) {
                if (r == 3 && !two) continue;                              // row only the absent second output row needs
                const float4 t4 = *reinterpret_cast<const float4*>(hb + r * (C::HS_COLS * C::HS_STRIDE) + ic * cstep);
                d[r][0] = make_float2(t4.x, t4.y); d[r][1] = make_float2(t4.z, t4.w);
              }
#pragma unroll
              for (int a = 0; a < 2; ++a) {
                const int kl = ic - a;
                if (kl < 0 || kl > 2) continue;
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
                  for (int j = 0; j < 2; ++j) acc[0][a][j] = ffma2(d[ky][j], w[ky][kl][j], acc[0][a][j]);
                  if (two) {
#pragma unroll
                    for (int j = 0; j < 2; ++j) acc[1][a][j] = ffma2(d[ky + 1][j], w[ky][kl][j], acc[1][a][j]);
                  }
                }
              }
            }
            constexpr float kOut = 6.0f * kActScale;
#pragma unroll
            for (int ro = 0; ro < 2; ++ro) {
              if (ro == 1 && !two) continue;
#pragma unroll
              for (int a = 0; a < 2; ++a) {
                const int col = ox + (mir ? 1 - a : a);
                if (col >= C::WO) continue;                                // odd width: the last pair has one column
                const int m2 = f * C::M2F + (oy + ro) * C::WO + col;
                uint32_t h0, l0, h1, l1;
                split2_f16<false>(__saturatef(acc[ro][a][0].x) * kOut, __saturatef(acc[ro][a][0].y) * kOut, h0, l0);
                split2_f16<false>(__saturatef(acc[ro][a][1].x) * kOut, __saturatef(acc[ro][a][1].y) * kOut, h1, l1);
                uint8_t* dst = sA2 + (m2 >> 7) * (128 * C::NC * 2) + ((m2 & 127) >> 3) * 128 + kg * 2048 + (m2 & 7) * 16 + qh * 8;
                *reinterpret_cast<uint2*>(dst) = make_uint2(h0, h1);
                *reinterpret_cast<uint2*>(dst + C::A2_PLANE) = make_uint2(l0, l1);
              }
            }
          }
        } else
        {
          // Item = (8 hidden channels, two vertically adjacent output rows, 8 lanes along x): the 3x3
          // windows of the two rows share (S=1: 2 of 4, S=2: 1 of 5) input rows and all nine tap vectors,
          // which cuts the shared-memory loads per output by ~40 % against one pixel per thread.
          // Hidden values are stored as relu6(h)/6 in [0,1] and the bias row holds bdw/6, so the
          // activation is a single saturate and the fp16 pre-scale becomes 6 * kActScale.
          constexpr int NKG = C::NC / 8;
          constexpr int GX = (C::WO >= 8) ? 8 : 4, GY = 8 / GX;            // quarter-warp footprint
          constexpr int XG = (C::WO + GX - 1) / GX;                        // x groups per output row
          // small maps (8x8, 4x4) have fewer row-pair items than worker threads: one output row per item
          // there, so that every thread has work and the per-chunk dependency chain is half as long
          // (chosen when at most a quarter of the threads would have a row-pair item: with half of them busy the
          // extra window loads of single rows cost more than the idle warps)
          constexpr int RPI = (4 * C::FACES * ((C::RO + 1) / 2) * ((C::WO + GX - 1) / GX) * GX * NKG <= NWT) ? 1 : 2;
          constexpr int RP = (C::RO + RPI - 1) / RPI, RPG = (RP + GY - 1) / GY;   // row pairs (rows), groups of them
          constexpr int PER_FACE = XG * RPG;
          constexpr int NR = (RPI - 1) * C::STRIDE + 3;                    // window rows of an item
          const int per_kg = nfaces * PER_FACE;
          const int l8 = tid & 7, lx = l8 % GX, ly = l8 / GX;
          // Stride 2: the window pixels of neighbouring lanes lie 2 * HS_STRIDE floats apart, an even number
          // of 16-byte bank groups, so lanes l and l+4 of a quarter-warp would collide on every window load.
          // Lanes 4-7 therefore take the two channel quads of their octet in the opposite order (q0, q1 are
          // the float offsets of the first / second quad); only the final operand store swaps them back.
          const bool swz = (C::STRIDE == 2) && (l8 & 4);
          const int q0 = swz ? 4 : 0, q1 = 4 - q0;
          {
            const int kg_end = (grp + 1) * KPG;                              // this group's channel octets
            int kg = grp * KPG, it = gtid >> 3;
            while (it >= per_kg && kg < kg_end) { it -= per_kg; ++kg; }
            while (kg < kg_end) {
              const int f = it / PER_FACE, r2 = it - f * PER_FACE;
              const int rpg = r2 / XG, xg = r2 - rpg * XG;
              // single rows with GY == 2: the two rows of a quarter-warp lie RPG rows apart (an even number),
              // which keeps the two half-rows of lanes on disjoint bank groups
              const int ox = xg * GX + lx, oy = (RPI == 2) ? 2 * (rpg * GY + ly) : rpg + RPG * ly;
              if (ox < C::WO && oy < C::RO) {
                const float* wbase = dwc + kg * 8;
                const float* h0 = sH + (size_t)(f * C::HS_FACE + (oy * C::STRIDE) * C::HS_COLS + ox * C::STRIDE) * C::HS_STRIDE + kg * 8;
                const bool two = (RPI == 2) && (oy + 1 < C::RO);             // second output row exists
                float2 acc0[4], acc1[4];                                     // channel pairs
                {
                  const float4 a = *reinterpret_cast<const float4*>(wbase + 9 * C::DWS + q0);
                  const float4 e = *reinterpret_cast<const float4*>(wbase + 9 * C::DWS + q1);
                  acc0[0] = make_float2(a.x, a.y); acc0[1] = make_float2(a.z, a.w); acc0[2] = make_float2(e.x, e.y); acc0[3] = make_float2(e.z, e.w);
  #pragma unroll
                  for (int j = 0; j < 4; ++j) acc1[j] = acc0[j];
                }
  #pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                  float2 w[3][4];
  #pragma unroll
                  for (int dy = 0; dy < 3; ++dy) {
                    const float4 a = *reinterpret_cast<const float4*>(wbase + (dy * 3 + dx) * C::DWS + q0);
                    const float4 e = *reinterpret_cast<const float4*>(wbase + (dy * 3 + dx) * C::DWS + q1);
                    w[dy][0] = make_float2(a.x, a.y); w[dy][1] = make_float2(a.z, a.w);
                    w[dy][2] = make_float2(e.x, e.y); w[dy][3] = make_float2(e.z, e.w);
                  }
  #pragma unroll
                  for (int wr = 0; wr < NR; ++wr) {
                    if (wr >= 3 && !two) continue;                           // rows only the (absent) second pixel needs
                    const float* hp = h0 + (wr * C::HS_COLS + dx) * C::HS_STRIDE;
                    const float4 a = *reinterpret_cast<const float4*>(hp + q0);
                    const float4 e = *reinterpret_cast<const float4*>(hp + q1);
                    const float2 d[4] = {make_float2(a.x, a.y), make_float2(a.z, a.w), make_float2(e.x, e.y), make_float2(e.z, e.w)};
                    if (wr < 3) {
  #pragma unroll
                      for (int j = 0; j < 4; ++j) acc0[j] = ffma2(d[j], w[wr][j], acc0[j]);
                    }
                    if (RPI == 2 && wr >= C::STRIDE) {
  #pragma unroll
                      for (int j = 0; j < 4; ++j) acc1[j] = ffma2(d[j], w[wr - C::STRIDE][j], acc1[j]);
                    }
                  }
                }
                constexpr float kOut = 6.0f * kActScale;                   // relu6(x) * kActScale = sat(x/6) * 384
                const int m2 = f * C::M2F + oy * C::WO + ox;
                {
                  uint32_t h[4], l[4];
  #pragma unroll
                  for (int j = 0; j < 4; ++j)
                    split2_f16<false>(__saturatef(acc0[j].x) * kOut, __saturatef(acc0[j].y) * kOut, h[j], l[j]);
                  uint8_t* dst = sA2 + (m2 >> 7) * (128 * C::NC * 2) + ((m2 & 127) >> 3) * 128 + kg * 2048 + (m2 & 7) * 16;
                  *reinterpret_cast<uint4*>(dst) = swz ? make_uint4(h[2], h[3], h[0], h[1]) : make_uint4(h[0], h[1], h[2], h[3]);
                  *reinterpret_cast<uint4*>(dst + C::A2_PLANE) = swz ? make_uint4(l[2], l[3], l[0], l[1]) : make_uint4(l[0], l[1], l[2], l[3]);
                }
                if (two) {
                  const int m3 = m2 + C::WO;
                  uint32_t h[4], l[4];
  #pragma unroll
                  for (int j = 0; j < 4; ++j)
                    split2_f16<false>(__saturatef(acc1[j].x) * kOut, __saturatef(acc1[j].y) * kOut, h[j], l[j]);
                  uint8_t* dst = sA2 + (m3 >> 7) * (128 * C::NC * 2) + ((m3 & 127) >> 3) * 128 + kg * 2048 + (m3 & 7) * 16;
                  *reinterpret_cast<uint4*>(dst) = swz ? make_uint4(h[2], h[3], h[0], h[1]) : make_uint4(h[0], h[1], h[2], h[3]);
                  *reinterpret_cast<uint4*>(dst + C::A2_PLANE) = swz ? make_uint4(l[2], l[3], l[0], l[1]) : make_uint4(l[0], l[1], l[2], l[3]);
                }
              }
              it += TPG / 8;
              while (it >= per_kg && kg < kg_end) { it -= per_kg; ++kg; }
            }
          }
        }
        SYN_TRACE(0, c, 5);
        if constexpr (LATE_G1) {
          if (more) wn = chunk_slot(g + 1, c + 1);
          issue_g1(more && wg < slabs1, acc1[0], wg, wn);
        }
        fence_proxy_async_smem();
        group_bar_sync<TPG>(grp);   // A2 of this chunk is complete
        {
          // ---- GEMM2: D2 += A2 * W3c^T on this warpgroup's items (accumulators stay in registers over the chunks);
          const uint32_t w_lo = smem_desc_lo(smem_u32(wch + C::CH_W3), LBO_W3);
          const int items2 = ((M2 + 63) >> 6) * NSPL;
#pragma unroll
          for (int u = 0; u < IPW; ++u) {                            // one group per item (empty if it has none)
            const int it = wg + u * NWG;
            if (it < items2) {                                       // warpgroup-uniform
              const int s2 = it / NSPL, pc = it - s2 * NSPL;
              const uint32_t a_lo = smem_desc_lo(smem_u32(sA2 + (s2 >> 1) * (128 * C::NC * 2)) + (s2 & 1) * 1024, 2048);
              const uint32_t b_lo = w_lo + ((pc * (N2 / 8) * 128) >> 4);
              if (p.npass == 1) fused_mma_group<N2, C::NC / 16, 1>(acc2[u], d_hi, a_lo, C::A2_PLANE, 4096, b_lo, C::W3_PLANE, 2 * LBO_W3, c > 0);
              else fused_mma_group<N2, C::NC / 16, 3>(acc2[u], d_hi, a_lo, C::A2_PLANE, 4096, b_lo, C::W3_PLANE, 2 * LBO_W3, c > 0);
            } else {
              wgmma_fence();
              wgmma_commit();
            }
          }
        }
        // GEMM2 is retired at once: kept in flight under the next EPI1, ptxas serialises every MMA of the kernel (it
        // cannot prove that EPI1 reads no register of the pending GEMM2)
        wgmma_wait<0>();
        if constexpr (C::WSTREAM) mbar_arrive(smem_u32(&bar_wempty[slot]));   // the chunk's slot may be refilled
        SYN_TRACE(0, c, 6);
        if (more) {
          SYN_TRACE(0, c + 1, 0);
          SYN_TRACE(0, c + 1, 1);
          gemm1_epi1(c + 1, wn);
        }
      }
      SYN_TRACE(0, 63, 1);

      if (tile + (int)gridDim.x < ntiles) prep(tile + gridDim.x);   // XA is free: every GEMM1 of this tile is done
      prefetch_x(tile + 2 * (int)gridDim.x);
      // ---- EPI2: s3*D2 + b3 (+ skip) -> global NHWC --------------------------------------------------
      SYN_TRACE(0, 63, 2);
      // GEMM2 row m2 -> output pixel of the tile (tiles are contiguous in NHWC memory); -1 = no pixel
      auto out_pixel = [&](int m2) -> int {
        if (m2 >= M2) return -1;
        return m2;
      };
      const int items2 = ((M2 + 63) >> 6) * NSPL;
#pragma unroll
      for (int u = 0; u < IPW; ++u) {
        const int it = wg + u * NWG;
        if (it >= items2) break;
        const int s2 = it / NSPL, pc = it - s2 * NSPL;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int pix = out_pixel(64 * s2 + acc_row(row, 2 * h));
          if (pix < 0) continue;
          float* orow = p.y + ((size_t)(f0 * C::WO + oy0) * C::WO + pix) * C::COUT;
          const float* xrow = p.x + ((size_t)(f0 * C::W + oy0) * C::W + pix) * C::CIN;   // skip: same pixel, CIN == COUT
          float2 res[N2 / 8];
          if constexpr (C::RES) {                                   // all skip loads in flight before the first use
#pragma unroll
            for (int q = 0; q < N2 / 8; ++q) {
              const int j = pc * N2 + acc_col(row, 4 * q);
              res[q] = j < C::COUT ? __ldg(reinterpret_cast<const float2*>(xrow + j)) : make_float2(0.f, 0.f);
            }
          }
#pragma unroll
          for (int q = 0; q < N2 / 8; ++q) {
            const int i = 4 * q + 2 * h, j = pc * N2 + acc_col(row, i);
            if (j < C::COUT) {                                      // COUT is even: pairs never straddle it
              const float2 bb = *reinterpret_cast<const float2*>(sB3 + j);
              const float2 sc = *reinterpret_cast<const float2*>(sB3 + C::COUT_P + j);
              float2 o = make_float2(fmaf(acc2[u][i], sc.x, bb.x), fmaf(acc2[u][i + 1], sc.y, bb.y));
              if constexpr (C::RES) { o.x += res[q].x; o.y += res[q].y; }
              *reinterpret_cast<float2*>(orow + j) = o;
            }
          }
        }
      }
      SYN_TRACE(0, 63, 4);
    }
  } else if (warp == NWW) {
    // =============================== weight loader ================================================
    // The whole warp runs this control flow convergently and every batch of bulk copies sits under one elect.sync.
    const int my_tiles = (ntiles > (int)blockIdx.x) ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const uint32_t total_chunks = (uint32_t)my_tiles * C::NCHUNK;
    auto load_chunk = [&](uint32_t gi) {                     // streaming: chunk gi -> slot gi % WSTAGES
      const uint32_t slot = gi % C::WSTAGES, c = gi % C::NCHUNK;
      mbar_expect_tx(smem_u32(&bar_wfull[slot]), C::CHUNK_BYTES);
      bulk_g2s(smem_u32(sWch + slot * C::CHUNK_BYTES), p.wimg + C::B3_BYTES + (size_t)c * C::CHUNK_BYTES, C::CHUNK_BYTES,
               smem_u32(&bar_wfull[slot]));
    };
    if (elect_one()) {
      if constexpr (C::WSTREAM) {
        mbar_expect_tx(smem_u32(&bar_w), C::B3_BYTES);
        bulk_g2s(smem_u32(smem + C::S_B3), p.wimg, C::B3_BYTES, smem_u32(&bar_w));
        for (uint32_t k = 0; k < (uint32_t)C::WSTAGES; ++k)
          if (total_chunks > k) load_chunk(k);
      } else {
        mbar_expect_tx(smem_u32(&bar_w), C::W_BYTES);
        bulk_g2s(smem_u32(smem + C::S_B3), p.wimg, C::W_BYTES, smem_u32(&bar_w));
      }
    }
    __syncwarp();
    if constexpr (C::WSTREAM) {
      // chunk gi reuses the slot of chunk gi - WSTAGES once every worker's GEMM2 of that chunk is done
      for (uint32_t gi = C::WSTAGES; gi < total_chunks; ++gi) {
        mbar_wait(smem_u32(&bar_wempty[gi % C::WSTAGES]), (gi / C::WSTAGES - 1) & 1, p.err);
        if (elect_one()) load_chunk(gi);
        __syncwarp();
      }
    }
  }
}

// Face groups of a launch: {split, face_groups}.  FACES == 2: full two-face groups fill whole waves of `sms`
// CTAs; the remainder becomes single-face groups when those still fit in one wave.
template <class C>
inline void fused_tile_plan(int batch, int sms, int& split, int& face_groups) {
  if constexpr (C::FACES == 2) {
    const int full = batch / 2, odd = batch & 1, rem = full % sms;
    split = (2 * rem + odd <= sms) ? full - rem : full;
    face_groups = split + (batch - 2 * split);              // every face past the two-face groups is its own group
  } else {
    split = 0;
    face_groups = (batch + C::FACES - 1) / C::FACES;
  }
}

// ---- the instantiations used by the backbone (SURVEY.md section 8(a) shape table) -------------------
// Block 3 takes 48-channel chunks (3 per tile: fewer per-chunk barrier round trips).  The strip heights of blocks 3-6
// are bounded by shared memory: the block input (XA) is staged there next to the hidden window.
//                          CIN CHID NC COUT  W  S  RO FACES RES   weight ring slots (0 = resident)
using FusedB2 = FusedCfg<16, 96, 32, 24, 60, 2, 6, 1, false, 0>;              // features[2]
using FusedB3 = FusedCfg<24, 144, 48, 24, 30, 1, 6, 1, true, 0>;             // features[3]
using FusedB4 = FusedCfg<24, 144, 16, 32, 30, 2, 5, 1, false, 0>;             // features[4]
using FusedB56 = FusedCfg<32, 192, 64, 32, 15, 1, 5, 1, true, 0>;            // features[5], [6]
using FusedB7 = FusedCfg<32, 192, 64, 64, 15, 2, 8, 1, false, 0>;             // features[7]
using FusedB8 = FusedCfg<64, 384, 64, 64, 8, 1, 8, 2, true, 3>;                // features[8..10]
using FusedB11 = FusedCfg<64, 384, 64, 96, 8, 1, 8, 2, false, 2>;              // features[11]
using FusedB12 = FusedCfg<96, 576, 32, 96, 8, 1, 8, 2, true, 3>;               // features[12], [13]
using FusedB14 = FusedCfg<96, 576, 32, 160, 8, 2, 4, 2, false, 3>;             // features[14]
// blocks 15-17: four faces per tile (64 GEMM rows = one MMA slab), so that the 64 x COUT fp32 D2 accumulator fits the
// registers of the worker warpgroups
using FusedB15 = FusedCfg<160, 960, 32, 160, 4, 1, 4, 4, true, 3>;             // features[15], [16]
using FusedB17 = FusedCfg<160, 960, 32, 320, 4, 1, 4, 4, false, 2>;            // features[17]

}  // namespace syn
