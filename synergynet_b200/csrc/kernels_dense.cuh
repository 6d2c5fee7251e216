// 3DMM reconstruction on tensor cores (wgmma; reference model_building.py:106-139, reconstruct_vertex_62):
//   S[b, 3v+c] = u[3v+c] + sum_k W[3v+c, k] * alpha[b, k]      (k = 40 shape + 10 expression)
//   V[b, i, v] = sum_c P[b, i, c] * S[b, 3v+c] + t[b, i];   V[b, 1, v] = 121 - V[b, 1, v]
// The basis product is a GEMM with M = vertices, N = faces, K = 50 (padded to 64); running it once per
// coordinate plane (x, y, z) puts the three coordinates of vertex v in the SAME accumulator position of the
// same thread, so the 3x3 pose transform is per-thread arithmetic.  The kernel is HBM-write bound:
// 638,580 B per face (dense).
//
//   dense_alpha_kernel     params (B,62) -> de-whitened pose (B,12) fp32 + alpha as fp16 hi/lo B tiles
//   dense_recon_tc_kernel  persistent; item = (128-vertex tile, 64-face tile), vertex-tile major; the
//                          96 KB basis tile (3 planes x hi/lo) stays in smem while the CTA walks over
//                          the face tiles
//     warp 16: loader (bulk copies of basis tiles and alpha / pose tiles)
//     warps 0-15: four warpgroups; warpgroup w runs the MMAs (3 planes x 3 passes x 4 K-steps, N = 32) of
//                 vertices 64 (w & 1) .. +63 x faces 32 (w >> 1) .. +31 of every item and their epilogue
// Split-16x3 precision scheme of kernels_tc.cuh; basis rows are pre-scaled per vertex row and alpha
// per coefficient (both powers of two, folded back exactly in the epilogue / the basis image); a face whose scaled
// coefficients leave the fp16 range is further divided by a per-face power of two (dense_alpha_kernel).
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace syn {

constexpr int kDnK = 64;                                  // padded coefficient count
constexpr int kDnFaces = 64;                              // faces per tile (MMA N)
constexpr int kDnAPlane = 128 * kDnK * 2;                 // 16 KB: one plane (hi or lo) of one coordinate
constexpr int kDnATile = 3 * 2 * kDnAPlane;               // 96 KB per 128-vertex tile: [x|y|z][hi|lo]
constexpr int kDnBPlane = kDnFaces * kDnK * 2;            // 8 KB
constexpr int kDnBTile = 2 * kDnBPlane;                   // 16 KB per face tile: [hi|lo]
constexpr int kDnPoseStride = 20;                        // floats per face: [R|t] (12), crop->image affine kx, sx, ky, sy, kz, face scale fs, pad
constexpr int kDnPoseTile = kDnFaces * kDnPoseStride * 4; // 5 KB
constexpr int kDnBSlot = kDnBTile + kDnPoseTile;
constexpr int kDnMetaTile = 128 * 6 * 4;                  // per vertex tile: u[3][128], 1/rowscale[3][128]
constexpr int kDnBSlots = 4;                              // alpha/pose ring: loads run 3 items ahead of the MMAs
constexpr int kDnSmem = kDnATile + 2 * kDnMetaTile + kDnBSlots * kDnBSlot + 1024;
constexpr int kDnEpiWarps = 16;                          // four warpgroups: MMA + epilogue
constexpr int kDnThreads = (kDnEpiWarps + 1) * 32;

// ---- pre-pass -----------------------------------------------------------------------------------------
// alpha image: per face tile [hi plane 64 faces x 64 k][lo plane], canonical K-major (SBO 128, LBO 1024);
// pose: (tiles*64, kDnPoseStride) fp32 rows [R|t] (model_building.py:27-29) + crop -> image affine, identity / zero
// rows past the batch.  One thread per (face, group of 8 coefficients): a 512-thread CTA per face tile, every uint4 of
// the image and every float4 of the pose rows is produced by its own thread (the first version -- one thread per face
// walking all 62 parameters -- took as long as a tenth of the dense reconstruction it feeds).
constexpr int kDnAlphaThreads = kDnFaces * (kDnK / 8);
__global__ void __launch_bounds__(kDnAlphaThreads) dense_alpha_kernel(const float* __restrict__ params, const float* __restrict__ mean,
                                                                      const float* __restrict__ stdv, const float* __restrict__ ascale,
                                                                      uint8_t* __restrict__ aimg, float* __restrict__ pose, int batch,
                                                                      int whitening, const float* __restrict__ roi5,
                                                                      int* __restrict__ sat) {
  // the reconstruction kernel may start its prologue (barriers, basis planes) now; it waits for this grid
  // (griddepcontrol.wait) before it touches the alpha image or the pose rows
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int f = threadIdx.x & (kDnFaces - 1), kg = threadIdx.x / kDnFaces, tile = blockIdx.x;
  const int b = tile * kDnFaces + f;
  const bool live = b < batch;
  auto param = [&](int j) {                                  // de-whitened parameter j of face b (model_building.py:117)
    float v = 0.f;
    if (live) {
      v = params[(size_t)b * kNumParams + j];
      if (whitening) v = v * stdv[j] + mean[j];
    }
    return v;
  };
  float a[8], amax = 0.f;
  bool nonfinite = false;                                    // NaN / +-Inf: the split clamps it (fmaxf drops a NaN)
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = kg * 8 + j;
    a[j] = (k < kNumAlpha) ? param(12 + k) * ascale[k] : 0.f;
    amax = fmaxf(amax, fabsf(a[j]));
    nonfinite = nonfinite || !(fabsf(a[j]) <= FLT_MAX);
  }
  if (nonfinite) *sat = 1;                                   // sticky, cleared by syn_poll_saturation
  // Face scale: ascale bounds |alpha_k * ascale_k| by 2^10 within 8 sigma of the mean, but a face further out (or raw
  // coefficients with whitening off) would hit split2_f16's clamp at 60000.  Such a face is divided by a power of two
  // fs that brings its largest scaled coefficient into [2^14, 2^15); the epilogues multiply the accumulator by fs
  // (exact).  Faces inside the clamp keep fs = 1 and their results bit for bit.
  __shared__ float s_amax[kDnK / 8][kDnFaces];
  s_amax[kg][f] = amax;
  __syncthreads();
#pragma unroll
  for (int g = 0; g < kDnK / 8; ++g) amax = fmaxf(amax, s_amax[g][f]);
  float fs = 1.f, fs_inv = 1.f;
  if (amax > 60000.f && isfinite(amax)) {
    const int ex = ((__float_as_int(amax) >> 23) & 0xff) - 126;     // amax in [2^(ex-1), 2^ex)
    fs = __int_as_float((ex - 15 + 127) << 23);
    fs_inv = __int_as_float((127 - ex + 15) << 23);
  }
  // pose row: float4 #kg of [R|t] (kg 0..2), crop -> image affine kx,sx,ky,sy (3), kz,fs,0,0 (4)
  // (utils/inference.py:127-138: x*kx+sx, y*ky+sy, z*kz; identity if absent)
  if (kg < kDnPoseStride / 4) {
    float4 v;
    if (kg < 3) {
      v = make_float4(param(4 * kg), param(4 * kg + 1), param(4 * kg + 2), param(4 * kg + 3));
    } else {
      const bool has = roi5 != nullptr && live;
      const float* r = roi5 + (size_t)b * 5;
      if (kg == 3) v = make_float4(has ? r[0] : 1.f, has ? r[1] : 0.f, has ? r[2] : 1.f, has ? r[3] : 0.f);
      else v = make_float4(has ? r[4] : 1.f, fs, 0.f, 0.f);
    }
    *reinterpret_cast<float4*>(pose + (size_t)(tile * kDnFaces + f) * kDnPoseStride + 4 * kg) = v;
  }
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) tc::split2_f16(a[2 * j] * fs_inv, a[2 * j + 1] * fs_inv, h[j], l[j]);
  uint8_t* hi = aimg + (size_t)tile * kDnBTile + kg * 1024 + f * 16;   // (f >> 3) * 128 + (f & 7) * 16 = f * 16
  *reinterpret_cast<uint4*>(hi) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(hi + kDnBPlane) = make_uint4(l[0], l[1], l[2], l[3]);
}

struct DenseArgs {
  const uint8_t* basis_img;   // [vertex tiles][x|y|z][hi|lo][128 x 64] canonical (SBO 128, LBO 2048)
  const float* meta;          // [vertex tiles][6][128]: u_x,u_y,u_z, 1/rowscale_x,_y,_z
  const uint8_t* alpha_img;   // from dense_alpha_kernel
  const float* pose;
  float* out;                 // (B,3,nver)
  int batch, nver, n_vtiles, n_ftiles, transform;
  int affine;                 // apply the per-face crop -> image affine stored behind the pose rows
  long long* trace;           // debug (SYN_DENSE_TRACE): clock64 stamps of CTA 0, 8 events x 64 items x {team 0, unused, loader}
  int* err;
};

// Synchronisation (item i uses B slot i % kDnBSlots; items are processed in order by every warpgroup):
//   bar_a        basis tile + meta landed (one phase per vertex tile)       loader -> compute warps
//   bar_bfull[s] alpha + pose tile landed                                    loader -> compute warps
//   bar_done[s]  all 512 compute threads are done with the item in slot s (its B slot, and -- at a vertex-tile
//                change -- the basis tile and its meta rows may be overwritten)                  -> loader
__global__ void __launch_bounds__(kDnThreads, 1) dense_recon_tc_kernel(const DenseArgs p) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_a, bar_bfull[kDnBSlots], bar_done[kDnBSlots];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  float* sMeta = reinterpret_cast<float*>(smem + kDnATile);          // 2 slots (vertex-tile load parity)
  uint8_t* sB = smem + kDnATile + 2 * kDnMetaTile;                   // kDnBSlots slots of alpha + pose

  const int tid = threadIdx.x, warp = tid >> 5;
  const int items = p.n_vtiles * p.n_ftiles;
  const int per = (items + gridDim.x - 1) / gridDim.x;
  const int it0 = min((int)blockIdx.x * per, items), it1 = min(it0 + per, items);

  if (tid == 0) {
    mbar_init(smem_u32(&bar_a), 1);
    for (int i = 0; i < kDnBSlots; ++i) {
      mbar_init(smem_u32(&bar_bfull[i]), 1);
      mbar_init(smem_u32(&bar_done[i]), kDnEpiWarps * 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < kDnEpiWarps) {
    // ------------------------------ MMA + epilogue ------------------------------------------------
    const int t = tid & 127, wg = tid >> 7, slab = wg & 1, fh = wg >> 1;
    const int vt0 = it0 / p.n_ftiles;
    int cur_vt = -1;
    float ux[2] = {}, uy[2] = {}, uz[2] = {}, ox[2] = {}, oy[2] = {}, oz[2] = {};
    const uint32_t d_hi = smem_desc_hi(128);
    const uint32_t a_lo = smem_desc_lo(smem_u32(sA) + slab * 1024, 2048);
    for (int it = it0, i = 0; it < it1; ++it, ++i) {
      const int vt = it / p.n_ftiles, ft = it - vt * p.n_ftiles;
      const int sb = i % kDnBSlots;
      mbar_wait(smem_u32(&bar_bfull[sb]), (uint32_t)(i / kDnBSlots) & 1, p.err);
      if (vt != cur_vt) {             // new basis tile and its meta rows
        cur_vt = vt;
        mbar_wait(smem_u32(&bar_a), (uint32_t)(vt - vt0) & 1, p.err);
        const float* m = sMeta + ((vt - vt0) & 1) * (kDnMetaTile / 4);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int lv = 64 * slab + acc_row(t, 2 * h);
          ux[h] = m[0 * 128 + lv]; uy[h] = m[1 * 128 + lv]; uz[h] = m[2 * 128 + lv];
          ox[h] = m[3 * 128 + lv]; oy[h] = m[4 * 128 + lv]; oz[h] = m[5 * 128 + lv];
        }
      }
      const uint32_t b_lo = smem_desc_lo(smem_u32(sB + sb * kDnBSlot) + fh * 4 * 128, 1024);   // faces 32 fh ..
      float acc[3][16];
      wgmma_fence();
#pragma unroll
      for (int plane = 0; plane < 3; ++plane) {
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
          const uint32_t a_off = (plane * 2 + (pass == 2 ? 1 : 0)) * kDnAPlane;   // W: hi,hi,lo
          const uint32_t b_off = (pass == 1 ? kDnBPlane : 0);                     // alpha: hi,lo,hi
#pragma unroll
          for (int ks = 0; ks < kDnK / 16; ++ks)
            wgmma_f16<32>(acc[plane], desc64(d_hi, a_lo + ((a_off + ks * 4096) >> 4)),
                          desc64(d_hi, b_lo + ((b_off + ks * 2048) >> 4)), (pass > 0 || ks > 0) ? 1u : 0u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      const float* pose_tile = reinterpret_cast<const float*>(sB + sb * kDnBSlot + kDnBTile);
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int h = (q >> 1) & 1;
        const int v = vt * 128 + 64 * slab + acc_row(t, q);
        const int fl = 32 * fh + acc_col(t, q), b = ft * kDnFaces + fl;
        if (v < p.nver && b < p.batch) {
          const float* pose = pose_tile + fl * kDnPoseStride;
          const float4 r0 = *reinterpret_cast<const float4*>(pose);
          const float4 r1 = *reinterpret_cast<const float4*>(pose + 4);
          const float4 r2 = *reinterpret_cast<const float4*>(pose + 8);
          const float fs = pose[17];                             // face scale (dense_alpha_kernel)
          const float X = fmaf(acc[0][q] * fs, ox[h], ux[h]), Y = fmaf(acc[1][q] * fs, oy[h], uy[h]),
                      Z = fmaf(acc[2][q] * fs, oz[h], uz[h]);
          float vx = fmaf(r0.x, X, fmaf(r0.y, Y, fmaf(r0.z, Z, r0.w)));
          float vy = fmaf(r1.x, X, fmaf(r1.y, Y, fmaf(r1.z, Z, r1.w)));
          float vz = fmaf(r2.x, X, fmaf(r2.y, Y, fmaf(r2.z, Z, r2.w)));
          if (p.transform) vy = (float)(kImg + 1) - vy;          // model_building.py:129,137
          if (p.affine) {                                        // utils/inference.py:131-136, numpy's fp32 mul then add
            const float4 a4 = *reinterpret_cast<const float4*>(pose + 12);
            vx = __fadd_rn(__fmul_rn(vx, a4.x), a4.y);
            vy = __fadd_rn(__fmul_rn(vy, a4.z), a4.w);
            vz = __fmul_rn(vz, pose[16]);
          }
          float* o = p.out + (size_t)b * 3 * p.nver + v;
          __stcs(o, vx); __stcs(o + p.nver, vy); __stcs(o + 2 * (size_t)p.nver, vz);   // write-once stream
        }
      }
      mbar_arrive(smem_u32(&bar_done[sb]));
    }
  } else if (warp == kDnEpiWarps) {
    // ------------------------------ loader (converged warp, bulk copies under elect.sync) -----------------
    auto load_b = [&](int it, int s) {
      if (elect_one()) {
        const int ft = it % p.n_ftiles;
        uint8_t* dst = sB + s * kDnBSlot;
        mbar_expect_tx(smem_u32(&bar_bfull[s]), kDnBSlot);
        bulk_g2s(smem_u32(dst), p.alpha_img + (size_t)ft * kDnBTile, kDnBTile, smem_u32(&bar_bfull[s]));
        bulk_g2s(smem_u32(dst + kDnBTile), p.pose + (size_t)ft * kDnFaces * kDnPoseStride, kDnPoseTile, smem_u32(&bar_bfull[s]));
      }
      __syncwarp();
    };
    auto done_wait = [&](int j) {                                   // every compute thread finished item j (>= 0)
      mbar_wait(smem_u32(&bar_done[j % kDnBSlots]), (uint32_t)(j / kDnBSlots) & 1, p.err);
    };
    int cur_vt = -1;
    const int vt0 = it0 / p.n_ftiles;
    asm volatile("griddepcontrol.wait;" ::: "memory");               // alpha image / pose rows come from the pre-pass
    for (int k = 0; k < kDnBSlots - 1; ++k)
      if (it0 + k < it1) load_b(it0 + k, k);
    for (int it = it0, i = 0; it < it1; ++it, ++i) {
      const int vt = it / p.n_ftiles;
      if (vt != cur_vt) {
        // the basis tile in smem is overwritten: every thread must be done with item i-1 (its MMAs read the old tile)
        if (i >= 1) done_wait(i - 1);
        cur_vt = vt;
        if (elect_one()) {
          mbar_expect_tx(smem_u32(&bar_a), kDnATile + kDnMetaTile);
          bulk_g2s(smem_u32(sA), p.basis_img + (size_t)vt * kDnATile, kDnATile, smem_u32(&bar_a));
          bulk_g2s(smem_u32(sMeta + ((vt - vt0) & 1) * (kDnMetaTile / 4)), p.meta + (size_t)vt * 6 * 128, kDnMetaTile,
                   smem_u32(&bar_a));
        }
        __syncwarp();
      }
      // prefetch alpha/pose three items ahead into the slot last used by item i-1
      if (it + kDnBSlots - 1 < it1) {
        if (i >= 1) done_wait(i - 1);
        load_b(it + kDnBSlots - 1, (i + kDnBSlots - 1) % kDnBSlots);
      }
    }
  }
}


// -------------------------------------------------------------------------------------------------------------------
// Face-major variant for the dense mesh (configs[2]).  The kernel above walks vertex-tile major: a CTA writes 512 B
// to each of 64 faces x 3 rows and moves on to OTHER faces, so every DRAM page is touched once per visit.  Here a CTA
// keeps one 64-face tile and walks over consecutive vertex tiles: each of its 192 output rows grows by 512 contiguous
// bytes per item.  The price is a new basis tile per item; it streams from L2 (40 MB image, resident in the 50 MB L2)
// coordinate plane by coordinate plane (32 KB = hi + lo of one coordinate) through a 4-slot ring, ahead of the MMAs.
//
// WHOLE-SECTOR STORES.  The output rows of the reference layout (B,3,53215) fp32 start on every 4-byte phase, so a warp
// that stores "lane = vertex" always writes two partial 32-byte sectors per 128 bytes; the same bytes written as whole
// aligned sectors are much cheaper for the memory system.  So the epilogue does not store from the accumulator layout:
// a TEAM (one warpgroup: 128 vertices = two 64-row MMA slabs, 16 faces) stages 24 output rows (8 faces x 3 coordinates)
// at a time in shared memory and writes them back out with the lane -> address mapping shifted by each row's own
// phase (address / 4 mod 8), so that every warp store covers whole aligned sectors.  The <= 7 floats that fall off the
// end of a row piece are carried (sCarry) into the next item's piece of the same row; only the two ends of a CTA's
// band are written with bounds-checked stores.
//   bar_pfull[slot]   plane landed                                                    loader -> teams
//   bar_pempty[slot]  all 512 team threads' MMAs that read the plane are complete     teams -> loader
//   bar_mfull[slot]   meta rows of item i (slot i % 4) landed                         loader -> teams
//   bar_bfull         alpha + pose tile of the CTA's face tile landed (once)
constexpr int kFmPlane = 2 * kDnAPlane;                   // 32 KB: [hi|lo] of one coordinate of one vertex tile
constexpr int kFmPSlots = 4, kFmMetaSlots = 4;
constexpr int kFmTeams = 4;                               // one warpgroup each: faces 16t .. 16t+15 of the item
constexpr int kFmSubFaces = 8;                            // faces staged per sub-round -> 24 rows
constexpr int kFmRows = 3 * kFmSubFaces;
// floats per staged row (position = vertex within the tile).  128 + 4: the accumulator layout writes rows 6 apart from
// the four lanes of a quad; the pad puts them on four different groups of 8 banks
constexpr int kFmPitch = 132;
constexpr int kFmStage = kFmRows * kFmPitch * 4;          // per team: 12.4 KB
constexpr int kFmCarry = 16 * 3 * 8 * 4;                  // per team: 48 rows x 8 floats
constexpr int kFmSmem = kFmPSlots * kFmPlane + kFmMetaSlots * kDnMetaTile + kDnBSlot + kFmTeams * (kFmStage + kFmCarry) + 1024;
static_assert(kDnATile == 3 * kFmPlane, "basis tile = three coordinate planes");
static_assert(kFmSmem + 512 <= 227 * 1024, "shared memory");
static_assert(kDnEpiWarps == 4 * kFmTeams && kDnFaces == 16 * kFmTeams, "team shape");

// Bounds-checked write-out of dense_recon_fm_kernel for the first / last item of a CTA's band and for ragged face tiles
// (kept out of line: the hot path then needs no predicates).  Same mapping as the fast path in the kernel.
__device__ __forceinline__ void fm_write_edge(const DenseArgs& p, const float* Tw, float* crw, float* piece, int bq, int wq, int lane,
                                           bool first, bool last, int nvalid) {
#pragma unroll 1
  for (int k = 0; k < kFmRows / 4; ++k, piece += 4 * (size_t)p.nver) {
    if (bq + (wq + 4 * k) / 3 >= p.batch) continue;
    const int phase = (int)((reinterpret_cast<uintptr_t>(piece) >> 2) & 7u);
    const float* src = Tw + 4 * k * kFmPitch - phase;
    float* cr = crw + 4 * k * 8;
    const bool low = lane < phase;
    const float v0 = *(low ? cr : src);                              // `first`: garbage below phase, not stored
    const float v1 = src[32], v2 = src[64], v3 = src[96];
    float ov = 0.f;
    if (low) { ov = src[128]; *cr = ov; }
    float* win = piece - phase + lane;
    const int lo = first ? phase : 0;                                // floats below belong to the previous band's CTA
    const int hi = last ? phase + nvalid : 128;                      // the last item also flushes what it would carry
    if (lane >= lo && lane < hi) win[0] = v0;
    if (32 + lane < hi) win[32] = v1;
    if (64 + lane < hi) win[64] = v2;
    if (96 + lane < hi) win[96] = v3;
    if (low && 128 + lane < hi) win[128] = ov;
  }
}

template <bool kTrace, bool kAffine>
__global__ void __launch_bounds__(kDnThreads, 1) dense_recon_fm_kernel(const DenseArgs p) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_pfull[kFmPSlots], bar_pempty[kFmPSlots], bar_mfull[kFmMetaSlots], bar_bfull;
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sP = smem;                                                                      // plane ring
  float* sMeta = reinterpret_cast<float*>(smem + kFmPSlots * kFmPlane);                   // kFmMetaSlots meta tiles
  uint8_t* sB = smem + kFmPSlots * kFmPlane + kFmMetaSlots * kDnMetaTile;                 // alpha + pose tile of this CTA's face tile
  float* sStage = reinterpret_cast<float*>(sB + kDnBSlot);                                // [team][row][kFmPitch]
  float* sCarry = sStage + kFmTeams * (kFmStage / 4);                                     // [team][48 rows][8]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // Work split: CTA = (face tile ft, BAND of consecutive vertex tiles); the bands are the same for every face tile and
  // the CTAs of one band are neighbours in the grid, so the CTAs that need a given basis tile ask for it at about the
  // same time and all but the first hit in L2 (a plain contiguous split of the item list gives every face tile its own
  // band boundaries, and the basis image is read several times from DRAM).
  const int n_bands = max(1, (int)gridDim.x / p.n_ftiles);
  const int band_len = (p.n_vtiles + n_bands - 1) / n_bands;
  const int ft = (int)blockIdx.x % p.n_ftiles, my_band = (int)blockIdx.x / p.n_ftiles;
  const int vt_lo = min(my_band * band_len, p.n_vtiles), vt_hi = (my_band < n_bands) ? min(vt_lo + band_len, p.n_vtiles) : vt_lo;
  const int n_items = vt_hi - vt_lo;                                 // item i = vertex tile vt_lo + i

  if (tid == 0) {
    for (int i = 0; i < kFmPSlots; ++i) {
      mbar_init(smem_u32(&bar_pfull[i]), 1);
      mbar_init(smem_u32(&bar_pempty[i]), kDnEpiWarps * 32);
    }
    for (int i = 0; i < kFmMetaSlots; ++i) mbar_init(smem_u32(&bar_mfull[i]), 1);
    mbar_init(smem_u32(&bar_bfull), 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < kDnEpiWarps) {
    // ------------------------------ 4 teams (warpgroups), every team works on every item ------------------------------
    const int team = warp >> 2, t = tid & 127, wq = warp & 3;
    const int f0 = team * 16;                                        // first face (within the tile) of this team
    float* stage = sStage + team * (kFmStage / 4);
    float* carry = sCarry + team * (kFmCarry / 4);
    const float* pose_tile = reinterpret_cast<const float*>(sB + kDnBTile);
    const uint32_t d_hi = smem_desc_hi(128);
    const uint32_t b_lo = smem_desc_lo(smem_u32(sB) + (f0 / 8) * 128, 1024);   // alpha rows of faces f0 .. f0 + 15
    for (int i = 0; i < n_items; ++i) {
      const int vt = vt_lo + i;
      const bool tr = kTrace && blockIdx.x == 0 && tid == 0 && i < 64;
      if (tr) p.trace[i * 8 + 0] = clock64();
      mbar_wait_inl(smem_u32(&bar_bfull), 0, p.err);                                       // alpha / pose tile visible
      mbar_wait_inl(smem_u32(&bar_mfull[i % kFmMetaSlots]), (uint32_t)(i / kFmMetaSlots) & 1, p.err);   // meta rows visible
      // this thread's four vertices: 64 s + acc_row(t, 2 h), s = MMA slab, h = row half
      float ux[4], uy[4], uz[4], ox[4], oy[4], oz[4];
      {
        const float* m = sMeta + (i % kFmMetaSlots) * (kDnMetaTile / 4);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int lv = 64 * (u >> 1) + acc_row(t, 2 * (u & 1));
          ux[u] = m[0 * 128 + lv]; uy[u] = m[1 * 128 + lv]; uz[u] = m[2 * 128 + lv];
          ox[u] = m[3 * 128 + lv]; oy[u] = m[4 * 128 + lv]; oz[u] = m[5 * 128 + lv];
        }
      }
      if (tr) p.trace[i * 8 + 1] = clock64();
      float acc[3][2][8];                                            // [coordinate][slab][16 faces]
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int q = 3 * i + c, slot = q % kFmPSlots;
        mbar_wait_inl(smem_u32(&bar_pfull[slot]), (uint32_t)(q / kFmPSlots) & 1, p.err);
        const uint32_t a_lo = smem_desc_lo(smem_u32(sP + slot * kFmPlane), 2048);
        wgmma_fence();
#pragma unroll
        for (int sl = 0; sl < 2; ++sl)
#pragma unroll
          for (int pass = 0; pass < 3; ++pass) {
            const uint32_t a_off = sl * 1024 + (pass == 2 ? kDnAPlane : 0);        // W: hi,hi,lo
            const uint32_t b_off = (pass == 1 ? kDnBPlane : 0);                     // alpha: hi,lo,hi
#pragma unroll
            for (int ks = 0; ks < kDnK / 16; ++ks)
              wgmma_f16<16>(acc[c][sl], desc64(d_hi, a_lo + ((a_off + ks * 4096) >> 4)),
                            desc64(d_hi, b_lo + ((b_off + ks * 2048) >> 4)), (pass > 0 || ks > 0) ? 1u : 0u);
          }
        wgmma_commit();
      }
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < 3; ++c) mbar_arrive(smem_u32(&bar_pempty[(3 * i + c) % kFmPSlots]));   // planes may be refilled
      // face scales (dense_alpha_kernel) of this thread's four faces, applied to the accumulators before the epilogue
      // (exact: powers of two; the same values as fmaf(acc * fs, ox, ux) in dense_recon_tc_kernel)
#pragma unroll
      for (int sr = 0; sr < 2; ++sr)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float fs = pose_tile[(f0 + sr * kFmSubFaces + 2 * (t & 3) + e) * kDnPoseStride + 17];
#pragma unroll
          for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int sl = 0; sl < 2; ++sl)
#pragma unroll
              for (int h = 0; h < 2; ++h) acc[c][sl][4 * sr + 2 * h + e] *= fs;
        }
      if (tr) p.trace[i * 8 + 2] = clock64();
      const bool first = i == 0, last = i == n_items - 1;
      const bool edge = first || last || (ft + 1) * kDnFaces > p.batch;     // CTA-uniform
      const int nvalid = min(128, p.nver - vt * 128);
      float* item_row0 = p.out + ((size_t)(ft * kDnFaces + f0) * 3 + wq) * p.nver + (size_t)vt * 128;   // face f0, row wq
#pragma unroll
      for (int sr = 0; sr < 2; ++sr) {                               // faces 8 sr .. 8 sr + 7 of the team = accumulator values 4 sr ..
        const int bq = ft * kDnFaces + f0 + sr * kFmSubFaces;        // first face (batch index) of the sub-round
        // ---- stage: row (face, coordinate), position = vertex (no shift: the reader applies the phase)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int fl = 2 * (t & 3) + e;                            // face within the sub-round
          const float* pose = pose_tile + (f0 + sr * kFmSubFaces + fl) * kDnPoseStride;
          const float4 r0 = *reinterpret_cast<const float4*>(pose);
          const float4 r1 = *reinterpret_cast<const float4*>(pose + 4);
          const float4 r2 = *reinterpret_cast<const float4*>(pose + 8);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int sl = u >> 1, h = u & 1, vi = 4 * sr + 2 * h + e;
            const float X = fmaf(acc[0][sl][vi], ox[u], ux[u]), Y = fmaf(acc[1][sl][vi], oy[u], uy[u]),
                        Z = fmaf(acc[2][sl][vi], oz[u], uz[u]);
            float vx = fmaf(r0.x, X, fmaf(r0.y, Y, fmaf(r0.z, Z, r0.w)));
            float vy = fmaf(r1.x, X, fmaf(r1.y, Y, fmaf(r1.z, Z, r1.w)));
            float vz = fmaf(r2.x, X, fmaf(r2.y, Y, fmaf(r2.z, Z, r2.w)));
            if (p.transform) vy = (float)(kImg + 1) - vy;            // model_building.py:129,137
            if (kAffine) {                                           // utils/inference.py:131-136, numpy's fp32 mul then add
              const float4 a4 = *reinterpret_cast<const float4*>(pose + 12);
              vx = __fadd_rn(__fmul_rn(vx, a4.x), a4.y);
              vy = __fadd_rn(__fmul_rn(vy, a4.z), a4.w);
              vz = __fmul_rn(vz, pose[16]);
            }
            const int lv = 64 * sl + acc_row(t, 2 * h);
            stage[(fl * 3 + 0) * kFmPitch + lv] = vx;
            stage[(fl * 3 + 1) * kFmPitch + lv] = vy;
            stage[(fl * 3 + 2) * kFmPitch + lv] = vz;
          }
        }
        asm volatile("bar.sync %0, 128;" ::"r"(team + 1) : "memory");
        // ---- write out: warp wq takes rows wq + 4k.  Window position pos (0 = the sector boundary at or below the row
        // piece) holds vertex pos - phase of this item, or, below phase, the previous item's overhang.  Lane j stores
        // positions j, 32 + j, 64 + j, 96 + j: every warp store is four whole aligned sectors.
        const float* Tw = stage + wq * kFmPitch + lane;
        float* crw = carry + (sr * kFmRows + wq) * 8 + lane;
        float* piece = item_row0 + (size_t)(sr * kFmRows) * p.nver;   // row wq of the sub-round, first float of the piece
        if (!edge) {
#pragma unroll
          for (int k = 0; k < kFmRows / 4; ++k, piece += 4 * (size_t)p.nver) {
            const int phase = (int)((reinterpret_cast<uintptr_t>(piece) >> 2) & 7u);
            const float* src = Tw + 4 * k * kFmPitch - phase;
            float* cr = crw + 4 * k * 8;
            const bool low = lane < phase;
            const float v0 = *(low ? cr : src);
            const float v1 = src[32], v2 = src[64], v3 = src[96];
            if (low) *cr = src[128];                               // this item's overhang (vertices 128 - phase .. 127)
            float* win = piece - phase + lane;
            win[0] = v0; win[32] = v1; win[64] = v2; win[96] = v3;
          }
        } else {                                                   // first / last item of the band, ragged face tile
          fm_write_edge(p, Tw, crw, piece, bq, wq, lane, first, last, nvalid);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(team + 1) : "memory");   // the staging rows are rewritten next
      }
      if (tr) p.trace[i * 8 + 4] = clock64();
    }
  } else if (warp == kDnEpiWarps) {
    // ------------------------------ loader (converged warp, elect.sync) ------------------------------
    int next_plane = 0;                                               // next plane to request (plane q = 3 * item + coordinate)
    const uint64_t keep = l2_policy_evict_last();                     // the basis image is re-read once per face tile
    // Request planes up to (and including) `upto`.  Plane q reuses the slot of plane q - kFmPSlots, whose MMAs must be
    // complete (bar_pempty, consumed strictly in order).  The meta rows of item v go to slot v % 4, last read by the
    // teams at the start of item v - 4, before they released any plane of item v - 2, which is waited for here.
    auto request_planes = [&](int upto) {
      upto = min(upto, 3 * n_items - 1);
      for (; next_plane <= upto; ++next_plane) {
        const int q = next_plane, slot = q % kFmPSlots, v = q / 3, c = q - 3 * v;
        if (q >= kFmPSlots) mbar_wait_inl(smem_u32(&bar_pempty[slot]), (uint32_t)(q / kFmPSlots - 1) & 1, p.err);
        if (kTrace && blockIdx.x == 0 && lane == 0 && v < 64) p.trace[(128 + v) * 8 + c] = clock64();
        if (elect_one()) {
          mbar_expect_tx(smem_u32(&bar_pfull[slot]), kFmPlane);
          bulk_g2s_hint(smem_u32(sP + slot * kFmPlane), p.basis_img + (size_t)(vt_lo + v) * kDnATile + (size_t)c * kFmPlane,
                        kFmPlane, smem_u32(&bar_pfull[slot]), keep);
          if (c == 0) {
            const int ms = v % kFmMetaSlots;
            mbar_expect_tx(smem_u32(&bar_mfull[ms]), kDnMetaTile);
            bulk_g2s_hint(smem_u32(sMeta + ms * (kDnMetaTile / 4)), p.meta + (size_t)(vt_lo + v) * 6 * 128, kDnMetaTile,
                          smem_u32(&bar_mfull[ms]), keep);
          }
        }
        __syncwarp();
      }
    };
    request_planes(kFmPSlots - 1);                                   // planes 0..3 in flight before the first MMA
    // programmatic dependent launch: everything above overlaps the pre-pass; its output is first touched here
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (n_items > 0) {                                               // alpha + pose of this CTA's face tile: once
      if (elect_one()) {
        mbar_expect_tx(smem_u32(&bar_bfull), kDnBSlot);
        bulk_g2s(smem_u32(sB), p.alpha_img + (size_t)ft * kDnBTile, kDnBTile, smem_u32(&bar_bfull));
        bulk_g2s(smem_u32(sB + kDnBTile), p.pose + (size_t)ft * kDnFaces * kDnPoseStride, kDnPoseTile, smem_u32(&bar_bfull));
      }
      __syncwarp();
    }
    request_planes(3 * n_items - 1);
  }
}

}  // namespace syn
