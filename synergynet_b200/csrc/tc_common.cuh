// wgmma / mbarrier / bulk-copy primitives for sm_90a (Hopper), as inline PTX.
//
// Operand layout used throughout: K-major, no swizzle ("interleaved") canonical GMMA layout.
// A tile of R rows x K columns of 16-bit values is stored as 8x8 core matrices of 128 contiguous
// bytes (8 rows x 16 bytes); element (r, k) lives at byte
//     (r / 8) * SBO + (k / 8) * LBO + (r % 8) * 16 + (k % 8) * 2
// with LBO = stride between core matrices along K and SBO = stride between 8-row groups
// (cute::GMMA::make_gmma_desc<Major::K>, LayoutType::INTERLEAVE: ((8,n),2):((1,SBO),LBO) in
// uint128 units).  One wgmma consumes K = 16 (two core matrices along K).
//
// Accumulators live in the registers of the issuing warpgroup (128 threads).  m64nNk16 with fp32
// accumulators: thread t of the warpgroup holds N/2 values; value i belongs to
//     row = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),   column = 8 * (i / 4) + 2 * (t % 4) + i % 2
// (acc_row / acc_col below).  A piece of columns [n0, n0 + n) of a wider accumulator therefore
// starts at value n0 / 2, and its B operand at byte (n0 / 8) * SBO of the B tile.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace syn {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor) ---------------------------------
// bits [0,14) start>>4, [16,30) LBO>>4, [32,46) SBO>>4, [49,52) base offset = 0, [62,64) layout (0 = interleave)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// The two 32-bit halves separately: callers keep `hi` and a base `lo` in registers and only add
// (byte offset >> 4) to `lo` per instruction instead of rebuilding the 64-bit descriptor.
__device__ __forceinline__ uint32_t smem_desc_lo(uint32_t smem_addr, uint32_t lbo_bytes) {
  return ((smem_addr & 0x3FFFFu) >> 4) | (((lbo_bytes >> 4) & 0x3FFFu) << 16);
}
__device__ __forceinline__ uint32_t smem_desc_hi(uint32_t sbo_bytes) { return (sbo_bytes >> 4) & 0x3FFFu; }
__device__ __forceinline__ uint64_t desc64(uint32_t hi, uint32_t lo) { return ((uint64_t)hi << 32) | lo; }

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must not hang the GPU.  After ~2 s of wall
// clock (or as soon as any other thread has already timed out) the caller-provided sticky flag is
// raised and the wait returns, so the kernel drains with garbage instead of spinning forever.
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Slow path: plain try_wait polling without a suspend-time hint (wake-up latency matters more than the issue slots
// the polling warps take).  The sticky flag (a global load) and the wall clock are only looked at every 256 polls.
__device__ __forceinline__ bool mbar_wait_spin(uint32_t bar, uint32_t parity, int* err_flag) {
  const uint64_t t0 = globaltimer_ns();
  for (uint32_t it = 1;; ++it) {
    if (mbar_try_wait(bar, parity)) return true;
    if ((it & 255u) == 0) {
      if (err_flag != nullptr && *reinterpret_cast<volatile int*>(err_flag) != 0) return false;
      if (globaltimer_ns() - t0 > 2000000000ull) {
        // the flag lives in mapped pinned host memory (the host reads it without a device sync): plain store
        if (err_flag != nullptr) { *reinterpret_cast<volatile int*>(err_flag) = 1; __threadfence_system(); }
        return false;
      }
    }
  }
}
__device__ __noinline__ bool mbar_wait_slow(uint32_t bar, uint32_t parity, int* err_flag) {
  return mbar_wait_spin(bar, parity, err_flag);
}
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, int* err_flag) {
  if (mbar_try_wait(bar, parity)) return true;
  return mbar_wait_slow(bar, parity, err_flag);
}
// always-inline flavour for kernels whose hot loop is made of global stores (dense_recon_fm_kernel): a real call in a
// kernel makes ptxas keep the global-memory descriptor in a vector register and copy it to a uniform register pair
// (2 x R2UR) in front of every LDG / STG; the spin loop inlined costs less code than that.
__device__ __forceinline__ bool mbar_wait_inl(uint32_t bar, uint32_t parity, int* err_flag) {
  if (mbar_try_wait(bar, parity)) return true;
  return mbar_wait_spin(bar, parity, err_flag);
}

// ---- proxies / fences ----------------------------------------------------------------------------
// One lane of a converged warp (elect.sync, full mask).  Code under `if (elect_one())` is known to the
// compiler to run on a single thread, so bulk-copy operands come straight from uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n .reg .pred p;\n elect.sync _|p, 0xffffffff;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(pred));
  return pred != 0;
}

// generic-proxy st.shared -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// ---- wgmma: issued by all 128 threads of a warpgroup, convergently ------------------------------
// fence before the first wgmma that reads accumulator registers written by ordinary instructions
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this warpgroup are still pending
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D(64 x N, fp32, registers) (+)= A(64 x 16, fp16, smem) * B(N x 16, fp16, smem)^T; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_m64n8k16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0,%1,%2,%3}, %4, %5, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n16k16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n32k16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n64k16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n256k16_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(scale_d)
      : "memory");
}

// N known at compile time (multiple of 8, <= 256): one instruction where the shape exists, else 64/32/16/8-column
// pieces (B advanced by (n0 / 8) * 128 bytes: every B tile of this library has SBO = 128)
template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  static_assert(N % 8 == 0 && N > 0 && N <= 256, "wgmma N");
  if constexpr (N == 256) wgmma_m64n256k16_f16(d, adesc, bdesc, scale_d);
  else if constexpr (N == 128) wgmma_m64n128k16_f16(d, adesc, bdesc, scale_d);
  else if constexpr (N == 64) wgmma_m64n64k16_f16(d, adesc, bdesc, scale_d);
  else if constexpr (N == 32) wgmma_m64n32k16_f16(d, adesc, bdesc, scale_d);
  else if constexpr (N == 16) wgmma_m64n16k16_f16(d, adesc, bdesc, scale_d);
  else if constexpr (N == 8) wgmma_m64n8k16_f16(d, adesc, bdesc, scale_d);
  else {
    constexpr int P = N >= 128 ? 128 : N >= 64 ? 64 : N >= 32 ? 32 : N >= 16 ? 16 : 8;
    wgmma_f16<P>(d, adesc, bdesc, scale_d);
    wgmma_f16<N - P>(d + P / 2, adesc, bdesc + (uint64_t)((P / 8) * 128 >> 4), scale_d);
  }
}
// N chosen at run time (multiple of 16, <= 256): 64-column blocks at fixed register offsets, the last partial
// block as 32 / 16 pieces.  d must hold 128 values.
__device__ __forceinline__ void wgmma_f16_rt(float* d, int n, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const int rem = n - 64 * b;
    const uint64_t bd = bdesc + (uint64_t)(b * 8 * 128 >> 4);
    if (rem >= 64) {
      wgmma_m64n64k16_f16(d + 32 * b, adesc, bd, scale_d);
    } else if (rem > 0) {
      if (rem >= 32) wgmma_m64n32k16_f16(d + 32 * b, adesc, bd, scale_d);
      if (rem == 16) wgmma_m64n16k16_f16(d + 32 * b, adesc, bd, scale_d);
      if (rem == 48) wgmma_m64n16k16_f16(d + 32 * b + 16, adesc, bd + (uint64_t)(4 * 128 >> 4), scale_d);
    }
  }
}
// position of accumulator value i of thread t (0..127 inside its warpgroup)
__device__ __forceinline__ int acc_row(int t, int i) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int acc_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// ---- bulk async copy global -> shared (TMA engine, no tensor map), completes on an mbarrier ------
// size multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// Same copy with an L2 eviction-priority hint.  evict_last keeps a re-read working set (the 40 MB dense basis image,
// read once per 64-face tile) resident in the 50 MB L2 while a write-once stream several times its size flows through.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar), "l"(policy)
               : "memory");
}

// ---- fp32 pairs (two scalar FMAs / multiplies; the depthwise code is written on float2 operands) ----------
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// ---- fp32 -> (hi, lo) bf16 split: x ~= hi + lo with |x - hi - lo| <= 2^-17 |x| ----------------------
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// ---- fp32 -> (hi, lo) fp16 split: 11 + 11 mantissa bits, |x - hi - lo| <= 2^-22 |x| while lo stays a
// normal fp16 number.  Callers pre-scale by a power of two (kActScale for activations, a per-channel
// scale for weights) so that this holds over the value range that matters, and clamp to the fp16 range.
constexpr float kActScale = 64.0f;           // relu6 range [0,6] -> [0,384]; block inputs: |x| < 1000
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  x = fminf(fmaxf(x, -60000.f), 60000.f);
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
// true when the clamp of an activation split (x * kActScale to +-60000) would change x: |x| > 937.5, +-Inf or NaN.
// Scaling by a power of two is exact, so the test is made on x itself (no multiply); NaN fails every comparison.
__device__ __forceinline__ bool act_clamped(float x) { return !(fabsf(x) <= 60000.f / kActScale); }
__device__ __forceinline__ uint32_t pack_f16x2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}
// split two fp32 values (already multiplied by their power-of-two scale) into packed hi and lo words;
// CLAMP = false when the inputs are known to be inside the fp16 range (ReLU6 outputs x kActScale)
template <bool CLAMP = true>
__device__ __forceinline__ void split2_f16(float a, float b, uint32_t& hi, uint32_t& lo) {
  if (CLAMP) {
    a = fminf(fmaxf(a, -60000.f), 60000.f);
    b = fminf(fmaxf(b, -60000.f), 60000.f);
  }
  const __half2 h = __floats2half2_rn(a, b);                 // one cvt.rn.f16x2.f32
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

}  // namespace tc
}  // namespace syn
