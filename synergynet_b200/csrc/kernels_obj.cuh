// The OBJ text of write_obj (utils/inference.py:8-23) and write_obj_with_colors (artistic.py:19-31) for B meshes in one
// call (syn_obj_plan, syn_obj_write).  Every line's bytes come from obj_math.h, which the host emulation the CPU tests
// hold to Python's str.format compiles too.
//
// Mesh b's text is its vertex lines, then the triangle lines.  The triangle lines are the same for every mesh, so they
// are formatted once, into mesh 0's text, and copied into the others.
//   plan:  obj_len_kernel     one thread per line: its byte count; one block sum per 256 lines
//          obj_scan_kernel    one CTA: the triangle text's size T and block bases, then the vertex block bases across
//                             meshes (the last vertex block of each mesh carries T): the byte offset of every block and
//                             of every mesh (B + 1)
//   write: obj_write_kernel   the line lengths again, a block scan, each thread stores its line at its block's base
//          obj_copy_kernel    mesh 0's triangle text into meshes 1..B-1
// Every store is checked against the output's size, so a caller's buffer smaller than the plan's total loses text
// instead of memory beyond it; nothing reads the output before writing it.
#pragma once
#include "common.cuh"
#include "obj_math.h"

namespace syn {

constexpr int kObjThreads = 256;

struct ObjArgs {
  const float* v;              // coordinate k of vertex i of mesh b: v[b * sb + i * sv + k * sc]
  long long sb;
  int sv, sc;
  const int32_t* keep;         // vertex line i prints vertex keep[i] (nullptr: vertex i)
  int n;                       // vertex lines per mesh
  const int64_t* colors;       // BGR colour of line i of mesh b: colors[b * cb + 3 i + 0..2] (nullptr: no colours)
  long long cb;
  int color_dot0;
  const int64_t* tri;          // (ntri, 3)
  int ntri, tri_order, tri_dot0;   // tri_order 0: columns 2, 1, 0 (write_obj); 1: 0, 1, 2 (write_obj_with_colors)
  int batch, vblocks, tblocks;     // blocks of vertex lines per mesh, blocks of triangle lines
};

// line `line` of block `blk`: its length, and (out != nullptr) its bytes at out
__device__ __forceinline__ int obj_line(const ObjArgs& a, int blk, int t, char* out) {
  const int nv = a.batch * a.vblocks;
  if (blk < nv) {
    const int b = blk / a.vblocks;
    const long long i = (long long)(blk - b * a.vblocks) * kObjThreads + t;
    if (i >= a.n) return 0;
    const long long vi = a.keep ? a.keep[i] : i;
    const float* p = a.v + b * a.sb + vi * a.sv;
    const float x = p[0], y = p[a.sc], z = p[2LL * a.sc];
    const int64_t* c = a.colors ? a.colors + b * a.cb + 3LL * i : nullptr;
    return out ? omath::vertex_line_write(x, y, z, c, a.color_dot0, out) : omath::vertex_line_len(x, y, z, c, a.color_dot0);
  }
  const long long i = (long long)(blk - nv) * kObjThreads + t;
  if (i >= a.ntri) return 0;
  const int64_t* r = a.tri + 3LL * i;
  const int64_t f0 = a.tri_order ? r[0] : r[2], f2 = a.tri_order ? r[2] : r[0];
  return out ? omath::tri_line_write(f0, r[1], f2, a.tri_dot0, out) : omath::tri_line_len(f0, r[1], f2, a.tri_dot0);
}

// exclusive scan of v over the CTA (blockDim.x a multiple of 32, at most 1024); *total = the CTA's sum
template <typename T>
__device__ __forceinline__ T obj_block_scan(T v, T* total) {
  __shared__ T warp_sum[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  T inc = v;
  for (int d = 1; d < 32; d <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += u;
  }
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    T s = lane < n_warps ? warp_sum[lane] : T(0);
    for (int d = 1; d < 32; d <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += u;
    }
    if (lane < n_warps) warp_sum[lane] = s;     // inclusive warp prefix
  }
  __syncthreads();
  const T before = warp ? warp_sum[warp - 1] : T(0);
  *total = warp_sum[n_warps - 1];
  __syncthreads();                              // warp_sum is reused by the next call
  return before + inc - v;
}

// sums[blk] = bytes of block blk's lines
__global__ void __launch_bounds__(kObjThreads) obj_len_kernel(ObjArgs a, long long* sums) {
  const int len = obj_line(a, blockIdx.x, threadIdx.x, nullptr);
  int total;
  obj_block_scan<int>(len, &total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

constexpr int kObjScanThreads = 1024;

// ws[0] = T; ws[1 + blk]: the block sums in, the block bases out (vertex blocks: byte offset in the output; triangle
// blocks: byte offset in the triangle text).  offsets[b] = first byte of mesh b, offsets[batch] = the total.
__global__ void __launch_bounds__(kObjScanThreads) obj_scan_kernel(int batch, int vblocks, int tblocks, long long* ws, long long* offsets) {
  long long* blocks = ws + 1;
  const int nv = batch * vblocks;
  long long carry = 0, total;
  for (long long j0 = 0; j0 < tblocks; j0 += blockDim.x) {
    const long long j = j0 + threadIdx.x;
    const long long s = j < tblocks ? blocks[nv + j] : 0;
    const long long ex = obj_block_scan<long long>(s, &total);
    if (j < tblocks) blocks[nv + j] = carry + ex;
    carry += total;
  }
  const long long tri_bytes = carry;
  carry = 0;
  for (long long j0 = 0; j0 < nv; j0 += blockDim.x) {
    const long long j = j0 + threadIdx.x;
    const long long s = j < nv ? blocks[j] + (j % vblocks == vblocks - 1 ? tri_bytes : 0) : 0;
    const long long ex = obj_block_scan<long long>(s, &total);
    if (j < nv) {
      blocks[j] = carry + ex;
      if (j % vblocks == 0) offsets[j / vblocks] = carry + ex;
    }
    carry += total;
  }
  if (vblocks == 0)                             // no vertex line: every mesh is the triangle text alone
    for (int b = threadIdx.x; b < batch; b += blockDim.x) offsets[b] = b * tri_bytes;
  if (threadIdx.x == 0) {
    ws[0] = tri_bytes;
    offsets[batch] = vblocks ? carry : batch * tri_bytes;
  }
}

__global__ void __launch_bounds__(kObjThreads) obj_write_kernel(ObjArgs a, const long long* ws, const long long* offsets, char* out,
                                                                long long out_bytes) {
  const int len = obj_line(a, blockIdx.x, threadIdx.x, nullptr);
  int total;
  const int local = obj_block_scan<int>(len, &total);
  if (!len) return;
  const int nv = a.batch * a.vblocks;
  long long at = ws[1 + blockIdx.x] + local;
  if ((int)blockIdx.x >= nv) at += offsets[1] - ws[0];           // mesh 0's triangle text
  if (at < 0 || at + len > out_bytes) return;
  obj_line(a, blockIdx.x, threadIdx.x, out + at);
}

// grid (x, batch - 1): mesh 0's triangle text (T = ws[0] bytes, ending at offsets[1]) into mesh 1 + blockIdx.y
__global__ void __launch_bounds__(kObjThreads) obj_copy_kernel(const long long* ws, const long long* offsets, char* out, long long out_bytes) {
  const long long n = ws[0];
  const long long src = offsets[1] - n, dst = offsets[blockIdx.y + 2] - n;
  if (src < 0 || dst < 0 || src + n > out_bytes || dst + n > out_bytes) return;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[dst + i] = out[src + i];
}

}  // namespace syn
