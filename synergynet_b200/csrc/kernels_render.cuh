// Sim3DR on the GPU (SURVEY.md section 8 row f2): vertex normals, per-vertex lighting and z-buffer rasterisation of a
// BATCH of meshes that share one triangle list -- the consumer of the dense vertices `syn_reconstruct_image` leaves in
// HBM, which it reads in place (plane-major (B,3,N) or the reference's interleaved (N,3): element strides).
//
// The reference (Sim3DR/lib/rasterize_kernel.cpp) is one serial loop over triangles with a read-modify-write depth
// buffer.  Its result per pixel is "the triangle of greatest interpolated depth, first one on ties" (strict `>` test,
// :241), which is order-free once written as the maximum of a 64-bit key (render_math.h):
//   pass 1  raster_depth_kernel    one thread per (mesh, triangle); atomicMax of the key over the pixels of its bounding
//                                  box; bounding boxes above 64 pixels are walked by the whole warp
//   pass 2  raster_resolve_kernel  one thread per pixel: the LAST mesh that covers it wins (the reference draws meshes
//                                  one after the other onto the same image, utils/render.py:41-45, each with a fresh
//                                  depth buffer), barycentric weights recomputed from the winning triangle, colours
//                                  interpolated and written as the reference's (unsigned char) expression.
// The frame axis (syn_render_frames_plan / syn_rasterize_frames: the meshes of N frames, frame f owning a contiguous
// range of them) keeps the same per-pixel arithmetic, but a mesh's keys live only in its pixel box -- the union of its
// triangles' clamped boxes -- so the workspace is the sum of the box areas instead of B x H x W:
//   pass 0  mesh_box_kernel + mesh_box_scan_kernel   the boxes, and their areas' exclusive prefix sum (key offsets)
//   pass 1  raster_depth_kernel                      unchanged, each key addressed inside its mesh's box
//   pass 2  raster_resolve_frames_kernel             one thread per (frame, pixel) over that frame's meshes only
// and the overlay blend of utils/render.py:45 (cv2.addWeighted) runs as add_weighted_u8_kernel.
// Vertex normals are the sum of the incident face normals IN TRIANGLE ORDER (:189-199): a per-vertex incidence list,
// ascending by construction (syn_mesh_incidence_host), replaces the scatter loop, so the float sums associate exactly
// as the reference's do.  All arithmetic comes from render_math.h (no FMA contraction): normals and rasterisation are
// bit-exact against the reference; lighting is numpy float32 arithmetic except powf (see rmath::powi).
#pragma once
#include "common.cuh"
#include "render_math.h"

namespace syn {

struct MeshView {        // B meshes over one topology
  const float* v;        // coordinate k of vertex i of mesh b: v[b * sb + i * sv + k * sc]
  long long sb;
  int sv, sc;
  int nver, batch;
};

__device__ __forceinline__ void load_vertex(const MeshView& m, int b, int i, float* p) {
  const float* q = m.v + (size_t)b * m.sb + (size_t)i * m.sv;
  p[0] = __ldg(q);
  p[1] = __ldg(q + m.sc);
  p[2] = __ldg(q + 2 * m.sc);
}

// ---- normals -------------------------------------------------------------------------------------------------------
__global__ void tri_normal_kernel(MeshView m, const int32_t* __restrict__ tri, int ntri, float* __restrict__ tn) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= ntri) return;
  const int i0 = __ldg(tri + 3 * i), i1 = __ldg(tri + 3 * i + 1), i2 = __ldg(tri + 3 * i + 2);
  float n[3] = {0.f, 0.f, 0.f};
  if ((unsigned)i0 < (unsigned)m.nver && (unsigned)i1 < (unsigned)m.nver && (unsigned)i2 < (unsigned)m.nver) {
    float p0[3], p1[3], p2[3];
    load_vertex(m, b, i0, p0);
    load_vertex(m, b, i1, p1);
    load_vertex(m, b, i2, p2);
    rmath::tri_normal(p0, p1, p2, n);
  }
  float* o = tn + ((size_t)b * ntri + i) * 3;
  o[0] = n[0]; o[1] = n[1]; o[2] = n[2];
}

// inc_start (nver + 1), inc_tri (3 * ntri): triangles incident to each vertex, ascending, one entry per corner
__global__ void vertex_normal_kernel(int nver, int ntri, const float* __restrict__ tn, const int32_t* __restrict__ inc_start,
                                     const int32_t* __restrict__ inc_tri, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= nver) return;
  float n[3] = {0.f, 0.f, 0.f};
  const int e0 = __ldg(inc_start + i), e1 = __ldg(inc_start + i + 1);
  const float* base = tn + (size_t)b * ntri * 3;
  for (int e = e0; e < e1; ++e) {
    const float* t = base + (size_t)__ldg(inc_tri + e) * 3;
    n[0] = rmath::add(n[0], t[0]);
    n[1] = rmath::add(n[1], t[1]);
    n[2] = rmath::add(n[2], t[2]);
  }
  rmath::normalize3(n);
  float* o = out + ((size_t)b * nver + i) * 3;
  o[0] = n[0]; o[1] = n[1]; o[2] = n[2];
}

// ---- lighting ------------------------------------------------------------------------------------------------------
// per-mesh coordinate extremes as order-preserving unsigneds; stats[b][0..2] = max of ~ordered(x) (i.e. the minimum),
// stats[b][3..5] = max of ordered(x); zero-initialised by the caller (cudaMemsetAsync)
__global__ void mesh_extent_kernel(MeshView m, unsigned* __restrict__ stats) {
  const int b = blockIdx.y;
  unsigned lo[3] = {0u, 0u, 0u}, hi[3] = {0u, 0u, 0u};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m.nver; i += gridDim.x * blockDim.x) {
    float p[3];
    load_vertex(m, b, i, p);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const unsigned o = rmath::float_ordered(p[k]);
      lo[k] = max(lo[k], ~o);
      hi[k] = max(hi[k], o);
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    lo[k] = __reduce_max_sync(0xFFFFFFFFu, lo[k]);
    hi[k] = __reduce_max_sync(0xFFFFFFFFu, hi[k]);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      atomicMax(stats + b * 6 + k, lo[k]);
      atomicMax(stats + b * 6 + 3 + k, hi[k]);
    }
  }
}

// light[b][i][0..2] (Sim3DR/lighting.py:37-66); with a texture (nver,3): colours = texture * light (:74)
__global__ void vertex_light_kernel(MeshView m, const float* __restrict__ normals, const unsigned* __restrict__ stats,
                                    rmath::LightCfg cfg, const float* __restrict__ texture, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= m.nver) return;
  rmath::NormStats s;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    s.mn[k] = rmath::ordered_float(~stats[b * 6 + k]);
    s.mx[k] = rmath::ordered_float(stats[b * 6 + 3 + k]);
  }
  float p[3], l[3];
  load_vertex(m, b, i, p);
  const float* n = normals + ((size_t)b * m.nver + i) * 3;
  const float nn[3] = {n[0], n[1], n[2]};
  rmath::vertex_light(p, nn, s, cfg, l);
  float* o = out + ((size_t)b * m.nver + i) * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) o[k] = texture ? rmath::mul(__ldg(texture + (size_t)i * 3 + k), l[k]) : l[k];
}

// ---- rasterisation -------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool load_tri(const MeshView& m, int b, const int32_t* __restrict__ tri, int i, int w, int h,
                                         rmath::TriSetup& t) {
  const int i0 = __ldg(tri + 3 * i), i1 = __ldg(tri + 3 * i + 1), i2 = __ldg(tri + 3 * i + 2);
  if ((unsigned)i0 >= (unsigned)m.nver || (unsigned)i1 >= (unsigned)m.nver || (unsigned)i2 >= (unsigned)m.nver) return false;
  float p[3];
  load_vertex(m, b, i0, p); t.x0 = p[0]; t.y0 = p[1]; t.z0 = p[2];
  load_vertex(m, b, i1, p); t.x1 = p[0]; t.y1 = p[1]; t.z1 = p[2];
  load_vertex(m, b, i2, p); t.x2 = p[0]; t.y2 = p[1]; t.z2 = p[2];
  return rmath::tri_setup(t, w, h);
}

constexpr int kRasterSmallBox = 64;     // bounding boxes up to this many pixels are walked by the owning thread

// keys: zero = empty.  BOXED = false (syn_rasterize): the (B, h, w) canvas of every mesh; boxes / key_off are not read.
// BOXED = true (the frame axis): mesh b keys only its pixel box boxes[b] = (x0, y0, x1, y1), in the box-many slots at
// keys + key_off[b] (mesh_box_kernel / mesh_box_scan_kernel plan them).  The canvas instantiation is the one-image kernel
// as it was before the frame axis existed, instruction for instruction.  One thread per (mesh, triangle).
template <bool BOXED>
__global__ void raster_depth_kernel(MeshView m, const int32_t* __restrict__ tri, int ntri, int w, int h,
                                    unsigned long long* __restrict__ keys, const int4* __restrict__ boxes,
                                    const long long* __restrict__ key_off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31;
  rmath::TriSetup t;
  const bool live = (i < ntri) && load_tri(m, b, tri, i, w, h, t);
  unsigned long long* kb = keys + (size_t)b * w * h;     // key of pixel (x, y): kb[y * ks + x]
  int ks = w;
  if constexpr (BOXED) {                                  // the box's row-major slots, addressed from the canvas origin
    const int4 q = boxes[b];
    ks = q.z - q.x + 1;
    kb = keys + key_off[b] - ((long long)q.y * ks + q.x);
  }
  int bw = 0, area = 0;
  if (live) { bw = t.xmax - t.xmin + 1; area = bw * (t.ymax - t.ymin + 1); }
  if (live && area <= kRasterSmallBox) {
    for (int y = t.ymin; y <= t.ymax; ++y)
      for (int x = t.xmin; x <= t.xmax; ++x) {
        uint64_t key;
        if (rmath::pixel_key(t, (uint32_t)i, x, y, key)) atomicMax(kb + (size_t)y * ks + x, (unsigned long long)key);
      }
  }
  // large boxes: the warp walks them together, one triangle at a time
  unsigned big = __ballot_sync(0xFFFFFFFFu, live && area > kRasterSmallBox);
  while (big) {
    const int src = __ffs(big) - 1;
    big &= big - 1;
    rmath::TriSetup s;
    s.x0 = __shfl_sync(0xFFFFFFFFu, t.x0, src); s.y0 = __shfl_sync(0xFFFFFFFFu, t.y0, src); s.z0 = __shfl_sync(0xFFFFFFFFu, t.z0, src);
    s.x1 = __shfl_sync(0xFFFFFFFFu, t.x1, src); s.y1 = __shfl_sync(0xFFFFFFFFu, t.y1, src); s.z1 = __shfl_sync(0xFFFFFFFFu, t.z1, src);
    s.x2 = __shfl_sync(0xFFFFFFFFu, t.x2, src); s.y2 = __shfl_sync(0xFFFFFFFFu, t.y2, src); s.z2 = __shfl_sync(0xFFFFFFFFu, t.z2, src);
    s.xmin = __shfl_sync(0xFFFFFFFFu, t.xmin, src); s.ymin = __shfl_sync(0xFFFFFFFFu, t.ymin, src);
    const int sbw = __shfl_sync(0xFFFFFFFFu, bw, src), sarea = __shfl_sync(0xFFFFFFFFu, area, src);
    const int si = __shfl_sync(0xFFFFFFFFu, i, src);
    for (int q = lane; q < sarea; q += 32) {
      const int y = s.ymin + q / sbw, x = s.xmin + q % sbw;
      uint64_t key;
      if (rmath::pixel_key(s, (uint32_t)si, x, y, key)) atomicMax(kb + (size_t)y * ks + x, (unsigned long long)key);
    }
  }
}

// The winning triangle `key` of mesh b at pixel (x, y): barycentric weights recomputed from its vertices, colours
// interpolated, written as the reference's (unsigned char) expression over the pixel's bytes (:239-255).  The pixel is
// row `row`, column x of the (h, w, c) images src and dst (row = y, or h - 1 - y when drawing upside down).
__device__ __forceinline__ void shade_pixel(const MeshView& m, int b, const int32_t* __restrict__ tri, const float* __restrict__ colors,
                                            int c, int w, int x, int y, int row, unsigned long long key, float alpha,
                                            const unsigned char* src, unsigned char* dst) {
  const int i = (int)rmath::key_tri(key);
  const int i0 = __ldg(tri + 3 * i), i1 = __ldg(tri + 3 * i + 1), i2 = __ldg(tri + 3 * i + 2);
  float p0[3], p1[3], p2[3];
  load_vertex(m, b, i0, p0);
  load_vertex(m, b, i1, p1);
  load_vertex(m, b, i2, p2);
  const rmath::Bary bw = rmath::barycentric((float)x, (float)y, p0[0], p0[1], p1[0], p1[1], p2[0], p2[1]);
  const float* cb = colors + (size_t)b * m.nver * c;
  const size_t at = ((size_t)row * w + x) * c;
  src += at;
  dst += at;
  for (int k = 0; k < c; ++k) {
    const float pc = rmath::interp(bw, __ldg(cb + (size_t)i0 * c + k), __ldg(cb + (size_t)i1 * c + k), __ldg(cb + (size_t)i2 * c + k));
    dst[k] = rmath::blend_u8(src[k], alpha, pc);
  }
}

// One thread per pixel.  image (h, w, c) uint8 is updated in place; depth_out (optional, (B,h,w) fp32) receives the
// reference's depth buffer of every mesh (-1e8 where nothing was drawn).
__global__ void raster_resolve_kernel(MeshView m, const int32_t* __restrict__ tri, const float* __restrict__ colors, int c,
                                      int w, int h, float alpha, int reverse, const unsigned long long* __restrict__ keys,
                                      unsigned char* __restrict__ image, float* __restrict__ depth_out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const size_t pix = (size_t)y * w + x;
  bool drawn = false;
  for (int b = m.batch - 1; b >= 0; --b) {
    const unsigned long long key = keys[(size_t)b * w * h + pix];
    if (depth_out) depth_out[(size_t)b * w * h + pix] = key ? rmath::key_depth(key) : rmath::kDepthInit;
    if (key == 0ull || drawn) continue;
    drawn = true;                       // later meshes overwrite earlier ones (alpha == 1)
    shade_pixel(m, b, tri, colors, c, w, x, y, reverse ? h - 1 - y : y, key, alpha, image, image);
    if (!depth_out) break;
  }
}

// ---- the frame axis: meshes grouped by frame, keys in per-mesh boxes ---------------------------------------------------------
// Pass 0a: acc (M,4) int32, set to 0x7F7F7F7F bytes by the caller, receives min x0, min y0, min -x1, min -y1 over the
// triangles load_tri draws (the same skips: bad indices, boxes empty after clamping).  One thread per (mesh, triangle).
__global__ void mesh_box_kernel(MeshView m, const int32_t* __restrict__ tri, int ntri, int w, int h, int* __restrict__ acc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  rmath::TriSetup t;
  const bool live = (i < ntri) && load_tri(m, b, tri, i, w, h, t);
  const int big = 0x7F7F7F7F;
  const int v[4] = {live ? t.xmin : big, live ? t.ymin : big, live ? -t.xmax : big, live ? -t.ymax : big};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = __reduce_min_sync(0xFFFFFFFFu, v[k]);
    if ((threadIdx.x & 31) == 0 && r != big) atomicMin(acc + 4 * b + k, r);
  }
}

// Pass 0b, one CTA: acc -> the boxes (x0, y0, x1, y1) in place (an empty mesh: (0, 0, -1, -1), area 0) and key_off (M+1)
// = the exclusive prefix sum of the box areas; key_off[M] is the key count of the whole call.
constexpr int kBoxScanThreads = 1024;
__global__ void __launch_bounds__(kBoxScanThreads) mesh_box_scan_kernel(int nmesh, int* __restrict__ acc, long long* __restrict__ key_off) {
  __shared__ long long part[kBoxScanThreads];
  const int tid = threadIdx.x, per = (nmesh + kBoxScanThreads - 1) / kBoxScanThreads;
  const int j0 = min(tid * per, nmesh), j1 = min(j0 + per, nmesh);
  long long s = 0;
  for (int j = j0; j < j1; ++j) {
    int* q = acc + 4 * j;
    rmath::PixBox bx;
    bx.x0 = q[0]; bx.y0 = q[1]; bx.x1 = -q[2]; bx.y1 = -q[3];
    if (bx.x1 < bx.x0 || bx.y1 < bx.y0) bx = rmath::pix_box_empty();
    q[0] = bx.x0; q[1] = bx.y0; q[2] = bx.x1; q[3] = bx.y1;
    s += rmath::pix_box_area(bx);
  }
  part[tid] = s;
  __syncthreads();
  for (int d = 1; d < kBoxScanThreads; d <<= 1) {        // inclusive scan of the per-thread sums
    const long long add = tid >= d ? part[tid - d] : 0ll;
    __syncthreads();
    part[tid] += add;
    __syncthreads();
  }
  long long base = part[tid] - s;
  for (int j = j0; j < j1; ++j) {
    key_off[j] = base;
    const int* q = acc + 4 * j;
    rmath::PixBox bx;
    bx.x0 = q[0]; bx.y0 = q[1]; bx.x1 = q[2]; bx.y1 = q[3];
    base += rmath::pix_box_area(bx);
  }
  if (tid == kBoxScanThreads - 1) key_off[nmesh] = part[tid];
}

// Pass 2 of the frame axis: one thread per (frame, pixel), grid.z = frame.  Frame f's meshes [mesh_start[f],
// mesh_start[f+1]) are walked last to first; the first whose box holds the pixel and whose key there is set is drawn (alpha
// = 1, so it overwrites whatever the earlier meshes drew), as raster_resolve_kernel draws a one-image batch.  src and dst
// are (N, h, w, c) stacks and may be the same buffer; an undrawn pixel is copied.
__global__ void raster_resolve_frames_kernel(MeshView m, const int32_t* __restrict__ tri, const float* __restrict__ colors, int c,
                                             int w, int h, const int32_t* __restrict__ mesh_start, const int4* __restrict__ boxes,
                                             const long long* __restrict__ key_off, const unsigned long long* __restrict__ keys,
                                             const unsigned char* src, unsigned char* dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= w || y >= h) return;
  const size_t pix = (((size_t)f * h + y) * w + x) * c;
  const int b0 = mesh_start[f];
  for (int b = mesh_start[f + 1] - 1; b >= b0; --b) {
    const int4 q = boxes[b];
    if (x < q.x || x > q.z || y < q.y || y > q.w) continue;
    rmath::PixBox box;
    box.x0 = q.x; box.y0 = q.y; box.x1 = q.z; box.y1 = q.w;
    const unsigned long long key = keys[key_off[b] + rmath::pix_box_slot(box, x, y)];
    if (key == 0ull) continue;
    const size_t frame = (size_t)f * h * w * c;
    shade_pixel(m, b, tri, colors, c, w, x, y, y, key, 1.0f, src + frame, dst + frame);
    return;
  }
  if (src != dst)
    for (int k = 0; k < c; ++k) dst[pix + k] = src[pix + k];
}

// out = cv2.addWeighted(a, 1 - alpha, b, alpha, 0) over n bytes (rmath::add_weighted_u8).  vec: n % 16 == 0 and all three
// pointers 16-byte aligned, sixteen bytes per load.  out may be a or b.
__global__ void add_weighted_u8_kernel(const unsigned char* a, const unsigned char* b, double alpha, unsigned char* out, long long n,
                                       int vec) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (vec) {
    union V { uint4 v; unsigned char c[16]; };
    for (long long q = t; q < n / 16; q += stride) {
      V va, vb, vo;
      va.v = reinterpret_cast<const uint4*>(a)[q];
      vb.v = reinterpret_cast<const uint4*>(b)[q];
#pragma unroll
      for (int k = 0; k < 16; ++k) vo.c[k] = rmath::add_weighted_u8(va.c[k], vb.c[k], alpha);
      reinterpret_cast<uint4*>(out)[q] = vo.v;
    }
  } else {
    for (long long i = t; i < n; i += stride) out[i] = rmath::add_weighted_u8(a[i], b[i], alpha);
  }
}

// ---- NMS (SURVEY.md section 8 row f3: FaceBoxes/utils/nms/cpu_nms.pyx:17-68, py_cpu_nms.py:10-38) -----------------------
// dets (n, 5) fp32 [x1 y1 x2 y2 score], ALREADY in the order the greedy loop visits them (descending score).
// mask[i][j / 64] bit (j % 64) = box j (> i) is suppressed by box i.  ge != 0: `ovr >= thresh` in double (cpu_nms.pyx:65,
// thresh is a C double there); ge == 0: py_cpu_nms keeps `ovr <= thresh` in float32, i.e. suppresses on `!(ovr <= thresh)`,
// so a NaN overlap (a box with a NaN or +-inf-minus-inf coordinate) is suppressed there and kept by cpu_nms.
// Segmented (syn_nms_batch): n_dev != nullptr, grid.z = frame.  Frame f owns rows [f * n, (f + 1) * n) of dets and a mask
// block sized for n rows, of which its own count n_dev[f] <= n are valid and laid out with ITS OWN word count, so the
// bits (and the scan below) are those of a one-image call with that count.  The grid is sized for n.
__device__ __forceinline__ int nms_segment(const int32_t* n_dev, int& n, int fr) {      // -> rows per frame; n = the frame's count
  const int cap = n;
  if (n_dev) n = max(0, min(n_dev[fr], cap));
  return cap;
}

__global__ void nms_mask_kernel(const float* __restrict__ dets, int n, double thresh, int ge, unsigned long long* __restrict__ mask,
                                const int32_t* __restrict__ n_dev) {
  {
    const int cap = nms_segment(n_dev, n, blockIdx.z);
    dets += (size_t)blockIdx.z * cap * 5;
    mask += (size_t)blockIdx.z * cap * ((cap + 63) / 64);
  }
  const int words = (n + 63) / 64;
  const int i = blockIdx.y * blockDim.y + threadIdx.y, wj = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || wj >= words) return;
  unsigned long long bits = 0ull;
  const int j0 = wj * 64;
  if (j0 + 63 > i) {
    const float a[4] = {dets[i * 5], dets[i * 5 + 1], dets[i * 5 + 2], dets[i * 5 + 3]};
    const float area_a = rmath::box_area(a[0], a[1], a[2], a[3]);
    const float thr_f = (float)thresh;
    for (int jj = 0; jj < 64; ++jj) {
      const int j = j0 + jj;
      if (j <= i || j >= n) continue;
      const float bq[4] = {dets[j * 5], dets[j * 5 + 1], dets[j * 5 + 2], dets[j * 5 + 3]};
      const float ovr = rmath::box_overlap(a, area_a, bq, rmath::box_area(bq[0], bq[1], bq[2], bq[3]));
      const bool sup = ge ? ((double)ovr >= thresh) : !(ovr <= thr_f);
      if (sup) bits |= 1ull << jj;
    }
  }
  mask[(size_t)i * words + wj] = bits;
}

// The greedy scan itself, 64 boxes (one mask word) at a time, one CTA:
//   A  warp 0 resolves the block: the 64 x 64 diagonal of the bit matrix sits in two registers per lane, box b of the
//      block survives iff its bit in `removed` is still clear when its turn comes, and then its diagonal word joins the
//      running word -- 64 shuffle steps, no memory traffic;
//   B  all threads OR the rows of the boxes that survived into `removed` for the words to the right of the block, four
//      independent loads in flight per thread (a box-by-box scan would pay one dependent L2 round trip per kept box).
// keep (n) int32 receives the kept indices in visiting order, *n_keep their number: the serial greedy list, exactly.
// Segmented: one CTA per frame (blockIdx.x), frame f's keep list at keep + f * n and its count at n_keep[f].
constexpr int kNmsScanThreads = 1024;
__global__ void __launch_bounds__(kNmsScanThreads) nms_scan_kernel(const unsigned long long* __restrict__ mask, int n,
                                                                   int32_t* __restrict__ keep, int32_t* __restrict__ n_keep,
                                                                   const int32_t* __restrict__ n_dev) {
  extern __shared__ unsigned long long removed[];          // words entries
  __shared__ int rows[64];
  __shared__ int n_rows, total;
  {
    const int cap = nms_segment(n_dev, n, blockIdx.x);
    mask += (size_t)blockIdx.x * cap * ((cap + 63) / 64);
    keep += (size_t)blockIdx.x * cap;
    n_keep += blockIdx.x;
  }
  const int words = (n + 63) / 64, tid = threadIdx.x, lane = tid & 31;
  for (int wq = tid; wq < words; wq += kNmsScanThreads) removed[wq] = 0ull;
  if (tid == 0) total = 0;
  __syncthreads();
  for (int blk = 0; blk < words; ++blk) {
    const int base = blk * 64, cnt = min(64, n - base);
    if (tid < 32) {
      const unsigned long long d0 = (lane < cnt) ? mask[(size_t)(base + lane) * words + blk] : 0ull;
      const unsigned long long d1 = (lane + 32 < cnt) ? mask[(size_t)(base + 32 + lane) * words + blk] : 0ull;
      unsigned long long cur = removed[blk], keepbits = 0ull;
      for (int b = 0; b < cnt; ++b) {
        const unsigned long long db = __shfl_sync(0xFFFFFFFFu, (b < 32) ? d0 : d1, b & 31);
        if (!((cur >> b) & 1ull)) { keepbits |= 1ull << b; cur |= db; }
      }
      const int t0 = total;
#pragma unroll
      for (int hlf = 0; hlf < 2; ++hlf) {
        const int b = lane + 32 * hlf;
        if ((keepbits >> b) & 1ull) {
          const int pos = __popcll(keepbits & ((1ull << b) - 1ull));
          keep[t0 + pos] = base + b;
          rows[pos] = base + b;
        }
      }
      __syncwarp();
      if (lane == 0) { n_rows = __popcll(keepbits); total = t0 + __popcll(keepbits); }
    }
    __syncthreads();
    const int nr = n_rows, rem = words - blk - 1;
    const int pairs = nr * rem;
    for (int p0 = tid; p0 < pairs; p0 += 4 * kNmsScanThreads) {
      unsigned long long v[4];
      int wq[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int p = p0 + u * kNmsScanThreads;
        v[u] = 0ull; wq[u] = 0;
        if (p < pairs) {
          const int r = p / rem;
          wq[u] = blk + 1 + (p - r * rem);
          v[u] = mask[(size_t)rows[r] * words + wq[u]];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (v[u]) atomicOr(&removed[wq[u]], v[u]);
    }
    __syncthreads();
  }
  if (tid == 0) *n_keep = total;
}

}  // namespace syn
