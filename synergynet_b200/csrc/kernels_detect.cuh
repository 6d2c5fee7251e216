// FaceBoxes post-processing on the GPU (SURVEY.md section 8 row f3): prior boxes, box decode, score filter, top-k ordering.
// Replaces FaceBoxes/FaceBoxes.py:98-120 (+ utils/prior_box.py:12-48, utils/box_utils.py:177-195); the greedy NMS that
// follows (:122-127) is nms_mask_kernel / nms_scan_kernel in kernels_render.cuh.
//
// Prior boxes are a closed form of the prior index (no table in memory): the reference builds them in Python doubles
// and rounds to float32 once (`torch.Tensor(anchors)`), which is what prior_of() does.  The decode is float32 torch
// arithmetic, one rounding per operation; only exp() has no bit pattern to match (torch's CPU kernel is a Sleef
// vector exp), so boxes agree to ~1e-7 relative and the ordering / NMS index work is exact given equal scores.
#pragma once
#include "common.cuh"
#include "render_math.h"

namespace syn {

// cfg of FaceBoxes/utils/config.py: min_sizes [[32, 64, 128], [256], [512]], steps [32, 64, 128], variance [0.1, 0.2]
__host__ __device__ inline int fb_cells(int size, int step) { return (size + step - 1) / step; }      // ceil(size / step), prior_box.py:19
__host__ __device__ inline int faceboxes_num_priors(int h, int w) {
  return 21 * fb_cells(h, 32) * fb_cells(w, 32) + fb_cells(h, 64) * fb_cells(w, 64) + fb_cells(h, 128) * fb_cells(w, 128);
}

// prior `idx` -> (cx, cy, s_kx, s_ky), the order of prior_box.py:23-43: level, row i, column j, then 16 + 4 + 1 anchors
__device__ inline void prior_of(int idx, int h, int w, float* p) {
  const int n0 = 21 * fb_cells(h, 32) * fb_cells(w, 32), n1 = fb_cells(h, 64) * fb_cells(w, 64);
  double cx, cy, ms, step;
  if (idx < n0) {
    const int cell = idx / 21, a = idx - cell * 21, cols = fb_cells(w, 32);
    const int i = cell / cols, j = cell - i * cols;
    step = 32.0;
    if (a < 16) { ms = 32.0; cx = j + 0.25 * (a & 3); cy = i + 0.25 * (a >> 2); }
    else if (a < 20) { ms = 64.0; cx = j + 0.5 * ((a - 16) & 1); cy = i + 0.5 * ((a - 16) >> 1); }
    else { ms = 128.0; cx = j + 0.5; cy = i + 0.5; }
  } else if (idx < n0 + n1) {
    const int cell = idx - n0, cols = fb_cells(w, 64);
    step = 64.0; ms = 256.0; cx = cell % cols + 0.5; cy = cell / cols + 0.5;
  } else {
    const int cell = idx - n0 - n1, cols = fb_cells(w, 128);
    step = 128.0; ms = 512.0; cx = cell % cols + 0.5; cy = cell / cols + 0.5;
  }
  p[0] = (float)(cx * step / (double)w);
  p[1] = (float)(cy * step / (double)h);
  p[2] = (float)(ms / (double)w);
  p[3] = (float)(ms / (double)h);
}

// Per-frame parameters of one decode launch (grid.y = frame), passed by value: one image, a stack of equal frames or a
// list of images of any sizes.  Frame f's priors are rows p0 .. p0 + np - 1 of loc / conf; its candidate count sits at
// cand[c0] and its candidate indices at cand[i0 ..]; box_scale_w / _h are the network input's width / height
// (FaceBoxes.py:101), scale the shrink factor (:104).
constexpr int kDecodeMaxFrames = SYN_FB_MAX_FRAMES;
struct FbDecodeFrames {
  int h[kDecodeMaxFrames], w[kDecodeMaxFrames], np[kDecodeMaxFrames], p0[kDecodeMaxFrames], c0[kDecodeMaxFrames], i0[kDecodeMaxFrames];
  float box_scale_w[kDecodeMaxFrames], box_scale_h[kDecodeMaxFrames], scale[kDecodeMaxFrames];
};

// cand[c0] = number of priors whose face score conf[:, 1] exceeds the threshold (FaceBoxes.py:112), cand[i0..] = their
// indices.  grid.y = frame, the grid sized for the frame with the most priors.
__global__ void faceboxes_select_kernel(const float* __restrict__ conf, const __grid_constant__ FbDecodeFrames t, float thresh,
                                        int32_t* __restrict__ cand) {
  const int f = blockIdx.y, np = t.np[f];
  conf += (size_t)t.p0[f] * 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < np && conf[2 * i + 1] > thresh) cand[t.i0[f] + atomicAdd(cand + t.c0[f], 1)] = i;
}

// Rank of every candidate in descending score order (ties: the higher prior index first = a stable ascending argsort
// read backwards, :117), the first top_k decoded and written in that order as rows [x1 y1 x2 y2 score] (:121).
// grid.y = frame, which builds its own priors and ranks its own candidates into its own (top_k,5) block and count.
__global__ void faceboxes_rank_decode_kernel(const float* __restrict__ loc, const float* __restrict__ conf,
                                             const __grid_constant__ FbDecodeFrames t, int top_k, const int32_t* __restrict__ cand,
                                             float* __restrict__ dets, int32_t* __restrict__ n_dets) {
  const int fr = blockIdx.y, h = t.h[fr], w = t.w[fr];
  const float box_scale_w = t.box_scale_w[fr], box_scale_h = t.box_scale_h[fr], scale = t.scale[fr];
  loc += (size_t)t.p0[fr] * 4; conf += (size_t)t.p0[fr] * 2; dets += (size_t)fr * top_k * 5; n_dets += fr;
  const int n = cand[t.c0[fr]];
  cand += t.i0[fr] - 1;                                                   // cand[1 + c] = candidate c, as below
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_dets = min(n, top_k);
  if ((int)(blockIdx.x * blockDim.x) >= n) return;                       // whole CTA: the grid is sized for every prior
  __shared__ float ss[512];
  __shared__ int si[512];
  {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = c < n;
    const int i = live ? cand[1 + c] : 0;
    const float s = live ? conf[2 * i + 1] : 0.f;
    int rank = 0;
    for (int t0 = 0; t0 < n; t0 += 512) {                                 // all candidates, 512 at a time through shared memory
      const int tn = min(512, n - t0);
      for (int e = threadIdx.x; e < tn; e += blockDim.x) {
        const int j = cand[1 + t0 + e];
        si[e] = j;
        ss[e] = conf[2 * j + 1];
      }
      __syncthreads();
      if (live)
        for (int q = 0; q < tn; ++q) rank += (ss[q] > s) || (ss[q] == s && si[q] > i);
      __syncthreads();
    }
    if (!live) return;
    if (rank >= top_k) return;
    float p[4];
    prior_of(i, h, w, p);
    const float* l = loc + 4 * (size_t)i;
    using namespace rmath;
    const float cx = add(p[0], mul(mul(l[0], 0.1f), p[2])), cy = add(p[1], mul(mul(l[1], 0.1f), p[3]));       // box_utils.py:191
    const float bw = mul(p[2], expf(mul(l[2], 0.2f))), bh = mul(p[3], expf(mul(l[3], 0.2f)));                  // :192
    const float x1 = sub(cx, dvd(bw, 2.0f)), y1 = sub(cy, dvd(bh, 2.0f));                                       // :193
    const float x2 = add(bw, x1), y2 = add(bh, y1);                                                             // :194
    float* o = dets + 5 * (size_t)rank;
    o[0] = dvd(mul(x1, box_scale_w), scale);                                                                    // FaceBoxes.py:104
    o[1] = dvd(mul(y1, box_scale_h), scale);
    o[2] = dvd(mul(x2, box_scale_w), scale);
    o[3] = dvd(mul(y2, box_scale_h), scale);
    o[4] = s;
  }
}

}  // namespace syn

// ---- the detector network (FaceBoxes/models/faceboxes.py:8-150) -------------------------------------------------------
// 33 small convolutions on one image of arbitrary size (0.7 GMAC at 720 x 1080), or on a stack of equally sized frames.  A first, plain H100 path: fp32 FMA on
// CUDA cores as a shared-memory-tiled implicit GEMM (M = output pixels, N = output channels, K = kh*kw*cin), BatchNorm
// folded into weights and bias on the host in float64, activation and the channel concatenations fused into the store
// (every layer writes its slice of the NHWC tensor the next layer reads).  NHWC is also how the image arrives (H,W,3
// BGR uint8): the mean subtraction of FaceBoxes.py:92 happens in the first layer's gather.
namespace syn {

// The frame axis: images of any sizes, every map packed back to back (frame f's pixels follow frame f-1's).  One FbLevel per
// frame and map size of the network (image, conv1, pool1, conv2, the three detection sources and the heads' view of
// them), built on the host per call and uploaded in one copy.
struct FbLevel {
  int pix0;                // first pixel of this frame in the packed map = sum of h * w over earlier frames
  int h, w;                // this frame's map size
  int prior0;              // detection sources: first prior of this source in the packed (sum P) prior axis
  int ppp;                 // the loc / conf heads' view of a source: its priors per pixel (21 or 1); 0 for every other map
};

struct FbConvArgs {
  const float* x;          // NHWC input (h, w, cin_stride channels per pixel; this layer reads channels [cin_off, cin_off + cin))
  const uint8_t* x_u8;     // first layer: raw image (h, w, 3); value = (float)u8 - mean[c]
  const float* wk;         // [K = kh*kw*cin][cout] fp32, BN scale folded
  const float* bias;       // [cout]
  float* y;                // NHWC output, cout_stride channels per pixel, written at channel offset cout_off
  int h, w, cin, cin_stride, cin_off;
  int ho, wo, cout, cout_stride, cout_off;
  int k, stride, pad;
  int act;                 // 0 linear, 1 ReLU, 2 CReLU: channel c gets relu(v), channel c + cout gets relu(-v)  (faceboxes.py:60-64)
  float mean[3];
  // frame axis (FRAMES instantiations only): the packed maps of `frames` images of any sizes; gin / gout: the per-frame
  // geometry of this layer's input and output map.  Keep this layout (no field in the padding after `frames`): the
  // one-image instantiations' machine code depends on it.
  int frames;
  const FbLevel* gin;
  const FbLevel* gout;
};

// Frame axis: rows of the GEMM = pixels of the packed output map
__device__ __forceinline__ int fb_rows(const FbConvArgs& a) {
  const FbLevel l = a.gout[a.frames - 1];
  return l.pix0 + l.h * l.w;
}

constexpr int FB_BM = 64, FB_BN = 64, FB_BK = 16;

// Frame of packed pixel (GEMM row) m: the last frame whose first pixel is <= m.  Every frame has >= 1 pixel per level.
__device__ __forceinline__ int fb_frame_of(const FbLevel* g, int frames, int m) {
  int lo = 0, hi = frames - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&g[mid].pix0) <= m) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// One GEMM row's input geometry on the frame axis, looked up once per row per tile: its frame's input size, its output
// pixel (oy, ox) and the element offset of its frame's input map.  A 64-row tile may straddle frames of different sizes.
struct FbRow { int h, w, oy, ox; size_t xo; };
__device__ __forceinline__ FbRow fb_row_geo(const FbConvArgs& a, int m) {
  const int fr = fb_frame_of(a.gout, a.frames, m);
  const FbLevel gi = a.gin[fr];
  const int pix = m - a.gout[fr].pix0, wo = a.gout[fr].w;
  FbRow r;
  r.h = gi.h; r.w = gi.w; r.oy = pix / wo; r.ox = pix - r.oy * wo;
  r.xo = (size_t)gi.pix0 * (a.x_u8 ? 3 : a.cin_stride);
  return r;
}

// Frame axis: where output row m stores its cout channels (before cout_off)
__device__ __forceinline__ float* fb_row_out(const FbConvArgs& a, int m) {
  const FbLevel go = a.gout[fb_frame_of(a.gout, a.frames, m)];
  // a head writes its frame's slice of the packed (sum P, 4) / (sum P, 2) block: cout_stride / ppp floats per prior
  const size_t base = go.ppp ? (size_t)go.prior0 * (a.cout_stride / go.ppp) : (size_t)go.pix0 * a.cout_stride;
  return a.y + base + (size_t)(m - go.pix0) * a.cout_stride;
}

// One input value of the one-image implicit GEMM: element `kidx` = (kh, kw, ci) of output row m's patch (0 outside the
// image); MT = rows of the GEMM
__device__ __forceinline__ float fb_gather1(const FbConvArgs& a, int kidx, int m, int K, int M, int MT) {
  if (kidx >= K || m >= MT) return 0.f;
  const int pix = m;
  const int ci = kidx % a.cin, t = kidx / a.cin, kw = t % a.k, kh = t / a.k;
  const int oy = pix / a.wo, ox = pix - oy * a.wo;
  const int iy = oy * a.stride - a.pad + kh, ix = ox * a.stride - a.pad + kw;
  if (iy < 0 || iy >= a.h || ix < 0 || ix >= a.w) return 0.f;
  if (a.x_u8) return (float)a.x_u8[((size_t)iy * a.w + ix) * 3 + ci] - (ci == 0 ? a.mean[0] : ci == 1 ? a.mean[1] : a.mean[2]);
  return a.x[((size_t)iy * a.w + ix) * a.cin_stride + a.cin_off + ci];
}

// The same on the frame axis, against row r's own frame (live: r is a row of the GEMM)
__device__ __forceinline__ float fb_gather_row(const FbConvArgs& a, const FbRow& r, bool live, int kidx, int K) {
  if (kidx >= K || !live) return 0.f;
  const int ci = kidx % a.cin, t = kidx / a.cin, kw = t % a.k, kh = t / a.k;
  const int iy = r.oy * a.stride - a.pad + kh, ix = r.ox * a.stride - a.pad + kw;
  if (iy < 0 || iy >= r.h || ix < 0 || ix >= r.w) return 0.f;
  if (a.x_u8) return (float)a.x_u8[r.xo + ((size_t)iy * r.w + ix) * 3 + ci] - (ci == 0 ? a.mean[0] : ci == 1 ? a.mean[1] : a.mean[2]);
  return a.x[r.xo + ((size_t)iy * r.w + ix) * a.cin_stride + a.cin_off + ci];
}

// VEC: cin, cin_stride, cin_off and cout are multiples of 4 (every layer but conv1 and the 42- / 2-channel heads): a
// thread fetches ONE float4 of the A tile (4 consecutive input channels of one patch position: contiguous in NHWC) and
// one float4 of the B tile per K step instead of four scalars each.  Either way the next step's operands are fetched
// into registers before the current step's FMAs and stored to shared memory after them, so the global-load latency of
// the long-K, small-M layers (conv2, the stride-2 3x3s, the heads: 72-144 K steps on a few dozen CTAs) is hidden.
// FRAMES (syn_fb_forward_images, syn_fb_forward_batch) only changes which frame a row addresses: the K order and the
// fmaf chain of every accumulator are the one-image kernel's, so each output element has the one-image bits.
template <bool VEC, bool FRAMES>
__global__ void __launch_bounds__(256) fb_conv_kernel(const FbConvArgs a) {
  __shared__ __align__(16) float sA[FB_BK][FB_BM + 4];
  __shared__ __align__(16) float sB[FB_BK][FB_BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;            // thread = 4 pixels (ty) x 4 channels (tx)
  const int m0 = blockIdx.x * FB_BM, n0 = blockIdx.y * FB_BN;
  const int M = a.ho * a.wo, K = a.k * a.k * a.cin, MT = FRAMES ? fb_rows(a) : M;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float ra[4], rb[4];
  // VEC mapping: A -- pixel tid / 4, K quad tid % 4 (four neighbouring threads read 64 contiguous bytes);
  //              B -- K row tid / 16, channel quad tid % 16
  const int a_mm = tid >> 2, a_kq = tid & 3, b_kk = tid >> 4, b_nq = tid & 15;
  // the row this thread gathers (VEC: pixel a_mm; scalar: pixel tid % 64 of every K row it fetches)
  int v_oy = 0, v_ox = 0, v_h = a.h, v_w = a.w;
  const float* v_x = a.x;
  FbRow row{};
  if constexpr (FRAMES) {
    row = fb_row_geo(a, m0 + (VEC ? a_mm : tid % FB_BM));
    v_oy = row.oy; v_ox = row.ox; v_h = row.h; v_w = row.w;
    v_x += row.xo;
  } else if (VEC) {
    const int pix = m0 + a_mm;
    v_oy = pix / a.wo; v_ox = pix - v_oy * a.wo;
  }
  auto fetch = [&](int k0) {
    if (VEC) {
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = make_float4(0.f, 0.f, 0.f, 0.f);
      const int kidx = k0 + a_kq * 4;
      if (kidx < K && m0 + a_mm < MT) {
        const int ci = kidx % a.cin, t = kidx / a.cin, kw = t % a.k, kh = t / a.k;
        const int iy = v_oy * a.stride - a.pad + kh, ix = v_ox * a.stride - a.pad + kw;
        if (iy >= 0 && iy < v_h && ix >= 0 && ix < v_w)
          va = __ldg(reinterpret_cast<const float4*>(v_x + ((size_t)iy * v_w + ix) * a.cin_stride + a.cin_off + ci));
      }
      const int kb = k0 + b_kk, n = n0 + b_nq * 4;
      if (kb < K && n < a.cout) vb = __ldg(reinterpret_cast<const float4*>(a.wk + (size_t)kb * a.cout + n));
      ra[0] = va.x; ra[1] = va.y; ra[2] = va.z; ra[3] = va.w;
      rb[0] = vb.x; rb[1] = vb.y; rb[2] = vb.z; rb[3] = vb.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = tid + j * 256, kk = e / FB_BM, mm = e - kk * FB_BM;
        if constexpr (FRAMES) ra[j] = fb_gather_row(a, row, m0 + mm < MT, k0 + kk, K);
        else ra[j] = fb_gather1(a, k0 + kk, m0 + mm, K, M, MT);
        const int kb = k0 + e / FB_BN, n = n0 + e % FB_BN;
        rb[j] = (kb < K && n < a.cout) ? a.wk[(size_t)kb * a.cout + n] : 0.f;
      }
    }
  };
  auto stash = [&]() {
    if (VEC) {
#pragma unroll
      for (int j = 0; j < 4; ++j) sA[a_kq * 4 + j][a_mm] = ra[j];
      *reinterpret_cast<float4*>(&sB[b_kk][b_nq * 4]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = tid + j * 256;
        sA[e / FB_BM][e % FB_BM] = ra[j];
        sB[e / FB_BN][e % FB_BN] = rb[j];
      }
    }
  };
  fetch(0);
  stash();
  __syncthreads();
  for (int k0 = 0; k0 < K; k0 += FB_BK) {
    const bool more = k0 + FB_BK < K;
    if (more) fetch(k0 + FB_BK);
#pragma unroll
    for (int kk = 0; kk < FB_BK; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&sA[kk][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&sB[kk][tx * 4]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w}, bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
    if (more) {
      stash();
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= MT) continue;
    float* o = (FRAMES ? fb_row_out(a, m) : a.y + (size_t)m * a.cout_stride) + a.cout_off;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= a.cout) continue;
      const float v = acc[i][j] + a.bias[n];
      if (a.act == 0) o[n] = v;
      else if (a.act == 1) o[n] = fmaxf(v, 0.f);
      else { o[n] = fmaxf(v, 0.f); o[n + a.cout] = fmaxf(-v, 0.f); }
    }
  }
}

// Layers with at most 8 output channels and a long K (the 4- / 2-channel heads on the stride-64 / -128 maps: K = 2304,
// 204 or 54 pixels): a 64 x 64 tile would run 144 serial K steps on one or two CTAs.  Here a CTA of 128 threads owns ONE
// output pixel, the threads stride over K and the partial sums meet in a warp-shuffle + shared-memory reduction.
// FRAMES: blockIdx.x = packed output pixel, its frame looked up once; the K stride and the reduction tree are unchanged.
constexpr int FB_SMALLN = 8;
template <bool FRAMES>
__global__ void __launch_bounds__(128) fb_conv_smalln_kernel(const FbConvArgs a) {
  __shared__ float red[4][FB_SMALLN];
  const int m = blockIdx.x, tid = threadIdx.x;
  const int M = a.ho * a.wo, K = a.k * a.k * a.cin, MT = FRAMES ? fb_rows(a) : M;
  FbRow row{};
  if constexpr (FRAMES) row = fb_row_geo(a, m);
  float acc[FB_SMALLN];
#pragma unroll
  for (int n = 0; n < FB_SMALLN; ++n) acc[n] = 0.f;
  for (int k = tid; k < K; k += 128) {
    float v;
    if constexpr (FRAMES) v = fb_gather_row(a, row, m < MT, k, K);
    else v = fb_gather1(a, k, m, K, M, MT);
    const float* wr = a.wk + (size_t)k * a.cout;
#pragma unroll
    for (int n = 0; n < FB_SMALLN; ++n)
      if (n < a.cout) acc[n] = fmaf(v, wr[n], acc[n]);
  }
#pragma unroll
  for (int n = 0; n < FB_SMALLN; ++n) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc[n] += __shfl_xor_sync(0xFFFFFFFFu, acc[n], off);
    if ((tid & 31) == 0) red[tid >> 5][n] = acc[n];
  }
  __syncthreads();
  if (tid < a.cout) {
    const float v = ((red[0][tid] + red[1][tid]) + (red[2][tid] + red[3][tid])) + a.bias[tid];
    float* o = (FRAMES ? fb_row_out(a, m) : a.y + (size_t)m * a.cout_stride) + a.cout_off;
    if (a.act == 0) o[tid] = v;
    else if (a.act == 1) o[tid] = fmaxf(v, 0.f);
    else { o[tid] = fmaxf(v, 0.f); o[tid + a.cout] = fmaxf(-v, 0.f); }
  }
}

// The pools on the frame axis: element i of the packed output map -> (frame, pixel, channel) and that frame's input map
struct FbPoolFrames {
  const FbLevel* gin;
  const FbLevel* gout;
  int frames, rows;        // rows: pixels of the packed output map
};

// F.max_pool2d(x, 3, stride 2, padding 1) (faceboxes.py:121,123), NHWC.  FRAMES: the packed maps of fr.frames images
template <bool FRAMES>
__global__ void fb_maxpool_kernel(const float* __restrict__ x, int h, int w, int c, float* __restrict__ y, int ho, int wo,
                                  const FbPoolFrames fr) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int ch, ox, oy;
  if (FRAMES) {
    if (i >= (size_t)fr.rows * c) return;
    const int q = (int)(i / c), f = fb_frame_of(fr.gout, fr.frames, q);
    const FbLevel gi = fr.gin[f], go = fr.gout[f];
    ch = (int)(i - (size_t)q * c); oy = (q - go.pix0) / go.w; ox = q - go.pix0 - oy * go.w;
    h = gi.h; w = gi.w;
    x += (size_t)gi.pix0 * c;
  } else {
    if (i >= (size_t)ho * wo * c) return;
    ch = (int)(i % c); ox = (int)((i / c) % wo); oy = (int)(i / ((size_t)c * wo));
  }
  float m = -INFINITY;
  for (int dy = 0; dy < 3; ++dy)
    for (int dx = 0; dx < 3; ++dx) {
      const int iy = oy * 2 - 1 + dy, ix = ox * 2 - 1 + dx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) m = fmaxf(m, x[((size_t)iy * w + ix) * c + ch]);
    }
  y[i] = m;
}

// F.avg_pool2d(x, 3, stride 1, padding 1) (faceboxes.py:37): count_include_pad defaults to True, the divisor is always 9.
// FRAMES: the packed maps of fr.frames images (input and output share one geometry)
template <bool FRAMES>
__global__ void fb_avgpool_kernel(const float* __restrict__ x, int h, int w, int c, float* __restrict__ y, const FbPoolFrames fr) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int ch, ox, oy;
  if (FRAMES) {
    if (i >= (size_t)fr.rows * c) return;
    const int q = (int)(i / c), f = fb_frame_of(fr.gout, fr.frames, q);
    const FbLevel g = fr.gout[f];
    ch = (int)(i - (size_t)q * c); oy = (q - g.pix0) / g.w; ox = q - g.pix0 - oy * g.w;
    h = g.h; w = g.w;
    x += (size_t)g.pix0 * c;
  } else {
    if (i >= (size_t)h * w * c) return;
    ch = (int)(i % c); ox = (int)((i / c) % w); oy = (int)(i / ((size_t)c * w));
  }
  float s = 0.f;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      const int iy = oy + dy, ix = ox + dx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) s += x[((size_t)iy * w + ix) * c + ch];
    }
  y[i] = s / 9.0f;
}

// nn.Softmax(dim=-1) over the (P, 2) class scores (faceboxes.py:92,143); on the frame axis np = sum of every P_i
__global__ void fb_softmax2_kernel(float* __restrict__ conf, int np) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const float a = conf[2 * i], b = conf[2 * i + 1], m = fmaxf(a, b);
  const float ea = expf(a - m), eb = expf(b - m), s = ea + eb;
  conf[2 * i] = ea / s;
  conf[2 * i + 1] = eb / s;
}

}  // namespace syn
