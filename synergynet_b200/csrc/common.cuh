// Shared helpers for the sm_90a SynergyNet hot-path library.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/synergy_b200.h"

namespace syn {

// ---- error plumbing (no exceptions cross the C ABI) ---------------------------------------------
inline char* last_error_buf() {
  static thread_local char buf[512] = "";
  return buf;
}
inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

#define SYN_CUDA(call)                                                                   \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess)                                                              \
      return ::syn::fail(SYN_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call,      \
                         cudaGetErrorString(e__));                                       \
  } while (0)

#define SYN_LAUNCH_CHECK(name)                                                           \
  do {                                                                                   \
    cudaError_t e__ = cudaGetLastError();                                                \
    if (e__ != cudaSuccess)                                                              \
      return ::syn::fail(SYN_ERR_CUDA, "launch %s -> %s", name, cudaGetErrorString(e__)); \
  } while (0)

// SYN_ERR_STATE with the formatted message when `st` is capturing a CUDA graph (or holds an invalidated capture).  Called
// before a step that a graph cannot record: a workspace growth (its cudaDeviceSynchronize is illegal under capture and
// would invalidate it, and its cudaFree would leave earlier replays reading freed memory) or a copy from a host buffer
// the next call rewrites.  Every call site comes before the entry's first launch, so a refused call records nothing
// and the caller can end the capture cleanly.
inline int refuse_capture(cudaStream_t st, const char* fmt, ...) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  SYN_CUDA(cudaStreamIsCapturing(st, &cs));
  if (cs == cudaStreamCaptureStatusNone) return SYN_OK;
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return SYN_ERR_STATE;
}
// the end of a growth refusal's message
#define SYN_EAGER_FIRST " cannot grow while the stream is capturing a CUDA graph: make an eager call before capture at this size or larger"

// The cudaMalloc of every workspace growth site.  fill >= 0 (syn_debug_fill_on_grow / syn_fb_debug_fill_on_grow) sets
// every byte of the new buffer to `fill` before the growing call launches anything, so that a call which grows its own
// workspace runs on poison, not on the zeroed pages a fresh allocation usually returns.  Growth sites run with the
// device idle and never under capture, so the blocking memset orders before every stream of the handle.
template <class T>
inline cudaError_t grow_alloc(T** p, size_t bytes, int fill) {
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), bytes);
  if (e == cudaSuccess && fill >= 0) e = cudaMemset(*p, fill, bytes);
  if (e == cudaSuccess && fill >= 0) e = cudaDeviceSynchronize();
  return e;
}

// One buffer of a debug fill (syn_debug_fill_workspaces): `bytes` bytes at p set to `byte` on stream st, counted in *total.
inline cudaError_t fill_buffer(void* p, size_t bytes, int byte, cudaStream_t st, size_t* total) {
  if (p == nullptr || bytes == 0) return cudaSuccess;
  *total += bytes;
  return cudaMemsetAsync(p, byte, bytes, st);
}

// ---- network geometry (reference backbone_nets/mobilenetv2_backbone.py:108-138) ---------------
constexpr int kImg = 120;
constexpr int kNumConv = 52;
constexpr int kLastCh = 1280;
constexpr int kNumParams = 62;       // 12 pose + 40 shape + 10 expression
constexpr int kNumShp = 40, kNumExp = 10, kNumAlpha = 50;

enum ConvKind { kStem = 0, kExpand = 1, kDepthwise = 2, kProject = 3, kLast = 4 };

struct ConvDesc {
  int kind, block, cin, cout, ksize, stride, groups, relu6, h_in, h_out, residual;
};

struct Plan {
  ConvDesc conv[kNumConv];
  int n;
};

inline Plan make_plan() {
  static const int stages[7][4] = {{1, 16, 1, 1}, {6, 24, 2, 2}, {6, 32, 3, 2}, {6, 64, 4, 2},
                                   {6, 96, 3, 1}, {6, 160, 3, 2}, {6, 320, 1, 1}};
  Plan p;
  p.n = 0;
  int h = kImg, ho = (h + 2 - 3) / 2 + 1;
  p.conv[p.n++] = ConvDesc{kStem, 0, 3, 32, 3, 2, 1, 1, h, ho, 0};
  h = ho;
  int cin = 32, blk = 1;
  for (int s = 0; s < 7; ++s) {
    const int t = stages[s][0], c = stages[s][1], n = stages[s][2], st = stages[s][3];
    for (int i = 0; i < n; ++i) {
      const int stride = (i == 0) ? st : 1;
      const int hid = cin * t;
      if (t != 1) p.conv[p.n++] = ConvDesc{kExpand, blk, cin, hid, 1, 1, 1, 1, h, h, 0};
      ho = (h + 2 - 3) / stride + 1;
      p.conv[p.n++] = ConvDesc{kDepthwise, blk, hid, hid, 3, stride, hid, 1, h, ho, 0};
      p.conv[p.n++] =
          ConvDesc{kProject, blk, hid, c, 1, 1, 1, 0, ho, ho, (stride == 1 && cin == c) ? 1 : 0};
      h = ho;
      cin = c;
      ++blk;
    }
  }
  p.conv[p.n++] = ConvDesc{kLast, blk, cin, kLastCh, 1, 1, 1, 1, h, h, 0};
  return p;
}

inline const Plan& plan() {
  static const Plan p = make_plan();
  return p;
}

__device__ __forceinline__ float relu6f(float v) { return fminf(fmaxf(v, 0.f), 6.f); }

}  // namespace syn
