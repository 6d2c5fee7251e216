// Text of the reference's OBJ writers (utils/inference.py:8-23 write_obj; artistic.py:19-31 and
// uv_texture_realFaces.py:21-33 write_obj_with_colors), shared by the CUDA kernels (kernels_obj.cuh) and by the host
// emulation the CPU tests run (tests/host_emul/obj_emul.cpp compiles this header with g++).
//
// Three fields, each a length function and a write function that stores exactly that many bytes:
//   * f4: '{:.4f}'.format(np.float32 x).  NumPy formats a float32 through Python float, so the text is the exact binary
//     value rounded to 4 decimals, ties to even.  Exact integer arithmetic, no printf, no floating-point rounding:
//     x = m 2^e with m < 2^24.  For e >= 0 the integer part m << e (< 2^128) is printed, then ".0000".  For e < 0, with
//     k = -e, s = m 10^4 (< 2^38), q = s >> k rounded half to even on the k dropped bits (q = 0 for k >= 64), printed as
//     q / 10^4 "." (q % 10^4 on 4 digits).  The sign bit always prints ("-0.0000"); a NaN of either sign is "nan",
//     infinities are "inf" / "-inf".
//   * int: '{}' of an integer NumPy scalar: its decimal digits, any int64.
//   * n0: '{}' of an integral float scalar below 1e16 in magnitude: repr of the double, the digits then ".0".  The value
//     travels as an int64; kNegZero (INT64_MIN, which the form never reaches) stands for -0.0 and prints "-0.0".
// num() is int or n0 by a flag.  A vertex line is "v x y z\n", or "v x y z c2 c1 c0\n" with colours (BGR stored, RGB
// written); a triangle line is "f a b c\n" of the three indices in the order the caller passes them.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define SYN_OM_HD __host__ __device__ __forceinline__
#else
#define SYN_OM_HD inline
#endif

namespace syn {
namespace omath {

constexpr int64_t kNegZero = INT64_MIN;

SYN_OM_HD uint32_t float_bits(float x) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(x);
#else
  uint32_t u;
  memcpy(&u, &x, 4);
  return u;
#endif
}

SYN_OM_HD int u64_digits(uint64_t v) {
  int n = 1;
  while (v >= 10) { v /= 10; ++n; }
  return n;
}

SYN_OM_HD int u128_digits(unsigned __int128 v) {
  const uint64_t e19 = 10000000000000000000ull;
  if (v >> 64 == 0) return u64_digits((uint64_t)v);
  const unsigned __int128 hi = v / e19;
  return (hi >> 64 == 0 ? u64_digits((uint64_t)hi) : 19 + u64_digits((uint64_t)(hi / e19))) + 19;
}

// the n digits of v, most significant first, at p[0..n-1]
SYN_OM_HD void put_u64(char* p, uint64_t v, int n) {
  for (int i = n - 1; i >= 0; --i) { p[i] = (char)('0' + v % 10); v /= 10; }
}

SYN_OM_HD void put_u128(char* p, unsigned __int128 v, int n) {
  const uint64_t e19 = 10000000000000000000ull;
  while (n > 19) {                                    // 19 low digits at a time
    put_u64(p + n - 19, (uint64_t)(v % e19), 19);
    v /= e19;
    n -= 19;
  }
  put_u64(p, (uint64_t)v, n);
}

// the decomposition of a finite float32: |x| = ip + q / 10^4 rounded as '{:.4f}' rounds it (big: ip is (m << e))
struct F4 {
  int kind;               // 0 finite, 1 nan, 2 inf
  bool neg;
  bool big;               // e >= 0: the integer part is m << e and the decimals are 0
  unsigned __int128 ip;   // big: the integer part
  uint64_t q;             // !big: |x| 10^4 rounded half to even
};

SYN_OM_HD F4 f4_split(float x) {
  const uint32_t u = float_bits(x);
  F4 r;
  r.neg = (u >> 31) != 0;
  const int be = (int)((u >> 23) & 255);
  const uint32_t frac = u & 0x7FFFFF;
  r.kind = be == 255 ? (frac ? 1 : 2) : 0;
  r.big = false;
  r.ip = 0;
  r.q = 0;
  if (r.kind) return r;
  const uint64_t m = be ? (frac | 0x800000u) : frac;
  const int e = be ? be - 150 : -149;
  if (e >= 0) {
    r.big = true;
    r.ip = (unsigned __int128)m << e;
    return r;
  }
  const int k = -e;
  if (k >= 64) return r;                              // s < 2^38 <= 2^(k-1): rounds to 0
  const uint64_t s = m * 10000u;
  uint64_t q = s >> k;
  const uint64_t rem = s & ((1ull << k) - 1), half = 1ull << (k - 1);
  if (rem > half || (rem == half && (q & 1))) ++q;
  r.q = q;
  return r;
}

SYN_OM_HD int f4_len(float x) {
  const F4 f = f4_split(x);
  if (f.kind == 1) return 3;
  if (f.kind == 2) return 3 + f.neg;
  if (f.big) return f.neg + u128_digits(f.ip) + 5;
  return f.neg + u64_digits(f.q / 10000) + 5;
}

SYN_OM_HD int f4_write(float x, char* p) {
  const F4 f = f4_split(x);
  if (f.kind == 1) { p[0] = 'n'; p[1] = 'a'; p[2] = 'n'; return 3; }
  int n = 0;
  if (f.neg) p[n++] = '-';
  if (f.kind == 2) { p[n] = 'i'; p[n + 1] = 'n'; p[n + 2] = 'f'; return n + 3; }
  uint64_t dec = 0;
  if (f.big) {
    const int d = u128_digits(f.ip);
    put_u128(p + n, f.ip, d);
    n += d;
  } else {
    const int d = u64_digits(f.q / 10000);
    put_u64(p + n, f.q / 10000, d);
    n += d;
    dec = f.q % 10000;
  }
  p[n++] = '.';
  put_u64(p + n, dec, 4);
  return n + 4;
}

SYN_OM_HD uint64_t magnitude(int64_t v) { return v < 0 ? 0 - (uint64_t)v : (uint64_t)v; }

SYN_OM_HD int int_len(int64_t v) { return (v < 0) + u64_digits(magnitude(v)); }

SYN_OM_HD int int_write(int64_t v, char* p) {
  const int s = v < 0, d = u64_digits(magnitude(v));
  if (s) p[0] = '-';
  put_u64(p + s, magnitude(v), d);
  return s + d;
}

SYN_OM_HD int n0_len(int64_t v) { return v == kNegZero ? 4 : int_len(v) + 2; }

SYN_OM_HD int n0_write(int64_t v, char* p) {
  if (v == kNegZero) { p[0] = '-'; p[1] = '0'; p[2] = '.'; p[3] = '0'; return 4; }
  const int n = int_write(v, p);
  p[n] = '.';
  p[n + 1] = '0';
  return n + 2;
}

SYN_OM_HD int num_len(int64_t v, int dot0) { return dot0 ? n0_len(v) : int_len(v); }
SYN_OM_HD int num_write(int64_t v, int dot0, char* p) { return dot0 ? n0_write(v, p) : int_write(v, p); }

// "v x y z\n", or with colours (c = the BGR triple of the vertex) "v x y z c[2] c[1] c[0]\n"
SYN_OM_HD int vertex_line_len(float x, float y, float z, const int64_t* c, int dot0) {
  int n = 2 + f4_len(x) + 1 + f4_len(y) + 1 + f4_len(z) + 1;
  if (c) n += num_len(c[2], dot0) + 1 + num_len(c[1], dot0) + 1 + num_len(c[0], dot0) + 1;
  return n;
}

SYN_OM_HD int vertex_line_write(float x, float y, float z, const int64_t* c, int dot0, char* p) {
  int n = 0;
  p[n++] = 'v';
  p[n++] = ' ';
  n += f4_write(x, p + n);
  p[n++] = ' ';
  n += f4_write(y, p + n);
  p[n++] = ' ';
  n += f4_write(z, p + n);
  if (c) {
    for (int k = 2; k >= 0; --k) {
      p[n++] = ' ';
      n += num_write(c[k], dot0, p + n);
    }
  }
  p[n++] = '\n';
  return n;
}

// "f a b c\n"
SYN_OM_HD int tri_line_len(int64_t a, int64_t b, int64_t c, int dot0) {
  return 2 + num_len(a, dot0) + 1 + num_len(b, dot0) + 1 + num_len(c, dot0) + 1;
}

SYN_OM_HD int tri_line_write(int64_t a, int64_t b, int64_t c, int dot0, char* p) {
  int n = 0;
  p[n++] = 'f';
  p[n++] = ' ';
  n += num_write(a, dot0, p + n);
  p[n++] = ' ';
  n += num_write(b, dot0, p + n);
  p[n++] = ' ';
  n += num_write(c, dot0, p + n);
  p[n++] = '\n';
  return n;
}

}  // namespace omath
}  // namespace syn
