// Serial host emulation of the OBJ kernels (synergynet_b200/csrc/kernels_obj.cuh): the lines of one mesh formatted one
// after the other by the same obj_math.h functions, plus the field sweeps tests/test_obj_emulation.py holds to
// snprintf("%.4f") and to Python's str.format.
// Build: g++ -O2 -shared -fPIC -pthread (the tests do it).
#include "../../synergynet_b200/csrc/obj_math.h"

#include <algorithm>
#include <stdio.h>
#include <string.h>
#include <thread>
#include <vector>

using namespace syn::omath;

extern "C" {

// '{:.4f}' of each of n floats, each followed by '\n', into out (NULL: lengths only); returns the bytes
int64_t emul_f4(const float* x, int64_t n, char* out) {
  int64_t at = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int len = f4_len(x[i]);
    if (out) {
      if (f4_write(x[i], out + at) != len) return -1;
      out[at + len] = '\n';
    }
    at += len + 1;
  }
  return at;
}

// '{}' of each of n int64 (dot0: the N.0 form), each followed by '\n'
int64_t emul_num(const int64_t* v, int64_t n, int dot0, char* out) {
  int64_t at = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int len = num_len(v[i], dot0);
    if (out) {
      if (num_write(v[i], dot0, out + at) != len) return -1;
      out[at + len] = '\n';
    }
    at += len + 1;
  }
  return at;
}

// every float32 of both signs with biased exponent in [be_lo, be_hi] (all mantissas), and every odd multiple of 2^-5
// float32 holds (ties == 1), formatted by f4 and by snprintf("%.4f") of the double: the count of differences; *first
// receives the bits of the first one
int64_t emul_f4_sweep(int be_lo, int be_hi, int ties, uint32_t* first) {
  const int n_threads = (int)std::max(1u, std::thread::hardware_concurrency());
  std::vector<int64_t> bad(n_threads, 0);
  std::vector<uint32_t> where(n_threads, 0);
  const uint64_t count = ties ? (1u << 23) : (uint64_t)(be_hi - be_lo + 1) << 23;
  std::vector<std::thread> pool;
  for (int t = 0; t < n_threads; ++t)
    pool.emplace_back([&, t] {
      char a[64], b[64];
      for (uint64_t j = t; j < count; j += n_threads)
        for (int s = 0; s < 2; ++s) {
          float x;
          if (ties) x = (float)(2 * j + 1) * 0.03125f;
          else {
            const uint32_t u = (uint32_t)(((uint64_t)be_lo << 23) + j);
            memcpy(&x, &u, 4);
          }
          if (s) x = -x;
          const int n = f4_write(x, a);
          const int m = snprintf(b, sizeof b, "%.4f", (double)x);
          if (n != f4_len(x) || n != m || memcmp(a, b, n)) {
            if (!bad[t]++) memcpy(&where[t], &x, 4);
          }
        }
    });
  for (auto& th : pool) th.join();
  int64_t total = 0;
  for (int t = 0; t < n_threads; ++t) {
    if (bad[t] && !total) *first = where[t];
    total += bad[t];
  }
  return total;
}

// the text of one mesh as the kernels write it: n vertex lines of rows xyz (n,3) float32 (already the kept vertices),
// colours (n,3) int64 or NULL, then ntri triangle lines of tri (ntri,3) int64 in tri_order; out NULL: length only
int64_t emul_obj(const float* xyz, int n, const int64_t* colors, int colors_dot0, const int64_t* tri, int ntri, int tri_order,
                 int tri_dot0, char* out) {
  int64_t at = 0;
  for (int i = 0; i < n; ++i) {
    const float* p = xyz + 3LL * i;
    const int64_t* c = colors ? colors + 3LL * i : nullptr;
    const int len = vertex_line_len(p[0], p[1], p[2], c, colors_dot0);
    if (out && vertex_line_write(p[0], p[1], p[2], c, colors_dot0, out + at) != len) return -1;
    at += len;
  }
  for (int i = 0; i < ntri; ++i) {
    const int64_t* r = tri + 3LL * i;
    const int64_t a = tri_order ? r[0] : r[2], b = r[1], c = tri_order ? r[2] : r[0];
    const int len = tri_line_len(a, b, c, tri_dot0);
    if (out && tri_line_write(a, b, c, tri_dot0, out + at) != len) return -1;
    at += len;
  }
  return at;
}

}  // extern "C"
