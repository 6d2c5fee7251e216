// UV texture sampling of artistic.py:126-131 and uv_texture_realFaces.py:103-114 for many faces at once: each face reads
// its own UV map at the kept vertices' texels.  The host resolves every texel of np.flip(map, 0)[coord_u, coord_v][keep]
// to a (row, column) of the unflipped map (numpy's wrap of negative indices included), once per map size, so the kernel
// is a gather: one thread per (face, kept vertex), three bytes in, three floats (and optionally three int64) out.
#pragma once
#include "common.cuh"

namespace syn {

constexpr int kUvThreads = 256;

// maps: packed uint8 (h, w, 3) maps, map m at byte table[3m] with width table[3m+2]; texels (n_maps, n_keep, 2) int32:
// (row, column) of kept vertex i in map m; face_map[f]: the map of face f.  texture (F, n_keep, 3) float32 = byte / 255
// and colors (F, n_keep, 3) int64 = byte, each skipped when nullptr.
__global__ void uv_sample_kernel(const uint8_t* __restrict__ maps, const long long* __restrict__ table,
                                 const int32_t* __restrict__ texels, int n_keep, const int32_t* __restrict__ face_map,
                                 float* __restrict__ texture, long long* __restrict__ colors) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
  if (i >= n_keep) return;
  const int m = __ldg(face_map + f);
  const long long off = __ldg(table + 3 * m), w = __ldg(table + 3 * m + 2);
  const int2 rc = __ldg(reinterpret_cast<const int2*>(texels) + (size_t)m * n_keep + i);
  const uint8_t* p = maps + off + 3 * ((long long)rc.x * w + rc.y);
  const size_t o = ((size_t)f * n_keep + i) * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint8_t c = __ldg(p + k);
    if (texture) texture[o + k] = (float)c / 255.0f;    // IEEE division: numpy's colors_uv.astype(np.float32) / 255.0
    if (colors) colors[o + k] = c;
  }
}

}  // namespace syn
