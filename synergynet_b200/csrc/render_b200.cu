// C ABI of the stages either side of the 3DMM path (SURVEY.md section 8 rows f2, f3): Sim3DR normals / lighting /
// rasterisation of the dense meshes, the FaceBoxes box decode + greedy NMS that produces the crops, the crop + resize
// that turns boxes (or an oversized detector input) into network inputs, and the pose axes drawn over the frames.
// Handle-free: device pointers and workspaces belong to the caller (include/synergy_b200.h states the sizes).
#include "kernels_render.cuh"
#include "kernels_detect.cuh"
#include "kernels_resize.cuh"
#include "kernels_draw.cuh"
#include "kernels_obj.cuh"
#include "kernels_uv.cuh"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <new>
#include <vector>

using namespace syn;

namespace {

int check_mesh(const float* v, long long sb, int sv, int sc, int batch, int nver, MeshView& m) {
  if (!v || batch <= 0 || nver <= 0 || sv <= 0 || sc <= 0 || (batch > 1 && sb <= 0))
    return fail(SYN_ERR_INVALID, "mesh view: null pointer, empty batch or non-positive stride");
  m.v = v; m.sb = sb; m.sv = sv; m.sc = sc; m.nver = nver; m.batch = batch;
  return SYN_OK;
}

// the shared checks of the frame-axis entries: the mesh view, the frame size and mesh_start_host (n_frames + 1 entries,
// 0 = mesh_start[0] <= ... <= mesh_start[n_frames] = n_meshes); meshes and frames each sit on one grid axis
int check_frames(const float* v, long long sb, int sv, int sc, int n_meshes, int nver, const int32_t* mesh_start_host, int n_frames,
                 int height, int width, MeshView& m, const char* who, const char* unit = "frame") {
  if (!v || !mesh_start_host || n_meshes <= 0 || nver <= 0 || sv <= 0 || sc <= 0 || (n_meshes > 1 && sb <= 0))
    return fail(SYN_ERR_INVALID, "%s: null pointer, no mesh or non-positive stride", who);
  if (n_frames <= 0 || n_frames > 65535 || n_meshes > 65535)
    return fail(SYN_ERR_INVALID, "%s: %d %ss and %d meshes (1..65535 of each per call)", who, n_frames, unit, n_meshes);
  if (height <= 0 || width <= 0) return fail(SYN_ERR_INVALID, "%s: frame size %dx%d", who, height, width);
  if (mesh_start_host[0] != 0 || mesh_start_host[n_frames] != n_meshes)
    return fail(SYN_ERR_SHAPE, "%s: mesh_start runs from %d to %d, must run from 0 to %d meshes", who, mesh_start_host[0],
                mesh_start_host[n_frames], n_meshes);
  for (int f = 0; f < n_frames; ++f)
    if (mesh_start_host[f + 1] < mesh_start_host[f])
      return fail(SYN_ERR_SHAPE, "%s: mesh_start is not monotone at %s %d (%d after %d)", who, unit, f, mesh_start_host[f + 1],
                  mesh_start_host[f]);
  return check_mesh(v, sb, sv, sc, n_meshes, nver, m);
}

// the shared checks of the image-list entries: check_frames, then the image table (n_images,3) int64 (offset, h, w) --
// the images in memory order, disjoint, inside the image bytes, each offset a multiple of the channel count -- and the
// device copies.  Fills the kernels' ImageAxis.
int check_images(const float* v, long long sb, int sv, int sc, int n_meshes, int nver, const int32_t* mesh_start_host,
                 const int32_t* mesh_start_dev, const int64_t* table_host, const int64_t* table_dev, int n_images, int64_t image_bytes,
                 int channels, MeshView& m, ImageAxis& ax, const char* who) {
  if (!table_host || !table_dev || !mesh_start_dev) return fail(SYN_ERR_INVALID, "%s: null pointer", who);
  if (int rc = check_frames(v, sb, sv, sc, n_meshes, nver, mesh_start_host, n_images, 1, 1, m, who, "image")) return rc;
  if (channels <= 0 || image_bytes < 0)
    return fail(SYN_ERR_SHAPE, "%s: %d image channels, %lld image bytes", who, channels, (long long)image_bytes);
  int64_t end = 0;
  for (int f = 0; f < n_images; ++f) {
    const int64_t off = table_host[3 * f], h = table_host[3 * f + 1], w = table_host[3 * f + 2];
    if (h < 1 || w < 1 || h > INT32_MAX || w > INT32_MAX)
      return fail(SYN_ERR_SHAPE, "%s: image %d is %lldx%lld", who, f, (long long)h, (long long)w);
    if (off < end || off > image_bytes || h > (image_bytes - off) / channels / w)
      return fail(SYN_ERR_SHAPE, "%s: image %d (%lldx%lld at byte %lld) does not fit the %lld image bytes after the image before it",
                  who, f, (long long)h, (long long)w, (long long)off, (long long)image_bytes);
    if (off % channels)
      return fail(SYN_ERR_SHAPE, "%s: image %d starts at byte %lld, not a multiple of its %d channels", who, f, (long long)off, channels);
    end = off + channels * h * w;
  }
  ax.mesh_start = mesh_start_dev;
  ax.table = reinterpret_cast<const long long*>(table_dev);
  ax.n = n_images;
  return SYN_OK;
}

// the host planner of both crop entries; frames_host == nullptr: one image
int crop_plan(const int32_t* rois_host, const int32_t* frames_host, int n_frames, int batch, int out_h, int out_w, int mode,
              void* plan_out, int64_t plan_bytes, const char* who) {
  if (!rois_host || !plan_out || batch <= 0) return fail(SYN_ERR_INVALID, "%s: null pointer or empty batch", who);
  if (out_h < 1 || out_w < 1) return fail(SYN_ERR_INVALID, "%s: output size %dx%d", who, out_h, out_w);
  if (mode != SYN_INTER_LINEAR && mode != SYN_INTER_LANCZOS4)
    return fail(SYN_ERR_UNSUPPORTED, "%s: interpolation %d (only INTER_LINEAR = 1 and INTER_LANCZOS4 = 4)", who, mode);
  for (int b = 0; b < batch; ++b) {
    const int32_t* r = rois_host + 4 * b;
    if (r[2] <= r[0] || r[3] <= r[1])        // crop_img would return an empty array, which cv2.resize rejects
      return fail(SYN_ERR_SHAPE, "%s: ROI %d (%d,%d,%d,%d) is empty", who, b, r[0], r[1], r[2], r[3]);
    if (frames_host && (frames_host[b] < 0 || frames_host[b] >= n_frames))
      return fail(SYN_ERR_SHAPE, "%s: ROI %d names frame %d of %d", who, b, frames_host[b], n_frames);
  }
  if (plan_bytes < syn_crop_resize_plan_size(batch, out_h, out_w, mode))
    return fail(SYN_ERR_SHAPE, "%s: plan buffer of %lld bytes, %lld needed", who, (long long)plan_bytes,
                (long long)syn_crop_resize_plan_size(batch, out_h, out_w, mode));
  rsz::build_plan(rois_host, batch, out_h, out_w, mode, plan_out, frames_host);
  return SYN_OK;
}

// the launch of both crop entries; n_frames == 0: one image, the plan's frame indices are not read
int crop_launch(const uint8_t* image_dev, int n_frames, int height, int width, int channels, const void* plan_dev, int batch,
                int out_h, int out_w, int mode, uint8_t* out_dev, int64_t stride_roi, int64_t stride_y, int64_t stride_x,
                int64_t stride_c, cudaStream_t st, const char* who) {
  if (!image_dev || !plan_dev || !out_dev || batch <= 0) return fail(SYN_ERR_INVALID, "%s: null pointer or empty batch", who);
  if (height < 1 || width < 1 || out_h < 1 || out_w < 1)
    return fail(SYN_ERR_INVALID, "%s: image %dx%d, output %dx%d", who, height, width, out_h, out_w);
  if (channels != 3) return fail(SYN_ERR_UNSUPPORTED, "%s: %d channels (BGR images only)", who, channels);
  if (mode != SYN_INTER_LINEAR && mode != SYN_INTER_LANCZOS4)
    return fail(SYN_ERR_UNSUPPORTED, "%s: interpolation %d (only INTER_LINEAR = 1 and INTER_LANCZOS4 = 4)", who, mode);
  if (batch > 65535) return fail(SYN_ERR_SHAPE, "%s: %d ROIs exceed one launch's grid", who, batch);
  const dim3 grid((out_w + kResizeBX - 1) / kResizeBX, (out_h + kResizeBY - 1) / kResizeBY, batch), block(kResizeBX, kResizeBY);
  if (mode == SYN_INTER_LANCZOS4)
    crop_resize_kernel<8><<<grid, block, 0, st>>>(image_dev, height, width, plan_dev, batch, out_h, out_w, out_dev, stride_roi,
                                                  stride_y, stride_x, stride_c, n_frames);
  else
    crop_resize_kernel<2><<<grid, block, 0, st>>>(image_dev, height, width, plan_dev, batch, out_h, out_w, out_dev, stride_roi,
                                                  stride_y, stride_x, stride_c, n_frames);
  SYN_LAUNCH_CHECK("crop_resize_kernel");
  return SYN_OK;
}

// frame f of a decode launch's table
FbDecodeFrames decode_frame(FbDecodeFrames t, int f, int h, int w, float box_scale_w, float box_scale_h, float scale, int p0, int c0,
                            int i0) {
  t.h[f] = h; t.w[f] = w; t.np[f] = faceboxes_num_priors(h, w); t.p0[f] = p0; t.c0[f] = c0; t.i0[f] = i0;
  t.box_scale_w[f] = box_scale_w; t.box_scale_h[f] = box_scale_h; t.scale[f] = scale;
  return t;
}

// the two decode launches of every decode entry: grid.y = frame, grid.x sized for np_max priors; counts already zeroed
int decode_launch(const float* loc, const float* conf, const FbDecodeFrames& t, int n_frames, int np_max, float conf_thresh, int top_k,
                  int32_t* cand, float* dets, int32_t* n_dets, cudaStream_t st) {
  faceboxes_select_kernel<<<dim3((np_max + 255) / 256, n_frames), 256, 0, st>>>(conf, t, conf_thresh, cand);
  SYN_LAUNCH_CHECK("faceboxes_select_kernel");
  faceboxes_rank_decode_kernel<<<dim3((np_max + 127) / 128, n_frames), 128, 0, st>>>(loc, conf, t, top_k, cand,
                                                                                                        dets, n_dets);
  SYN_LAUNCH_CHECK("faceboxes_rank_decode_kernel");
  return SYN_OK;
}

// both lighting entries: texture_dev NULL (light only), or mesh b's (nver,3) texture at texture_dev + b * tb
int mesh_lighting(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch, int nver,
                  const float* normals_dev, const syn_light_cfg_t* cfg, const float* texture_dev, int64_t tb, uint32_t* stats_ws_dev,
                  float* colors_dev, void* stream, const char* who) {
  MeshView m;
  if (int rc = check_mesh(vertices_dev, stride_mesh, stride_vertex, stride_coord, batch, nver, m)) return rc;
  if (!normals_dev || !cfg || !stats_ws_dev || !colors_dev) return fail(SYN_ERR_INVALID, "%s: null pointer", who);
  rmath::LightCfg c;
  c.intensity_ambient = cfg->intensity_ambient;
  c.intensity_directional = cfg->intensity_directional;
  c.intensity_specular = cfg->intensity_specular;
  c.specular_exp = cfg->specular_exp;
  for (int k = 0; k < 3; ++k) {
    c.color_ambient[k] = cfg->color_ambient[k];
    c.color_directional[k] = cfg->color_directional[k];
    c.light_pos[k] = cfg->light_pos[k];
    c.view_pos[k] = cfg->view_pos[k];
  }
  cudaStream_t st = (cudaStream_t)stream;
  SYN_CUDA(cudaMemsetAsync(stats_ws_dev, 0, sizeof(uint32_t) * 6 * batch, st));
  const int blocks = min((nver + 255) / 256, 64);
  mesh_extent_kernel<<<dim3(blocks, batch), 256, 0, st>>>(m, stats_ws_dev);
  SYN_LAUNCH_CHECK("mesh_extent_kernel");
  vertex_light_kernel<<<dim3((nver + 255) / 256, batch), 256, 0, st>>>(m, normals_dev, stats_ws_dev, c, texture_dev, (long long)tb,
                                                                        colors_dev);
  SYN_LAUNCH_CHECK("vertex_light_kernel");
  return SYN_OK;
}

int64_t obj_blocks(int n) { return ((int64_t)n + kObjThreads - 1) / kObjThreads; }

// the shared checks of the two OBJ entries; fills the kernels' arguments
int check_obj(const syn_obj_desc_t* d, const void* ws, int64_t ws_bytes, ObjArgs& a, const char* who) {
  if (!d || !d->vertices || !ws || (d->keep_host && !d->keep_dev) || (d->ntri > 0 && !d->triangles))
    return fail(SYN_ERR_INVALID, "%s: null pointer", who);
  if (d->keep_dev && !d->keep_host)
    return fail(SYN_ERR_INVALID, "%s: keep_dev without keep_host (the kept indices are checked on the host)", who);
  if (d->batch < 1 || d->batch > 65535 || d->nver < 1 || d->ntri < 0 || (d->keep_host && d->n_keep < 0))
    return fail(SYN_ERR_INVALID, "%s: %d meshes (1..65535), %d vertices, %d kept, %d triangles", who, d->batch, d->nver,
                d->keep_host ? d->n_keep : d->nver, d->ntri);
  if (d->stride_vertex < 1 || d->stride_coord < 1 || (d->batch > 1 && d->stride_mesh < 1) || d->colors_stride_mesh < 0)
    return fail(SYN_ERR_INVALID, "%s: strides mesh %lld, vertex %d, coordinate %d, colour mesh %lld", who, (long long)d->stride_mesh,
                d->stride_vertex, d->stride_coord, (long long)d->colors_stride_mesh);
  if ((d->tri_order | d->tri_dot0 | d->colors_dot0) & ~1)
    return fail(SYN_ERR_INVALID, "%s: flags tri_order %d, tri_dot0 %d, colors_dot0 %d (each 0 or 1)", who, d->tri_order, d->tri_dot0,
                d->colors_dot0);
  const int n = d->keep_host ? d->n_keep : d->nver;
  if (d->keep_host)
    for (int i = 0; i < n; ++i)
      if (d->keep_host[i] < 0 || d->keep_host[i] >= d->nver)
        return fail(SYN_ERR_INVALID, "%s: keep[%d] = %d lies outside [0, %d)", who, i, d->keep_host[i], d->nver);
  if ((int64_t)d->batch * obj_blocks(n) + obj_blocks(d->ntri) > INT32_MAX)
    return fail(SYN_ERR_INVALID, "%s: %d meshes of %d vertex lines and %d triangles exceed one launch's %d blocks of %d lines", who,
                d->batch, n, d->ntri, INT32_MAX, kObjThreads);
  if (ws_bytes < syn_obj_workspace_size(d->batch, n, d->ntri))
    return fail(SYN_ERR_SHAPE, "%s: workspace of %lld bytes, %lld needed", who, (long long)ws_bytes,
                (long long)syn_obj_workspace_size(d->batch, n, d->ntri));
  a.v = d->vertices; a.sb = d->batch > 1 ? d->stride_mesh : 0; a.sv = d->stride_vertex; a.sc = d->stride_coord;
  a.keep = d->keep_host ? d->keep_dev : nullptr; a.n = n;
  a.colors = d->colors; a.cb = d->colors_stride_mesh; a.color_dot0 = d->colors_dot0;
  a.tri = d->triangles; a.ntri = d->ntri; a.tri_order = d->tri_order; a.tri_dot0 = d->tri_dot0;
  a.batch = d->batch; a.vblocks = (int)obj_blocks(n); a.tblocks = (int)obj_blocks(d->ntri);
  return SYN_OK;
}

}  // namespace

extern "C" {

int syn_mesh_incidence_host(const int32_t* tri_host, int ntri, int nver, int32_t* start_out, int32_t* list_out) {
  if (!tri_host || !start_out || !list_out || ntri < 0 || nver <= 0) return fail(SYN_ERR_INVALID, "syn_mesh_incidence_host: bad argument");
  for (int i = 0; i < 3 * ntri; ++i)
    if (tri_host[i] < 0 || tri_host[i] >= nver) return fail(SYN_ERR_SHAPE, "triangle %d references vertex %d of %d", i / 3, tri_host[i], nver);
  for (int v = 0; v <= nver; ++v) start_out[v] = 0;
  for (int i = 0; i < 3 * ntri; ++i) ++start_out[tri_host[i] + 1];
  for (int v = 0; v < nver; ++v) start_out[v + 1] += start_out[v];
  std::vector<int32_t> fill(start_out, start_out + nver);
  for (int t = 0; t < ntri; ++t)                 // triangles in order: every vertex's list comes out ascending
    for (int k = 0; k < 3; ++k) list_out[fill[tri_host[3 * t + k]]++] = t;
  return SYN_OK;
}

int syn_mesh_normals(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch, int nver,
                     const int32_t* tri_dev, int ntri, const int32_t* inc_start_dev, const int32_t* inc_tri_dev,
                     float* tri_normals_ws_dev, float* normals_dev, void* stream) {
  MeshView m;
  if (int rc = check_mesh(vertices_dev, stride_mesh, stride_vertex, stride_coord, batch, nver, m)) return rc;
  if (!tri_dev || ntri <= 0 || !inc_start_dev || !inc_tri_dev || !tri_normals_ws_dev || !normals_dev)
    return fail(SYN_ERR_INVALID, "syn_mesh_normals: null pointer or no triangles");
  cudaStream_t st = (cudaStream_t)stream;
  tri_normal_kernel<<<dim3((ntri + 255) / 256, batch), 256, 0, st>>>(m, tri_dev, ntri, tri_normals_ws_dev);
  SYN_LAUNCH_CHECK("tri_normal_kernel");
  vertex_normal_kernel<<<dim3((nver + 255) / 256, batch), 256, 0, st>>>(nver, ntri, tri_normals_ws_dev, inc_start_dev, inc_tri_dev, normals_dev);
  SYN_LAUNCH_CHECK("vertex_normal_kernel");
  return SYN_OK;
}

int syn_mesh_lighting(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch, int nver,
                      const float* normals_dev, const syn_light_cfg_t* cfg, const float* texture_dev, uint32_t* stats_ws_dev,
                      float* colors_dev, void* stream) {
  return mesh_lighting(vertices_dev, stride_mesh, stride_vertex, stride_coord, batch, nver, normals_dev, cfg, texture_dev, 0,
                       stats_ws_dev, colors_dev, stream, "syn_mesh_lighting");
}

int syn_mesh_lighting_textures(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch,
                               int nver, const float* normals_dev, const syn_light_cfg_t* cfg, const float* texture_dev,
                               int64_t texture_stride_mesh, uint32_t* stats_ws_dev, float* colors_dev, void* stream) {
  const char* who = "syn_mesh_lighting_textures";
  if (!texture_dev) return fail(SYN_ERR_INVALID, "%s: null texture", who);
  if (texture_stride_mesh < 0 || (texture_stride_mesh > 0 && texture_stride_mesh < 3LL * nver))
    return fail(SYN_ERR_INVALID, "%s: texture mesh stride %lld (0, or at least 3 * %d)", who, (long long)texture_stride_mesh, nver);
  return mesh_lighting(vertices_dev, stride_mesh, stride_vertex, stride_coord, batch, nver, normals_dev, cfg, texture_dev,
                       texture_stride_mesh, stats_ws_dev, colors_dev, stream, who);
}

int syn_rasterize(uint8_t* image_dev, int height, int width, int channels, const float* vertices_dev, int64_t stride_mesh,
                  int stride_vertex, int stride_coord, int batch, int nver, const int32_t* tri_dev, int ntri,
                  const float* colors_dev, float alpha, int reverse, uint64_t* keys_ws_dev, float* depth_out_dev, void* stream) {
  MeshView m;
  if (int rc = check_mesh(vertices_dev, stride_mesh, stride_vertex, stride_coord, batch, nver, m)) return rc;
  if (!image_dev || !tri_dev || !colors_dev || !keys_ws_dev || height <= 0 || width <= 0 || channels <= 0 || ntri < 0)
    return fail(SYN_ERR_INVALID, "syn_rasterize: null pointer or empty image");
  if (alpha != 1.0f)
    return fail(SYN_ERR_UNSUPPORTED, "syn_rasterize: alpha = %g; only alpha = 1 (the value Sim3DR.rasterize always passes) has an "
                                     "order-free result", (double)alpha);
  cudaStream_t st = (cudaStream_t)stream;
  SYN_CUDA(cudaMemsetAsync(keys_ws_dev, 0, sizeof(uint64_t) * (size_t)batch * height * width, st));
  if (ntri > 0) {
    raster_depth_kernel<false><<<dim3((ntri + 255) / 256, batch), 256, 0, st>>>(m, tri_dev, ntri, width, height,
                                                                         reinterpret_cast<unsigned long long*>(keys_ws_dev), nullptr,
                                                                         nullptr, ImageAxis{});
    SYN_LAUNCH_CHECK("raster_depth_kernel");
  }
  raster_resolve_kernel<<<dim3((width + 31) / 32, (height + 7) / 8), dim3(32, 8), 0, st>>>(
      m, tri_dev, colors_dev, channels, width, height, alpha, reverse, reinterpret_cast<const unsigned long long*>(keys_ws_dev),
      image_dev, depth_out_dev);
  SYN_LAUNCH_CHECK("raster_resolve_kernel");
  return SYN_OK;
}

int syn_render_frames_plan(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int n_meshes, int nver,
                           const int32_t* tri_dev, int ntri, const int32_t* mesh_start_host, int n_frames, int height, int width,
                           int32_t* boxes_dev, int64_t* key_off_dev, void* stream) {
  const char* who = "syn_render_frames_plan";
  MeshView m;
  if (int rc = check_frames(vertices_dev, stride_mesh, stride_vertex, stride_coord, n_meshes, nver, mesh_start_host, n_frames, height,
                            width, m, who))
    return rc;
  if (!tri_dev || ntri < 0 || !boxes_dev || !key_off_dev) return fail(SYN_ERR_INVALID, "%s: null pointer or negative triangle count", who);
  cudaStream_t st = (cudaStream_t)stream;
  SYN_CUDA(cudaMemsetAsync(boxes_dev, 0x7F, sizeof(int32_t) * 4 * (size_t)n_meshes, st));
  if (ntri > 0) {
    mesh_box_kernel<false><<<dim3((ntri + 255) / 256, n_meshes), 256, 0, st>>>(m, tri_dev, ntri, width, height, boxes_dev, ImageAxis{});
    SYN_LAUNCH_CHECK("mesh_box_kernel");
  }
  mesh_box_scan_kernel<<<1, kBoxScanThreads, 0, st>>>(n_meshes, boxes_dev, reinterpret_cast<long long*>(key_off_dev));
  SYN_LAUNCH_CHECK("mesh_box_scan_kernel");
  return SYN_OK;
}

int syn_rasterize_frames(const uint8_t* frames_dev, uint8_t* solid_dev, int n_frames, int height, int width, int channels,
                         const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int n_meshes, int nver,
                         const int32_t* tri_dev, int ntri, const float* colors_dev, int color_channels, const int32_t* mesh_start_host,
                         const int32_t* mesh_start_dev, const int32_t* boxes_dev, const int64_t* key_off_dev, int64_t n_keys,
                         uint64_t* keys_ws_dev, int64_t keys_ws_count, void* stream) {
  const char* who = "syn_rasterize_frames";
  MeshView m;
  if (int rc = check_frames(vertices_dev, stride_mesh, stride_vertex, stride_coord, n_meshes, nver, mesh_start_host, n_frames, height,
                            width, m, who))
    return rc;
  if (!frames_dev || !solid_dev || !tri_dev || !colors_dev || !mesh_start_dev || !boxes_dev || !key_off_dev || !keys_ws_dev || ntri < 0)
    return fail(SYN_ERR_INVALID, "%s: null pointer or negative triangle count", who);
  if (channels <= 0 || channels != color_channels)
    return fail(SYN_ERR_SHAPE, "%s: %d image channels, colours of %d channels", who, channels, color_channels);
  if (n_keys < 0 || keys_ws_count < n_keys)
    return fail(SYN_ERR_SHAPE, "%s: key workspace of %lld slots, the plan needs %lld", who, (long long)keys_ws_count, (long long)n_keys);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(keys_ws_dev);
  const int4* boxes = reinterpret_cast<const int4*>(boxes_dev);
  const long long* off = reinterpret_cast<const long long*>(key_off_dev);
  if (n_keys > 0) {
    SYN_CUDA(cudaMemsetAsync(keys_ws_dev, 0, sizeof(uint64_t) * (size_t)n_keys, st));
    if (ntri > 0) {
      raster_depth_kernel<true><<<dim3((ntri + 255) / 256, n_meshes), 256, 0, st>>>(m, tri_dev, ntri, width, height, keys, boxes, off,
                                                                                    ImageAxis{});
      SYN_LAUNCH_CHECK("raster_depth_kernel");
    }
  }
  raster_resolve_frames_kernel<false><<<dim3((width + 31) / 32, (height + 7) / 8, n_frames), dim3(32, 8), 0, st>>>(
      m, tri_dev, colors_dev, channels, width, height, mesh_start_dev, boxes, off, keys, frames_dev, solid_dev, ImageAxis{});
  SYN_LAUNCH_CHECK("raster_resolve_frames_kernel");
  return SYN_OK;
}

int syn_render_images_plan(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int n_meshes, int nver,
                           const int32_t* tri_dev, int ntri, const int32_t* mesh_start_host, const int32_t* mesh_start_dev,
                           const int64_t* images_host, const int64_t* images_dev, int n_images, int64_t image_bytes, int channels,
                           int32_t* boxes_dev, int64_t* key_off_dev, void* stream) {
  const char* who = "syn_render_images_plan";
  MeshView m;
  ImageAxis ax;
  if (int rc = check_images(vertices_dev, stride_mesh, stride_vertex, stride_coord, n_meshes, nver, mesh_start_host, mesh_start_dev,
                            images_host, images_dev, n_images, image_bytes, channels, m, ax, who))
    return rc;
  if (!tri_dev || ntri < 0 || !boxes_dev || !key_off_dev) return fail(SYN_ERR_INVALID, "%s: null pointer or negative triangle count", who);
  cudaStream_t st = (cudaStream_t)stream;
  SYN_CUDA(cudaMemsetAsync(boxes_dev, 0x7F, sizeof(int32_t) * 4 * (size_t)n_meshes, st));
  if (ntri > 0) {
    mesh_box_kernel<true><<<dim3((ntri + 255) / 256, n_meshes), 256, 0, st>>>(m, tri_dev, ntri, 0, 0, boxes_dev, ax);
    SYN_LAUNCH_CHECK("mesh_box_kernel");
  }
  mesh_box_scan_kernel<<<1, kBoxScanThreads, 0, st>>>(n_meshes, boxes_dev, reinterpret_cast<long long*>(key_off_dev));
  SYN_LAUNCH_CHECK("mesh_box_scan_kernel");
  return SYN_OK;
}

int syn_rasterize_images(const uint8_t* images_dev, uint8_t* solid_dev, int64_t image_bytes, const int64_t* table_host,
                         const int64_t* table_dev, int n_images, int channels, const float* vertices_dev, int64_t stride_mesh,
                         int stride_vertex, int stride_coord, int n_meshes, int nver, const int32_t* tri_dev, int ntri,
                         const float* colors_dev, int color_channels, const int32_t* mesh_start_host, const int32_t* mesh_start_dev,
                         const int32_t* boxes_dev, const int64_t* key_off_dev, int64_t n_keys, uint64_t* keys_ws_dev,
                         int64_t keys_ws_count, void* stream) {
  const char* who = "syn_rasterize_images";
  MeshView m;
  ImageAxis ax;
  if (int rc = check_images(vertices_dev, stride_mesh, stride_vertex, stride_coord, n_meshes, nver, mesh_start_host, mesh_start_dev,
                            table_host, table_dev, n_images, image_bytes, channels, m, ax, who))
    return rc;
  if (!images_dev || !solid_dev || !tri_dev || !colors_dev || !boxes_dev || !key_off_dev || !keys_ws_dev || ntri < 0)
    return fail(SYN_ERR_INVALID, "%s: null pointer or negative triangle count", who);
  if (channels != color_channels)
    return fail(SYN_ERR_SHAPE, "%s: %d image channels, colours of %d channels", who, channels, color_channels);
  if (n_keys < 0 || keys_ws_count < n_keys)
    return fail(SYN_ERR_SHAPE, "%s: key workspace of %lld slots, the plan needs %lld", who, (long long)keys_ws_count, (long long)n_keys);
  // pixel slots from the first image's first byte to the last image's end
  const int64_t first = table_host[0], last = table_host[3 * (n_images - 1)];
  const int64_t slots = (last - first) / channels + table_host[3 * (n_images - 1) + 1] * table_host[3 * (n_images - 1) + 2];
  if ((slots + 255) / 256 > INT32_MAX) return fail(SYN_ERR_SHAPE, "%s: %lld pixel slots exceed one launch's grid", who, (long long)slots);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(keys_ws_dev);
  const int4* boxes = reinterpret_cast<const int4*>(boxes_dev);
  const long long* off = reinterpret_cast<const long long*>(key_off_dev);
  if (n_keys > 0) {
    SYN_CUDA(cudaMemsetAsync(keys_ws_dev, 0, sizeof(uint64_t) * (size_t)n_keys, st));
    if (ntri > 0) {
      raster_depth_kernel<true, true><<<dim3((ntri + 255) / 256, n_meshes), 256, 0, st>>>(m, tri_dev, ntri, 0, 0, keys, boxes, off, ax);
      SYN_LAUNCH_CHECK("raster_depth_kernel");
    }
  }
  raster_resolve_frames_kernel<true><<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(m, tri_dev, colors_dev, channels, 0, 0, mesh_start_dev,
                                                                                     boxes, off, keys, images_dev, solid_dev, ax);
  SYN_LAUNCH_CHECK("raster_resolve_frames_kernel");
  return SYN_OK;
}

int syn_add_weighted_u8(const uint8_t* a_dev, const uint8_t* b_dev, double alpha, uint8_t* out_dev, int64_t n, void* stream) {
  if (!a_dev || !b_dev || !out_dev || n < 0) return fail(SYN_ERR_INVALID, "syn_add_weighted_u8: null pointer or negative size");
  if (!std::isfinite(alpha)) return fail(SYN_ERR_INVALID, "syn_add_weighted_u8: alpha %g is not finite", alpha);
  if (n == 0) return SYN_OK;
  const bool vec = n % 16 == 0 && ((reinterpret_cast<uintptr_t>(a_dev) | reinterpret_cast<uintptr_t>(b_dev) |
                                    reinterpret_cast<uintptr_t>(out_dev)) & 15) == 0;
  const long long work = vec ? n / 16 : n;
  const int blocks = (int)std::min<long long>((work + 255) / 256, 1 << 20);
  add_weighted_u8_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a_dev, b_dev, alpha, out_dev, (long long)n, vec ? 1 : 0);
  SYN_LAUNCH_CHECK("add_weighted_u8_kernel");
  return SYN_OK;
}

int syn_draw_lines(uint8_t* images_dev, int64_t image_bytes, const int64_t* frames_host, const int64_t* frames_dev, int n_frames,
                   const int32_t* seg_start_host, const int32_t* seg_start_dev, const int32_t* segs_dev, int n_segs, int thickness,
                   int line_type, void* stream) {
  const char* who = "syn_draw_lines";
  if (!images_dev || !frames_host || !frames_dev || !seg_start_host || !seg_start_dev || (n_segs > 0 && !segs_dev))
    return fail(SYN_ERR_INVALID, "%s: null pointer", who);
  if (n_frames <= 0 || n_segs < 0 || image_bytes < 0)
    return fail(SYN_ERR_INVALID, "%s: %d frames, %d segments, %lld image bytes", who, n_frames, n_segs, (long long)image_bytes);
  if (thickness != dmath::kThickness)
    return fail(SYN_ERR_UNSUPPORTED, "%s: thickness %d (only %d, the thickness of draw_axis, is restated)", who, thickness,
                dmath::kThickness);
  if (line_type != 8) return fail(SYN_ERR_UNSUPPORTED, "%s: line type %d (only LINE_8 = 8)", who, line_type);
  if (seg_start_host[0] != 0 || seg_start_host[n_frames] != n_segs)
    return fail(SYN_ERR_SHAPE, "%s: seg_start runs from %d to %d, must run from 0 to %d segments", who, seg_start_host[0],
                seg_start_host[n_frames], n_segs);
  for (int f = 0; f < n_frames; ++f)
    if (seg_start_host[f + 1] < seg_start_host[f])
      return fail(SYN_ERR_SHAPE, "%s: seg_start is not monotone at frame %d (%d after %d)", who, f, seg_start_host[f + 1],
                  seg_start_host[f]);
  int64_t end = 0;                                   // the frames in memory order, disjoint, inside the image bytes
  for (int f = 0; f < n_frames; ++f) {
    const int64_t off = frames_host[3 * f], h = frames_host[3 * f + 1], w = frames_host[3 * f + 2];
    if (h < 1 || w < 1 || h > INT32_MAX || w > INT32_MAX)
      return fail(SYN_ERR_SHAPE, "%s: frame %d is %lldx%lld", who, f, (long long)h, (long long)w);
    if (off < end || off > image_bytes || h > (image_bytes - off) / 3 / w)
      return fail(SYN_ERR_SHAPE, "%s: frame %d (%lldx%lld at byte %lld) does not fit the %lld image bytes after the frame before it", who,
                  f, (long long)h, (long long)w, (long long)off, (long long)image_bytes);
    end = off + 3 * h * w;
  }
  if (n_segs == 0) return SYN_OK;
  draw_lines_kernel<<<n_frames, kDrawThreads, 0, (cudaStream_t)stream>>>(images_dev, reinterpret_cast<const long long*>(frames_dev),
                                                                       seg_start_dev, segs_dev);
  SYN_LAUNCH_CHECK("draw_lines_kernel");
  return SYN_OK;
}

int syn_uv_sample(const uint8_t* maps_dev, int64_t map_bytes, const int64_t* maps_host, const int64_t* maps_table_dev, int n_maps,
                  const int32_t* texels_host, const int32_t* texels_dev, int n_keep, const int32_t* face_map_host,
                  const int32_t* face_map_dev, int n_faces, float* texture_dev, int64_t* colors_dev, void* stream) {
  const char* who = "syn_uv_sample";
  if (!maps_dev || !maps_host || !maps_table_dev || !texels_host || !texels_dev || !face_map_host || !face_map_dev ||
      (!texture_dev && !colors_dev))
    return fail(SYN_ERR_INVALID, "%s: null pointer", who);
  if (reinterpret_cast<uintptr_t>(texels_dev) % 8)
    return fail(SYN_ERR_INVALID, "%s: texels_dev is not 8-byte aligned", who);
  if (n_maps < 1 || n_keep < 1 || n_faces < 1 || n_faces > 65535 || map_bytes < 0)
    return fail(SYN_ERR_INVALID, "%s: %d maps, %d kept vertices, %d faces (1..65535), %lld map bytes", who, n_maps, n_keep, n_faces,
                (long long)map_bytes);
  int64_t end = 0;                                   // the maps in memory order, disjoint, inside the map bytes
  for (int m = 0; m < n_maps; ++m) {
    const int64_t off = maps_host[3 * m], h = maps_host[3 * m + 1], w = maps_host[3 * m + 2];
    if (h < 1 || w < 1 || h > INT32_MAX || w > INT32_MAX) return fail(SYN_ERR_SHAPE, "%s: map %d is %lldx%lld", who, m, (long long)h, (long long)w);
    if (off < end || off > map_bytes || h > (map_bytes - off) / 3 / w)
      return fail(SYN_ERR_SHAPE, "%s: map %d (%lldx%lld at byte %lld) does not fit the %lld map bytes after the map before it", who, m,
                  (long long)h, (long long)w, (long long)off, (long long)map_bytes);
    end = off + 3 * h * w;
    const int32_t* t = texels_host + 2 * (int64_t)m * n_keep;
    for (int i = 0; i < n_keep; ++i)
      if (t[2 * i] < 0 || t[2 * i] >= h || t[2 * i + 1] < 0 || t[2 * i + 1] >= w)
        return fail(SYN_ERR_SHAPE, "%s: texel %d of map %d is (%d, %d), outside its %lldx%lld", who, i, m, t[2 * i], t[2 * i + 1],
                    (long long)h, (long long)w);
  }
  for (int f = 0; f < n_faces; ++f)
    if (face_map_host[f] < 0 || face_map_host[f] >= n_maps)
      return fail(SYN_ERR_SHAPE, "%s: face %d names map %d of %d", who, f, face_map_host[f], n_maps);
  uv_sample_kernel<<<dim3((n_keep + kUvThreads - 1) / kUvThreads, n_faces), kUvThreads, 0, (cudaStream_t)stream>>>(
      maps_dev, reinterpret_cast<const long long*>(maps_table_dev), texels_dev, n_keep, face_map_dev, texture_dev,
      reinterpret_cast<long long*>(colors_dev));
  SYN_LAUNCH_CHECK("uv_sample_kernel");
  return SYN_OK;
}

int64_t syn_obj_workspace_size(int batch, int n_lines, int ntri) {
  if (batch < 1 || batch > 65535 || n_lines < 0 || ntri < 0 || (int64_t)batch * obj_blocks(n_lines) + obj_blocks(ntri) > INT32_MAX)
    return -1;
  return (int64_t)sizeof(long long) * (1 + batch * obj_blocks(n_lines) + obj_blocks(ntri));
}

int syn_obj_plan(const syn_obj_desc_t* desc, void* ws_dev, int64_t ws_bytes, int64_t* offsets_dev, void* stream) {
  const char* who = "syn_obj_plan";
  ObjArgs a;
  if (int rc = check_obj(desc, ws_dev, ws_bytes, a, who)) return rc;
  if (!offsets_dev) return fail(SYN_ERR_INVALID, "%s: null pointer", who);
  cudaStream_t st = (cudaStream_t)stream;
  long long* ws = static_cast<long long*>(ws_dev);
  const long long blocks = (long long)a.batch * a.vblocks + a.tblocks;
  if (blocks > 0) {
    obj_len_kernel<<<(unsigned)blocks, kObjThreads, 0, st>>>(a, ws + 1);
    SYN_LAUNCH_CHECK("obj_len_kernel");
  }
  obj_scan_kernel<<<1, kObjScanThreads, 0, st>>>(a.batch, a.vblocks, a.tblocks, ws, reinterpret_cast<long long*>(offsets_dev));
  SYN_LAUNCH_CHECK("obj_scan_kernel");
  return SYN_OK;
}

int syn_obj_write(const syn_obj_desc_t* desc, const void* ws_dev, int64_t ws_bytes, const int64_t* offsets_dev, uint8_t* out_dev,
                  int64_t out_bytes, void* stream) {
  const char* who = "syn_obj_write";
  ObjArgs a;
  if (int rc = check_obj(desc, ws_dev, ws_bytes, a, who)) return rc;
  if (!offsets_dev || !out_dev || out_bytes < 0)
    return fail(SYN_ERR_INVALID, "%s: null pointer or %lld output bytes", who, (long long)out_bytes);
  cudaStream_t st = (cudaStream_t)stream;
  const long long* ws = static_cast<const long long*>(ws_dev);
  const long long* off = reinterpret_cast<const long long*>(offsets_dev);
  char* out = reinterpret_cast<char*>(out_dev);
  const long long blocks = (long long)a.batch * a.vblocks + a.tblocks;
  if (blocks > 0) {
    obj_write_kernel<<<(unsigned)blocks, kObjThreads, 0, st>>>(a, ws, off, out, (long long)out_bytes);
    SYN_LAUNCH_CHECK("obj_write_kernel");
  }
  if (a.batch > 1 && a.ntri > 0) {
    obj_copy_kernel<<<dim3(128, a.batch - 1), kObjThreads, 0, st>>>(ws, off, out, (long long)out_bytes);
    SYN_LAUNCH_CHECK("obj_copy_kernel");
  }
  return SYN_OK;
}

int syn_nms(const float* dets_dev, int n, double thresh, int mode, uint64_t* mask_ws_dev, int32_t* keep_dev, int32_t* n_keep_dev,
            void* stream) {
  if (n < 0 || !n_keep_dev || (n > 0 && (!dets_dev || !mask_ws_dev || !keep_dev))) return fail(SYN_ERR_INVALID, "syn_nms: bad argument");
  if (mode != SYN_NMS_CPU_NMS && mode != SYN_NMS_PY_CPU_NMS) return fail(SYN_ERR_INVALID, "syn_nms: unknown mode %d", mode);
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {                                   // nms_wrapper.py:16-17: no detections, empty keep list
    SYN_CUDA(cudaMemsetAsync(n_keep_dev, 0, sizeof(int32_t), st));
    return SYN_OK;
  }
  const int words = (n + 63) / 64;
  if ((size_t)words * 8 > 200 * 1024) return fail(SYN_ERR_SHAPE, "syn_nms: %d boxes exceed the scan kernel's shared memory", n);
  nms_mask_kernel<<<dim3((words + 31) / 32, (n + 7) / 8), dim3(32, 8), 0, st>>>(dets_dev, n, thresh, mode == SYN_NMS_CPU_NMS ? 1 : 0,
                                                                               reinterpret_cast<unsigned long long*>(mask_ws_dev), nullptr);
  SYN_LAUNCH_CHECK("nms_mask_kernel");
  if (words * 8 > 48 * 1024)
    SYN_CUDA(cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, words * 8));
  nms_scan_kernel<<<1, kNmsScanThreads, words * 8, st>>>(reinterpret_cast<const unsigned long long*>(mask_ws_dev), n, keep_dev, n_keep_dev,
                                                         nullptr);
  SYN_LAUNCH_CHECK("nms_scan_kernel");
  return SYN_OK;
}

int syn_nms_batch(const float* dets_dev, const int32_t* n_dev, int n_frames, int rows_per_frame, double thresh, int mode,
                  uint64_t* mask_ws_dev, int32_t* keep_dev, int32_t* n_keep_dev, void* stream) {
  if (!dets_dev || !n_dev || !mask_ws_dev || !keep_dev || !n_keep_dev || n_frames <= 0 || rows_per_frame <= 0)
    return fail(SYN_ERR_INVALID, "syn_nms_batch: null pointer, no frame or no row");
  if (n_frames > SYN_FB_MAX_FRAMES) return fail(SYN_ERR_INVALID, "syn_nms_batch: %d frames, at most %d per call", n_frames, SYN_FB_MAX_FRAMES);
  if (mode != SYN_NMS_CPU_NMS && mode != SYN_NMS_PY_CPU_NMS) return fail(SYN_ERR_INVALID, "syn_nms_batch: unknown mode %d", mode);
  cudaStream_t st = (cudaStream_t)stream;
  const int n = rows_per_frame, words = (n + 63) / 64;
  if ((size_t)words * 8 > 200 * 1024) return fail(SYN_ERR_SHAPE, "syn_nms_batch: %d boxes exceed the scan kernel's shared memory", n);
  nms_mask_kernel<<<dim3((words + 31) / 32, (n + 7) / 8, n_frames), dim3(32, 8), 0, st>>>(
      dets_dev, n, thresh, mode == SYN_NMS_CPU_NMS ? 1 : 0, reinterpret_cast<unsigned long long*>(mask_ws_dev), n_dev);
  SYN_LAUNCH_CHECK("nms_mask_kernel");
  if (words * 8 > 48 * 1024)
    SYN_CUDA(cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, words * 8));
  nms_scan_kernel<<<n_frames, kNmsScanThreads, words * 8, st>>>(reinterpret_cast<const unsigned long long*>(mask_ws_dev), n, keep_dev,
                                                                n_keep_dev, n_dev);
  SYN_LAUNCH_CHECK("nms_scan_kernel");
  return SYN_OK;
}

int64_t syn_crop_resize_plan_size(int batch, int out_h, int out_w, int mode) {
  if (batch <= 0 || out_h <= 0 || out_w <= 0 || (mode != SYN_INTER_LINEAR && mode != SYN_INTER_LANCZOS4)) return -1;
  return rsz::plan_bytes(batch, out_h, out_w, rsz::taps_of(mode));
}

int syn_crop_resize_plan_host(const int32_t* rois_host, int batch, int out_h, int out_w, int mode, void* plan_out,
                              int64_t plan_bytes) {
  return crop_plan(rois_host, nullptr, 0, batch, out_h, out_w, mode, plan_out, plan_bytes, "syn_crop_resize_plan_host");
}

int syn_crop_resize_plan_frames_host(const int32_t* rois_host, const int32_t* frames_host, int n_frames, int batch, int out_h,
                                     int out_w, int mode, void* plan_out, int64_t plan_bytes) {
  const char* who = "syn_crop_resize_plan_frames_host";
  if (!frames_host || n_frames <= 0) return fail(SYN_ERR_INVALID, "%s: null frame list or no frame", who);
  return crop_plan(rois_host, frames_host, n_frames, batch, out_h, out_w, mode, plan_out, plan_bytes, who);
}

int syn_crop_resize(const uint8_t* image_dev, int height, int width, int channels, const void* plan_dev, int batch, int out_h,
                    int out_w, int mode, uint8_t* out_dev, int64_t stride_roi, int64_t stride_y, int64_t stride_x, int64_t stride_c,
                    void* stream) {
  return crop_launch(image_dev, 0, height, width, channels, plan_dev, batch, out_h, out_w, mode, out_dev, stride_roi, stride_y,
                     stride_x, stride_c, (cudaStream_t)stream, "syn_crop_resize");
}

int syn_crop_resize_batch(const uint8_t* images_dev, int n_frames, int height, int width, int channels, const void* plan_dev,
                          int batch, int out_h, int out_w, int mode, uint8_t* out_dev, int64_t stride_roi, int64_t stride_y,
                          int64_t stride_x, int64_t stride_c, void* stream) {
  if (n_frames <= 0) return fail(SYN_ERR_INVALID, "syn_crop_resize_batch: %d frames", n_frames);
  return crop_launch(images_dev, n_frames, height, width, channels, plan_dev, batch, out_h, out_w, mode, out_dev, stride_roi,
                     stride_y, stride_x, stride_c, (cudaStream_t)stream, "syn_crop_resize_batch");
}

int64_t syn_crop_resize_images_plan_size(int batch, const int32_t* out_h_host, const int32_t* out_w_host, int mode) {
  if (batch <= 0 || !out_h_host || !out_w_host || (mode != SYN_INTER_LINEAR && mode != SYN_INTER_LANCZOS4)) return -1;
  int64_t n = (int64_t)sizeof(CropImagesRoi) * batch;
  for (int b = 0; b < batch; ++b) {
    if (out_h_host[b] < 1 || out_w_host[b] < 1) return -1;
    n += rsz::plan_bytes(1, out_h_host[b], out_w_host[b], rsz::taps_of(mode));
  }
  return n;
}

int syn_crop_resize_plan_images_host(const int32_t* rois_host, const int32_t* images_host, int n_images, const int32_t* heights_host,
                                     const int32_t* widths_host, int batch, const int32_t* out_h_host, const int32_t* out_w_host,
                                     int mode, void* plan_out, int64_t plan_bytes) {
  const char* who = "syn_crop_resize_plan_images_host";
  if (!rois_host || !images_host || !heights_host || !widths_host || !out_h_host || !out_w_host || !plan_out || batch <= 0)
    return fail(SYN_ERR_INVALID, "%s: null pointer or empty batch", who);
  if (n_images <= 0) return fail(SYN_ERR_INVALID, "%s: %d images", who, n_images);
  if (mode != SYN_INTER_LINEAR && mode != SYN_INTER_LANCZOS4)
    return fail(SYN_ERR_UNSUPPORTED, "%s: interpolation %d (only INTER_LINEAR = 1 and INTER_LANCZOS4 = 4)", who, mode);
  for (int i = 0; i < n_images; ++i)
    if (heights_host[i] < 1 || widths_host[i] < 1) return fail(SYN_ERR_INVALID, "%s: image %d is %dx%d", who, i, heights_host[i], widths_host[i]);
  for (int b = 0; b < batch; ++b) {
    const int32_t* r = rois_host + 4 * b;
    if (out_h_host[b] < 1 || out_w_host[b] < 1) return fail(SYN_ERR_INVALID, "%s: ROI %d output %dx%d", who, b, out_h_host[b], out_w_host[b]);
    if (r[2] <= r[0] || r[3] <= r[1]) return fail(SYN_ERR_SHAPE, "%s: ROI %d (%d,%d,%d,%d) is empty", who, b, r[0], r[1], r[2], r[3]);
    if (images_host[b] < 0 || images_host[b] >= n_images)
      return fail(SYN_ERR_SHAPE, "%s: ROI %d names image %d of %d", who, b, images_host[b], n_images);
  }
  const int64_t need = syn_crop_resize_images_plan_size(batch, out_h_host, out_w_host, mode);
  if (plan_bytes < need) return fail(SYN_ERR_SHAPE, "%s: plan buffer of %lld bytes, %lld needed", who, (long long)plan_bytes, (long long)need);
  std::vector<long long> src(n_images + 1, 0);
  for (int i = 0; i < n_images; ++i) src[i + 1] = src[i] + 3LL * heights_host[i] * widths_host[i];
  CropImagesRoi* hdr = static_cast<CropImagesRoi*>(plan_out);
  long long out = 0, at = (long long)sizeof(CropImagesRoi) * batch;
  for (int b = 0; b < batch; ++b) {
    const int im = images_host[b];
    hdr[b] = CropImagesRoi{src[im], heights_host[im], widths_host[im], out_h_host[b], out_w_host[b], out, at};
    rsz::build_plan(rois_host + 4 * b, 1, out_h_host[b], out_w_host[b], mode, static_cast<char*>(plan_out) + at);
    out += 3LL * out_h_host[b] * out_w_host[b];
    at += rsz::plan_bytes(1, out_h_host[b], out_w_host[b], rsz::taps_of(mode));
  }
  return SYN_OK;
}

int syn_crop_resize_images(const uint8_t* images_dev, const void* plan_dev, int batch, const int32_t* out_h_host, const int32_t* out_w_host,
                           int mode, int planar, uint8_t* out_dev, void* stream) {
  const char* who = "syn_crop_resize_images";
  if (!images_dev || !plan_dev || !out_dev || !out_h_host || !out_w_host || batch <= 0)
    return fail(SYN_ERR_INVALID, "%s: null pointer or empty batch", who);
  if (mode != SYN_INTER_LINEAR && mode != SYN_INTER_LANCZOS4)
    return fail(SYN_ERR_UNSUPPORTED, "%s: interpolation %d (only INTER_LINEAR = 1 and INTER_LANCZOS4 = 4)", who, mode);
  if (planar != 0 && planar != 1) return fail(SYN_ERR_INVALID, "%s: planar = %d", who, planar);
  if (batch > 65535) return fail(SYN_ERR_SHAPE, "%s: %d ROIs exceed one launch's grid", who, batch);
  int mh = 0, mw = 0;
  for (int b = 0; b < batch; ++b) {
    if (out_h_host[b] < 1 || out_w_host[b] < 1) return fail(SYN_ERR_INVALID, "%s: ROI %d output %dx%d", who, b, out_h_host[b], out_w_host[b]);
    mh = std::max(mh, (int)out_h_host[b]);
    mw = std::max(mw, (int)out_w_host[b]);
  }
  const dim3 grid((mw + kResizeBX - 1) / kResizeBX, (mh + kResizeBY - 1) / kResizeBY, batch), block(kResizeBX, kResizeBY);
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == SYN_INTER_LANCZOS4) crop_resize_images_kernel<8><<<grid, block, 0, st>>>(images_dev, plan_dev, out_dev, planar);
  else crop_resize_images_kernel<2><<<grid, block, 0, st>>>(images_dev, plan_dev, out_dev, planar);
  SYN_LAUNCH_CHECK("crop_resize_images_kernel");
  return SYN_OK;
}

int syn_faceboxes_num_priors(int im_height, int im_width) {
  if (im_height <= 0 || im_width <= 0) return -1;
  return faceboxes_num_priors(im_height, im_width);
}

int syn_faceboxes_decode(const float* loc_dev, const float* conf_dev, int im_height, int im_width, float box_scale_w,
                         float box_scale_h, float scale, float conf_thresh, int top_k, int32_t* cand_ws_dev, float* dets_dev,
                         int32_t* n_dets_dev, void* stream) {
  if (!loc_dev || !conf_dev || !cand_ws_dev || !dets_dev || !n_dets_dev || im_height <= 0 || im_width <= 0 || top_k <= 0 || !(scale > 0.f))
    return fail(SYN_ERR_INVALID, "syn_faceboxes_decode: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int np = faceboxes_num_priors(im_height, im_width);
  SYN_CUDA(cudaMemsetAsync(n_dets_dev, 0, sizeof(int32_t), st));
  SYN_CUDA(cudaMemsetAsync(cand_ws_dev, 0, sizeof(int32_t), st));
  return decode_launch(loc_dev, conf_dev, decode_frame(FbDecodeFrames{}, 0, im_height, im_width, box_scale_w, box_scale_h, scale, 0, 0, 1),
                       1, np, conf_thresh, top_k, cand_ws_dev, dets_dev, n_dets_dev, st);
}

int syn_faceboxes_decode_batch(const float* loc_dev, const float* conf_dev, int n_frames, int im_height, int im_width,
                               float box_scale_w, float box_scale_h, float scale, float conf_thresh, int top_k, int32_t* cand_ws_dev,
                               float* dets_dev, int32_t* n_dets_dev, void* stream) {
  if (!loc_dev || !conf_dev || !cand_ws_dev || !dets_dev || !n_dets_dev || n_frames <= 0 || im_height <= 0 || im_width <= 0 ||
      top_k <= 0 || !(scale > 0.f))
    return fail(SYN_ERR_INVALID, "syn_faceboxes_decode_batch: bad argument");
  if (n_frames > SYN_FB_MAX_FRAMES)
    return fail(SYN_ERR_INVALID, "syn_faceboxes_decode_batch: %d frames, at most %d per call", n_frames, SYN_FB_MAX_FRAMES);
  cudaStream_t st = (cudaStream_t)stream;
  const int np = faceboxes_num_priors(im_height, im_width);
  FbDecodeFrames t{};
  for (int f = 0; f < n_frames; ++f)                     // frame f: rows f * np.., candidates in its (np + 1) block
    t = decode_frame(t, f, im_height, im_width, box_scale_w, box_scale_h, scale, f * np, f * (np + 1), f * (np + 1) + 1);
  SYN_CUDA(cudaMemsetAsync(n_dets_dev, 0, sizeof(int32_t) * n_frames, st));
  SYN_CUDA(cudaMemset2DAsync(cand_ws_dev, sizeof(int32_t) * (np + 1), 0, sizeof(int32_t), n_frames, st));   // every frame's count
  return decode_launch(loc_dev, conf_dev, t, n_frames, np, conf_thresh, top_k, cand_ws_dev, dets_dev, n_dets_dev, st);
}

int syn_faceboxes_decode_images(const float* loc_dev, const float* conf_dev, int n_images, const int32_t* heights_host,
                                const int32_t* widths_host, const float* scale_host, float conf_thresh, int top_k, int32_t* cand_ws_dev,
                                float* dets_dev, int32_t* n_dets_dev, void* stream) {
  const char* who = "syn_faceboxes_decode_images";
  if (!loc_dev || !conf_dev || !heights_host || !widths_host || !scale_host || !cand_ws_dev || !dets_dev || !n_dets_dev || top_k <= 0)
    return fail(SYN_ERR_INVALID, "%s: null pointer or top_k < 1", who);
  if (n_images <= 0 || n_images > SYN_FB_MAX_FRAMES)
    return fail(SYN_ERR_INVALID, "%s: %d images, 1..%d per call", who, n_images, SYN_FB_MAX_FRAMES);
  FbDecodeFrames t{};
  int p0 = 0, np_max = 0;
  for (int f = 0; f < n_images; ++f) {
    if (heights_host[f] < 1 || widths_host[f] < 1 || !(scale_host[f] > 0.f))
      return fail(SYN_ERR_INVALID, "%s: image %d is %dx%d at scale %g", who, f, heights_host[f], widths_host[f], (double)scale_host[f]);
    const int np = faceboxes_num_priors(heights_host[f], widths_host[f]);
    // priors at p0.. of the packed (sum P) rows; the n_images counts first in cand_ws, then every image's indices
    t = decode_frame(t, f, heights_host[f], widths_host[f], (float)widths_host[f], (float)heights_host[f], scale_host[f], p0, f,
                     n_images + p0);
    p0 += np;
    np_max = std::max(np_max, np);
  }
  cudaStream_t st = (cudaStream_t)stream;
  SYN_CUDA(cudaMemsetAsync(n_dets_dev, 0, sizeof(int32_t) * n_images, st));
  SYN_CUDA(cudaMemsetAsync(cand_ws_dev, 0, sizeof(int32_t) * n_images, st));
  return decode_launch(loc_dev, conf_dev, t, n_images, np_max, conf_thresh, top_k, cand_ws_dev, dets_dev, n_dets_dev, st);
}

}  // extern "C"

// ---- the detector network: host side (FaceBoxes/models/faceboxes.py:68-150) ------------------------------------------------
namespace {

struct FbLayer { const char* name; int cin, cout, k, stride, pad, bn, act; };
// execution order; inception layers are 2 + 7 * block + {0 branch1x1, 1 branch1x1_2, 2 branch3x3_reduce, 3 branch3x3,
// 4 branch3x3_reduce_2, 5 branch3x3_2, 6 branch3x3_3} (faceboxes.py:21-47)
const FbLayer kFbLayers[33] = {
    {"conv1", 3, 24, 7, 4, 3, 1, 2},         {"conv2", 48, 64, 5, 2, 2, 1, 2},
    {"inception1.branch1x1", 128, 32, 1, 1, 0, 1, 1},       {"inception1.branch1x1_2", 128, 32, 1, 1, 0, 1, 1},
    {"inception1.branch3x3_reduce", 128, 24, 1, 1, 0, 1, 1}, {"inception1.branch3x3", 24, 32, 3, 1, 1, 1, 1},
    {"inception1.branch3x3_reduce_2", 128, 24, 1, 1, 0, 1, 1}, {"inception1.branch3x3_2", 24, 32, 3, 1, 1, 1, 1},
    {"inception1.branch3x3_3", 32, 32, 3, 1, 1, 1, 1},
    {"inception2.branch1x1", 128, 32, 1, 1, 0, 1, 1},       {"inception2.branch1x1_2", 128, 32, 1, 1, 0, 1, 1},
    {"inception2.branch3x3_reduce", 128, 24, 1, 1, 0, 1, 1}, {"inception2.branch3x3", 24, 32, 3, 1, 1, 1, 1},
    {"inception2.branch3x3_reduce_2", 128, 24, 1, 1, 0, 1, 1}, {"inception2.branch3x3_2", 24, 32, 3, 1, 1, 1, 1},
    {"inception2.branch3x3_3", 32, 32, 3, 1, 1, 1, 1},
    {"inception3.branch1x1", 128, 32, 1, 1, 0, 1, 1},       {"inception3.branch1x1_2", 128, 32, 1, 1, 0, 1, 1},
    {"inception3.branch3x3_reduce", 128, 24, 1, 1, 0, 1, 1}, {"inception3.branch3x3", 24, 32, 3, 1, 1, 1, 1},
    {"inception3.branch3x3_reduce_2", 128, 24, 1, 1, 0, 1, 1}, {"inception3.branch3x3_2", 24, 32, 3, 1, 1, 1, 1},
    {"inception3.branch3x3_3", 32, 32, 3, 1, 1, 1, 1},
    {"conv3_1", 128, 128, 1, 1, 0, 1, 1},    {"conv3_2", 128, 256, 3, 2, 1, 1, 1},
    {"conv4_1", 256, 128, 1, 1, 0, 1, 1},    {"conv4_2", 128, 256, 3, 2, 1, 1, 1},
    {"loc.0", 128, 84, 3, 1, 1, 0, 0},       {"loc.1", 256, 4, 3, 1, 1, 0, 0},       {"loc.2", 256, 4, 3, 1, 1, 0, 0},
    {"conf.0", 128, 42, 3, 1, 1, 0, 0},      {"conf.1", 256, 2, 3, 1, 1, 0, 0},      {"conf.2", 256, 2, 3, 1, 1, 0, 0},
};

inline int conv_out(int n, int k, int s, int p) { return (n + 2 * p - k) / s + 1; }

}  // namespace

// map sizes of the network on the frame axis: 0 image, 1 conv1, 2 pool1, 3 conv2, 4 / 5 / 6 detection sources 0 / 1 / 2,
// 7 / 8 / 9 the heads' view of sources 0 / 1 / 2 (their frames' slices of the packed prior axis)
constexpr int kFbLevels = 10;

struct syn_fb {
  int device = 0;
  std::vector<float> w[33], b[33];          // folded [K][cout] weights and bias, host
  bool set[33] = {};
  float* d_w[33] = {};
  float* d_b[33] = {};
  bool committed = false;
  // activation workspace, grown (never shrunk) to the bytes a call needs
  float *c1 = nullptr, *p1 = nullptr, *c2 = nullptr, *xa = nullptr, *xb = nullptr, *avg = nullptr, *r1 = nullptr, *r2 = nullptr,
        *t3 = nullptr, *c31 = nullptr, *c32 = nullptr, *c41 = nullptr, *c42 = nullptr;
  size_t ws_sizes[13] = {};                 // bytes of c1 ... c42, in that order
  // frame-axis geometry, FbLevel[kFbLevels][frames]: built on the host per call, one copy to the device
  FbLevel geo_host[kFbLevels * SYN_FB_MAX_FRAMES] = {};
  FbLevel* geo_dev = nullptr;
  int fill_on_grow = -1;                    // debug: byte every workspace growth fills its new buffers with (-1: off)
  int64_t launches = 0;
};

namespace {

void fb_free_ws(syn_fb* f) {
  float** bufs[] = {&f->c1, &f->p1, &f->c2, &f->xa, &f->xb, &f->avg, &f->r1, &f->r2, &f->t3, &f->c31, &f->c32, &f->c41, &f->c42};
  for (float** q : bufs) { cudaFree(*q); *q = nullptr; }
  for (size_t& b : f->ws_sizes) b = 0;
  cudaFree(f->geo_dev);
  f->geo_dev = nullptr;
}

struct FbGeom { int h1, w1, hp1, wp1, h2, w2, h3, w3, h4, w4, h5, w5; };
inline FbGeom fb_geom(int h, int w) {
  FbGeom g;
  g.h1 = conv_out(h, 7, 4, 3); g.w1 = conv_out(w, 7, 4, 3);
  g.hp1 = conv_out(g.h1, 3, 2, 1); g.wp1 = conv_out(g.w1, 3, 2, 1);
  g.h2 = conv_out(g.hp1, 5, 2, 2); g.w2 = conv_out(g.wp1, 5, 2, 2);
  g.h3 = conv_out(g.h2, 3, 2, 1); g.w3 = conv_out(g.w2, 3, 2, 1);
  g.h4 = conv_out(g.h3, 3, 2, 1); g.w4 = conv_out(g.w3, 3, 2, 1);
  g.h5 = conv_out(g.h4, 3, 2, 1); g.w5 = conv_out(g.w4, 3, 2, 1);
  return g;
}

// Pixels of every level summed over the frames of a call -> every buffer is the packed map of its level.  A buffer that
// is too small for the call is reallocated with the device idle (like Workspace::ensure of the backbones); one that is
// large enough is kept, so a stream of calls of different sizes stops allocating once it has met its largest.
int fb_workspace(syn_fb* f, const size_t* pix, cudaStream_t st, const char* who, int height, int width) {
  const size_t floats[13] = {pix[1] * 48, pix[2] * 48, pix[3] * 128, pix[4] * 128, pix[4] * 128, pix[4] * 128, pix[4] * 24,
                             pix[4] * 24, pix[4] * 32, pix[4] * 128, pix[5] * 256, pix[5] * 128, pix[6] * 256};
  bool fits = f->geo_dev != nullptr;
  for (int k = 0; k < 13; ++k) fits = fits && sizeof(float) * floats[k] <= f->ws_sizes[k];
  if (fits) return SYN_OK;
  if (int rc = refuse_capture(st, "%s: a %dx%d input: the detector workspace" SYN_EAGER_FIRST, who, height, width)) return rc;
  SYN_CUDA(cudaDeviceSynchronize());
  size_t keep[13];
  for (int k = 0; k < 13; ++k) keep[k] = std::max(f->ws_sizes[k], sizeof(float) * floats[k]);
  fb_free_ws(f);
  float** bufs[13] = {&f->c1, &f->p1, &f->c2, &f->xa, &f->xb, &f->avg, &f->r1, &f->r2, &f->t3, &f->c31, &f->c32, &f->c41, &f->c42};
  for (int k = 0; k < 13; ++k) {
    f->ws_sizes[k] = keep[k];
    SYN_CUDA(grow_alloc(bufs[k], f->ws_sizes[k], f->fill_on_grow));
  }
  SYN_CUDA(grow_alloc(&f->geo_dev, sizeof(f->geo_host), f->fill_on_grow < 0 ? -1 : 0));
  return SYN_OK;
}

// The frame axis of one call: its frame count and, per level, the device geometry and the packed pixel count
struct FbFrames {
  int n;
  const FbLevel* geo;      // device FbLevel[kFbLevels][n]
  size_t pix[kFbLevels];
  const FbLevel* level(int l) const { return geo + (size_t)l * n; }
};

// R == nullptr: the one-image kernels on an h x w input.  Otherwise their FRAMES instantiations on the packed maps of
// R->n frames: lin / lout = input / output level.
int fb_conv(syn_fb* f, int idx, const float* x, const uint8_t* x_u8, int h, int w, int cin_stride, int cin_off, float* y,
            int cout_stride, int cout_off, cudaStream_t st, const FbFrames* R = nullptr, int lin = 0, int lout = 0) {
  const FbLayer& L = kFbLayers[idx];
  FbConvArgs a;
  a.x = x; a.x_u8 = x_u8; a.wk = f->d_w[idx]; a.bias = f->d_b[idx]; a.y = y;
  a.h = h; a.w = w; a.cin = L.cin; a.cin_stride = cin_stride; a.cin_off = cin_off;
  a.ho = conv_out(h, L.k, L.stride, L.pad); a.wo = conv_out(w, L.k, L.stride, L.pad);
  a.cout = L.cout; a.cout_stride = cout_stride; a.cout_off = cout_off;
  a.k = L.k; a.stride = L.stride; a.pad = L.pad; a.act = L.act;
  a.mean[0] = 104.f; a.mean[1] = 117.f; a.mean[2] = 123.f;          // FaceBoxes.py:92
  a.frames = R ? R->n : 0;
  a.gin = R ? R->level(lin) : nullptr;
  a.gout = R ? R->level(lout) : nullptr;
  const int M = R ? (int)R->pix[lout] : a.ho * a.wo;
  const dim3 grid((M + FB_BM - 1) / FB_BM, (L.cout + FB_BN - 1) / FB_BN);
  const bool vec = x_u8 == nullptr && L.cin % 4 == 0 && cin_stride % 4 == 0 && cin_off % 4 == 0 && L.cout % 4 == 0 &&
                   (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const bool smalln = L.cout <= FB_SMALLN && L.k * L.k * L.cin >= 512;
  if (R) {
    if (smalln) fb_conv_smalln_kernel<true><<<M, 128, 0, st>>>(a);
    else if (vec) fb_conv_kernel<true, true><<<grid, 256, 0, st>>>(a);
    else fb_conv_kernel<false, true><<<grid, 256, 0, st>>>(a);
  } else {
    if (smalln) fb_conv_smalln_kernel<false><<<M, 128, 0, st>>>(a);
    else if (vec) fb_conv_kernel<true, false><<<grid, 256, 0, st>>>(a);
    else fb_conv_kernel<false, false><<<grid, 256, 0, st>>>(a);
  }
  SYN_LAUNCH_CHECK("fb_conv_kernel");
  ++f->launches;
  return SYN_OK;
}

// A debug run (syn_fb_debug_forward_until): the production launch sequence, stopped right after launch `stage`, whose
// whole destination tensor is copied to `out` on the same stream.  Production calls pass nullptr.
constexpr int kFbStages = 39;
struct FbStop {
  int stage;
  float* out;
  int64_t numel;
};

int fb_stop_copy(const FbStop* d, const float* src, size_t n, cudaStream_t st) {
  if (d->numel != (int64_t)n)
    return fail(SYN_ERR_SHAPE, "syn_fb_debug_forward_until: stage %d writes %lld floats, out_numel is %lld", d->stage,
                (long long)n, (long long)d->numel);
  SYN_CUDA(cudaMemcpyAsync(d->out, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return SYN_OK;
}

// after launch s: return from the enclosing function if a debug run stops there
#define SYN_FB_STOP(d, s, src, n, st) \
  do { if ((d) != nullptr && (d)->stage == (s)) return fb_stop_copy((d), (src), (n), (st)); } while (0)

// The argument checks of every detector entry, before anything is read or launched: `frames` == 0 is one image of
// heights[0] x widths[0], else `frames` images of any sizes packed back to back.
int fb_check(const syn_fb* f, const uint8_t* image_dev, int frames, const int32_t* heights, const int32_t* widths, const float* loc_dev,
             const float* conf_dev, const char* who) {
  if (frames < 0 || frames > SYN_FB_MAX_FRAMES) return fail(SYN_ERR_INVALID, "%s: %d frames, 1..%d per call", who, frames, SYN_FB_MAX_FRAMES);
  if (!f || !image_dev || !loc_dev || !conf_dev || !heights || !widths) return fail(SYN_ERR_INVALID, "%s: bad argument", who);
  for (int i = 0; i < std::max(frames, 1); ++i) {
    if (heights[i] <= 0 || widths[i] <= 0) return fail(SYN_ERR_INVALID, "%s: bad argument: image %d is %dx%d", who, i, heights[i], widths[i]);
    const FbGeom g = fb_geom(heights[i], widths[i]);
    if (g.h3 != fb_cells(heights[i], 32) || g.w3 != fb_cells(widths[i], 32) || g.h4 != fb_cells(heights[i], 64) ||
        g.w4 != fb_cells(widths[i], 64) || g.h5 != fb_cells(heights[i], 128) || g.w5 != fb_cells(widths[i], 128))
      return fail(SYN_ERR_SHAPE, "%s: feature maps of a %dx%d input do not match the prior grid", who, heights[i], widths[i]);
  }
  if (!f->committed) return fail(SYN_ERR_STATE, "%s before syn_fb_commit", who);
  return SYN_OK;
}

// syn_fb_forward's launch sequence; `stop` (nullable) ends it early.  Stages are the launches in order, see the table
// at syn_fb_debug_forward_until in include/synergy_b200.h.  frames == 0: one image (heights[0] x widths[0]).  frames >= 1
// (syn_fb_forward_images, and syn_fb_forward_batch with one size): the same 39 launches over the packed maps of every
// frame; loc / conf are the packed (sum P, 4) / (sum P, 2), frame i's priors after those of frames 0 .. i-1.
int fb_forward_body(syn_fb* f, const uint8_t* image_dev, int frames, const int32_t* heights, const int32_t* widths, float* loc_dev,
                    float* conf_dev, cudaStream_t st, const FbStop* stop, const char* who) {
  if (int rc = fb_check(f, image_dev, frames, heights, widths, loc_dev, conf_dev, who)) return rc;
  SYN_CUDA(cudaSetDevice(f->device));
  const int nf = std::max(frames, 1), height = heights[0], width = widths[0];
  // every level of every frame: size, first packed pixel, and for the detection sources the first prior
  FbFrames R{nf, nullptr, {}};
  size_t np_all = 0;
  for (int i = 0; i < nf; ++i) {
    const FbGeom g = fb_geom(heights[i], widths[i]);
    const int hw[kFbLevels][2] = {{heights[i], widths[i]}, {g.h1, g.w1}, {g.hp1, g.wp1}, {g.h2, g.w2}, {g.h3, g.w3}, {g.h4, g.w4},
                                  {g.h5, g.w5}, {g.h3, g.w3}, {g.h4, g.w4}, {g.h5, g.w5}};
    const int s1 = (int)np_all + 21 * g.h3 * g.w3, s2 = s1 + g.h4 * g.w4;
    const int prior[kFbLevels] = {0, 0, 0, 0, 0, 0, 0, (int)np_all, s1, s2}, ppp[kFbLevels] = {0, 0, 0, 0, 0, 0, 0, 21, 1, 1};
    for (int l = 0; l < kFbLevels; ++l) {
      f->geo_host[l * nf + i] = FbLevel{(int)R.pix[l], hw[l][0], hw[l][1], prior[l], ppp[l]};
      R.pix[l] += (size_t)hw[l][0] * hw[l][1];
    }
    np_all += (size_t)faceboxes_num_priors(heights[i], widths[i]);
  }
  if (frames && (R.pix[0] * 3 > (size_t)INT32_MAX || np_all * 4 > (size_t)INT32_MAX))
    return fail(SYN_ERR_SHAPE, "%s: %zu pixels in one call exceed the packed maps' int32 indices", who, R.pix[0]);
  // the frame paths copy this call's geometry from geo_host, which the next call rewrites: a graph would replay the
  // copy from whatever the host buffer then holds.  Only the one-image path (frames == 0) can be captured.
  if (frames)
    if (int rc = refuse_capture(st, "%s: %d frames: the frame paths cannot be captured in a CUDA graph (their per-call geometry "
                                    "is copied from host memory); capture syn_fb_forward, one image per call", who, frames))
      return rc;
  if (int rc = fb_workspace(f, R.pix, st, who, height, width)) return rc;
  R.geo = f->geo_dev;
  if (frames) SYN_CUDA(cudaMemcpyAsync(f->geo_dev, f->geo_host, sizeof(FbLevel) * kFbLevels * nf, cudaMemcpyHostToDevice, st));
  if (stop) {
    // A debug run copies a stage's whole destination, slices that later launches write included: start from a zeroed
    // workspace so that those slices read 0 instead of whatever an earlier call (another image, another frame count) left.
    float* bufs[13] = {f->c1, f->p1, f->c2, f->xa, f->xb, f->avg, f->r1, f->r2, f->t3, f->c31, f->c32, f->c41, f->c42};
    for (int k = 0; k < 13; ++k) SYN_CUDA(cudaMemsetAsync(bufs[k], 0, f->ws_sizes[k], st));
  }
  const FbFrames* Rp = frames ? &R : nullptr;
  const FbGeom g = fb_geom(height, width);            // the one-image launches' sizes
  auto pool_frames = [&](int lin, int lout) { return FbPoolFrames{R.level(lin), R.level(lout), nf, (int)R.pix[lout]}; };
  auto pool_grid = [](size_t n) { return dim3((unsigned)((n + 255) / 256)); };
  const size_t n1 = R.pix[1], np1 = R.pix[2], n2 = R.pix[3], n3 = R.pix[4], n4 = R.pix[5], n5 = R.pix[6];
  const size_t np = np_all;
  // conv1 (CReLU) -> max-pool -> conv2 (CReLU) -> max-pool                                          faceboxes.py:120-123
  if (int rc = fb_conv(f, 0, nullptr, image_dev, height, width, 3, 0, f->c1, 48, 0, st, Rp, 0, 1)) return rc;
  SYN_FB_STOP(stop, 0, f->c1, n1 * 48, st);
  if (frames) fb_maxpool_kernel<true><<<pool_grid(np1 * 48), 256, 0, st>>>(f->c1, 0, 0, 48, f->p1, 0, 0, pool_frames(1, 2));
  else fb_maxpool_kernel<false><<<pool_grid(np1 * 48), 256, 0, st>>>(f->c1, g.h1, g.w1, 48, f->p1, g.hp1, g.wp1, FbPoolFrames{});
  SYN_LAUNCH_CHECK("fb_maxpool_kernel");
  ++f->launches;
  SYN_FB_STOP(stop, 1, f->p1, np1 * 48, st);
  if (int rc = fb_conv(f, 1, f->p1, nullptr, g.hp1, g.wp1, 48, 0, f->c2, 128, 0, st, Rp, 2, 3)) return rc;
  SYN_FB_STOP(stop, 2, f->c2, n2 * 128, st);
  if (frames) fb_maxpool_kernel<true><<<pool_grid(n3 * 128), 256, 0, st>>>(f->c2, 0, 0, 128, f->xa, 0, 0, pool_frames(3, 4));
  else fb_maxpool_kernel<false><<<pool_grid(n3 * 128), 256, 0, st>>>(f->c2, g.h2, g.w2, 128, f->xa, g.h3, g.w3, FbPoolFrames{});
  SYN_LAUNCH_CHECK("fb_maxpool_kernel");
  ++f->launches;
  SYN_FB_STOP(stop, 3, f->xa, n3 * 128, st);
  // three inception blocks: every branch writes its 32-channel slice of the next 128-channel tensor     :124-126, :33-47
  float *x = f->xa, *y = f->xb;
  for (int blk = 0; blk < 3; ++blk) {
    const int L0 = 2 + 7 * blk, s0 = 4 + 8 * blk;
    if (int rc = fb_conv(f, L0 + 0, x, nullptr, g.h3, g.w3, 128, 0, y, 128, 0, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 0, y, n3 * 128, st);
    if (frames) fb_avgpool_kernel<true><<<pool_grid(n3 * 128), 256, 0, st>>>(x, 0, 0, 128, f->avg, pool_frames(4, 4));
    else fb_avgpool_kernel<false><<<pool_grid(n3 * 128), 256, 0, st>>>(x, g.h3, g.w3, 128, f->avg, FbPoolFrames{});
    SYN_LAUNCH_CHECK("fb_avgpool_kernel");
    ++f->launches;
    SYN_FB_STOP(stop, s0 + 1, f->avg, n3 * 128, st);
    if (int rc = fb_conv(f, L0 + 1, f->avg, nullptr, g.h3, g.w3, 128, 0, y, 128, 32, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 2, y, n3 * 128, st);
    if (int rc = fb_conv(f, L0 + 2, x, nullptr, g.h3, g.w3, 128, 0, f->r1, 24, 0, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 3, f->r1, n3 * 24, st);
    if (int rc = fb_conv(f, L0 + 3, f->r1, nullptr, g.h3, g.w3, 24, 0, y, 128, 64, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 4, y, n3 * 128, st);
    if (int rc = fb_conv(f, L0 + 4, x, nullptr, g.h3, g.w3, 128, 0, f->r2, 24, 0, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 5, f->r2, n3 * 24, st);
    if (int rc = fb_conv(f, L0 + 5, f->r2, nullptr, g.h3, g.w3, 24, 0, f->t3, 32, 0, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 6, f->t3, n3 * 32, st);
    if (int rc = fb_conv(f, L0 + 6, f->t3, nullptr, g.h3, g.w3, 32, 0, y, 128, 96, st, Rp, 4, 4)) return rc;
    SYN_FB_STOP(stop, s0 + 7, y, n3 * 128, st);
    float* t = x; x = y; y = t;
  }
  // x = inception3 output (detection source 0); conv3_x, conv4_x give sources 1 and 2                  :127-135
  if (int rc = fb_conv(f, 23, x, nullptr, g.h3, g.w3, 128, 0, f->c31, 128, 0, st, Rp, 4, 4)) return rc;
  SYN_FB_STOP(stop, 28, f->c31, n3 * 128, st);
  if (int rc = fb_conv(f, 24, f->c31, nullptr, g.h3, g.w3, 128, 0, f->c32, 256, 0, st, Rp, 4, 5)) return rc;
  SYN_FB_STOP(stop, 29, f->c32, n4 * 256, st);
  if (int rc = fb_conv(f, 25, f->c32, nullptr, g.h4, g.w4, 256, 0, f->c41, 128, 0, st, Rp, 5, 5)) return rc;
  SYN_FB_STOP(stop, 30, f->c41, n4 * 128, st);
  if (int rc = fb_conv(f, 26, f->c41, nullptr, g.h4, g.w4, 128, 0, f->c42, 256, 0, st, Rp, 5, 6)) return rc;
  SYN_FB_STOP(stop, 31, f->c42, n5 * 256, st);
  // heads: NHWC output of each source IS permute(0,2,3,1).view(-1) (:137-142); the three sources are concatenated by
  // offset (one image), or by each frame's prior offsets (the frame axis: the head levels 7..9)
  float* loc1 = frames ? loc_dev : loc_dev + n3 * 84;
  float* loc2 = frames ? loc_dev : loc_dev + n3 * 84 + n4 * 4;
  float* conf1 = frames ? conf_dev : conf_dev + n3 * 42;
  float* conf2 = frames ? conf_dev : conf_dev + n3 * 42 + n4 * 2;
  if (int rc = fb_conv(f, 27, x, nullptr, g.h3, g.w3, 128, 0, loc_dev, 84, 0, st, Rp, 4, 7)) return rc;
  SYN_FB_STOP(stop, 32, loc_dev, np * 4, st);
  if (int rc = fb_conv(f, 28, f->c32, nullptr, g.h4, g.w4, 256, 0, loc1, 4, 0, st, Rp, 5, 8)) return rc;
  SYN_FB_STOP(stop, 33, loc_dev, np * 4, st);
  if (int rc = fb_conv(f, 29, f->c42, nullptr, g.h5, g.w5, 256, 0, loc2, 4, 0, st, Rp, 6, 9)) return rc;
  SYN_FB_STOP(stop, 34, loc_dev, np * 4, st);
  if (int rc = fb_conv(f, 30, x, nullptr, g.h3, g.w3, 128, 0, conf_dev, 42, 0, st, Rp, 4, 7)) return rc;
  SYN_FB_STOP(stop, 35, conf_dev, np * 2, st);
  if (int rc = fb_conv(f, 31, f->c32, nullptr, g.h4, g.w4, 256, 0, conf1, 2, 0, st, Rp, 5, 8)) return rc;
  SYN_FB_STOP(stop, 36, conf_dev, np * 2, st);
  if (int rc = fb_conv(f, 32, f->c42, nullptr, g.h5, g.w5, 256, 0, conf2, 2, 0, st, Rp, 6, 9)) return rc;
  SYN_FB_STOP(stop, 37, conf_dev, np * 2, st);
  fb_softmax2_kernel<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(conf_dev, (int)np);
  SYN_LAUNCH_CHECK("fb_softmax2_kernel");
  ++f->launches;
  SYN_FB_STOP(stop, 38, conf_dev, np * 2, st);
  return SYN_OK;
}

#undef SYN_FB_STOP

}  // namespace

extern "C" {

int syn_fb_num_layers(void) { return 33; }

int syn_fb_layer_desc(int idx, syn_fb_layer_desc_t* out) {
  if (idx < 0 || idx >= 33 || !out) return fail(SYN_ERR_INVALID, "syn_fb_layer_desc: bad index %d", idx);
  const FbLayer& L = kFbLayers[idx];
  out->name = L.name; out->cin = L.cin; out->cout = L.cout; out->ksize = L.k; out->stride = L.stride; out->pad = L.pad;
  out->has_bn = L.bn; out->activation = L.act;
  return SYN_OK;
}

int syn_fb_create(int device, syn_fb_t** out) {
  if (!out) return fail(SYN_ERR_INVALID, "syn_fb_create: null out");
  SYN_CUDA(cudaSetDevice(device));
  syn_fb* f = new (std::nothrow) syn_fb();
  if (!f) return fail(SYN_ERR_NOMEM, "syn_fb_create: out of host memory");
  f->device = device;
  *out = f;
  return SYN_OK;
}

void syn_fb_destroy(syn_fb_t* f) {
  if (!f) return;
  cudaSetDevice(f->device);
  fb_free_ws(f);
  for (int i = 0; i < 33; ++i) { cudaFree(f->d_w[i]); cudaFree(f->d_b[i]); }
  delete f;
}

int syn_fb_set_layer(syn_fb_t* f, int idx, const float* w_host, int64_t w_numel, const float* bias_host, const float* bn_weight_host,
                     const float* bn_bias_host, const float* bn_mean_host, const float* bn_var_host, float eps) {
  if (!f || !w_host || idx < 0 || idx >= 33) return fail(SYN_ERR_INVALID, "syn_fb_set_layer: bad argument");
  const FbLayer& L = kFbLayers[idx];
  const int64_t want = (int64_t)L.cout * L.cin * L.k * L.k;
  if (w_numel != want) return fail(SYN_ERR_SHAPE, "syn_fb_set_layer: %s expects %lld weights, got %lld", L.name, (long long)want, (long long)w_numel);
  if (L.bn && (!bn_weight_host || !bn_bias_host || !bn_mean_host || !bn_var_host)) return fail(SYN_ERR_INVALID, "syn_fb_set_layer: %s needs its BatchNorm", L.name);
  if (!L.bn && !bias_host) return fail(SYN_ERR_INVALID, "syn_fb_set_layer: %s needs its bias", L.name);
  const int K = L.k * L.k * L.cin;
  f->w[idx].assign((size_t)K * L.cout, 0.f);
  f->b[idx].assign(L.cout, 0.f);
  for (int co = 0; co < L.cout; ++co) {
    double sc = 1.0, sh = 0.0;
    if (L.bn) {                                            // eval BatchNorm2d: y = (x - mean) / sqrt(var + eps) * weight + bias
      sc = (double)bn_weight_host[co] / std::sqrt((double)bn_var_host[co] + (double)eps);
      sh = (double)bn_bias_host[co] - (double)bn_mean_host[co] * sc;
    } else {
      sh = bias_host[co];
    }
    f->b[idx][co] = (float)sh;
    for (int ci = 0; ci < L.cin; ++ci)
      for (int kh = 0; kh < L.k; ++kh)
        for (int kw = 0; kw < L.k; ++kw)                   // OIHW -> [(kh, kw, ci)][co]
          f->w[idx][((size_t)(kh * L.k + kw) * L.cin + ci) * L.cout + co] =
              (float)((double)w_host[(((size_t)co * L.cin + ci) * L.k + kh) * L.k + kw] * sc);
  }
  f->set[idx] = true;
  f->committed = false;
  return SYN_OK;
}

int syn_fb_commit(syn_fb_t* f) {
  if (!f) return fail(SYN_ERR_INVALID, "syn_fb_commit: null handle");
  SYN_CUDA(cudaSetDevice(f->device));
  for (int i = 0; i < 33; ++i)
    if (!f->set[i]) return fail(SYN_ERR_STATE, "syn_fb_commit: layer %s was never set", kFbLayers[i].name);
  for (int i = 0; i < 33; ++i) {
    cudaFree(f->d_w[i]); cudaFree(f->d_b[i]);
    f->d_w[i] = f->d_b[i] = nullptr;
    SYN_CUDA(cudaMalloc(&f->d_w[i], f->w[i].size() * sizeof(float)));
    SYN_CUDA(cudaMalloc(&f->d_b[i], f->b[i].size() * sizeof(float)));
    SYN_CUDA(cudaMemcpy(f->d_w[i], f->w[i].data(), f->w[i].size() * sizeof(float), cudaMemcpyHostToDevice));
    SYN_CUDA(cudaMemcpy(f->d_b[i], f->b[i].data(), f->b[i].size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  f->committed = true;
  return SYN_OK;
}

int64_t syn_fb_launch_count(const syn_fb_t* f) { return f ? f->launches : 0; }

int syn_fb_debug_fill_workspaces(syn_fb_t* f, int byte, size_t* bytes_filled, void* stream) {
  const char* who = "syn_fb_debug_fill_workspaces";
  if (!f || byte < 0 || byte > 255) return fail(SYN_ERR_INVALID, "%s: null handle or byte %d", who, byte);
  cudaStream_t st = (cudaStream_t)stream;
  SYN_CUDA(cudaSetDevice(f->device));
  if (int rc = refuse_capture(st, "%s: a fill is never recorded into a CUDA graph", who)) return rc;
  float* bufs[13] = {f->c1, f->p1, f->c2, f->xa, f->xb, f->avg, f->r1, f->r2, f->t3, f->c31, f->c32, f->c41, f->c42};
  size_t total = 0;
  for (int k = 0; k < 13; ++k) SYN_CUDA(fill_buffer(bufs[k], f->ws_sizes[k], byte, st, &total));
  // the geometry table holds pixel offsets: cleared, never filled with a byte pattern that could turn into an address
  SYN_CUDA(fill_buffer(f->geo_dev, sizeof(f->geo_host), 0, st, &total));
  if (bytes_filled) *bytes_filled = total;
  return SYN_OK;
}

int syn_fb_debug_fill_on_grow(syn_fb_t* f, int byte) {
  if (!f || byte < -1 || byte > 255) return fail(SYN_ERR_INVALID, "syn_fb_debug_fill_on_grow: null handle or byte %d", byte);
  f->fill_on_grow = byte;
  return SYN_OK;
}

int syn_fb_forward(syn_fb_t* f, const uint8_t* image_dev, int height, int width, float* loc_dev, float* conf_dev, void* stream) {
  return fb_forward_body(f, image_dev, 0, &height, &width, loc_dev, conf_dev, (cudaStream_t)stream, nullptr, "syn_fb_forward");
}

int syn_fb_forward_batch(syn_fb_t* f, const uint8_t* images_dev, int n_frames, int height, int width, float* loc_dev, float* conf_dev,
                         void* stream) {
  if (n_frames <= 0) return fail(SYN_ERR_INVALID, "syn_fb_forward_batch: %d frames", n_frames);
  const std::vector<int32_t> hs(std::min(n_frames, SYN_FB_MAX_FRAMES + 1), height), ws(hs.size(), width);   // one size, every frame
  return fb_forward_body(f, images_dev, n_frames, hs.data(), ws.data(), loc_dev, conf_dev, (cudaStream_t)stream, nullptr,
                         "syn_fb_forward_batch");
}

int syn_fb_forward_images(syn_fb_t* f, const uint8_t* images_dev, int n_images, const int32_t* heights_host, const int32_t* widths_host,
                          float* loc_dev, float* conf_dev, void* stream) {
  if (n_images <= 0) return fail(SYN_ERR_INVALID, "syn_fb_forward_images: %d images", n_images);
  return fb_forward_body(f, images_dev, n_images, heights_host, widths_host, loc_dev, conf_dev, (cudaStream_t)stream, nullptr,
                         "syn_fb_forward_images");
}

int syn_fb_debug_forward_until(syn_fb_t* f, const uint8_t* image_dev, int height, int width, int stage, float* out_dev,
                               int64_t out_numel, float* loc_dev, float* conf_dev, void* stream) {
  if (stage < 0 || stage >= kFbStages)
    return fail(SYN_ERR_INVALID, "syn_fb_debug_forward_until: stage %d outside 0..%d", stage, kFbStages - 1);
  if (!f || !out_dev) return fail(SYN_ERR_INVALID, "syn_fb_debug_forward_until: null handle or output");
  const FbStop stop{stage, out_dev, out_numel};
  return fb_forward_body(f, image_dev, 0, &height, &width, loc_dev, conf_dev, (cudaStream_t)stream, &stop, "syn_fb_debug_forward_until");
}

int syn_fb_debug_forward_batch_until(syn_fb_t* f, const uint8_t* images_dev, int n_frames, int height, int width, int stage,
                                     float* out_dev, int64_t out_numel, float* loc_dev, float* conf_dev, void* stream) {
  const char* who = "syn_fb_debug_forward_batch_until";
  if (stage < 0 || stage >= kFbStages) return fail(SYN_ERR_INVALID, "%s: stage %d outside 0..%d", who, stage, kFbStages - 1);
  if (!f || !out_dev) return fail(SYN_ERR_INVALID, "%s: null handle or output", who);
  if (n_frames <= 0) return fail(SYN_ERR_INVALID, "%s: %d frames", who, n_frames);
  const std::vector<int32_t> hs(std::min(n_frames, SYN_FB_MAX_FRAMES + 1), height), ws(hs.size(), width);
  const FbStop stop{stage, out_dev, out_numel};
  return fb_forward_body(f, images_dev, n_frames, hs.data(), ws.data(), loc_dev, conf_dev, (cudaStream_t)stream, &stop, who);
}

int syn_fb_debug_forward_images_until(syn_fb_t* f, const uint8_t* images_dev, int n_images, const int32_t* heights_host,
                                      const int32_t* widths_host, int stage, float* out_dev, int64_t out_numel, float* loc_dev,
                                      float* conf_dev, void* stream) {
  const char* who = "syn_fb_debug_forward_images_until";
  if (stage < 0 || stage >= kFbStages) return fail(SYN_ERR_INVALID, "%s: stage %d outside 0..%d", who, stage, kFbStages - 1);
  if (!f || !out_dev) return fail(SYN_ERR_INVALID, "%s: null handle or output", who);
  if (n_images <= 0) return fail(SYN_ERR_INVALID, "%s: %d images", who, n_images);
  const FbStop stop{stage, out_dev, out_numel};
  return fb_forward_body(f, images_dev, n_images, heights_host, widths_host, loc_dev, conf_dev, (cudaStream_t)stream, &stop, who);
}

}  // extern "C"
