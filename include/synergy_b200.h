/*
 * synergy_b200.h -- C ABI of the H100 (sm_90a) SynergyNet inference hot path.
 *
 * The reference (choyingw/SynergyNet) has no native boundary for this path: it is a Python
 * nn.Module API (model_building.py:65-165, synergy3DMM.py:70-207) whose arithmetic runs inside
 * PyTorch.  This library sits *under* a Python shim with the same class/method names
 * (synergynet_b200/model_building.py, synergynet_b200/synergy3DMM.py) and is bound with ctypes
 * (synergynet_b200/_lib.py); INTEGRATION.md shows the stub a reference maintainer would add.
 * Each entry point cites the reference code it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every function returns SYN_OK (0) or a SYN_ERR_* code; no exceptions cross the boundary;
 *     syn_last_error() returns a thread-local message for the last failing call.
 *   - plain pointers and sizes only.  "_dev" pointers are device memory on the handle's GPU and
 *     are owned by the caller; "_host" pointers are host memory.  `stream` is a cudaStream_t
 *     (passed as void*); work is enqueued on it and NOT synchronised unless stated.
 *   - one handle per device; a handle is not re-entrant (one call at a time per handle), but
 *     different handles may be driven from different host threads (nn.DataParallel replicas,
 *     main_train.py:176).
 *   - CUDA graphs: an entry that takes a `stream` may be captured on it once an eager call of the
 *     same size has run on that handle (workspaces grow, never shrink, and only eagerly).  A replay
 *     runs with the arguments fixed at capture: the workspace pointers, the tile plans and the
 *     syn_set_center_crop margin of that moment.  Replays are valid while no call grows that
 *     handle's workspace and no syn_*commit, syn_resnet_select or syn_mbv1_set_widen runs; the
 *     caller orders replays against eager calls of the same handle (they share its workspace).
 *     A call that would grow a workspace while its stream is capturing, and the detector's frame
 *     paths (syn_fb_forward_batch / _images: their per-call geometry comes from host memory),
 *     return SYN_ERR_STATE before they launch anything, leaving the capture valid.  The host
 *     pipelines (syn_forward_landmarks_host*, _submit) run on the library's own streams and wait on
 *     the host: never call them during a capture (the Python Engine refuses).
 *   - tensors are fp32 and contiguous in the layouts the reference uses.
 */
#ifndef SYNERGY_H100_H_
#define SYNERGY_H100_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SYN_ABI_VERSION 1

enum {
  SYN_OK = 0,
  SYN_ERR_INVALID = 1,   /* bad argument (null pointer, negative size, unknown layer ...)      */
  SYN_ERR_CUDA = 2,      /* a CUDA runtime call or kernel launch failed                         */
  SYN_ERR_STATE = 3,     /* call order violated (e.g. forward before syn_commit)               */
  SYN_ERR_SHAPE = 4,     /* "length of params mismatch" (model_building.py:116-119) and alike  */
  SYN_ERR_NOMEM = 5,
  SYN_ERR_UNSUPPORTED = 6 /* not an sm_90 device, or an engine the build does not contain      */
};

/* Compute engines for the 1x1 convolutions / basis products (syn_set_engine). */
enum {
  SYN_ENGINE_SIMT_FP32 = 0,   /* CUDA-core fp32 FMA everywhere (bring-up / cross-check path)     */
  SYN_ENGINE_TC_SPLIT3 = 1,   /* wgmma, operands split in fp16 hi+lo with exact power-of-two        */
                              /* pre-scaling, 3 MMAs per product (hi*hi + hi*lo + lo*hi), fp32      */
                              /* accumulation in registers: meets the 1e-4 parity bar (a bf16 split, */
                              /* first version, measured 1.7e-4 and was dropped); convs unfused      */
  SYN_ENGINE_TC_BF16X3 = 1,   /* old name of SYN_ENGINE_TC_SPLIT3                                    */
  SYN_ENGINE_TC_FUSED = 2,    /* default: the same arithmetic with the stem + all 17 inverted-       */
                              /* residual blocks each fused into one kernel (expand -> depthwise ->  */
                              /* project, hidden tensor on chip), last conv fused with the pooling   */
  SYN_ENGINE_TC_FUSED_1PASS = 3 /* NOT parity-grade, never the default: engine 2 with ONE fp16 MMA per */
                              /* product (hi*hi only) in the backbone.  Exists to show how much of    */
                              /* the step is the 3x precision tax; misses the 1e-4 bar (SURVEY fact 6) */
};

typedef struct syn_handle syn_handle_t;

/* Geometry of convolution `layer` (0..51) in execution order; lets the host check a checkpoint
 * against the compiled-in MobileNetV2 plan (mobilenetv2_backbone.py:108-138). */
typedef struct {
  int32_t cin, cout, ksize, stride, groups, relu6, h_in, h_out, residual;
} syn_conv_desc_t;

int         syn_abi_version(void);
const char* syn_last_error(void);
int         syn_num_conv_layers(void);                       /* 52 */
int         syn_conv_desc(int layer, syn_conv_desc_t* out);

/* Lifetime.  Replaces nn.Module construction + .cuda() (model_building.py:66-101). */
int  syn_create(int device, syn_handle_t** out);
void syn_destroy(syn_handle_t* h);

/* ---- weights: host pointers in the reference's own layouts; copied during the call ----------
 * Conv2d weight is OIHW fp32 (cout, cin/groups, k, k); BatchNorm2d is eval-mode
 * (weight, bias, running_mean, running_var, eps) and is folded into the convolution by
 * syn_commit.  Replaces ConvBNReLU / InvertedResidual parameter storage
 * (mobilenetv2_backbone.py:33-68). */
int syn_set_conv_bn(syn_handle_t* h, int layer, const float* w_host, int64_t w_numel,
                    const float* bn_weight_host, const float* bn_bias_host,
                    const float* bn_mean_host, const float* bn_var_host, float eps);
/* classifier_ori / classifier_shape / classifier_exp Linear layers, weights (out,1280) row
 * major (mobilenetv2_backbone.py:147-158). */
int syn_set_heads(syn_handle_t* h, const float* w_ori_host, const float* b_ori_host,
                  const float* w_shape_host, const float* b_shape_host,
                  const float* w_exp_host, const float* b_exp_host);
/* param_mean / param_std, 62 floats each (model_building.py:87-88). */
int syn_set_whitening(syn_handle_t* h, const float* mean_host, const float* std_host);
/* Landmark basis buffers u_base (3*n_pts), w_shp_base (3*n_pts,40), w_exp_base (3*n_pts,10),
 * rows xyz-interleaved (model_building.py:99-101, utils/params.py:30-32). */
int syn_set_basis_sparse(syn_handle_t* h, const float* u_base_host, const float* w_shp_base_host,
                         const float* w_exp_base_host, int n_pts);
/* Dense basis buffers u (3*n_vert), w_shp (3*n_vert,40), w_exp (3*n_vert,10)
 * (model_building.py:89-91).  Optional: only needed for dense reconstruction. */
int syn_set_basis_dense(syn_handle_t* h, const float* u_host, const float* w_shp_host,
                        const float* w_exp_host, int64_t n_vert);
/* Fold BN, re-lay-out for the kernels, upload.  Must follow the setters, may be repeated. */
int syn_commit(syn_handle_t* h);

int syn_set_engine(syn_handle_t* h, int engine);
int syn_get_engine(const syn_handle_t* h);

/* ---- compute, device buffers ------------------------------------------------------------------
 * syn_forward: I2P.forward_test / MobileNetV2._forward_impl (model_building.py:59-62,
 * mobilenetv2_backbone.py:173-189).  x_dev (B,3,120,120) NCHW -> params62_dev (B,62) whitened
 * parameters [ori12|shape40|exp10]; pool1280_dev (B,1280) may be NULL. */
int syn_forward(syn_handle_t* h, const float* x_dev, int batch, float* params62_dev,
                float* pool1280_dev, void* stream);
/* syn_reconstruct: reconstruct_vertex_62 (model_building.py:106-139; benchmark.py:76-97).
 * params62_dev (B,62) -> out_dev (B,3,N) with N = n_pts (dense=0) or n_vert (dense=1). */
int syn_reconstruct(syn_handle_t* h, const float* params62_dev, int batch, int dense,
                    int whitening, int transform, float* out_dev, void* stream);
/* forward_test + reconstruct_vertex_62(dense=False) without leaving the device
 * (benchmark.py:125-127 then :153-166).  params62_dev may be NULL. */
int syn_forward_landmarks(syn_handle_t* h, const float* x_dev, int batch, float* params62_dev,
                          float* lmk_dev, void* stream);

/* ---- image-space outputs of get_all_outputs (SURVEY.md section 8 f1) ----------------------------------------
 * _predict_vertices (utils/inference.py:127-138) fused into the reconstruction: vertices leave the GPU already in the
 * coordinates of the original image.  roi5_dev (B,5) fp32 = kx, sx, ky, sy, kz with kx = (ex-sx)/120, ky = (ey-sy)/120,
 * kz = (kx+ky)/2 evaluated in double on the host like the reference's Python scalars; whitening and the y flip are on. */
int syn_reconstruct_image(syn_handle_t* h, const float* params62_dev, int batch, int dense, const float* roi5_dev,
                          float* out_dev, void* stream);
/* parse_pose + predict_pose (utils/inference.py:33-62,86-92,146-157) for B whitened vectors: angles_dev (B,3) fp64
 * degrees [pitch-like x, yaw-like y, roll-like z in the reference's order], t3d_dev (B,3) fp32 (image coordinates when
 * roi5_dev is given, crop coordinates when NULL).  One deliberate departure from the reference: the fp32 cross product
 * gives |R20| = 1 + 2^-23 for some camera rows at yaw +-90 degrees, where the reference's math.asin raises; every
 * |R20| >= 1 takes the gimbal-lock branch of R20's sign, the reference's own value at R20 = +-1 (x = +90 for -1). */
int syn_pose_decode(syn_handle_t* h, const float* params62_dev, int batch, const float* roi5_dev, double* angles_dev,
                    float* t3d_dev, void* stream);
/* CenterCrop(margin, mode='test') of the reference loader (utils/ddfa.py:162-243, benchmark.py:116): the uint8 entry
 * points read the `margin`-pixel frame of every crop as 0 before normalising.  0 (default) = off. */
int syn_set_center_crop(syn_handle_t* h, int margin);

/* ---- compute, host buffers (the end-to-end call: H2D of the crops, forward, landmarks, D2H) --
 * x_host (B,3,120,120) fp32, lmk_host (B,3,68), params62_host (B,62) or NULL.  Pinned host
 * memory is recommended; chunks are pipelined over internal streams.  Synchronous. */
int syn_forward_landmarks_host(syn_handle_t* h, const float* x_host, int batch,
                               float* params62_host, float* lmk_host);

/* ---- uint8 crops (SURVEY.md section 8 f1): the reference normalises on the host,
 * `(img - 127.5) / 128` (synergy3DMM.py:192, benchmark.py:116 Normalize(mean=127.5, std=128)); these
 * entry points take the raw uint8 (B,3,120,120) planar crops and apply the same fp32 arithmetic on the
 * device (bit-identical values, 4x fewer bytes over PCIe / HBM). */
int syn_forward_landmarks_u8(syn_handle_t* h, const uint8_t* x_u8_dev, int batch, float* params62_dev,
                             float* lmk_dev, void* stream);
int syn_forward_landmarks_host_u8(syn_handle_t* h, const uint8_t* x_u8_host, int batch,
                                  float* params62_host, float* lmk_host);
/* The same call split in two, for a loader loop that keeps the GPU busy (benchmark.py:119-132 iterates a DataLoader
 * with pinned memory and non_blocking copies): submit enqueues H2D + forward + landmarks + D2H and returns a ticket;
 * syn_host_wait(ticket) returns once lmk_host / params62_host of that call are filled.  Up to two calls may be in flight
 * (the second one's copies run under the first one's kernels); a third submit waits for the oldest.  The host buffers
 * (pinned) must stay valid until their ticket has been waited for.  x_is_u8: 0 = fp32 normalised crops, 1 = raw uint8. */
int syn_forward_landmarks_host_submit(syn_handle_t* h, const void* x_host, int x_is_u8, int batch, float* params62_host,
                                      float* lmk_host, int* ticket);
int syn_host_wait(syn_handle_t* h, int ticket);

/* ---- PointNet refinement heads and the training-forward losses (SURVEY.md section 8 a10 / f4) -------------
 * net 0 = MLP_for (backbone_nets/pointnet_backbone.py:7-64): layer 0..8 = conv1..conv9 (+bn1..bn9);
 * net 1 = MLP_rev (:67-106): layer 0..4 = conv1..conv5, 5/6/7 = conv6_1 / conv6_2 / conv6_3 (+their BN).
 * Conv1d weights are (cout, cin, 1) fp32 host arrays, BatchNorm1d is eval-mode and folded at commit. */
int syn_pointnet_set_layer(syn_handle_t* h, int net, int layer, const float* w_host, int cout, int cin,
                           const float* conv_bias_host, const float* bn_weight_host, const float* bn_bias_host,
                           const float* bn_mean_host, const float* bn_var_host, float eps);
int syn_pointnet_commit(syn_handle_t* h, int net);            /* after syn_commit */
/* MLP_for.forward(x, avgpool, shape_code, expr_code) (pointnet_backbone.py:31-64) as called at
 * model_building.py:149-150: lmk_dev (B,3,68), pool1280_dev (B,1280), params62_dev (B,62; columns 12:52 and
 * 52:62 are the shape / expression codes) -> residual_dev (B,3,68) = point_residual and/or
 * refined_dev (B,3,68) = lmk + 0.05 * point_residual (either may be NULL). */
int syn_mlp_for(syn_handle_t* h, const float* lmk_dev, const float* pool1280_dev, const float* params62_dev,
                int batch, float* residual_dev, float* refined_dev, void* stream);
/* MLP_rev.forward (pointnet_backbone.py:90-106, model_building.py:153): lmk_dev (B,3,68) -> (B,62). */
int syn_mlp_rev(syn_handle_t* h, const float* lmk_dev, int batch, float* params62_dev, void* stream);
/* WingLoss(omega=10, epsilon=2) (loss_definition.py:8-27): mean over the B*3*n_pts coordinates -> out_dev[0]. */
int syn_wing_loss(syn_handle_t* h, const float* pred_dev, const float* target_dev, int batch, int n_pts,
                  float* out_dev, void* stream);
/* ParamLoss (loss_definition.py:29-42), one value per sample -> out_dev (B): mode 0 = 'normal', 1 = 'only_3dmm'
 * (input[:, :50] against target[:, 12:62], as the reference does). */
int syn_param_loss(syn_handle_t* h, const float* input_dev, const float* target_dev, int batch, int mode,
                   float* out_dev, void* stream);

/* ---- ResNet-50 backbone variant (BASELINE.json configs[4]; backbone_nets/resnet_backbone.py:227-249) -----------
 * 53 convolutions in execution order: 0 = conv1 (7x7/s2); then per Bottleneck conv1, conv2, conv3 and -- first block of a
 * stage -- downsample.0 (syn_resnet_conv_desc gives each one's geometry).  Weights OIHW fp32 + eval BatchNorm2d, as
 * for syn_set_conv_bn.  Heads: the four Linear layers concatenated in the reference's OUTPUT order
 * fc_ori | fc_shape | fc_exp | fc_tex -> (102, 2048) weights, (102) bias (:242-246).
 * syn_resnet50_forward: x_dev (B,3,120,120) NCHW -> out102_dev (B,102) exactly what ResNet._forward_impl returns;
 * pool2048_dev (B,2048) = the flattened avgpool, may be NULL.  (The reference's I2P unpacks two values from this
 * backbone and fails, SURVEY.md fact 4; the Python shim adapts: params = out[:, :62], pool = the 2048-d feature.)
 * Every forward and debug run of the ResNet, MobileNetV1 and GhostNet backbones (syn_resnet50_forward,
 * syn_resnet_forward, syn_mbv1_forward, syn_ghost_forward, syn_debug_resnet_until, syn_debug_mbv1_until,
 * syn_debug_ghost_until) takes 1 <= B <= 65535 faces per call, and returns
 * SYN_ERR_INVALID before any launch otherwise. */
int syn_resnet_num_convs(void);                              /* 53 */
int syn_resnet_conv_desc(int idx, syn_conv_desc_t* out);
int syn_resnet_set_conv(syn_handle_t* h, int idx, const float* w_host, int64_t w_numel, const float* bn_weight_host,
                        const float* bn_bias_host, const float* bn_mean_host, const float* bn_var_host, float eps);
int syn_resnet_set_heads(syn_handle_t* h, const float* w102x2048_host, const float* b102_host);
int syn_resnet_commit(syn_handle_t* h);                      /* after syn_commit */
int syn_resnet50_forward(syn_handle_t* h, const float* x_dev, int batch, float* out102_dev, float* pool2048_dev,
                         void* stream);
/* The other ResNet factories the reference's I2P builds (model_building.py:44-45; resnet_backbone.py:282-391), named by
 * (depth, width_per_group): resnet18 (18, 64), resnet34 (34, 64), resnet50 (50, 64), resnet101 (101, 64), resnet152
 * (152, 64), wide_resnet50_2 (50, 128), wide_resnet101_2 (101, 128).  18 / 34 use BasicBlock (:50-88: conv1 3x3 carries
 * the stride, conv2 3x3 adds the shortcut), the others Bottleneck (:90-136, width = planes * width_per_group / 64).
 * Convolutions in state-dict order: 0 = conv1 (7x7/s2); then per block conv1, conv2 (, conv3) and, where the block has
 * one (stride != 1 or inplanes != planes * expansion, :210-214), downsample.0.  `residual` marks the conv that adds the
 * shortcut.  Anything but the seven pairs is SYN_ERR_INVALID; syn_resnet_arch_num_convs then returns -1.
 * syn_resnet_select picks the arch of the handle and forgets the ResNet weights set so far; a handle that never calls it
 * holds resnet50.  syn_resnet_set_conv / _set_heads / _commit act on the selected arch; the heads are (102, 512) for
 * 18 / 34 and (102, 2048) otherwise.  syn_resnet50_forward refuses any other committed arch.
 * syn_resnet_forward: x_dev (B,3,120,120) NCHW fp32 crops, or raw uint8 crops when x_is_u8 (normalised in the stem as
 * (v - 127.5) / 128, with the syn_set_center_crop frame), -> out102_dev (B,102) = what ResNet._forward_impl returns;
 * pool_dev (B,512 or 2048) = the flattened avgpool, may be NULL. */
int syn_resnet_arch_num_convs(int depth, int width_per_group);
int syn_resnet_arch_conv_desc(int depth, int width_per_group, int idx, syn_conv_desc_t* out);
int syn_resnet_select(syn_handle_t* h, int depth, int width_per_group);
int syn_resnet_forward(syn_handle_t* h, const void* x_dev, int x_is_u8, int batch, float* out102_dev, float* pool_dev,
                       void* stream);

/* ---- MobileNetV1 backbones (backbone_nets/mobilenetv1_backbone.py:21-140, prelu=False) ------------------------------
 * Five widths, named by widen_code = 100 x the widen factor: SYN_MBV1_2 (200, mobilenet_2), SYN_MBV1_1 (100),
 * SYN_MBV1_075 (75), SYN_MBV1_05 (50), SYN_MBV1_025 (25); every channel count is int(c * widen).  27 convolutions in
 * execution order: 0 = conv1 (3x3/s2, 3 -> 32w), then per DepthWiseBlock dw2_1 .. dw6 its conv_dw (3x3 depthwise,
 * stride 1 or 2) and its conv_sep (1x1) -- syn_mbv1_conv_desc gives each one's geometry (groups = cin for a depthwise).
 * syn_mbv1_set_widen selects the width of the handle and forgets the MobileNetV1 weights set so far; then every conv
 * takes OIHW fp32 weights + eval BatchNorm2d as for syn_resnet_set_conv, and the heads the four Linear layers
 * concatenated in the reference's OUTPUT order fc_ori | fc_shape | fc_exp | fc_tex -> (102, 1024w) weights, (102)
 * bias (:95-98, :132-138).  syn_mbv1_commit comes after syn_commit (the shared library state); BatchNorm is folded in
 * float64.  syn_mbv1_forward: x_dev (B,3,120,120) NCHW fp32 crops, or raw uint8 crops when x_is_u8 (normalised as
 * (v - 127.5) / 128, with the syn_set_center_crop frame), -> out102_dev (B,102) = what MobileNet.forward returns;
 * pool_dev (B,1024w) = the flattened avgpool, may be NULL.  (The reference's I2P unpacks two values from this backbone
 * along dim 0; the Python shim adapts as for ResNet-50: params = out[:, :62], pool = the 1024w-d feature.) */
enum { SYN_MBV1_2 = 200, SYN_MBV1_1 = 100, SYN_MBV1_075 = 75, SYN_MBV1_05 = 50, SYN_MBV1_025 = 25 };
int syn_mbv1_num_convs(void);                                /* 27 */
int syn_mbv1_conv_desc(int widen_code, int idx, syn_conv_desc_t* out);
int syn_mbv1_set_widen(syn_handle_t* h, int widen_code);
int syn_mbv1_set_conv(syn_handle_t* h, int idx, const float* w_host, int64_t w_numel, const float* bn_weight_host,
                      const float* bn_bias_host, const float* bn_mean_host, const float* bn_var_host, float eps);
int syn_mbv1_set_heads(syn_handle_t* h, const float* w102xC_host, const float* b102_host);
int syn_mbv1_commit(syn_handle_t* h);                        /* after syn_commit */
int syn_mbv1_forward(syn_handle_t* h, const void* x_dev, int x_is_u8, int batch, float* out102_dev, float* pool_dev,
                     void* stream);

/* ---- GhostNet backbone (backbone_nets/ghostnet_backbone.py, ghostnet() at width 1.0, eval) ----------------------------
 * 95 convolutions in state-dict order: 0 = conv_stem (3x3/s2, 3 -> 16); per GhostBottleneck ghost1.primary_conv (1x1),
 * ghost1.cheap_operation (3x3 depthwise), conv_dw (k x k/s2 depthwise, stride-2 blocks), se.conv_reduce and
 * se.conv_expand (1x1 with bias, SE blocks), ghost2.primary_conv, ghost2.cheap_operation (`residual` = 1: its pass adds
 * the shortcut), shortcut.0 (k x k depthwise) and shortcut.2 (1x1) where the block has them; then blocks.9.0.conv
 * (1x1 160 -> 960) and conv_head (1x1 960 -> 1280 with bias).  syn_ghost_conv_desc gives each one's geometry (groups =
 * cin for a depthwise; the SE convs and conv_head have h_in = h_out = 1).  Every conv with a BatchNorm takes OIHW fp32
 * weights + eval BatchNorm2d through syn_ghost_set_conv; the SE convs and conv_head take weights and their (cout) bias
 * through syn_ghost_set_conv_bias; a conv given to the wrong setter, or of the wrong size, is refused.  Heads: the four
 * Linear layers concatenated in the reference's OUTPUT order classifier_ori | classifier_shape | classifier_exp |
 * classifier_texture -> (102, 1280) weights, (102) bias.  syn_ghost_commit comes after syn_commit; BatchNorm is folded
 * in float64.  syn_ghost_forward: x_dev as for syn_mbv1_forward -> out102_dev (B,102) = what GhostNet.forward returns;
 * feat1280_dev (B,1280) = the conv_head output after its ReLU (what the heads read), may be NULL.  B is bounded as for
 * the other conv+BN backbones. */
int syn_ghost_num_convs(void);                               /* 95 */
int syn_ghost_conv_desc(int idx, syn_conv_desc_t* out);
int syn_ghost_set_conv(syn_handle_t* h, int idx, const float* w_host, int64_t w_numel, const float* bn_weight_host,
                       const float* bn_bias_host, const float* bn_mean_host, const float* bn_var_host, float eps);
int syn_ghost_set_conv_bias(syn_handle_t* h, int idx, const float* w_host, int64_t w_numel, const float* b_host);
int syn_ghost_set_heads(syn_handle_t* h, const float* w102x1280_host, const float* b102_host);
int syn_ghost_commit(syn_handle_t* h);                       /* after syn_commit */
int syn_ghost_forward(syn_handle_t* h, const void* x_dev, int x_is_u8, int batch, float* out102_dev, float* feat1280_dev,
                      void* stream);

/* ---- Sim3DR: vertex normals, lighting, z-buffer rasterisation (SURVEY.md section 8 row f2) -------------------------
 * Handle-free; every pointer is caller-owned device memory unless it says _host.  B meshes share one triangle list
 * tri_dev (ntri,3) int32, 0-based (utils/render.py:32-33).  Vertices are read in place through element strides:
 * coordinate k of vertex i of mesh b = vertices_dev[b*stride_mesh + i*stride_vertex + k*stride_coord], i.e.
 * (nver, 1) for the dense output (B,3,nver) of syn_reconstruct / syn_reconstruct_image (stride_mesh = 3*nver) and
 * (3, 1) for the (nver,3) arrays the reference passes (Sim3DR/Sim3DR.py:8-29).  normals / colours are (B,nver,3).
 * Normals and rasterisation return the reference's bits (csrc/render_math.h explains how); lighting is its float32
 * arithmetic except x**5, where numpy's powf has no portable bit pattern (<= 1 ulp). */
typedef struct {        /* Sim3DR/lighting.py:24-32 (RenderPipeline.__init__) */
  float intensity_ambient, intensity_directional, intensity_specular;
  float color_ambient[3], color_directional[3], light_pos[3], view_pos[3];
  int32_t specular_exp;
} syn_light_cfg_t;

/* One-time index work per topology: the triangles incident to each vertex, ascending (start_out: nver+1 entries,
 * list_out: 3*ntri), so that vertex normals add up in the reference's order (rasterize_kernel.cpp:189-199).
 * SYN_ERR_SHAPE if a triangle references a vertex outside [0, nver). */
int syn_mesh_incidence_host(const int32_t* tri_host, int ntri, int nver, int32_t* start_out, int32_t* list_out);
/* Sim3DR.get_normal (Sim3DR/Sim3DR.py:8-11 -> rasterize_kernel.cpp:158-213).  tri_normals_ws_dev: B*ntri*3 floats. */
int syn_mesh_normals(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch, int nver,
                     const int32_t* tri_dev, int ntri, const int32_t* inc_start_dev, const int32_t* inc_tri_dev,
                     float* tri_normals_ws_dev, float* normals_dev, void* stream);
/* RenderPipeline.__call__ up to the rasterize call (Sim3DR/lighting.py:37-75): colours = clip(ambient + diffuse +
 * specular, 0, 1), times texture_dev (nver,3) when that is not NULL.  stats_ws_dev: 6*B uint32. */
int syn_mesh_lighting(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch, int nver,
                      const float* normals_dev, const syn_light_cfg_t* cfg, const float* texture_dev, uint32_t* stats_ws_dev,
                      float* colors_dev, void* stream);
/* syn_mesh_lighting with one texture per mesh: mesh b's colours are its light times the (nver,3) float32 texture at
 * texture_dev + b * texture_stride_mesh.  A stride of 0 shares one texture, with the bits of syn_mesh_lighting; otherwise
 * the stride is at least 3 * nver.  The (B,nver,3) textures syn_uv_sample writes take stride 3 * nver (artistic.py and
 * uv_texture_realFaces.py light each face with its own UV colours).  SYN_ERR_INVALID for a NULL texture or a stride
 * outside those values, and the refusals of syn_mesh_lighting, before any launch. */
int syn_mesh_lighting_textures(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int batch,
                               int nver, const float* normals_dev, const syn_light_cfg_t* cfg, const float* texture_dev,
                               int64_t texture_stride_mesh, uint32_t* stats_ws_dev, float* colors_dev, void* stream);
/* Sim3DR.rasterize (Sim3DR/Sim3DR.py:14-29 -> rasterize_kernel.cpp:217-287): draws the B meshes, in order, onto
 * image_dev (height,width,channels) uint8, each with its own depth buffer as the reference's per-face calls have
 * (utils/render.py:41-45).  colors_dev (B,nver,channels).  alpha must be 1 (the only value the reference's Python
 * API can pass; SYN_ERR_UNSUPPORTED otherwise).  keys_ws_dev: B*height*width uint64.  depth_out_dev: NULL, or
 * (B,height,width) floats that receive each mesh's final depth buffer (-1e8 where nothing was drawn). */
int syn_rasterize(uint8_t* image_dev, int height, int width, int channels, const float* vertices_dev, int64_t stride_mesh,
                  int stride_vertex, int stride_coord, int batch, int nver, const int32_t* tri_dev, int ntri,
                  const float* colors_dev, float alpha, int reverse, uint64_t* keys_ws_dev, float* depth_out_dev, void* stream);

/* The overlay stage of utils/render.py:38-47 for a stack of frames (the reference runs it once per image): n_frames
 * equally sized frames, frame f owning meshes [mesh_start[f], mesh_start[f+1]) of the n_meshes meshes, in draw order.
 * Each frame's solid overlay is what syn_rasterize draws onto a copy of that frame with that frame's meshes
 * (Sim3DR/lighting.py:37-72 for the colours, rasterize_kernel.cpp:217-287 for the z-buffer, alpha 1, no reverse, no
 * depth output).  A mesh keys only its pixel box -- the union of its triangles' boxes clamped to the frame -- so the key
 * workspace is the sum of the box areas, not n_meshes * height * width.  Two steps:
 *   syn_render_frames_plan writes boxes_dev (n_meshes,4) int32 (x0, y0, x1, y1; an empty or off-frame mesh: (0,0,-1,-1))
 *   and key_off_dev (n_meshes+1) int64, the exclusive prefix sum of the box areas: key_off_dev[n_meshes] is the number
 *   of uint64 key slots syn_rasterize_frames needs.  Reading it back is the one host synchronisation of the stage.
 *   syn_rasterize_frames reads frames_dev (n_frames,height,width,channels) uint8 and writes the solid overlays to
 *   solid_dev (same shape; it may be frames_dev, to draw in place -- later meshes of a frame can so be drawn by a later
 *   call onto what an earlier call drew, with the same bytes as one call).  colors_dev (n_meshes,nver,color_channels)
 *   as syn_mesh_lighting writes them; mesh_start_dev is mesh_start_host on the device; n_keys = key_off_dev[n_meshes];
 *   keys_ws_dev holds keys_ws_count >= n_keys uint64.
 * Both take the vertices through element strides as syn_rasterize does, and check mesh_start_host before any launch:
 * mesh_start[0] = 0, monotone, mesh_start[n_frames] = n_meshes (SYN_ERR_SHAPE otherwise).  1..65535 frames and meshes
 * per call.  A channel mismatch or a key workspace smaller than n_keys is SYN_ERR_SHAPE. */
int syn_render_frames_plan(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int n_meshes, int nver,
                           const int32_t* tri_dev, int ntri, const int32_t* mesh_start_host, int n_frames, int height, int width,
                           int32_t* boxes_dev, int64_t* key_off_dev, void* stream);
int syn_rasterize_frames(const uint8_t* frames_dev, uint8_t* solid_dev, int n_frames, int height, int width, int channels,
                         const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int n_meshes, int nver,
                         const int32_t* tri_dev, int ntri, const float* colors_dev, int color_channels, const int32_t* mesh_start_host,
                         const int32_t* mesh_start_dev, const int32_t* boxes_dev, const int64_t* key_off_dev, int64_t n_keys,
                         uint64_t* keys_ws_dev, int64_t keys_ws_count, void* stream);
/* The same overlay stage (utils/render.py:31-53, per image; rasterize_kernel.cpp:217-287 for the z-buffer) for a list of
 * images of different sizes, drawn in one pass.  Image f is (h, w, channels) uint8 at byte offset off of the image table
 * (n_images,3) int64 (off, h, w).  The table comes as images_host (checked here) and images_dev (its device copy, which
 * the kernels read).  The images lie in memory order, disjoint, inside the image_bytes of the pack, and every off is a
 * multiple of channels: a packed image list, an equal-size stack, or a slice of either.  Image f owns meshes
 * [mesh_start[f], mesh_start[f+1]) of the n_meshes meshes, in draw order; mesh_start comes as mesh_start_host (checked)
 * and mesh_start_dev (read by the kernels).  Each mesh's pixel box is clamped to its OWN image, so a mesh off its image
 * draws nothing, even where a larger image of the list would hold it.  Nothing outside an image's own bytes is written.
 *   syn_render_images_plan writes boxes_dev and key_off_dev as syn_render_frames_plan does.
 *   syn_rasterize_images reads images_dev and writes the solid overlays to solid_dev (the same layout; it may be
 *   images_dev, to draw in place).  Image f's bytes are what syn_rasterize_frames draws onto a one-frame stack of that
 *   image with its meshes.  colors_dev (n_meshes,nver,color_channels); n_keys = key_off_dev[n_meshes]; keys_ws_dev holds
 *   keys_ws_count >= n_keys uint64.
 * All checks run before any launch.  SYN_ERR_INVALID: a null pointer, or not 1..65535 images and meshes.  SYN_ERR_SHAPE:
 * a table that is out of order, overlaps, does not fit the image bytes or has an offset that is not a multiple of
 * channels; a mesh_start that does not run monotonically from 0 to n_meshes; image and colour channels that differ; a
 * key workspace smaller than n_keys.  Host arrays are read during the call only. */
int syn_render_images_plan(const float* vertices_dev, int64_t stride_mesh, int stride_vertex, int stride_coord, int n_meshes, int nver,
                           const int32_t* tri_dev, int ntri, const int32_t* mesh_start_host, const int32_t* mesh_start_dev,
                           const int64_t* images_host, const int64_t* images_dev, int n_images, int64_t image_bytes, int channels,
                           int32_t* boxes_dev, int64_t* key_off_dev, void* stream);
int syn_rasterize_images(const uint8_t* images_dev, uint8_t* solid_dev, int64_t image_bytes, const int64_t* table_host,
                         const int64_t* table_dev, int n_images, int channels, const float* vertices_dev, int64_t stride_mesh,
                         int stride_vertex, int stride_coord, int n_meshes, int nver, const int32_t* tri_dev, int ntri,
                         const float* colors_dev, int color_channels, const int32_t* mesh_start_host, const int32_t* mesh_start_dev,
                         const int32_t* boxes_dev, const int64_t* key_off_dev, int64_t n_keys, uint64_t* keys_ws_dev,
                         int64_t keys_ws_count, void* stream);
/* cv2.addWeighted(a, 1 - alpha, b, alpha, 0) on n uint8 values (utils/render.py:45), byte for byte with OpenCV 4.x:
 * out = saturate(round_half_even(fmaf(a, (float)(1 - alpha), b * (float)alpha))), 1 - alpha in double (csrc/render_math.h
 * add_weighted_u8).  out_dev may be a_dev or b_dev.  Any finite alpha; otherwise SYN_ERR_INVALID. */
int syn_add_weighted_u8(const uint8_t* a_dev, const uint8_t* b_dev, double alpha, uint8_t* out_dev, int64_t n, void* stream);
/* The pose axes of draw_axis (utils/inference.py:199-244, three cv2.line calls of thickness 4 per face, called once per
 * face in rect order by singleImage.py:112-117) for many images at once: cv2.line(img, p0, p1, colour, 4) with LINE_8
 * and shift 0, byte for byte with OpenCV 4.x (csrc/draw_math.h), for every segment, drawn IN PLACE.
 *   images_dev: image_bytes uint8; image f is (h, w, 3) BGR at byte offset off of the frame table (n_frames,3) int64
 *     (off, h, w), given as frames_host (checked here) and frames_dev (its device copy, which the kernel reads); the
 *     images lie in memory order, disjoint, inside the image bytes (an equal-size stack, or an ImagePack).
 *   segs_dev (n_segs,5) int32: x0, y0, x1, y1 and the colour b | g << 8 | r << 16; image f owns segments
 *     [seg_start[f], seg_start[f+1]), in draw order: where segments overlap, the later one's colour is left.  seg_start
 *     comes as seg_start_host (checked here) and seg_start_dev (read by the kernel).
 * A segment that leaves its image is clipped to it; nothing outside an image's own bytes is written.  thickness other
 * than 4 or line_type other than 8 is SYN_ERR_UNSUPPORTED, a null pointer or a negative count SYN_ERR_INVALID, a
 * seg_start that does not run monotonically from 0 to n_segs or a frame table that does not fit SYN_ERR_SHAPE, all
 * before any launch.  No allocation and no synchronisation (graph capture is fine); host arrays are read during the
 * call only. */
int syn_draw_lines(uint8_t* images_dev, int64_t image_bytes, const int64_t* frames_host, const int64_t* frames_dev, int n_frames,
                   const int32_t* seg_start_host, const int32_t* seg_start_dev, const int32_t* segs_dev, int n_segs, int thickness,
                   int line_type, void* stream);
/* The UV colours of artistic.py:126-131 / uv_texture_realFaces.py:103-114 for n_faces faces, each with its own map:
 * colors_uv = np.flip(map, 0)[coord_u, coord_v][keep], as float32 / 255 (the texture the overlay lights) and as the
 * bytes themselves (the int64 colour rows syn_obj_write prints with colors_dot0 = 1, "233.0").
 *   maps_dev: map_bytes uint8; map m is (h, w, 3) at byte offset off of the map table (n_maps,3) int64 (off, h, w), given
 *     as maps_host (checked here) and maps_table_dev (its device copy, which the kernel reads): the layout of the image
 *     tables of syn_draw_lines and syn_rasterize_images.
 *   texels_host / texels_dev (n_maps, n_keep, 2) int32: the (row, column) of the UNFLIPPED map m that kept vertex i reads,
 *     resolved on the host (the flip and numpy's negative-index wrap included); texels_dev 8-byte aligned.
 *   face_map_host / face_map_dev (n_faces) int32: the map of each face.
 *   texture_dev (n_faces, n_keep, 3) float32 and colors_dev (n_faces, n_keep, 3) int64; either may be NULL, not both.
 * SYN_ERR_INVALID for a null pointer, a misaligned texels_dev, or counts outside 1..65535 faces, >= 1 map and kept
 * vertex; SYN_ERR_SHAPE for a map table that is out of order, overlaps or does not fit the map bytes, a texel outside
 * its map, or a face naming no map; all before the one launch.  No allocation and no synchronisation (graph capture is
 * fine); host arrays are read during the call only. */
int syn_uv_sample(const uint8_t* maps_dev, int64_t map_bytes, const int64_t* maps_host, const int64_t* maps_table_dev, int n_maps,
                  const int32_t* texels_host, const int32_t* texels_dev, int n_keep, const int32_t* face_map_host,
                  const int32_t* face_map_dev, int n_faces, float* texture_dev, int64_t* colors_dev, void* stream);

/* ---- OBJ text of dense meshes (utils/inference.py:8-23 write_obj; artistic.py:19-31 and uv_texture_realFaces.py:21-33
 * write_obj_with_colors) -------------------------------------------------------------------------------------------
 * The bytes those functions write for B meshes, each mesh's text its vertex lines then its triangle lines:
 *   vertex line   'v {:.4f} {:.4f} {:.4f}\n' of the float32 coordinates 0, 1, 2 (the exact binary value rounded to 4
 *                 decimals, ties to even; "nan", "inf", "-inf"; the sign bit always prints), with colours followed by
 *                 ' {} {} {}' of colours[i, 2], [i, 1], [i, 0] before the newline;
 *   triangle line 'f {} {} {}\n' of triangles[i, 2], [i, 1], [i, 0] (tri_order 0, write_obj) or [i, 0], [i, 1], [i, 2]
 *                 (tri_order 1, write_obj_with_colors), the indices as given.
 * A '{}' field is the int64's digits, or with its dot0 flag the repr of an integral float below 1e16 ("233.0"; the
 * value INT64_MIN stands for -0.0 and prints "-0.0").  Coordinate k of vertex i of mesh b is
 * vertices[b * stride_mesh + i * stride_vertex + k * stride_coord] (the (B,3,N) output of syn_reconstruct_image and
 * (N,3) arrays alike).  keep_host / keep_dev: NULL (vertex line i prints vertex i, nver lines), or n_keep vertex
 * indices (line i prints vertex keep[i]: vertices[:, keep] without a gather copy).  colors: NULL, or int64 (n, 3) rows
 * of line i at colors[b * colors_stride_mesh + 3 i]; stride 0 shares one colour table between the meshes.
 * triangles: int64 (ntri, 3), the same text for every mesh. */
typedef struct {
  const float* vertices;
  int64_t stride_mesh;
  int32_t stride_vertex, stride_coord, batch, nver;
  const int32_t* keep_host;
  const int32_t* keep_dev;
  int32_t n_keep;
  const int64_t* colors;
  int64_t colors_stride_mesh;
  int32_t colors_dot0;
  const int64_t* triangles;
  int32_t ntri, tri_order, tri_dot0;
} syn_obj_desc_t;
/* Bytes of the workspace syn_obj_plan fills and syn_obj_write reads for batch meshes of n_lines vertex lines and ntri
 * triangles; -1 for a negative count, a batch outside 1..65535, or more than INT32_MAX blocks of 256 lines
 * (batch * ceil(n_lines / 256) + ceil(ntri / 256)), the sizes both entries refuse. */
int64_t syn_obj_workspace_size(int batch, int n_lines, int ntri);
/* The byte offset of every mesh's text: offsets_dev (batch + 1) int64, mesh b's text at [offsets[b], offsets[b+1]),
 * offsets[batch] the total the caller allocates for syn_obj_write (the one value it needs on the host).  Two launches.
 * SYN_ERR_INVALID before any launch for a null pointer, keep_dev without keep_host, batch outside 1..65535, nver < 1,
 * n_keep or ntri < 0, more than INT32_MAX blocks of 256 lines, a keep index outside [0, nver), a non-positive vertex
 * stride (stride_mesh too when batch > 1), a negative colour stride, a flag other than 0 or 1; SYN_ERR_SHAPE for a
 * workspace below syn_obj_workspace_size.  No allocation and no
 * synchronisation (graph capture is fine); keep_host is read during the call only. */
int syn_obj_plan(const syn_obj_desc_t* desc, void* ws_dev, int64_t ws_bytes, int64_t* offsets_dev, void* stream);
/* The text itself into out_dev (out_bytes, offsets[batch] of the plan of the same desc, workspace and offsets): one
 * launch, and one more that copies mesh 0's triangle text to the others when batch > 1 and ntri > 0.  Every byte of
 * [0, offsets[batch]) is written; a store past out_bytes is dropped.  The refusals of syn_obj_plan, and SYN_ERR_INVALID
 * for a null out_dev or offsets_dev or a negative out_bytes. */
int syn_obj_write(const syn_obj_desc_t* desc, const void* ws_dev, int64_t ws_bytes, const int64_t* offsets_dev, uint8_t* out_dev,
                  int64_t out_bytes, void* stream);

/* ---- FaceBoxes post-processing (SURVEY.md section 8 row f3) -----------------------------------------------------------
 * These entries take the detector network's outputs (syn_fb_forward below, or any other producer). */
enum {
  SYN_NMS_CPU_NMS = 0,     /* FaceBoxes/utils/nms/cpu_nms.pyx:17-68, the path nms_wrapper.py:13-18 takes: suppress on   */
                           /* ovr >= thresh, compared in double                                                       */
  SYN_NMS_PY_CPU_NMS = 1   /* FaceBoxes/utils/nms/py_cpu_nms.py:10-38: keep on ovr <= thresh, compared in float32     */
                           /* (a NaN overlap, from a box with a NaN coordinate, fails that test: the box is dropped)   */
};
/* Greedy NMS of dets_dev (n,5) fp32 rows [x1 y1 x2 y2 score] ALREADY in descending score order (FaceBoxes.py:116-121
 * sorts before it calls nms).  keep_dev (n) int32 receives the kept row indices in order, *n_keep_dev their count:
 * the index list either reference function returns, bit for bit.  mask_ws_dev: n * ceil(n/64) uint64. */
int syn_nms(const float* dets_dev, int n, double thresh, int mode, uint64_t* mask_ws_dev, int32_t* keep_dev, int32_t* n_keep_dev,
            void* stream);
/* The same greedy loop (FaceBoxes.py:122-127) for n_frames frames in two launches, with no host round trip after the
 * decode: dets_dev (n_frames, rows_per_frame, 5), frame f's first min(n_dev[f], rows_per_frame) rows are its boxes
 * (n_dev: the device counts syn_faceboxes_decode_batch wrote).  keep_dev (n_frames, rows_per_frame) int32 and n_keep_dev
 * (n_frames) receive every frame's list and count, each what syn_nms returns for that frame alone (a frame with no box:
 * count 0).  mask_ws_dev: n_frames * rows_per_frame * ceil(rows_per_frame/64) uint64.  n_frames <= SYN_FB_MAX_FRAMES. */
int syn_nms_batch(const float* dets_dev, const int32_t* n_dev, int n_frames, int rows_per_frame, double thresh, int mode,
                  uint64_t* mask_ws_dev, int32_t* keep_dev, int32_t* n_keep_dev, void* stream);
/* Number of prior boxes for an im_height x im_width network input (utils/prior_box.py:19-43); -1 on bad sizes. */
int syn_faceboxes_num_priors(int im_height, int im_width);
/* FaceBoxes.__call__ between the network and the NMS (FaceBoxes/FaceBoxes.py:98-121): priors, decode
 * (utils/box_utils.py:177-195, variances 0.1 / 0.2), `boxes * scale_bbox / scale`, `scores > conf_thresh`, descending
 * order (ties: higher prior index first), first top_k.  loc_dev (P,4), conf_dev (P,2) softmax output, P =
 * syn_faceboxes_num_priors.  dets_dev (top_k,5), *n_dets_dev = rows written.  cand_ws_dev: P+1 int32. */
int syn_faceboxes_decode(const float* loc_dev, const float* conf_dev, int im_height, int im_width, float box_scale_w,
                         float box_scale_h, float scale, float conf_thresh, int top_k, int32_t* cand_ws_dev, float* dets_dev,
                         int32_t* n_dets_dev, void* stream);
/* FaceBoxes.py:98-121 for n_frames network inputs of one size in two launches: loc_dev (n_frames,P,4), conf_dev
 * (n_frames,P,2) as syn_fb_forward_batch writes them.  Every frame has its own candidates, its own ranking (same tie
 * rule), its own (top_k,5) block of dets_dev (n_frames,top_k,5) and its own count in n_dets_dev (n_frames).
 * cand_ws_dev: n_frames * (P+1) int32.  n_frames <= SYN_FB_MAX_FRAMES. */
int syn_faceboxes_decode_batch(const float* loc_dev, const float* conf_dev, int n_frames, int im_height, int im_width,
                               float box_scale_w, float box_scale_h, float scale, float conf_thresh, int top_k, int32_t* cand_ws_dev,
                               float* dets_dev, int32_t* n_dets_dev, void* stream);
/* FaceBoxes.py:98-121 (FaceBoxes.__call__ once per image) for n_images network inputs of any sizes in the same two
 * launches: loc_dev (sum P_i,4), conf_dev (sum P_i,2) as syn_fb_forward_images writes them, P_i =
 * syn_faceboxes_num_priors(heights_host[i], widths_host[i]) and image i's priors after those of images 0..i-1.  Image i
 * decodes with box scale (widths_host[i], heights_host[i]) (:101) and shrink factor scale_host[i] (:104) into its own
 * (top_k,5) block of dets_dev (n_images,top_k,5) and its own count in n_dets_dev (n_images): the rows and count
 * syn_faceboxes_decode gives for that image alone.  cand_ws_dev: n_images + sum P_i int32.  1 <= n_images <=
 * SYN_FB_MAX_FRAMES; sizes < 1 or a scale that is not > 0 are SYN_ERR_INVALID before anything is launched. */
int syn_faceboxes_decode_images(const float* loc_dev, const float* conf_dev, int n_images, const int32_t* heights_host,
                                const int32_t* widths_host, const float* scale_host, float conf_thresh, int top_k, int32_t* cand_ws_dev,
                                float* dets_dev, int32_t* n_dets_dev, void* stream);

/* ---- crop + resize of uint8 BGR images (crop_img + cv2.resize) ---------------------------------------------------------
 * The face crops of get_all_outputs (utils/inference.py:95-125 crop_img, then cv2.resize to 120x120: INTER_LANCZOS4 in
 * synergy3DMM.py:187-188 / model_building.py:286-287, INTER_LINEAR in singleImage.py:76-77 / artistic.py:95) and the
 * detector's shrink of oversized images (FaceBoxes/FaceBoxes.py:62-79, cv2.resize's default INTER_LINEAR; ROI = the whole
 * image).  The output is OpenCV's, byte for byte, including the fast 2x2 area path INTER_LINEAR takes for an exact
 * halving (csrc/resize_math.h states the arithmetic).  Handle-free, in two steps like syn_mesh_incidence_host +
 * syn_mesh_normals: the host planner turns rois_host (B,4) int32 x0, y0, x1, y1 (crop_img's int(round(v)), may reach
 * outside the image: crop pixels there are 0) into one plan buffer of syn_crop_resize_plan_size bytes (-1 on bad
 * arguments) with the per-axis tap tables; the caller uploads it and syn_crop_resize reads image_dev (height,width,3)
 * uint8 and writes B outputs of out_h x out_w x 3 through element strides: channel c of pixel (y, x) of ROI b is
 * out_dev[b*stride_roi + y*stride_y + x*stride_x + c*stride_c] -- (3*h*w, w, 1, h*w) for planar (B,3,h,w) crops, (0, 3*w,
 * 3, 1) for one interleaved (h,w,3) image.  batch, out_h, out_w and mode must be the ones the plan was built with.
 * Empty ROIs are SYN_ERR_SHAPE, sizes < 1 SYN_ERR_INVALID, channels != 3 and other modes SYN_ERR_UNSUPPORTED. */
enum {
  SYN_INTER_LINEAR = 1,    /* cv::INTER_LINEAR   */
  SYN_INTER_LANCZOS4 = 4   /* cv::INTER_LANCZOS4 */
};
int64_t syn_crop_resize_plan_size(int batch, int out_h, int out_w, int mode);
int syn_crop_resize_plan_host(const int32_t* rois_host, int batch, int out_h, int out_w, int mode, void* plan_out,
                              int64_t plan_bytes);
int syn_crop_resize(const uint8_t* image_dev, int height, int width, int channels, const void* plan_dev, int batch, int out_h,
                    int out_w, int mode, uint8_t* out_dev, int64_t stride_roi, int64_t stride_y, int64_t stride_x, int64_t stride_c,
                    void* stream);
/* The same stage for a stack of equally sized frames in ONE launch: the crops of every face of every frame
 * (synergy3DMM.py:186-188 once per face per image), or the detector's shrink of every frame (FaceBoxes.py:62-79; ROI =
 * the whole frame, interleaved output).  The planner also takes frames_host (B): ROI b is cut out of frame
 * frames_host[b] of n_frames (outside 0..n_frames-1: SYN_ERR_SHAPE); the plan has syn_crop_resize_plan_size bytes and
 * the same tables.  images_dev (n_frames,height,width,3).  Output bytes are those of syn_crop_resize on each frame. */
int syn_crop_resize_plan_frames_host(const int32_t* rois_host, const int32_t* frames_host, int n_frames, int batch, int out_h,
                                     int out_w, int mode, void* plan_out, int64_t plan_bytes);
int syn_crop_resize_batch(const uint8_t* images_dev, int n_frames, int height, int width, int channels, const void* plan_dev,
                          int batch, int out_h, int out_w, int mode, uint8_t* out_dev, int64_t stride_roi, int64_t stride_y,
                          int64_t stride_x, int64_t stride_c, void* stream);
/* The same stage for a list of images of any sizes in ONE launch, every ROI with its own output size: the crops of every
 * face of every image (synergy3DMM.py:186-188 once per face per image), or the detector's shrink of every oversized image
 * to its own size (FaceBoxes.py:62-79, a different scale per image).  images_dev: n_images uint8 BGR images packed back to
 * back, image i (heights_host[i] x widths_host[i] x 3) at byte sum_{j<i} 3 h_j w_j.  ROI b reads image images_host[b] and
 * is resized to out_h_host[b] x out_w_host[b]; its output follows the outputs of ROIs 0..b-1 (3 out_h out_w bytes each),
 * planar (3,h,w) when planar = 1, interleaved (h,w,3) when planar = 0.  The plan, syn_crop_resize_images_plan_size bytes
 * (-1 for a bad argument), is CropImagesRoi[batch] followed by, for every ROI, the bytes syn_crop_resize_plan_host makes
 * for that ROI alone.  Output bytes are those of syn_crop_resize on each image.  Null pointers, an empty batch, sizes < 1
 * and an unknown mode fail before anything is written or launched; an image index outside 0..n_images-1 is
 * SYN_ERR_SHAPE. */
int64_t syn_crop_resize_images_plan_size(int batch, const int32_t* out_h_host, const int32_t* out_w_host, int mode);
int syn_crop_resize_plan_images_host(const int32_t* rois_host, const int32_t* images_host, int n_images, const int32_t* heights_host,
                                     const int32_t* widths_host, int batch, const int32_t* out_h_host, const int32_t* out_w_host,
                                     int mode, void* plan_out, int64_t plan_bytes);
int syn_crop_resize_images(const uint8_t* images_dev, const void* plan_dev, int batch, const int32_t* out_h_host, const int32_t* out_w_host,
                           int mode, int planar, uint8_t* out_dev, void* stream);

/* The detector network (FaceBoxes/models/faceboxes.py:68-150, FaceBoxesNet in 'test' phase) on ONE image of any size
 * (syn_fb_forward), on a stack of frames of one size (syn_fb_forward_batch), or on a list of images of any sizes
 * (syn_fb_forward_images).
 * A separate handle: the detector has its own weights and workspace and does not touch syn_handle_t.  Like syn_handle_t
 * it is bound to one device and is not re-entrant (its activation workspace is shared by consecutive calls, which are
 * ordered by the stream they are enqueued on).  The workspace only grows: a call that needs more bytes than an earlier
 * one synchronises the device and reallocates (SYN_ERR_STATE under capture), a call that fits runs without any
 * synchronisation.  Only syn_fb_forward can be captured in a CUDA graph (see the conventions at the top).
 * 33 convolutions in execution order (syn_fb_layer_desc names them with the reference's state_dict prefixes:
 * "conv1", "inception2.branch3x3_2", "loc.0" ...): layers with has_bn take the conv weight (OIHW fp32, no bias) and
 * the eval-mode BatchNorm2d of the same block (<name>.conv.weight / <name>.bn.*), the six head layers take weight +
 * bias.  activation: 0 none, 1 ReLU (BasicConv2d, :8-18), 2 CReLU (:50-64, output has 2*cout channels). */
typedef struct syn_fb syn_fb_t;
typedef struct {
  const char* name;
  int32_t cin, cout, ksize, stride, pad, has_bn, activation;
} syn_fb_layer_desc_t;
int  syn_fb_num_layers(void);                                 /* 33 */
int  syn_fb_layer_desc(int idx, syn_fb_layer_desc_t* out);
int  syn_fb_create(int device, syn_fb_t** out);
void syn_fb_destroy(syn_fb_t* f);
int  syn_fb_set_layer(syn_fb_t* f, int idx, const float* w_host, int64_t w_numel, const float* bias_host, const float* bn_weight_host,
                      const float* bn_bias_host, const float* bn_mean_host, const float* bn_var_host, float eps);
int  syn_fb_commit(syn_fb_t* f);
/* FaceBoxes.__call__ lines 88-96: image_dev (height,width,3) uint8 BGR as cv2 delivers it (already rescaled by the caller,
 * :62-79); the mean (104,117,123) is subtracted on the fly.  loc_dev (P,4) and conf_dev (P,2, softmax applied) are what
 * `self.net(img)` returns, P = syn_faceboxes_num_priors(height, width); feed them to syn_faceboxes_decode + syn_nms. */
int  syn_fb_forward(syn_fb_t* f, const uint8_t* image_dev, int height, int width, float* loc_dev, float* conf_dev, void* stream);
int64_t syn_fb_launch_count(const syn_fb_t* f);
/* FaceBoxes.__call__ lines 88-96 for n_frames images of one size in the SAME 39 launches (syn_fb_launch_count grows by 39
 * whatever n_frames is): images_dev (n_frames,height,width,3) uint8 BGR -> loc_dev (n_frames,P,4), conf_dev
 * (n_frames,P,2).  This is syn_fb_forward_images with every size equal.  Rows of every convolution's implicit GEMM run
 * over the packed pixels of all frames; each output element is computed by the one-image kernel's arithmetic in its
 * order, so frame i's outputs are, bit for bit, syn_fb_forward's for image i.  The workspace grows to n_frames times the
 * one-image maps (15.5 MB per 720 x 1080 frame, so about 1 GB at SYN_FB_MAX_FRAMES); more frames per call are
 * SYN_ERR_INVALID, callers split the stack. */
#define SYN_FB_MAX_FRAMES 64
int  syn_fb_forward_batch(syn_fb_t* f, const uint8_t* images_dev, int n_frames, int height, int width, float* loc_dev,
                          float* conf_dev, void* stream);
/* FaceBoxes.__call__ lines 88-96 (FaceBoxes/FaceBoxes.py, once per image) for n_images images of any sizes in the SAME 39
 * launches: images_dev holds them packed back to back, image i (heights_host[i] x widths_host[i] x 3 uint8 BGR) at byte
 * sum_{j<i} 3 h_j w_j; loc_dev (sum P_i,4) and conf_dev (sum P_i,2) get image i's priors after those of images 0..i-1.
 * Every map of the network is packed the same way; each launch takes a per-image geometry table (map sizes and first
 * pixel of every image at every map size), uploaded with one asynchronous copy per call.  Image i's outputs are, bit for
 * bit, syn_fb_forward's on image i alone.  1 <= n_images <= SYN_FB_MAX_FRAMES; null pointers and sizes < 1 fail before
 * anything is launched. */
int  syn_fb_forward_images(syn_fb_t* f, const uint8_t* images_dev, int n_images, const int32_t* heights_host, const int32_t* widths_host,
                           float* loc_dev, float* conf_dev, void* stream);
/* Per-stage tests of the detector network.  Runs syn_fb_forward's launch sequence unchanged and returns right after launch
 * `stage` (0..38), having copied (on the stream) the whole tensor that launch wrote to out_dev, which holds out_numel
 * floats (SYN_ERR_SHAPE if that is not the tensor's size).  The activation workspace is zeroed first, so channel slices
 * of that tensor which later launches would write read 0.  NHWC maps of an h x w image, n3/n4/n5 = the pixels of the
 * stride-32/64/128 maps, P = syn_faceboxes_num_priors(h, w):
 *   0 conv1 (CReLU, 48 ch)   1 max-pool (48 ch)   2 conv2 (CReLU, 128 ch)   3 max-pool (128 ch: inception1's input)
 *   4 + 8b .. 11 + 8b, inception b = 0..2: branch1x1 -> block output (all 128 ch; it owns 0..31), avg-pool of the
 *     block input (128 ch), branch1x1_2 -> block output (owns 32..63), branch3x3_reduce (24 ch), branch3x3 -> block
 *     output (owns 64..95), branch3x3_reduce_2 (24 ch), branch3x3_2 (32 ch), branch3x3_3 -> block output (owns 96..127)
 *   28 conv3_1 (128 ch)   29 conv3_2 (256 ch)   30 conv4_1 (128 ch)   31 conv4_2 (256 ch)
 *   32..34 loc.0..2 -> the whole loc_dev (P*4; loc.k owns offsets from 0, n3*84, n3*84 + n4*4)
 *   35..37 conf.0..2 -> the whole conf_dev (P*2 logits; offsets 0, n3*42, n3*42 + n4*2)   38 softmax -> conf_dev (P*2)
 * The block input is stage 3 for inception1 and the previous block's stage 11 + 8b otherwise. */
int  syn_fb_debug_forward_until(syn_fb_t* f, const uint8_t* image_dev, int height, int width, int stage, float* out_dev,
                                int64_t out_numel, float* loc_dev, float* conf_dev, void* stream);
/* syn_fb_forward_batch stopped after launch `stage` of the same table: out_dev receives the (n_frames,h,w,c) stack of that
 * launch's maps, or the whole (n_frames,P*4) loc / (n_frames,P*2) conf for stages 32..38. */
int  syn_fb_debug_forward_batch_until(syn_fb_t* f, const uint8_t* images_dev, int n_frames, int height, int width, int stage,
                                      float* out_dev, int64_t out_numel, float* loc_dev, float* conf_dev, void* stream);
/* syn_fb_forward_images stopped after launch `stage` of the same table: out_dev receives every image's map of that launch
 * packed back to back (image i's (h_i,w_i,c) map after those of images 0..i-1), or the whole packed (sum P_i * 4) loc /
 * (sum P_i * 2) conf for stages 32..38. */
int  syn_fb_debug_forward_images_until(syn_fb_t* f, const uint8_t* images_dev, int n_images, const int32_t* heights_host,
                                       const int32_t* widths_host, int stage, float* out_dev, int64_t out_numel, float* loc_dev,
                                       float* conf_dev, void* stream);

/* ---- introspection ---------------------------------------------------------------------------*/
/* Number of kernels this handle has launched since creation (bench.py "gpu_launches"). */
int64_t syn_launch_count(const syn_handle_t* h);
/* Per-launch device timing of the LAST device-buffer call (syn_forward / syn_forward_landmarks[_u8] /
 * syn_reconstruct): with timing on, a CUDA event is recorded on the caller's stream behind every kernel.
 * syn_get_timings synchronises and returns up to max_entries durations (ms) with the kernel labels
 * (static strings; names_out may be NULL).  Used by bench.py for the per-kernel roofline. */
int syn_set_timing(syn_handle_t* h, int on);
int syn_get_timings(syn_handle_t* h, float* ms_out, const char** names_out, int max_entries, int* n_out);
/* Synchronise the device and report (then clear) the sticky flag a bounded in-kernel wait raises
 * when it times out (pipeline protocol bug); *flag_out = 0 means no kernel ever timed out.
 * While the flag is raised every compute entry point returns SYN_ERR_CUDA instead of results. */
int syn_poll_error(syn_handle_t* h, int* flag_out);
/* The same flag WITHOUT synchronising or clearing (it lives in mapped host memory): cheap enough to
 * call after any host-side synchronisation point. */
int syn_peek_error(const syn_handle_t* h, int* flag_out);
/* Synchronise and report (then clear) the sticky "activation clamped" flag of this handle: the
 * split-fp16 engines scale an activation by 64 and clamp it to +-60000 before the fp16 hi/lo split, so
 * an input with |x| > 937.5, +-Inf or NaN is changed (NaN is read as -937.5).  The flag is raised
 * wherever that happens: the fused block kernel's input (the fp32 crop at the stem and the inputs of
 * blocks 2-17; engines 2, 3), the tail kernel's input (the block-17 output; engines 2, 3) and the input
 * of every expand conv and of conv 51 on the unfused tensor-core engine (engine 1).  The GEMM layers
 * (ResNets, MobileNetV1, PointNet heads) scale every finite input into range and raise it for a +-Inf
 * or NaN input value (or a value about twice the row maximum they were given or more); the dense reconstruction raises it for a +-Inf or NaN coefficient.  The fp32
 * engine (SYN_ENGINE_SIMT_FP32) has no such limit.  *flag_out != 0: results of engines 1-3 (or of the
 * GEMM layers and the dense mesh) are suspect. */
int syn_poll_saturation(syn_handle_t* h, int* flag_out);
/* Run the backbone on x_dev but stop after convolution `layer` (0..51) and copy its NHWC
 * activation (batch*h_out*h_out*cout floats, residual already added for project convs) to
 * out_dev.  Per-layer parity tests only. */
int syn_debug_forward_until(syn_handle_t* h, const float* x_dev, int batch, int layer,
                            float* out_dev, void* stream);

/* Per-stage tests of the GEMM layers.  Both run the production launch sequence unchanged up to `stage` and copy that
 * stage's fp32 output to out_dev and, when the stage records them, its per-row maxima (fp32 bit patterns, what the next
 * GEMM scales its rows by) to rowmax_dev (nullable; left untouched for a stage that records none).
 * ResNet-50 (NHWC rows, one per pixel): 0 stem (B*3600 x 64), 1 max-pool (B*900 x 64), 1 + i conv i of
 * syn_resnet_conv_desc (i = 1..52; a block's downsample runs before its conv3 and records no row maxima), 54 avgpool
 * (B x 2048), 55 heads (B x 102, no row maxima).  For the selected arch with n convs (syn_resnet_arch_num_convs):
 * 1 + i conv i of syn_resnet_arch_conv_desc (i = 1..n-1; a downsample runs before the conv that adds it), n + 1 avgpool
 * (B x 512 or 2048), n + 2 heads.  x_dev: fp32 crops. */
int syn_debug_resnet_until(syn_handle_t* h, const float* x_dev, int batch, int stage, float* out_dev, unsigned* rowmax_dev,
                           void* stream);
/* MobileNetV1 (NHWC rows, one per pixel; C_i = cout of conv i of syn_mbv1_conv_desc): 0 stem (B*3600 x C_0),
 * 2j - 1 / 2j conv_dw / conv_sep of block j = 1..13 (B*HO*HO x C_i; every stage records row maxima except the conv_seps
 * of blocks 1..12), 27 avgpool (B x 1024w), 28 heads (B x 102, no row maxima).  x_dev: fp32 crops. */
int syn_debug_mbv1_until(syn_handle_t* h, const float* x_dev, int batch, int stage, float* out_dev, unsigned* rowmax_dev,
                         void* stream);
/* GhostNet: one stage per launch output, in launch order -- stem; per block the primary GEMM's x1, the ghost concat
 * [x1 | cheap(x1)], conv_dw, the SE pooled vector / conv_reduce (its columns padded to a multiple of 8 with exact zeros)
 * / conv_expand / gated map, ghost2's x1, the shortcut's depthwise / pointwise outputs, and ghost2's concat with the
 * shortcut added; then ConvBnAct, avgpool, conv_head, heads (the last stage; 111 in all).  syn_ghost_stage_desc gives
 * each stage's rows per face (pixels, or 1), its columns and whether it records row maxima (max |row| as fp32 bits).
 * x_dev: fp32 crops. */
int syn_ghost_num_stages(void);                              /* 111 */
int syn_ghost_stage_desc(int stage, int* rows_per_face, int* cols, int* has_rowmax);
int syn_debug_ghost_until(syn_handle_t* h, const float* x_dev, int batch, int stage, float* out_dev, unsigned* rowmax_dev,
                          void* stream);
/* PointNet heads (rows = B*68 point-major, or B): net 0 = MLP_for: 0..4 conv1..conv5 (64, 64, 64, 128, 1024 columns;
 * conv5 is written only by this call, without row maxima), 5 the max-pooled global features (B x 1024), 6 the face vector
 * (B x 2360), 7 conv6's face part (B x 512, no row maxima), 8 conv6's point part (512), 9 conv7 (256), 10 conv8 (128),
 * 11 conv9 (3, no row maxima), 12 point_residual (B,3,68).  pool1280_dev / params62_dev as for syn_mlp_for.
 * net 1 = MLP_rev (pool1280_dev / params62_dev unused): 0..4 as above, 5 the global features (B x 1024), 6 the heads (B x 62). */
int syn_debug_pointnet_until(syn_handle_t* h, int net, const float* lmk_dev, const float* pool1280_dev,
                             const float* params62_dev, int batch, int stage, float* out_dev, unsigned* rowmax_dev,
                             void* stream);
/* One tc_gemm_kernel launch on a temporary layer built from host weights w_host (N x K fp32, K in the GEMM's k order,
 * bias_host N): out[m, n] = act(sum_k A[m, k] W[n, k] + bias[n] + addend[m / addend_group, n] + residual[m, n]),
 * act 0 none / 2 ReLU.  ksize = 0: plain rows, a_dev [M][lda]; ksize > 0: implicit GEMM over the ksize x ksize x C patch
 * of NHWC a_dev (M / (HO*WO) maps of H x W x C, K = ksize*ksize*C).  rowmax_in_dev: the caller's max|a| per row (per
 * input pixel in conv mode), as fp32 bits.  residual_dev, addend_dev, colmax_dev (zeroed by the caller) and
 * rowmax_out_dev are nullable.  K and C must be multiples of 8.  Synchronises the stream. */
int syn_debug_gemm(syn_handle_t* h, const float* w_host, const float* bias_host, int N, int K, int act, int ksize,
                   int stride, int pad, int H, int W, int C, const float* a_dev, int M, int lda, const unsigned* rowmax_in_dev,
                   const float* residual_dev, const float* addend_dev, int addend_group, unsigned* colmax_dev,
                   int colmax_group, float* out_dev, unsigned* rowmax_out_dev, void* stream);

/* Host-only: the face-group plan the fused engine uses for a launch over `batch` faces on a GPU with
 * `sms` SMs and `faces_per_tile` (1, 2 or 4) faces per full tile.  Groups [0, *split) hold
 * faces_per_tile faces each; for two-face tiles the groups [*split, *face_groups) hold ONE face each
 * (the partial last wave is split so that more SMs share it), otherwise the last group may be
 * partial.  Lets the host logic be tested without a GPU. */
int syn_debug_tile_plan(int batch, int sms, int faces_per_tile, int* split, int* face_groups);

/* Poisoned-workspace tests only; no product path calls these.  A handle's workspaces only grow and are never cleared, so
 * a call smaller than an earlier one runs on that call's bytes past its own extent.  syn_debug_fill_workspaces sets every
 * byte of every device buffer the handle has grown -- at its allocated size, not the last call's -- to `byte` (0..255)
 * with stream-ordered memsets on `stream`, and reports the total in *bytes_filled (nullable): the MobileNetV2 activations,
 * d_params_tmp and d_pool_tmp, the uint8 crops' fp32 scratch, the reconstruction tiles, the host pipelines' staging
 * buffers (their streams wait for the fill), the PointNet workspace and the conv+BN backbone workspaces.  Weights, packed
 * bases, plans and the error and saturation flags are not touched.  syn_fb_debug_fill_workspaces does the same for the
 * detector's 13 activation buffers; its geometry table (pixel offsets) is cleared to 0 and counted, never filled with
 * `byte`.  Both refuse a capturing stream with SYN_ERR_STATE, so a fill is never recorded into a graph.
 * syn_debug_fill_on_grow / syn_fb_debug_fill_on_grow: every later workspace growth of the handle sets its new buffers
 * to `byte` right after allocating them (the detector's geometry table to 0); -1 (the default) turns this off. */
int syn_debug_fill_workspaces(syn_handle_t* h, int byte, size_t* bytes_filled, void* stream);
int syn_debug_fill_on_grow(syn_handle_t* h, int byte);
int syn_fb_debug_fill_workspaces(syn_fb_t* f, int byte, size_t* bytes_filled, void* stream);
int syn_fb_debug_fill_on_grow(syn_fb_t* f, int byte);

#ifdef __cplusplus
}
#endif
#endif  /* SYNERGY_H100_H_ */
