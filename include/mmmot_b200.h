/*
 * mmmot_b200.h — C ABI of libmmmot_sm90a.so
 *
 * CUDA-native (sm_90a, H100) implementation of mmMOT's per-frame-pair association forward.
 * The reference (ZwwWayne/mmMOT) has no FFI of its own: its boundary is the Python class
 * modules/tracking_net.py:15 `TrackingNet` and the function solvers.py:9 `ortools_solve`.
 * Each entry point below replaces one group of ATen/OR-tools calls behind that boundary; the
 * reference lines replaced are cited per function.  INTEGRATION.md shows the ctypes binding.
 *
 * Conventions
 *   - plain pointers + sizes only; every pointer is a DEVICE pointer unless marked host.
 *   - no allocation, no ownership transfer, stateless, stream-ordered (last argument is a
 *     cudaStream_t passed as void*), thread-safe across streams.
 *   - return 0 on success, a negative MMMOT_E_* on a bad argument, or a positive cudaError_t.
 *   - every `workspace` starts with a 256-byte STATUS BLOCK (included in the mmmot_*_workspace sizes): stages raise
 *     flags in it while they run and never clear it.  Protocol: mmmot_status_reset(ws) -> stages ... -> mmmot_status_check(ws).
 *   - all real data is fp32; `stats` scratch is fp64.
 *   - "group" = one GroupNorm domain.  A frame-pair with N previous / M next detections has
 *     L = N + M detections; all pairs of one call share N, M, crop size H x W.
 *   - feature tensors are channel-major: feats[pair][stack 0..2][512][L]
 *     (stack 0 = image, 1 = LiDAR, 2 = fused; reference: modules/tracking_net.py:40,131-145).
 */
#ifndef MMMOT_B200_H
#define MMMOT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMMOT_ABI_VERSION 3

enum {
  MMMOT_E_ARG = -1,        /* null pointer / non-positive size / unsupported enum */
  MMMOT_E_WORKSPACE = -2,  /* workspace too small */
  MMMOT_E_SHAPE = -3,      /* shape constraint violated (see function comment) */
  MMMOT_E_RANGE = -4       /* an activation left FP16's range (|x| >= 65504) on the tensor-core path: the result
                              of the stage that raised it is clamped, i.e. WRONG (mmmot_status_check) */
};

/* fusion_module_{A,B,C}: reference modules/fusion_net.py:73,45,6 */
enum { MMMOT_FUSION_A = 0, MMMOT_FUSION_B = 1, MMMOT_FUSION_C = 2 };
/* batch_multiply / batch_minus_abs / batch_minus: reference modules/gcn.py:6,17,32 */
enum { MMMOT_AFF_MULTIPLY = 0, MMMOT_AFF_MINUS_ABS = 1, MMMOT_AFF_MINUS = 2 };
/* softmax_mode: reference modules/tracking_net.py:109-124 */
enum { MMMOT_SM_NONE = 0, MMMOT_SM_SINGLE = 1, MMMOT_SM_DUAL = 2, MMMOT_SM_DUAL_ADD = 3, MMMOT_SM_DUAL_MAX = 4 };
/* NewEndIndicator_v2 mode: reference modules/new_end.py:69-74 (mean / max of the normalised map over the other frame) */
enum { MMMOT_END_AVG = 0, MMMOT_END_MAX = 1 };

/*
 * Prepared weights.  Produced once per checkpoint by the host (mmmot_b200/weights.py) from the
 * reference state_dict: eval-mode BatchNorm folded into the preceding conv, the two constant
 * STN transforms (SURVEY F4) folded into the PointNet convs they feed, every matrix stored
 * TRANSPOSED as Wt[K][Cout] (K-major rows, Cout contiguous).
 */
enum mmmot_weight_id {
  /* VGG16-BN trunk, 13 convs: Wt[(ky*3+kx)*Cin + ci][Cout], bias[Cout]  (appear_net.py:166-172) */
  MMMOT_W_VGG_WT0 = 0,            /* .. +12 */
  MMMOT_W_VGG_B0 = 13,            /* .. +12 */
  /* SkipPool heads s=0..3, 10 tensors each (appear_net.py:18-32):
     +0 gn0_w[C] +1 gn0_b[C] +2 w1t[C][mid] +3 b1[mid] +4 gn1_w +5 gn1_b +6 w2t[mid][128] +7 b2 +8 gn2_w +9 gn2_b */
  MMMOT_W_SKIP0 = 26,             /* .. +39 */
  /* PointNet trunk (point_net.py:115-138), layer i=1..5: +0 wt[Cin][Cout] +1 b +2 gn_w +3 gn_b */
  MMMOT_W_PN_L1 = 66,             /* .. 5 layers x 4 = 20 */
  /* PointNet head (point_net.py:25-41) */
  MMMOT_W_PN_WHAT = 86,           /* [64][512]   local-feature part of conv1, T2 folded in   */
  MMMOT_W_PN_WHGT = 87,           /* [1024][512] global-feature part of conv1                */
  MMMOT_W_PN_BH = 88, MMMOT_W_PN_GHW = 89, MMMOT_W_PN_GHB = 90,
  MMMOT_W_PN_WOT = 91,            /* [512][512] conv2 */
  MMMOT_W_PN_BO = 92, MMMOT_W_PN_GOW = 93, MMMOT_W_PN_GOB = 94,
  /* fusion (fusion_net.py): A uses WPT as the [1024][512] matrix; B uses WPT/WIT; C adds gates */
  MMMOT_W_FU_WPT = 95, MMMOT_W_FU_BP = 96, MMMOT_W_FU_GPW = 97, MMMOT_W_FU_GPB = 98,
  MMMOT_W_FU_WIT = 99, MMMOT_W_FU_BI = 100, MMMOT_W_FU_GIW = 101, MMMOT_W_FU_GIB = 102,
  MMMOT_W_FU_GATE_PT = 103, MMMOT_W_FU_GATE_PB = 104, MMMOT_W_FU_GATE_IT = 105, MMMOT_W_FU_GATE_IB = 106,
  /* w_det (tracking_net.py:92-100), BN folded */
  MMMOT_W_WD_W1T = 107, MMMOT_W_WD_B1 = 108, MMMOT_W_WD_W2T = 109, MMMOT_W_WD_B2 = 110,
  MMMOT_W_WD_W3 = 111, MMMOT_W_WD_B3 = 112,
  /* affinity (gcn.py:59-66) + new/end conv0 (new_end.py:48-52) stacked as one [512][1024] matrix */
  MMMOT_W_AF_W01T = 113, MMMOT_W_AF_B01 = 114,
  MMMOT_W_AF_G1W = 115, MMMOT_W_AF_G1B = 116,   /* conv1.1  GN(512,512) */
  MMMOT_W_AF_G0W = 117, MMMOT_W_AF_G0B = 118,   /* w_new_end.conv0.1  GN(1,512) */
  MMMOT_W_AF_W2T = 119, MMMOT_W_AF_B2 = 120, MMMOT_W_AF_G2W = 121, MMMOT_W_AF_G2B = 122,
  MMMOT_W_AF_W3T = 123, MMMOT_W_AF_B3 = 124, MMMOT_W_AF_G3W = 125, MMMOT_W_AF_G3B = 126,
  MMMOT_W_AF_W4 = 127, MMMOT_W_AF_B4 = 128,
  /* new/end 1-D MLP (new_end.py:53-60) */
  MMMOT_W_NE_W1T = 129, MMMOT_W_NE_B1 = 130, MMMOT_W_NE_G1W = 131, MMMOT_W_NE_G1B = 132,
  MMMOT_W_NE_W2T = 133, MMMOT_W_NE_B2 = 134, MMMOT_W_NE_G2W = 135, MMMOT_W_NE_G2B = 136,
  MMMOT_W_NE_W3 = 137, MMMOT_W_NE_B3 = 138,
  /* ---- tensor-core operands: the same matrices split into FP16 hi/lo and pre-tiled in the wgmma
     canonical K-major core-matrix layout  [k chunk 32][m tile 128][hi|lo][k group 4][m group 16][8][8]
     (zero padded to multiples of 128 rows / 32 k); see weights.py::pack_tc.  VGG layer 0 (fp32 NCHW crops) uses
     the K order k = ci*9 + (ky*3+kx); layers 1..12 (packed FP16 NHWC activations) use k = (ky*3+kx)*Cin + ci. */
  MMMOT_W_VGG_WP0 = 139,          /* .. +12 */
  MMMOT_W_PN_WP1 = 152,           /* .. +4 : PointNet trunk layers 1..5 */
  MMMOT_W_PN_WHAP = 157,
  MMMOT_W_AF_W01P = 158, MMMOT_W_AF_W2P = 159, MMMOT_W_AF_W3P = 160,
  /* ---- training-mode operands (SURVEY 8f N4): the UNFOLDED conv weights / biases and the BatchNorm affines of the
     layers whose BatchNorm uses batch statistics in .train() */
  MMMOT_W_VGG_RAWW0 = 161,        /* .. +12 : Wt[(ky*3+kx)*Cin + ci][Cout], not folded */
  MMMOT_W_VGG_RAWB0 = 174,        /* .. +12 */
  MMMOT_W_VGG_BNW0 = 187,         /* .. +12 : BatchNorm2d weight */
  MMMOT_W_VGG_BNB0 = 200,         /* .. +12 : BatchNorm2d bias */
  MMMOT_W_WD_RAW0 = 213,          /* .. +7  : w_det w1t b1 bn1_w bn1_b w2t b2 bn2_w bn2_b */
  /* ---- packed tensor-core tiles of the per-detection contractions (fusion linears, gates, w_det; BN folded) */
  MMMOT_W_FU_WPP = 221, MMMOT_W_FU_WIP = 222, MMMOT_W_FU_GATE_PP = 223, MMMOT_W_FU_GATE_IP = 224,
  MMMOT_W_WD_W1P = 225, MMMOT_W_WD_W2P = 226,
  /* the two 64-output VGG layers again, compact for the pixel-major kernel: [k chunk][hi|lo][k group 4][row group 8][8][8] */
  MMMOT_W_VGG_WPX0 = 227,         /* .. +1 */
  /* packed tiles of the remaining small contractions: new/end MLP, PointNet per-detection parts */
  MMMOT_W_NE_W1P = 229, MMMOT_W_NE_W2P = 230, MMMOT_W_PN_WHGP = 231, MMMOT_W_PN_WOP = 232,
  MMMOT_W_COUNT = 233
};

typedef struct mmmot_weights {
  const float* w[MMMOT_W_COUNT];
  /* for the packed tensor-core operands (ids >= MMMOT_W_VGG_WP0): 2^-s, where the packed FP16 tiles
     hold W * 2^s (power-of-two pre-scaling keeps the lo terms in FP16's normal range) */
  float tc_scale[MMMOT_W_COUNT];
  /* width of PointNet's input points, a property of the checkpoint (point_net.feat.conv1.weight.shape[1]): 3 = xyz,
     4 = xyz + LiDAR reflectance (reference without_reflectivity: False, modules/tracking_net.py:41) */
  int point_channels;
} mmmot_weights;

int mmmot_abi_version(void);

/* Status block of a workspace (see Conventions).  reset: stream-ordered clear.  check: copies the status word back,
 * SYNCHRONISES the stream and returns 0 or MMMOT_E_RANGE.  The tensor-core engines feed activations to the MMA units
 * as FP16 hi/lo pairs; a value with |x| >= 65504 saturates in that conversion, which these calls make loud. */
int mmmot_status_reset(void* workspace, void* stream);
int mmmot_status_check(const void* workspace, void* stream);
/* Small stream-ordered host -> device transfer that uses NEITHER the copy engine NOR a host synchronisation: a kernel
 * reads `count` int32 words straight from PINNED (page-locked, mapped) host memory.  For the CSR offsets that accompany
 * a sub-batch: a cudaMemcpyAsync of them would queue on the copy engine behind the bulk input copies of the NEXT
 * sub-batch (stalling the compute stream for milliseconds), a pageable copy blocks the calling thread.  The source
 * must stay untouched until the stream has passed this call.  MMMOT_E_ARG if `src_pinned_host` is not pinned. */
int mmmot_fetch_pinned_i32(int* dst_device, const int* src_pinned_host, long count, void* stream);
/* number of SMs / name of the current device: lets the host fail loudly when no sm_90 GPU is present */
int mmmot_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------
 * Appearance: VGG16-BN trunk + 4 SkipPool heads -> stack 0 of feats.
 * Replaces AppearanceNet.forward, reference modules/appear_net.py:166-190 (+ vgg.py:67-80).
 *   crops  [n_img][3][H][W]   (H, W multiples of 32), n_img = pairs*L
 *   feats  [pairs][3][512][L] ; writes feats[p][0][:][l] for image p*L + l
 * workspace: mmmot_appearance_workspace(n_img, H, W) bytes.
 */
size_t mmmot_appearance_workspace(int n_img, int H, int W);
int mmmot_appearance_fwd(const mmmot_weights* wts, const float* crops, int n_img, int H, int W,
                         int L, float* feats, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * PointNet encoder over ragged per-detection point sets -> stack 1 of feats.
 * Replaces PointNet_v1.forward, reference modules/point_net.py:25-44,115-153.
 *   points     [P_total][C]  C = wts->point_channels: xyz, or xyz + reflectance (16-byte aligned rows), detections
 *                            concatenated in order; any other point_channels (or misaligned 4-channel points) returns
 *                            MMMOT_E_ARG before any CUDA call
 *   det_split  [pairs*L + 1] int32 CSR offsets into points (device)
 *   h_det_split same array on the HOST (used only to size the launch; the reference reads it
 *               with .item() per detection, point_net.py:33-35,140-142)
 * Every pair is one GroupNorm domain (all points of its L detections).
 */
size_t mmmot_pointnet_workspace(int pairs, int L, long p_total);
int mmmot_pointnet_fwd(const mmmot_weights* wts, const float* points, const int* det_split,
                       const int* h_det_split, int pairs, int L, float* feats,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fusion A/B/C -> stack 2 of feats, then the detection-score branch on all 3 stacks.
 * Replaces fusion_module_{A,B,C}.forward (modules/fusion_net.py:31-42,62-70,85-92) and
 * TrackingNet.determine_det eval branch (modules/tracking_net.py:149-163).
 *   det_scores [pairs][3][L]   = s - [s < neg_threshold],  s = sigmoid(w_det(feats)) if score_flags & MMMOT_SCORE_SIGMOID
 *                                ('cls' in score_arch, tracking_net.py:153-156) else w_det(feats);
 *                                the threshold step is skipped without MMMOT_SCORE_THRESHOLD.
 */
enum { MMMOT_SCORE_SIGMOID = 1, MMMOT_SCORE_THRESHOLD = 2 };
size_t mmmot_fusion_det_workspace(int pairs, int L);
int mmmot_fusion_det_fwd(const mmmot_weights* wts, int fusion_arch, int score_flags, float neg_threshold,
                         int pairs, int L, float* feats, float* det_scores,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training-mode variants (SURVEY.md 8f row N4) of the two stages that contain BatchNorm: in .train() the reference's
 * BatchNorm2d layers of the VGG trunk (modules/vgg.py:67-80) and BatchNorm1d layers of w_det (modules/tracking_net.py:
 * 92-100) use the statistics of the current batch, and det_scores stay raw logits (tracking_net.py:152-162).  FP32 FFMA
 * engine; one frame-pair = one batch (the reference trains on one sample per step, tracking_model.py:50-66).
 *   mmmot_appearance_train_fwd: as mmmot_appearance_fwd; bn_stats [13][2][512] = per layer (batch mean | biased batch
 *     variance) per channel, for the caller's running-average update.
 *   mmmot_w_det_train_fwd: feats [3][512][L] of one pair -> det_scores [3][L] raw logits; bn_stats [2][2][512].
 *     drop_mask2 / drop_mask3 (NULL = none): DropBlock2D weights of the two deepest SkipPool heads
 *     (modules/appear_net.py:27-30,143-152; modules/dropblock.py:28-55), [n_img][H/16][W/16] and [n_img][H/32][W/32] =
 *     block_mask * numel / sum.  The caller draws the Bernoulli seeds (the reference draws them with torch's CPU generator,
 *     which a bit-matching run has to share) and max-pools them into blocks; the library applies them before the mean.
 *   mmmot_pointnet_train_fwd: as mmmot_pointnet_fwd on the FP32 engine, with the optional nn.Dropout mask of the head
 *     activation (modules/point_net.py:29-30): head_drop_mask [512][P], values {0, 1/(1-p)}, NULL = none.
 * Fusion and affinity have neither BatchNorm nor dropout: the eval entry points serve both modes
 * (mmmot_fusion_det_fwd's det_scores are simply overwritten by mmmot_w_det_train_fwd's).  Forward only: no gradients.
 */
size_t mmmot_appearance_train_workspace(int n_img, int H, int W);
int mmmot_appearance_train_fwd(const mmmot_weights* wts, const float* crops, int n_img, int H, int W, int L,
                               float* feats, float* bn_stats, const float* drop_mask2, const float* drop_mask3,
                               void* workspace, size_t workspace_bytes, void* stream);
size_t mmmot_pointnet_train_workspace(int pairs, int L, long p_total);
int mmmot_pointnet_train_fwd(const mmmot_weights* wts, const float* points, const int* det_split, const int* h_det_split,
                             int pairs, int L, const float* head_drop_mask, float* feats, void* workspace,
                             size_t workspace_bytes, void* stream);
size_t mmmot_w_det_train_workspace(int L);
int mmmot_w_det_train_fwd(const mmmot_weights* wts, int L, const float* feats, float* det_scores, float* bn_stats,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pairwise affinity + start/end indicator + softmax mode.
 * Replaces affinity_module.forward (modules/gcn.py:68-82), NewEndIndicator_v2.forward
 * (modules/new_end.py:62-82, modes 'avg' and 'max') and TrackingNet.associate (tracking_net.py:106-126).
 * The 3 x 512 x N x M pairwise tensor is generated tile by tile inside the first contraction's operand producers
 * (csrc/gemm_gen.cuh) and never stored; GroupNorm + ReLU between the MLP layers is applied by the next layer's
 * producers, so each layer output crosses HBM once as fp32.
 *   link  [pairs][3][N][M]
 *   new_s [pairs][3][M]   end_s [pairs][3][N]   (un-padded; the host pads with zeros as
 *                                                tracking_net.py:183-189 does)
 */
size_t mmmot_affinity_workspace(int pairs, int n, int m);
int mmmot_affinity_fwd(const mmmot_weights* wts, int affinity_op, int softmax_mode, int end_mode,
                       int pairs, int n, int m, const float* feats,
                       float* link, float* new_s, float* end_s,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Association integer programme for 2-frame pairs, solved exactly as a rectangular
 * assignment problem (SURVEY F9).  Replaces ortools_solve, reference solvers.py:9-138.
 *   det [pairs][L], link [pairs][N][M], new_s/end_s [pairs][L] (zero-padded like the reference's
 *   forward output); strides in floats between consecutive pairs are given explicitly so the
 *   solver can read the test_mode stack straight out of the forward outputs.
 *   outputs (fp32 0/1, same layout as solvers.py:116-131):
 *   a_det [pairs][L], a_link [pairs][N][M], a_new [pairs][L], a_end [pairs][L]
 *   match [pairs][N] int32: column matched to previous detection j, or -1.
 */
size_t mmmot_lp_workspace(int pairs, int n, int m);
int mmmot_lp_assign(const float* det, long det_stride, const float* link, long link_stride,
                    const float* new_s, long new_stride, const float* end_s, long end_stride,
                    int pairs, int n, int m,
                    float* a_det, float* a_link, float* a_new, float* a_end, int* match,
                    void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Association integer programme of samples of K >= 2 frames (reference solvers.py:9-138 for any len(det_split)),
 * solved exactly as a min-cost flow (csrc/flow_assign.cu).  All samples share the frame counts.
 *   counts [frames] (HOST): detections per frame, n_0 .. n_{K-1};  L = sum of counts
 *   det, new_s, end_s [samples][L] (zero-padded like the reference's forward output), links [samples][..]: one
 *   sample's link matrices back to back, [n0][n1], then [n1][n2], ...; strides in floats between samples.
 *   outputs (fp32 0/1, same layout as solvers.py:116-131):
 *   a_det, a_new, a_end [samples][L], a_links [samples][..] packed like links (dense between samples)
 *   match [samples][L - n_{K-1}] int32: each non-last-frame detection's successor index in the next frame, or -1.
 * MMMOT_E_ARG, before any CUDA call, for null pointers, samples <= 0, frames < 2 or a count <= 0; MMMOT_E_SHAPE for
 * frames > 64 or an L whose solver state does not fit one SM's shared memory (L > 4469).  Run time grows about as L^3:
 * one sample of dense random scores took 14 s at L = 2048 and 116 s at L = 4469 in a single launch on an H100 80GB HBM3
 * (700 W, 1980 MHz; profiles/flow_times_cap.json), against 2.6 s for 128 samples of L = 1024.
 */
size_t mmmot_flow_workspace(int samples, int frames, const int* counts);
int mmmot_flow_assign(const float* det, long det_stride, const float* links, long links_stride,
                      const float* new_s, long new_stride, const float* end_s, long end_stride,
                      int samples, int frames, const int* counts,
                      float* a_det, float* a_links, float* a_new, float* a_end, int* match,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Per-detection LiDAR cropping (SURVEY.md 8f row N1 — the step right before the hot path).
 * Replaces the host loop of reference point_cloud/preprocess.py:72-81 / box_np_ops.py:688-699 /
 * geometry.py:96-114.  planes[n_boxes][6][4]: inward plane equations (nx, ny, nz, d) of each rotated box,
 * prepared by the host exactly as the reference's numpy code does (mmmot_b200/lidar_crop.py), float64 when
 * planes_f64 != 0 (the reference's real pipeline: box_camera_to_lidar yields float64 boxes) else float32; a point is
 * inside iff x*nx + y*ny + z*nz + d < 0 for all six (evaluated in that precision, in the reference's operation
 * order, unfused).
 * Two steps because the output size is data dependent:
 *   mmmot_crop_count   -> split[n_boxes + 1] (device) CSR offsets; an empty box counts one (zero) point
 *   mmmot_crop_scatter -> out_points[split[n_boxes]][out_channels], scene order preserved inside a box
 * Both need the same workspace (mmmot_crop_workspace bytes) and the count step's contents are consumed by scatter.
 */
size_t mmmot_crop_workspace(int n_points, int n_boxes);
int mmmot_crop_count(const float* points, int n_points, int stride, const void* planes, int planes_f64, int n_boxes,
                     int* split, void* workspace, size_t workspace_bytes, void* stream);
int mmmot_crop_scatter(const float* points, int n_points, int stride, const void* planes, int planes_f64, int n_boxes,
                       const int* split, int out_channels, float* out_points, void* workspace,
                       size_t workspace_bytes, void* stream);

/*
 * Per-frame LiDAR preparation of many frames in one call (SURVEY.md 8f row N1): reference
 * point_cloud/preprocess.py:64-93 (read_and_prep_points minus the file read) — the camera field-of-view cull
 * (box_np_ops.py:629-640) followed by each detection's region, its 3-D box or the frustum of its 2-D image box
 * (box_np_ops.py:643-653).  Same predicate and kernels as mmmot_crop_*, always in float64.
 *   points [frame_offsets[n_frames]][stride] (device, stride 3 or 4): the frames' scans concatenated in frame order
 *   frame_offsets [n_frames + 1] (HOST): frame f's scan is points[frame_offsets[f] .. frame_offsets[f + 1]);
 *                 starts at 0, non-decreasing
 *   fov_planes [n_frames][6][4] (device, float64): each frame's field-of-view planes
 *   det_planes [n_dets][6][4] (device, float64): each detection's region
 *   det_frame  [n_dets] (HOST): frame of each detection; non-decreasing (detections grouped by frame, in frame order)
 * A point belongs to detection d when it is inside its frame's field of view AND inside d's region.
 *   mmmot_prep_count   -> split[n_dets + 1] (device) global CSR offsets; an empty detection counts one (zero) point
 *   mmmot_prep_scatter -> out_points[split[n_dets]][out_channels] (out_channels 3..4, <= stride), scan order inside
 *                         a detection, detections in order
 * Both take the same arguments and the same workspace (mmmot_prep_workspace bytes, max_frame_points = the largest
 * frame's point count); the count step's contents are consumed by scatter.  The launch count does not depend on
 * n_frames.  MMMOT_E_ARG on bad offsets or frame indices.
 */
size_t mmmot_prep_workspace(int max_frame_points, int n_frames, int n_dets);
int mmmot_prep_count(const float* points, const int* frame_offsets, int n_frames, int stride, const double* fov_planes,
                     const double* det_planes, const int* det_frame, int n_dets, int* split, void* workspace,
                     size_t workspace_bytes, void* stream);
int mmmot_prep_scatter(const float* points, const int* frame_offsets, int n_frames, int stride,
                       const double* fov_planes, const double* det_planes, const int* det_frame, int n_dets,
                       const int* split, int out_channels, float* out_points, void* workspace,
                       size_t workspace_bytes, void* stream);

/*
 * Per-detection image crop-and-resize (SURVEY.md 8f row N2 — the image-side step right before the hot path).
 * Replaces reference dataset/test_seq_dataset.py:212-218 (PIL crop + 224x224 BILINEAR resize per detection) and
 * utils/build_util.py:137-142 (ToTensor + Normalize): image uint8 [img_h][img_w][3] (device), boxes int32
 * [n_det][4] = (x1, y1, x2, y2) integer crop boxes (floor/ceil of the detection boxes, taken on the host like the
 * reference; may reach outside the image: PIL pads with 0), row_off int64 [n_det + 1] = prefix sum of the crop
 * heights (y2 - y1), total_rows = row_off[n_det], max_crop_h = largest crop height, mean_std = 6 host floats
 * (mean r,g,b then std r,g,b).  out fp32 [n_det][3][out_size][out_size], bit-identical to the reference's PIL +
 * torchvision result (Pillow 8-bit two-pass resampler reproduced in fixed point).  taps = the filter-tap stride:
 * max over boxes and axes of ceil(max(crop side / out_size, 1)) * 2 + 1, at most mmmot_crop_resize_max_taps().
 */
int mmmot_crop_resize_max_taps(void);
size_t mmmot_crop_resize_workspace(int n_det, long total_rows, int out_size, int taps);
int mmmot_crop_resize(const unsigned char* image, int img_h, int img_w, const int* boxes, const long long* row_off,
                      int n_det, long total_rows, int max_crop_h, int out_size, int taps, const float* mean_std,
                      float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Contraction engine selection: 0 = auto (wgmma tensor-core engine for large problems, FP32 FFMA
 * engine for tiny ones), 1 = force the FP32 FFMA engine, 2 = force the tensor-core engine.  Both engines
 * implement the same contraction; the switch exists for A/B parity tests and profiling. */
int mmmot_set_engine(int engine);

/* Accuracy / speed knob of the tensor-core conv engine.  The tensor core's fp32 accumulator rounds toward zero at
 * every K=16 step, so K chains longer than `chunks` x 32 are accumulated in several passes whose partial sums are
 * added in fp32 round-to-nearest.  0 = single pass (fastest), 36 (default) splits the K >= 2304 layers, 72 only the
 * K = 4608 layers. */
int mmmot_set_kseg(int chunks);

/* Profiling / A-B experiments (tools/stage_times.py, TC_DBG=...).  Results are WRONG with any of bits 0-3 set;
 * the other bits select an alternative implementation of the same arithmetic.  Default 0.
 *   bit 0 (1)    skip epilogue work          bit 1 (2)   skip weight loads
 *   bit 2 (4)    skip operand loads          bit 3 (8)   skip MMA issue
 *   bit 4 (16)   PointNet's layer-5 and head GroupNorm statistics by a statistics-only pass of the contraction itself
 *                instead of from the input's moments (mmmot_debug_pn_stats)
 *   bit 5 (32)   first VGG layer as the direct FP32 FFMA kernel instead of im2col + tensor cores
 *   bit 6 (64)   64-channel layers on the channel-major kernel instead of the pixel-major one
 *   bit 7 (128)  pixel-major epilogue with 16-byte stores instead of whole 32-byte sectors
 *   bit 8 (256)  pixel-major kernel without halo boxes (nine boxes per channel chunk)
 *   bit 9 (512)  no fused max-pool in the conv epilogues (separate max-pool kernel)
 *   bit 10 (1024) generated-operand engine (csrc/gemm_gen.cuh): producers without the software pipeline, every GEN
 *   bit 12 (4096) generated-operand engine: GEN_NORM producers with the software pipeline (prefetching variant)
 *   bit 13 (8192) PointNet layers 3, 4 through norm_split + the TMA-fed kernel instead of GEN_NORM producers
 *   bit 14 (16384) first VGG layer with a separate im2col pre-pass instead of in-kernel operand producers */
int mmmot_set_debug(int flags);

/* Test hook: one launch of the FP32 FFMA engine in any operand mode, with its GroupNorm partials (device pointers).
 * mode 0: x = X, mode 1: x = relu(X*sc[g][k] + sh[g][k]) (sc, sh [groups][K]).  Y[g*y_gs + co*y_ms + col] (or NULL) =
 * Wt^T x + bias (+ ReLU if relu), Wt [K][M] fp32, M a multiple of 64; x read at X[g*x_gs + k*x_ks + col].  Columns:
 * uniform tiling (tile_tab NULL) `groups` groups of S columns in 128-column tiles, or tile_tab int4 [num_tiles] {group,
 * first absolute column, length <= 128, 0} with x_gs = y_gs = 0.  part (or NULL): double2 [num_tiles][M] = (sum, sum of
 * squares) of each tile's columns.  mode 2-4 pairwise multiply / |minus| / minus: x[k][s] = f(F[g][k][i],
 * F[g][k][n + j]), s = i*m + j, F = X [groups][K][Lf], uniform tiling with S = n*m, Lf >= n + m, Y as mode 0; mode 5
 * 3x3 / pad 1 convolution: X = in[img][Cin][H][W], K = 9*Cin, x[k][s] = im2col with k = (ky*3 + kx)*Cin + ci and s =
 * (img, y, x), Y = out[img][M][H][W], uniform tiling with groups = 1, S = n_img*H*W, x_gs = y_gs = 0 (x_ks, y_ms
 * unused).  addend (or NULL): Y += addend[co*ld_add + seg[c]] before the ReLU, c the column (absolute for table
 * tiling, inside the group otherwise).  MMMOT_E_ARG, before any CUDA call, for any other combination. */
int mmmot_debug_simt_op(int mode, int M, int K, const float* Wt, const float* bias, int relu, const float* X, long x_gs,
                        long x_ks, const float* sc, const float* sh, int n, int m, int Lf, int H, int W, int Cin, int S,
                        int groups, const void* tile_tab, int num_tiles, const float* addend, const int* seg, int ld_add,
                        float* Y, long y_gs, long y_ms, void* part, void* stream);

/* Test hooks of the generated-operand tensor-core engine (csrc/gemm_gen.cuh), run through the same launch code as the
 * affinity, PointNet and fusion stages.  gen: 0-2 = pairwise multiply / |minus| / minus (MMMOT_AFF_*), 3 = GroupNorm +
 * ReLU of an fp32 source (GEN_NORM), 4 = an fp32 source as it is (GEN_COPY).
 * gen_prefetch: 1 if the launch takes the software-pipelined (prefetching) producers, else 0, under the current
 *   mmmot_set_debug state; computed on the host without any CUDA call.  m: detections of a pairwise launch.
 * gen_staged: 1 if that variant stages the pairwise sources in shared memory by TMA (GEN_PAIR_* at m == 128 without
 *   bit 10), else 0; computed on the host like gen_prefetch.
 * gen: Y[row][y_ms] (fp32 channels-last, first M channels written, or NULL) = op(x) W^T + bias (+ ReLU if relu), Wp =
 *   packed FP16 hi/lo tiles of W [M][K] (weights.py::pack_tc).  Columns (operand rows):
 *     uniform tiling (tile_tab NULL): `groups` groups of S columns, 256-column tiles; column s of group g reads source
 *       row g*x_gs + s (pairwise: s = i*m + j of the group's feature stack) and writes row g*y_gs + s;
 *     tile table (GEN_NORM / GEN_COPY only; x_gs, y_gs ignored): tile_tab int4 [num_tiles] {group, first absolute row,
 *       length <= 256, 0}.
 *   Source: pairwise src = feature stacks fcl [groups][Lf][K] with rows [0, n) objects, [n, n + m) detections, Lf = n + m;
 *   GEN_NORM / GEN_COPY src = fp32 rows of ld_src floats (multiple of 8, >= K; the first K are read), GEN_NORM
 *   x = relu(src*gsc[g][k] + gsh[g][k]) with gsc/gsh [groups][K], K <= 512.  part (or NULL): double2
 *   [num_tiles*2][M] = (sum, sum of squares) of each tile's column half (tile*2 + half).  prefetched (host, or NULL):
 *   the variant taken, as gen_prefetch. */
int mmmot_debug_gen_prefetch(int gen, int m);
int mmmot_debug_gen_staged(int gen, int m);
int mmmot_debug_gen(int gen, int M, int K, const void* Wp, float wp_scale, const float* bias, int relu, const float* src,
                    int ld_src, const float* gsc, const float* gsh, int n, int m, int Lf, int S, int groups, long x_gs,
                    long y_gs, const void* tile_tab, int num_tiles, float* Y, long y_ms, void* part, int* prefetched,
                    void* stream);

/* Test hook of PointNet's tensor-core trunk over ragged detections (csrc/pointnet.cu).  From the CSR offsets det_split
 * [pairs*L + 1] (device; h_det_split the same on the host) it builds, as mmmot_pointnet_fwd does: tiles int4 [n_tiles]
 * {pair, first point, length <= 256, 0}, cnt [pairs] points per pair, gstart [pairs + 1] first tile of each pair, seg
 * [P] detection of each point, ctab int4 [2*n_tiles] chunk descriptors ((first detection << 1) | chunk complete and
 * inside one detection, per 32-column chunk of each tile half).  *n_tiles (host, or NULL) = tile count;
 * MMMOT_E_WORKSPACE if it exceeds max_tiles.  If Wp is not NULL it then runs one matrix-mode contraction on those tables
 * as the trunk issues it: X = FP16 planes [2][P][K] (Xhi), Y [P][M] fp32 (or NULL), part [n_tiles*2][M] double2 (or
 * NULL), addend [det][ld_add] per-detection addend (or NULL), segsum (or NULL): [det][M] sums over each detection's
 * points of relu(y*sc[pair][co] + sh[pair][co]) in 2^-32 fixed point, accumulated (the caller zeroes it). */
int mmmot_debug_pn_contraction(const int* det_split, const int* h_det_split, int pairs, int L, long max_tiles, void* tiles,
                               int* cnt, int* gstart, int* seg, void* ctab, long* n_tiles, const void* Wp, float wp_scale,
                               const float* bias, int M, int K, const void* Xhi, float* Y, void* part, const float* addend,
                               int ld_add, unsigned long long* segsum, const float* sc, const float* sh, void* stream);

/* Test hook of the GroupNorm statistics of PointNet's two widest tensor-core layers (csrc/pointnet.cu), computed as
 * mmmot_pointnet_fwd computes them under the current mmmot_set_debug bits: y = x Wt + bias (+ addend[det]) over the
 * FP16 planes X [2][P][K] (Xhi) of the ragged detections det_split [pairs*L + 1] (device; h_det_split on the host);
 * K = 128 (layer 5, no addend) or 64 (head); M <= 1024, a multiple of 64; addend [det][M] or NULL.  Default: from the
 * input's moments, Wt [K][M] fp32 (Wp ignored); bit 4: a statistics-only contraction with the packed tiles Wp / wp_scale
 * (Wt ignored).  Then GroupNorm(M, M) per pair: sc / sh [pairs][M] (gamma, beta [M]).  Optional copies out: stats
 * [pairs][M][2] (sum y, sum y^2) fp64; default path only: mom [pairs][K*K + K] = (sum x x^T row-major, sum x) fp64 and,
 * for K = 64, detsum [det][64] = per-detection sums of x in 2^-32 fixed point.  workspace: the tensor-core PointNet
 * workspace, mmmot_pointnet_workspace(pairs, L, P) bytes with L >= 16 or under mmmot_set_engine(2) (otherwise that
 * function sizes the FP32 path's smaller layout and this hook returns MMMOT_E_WORKSPACE). */
int mmmot_debug_pn_stats(const int* det_split, const int* h_det_split, int pairs, int L, const void* Xhi, int K,
                         const float* Wt, const void* Wp, float wp_scale, const float* bias, int M, const float* addend,
                         const float* gamma, const float* beta, float* sc, float* sh, double* stats, double* mom,
                         unsigned long long* detsum, void* workspace, size_t workspace_bytes, void* stream);

/* Test hook of the TMA-fed tensor-core engine in matrix mode on uniform tiling: Y[rows][M] fp32 (channels-last) =
 * X W^T + bias, X two FP16 planes (hi, lo) [2][rows][K]. */
int mmmot_debug_linear_planar(const void* Wp, float wp_scale, const float* bias, const void* Xhi, float* Y,
                              int M, int K, long rows, void* stream);

/* Test hooks of the VGG trunk's convolutions, run through the same launch code as mmmot_appearance_fwd.
 * conv_plan: the launch plan of one 3x3 conv layer (n_img x H x W, C -> M channels), computed on the host without any
 *   CUDA call, under the current mmmot_set_debug / mmmot_set_kseg state.  want_pool: the caller takes a fused 2x2
 *   max-pool; use_kseg: the caller provides K-segment scratch.  plan[8] (host) = {pixel-major kernel, halo boxes,
 *   fused pool, box x, box y, box images, K segments, column tiles}.
 * conv_layer: 3x3 pad 1 + bias + ReLU on NHWC planes X[2][n][H][W][C] (x_plane apart) -> Y[2][n][H][W][M] (y_plane
 *   apart), or, when *did_pool (host) comes back 1, the 2x2 max-pooled map Y[2][n][H/2][W/2][M] (y_plane_pooled apart;
 *   y_plane_pooled > 0 and did_pool != NULL ask for the fused pool).  Wpx (or NULL): compact N = 64 tiles of a 64-output
 *   layer (weights.py::pack_px).  pool_sum (or NULL): [n][M] per-image sums of the pooled map in 2^-32 fixed point,
 *   accumulated (the caller zeroes it), filled only when the channel-major kernel fuses the pool.  kseg_scratch (or NULL):
 *   fp32 [column tiles * 256][M].  status: a status word (bit 0 = FP16 range).  plan (host, or NULL): as conv_plan.
 * vgg_conv0: the first VGG layer, fp32 NCHW crops [n][3][H][W] -> Y[2][n][H][W][64] (y_plane apart), bias + ReLU.
 *   wt [27][64] fp32 (k = (ky*3+kx)*3 + ci, debug bit 5), Wp / Wpx packed tiles with k = ci*9 + ky*3 + kx, cols
 *   [2][n*H*W][32] FP16 scratch of the im2col variant.  variant (host, or NULL) receives 0 = taps generated in the
 *   contraction kernel, 1 = im2col + matrix contraction, 2 = FP32 FFMA. */
int mmmot_debug_conv_plan(int n_img, int H, int W, int C, int M, int want_pool, int use_kseg, int* plan);
int mmmot_debug_conv_layer(const void* Wp, const void* Wpx, float wp_scale, const float* bias, const void* Xhi, long x_plane,
                           int n_img, int H, int W, int C, int M, void* Yhi, long y_plane, long y_plane_pooled,
                           int* did_pool, unsigned long long* pool_sum, float* kseg_scratch, int* status, int* plan,
                           void* stream);
int mmmot_debug_vgg_conv0(const float* crops, int n_img, int H, int W, const float* wt, const float* bias, const void* Wp,
                          float wp_scale, const void* Wpx, void* Yhi, long y_plane, void* cols, int* status, int* variant,
                          void* stream);

/* Test hooks of the kernels between the contractions.
 * stage_layout: where one run of a stage leaves its intermediates in the caller's workspace, computed on the host without
 *   any CUDA call from the same carve of the workspace the stage runs.  stage 0 = mmmot_affinity_fwd of shape
 *   (pairs, n, m), stage 1 = mmmot_fusion_det_fwd of shape (pairs, L = n; m ignored), stage 2 = mmmot_pointnet_fwd of
 *   shape (pairs, L = n, P = m points in all).  offsets (host, room for 32 entries whatever the stage) receives byte
 *   offsets from the start of the workspace, G = 3 pairs groups g = pair*3 + stack, NM = n*m, ldv = G*(n + m),
 *   "TC" the tensor-core path, "FP32" the FP32-engine path:
 *     stage 0, 31 offsets (entries [16].. are scratch the stage reuses; each holds what its last writer left):
 *       [0] y01   first layer [conv1.0 ; new/end conv0]: TC [g*NM + i*m + j][1024], FP32 [g][1024][NM]
 *       [1] y3    third affinity layer: TC [g*NM + s][128], FP32 [g][128][NM]
 *       [2] z     link logits [g][NM] (softmax_mode != NONE; with NONE they go straight to link)
 *       [3] fcl   TC only: the feature stacks channels-last [g][n + m][512]
 *       [4] sc0 [5] sh0   GroupNorm(1, 512) affine of new/end conv0 [g][512]
 *       [6] sc3 [7] sh3   GroupNorm affine of the third layer [g][128]
 *       [8] v     new/end row and column means (or maxima), column col = g*(n + m) + j (new) or + m + i (end):
 *                 TC [col][512], FP32 [512][ldv]
 *       [9] h2    second new/end MLP layer: TC [col][128], FP32 [128][ldv]
 *       [10] nsc2 [11] nsh2  its GroupNorm affine [2g + (0 new | 1 end)][128]
 *       [12] rmax [13] rsum  softmax over j per row [g][n];  [14] cmax [15] csum  over i per column [g][m]
 *       [16] y2   second affinity layer (before its GroupNorm): TC [g*NM + s][512], FP32 [g][512][NM]
 *       [17] sc1 [18] sh1   GroupNorm(512, 512) affine of the first affinity layer (channels 0..511 of y01) [g][512]
 *       [19] sc2 [20] sh2   GroupNorm(512, 512) affine of the second affinity layer [g][512]
 *       [21] h1   first new/end MLP layer (before its GroupNorm): TC [col][512], FP32 [512][ldv]
 *       [22] nsc1 [23] nsh1  its GroupNorm(1, 512) affine [2g + (0 new | 1 end)][512]
 *       [24] stats  fp64 (sum, sum of squares) [G][1024][2], written by layers 1, 2 and 3 in turn: at the end the
 *                 first [g][128][2] hold the third layer's
 *       [25] nstats fp64 [2G][512][2], written by both new/end layers: at the end the first [2g + e][128][2] hold
 *                 the second layer's
 *       [26] part  fp64 (sum, sum of squares) per column-tile partial, [tile*k + half][channel] with k = 2 on TC
 *                 (256-column tiles, two halves) and 1 on FP32 (128-column tiles), tiles g*tpg .. (g+1)*tpg - 1 of
 *                 group g; at the end the third layer's [G*tpg*k][128]
 *       [27] npart  the same for the new/end tiles of the table: at the end the second new/end layer's
 *                 [ne_tiles*k][128]
 *       [28] tiles  int4 {group 2g + e, first column col, length, 0}: per g, the new columns in tiles of 256 (TC) or
 *                 128 (FP32), then the end columns
 *       [29] cnt  int [2G] columns per new/end group (m new, n end)   [30] gstart  int [2G + 1] first tile per group
 *       The statistics of the first affinity layer, the second and the first new/end layer do not survive the stage.
 *     stage 1, 2 offsets:
 *       [0] f3    TC only: detection-major rows [(pair*L + l)*3 + stack][512]
 *       [1] h2    second w_det layer (after its ReLU): TC [(pair*L + l)*3 + stack][256], FP32 [g][256][L]
 *     stage 2, 27 offsets (carve order; ndet = pairs*L detections, d = pair*L + l; a buffer a path does not use has
 *     size 0 there; sc / sh / stats / part are reused layer after layer and end as conv2's):
 *       [0] xt    FP32: 3-channel points channel-major [3][P] (4-channel points are transposed into t1 instead, which
 *                 layer 3 then overwrites; xt stays untouched)
 *       [1] y1    FP32: layer 1 (C -> 64, before its GroupNorm) [64][P]
 *       [2] t0    TC: layer 4 [P][128];  FP32: layer 4 [128][P]
 *       [3] t1    TC: layer 3 [P][64];   FP32: layer 3 [64][P]
 *       [4] big   FP32: [1024][P], layer 5, whose first 512 rows the head (64 -> 512 + U addend, before its GroupNorm)
 *                 then overwrites
 *       [5] segsum  TC: 2^-32 fixed-point per-detection sums, u64; at the end the head's [ndet][512]
 *       [6] x1p   TC: relu(GN(layer 1)) as FP16 planes [2][P][64] (hi, lo)
 *       [7] xp    TC: relu(GN(layer 4)) as FP16 planes [2][P][128]
 *       [8] gmean per-detection mean of relu(GN(layer 5)): TC [ndet][1024], FP32 [1024][ndet]
 *       [9] u     FP32: U = Wh[:, 64:] gmean [512][ndet]     [10] ut  TC: U [ndet][512]
 *       [11] hmean  per-detection mean of relu(GN(head)): TC [ndet][512], FP32 [512][ndet]
 *       [12] o    conv2 (512 -> 512, before its GroupNorm): TC [ndet][512], FP32 [512][ndet]
 *       [13] sc1 [14] sh1   FP32: layer 1's GroupNorm affine [pairs][64]
 *       [15] sc [16] sh     [pairs][1024]; at the end the first [pairs][512] hold conv2's GroupNorm(16, 512) affine
 *       [17] stats          [pairs][1024][2] fp64; at the end the first [pairs][512][2] hold conv2's (sum, sum of squares)
 *       [18] mom  [19] part  moments / partials scratch   [20] gstart [pairs + 1]   [21] sstart (TC) [pairs + 1]
 *       [22] seg [P] detection of each point   [23] cnt [pairs] points per pair
 *       [24] tiles int4 {pair, first point, length, 0} (256-point tiles on TC, 128 on FP32)   [25] ctab (TC) int4
 *       [26] end  = mmmot_pointnet_workspace(pairs, L, P)
 *   *tensor_cores (host, or NULL) = 1 if that stage takes the tensor-core path under the current mmmot_set_engine.
 * skip_heads: the four SkipPool heads of mmmot_appearance_fwd on pooled vectors pooledS [n_img][C_S] (C = 128, 256, 512,
 *   512) chosen by the caller -> feats[pair][0][S*128 + t][l] for image pair*L + l; a NULL pooledS skips head S. */
int mmmot_debug_stage_layout(int stage, int pairs, int n, int m, size_t* offsets, int* tensor_cores);
int mmmot_debug_skip_heads(const mmmot_weights* wts, const float* pooled0, const float* pooled1, const float* pooled2,
                           const float* pooled3, int n_img, int L, float* feats, void* stream);

/* Per-launch timing of the hot kernels with CUDA events on the launching stream; used by bench.py's roofline
 * figures.  Every timed launch carries a tag = (stage, layer) — mmmot_timing_tag_count() tags, named by
 * mmmot_timing_tag_name() — and its ALGORITHMIC work (FLOPs; compulsory HBM bytes of that launch).
 * collect_tags() fills arrays of tag_count entries (any may be NULL) with the summed duration (ms), FLOPs, bytes and
 * launch count per tag since the last collect; collect() returns the totals over the 3x3-conv contractions of the
 * VGG trunk (layers 1..12, FLOPs = 2*Cout*9Cin*pixels), the dominant kernels. */
int mmmot_timing_enable(int on);
int mmmot_timing_tag_count(void);
const char* mmmot_timing_tag_name(int tag);
int mmmot_timing_collect_tags(double* ms, double* flop, double* bytes, long* launches);
int mmmot_timing_collect(double* total_ms, double* total_flop, long* launches);

/* counts kernel launches made through this library since process start (bench.py gpu_launches) */
unsigned long long mmmot_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* MMMOT_B200_H */
