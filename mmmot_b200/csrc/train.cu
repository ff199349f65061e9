// Training-mode w_det (SURVEY.md 8f row N4).  In .train() the reference's BatchNorm1d layers of w_det
// (modules/tracking_net.py:92-100) normalise with the statistics of the CURRENT batch (biased variance) and the
// detection scores stay raw logits (tracking_net.py:152-162).  The VGG trunk's training mode lives with its eval mode
// in appearance.cu; the rest of the forward (GroupNorm layers, PointNet, fusion, affinity) is the same in both modes.
// This runs on the FP32 FFMA engine (gemm_simt.cuh): contraction with per-tile (sum, sumsq) partials -> fixed-order
// reduction -> per-channel affine.  The batch statistics are returned so that the host can update the module's
// running averages like torch does.
#include "gemm_simt.cuh"
#include "norm_ops.cuh"

namespace {

// det_scores[g][l] = w3 . relu(h2[g][:, l]*sc + sh) + b3   (raw logits: tracking_net.py:152, training branch)
__global__ void det_logit_kernel(const float* __restrict__ h2, const float* __restrict__ sc, const float* __restrict__ sh,
                                 const float* __restrict__ w3, const float* __restrict__ b3, int G, int L,
                                 float* __restrict__ out) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= G * L) return;
  int g = idx / L, l = idx - g * L;
  const float* col = h2 + (long)g * 256 * L + l;
  float a = b3[0];
  for (int c = 0; c < 256; c++) a = fmaf(w3[c], fmaxf(fmaf(col[(long)c * L], sc[c], sh[c]), 0.f), a);
  out[idx] = a;
}

}  // namespace

// w_det in training mode on the three stacks of ONE frame-pair: conv -> BatchNorm1d(batch statistics over the 3 x L
// values of a channel) -> ReLU, twice, then the last conv; raw logits out (no sigmoid, no threshold).
// bn_stats: [2][2][512] = (layer, mean | biased var, channel)
extern "C" size_t mmmot_w_det_train_workspace(int L) {
  MmArena a(nullptr, 0);
  a.take<float>(3 * 512 * (size_t)L); a.take<float>(3 * 256 * (size_t)L);
  a.take<float>(3 * 512); a.take<float>(3 * 512);
  a.take<double>(512 * 2); a.take<double2>((size_t)3 * mm_cdiv(L, 128) * 512);
  return a.off;
}

extern "C" int mmmot_w_det_train_fwd(const mmmot_weights* wts, int L, const float* feats, float* det_scores, float* bn_stats,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  if (!wts || !feats || !det_scores || !bn_stats || !workspace || L <= 0) return MMMOT_E_ARG;
  if (!wts->w[MMMOT_W_WD_RAW0]) return MMMOT_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  MmArena ar(workspace, workspace_bytes);
  float* h1 = ar.take<float>(3 * 512 * (size_t)L);
  float* h2 = ar.take<float>(3 * 256 * (size_t)L);
  float* sc = ar.take<float>(3 * 512);
  float* sh = ar.take<float>(3 * 512);
  double* stats = ar.take<double>(512 * 2);
  double2* part = ar.take<double2>((size_t)3 * mm_cdiv(L, 128) * 512);
  if (!ar.ok()) return MMMOT_E_WORKSPACE;
  const float* const* R = &wts->w[MMMOT_W_WD_RAW0];   // w1t b1 bn1w bn1b w2t b2 bn2w bn2b
  const int tpg = mm_cdiv(L, 128), G = 3;
  GemmP p = gemm_defaults();
  p.Wt = R[0]; p.bias = R[1]; p.ldw = 512; p.M = 512; p.K = 512;
  p.S = L; p.tiles_per_group = tpg; p.num_tiles = tpg * G;
  p.X = feats; p.x_gs = 512L * L; p.x_ks = L;
  p.Y = h1; p.y_gs = 512L * L; p.y_ms = L;
  p.part = part;
  MM_TRY(gemm_simt_launch<XM_DIRECT>(p, st));
  MM_TRY(stats_reduce(part, 512, 1, tpg * G, nullptr, stats, st));            // one BatchNorm domain: all 3 stacks
  MM_TRY(gn_finalize(stats, R[2], R[3], nullptr, 3 * L, 1, 512, 1, sc, sh, st));
  bn_export_kernel<<<4, 128, 0, st>>>(stats, 512, 3.0 * L, bn_stats);
  MM_LAUNCH_CHECK();
  for (int g = 1; g < G; g++) {   // the operand generator indexes the affine per group
    MM_CUDA(cudaMemcpyAsync(sc + g * 512, sc, 512 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    MM_CUDA(cudaMemcpyAsync(sh + g * 512, sh, 512 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  p.Wt = R[4]; p.bias = R[5]; p.ldw = 256; p.M = 256;
  p.X = h1; p.sc = sc; p.sh = sh;
  p.Y = h2; p.y_gs = 256L * L;
  MM_TRY(gemm_simt_launch<XM_NORM_RELU>(p, st));
  MM_TRY(stats_reduce(part, 256, 1, tpg * G, nullptr, stats, st));
  MM_TRY(gn_finalize(stats, R[6], R[7], nullptr, 3 * L, 1, 256, 1, sc, sh, st));
  bn_export_kernel<<<2, 128, 0, st>>>(stats, 256, 3.0 * L, bn_stats + 1024);
  MM_LAUNCH_CHECK();
  det_logit_kernel<<<mm_cdiv(G * L, 128), 128, 0, st>>>(h2, sc, sh, wts->w[MMMOT_W_WD_W3], wts->w[MMMOT_W_WD_B3], G, L,
                                                       det_scores);
  MM_LAUNCH_CHECK();
  return 0;
}
