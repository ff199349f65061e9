// Appearance branch: VGG16-BN trunk + 4 SkipPool heads.
// Replaces reference modules/appear_net.py:166-190 (vgg_forward + SkipPool.forward :27-32).
// Eval mode (mmmot_appearance_fwd) folds BatchNorm into the convolutions.  Training mode (mmmot_appearance_train_fwd,
// SURVEY.md 8f row N4) runs the FP32 trunk with the unfolded weights and normalises every conv with the statistics of
// the current batch (modules/vgg.py:67-80 under .train()), which it returns for the host's running-average update.
#include <cuda_fp16.h>

#include "gemm_tma.cuh"
#include "norm_ops.cuh"

namespace {

// VGG16 "D" (reference modules/vgg.py:87-90): cout per conv, and whether a 2x2 max-pool follows.
const int kVggCout[13] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
const int kVggCin[13] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
const bool kPoolAfter[13] = {false, true, false, true, false, false, true, false, false, true, false, false, true};
// skip map s is the output of the pool after conv 3, 6, 9, 12 (reference appear_net.py:139-152:
// the first pool does not close a stage)
const int kSkipAfter[13] = {-1, -1, -1, 0, -1, -1, 1, -1, -1, 2, -1, -1, 3};
const int kSkipC[4] = {128, 256, 512, 512};

// 2x2 / stride 2 max-pool, NCHW.  One thread per output pixel pair-row; float2 loads.
__global__ void maxpool2_kernel(const float* __restrict__ in, float* __restrict__ out, long n_out,
                                int Ho, int Wo) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_out) return;
  int xo = (int)(idx % Wo);
  long t = idx / Wo;
  int yo = (int)(t % Ho);
  long plane = t / Ho;
  const float* src = in + (plane * (2 * Ho) + 2 * yo) * (long)(2 * Wo) + 2 * xo;
  float2 a = *reinterpret_cast<const float2*>(src);
  float2 b = *reinterpret_cast<const float2*>(src + 2 * Wo);
  out[idx] = fmaxf(fmaxf(a.x, a.y), fmaxf(b.x, b.y));
}

// Global average pool of every (img, channel) plane: one warp per plane.
// mask (optional, training): DropBlock weights [img][hw] = block_mask * numel / sum (modules/dropblock.py:49-53),
// applied before the SkipPool head's average pool (modules/appear_net.py:27-30); C = channels per image
__global__ void plane_mean_kernel(const float* __restrict__ in, float* __restrict__ out, long planes, int hw,
                                  const float* __restrict__ mask, int C) {
  long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (w >= planes) return;
  const float* src = in + w * hw;
  const float* mk = mask ? mask + (w / C) * hw : nullptr;
  float s = 0.f;
  for (int i = lane; i < hw; i += 32) s += mk ? src[i] * mk[i] : src[i];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[w] = s / (float)hw;
}

// training-mode BatchNorm + ReLU: y[img][c][hw] = relu(y*sc[c] + sh[c]) in place
__global__ void bn_relu_kernel(float* __restrict__ y, const float* __restrict__ sc, const float* __restrict__ sh, int C,
                               int hw, long n) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int c = (int)((idx / hw) % C);
  y[idx] = fmaxf(fmaf(y[idx], sc[c], sh[c]), 0.f);
}

// ---- FP16 hi/lo planes, NHWC: activations of the tensor-core trunk ([2][n][H][W][C]) ----
// 2x2 / stride 2 max-pool, 8 channels per thread (128-bit loads).  The max IS one of the four inputs, so its
// (hi, lo) pair is copied, not re-split.
__global__ void maxpool2_planar_kernel(const __half* __restrict__ in, __half* __restrict__ out, long n_out8,
                                       int Ho, int Wo, int C, long plane_in, long plane_out) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_out8) return;
  const int c8n = C >> 3;
  const int c = (int)(idx % c8n) * 8;
  long t = idx / c8n;
  const int xo = (int)(t % Wo);
  t /= Wo;
  const int yo = (int)(t % Ho);
  const long img = t / Ho;
  const long rs = (long)2 * Wo * C;
  const __half* src = in + ((img * 2 * Ho + 2 * yo) * 2 * Wo + 2 * xo) * (long)C + c;
  const long offs[4] = {0, (long)C, rs, rs + C};
  uint4 bh, bl;
  float best[8];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint4 h = *reinterpret_cast<const uint4*>(src + offs[k]);
    const uint4 l = *reinterpret_cast<const uint4*>(src + offs[k] + plane_in);
    const __half* hh = reinterpret_cast<const __half*>(&h);
    const __half* ll = reinterpret_cast<const __half*>(&l);
    __half* oh = reinterpret_cast<__half*>(&bh);
    __half* ol = reinterpret_cast<__half*>(&bl);
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const float f = __half2float(hh[e]) + __half2float(ll[e]);
      if (k == 0 || f > best[e]) { best[e] = f; oh[e] = hh[e]; ol[e] = ll[e]; }
    }
  }
  __half* dst = out + ((img * Ho + yo) * (long)Wo + xo) * C + c;
  *reinterpret_cast<uint4*>(dst) = bh;
  *reinterpret_cast<uint4*>(dst + plane_out) = bl;
}

// global average of every (img, channel) over the hw pixels of a planar NHWC map -> pooled[img][C] fp32
__global__ void plane_mean_planar_kernel(const __half* __restrict__ in, float* __restrict__ out, long n_img,
                                         int hw, int C, long plane) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_img * C) return;
  const int c = (int)(idx % C);
  const long img = idx / C;
  const __half* src = in + img * hw * (long)C + c;
  float s = 0.f;
  for (int i = 0; i < hw; i++) s += __half2float(src[(long)i * C]) + __half2float(src[(long)i * C + plane]);
  out[idx] = s / (float)hw;
}

// pooled[img][c] = sum[img][c] * 2^-32 / hw : the fixed-point per-image sums of the fused pool epilogue -> SkipPool's average
__global__ void pool_sum_mean_kernel(const unsigned long long* __restrict__ sum, float* __restrict__ out, long n, float inv_hw) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n) out[idx] = (float)((double)sum[idx] * (1.0 / 4294967296.0) * (double)inv_hw);
}

// First VGG layer (3 -> 64, K = 27) of the tensor-core trunk: too thin for the MMA path (memory-bound: 1 MB of
// output per crop), so a direct FP32 FFMA kernel writes the FP16 hi/lo NHWC planes the next layer's TMA loads
// read.  Each thread: 2 horizontally adjacent pixels x 16 channels (weights from smem as 128-bit loads);
// CTA = 64 pixel pairs x 4 channel groups.  wt: [(ky*3+kx)*3 + ci][64] (BN folded), ReLU fused.  W % 2 == 0.
__global__ void __launch_bounds__(256, 4) conv0_packed_kernel(const float* __restrict__ in, const float* __restrict__ wt,
                                                              const float* __restrict__ bias, long n_pairs, int H, int W,
                                                              __half* __restrict__ out, long plane, int* status) {
  __shared__ __align__(16) float ws[27 * 64];
  __shared__ float bs[64];
  for (int i = threadIdx.x; i < 27 * 64; i += 256) ws[i] = wt[i];
  if (threadIdx.x < 64) bs[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  // warp-uniform channel group (weight reads are smem broadcasts); lanes = 32 consecutive pixel pairs
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long pr = (long)blockIdx.x * 64 + (warp >> 2) * 32 + lane;
  const int cg = (warp & 3) * 16;
  if (pr >= n_pairs) return;
  const int wp = W >> 1, hw = H * W;
  const long row = pr / wp;                // (img, y)
  const int x0 = (int)(pr - row * wp) * 2;
  const long img = row / H;
  const int y = (int)(row - img * H);
  const float* src = in + img * 3 * hw;
  float acc[2][16];
#pragma unroll
  for (int p = 0; p < 2; p++)
#pragma unroll
    for (int c = 0; c < 16; c++) acc[p][c] = bs[cg + c];
#pragma unroll
  for (int ci = 0; ci < 3; ci++) {
#pragma unroll
    for (int ky = 0; ky < 3; ky++) {
      const int yy = y + ky - 1;
      const bool oky = yy >= 0 && yy < H;
      const float* rowp = src + (long)ci * hw + (long)yy * W + x0;
      float v[4];
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const int xx = x0 + t - 1;
        v[t] = (oky && xx >= 0 && xx < W) ? __ldg(rowp + t - 1) : 0.f;
      }
#pragma unroll
      for (int kx = 0; kx < 3; kx++) {
        const float4* wr = reinterpret_cast<const float4*>(ws + ((ky * 3 + kx) * 3 + ci) * 64 + cg);
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const float4 t4 = wr[q];
#pragma unroll
          for (int p = 0; p < 2; p++) {
            acc[p][4 * q] = fmaf(v[p + kx], t4.x, acc[p][4 * q]);
            acc[p][4 * q + 1] = fmaf(v[p + kx], t4.y, acc[p][4 * q + 1]);
            acc[p][4 * q + 2] = fmaf(v[p + kx], t4.z, acc[p][4 * q + 2]);
            acc[p][4 * q + 3] = fmaf(v[p + kx], t4.w, acc[p][4 * q + 3]);
          }
        }
      }
    }
  }
  const long pix0 = row * W + x0;
#pragma unroll
  for (int p = 0; p < 2; p++) {
    __half h[16], l[16];
#pragma unroll
    for (int c = 0; c < 16; c++) {
      tma::split_f16(fmaxf(acc[p][c], 0.f), h[c], l[c]);
      mm_range_flag(status, acc[p][c]);
    }
    __half* dst = out + (pix0 + p) * 64 + cg;
    reinterpret_cast<uint4*>(dst)[0] = reinterpret_cast<uint4*>(h)[0];
    reinterpret_cast<uint4*>(dst)[1] = reinterpret_cast<uint4*>(h)[1];
    reinterpret_cast<uint4*>(dst + plane)[0] = reinterpret_cast<uint4*>(l)[0];
    reinterpret_cast<uint4*>(dst + plane)[1] = reinterpret_cast<uint4*>(l)[1];
  }
}

// First VGG layer on the tensor cores: the 3-channel fp32 NCHW crop is expanded to the 27 (+5 zero) taps of every
// pixel, k = ci*9 + ky*3 + kx, as FP16 hi/lo planes [2][pixels][32]; the layer is then a K=32 contraction on the TMA
// engine whose epilogue writes the NHWC planes conv 1 reads.  One thread per pixel, 64 B per plane.
__global__ void __launch_bounds__(256) im2col27_kernel(const float* __restrict__ in, long n_pix, int H, int W,
                                                       __half* __restrict__ out, long plane, int* status) {
  const long pix = (long)blockIdx.x * 256 + threadIdx.x;
  if (pix >= n_pix) return;
  const int hw = H * W;
  const long img = pix / hw;
  const int r = (int)(pix - img * hw);
  const int y = r / W, x = r - y * W;
  const float* src = in + img * 3 * hw;
  __align__(16) __half h[32], l[32];
  float amax = 0.f;
#pragma unroll
  for (int ci = 0; ci < 3; ci++)
#pragma unroll
    for (int ky = 0; ky < 3; ky++)
#pragma unroll
      for (int kx = 0; kx < 3; kx++) {
        const int yy = y + ky - 1, xx = x + kx - 1;
        const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(src + (long)ci * hw + yy * W + xx) : 0.f;
        tma::split_f16(v, h[ci * 9 + ky * 3 + kx], l[ci * 9 + ky * 3 + kx]);
        amax = fmaxf(amax, fabsf(v));
      }
  mm_range_flag(status, amax);
#pragma unroll
  for (int k = 27; k < 32; k++) { h[k] = __ushort_as_half(0); l[k] = __ushort_as_half(0); }
  uint4* dh = reinterpret_cast<uint4*>(out + pix * 32);
  uint4* dl = reinterpret_cast<uint4*>(out + plane + pix * 32);
#pragma unroll
  for (int q = 0; q < 4; q++) {
    dh[q] = reinterpret_cast<const uint4*>(h)[q];
    dl[q] = reinterpret_cast<const uint4*>(l)[q];
  }
}

__device__ __forceinline__ float block_sum_128(float v, float* red) {
  // 128 threads (4 warps)
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return red[0] + red[1] + red[2] + red[3];
}

// One CTA (128 threads) per image per head: GN(1,C) -> 1x1 conv -> GN(1,mid) -> ReLU -> 1x1 conv
// -> GN(1,128) -> ReLU.  GN(1,C) on a C x 1 x 1 input is a per-detection layer norm over channels.
__global__ void __launch_bounds__(128) skip_head_kernel(
    const float* __restrict__ pooled,  // [n_img][C]
    const float* __restrict__ g0w, const float* __restrict__ g0b, const float* __restrict__ w1t,
    const float* __restrict__ b1, const float* __restrict__ g1w, const float* __restrict__ g1b,
    const float* __restrict__ w2t, const float* __restrict__ b2, const float* __restrict__ g2w,
    const float* __restrict__ g2b, int C, int mid, int L, int head, float* __restrict__ feats) {
  __shared__ float v[512];
  __shared__ float h[128];
  __shared__ float red[4];
  const int img = blockIdx.x, t = threadIdx.x;
  const float eps = 1e-5f;
  float s = 0.f;
  for (int c = t; c < C; c += 128) { float x = pooled[(long)img * C + c]; v[c] = x; s += x; }
  float mean = block_sum_128(s, red) / C;
  s = 0.f;
  for (int c = t; c < C; c += 128) { float d = v[c] - mean; s += d * d; }
  float rstd = rsqrtf(block_sum_128(s, red) / C + eps);
  for (int c = t; c < C; c += 128) v[c] = (v[c] - mean) * rstd * g0w[c] + g0b[c];
  __syncthreads();
  // conv C -> mid
  float a = 0.f;
  if (t < mid) {
    a = b1[t];
    for (int c = 0; c < C; c++) a = fmaf(w1t[(long)c * mid + t], v[c], a);
  }
  mean = block_sum_128(t < mid ? a : 0.f, red) / mid;
  float d = t < mid ? a - mean : 0.f;
  rstd = rsqrtf(block_sum_128(d * d, red) / mid + eps);
  if (t < mid) h[t] = fmaxf(d * rstd * g1w[t] + g1b[t], 0.f);
  __syncthreads();
  // conv mid -> 128
  a = b2[t];
  for (int c = 0; c < mid; c++) a = fmaf(w2t[c * 128 + t], h[c], a);
  mean = block_sum_128(a, red) / 128.f;
  d = a - mean;
  rstd = rsqrtf(block_sum_128(d * d, red) / 128.f + eps);
  float o = fmaxf(d * rstd * g2w[t] + g2b[t], 0.f);
  const int pair = img / L, l = img - pair * L;
  feats[(((long)pair * 3 + 0) * 512 + head * 128 + t) * L + l] = o;
}

// First VGG layer (3 -> 64, bias + ReLU): fp32 NCHW crops -> FP16 hi/lo NHWC planes Y[2][n][H][W][64], y_plane apart.
//   FFMA (debug bit 32): conv0_packed_kernel on wt [(ky*3+kx)*3 + ci][64]
//   GEN27: taps generated by the contraction kernel's producers (needs the compact Wpx, H*W % 256 == 0, W <= 512)
//   otherwise (or debug bit 16384): im2col27_kernel into cols [2][n*H*W][32] + the matrix contraction on Wp (and Wpx)
// variant (optional) receives 0 = GEN27, 1 = im2col + matrix, 2 = FFMA.
static int vgg_conv0_launch(const float* crops, int n_img, int H, int W, const float* wt, const float* bias, const uint4* Wp,
                            float wp_scale, const uint4* Wpx, __half* Y, long y_plane, __half* cols, int* status,
                            int* variant, cudaStream_t st) {
  const long n_pix = (long)n_img * H * W;
  const int dbg = mm_debug_flags();
  if (dbg & 32) {   // A/B: direct FP32 FFMA first layer
    if (variant) *variant = 2;
    if (!wt || (W & 1)) return MMMOT_E_ARG;
    conv0_packed_kernel<<<mm_cdiv(n_pix / 2, 64), 256, 0, st>>>(crops, wt, bias, n_pix / 2, H, W, Y, y_plane, status);
    MM_LAUNCH_CHECK();
  } else if (Wpx && !(dbg & 16384) && ((long)H * W) % 256 == 0 && W <= 512) {
    // taps generated inside the contraction kernel (no im2col matrix in HBM)
    if (variant) *variant = 0;
    MM_TRY(gemm_tma_px_launch_gen27(crops, n_img, H, W, Wpx, wp_scale, bias, Y, y_plane, status, st));
  } else {
    if (variant) *variant = 1;
    if (!Wp || !cols) return MMMOT_E_ARG;
    if (n_pix >= (1L << 31)) return MMMOT_E_SHAPE;
    im2col27_kernel<<<mm_cdiv(n_pix, 256), 256, 0, st>>>(crops, n_pix, H, W, cols, n_pix * 32, status);
    MM_LAUNCH_CHECK();
    GemmP p = gemm_defaults();
    p.bias = bias; p.M = 64; p.K = 32; p.relu = 1;
    p.S = (int)n_pix; p.tiles_per_group = mm_cdiv(n_pix, tc::BN); p.num_tiles = p.tiles_per_group;
    p.Y = reinterpret_cast<float*>(Y); p.y_ms = 64;
    MM_TRY(gemm_tma_launch_mat(p, Wp, wp_scale, cols, n_pix * 32, n_pix, 32, tma::OUT_PLANAR, y_plane, st, nullptr, status,
                               nullptr, Wpx));
  }
  return 0;
}

// What the FP32 trunk needs in training mode: the BatchNorm scratch, where the batch statistics go, and the DropBlock
// weights of the two deepest skip maps
struct VggTrain {
  double2* part;              // per-tile (sum, sumsq) partials of one conv
  double* stats;              // their fixed-order per-channel reduction
  float *sc, *sh;             // per-channel affine
  float* bn_stats;            // [13][2][512]: batch mean | biased batch variance of every conv
  const float* drop_mask[2];  // DropBlock weights [img][hw] of skip maps 2 and 3 (optional)
};

// The appearance stage's workspace: the two activation buffers and the pooled skip maps, then the tensor-core trunk's
// scratch (eval) or the BatchNorm scratch (training)
struct AppWs {
  float* buf[2];
  float* pooled[4];
  float* kseg_scratch;            // K-segment partial sums, tile order (largest: 256 ch at H/4 x W/4)
  unsigned long long* pool_sum;   // per-image sums of a pooled skip map (fused pool epilogue)
  VggTrain tr;
};
AppWs carve_appearance(MmArena& a, int n_img, int H, int W, bool train) {
  AppWs w = {};
  const size_t act = (size_t)n_img * 64 * H * W;
  w.buf[0] = a.take<float>(act);
  w.buf[1] = a.take<float>(act);
  for (int s = 0; s < 4; s++) w.pooled[s] = a.take<float>((size_t)n_img * kSkipC[s]);
  if (train) {
    w.tr.sc = a.take<float>(512);
    w.tr.sh = a.take<float>(512);
    w.tr.stats = a.take<double>(512 * 2);
    w.tr.part = a.take<double2>((size_t)mm_cdiv((long)n_img * H * W, 128) * 64);   // tiles x channels: largest at conv 0/1
  } else {
    w.kseg_scratch = a.take<float>((size_t)(n_img + 16) * H * W * 16);
    w.pool_sum = a.take<unsigned long long>((size_t)n_img * 512);
  }
  return w;
}

// The VGG trunk on the FP32 FFMA engine: fp32 NCHW activations in buf[0] / buf[1], the skip maps' global averages into
// pooled[s].  Eval (tr == nullptr): BatchNorm folded into the weights, ReLU in the conv's epilogue, every conv timed.
// Training: the conv with the unfolded weights, then BatchNorm2d on the statistics over (batch, H, W) (biased variance,
// eps 1e-5) and ReLU in place; the DropBlock weights scale skip maps 2 and 3 before their average.
int vgg_fp32_trunk(const mmmot_weights* wts, const float* crops, int n_img, int H, int W, float* const* buf,
                   float* const* pooled, const VggTrain* tr, cudaStream_t st) {
  const float* cur = crops;
  int which = 0, h = H, w = W;
  const bool timed = !tr && mm_timing_on();
  for (int i = 0; i < 13; i++) {
    GemmP p = gemm_defaults();
    p.Wt = wts->w[(tr ? MMMOT_W_VGG_RAWW0 : MMMOT_W_VGG_WT0) + i];
    p.bias = wts->w[(tr ? MMMOT_W_VGG_RAWB0 : MMMOT_W_VGG_B0) + i];
    p.ldw = kVggCout[i];
    p.M = kVggCout[i];
    p.K = 9 * kVggCin[i];
    p.Cin = kVggCin[i];
    p.H = h; p.W = w;
    p.S = n_img * h * w;
    p.X = cur;
    p.Y = buf[which];
    p.relu = !tr;
    p.part = tr ? tr->part : nullptr;
    p.tiles_per_group = mm_cdiv(p.S, 128);
    p.num_tiles = p.tiles_per_group;
    if (timed) mm_timing_begin(st, MM_T_VGG0 + i, 2.0 * p.M * (double)p.K * (double)p.S, 4.0 * (double)p.S * (p.Cin + p.M));
    MM_TRY(gemm_simt_launch<XM_CONV3>(p, st));
    if (timed) mm_timing_end(st);
    if (tr) {
      MM_TRY(stats_reduce(tr->part, p.M, 1, p.num_tiles, nullptr, tr->stats, st));
      MM_TRY(gn_finalize(tr->stats, wts->w[MMMOT_W_VGG_BNW0 + i], wts->w[MMMOT_W_VGG_BNB0 + i], nullptr, p.S, 1, p.M, 1,
                         tr->sc, tr->sh, st));
      bn_export_kernel<<<mm_cdiv(p.M, 128), 128, 0, st>>>(tr->stats, p.M, (double)p.S, tr->bn_stats + (long)i * 1024);
      MM_LAUNCH_CHECK();
      const long n = (long)p.S * p.M;
      bn_relu_kernel<<<mm_cdiv(n, 256), 256, 0, st>>>(buf[which], tr->sc, tr->sh, p.M, h * w, n);
      MM_LAUNCH_CHECK();
    }
    cur = buf[which]; which ^= 1;
    if (kPoolAfter[i]) {
      h /= 2; w /= 2;
      long n_out = (long)n_img * kVggCout[i] * h * w;
      maxpool2_kernel<<<mm_cdiv(n_out, 256), 256, 0, st>>>(cur, buf[which], n_out, h, w);
      MM_LAUNCH_CHECK();
      cur = buf[which]; which ^= 1;
      int s = kSkipAfter[i];
      if (s >= 0) {
        long planes = (long)n_img * kSkipC[s];
        const float* mask = tr && s >= 2 ? tr->drop_mask[s - 2] : nullptr;
        plane_mean_kernel<<<mm_cdiv(planes * 32, 256), 256, 0, st>>>(cur, pooled[s], planes, h * w, mask, kSkipC[s]);
        MM_LAUNCH_CHECK();
      }
    }
  }
  return 0;
}

}  // namespace

// Test hook: the first VGG layer exactly as mmmot_appearance_fwd runs it (vgg_conv0_launch).
extern "C" int mmmot_debug_vgg_conv0(const float* crops, int n_img, int H, int W, const float* wt, const float* bias,
                                     const void* Wp, float wp_scale, const void* Wpx, void* Yhi, long y_plane, void* cols,
                                     int* status, int* variant, void* stream) {
  if (!crops || !bias || !Yhi || n_img <= 0 || H <= 0 || W <= 0) return MMMOT_E_ARG;
  return vgg_conv0_launch(crops, n_img, H, W, wt, bias, (const uint4*)Wp, wp_scale, (const uint4*)Wpx, (__half*)Yhi, y_plane,
                          (__half*)cols, status, variant, (cudaStream_t)stream);
}

int mm_launch_skip_heads(const mmmot_weights* wts, float* const* pooled, int n_img, int L, float* feats, cudaStream_t st);

extern "C" size_t mmmot_appearance_workspace(int n_img, int H, int W) {
  MmArena a(nullptr, 0);
  carve_appearance(a, n_img, H, W, false);
  return a.off;
}

extern "C" size_t mmmot_appearance_train_workspace(int n_img, int H, int W) {
  MmArena a(nullptr, 0);
  carve_appearance(a, n_img, H, W, true);
  return a.off;
}

extern "C" int mmmot_appearance_fwd(const mmmot_weights* wts, const float* crops, int n_img, int H,
                                    int W, int L, float* feats, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (!wts || !crops || !feats || !workspace || n_img <= 0 || L <= 0) return MMMOT_E_ARG;
  if (H % 32 || W % 32 || H <= 0 || W <= 0 || n_img % L) return MMMOT_E_SHAPE;
  cudaStream_t st = (cudaStream_t)stream;
  MmArena ar(workspace, workspace_bytes);
  AppWs ws = carve_appearance(ar, n_img, H, W, false);
  if (!ar.ok()) return MMMOT_E_WORKSPACE;

  // Tensor-core trunk: activations live as FP16 hi/lo NHWC planes between layers; the epilogue of one conv
  // writes exactly what the next conv's TMA loads read (3x3 taps = shifted boxes, padding = TMA zero fill).
  // engine choice depends on per-pair shapes only (never on the batch size), so batched, looped and sharded runs
  // take the same path and stay bit-identical
  const bool tc_trunk = mm_engine() == 2 || (mm_engine() == 0 && (long)L * H * W >= 32768);
  if (tc_trunk) {
    __half* hb[2] = {reinterpret_cast<__half*>(ws.buf[0]), reinterpret_cast<__half*>(ws.buf[1])};
    const __half* cur = nullptr;
    long cur_plane = 0;
    int which = 0, h = H, w = W;
    const bool timed = mm_timing_on();   // roofline hook: every launch tagged (stage, layer)
    int* status = ar.status();
    for (int i = 0; i < 13; i++) {
      const int cout = kVggCout[i], cin = kVggCin[i];
      const long plane_out = (long)n_img * h * w * cout;
      int pooled_in_epilogue = 0;
      // algorithmic FLOPs 2*Cout*9Cin*pixels; compulsory bytes: activation in + activation out at 4 B per element
      // (the pooled map when the 2x2 max-pool is fused into the epilogue)
      if (timed) mm_timing_begin(st, MM_T_VGG0 + i, 2.0 * cout * 9.0 * cin * (double)n_img * h * w,
                                 4.0 * (double)n_img * h * w * (cin + (i == 1 ? cout / 4.0 : cout)));
      if (i == 0) {
        // im2col taps (if that variant runs) in the other activation buffer, dead once the contraction has run
        MM_TRY(vgg_conv0_launch(crops, n_img, h, w, wts->w[MMMOT_W_VGG_WT0], wts->w[MMMOT_W_VGG_B0],
                                (const uint4*)wts->w[MMMOT_W_VGG_WP0], wts->tc_scale[MMMOT_W_VGG_WP0],
                                (const uint4*)wts->w[MMMOT_W_VGG_WPX0], hb[which], plane_out, hb[which ^ 1], status,
                                nullptr, st));
      } else {
        GemmP p = gemm_defaults();
        p.bias = wts->w[MMMOT_W_VGG_B0 + i];
        p.M = cout;
        p.relu = 1;
        // a pooled layer asks for the 2x2 max-pool to be fused into the epilogue; a skip map's global average (SkipPool)
        // rides along as per-image fixed-point sums
        const bool skip_layer = kPoolAfter[i] && kSkipAfter[i] >= 0;
        if (skip_layer) MM_CUDA(cudaMemsetAsync(ws.pool_sum, 0, (size_t)n_img * cout * sizeof(unsigned long long), st));
        MM_TRY(gemm_tma_launch_conv(p, (const uint4*)wts->w[MMMOT_W_VGG_WP0 + i], wts->tc_scale[MMMOT_W_VGG_WP0 + i], cur,
                                    cur_plane, n_img, h, w, cin, hb[which], plane_out, st, ws.kseg_scratch,
                                    kPoolAfter[i] ? plane_out / 4 : 0, &pooled_in_epilogue, status,
                                    skip_layer ? ws.pool_sum : nullptr, i == 1 ? (const uint4*)wts->w[MMMOT_W_VGG_WPX0 + 1] : nullptr));
      }
      if (timed) mm_timing_end(st);
      cur = hb[which]; cur_plane = plane_out; which ^= 1;
      if (kPoolAfter[i]) {
        h /= 2; w /= 2;
        const long plane_p = (long)n_img * h * w * cout;
        // compulsory bytes: separate pool = read the map + write the pooled one (+ read it again for the mean); fused =
        // the per-image sums only
        if (timed) mm_timing_begin(st, MM_T_VGG_POOL, 0.0, pooled_in_epilogue ? 12.0 * n_img * cout : 4.0 * 6.0 * plane_p);
        if (pooled_in_epilogue) {
          cur_plane = plane_p;
        } else {
          const long n8 = plane_p / 8;
          maxpool2_planar_kernel<<<mm_cdiv(n8, 256), 256, 0, st>>>(cur, hb[which], n8, h, w, cout, cur_plane, plane_p);
          MM_LAUNCH_CHECK();
          cur = hb[which]; cur_plane = plane_p; which ^= 1;
        }
        int s = kSkipAfter[i];
        if (s >= 0 && pooled_in_epilogue && i > 1) {
          const long nn = (long)n_img * kSkipC[s];
          pool_sum_mean_kernel<<<mm_cdiv(nn, 256), 256, 0, st>>>(ws.pool_sum, ws.pooled[s], nn, 1.0f / (float)(h * w));
          MM_LAUNCH_CHECK();
        } else if (s >= 0) {
          plane_mean_planar_kernel<<<mm_cdiv((long)n_img * kSkipC[s], 128), 128, 0, st>>>(cur, ws.pooled[s], n_img, h * w,
                                                                                         kSkipC[s], cur_plane);
          MM_LAUNCH_CHECK();
        }
        if (timed) mm_timing_end(st);
      }
    }
  } else {
    MM_TRY(vgg_fp32_trunk(wts, crops, n_img, H, W, ws.buf, ws.pooled, nullptr, st));
  }
  return mm_launch_skip_heads(wts, ws.pooled, n_img, L, feats, st);
}

extern "C" int mmmot_appearance_train_fwd(const mmmot_weights* wts, const float* crops, int n_img, int H, int W, int L,
                                          float* feats, float* bn_stats, const float* drop_mask2,
                                          const float* drop_mask3, void* workspace, size_t workspace_bytes,
                                          void* stream) {
  if (!wts || !crops || !feats || !bn_stats || !workspace || n_img <= 0 || L <= 0) return MMMOT_E_ARG;
  if (H % 32 || W % 32 || H <= 0 || W <= 0 || n_img % L) return MMMOT_E_SHAPE;
  if (!wts->w[MMMOT_W_VGG_RAWW0]) return MMMOT_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  MmArena ar(workspace, workspace_bytes);
  AppWs ws = carve_appearance(ar, n_img, H, W, true);
  if (!ar.ok()) return MMMOT_E_WORKSPACE;
  ws.tr.bn_stats = bn_stats;
  ws.tr.drop_mask[0] = drop_mask2;
  ws.tr.drop_mask[1] = drop_mask3;
  MM_TRY(vgg_fp32_trunk(wts, crops, n_img, H, W, ws.buf, ws.pooled, &ws.tr, st));
  return mm_launch_skip_heads(wts, ws.pooled, n_img, L, feats, st);
}

// the four SkipPool heads on the pooled maps -> stack 0 of feats (eval and training mode); a NULL
// map skips its head (mmmot_debug_skip_heads)
int mm_launch_skip_heads(const mmmot_weights* wts, float* const* pooled, int n_img, int L, float* feats, cudaStream_t st) {
  for (int s = 0; s < 4; s++) {
    if (!pooled[s]) continue;
    const float* const* q = &wts->w[MMMOT_W_SKIP0 + 10 * s];
    int C = kSkipC[s], mid = C / 4 > 64 ? C / 4 : 64;
    skip_head_kernel<<<n_img, 128, 0, st>>>(pooled[s], q[0], q[1], q[2], q[3], q[4], q[5], q[6], q[7],
                                            q[8], q[9], C, mid, L, s, feats);
    MM_LAUNCH_CHECK();
  }
  return 0;
}

// Test hook: the SkipPool heads on pooled vectors the caller chooses, through mm_launch_skip_heads.
extern "C" int mmmot_debug_skip_heads(const mmmot_weights* wts, const float* pooled0, const float* pooled1,
                                      const float* pooled2, const float* pooled3, int n_img, int L, float* feats,
                                      void* stream) {
  if (!wts || !feats || n_img <= 0 || L <= 0 || n_img % L) return MMMOT_E_ARG;
  float* const pooled[4] = {const_cast<float*>(pooled0), const_cast<float*>(pooled1), const_cast<float*>(pooled2),
                            const_cast<float*>(pooled3)};
  return mm_launch_skip_heads(wts, pooled, n_img, L, feats, (cudaStream_t)stream);
}
