// Appearance branch on a ResNet-50/101/152 trunk + 4 SkipPool heads (eval mode, BatchNorm folded).
// Replaces reference modules/appear_net.py:60-83 (AppearanceNet with appear_arch resnetXX and skip pooling), :174-176
// (res_forward), :213-256 (the Resnet wrapper) and torchvision's Bottleneck v1.5 (the stride on the 3x3 conv).
//
// One graph, two engines (the choice depends on per-pair shapes only, as in mmmot_appearance_fwd):
//   tensor cores: activations live as FP16 hi/lo NHWC planes [2][n][h][w][C] between layers; stride-1 1x1 convs are
//     matrix contractions straight on the planes, stride-1 3x3 convs the TMA conv kernel (3x3 taps = shifted boxes),
//     the stem and every stride-2 conv a gather into hi/lo rows followed by a matrix contraction.
//   FP32 FFMA engine: activations channel-major [C][n][h][w] fp32; stride-1 1x1 convs read them directly, every other
//     conv after an fp32 gather into [K][pixels].
// The residual add + ReLU is a separate elementwise kernel on both engines (DESIGN.md §5.1, "ResNet appearance trunk").
#include <cuda_fp16.h>

#include <algorithm>
#include <utility>

#include "gemm_tma.cuh"

int mm_simt_direct(const GemmP& p, cudaStream_t st);
int mm_launch_plane_mean_planar(const __half* in, float* pooled, int n_img, int hw, int C, long plane, cudaStream_t st);

namespace {

constexpr int kStemK = 147, kStemKp = 160;   // 7x7x3 taps; the packed tiles' K, zero-padded to a multiple of 32

// ---- tensor-core engine: FP16 hi/lo planes ----

// Stem taps of the fp32 NCHW crops [n][3][H][W] (7x7, stride 2, pad 3) -> rows [2][n*Ho*Wo][160], k = (ky*7+kx)*3 + ci,
// k >= 147 zero.  One thread per (output pixel, group of 8 k).
__global__ void stem_gather_planar_kernel(const float* __restrict__ in, long n_items, int H, int W, int Ho, int Wo,
                                          __half* __restrict__ out, long plane, int* status) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;
  const int kg = (int)(idx % (kStemKp / 8));
  const long pix = idx / (kStemKp / 8);
  const int hwo = Ho * Wo;
  const long img = pix / hwo;
  const int r = (int)(pix - img * hwo);
  const int yo = r / Wo, xo = r - yo * Wo;
  const float* src = in + img * 3 * (long)H * W;
  __align__(16) __half h[8], l[8];
  float amax = 0.f;
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const int k = kg * 8 + e;
    float v = 0.f;
    if (k < kStemK) {
      const int tap = k / 3, ci = k - tap * 3;
      const int yy = 2 * yo + tap / 7 - 3, xx = 2 * xo + tap % 7 - 3;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = __ldg(src + ((long)ci * H + yy) * W + xx);
    }
    tma::split_f16(v, h[e], l[e]);
    amax = fmaxf(amax, fabsf(v));
  }
  mm_range_flag(status, amax);
  *reinterpret_cast<uint4*>(out + pix * kStemKp + kg * 8) = *reinterpret_cast<const uint4*>(h);
  *reinterpret_cast<uint4*>(out + plane + pix * kStemKp + kg * 8) = *reinterpret_cast<const uint4*>(l);
}

// Taps of a ks x ks / stride s / pad p conv on NHWC planes [2][n][H][W][C] -> rows [2][n*Ho*Wo][ks*ks*C],
// k = (ky*ks+kx)*C + ci; out-of-image taps are zero.  The (hi, lo) pairs are copied, not re-split.  One thread per
// (output pixel, tap, 8 channels).
__global__ void gather_planar_kernel(const __half* __restrict__ in, long in_plane, int H, int W, int C, int ks, int stride,
                                     int pad, int Ho, int Wo, long n_items, __half* __restrict__ out, long out_plane) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;
  const int c8n = C >> 3, taps = ks * ks;
  const int c = (int)(idx % c8n) * 8;
  long t = idx / c8n;
  const int tap = (int)(t % taps);
  const long pix = t / taps;
  const int hwo = Ho * Wo;
  const long img = pix / hwo;
  const int r = (int)(pix - img * hwo);
  const int yo = r / Wo, xo = r - yo * Wo;
  const int yy = yo * stride + tap / ks - pad, xx = xo * stride + tap % ks - pad;
  uint4 h = make_uint4(0, 0, 0, 0), l = h;
  if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
    const __half* src = in + ((img * H + yy) * W + xx) * (long)C + c;
    h = *reinterpret_cast<const uint4*>(src);
    l = *reinterpret_cast<const uint4*>(src + in_plane);
  }
  __half* dst = out + pix * (long)taps * C + (long)tap * C + c;
  *reinterpret_cast<uint4*>(dst) = h;
  *reinterpret_cast<uint4*>(dst + out_plane) = l;
}

// 3x3 / stride 2 / pad 1 max-pool on NHWC planes; padding never wins (PyTorch pads with -inf).  The max IS one of the
// inputs, so its (hi, lo) pair is copied.  One thread per (output pixel, 8 channels).
__global__ void maxpool3s2_planar_kernel(const __half* __restrict__ in, long in_plane, int H, int W, int C, int Ho, int Wo,
                                         long n_items, __half* __restrict__ out, long out_plane) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;
  const int c8n = C >> 3;
  const int c = (int)(idx % c8n) * 8;
  const long pix = idx / c8n;
  const int hwo = Ho * Wo;
  const long img = pix / hwo;
  const int r = (int)(pix - img * hwo);
  const int yo = r / Wo, xo = r - yo * Wo;
  float best[8];
  uint4 bh = make_uint4(0, 0, 0, 0), bl = bh;
  __half* oh = reinterpret_cast<__half*>(&bh);
  __half* ol = reinterpret_cast<__half*>(&bl);
#pragma unroll
  for (int e = 0; e < 8; e++) best[e] = -INFINITY;
  for (int t = 0; t < 9; t++) {
    const int yy = 2 * yo + t / 3 - 1, xx = 2 * xo + t % 3 - 1;
    if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
    const __half* src = in + ((img * H + yy) * W + xx) * (long)C + c;
    const uint4 h = *reinterpret_cast<const uint4*>(src);
    const uint4 l = *reinterpret_cast<const uint4*>(src + in_plane);
    const __half* hh = reinterpret_cast<const __half*>(&h);
    const __half* ll = reinterpret_cast<const __half*>(&l);
#pragma unroll
    for (int e = 0; e < 8; e++) {
      const float f = __half2float(hh[e]) + __half2float(ll[e]);
      if (f > best[e]) { best[e] = f; oh[e] = hh[e]; ol[e] = ll[e]; }
    }
  }
  __half* dst = out + pix * (long)C + c;
  *reinterpret_cast<uint4*>(dst) = bh;
  *reinterpret_cast<uint4*>(dst + out_plane) = bl;
}

// y = relu(y + id) on planes (8 elements per thread): both sums of hi + lo are exact in fp32, their sum rounds once and
// is split again.  Raises the FP16 range flag instead of clamping silently: on the value stored (a sum >= 65504), and on
// a NaN sum, which the ReLU would otherwise turn into 0.  A large negative sum is stored exactly (as 0) and is not flagged.
__global__ void add_relu_planar_kernel(__half* __restrict__ y, long y_plane, const __half* __restrict__ id, long id_plane,
                                       long n8, int* status) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n8) return;
  const uint4 ah = reinterpret_cast<const uint4*>(y)[idx], al = reinterpret_cast<const uint4*>(y + y_plane)[idx];
  const uint4 bh = reinterpret_cast<const uint4*>(id)[idx], bl = reinterpret_cast<const uint4*>(id + id_plane)[idx];
  const __half* a0 = reinterpret_cast<const __half*>(&ah);
  const __half* a1 = reinterpret_cast<const __half*>(&al);
  const __half* b0 = reinterpret_cast<const __half*>(&bh);
  const __half* b1 = reinterpret_cast<const __half*>(&bl);
  __align__(16) __half h[8], l[8];
  bool bad = false;
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const float sum = (__half2float(a0[e]) + __half2float(a1[e])) + (__half2float(b0[e]) + __half2float(b1[e]));
    tma::split_f16(fmaxf(sum, 0.f), h[e], l[e]);
    bad |= !(sum < MM_F16_MAX);          // also true for NaN
  }
  if (bad) mm_range_flag(status, INFINITY);
  reinterpret_cast<uint4*>(y)[idx] = *reinterpret_cast<const uint4*>(h);
  reinterpret_cast<uint4*>(y + y_plane)[idx] = *reinterpret_cast<const uint4*>(l);
}

// ---- FP32 engine: channel-major [C][n][h][w] ----

// Taps of a ks x ks / stride s / pad p conv -> cols [ks*ks*C][n*Ho*Wo], k = (ky*ks+kx)*C + ci.  Element (img, c, y, x)
// of the source is in[img*s_img + c*s_c + y*W + x]: the crops (NCHW, s_img = 3HW, s_c = HW) and the channel-major
// activations (s_img = HW, s_c = n*HW) alike.  One thread per (k, output pixel).
__global__ void gather_f32_kernel(const float* __restrict__ in, long s_img, long s_c, int H, int W, int C, int ks,
                                  int stride, int pad, int Ho, int Wo, long n_out, long n_items, float* __restrict__ out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;
  const long pix = idx % n_out;
  const int k = (int)(idx / n_out);
  const int tap = k / C, ci = k - tap * C;
  const int hwo = Ho * Wo;
  const long img = pix / hwo;
  const int r = (int)(pix - img * hwo);
  const int yo = r / Wo, xo = r - yo * Wo;
  const int yy = yo * stride + tap / ks - pad, xx = xo * stride + tap % ks - pad;
  out[idx] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(in + img * s_img + ci * s_c + (long)yy * W + xx) : 0.f;
}

// 3x3 / stride 2 / pad 1 max-pool of every (c, img) plane
__global__ void maxpool3s2_f32_kernel(const float* __restrict__ in, int H, int W, int Ho, int Wo, long n_items,
                                      float* __restrict__ out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;
  const int hwo = Ho * Wo;
  const long plane = idx / hwo;
  const int r = (int)(idx - plane * hwo);
  const int yo = r / Wo, xo = r - yo * Wo;
  const float* src = in + plane * (long)H * W;
  float best = -INFINITY;
  for (int t = 0; t < 9; t++) {
    const int yy = 2 * yo + t / 3 - 1, xx = 2 * xo + t % 3 - 1;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) best = fmaxf(best, src[yy * W + xx]);
  }
  out[idx] = best;
}

__global__ void add_relu_f32_kernel(float* __restrict__ y, const float* __restrict__ id, long n) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n) y[idx] = fmaxf(y[idx] + id[idx], 0.f);
}

// pooled[img][c] = mean over hw of x[c][img][hw]: one warp per (img, c)
__global__ void mean_cm_f32_kernel(const float* __restrict__ x, int n_img, int hw, int C, float* __restrict__ pooled) {
  const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long)n_img * C) return;
  const int c = (int)(w % C);
  const long img = w / C;
  const float* src = x + ((long)c * n_img + img) * hw;
  float s = 0.f;
  for (int i = lane; i < hw; i += 32) s += src[i];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) pooled[w] = s / (float)hw;
}

// ---- SkipPool heads of the ResNet stages (C = 256..2048, mid = C/4 = 64..512) ----
__device__ __forceinline__ float block_sum_512(float v, float* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; i++) s += red[i];
  return s;
}

// One CTA (512 threads) per image: GN(1,C) -> 1x1 conv C -> mid -> GN(1,mid) -> ReLU -> 1x1 conv mid -> 128 -> GN(1,128)
// -> ReLU (reference appear_net.py:19-25), the arithmetic of appearance.cu's skip_head_kernel on wider vectors.
__global__ void __launch_bounds__(512) skip_head_wide_kernel(
    const float* __restrict__ pooled,  // [n_img][C]
    const float* __restrict__ g0w, const float* __restrict__ g0b, const float* __restrict__ w1t,
    const float* __restrict__ b1, const float* __restrict__ g1w, const float* __restrict__ g1b,
    const float* __restrict__ w2t, const float* __restrict__ b2, const float* __restrict__ g2w,
    const float* __restrict__ g2b, int C, int mid, int L, int head, float* __restrict__ feats) {
  __shared__ float v[2048];
  __shared__ float h[512];
  __shared__ float red[16];
  const int img = blockIdx.x, t = threadIdx.x;
  const float eps = 1e-5f;
  float s = 0.f;
  for (int c = t; c < C; c += 512) { const float x = pooled[(long)img * C + c]; v[c] = x; s += x; }
  float mean = block_sum_512(s, red) / C;
  s = 0.f;
  for (int c = t; c < C; c += 512) { const float d = v[c] - mean; s += d * d; }
  float rstd = rsqrtf(block_sum_512(s, red) / C + eps);
  for (int c = t; c < C; c += 512) v[c] = (v[c] - mean) * rstd * g0w[c] + g0b[c];
  __syncthreads();
  float a = 0.f;
  if (t < mid) {
    a = b1[t];
    for (int c = 0; c < C; c++) a = fmaf(w1t[(long)c * mid + t], v[c], a);
  }
  mean = block_sum_512(t < mid ? a : 0.f, red) / mid;
  float d = t < mid ? a - mean : 0.f;
  rstd = rsqrtf(block_sum_512(d * d, red) / mid + eps);
  if (t < mid) h[t] = fmaxf(d * rstd * g1w[t] + g1b[t], 0.f);
  __syncthreads();
  a = 0.f;
  if (t < 128) {
    a = b2[t];
    for (int c = 0; c < mid; c++) a = fmaf(w2t[c * 128 + t], h[c], a);
  }
  mean = block_sum_512(t < 128 ? a : 0.f, red) / 128.f;
  d = t < 128 ? a - mean : 0.f;
  rstd = rsqrtf(block_sum_512(d * d, red) / 128.f + eps);
  if (t < 128) {
    const float o = fmaxf(d * rstd * g2w[t] + g2b[t], 0.f);
    const int pair = img / L, l = img - pair * L;
    feats[(((long)pair * 3 + 0) * 512 + head * 128 + t) * L + l] = o;
  }
}

int launch_heads(const mmmot_resnet_weights* rw, float* const* pooled, int n_img, int L, float* feats, cudaStream_t st) {
  for (int s = 0; s < 4; s++) {
    const float* const* q = rw->head[s];
    const int C = 256 << s;
    skip_head_wide_kernel<<<n_img, 512, 0, st>>>(pooled[s], q[0], q[1], q[2], q[3], q[4], q[5], q[6], q[7], q[8], q[9], C,
                                                 C / 4, L, s, feats);
    MM_LAUNCH_CHECK();
  }
  return 0;
}

// ---- FPN head (reference appear_net.py:83-104,192-210; DESIGN.md §5.1, "FPN head") ----
// H and W are multiples of 32, so every top-down interpolate is an exact 2x bilinear upsample, which preserves the
// spatial mean: avgpool(out) = sum over the four levels of the mean of their ReLU'd laterals.  The laterals are
// therefore only ever reduced to per-image channel means; no 512-channel map exists.

// Tables of one level's lateral on the tensor cores (h x w pixels per image, L images per pair): seg[pix] = image of
// pixel pix; tiles: per pair, ceil(L*hw / 256) column tiles {pair, first pixel, length} that start at the pair's first
// pixel, so how a pair's pixels fall into 32-column chunks does not depend on the pair's place in the batch; sc / sh
// [pairs][512] = 1 / 0 (the epilogue's per-group affine).  One thread per item of the largest of the three.
__global__ void fpn_tables_kernel(int n_img, int hw, int L, int tpp, int* __restrict__ seg, int4* __restrict__ tiles,
                                  float* __restrict__ sc, float* __restrict__ sh) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int pairs = n_img / L;
  const long per_pair = (long)L * hw;
  if (idx < (long)n_img * hw) seg[idx] = (int)(idx / hw);
  if (idx < (long)pairs * tpp) {
    const int pair = (int)(idx / tpp), j = (int)(idx - (long)pair * tpp);
    const long c0 = pair * per_pair + (long)j * tc::BN;
    tiles[idx] = make_int4(pair, (int)c0, (int)min((long)tc::BN, per_pair - (long)j * tc::BN), 0);
  }
  if (idx < (long)pairs * 512) { sc[idx] = 1.f; sh[idx] = 0.f; }
}

// means[img][c] = segsum[img][c] * 2^-32 / hw
__global__ void fpn_segsum_mean_kernel(const unsigned long long* __restrict__ segsum, long n, int hw,
                                       float* __restrict__ means) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n) means[idx] = (float)((double)segsum[idx] * (1.0 / 4294967296.0) / (double)hw);
}

// One CTA (512 threads) per image: v = sum of the four level means [4][n_img][512], then ReLU(W_last v + b_last) with
// conv_last.2 (BatchNorm) folded into conv_last.1 -> stack 0 of feats.  On the tensor cores the level means come from
// 2^-32 fixed-point sums (fpn_segsum_mean_kernel): each per-(image, channel) sum of ReLU'd lateral values must stay
// below 2^32 (at 224 x 224, an average lateral value below 1.3e6 on level 0).
__global__ void __launch_bounds__(512) fpn_head_kernel(const float* __restrict__ means, int n_img,
                                                       const float* __restrict__ wt, const float* __restrict__ bias,
                                                       int L, float* __restrict__ feats) {
  __shared__ float v[512];
  const int img = blockIdx.x, t = threadIdx.x;
  const long lv = (long)n_img * 512, o = (long)img * 512 + t;
  v[t] = ((means[o] + means[lv + o]) + means[2 * lv + o]) + means[3 * lv + o];
  __syncthreads();
  float a = bias[t];
  for (int c = 0; c < 512; c++) a = fmaf(wt[c * 512 + t], v[c], a);
  const int pair = img / L, l = img - pair * L;
  feats[(((long)pair * 3 + 0) * 512 + t) * L + l] = fmaxf(a, 0.f);
}

// ---- the trunk ----

int total_convs(const int* blocks) { return 1 + 3 * (blocks[0] + blocks[1] + blocks[2] + blocks[3]) + 4; }

// K-segment scratch of the tensor-core 3x3 convs whose K reaches 2304 (layer3: 256 channels at H/16, layer4: 512 at
// H/32): column tiles x 256 x M floats of the plan the launcher takes
size_t kseg_floats(int n_img, int H, int W) {
  size_t m = 0;
  for (int s = 2; s < 4; s++) {
    const int C = 64 << s, h = H >> (s + 2), w = W >> (s + 2);
    const ConvPlan c = conv_plan(C, false, n_img, h, w, C, false, true, 0, 36);
    m = std::max(m, (size_t)c.num_tiles * tc::BN * C);
  }
  return m;
}

// Workspace: five activation buffers (x, conv1, conv2, conv3 / block output, downsample), the gather rows, the K-segment
// scratch and the pooled skip maps.  Sizes in fp32 elements, which equal the bytes / 4 of the FP16 hi/lo planes of the
// same tensor, so one carve serves both engines.  Largest tensors, in units of n*H*W: stem output (64 ch at H/2) and
// layer1 output (256 at H/4) 16; conv1/conv2 outputs 8 (layer2's first conv1, 128 ch at H/4); gathers 40 (stem: 160 taps
// at H/2 as hi/lo rows; the FP32 engine's 147 taps, layer1's 576 at H/4).
struct ResWs {
  float* act[5];
  float* cols;
  float* kseg;
  float* pooled[4];
};
ResWs carve_resnet(MmArena& a, int n_img, int H, int W) {
  ResWs w = {};
  const size_t nhw = (size_t)n_img * H * W;
  w.act[0] = a.take<float>(nhw * 16);
  w.act[1] = a.take<float>(nhw * 8);
  w.act[2] = a.take<float>(nhw * 8);
  w.act[3] = a.take<float>(nhw * 16);
  w.act[4] = a.take<float>(nhw * 16);
  w.cols = a.take<float>(nhw * 40);
  w.kseg = a.take<float>(kseg_floats(n_img, H, W));
  for (int s = 0; s < 4; s++) w.pooled[s] = a.take<float>((size_t)n_img * (256 << s));
  return w;
}

// The FPN head's scratch, behind the trunk's: the level means [4][n_img][512], one level's fixed-point sums and the
// tables of the largest level (H/4 x W/4).  The FP32 engine's laterals ([512][n*hw], at most n*H*W*32 floats) go
// through the trunk's gather scratch.
struct FpnWs {
  float* means;
  unsigned long long* segsum;
  float *sc, *sh;
  int* seg;
  int4 *tiles, *ctab;
};
int fpn_tiles_per_pair(int L, int hw) { return mm_cdiv((long)L * hw, tc::BN); }
FpnWs carve_fpn(MmArena& a, int n_img, int H, int W, int L) {
  FpnWs f = {};
  const int hw0 = (H / 4) * (W / 4), pairs = mm_cdiv(n_img, L);
  const size_t max_tiles = (size_t)pairs * fpn_tiles_per_pair(L, hw0);
  f.means = a.take<float>((size_t)4 * n_img * 512);
  f.segsum = a.take<unsigned long long>((size_t)n_img * 512);
  f.sc = a.take<float>((size_t)pairs * 512);
  f.sh = a.take<float>((size_t)pairs * 512);
  f.seg = a.take<int>((size_t)n_img * hw0);
  f.tiles = a.take<int4>(max_tiles);
  f.ctab = a.take<int4>(2 * max_tiles);
  return f;
}

// One conv of the graph on either engine.  x / y: the engine's activation layout at (h, w) / (h/stride, w/stride).
struct Trunk {
  const mmmot_resnet_weights* rw;
  int n_img;
  bool tc;
  bool timed;
  float* cols;
  float* kseg;
  int* status;
  cudaStream_t st;

  // taps of a ks x ks / stride / pad ks/2 conv of x (Cin channels at h x w) -> out: hi/lo rows [2][n_out][ks*ks*Cin]
  // (tensor cores) or fp32 [ks*ks*Cin][n_out] (FP32 engine), k = (ky*ks+kx)*Cin + ci
  int gather(const float* x, int h, int w, int Cin, int ks, int stride, float* out) const {
    const int ho = h / stride, wo = w / stride;
    const long n_out = (long)n_img * ho * wo, n_in = (long)n_img * h * w;
    if (tc) {
      const long items = n_out * ks * ks * (Cin / 8);
      gather_planar_kernel<<<mm_cdiv(items, 256), 256, 0, st>>>(reinterpret_cast<const __half*>(x), n_in * Cin, h, w, Cin,
                                                                ks, stride, ks / 2, ho, wo, items,
                                                                reinterpret_cast<__half*>(out), n_out * ks * ks * Cin);
    } else {
      const long items = (long)ks * ks * Cin * n_out;
      gather_f32_kernel<<<mm_cdiv(items, 256), 256, 0, st>>>(x, (long)h * w, n_in, h, w, Cin, ks, stride, ks / 2, ho, wo,
                                                             n_out, items, out);
    }
    MM_LAUNCH_CHECK();
    return 0;
  }

  // the stem's taps of the fp32 NCHW crops -> out: hi/lo rows [2][n_out][160] (tensor cores, FP16 range flag raised on
  // an input |x| >= 65504) or fp32 [147][n_out] (FP32 engine)
  int stem_gather(const float* crops, int H, int W, float* out) const {
    const int ho = H / 2, wo = W / 2;
    const long n_out = (long)n_img * ho * wo;
    if (tc) {
      const long items = n_out * (kStemKp / 8);
      stem_gather_planar_kernel<<<mm_cdiv(items, 256), 256, 0, st>>>(crops, items, H, W, ho, wo,
                                                                     reinterpret_cast<__half*>(out), n_out * kStemKp, status);
    } else {
      const long items = kStemK * n_out;
      gather_f32_kernel<<<mm_cdiv(items, 256), 256, 0, st>>>(crops, 3L * H * W, (long)H * W, H, W, 3, 7, 2, 3, ho, wo, n_out,
                                                             items, out);
    }
    MM_LAUNCH_CHECK();
    return 0;
  }

  // ks x ks conv, stride 1 or 2, pad ks/2; Cin -> M; relu in the epilogue
  int conv(int i, const float* x, int h, int w, int Cin, int ks, int stride, int M, bool relu, float* y) const {
    const int ho = h / stride, wo = w / stride;
    const long n_out = (long)n_img * ho * wo, n_in = (long)n_img * h * w;
    const int tag = stride == 2 ? MM_T_RES_S2 : ks == 1 ? MM_T_RES_1X1 : MM_T_RES_3X3;
    const double K = (double)ks * ks * Cin;
    if (timed) mm_timing_begin(st, tag, 2.0 * M * K * n_out, 4.0 * (double)(n_in * Cin + n_out * M));
    GemmP p = gemm_defaults();
    p.bias = rw->bias[i]; p.M = M; p.relu = relu;
    if (tc) {
      const __half* xh = reinterpret_cast<const __half*>(x);
      __half* yh = reinterpret_cast<__half*>(y);
      if (ks == 3 && stride == 1) {
        // K-segmented accumulation (mmmot_set_kseg) where K >= 2304, as in the VGG trunk's deep layers
        MM_TRY(gemm_tma_launch_conv(p, (const uint4*)rw->wp[i], rw->wp_scale[i], xh, n_in * Cin, n_img, h, w, Cin, yh,
                                    n_out * M, st, 9 * Cin >= 2304 ? kseg : nullptr, 0, nullptr, status));
      } else {
        const __half* rows = xh;
        long rows_plane = n_in * Cin;
        if (stride != 1) {
          MM_TRY(gather(x, h, w, Cin, ks, stride, cols));
          rows_plane = n_out * ks * ks * Cin;
          rows = reinterpret_cast<const __half*>(cols);
        }
        p.K = (int)K; p.S = (int)n_out; p.tiles_per_group = mm_cdiv(n_out, tc::BN); p.num_tiles = p.tiles_per_group;
        p.Y = y; p.y_ms = M;
        MM_TRY(gemm_tma_launch_mat(p, (const uint4*)rw->wp[i], rw->wp_scale[i], rows, rows_plane, n_out, (int)K,
                                   tma::OUT_PLANAR, n_out * M, st, nullptr, status));
      }
    } else {
      const float* xin = x;
      if (ks != 1 || stride != 1) {
        MM_TRY(gather(x, h, w, Cin, ks, stride, cols));
        xin = cols;
      }
      p.Wt = rw->wt[i]; p.ldw = M; p.K = (int)K;
      p.S = (int)n_out; p.tiles_per_group = mm_cdiv(n_out, 128); p.num_tiles = p.tiles_per_group;
      p.X = xin; p.x_ks = n_out;
      p.Y = y; p.y_ms = n_out;
      MM_TRY(mm_simt_direct(p, st));
    }
    if (timed) mm_timing_end(st);
    return 0;
  }

  // stem (7x7 / 2 / pad 3, 3 -> 64, ReLU) of the fp32 NCHW crops -> y at H/2
  int stem(const float* crops, int H, int W, float* y) const {
    const int ho = H / 2, wo = W / 2;
    const long n_out = (long)n_img * ho * wo;
    if (timed) mm_timing_begin(st, MM_T_RES_STEM, 2.0 * 64 * kStemK * n_out, 4.0 * ((double)n_img * 3 * H * W + n_out * 64));
    GemmP p = gemm_defaults();
    p.bias = rw->bias[0]; p.M = 64; p.relu = 1;
    p.S = (int)n_out; p.Y = y;
    MM_TRY(stem_gather(crops, H, W, cols));
    if (tc) {
      const __half* c = reinterpret_cast<const __half*>(cols);
      p.K = kStemKp; p.tiles_per_group = mm_cdiv(n_out, tc::BN); p.num_tiles = p.tiles_per_group; p.y_ms = 64;
      MM_TRY(gemm_tma_launch_mat(p, (const uint4*)rw->wp[0], rw->wp_scale[0], c, n_out * kStemKp, n_out, kStemKp,
                                 tma::OUT_PLANAR, n_out * 64, st, nullptr, status));
    } else {
      p.Wt = rw->wt[0]; p.ldw = 64; p.K = kStemK;
      p.tiles_per_group = mm_cdiv(n_out, 128); p.num_tiles = p.tiles_per_group;
      p.X = cols; p.x_ks = n_out; p.y_ms = n_out;
      MM_TRY(mm_simt_direct(p, st));
    }
    if (timed) mm_timing_end(st);
    return 0;
  }

  // 3x3 / 2 / pad 1 max-pool of the 64-channel stem output at (h, w)
  int maxpool(const float* x, int h, int w, float* y) const {
    const int ho = h / 2, wo = w / 2;
    const long n_in = (long)n_img * h * w * 64, n_out = (long)n_img * ho * wo * 64;
    if (timed) mm_timing_begin(st, MM_T_RES_MAXPOOL, 0.0, 4.0 * (double)(n_in + n_out));
    if (tc) {
      const long items = n_out / 8;
      maxpool3s2_planar_kernel<<<mm_cdiv(items, 256), 256, 0, st>>>(reinterpret_cast<const __half*>(x), n_in, h, w, 64, ho,
                                                                    wo, items, reinterpret_cast<__half*>(y), n_out);
    } else {
      maxpool3s2_f32_kernel<<<mm_cdiv(n_out, 256), 256, 0, st>>>(x, h, w, ho, wo, n_out, y);
    }
    MM_LAUNCH_CHECK();
    if (timed) mm_timing_end(st);
    return 0;
  }

  // y = relu(y + id), n elements
  int add_relu(float* y, const float* id, long n) const {
    if (timed) mm_timing_begin(st, MM_T_RES_ADD, (double)n, 12.0 * (double)n);
    if (tc) {
      add_relu_planar_kernel<<<mm_cdiv(n / 8, 256), 256, 0, st>>>(reinterpret_cast<__half*>(y), n,
                                                                  reinterpret_cast<const __half*>(id), n, n / 8, status);
    } else {
      add_relu_f32_kernel<<<mm_cdiv(n, 256), 256, 0, st>>>(y, id, n);
    }
    MM_LAUNCH_CHECK();
    if (timed) mm_timing_end(st);
    return 0;
  }

  // per-image channel means of a stage output (C channels at h x w) -> pooled [n_img][C]
  int mean(const float* x, int h, int w, int C, float* pooled) const {
    if (timed) mm_timing_begin(st, MM_T_RES_HEADS, (double)n_img * C * h * w, 4.0 * (double)n_img * C * (h * w + 1));
    const long n = (long)n_img * h * w * C;
    if (tc) {
      MM_TRY(mm_launch_plane_mean_planar(reinterpret_cast<const __half*>(x), pooled, n_img, h * w, C, n, st));
    } else {
      mean_cm_f32_kernel<<<mm_cdiv((long)n_img * C * 32, 256), 256, 0, st>>>(x, n_img, h * w, C, pooled);
      MM_LAUNCH_CHECK();
    }
    if (timed) mm_timing_end(st);
    return 0;
  }

  // FPN lateral k of a stage output x (C channels at h x w, L images per pair): the per-image channel means of
  // relu(fpn_in[k] conv + folded BatchNorm) -> means [n_img][512].  Tensor cores: the contraction's segment-sum
  // epilogue (Y = nullptr: nothing stored) over per-pair column tiles; FP32 engine: the lateral map into cols, then
  // its means.
  int lateral(const mmmot_fpn_weights* fw, int k, const float* x, int h, int w, int C, int L, const FpnWs& f,
              float* means) const {
    const int hw = h * w;
    const long n_pix = (long)n_img * hw;
    if (timed) mm_timing_begin(st, MM_T_FPN_LAT, 2.0 * 512 * C * n_pix, 4.0 * (double)n_pix * C);
    GemmP p = gemm_defaults();
    p.bias = fw->lat_bias[k]; p.M = 512; p.K = C;
    if (tc) {
      const int pairs = n_img / L, tpp = fpn_tiles_per_pair(L, hw);
      const long items = std::max(n_pix, (long)pairs * 512);
      fpn_tables_kernel<<<mm_cdiv(items, 256), 256, 0, st>>>(n_img, hw, L, tpp, f.seg, f.tiles, f.sc, f.sh);
      MM_LAUNCH_CHECK();
      tma::seg_chunk_tab_kernel<<<mm_cdiv(pairs * tpp * 2, 128), 128, 0, st>>>(f.tiles, pairs * tpp, f.seg, f.ctab);
      MM_LAUNCH_CHECK();
      MM_CUDA(cudaMemsetAsync(f.segsum, 0, (size_t)n_img * 512 * sizeof(unsigned long long), st));
      p.tile_tab = f.tiles; p.num_tiles = pairs * tpp;
      p.seg = f.seg; p.sc = f.sc; p.sh = f.sh;
      MM_TRY(gemm_tma_launch_mat(p, (const uint4*)fw->lat_wp[k], fw->lat_wp_scale[k], reinterpret_cast<const __half*>(x),
                                 n_pix * C, n_pix, C, tc::OUT_CL, 0, st, f.segsum, status, f.ctab));
      fpn_segsum_mean_kernel<<<mm_cdiv((long)n_img * 512, 256), 256, 0, st>>>(f.segsum, (long)n_img * 512, hw, means);
    } else {
      p.relu = 1;
      p.Wt = fw->lat_wt[k]; p.ldw = 512;
      p.S = (int)n_pix; p.tiles_per_group = mm_cdiv(n_pix, 128); p.num_tiles = p.tiles_per_group;
      p.X = x; p.x_ks = n_pix;
      p.Y = cols; p.y_ms = n_pix;
      MM_TRY(mm_simt_direct(p, st));
      mean_cm_f32_kernel<<<mm_cdiv((long)n_img * 512 * 32, 256), 256, 0, st>>>(cols, n_img, hw, 512, means);
    }
    MM_LAUNCH_CHECK();
    if (timed) mm_timing_end(st);
    return 0;
  }
};

// Trunk setup shared by the entry points: the engine (per-pair shapes only, never the batch size, as in
// mmmot_appearance_fwd) and the scratch of a carved workspace.
Trunk make_trunk(const mmmot_resnet_weights* rw, int n_img, int H, int W, int L, const ResWs& ws, int* status,
                 cudaStream_t st) {
  Trunk t;
  t.rw = rw; t.n_img = n_img;
  t.tc = mm_use_tc((long)L * H * W >= 32768);
  t.timed = mm_timing_on();
  t.cols = ws.cols; t.kseg = ws.kseg; t.status = status; t.st = st;
  return t;
}

// The trunk on the fp32 NCHW crops: stem, max-pool, layer1..layer4.  on_stage(s, x, h, w, C) runs on the output of
// layer s+1 (C = 256 << s channels at h x w, in the engine's layout) while it is live.
template <class OnStage>
int run_trunk(const Trunk& t, const float* crops, int H, int W, const ResWs& ws, OnStage on_stage) {
  const mmmot_resnet_weights* rw = t.rw;
  const int n_img = t.n_img;
  // buffers: x (block input), t1 (conv1), t2 (conv2), y (conv3, then the block output), d (downsample)
  float *x = ws.act[0], *t1 = ws.act[1], *t2 = ws.act[2], *y = ws.act[3], *d = ws.act[4];
  MM_TRY(t.stem(crops, H, W, y));
  int h = H / 2, w = W / 2;
  MM_TRY(t.maxpool(y, h, w, x));
  h /= 2; w /= 2;
  int ci = 1, cin = 64;
  for (int s = 0; s < 4; s++) {
    const int width = 64 << s, cout = 4 * width;
    for (int b = 0; b < rw->blocks[s]; b++) {
      const int stride = (b == 0 && s > 0) ? 2 : 1;
      const int ho = h / stride, wo = w / stride;
      MM_TRY(t.conv(ci, x, h, w, cin, 1, 1, width, true, t1));
      MM_TRY(t.conv(ci + 1, t1, h, w, width, 3, stride, width, true, t2));
      MM_TRY(t.conv(ci + 2, t2, ho, wo, width, 1, 1, cout, false, y));
      const float* id = x;
      if (b == 0) {
        MM_TRY(t.conv(ci + 3, x, h, w, cin, 1, stride, cout, false, d));
        id = d;
      }
      MM_TRY(t.add_relu(y, id, (long)n_img * ho * wo * cout));
      ci += b == 0 ? 4 : 3;
      std::swap(x, y);
      h = ho; w = wo; cin = cout;
    }
    MM_TRY(on_stage(s, x, h, w, cout));
  }
  return 0;
}

// The trunk's arguments, checked before any CUDA call: the block counts, the shapes, every conv's pointers.
int check_trunk(const mmmot_resnet_weights* rw, int n_img, int H, int W, int L) {
  for (int s = 0; s < 4; s++)
    if (rw->blocks[s] < 1 || rw->blocks[s] > MMMOT_RESNET_MAX_CONVS) return MMMOT_E_ARG;
  if (total_convs(rw->blocks) > MMMOT_RESNET_MAX_CONVS) return MMMOT_E_ARG;
  if (H <= 0 || W <= 0 || H % 32 || W % 32 || n_img % L) return MMMOT_E_SHAPE;
  if ((long)n_img * (H / 2) * (W / 2) >= (1L << 31)) return MMMOT_E_SHAPE;
  const int nconv = total_convs(rw->blocks);
  for (int i = 0; i < nconv; i++)
    if (!rw->wt[i] || !rw->bias[i] || !rw->wp[i]) return MMMOT_E_ARG;
  return 0;
}

constexpr int kFpnMaxTcBlocks3 = 23;   // layer3 blocks of ResNet-101: the deepest FPN trunk run on the tensor cores

bool fpn_weights_ok(const mmmot_fpn_weights* fw) {
  if (!fw || !fw->last_wt || !fw->last_bias) return false;
  for (int k = 0; k < 4; k++)
    if (!fw->lat_wt[k] || !fw->lat_bias[k] || !fw->lat_wp[k]) return false;
  return true;
}

int launch_fpn_head(const mmmot_fpn_weights* fw, const float* means, int n_img, int L, float* feats, bool timed,
                    cudaStream_t st) {
  if (timed) mm_timing_begin(st, MM_T_FPN_HEAD, 2.0 * 512 * 512 * n_img, 4.0 * (512.0 * 512 + 4.0 * 512 * n_img));
  fpn_head_kernel<<<n_img, 512, 0, st>>>(means, n_img, fw->last_wt, fw->last_bias, L, feats);
  MM_LAUNCH_CHECK();
  if (timed) mm_timing_end(st);
  return 0;
}

}  // namespace

extern "C" size_t mmmot_appearance_resnet_workspace(int n_img, int H, int W) {
  if (n_img <= 0 || H <= 0 || W <= 0) return 0;
  MmArena a(nullptr, 0);
  carve_resnet(a, n_img, H, W);
  return a.off;
}

extern "C" int mmmot_appearance_resnet_fwd(const mmmot_weights* wts, const mmmot_resnet_weights* rw, const float* crops,
                                           int n_img, int H, int W, int L, float* feats, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  (void)wts;
  if (!rw || !crops || !feats || !workspace || n_img <= 0 || L <= 0) return MMMOT_E_ARG;
  MM_TRY(check_trunk(rw, n_img, H, W, L));
  for (int s = 0; s < 4; s++)
    for (int j = 0; j < 10; j++)
      if (!rw->head[s][j]) return MMMOT_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  MmArena ar(workspace, workspace_bytes);
  ResWs ws = carve_resnet(ar, n_img, H, W);
  if (!ar.ok()) return MMMOT_E_WORKSPACE;

  const Trunk t = make_trunk(rw, n_img, H, W, L, ws, ar.status(), st);
  MM_TRY(run_trunk(t, crops, H, W, ws, [&](int s, const float* x, int h, int w, int C) {
    return t.mean(x, h, w, C, ws.pooled[s]);
  }));
  if (t.timed) mm_timing_begin(st, MM_T_RES_HEADS, 0.0, 0.0);
  MM_TRY(launch_heads(rw, ws.pooled, n_img, L, feats, st));
  if (t.timed) mm_timing_end(st);
  return 0;
}

extern "C" size_t mmmot_appearance_resnet_fpn_workspace(int n_img, int H, int W, int L) {
  if (n_img <= 0 || H <= 0 || W <= 0 || L <= 0) return 0;
  MmArena a(nullptr, 0);
  carve_resnet(a, n_img, H, W);
  carve_fpn(a, n_img, H, W, L);
  return a.off;
}

extern "C" int mmmot_appearance_resnet_fpn_fwd(const mmmot_resnet_weights* rw, const mmmot_fpn_weights* fw,
                                               const float* crops, int n_img, int H, int W, int L, float* feats,
                                               void* workspace, size_t workspace_bytes, void* stream) {
  if (!rw || !crops || !feats || !workspace || n_img <= 0 || L <= 0) return MMMOT_E_ARG;
  MM_TRY(check_trunk(rw, n_img, H, W, L));
  if (!fpn_weights_ok(fw)) return MMMOT_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  MmArena ar(workspace, workspace_bytes);
  ResWs ws = carve_resnet(ar, n_img, H, W);
  FpnWs f = carve_fpn(ar, n_img, H, W, L);
  if (!ar.ok()) return MMMOT_E_WORKSPACE;

  Trunk t = make_trunk(rw, n_img, H, W, L, ws, ar.status(), st);
  // No GroupNorm follows this head, so the trunk's tensor-core error reaches the features undamped: the contractions'
  // accumulation bias adds up block by block, and at ResNet-152's 36 layer3 blocks it takes the link scores past 1e-4
  // (DESIGN.md §5.1, "FPN head").  Trunks deeper than ResNet-101 run on the FP32 engine in every engine mode.
  if (rw->blocks[2] > kFpnMaxTcBlocks3) t.tc = false;
  MM_TRY(run_trunk(t, crops, H, W, ws, [&](int s, const float* x, int h, int w, int C) {
    return t.lateral(fw, s, x, h, w, C, L, f, f.means + (long)s * n_img * 512);
  }));
  return launch_fpn_head(fw, f.means, n_img, L, feats, t.timed, st);
}

// Test hook of the FPN head, through the code mmmot_appearance_resnet_fpn_fwd runs.  See include/mmmot_b200.h.
extern "C" int mmmot_debug_fpn_op(int op, const mmmot_fpn_weights* fw, int level, int n_img, int h, int w, int L,
                                  const void* X, float* Y, void* workspace, size_t workspace_bytes, void* stream) {
  if (op < 0 || op > 1 || !fpn_weights_ok(fw) || !X || !Y || n_img <= 0 || L <= 0 || n_img % L) return MMMOT_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (op == 1) return launch_fpn_head(fw, (const float*)X, n_img, L, Y, false, st);
  if (level < 0 || level > 3 || h <= 0 || w <= 0 || !workspace) return MMMOT_E_ARG;
  const int H = h << (level + 2), W = w << (level + 2);
  if ((long)n_img * (H / 2) * (W / 2) >= (1L << 31)) return MMMOT_E_SHAPE;
  MmArena ar(workspace, workspace_bytes);
  ResWs ws = carve_resnet(ar, n_img, H, W);
  FpnWs f = carve_fpn(ar, n_img, H, W, L);
  if (!ar.ok()) return MMMOT_E_WORKSPACE;
  Trunk t = make_trunk(nullptr, n_img, H, W, L, ws, ar.status(), st);
  t.tc = mm_engine() != 1;
  t.timed = false;
  return t.lateral(fw, level, (const float*)X, h, w, 256 << level, L, f, Y);
}

// Test hook: one launch kind of the ResNet trunk through the Trunk members mmmot_appearance_resnet_fwd calls, on the
// engine mmmot_set_engine selects (1 = FP32 engine, 0 or 2 = tensor cores).  See include/mmmot_b200.h.
extern "C" int mmmot_debug_resnet_op(int op, const mmmot_resnet_weights* rw, int conv, int n_img, int H, int W, int C,
                                     int ks, int stride, int M, int relu, int L, const void* X, const void* id, void* Y,
                                     void* cols, float* kseg, int* status, void* stream) {
  if (op < 0 || op > 7 || n_img <= 0 || H <= 0 || W <= 0 || !Y) return MMMOT_E_ARG;
  if (op != 5 && !X) return MMMOT_E_ARG;
  if ((op == 2 || op == 3 || op == 7) && !rw) return MMMOT_E_ARG;
  if ((op == 0 || op == 3) && (C <= 0 || C % 32 || (ks != 1 && ks != 3) || (stride != 1 && stride != 2) || H % stride ||
                               W % stride))
    return MMMOT_E_ARG;
  if (op == 3 && (conv < 0 || conv >= MMMOT_RESNET_MAX_CONVS || M <= 0 || M % 64 || !rw->bias[conv] || !rw->wp[conv] ||
                  !rw->wt[conv]))
    return MMMOT_E_ARG;
  if (op == 2 && (!rw->wt[0] || !rw->bias[0] || !rw->wp[0])) return MMMOT_E_ARG;
  if ((op == 2 || op == 3) && !cols) return MMMOT_E_ARG;
  if ((op == 1 || op == 2 || op == 4) && (H % 2 || W % 2)) return MMMOT_E_ARG;
  if (op == 4 && C != 64) return MMMOT_E_ARG;
  if (op == 5 && (!id || C <= 0 || ((long)n_img * H * W * C) % 8)) return MMMOT_E_ARG;
  if (op == 6 && (C <= 0 || C > 2048)) return MMMOT_E_ARG;
  if (op == 7 && (L <= 0 || n_img % L)) return MMMOT_E_ARG;
  Trunk t;
  t.rw = rw; t.n_img = n_img; t.tc = mm_engine() != 1; t.timed = false;
  t.cols = (float*)cols; t.kseg = kseg; t.status = status; t.st = (cudaStream_t)stream;
  const float* x = (const float*)X;
  float* y = (float*)Y;
  switch (op) {
    case 0: return t.gather(x, H, W, C, ks, stride, y);
    case 1: return t.stem_gather(x, H, W, y);
    case 2: return t.stem(x, H, W, y);
    case 3: return t.conv(conv, x, H, W, C, ks, stride, M, relu != 0, y);
    case 4: return t.maxpool(x, H, W, y);
    case 5: return t.add_relu(y, (const float*)id, (long)n_img * H * W * C);
    case 6: return t.mean(x, H, W, C, y);
    default: {
      float* pooled[4];
      float* base = const_cast<float*>(x);
      for (int s = 0; s < 4; s++) { pooled[s] = base; base += (long)n_img * (256 << s); }
      return launch_heads(rw, pooled, n_img, L, y, t.st);
    }
  }
}
