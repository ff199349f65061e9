// Library-wide entry points of libmmmot_sm90a.so (see include/mmmot_b200.h).
#include <algorithm>
#include <atomic>

#include "common.cuh"

static std::atomic<unsigned long long> g_launches{0};

void mm_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

extern "C" unsigned long long mmmot_launch_count(void) { return g_launches.load(); }

extern "C" int mmmot_abi_version(void) { return MMMOT_ABI_VERSION; }

int mm_sm_count(int* sms) {
  static std::atomic<int> cache[64];
  int dev = 0;
  MM_CUDA(cudaGetDevice(&dev));
  int v = cache[dev & 63].load(std::memory_order_relaxed);
  if (!v) {
    MM_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    cache[dev & 63].store(v, std::memory_order_relaxed);
  }
  *sms = v;
  return 0;
}

// ---- status block (first MM_STATUS_BYTES of every workspace) ----
extern "C" int mmmot_status_reset(void* workspace, void* stream) {
  if (!workspace) return MMMOT_E_ARG;
  MM_CUDA(cudaMemsetAsync(workspace, 0, MM_STATUS_BYTES, (cudaStream_t)stream));
  return 0;
}

extern "C" int mmmot_status_check(const void* workspace, void* stream) {
  if (!workspace) return MMMOT_E_ARG;
  int word = 0;
  MM_CUDA(cudaMemcpyAsync(&word, workspace, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  MM_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return (word & 1) ? MMMOT_E_RANGE : 0;
}

// ---- pinned-host fetch (see header): zero-copy read over PCIe by a kernel, stream-ordered ----
__global__ void fetch_pinned_i32_kernel(int* __restrict__ dst, const int* __restrict__ src, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) dst[i] = src[i];
}

extern "C" int mmmot_fetch_pinned_i32(int* dst_device, const int* src_pinned_host, long count, void* stream) {
  if (!dst_device || !src_pinned_host || count < 0) return MMMOT_E_ARG;
  if (count == 0) return 0;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, src_pinned_host) != cudaSuccess || at.type != cudaMemoryTypeHost || !at.devicePointer) {
    (void)cudaGetLastError();
    return MMMOT_E_ARG;     // pageable (unregistered) or device memory
  }
  const void* dsrc = at.devicePointer;
  const int blocks = (int)std::min<long>(mm_cdiv(count, 256), 32);
  fetch_pinned_i32_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(dst_device, (const int*)dsrc, count);
  MM_LAUNCH_CHECK();
  return 0;
}

extern "C" int mmmot_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  MM_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  MM_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Optional per-launch timing of the hot kernels, used by bench.py for the roofline figures: CUDA events recorded on
// the launching stream around every tagged launch while enabled; mmmot_timing_collect*() synchronises on the
// events and returns the totals (per tag = per (stage, layer)).
#include <mutex>
#include <vector>

namespace {
std::mutex g_tmu;
bool g_timing = false;
struct Span { cudaEvent_t a, b; int tag; double flop, bytes; };
std::vector<Span> g_spans;
const char* const kTagNames[MM_T_COUNT] = {
    "vgg.conv0", "vgg.conv1", "vgg.conv2", "vgg.conv3", "vgg.conv4", "vgg.conv5", "vgg.conv6", "vgg.conv7", "vgg.conv8",
    "vgg.conv9", "vgg.conv10", "vgg.conv11", "vgg.conv12", "vgg.pool_mean_heads",
    "pointnet.l1_3to64", "pointnet.l2_64to64", "pointnet.l3_64to64", "pointnet.l4_64to128", "pointnet.norm_split",
    "pointnet.l5_128to1024_stats", "pointnet.l5_128to1024_segsum", "pointnet.head_64to512_stats",
    "pointnet.head_64to512_segsum",
    "affinity.l1_pair_512to1024", "affinity.newend_means", "affinity.l2_512to512", "affinity.l3_512to128",
    "affinity.logit", "lp.assign", "pointnet.moments_128", "pointnet.moments_64",
    "pointnet.moments_finalize", "lp.flow"};
}  // namespace

bool mm_timing_on() { return g_timing; }

void mm_timing_begin(cudaStream_t st, int tag, double flop, double bytes) {
  std::lock_guard<std::mutex> l(g_tmu);
  Span s;
  cudaEventCreate(&s.a);
  cudaEventCreate(&s.b);
  s.tag = tag; s.flop = flop; s.bytes = bytes;
  cudaEventRecord(s.a, st);
  g_spans.push_back(s);
}

void mm_timing_end(cudaStream_t st) {
  std::lock_guard<std::mutex> l(g_tmu);
  if (!g_spans.empty()) cudaEventRecord(g_spans.back().b, st);
}

extern "C" int mmmot_timing_enable(int on) {
  std::lock_guard<std::mutex> l(g_tmu);
  g_timing = on != 0;
  return 0;
}

extern "C" int mmmot_timing_tag_count(void) { return MM_T_COUNT; }
extern "C" const char* mmmot_timing_tag_name(int tag) { return (tag >= 0 && tag < MM_T_COUNT) ? kTagNames[tag] : ""; }

// ms / flop / bytes / launches: arrays of mmmot_timing_tag_count() entries (any may be null)
extern "C" int mmmot_timing_collect_tags(double* ms, double* flop, double* bytes, long* launches) {
  std::lock_guard<std::mutex> l(g_tmu);
  for (int t = 0; t < MM_T_COUNT; t++) {
    if (ms) ms[t] = 0.0;
    if (flop) flop[t] = 0.0;
    if (bytes) bytes[t] = 0.0;
    if (launches) launches[t] = 0;
  }
  int rc = 0;
  for (auto& s : g_spans) {
    float t = 0.f;
    cudaError_t e = cudaEventSynchronize(s.b);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&t, s.a, s.b);
    if (e != cudaSuccess) rc = (int)e;
    else {
      if (ms) ms[s.tag] += t;
      if (flop) flop[s.tag] += s.flop;
      if (bytes) bytes[s.tag] += s.bytes;
      if (launches) launches[s.tag] += 1;
    }
    cudaEventDestroy(s.a);
    cudaEventDestroy(s.b);
  }
  g_spans.clear();
  return rc;
}

// totals over the 3x3-conv contractions of the VGG trunk (layers 1..12), the dominant kernels
extern "C" int mmmot_timing_collect(double* total_ms, double* total_flop, long* launches) {
  double ms[MM_T_COUNT], fl[MM_T_COUNT];
  long n[MM_T_COUNT];
  int rc = mmmot_timing_collect_tags(ms, fl, nullptr, n);
  if (rc) return rc;
  double a = 0.0, b = 0.0;
  long c = 0;
  for (int t = MM_T_VGG0 + 1; t <= MM_T_VGG0 + 12; t++) { a += ms[t]; b += fl[t]; c += n[t]; }
  if (total_ms) *total_ms = a;
  if (total_flop) *total_flop = b;
  if (launches) *launches = c;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Engine selection + single-contraction test hook.
#include "gemm_gen.cuh"

namespace { int g_engine = 0; int g_dbg = 0; int g_kseg = 36; }
int mm_kseg_chunks() { return g_kseg; }
extern "C" int mmmot_set_kseg(int chunks) { if (chunks < 0) return MMMOT_E_ARG; g_kseg = chunks; return 0; }
int mm_debug_flags() { return g_dbg; }
extern "C" int mmmot_set_debug(int flags) { g_dbg = flags; return 0; }

int mm_engine() { return g_engine; }

extern "C" int mmmot_set_engine(int engine) {
  if (engine < 0 || engine > 2) return MMMOT_E_ARG;
  g_engine = engine;
  return 0;
}

// One launch of the FP32 engine (gemm_simt.cuh) in any operand mode, with its GroupNorm partials, in the channel-major
// layout the PointNet, affinity, fusion and w_det stages give it, and every field the modes read: the pairwise
// generator's (n, m, Lf), the 3x3 convolution's (H, W, Cin) and the per-detection addend of the epilogue.
extern "C" int mmmot_debug_simt_op(int mode, int M, int K, const float* Wt, const float* bias, int relu, const float* X,
                                   long x_gs, long x_ks, const float* sc, const float* sh, int n, int m, int Lf, int H,
                                   int W, int Cin, int S, int groups, const void* tile_tab, int num_tiles,
                                   const float* addend, const int* seg, int ld_add, float* Y, long y_gs, long y_ms,
                                   void* part, void* stream) {
  if (mode < XM_DIRECT || mode > XM_CONV3 || M <= 0 || M % 64 || K <= 0 || !Wt || !X) return MMMOT_E_ARG;
  if (mode == XM_NORM_RELU && (!sc || !sh)) return MMMOT_E_ARG;
  if (addend && (!seg || ld_add <= 0)) return MMMOT_E_ARG;
  const bool pair = mode >= XM_PAIR_MUL && mode <= XM_PAIR_SUB;
  if (tile_tab) {
    if (num_tiles <= 0 || x_gs || y_gs || pair || mode == XM_CONV3) return MMMOT_E_ARG;
  } else if (S <= 0 || groups <= 0) {
    return MMMOT_E_ARG;
  }
  if (pair && (n <= 0 || m <= 0 || Lf < n + m || (long)n * m != S)) return MMMOT_E_ARG;
  if (mode == XM_CONV3 && (H <= 0 || W <= 0 || Cin <= 0 || K != 9 * Cin || groups != 1 || S % ((long)H * W) ||
                           x_gs || y_gs))
    return MMMOT_E_ARG;
  GemmP p = gemm_defaults();
  p.Wt = Wt; p.ldw = M; p.bias = bias; p.M = M; p.K = K; p.relu = relu;
  if (tile_tab) {
    p.tile_tab = (const int4*)tile_tab; p.num_tiles = num_tiles;
  } else {
    p.S = S; p.tiles_per_group = mm_cdiv(S, 128); p.num_tiles = p.tiles_per_group * groups;
  }
  p.X = X; p.x_gs = x_gs; p.x_ks = x_ks; p.sc = sc; p.sh = sh;
  p.n = n; p.m = m; p.Lf = Lf;
  p.H = H; p.W = W; p.Cin = Cin;
  p.addend = addend; p.seg = seg; p.ld_add = ld_add;
  p.Y = Y; p.y_gs = y_gs; p.y_ms = y_ms;
  p.part = (double2*)part;
  cudaStream_t st = (cudaStream_t)stream;
  switch (mode) {
    case XM_DIRECT: return gemm_simt_launch<XM_DIRECT>(p, st);
    case XM_NORM_RELU: return gemm_simt_launch<XM_NORM_RELU>(p, st);
    case XM_PAIR_MUL: return gemm_simt_launch<XM_PAIR_MUL>(p, st);
    case XM_PAIR_ABS: return gemm_simt_launch<XM_PAIR_ABS>(p, st);
    case XM_PAIR_SUB: return gemm_simt_launch<XM_PAIR_SUB>(p, st);
    default: return gemm_simt_launch<XM_CONV3>(p, st);
  }
}

// The producer variant gemm_gen_launch takes (1 = prefetching), computed on the host without any CUDA call.
extern "C" int mmmot_debug_gen_prefetch(int gen, int m) {
  if (gen < gen::GEN_PAIR_MUL || gen > gen::GEN_COPY) return MMMOT_E_ARG;
  return gen_prefetch(gen, m, mm_debug_flags()) ? 1 : 0;
}

// Whether that variant stages the pairwise sources in shared memory by TMA (1) or not, on the host, no CUDA call.
extern "C" int mmmot_debug_gen_staged(int gen, int m) {
  if (gen < gen::GEN_PAIR_MUL || gen > gen::GEN_COPY) return MMMOT_E_ARG;
  return gen_staged(gen, m, mm_debug_flags()) ? 1 : 0;
}

// One contraction of the generated-operand tensor-core engine (gemm_gen.cuh) through gemm_gen_launch, with the
// arguments the affinity, PointNet and fusion stages pass it.
extern "C" int mmmot_debug_gen(int gen, int M, int K, const void* Wp, float wp_scale, const float* bias, int relu,
                               const float* src, int ld_src, const float* gsc, const float* gsh, int n, int m, int Lf, int S,
                               int groups, long x_gs, long y_gs, const void* tile_tab, int num_tiles, float* Y, long y_ms,
                               void* part, int* prefetched, void* stream) {
  if (M <= 0 || K <= 0) return MMMOT_E_ARG;
  GemmP p = gemm_defaults();
  p.bias = bias; p.M = M; p.K = K; p.relu = relu;
  if (tile_tab) {
    if (num_tiles <= 0) return MMMOT_E_ARG;
    p.tile_tab = (const int4*)tile_tab; p.num_tiles = num_tiles;
  } else {
    if (S <= 0 || groups <= 0) return MMMOT_E_ARG;
    p.S = S; p.tiles_per_group = mm_cdiv(S, tc::BN); p.num_tiles = p.tiles_per_group * groups;
    p.x_gs = x_gs; p.y_gs = y_gs;
  }
  p.Y = Y; p.y_ms = y_ms;
  p.part = (double2*)part;
  const uint4* w = (const uint4*)Wp;
  cudaStream_t st = (cudaStream_t)stream;
  switch (gen) {
    case gen::GEN_PAIR_MUL: return gemm_gen_launch<gen::GEN_PAIR_MUL>(p, w, wp_scale, src, ld_src, gsc, gsh, n, m, Lf, st, prefetched);
    case gen::GEN_PAIR_ABS: return gemm_gen_launch<gen::GEN_PAIR_ABS>(p, w, wp_scale, src, ld_src, gsc, gsh, n, m, Lf, st, prefetched);
    case gen::GEN_PAIR_SUB: return gemm_gen_launch<gen::GEN_PAIR_SUB>(p, w, wp_scale, src, ld_src, gsc, gsh, n, m, Lf, st, prefetched);
    case gen::GEN_NORM: return gemm_gen_launch<gen::GEN_NORM>(p, w, wp_scale, src, ld_src, gsc, gsh, n, m, Lf, st, prefetched);
    case gen::GEN_COPY: return gemm_gen_launch<gen::GEN_COPY>(p, w, wp_scale, src, ld_src, gsc, gsh, n, m, Lf, st, prefetched);
    default: return MMMOT_E_ARG;
  }
}

// ---------------------------------------------------------------------------------------------
// Test hooks for the TMA-fed tensor-core engine (planar FP16 hi/lo channels-last operands).
// Y[rows][M] fp32 (channels-last) = X W^T + bias ; X given as planes Xhi[rows][K], Xlo = Xhi + rows*K
extern "C" int mmmot_debug_linear_planar(const void* Wp, float wp_scale, const float* bias, const void* Xhi,
                                         float* Y, int M, int K, long rows, void* stream) {
  if (!Wp || !Xhi || !Y || M <= 0 || K <= 0 || rows <= 0) return MMMOT_E_ARG;
  GemmP p = gemm_defaults();
  p.bias = bias; p.M = M; p.K = K;
  p.S = (int)rows; p.tiles_per_group = mm_cdiv(rows, tc::BN); p.num_tiles = p.tiles_per_group;
  p.Y = Y; p.y_ms = M;
  return gemm_tma_launch_mat(p, (const uint4*)Wp, wp_scale, (const __half*)Xhi, rows * (long)K, rows, K, tc::OUT_CL, 0,
                             (cudaStream_t)stream);
}

static void conv_plan_words(const ConvPlan& c, int* plan) {
  const int v[8] = {c.px, c.halo, c.pool, c.bx, c.by, c.bi, c.ksegs, c.num_tiles};
  for (int i = 0; i < 8; i++) plan[i] = v[i];
}

// The launch plan gemm_tma_launch_conv takes for one VGG layer, computed on the host without any CUDA call.
extern "C" int mmmot_debug_conv_plan(int n_img, int H, int W, int C, int M, int want_pool, int use_kseg, int* plan) {
  if (!plan || n_img <= 0 || H <= 0 || W <= 0 || C <= 0 || C % tc::BK || M <= 0) return MMMOT_E_ARG;
  conv_plan_words(conv_plan(M, false, n_img, H, W, C, want_pool != 0, use_kseg != 0, mm_debug_flags(), mm_kseg_chunks()),
                  plan);
  return 0;
}

// One VGG conv layer (3x3 pad 1 + bias + ReLU) through gemm_tma_launch_conv with the arguments mmmot_appearance_fwd
// passes it.
extern "C" int mmmot_debug_conv_layer(const void* Wp, const void* Wpx, float wp_scale, const float* bias, const void* Xhi,
                                      long x_plane, int n_img, int H, int W, int C, int M, void* Yhi, long y_plane,
                                      long y_plane_pooled, int* did_pool, unsigned long long* pool_sum, float* kseg_scratch,
                                      int* status, int* plan, void* stream) {
  if (!Wp || !bias || !Xhi || !Yhi || n_img <= 0 || H <= 0 || W <= 0 || M <= 0) return MMMOT_E_ARG;
  GemmP p = gemm_defaults();
  p.bias = bias; p.M = M; p.relu = 1;
  ConvPlan c;
  const int rc = gemm_tma_launch_conv(p, (const uint4*)Wp, wp_scale, (const __half*)Xhi, x_plane, n_img, H, W, C,
                                      (__half*)Yhi, y_plane, (cudaStream_t)stream, kseg_scratch, y_plane_pooled, did_pool,
                                      status, pool_sum, (const uint4*)Wpx, &c);
  if (plan && rc != MMMOT_E_ARG) conv_plan_words(c, plan);
  return rc;
}

// ---------------------------------------------------------------------------------------------
// Where the affinity (stage 0), fusion / detection-score (stage 1) and PointNet (stage 2) stages leave their
// intermediates, on the host.
int mm_affinity_layout(int pairs, int n, int m, size_t* off, int* tensor_cores);
int mm_fusion_det_layout(int pairs, int L, size_t* off, int* tensor_cores);
int mm_pointnet_layout(int pairs, int L, long P, size_t* off, int* tensor_cores);

extern "C" int mmmot_debug_stage_layout(int stage, int pairs, int n, int m, size_t* offsets, int* tensor_cores) {
  if (!offsets || pairs <= 0 || n <= 0) return MMMOT_E_ARG;
  if (stage == 0) return m <= 0 ? MMMOT_E_ARG : mm_affinity_layout(pairs, n, m, offsets, tensor_cores);
  if (stage == 1) return mm_fusion_det_layout(pairs, n, offsets, tensor_cores);
  if (stage == 2) return m <= 0 ? MMMOT_E_ARG : mm_pointnet_layout(pairs, n, m, offsets, tensor_cores);
  return MMMOT_E_ARG;
}
