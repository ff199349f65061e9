// Exact solver for the association programme of samples of K >= 2 frames.
// Replaces reference solvers.py:9-138 (ortools_solve) for any len(det_split); csrc/lp_assign.cu keeps K = 2.
//
// Multiplying each "new + predecessors = det" row (solvers.py:103-109) by -1 leaves every variable with at most one +1
// and one -1 in the constraint matrix: a network matrix, so LP = MIP and the programme is a min-cost flow.
//   nodes  S, T, and per detection d an in_d and an out_d;   every arc has capacity 1 and cost -score:
//   S -> in_d (new_d)   in_d -> out_d (det_d)   out_d -> T (end_d)   out_j -> in_k, j in frame f, k in f + 1 (link_f[j][k])
// The optimum is the minimum-cost flow of free value.  Frame 0's new = det and the last frame's end = det
// (solvers.py:99-101, 110-111) hold because those nodes have no other inflow / outflow.
//
// Successive shortest paths in fp64, one WARP per sample, all state in shared memory.  Initial potentials are the
// shortest-path distances of the (acyclic) network, swept frame by frame.  Each augmentation is a dense Dijkstra on
// reduced costs (warp arg-min over the unsettled nodes), stopped when T is settled; potentials then move by
// min(d(v), d(T)), so the new pi(T) is the cost of the path found, and the path is augmented only if that cost is
// strictly below 0.  Node throughput is 1, so the flow is three per-detection arrays (successor, predecessor, on) and
// the residual arcs are implicit.  Deterministic: equal distances settle the smaller node index first (T = node 1,
// so it wins every tie), a relaxation must improve strictly, and a path of profit exactly 0 is not augmented.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kMaxFrames = 64;
constexpr int kMaxWarpsPerCta = 4;
constexpr size_t kSmemCap = 227 * 1024;
// pred[d]: local index of the linked previous-frame detection, kNone or kNew (S -> in_d carries flow);
// succ[d]: local index in the next frame, kNone or kEnd (out_d -> T carries flow)
constexpr int kNone = -1, kNew = -2, kEnd = -2;
constexpr int kS = 0, kT = 1;
__device__ __forceinline__ int node_in(int d) { return 2 + 2 * d; }
__device__ __forceinline__ int node_out(int d) { return 3 + 2 * d; }

struct FlowShape {
  int frames, L;
  int off[kMaxFrames + 1];  // first detection of each frame in the sample; off[frames] = L
  long loff[kMaxFrames];    // first element of link matrix f in a sample's links; loff[frames - 1] = all link elements
};

__host__ __device__ inline size_t flow_warp_bytes(long L) {
  size_t V = 2 * (size_t)L + 2;
  size_t b = V * 2 * sizeof(double)   // pi, dist
             + V * sizeof(int)        // parent
             + (size_t)L * 2 * sizeof(int)  // pred, succ
             + (size_t)L * 2 + V;     // frame of each detection, on, settled
  return (b + 15) / 16 * 16;
}

__global__ void __launch_bounds__(kMaxWarpsPerCta * 32) flow_assign_kernel(
    const float* __restrict__ det, long det_stride, const float* __restrict__ links, long links_stride,
    const float* __restrict__ new_s, long new_stride, const float* __restrict__ end_s, long end_stride,
    int samples, int warps_per_cta, const __grid_constant__ FlowShape sh, float* __restrict__ a_det,
    float* __restrict__ a_links, float* __restrict__ a_new, float* __restrict__ a_end, int* __restrict__ match) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sample = blockIdx.x * warps_per_cta + warp;
  if (warp >= warps_per_cta || sample >= samples) return;
  const int K = sh.frames, L = sh.L, V = 2 * L + 2;
  unsigned char* base = smem + (size_t)warp * flow_warp_bytes(L);
  double* pi = (double*)base;
  double* dist = pi + V;
  int* par = (int*)(dist + V);
  int* pred = par + V;
  int* succ = pred + L;
  unsigned char* fr = (unsigned char*)(succ + L);
  unsigned char* on = fr + L;
  unsigned char* settled = on + L;

  const float* ds = det + (long)sample * det_stride;
  const float* ns = new_s + (long)sample * new_stride;
  const float* es = end_s + (long)sample * end_stride;
  const float* lk = links + (long)sample * links_stride;
  const double INF = INFINITY;

  for (int f = 0; f < K; f++)
    for (int i = sh.off[f] + lane; i < sh.off[f + 1]; i += 32) { fr[i] = (unsigned char)f; pred[i] = succ[i] = kNone; on[i] = 0; }
  // initial potentials: shortest distances from S over the acyclic network, frame by frame
  if (lane == 0) pi[kS] = 0.0;
  for (int f = 0; f < K; f++) {
    const int o = sh.off[f], nf = sh.off[f + 1] - o;
    for (int k = lane; k < nf; k += 32) {
      double m = -(double)ns[o + k];
      if (f > 0) {
        const int po = sh.off[f - 1];
        const float* col = lk + sh.loff[f - 1] + k;
        for (int j = 0; j < o - po; j++) m = fmin(m, pi[node_out(po + j)] - (double)col[(long)j * nf]);
      }
      pi[node_in(o + k)] = m;
      pi[node_out(o + k)] = m - (double)ds[o + k];
    }
    __syncwarp();   // frame f + 1 reads frame f's out potentials from other lanes
  }
  {
    double m = INF;
    for (int i = lane; i < L; i += 32) m = fmin(m, pi[node_out(i)] - (double)es[i]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) pi[kT] = m;
  }
  __syncwarp();

  // every augmentation raises the flow value by one and S has L unit arcs: at most L of them
  for (int aug = 0; aug < L; aug++) {
    for (int v = lane; v < V; v += 32) { dist[v] = INF; par[v] = -1; settled[v] = 0; }
    __syncwarp();
    if (lane == 0) dist[kS] = 0.0;
    __syncwarp();
    bool reached = false;
    // every pass settles one more node, so V passes bound the search
    for (int pass = 0; pass < V; pass++) {
      double best = INF;
      int bu = 0x7fffffff;
      for (int v = lane; v < V; v += 32)
        if (!settled[v] && dist[v] < best) { best = dist[v]; bu = v; }   // ascending v per lane: first minimum kept
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        double ob = __shfl_xor_sync(0xffffffffu, best, o);
        int ov = __shfl_xor_sync(0xffffffffu, bu, o);
        if (ob < best || (ob == best && ov < bu)) { best = ob; bu = ov; }
      }
      if (bu == 0x7fffffff) break;   // nothing left that S reaches
      // every lane has scanned dist[] / settled[] before the relaxations below write them from other lanes
      __syncwarp();
      const int u = bu;
      const double du = best, pu = pi[u];
      if (lane == 0) settled[u] = 1;
      if (u == kT) { reached = true; break; }
      // reduced cost c + pi(u) - pi(v) is >= 0 in exact arithmetic; fp64 rounding can leave it at -eps, clamped to 0
      auto relax = [&](int v, double c) {
        if (settled[v]) return;
        const double nd = du + fmax(c + pu - pi[v], 0.0);
        if (nd < dist[v]) { dist[v] = nd; par[v] = u; }
      };
      if (u == kS) {
        for (int i = lane; i < L; i += 32)
          if (pred[i] != kNew) relax(node_in(i), -(double)ns[i]);
      } else if (!(u & 1)) {   // in_i: its one residual arc other than the way back to S
        const int i = (u - 2) >> 1;
        if (lane == 0) {
          if (!on[i]) {
            relax(node_out(i), -(double)ds[i]);
          } else if (pred[i] >= 0) {
            const int f = fr[i], nf = sh.off[f + 1] - sh.off[f];
            relax(node_out(sh.off[f - 1] + pred[i]), (double)lk[sh.loff[f - 1] + (long)pred[i] * nf + (i - sh.off[f])]);
          }
        }
      } else {                 // out_i: T, back to in_i, and the next frame's row of links
        const int i = (u - 3) >> 1, f = fr[i];
        if (lane == 0) {
          if (succ[i] != kEnd) relax(kT, -(double)es[i]);
          if (on[i]) relax(node_in(i), (double)ds[i]);
        }
        if (f + 1 < K) {
          const int o1 = sh.off[f + 1], n1 = sh.off[f + 2] - o1;
          const float* lrow = lk + sh.loff[f] + (long)(i - sh.off[f]) * n1;
          for (int k = lane; k < n1; k += 32)
            if (k != succ[i]) relax(node_in(o1 + k), -(double)lrow[k]);
        }
      }
      __syncwarp();
    }
    if (!reached) break;
    const double D = dist[kT];
    for (int v = lane; v < V; v += 32) pi[v] += fmin(dist[v], D);
    __syncwarp();
    if (!(pi[kT] < 0.0)) break;   // the cheapest S -> T path has profit <= 0
    // augment along the path (serial, at most V arcs); a link is cleared only if it is still the one the arc removes,
    // so the arcs may be applied in any order
    if (lane == 0) {
      int v = kT;
      for (int step = 0; step < V && v != kS; step++) {
        const int p = par[v];
        if (p == kS) {
          pred[(v - 2) >> 1] = kNew;
        } else if (v == kT) {
          succ[(p - 2) >> 1] = kEnd;
        } else {
          const int a = (p - 2) >> 1, b = (v - 2) >> 1;
          const int la = a - sh.off[fr[a]], lb = b - sh.off[fr[b]];
          if (a == b) on[a] = (p & 1) ? 0 : 1;                      // in -> out adds the detection, out -> in removes it
          else if (p & 1) { succ[a] = lb; pred[b] = la; }             // out_a -> in_b adds link a -> b
          else { if (succ[b] == la) succ[b] = kNone; if (pred[a] == lb) pred[a] = kNone; }   // in_a -> out_b removes b -> a
        }
        v = p;
      }
    }
    __syncwarp();
  }

  // ---- the 0/1 solution in ortools_solve's layout (solvers.py:115-138), links packed frame pair by frame pair ----
  const int nl = L - (sh.off[K] - sh.off[K - 1]);
  float* od = a_det + (long)sample * L;
  float* on_ = a_new + (long)sample * L;
  float* oe = a_end + (long)sample * L;
  float* ol = a_links + (long)sample * sh.loff[K - 1];
  int* om = match + (long)sample * nl;
  for (int i = lane; i < L; i += 32) {
    od[i] = on[i] ? 1.f : 0.f;
    on_[i] = pred[i] == kNew ? 1.f : 0.f;
    oe[i] = succ[i] == kEnd ? 1.f : 0.f;
    if (i < nl) {
      const int s = succ[i], f = fr[i];
      om[i] = s >= 0 ? s : -1;
      if (s >= 0) ol[sh.loff[f] + (long)(i - sh.off[f]) * (sh.off[f + 2] - sh.off[f + 1]) + s] = 1.f;
    }
  }
}

}  // namespace

extern "C" size_t mmmot_flow_workspace(int samples, int frames, const int* counts) {
  (void)samples; (void)frames; (void)counts;
  return 256;  // all solver state lives in shared memory; kept non-zero so callers can always pass a buffer
}

extern "C" int mmmot_flow_assign(const float* det, long det_stride, const float* links, long links_stride,
                                 const float* new_s, long new_stride, const float* end_s, long end_stride, int samples,
                                 int frames, const int* counts, float* a_det, float* a_links, float* a_new,
                                 float* a_end, int* match, void* workspace, size_t workspace_bytes, void* stream) {
  (void)workspace; (void)workspace_bytes;
  if (!det || !links || !new_s || !end_s || !counts || !a_det || !a_links || !a_new || !a_end || !match)
    return MMMOT_E_ARG;
  if (samples <= 0 || frames < 2) return MMMOT_E_ARG;
  long L = 0;   // every count is checked before any shape limit: a bad count is MMMOT_E_ARG whatever the shape
  for (int f = 0; f < frames; f++) {
    if (counts[f] <= 0) return MMMOT_E_ARG;
    L += counts[f];
  }
  if (frames > kMaxFrames || flow_warp_bytes(L) > kSmemCap) return MMMOT_E_SHAPE;
  FlowShape sh;
  sh.frames = frames;
  long nlink = 0;
  L = 0;
  for (int f = 0; f < frames; f++) {
    sh.off[f] = (int)L;
    sh.loff[f] = nlink;
    L += counts[f];
    if (f + 1 < frames) nlink += (long)counts[f] * counts[f + 1];
  }
  sh.off[frames] = (int)L;
  sh.loff[frames - 1] = nlink;
  sh.L = (int)L;
  const size_t wb = flow_warp_bytes(sh.L);
  const int wpc = (int)(kSmemCap / wb < (size_t)kMaxWarpsPerCta ? kSmemCap / wb : kMaxWarpsPerCta);
  const size_t smem = wb * wpc;
  cudaStream_t st = (cudaStream_t)stream;
  MM_CUDA(cudaFuncSetAttribute(flow_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // size varies: set per call
  MM_CUDA(cudaMemsetAsync(a_links, 0, (size_t)samples * nlink * sizeof(float), st));
  const bool timed = mm_timing_on();
  if (timed) mm_timing_begin(st, MM_T_FLOW, 0.0, 4.0 * samples * ((double)nlink * 2 + 7.0 * L));
  flow_assign_kernel<<<mm_cdiv(samples, wpc), wpc * 32, smem, st>>>(det, det_stride, links, links_stride, new_s,
                                                                     new_stride, end_s, end_stride, samples, wpc, sh,
                                                                     a_det, a_links, a_new, a_end, match);
  MM_LAUNCH_CHECK();
  if (timed) mm_timing_end(st);
  return 0;
}
