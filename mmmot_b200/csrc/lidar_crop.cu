// Per-detection LiDAR preparation on the GPU (SURVEY.md §8f row N1: the step immediately before the hot path).
// Replaces the per-box host loops of reference point_cloud/preprocess.py:64-93: the camera field-of-view cull
// (box_np_ops.remove_outside_points), then per detection either its rotated 3-D box (remove_points_outside_boxes ->
// box_np_ops.points_in_rbbox) or the view frustum of its 2-D image box (box_np_ops.get_frustum_points); every one
// ends in geometry._points_in_convex_polygon_3d_jit (geometry.py:96-114).
//
// Every region (field of view, 3-D box, 2-D frustum) is six inward-facing plane equations prepared on the host
// exactly as the reference's numpy code computes them (mmmot_b200/lidar_crop.py); the kernels evaluate the
// reference's membership predicate  sign = x*nx + y*ny + z*nz + d ; inside <=> sign < 0 for all 6 planes  with the
// same operation order and NO fused multiply-add, in the precision of the plane equations: float64 in the
// reference's real pipeline (camera_to_lidar promotes every plane set to float64, box_np_ops.py:584-589, so numba
// evaluates the predicate in float64 on the float32 points), float32 when the caller hands float32 boxes to
// mmmot_crop_*.  Membership is bit-identical to the reference in both cases.
// Output = the packed per-detection point list + CSR offsets that mmmot_pointnet_fwd consumes; point order inside
// a detection is the scan order (stable compaction); an empty detection yields one all-zero point
// (preprocess.py:78-79, 89-90).  Several frames go through one call: detections are grouped by frame, a detection
// only sees its own frame's points, and the offsets are global.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;              // threads per CTA
constexpr int kRounds = 4;                 // points per thread
constexpr int kTile = kThreads * kRounds;  // points per CTA: one count per (detection, tile)
constexpr int kSlots = kTile / 32;         // warp-sized slots of a tile, slot s = round * 8 + warp, in scan order
constexpr int kChunk = 64;                 // detections whose planes sit in shared memory at once

__device__ __forceinline__ bool inside_box(const float* __restrict__ pl, float x, float y, float z) {
  // pl: 6 planes x (nx, ny, nz, d)
#pragma unroll
  for (int k = 0; k < 6; k++) {
    float s = __fadd_rn(__fmul_rn(x, pl[4 * k]), __fmul_rn(y, pl[4 * k + 1]));
    s = __fadd_rn(s, __fmul_rn(z, pl[4 * k + 2]));
    s = __fadd_rn(s, pl[4 * k + 3]);
    if (s >= 0.f) return false;
  }
  return true;
}
__device__ __forceinline__ bool inside_box(const double* __restrict__ pl, float xf, float yf, float zf) {
  const double x = xf, y = yf, z = zf;
#pragma unroll
  for (int k = 0; k < 6; k++) {
    double s = __dadd_rn(__dmul_rn(x, pl[4 * k]), __dmul_rn(y, pl[4 * k + 1]));
    s = __dadd_rn(s, __dmul_rn(z, pl[4 * k + 2]));
    s = __dadd_rn(s, pl[4 * k + 3]);
    if (s >= 0.0) return false;
  }
  return true;
}

// first index i in [0, n) with a[i] >= key (a non-decreasing), n if none
__device__ __forceinline__ int lower_bound(const int* __restrict__ a, int n, int key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One CTA per (tile of kTile points, frame).  It loads its points once, tests the frame's field of view once per
// point (FOV), then tests the points that passed against every detection of the frame, kChunk detections at a time
// from shared memory, keeping one ballot per (detection, slot).  A slot whose points all failed skips the detections.
//   count   (!SCATTER): counts[d][tile] = points of the tile inside detection d
//   scatter ( SCATTER): counts holds the exclusive per-detection tile offsets; each inside point goes to
//                       split[d] + counts[d][tile] + (inside points of d before it in the tile)
template <typename T, bool FOV, bool SCATTER>
__global__ void __launch_bounds__(kThreads, 4) crop_tile_kernel(const float* __restrict__ pts, int stride,
                                                             const int* __restrict__ frame_off,
                                                             const double* __restrict__ fov_planes,
                                                             const T* __restrict__ planes,
                                                             const int* __restrict__ det_frame, int n_det,
                                                             int max_tiles, int* __restrict__ counts,
                                                             const int* __restrict__ split, int out_c,
                                                             float* __restrict__ out) {
  __shared__ T pl[kChunk * 24];
  __shared__ double fpl[24];
  __shared__ unsigned bal[kChunk][kSlots];
  __shared__ int pre[SCATTER ? kChunk : 1][kSlots];
  const int f = blockIdx.y, tile = blockIdx.x;
  const int p0 = frame_off[f], P = frame_off[f + 1] - p0;
  if (tile * kTile >= P) return;                                   // uniform: the frame has fewer tiles
  const int d0 = lower_bound(det_frame, n_det, f), d1 = lower_bound(det_frame, n_det, f + 1);
  if (d0 == d1) return;
  if (FOV && threadIdx.x < 24) fpl[threadIdx.x] = fov_planes[f * 24 + threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nch = SCATTER ? out_c : 3;
  float v[kRounds][4];
  bool ok[kRounds];
  unsigned any[kRounds];
#pragma unroll
  for (int r = 0; r < kRounds; r++) {
    const int p = tile * kTile + r * kThreads + threadIdx.x;
    ok[r] = p < P;
    const float* src = pts + (long)(p0 + (ok[r] ? p : 0)) * stride;
#pragma unroll
    for (int c = 0; c < 4; c++) v[r][c] = (ok[r] && c < nch) ? src[c] : 0.f;
    if (FOV && ok[r]) ok[r] = inside_box(fpl, v[r][0], v[r][1], v[r][2]);
    any[r] = __ballot_sync(0xffffffffu, ok[r]);
  }
  for (int c0 = d0; c0 < d1; c0 += kChunk) {
    const int nc = min(kChunk, d1 - c0);
    __syncthreads();                                               // the previous chunk's shared data is consumed
    for (int i = threadIdx.x; i < nc * 24; i += kThreads) pl[i] = planes[(long)c0 * 24 + i];
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kRounds; r++) {
      const int s = r * (kThreads / 32) + warp;
      for (int j = 0; j < nc; j++) {
        unsigned b = 0;
        if (any[r]) b = __ballot_sync(0xffffffffu, ok[r] && inside_box(pl + 24 * j, v[r][0], v[r][1], v[r][2]));
        if (lane == 0) bal[j][s] = b;
      }
    }
    __syncthreads();
    if constexpr (!SCATTER) {
      if (threadIdx.x < nc) {
        int c = 0;
#pragma unroll
        for (int s = 0; s < kSlots; s++) c += __popc(bal[threadIdx.x][s]);
        counts[(long)(c0 + threadIdx.x) * max_tiles + tile] = c;
      }
    } else {
      if (threadIdx.x < nc) {
        int a = 0;
#pragma unroll
        for (int s = 0; s < kSlots; s++) {
          pre[threadIdx.x][s] = a;
          a += __popc(bal[threadIdx.x][s]);
        }
      }
      __syncthreads();
#pragma unroll
      for (int r = 0; r < kRounds; r++) {
        if (!any[r]) continue;
        const int s = r * (kThreads / 32) + warp;
        for (int j = 0; j < nc; j++) {
          const unsigned b = bal[j][s];
          if (!((b >> lane) & 1u)) continue;
          const int d = c0 + j;
          const long dst = (long)split[d] + counts[(long)d * max_tiles + tile] + pre[j][s] + __popc(b & ((1u << lane) - 1u));
#pragma unroll
          for (int c = 0; c < 4; c++)
            if (c < out_c) out[dst * out_c + c] = v[r][c];
        }
      }
    }
  }
}

// per detection: exclusive scan of its frame's tile counts (in place) + total; one CTA per detection
__global__ void __launch_bounds__(256) crop_scan_tiles_kernel(int* __restrict__ counts, int max_tiles,
                                                              const int* __restrict__ frame_off,
                                                              const int* __restrict__ det_frame,
                                                              int* __restrict__ totals) {
  __shared__ int carry;
  __shared__ int wsum[8];
  const int b = blockIdx.x, f = det_frame[b];
  const int tiles = (frame_off[f + 1] - frame_off[f] + kTile - 1) / kTile;
  int* row = counts + (long)b * max_tiles;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int t0 = 0; t0 < tiles; t0 += 256) {
    const int t = t0 + threadIdx.x;
    const int v = t < tiles ? row[t] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = x;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < (threadIdx.x >> 5); w++) woff += wsum[w];
    const int incl = x + woff + carry;
    if (t < tiles) row[t] = incl - v;
    __syncthreads();
    if (threadIdx.x == 255) carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[b] = carry;
}

// split[0] = 0, split[b+1] = split[b] + max(total_b, 1) (an empty detection keeps one zero point); one CTA
__global__ void __launch_bounds__(1024) crop_scan_dets_kernel(const int* __restrict__ totals, int n,
                                                              int* __restrict__ split) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    carry = 0;
    split[0] = 0;
  }
  __syncthreads();
  for (int b0 = 0; b0 < n; b0 += 1024) {
    const int b = b0 + threadIdx.x;
    const int v = b < n ? max(totals[b], 1) : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    const int incl = x + (warp ? wsum[warp - 1] : 0) + carry;
    if (b < n) split[b + 1] = incl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
}

// detections with no point inside: one all-zero point
__global__ void crop_fill_empty_kernel(const int* __restrict__ totals, const int* __restrict__ split, int n,
                                       int out_c, float* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n || totals[b] > 0) return;
  for (int c = 0; c < out_c; c++) out[(long)split[b] * out_c + c] = 0.f;
}

// Workspace: counts [n_det][max_tiles] | totals [n_det] | frame_off [n_frames + 1] | det_frame [n_det]
struct Ws {
  int *counts, *totals, *frame_off, *det_frame;
};
size_t ws_bytes(int max_tiles, int n_frames, int n_det) {
  return mm_align((size_t)max_tiles * n_det * sizeof(int)) + mm_align((size_t)n_det * sizeof(int)) +
         mm_align((size_t)(n_frames + 1) * sizeof(int)) + mm_align((size_t)n_det * sizeof(int));
}
Ws ws_carve(void* w, int max_tiles, int n_frames, int n_det) {
  char* p = (char*)w;
  Ws r;
  r.counts = (int*)p;
  p += mm_align((size_t)max_tiles * n_det * sizeof(int));
  r.totals = (int*)p;
  p += mm_align((size_t)n_det * sizeof(int));
  r.frame_off = (int*)p;
  p += mm_align((size_t)(n_frames + 1) * sizeof(int));
  r.det_frame = (int*)p;
  return r;
}

// Host-side validation shared by every entry point: frame offsets start at 0 and never decrease, detections are
// grouped by frame in frame order.  Returns the tile count of the largest frame, or MMMOT_E_ARG.
int check_frames(const int* frame_off, int n_frames, const int* det_frame, int n_det) {
  if (!frame_off || n_frames <= 0 || n_det <= 0 || frame_off[0] != 0) return MMMOT_E_ARG;
  int max_p = 0;
  for (int f = 0; f < n_frames; f++) {
    if (frame_off[f + 1] < frame_off[f]) return MMMOT_E_ARG;
    max_p = std::max(max_p, frame_off[f + 1] - frame_off[f]);
  }
  if (max_p <= 0) return MMMOT_E_ARG;
  if (det_frame)
    for (int d = 0; d < n_det; d++)
      if (det_frame[d] < 0 || det_frame[d] >= n_frames || (d && det_frame[d] < det_frame[d - 1])) return MMMOT_E_ARG;
  return mm_cdiv(max_p, kTile);
}

// count phase: per-(detection, tile) counts -> per-detection tile offsets and totals -> split.  det_frame == NULL
// means every detection belongs to frame 0.  Uploads the frame table into the workspace for the scatter phase.
template <typename T, bool FOV>
int crop_count(const float* pts, int stride, const int* frame_off, int n_frames, const double* fov, const T* planes,
               const int* det_frame, int n_det, int* split, void* workspace, size_t workspace_bytes,
               cudaStream_t st) {
  const int max_tiles = check_frames(frame_off, n_frames, det_frame, n_det);
  if (max_tiles < 0) return max_tiles;
  if (workspace_bytes < ws_bytes(max_tiles, n_frames, n_det)) return MMMOT_E_WORKSPACE;
  const Ws w = ws_carve(workspace, max_tiles, n_frames, n_det);
  MM_CUDA(cudaMemcpyAsync(w.frame_off, frame_off, (n_frames + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
  if (det_frame)
    MM_CUDA(cudaMemcpyAsync(w.det_frame, det_frame, n_det * sizeof(int), cudaMemcpyHostToDevice, st));
  else
    MM_CUDA(cudaMemsetAsync(w.det_frame, 0, n_det * sizeof(int), st));
  crop_tile_kernel<T, FOV, false><<<dim3(max_tiles, n_frames), kThreads, 0, st>>>(
      pts, stride, w.frame_off, fov, planes, w.det_frame, n_det, max_tiles, w.counts, nullptr, 0, nullptr);
  MM_LAUNCH_CHECK();
  crop_scan_tiles_kernel<<<n_det, 256, 0, st>>>(w.counts, max_tiles, w.frame_off, w.det_frame, w.totals);
  MM_LAUNCH_CHECK();
  crop_scan_dets_kernel<<<1, 1024, 0, st>>>(w.totals, n_det, split);
  MM_LAUNCH_CHECK();
  return 0;
}

// scatter phase: consumes the workspace the count phase filled (same arguments)
template <typename T, bool FOV>
int crop_scatter(const float* pts, int stride, const int* frame_off, int n_frames, const double* fov, const T* planes,
                 const int* det_frame, int n_det, const int* split, int out_c, float* out, void* workspace,
                 size_t workspace_bytes, cudaStream_t st) {
  const int max_tiles = check_frames(frame_off, n_frames, det_frame, n_det);
  if (max_tiles < 0) return max_tiles;
  if (out_c < 3 || out_c > 4 || out_c > stride) return MMMOT_E_ARG;
  if (workspace_bytes < ws_bytes(max_tiles, n_frames, n_det)) return MMMOT_E_WORKSPACE;
  const Ws w = ws_carve(workspace, max_tiles, n_frames, n_det);
  crop_tile_kernel<T, FOV, true><<<dim3(max_tiles, n_frames), kThreads, 0, st>>>(
      pts, stride, w.frame_off, fov, planes, w.det_frame, n_det, max_tiles, w.counts, split, out_c, out);
  MM_LAUNCH_CHECK();
  crop_fill_empty_kernel<<<mm_cdiv(n_det, 128), 128, 0, st>>>(w.totals, split, n_det, out_c, out);
  MM_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" size_t mmmot_crop_workspace(int n_points, int n_boxes) {
  if (n_points <= 0 || n_boxes <= 0) return 0;
  return ws_bytes(mm_cdiv(n_points, kTile), 1, n_boxes);
}

extern "C" int mmmot_crop_count(const float* points, int n_points, int stride, const void* planes, int planes_f64,
                                int n_boxes, int* split, void* workspace, size_t workspace_bytes, void* stream) {
  if (!points || !planes || !split || !workspace || n_points <= 0 || n_boxes <= 0 || stride < 3) return MMMOT_E_ARG;
  const int frame_off[2] = {0, n_points};
  cudaStream_t st = (cudaStream_t)stream;
  if (planes_f64)
    return crop_count<double, false>(points, stride, frame_off, 1, nullptr, (const double*)planes, nullptr, n_boxes,
                                     split, workspace, workspace_bytes, st);
  return crop_count<float, false>(points, stride, frame_off, 1, nullptr, (const float*)planes, nullptr, n_boxes, split,
                                  workspace, workspace_bytes, st);
}

extern "C" int mmmot_crop_scatter(const float* points, int n_points, int stride, const void* planes, int planes_f64,
                                  int n_boxes, const int* split, int out_channels, float* out_points, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  if (!points || !planes || !split || !out_points || !workspace || n_points <= 0 || n_boxes <= 0) return MMMOT_E_ARG;
  const int frame_off[2] = {0, n_points};
  cudaStream_t st = (cudaStream_t)stream;
  if (planes_f64)
    return crop_scatter<double, false>(points, stride, frame_off, 1, nullptr, (const double*)planes, nullptr, n_boxes,
                                       split, out_channels, out_points, workspace, workspace_bytes, st);
  return crop_scatter<float, false>(points, stride, frame_off, 1, nullptr, (const float*)planes, nullptr, n_boxes,
                                    split, out_channels, out_points, workspace, workspace_bytes, st);
}

extern "C" size_t mmmot_prep_workspace(int max_frame_points, int n_frames, int n_dets) {
  if (max_frame_points <= 0 || n_frames <= 0 || n_dets <= 0) return 0;
  return ws_bytes(mm_cdiv(max_frame_points, kTile), n_frames, n_dets);
}

extern "C" int mmmot_prep_count(const float* points, const int* frame_offsets, int n_frames, int stride,
                                const double* fov_planes, const double* det_planes, const int* det_frame, int n_dets,
                                int* split, void* workspace, size_t workspace_bytes, void* stream) {
  if (!points || !fov_planes || !det_planes || !det_frame || !split || !workspace || stride < 3 || stride > 4)
    return MMMOT_E_ARG;
  return crop_count<double, true>(points, stride, frame_offsets, n_frames, fov_planes, det_planes, det_frame, n_dets,
                                  split, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int mmmot_prep_scatter(const float* points, const int* frame_offsets, int n_frames, int stride,
                                  const double* fov_planes, const double* det_planes, const int* det_frame,
                                  int n_dets, const int* split, int out_channels, float* out_points, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  if (!points || !fov_planes || !det_planes || !det_frame || !split || !out_points || !workspace || stride < 3 ||
      stride > 4)
    return MMMOT_E_ARG;
  return crop_scatter<double, true>(points, stride, frame_offsets, n_frames, fov_planes, det_planes, det_frame,
                                    n_dets, split, out_channels, out_points, workspace, workspace_bytes,
                                    (cudaStream_t)stream);
}
