// PointNet encoder over ragged per-detection LiDAR point sets.
// Replaces reference modules/point_net.py:25-44 (PointNet_v1.forward) and :115-153
// (PointNetfeatGN.forward).  Uses two identities proven in SURVEY F4 / B-9:
//   * both STN transforms are input-independent constants -> folded into conv1 / conv2 / head
//     weights by the host weight packer (the STN convs are never executed);
//   * the 1088-wide head conv splits into a 64-wide per-point part plus a per-detection
//     addend  Wh[:,64:] * mean_det(x5)  (1088 -> 64 MACs per point per output channel).
// Per-detection pooling is a MEAN (SURVEY F5).  One frame-pair = one GroupNorm domain.
#include <algorithm>
#include <atomic>
#include <vector>

#include "norm_ops.cuh"
#include "gemm_gen.cuh"
#include "tc_ops.cuh"

namespace {

// xt [C][P] = pts [P][C] transposed (C = 3 or 4 point channels)
__global__ void transpose_points_kernel(const float* __restrict__ pts, int C, float* __restrict__ xt, long P) {
  long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  for (int k = 0; k < C; k++) xt[k * P + p] = pts[p * C + k];
}

// First trunk layer (C -> 64, C = 3 xyz or 4 xyz + reflectance) on the tensor-core path.  With K = C a contraction
// kernel is all epilogue, so the layer is never materialised in fp32: one kernel accumulates its GroupNorm statistics, a
// second recomputes it, applies GroupNorm + ReLU and writes the FP16 hi/lo planes layer 2's TMA loads read.  Both evaluate
//   y = fma(w2, z, fma(w1, y, fma(w0, x, b)))  and, with C = 4, then  y = fma(w3, r, y)
// in this order, so the statistics describe exactly the values normalised and 3-channel points take the same arithmetic
// as before the reflectance channel existed.  C is a runtime argument, uniform per launch.
// pts [P][C] (16-byte rows when C = 4), wt [C][64], part[(tile*2 + h)*64 + c] (h = first / second half of the tile's
// points, fp64 sums).  The stats kernel stages the tile's points as 16-byte rows whatever C (3-channel rows padded with
// r = 0, w3 = 0) and runs one loop for both widths: fma(0, 0, y) = y exactly (up to the sign of a zero, which no sum or
// square sees), so the statistics of 3-channel points are the ones the 3-term chain gives.  The apply kernel, whose
// outputs carry the sign of a zero into the FP16 planes, takes the fourth fma only when C = 4.  The fp64 sums are
// latency-bound: the stats kernel is held to 32 registers, eight CTAs per SM.
__global__ void __launch_bounds__(256, 8) pn_l1_stats_kernel(const float* __restrict__ pts, int C, const int4* __restrict__ tiles,
                                                          const float* __restrict__ wt, const float* __restrict__ bias,
                                                          double2* __restrict__ part) {
  __shared__ float4 sp[256];
  __shared__ double2 red[4][64];
  const int4 tt = tiles[blockIdx.x];          // (pair, first point, length <= 256, -)
  if (threadIdx.x < tt.z) {                   // one point per thread (a tile holds at most 256)
    const long r = (long)tt.y + threadIdx.x;
    sp[threadIdx.x] = C == 4 ? __ldg(reinterpret_cast<const float4*>(pts) + r)
                             : make_float4(__ldg(pts + r * 3), __ldg(pts + r * 3 + 1), __ldg(pts + r * 3 + 2), 0.f);
  }
  __syncthreads();
  const int c = threadIdx.x & 63, qd = threadIdx.x >> 6;
  const float w0 = wt[c], w1 = wt[64 + c], w2 = wt[128 + c], w3 = C == 4 ? wt[192 + c] : 0.f, b = bias[c];
  double s1 = 0.0, s2 = 0.0;
  const int p1 = min(tt.z, (qd + 1) * 64);
  for (int p = qd * 64; p < p1; p++) {
    const float4 q = sp[p];
    const float y = fmaf(w3, q.w, fmaf(w2, q.z, fmaf(w1, q.y, fmaf(w0, q.x, b))));
    s1 += (double)y;
    s2 += (double)y * (double)y;
  }
  red[qd][c] = make_double2(s1, s2);
  __syncthreads();
  if (threadIdx.x < 128) {
    const int h = threadIdx.x >> 6;
    const double2 a = red[2 * h][c], d = red[2 * h + 1][c];
    part[((long)blockIdx.x * 2 + h) * 64 + c] = make_double2(a.x + d.x, a.y + d.y);
  }
}
// x1p planes [2][P][64] = split(relu(GN(y)))  ;  thread = (point, 4 channels)
__global__ void __launch_bounds__(256) pn_l1_apply_kernel(const float* __restrict__ pts, int C, const float* __restrict__ wt,
                                                          const float* __restrict__ bias, const float* __restrict__ sc,
                                                          const float* __restrict__ sh, const int* __restrict__ seg,
                                                          int L, long P, __half* __restrict__ out, int* status) {
  const long idx = (long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= P * 16) return;
  const long row = idx >> 4;
  const int c = (int)(idx & 15) * 4;
  const int g = seg[row] / L;
  float4 q;
  if (C == 4) q = __ldg(reinterpret_cast<const float4*>(pts) + row);
  else q = make_float4(__ldg(pts + row * 3), __ldg(pts + row * 3 + 1), __ldg(pts + row * 3 + 2), 0.f);
  const float4 w0 = *reinterpret_cast<const float4*>(wt + c), w1 = *reinterpret_cast<const float4*>(wt + 64 + c),
               w2 = *reinterpret_cast<const float4*>(wt + 128 + c), b = *reinterpret_cast<const float4*>(bias + c);
  float4 v;
  v.x = fmaf(w2.x, q.z, fmaf(w1.x, q.y, fmaf(w0.x, q.x, b.x)));
  v.y = fmaf(w2.y, q.z, fmaf(w1.y, q.y, fmaf(w0.y, q.x, b.y)));
  v.z = fmaf(w2.z, q.z, fmaf(w1.z, q.y, fmaf(w0.z, q.x, b.z)));
  v.w = fmaf(w2.w, q.z, fmaf(w1.w, q.y, fmaf(w0.w, q.x, b.w)));
  if (C == 4) {
    const float4 w3 = *reinterpret_cast<const float4*>(wt + 192 + c);
    v.x = fmaf(w3.x, q.w, v.x); v.y = fmaf(w3.y, q.w, v.y); v.z = fmaf(w3.z, q.w, v.z); v.w = fmaf(w3.w, q.w, v.w);
  }
  const float4 a = *reinterpret_cast<const float4*>(sc + (long)g * 64 + c);
  const float4 s = *reinterpret_cast<const float4*>(sh + (long)g * 64 + c);
  float4 r;
  r.x = fmaxf(fmaf(v.x, a.x, s.x), 0.f);
  r.y = fmaxf(fmaf(v.y, a.y, s.y), 0.f);
  r.z = fmaxf(fmaf(v.z, a.z, s.z), 0.f);
  r.w = fmaxf(fmaf(v.w, a.w, s.w), 0.f);
  split4_store(r, out + row * 64 + c, out + P * 64 + row * 64 + c, status);
}

// seg[p] = detection owning point p (binary search in the CSR offsets)
__global__ void point_segment_kernel(const int* __restrict__ split, int ndet, long P, int* __restrict__ seg) {
  long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  int lo = 0, hi = ndet;  // split[lo] <= p < split[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (split[mid] <= p) lo = mid; else hi = mid;
  }
  seg[p] = lo;
}

// out[c][d] = mean over the detection's points of relu(Y[c][p]*sc[pair][c] + sh[pair][c]).
// One warp per (c, d); lanes stride the segment (coalesced).
__global__ void segment_mean_kernel(const float* __restrict__ Y, long P, const int* __restrict__ split,
                                    const float* __restrict__ sc, const float* __restrict__ sh, int C,
                                    int ndet, int L, float* __restrict__ out, const float* __restrict__ mask = nullptr) {
  long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (w >= (long)C * ndet) return;
  int d = (int)(w % ndet), c = (int)(w / ndet);
  int pair = d / L;
  float a = sc[(long)pair * C + c], b = sh[(long)pair * C + c];
  int s = split[d], e = split[d + 1];
  const float* row = Y + (long)c * P;
  float acc = 0.f;
  if (mask) {   // training-mode Dropout of the head activation (point_net.py:29-30): mask[c][p] in {0, 1/(1-p)}
    const float* mrow = mask + (long)c * P;
    for (int p = s + lane; p < e; p += 32) acc += fmaxf(fmaf(row[p], a, b), 0.f) * mrow[p];
  } else {
    for (int p = s + lane; p < e; p += 32) acc += fmaxf(fmaf(row[p], a, b), 0.f);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[(long)c * ndet + d] = e > s ? acc / (float)(e - s) : 0.f;
}

// feats[pair][1][c][l] = relu(O[c][d]*sc[pair][c] + sh[pair][c])
__global__ void pointnet_out_kernel(const float* __restrict__ O, const float* __restrict__ sc,
                                    const float* __restrict__ sh, int ndet, int L,
                                    float* __restrict__ feats) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 512L * ndet) return;
  int d = (int)(idx % ndet), c = (int)(idx / ndet);
  int pair = d / L, l = d - pair * L;
  float v = fmaxf(fmaf(O[idx], sc[pair * 512 + c], sh[pair * 512 + c]), 0.f);
  feats[(((long)pair * 3 + 1) * 512 + c) * L + l] = v;
}

// out[c][d] = segsum[d][c] * 2^-32 / (points of detection d)   (fixed-point sums of the fused segment-sum epilogue)
__global__ void segsum_mean_kernel(const unsigned long long* __restrict__ segsum, const int* __restrict__ split,
                                   int C, int ndet, float* __restrict__ out) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)C * ndet) return;
  const int d = (int)(idx / C), c = (int)(idx - (long)d * C);
  const int cnt = split[d + 1] - split[d];
  out[(long)c * ndet + d] = cnt > 0 ? (float)((double)segsum[idx] * (1.0 / 4294967296.0) / (double)cnt) : 0.f;
}

// channels-last variant: out[d][C] (the layout the tensor-core per-detection contractions read as rows)
__global__ void segsum_mean_cl_kernel(const unsigned long long* __restrict__ segsum, const int* __restrict__ split,
                                      int C, int ndet, float* __restrict__ out) {
  long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)C * ndet) return;
  const int d = (int)(idx / C);
  const int cnt = split[d + 1] - split[d];
  out[idx] = cnt > 0 ? (float)((double)segsum[idx] * (1.0 / 4294967296.0) / (double)cnt) : 0.f;
}
// feats[pair][1][c][l] = relu(O[d][c]*sc[pair][c] + sh[pair][c]) from channels-last O (32 x 32 tiles through smem)
__global__ void pointnet_out_cl_kernel(const float* __restrict__ O, const float* __restrict__ sc, const float* __restrict__ sh,
                                       int L, float* __restrict__ feats) {
  __shared__ float tile[32][33];
  const int pair = blockIdx.z, c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int l = l0 + i, c = c0 + threadIdx.x;
    if (l < L) tile[i][threadIdx.x] = fmaxf(fmaf(O[((long)pair * L + l) * 512 + c], sc[pair * 512 + c], sh[pair * 512 + c]), 0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, l = l0 + threadIdx.x;
    if (l < L) feats[(((long)pair * 3 + 1) * 512 + c) * L + l] = tile[threadIdx.x][i];
  }
}

// Column-tile table of the ragged per-pair point ranges, built ON THE DEVICE from the CSR offsets (the host only
// needs the tile count for its launch geometry): no pageable host->device copy, so the calling thread never blocks on
// the stream and can keep enqueueing.  gstart[p] = first tile of pair p (one thread: pairs is small), then one thread
// per pair fills its tiles {pair, first point, length <= tw}.
__global__ void pn_tiles_kernel(const int* __restrict__ split, int pairs, int L, int tw, int* __restrict__ cnt,
                                int* __restrict__ gstart, int4* __restrict__ tiles) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int p = 0; p < pairs; p++) {
      const int n = split[(p + 1) * L] - split[p * L];
      cnt[p] = n;
      gstart[p] = acc;
      acc += (n + tw - 1) / tw;
    }
    gstart[pairs] = acc;
  }
  __syncthreads();   // single CTA: the prefix is visible to all its threads
  for (int p = threadIdx.x; p < pairs; p += blockDim.x) {
    const int s0 = split[p * L], e = split[(p + 1) * L];
    int t = gstart[p];
    for (int c = s0; c < e; c += tw) tiles[t++] = make_int4(p, c, min(tw, e - c), 0);
  }
}

// ---------------- GroupNorm statistics of the two widest layers from the moments of their input ----------------
// GroupNorm(C, C) over a pair's n points of y = W x + b (+ a[det]) needs, per output channel, only the mean and the
// variance of y, and both follow from the input's moments: S1 = sum x, S2 = sum x x^T (C x C) and, with an addend,
// the per-detection sums of x.  Building them costs C^2 MACs per point instead of the layer's C x M (M = 8C here).
namespace pnm {
constexpr int KC = 32;        // points per pipeline stage
constexpr int NSTG = 4;       // pipeline stages
constexpr int SLICE = 32;     // tiles (of 256 points) per CTA

template <int C> __host__ __device__ constexpr int threads() { return (C / 32) * (C / 32) * 32; }   // one warp per 32 x 32 block of S2
template <int C> __host__ __device__ constexpr size_t ring_bytes() { return (size_t)NSTG * 2 * KC * (C + 8) * sizeof(__half); }
// ring + the fp64 accumulators of S2 (32 per thread, kept in shared memory: in registers they would spill)
template <int C> constexpr size_t smem_bytes() { return ring_bytes<C>() + 32 * sizeof(double) * threads<C>(); }
constexpr long part_doubles(long max_tiles, int pairs) { return (max_tiles / SLICE + pairs) * (128L * 128 + 128); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Moments of the FP16 hi/lo planes X [2][P][C] (x = hi + lo), one CTA per slice: slice j of pair p is the pair's tiles
// gstart[p] + j*SLICE .. (at most SLICE, never past the pair), a contiguous range of its points; sstart [pairs + 1] =
// first slice of each pair.  part[slice][C*C + C] (fp64) = S2 row-major, then S1, over the slice's points.
// S2 ~ XhT Xh + XhT Xl + XlT Xh on mma.sync (points are the K dimension, so both operands are read transposed from the
// channels-last rows with ldmatrix.trans); the fp32 accumulators restart at every 256-point tile and are added into
// fp64 ones, so no fp32 chain spans more than one tile.  S1 in fp64 (x = hi + lo is exact in fp32).
// DET: also detsum[det][C] += the detection's sums of x in 2^-32 fixed point (integer adds: order-independent).
// Every partial depends only on the pair's data, never on the grid or on the rest of the batch.
template <int C, bool DET>
__global__ void __launch_bounds__(threads<C>(), 1)
pn_moments_kernel(const __half* __restrict__ X, long P, const int4* __restrict__ tiles, const int* __restrict__ gstart,
                  const int* __restrict__ sstart, int pairs, const int* __restrict__ seg, double* __restrict__ part,
                  unsigned long long* __restrict__ detsum) {
  constexpr int NT = threads<C>(), LD = C + 8, PLANE = KC * LD, STAGE = 2 * PLANE;   // smem rows padded: no conflicts
  constexpr int Q = NT / C, R = KC / Q;     // per-channel sums: thread (c, q) takes rows [q R, q R + R) of each stage
  constexpr int CH = C / 8;                  // 16-byte chunks per row
  extern __shared__ __align__(16) __half sm[];
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int lo = 0, hi = pairs;                    // the pair: sstart[lo] <= s < sstart[lo + 1]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sstart[mid] <= s) lo = mid; else hi = mid;
  }
  const int t0 = gstart[lo] + (s - sstart[lo]) * SLICE, t1 = min(t0 + SLICE, gstart[lo + 1]);
  const long r0 = tiles[t0].y;
  const int n = (int)(tiles[t1 - 1].y + tiles[t1 - 1].z - r0);
  const int nst = (n + KC - 1) / KC;
  const uint32_t sbase = tc::smem_u32(sm);

  auto load = [&](int k) {
    const uint32_t dst0 = sbase + (uint32_t)((k % NSTG) * STAGE * 2);
#pragma unroll
    for (int i = tid; i < 2 * KC * CH; i += NT) {
      const int pl = i / (KC * CH), row = (i / CH) % KC, ch = i % CH;
      const int r = k * KC + row;
      const __half* src = r < n ? X + pl * P * C + (r0 + r) * C + ch * 8 : X;
      cp_async16(dst0 + (uint32_t)((pl * PLANE + row * LD + ch * 8) * 2), src, r < n ? 16 : 0);   // zero-fills the tail
    }
  };

  const int wi = warp / (C / 32), wj = warp % (C / 32);
  float acc[2][4][4];
  double* acc64 = reinterpret_cast<double*>(reinterpret_cast<char*>(sm) + ring_bytes<C>()) + tid;   // [32][NT]
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int e = 0; e < 4; e++) { acc[a][b][e] = 0.f; acc64[((a * 4 + b) * 4 + e) * NT] = 0.0; }
  const int c = tid % C, q = tid / C;
  double s1 = 0.0;
  int dcur = -1;
  long long run = 0;

#pragma unroll
  for (int k = 0; k < NSTG - 1; k++) {
    if (k < nst) load(k);
    cp_commit();
  }
  for (int k = 0; k < nst; k++) {
    cp_wait<NSTG - 2>();
    __syncthreads();                         // stage k landed for all; stage k - 1's buffer is free
    if (k + NSTG - 1 < nst) load(k + NSTG - 1);
    cp_commit();
    const uint32_t st_hi = sbase + (uint32_t)((k % NSTG) * STAGE * 2), st_lo = st_hi + PLANE * 2;
#pragma unroll
    for (int ks = 0; ks < KC / 16; ks++) {
      uint32_t ah[2][4], al[2][4];
      const int ka = ks * 16 + (lane & 7) + ((lane >> 4) & 1) * 8;
#pragma unroll
      for (int mt = 0; mt < 2; mt++) {
        const uint32_t off = (uint32_t)((ka * LD + wi * 32 + mt * 16 + ((lane >> 3) & 1) * 8) * 2);
        ldsm_x4_t(st_hi + off, ah[mt]);
        ldsm_x4_t(st_lo + off, al[mt]);
      }
      const int kb = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int np = 0; np < 2; np++) {
        uint32_t bh[4], bl[4];
        const uint32_t off = (uint32_t)((kb * LD + wj * 32 + np * 16 + ((lane >> 4) & 1) * 8) * 2);
        ldsm_x4_t(st_hi + off, bh);
        ldsm_x4_t(st_lo + off, bl);
#pragma unroll
        for (int mt = 0; mt < 2; mt++)
#pragma unroll
          for (int h = 0; h < 2; h++) {
            float (&d)[4] = acc[mt][np * 2 + h];
            mma16816(d, ah[mt], bh[2 * h], bh[2 * h + 1]);
            mma16816(d, ah[mt], bl[2 * h], bl[2 * h + 1]);
            mma16816(d, al[mt], bh[2 * h], bh[2 * h + 1]);
          }
      }
    }
    {
      const __half* xs = sm + (k % NSTG) * STAGE + q * R * LD + c;
#pragma unroll 4
      for (int rr = 0; rr < R; rr++) {
        const int r = k * KC + q * R + rr;
        if (r >= n) break;
        const float x = __half2float(xs[rr * LD]) + __half2float(xs[PLANE + rr * LD]);
        s1 += (double)x;
        if (DET) {
          const int d = seg[r0 + r];
          if (d != dcur) {
            if (dcur >= 0) atomicAdd(detsum + (long)dcur * C + c, (unsigned long long)run);
            dcur = d;
            run = 0;
          }
          run += __float2ll_rn(x * 4294967296.f);
        }
      }
    }
    if ((k & 7) == 7 || k == nst - 1) {      // end of a 256-point tile
#pragma unroll
      for (int a = 0; a < 2; a++)
#pragma unroll
        for (int b = 0; b < 4; b++)
#pragma unroll
          for (int e = 0; e < 4; e++) { acc64[((a * 4 + b) * 4 + e) * NT] += (double)acc[a][b][e]; acc[a][b][e] = 0.f; }
    }
  }
  if (DET && dcur >= 0) atomicAdd(detsum + (long)dcur * C + c, (unsigned long long)run);

  double* out = part + (long)s * (C * C + C);
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++) {
      const int i = wi * 32 + a * 16 + (lane >> 2), j = wj * 32 + b * 8 + 2 * (lane & 3);
      const double* v = acc64 + (a * 4 + b) * 4 * NT;
      *reinterpret_cast<double2*>(out + (long)i * C + j) = make_double2(v[0], v[NT]);
      *reinterpret_cast<double2*>(out + (long)(i + 8) * C + j) = make_double2(v[2 * NT], v[3 * NT]);
    }
  cp_wait<0>();
  __syncthreads();                           // every stage read: the ring holds the S1 reduction now
  double* red = reinterpret_cast<double*>(sm);
  red[q * C + c] = s1;
  __syncthreads();
  if (tid < C) {
    double v = 0.0;
#pragma unroll
    for (int g = 0; g < Q; g++) v += red[g * C + tid];
    out[C * C + tid] = v;
  }
}

// sstart[p] = first slice of pair p (pairs + 1 entries) from the tile starts gstart (one thread: pairs is small)
__global__ void pn_slices_kernel(const int* __restrict__ gstart, int pairs, int* __restrict__ sstart) {
  int acc = 0;
  for (int p = 0; p < pairs; p++) {
    sstart[p] = acc;
    acc += (gstart[p + 1] - gstart[p] + SLICE - 1) / SLICE;
  }
  sstart[pairs] = acc;
}

// mom[p][e] = sum over pair p's slices, in slice order, of part[slice][e]   (E = C*C + C)
__global__ void pn_moments_reduce_kernel(const double* __restrict__ part, const int* __restrict__ sstart, int E,
                                         double* __restrict__ mom) {
  const int p = blockIdx.y, e = blockIdx.x * 256 + threadIdx.x;
  if (e >= E) return;
  double a = 0.0;
  for (int s = sstart[p]; s < sstart[p + 1]; s++) a += part[(long)s * E + e];
  mom[(long)p * E + e] = a;
}

// stats[p][o] = (sum y, sum y^2) over pair p's n points of y = x Wt[:, o] + bias[o] (+ addend[det][o]), the format
// gn_finalize reads, from the pair's moments mom[p] = (S2, S1) in centred form (no cancellation in y):
//   mu = S1 / n,  Cov = S2 / n - mu mu^T,  mean = w.mu + b,  var = w^T Cov w.
// With the addend a_d = addend[d] + b (per detection d of n_d points with sums s1_d = detsum[d] 2^-32) and its
// point-weighted mean abar:  mean = w.mu + abar,  var += (2/n) sum_d (a_d - abar) w.(s1_d - n_d mu)
//                                                       + (1/n) sum_d n_d (a_d - abar)^2.
// Wt [C][M] are the fp32 master weights.  CTA = 64 output channels x 4 row groups of the quadratic form.
template <int C>
__global__ void __launch_bounds__(256) pn_moments_stats_kernel(const double* __restrict__ mom, const int* __restrict__ cnt,
                                                               const float* __restrict__ Wt, const float* __restrict__ bias,
                                                               int M, const float* __restrict__ addend,
                                                               const unsigned long long* __restrict__ detsum,
                                                               const int* __restrict__ det_split, int L,
                                                               double* __restrict__ stats) {
  __shared__ float ws[C][64];
  __shared__ double mu[C];
  __shared__ double cv[8][C];
  __shared__ double red[4][64];
  const int p = blockIdx.y, o0 = blockIdx.x * 64, ol = threadIdx.x & 63, q = threadIdx.x >> 6, o = o0 + ol;
  const double* S2 = mom + (long)p * (C * C + C);
  const double n = (double)cnt[p];
  for (int i = threadIdx.x; i < C * 64; i += 256) ws[i / 64][i % 64] = o0 + i % 64 < M ? Wt[(long)(i / 64) * M + o0 + i % 64] : 0.f;
  for (int i = threadIdx.x; i < C; i += 256) mu[i] = S2[C * C + i] / n;
  __syncthreads();
  double wmu = 0.0;
  for (int k = 0; k < C; k++) wmu += (double)ws[k][ol] * mu[k];
  double var = 0.0;
  for (int i0 = 0; i0 < C; i0 += 8) {
    for (int e = threadIdx.x; e < 8 * C; e += 256) {
      const int r = e / C, j = e % C;
      cv[r][j] = S2[(long)(i0 + r) * C + j] / n - mu[i0 + r] * mu[j];
    }
    __syncthreads();
    for (int r = 2 * q; r < 2 * q + 2; r++) {
      double t = 0.0;
      for (int j = 0; j < C; j++) t += cv[r][j] * (double)ws[j][ol];
      var += (double)ws[i0 + r][ol] * t;
    }
    __syncthreads();
  }
  const bool valid = o < M;
  double mean = wmu + (valid ? (double)bias[o] : 0.0);
  if (addend && valid) {
    const double b = (double)bias[o];
    double abar = 0.0;
    for (int l = 0; l < L; l++) {
      const int d = p * L + l;
      abar += (double)(det_split[d + 1] - det_split[d]) * ((double)addend[(long)d * M + o] + b);
    }
    abar /= n;
    double cross = 0.0, between = 0.0;
    for (int l = q; l < L; l += 4) {
      const int d = p * L + l;
      const double nd = (double)(det_split[d + 1] - det_split[d]);
      const double a = (double)addend[(long)d * M + o] + b - abar;
      double ws1 = 0.0;
      for (int k = 0; k < C; k++)
        ws1 += (double)ws[k][ol] * ((double)(long long)detsum[(long)d * C + k] * (1.0 / 4294967296.0) - nd * mu[k]);
      cross += a * ws1;
      between += nd * a * a;
    }
    var += (2.0 * cross + between) / n;
    mean = wmu + abar;
  }
  red[q][ol] = var;
  __syncthreads();
  if (q == 0 && valid) {
    const double v = fmax(red[0][ol] + red[1][ol] + red[2][ol] + red[3][ol], 0.0);
    stats[((long)p * M + o) * 2] = n * mean;
    stats[((long)p * M + o) * 2 + 1] = n * (v + mean * mean);
  }
}
}  // namespace pnm

struct PnWs {
  float *xt, *y1, *t0, *t1, *big, *gmean, *u, *ut, *hmean, *o;
  unsigned long long* segsum;   // tensor-core path: [ndet][1024] fixed-point per-detection sums
  __half *x1p, *xp;     // tensor-core path: FP16 hi/lo planes of normalised activations [2][P][64], [2][P][128]
  float *sc1, *sh1, *sc, *sh;
  double *stats, *mom;  // mom (tensor-core path): [pairs][128*128 + 128] input moments of the widest layers
  double2* part;        // tensor-core path: also the moments kernel's per-slice partials (used one at a time)
  int *seg, *cnt, *gstart, *sstart;
  int4 *tiles, *ctab;
};

// capacity of the tile tables: 128-point tiles over `pairs` ragged ranges of P points; also bounds 2 partials per 256-wide tile
long pn_max_tiles(long P, int pairs) { return P / 128 + 2 * pairs + 2; }

// use_tc: the tensor-core path never materialises the 1024-wide activation (537 MB per frame-pair at cfg4), reads the
// points row-major (no xt), never stores layer 1 in fp32 (no y1) and keeps U channels-last (ut; the FP32 path: u)
PnWs carve(MmArena& a, int pairs, int L, long P, bool use_tc) {
  const long max_tiles = pn_max_tiles(P, pairs);
  PnWs w;
  long nd = (long)pairs * L;
  w.xt = a.take<float>(use_tc ? 0 : 3 * P);   // 3-channel points only: pointnet_fp32 transposes 4-channel ones into t1
  w.y1 = a.take<float>(use_tc ? 0 : 64 * P);
  w.t0 = a.take<float>(128 * P);
  w.t1 = a.take<float>(64 * P);
  w.big = a.take<float>(use_tc ? 0 : 1024 * P);
  w.segsum = a.take<unsigned long long>(1024 * nd);
  w.x1p = a.take<__half>(2 * 64 * P);
  w.xp = a.take<__half>(2 * 128 * P);
  w.gmean = a.take<float>(1024 * nd);
  w.u = a.take<float>(use_tc ? 0 : 512 * nd);
  w.ut = a.take<float>(use_tc ? 512 * nd : 0);
  w.hmean = a.take<float>(512 * nd);
  w.o = a.take<float>(512 * nd);
  w.sc1 = a.take<float>((size_t)pairs * 64);
  w.sh1 = a.take<float>((size_t)pairs * 64);
  w.sc = a.take<float>((size_t)pairs * 1024);
  w.sh = a.take<float>((size_t)pairs * 1024);
  w.stats = a.take<double>((size_t)pairs * 1024 * 2);
  w.mom = a.take<double>(use_tc ? (size_t)pairs * (128 * 128 + 128) : 0);
  w.part = a.take<double2>(use_tc ? std::max((size_t)max_tiles * 1024, (size_t)(pnm::part_doubles(max_tiles, pairs) + 1) / 2)
                                  : (size_t)max_tiles * 1024);
  w.gstart = a.take<int>(pairs + 1);
  w.sstart = a.take<int>(use_tc ? pairs + 1 : 0);
  w.seg = a.take<int>(P);
  w.cnt = a.take<int>(pairs);
  w.tiles = a.take<int4>(max_tiles);
  w.ctab = a.take<int4>(2 * max_tiles);
  return w;
}

// The host's checks of the CSR offsets h_det_split [pairs*L + 1]: MMMOT_E_SHAPE unless the first is 0, P > 0 and every
// detection owns at least one point.  n_tiles: column tiles of at most tw points over each pair's point range (tiles
// never straddle two pairs: one pair = one GroupNorm domain); the host needs only this count for its launch geometry.
// max_tiles: how many the tables of a carved workspace hold.
struct PnShape { long P, n_tiles, max_tiles; };
int pn_shape(const int* h_det_split, int pairs, int L, int tw, PnShape& s) {
  const int ndet = pairs * L;
  s.P = h_det_split[ndet];
  if (h_det_split[0] != 0 || s.P <= 0) return MMMOT_E_SHAPE;
  for (int d = 0; d < ndet; d++)
    if (h_det_split[d + 1] <= h_det_split[d]) return MMMOT_E_SHAPE;
  s.n_tiles = 0;
  for (int p = 0; p < pairs; p++) s.n_tiles += mm_cdiv((long)h_det_split[(p + 1) * L] - h_det_split[p * L], tw);
  s.max_tiles = pn_max_tiles(s.P, pairs);
  return 0;
}

// The tables of the ragged per-pair point ranges, built on the device from the CSR offsets det_split [pairs*L + 1]:
// tiles [n_tiles] {pair, first point, length <= tw, 0}, cnt [pairs] points per pair, gstart [pairs + 1] first tile of
// each pair, seg [P] detection of each point and, if ctab is set, the chunk descriptors of the tensor-core epilogue
// (tma::seg_chunk_tab_kernel, [2*n_tiles]).
int pn_tables(const int* det_split, int pairs, int L, long P, int tw, long n_tiles, int* cnt, int* gstart, int4* tiles,
              int* seg, int4* ctab, cudaStream_t st) {
  pn_tiles_kernel<<<1, 256, 0, st>>>(det_split, pairs, L, tw, cnt, gstart, tiles);
  MM_LAUNCH_CHECK();
  point_segment_kernel<<<mm_cdiv(P, 256), 256, 0, st>>>(det_split, pairs * L, P, seg);
  MM_LAUNCH_CHECK();
  if (ctab) {
    tma::seg_chunk_tab_kernel<<<mm_cdiv(n_tiles * 2, 128), 128, 0, st>>>(tiles, (int)n_tiles, seg, ctab);
    MM_LAUNCH_CHECK();
  }
  return 0;
}

template <int C, bool DET>
int pn_moments_launch(const PnWs& w, const __half* X, long P, int pairs, long n_slices, cudaStream_t st) {
  static std::atomic<unsigned long long> smem_set{0};
  MM_TRY(mm_ensure_smem(pnm::pn_moments_kernel<C, DET>, pnm::smem_bytes<C>(), smem_set));
  pnm::pn_moments_kernel<C, DET><<<(int)n_slices, pnm::threads<C>(), pnm::smem_bytes<C>(), st>>>(
      X, P, w.tiles, w.gstart, w.sstart, pairs, w.seg, (double*)w.part, w.segsum);
  MM_LAUNCH_CHECK();
  return 0;
}

// GroupNorm(M, M) statistics w.stats [pairs][M] (sum, sum of squares per pair and channel) of the tensor-core path's
// widest layers, y = x Wt + bias (+ addend[det], [ndet][M]) over the FP16 hi/lo planes X [2][P][K], K = 128 (layer 5,
// 128 -> 1024) or 64 (head, 64 -> 512, with the addend).  Default: from the input's moments (pnm above); Wt [K][M] are
// the fp32 master weights.  Debug bit 4: the contraction itself with only its GroupNorm partials kept (Wp / wps, the
// packed tiles), then their fixed-order reduction.  Tables (tiles, gstart, cnt, seg, ctab) as pn_tables left them.
int pn_wide_stats(const PnWs& w, const int* h_det_split, const int* det_split, long P, int pairs, int L, long n_tiles,
                  const __half* X, int K, const float* Wt, const uint4* Wp, float wps, const float* bias, int M,
                  const float* addend, cudaStream_t st) {
  const bool timed = mm_timing_on();
  if (mm_debug_flags() & MM_DBG_PN_STATS_PASS) {
    GemmP p = gemm_defaults();
    p.bias = bias; p.M = M; p.K = K;
    p.tile_tab = w.tiles; p.num_tiles = (int)n_tiles;
    p.Y = nullptr; p.y_ms = M;
    p.part = w.part;
    if (addend) { p.addend = addend; p.seg = w.seg; p.ld_add = M; }
    if (timed) mm_timing_begin(st, K == 128 ? MM_T_PN_L5A : MM_T_PN_HEADA, 2.0 * M * K * (double)P, 4.0 * K * (double)P);
    MM_TRY(gemm_tma_launch_mat(p, Wp, wps, X, P * K, P, K, tc::OUT_CL, 0, st, nullptr, nullptr, addend ? w.ctab : nullptr));
    if (timed) mm_timing_end(st);
    return stats_reduce(w.part, M, pairs, 0, w.gstart, w.stats, st, 2);
  }
  long n_slices = 0;
  for (int p = 0; p < pairs; p++)
    n_slices += mm_cdiv(mm_cdiv((long)h_det_split[(p + 1) * L] - h_det_split[p * L], tc::BN), pnm::SLICE);
  const int E = K * K + K;
  if (timed) mm_timing_begin(st, MM_T_PN_MOMFIN, 0.0, 0.0);
  pnm::pn_slices_kernel<<<1, 1, 0, st>>>(w.gstart, pairs, w.sstart);
  MM_LAUNCH_CHECK();
  if (timed) mm_timing_end(st);
  // algorithmic work: S2 (2 K^2 FLOPs per point; the MMAs issue three times that); compulsory traffic: the two FP16
  // planes (and the point -> detection map with the per-detection sums)
  if (K == 128) {
    if (timed) mm_timing_begin(st, MM_T_PN_MOM128, 2.0 * K * K * (double)P, 4.0 * K * (double)P);
    MM_TRY((pn_moments_launch<128, false>(w, X, P, pairs, n_slices, st)));
  } else {
    MM_CUDA(cudaMemsetAsync(w.segsum, 0, (size_t)pairs * L * 64 * sizeof(unsigned long long), st));
    if (timed) mm_timing_begin(st, MM_T_PN_MOM64, 2.0 * K * K * (double)P, (4.0 * K + 4.0) * (double)P);
    MM_TRY((pn_moments_launch<64, true>(w, X, P, pairs, n_slices, st)));
  }
  if (timed) mm_timing_end(st);
  // slice partials in, pair moments out; the quadratic forms w^T Cov w (2 K^2 FLOPs per pair and channel)
  if (timed) mm_timing_begin(st, MM_T_PN_MOMFIN, 2.0 * K * K * (double)M * pairs, 8.0 * E * (double)(n_slices + pairs));
  pnm::pn_moments_reduce_kernel<<<dim3(mm_cdiv(E, 256), pairs), 256, 0, st>>>((const double*)w.part, w.sstart, E, w.mom);
  MM_LAUNCH_CHECK();
  if (K == 128)
    pnm::pn_moments_stats_kernel<128><<<dim3(mm_cdiv(M, 64), pairs), 256, 0, st>>>(w.mom, w.cnt, Wt, bias, M, nullptr, nullptr,
                                                                                   det_split, L, w.stats);
  else
    pnm::pn_moments_stats_kernel<64><<<dim3(mm_cdiv(M, 64), pairs), 256, 0, st>>>(w.mom, w.cnt, Wt, bias, M, addend, w.segsum,
                                                                                  det_split, L, w.stats);
  MM_LAUNCH_CHECK();
  if (timed) mm_timing_end(st);
  return 0;
}

// Layer 5 (K = 128 -> M = 1024) or the head (64 -> 512, addend U): statistics only (pn_wide_stats), then a recompute with
// GroupNorm + ReLU + per-detection sums in its epilogue, out [ndet][M] the per-detection means.  The M x P activation
// (537 MB per frame-pair at cfg4 for layer 5) is never written.  tag times the recompute; status goes to gn_finalize.
int pn_wide_layer(const PnWs& w, const int* h_det_split, const int* det_split, long P, int pairs, int L, long n_tiles,
                  const __half* X, int K, const float* Wt, const uint4* Wp, float wps, const float* bias, int M,
                  const float* addend, const float* gamma, const float* beta, float* out, int tag, int* status,
                  cudaStream_t st) {
  const int ndet = pairs * L;
  MM_TRY(pn_wide_stats(w, h_det_split, det_split, P, pairs, L, n_tiles, X, K, Wt, Wp, wps, bias, M, addend, st));
  MM_TRY(gn_finalize(w.stats, gamma, beta, w.cnt, 0, pairs, M, 1, w.sc, w.sh, st, 0, 0, status));
  MM_CUDA(cudaMemsetAsync(w.segsum, 0, (size_t)ndet * M * sizeof(unsigned long long), st));
  GemmP p = gemm_defaults();
  p.bias = bias; p.M = M; p.K = K;
  p.tile_tab = w.tiles; p.num_tiles = (int)n_tiles;
  p.y_ms = M;
  if (addend) { p.addend = addend; p.ld_add = M; }
  p.sc = w.sc; p.sh = w.sh; p.seg = w.seg;
  const bool timed = mm_timing_on();
  if (timed) mm_timing_begin(st, tag, 2.0 * M * K * (double)P, 4.0 * K * (double)P);
  MM_TRY(gemm_tma_launch_mat(p, Wp, wps, X, P * K, P, K, tc::OUT_CL, 0, st, w.segsum, nullptr, w.ctab));
  if (timed) mm_timing_end(st);
  segsum_mean_cl_kernel<<<mm_cdiv((long)M * ndet, 256), 256, 0, st>>>(w.segsum, det_split, M, ndet, out);
  MM_LAUNCH_CHECK();
  return 0;
}

// Tensor-core path: channels-last activations; layers 2-4 write fp32 Y[p][cout] + GroupNorm partials, layer 1 and the
// two widest layers are recomputed instead of stored.  Layer 1's FP16 planes (x1p) are kept for the head.
int pointnet_tc(const mmmot_weights* wts, const float* points, const int* det_split, const int* h_det_split, int pairs,
                int L, long P, long n_tiles, const PnWs& w, int* status, float* feats, cudaStream_t st) {
  const int ndet = pairs * L;
  const bool timed = mm_timing_on();
  const double cols = (double)P;
  // layer 1 (C -> 64): its statistics, then the layer recomputed, normalised and split into x1p
  const int C = wts->point_channels;
  const float* const* l1 = &wts->w[MMMOT_W_PN_L1];
  if (timed) mm_timing_begin(st, MM_T_PN_L1, 2.0 * 64 * C * cols, 4.0 * C * cols);
  pn_l1_stats_kernel<<<(int)n_tiles, 256, 0, st>>>(points, C, w.tiles, l1[0], l1[1], w.part);
  MM_LAUNCH_CHECK();
  if (timed) mm_timing_end(st);
  MM_TRY(stats_reduce(w.part, 64, pairs, 0, w.gstart, w.stats, st, 2));
  MM_TRY(gn_finalize(w.stats, l1[2], l1[3], w.cnt, 0, pairs, 64, 1, w.sc, w.sh, st, 0, 0, status));
  if (timed) mm_timing_begin(st, MM_T_PN_L1, 0.0, (4.0 * C + 4.0 * 64) * cols);
  pn_l1_apply_kernel<<<mm_cdiv(P * 16, 256), 256, 0, st>>>(points, C, l1[0], l1[1], w.sc, w.sh, w.seg, L, P, w.x1p, status);
  MM_LAUNCH_CHECK();
  if (timed) mm_timing_end(st);
  float* const ys[3] = {w.t0, w.t1, w.t0};             // outputs of layers 2, 3, 4
  const bool gen_mid = !(mm_debug_flags() & MM_DBG_PN_NORM_SPLIT);   // layers 3, 4 through norm_split + the TMA-fed kernel
  for (int i = 1; i < 4; i++) {
    const float* const* q = &wts->w[MMMOT_W_PN_L1 + 4 * i];
    const int cin = 64, cout = i == 3 ? 128 : 64;
    GemmP p = gemm_defaults();
    p.bias = q[1]; p.M = cout; p.K = cin;
    p.tile_tab = w.tiles; p.num_tiles = (int)n_tiles;
    p.Y = ys[i - 1]; p.y_ms = cout;
    p.part = w.part;
    const uint4* wp = (const uint4*)wts->w[MMMOT_W_PN_WP1 + i];
    const float wps = wts->tc_scale[MMMOT_W_PN_WP1 + i];
    // compulsory traffic: activation in (4 B per element) + fp32 activation out
    if (timed) mm_timing_begin(st, MM_T_PN_L2 + (i - 1), 2.0 * cout * cin * cols, 4.0 * (cin + cout) * cols);
    if (gen_mid && i > 1) {
      // layers 3, 4: GroupNorm + ReLU of the previous layer applied by this contraction's operand producers
      // (gemm_gen.cuh) straight from its fp32 output: no normalised copy is written
      MM_TRY((gemm_gen_launch<gen::GEN_NORM>(p, wp, wps, ys[i - 2], cin, P, w.sc, w.sh, 0, 0, 0, st)));
    } else {                                                // FP16 hi/lo planes [2][P][cin] via TMA
      MM_TRY(gemm_tma_launch_mat(p, wp, wps, i == 1 ? w.x1p : w.xp, P * cin, P, cin, tc::OUT_CL, 0, st));
    }
    if (timed) mm_timing_end(st);
    MM_TRY(stats_reduce(w.part, cout, pairs, 0, w.gstart, w.stats, st, 2));
    MM_TRY(gn_finalize(w.stats, q[2], q[3], w.cnt, 0, pairs, cout, 1, w.sc, w.sh, st, 0, 0, status));
    if (!gen_mid || i == 3) {                           // otherwise consumed in place by the next layer's producers
      if (timed) mm_timing_begin(st, MM_T_PN_NORM, 0.0, 8.0 * cout * cols);
      MM_TRY(norm_split(ys[i - 1], cout, w.sc, w.sh, cout, P, 0, w.seg, L, w.xp, st, status));
      if (timed) mm_timing_end(st);
    }
  }
  const float* const* l5 = &wts->w[MMMOT_W_PN_L1 + 16];
  MM_TRY(pn_wide_layer(w, h_det_split, det_split, P, pairs, L, n_tiles, w.xp, 128, l5[0],
                       (const uint4*)wts->w[MMMOT_W_PN_WP1 + 4], wts->tc_scale[MMMOT_W_PN_WP1 + 4], l5[1], 1024, nullptr,
                       l5[2], l5[3], w.gmean, MM_T_PN_L5B, status, st));
  {
    // U[det][512] = gmean[det][1024] Wh[:, 64:]^T  (the per-detection part of point_net.py:27-28's conv1), on the
    // tensor cores over channels-last rows; its output is directly the [det][512] addend table of the head
    GemmP p = gemm_defaults();
    p.M = 512; p.K = 1024;
    p.S = ndet; p.tiles_per_group = mm_cdiv(ndet, tc::BN); p.num_tiles = p.tiles_per_group;
    p.x_gs = ndet;
    p.Y = w.ut; p.y_gs = ndet; p.y_ms = 512;
    MM_TRY((gemm_gen_launch<gen::GEN_COPY>(p, (const uint4*)wts->w[MMMOT_W_PN_WHGP], wts->tc_scale[MMMOT_W_PN_WHGP], w.gmean, 1024, 0,
                                           nullptr, nullptr, 0, 0, 0, st)));
  }
  MM_TRY(pn_wide_layer(w, h_det_split, det_split, P, pairs, L, n_tiles, w.x1p, 64, wts->w[MMMOT_W_PN_WHAT],
                       (const uint4*)wts->w[MMMOT_W_PN_WHAP], wts->tc_scale[MMMOT_W_PN_WHAP], wts->w[MMMOT_W_PN_BH], 512,
                       w.ut, wts->w[MMMOT_W_PN_GHW], wts->w[MMMOT_W_PN_GHB], w.hmean, MM_T_PN_HEADB, nullptr, st));
  // conv2 512 -> 512 over the pair's L detections, GroupNorm(16,512), ReLU (point_net.py:40-41), on the tensor cores
  const int tpg2 = mm_cdiv(L, tc::BN);
  GemmP p = gemm_defaults();
  p.bias = wts->w[MMMOT_W_PN_BO]; p.M = 512; p.K = 512;
  p.S = L; p.tiles_per_group = tpg2; p.num_tiles = tpg2 * pairs;
  p.x_gs = L;
  p.Y = w.o; p.y_gs = L; p.y_ms = 512;
  p.part = w.part;
  MM_TRY((gemm_gen_launch<gen::GEN_COPY>(p, (const uint4*)wts->w[MMMOT_W_PN_WOP], wts->tc_scale[MMMOT_W_PN_WOP], w.hmean, 512, 0,
                                         nullptr, nullptr, 0, 0, 0, st)));
  MM_TRY(stats_reduce(w.part, 512, pairs, tpg2, nullptr, w.stats, st, 2));
  MM_TRY(gn_finalize(w.stats, wts->w[MMMOT_W_PN_GOW], wts->w[MMMOT_W_PN_GOB], nullptr, L, pairs, 512, 32, w.sc, w.sh, st));
  pointnet_out_cl_kernel<<<dim3(mm_cdiv(L, 32), 16, pairs), dim3(32, 8), 0, st>>>(w.o, w.sc, w.sh, L, feats);
  MM_LAUNCH_CHECK();
  return 0;
}

// FP32 path (also the training forward): channel-major activations [C][P], every layer stored
int pointnet_fp32(const mmmot_weights* wts, const float* points, const int* det_split, int pairs, int L, long P,
                  long n_tiles, const PnWs& w, const float* head_mask, float* feats, cudaStream_t st) {
  const int ndet = pairs * L;
  const int C = wts->point_channels;
  // the carve holds 3P floats for xt; 4-channel points are transposed into t1 (64P floats), which nothing reads before
  // layer 3 writes it
  float* const xt = C == 4 ? w.t1 : w.xt;
  transpose_points_kernel<<<mm_cdiv(P, 256), 256, 0, st>>>(points, C, xt, P);
  MM_LAUNCH_CHECK();
  // trunk: C -> 64 -> 64 -> 64 -> 128 -> 1024, each conv + GroupNorm(cout, cout) over the pair's points + ReLU
  const int cin[5] = {C, 64, 64, 64, 128}, cout[5] = {64, 64, 64, 128, 1024};
  const float* src[5] = {xt, w.y1, w.t0, w.t1, w.t0};
  float* dst[5] = {w.y1, w.t0, w.t1, w.t0, w.big};
  for (int i = 0; i < 5; i++) {
    const float* const* q = &wts->w[MMMOT_W_PN_L1 + 4 * i];
    GemmP p = gemm_defaults();
    p.Wt = q[0]; p.bias = q[1]; p.ldw = cout[i]; p.M = cout[i]; p.K = cin[i];
    p.tile_tab = w.tiles; p.num_tiles = (int)n_tiles;
    p.X = src[i]; p.x_ks = P;
    p.Y = dst[i]; p.y_ms = P;
    p.part = w.part;
    if (i == 0) {
      MM_TRY(gemm_simt_launch<XM_DIRECT>(p, st));
    } else {
      p.sc = (i == 1) ? w.sc1 : w.sc;
      p.sh = (i == 1) ? w.sh1 : w.sh;
      MM_TRY(gemm_simt_launch<XM_NORM_RELU>(p, st));
    }
    MM_TRY(stats_reduce(w.part, cout[i], pairs, 0, w.gstart, w.stats, st));
    MM_TRY(gn_finalize(w.stats, q[2], q[3], w.cnt, 0, pairs, cout[i], 1, i == 0 ? w.sc1 : w.sc,
                       i == 0 ? w.sh1 : w.sh, st));
  }
  // per-detection mean of the 1024-d feature (reference point_net.py:140-146)
  segment_mean_kernel<<<mm_cdiv(1024L * ndet * 32, 256), 256, 0, st>>>(w.big, P, det_split, w.sc, w.sh,
                                                                       1024, ndet, L, w.gmean);
  MM_LAUNCH_CHECK();
  // U = Wh[:,64:] * gmean  (the per-detection part of point_net.py:27-28's conv1)
  {
    GemmP p = gemm_defaults();
    p.Wt = wts->w[MMMOT_W_PN_WHGT]; p.ldw = 512; p.M = 512; p.K = 1024;
    p.S = ndet; p.tiles_per_group = mm_cdiv(ndet, 128); p.num_tiles = p.tiles_per_group;
    p.X = w.gmean; p.x_ks = ndet;
    p.Y = w.u; p.y_ms = ndet;
    MM_TRY(gemm_simt_launch<XM_DIRECT>(p, st));
  }
  // head: Wh[:, :64] * x_local + U[:, det(p)] + b -> GroupNorm(512,512) -> ReLU -> per-detection mean
  {
    GemmP p = gemm_defaults();
    p.Wt = wts->w[MMMOT_W_PN_WHAT]; p.bias = wts->w[MMMOT_W_PN_BH]; p.ldw = 512; p.M = 512; p.K = 64;
    p.tile_tab = w.tiles; p.num_tiles = (int)n_tiles;
    p.X = w.y1; p.x_ks = P; p.sc = w.sc1; p.sh = w.sh1;
    p.Y = w.big; p.y_ms = P;
    p.part = w.part;
    p.addend = w.u; p.seg = w.seg; p.ld_add = ndet;
    MM_TRY(gemm_simt_launch<XM_NORM_RELU>(p, st));
    MM_TRY(stats_reduce(w.part, 512, pairs, 0, w.gstart, w.stats, st));
    MM_TRY(gn_finalize(w.stats, wts->w[MMMOT_W_PN_GHW], wts->w[MMMOT_W_PN_GHB], w.cnt, 0, pairs, 512, 1,
                       w.sc, w.sh, st));
    segment_mean_kernel<<<mm_cdiv(512L * ndet * 32, 256), 256, 0, st>>>(w.big, P, det_split, w.sc, w.sh,
                                                                        512, ndet, L, w.hmean, head_mask);
    MM_LAUNCH_CHECK();
  }
  // conv2 512 -> 512 over the pair's L detections, GroupNorm(16,512), ReLU (point_net.py:40-41)
  GemmP p = gemm_defaults();
  p.Wt = wts->w[MMMOT_W_PN_WOT]; p.bias = wts->w[MMMOT_W_PN_BO]; p.ldw = 512; p.M = 512; p.K = 512;
  p.S = L; p.tiles_per_group = mm_cdiv(L, 128); p.num_tiles = p.tiles_per_group * pairs;
  p.X = w.hmean; p.x_gs = L; p.x_ks = ndet;
  p.Y = w.o; p.y_gs = L; p.y_ms = ndet;
  p.part = w.part;
  MM_TRY(gemm_simt_launch<XM_DIRECT>(p, st));
  MM_TRY(stats_reduce(w.part, 512, pairs, p.tiles_per_group, nullptr, w.stats, st));
  MM_TRY(gn_finalize(w.stats, wts->w[MMMOT_W_PN_GOW], wts->w[MMMOT_W_PN_GOB], nullptr, L, pairs, 512, 32,
                     w.sc, w.sh, st));
  pointnet_out_kernel<<<mm_cdiv(512L * ndet, 256), 256, 0, st>>>(w.o, w.sc, w.sh, ndet, L, feats);
  MM_LAUNCH_CHECK();
  return 0;
}

}  // namespace

// engine choice from the per-pair shape only (see appearance.cu)
static bool pointnet_use_tc(int L) { return mm_use_tc(L >= 16); }

extern "C" size_t mmmot_pointnet_workspace(int pairs, int L, long p_total) {
  MmArena a(nullptr, 0);
  carve(a, pairs, L, p_total, pointnet_use_tc(L));
  return a.off;
}

extern "C" size_t mmmot_pointnet_train_workspace(int pairs, int L, long p_total) {
  MmArena a(nullptr, 0);
  carve(a, pairs, L, p_total, false);
  return a.off;
}

// mmmot_debug_stage_layout, stage 2: where mmmot_pointnet_fwd leaves its intermediates (a dry carve; no CUDA call)
int mm_pointnet_layout(int pairs, int L, long P, size_t* off, int* tensor_cores) {
  MmArena a(nullptr, 0);
  const bool use_tc = pointnet_use_tc(L);
  const PnWs w = carve(a, pairs, L, P, use_tc);
  const void* const bufs[26] = {w.xt, w.y1, w.t0, w.t1, w.big, w.segsum, w.x1p, w.xp, w.gmean, w.u, w.ut, w.hmean, w.o,
                                w.sc1, w.sh1, w.sc, w.sh, w.stats, w.mom, w.part, w.gstart, w.sstart, w.seg, w.cnt,
                                w.tiles, w.ctab};
  for (int i = 0; i < 26; i++) off[i] = (size_t)reinterpret_cast<uintptr_t>(bufs[i]);
  off[26] = a.off;
  if (tensor_cores) *tensor_cores = use_tc ? 1 : 0;
  return 0;
}

// train: FP32 engine; head_mask (optional) = the Dropout mask of the head activation, [512][P] with values {0, 1/(1-p)}
static int pointnet_impl(const mmmot_weights* wts, const float* points, const int* det_split, const int* h_det_split,
                         int pairs, int L, float* feats, void* workspace, size_t workspace_bytes, void* stream, bool train,
                         const float* head_mask) {
  if (!wts || !points || !det_split || !h_det_split || !feats || !workspace || pairs <= 0 || L <= 0)
    return MMMOT_E_ARG;
  // points [P][point_channels]: xyz, or xyz + reflectance in 16-byte rows
  if (wts->point_channels != 3 && !(wts->point_channels == 4 && (reinterpret_cast<uintptr_t>(points) & 15) == 0))
    return MMMOT_E_ARG;
  const bool use_tc = !train && pointnet_use_tc(L);
  const int tw = use_tc ? tc::BN : 128;
  PnShape s;
  MM_TRY(pn_shape(h_det_split, pairs, L, tw, s));
  MmArena ar(workspace, workspace_bytes);
  const PnWs w = carve(ar, pairs, L, s.P, use_tc);
  if (!ar.ok() || s.n_tiles > s.max_tiles) return MMMOT_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  MM_TRY(pn_tables(det_split, pairs, L, s.P, tw, s.n_tiles, w.cnt, w.gstart, w.tiles, w.seg, use_tc ? w.ctab : nullptr, st));
  if (use_tc) return pointnet_tc(wts, points, det_split, h_det_split, pairs, L, s.P, s.n_tiles, w, ar.status(), feats, st);
  return pointnet_fp32(wts, points, det_split, pairs, L, s.P, s.n_tiles, w, head_mask, feats, st);
}

extern "C" int mmmot_pointnet_fwd(const mmmot_weights* wts, const float* points, const int* det_split,
                                  const int* h_det_split, int pairs, int L, float* feats,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  return pointnet_impl(wts, points, det_split, h_det_split, pairs, L, feats, workspace, workspace_bytes, stream, false, nullptr);
}

extern "C" int mmmot_pointnet_train_fwd(const mmmot_weights* wts, const float* points, const int* det_split,
                                        const int* h_det_split, int pairs, int L, const float* head_drop_mask, float* feats,
                                        void* workspace, size_t workspace_bytes, void* stream) {
  return pointnet_impl(wts, points, det_split, h_det_split, pairs, L, feats, workspace, workspace_bytes, stream, true,
                       head_drop_mask);
}

// PointNet's tables over ragged per-pair point ranges (pn_tables, 256-point tiles as on the tensor-core path), then
// optionally one matrix-mode contraction on them exactly as the tensor-core path issues it: FP16 planes X[2][P][K], tile
// table, and per launch Y / part (statistics), addend (head) or segsum (second passes).
extern "C" int mmmot_debug_pn_contraction(const int* det_split, const int* h_det_split, int pairs, int L, long max_tiles,
                                          void* tiles, int* cnt, int* gstart, int* seg, void* ctab, long* n_tiles,
                                          const void* Wp, float wp_scale, const float* bias, int M, int K, const void* Xhi,
                                          float* Y, void* part, const float* addend, int ld_add,
                                          unsigned long long* segsum, const float* sc, const float* sh, void* stream) {
  if (!det_split || !h_det_split || pairs <= 0 || L <= 0 || !tiles || !cnt || !gstart || !seg || !ctab) return MMMOT_E_ARG;
  PnShape s;
  MM_TRY(pn_shape(h_det_split, pairs, L, tc::BN, s));
  if (n_tiles) *n_tiles = s.n_tiles;
  if (s.n_tiles > max_tiles) return MMMOT_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  MM_TRY(pn_tables(det_split, pairs, L, s.P, tc::BN, s.n_tiles, cnt, gstart, (int4*)tiles, seg, (int4*)ctab, st));
  if (!Wp) return 0;
  if (!Xhi) return MMMOT_E_ARG;
  GemmP p = gemm_defaults();
  p.bias = bias; p.M = M; p.K = K;
  p.tile_tab = (const int4*)tiles; p.num_tiles = (int)s.n_tiles;
  p.Y = Y; p.y_ms = M;
  p.part = (double2*)part;
  p.addend = addend; p.ld_add = ld_add;
  p.sc = sc; p.sh = sh;
  if (addend || segsum) p.seg = seg;
  return gemm_tma_launch_mat(p, (const uint4*)Wp, wp_scale, (const __half*)Xhi, s.P * K, s.P, K, tc::OUT_CL, 0, st, segsum,
                             nullptr, (const int4*)ctab);
}

// The GroupNorm statistics of PointNet's widest layers exactly as the tensor-core path computes them (pn_wide_stats under the
// current debug bits), then gn_finalize.  The workspace is a PointNet one (mmmot_pointnet_workspace(pairs, L, P)).
extern "C" int mmmot_debug_pn_stats(const int* det_split, const int* h_det_split, int pairs, int L, const void* Xhi, int K,
                                    const float* Wt, const void* Wp, float wp_scale, const float* bias, int M,
                                    const float* addend, const float* gamma, const float* beta, float* sc, float* sh,
                                    double* stats, double* mom, unsigned long long* detsum, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (!det_split || !h_det_split || pairs <= 0 || L <= 0 || !Xhi || !bias || !gamma || !beta || !sc || !sh || !workspace)
    return MMMOT_E_ARG;
  if (!(K == 64 || (K == 128 && !addend)) || M <= 0 || M > 1024 || M % 64) return MMMOT_E_ARG;
  const bool two_pass = mm_debug_flags() & MM_DBG_PN_STATS_PASS;
  if (two_pass ? !Wp : !Wt) return MMMOT_E_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int ndet = pairs * L;
  PnShape s;
  MM_TRY(pn_shape(h_det_split, pairs, L, tc::BN, s));
  MmArena ar(workspace, workspace_bytes);
  const PnWs w = carve(ar, pairs, L, s.P, true);
  if (!ar.ok() || s.n_tiles > s.max_tiles) return MMMOT_E_WORKSPACE;
  MM_TRY(pn_tables(det_split, pairs, L, s.P, tc::BN, s.n_tiles, w.cnt, w.gstart, w.tiles, w.seg, w.ctab, st));
  MM_TRY(pn_wide_stats(w, h_det_split, det_split, s.P, pairs, L, s.n_tiles, (const __half*)Xhi, K, Wt, (const uint4*)Wp,
                       wp_scale, bias, M, addend, st));
  MM_TRY(gn_finalize(w.stats, gamma, beta, w.cnt, 0, pairs, M, 1, sc, sh, st));
  if (stats) MM_CUDA(cudaMemcpyAsync(stats, w.stats, (size_t)pairs * M * 2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (mom && !two_pass)
    MM_CUDA(cudaMemcpyAsync(mom, w.mom, (size_t)pairs * (K * K + K) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (detsum && K == 64 && !two_pass)
    MM_CUDA(cudaMemcpyAsync(detsum, w.segsum, (size_t)ndet * 64 * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
  return 0;
}
