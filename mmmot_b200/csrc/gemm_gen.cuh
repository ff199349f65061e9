// Tensor-core contraction engine, GENERATED-operand variant (sm_90a, wgmma): the affinity MLP.
//
// Same arithmetic as gemm_tma.cuh (FP16 hi/lo split operands, 3 MMAs per k-step, FP32 accumulate) but the
// activation operand never exists in HBM in operand form: eight producer warps build each [256 columns x 32 k]
// FP16 hi/lo block in shared memory, in the canonical K-major layout, from
//   GEN_PAIR_*  the two feature slabs of the frame-pair:  x[(i,j)][k] = f[i][k] (*|-) f[N+j][k]   (reference
//               modules/gcn.py:6-41; the 3 x 512 x N x M tensor is never stored), or
//   GEN_NORM    the previous layer's fp32 output:  x[s][k] = relu(y[s][k]*sc[g][k] + sh[g][k])   (GroupNorm + ReLU of
//               the producer layer applied on the fly; no normalised copy of the activation is ever written), or
//   GEN_COPY    an fp32 channels-last activation as it is (the small per-detection contractions: fusion, w_det).
// All activations are channels-last ([row][channel]).  A producer thread owns one 8-wide k group of four columns per
// chunk: one 256-bit load per (column, source) — a quarter warp reads eight rows, the four quarters the four k groups
// of the same 128-byte lines — and one 16-byte shared-memory store per (column, plane); the epilogue writes a warp's
// 32 channels of one column as one 128-byte line.  (Load/store instructions and their L1 wavefronts, not the FP32
// pipe, are what the producers compete for with the epilogue.)
//
// CTA (512 threads, persistent, one per SM): warps 0-7 are two consumer warpgroups (warpgroup h issues the wgmma chains
// of the tile's 128 rows x column half h and runs that half's epilogue), warps 8-15 operand producers; the first
// producer thread also fetches each chunk's pre-tiled FP16 hi/lo weight block (cp.async.bulk) and, for the pairwise
// producers at m == 128, the chunk's fp32 sources (TMA, see gemm_gen_kernel).  One mbarrier per stage collects the
// weight expect_tx and the eight producer warps' arrivals.  The consumers hold 128 accumulator registers
// each and take registers from the producers (setmaxnreg).  The accumulator image of a finished tile overlays
// stages 0-1 of the ring, so the producers start the next tile once the epilogue has read it.
#pragma once
#include "gemm_tma.cuh"

namespace gen {

using namespace tc;

enum { GEN_PAIR_MUL = 0, GEN_PAIR_ABS = 1, GEN_PAIR_SUB = 2, GEN_NORM = 3, GEN_COPY = 4 };   // GEN_PAIR_* == MMMOT_AFF_*

constexpr int G_EPI_WARPS = 8, G_PROD_WARP0 = 8, G_PROD_WARPS = 8;
constexpr int G_THREADS = (G_PROD_WARP0 + G_PROD_WARPS) * 32;   // 512
constexpr int G_CONS_REGS = 176, G_PROD_REGS = 80;
static_assert(256 * G_CONS_REGS + 256 * G_PROD_REGS <= launch_regs(G_THREADS) * G_THREADS, "register split exceeds the CTA's pool");
// Staged pairwise sources (PAIRED GEN_PAIR_*): per stage, the chunk's [128 detections x 32 channels] fp32 box in the
// stage's otherwise unused 16 KB slot at A_SUB (128-byte swizzle), and the two object rows [2 x 32] fp32 beside the
// barriers (G_OBJ_BYTES per stage).
constexpr int G_DET_BYTES = 128 * BK * 4, G_OBJ_BYTES = 2 * BK * 4;
static_assert(G_DET_BYTES == A_SUB && A_SUB % 1024 == 0, "the detection box fills the stage's free 1024-aligned slot");
constexpr int G_SRC_AHEAD = STAGES - 1;   // chunks whose sources are in flight while the producers convert one
constexpr size_t G_SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 + 256 + STAGES * G_OBJ_BYTES;
constexpr int G_MAX_K = 512;   // producer-side GroupNorm affine staged in shared memory
__host__ __device__ constexpr bool staged(int GEN, bool PAIRED) { return PAIRED && GEN <= GEN_PAIR_SUB; }

struct GenP {
  TcP t;               // .g: M, K, bias, S (columns per group), tiles_per_group, num_tiles, Y / y_gs / y_ms (fp32
                       // channels-last: row = g*y_gs + column), part
  const float* src;    // PAIR: fcl [G][Lf][K] channels-last feature stacks; NORM: fp32 channels-last [G*S][ld_src]
  int ld_src;          // NORM: floats per source row (its first K channels are read)
  const float* gsc;    // NORM: GroupNorm affine of the SOURCE layer, [G][K]
  const float* gsh;
  int n, m, Lf;        // PAIR: columns s = i*m + j, objs = feature rows [0, n), dets = [n, n + m), Lf = n + m
  // FP16 range: the producers do not track the magnitudes they convert (their instruction stream is the kernel's
  // bottleneck); the callers bound the operand instead — PAIR: feats_cl_check_kernel on the feature stacks, NORM:
  // gn_finalize's bound sqrt(count)*|gamma| + |beta| on the normalised values (both raise the status flag).
};

__device__ __forceinline__ void lds128(uint32_t addr, float4& v) {
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
}
__device__ __forceinline__ void ld_global_256(const float* p, float (&v)[8]) {
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%8];\n\tld.global.nc.v4.f32 {%4, %5, %6, %7}, [%8+16];"
               : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]), "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7])
               : "l"(p));
}

// PAIRED: pipelined producers.  GEN_PAIR_*: only for m == 128, where a 256-column tile is two whole object rows i0,
// i0 + 1 against all 128 detections and the thread's four items are {row i0, row i0 + 1} x {j = cb, j = cb + 64}.  The
// chunk's sources (the detection box and the two object rows, map_det / map_obj) are staged in shared memory by TMA,
// G_SRC_AHEAD chunks ahead of the conversion; the producers hold no prefetch in registers.
// GEN_NORM, GEN_COPY: the next chunk's source vectors are loaded into registers before the current chunk is converted
// (any shape; GEN_NORM then re-reads the GroupNorm affine from shared memory per pair of items).
template <int GEN, bool PAIRED>
static __global__ void __launch_bounds__(G_THREADS, 1)
gemm_gen_kernel(const GenP P, const __grid_constant__ CUtensorMap map_det, const __grid_constant__ CUtensorMap map_obj) {
  const GemmP& p = P.t.g;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(16) float s_gsc[GEN == GEN_NORM ? G_MAX_K : 4], s_gsh[GEN == GEN_NORM ? G_MAX_K : 4];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t bar0 = base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (STAGES + s); };
  const uint32_t free_bar = bar0 + 8u * (2 * STAGES);   // the epilogue has read the accumulator image
  // staged sources: src_full(s) collects the TMA bytes of stage s's sources, src_empty(s) one arrive per producer warp
  // once it has converted them
  auto src_full = [&](int s) { return bar0 + 8u * (2 * STAGES + 1 + s); };
  auto src_empty = [&](int s) { return bar0 + 8u * (3 * STAGES + 1 + s); };
  const uint32_t obj0 = bar0 + 256;                       // object rows, G_OBJ_BYTES per stage
  float* img = reinterpret_cast<float*>(sm);              // accumulator image [128][BN] fp32 over stages 0-1

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mgroups = P.t.m_tiles;
  const long total_tiles = (long)p.num_tiles * mgroups;
  const int KC = P.t.k_chunks;

  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(full_bar(s), 1 + G_PROD_WARPS);   // weight expect_tx arrive + one arrive per producer warp
      mbar_init(empty_bar(s), G_EPI_WARPS);       // one arrive per consumer warp once its wgmmas have read the stage
      if (staged(GEN, PAIRED)) {
        mbar_init(src_full(s), 1);
        mbar_init(src_empty(s), G_PROD_WARPS);
      }
    }
    mbar_init(free_bar, G_EPI_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // column tile -> group / first column / valid length
  // (table tiling: {group, first ABSOLUTE row, length}; x_gs and y_gs are 0 then)
  auto tile_cols = [&](int nt, int& g, int& c0, int& len) {
    if (p.tile_tab) { const int4 tt = p.tile_tab[nt]; g = tt.x; c0 = tt.y; len = tt.z; return; }
    g = nt / p.tiles_per_group;
    c0 = (nt - g * p.tiles_per_group) * BN;
    len = min(BN, p.S - c0);
  };

  if (warp < G_EPI_WARPS) {
    // =============================== CONSUMERS: wgmma + epilogue ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(G_CONS_REGS));
    const int q = warp & 3, half = warp >> 2;
    uint32_t it = 0;
    float acc[2][64];      // rows 64 mb + fragment row, columns 128 half + fragment column
    auto clear_acc = [&]() {
#pragma unroll
      for (int mb = 0; mb < 2; mb++)
#pragma unroll
        for (int i = 0; i < 64; i++) acc[mb][i] = 0.f;
    };
    if (!staged(GEN, PAIRED)) clear_acc();
    for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int mg = (int)(t % mgroups);
      const int nt = (int)(t / mgroups);
      int g, c0, len;
      tile_cols(nt, g, c0, len);
      // The first wgmma of each chain ignores the accumulators (scale_d = 0).  Staged pairwise variant: clearing them
      // here rather than once per CTA leaves them dead from the image dump to the next tile, so the epilogue has their
      // registers (no spills).
      if (staged(GEN, PAIRED)) clear_acc();
      for (int kc = 0; kc < KC; kc++, it++) {
        const int s = it % STAGES;
        mbar_wait(full_bar(s), (it / STAGES) & 1);
        const uint32_t sa = base + s * STAGE_BYTES, sb = sa + 2 * A_SUB + half * (128 / 8) * 128;
        if (!(P.t.dbg & 8)) {
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 2; ks++) {
            const uint64_t b_hi = smem_desc(sb + ks * 2 * B_LBO, B_LBO, SBO);
            const uint64_t b_lo = smem_desc(sb + B_HALF + ks * 2 * B_LBO, B_LBO, SBO);
#pragma unroll
            for (int mb = 0; mb < 2; mb++) {
              const uint32_t a = sa + mb * 8 * SBO + ks * 2 * A_LBO;
              const uint64_t a_hi = smem_desc(a, A_LBO, SBO), a_lo = smem_desc(a + A_HALF, A_LBO, SBO);
              wgmma_n128(acc[mb], a_hi, b_hi, (kc | ks) ? 1u : 0u);
              wgmma_n128(acc[mb], a_hi, b_lo, 1u);
              wgmma_n128(acc[mb], a_lo, b_hi, 1u);
            }
          }
          wgmma_commit();
        }
        wgmma_wait<1>();   // the previous chunk's wgmmas are done: release its stage
        if (kc > 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar((it - 1) % STAGES)); }
      }
      wgmma_wait<0>();
      fence_acc(acc[0]);
      fence_acc(acc[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar((it - 1) % STAGES));
      bar_sync(7, G_EPI_WARPS * 32);   // both warpgroups are past their wgmmas: stages 0-1 may be overwritten
      acc_dump(acc[0], img, BN, 0, half * 128);
      acc_dump(acc[1], img, BN, 64, half * 128);
      bar_sync(7, G_EPI_WARPS * 32);
      {
        const int co = mg * 128 + q * 32 + lane;
        const bool rowok = co < p.M;
        const float bv = (rowok && p.bias) ? __ldg(p.bias + co) : 0.f;
        double f1 = 0.0, f2 = 0.0;   // (sum, sum of squares) over this thread's 128 columns: four shifted chunk sums
        // channels-last: a warp's 32 consecutive channels of one column are one 128-byte line
        float* dst = p.Y + ((long)g * p.y_gs + c0 + half * 128) * p.y_ms + co;
#pragma unroll 1
        for (int cc = 0; cc < 4; cc++) {
          const int col0 = half * 128 + cc * 32;
          if (col0 >= len) break;   // warp-uniform
          uint32_t v[32];
          acc_ld32(img, BN, q * 32 + lane, col0, v);
          if (P.t.dbg & 1) continue;
          float s1 = 0.f, s2 = 0.f, pv = 0.f;
          if (col0 + 32 <= len) {
            if (p.relu) epi_fast<true>(v, P.t.out_scale, bv, pv, s1, s2);
            else epi_fast<false>(v, P.t.out_scale, bv, pv, s1, s2);
          } else {
            float t = 0.f;
#pragma unroll
            for (int j = 0; j < 32; j++) {
              float x = fmaf(__uint_as_float(v[j]), P.t.out_scale, bv);
              if (p.relu) x = fmaxf(x, 0.f);
              v[j] = __float_as_uint(x);
              if (col0 + j < len) t += x;            // columns beyond the group are not counted (and not stored)
            }
            pv = t / (float)(len - col0);
#pragma unroll
            for (int j = 0; j < 32; j++)
              if (col0 + j < len) { const float d = __uint_as_float(v[j]) - pv; s1 += d; s2 = fmaf(d, d, s2); }
          }
          stat_fold(f1, f2, min(32, len - col0), pv, s1, s2);
          if (p.Y && rowok) {
            float* d = dst + (long)cc * 32 * p.y_ms;
            if (col0 + 32 <= len) {
#pragma unroll
              for (int j = 0; j < 32; j++) { *d = __uint_as_float(v[j]); d += p.y_ms; }
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (col0 + j < len) d[(long)j * p.y_ms] = __uint_as_float(v[j]);
            }
          }
        }
        if (p.part && rowok) p.part[((long)nt * 2 + half) * p.M + co] = make_double2(f1, f2);
      }
      fence_async_smem();   // the image's generic-proxy reads precede the next tile's operand and weight writes
      __syncwarp();
      if (lane == 0) mbar_arrive(free_bar);
    }
  } else {
    // =============================== OPERAND PRODUCERS (+ weight loads) ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(G_PROD_REGS));
    // thread = (k group kg of 8, four columns cb + 64 r).  Per chunk every item is converted, split into FP16 hi/lo
    // and written as one 16-byte piece per plane of the canonical K-major layout:
    //   byte offset = kg * B_LBO + (column / 8) * 128 + (column % 8) * 16
    // (a quarter warp = one kg, eight consecutive columns -> 128 contiguous bytes: conflict-free).
    // PAIRED GEN_NORM / GEN_COPY: the 256-bit source loads of chunk c+1 are issued before chunk c is converted (two
    // register sets, ping-pong), so the L2 transfer of one chunk overlaps the conversion of the previous one; the generic
    // pairwise variant (8 source vectors per chunk) has no registers for that and only overlaps its loads with the wait
    // for the ring slot.  PAIRED GEN_PAIR_*: the sources come through shared memory (STAGED, below).
    constexpr bool STAGED = staged(GEN, PAIRED);
    constexpr bool PREFETCH = PAIRED && !STAGED;
    constexpr bool ROWS = GEN == GEN_NORM || GEN == GEN_COPY;      // the operand is a function of one fp32 source row
    constexpr int NA = (ROWS || !PAIRED) ? 4 : 2;                  // source vectors of 8 floats per chunk: a / y ...
    constexpr int NB = ROWS ? 0 : (PAIRED ? 2 : 4);                // ... and b
    const int pt = tid - G_PROD_WARP0 * 32;   // 0..255
    const int kg = (pt >> 3) & 3;
    const int cb = (pt & 7) + 8 * (pt >> 5);
    const uint32_t off0 = (uint32_t)kg * B_LBO + (uint32_t)(cb >> 3) * 128u + (uint32_t)(cb & 7) * 16u;   // + r * 1024
    uint32_t it = 0, wcount = 0;
    int g_staged = -1;
    struct Raw { float a[NA][8]; float b[NB ? NB : 1][8]; };
    for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int mg = (int)(t % mgroups);
      const int nt = (int)(t / mgroups);
      int g, c0, len;
      tile_cols(nt, g, c0, len);
      if (wcount > 0) mbar_wait(free_bar, (wcount - 1) & 1);   // the previous tile's accumulator image has been read
      wcount++;
      unsigned okmask = 0;
      // 32-bit element offsets of the items' rows (this thread's k group) relative to the tile's / group's base
      const float* tbase = ROWS ? P.src + ((long)g * p.x_gs + c0) * P.ld_src : P.src + (long)g * P.Lf * p.K;
      int oa[NA], ob[NB ? NB : 1];
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int col = cb + 64 * r;
        if (col < len) okmask |= 1u << r;
        const int cc = min(col, len - 1);
        if (ROWS) {
          oa[r] = cc * P.ld_src + kg * 8;
        } else {
          const int s = c0 + cc;
          const int i = s / P.m, j = s - i * P.m;
          if (!PAIRED) {
            oa[r] = i * p.K + kg * 8;
            ob[r] = (P.n + j) * p.K + kg * 8;
          } else {
            if (!(r & 1)) oa[r >> 1] = i * p.K + kg * 8;          // r = 0, 2: the two rows i
            if (r < 2) ob[r] = (P.n + j) * p.K + kg * 8;          // r = 0, 1: the two detections j
          }
        }
      }
      if (GEN == GEN_NORM && g != g_staged) {   // same decision in every producer thread: stage the group's affine
        asm volatile("bar.sync 1, %0;" ::"n"(G_PROD_WARPS * 32) : "memory");   // previous tile's readers are done
        for (int k = pt; k < p.K; k += G_PROD_WARPS * 32) {
          s_gsc[k] = __ldg(P.gsc + (long)g * p.K + k);
          s_gsh[k] = __ldg(P.gsh + (long)g * p.K + k);
        }
        asm volatile("bar.sync 1, %0;" ::"n"(G_PROD_WARPS * 32) : "memory");
        g_staged = g;
      }
      auto load = [&](Raw& R, int kc) {
        if (P.t.dbg & 4) return;
#pragma unroll
        for (int r = 0; r < NA; r++) ld_global_256(tbase + oa[r] + kc * BK, R.a[r]);
#pragma unroll
        for (int r = 0; r < NB; r++) ld_global_256(tbase + ob[r] + kc * BK, R.b[r]);
      };
      // wait for the ring slot, convert + store the chunk, publish it
      auto emit = [&](const Raw& R, int kc) {
        const int s = it % STAGES;
        mbar_wait(empty_bar(s), ((it / STAGES) & 1) ^ 1u);
        if (pt == 0) {   // the chunk's weight block
          if (P.t.dbg & 2) {
            mbar_arrive(full_bar(s));
          } else {
            mbar_expect_tx(full_bar(s), A_SUB);
            bulk_g2s(base + s * STAGE_BYTES, reinterpret_cast<const uint8_t*>(P.t.Wp) + ((size_t)kc * P.t.m_tiles + mg) * A_SUB,
                     A_SUB, full_bar(s));
          }
        }
        uint8_t* bh = sm + s * STAGE_BYTES + 2 * A_SUB + off0;
        if (!(P.t.dbg & 4)) {
          const uint32_t sca = smem_u32(s_gsc + kc * BK + kg * 8), sha = smem_u32(s_gsh + kc * BK + kg * 8);
          float4 sc0, sc1, sh0, sh1;
#pragma unroll
          for (int r = 0; r < 4; r++) {
            float x[8];
            if (GEN == GEN_NORM) {
              const float(&y)[8] = R.a[r];
              // prefetching variant: the affine is re-read from shared memory per pair of items (volatile asm) instead
              // of holding the eight (scale, shift) pairs across the chunk: 16 registers for the prefetched vectors
              if (!PAIRED ? r == 0 : !(r & 1)) { lds128(sca, sc0); lds128(sca + 16, sc1); lds128(sha, sh0); lds128(sha + 16, sh1); }
              x[0] = fmaxf(fmaf(y[0], sc0.x, sh0.x), 0.f); x[1] = fmaxf(fmaf(y[1], sc0.y, sh0.y), 0.f);
              x[2] = fmaxf(fmaf(y[2], sc0.z, sh0.z), 0.f); x[3] = fmaxf(fmaf(y[3], sc0.w, sh0.w), 0.f);
              x[4] = fmaxf(fmaf(y[4], sc1.x, sh1.x), 0.f); x[5] = fmaxf(fmaf(y[5], sc1.y, sh1.y), 0.f);
              x[6] = fmaxf(fmaf(y[6], sc1.z, sh1.z), 0.f); x[7] = fmaxf(fmaf(y[7], sc1.w, sh1.w), 0.f);
            } else if (GEN == GEN_COPY) {
#pragma unroll
              for (int e = 0; e < 8; e++) x[e] = R.a[r][e];
            } else {
              const float(&av)[8] = R.a[PAIRED ? (r >> 1) : r];
              const float(&bv)[8] = R.b[NB ? (PAIRED ? (r & 1) : r) : 0];
#pragma unroll
              for (int e = 0; e < 8; e++) {
                if (GEN == GEN_PAIR_MUL) x[e] = av[e] * bv[e];
                else if (GEN == GEN_PAIR_ABS) x[e] = fabsf(av[e] - bv[e]) * 0.5f;   // == |(a - b) / 2| exactly; |.| folds into the FMUL
                else x[e] = (av[e] - bv[e]) * 0.5f;
              }
            }
            uint32_t h[4], l[4];
#pragma unroll
            for (int q = 0; q < 4; q++) split_f16x2(x[2 * q], x[2 * q + 1], h[q], l[q]);
            if (!((okmask >> r) & 1u)) { h[0] = h[1] = h[2] = h[3] = 0u; l[0] = l[1] = l[2] = l[3] = 0u; }   // beyond the group
            *reinterpret_cast<uint4*>(bh + r * 1024) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4*>(bh + B_HALF + r * 1024) = make_uint4(l[0], l[1], l[2], l[3]);
          }
        }
        fence_async_smem();   // generic-proxy writes -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(full_bar(s));
        it++;
      };
      if (STAGED) {
        // Per chunk, the first producer thread loads the detection box [128 rows x 32 channels] (rows g*Lf + n ..,
        // 128-byte swizzle: 16-byte unit u of box row j at unit u ^ (j & 7)) into the stage's free slot at A_SUB and the
        // two object rows i0, i0 + 1 into the stage's object area, G_SRC_AHEAD chunks ahead.  The slot of chunk c + 2
        // was last read by chunk c - 1, so the refill waits only for every producer warp to be done with that one.
        // A quarter warp's eight detections j = cb + 64 b share a k group and have eight different j & 7: its 16-byte
        // reads hit eight different bank groups.
        const bool gen_ops = !(P.t.dbg & 4);
        const int row_det = g * P.Lf + P.n, row_obj = g * P.Lf + c0 / P.m;
        auto issue = [&](uint32_t pos, int kc) {
          const int s = pos % STAGES;
          mbar_wait(src_empty(s), ((pos / STAGES) & 1) ^ 1u);
          mbar_expect_tx(src_full(s), G_DET_BYTES + G_OBJ_BYTES);
          tma::tma_load_2d(base + s * STAGE_BYTES + A_SUB, &map_det, kc * BK, row_det, src_full(s));
          tma::tma_load_2d(obj0 + s * G_OBJ_BYTES, &map_obj, kc * BK, row_obj, src_full(s));
        };
        if (pt == 0 && gen_ops)
          for (int kc = 0; kc < KC && kc < G_SRC_AHEAD; kc++) issue(it + kc, kc);
        const uint32_t u0 = (uint32_t)(((2 * kg) ^ (cb & 7)) * 16), u1 = (uint32_t)(((2 * kg + 1) ^ (cb & 7)) * 16);
        for (int kc = 0; kc < KC; kc++) {
          const int s = it % STAGES;
          mbar_wait(empty_bar(s), ((it / STAGES) & 1) ^ 1u);
          if (pt == 0) {   // the chunk's weight block
            if (P.t.dbg & 2) {
              mbar_arrive(full_bar(s));
            } else {
              mbar_expect_tx(full_bar(s), A_SUB);
              bulk_g2s(base + s * STAGE_BYTES, reinterpret_cast<const uint8_t*>(P.t.Wp) + ((size_t)kc * P.t.m_tiles + mg) * A_SUB,
                       A_SUB, full_bar(s));
            }
          }
          if (gen_ops) {
            uint8_t* bh = sm + s * STAGE_BYTES + 2 * A_SUB + off0;
            const uint32_t db = base + s * STAGE_BYTES + A_SUB + (uint32_t)cb * 128u, ob = obj0 + s * G_OBJ_BYTES + kg * 32;
            mbar_wait(src_full(s), (it / STAGES) & 1);
            float4 d[2][2];   // detections j = cb, cb + 64: channels kg*8 .. kg*8 + 7
            lds128(db + u0, d[0][0]); lds128(db + u1, d[0][1]);
            lds128(db + 64 * 128 + u0, d[1][0]); lds128(db + 64 * 128 + u1, d[1][1]);
#pragma unroll
            for (int a = 0; a < 2; a++) {
              float4 o[2];    // object row i0 + a (every lane of a k group reads the same 32 bytes: a broadcast)
              lds128(ob + a * BK * 4, o[0]); lds128(ob + a * BK * 4 + 16, o[1]);
              const float av[8] = {o[0].x, o[0].y, o[0].z, o[0].w, o[1].x, o[1].y, o[1].z, o[1].w};
#pragma unroll
              for (int b = 0; b < 2; b++) {
                const int r = 2 * a + b;
                const float bv[8] = {d[b][0].x, d[b][0].y, d[b][0].z, d[b][0].w, d[b][1].x, d[b][1].y, d[b][1].z, d[b][1].w};
                float x[8];
#pragma unroll
                for (int e = 0; e < 8; e++) {
                  if (GEN == GEN_PAIR_MUL) x[e] = av[e] * bv[e];
                  else if (GEN == GEN_PAIR_ABS) x[e] = fabsf(av[e] - bv[e]) * 0.5f;
                  else x[e] = (av[e] - bv[e]) * 0.5f;
                }
                uint32_t h[4], l[4];
#pragma unroll
                for (int q = 0; q < 4; q++) split_f16x2(x[2 * q], x[2 * q + 1], h[q], l[q]);
                if (!((okmask >> r) & 1u)) { h[0] = h[1] = h[2] = h[3] = 0u; l[0] = l[1] = l[2] = l[3] = 0u; }
                *reinterpret_cast<uint4*>(bh + r * 1024) = make_uint4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<uint4*>(bh + B_HALF + r * 1024) = make_uint4(l[0], l[1], l[2], l[3]);
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(src_empty(s));   // this warp is done with the stage's sources
          }
          fence_async_smem();   // generic-proxy writes -> visible to the tensor core (async proxy)
          __syncwarp();
          if (lane == 0) mbar_arrive(full_bar(s));
          if (pt == 0 && gen_ops && kc + G_SRC_AHEAD < KC) issue(it + G_SRC_AHEAD, kc + G_SRC_AHEAD);
          it++;
        }
      } else if (PREFETCH) {
        Raw R0, R1;
        load(R0, 0);
        for (int kc = 0; kc < KC; kc += 2) {
          if (kc + 1 < KC) load(R1, kc + 1);
          emit(R0, kc);
          if (kc + 1 < KC) {
            if (kc + 2 < KC) load(R0, kc + 2);
            emit(R1, kc + 1);
          }
        }
      } else {
        for (int kc = 0; kc < KC; kc++) {
          Raw R;
          load(R, kc);
          emit(R, kc);
        }
      }
    }
  }
}

}  // namespace gen

// Host launcher.  g: M, K (multiple of 32, <= 512 for GEN_NORM), bias, S / tiles_per_group / num_tiles (uniform column
// tiling, 256 columns per tile) or tile_tab (GEN_NORM, GEN_COPY: ragged groups, absolute rows), x_gs (NORM: source rows per group), Y / y_gs / y_ms = fp32 channels-last output (or
// null), part = two GroupNorm partials per tile (stats_reduce(..., mult = 2)).  Wp = weights packed by
// weights.py::pack_tc.  PAIR: src = fcl [G][Lf][K]; NORM: src = [G*x_gs][ld_src] fp32, gsc/gsh [G][K].
template <int GEN, bool PAIRED>
static int gemm_gen_launch_t(const GemmP& g, const uint4* Wp, float out_scale, const float* src, int ld_src,
                           const float* gsc, const float* gsh, int n, int m, int Lf, cudaStream_t st) {
  if (!Wp || !src || g.num_tiles <= 0 || g.K % tc::BK) return MMMOT_E_ARG;
  if (g.tile_tab && ((GEN != gen::GEN_NORM && GEN != gen::GEN_COPY) || g.x_gs || g.y_gs)) return MMMOT_E_ARG;
  if (GEN == gen::GEN_NORM && (g.K > gen::G_MAX_K || !gsc || !gsh)) return MMMOT_E_ARG;
  if ((GEN == gen::GEN_NORM || GEN == gen::GEN_COPY) && (ld_src < g.K || (ld_src & 7))) return MMMOT_E_ARG;
  int sms = 0;
  MM_TRY(mm_sm_count(&sms));
  static std::atomic<unsigned long long> attr{0};
  MM_TRY(mm_ensure_smem(gen::gemm_gen_kernel<GEN, PAIRED>, gen::G_SMEM_BYTES, attr));
  gen::GenP P;
  memset(&P, 0, sizeof(P));
  P.t.g = g;
  P.t.Wp = Wp;
  P.t.m_tiles = (g.M + 127) / 128;
  P.t.k_chunks = g.K / tc::BK;
  P.t.out_scale = out_scale;
  P.t.out_mode = tc::OUT_CL;
  P.t.dbg = mm_debug_flags();
  P.src = src; P.ld_src = ld_src; P.gsc = gsc; P.gsh = gsh;
  P.n = n; P.m = m; P.Lf = Lf;
  alignas(64) CUtensorMap map_det, map_obj;
  memset(&map_det, 0, sizeof(map_det));
  memset(&map_obj, 0, sizeof(map_obj));
  if (gen::staged(GEN, PAIRED)) {
    // two whole object rows per tile against all m = 128 detections; maps over the feature stacks [G * Lf][K]
    if (m != 128 || Lf != n + m || g.tile_tab || g.tiles_per_group <= 0) return MMMOT_E_ARG;
    const long rows = (long)(g.num_tiles / g.tiles_per_group) * Lf;
    MM_TRY(tma::make_map_2d_f32(&map_det, src, rows, g.K, 128, CU_TENSOR_MAP_SWIZZLE_128B));
    MM_TRY(tma::make_map_2d_f32(&map_obj, src, rows, g.K, 2, CU_TENSOR_MAP_SWIZZLE_NONE));
  }
  const long total = (long)g.num_tiles * P.t.m_tiles;
  const int grid = (int)(total < sms ? total : sms);
  gen::gemm_gen_kernel<GEN, PAIRED><<<grid, gen::G_THREADS, gen::G_SMEM_BYTES, st>>>(P, map_det, map_obj);
  MM_LAUNCH_CHECK();
  return 0;
}

// Producer variant gemm_gen_launch takes: the software-pipelined (prefetching, PAIRED) producers or the plain ones.
// Pure host logic, no CUDA call, so that tests can query it without a GPU (mmmot_debug_gen_prefetch).
// dbg: mmmot_set_debug state; bit 10 (1024) producers without the software pipeline (A/B runs), bit 12 (4096) GEN_NORM
// with it.  GEN_PAIR_* pipeline only at m == 128 (two whole rows per tile, see gemm_gen_kernel).
static inline bool gen_prefetch(int GEN, int m, int dbg) {
  if (dbg & 1024) return false;
  if (GEN == gen::GEN_NORM) return (dbg & 4096) != 0;
  if (GEN == gen::GEN_COPY) return true;
  return m == 128;
}

// Whether that variant stages the pairwise sources in shared memory by TMA (the pipelined GEN_PAIR_* producers).  Pure
// host logic, like gen_prefetch (mmmot_debug_gen_staged).
static inline bool gen_staged(int GEN, int m, int dbg) {
  return GEN <= gen::GEN_PAIR_SUB && gen_prefetch(GEN, m, dbg);
}

// prefetched (host, or NULL) receives the variant taken (gen_prefetch)
template <int GEN>
static int gemm_gen_launch(const GemmP& g, const uint4* Wp, float out_scale, const float* src, int ld_src,
                           const float* gsc, const float* gsh, int n, int m, int Lf, cudaStream_t st,
                           int* prefetched = nullptr) {
  const bool pipe = gen_prefetch(GEN, m, mm_debug_flags());
  if (prefetched) *prefetched = pipe ? 1 : 0;
  if (pipe) return gemm_gen_launch_t<GEN, true>(g, Wp, out_scale, src, ld_src, gsc, gsh, n, m, Lf, st);
  return gemm_gen_launch_t<GEN, false>(g, Wp, out_scale, src, ld_src, gsc, gsh, n, m, Lf, st);
}
