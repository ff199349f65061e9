// Tensor-core contraction engine, TMA-fed variant (sm_90a, wgmma).
//
// Same arithmetic as gemm_gen.cuh (FP16 hi/lo split operands, 3 MMAs per k-step, FP32 accumulate, fused epilogue)
// but the generated operand is not produced by threads: activations between tensor-core layers live in HBM as two
// FP16 planes (hi, lo), channels-last, and the TMA engine (cp.async.bulk.tensor, tiled mode, 64-byte swizzle) drops
// each [256 rows x 32 channels] box straight into shared memory in the wgmma K-major SWIZZLE_64B layout:
//   * 1x1 contraction: 2-D map [rows][C], box (32, 256)
//   * 3x3 convolution: 4-D map [img][H][W][C], box (32, bx, by, bi) with bx*by*bi = 256; the 9 taps are the
//     same box at shifted (x, y) coordinates and the zero padding is TMA's out-of-bounds fill — no im2col,
//     no boundary code, no index arithmetic on the SMs.
// CTA (384 threads, persistent, one per SM): warps 0-7 are two consumer warpgroups (warpgroup h issues the wgmma
// chains of the tile's 128 rows x column half h, then runs the epilogue of that half), warp 8 is the loader (weights
// by cp.async.bulk, operand boxes by TMA; warps 9-11 only complete its warpgroup).  Ring of 4 x 48 KB stages.
// gemm_tma_kernel<EPI> is instantiated once per consumer: EPI_MAT (mat_consumer, 1x1 contractions), EPI_CONV_IMAGE
// (conv_image_consumer: convs with GroupNorm partials, or under debug bit 11) and EPI_CONV_ACC (conv_acc_consumer: convs
// from the wgmma fragments, K segments included).  The first two hand each tile over as an accumulator image (128 x 256 fp32) over the
// ring's first 128 KB, so the loader starts the next tile once the epilogue has read it; their FP16 outputs are
// transposed through a per-warp smem scratch (store_rows) so each lane stores 64 contiguous bytes per plane.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace tma {

using namespace tc;

constexpr int T_THREADS = 384;
constexpr int T_EPI_WARPS = 8, T_LOAD_WARP = 8;   // warps 9-11 only complete the loader's warpgroup
constexpr int T_CONS_REGS = 232, T_LOAD_REGS = 40;
static_assert(256 * T_CONS_REGS + 128 * T_LOAD_REGS <= launch_regs(T_THREADS) * T_THREADS, "register split exceeds the CTA's pool");
constexpr int T_EPI_SCRATCH = 32 * 80;   // per epilogue warp: 32 pixels x (64 B of channels + 16 B pad)
// ring stage = one k chunk: the tile's weight block (hi | lo, 16 KB) and the operand box (hi, lo planes, 2 x 16 KB).
// Four such stages fill the shared memory three 64 KB stages would (tc::STAGE_BYTES has room for a second weight
// block this kernel never loads), so the loader runs one chunk further ahead of the MMAs.
constexpr int T_STAGES = 4;
constexpr int T_STAGE_BYTES = A_SUB + 2 * B_HALF;
constexpr size_t T_SMEM_BYTES = (size_t)T_STAGES * T_STAGE_BYTES + 1024 + 256 + T_EPI_WARPS * T_EPI_SCRATCH;
static_assert(T_SMEM_BYTES <= 227 * 1024, "gemm_tma_kernel exceeds the 227 KB of shared memory per block");
static_assert(T_STAGES * T_STAGE_BYTES >= 128 * BN * 4, "the accumulator image must fit in the ring it overlays");
// Conv kernel with the epilogue from the accumulators (gemm_tma_kernel<EPI_CONV_ACC>): no accumulator image and no
// per-warp scratch, but two staging buffers per consumer warpgroup, each [64-channel half of the m128 tile][32 pixels]
// [128 B] (FP16 hi in one, lo in the other, SWIZZLE_128B) that the TMA stores to the NHWC output planes.
constexpr int T_STG_BUF = 2 * 32 * 128;
constexpr size_t T_CONV_SMEM_BYTES = (size_t)T_STAGES * T_STAGE_BYTES + 2 * 2 * T_STG_BUF + 1024 + 256;
static_assert(T_CONV_SMEM_BYTES <= 227 * 1024, "EPI_CONV_ACC exceeds the 227 KB of shared memory per block");

enum { OUT_PLANAR = 3 };   // two FP16 planes Y_hi[row][y_ms], Y_lo = Y_hi + plane_elems (channels-last)
// gemm_tma_kernel's consumers: rows x C matrix; 3x3 conv through the accumulator image, or from the accumulators
enum { EPI_MAT = 0, EPI_CONV_IMAGE = 1, EPI_CONV_ACC = 2 };

struct TmaP {
  TcP t;                    // .g: M, K, bias, relu, part, Y, y_ms, y_gs, S/tiles ...
  int bx, by, bi;           // conv box (pixels): columns of a tile = (ii*by + yy)*bx + xx
  int tiles_x, tiles_y;     // conv tile grid per image group
  int n_img, H, W, C;       // conv geometry (C = input channels; 0 in a matrix launch)
  long plane_elems;         // output: distance (in fp16 elements) between the hi and lo planes
  int ksegs, kc_per_seg;    // conv: K is accumulated in `ksegs` passes of kc_per_seg chunks whose fp32
  float* acc_scratch;       // partial sums are combined in fp32 RN through acc_scratch: [tile*256 + column][M]
                            // (conv_image_consumer), or that range's blocks in fragment order (seg_fold)
  int halo, pool;           // halo: pixel-major kernel only (gemm_tma_px.cuh), vertical taps from one halo box
                            // pool: fused 2x2 max-pool in the conv epilogue (both kernels): the pooled map is written
  unsigned long long* pool_sum;   // channel-major conv + pool: if set, the pooled values are also summed per (image, channel)
                            // into pool_sum[img][M] as 2^-32 fixed point (SkipPool's global average, order-independent)
  unsigned long long* segsum;   // matrix mode: if set, nothing is stored; relu(x*sc[g][co] + sh[g][co]) is summed per
                            // detection (g.seg[column]) into segsum[det][M] as 2^-32 fixed point (order-independent)
  int* status;              // workspace status word (FP16 range flag of the planar outputs) or null
  int wcompact;             // pixel-major kernel: t.Wp holds the compact N = 64 tiles (8 KB per k chunk, weights.py::pack_px)
  const float* gen_src;     // pixel-major kernel, GEN27 variant: fp32 NCHW 3-channel crops [n_img][3][H][W]; the 27 (+5 zero)
                            // taps of every pixel (k = ci*9 + ky*3 + kx) are built in shared memory by producer warps
  const int4* chunk_tab;    // matrix mode with g.seg: per (column tile, half) the four 32-column chunks' descriptors
                            // (first detection index << 1) | (chunk complete and inside ONE detection); see
                            // seg_chunk_tab_kernel.  One uniform 16-byte load per subtile instead of a load + 12 shuffles.
};

// chunk descriptors of the table-tiled contractions over ragged per-detection columns (PointNet): tab[tile*2 + half]
static __global__ void seg_chunk_tab_kernel(const int4* __restrict__ tiles, int num_tiles, const int* __restrict__ seg,
                                            int4* __restrict__ tab) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= num_tiles * 2) return;
  const int4 tt = tiles[idx >> 1];
  const int half = idx & 1, c0 = tt.y, len = tt.z;
  int v[4];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    const int col0 = half * 128 + c * 32;
    v[c] = 0;
    if (col0 < len) {
      const int first = seg[c0 + col0], last = seg[c0 + min(col0 + 31, len - 1)];
      v[c] = (first << 1) | ((col0 + 32 <= len && first == last) ? 1 : 0);
    }
  }
  tab[idx] = make_int4(v[0], v[1], v[2], v[3]);
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t mbar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(mbar)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint32_t mbar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], "
      "[%6];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(mbar)
      : "memory");
}
// shared -> global box store (bulk async-group of the issuing thread); OOB elements of the box are not written
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's committed bulk stores have read their shared-memory source (read) / are complete
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// four 8x8 b16 matrices in mma fragment layout (thread (g, t) holds row g, columns 2t, 2t+1), stored transposed:
// lane l gives the address of row l % 8 of matrix l / 8, which receives column l % 8 of the fragment
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}
__device__ __forceinline__ void st_shared_u16(uint32_t addr, unsigned short v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
// K-major SWIZZLE_64B operand: rows of 64 bytes (32 fp16), 8-row groups 512 B apart (SBO), layout type 2.
__device__ __forceinline__ uint64_t smem_desc_sw64(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
// one 32-byte (whole sector) store as two 16-byte halves; dst 32-byte aligned
__device__ __forceinline__ void st_global_256(void* dst, const uint4& a, const uint4& b) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};\n\tst.global.v4.b32 [%0+16], {%5, %6, %7, %8};" ::"l"(dst),
               "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b.x), "r"(b.y), "r"(b.z), "r"(b.w)
               : "memory");
}
__device__ __forceinline__ void st_global_256(void* dst, const uint32_t* r) {
  st_global_256(dst, make_uint4(r[0], r[1], r[2], r[3]), make_uint4(r[4], r[5], r[6], r[7]));
}
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  unsigned short a, b;
  asm("{\n\t.reg .f32 f;\n\t"
      "cvt.rn.satfinite.f16.f32 %0, %2;\n\t"
      "cvt.f32.f16 f, %0;\n\t"
      "sub.f32 f, %2, f;\n\t"
      "cvt.rn.satfinite.f16.f32 %1, f;\n\t}"
      : "=h"(a), "=h"(b)
      : "f"(x));
  hi = __ushort_as_half(a);
  lo = __ushort_as_half(b);
}

// 2x2 max-pool of one 32-column chunk held by a thread (one channel): the chunk is 32/BX box rows of BX pixels, so its
// 16/BX row pairs hold BX/2 windows each: o[a*(BX/2) + b] = window (rows 2a, 2a+1; columns 2b, 2b+1).  BX <= 16.
template <int BX>
__device__ __forceinline__ void pool_chunk(const float (&x)[32], float (&o)[8]) {
#pragma unroll
  for (int a = 0; a < 16 / BX; a++)
#pragma unroll
    for (int b = 0; b < BX / 2; b++) {
      const int i = 2 * a * BX + 2 * b;
      o[a * (BX / 2) + b] = fmaxf(fmaxf(x[i], x[i + 1]), fmaxf(x[i + BX], x[i + BX + 1]));
    }
}

// ---- main loop: one K segment (chunks [kc_lo, kc_hi)) of this warpgroup's 128 rows x 128 columns (column half `half`),
// two m64n128 wgmma chains.  On return the accumulators are final and every ring stage they read has been released.
__device__ __forceinline__ void mma_segment(float (&acc)[2][64], const TmaP& P, uint32_t base, uint32_t bar0, int half,
                                            int lane, int kc_lo, int kc_hi, uint32_t& it) {
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (T_STAGES + s); };
  // The first wgmma of each chain ignores the accumulators (scale_d = 0); clearing them here rather than once per
  // CTA leaves them dead from the epilogue to the next item, so the epilogue has their registers (no spills).
#pragma unroll
  for (int mb = 0; mb < 2; mb++)
#pragma unroll
    for (int i = 0; i < 64; i++) acc[mb][i] = 0.f;
  for (int kc = kc_lo; kc < kc_hi; kc++, it++) {
    const int s = it % T_STAGES;
    mbar_wait(full_bar(s), (it / T_STAGES) & 1);
    const uint32_t sa = base + s * T_STAGE_BYTES, sb = sa + A_SUB + half * (128 / 8) * 512;
    if (!(P.t.dbg & MM_DBG_SKIP_MMA)) {
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ks++) {
        const uint64_t b_hi = smem_desc_sw64(sb + ks * 32), b_lo = smem_desc_sw64(sb + B_HALF + ks * 32);
#pragma unroll
        for (int mb = 0; mb < 2; mb++) {
          const uint32_t a = sa + mb * 8 * SBO + ks * 2 * A_LBO;
          const uint64_t a_hi = smem_desc(a, A_LBO, SBO), a_lo = smem_desc(a + A_HALF, A_LBO, SBO);
          wgmma_n128(acc[mb], a_hi, b_hi, ((kc - kc_lo) | ks) ? 1u : 0u);
          wgmma_n128(acc[mb], a_hi, b_lo, 1u);
          wgmma_n128(acc[mb], a_lo, b_hi, 1u);
        }
      }
      wgmma_commit();
    }
    wgmma_wait<1>();   // the previous chunk's wgmmas are done: release its stage
    if (kc > kc_lo) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar((it - 1) % T_STAGES)); }
  }
  wgmma_wait<0>();
  fence_acc(acc[0]);
  fence_acc(acc[1]);
  __syncwarp();
  if (lane == 0) mbar_arrive(empty_bar((it - 1) % T_STAGES));
}

__device__ __forceinline__ int opaque(int v) { asm volatile("" : "+r"(v)); return v; }

// Origin (dx, dy, di) inside a box (BX, BY, BI) (powers of two, lbx / lby their logs) of the 32 consecutive columns
// from column c0 (a multiple of 32), columns numbered (ii*BY + yy)*BX + xx.  Those 32 columns are themselves the box
// (min(BX, 32), min(BY, 32 / min(BX, 32)), ...) that store_box_dims gives the output tensor maps.
__device__ __forceinline__ void box_origin32(int c0, int BX, int BY, int lbx, int lby, int& dx, int& dy, int& di) {
  const int r = c0 >> lbx;
  dx = c0 & (BX - 1); dy = r & (BY - 1); di = r >> lby;
}

// column tile of a conv launch -> box origin (first image, y, x)
__device__ __forceinline__ void conv_origin(const TmaP& P, int nt, int& i0, int& y0, int& x0) {
  const int tx = nt % P.tiles_x;
  const int r = nt / P.tiles_x;
  const int ty = r % P.tiles_y;
  i0 = (r / P.tiles_y) * P.bi; y0 = ty * P.by; x0 = tx * P.bx;
}

// x[j] = (row j of the warp's 32, channel `lane`) -> FP16 hi / lo planes at dst, dst + plane_elems: the 32x32 block is
// transposed through the warp's smem scratch so that lane p stores the 32 channels (64 contiguous bytes per plane) of
// row p at dst (the lane's own row, if ok); amax tracks the magnitudes converted.
__device__ __forceinline__ void store_rows(const float (&x)[32], bool ok, __half* dst, long plane_elems, __half* scr,
                                           int lane, float& amax) {
  __half h[32], l[32];
#pragma unroll
  for (int j = 0; j < 32; j++) { split_f16(x[j], h[j], l[j]); amax = fmaxf(amax, fabsf(x[j])); }
#pragma unroll
  for (int pl = 0; pl < 2; pl++) {
#pragma unroll
    for (int j = 0; j < 32; j++) scr[j * 40 + lane] = pl ? l[j] : h[j];
    __syncwarp();
    if (ok) {
      // 256-bit stores: each instruction writes whole 32-byte sectors (16-byte pieces cost a partial-sector
      // write each and ran the first layers' epilogues at ~1.8 TB/s)
      const uint4* src = reinterpret_cast<const uint4*>(scr + lane * 40);
      __half* d = dst + (pl ? plane_elems : 0);
      const uint4 a = src[0], b = src[1], c = src[2], e = src[3];
      st_global_256(d, a, b);
      st_global_256(d + 16, c, e);
    }
    __syncwarp();
  }
}

// Channel-major conv consumers of gemm_tma_kernel<EPI_CONV_ACC>: the epilogue runs on the wgmma fragments in registers.
// Thread (warp w of warpgroup `half`, lane = 4g + t) holds, for m64 block mb and n8 block j, channels
// mg*128 + mb*64 + 16w + {g, g+8} at columns half*128 + 8j + {2t, 2t+1}: acc[mb][4j + {0, 1}] and acc[mb][4j + {2, 3}].
// Output: per 32 columns (or the 32 pooled pixels of a half) the FP16 hi and lo values go pixel-major into the
// warpgroup's two staging buffers (stmatrix.trans, 128-byte swizzle) and one thread stores them by TMA through the
// NHWC maps out_hi / out_lo, which clip partial boxes.  Only the warpgroup synchronises; the ring is never waited on.
// K-segmented launches fold their segments' partial sums first (seg_fold).
template <int BX>
__device__ __forceinline__ void conv_pool_epi(const TmaP& P, const float (&x)[2][64], int half, int w, int lane, int mg,
                                              int i0, int y0, int x0, int lby, float& amax, uint32_t buf) {
  const GemmP& p = P.t.g;
  const int g = lane >> 2, t = lane & 3;
  constexpr int NS = BX >= 8 ? 8 : 16;   // pooled values per channel row of the thread
  constexpr int BX8 = BX >= 8 ? BX / 8 : 1;
  const int PBY = P.by >> 1, lpby = lby - 1;          // pooled box rows
  const int Hp = P.H >> 1, Wp = P.W >> 1;
  float run[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  int cur = -1;                                        // image of the running sums
  auto flush = [&]() {
    // BX >= 4: the quad's four lanes hold the same channel and the same image, so they reduce to one atomic
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        float s = run[mb][h];
        if (BX >= 4) { s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2); }
        const int co = mg * 128 + mb * 64 + 16 * w + 8 * h + g;
        if ((BX >= 4 ? t == 0 : !(t & 1)) && cur >= 0 && cur < P.n_img && co < p.M)
          atomicAdd(P.pool_sum + (long)cur * p.M + co, __float2ull_rn(s * 4294967296.f));
        run[mb][h] = 0.f;
      }
  };
#pragma unroll
  for (int J = 0; J < NS; J++) {
    // pooled column pc (0..31 in the half, numbered like the columns in the pooled box (BX/2, by/2, bi)) and the
    // window's maximum for the thread's four channel rows
    float v[2][2];
    int pc;
    bool own = true;
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (BX >= 8) {   // vertical partner: the same thread's n8 block BX/8 further on
          const int j = (J / BX8) * (BX / 4) + J % BX8, jp = j + BX8;
          v[mb][h] = fmaxf(fmaxf(x[mb][4 * j + 2 * h], x[mb][4 * j + 2 * h + 1]),
                           fmaxf(x[mb][4 * jp + 2 * h], x[mb][4 * jp + 2 * h + 1]));
        } else {         // vertical partner: lane ^ 2 (BX = 4) or lane ^ 1 (BX = 2) of the same n8 block
          const float hm = fmaxf(x[mb][4 * J + 2 * h], x[mb][4 * J + 2 * h + 1]);
          v[mb][h] = fmaxf(hm, __shfl_xor_sync(0xffffffffu, hm, BX == 4 ? 2 : 1));
        }
      }
    if (BX >= 8) pc = 4 * J + t;
    else if (BX == 4) { pc = 2 * J + (t & 1); own = t < 2; }
    else { pc = 2 * J + (t >> 1); own = !(t & 1); }
    // pooled pixel -> (image, y, x) of the pooled map
    const int c = half * 32 + pc;
    const int r = c / (BX / 2);
    const int pimg = i0 + (r >> lpby), py = (y0 >> 1) + (r & (PBY - 1)), px = (x0 >> 1) + c % (BX / 2);
    const bool ok = own && pimg < P.n_img && py < Hp && px < Wp;
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int ch = 16 * w + 8 * h + g;
        if (mg * 128 + mb * 64 + ch < p.M) amax = fmaxf(amax, fabsf(v[mb][h]));
        if (own) {
          __half hi, lo;
          split_f16(v[mb][h], hi, lo);
          const uint32_t a = buf + mb * 4096 + pc * 128 + ((((ch >> 3) ^ (pc & 7)) << 4) | ((ch & 7) << 1));
          st_shared_u16(a, __half_as_ushort(hi));
          st_shared_u16(a + T_STG_BUF, __half_as_ushort(lo));
        }
      }
    if (P.pool_sum) {
      if (pimg != cur) {   // warp-uniform for BX >= 4 (one image per quad and J); BX = 2 flushes without shuffles
        flush();
        cur = pimg;
      }
#pragma unroll
      for (int mb = 0; mb < 2; mb++)
#pragma unroll
        for (int h = 0; h < 2; h++) run[mb][h] += ok ? v[mb][h] : 0.f;
    }
  }
  if (P.pool_sum) flush();
}

// K-segmented launches of conv_acc_consumer: fold segment `seg`'s fragments into the tile's running fp32 sums S, the
// same operations in the same order as conv_image_consumer, so the outputs are byte-identical: after segment 0
// S = RN(v s), after each later one S = fmaf(v, s, S).  S lives in acc_scratch between segments, one block per (tile,
// m-group) where the tile-order layout [tile*256 + column][M] puts it (256 x min(128, M - 128 mg) floats), in fragment
// order: float4 piece pc of m64 block mb of consumer thread tid at [mb][pc][tid], so a warp instruction covers 512
// contiguous bytes; m64 blocks of rows >= M are neither loaded nor stored (conv_plan takes this path for M % 64 == 0
// only, so every block is whole).  Every S of a batch is loaded and folded
// before any store, so no load waits on a store of the same boundary; a thread reads back only what it wrote, so
// program order suffices (ld.global.cg: the non-coherent path could return stale lines written by this kernel).
// On return acc holds S; after the last segment nothing is stored.
constexpr int SEG_BATCH = 8;   // float4 pieces loaded together
__device__ __forceinline__ void seg_fold(float (&acc)[2][64], const TmaP& P, int nt, int mg, int seg) {
  const GemmP& p = P.t.g;
  const float s = P.t.out_scale;
  float4* blk = reinterpret_cast<float4*>(P.acc_scratch + ((long)nt * BN * p.M + (long)mg * 128 * BN)) +
                (opaque(threadIdx.x) & 255);
#pragma unroll
  for (int mb = 0; mb < 2; mb++) {
    if (mg * 128 + mb * 64 >= p.M) continue;
    const float4* sp = blk + mb * 16 * 256;
    if (seg == 0) {
#pragma unroll
      for (int i = 0; i < 64; i++) acc[mb][i] = __fmul_rn(acc[mb][i], s);
      continue;
    }
#pragma unroll
    for (int b = 0; b < 16; b += SEG_BATCH) {
      float4 S[SEG_BATCH];
#pragma unroll
      for (int i = 0; i < SEG_BATCH; i++) S[i] = __ldcg(sp + (b + i) * 256);
#pragma unroll
      for (int i = 0; i < SEG_BATCH; i++) {
        float* v = &acc[mb][4 * (b + i)];
        v[0] = fmaf(v[0], s, S[i].x); v[1] = fmaf(v[1], s, S[i].y);
        v[2] = fmaf(v[2], s, S[i].z); v[3] = fmaf(v[3], s, S[i].w);
      }
    }
  }
  if (seg == P.ksegs - 1) return;
#pragma unroll
  for (int mb = 0; mb < 2; mb++) {
    if (mg * 128 + mb * 64 >= p.M) continue;
#pragma unroll
    for (int pc = 0; pc < 16; pc++)
      __stcg(blk + (mb * 16 + pc) * 256,
             make_float4(acc[mb][4 * pc], acc[mb][4 * pc + 1], acc[mb][4 * pc + 2], acc[mb][4 * pc + 3]));
  }
}

__device__ __forceinline__ void conv_acc_consumer(const TmaP& P, uint32_t base, uint32_t bar0, const CUtensorMap* out_hi,
                                                  const CUtensorMap* out_lo) {
  const GemmP& p = P.t.g;
  const int tid = threadIdx.x, half = tid >> 7;
  const bool elected = (tid & 127) == 0;
  const uint32_t stg = base + T_STAGES * T_STAGE_BYTES + half * 2 * T_STG_BUF;   // hi buffer; lo = hi + T_STG_BUF
  const int KC = P.t.k_chunks, mgroups = P.t.m_tiles;
  const long total_tiles = (long)p.num_tiles * mgroups;
  const int lbx = 31 - __clz(P.bx), lby = 31 - __clz(P.by);
  const float s = P.t.out_scale;
  uint32_t it = 0;
  float acc[2][64];
  float amax = 0.f;
  // write the staging buffers (fill), then store them: [mb] boxes of 64 channels at (x, y, img) of the output map
  auto stage = [&](auto&& fill, int mg, int cx, int cy, int ci) {
    if (elected) bulk_wait_read0();   // the previous stores have read the buffers
    bar_sync(8 + half, 128);
    fill();
    fence_async_smem();
    bar_sync(8 + half, 128);
    if (elected) {
#pragma unroll
      for (int mb = 0; mb < 2; mb++)
        if (mg * 128 + mb * 64 < p.M) {
          tma_store_4d(out_hi, stg + mb * 4096, mg * 128 + mb * 64, cx, cy, ci);
          tma_store_4d(out_lo, stg + T_STG_BUF + mb * 4096, mg * 128 + mb * 64, cx, cy, ci);
        }
      bulk_commit();
    }
  };

  for (long tl = blockIdx.x; tl < total_tiles; tl += gridDim.x) {
    const int mg_ = (int)(tl % mgroups);
    const int nt = (int)(tl / mgroups);
    int i0_, y0_, x0_;
    conv_origin(P, nt, i0_, y0_, x0_);
    {
      // K segments run back to back: the loader streams through their boundaries, where seg_fold carries the partial
      // sums through acc_scratch (single-pass launches: one segment of KC chunks)
      for (int seg = 0; seg < P.ksegs; seg++) {
        const int kc_lo = seg * P.kc_per_seg;
        mma_segment(acc, P, base, bar0, half, tid & 31, kc_lo, min(KC, kc_lo + P.kc_per_seg), it);
        if (P.ksegs > 1 && !(P.t.dbg & MM_DBG_SKIP_EPI)) seg_fold(acc, P, opaque(nt), opaque(mg_), seg);
      }
      if (P.t.dbg & MM_DBG_SKIP_EPI) continue;
      // Everything below derives from values laundered here, so the compiler cannot hoist the epilogue's lane and tile
      // arithmetic above the main loop, where it would be live next to the 128 accumulators.
      const int lane = opaque(threadIdx.x) & 31, w = (threadIdx.x >> 5) & 3, g = lane >> 2;
      const int mg = opaque(mg_), i0 = opaque(i0_), y0 = opaque(y0_), x0 = opaque(x0_);
      // bias (+ ReLU) in place: fmaf(v, s, b) as one pass, S + b after K segments (seg_fold left S in acc)
      const bool segmented = P.ksegs > 1;
#pragma unroll
      for (int mb = 0; mb < 2; mb++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int co = mg * 128 + mb * 64 + 16 * w + 8 * h + g;
          const float bv = (co < p.M && p.bias) ? __ldg(p.bias + co) : 0.f;
#pragma unroll
          for (int j = 0; j < 16; j++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
              float& v = acc[mb][4 * j + 2 * h + e];
              const float a = segmented ? __fadd_rn(v, bv) : fmaf(v, s, bv);
              v = p.relu ? fmaxf(a, 0.f) : a;
            }
        }
      if (P.pool) {
        int dx, dy, di;
        box_origin32(half * 32, P.bx >> 1, P.by >> 1, lbx - 1, lby - 1, dx, dy, di);
        stage([&]() {
          switch (P.bx) {
            case 32: conv_pool_epi<32>(P, acc, half, w, lane, mg, i0, y0, x0, lby, amax, stg); break;
            case 16: conv_pool_epi<16>(P, acc, half, w, lane, mg, i0, y0, x0, lby, amax, stg); break;
            case 8: conv_pool_epi<8>(P, acc, half, w, lane, mg, i0, y0, x0, lby, amax, stg); break;
            case 4: conv_pool_epi<4>(P, acc, half, w, lane, mg, i0, y0, x0, lby, amax, stg); break;
            default: conv_pool_epi<2>(P, acc, half, w, lane, mg, i0, y0, x0, lby, amax, stg); break;
          }
        }, mg, (x0 >> 1) + dx, (y0 >> 1) + dy, i0 + di);
        continue;
      }
#pragma unroll
      for (int cc = 0; cc < 4; cc++) {
        uint32_t hv[2][8], lv[2][8];   // [mb][2 jj + h]: n8 block 4cc + jj, channel row g + 8h
#pragma unroll
        for (int mb = 0; mb < 2; mb++)
#pragma unroll
          for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
              const float a0 = acc[mb][4 * (4 * cc + jj) + 2 * h], a1 = acc[mb][4 * (4 * cc + jj) + 2 * h + 1];
              if (mg * 128 + mb * 64 + 16 * w + 8 * h + g < p.M) amax = fmaxf(amax, fmaxf(fabsf(a0), fabsf(a1)));
              split_f16x2(a0, a1, hv[mb][2 * jj + h], lv[mb][2 * jj + h]);
            }
        int dx, dy, di;
        box_origin32(half * 128 + cc * 32, P.bx, P.by, lbx, lby, dx, dy, di);
        stage([&]() {
          // matrix q = lane / 8 of an x4: n8 block 2pr + q / 2, channels 16w + 8 (q & 1) ..; lane gives pixel row lane % 8
          const int q = lane >> 3, k = lane & 7;
#pragma unroll
          for (int mb = 0; mb < 2; mb++)
#pragma unroll
            for (int pr = 0; pr < 2; pr++) {
              const int px = 8 * (2 * pr + (q >> 1)) + k, c16 = 2 * w + (q & 1);
              const uint32_t a = stg + mb * 4096 + px * 128 + ((c16 ^ k) << 4);
              stmatrix_x4_trans(a, hv[mb][4 * pr], hv[mb][4 * pr + 1], hv[mb][4 * pr + 2], hv[mb][4 * pr + 3]);
              stmatrix_x4_trans(a + T_STG_BUF, lv[mb][4 * pr], lv[mb][4 * pr + 1], lv[mb][4 * pr + 2], lv[mb][4 * pr + 3]);
            }
        }, mg, x0 + dx, y0 + dy, i0 + di);
      }
    }
  }
  if (elected) bulk_wait0();
  mm_range_flag(P.status, amax);
}

// Matrix consumers of gemm_tma_kernel<EPI_MAT>, thread = one output channel of 128 image columns: bias, per-detection
// addend, ReLU, GroupNorm partials, then the per-detection sums (segsum) or the fp32 channels-last / planar FP16 store.
__device__ __forceinline__ void mat_consumer(const TmaP& P, uint8_t* sm, uint32_t base, uint32_t bar0) {
  const GemmP& p = P.t.g;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q = warp & 3, half = warp >> 2;
  const uint32_t free_bar = bar0 + 8u * (2 * T_STAGES);
  float* img = reinterpret_cast<float*>(sm);
  __half* scr = reinterpret_cast<__half*>(sm + T_STAGES * T_STAGE_BYTES + 256 + warp * T_EPI_SCRATCH);
  __half* yh = reinterpret_cast<__half*>(p.Y);
  const int KC = P.t.k_chunks, mgroups = P.t.m_tiles;
  const long total_tiles = (long)p.num_tiles * mgroups;
  uint32_t it = 0;       // k chunks consumed (ring position)
  float acc[2][64];      // rows 64 mb + fragment row, columns 128 half + fragment column
  float amax = 0.f;      // largest magnitude converted to FP16 by this thread (range guard)
  for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int mg = (int)(t % mgroups);
    const int nt = (int)(t / mgroups);
    int g, c0, len;
    tile_cols(p, nt, g, c0, len);
    mma_segment(acc, P, base, bar0, half, lane, 0, KC, it);
    acc_to_image(acc, img, half);
    const int co = mg * 128 + q * 32 + lane;
    const bool rowok = co < p.M;
    const float bv = (rowok && p.bias) ? __ldg(p.bias + co) : 0.f;
    double f1 = 0.0, f2 = 0.0;   // this thread's (sum, sum of squares) over its 128 columns: four shifted chunk sums
    const bool pass2 = P.segsum && !p.part && !p.Y && !p.relu;
    // Everything the four 32-column chunks need from global memory is fetched up front, so its latency is paid once
    // per subtile instead of once (or twice, seg -> addend) per chunk: the detection index at both ends of every
    // chunk (one load: lane 2c / 2c+1 holds chunk c's first / last column), the per-detection addend row of every
    // single-detection chunk, and the GroupNorm affine of the recomputing pass.
    const bool use_seg = p.seg && (p.addend || P.segsum);
    int4 ct = make_int4(0, 0, 0, 0);
    if (use_seg) ct = __ldg(P.chunk_tab + (long)nt * 2 + half);   // same address in every lane: one transaction
    const int cdesc[4] = {ct.x, ct.y, ct.z, ct.w};
    float adv[4] = {0.f, 0.f, 0.f, 0.f};
    unsigned one_det = 0;   // bit c: chunk c is complete and lies inside one detection
#pragma unroll
    for (int c = 0; c < 4; c++) {
      if (cdesc[c] & 1) {
        one_det |= 1u << c;
        if (p.addend && rowok) adv[c] = __ldg(p.addend + (long)(cdesc[c] >> 1) * p.ld_add + co);
      }
    }
    float na = 0.f, nb = 0.f;
    if (P.segsum && rowok) { na = __ldg(p.sc + (long)g * p.M + co); nb = __ldg(p.sh + (long)g * p.M + co); }
#pragma unroll 1
    for (int cc = 0; cc < 4; cc++) {
      const int col0 = half * 128 + cc * 32;
      if (col0 >= len) break;   // warp-uniform
      const int da = (cc == 0 ? ct.x : cc == 1 ? ct.y : cc == 2 ? ct.z : ct.w) >> 1;
      const float adc = cc == 0 ? adv[0] : cc == 1 ? adv[1] : cc == 2 ? adv[2] : adv[3];
      const bool single = (one_det >> cc) & 1u;
      const int nvalid = min(32, len - col0);
      uint32_t v[32];
      acc_ld32(img, BN, q * 32 + lane, col0, v);
      if (P.t.dbg & MM_DBG_SKIP_EPI) continue;
      float s1 = 0.f, s2 = 0.f, pv = 0.f;
      bool fast = col0 + 32 <= len;
      if (pass2 && fast) {
        // second (recomputing) pass, whole chunk inside one detection: bias, addend and the GroupNorm affine
        // fold into one fma per element; no statistics, nothing stored
        if (single) {
          if (rowok) {
            const float bva = bv + adc;
            const float a2 = P.t.out_scale * na, b2 = fmaf(bva, na, nb);
            float r0 = 0.f, r1 = 0.f;
#pragma unroll
            for (int j = 0; j < 32; j += 2) {
              r0 += fmaxf(fmaf(__uint_as_float(v[j]), a2, b2), 0.f);
              r1 += fmaxf(fmaf(__uint_as_float(v[j + 1]), a2, b2), 0.f);
            }
            atomicAdd(P.segsum + (long)da * p.M + co, __float2ull_rn((r0 + r1) * 4294967296.f));
          }
          continue;
        }
      }
      float bva = bv;
      if (fast && p.addend) {
        if (single) bva += adc;
        else fast = false;
      }
      if (fast) {
        if (p.relu) epi_fast<true>(v, P.t.out_scale, bva, pv, s1, s2);
        else epi_fast<false>(v, P.t.out_scale, bva, pv, s1, s2);
      } else if (p.addend) {   // per column: the chunk spans detections, or is partial
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 32; j++) {
          float x = fmaf(__uint_as_float(v[j]), P.t.out_scale, bv);
          const int col = col0 + j;
          if (rowok && col < len) x += __ldg(p.addend + (long)__ldg(p.seg + c0 + col) * p.ld_add + co);
          if (p.relu) x = fmaxf(x, 0.f);
          v[j] = __float_as_uint(x);
          if (col < len) t += x;
        }
        pv = t / (float)nvalid;
#pragma unroll
        for (int j = 0; j < 32; j++)
          if (j < nvalid) { const float d = __uint_as_float(v[j]) - pv; s1 += d; s2 = fmaf(d, d, s2); }
      } else epi_part(v, P.t.out_scale, bv, p.relu, col0, len, pv, s1, s2);
      stat_fold(f1, f2, nvalid, pv, s1, s2);
      if (P.segsum && rowok) {
        // GroupNorm + ReLU + per-detection sum fused into the (recomputing) second pass: the activation never
        // reaches HBM.  Run sums are fp32 in column order; runs are merged with integer atomics, so the result
        // does not depend on the order in which tiles finish.
        int dcur = da;
        float run = 0.f;
        if (single) {
          // common case: the whole 32-column chunk belongs to one detection
#pragma unroll
          for (int j = 0; j < 32; j++) run += fmaxf(fmaf(__uint_as_float(v[j]), na, nb), 0.f);
        } else {
#pragma unroll
          for (int j = 0; j < 32; j++) {
            if (j < nvalid) {
              const int d = __ldg(p.seg + c0 + col0 + j);
              if (d != dcur) {
                atomicAdd(P.segsum + (long)dcur * p.M + co, __float2ull_rn(run * 4294967296.f));
                run = 0.f; dcur = d;
              }
              run += fmaxf(fmaf(__uint_as_float(v[j]), na, nb), 0.f);
            }
          }
        }
        atomicAdd(P.segsum + (long)dcur * p.M + co, __float2ull_rn(run * 4294967296.f));
      }
      if (!p.Y || !rowok) continue;
      const long row0 = (long)g * p.y_gs + c0 + col0;
      if (P.t.out_mode == OUT_PLANAR && !(p.y_ms & 31)) {
        float xv[32];
#pragma unroll
        for (int j = 0; j < 32; j++) xv[j] = __uint_as_float(v[j]);
        store_rows(xv, lane < nvalid, yh + (row0 + lane) * p.y_ms + (co - lane), P.plane_elems, scr, lane, amax);
      } else if (P.t.out_mode == OUT_PLANAR) {
        __half* dst = yh + row0 * p.y_ms + co;
#pragma unroll
        for (int j = 0; j < 32; j++)
          if (j < nvalid) {
            __half h, l;
            split_f16(__uint_as_float(v[j]), h, l);
            amax = fmaxf(amax, fabsf(__uint_as_float(v[j])));
            dst[(long)j * p.y_ms] = h;
            dst[(long)j * p.y_ms + P.plane_elems] = l;
          }
      } else {   // OUT_CL fp32 channels-last
        store_cl(p.Y + row0 * p.y_ms + co, v, col0, len, p.y_ms);
      }
    }
    if (p.part && rowok) p.part[((long)nt * 2 + half) * p.M + co] = make_double2(f1, f2);
    image_release(free_bar, lane);
  }
  mm_range_flag(P.status, amax);
}

// Conv consumers of gemm_tma_kernel<EPI_CONV_IMAGE>, thread = one output channel of 128 image pixels: K segments
// combined through acc_scratch, or one pass with GroupNorm partials; planar FP16 NHWC, optionally 2x2 max-pooled.
__device__ __forceinline__ void conv_image_consumer(const TmaP& P, uint8_t* sm, uint32_t base, uint32_t bar0) {
  const GemmP& p = P.t.g;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q = warp & 3, half = warp >> 2;
  const uint32_t free_bar = bar0 + 8u * (2 * T_STAGES);
  float* img = reinterpret_cast<float*>(sm);
  __half* scr = reinterpret_cast<__half*>(sm + T_STAGES * T_STAGE_BYTES + 256 + warp * T_EPI_SCRATCH);
  __half* yh = reinterpret_cast<__half*>(p.Y);
  const int KC = P.t.k_chunks, mgroups = P.t.m_tiles;
  const long total_tiles = (long)p.num_tiles * mgroups;
  const int lbx = 31 - __clz(P.bx), lby = 31 - __clz(P.by);
  uint32_t it = 0;       // k chunks consumed (ring position)
  float acc[2][64], amax = 0.f;
  // ---- fused 2x2 max-pool (P.pool): the thread owns one channel of the tile's columns, so every pooling window of
  // its chunks is in its own registers.  NP pooled pixels per emission (8 for bx <= 16; 16 for bx == 32, where a
  // chunk is one box row and the previous chunk's horizontal maxima are kept); lane q < NP stores pooled pixel q's
  // 32 channels.  The pooled values are also summed per (image, channel) for SkipPool's global average.
  const int Hp = P.H >> 1, Wp = P.W >> 1;
  float hprev[16];            // bx == 32: horizontal maxima of the even row
  float psum = 0.f;           // running sum of this thread's pooled values of image psum_img
  int psum_img = -1;
  auto pool_flush = [&](int co_) {
    if (P.pool_sum && psum_img >= 0 && psum_img < P.n_img)
      atomicAdd(P.pool_sum + (long)psum_img * p.M + co_, __float2ull_rn(psum * 4294967296.f));
    psum = 0.f; psum_img = -1;
  };
  // o[q], q < np: pooled pixels of box rows (r0, r0 + 1), columns 2q', in box-row units r = ii*by + yy
  auto pool_emit = [&](const float (&o)[16], int np, int r0, int wq, int cb, int co_, int i0, int y0, int x0) {
    // pooled pixel q: box row r0 + 2*(q / wq), box column 2*(q % wq)      (wq = windows per row pair)
    float xs[32];
#pragma unroll
    for (int j = 0; j < 32; j++) xs[j] = j < 16 ? o[j] : 0.f;
    const int q = lane < np ? lane : 0;
    const int r = r0 + 2 * (q / wq), xx = 2 * (q - (q / wq) * wq);
    const int yy = r & (P.by - 1), ii = r >> lby;
    const int img = i0 + ii, y = y0 + yy, xg = x0 + xx;
    const bool ok = lane < np && img < P.n_img && y < P.H && xg < P.W;
    store_rows(xs, ok, yh + (((long)img * Hp + (y >> 1)) * Wp + (xg >> 1)) * p.y_ms + cb, P.plane_elems, scr, lane,
               amax);
    if (P.pool_sum) {
#pragma unroll
      for (int j = 0; j < 16; j++) {
        if (j < np) {
          const int rj = r0 + 2 * (j / wq), xj = 2 * (j - (j / wq) * wq);
          const int imj = i0 + (rj >> lby);
          const bool okj = imj < P.n_img && y0 + (rj & (P.by - 1)) < P.H && x0 + xj < P.W;
          if (imj != psum_img) { pool_flush(co_); psum_img = imj; }
          if (okj) psum += o[j];
        }
      }
    }
  };
  // one finished 32-column chunk (bias + ReLU applied) of channel co_: store it (x[j] = pixel column col0 + j, lane p
  // stores pixel col0 + p), or pool it and store the pooled map
  auto emit_conv = [&](const float (&x)[32], int cc, int col0, int co_, int i0, int y0, int x0) {
    if (!P.pool) {
      const int col = col0 + lane, r = col >> lbx;
      const int img = i0 + (r >> lby), y = y0 + (r & (P.by - 1)), xg = x0 + (col & (P.bx - 1));
      store_rows(x, img < P.n_img && y < P.H && xg < P.W, yh + (((long)img * P.H + y) * P.W + xg) * p.y_ms + co_ - lane,
                 P.plane_elems, scr, lane, amax);
      return;
    }
    float o[16];
    const int r0 = col0 >> lbx;
    if (P.bx == 32) {
      if (!(cc & 1)) {
#pragma unroll
        for (int b = 0; b < 16; b++) hprev[b] = fmaxf(x[2 * b], x[2 * b + 1]);
        return;
      }
#pragma unroll
      for (int b = 0; b < 16; b++) o[b] = fmaxf(hprev[b], fmaxf(x[2 * b], x[2 * b + 1]));
      pool_emit(o, 16, r0 - 1, 16, co_ - lane, co_, i0, y0, x0);
      return;
    }
    float o8[8];
    if (P.bx == 16) pool_chunk<16>(x, o8);
    else if (P.bx == 8) pool_chunk<8>(x, o8);
    else if (P.bx == 4) pool_chunk<4>(x, o8);
    else pool_chunk<2>(x, o8);
#pragma unroll
    for (int j = 0; j < 16; j++) o[j] = j < 8 ? o8[j] : 0.f;
    pool_emit(o, 8, r0, P.bx >> 1, co_ - lane, co_, i0, y0, x0);
  };
  for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int mg = (int)(t % mgroups);
    const int nt = (int)(t / mgroups);
    int i0, y0, x0;
    conv_origin(P, nt, i0, y0, x0);
    for (int seg = 0; seg < P.ksegs; seg++) {
      const int kc_lo = seg * P.kc_per_seg, kc_hi = min(KC, kc_lo + P.kc_per_seg);
      mma_segment(acc, P, base, bar0, half, lane, kc_lo, kc_hi, it);
      acc_to_image(acc, img, half);
      const int co = mg * 128 + q * 32 + lane;
      const bool rowok = co < p.M;
      const float bv = (rowok && p.bias) ? __ldg(p.bias + co) : 0.f;
      double f1 = 0.0, f2 = 0.0;   // single pass: GroupNorm partials over the tile's (always complete) chunks
#pragma unroll 1
      for (int cc = 0; cc < 4; cc++) {
        const int col0 = half * 128 + cc * 32;
        uint32_t v[32];
        acc_ld32(img, BN, q * 32 + lane, col0, v);
        float x[32];
        if (P.ksegs > 1) {
          // K segments: S = the segments' fmaf(v, s, S) in fp32 RN, then S + bv.  Partial sums live in TILE order,
          // scratch[(tile*256 + column)][M]: no pixel arithmetic, and a warp's 32 channels of one column are one
          // 128-byte access
          if (!rowok) continue;
          float* sp = P.acc_scratch + ((long)nt * BN + col0) * p.M + co;
          if (seg == 0 && seg < P.ksegs - 1) {
#pragma unroll
            for (int j = 0; j < 32; j++) __stcg(sp + (long)j * p.M, __uint_as_float(v[j]) * P.t.out_scale);
            continue;
          }
#pragma unroll
          for (int j = 0; j < 32; j++) x[j] = __ldcg(sp + (long)j * p.M);
          if (seg < P.ksegs - 1) {
#pragma unroll
            for (int j = 0; j < 32; j++) __stcg(sp + (long)j * p.M, fmaf(__uint_as_float(v[j]), P.t.out_scale, x[j]));
            continue;
          }
#pragma unroll
          for (int j = 0; j < 32; j++) {
            const float a = fmaf(__uint_as_float(v[j]), P.t.out_scale, x[j]) + bv;
            x[j] = p.relu ? fmaxf(a, 0.f) : a;
          }
        } else {
          if (P.t.dbg & MM_DBG_SKIP_EPI) continue;
          float s1 = 0.f, s2 = 0.f, pv = 0.f;
          if (p.relu) epi_fast<true>(v, P.t.out_scale, bv, pv, s1, s2);
          else epi_fast<false>(v, P.t.out_scale, bv, pv, s1, s2);
          stat_fold(f1, f2, 32, pv, s1, s2);
          if (!rowok) continue;
#pragma unroll
          for (int j = 0; j < 32; j++) x[j] = __uint_as_float(v[j]);
        }
        emit_conv(x, cc, col0, co, i0, y0, x0);
      }
      if (P.ksegs == 1 && p.part && rowok) p.part[((long)nt * 2 + half) * p.M + co] = make_double2(f1, f2);
      if (P.pool && seg == P.ksegs - 1 && rowok) pool_flush(co);
      image_release(free_bar, lane);
    }
  }
  mm_range_flag(P.status, amax);
}

template <int EPI>
static __global__ void __launch_bounds__(T_THREADS, 1)
gemm_tma_kernel(const TmaP P, const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                const __grid_constant__ CUtensorMap out_hi, const __grid_constant__ CUtensorMap out_lo) {
  const GemmP& p = P.t.g;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t bar0 = base + T_STAGES * T_STAGE_BYTES + (EPI == EPI_CONV_ACC ? 2 * 2 * T_STG_BUF : 0);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (T_STAGES + s); };
  const uint32_t free_bar = bar0 + 8u * (2 * T_STAGES);   // the epilogue has read the accumulator image

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mgroups = P.t.m_tiles;
  const long total_tiles = (long)p.num_tiles * mgroups;
  // K chunks: conv = 9 taps x (C / 32) channel chunks, K order k = tap*C + ci ; matrix = K / 32
  const int KC = P.t.k_chunks;

  if (tid == 0) {
    for (int s = 0; s < T_STAGES; s++) {
      mbar_init(full_bar(s), 1);              // the loader's single expect_tx arrive (weights + 2 operand boxes)
      mbar_init(empty_bar(s), T_EPI_WARPS);   // one arrive per consumer warp once its wgmmas have read the stage
    }
    mbar_init(free_bar, T_EPI_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < T_EPI_WARPS) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(T_CONS_REGS));
    if constexpr (EPI == EPI_MAT) mat_consumer(P, sm, base, bar0);
    else if constexpr (EPI == EPI_CONV_IMAGE) conv_image_consumer(P, sm, base, bar0);
    else conv_acc_consumer(P, base, bar0, &out_hi, &out_lo);
  } else {
    // =============================== LOADER (weights + operand boxes) ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(T_LOAD_REGS));
    if (warp == T_LOAD_WARP && lane == 0) {
      uint32_t it = 0, wcount = 0;
      for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int mg = (int)(t % mgroups);
        const int nt = (int)(t / mgroups);
        int g = 0, c0 = 0, len = BN, i0 = 0, y0 = 0, x0 = 0;
        if constexpr (EPI == EPI_MAT) tile_cols(p, nt, g, c0, len);
        else conv_origin(P, nt, i0, y0, x0);
        const int row0 = (int)((long)g * p.x_gs + c0);
        for (int kc = 0; kc < KC; kc++, it++) {
          if (kc % P.kc_per_seg == 0) {   // a new (tile, segment): the previous one's accumulator image has been read
            if (EPI != EPI_CONV_ACC && wcount > 0) mbar_wait(free_bar, (wcount - 1) & 1);
            wcount++;
          }
          const int s = it % T_STAGES;
          mbar_wait(empty_bar(s), ((it / T_STAGES) & 1) ^ 1);
          const uint32_t abytes = (uint32_t)A_SUB;
          const bool skipA = P.t.dbg & MM_DBG_SKIP_WEIGHTS, skipB = P.t.dbg & MM_DBG_SKIP_OPERANDS;
          mbar_expect_tx(full_bar(s), (skipA ? 0u : abytes) + (skipB ? 0u : 2u * B_HALF));
          const uint32_t sa = base + s * T_STAGE_BYTES, sb = sa + A_SUB;
          const uint8_t* src = reinterpret_cast<const uint8_t*>(P.t.Wp) + ((size_t)kc * P.t.m_tiles + mg) * A_SUB;
          if (!skipA) bulk_g2s(sa, src, abytes, full_bar(s));
          if (skipB) continue;
          if constexpr (EPI == EPI_MAT) {
            tma_load_2d(sb, &map_hi, kc * BK, row0, full_bar(s));
            tma_load_2d(sb + B_HALF, &map_lo, kc * BK, row0, full_bar(s));
          } else {
            const int cchunks = P.C / BK;
            const int tap = kc / cchunks, cc = kc - tap * cchunks;
            const int dx = tap % 3 - 1, dy = tap / 3 - 1;
            tma_load_4d(sb, &map_hi, cc * BK, x0 + dx, y0 + dy, i0, full_bar(s));
            tma_load_4d(sb + B_HALF, &map_lo, cc * BK, x0 + dx, y0 + dy, i0, full_bar(s));
          }
        }
      }
    }
    __syncwarp();
  }
}

// ---- host side: tensor maps through the driver entry point (no libcuda link dependency) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
// one tiled tensor map (unit element strides, no interleave, zero OOB fill); 900 + the CUresult on failure
static inline int encode_map(CUtensorMap* m, CUtensorMapDataType type, cuuint32_t rank, const void* basep,
                             const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                             CUtensorMapSwizzle swizzle, CUtensorMapL2promotion promo) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return MMMOT_E_ARG;
  const cuuint32_t es[4] = {1, 1, 1, 1};
  const CUresult r = fn(m, type, rank, const_cast<void*>(basep), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 900 + (int)r;
}
// fp16 [rows][C] matrix (row stride ld elements), box 32 x 256, 64-byte swizzle
static inline int make_map_2d(CUtensorMap* m, const void* basep, long rows, int C, long ld) {
  const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {32, 256};
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, basep, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
// fp32 [rows][C] matrix (row stride ld >= C elements, ld * 4 a multiple of 16), box 32 x box_rows: 128-byte box rows,
// so SWIZZLE_128B is allowed
static inline int make_map_2d_f32(CUtensorMap* m, const void* basep, long rows, int C, long ld, int box_rows,
                                  CUtensorMapSwizzle swizzle) {
  const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, basep, dims, strides, box, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
// fp16 NHWC [n_img][H][W][C], box (32, bx, by, bi)
static inline int make_map_4d(CUtensorMap* m, const void* basep, int n_img, int H, int W, int C, int bx, int by,
                              int bi) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n_img};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {32, (cuuint32_t)bx, (cuuint32_t)by, (cuuint32_t)bi};
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, basep, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// Output map of gemm_tma_kernel<EPI_CONV_ACC>: fp16 NHWC [n_img][H][W][M], box = 64 channels x the 32 consecutive
// columns of a (bx, by, bi) box (box_origin32), 128-byte swizzle (the staging buffers' layout)
static inline int make_map_4d_store(CUtensorMap* m, const void* basep, int n_img, int H, int W, int M, int bx, int by,
                                    int bi) {
  const int sx = bx < 32 ? bx : 32, sy = by < 32 / sx ? by : 32 / sx, si = 32 / (sx * sy);
  if (bx * by * bi < 64 || si > bi) return MMMOT_E_SHAPE;
  const cuuint64_t dims[4] = {(cuuint64_t)M, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n_img};
  const cuuint64_t strides[3] = {(cuuint64_t)M * 2, (cuuint64_t)W * M * 2, (cuuint64_t)H * W * M * 2};
  const cuuint32_t box[4] = {64, (cuuint32_t)sx, (cuuint32_t)sy, (cuuint32_t)si};
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, basep, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_NONE);
}

}  // namespace tma

#include "gemm_tma_px.cuh"

// launch parameters every TMA-fed launch sets; the rest of TmaP starts zero
static inline tma::TmaP tma_params(const GemmP& g, const uint4* Wp, float out_scale, int out_mode, long plane_elems,
                                   int* status) {
  tma::TmaP P;
  memset(&P, 0, sizeof(P));
  P.t.g = g;
  P.t.Wp = Wp;
  P.t.m_tiles = (g.M + 127) / 128;
  P.t.k_chunks = g.K / tc::BK;
  P.t.out_scale = out_scale;
  P.t.out_mode = out_mode;
  P.t.dbg = mm_debug_flags();
  P.plane_elems = plane_elems;
  P.status = status;
  return P;
}

// pixel-major kernel for 64-channel planar outputs (see gemm_tma_px.cuh); P fully prepared by the caller
static int gemm_tma_px_launch(tma::TmaP& P, const CUtensorMap& mh, const CUtensorMap& ml, int sms, cudaStream_t st) {
  static std::atomic<unsigned long long> attr{0};
  MM_TRY(mm_ensure_smem(tma::gemm_tma_px_kernel<false>, tma::PX_SMEM_BYTES, attr));
  const long total = P.t.g.num_tiles;
  const int grid = (int)(total < sms ? total : sms);
  tma::gemm_tma_px_kernel<false><<<grid, tma::PX_THREADS, tma::PX_SMEM_BYTES, st>>>(P, mh, ml);
  MM_LAUNCH_CHECK();
  return 0;
}

// First VGG layer (3 -> 64 channels, 3x3 / pad 1) straight from the fp32 NCHW crops: the K = 32 operand (27 taps + 5
// zeros per pixel, FP16 hi/lo) is generated in shared memory by the kernel's producer warps, so the im2col matrix
// (128 B per pixel written and read back) never exists.  Output: planar FP16 NHWC, bias + ReLU applied.
static int gemm_tma_px_launch_gen27(const float* crops, int n_img, int H, int W, const uint4* Wpx, float out_scale,
                                    const float* bias, __half* Yhi, long y_plane, int* status, cudaStream_t st) {
  if (!crops || !Wpx || !Yhi) return MMMOT_E_ARG;
  const long n_pix = (long)n_img * H * W;
  // a tile = 256 consecutive pixels of one image; staging buffer (256 + 2W + 2) x 3 floats in two 8 KB weight slots
  if (n_pix >= (1L << 31) || ((long)H * W) % tc::BN || (tc::BN + 2 * W + 2) * 12 > 2 * tma::PX_W_SLOT) return MMMOT_E_SHAPE;
  int sms = 0;
  MM_TRY(mm_sm_count(&sms));
  static std::atomic<unsigned long long> attr{0};
  MM_TRY(mm_ensure_smem(tma::gemm_tma_px_kernel<true>, tma::PX_SMEM_BYTES, attr));
  GemmP g = gemm_defaults();
  g.bias = bias; g.M = 64; g.K = 32; g.relu = 1;
  g.S = (int)n_pix; g.tiles_per_group = mm_cdiv(n_pix, tc::BN); g.num_tiles = g.tiles_per_group;
  g.Y = reinterpret_cast<float*>(Yhi); g.y_ms = 64;
  tma::TmaP P = tma_params(g, Wpx, out_scale, tma::OUT_PLANAR, y_plane, status);
  P.wcompact = 1;
  P.ksegs = 1; P.kc_per_seg = 1;
  P.gen_src = crops; P.n_img = n_img; P.H = H; P.W = W;
  alignas(64) CUtensorMap dummy;
  memset(&dummy, 0, sizeof(dummy));
  const long total = g.num_tiles;
  const int grid = (int)(total < sms ? total : sms);
  tma::gemm_tma_px_kernel<true><<<grid, tma::PX_GEN_THREADS, tma::PX_SMEM_BYTES, st>>>(P, dummy, dummy);
  MM_LAUNCH_CHECK();
  return 0;
}

#include "gemm_segsum.cuh"

// Whether a matrix-mode launch takes gemm_segsum_kernel (gemm_segsum.cuh): the per-detection-sum pass at K = 64 or 128
// with nothing stored, no statistics and no ReLU before the affine; MM_DBG_SEGSUM_GENERAL keeps gemm_tma_kernel (A/B
// runs).  Pure host logic, no CUDA call (mmmot_debug_segsum_kernel).
static inline bool segsum_dedicated(int K, bool segsum, bool y, bool part, bool relu, int dbg) {
  return segsum && !y && !part && !relu && (K == 64 || K == 128) && !(dbg & MM_DBG_SEGSUM_GENERAL);
}

template <int K>
static int gemm_segsum_launch(const tma::TmaP& P, const CUtensorMap& mh, const CUtensorMap& ml, int sms, cudaStream_t st) {
  static std::atomic<unsigned long long> attr{0};
  MM_TRY(mm_ensure_smem(tma::gemm_segsum_kernel<K>, tma::SegsumCfg<K>::SMEM, attr));
  const int mg_per = tma::segsum_mg_per(P.t.g.num_tiles, P.t.m_tiles, sms);
  const long units = (long)P.t.g.num_tiles * ((P.t.m_tiles + mg_per - 1) / mg_per);
  const int grid = (int)(units < sms ? units : sms);
  tma::gemm_segsum_kernel<K><<<grid, tma::SS_THREADS, tma::SegsumCfg<K>::SMEM, st>>>(P, mh, ml, mg_per);
  MM_LAUNCH_CHECK();
  return 0;
}

// 1x1 contraction on planar FP16 (hi, lo) channels-last activations X_hi[rows][ldx], X_lo = X_hi + x_plane.
// g: M, K (multiple of 32), bias, tiles, x_gs (rows per group), Y / y_ms / y_gs, part, addend...
static int gemm_tma_launch_mat(const GemmP& g, const uint4* Wp, float out_scale, const __half* Xhi, long x_plane,
                               long rows, int ldx, int out_mode, long y_plane, cudaStream_t st,
                               unsigned long long* segsum = nullptr, int* status = nullptr, const int4* chunk_tab = nullptr,
                               const uint4* Wpx = nullptr) {
  if (!Wp || g.num_tiles <= 0 || g.K % tc::BK) return MMMOT_E_ARG;
  int sms = 0;
  MM_TRY(mm_sm_count(&sms));
  static std::atomic<unsigned long long> attr{0};
  MM_TRY(mm_ensure_smem(tma::gemm_tma_kernel<tma::EPI_MAT>, tma::T_SMEM_BYTES, attr));
  tma::TmaP P = tma_params(g, Wp, out_scale, out_mode, y_plane, status);
  P.ksegs = 1; P.kc_per_seg = P.t.k_chunks;
  P.segsum = segsum;
  P.chunk_tab = chunk_tab;
  if (g.seg && (g.addend || segsum) && !chunk_tab) return MMMOT_E_ARG;
  alignas(64) CUtensorMap mh, ml;
  MM_TRY(tma::make_map_2d(&mh, Xhi, rows, g.K, ldx));
  MM_TRY(tma::make_map_2d(&ml, Xhi + x_plane, rows, g.K, ldx));
  if (out_mode == tma::OUT_PLANAR && g.M == 64 && g.y_ms == 64 && !g.part && !segsum && !g.addend && !g.tile_tab &&
      !(P.t.dbg & MM_DBG_CM64)) {
    if (Wpx) { P.t.Wp = Wpx; P.wcompact = 1; }
    return gemm_tma_px_launch(P, mh, ml, sms, st);
  }
  if (segsum_dedicated(g.K, segsum != nullptr, g.Y != nullptr, g.part != nullptr, g.relu != 0, P.t.dbg)) {
    if (!g.seg || !g.sc || !g.sh) return MMMOT_E_ARG;
    return g.K == 128 ? gemm_segsum_launch<128>(P, mh, ml, sms, st) : gemm_segsum_launch<64>(P, mh, ml, sms, st);
  }
  const long total = (long)g.num_tiles * P.t.m_tiles;
  const int grid = (int)(total < sms ? total : sms);
  tma::gemm_tma_kernel<tma::EPI_MAT><<<grid, tma::T_THREADS, tma::T_SMEM_BYTES, st>>>(P, mh, ml, mh, ml);
  MM_LAUNCH_CHECK();
  return 0;
}

// Waste of a box: padded / real pixels of the tile grid it induces.
static inline double conv_box_waste(int n_img, int H, int W, int bx, int by, int bi) {
  return (double)mm_cdiv(W, bx) * bx / W * mm_cdiv(H, by) * by / H * mm_cdiv(n_img, bi) * bi / n_img;
}

// Launch plan of a 3x3 convolution (gemm_tma_launch_conv).  Pure host logic, no CUDA call, so that tests can query
// the decision the launcher takes (mmmot_debug_conv_plan) on a machine without a GPU.
struct ConvPlan {
  int px;                  // pixel-major kernel (gemm_tma_px.cuh) instead of the channel-major one
  int halo;                // pixel-major: vertical taps from one (by + 2)-row halo box
  int pool;                // 2x2 max-pool fused into the epilogue
  int bx, by, bi;          // box of 256 pixels (powers of two)
  int ksegs, kc_per_seg;   // K accumulated in ksegs passes of kc_per_seg 32-wide chunks
  int tiles_x, tiles_y, num_tiles;   // column tiles (boxes); the channel-major kernel runs ceil(M/128) row tiles of each
  int acc_epi;             // channel-major, single-pass K: epilogue from the wgmma accumulators, TMA stores (EPI_CONV_ACC)
  int seg_acc;             // channel-major, K segments: the same kernel, partial sums folded from the fragments (seg_fold)
};
// want_pool: the caller takes a fused pooled map; use_kseg: the caller provides K-segment scratch.
// dbg / seg_chunks: mmmot_set_debug / mmmot_set_kseg state.
static inline ConvPlan conv_plan(int M, bool part, int n_img, int H, int W, int C, bool want_pool, bool use_kseg, int dbg,
                                 int seg_chunks) {
  ConvPlan c;
  memset(&c, 0, sizeof(c));
  // box of 256 pixels = bx * by * bi (powers of two): the shape with the least padding waste, widest first
  c.bx = 1; c.by = 1; c.bi = 256;
  double best = 1e30;
  for (int cx = 256; cx >= 1; cx >>= 1)
    for (int cy = 256 / cx; cy >= 1; cy >>= 1) {
      const int ci = 256 / (cx * cy);
      const double waste = conv_box_waste(n_img, H, W, cx, cy, ci);
      if (waste < best - 1e-9) { best = waste; c.bx = cx; c.by = cy; c.bi = ci; }
    }
  const int kchunks = 9 * C / tc::BK;
  // 64-channel outputs run on the pixel-major kernel (gemm_tma_px.cuh); it prefers a 16 x 16 single-image box
  // (vertical taps from one halo box, 2x2 pooling windows inside a warp) when that wastes no more than the best box
  c.px = M == 64 && !part && !(dbg & MM_DBG_CM64) && !(use_kseg && seg_chunks > 0 && kchunks > seg_chunks);
  if (c.px && conv_box_waste(1, H, W, 16, 16, 1) <= best + 1e-9) { c.bx = 16; c.by = 16; c.bi = 1; }
  if (c.px) {
    c.halo = (c.bi == 1 && c.bx >= 8 && c.bx * (c.by + 2) * 64 <= tma::PX_X_PLANE && !(dbg & MM_DBG_PX_NO_HALO)) ? 1 : 0;
    c.pool = want_pool && c.bx >= 2 && c.bx <= 16 && c.by >= 2 && !(H & 1) && !(W & 1) && !(dbg & MM_DBG_NO_FUSED_POOL);
  } else {
    // channel-major kernel: the 2x2 max-pool (and SkipPool's per-image sums) fused into the epilogue when every pooling
    // window lies inside one thread's chunks: box rows of <= 32 pixels, an even number of box rows per 128-column half
    c.pool = want_pool && c.bx >= 2 && c.bx <= 32 && c.by >= 2 && !(H & 1) && !(W & 1) && !(dbg & MM_DBG_NO_FUSED_POOL);
  }
  c.ksegs = 1; c.kc_per_seg = kchunks;
  if (use_kseg && seg_chunks > 0 && kchunks > seg_chunks) {
    c.ksegs = (kchunks + seg_chunks - 1) / seg_chunks;
    c.kc_per_seg = (kchunks + c.ksegs - 1) / c.ksegs;
  }
  c.tiles_x = mm_cdiv(W, c.bx); c.tiles_y = mm_cdiv(H, c.by);
  c.num_tiles = c.tiles_x * c.tiles_y * mm_cdiv(n_img, c.bi);
  // The accumulator epilogue stores 64-channel boxes; with K segments it also carries the partial sums between them
  // (seg_fold), so no segment boundary waits for an accumulator image.  GroupNorm partials (part) need the image.
  // seg_fold keeps whole m64 blocks of partial sums, so K segments need M % 64 == 0 (a partial block would not fit its
  // place in the [tiles*256][M] scratch); other M keep the image.  Debug bit 11 keeps the accumulator-image epilogue
  // (A/B runs).
  const bool acc = !c.px && !part && !(dbg & MM_DBG_CONV_IMAGE) && M >= 64;
  c.acc_epi = acc && c.ksegs == 1;
  c.seg_acc = acc && c.ksegs > 1 && M % 64 == 0;
  return c;
}

// 3x3 / pad 1 convolution on planar FP16 NHWC activations; output planar FP16 NHWC (ReLU via g.relu).
// acc_scratch (fp32 [tiles*256][M], tiles = ceil(W/bx)*ceil(H/by)*ceil(n/bi) <= padded pixel count) enables K-segmentation: chains longer than mmmot_set_kseg() chunks of 32 are
// accumulated in several passes and summed in fp32 RN, which bounds the tensor core's round-toward-zero
// accumulation error (DESIGN.md §4.2).  nullptr = single pass.
// pool_sum is filled only by the channel-major kernel's fused pool; plan (optional) receives the plan taken.
static int gemm_tma_launch_conv(const GemmP& g0, const uint4* Wp, float out_scale, const __half* Xhi, long x_plane,
                                int n_img, int H, int W, int C, __half* Yhi, long y_plane, cudaStream_t st,
                                float* acc_scratch = nullptr, long y_plane_pooled = 0, int* did_pool = nullptr,
                                int* status = nullptr, unsigned long long* pool_sum = nullptr, const uint4* Wpx = nullptr,
                                ConvPlan* plan = nullptr) {
  if (did_pool) *did_pool = 0;
  if (!Wp || C % tc::BK) return MMMOT_E_ARG;
  const ConvPlan c = conv_plan(g0.M, g0.part != nullptr, n_img, H, W, C, y_plane_pooled > 0 && did_pool,
                               acc_scratch != nullptr, mm_debug_flags(), mm_kseg_chunks());
  if (plan) *plan = c;
  int sms = 0;
  MM_TRY(mm_sm_count(&sms));
  GemmP g = g0;
  g.K = 9 * C;
  g.num_tiles = c.num_tiles;
  g.tile_tab = nullptr;
  g.Y = reinterpret_cast<float*>(Yhi);
  g.y_ms = g.M;
  tma::TmaP P = tma_params(g, Wp, out_scale, tma::OUT_PLANAR, c.pool ? y_plane_pooled : y_plane, status);
  P.bx = c.bx; P.by = c.by; P.bi = c.bi;
  P.halo = c.halo;
  P.pool = c.pool;
  if (c.pool) *did_pool = 1;
  if (c.pool && !c.px) P.pool_sum = pool_sum;
  P.tiles_x = c.tiles_x; P.tiles_y = c.tiles_y;
  P.n_img = n_img; P.H = H; P.W = W; P.C = C;
  P.ksegs = c.ksegs; P.kc_per_seg = c.kc_per_seg;
  if (c.ksegs > 1) P.acc_scratch = acc_scratch;
  alignas(64) CUtensorMap mh, ml;
  const int box_y = P.halo ? c.by + 2 : c.by;
  MM_TRY(tma::make_map_4d(&mh, Xhi, n_img, H, W, C, c.bx, box_y, c.bi));
  MM_TRY(tma::make_map_4d(&ml, Xhi + x_plane, n_img, H, W, C, c.bx, box_y, c.bi));
  if (c.px) {
    if (Wpx) { P.t.Wp = Wpx; P.wcompact = 1; }
    return gemm_tma_px_launch(P, mh, ml, sms, st);
  }
  const long total = (long)g.num_tiles * P.t.m_tiles;
  const int grid = (int)(total < sms ? total : sms);
  if (c.acc_epi || c.seg_acc) {
    static std::atomic<unsigned long long> attr{0};
    MM_TRY(mm_ensure_smem(tma::gemm_tma_kernel<tma::EPI_CONV_ACC>, tma::T_CONV_SMEM_BYTES, attr));
    const int sh = c.pool ? 1 : 0;
    alignas(64) CUtensorMap oh, ol;
    MM_TRY(tma::make_map_4d_store(&oh, Yhi, n_img, H >> sh, W >> sh, g.M, c.bx >> sh, c.by >> sh, c.bi));
    MM_TRY(tma::make_map_4d_store(&ol, Yhi + P.plane_elems, n_img, H >> sh, W >> sh, g.M, c.bx >> sh, c.by >> sh, c.bi));
    tma::gemm_tma_kernel<tma::EPI_CONV_ACC><<<grid, tma::T_THREADS, tma::T_CONV_SMEM_BYTES, st>>>(P, mh, ml, oh, ol);
  } else {
    static std::atomic<unsigned long long> attr{0};
    MM_TRY(mm_ensure_smem(tma::gemm_tma_kernel<tma::EPI_CONV_IMAGE>, tma::T_SMEM_BYTES, attr));
    tma::gemm_tma_kernel<tma::EPI_CONV_IMAGE><<<grid, tma::T_THREADS, tma::T_SMEM_BYTES, st>>>(P, mh, ml, mh, ml);
  }
  MM_LAUNCH_CHECK();
  return 0;
}
