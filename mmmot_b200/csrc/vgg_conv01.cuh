// First VGG block in one launch: layer 0 (3 -> 64, 3x3 / pad 1, bias + ReLU), layer 1 (64 -> 64, 3x3 / pad 1, bias +
// ReLU) and the 2x2 max-pool after it, from the fp32 NCHW crops to the pooled FP16 hi/lo NHWC planes conv 2 reads.
//
// The two-launch path (gemm_tma_px.cuh: GEN27, then the halo + pool kernel) writes layer 0's 64-channel full-resolution
// map to HBM and reads it back 3 * 18/16 times per channel chunk through TMA halo boxes.  Here a CTA computes, per
// 16 x 16 tile of layer-1 pixels, the 18 x 18 layer-0 pixels that tile needs (the halo ring is recomputed by the
// neighbouring tiles) and keeps them in shared memory only:
//   1. the tile's 20 x 20 x 3 crop neighbourhood is staged in shared memory (zero outside the image);
//   2. layer 0 runs on the tensor cores as in GEN27: K = 27 taps (+5 zeros), k = ci*9 + ky*3 + kx, FP16 hi/lo, three
//      MMAs per k16 step, then out_scale, bias, ReLU and split_f16x2; the A fragments are built in registers straight
//      from the staged crop.  Layer-0 pixels outside the image are stored as 0 (layer 1's zero padding), not relu(bias);
//   3. the 18 x 18 x 64 hi/lo image (81 KB) stays in shared memory; 16-byte chunk c of pixel p is stored at chunk
//      c ^ ((p >> 1) & 7), so the 8 rows of every ldmatrix below (pixels p0 + 2r) hit 8 different bank groups;
//   4. layer 1 takes its A operand (pixels x k) from registers, loaded by ldmatrix from that one image: a horizontal tap
//      is a shifted pixel index, not a shifted TMA box, so no swizzle-atom alignment is needed.  The weights stream
//      through a ring of 24 KB stages (one (kx, channel chunk) with its three vertical taps), as in the two-launch path;
//   5. the M rows are ordered so that each thread's accumulators hold whole pooling windows: consumer warpgroup h,
//      warp w, fragment row g (+8) of m-block mb is pixel (8h + 2w + mb, 2g (+1)); the 2x2 max is taken in registers,
//      then bias + ReLU (they commute with the max) and the FP16 split, and the pooled planes are stored directly.
// Accumulation order, per output element, is the two-launch path's: horizontal tap, channel chunk, vertical tap, k16
// step, then hi*hi, hi*lo, lo*hi; layer 0's is GEN27's.  The pooled planes are therefore bit-identical to it.
//
// CTA (384 threads, persistent, one per SM): warps 0-7 are two consumer warpgroups that run every phase of a tile
// together (staging, layer 0 with 3 of the 6 m64 blocks of 18 x 18 -> 384 padded rows each, layer 1 on 128 pixels each,
// pooled epilogue); warp 8 is the loader of the weight ring (warps 9-11 only complete its warpgroup).  The loader runs up
// to F01_STAGES stages ahead, so the next tile's first weight stages arrive while the consumers stage the crop and run
// layer 0; the next tile's crop loads are issued into registers before layer 1's MMAs and stored after them.
#pragma once

namespace tma {

constexpr int F01_TILE = 16;                       // layer-1 output tile: 16 x 16 pixels (8 x 8 pooled)
constexpr int F01_HALO = F01_TILE + 2;             // layer-0 pixels per side the tile needs
constexpr int F01_HPIX = F01_HALO * F01_HALO;      // 324 layer-0 pixels, in 6 m64 blocks (384 rows)
constexpr int F01_CROP = F01_TILE + 4;             // crop neighbourhood per side
constexpr int F01_CROP_N = 3 * F01_CROP * F01_CROP;
constexpr int F01_IMG_PLANE = F01_HPIX * 128;      // layer-0 image: [pixel][64 channels] FP16, per plane
constexpr int F01_STAGE = 3 * PX_W_SLOT;           // weight ring stage: three vertical taps of one (kx, channel chunk)
constexpr int F01_STAGES = 5;
constexpr int F01_W0_OFF = F01_STAGES * F01_STAGE;            // layer-0 weights, compact 8 KB tile (resident)
constexpr int F01_IMG_OFF = F01_W0_OFF + PX_W_SLOT;           // layer-0 image, hi then lo plane
constexpr int F01_CROP_OFF = F01_IMG_OFF + 2 * F01_IMG_PLANE;  // staged crop [ci][20][20] fp32
constexpr int F01_BAR_OFF = F01_CROP_OFF + F01_CROP_N * 4;
constexpr size_t F01_SMEM_BYTES = (size_t)F01_BAR_OFF + 16 * F01_STAGES + 1024;
static_assert(F01_SMEM_BYTES <= 227 * 1024, "vgg_conv01_kernel exceeds the 227 KB of shared memory per block");
static_assert(F01_IMG_OFF % 1024 == 0 && F01_BAR_OFF % 8 == 0, "vgg_conv01_kernel: shared-memory layout misaligned");
static_assert(6 * 64 >= F01_HPIX, "layer 0 runs 3 m64 blocks per consumer warpgroup");
constexpr int F01_THREADS = 384;
constexpr int F01_CONS_REGS = 232, F01_LOAD_REGS = 40;
static_assert(256 * F01_CONS_REGS + 128 * F01_LOAD_REGS <= launch_regs(F01_THREADS) * F01_THREADS,
              "vgg_conv01 register split exceeds the CTA's pool");

struct F01P {
  const float* crops;            // fp32 NCHW [n_img][3][H][W]
  int n_img, H, W;               // H, W multiples of 16
  int tiles_x, tiles_y;
  long num_tiles;
  const uint4* w0;               // layer 0: compact N = 64 tile of K = 32 (weights.py::pack_px)
  float scale0;
  const float* bias0;
  const uint4* w1;               // layer 1: 18 compact tiles, chunk (ky*3 + kx)*2 + cc
  float scale1;
  const float* bias1;
  __half* Y;                     // pooled FP16 NHWC planes [n_img][H/2][W/2][64], lo = hi + plane
  long plane;
  int* status;                   // FP16 range flag (crops, layer-0 and layer-1 outputs)
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T with A from registers (the m16n8k16 fragment layout per warp: a0 rows g,
// k 2t..2t+1; a1 rows g+8; a2, a3 the same at k + 8) and B from a shared-memory descriptor.
__device__ __forceinline__ void wgmma_n64_ra(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

static __global__ void __launch_bounds__(F01_THREADS, 1) vgg_conv01_kernel(const F01P P) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ float s_bias[2][64];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t bar0 = base + F01_BAR_OFF;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (F01_STAGES + s); };
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid < 128) s_bias[tid >> 6][tid & 63] = (tid < 64 ? P.bias0 : P.bias1)[tid & 63];
  for (int i = tid; i < PX_W_SLOT / 16; i += F01_THREADS)
    reinterpret_cast<uint4*>(sm + F01_W0_OFF)[i] = __ldg(P.w0 + i);
  fence_async_smem();   // generic-proxy writes of the layer-0 weights -> visible to the MMA's async proxy
  if (tid == 0) {
    for (int s = 0; s < F01_STAGES; s++) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), T_EPI_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int hw = P.H * P.W;
  auto tile_origin = [&](long t, int& img, int& y0, int& x0) {
    const int tx = (int)(t % P.tiles_x);
    const long r = t / P.tiles_x;
    y0 = (int)(r % P.tiles_y) * F01_TILE; x0 = tx * F01_TILE; img = (int)(r / P.tiles_y);
  };

  if (warp < T_EPI_WARPS) {
    // =============================== CONSUMERS ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(F01_CONS_REGS));
    const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t4 = lane & 3;
    const uint32_t img_hi = base + F01_IMG_OFF, w0s = base + F01_W0_OFF;
    const float* stg = reinterpret_cast<const float*>(sm + F01_CROP_OFF);
    float* stg_w = reinterpret_cast<float*>(sm + F01_CROP_OFF);
    uint32_t racc = 0;   // running max of the converted |hi| values of both layers (FP16 range guard)
    float amax = 0.f;    // largest |crop| value staged
    // layer-0 A fragment taps of this thread: k = 16 ks + 8 half + 2 t4 + e, as offsets ci*400 + ky*20 + kx into the
    // staged crop (-1: k >= 27, a zero column)
    int toff[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int k = (j >> 2) * 16 + ((j >> 1) & 1) * 8 + 2 * t4 + (j & 1);
      const int ci = k / 9, ky = (k % 9) / 3, kx = k % 3;
      toff[j] = k < 27 ? ci * F01_CROP * F01_CROP + ky * F01_CROP + kx : -1;
    }
    // layer-1 ldmatrix row of this lane: matrix lane >> 3 (rows g / g + 8, k 0-7 / 8-15), row lane & 7
    const int lx = 2 * (lane & 7) + ((lane >> 3) & 1), khalf = lane >> 4, ly = 8 * wg + 2 * w;
    const uint64_t w0_hi0 = smem_desc(w0s, PX_WC_LBO, SBO), w0_lo0 = smem_desc(w0s + 8 * SBO, PX_WC_LBO, SBO);
    const uint64_t w0_hi1 = smem_desc(w0s + 2 * PX_WC_LBO, PX_WC_LBO, SBO),
                   w0_lo1 = smem_desc(w0s + 8 * SBO + 2 * PX_WC_LBO, PX_WC_LBO, SBO);

    // crop neighbourhood of a tile: element i = (ci*20 + ry)*20 + rx, image pixel (y0 - 2 + ry, x0 - 2 + rx)
    constexpr int NPF = (F01_CROP_N + 255) / 256;
    float pf[NPF];
    auto load_crop = [&](long t) {
      int img, y0, x0;
      tile_origin(t, img, y0, x0);
      const float* src = P.crops + (long)img * 3 * hw;
#pragma unroll
      for (int u = 0; u < NPF; u++) {
        const int i = tid + 256 * u;
        const int ci = i / (F01_CROP * F01_CROP), rem = i - ci * F01_CROP * F01_CROP;
        const int gy = y0 - 2 + rem / F01_CROP, gx = x0 - 2 + rem % F01_CROP;
        pf[u] = (i < F01_CROP_N && gy >= 0 && gy < P.H && gx >= 0 && gx < P.W) ? __ldg(src + (long)ci * hw + gy * P.W + gx) : 0.f;
      }
    };
    if (blockIdx.x < P.num_tiles) load_crop(blockIdx.x);

    uint32_t it = 0;   // weight stages consumed (ring position)
    for (long t = blockIdx.x; t < P.num_tiles; t += gridDim.x) {
      int img, y0, x0;
      tile_origin(t, img, y0, x0);
      // ---- 1. stage the crop neighbourhood (the other warpgroup has finished reading the previous one: barrier 2 below)
#pragma unroll
      for (int u = 0; u < NPF; u++) {
        const int i = tid + 256 * u;
        if (i < F01_CROP_N) { stg_w[i] = pf[u]; amax = fmaxf(amax, fabsf(pf[u])); }
      }
      bar_sync(1, 256);   // crop staged; both warpgroups are past the previous tile's layer-1 reads of the image
      // ---- 2. layer 0 on this warpgroup's three m64 blocks of the 18 x 18 halo pixels
#pragma unroll 1
      for (int b = 0; b < 3; b++) {
        const int blk = wg * 3 + b;
        int hp[2], cbase[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          hp[h] = 64 * blk + 16 * w + g + 8 * h;
          cbase[h] = hp[h] < F01_HPIX ? (hp[h] / F01_HALO) * F01_CROP + hp[h] % F01_HALO : -1;
        }
        uint32_t ahi[2][4], alo[2][4];
#pragma unroll
        for (int ks = 0; ks < 2; ks++)
#pragma unroll
          for (int q = 0; q < 4; q++) {   // register q: row half q & 1, k half q >> 1
            const int h = q & 1, j = ks * 4 + (q >> 1) * 2;
            float v0 = 0.f, v1 = 0.f;
            if (cbase[h] >= 0) {
              if (toff[j] >= 0) v0 = stg[toff[j] + cbase[h]];
              if (toff[j + 1] >= 0) v1 = stg[toff[j + 1] + cbase[h]];
            }
            split_f16x2(v0, v1, ahi[ks][q], alo[ks][q]);
          }
        float a0[32];
        wgmma_fence();
        wgmma_n64_ra(a0, ahi[0], w0_hi0, 0u);
        wgmma_n64_ra(a0, ahi[0], w0_lo0, 1u);
        wgmma_n64_ra(a0, alo[0], w0_hi0, 1u);
        wgmma_n64_ra(a0, ahi[1], w0_hi1, 1u);
        wgmma_n64_ra(a0, ahi[1], w0_lo1, 1u);
        wgmma_n64_ra(a0, alo[1], w0_hi1, 1u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(a0);
        // epilogue: pixel hp[h], channels 8j + 2 t4 (+1) -> one f16x2 word per plane
#pragma unroll
        for (int h = 0; h < 2; h++) {
          if (cbase[h] < 0) continue;
          const int yy = y0 - 1 + hp[h] / F01_HALO, xx = x0 - 1 + hp[h] % F01_HALO;
          const bool inside = yy >= 0 && yy < P.H && xx >= 0 && xx < P.W;
          const uint32_t row = img_hi + (uint32_t)hp[h] * 128u + 4u * t4, sw = (uint32_t)((hp[h] >> 1) & 7);
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const int c = 8 * j + 2 * t4;
            uint32_t hi = 0u, lo = 0u;
            if (inside) {
              const float x0v = fmaxf(fmaf(a0[4 * j + 2 * h], P.scale0, s_bias[0][c]), 0.f);
              const float x1v = fmaxf(fmaf(a0[4 * j + 2 * h + 1], P.scale0, s_bias[0][c + 1]), 0.f);
              split_f16x2(x0v, x1v, hi, lo);
              mm_range_track2(racc, hi);
            }
            const uint32_t a = row + (((uint32_t)j ^ sw) << 4);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(hi) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + F01_IMG_PLANE), "r"(lo) : "memory");
          }
        }
      }
      bar_sync(1, 256);   // layer-0 image complete; every layer-0 read of the staged crop done
      if (t + gridDim.x < P.num_tiles) load_crop(t + gridDim.x);   // in flight during layer 1
      // ---- 3. layer 1: 6 ring stages (kx, cc) x 3 vertical taps x 2 k16 steps
      float acc[2][32];
#pragma unroll
      for (int mb = 0; mb < 2; mb++)
#pragma unroll
        for (int i = 0; i < 32; i++) acc[mb][i] = 0.f;
#pragma unroll 1
      for (int si = 0; si < 6; si++, it++) {
        const int kx = si >> 1, cc = si & 1;
        const int s = it % F01_STAGES;
        mbar_wait(full_bar(s), (it / F01_STAGES) & 1);
        const uint32_t sw = base + s * F01_STAGE;
#pragma unroll
        for (int ky = 0; ky < 3; ky++) {
          // One commit group per vertical tap: 12 MMAs on 32 A registers, retired before the next tap's ldmatrix
          // overwrites them (ptxas serialises every wgmma when A registers are redefined while a group is in flight).
          // The other warpgroup's MMAs fill the tensor pipe in between.
          uint32_t ah[2][2][4], al[2][2][4];
#pragma unroll
          for (int ks = 0; ks < 2; ks++)
#pragma unroll
            for (int mb = 0; mb < 2; mb++) {
              const int hp = (ly + mb + ky) * F01_HALO + lx + kx;
              const uint32_t c16 = (uint32_t)(cc * 4 + ks * 2 + khalf);
              const uint32_t a = img_hi + (uint32_t)hp * 128u + ((c16 ^ (uint32_t)((hp >> 1) & 7)) << 4);
              ldsm_x4(a, ah[ks][mb]);
              ldsm_x4(a + F01_IMG_PLANE, al[ks][mb]);
            }
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 2; ks++) {
            const uint32_t wo = sw + (uint32_t)(ky * PX_W_SLOT + ks * 2 * PX_WC_LBO);
            const uint64_t w_hi = smem_desc(wo, PX_WC_LBO, SBO), w_lo = smem_desc(wo + 8 * SBO, PX_WC_LBO, SBO);
#pragma unroll
            for (int mb = 0; mb < 2; mb++) {
              wgmma_n64_ra(acc[mb], ah[ks][mb], w_hi, (si | ky | ks) ? 1u : 0u);
              wgmma_n64_ra(acc[mb], ah[ks][mb], w_lo, 1u);
              wgmma_n64_ra(acc[mb], al[ks][mb], w_hi, 1u);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));   // this stage's weights are read
      }
      fence_acc(acc[0]);
      fence_acc(acc[1]);
      // ---- 4. 2x2 max-pool in registers (window = rows g, g + 8 of both m-blocks), bias + ReLU, FP16 split, store
      const long py = (y0 >> 1) + 4 * wg + w, px = (x0 >> 1) + g;
      __half* dst = P.Y + (((long)img * (P.H >> 1) + py) * (P.W >> 1) + px) * 64 + 2 * t4;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        float x[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const float m = fmaxf(fmaxf(acc[0][4 * j + e], acc[0][4 * j + 2 + e]), fmaxf(acc[1][4 * j + e], acc[1][4 * j + 2 + e]));
          x[e] = fmaxf(fmaf(m, P.scale1, s_bias[1][8 * j + 2 * t4 + e]), 0.f);
        }
        uint32_t hi, lo;
        split_f16x2(x[0], x[1], hi, lo);
        mm_range_track2(racc, hi);
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = hi;
        *reinterpret_cast<uint32_t*>(dst + P.plane + 8 * j) = lo;
      }
    }
    mm_range_flag(P.status, amax);
    mm_range_flag2(P.status, racc);
  } else {
    // =============================== LOADER: layer-1 weight ring ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(F01_LOAD_REGS));
    if (warp == T_LOAD_WARP && lane == 0) {
      uint32_t it = 0;
      for (long t = blockIdx.x; t < P.num_tiles; t += gridDim.x)
        for (int si = 0; si < 6; si++, it++) {
          const int s = it % F01_STAGES;
          const int kx = si >> 1, cc = si & 1;
          mbar_wait(empty_bar(s), ((it / F01_STAGES) & 1) ^ 1);
          mbar_expect_tx(full_bar(s), (uint32_t)F01_STAGE);
          for (int ky = 0; ky < 3; ky++)
            bulk_g2s(base + s * F01_STAGE + ky * PX_W_SLOT,
                     reinterpret_cast<const uint8_t*>(P.w1) + (size_t)((ky * 3 + kx) * 2 + cc) * PX_W_SLOT, PX_W_SLOT,
                     full_bar(s));
        }
    }
    __syncwarp();
  }
}

}  // namespace tma

// Whether the first VGG block (layers 0 and 1 + the 2x2 max-pool) of an n_img x H x W crop batch runs as the fused
// launch: pure host logic, so that tests can query it without a GPU.  It does where the two-launch path would run
// exactly the arithmetic it reproduces — layer 0 with in-kernel taps (GEN27: the compact tiles, H*W % 256 == 0,
// W <= 512) and layer 1 on the pixel-major kernel with 16 x 16 halo boxes and the fused pool (no K segments) — and
// the 16 x 16 tiles cover the image (H, W multiples of 16).  Debug bit 15 forces the two launches.
static inline bool vgg_conv01_fused(int n_img, int H, int W, bool compact_tiles, int dbg, int kseg) {
  if (!compact_tiles || (dbg & (MM_DBG_VGG0_FFMA | MM_DBG_VGG0_IM2COL | MM_DBG_VGG01_UNFUSED)) || n_img <= 0) return false;
  if (H % tma::F01_TILE || W % tma::F01_TILE || W > 512 || (long)n_img * H * W >= (1L << 31)) return false;
  const ConvPlan c = conv_plan(64, false, n_img, H, W, 64, true, true, dbg, kseg);
  return c.px && c.halo && c.pool && c.bx == tma::F01_TILE && c.by == tma::F01_TILE && c.bi == 1 && c.ksegs == 1;
}

// The fused first VGG block: crops [n_img][3][H][W] fp32 -> pooled planes Y[2][n_img][H/2][W/2][64] (y_plane apart).
// Wpx0 / Wpx1: the compact N = 64 tiles of layers 0 and 1 (weights.py::pack_px).
static int vgg_conv01_launch(const float* crops, int n_img, int H, int W, const uint4* Wpx0, float scale0,
                             const float* bias0, const uint4* Wpx1, float scale1, const float* bias1, __half* Y,
                             long y_plane, int* status, cudaStream_t st) {
  if (!crops || !Wpx0 || !Wpx1 || !bias0 || !bias1 || !Y) return MMMOT_E_ARG;
  if (n_img <= 0 || H % tma::F01_TILE || W % tma::F01_TILE || H <= 0 || W <= 0 || (long)n_img * H * W >= (1L << 31))
    return MMMOT_E_SHAPE;
  int sms = 0;
  MM_TRY(mm_sm_count(&sms));
  static std::atomic<unsigned long long> attr{0};
  MM_TRY(mm_ensure_smem(tma::vgg_conv01_kernel, tma::F01_SMEM_BYTES, attr));
  tma::F01P P;
  memset(&P, 0, sizeof(P));
  P.crops = crops; P.n_img = n_img; P.H = H; P.W = W;
  P.tiles_x = W / tma::F01_TILE; P.tiles_y = H / tma::F01_TILE;
  P.num_tiles = (long)P.tiles_x * P.tiles_y * n_img;
  P.w0 = Wpx0; P.scale0 = scale0; P.bias0 = bias0;
  P.w1 = Wpx1; P.scale1 = scale1; P.bias1 = bias1;
  P.Y = Y; P.plane = y_plane; P.status = status;
  const int grid = (int)(P.num_tiles < sms ? P.num_tiles : sms);
  tma::vgg_conv01_kernel<<<grid, tma::F01_THREADS, tma::F01_SMEM_BYTES, st>>>(P);
  MM_LAUNCH_CHECK();
  return 0;
}
