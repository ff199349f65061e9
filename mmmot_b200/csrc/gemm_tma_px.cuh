// Tensor-core contraction engine, pixel-major variant for 64-channel outputs (the first two VGG layers).
//
// With Cout = 64 the channel-major kernel (gemm_tma.cuh) pads the MMA's M from 64 to 128 — half of every
// tensor-core instruction is zeros.  Here the roles are swapped: the 256-pixel activation box is the A operand
// (K-major SWIZZLE_64B, as TMA writes it; consumer warpgroup h issues the m64n64 wgmma chains of pixels
// 128h..128h+127) and the packed weights are the B operand (N = 64, K-major canonical layout, only rows 0..63 of the
// packed tile are fetched).  The accumulators D[pixel][channel] go through a dedicated shared-memory image, so every
// epilogue thread owns 32 consecutive channels of one pixel and stores its 64 bytes per plane directly, and the
// loader fills the two ring stages of the next tile while the epilogue runs.
// Same arithmetic as the channel-major kernel: FP16 hi/lo split operands, D += Xhi*Whi + Xhi*Wlo + Xlo*Whi.
#pragma once

namespace tma {

// Halo mode (3x3 conv, one image per box): a stage holds the (by+2)-row box of ONE horizontal tap and channel chunk;
// its three vertical taps are the same shared-memory box read at start addresses dy*bx*64 B (whole swizzle atoms for
// bx >= 8), so the activation traffic from L2 — what bounds this layer — drops from 9 to 3*(by+2)/by boxes per
// chunk.  Optional fused 2x2 max-pool: with bx <= 16 a warp's 32 pixels are whole pooling windows (lanes l, l^1,
// l^bx, l^(bx+1)), so the pooled NHWC planes are written directly and the full-resolution activation never exists.
constexpr int PX_W_SLOT = 8192;                 // compact weight tile: [hi|lo][k group 4][row group 8][8][8] f16
constexpr int PX_W_LBO = 1024;
constexpr int PX_X_OFF = 3 * PX_W_SLOT;         // 24 KB: three tap slots
constexpr int PX_X_PLANE = 24576;               // up to 384 box rows x 64 B per plane
constexpr int PX_STAGE = PX_X_OFF + 2 * PX_X_PLANE;   // 72 KB
constexpr int PX_STAGES = 2;                   // 2 x 72 KB ring + the 64 KB accumulator image fit in 227 KB
constexpr int PX_IMG = 256 * 64 * 4;            // accumulator image [256 pixels][64 channels] fp32
constexpr size_t PX_SMEM_BYTES = (size_t)PX_STAGES * PX_STAGE + PX_IMG + 1024 + 256;

// Compact weight tiles (weights.py::pack_px): [k group 4][hi rows 0-63 | lo rows 0-63][8 rows][8 k], i.e. per k group a
// 128-row K-major block whose first 64 rows are W_hi and last 64 rows W_lo (one 8 KB copy per k chunk).
constexpr int PX_WC_LBO = 2048;

// CTA: warps 0-7 consumers (two warpgroups), warp 8 loader.  GEN27 variant: 20 warps; warps 9-11 only complete the
// loader's warpgroup and give up their registers (setmaxnreg), warps 12-19 are the operand producers.
constexpr int PX_THREADS = 288, PX_GEN_THREADS = 640, PX_GEN_WARP0 = 12;
constexpr int PX_CONS_REGS = 144, PX_LOAD_REGS = 24, PX_PROD_REGS = 80;   // GEN27 register split
static_assert(256 * PX_CONS_REGS + 128 * PX_LOAD_REGS + 256 * PX_PROD_REGS <= launch_regs(PX_GEN_THREADS) * PX_GEN_THREADS,
              "GEN27 register split exceeds the CTA's pool");

// GEN27 variant (first VGG layer): eight extra producer warps build the K = 32 activation operand of every tile — the 27
// taps of each pixel read from the fp32 NCHW crop, zero padding at the borders, FP16 hi/lo split — directly in the
// SWIZZLE_64B layout TMA would have written (row = pixel, 64 B per plane; 16-byte chunk c of row r lives at chunk
// c ^ ((r >> 1) & 3)).  Four warps (one group) complete a tile's full barrier.
constexpr int PX_GEN_WARPS = 4;

template <bool GEN27>
static __global__ void __launch_bounds__(GEN27 ? PX_GEN_THREADS : PX_THREADS, 1)
gemm_tma_px_kernel(const TmaP P, const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo) {
  const GemmP& p = P.t.g;
  extern __shared__ uint8_t smem_raw[];
  __shared__ float s_bias[64];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  float* img = reinterpret_cast<float*>(sm + PX_STAGES * PX_STAGE);
  const uint32_t bar0 = base + PX_STAGES * PX_STAGE + PX_IMG;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (PX_STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long total_tiles = p.num_tiles;
  const int KC = P.t.k_chunks;
  const bool conv = P.C > 0;                             // matrix launches leave the conv geometry 0
  const int cchunks = conv ? P.C / BK : KC;
  const int ntap = P.halo ? 3 : 1;                       // vertical taps served by one stage
  const int nstage = P.halo ? 3 * cchunks : KC;          // stages per tile
  const uint32_t xbytes = P.halo ? (uint32_t)(P.bx * (P.by + 2) * 64) : (uint32_t)B_HALF;

  if (tid < 64) s_bias[tid] = p.bias ? p.bias[tid] : 0.f;
  if (tid == 0) {
    for (int s = 0; s < PX_STAGES; s++) {
      mbar_init(full_bar(s), GEN27 ? 1 + PX_GEN_WARPS : 1);
      mbar_init(empty_bar(s), T_EPI_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < T_EPI_WARPS) {
    // =============================== CONSUMERS: wgmma + epilogue ===============================
    if (GEN27) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(PX_CONS_REGS));
    const int q = warp & 3, cb = (warp >> 2) * 32;   // pixel quadrant of each 128-pixel half, channel half
    const int lbx = 31 - __clz(max(P.bx, 1)), lby = 31 - __clz(max(P.by, 1));
    __half* yh = reinterpret_cast<__half*>(p.Y);
    uint32_t racc = 0;   // running max of the converted |hi| values (FP16 range guard)
    uint32_t it = 0;     // k stages consumed (ring position)
    const int wg = warp >> 2;
    float acc[2][32];    // pixels 128 wg + 64 mb + fragment row, channels = fragment column
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int i = 0; i < 32; i++) acc[mb][i] = 0.f;
    for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int nt = (int)t;
      int i0 = 0, y0 = 0, x0 = 0;
      if (conv) conv_origin(P, nt, i0, y0, x0);
      // ---- main loop: pixels 128 wg .. 128 wg + 127 x 64 channels, two m64n64 wgmma chains ----
      for (int si = 0; si < nstage; si++, it++) {
        const int s = it % PX_STAGES;
        mbar_wait(full_bar(s), (it / PX_STAGES) & 1);
        const uint32_t sw = base + s * PX_STAGE, sx = sw + PX_X_OFF;
        if (!(P.t.dbg & MM_DBG_SKIP_MMA)) {
          wgmma_fence();
          for (int ky = 0; ky < ntap; ky++) {
            const uint32_t xo = sx + (uint32_t)(ky * P.bx * 64 + wg * (128 * 64)), wo = sw + (uint32_t)(ky * PX_W_SLOT);
#pragma unroll
            for (int ks = 0; ks < 2; ks++) {
              uint64_t w_hi, w_lo;
              if (P.wcompact) {   // rows 0-63 W_hi, 64-127 W_lo
                w_hi = smem_desc(wo + ks * 2 * PX_WC_LBO, PX_WC_LBO, SBO);
                w_lo = smem_desc(wo + 8 * SBO + ks * 2 * PX_WC_LBO, PX_WC_LBO, SBO);
              } else {
                w_hi = smem_desc(wo + ks * 2 * PX_W_LBO, PX_W_LBO, SBO);
                w_lo = smem_desc(wo + PX_W_SLOT / 2 + ks * 2 * PX_W_LBO, PX_W_LBO, SBO);
              }
#pragma unroll
              for (int mb = 0; mb < 2; mb++) {
                const uint64_t x_hi = smem_desc_sw64(xo + mb * (64 * 64) + ks * 32);
                const uint64_t x_lo = smem_desc_sw64(xo + PX_X_PLANE + mb * (64 * 64) + ks * 32);
                wgmma_n64(acc[mb], x_hi, w_hi, (si | ky | ks) ? 1u : 0u);
                wgmma_n64(acc[mb], x_hi, w_lo, 1u);
                wgmma_n64(acc[mb], x_lo, w_hi, 1u);
              }
            }
          }
          wgmma_commit();
        }
        wgmma_wait<1>();   // the previous stage's wgmmas are done: release it
        if (si > 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar((it - 1) % PX_STAGES)); }
      }
      wgmma_wait<0>();
      fence_acc(acc[0]);
      fence_acc(acc[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar((it - 1) % PX_STAGES));
      bar_sync(7, T_EPI_WARPS * 32);   // the previous tile's epilogue has read the image
      acc_dump(acc[0], img, 64, wg * 128, 0);
      acc_dump(acc[1], img, 64, wg * 128 + 64, 0);
      bar_sync(7, T_EPI_WARPS * 32);
#pragma unroll 1
      for (int sub = 0; sub < 2; sub++) {
        const int col = sub * 128 + q * 32 + lane;
        bool ok;
        long o;
        if (conv) {
          const int xx = col & (P.bx - 1), r = col >> lbx;
          const int yy = r & (P.by - 1), ii = r >> lby;
          const int img = i0 + ii, y = y0 + yy, xg = x0 + xx;
          ok = img < P.n_img && y < P.H && xg < P.W;
          o = (((long)img * P.H + y) * P.W + xg) * 64 + cb;
        } else {
          const long row = (long)nt * BN + col;
          ok = row < p.S;
          o = row * 64 + cb;
        }
        uint32_t v[32];
        acc_ld32(img, 64, sub * 128 + q * 32 + lane, cb, v);
        if (P.t.dbg & MM_DBG_SKIP_EPI) continue;
        if (P.pool) {
          // 2x2 max over lanes l, l^1 (x) and l^bx (y); bias + ReLU commute with the max and are applied below
#pragma unroll
          for (int j = 0; j < 32; j++) {
            float a = __uint_as_float(v[j]);
            a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 1));
            a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, P.bx));
            v[j] = __float_as_uint(a);
          }
          const int xx = col & (P.bx - 1), r = col >> lbx;
          const int yy = r & (P.by - 1);
          const int y = y0 + yy, xg = x0 + xx;
          ok = ok && !(xx & 1) && !(yy & 1);
          o = (((long)(i0 + (r >> lby)) * (P.H >> 1) + (y >> 1)) * (P.W >> 1) + (xg >> 1)) * 64 + cb;
          if (!ok) continue;
        }
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int j = 0; j < 32; j += 2) {
          float x0v = fmaf(__uint_as_float(v[j]), P.t.out_scale, s_bias[cb + j]);
          float x1v = fmaf(__uint_as_float(v[j + 1]), P.t.out_scale, s_bias[cb + j + 1]);
          if (p.relu) { x0v = fmaxf(x0v, 0.f); x1v = fmaxf(x1v, 0.f); }
          split_f16x2(x0v, x1v, hi[j >> 1], lo[j >> 1]);
          mm_range_track2(racc, hi[j >> 1]);
        }
        if (GEN27) {
          // Line-coalesced stores.  A thread owns 64 B per plane of ONE pixel, so a warp-wide store of it touches 32
          // different 128-byte lines (32 LSU wavefronts per instruction; this epilogue is what bounds the layer).  The
          // two warps of a pixel quadrant (channel halves 0-31 / 32-63 of the same 32 pixels) exchange through an
          // 8 KB scratch [plane][pixel][128 B] (16-byte chunk c of pixel p at slot c ^ (p & 7): conflict-free both ways)
          // in an unused tail of the stage buffers; then one warp stores the hi plane, the other the lo plane, every
          // instruction writing 8 complete lines.
          const uint32_t scr = base + (uint32_t)((q >> 1) * PX_STAGE + PX_X_OFF + (q & 1) * PX_X_PLANE + 16384);
          const uint32_t rowa = scr + (uint32_t)lane * 128u;
#pragma unroll
          for (int k = 0; k < 4; k++) {
            const uint32_t slot = (uint32_t)((((cb >> 3) + k) ^ (lane & 7)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rowa + slot), "r"(hi[4 * k]), "r"(hi[4 * k + 1]),
                         "r"(hi[4 * k + 2]), "r"(hi[4 * k + 3]) : "memory");
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rowa + 4096u + slot), "r"(lo[4 * k]),
                         "r"(lo[4 * k + 1]), "r"(lo[4 * k + 2]), "r"(lo[4 * k + 3]) : "memory");
          }
          asm volatile("bar.sync %0, 64;" ::"r"(3 + q) : "memory");
          const int h = warp >> 2;                                   // plane this warp stores
          const long row0 = (long)nt * BN + sub * 128 + q * 32;
          __half* dstp = yh + (long)h * P.plane_elems + row0 * 64;
#pragma unroll
          for (int r = 0; r < 4; r++) {
            const int idx = r * 32 + lane, px = idx >> 2, c = (idx & 3) * 2;
            const uint32_t ra = scr + (uint32_t)h * 4096u + (uint32_t)px * 128u;
            uint32_t w[8];
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
                         : "r"(ra + (uint32_t)((c ^ (px & 7)) << 4)));
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
                         : "r"(ra + (uint32_t)(((c + 1) ^ (px & 7)) << 4)));
            if (row0 + px < p.S) st_global_256(dstp + (long)px * 64 + c * 8, w);
          }
          asm volatile("bar.sync %0, 64;" ::"r"(3 + q) : "memory");   // scratch free for the next subtile
        } else if (ok && !(P.t.dbg & MM_DBG_PX_ST16)) {
          // 256-bit stores: every instruction writes whole 32-byte sectors (two per plane per thread)
          st_global_256(yh + o, hi);
          st_global_256(yh + o + 16, hi + 8);
          st_global_256(yh + o + P.plane_elems, lo);
          st_global_256(yh + o + P.plane_elems + 16, lo + 8);
        } else if (ok) {
          uint4* dh = reinterpret_cast<uint4*>(yh + o);
          uint4* dl = reinterpret_cast<uint4*>(yh + o + P.plane_elems);
#pragma unroll
          for (int k = 0; k < 4; k++) {
            dh[k] = make_uint4(hi[4 * k], hi[4 * k + 1], hi[4 * k + 2], hi[4 * k + 3]);
            dl[k] = make_uint4(lo[4 * k], lo[4 * k + 1], lo[4 * k + 2], lo[4 * k + 3]);
          }
        }
      }
    }
    mm_range_flag2(P.status, racc);
  } else if (GEN27 && warp >= PX_GEN_WARP0) {
    // =============================== OPERAND PRODUCERS (first VGG layer) ===============================
    // Two groups of four warps take alternate tiles.  A tile is 256 consecutive pixels of ONE image (H*W is a multiple of
    // 256); the group first stages the pixels' 3-channel neighbourhood — the linear range [r0 - W - 1, r0 + 256 + W + 1)
    // of each channel, zero outside the image — in the stage's two unused weight slots with coalesced loads, then every
    // thread gathers the 27 taps of its two pixels from shared memory (left / right image borders by predicate).
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PX_PROD_REGS));
    const int pw = warp - PX_GEN_WARP0;
    const int grp = pw >> 2;
    const int pt = (pw & 3) * 32 + lane;        // 0..127: rows pt and pt + 128 of the group's tiles
    const int W = P.W, hw = P.H * P.W;
    const int span = BN + 2 * W + 2;
    float amax = 0.f;
    uint32_t it = (uint32_t)grp;
    for (long t = blockIdx.x + (long)grp * gridDim.x; t < total_tiles; t += 2L * gridDim.x, it += 2) {
      const int s = it % PX_STAGES;
      const long row0 = t * BN;
      const long img = row0 / hw;
      const int r0 = (int)(row0 - img * hw);
      const float* src = P.gen_src + img * 3 * hw;
      mbar_wait(empty_bar(s), ((it / PX_STAGES) & 1) ^ 1);
      float* stg = reinterpret_cast<float*>(sm + s * PX_STAGE + PX_W_SLOT);
      const int lin0 = r0 - W - 1;
      if (P.t.dbg & MM_DBG_SKIP_OPERANDS) {      // A/B: no operand generation (results wrong)
        __syncwarp();
        if (lane == 0) mbar_arrive(full_bar(s));
        continue;
      }
#pragma unroll 1
      for (int i0 = pt; i0 < 3 * span; i0 += 8 * 128) {
        float q[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {           // eight independent loads in flight per thread
          const int i = i0 + u * 128;
          const int ci = i / span, lin = lin0 + (i - ci * span);
          q[u] = (i < 3 * span && lin >= 0 && lin < hw) ? __ldg(src + (long)ci * hw + lin) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; u++)
          if (i0 + u * 128 < 3 * span) stg[i0 + u * 128] = q[u];
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");
      const uint32_t sx = base + s * PX_STAGE + PX_X_OFF;
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int rr = j * 128 + pt;
        const int x = (r0 + rr) % W;
        const bool xl = x > 0, xr = x < W - 1;
        const float* c = stg + rr + W + 1;
        float v[28];
#pragma unroll
        for (int ci = 0; ci < 3; ci++)
#pragma unroll
          for (int ky = 0; ky < 3; ky++)
#pragma unroll
            for (int kx = 0; kx < 3; kx++) {
              float q = c[ci * span + (ky - 1) * W + (kx - 1)];
              if (kx == 0 && !xl) q = 0.f;
              if (kx == 2 && !xr) q = 0.f;
              v[ci * 9 + ky * 3 + kx] = q;
              amax = fmaxf(amax, fabsf(q));
            }
        v[27] = 0.f;
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int k = 0; k < 28; k += 2) split_f16x2(v[k], v[k + 1], hi[k >> 1], lo[k >> 1]);
        hi[14] = hi[15] = lo[14] = lo[15] = 0u;
        const uint32_t rowaddr = sx + (uint32_t)rr * 64u, sw = (uint32_t)((rr >> 1) & 3);
#pragma unroll
        for (int cch = 0; cch < 4; cch++) {
          const uint32_t a = rowaddr + ((cch ^ sw) << 4);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(hi[4 * cch]), "r"(hi[4 * cch + 1]),
                       "r"(hi[4 * cch + 2]), "r"(hi[4 * cch + 3]) : "memory");
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a + PX_X_PLANE), "r"(lo[4 * cch]),
                       "r"(lo[4 * cch + 1]), "r"(lo[4 * cch + 2]), "r"(lo[4 * cch + 3]) : "memory");
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the MMA's async proxy
      __syncwarp();
      if (lane == 0) mbar_arrive(full_bar(s));
    }
    mm_range_flag(P.status, amax);
  } else {
    // =============================== LOADER ===============================
    if (GEN27) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PX_LOAD_REGS));
    if (warp == T_LOAD_WARP && lane == 0) {
      uint32_t it = 0;
      for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = (int)t;
        int i0 = 0, y0 = 0, x0 = 0;
        if (conv) conv_origin(P, nt, i0, y0, x0);
        for (int si = 0; si < nstage; si++, it++) {
          const int s = it % PX_STAGES;
          mbar_wait(empty_bar(s), ((it / PX_STAGES) & 1) ^ 1);
          mbar_expect_tx(full_bar(s), (uint32_t)ntap * PX_W_SLOT + (GEN27 ? 0u : 2u * xbytes));
          const uint32_t sw = base + s * PX_STAGE, sx = sw + PX_X_OFF;
          const int kx = P.halo ? si / cchunks : 0, cc = P.halo ? si - kx * cchunks : 0;
          for (int ky = 0; ky < ntap; ky++) {
            const int kc = P.halo ? (ky * 3 + kx) * cchunks + cc : si;
            if (P.wcompact) {
              // weights pre-packed for N = 64 (weights.py::pack_px): one 8 KB copy per k chunk
              bulk_g2s(sw + ky * PX_W_SLOT, reinterpret_cast<const uint8_t*>(P.t.Wp) + (size_t)kc * PX_W_SLOT, PX_W_SLOT, full_bar(s));
            } else {
              // rows 0..63 of the packed [hi|lo][k group 4][row group 16][8][8] tile -> compact 8 KB slot: 8 runs of 1 KB
              const uint8_t* src = reinterpret_cast<const uint8_t*>(P.t.Wp) + (size_t)kc * P.t.m_tiles * A_SUB;
#pragma unroll
              for (int r = 0; r < 8; r++)
                bulk_g2s(sw + ky * PX_W_SLOT + r * PX_W_LBO, src + r * A_LBO, 1024, full_bar(s));
            }
          }
          if (P.halo) {
            tma_load_4d(sx, &map_hi, cc * BK, x0 + kx - 1, y0 - 1, i0, full_bar(s));
            tma_load_4d(sx + PX_X_PLANE, &map_lo, cc * BK, x0 + kx - 1, y0 - 1, i0, full_bar(s));
          } else if (conv) {
            const int tap = si / cchunks, c2 = si - tap * cchunks;
            const int dx = tap % 3 - 1, dy = tap / 3 - 1;
            tma_load_4d(sx, &map_hi, c2 * BK, x0 + dx, y0 + dy, i0, full_bar(s));
            tma_load_4d(sx + PX_X_PLANE, &map_lo, c2 * BK, x0 + dx, y0 + dy, i0, full_bar(s));
          } else if (!GEN27) {
            tma_load_2d(sx, &map_hi, si * BK, nt * BN, full_bar(s));
            tma_load_2d(sx + PX_X_PLANE, &map_lo, si * BK, nt * BN, full_bar(s));
          }
        }
      }
    }
    __syncwarp();
  }
}

}  // namespace tma
