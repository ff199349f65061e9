// Per-detection-sum pass of PointNet's two widest contractions (sm_90a, wgmma): layer 5 (K = 128 -> M = 1024) and the
// head (K = 64 -> M = 512, plus the per-detection addend U[det][M]), recomputed with GroupNorm + ReLU + per-detection
// sums fused into the epilogue.  Same arithmetic as gemm_tma_kernel's segsum mode (FP16 hi/lo planes, three MMAs per
// k-step, fp32 accumulation, pre-scaled weights undone by out_scale), but shaped for chains of only 2 or 4 K chunks:
//   * work unit = one 256-column tile x a run of its m-groups (all M/128 of them unless the launch has fewer tiles
//     than SMs): the tile's whole operand, [256 x K] hi and lo, is loaded once by TMA into a resident slot (one
//     full / empty barrier pair per K chunk) and stays there while the weights stream through a ring of 16 KB
//     (kc, m-tile) blocks.  Operand chunk kc of the next unit is refilled as soon as both warpgroups have finished
//     the last m-group's chunk kc, so a unit's first m-group finds its operand already loaded.
//   * the epilogue works straight from the wgmma accumulators (no accumulator image): in the m64n128 D fragment a
//     thread holds rows 16w + lane/4 (+8) at columns 8i + 2(lane%4) + {0,1}, so a 32-column chunk of one row is 8
//     values in each lane of a quad.  Per (row, chunk): one fma + ReLU per value, an in-thread sum, and a transposing
//     quad reduction after which lane q of the quad holds chunk q's sum and issues its 2^-32 fixed-point atomic.  The
//     registers are free as soon as the sums are taken, and the loader never waits for an epilogue.  Each row's
//     affine (and the head's addend) is loaded while the warpgroup's last chains are still running.
//   * the two warpgroups take turns at the tensor core (ping-pong): warpgroup 1 issues an m-group's chains once
//     warpgroup 0 has issued its own, and warpgroup 0 the next m-group's once warpgroup 1 has, so each one's epilogue
//     runs while the other's MMAs do.  Issued together, both would reach their epilogues together and leave the tensor
//     core idle meanwhile.
//   * chunks spanning detections or the tile's end (chunk_tab bit 0 clear) go through a per-warp scratch in which lane
//     l < 16 holds row l's 32 consecutive columns (one chain at a time), and are split into per-detection runs exactly
//     as gemm_tma_kernel does.
// CTA: 384 threads, persistent, one per SM: warps 0-7 the two consumer warpgroups (warpgroup h: column half h),
// warp 8 the loader (warps 9-11 only complete its warpgroup).
#pragma once

namespace tma {

__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("barrier.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

constexpr int SS_THREADS = 384;
constexpr int SS_SCR_LD = 33;                        // scratch row stride (floats): lane l reads row l bank-conflict-free
constexpr int SS_SCRATCH = 16 * SS_SCR_LD * 4;       // per consumer warp: its 16 rows of one chain x 32 columns of one chunk
constexpr int SS_BAR_ISSUED0 = 1, SS_BAR_ISSUED1 = 2;   // named barriers: warpgroup 0 / 1 has issued an m-group's chains
static_assert(256 * T_CONS_REGS + 128 * T_LOAD_REGS <= launch_regs(SS_THREADS) * SS_THREADS,
              "register split exceeds the CTA's pool");

template <int K>
struct SegsumCfg {
  static constexpr int KC = K / BK;                  // K chunks of 32
  static constexpr int OP_BYTES = KC * 2 * B_HALF;   // the unit's operand: per chunk a (hi, lo) pair of 256 x 32 boxes
  // weight ring: one 16 KB (kc, m-tile) block per stage.  A block is read by warpgroup 0 and, one m-group's MMA time
  // later, by warpgroup 1, so the ring holds more than one m-group for the loader to run ahead.
  static constexpr int W_STAGES = K == 128 ? 5 : 8;
  static constexpr int BAR_BYTES = 256;
  static constexpr size_t SMEM = (size_t)OP_BYTES + (size_t)W_STAGES * A_SUB + BAR_BYTES + 8 * SS_SCRATCH + 1024;
  static_assert(K == 64 || K == 128, "gemm_segsum_kernel is built for K = 64 and K = 128");
  static_assert(8 * (2 * KC + 2 * W_STAGES) <= BAR_BYTES, "mbarriers exceed their area");
  static_assert(W_STAGES > KC, "the ring holds more than one m-group's weight blocks");
  static_assert(SMEM <= 227 * 1024, "gemm_segsum_kernel exceeds the 227 KB of shared memory per block");
};

// Units of a launch: column tile nt = u / upt takes m-groups [(u % upt) * mg_per, +mg_per) (clipped to m_tiles).
// mg_per: the longest run whose persistent schedule is no longer than any shorter run's, counting ceil(units / SMs)
// rounds of mg_per m-groups plus about one m-group's time per unit for its operand.  Large launches keep all m-groups
// of a tile in one unit; launches with fewer tiles than SMs split them so that every SM gets work.
static inline int segsum_mg_per(long n_tiles, int mgroups, int sms) {
  int best = mgroups;
  long best_cost = -1;
  for (int mp = mgroups; mp >= 1; mp--) {
    const long units = n_tiles * ((mgroups + mp - 1) / mp);
    const long cost = (units + sms - 1) / sms * (mp + 1);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = mp; }
  }
  return best;
}

template <int K>
static __global__ void __launch_bounds__(SS_THREADS, 1)
gemm_segsum_kernel(const TmaP P, const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                   int mg_per) {
  using Cfg = SegsumCfg<K>;
  constexpr int KC = Cfg::KC, WS = Cfg::W_STAGES;
  const GemmP& p = P.t.g;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;      // operand slot: chunk kc = hi box at base + kc*32 KB, lo box + 16 KB
  uint8_t* sm = smem_raw + (base - raw);
  const uint32_t wbase = base + Cfg::OP_BYTES;
  const uint32_t bar0 = wbase + WS * A_SUB;
  auto op_full = [&](int kc) { return bar0 + 8u * kc; };
  auto op_empty = [&](int kc) { return bar0 + 8u * (KC + kc); };
  auto w_full = [&](int s) { return bar0 + 8u * (2 * KC + s); };
  auto w_empty = [&](int s) { return bar0 + 8u * (2 * KC + WS + s); };
  float* scratch = reinterpret_cast<float*>(sm + Cfg::OP_BYTES + WS * A_SUB + Cfg::BAR_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mgroups = P.t.m_tiles;
  const int upt = (mgroups + mg_per - 1) / mg_per;
  const long units = (long)p.num_tiles * upt;

  if (tid == 0) {
    for (int kc = 0; kc < KC; kc++) {
      mbar_init(op_full(kc), 1);                  // the loader's expect_tx arrive (hi + lo box)
      mbar_init(op_empty(kc), T_EPI_WARPS);       // one arrive per consumer warp after the unit's last m-group
    }
    for (int s = 0; s < WS; s++) {
      mbar_init(w_full(s), 1);
      mbar_init(w_empty(s), T_EPI_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto tile_cols = [&](int nt, int& g, int& c0, int& len) {
    if (p.tile_tab) { int4 tt = p.tile_tab[nt]; g = tt.x; c0 = tt.y; len = tt.z; }
    else { g = nt / p.tiles_per_group; c0 = (nt - g * p.tiles_per_group) * BN; len = min(BN, p.S - c0); }
  };

  if (warp < T_EPI_WARPS) {
    // =============================== CONSUMERS: MMA + epilogue ===============================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(T_CONS_REGS));
    const int half = warp >> 2, w = warp & 3, quad = lane & 3;
    float* scr = scratch + warp * 16 * SS_SCR_LD;
    uint32_t it = 0, un = 0;   // weight blocks consumed (ring position), units processed
    bool first = true;         // no m-group issued yet by this warpgroup
    float acc[2][64];          // chain mb: rows 64 mb + fragment row, columns 128 half + fragment column
    for (long u = blockIdx.x; u < units; u += gridDim.x, un++) {
      const int nt = (int)(u / upt);
      const int mg0 = (int)(u - (long)nt * upt) * mg_per, mg1 = min(mgroups, mg0 + mg_per);
      int g = 0, c0 = 0, len = BN;
      tile_cols(nt, g, c0, len);
      const int4 ct = __ldg(P.chunk_tab + (long)nt * 2 + half);   // same address in every lane: one transaction
      // chunk quad of this lane: after the quad reduction it holds that chunk's sums and issues their atomics
      const int qdesc = quad == 0 ? ct.x : quad == 1 ? ct.y : quad == 2 ? ct.z : ct.w;
      const bool qsingle = qdesc & 1;
      const int qdet = qdesc >> 1;
      for (int mg = mg0; mg < mg1; mg++) {
        const bool last = mg == mg1 - 1;
        // this warpgroup's turn: warpgroup 1 after warpgroup 0 has issued this m-group, warpgroup 0 after warpgroup 1
        // has issued the previous one
        if (half) bar_sync(SS_BAR_ISSUED0, 256);
        else if (!first) bar_sync(SS_BAR_ISSUED1, 256);
        first = false;
        for (int kc = 0; kc < KC; kc++, it++) {
          const int s = it % WS;
          if (mg == mg0) mbar_wait(op_full(kc), un & 1);
          mbar_wait(w_full(s), (it / WS) & 1);
          const uint32_t sa = wbase + s * A_SUB, sb = base + kc * 2 * B_HALF + half * (128 / 8) * 512;
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 2; ks++) {
            const uint64_t b_hi = smem_desc_sw64(sb + ks * 32), b_lo = smem_desc_sw64(sb + B_HALF + ks * 32);
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
          wgmma_wait<1>();   // the previous chunk's wgmmas are done: release its weight block (and operand chunk)
          if (kc > 0) {
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(w_empty((it - 1) % WS));
              if (last) mbar_arrive(op_empty(kc - 1));
            }
          }
        }
        bar_arrive(half ? SS_BAR_ISSUED1 : SS_BAR_ISSUED0, 256);   // the last chunk is in flight: pass the turn
        // the epilogue's per-row constants, loaded while the chains run: the GroupNorm affine with bias and addend folded
        // in, y = relu(acc * a2 + b2), rows ri = 2 mb + h -> tile row 64 mb + 16 w + lane/4 + 8 h
        const int rbase = mg * 128 + 16 * w + (lane >> 2);
        float a2[4], b2[4][4];
#pragma unroll
        for (int ri = 0; ri < 4; ri++) {
          const int co = rbase + 64 * (ri >> 1) + 8 * (ri & 1);
          float na = 0.f, nb = 0.f, bv = 0.f;
          if (co < p.M) {
            na = __ldg(p.sc + (long)g * p.M + co);
            nb = __ldg(p.sh + (long)g * p.M + co);
            if (p.bias) bv = __ldg(p.bias + co);
          }
          a2[ri] = P.t.out_scale * na;
#pragma unroll
          for (int c = 0; c < 4; c++) {
            float adc = 0.f;
            if (p.addend && co < p.M) {
              const int d = (c == 0 ? ct.x : c == 1 ? ct.y : c == 2 ? ct.z : ct.w) >> 1;
              adc = __ldg(p.addend + (long)d * p.ld_add + co);
            }
            b2[ri][c] = fmaf(bv + adc, na, nb);
          }
        }
        wgmma_wait<0>();
        fence_acc(acc[0]);
        fence_acc(acc[1]);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(w_empty((it - 1) % WS));
          if (last) mbar_arrive(op_empty(KC - 1));
        }

        // ---- epilogue: GroupNorm affine + ReLU, summed per (row, 32-column chunk) ----
#pragma unroll
        for (int ri = 0; ri < 4; ri++) {
          const int mb = ri >> 1, h = ri & 1;
          const int co = rbase + 64 * mb + 8 * h;
          const bool rowok = co < p.M;
          float cs[4];   // this lane's part of chunk c's sum
#pragma unroll
          for (int c = 0; c < 4; c++) {
            float r0 = 0.f, r1 = 0.f;
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
              const int i = 16 * c + 4 * jj + 2 * h;
              r0 += fmaxf(fmaf(acc[mb][i], a2[ri], b2[ri][c]), 0.f);
              r1 += fmaxf(fmaf(acc[mb][i + 1], a2[ri], b2[ri][c]), 0.f);
            }
            cs[c] = r0 + r1;
          }
          // transposing quad reduction: after the xor-1 step lane q keeps chunks q&1 and (q&1) + 2, after the xor-2 step
          // chunk q alone, summed over the quad's four lanes
          const bool b0 = quad & 1, b1 = quad & 2;
          const float x = __shfl_xor_sync(0xffffffffu, b0 ? cs[0] : cs[1], 1);
          const float y = __shfl_xor_sync(0xffffffffu, b0 ? cs[2] : cs[3], 1);
          const float k0 = (b0 ? cs[1] : cs[0]) + x, k1 = (b0 ? cs[3] : cs[2]) + y;
          const float sum = (b1 ? k1 : k0) + __shfl_xor_sync(0xffffffffu, b1 ? k0 : k1, 2);
          if (qsingle && rowok)
            atomicAdd(P.segsum + (long)qdet * p.M + co, __float2ull_rn(sum * 4294967296.f));
        }
        // chunks that span detections or end inside the tile: per chain, lane l < 16 takes row l of the warp's 16 from
        // the scratch and splits it into per-detection runs (unrolled: the accumulators are indexed by c and mb)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const int desc = c == 0 ? ct.x : c == 1 ? ct.y : c == 2 ? ct.z : ct.w;
          const int col0 = half * 128 + c * 32;
          if ((desc & 1) || col0 >= len) continue;   // warp-uniform
#pragma unroll
          for (int mb = 0; mb < 2; mb++) {
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
              for (int jj = 0; jj < 4; jj++) {
                float* dst = scr + (8 * h + (lane >> 2)) * SS_SCR_LD + 8 * jj + 2 * quad;
                const int i = 16 * c + 4 * jj + 2 * h;
                dst[0] = acc[mb][i];
                dst[1] = acc[mb][i + 1];
              }
            __syncwarp();
            const int co = mg * 128 + mb * 64 + 16 * w + lane;
            if (lane < 16 && co < p.M) {
              const float bv = p.bias ? __ldg(p.bias + co) : 0.f;
              const float na = __ldg(p.sc + (long)g * p.M + co), nb = __ldg(p.sh + (long)g * p.M + co);
              const int nvalid = min(32, len - col0);
              const float* row = scr + lane * SS_SCR_LD;
              int dcur = desc >> 1;
              float run = 0.f;
              for (int j = 0; j < nvalid; j++) {
                float xv = fmaf(row[j], P.t.out_scale, bv);
                const int d = __ldg(p.seg + c0 + col0 + j);
                if (p.addend) xv += __ldg(p.addend + (long)d * p.ld_add + co);
                if (d != dcur) {
                  atomicAdd(P.segsum + (long)dcur * p.M + co, __float2ull_rn(run * 4294967296.f));
                  run = 0.f; dcur = d;
                }
                run += fmaxf(fmaf(xv, na, nb), 0.f);
              }
              atomicAdd(P.segsum + (long)dcur * p.M + co, __float2ull_rn(run * 4294967296.f));
            }
            __syncwarp();
          }
        }
      }
    }
    if (!half && !first) bar_sync(SS_BAR_ISSUED1, 256);   // matches warpgroup 1's arrive after the last m-group
  } else {
    // =============================== LOADER (operand chunks + weight blocks) ===============================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(T_LOAD_REGS));
    if (warp == T_LOAD_WARP && lane == 0) {
      uint32_t it = 0, un = 0;
      for (long u = blockIdx.x; u < units; u += gridDim.x, un++) {
        const int nt = (int)(u / upt);
        const int mg0 = (int)(u - (long)nt * upt) * mg_per, mg1 = min(mgroups, mg0 + mg_per);
        int g = 0, c0 = 0, len = BN;
        tile_cols(nt, g, c0, len);
        const int row0 = (int)((long)g * p.x_gs + c0);
        for (int mg = mg0; mg < mg1; mg++)
          for (int kc = 0; kc < KC; kc++, it++) {
            if (mg == mg0) {   // operand chunk kc, once the previous unit's last m-group has read it
              mbar_wait(op_empty(kc), (un & 1) ^ 1);
              mbar_expect_tx(op_full(kc), 2u * B_HALF);
              const uint32_t sb = base + kc * 2 * B_HALF;
              tma_load_2d(sb, &map_hi, kc * BK, row0, op_full(kc));
              tma_load_2d(sb + B_HALF, &map_lo, kc * BK, row0, op_full(kc));
            }
            const int s = it % WS;
            mbar_wait(w_empty(s), ((it / WS) & 1) ^ 1);
            mbar_expect_tx(w_full(s), (uint32_t)A_SUB);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(P.t.Wp) + ((size_t)kc * mgroups + mg) * A_SUB;
            bulk_g2s(wbase + s * A_SUB, src, (uint32_t)A_SUB, w_full(s));
          }
      }
    }
    __syncwarp();
  }
}

}  // namespace tma
