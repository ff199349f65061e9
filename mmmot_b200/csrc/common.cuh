// Shared helpers for libmmmot_sm90a.so (sm_90a only; no torch headers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/mmmot_b200.h"

#define MM_CUDA(x)                                    \
  do {                                                \
    cudaError_t _e = (x);                             \
    if (_e != cudaSuccess) return (int)_e;            \
  } while (0)

#define MM_LAUNCH_CHECK()                             \
  do {                                                \
    mm_count_launch();                                \
    cudaError_t _e = cudaGetLastError();              \
    if (_e != cudaSuccess) return (int)_e;            \
  } while (0)

#define MM_TRY(x)                                     \
  do {                                                \
    int _r = (x);                                     \
    if (_r != 0) return _r;                           \
  } while (0)

void mm_count_launch();
int mm_debug_flags();
int mm_kseg_chunks();  // K-segment length (in 32-wide chunks) of the tensor-core conv engine, 0 = off (mmmot_set_kseg)
int mm_engine();  // 0 auto, 1 FP32 FFMA engine, 2 tensor-core (wgmma) engine (mmmot_set_engine)
// Per-launch timing hook (mmmot_timing_*): every hot kernel of the path is bracketed by CUDA events on the launching
// stream while timing is enabled, tagged with (stage, layer) and its ALGORITHMIC work (FLOPs, compulsory HBM bytes).
enum {
  MM_T_VGG0 = 0,          // .. +12 : VGG conv i (tag 0 includes its im2col pre-pass)
  MM_T_VGG_POOL = 13,     // 2x2 max-pools + SkipPool plane means + heads
  MM_T_PN_L1 = 14,        // PointNet 3 -> 64 (statistics + apply)
  MM_T_PN_L2 = 15, MM_T_PN_L3 = 16, MM_T_PN_L4 = 17,
  MM_T_PN_NORM = 18,      // GroupNorm+ReLU -> FP16 planes passes between PointNet layers
  MM_T_PN_L5A = 19, MM_T_PN_L5B = 20,        // 128 -> 1024: statistics pass, normalise + segment-sum pass
  MM_T_PN_HEADA = 21, MM_T_PN_HEADB = 22,    // head 64 -> 512, two passes
  MM_T_AFF_L1 = 23, MM_T_AFF_MEAN = 24, MM_T_AFF_L2 = 25, MM_T_AFF_L3 = 26, MM_T_AFF_LOGIT = 27,
  MM_T_LP = 28,
  MM_T_PN_MOM128 = 29, MM_T_PN_MOM64 = 30,   // input moments of layer 5 and of the head (their GroupNorm statistics)
  MM_T_PN_MOMFIN = 31,                       // their slice tables, fixed-order reductions and fp64 statistics
  MM_T_FLOW = 32,         // association programme of K-frame samples (min-cost flow)
  MM_T_COUNT = 33
};
bool mm_timing_on();
void mm_timing_begin(cudaStream_t st, int tag, double flop, double bytes);
void mm_timing_end(cudaStream_t st);

// SM count of the CURRENT device (cached per device; the library may be used on several GPUs from one process)
int mm_sm_count(int* sms);
// Opt a kernel into > 48 KB of dynamic shared memory, once per (kernel, device): `done` is a per-call-site bit mask
// indexed by device ordinal.  Safe to race: setting the attribute twice is harmless.
#include <atomic>
template <typename K>
static inline int mm_ensure_smem(K kernel, size_t bytes, std::atomic<unsigned long long>& done) {
  int dev = 0;
  MM_CUDA(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(done.load(std::memory_order_acquire) & bit)) {
    MM_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    done.fetch_or(bit, std::memory_order_release);
  }
  return 0;
}

static inline size_t mm_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
static inline int mm_cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// GroupNorm partials of all three contraction engines.  A thread holds a run of k values of one channel in registers,
// takes their fp32 mean pv, sums d = y - pv (s1) and d^2 (s2) in fp32 and folds the run into its fp64 (sum y, sum y^2)
// as (k pv + s1, k pv^2 + 2 pv s1 + s2) -- a two-pass mean and variance per run, combined exactly in fp64.  The fp32
// rounding then scales with the spread of the run, not with its mean: summing y^2 directly loses about (mean/std)^2 of
// relative accuracy in var = sum y^2 / n - mean^2 (gn_finalize), the centred runs about mean/std, GroupNorm's own
// conditioning (DESIGN.md §4.2).  A pivot taken from the run's values instead (say its first) is worse than no shift
// when that value is far from the rest, as a rare positive value among ReLU zeros is.
__device__ __forceinline__ void stat_fold(double& f1, double& f2, int k, float pv, float s1, float s2) {
  const double p = pv, a = s1;
  f1 += k * p + a;
  f2 += p * (k * p + 2.0 * a) + (double)s2;
}

// Bump allocator over the caller-provided workspace.  The first MM_STATUS_BYTES of EVERY workspace are the status
// block (word 0 = range flag, see mmmot_status_reset / mmmot_status_check): all stages carve behind it, so a flag
// raised by one stage survives the stages that reuse the workspace after it.
constexpr size_t MM_STATUS_BYTES = 256;
struct MmArena {
  char* base;
  size_t cap, off;
  bool dry;  // dry run: only measure; take() returns the byte offset itself (mmmot_debug_stage_layout reads a carve that way)
  MmArena(void* p, size_t c) : base((char*)p), cap(c), off(MM_STATUS_BYTES), dry(p == nullptr) {}
  int* status() const { return dry ? nullptr : reinterpret_cast<int*>(base); }
  template <typename T>
  T* take(size_t n) {
    size_t bytes = mm_align(n * sizeof(T));
    char* r = dry ? reinterpret_cast<char*>(static_cast<uintptr_t>(off)) : base + off;
    off += bytes;
    return (T*)r;
  }
  bool ok() const { return dry || off <= cap; }
};

__device__ __forceinline__ float mm_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// FP16 range guard.  Activations enter the tensor cores as FP16 hi/lo pairs; cvt.rn.satfinite clamps |x| >= 65504
// silently, so every conversion site tracks the largest magnitude it converted and raises bit 0 of the workspace
// status word once per thread when the clamp was hit.  The host reads it with mmmot_status_check -> MMMOT_E_RANGE.
constexpr float MM_F16_MAX = 65504.f;
__device__ __forceinline__ void mm_range_flag(int* status, float amax) {
  if (status && !(amax < MM_F16_MAX)) atomicOr(status, 1);      // also catches NaN
}
// packed variant: acc = running max of |hi| over f16x2 words (starts at 0)
__device__ __forceinline__ void mm_range_track2(uint32_t& acc, uint32_t hi2) {
  asm("{\n\t.reg .b32 t;\n\tabs.f16x2 t, %1;\n\tmax.NaN.f16x2 %0, %0, t;\n\t}" : "+r"(acc) : "r"(hi2));
}
__device__ __forceinline__ void mm_range_flag2(int* status, uint32_t acc) {
  if (status && ((acc & 0xFFFFu) >= 0x7BFFu || (acc >> 16) >= 0x7BFFu)) atomicOr(status, 1);
}
