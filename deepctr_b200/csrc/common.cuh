// common.cuh — shared helpers for libb2ctr (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include "../../include/b2ctr.h"

namespace b2ctr {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define B2_REQUIRE(cond, ...)                         \
  do {                                                \
    if (!(cond)) {                                    \
      b2ctr::set_error(__VA_ARGS__);                  \
      return B2CTR_ERR_INVALID_ARG;                   \
    }                                                 \
  } while (0)

#define B2_CHECK_LAUNCH(name)                                                         \
  do {                                                                                \
    cudaError_t e__ = cudaGetLastError();                                             \
    if (e__ != cudaSuccess) {                                                         \
      b2ctr::set_error("%s: CUDA launch failed: %s", name, cudaGetErrorString(e__));  \
      return B2CTR_ERR_CUDA;                                                          \
    }                                                                                 \
    b2ctr::count_launch();                                                            \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// Device counter of embedding ids outside [0, vocabulary_size) seen by the gather / scatter kernels of the
// current device (one per device, allocated on first use, never freed).  Out-of-range ids read a ZERO row and
// are skipped by the update kernels (TF-GPU semantics, memory-safe); the host reads the counter with
// b2ctr_embed_oob_count and raises like TF-CPU does (SURVEY.md App. A.1).
unsigned long long* oob_counter();

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Grid for a grid-stride kernel: whole multiples of the SM count, capped by the work.
static inline int grid_for(int64_t work_items, int items_per_block, int blocks_per_sm) {
  int64_t need = ceil_div(work_items, items_per_block);
  int64_t cap = (int64_t)kNumSMs * blocks_per_sm;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

// bf16 hi/lo operand planes of the split-bf16 GEMM (b2ctr_split_planes): padded extent of a [rows, cols] matrix
static inline int64_t planes_rows_pad(int64_t rows) { return (rows + 255) / 256 * 256; }
static inline int64_t planes_cols_pad(int64_t cols) { return cols <= 64 ? 64 : (cols + 127) / 128 * 128; }

// ---- device helpers -------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 lo, __nv_bfloat16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

__device__ __forceinline__ float4 ldg_stream_f4(const float* p) {
  // read-once data (embedding rows, activations): do not allocate in L1
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ldg_stream_f1(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream_f4(float* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
// table row update without a return value: the add happens at the L2 slice (REDG.F32x4)
__device__ __forceinline__ void red_add_f4(float* p, float4 v) {
  asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void red_add_f1(float* p, float v) {
  asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// ---- L2 eviction-priority variants (createpolicy + .L2::cache_hint).  Used by the embedding kernels:
// the 26 dim-1 linear tables (104 MB at C2, twice the 50 MB L2) are marked evict_last, while the
// once-touched streams (embedding rows, activations, gradients) are marked evict_first.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float4 ldg_stream_f4_pol(const float* p, uint64_t pol) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ float ldg_f1_pol(const float* p, uint64_t pol) {
  float r;
  asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ void stg_stream_f4_pol(float* p, float4 v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void red_add_f4_pol(float* p, float4 v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void red_add_f1_pol(float* p, float v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol)
               : "memory");
}

__device__ __forceinline__ bool id_in_range(int64_t id, int64_t vocab) { return (uint64_t)id < (uint64_t)vocab; }
__device__ __forceinline__ void note_oob(unsigned long long* counter) {
  if (counter) atomicAdd(counter, 1ull);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// counter-based hash behind b2ctr_dropout's keep test: element i survives iff
// mix32(seed * 0x9E3779B97F4A7C15 + i) >= rate * 2^32 (also used by the attention kernels' dropout)
__device__ __forceinline__ uint32_t mix32(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
  return (uint32_t)((z ^ (z >> 31)) >> 32);
}

__device__ __forceinline__ int64_t load_idx(const void* p, int64_t off, int dtype) {
  return dtype == B2CTR_IDX_I64 ? reinterpret_cast<const int64_t*>(p)[off]
                                : (int64_t) reinterpret_cast<const int32_t*>(p)[off];
}

__device__ __forceinline__ float act_apply(float x, int act) {
  switch (act) {
    case B2CTR_ACT_RELU: return x > 0.f ? x : 0.f;
    case B2CTR_ACT_SIGMOID: return 1.f / (1.f + expf(-x));
    case B2CTR_ACT_TANH: return tanhf(x);
    default: return x;
  }
}
// derivative expressed through the activation OUTPUT y
__device__ __forceinline__ float act_grad_from_out(float y, int act) {
  switch (act) {
    case B2CTR_ACT_RELU: return y > 0.f ? 1.f : 0.f;
    case B2CTR_ACT_SIGMOID: return y * (1.f - y);
    case B2CTR_ACT_TANH: return 1.f - y * y;
    default: return 1.f;
  }
}

#endif  // __CUDACC__
}  // namespace b2ctr
