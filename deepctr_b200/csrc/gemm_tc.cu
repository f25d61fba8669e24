// gemm_tc.cu — fp32-in / fp32-out GEMM on the Hopper tensor cores (wgmma, sm_90a).
//
// Precision mode B2CTR_GEMM_BF16X3: every fp32 operand x is split into two bf16 values
//   x = hi + lo,  hi = bf16(x),  lo = bf16(x - hi)           (|x - hi - lo| <= 2^-17 |x|)
// and the product is accumulated in fp32 registers as  hi*hi + hi*lo + lo*hi  (the dropped lo*lo term is
// <= 2^-16 relative), i.e. three bf16 wgmma per K-step.  That keeps the reference's fp32 logits within the
// 1e-4 bar at ~1/3 of the bf16 tensor throughput instead of the FFMA pipe.
//
// Every kernel computes 128 x BN output tiles.  The fp32 -> (hi, lo) split is done once per operand into bf16
// planes in global memory (or the producer warps generate the A operand, CIN / DIN attention).  Operand tiles sit in
// shared memory in the 128-byte-swizzled layouts wgmma reads through matrix descriptors (K-major: 16-byte chunk
// index XOR row % 8; MN-major: 64-element atoms of 64 k-rows).  The accumulator lives in the registers of two
// consumer warpgroups.
//   gemm_planes_ws_kernel (variant 4, the default and the only production path): persistent, warp-specialised: TMA
//       or generating producer warps fill a stage ring guarded by mbarriers while the two consumer warpgroups
//       multiply and run the epilogue (plain outputs: staged in shared memory and stored with TMA).
//   gemm_planes_kernel (variant 3): non-persistent, cp.async, register epilogue.  It issues the same wgmma in the
//       same order per output element, so it is the reference the bit-exact tests compare variant 4 against.
#include <cuda.h>          // CUtensorMap + enums only: the encoder is resolved through the runtime (no libcuda link)
#include <cuda_bf16.h>
#include "common.cuh"

namespace b2ctr {

constexpr int kTM = 128;       // rows of the output tile: two warpgroups x 64
constexpr int kTK = 64;        // K elements per stage = one 128-byte swizzle atom of bf16
constexpr int kTcThreads = 256;   // gemm_planes_kernel: two warpgroups that both fill and multiply every stage

struct PlaneArgs {
  // K-major planes: [rows_pad, k_pad] (k contiguous).  MN-major planes: [k_pad, rows_pad] (row index
  // contiguous) - the natural layout of a row-major operand whose reduction dim is its row index
  // (wgrad: X^T, dZ^T; forward: W).  *_pitch = elements between consecutive plane rows.
  const __nv_bfloat16* a_hi; const __nv_bfloat16* a_lo;
  const __nv_bfloat16* b_hi; const __nv_bfloat16* b_lo;
  int64_t a_pitch, b_pitch;
  int a_mn, b_mn;
  float* c; const float* bias; float* ws;
  int64_t m, n, k_pad;
  int64_t ldc;
  int64_t k_per_split;
  float alpha;
  int act, accumulate, splits;
  // CIN mode (cin_on): the A operand is never stored anywhere - the producer warps GENERATE its bf16 hi/lo tile
  // in shared memory from the two factors of the outer product (deepctr/layers/interaction.py:287-297):
  //   A[r, i*hp + j] = t0[r*ld0 + i] * xk[r*ldk + j]   (j < h, i < m; zero otherwise),  r = (sample, embedding dim)
  // a_mn = 0: A is [rows, m*hp] (forward, M = r);  a_mn = 1: A^T, i.e. M = i*hp + j and K = r (filter gradient).
  const float* cin_t0; const float* cin_xk;
  int64_t cin_ld0, cin_ldk, cin_rows;
  int cin_m, cin_h, cin_hp, cin_on;
  // FOLD epilogue (CIN backward): dT0 [rows, cin_ld0] and dXk [rows, fold_ldx], both accumulated with red.add
  float* fold_dt0; float* fold_dxk; int64_t fold_ldx;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
// ---- warpgroup MMA (wgmma.mma_async, sm_90a) ----------------------------------------------------------------
// Shared-memory matrix descriptor with 128-byte swizzle: start address >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32 |
// layout SWIZZLE_128B (1) << 62.
//   K-major : rows of 128 B (64 bf16 along K), groups of 8 rows 1024 B apart (SBO); LBO unused (1).
//   MN-major: 64-element atoms along M/N 8192 B apart (LBO), groups of 8 k-rows 1024 B apart (SBO).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, int mn) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(mn ? 512 : 1) << 16) | (64ull << 32) | (1ull << 62);
}
// one K-step = 16 bf16 along K: 32 B inside the swizzled row (K-major) or 16 k-rows = 2048 B (MN-major)
__device__ __forceinline__ uint64_t wgmma_desc_k(uint32_t base, int ks, int mn) {
  return wgmma_desc(mn ? base + ks * 2048 : base + ks * 32, mn);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// m64nNk16, D (fp32, registers) += A (bf16, smem) * B (bf16, smem); TA / TB: 1 = operand stored MN-major
template <int N> struct Wgmma;
template <> struct Wgmma<32> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<64> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<128> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<256> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[128], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(1), "n"(TA), "n"(TB));
  }
};
// One 64-deep k-block of the split product for the 64 rows of the calling warpgroup: 4 K-steps x
// (hi*hi + hi*lo + lo*hi), committed as one wgmma group.  Stage at `st`: A hi / lo planes (kTM rows), then B hi / lo
// (BN rows); the warpgroup `wg` reads rows [64 wg, 64 wg + 64) of A, which start 8192 B into the plane in both
// layouts.  TA / TB (1 = MN-major) are template parameters and the accumulator is not touched between the MMAs and
// the commit: a control-flow join or a register access there makes ptxas close the group early (it then commits an
// empty group, and wgmma_wait<1> waits for the k-block just issued).  The caller fences the accumulator
// (fence_acc) only after wgmma_wait<0>.
template <int BN, int TA, int TB>
__device__ __forceinline__ void wg_kblock(float (&d)[BN / 2], uint32_t st, int wg) {
  constexpr uint32_t A_PLANE = kTM * 128, B_PLANE = BN * 128;
  const uint32_t a_hi = st + wg * 8192, a_lo = a_hi + A_PLANE, b_hi = st + 2 * A_PLANE, b_lo = b_hi + B_PLANE;
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < kTK / 16; ++ks) {
    const uint64_t dah = wgmma_desc_k(a_hi, ks, TA), dal = wgmma_desc_k(a_lo, ks, TA);
    const uint64_t dbh = wgmma_desc_k(b_hi, ks, TB), dbl = wgmma_desc_k(b_lo, ks, TB);
    Wgmma<BN>::template mma<TA, TB>(d, dah, dbh);
    Wgmma<BN>::template mma<TA, TB>(d, dah, dbl);
    Wgmma<BN>::template mma<TA, TB>(d, dal, dbh);
  }
  wgmma_commit();
}
// Half a k-block (K-steps KS0, KS0 + 1) of the split product for all 128 rows of the tile, from ONE warpgroup (the
// ping-pong consumers): 12 wgmma committed as one group, alternating between the accumulators of the two 64-row
// halves so that consecutive MMAs do not depend on each other.  Each accumulator sees its K-steps and the three
// products in wg_kblock's order, so the sums are bit-identical.  (Issuing one half's 12 dependent MMAs and then the
// other's halves the tensor-pipe throughput.)
template <int BN, int TA, int TB, int KS0>
__device__ __forceinline__ void tile_kblock_half(float (&d0)[BN / 2], float (&d1)[BN / 2], uint32_t st) {
  constexpr uint32_t A_PLANE = kTM * 128, B_PLANE = BN * 128;
  const uint32_t a_hi = st, a_lo = a_hi + A_PLANE, b_hi = st + 2 * A_PLANE, b_lo = b_hi + B_PLANE;
  wgmma_fence();
#pragma unroll
  for (int ks = KS0; ks < KS0 + 2; ++ks) {
    const uint64_t dah0 = wgmma_desc_k(a_hi, ks, TA), dal0 = wgmma_desc_k(a_lo, ks, TA);
    const uint64_t dah1 = wgmma_desc_k(a_hi + 8192, ks, TA), dal1 = wgmma_desc_k(a_lo + 8192, ks, TA);
    const uint64_t dbh = wgmma_desc_k(b_hi, ks, TB), dbl = wgmma_desc_k(b_lo, ks, TB);
    Wgmma<BN>::template mma<TA, TB>(d0, dah0, dbh);
    Wgmma<BN>::template mma<TA, TB>(d1, dah1, dbh);
    Wgmma<BN>::template mma<TA, TB>(d0, dah0, dbl);
    Wgmma<BN>::template mma<TA, TB>(d1, dah1, dbl);
    Wgmma<BN>::template mma<TA, TB>(d0, dal0, dbh);
    Wgmma<BN>::template mma<TA, TB>(d1, dal1, dbh);
  }
  wgmma_commit();
}
// Calls f(Major<a_mn>, Major<b_mn>) with the operand majorness as compile-time constants: the consumer loop is
// instantiated per layout and the branch runs once per launch, outside every k-block.
template <int V> struct Major { static constexpr int value = V; };
template <class F>
__device__ __forceinline__ void with_majorness(int a_mn, int b_mn, F&& f) {
  if (a_mn) {
    if (b_mn) f(Major<1>{}, Major<1>{});
    else f(Major<1>{}, Major<0>{});
  } else {
    if (b_mn) f(Major<0>{}, Major<1>{});
    else f(Major<0>{}, Major<0>{});
  }
}

// Epilogue straight from the accumulator fragment of m64nBN: thread (warp w of the warpgroup, lane l) holds rows
// row0 + 16w + l/4 (+ 8) and columns n0 + 8i + 2(l % 4) + {0, 1} in d[4i + {0, 1}] (and d[4i + {2, 3}] for the
// row + 8).  Each group of four lanes writes 32 contiguous bytes of a row.  C = act(alpha acc [+ C] [+ bias]);
// split-K slices go to the workspace instead (ws[z][m][n], reduced by tc_splitk_reduce_kernel).  The persistent
// kernel uses it for what store_acc_tma cannot store (accumulate, unaligned C, split-K with n % 4 != 0).
template <int BN>
__device__ __forceinline__ void store_acc(const PlaneArgs& g, const float (&d)[BN / 2], int64_t row0, int64_t n0,
                                          int64_t z) {
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const bool vec = (g.ldc % 2 == 0) && ((reinterpret_cast<uintptr_t>(g.c) & 7) == 0);
  const bool vec_ws = g.n % 2 == 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t gm = row0 + w * 16 + (lane >> 2) + 8 * h;
    if (gm >= g.m) continue;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int64_t gn = n0 + 8 * i + 2 * (lane & 3);
      if (gn >= g.n) continue;
      const bool two = gn + 1 < g.n;
      float v0 = g.alpha * d[4 * i + 2 * h], v1 = g.alpha * d[4 * i + 2 * h + 1];
      if (g.splits > 1) {
        float* wp = g.ws + (z * g.m + gm) * g.n + gn;
        if (two && vec_ws) *reinterpret_cast<float2*>(wp) = make_float2(v0, v1);
        else {
          wp[0] = v0;
          if (two) wp[1] = v1;
        }
        continue;
      }
      float* cp = g.c + gm * g.ldc + gn;
      if (two && vec) {
        if (g.accumulate) {
          const float2 o = *reinterpret_cast<const float2*>(cp);
          v0 += o.x; v1 += o.y;
        }
        if (g.bias) { v0 += __ldg(g.bias + gn); v1 += __ldg(g.bias + gn + 1); }
        *reinterpret_cast<float2*>(cp) = make_float2(act_apply(v0, g.act), act_apply(v1, g.act));
      } else {
        if (g.accumulate) v0 += cp[0];
        if (g.bias) v0 += g.bias[gn];
        cp[0] = act_apply(v0, g.act);
        if (two) {
          if (g.accumulate) v1 += cp[1];
          if (g.bias) v1 += g.bias[gn + 1];
          cp[1] = act_apply(v1, g.act);
        }
      }
    }
  }
}

__device__ __forceinline__ unsigned char* align1024(unsigned char* p) {
  return reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

__global__ void tc_splitk_reduce_kernel(const PlaneArgs g) {
  const int64_t total = g.m * g.n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t gm = i / g.n, gn = i - gm * g.n;
    float v = 0.f;
    for (int z = 0; z < g.splits; ++z) v += g.ws[(int64_t)z * total + i];
    if (g.accumulate) v += g.c[gm * g.ldc + gn];
    if (g.bias) v += g.bias[gn];
    g.c[gm * g.ldc + gn] = act_apply(v, g.act);
  }
}
// The same reduction for n % 4 == 0: a thread owns four consecutive outputs of a row, loads the slices' float4 partials
// kReduceBatch at a time (all in flight before the first add) and adds them in ascending z from 0.f, then accumulate,
// bias and activation, as tc_splitk_reduce_kernel does: bit-identical results.  The scalar kernel issued one load per
// add from a loop with a run-time trip count, so at 256 x 128 x 64 slices its 32768 threads were load-latency-bound.
constexpr int kReduceBatch = 16;
__global__ void __launch_bounds__(128) tc_splitk_reduce4_kernel(const PlaneArgs g) {
  const int64_t total4 = g.m * g.n / 4;
  const float4* ws = reinterpret_cast<const float4*>(g.ws);
  const bool vec_c = g.ldc % 4 == 0 && ((reinterpret_cast<uintptr_t>(g.c) & 15) == 0);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int z0 = 0; z0 < g.splits; z0 += kReduceBatch) {
      float4 p[kReduceBatch];
#pragma unroll
      for (int j = 0; j < kReduceBatch; ++j)
        if (z0 + j < g.splits) p[j] = __ldcs(ws + (int64_t)(z0 + j) * total4 + i);
#pragma unroll
      for (int j = 0; j < kReduceBatch; ++j)
        if (z0 + j < g.splits) {
          v[0] += p[j].x; v[1] += p[j].y; v[2] += p[j].z; v[3] += p[j].w;
        }
    }
    const int64_t gm = (4 * i) / g.n, gn = 4 * i - gm * g.n;
    float* cp = g.c + gm * g.ldc + gn;
    if (g.accumulate) {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] += cp[e];
    }
    if (g.bias) {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] += __ldg(g.bias + gn + e);
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = act_apply(v[e], g.act);
    if (vec_c) *reinterpret_cast<float4*>(cp) = make_float4(v[0], v[1], v[2], v[3]);
    else {
#pragma unroll
      for (int e = 0; e < 4; ++e) cp[e] = v[e];
    }
  }
}
// split-K reduction of a persistent-kernel launch: the float4 kernel when the workspace rows allow it, with blocks
// small enough that the grid covers the SMs (256 x 128 is 8192 threads, 128 x 64 only 2048)
static void splitk_reduce(const PlaneArgs& pa, cudaStream_t st) {
  if (pa.n % 4 != 0 || ((uintptr_t)pa.ws & 15) != 0) {
    tc_splitk_reduce_kernel<<<grid_for(pa.m * pa.n, 256, 4), 256, 0, st>>>(pa);
    return;
  }
  const int64_t total4 = pa.m * pa.n / 4;
  int tpb = 128;
  while (tpb > 32 && ceil_div(total4, tpb) < kNumSMs) tpb /= 2;
  tc_splitk_reduce4_kernel<<<grid_for(total4, tpb, 2048 / tpb), tpb, 0, st>>>(pa);
}

// ================================================================================================
// Operand planes and the non-persistent reference kernel (variant 3)
// The fp32 -> (hi, lo) bf16 split is done ONCE per operand by a streaming kernel into planes in workspace memory,
// so no CTA re-converts an operand tile another CTA also reads.  A row-contiguous operand keeps its layout
// (MN-major planes, the wgmma descriptors do the transposition); only a row-contiguous B under a 32-wide N tile
// (an MN-major tile is one 64-wide atom) goes through the transposing split into K-major planes.
// ================================================================================================
// dst planes [rows_pad, k_pad] <- src(r, k) = p[r*sr + k*sk]; zero outside [rows, k).
// K-contiguous source: thread = (row, 8 consecutive k).
__global__ void __launch_bounds__(256)
    split_planes_kernel(const float* __restrict__ p, int64_t sr, int64_t rows, int64_t k, int64_t rows_pad,
                        int64_t k_pad, __nv_bfloat16* hi, __nv_bfloat16* lo, int vec_ok) {
  const int64_t chunks = k_pad / 8;
  const int64_t total = rows_pad * chunks;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / chunks;
    const int64_t k0 = (t - r * chunks) * 8;
    float v[8];
    if (r < rows && vec_ok && k0 + 8 <= k) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(p + r * sr + k0));
      const float4 b = __ldg(reinterpret_cast<const float4*>(p + r * sr + k0) + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (r < rows && k0 + j < k) ? __ldg(p + r * sr + k0 + j) : 0.f;
    }
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v[2 * j]), h1 = __float2bfloat16_rn(v[2 * j + 1]);
      h[j] = pack_bf16(h0, h1);
      l[j] = pack_bf16(__float2bfloat16_rn(v[2 * j] - __bfloat162float(h0)),
                       __float2bfloat16_rn(v[2 * j + 1] - __bfloat162float(h1)));
    }
    *reinterpret_cast<uint4*>(hi + r * k_pad + k0) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(lo + r * k_pad + k0) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}
// Row-contiguous source (src(r,k) = p[k*sk + r]): 64 x 64 tile transposed through shared memory.
__global__ void __launch_bounds__(256)
    split_planes_t_kernel(const float* __restrict__ p, int64_t sk, int64_t rows, int64_t k, int64_t rows_pad,
                          int64_t k_pad, __nv_bfloat16* hi, __nv_bfloat16* lo) {
  __shared__ float tile[64][65];
  const int64_t r0 = (int64_t)blockIdx.x * 64, k0 = (int64_t)blockIdx.y * 64;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;   // 64 x 4
#pragma unroll 4
  for (int kk = ty; kk < 64; kk += 4) {
    const int64_t gr = r0 + tx, gk = k0 + kk;
    tile[kk][tx] = (gr < rows && gk < k) ? __ldg(p + gk * sk + gr) : 0.f;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 64 * 8; t += 256) {
    const int r = t >> 3, c = t & 7;
    const int64_t gr = r0 + r;
    if (gr >= rows_pad) continue;
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float v0 = tile[c * 8 + 2 * j][r], v1 = tile[c * 8 + 2 * j + 1][r];
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v0), h1 = __float2bfloat16_rn(v1);
      h[j] = pack_bf16(h0, h1);
      l[j] = pack_bf16(__float2bfloat16_rn(v0 - __bfloat162float(h0)), __float2bfloat16_rn(v1 - __bfloat162float(h1)));
    }
    *reinterpret_cast<uint4*>(hi + gr * k_pad + k0 + c * 8) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(lo + gr * k_pad + k0 + c * 8) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

// Multi-stage cp.async ring: the copies of k-block kb + STAGES - 1 are in flight while k-block kb is multiplied.
// CTAs per SM follow from the stage footprint: a single-stage 128x128 tile (65 KB) fits twice, so short-K GEMMs
// (dgrad of the first layer: K = 256 = 4 k-blocks) overlap one CTA's epilogue with its neighbour's main loop.
template <int BN, int STAGES>
__global__ void __launch_bounds__(kTcThreads, (STAGES * (2 * kTM * 128 + 2 * BN * 128) + 1024 <= 113 * 1024) ? 2 : 1)
    gemm_planes_kernel(const PlaneArgs g) {
  constexpr int A_PLANE = kTM * 128;
  constexpr int B_PLANE = BN * 128;
  constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* tiles = align1024(smem_raw);

  const int tid = threadIdx.x, wg = tid >> 7;
  const int64_t m0 = (int64_t)blockIdx.y * kTM, n0 = (int64_t)blockIdx.x * BN;
  const int64_t kbeg = (int64_t)blockIdx.z * g.k_per_split;
  const int64_t kend = kbeg + g.k_per_split < g.k_pad ? kbeg + g.k_per_split : g.k_pad;
  const int nkb = kend > kbeg ? (int)((kend - kbeg) / kTK) : 0;

  auto load = [&](int kb) {
    const uint32_t st = smem_u32(tiles + (size_t)(kb % STAGES) * STAGE);
    const int64_t k0 = kbeg + (int64_t)kb * kTK;
#pragma unroll
    for (int t = tid; t < kTM * 8; t += kTcThreads) {
      uint32_t off;
      int64_t src;
      if (g.a_mn) {   // chunk c of k-row kk: 8 consecutive m inside atom c/8
        const int kk = t / (kTM / 8), c = t % (kTM / 8);
        off = (c >> 3) * 8192 + kk * 128 + (((c & 7) ^ (kk & 7)) << 4);
        src = (k0 + kk) * g.a_pitch + m0 + c * 8;
      } else {
        const int r = t >> 3, c = t & 7;
        off = r * 128 + ((c ^ (r & 7)) << 4);
        src = (m0 + r) * g.a_pitch + k0 + c * 8;
      }
      cp_async16(st + off, g.a_hi + src);
      cp_async16(st + A_PLANE + off, g.a_lo + src);
    }
#pragma unroll
    for (int t = tid; t < BN * 8; t += kTcThreads) {
      uint32_t off;
      int64_t src;
      if (g.b_mn) {
        const int kk = t / (BN / 8), c = t % (BN / 8);
        off = (c >> 3) * 8192 + kk * 128 + (((c & 7) ^ (kk & 7)) << 4);
        src = (k0 + kk) * g.b_pitch + n0 + c * 8;
      } else {
        const int r = t >> 3, c = t & 7;
        off = r * 128 + ((c ^ (r & 7)) << 4);
        src = (n0 + r) * g.b_pitch + k0 + c * 8;
      }
      cp_async16(st + 2 * A_PLANE + off, g.b_hi + src);
      cp_async16(st + 2 * A_PLANE + B_PLANE + off, g.b_lo + src);
    }
  };

  float d[BN / 2];
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) d[j] = 0.f;
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkb) load(s);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  with_majorness(g.a_mn, g.b_mn, [&](auto ta, auto tb) {
    for (int kb = 0; kb < nkb; ++kb) {
      // the slot of k-block kb + STAGES - 1 was last read by k-block kb - 1, retired below
      if (kb + STAGES - 1 < nkb) load(kb + STAGES - 1);
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 1) : "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      wg_kblock<BN, decltype(ta)::value, decltype(tb)::value>(d, smem_u32(tiles + (size_t)(kb % STAGES) * STAGE), wg);
      wgmma_wait<0>();
      __syncthreads();
    }
  });
  asm volatile("cp.async.wait_all;" ::: "memory");
  fence_acc(d);
  store_acc<BN>(g, d, m0 + wg * 64, n0, blockIdx.z);
}

template <int BN, int STAGES>
static cudaError_t launch_planes(const PlaneArgs& pa, cudaStream_t st) {
  constexpr size_t smem = (size_t)STAGES * (2 * kTM * 128 + 2 * BN * 128) + 1024;
  dim3 grid((unsigned)ceil_div(pa.n, BN), (unsigned)ceil_div(pa.m, kTM), (unsigned)pa.splits);
  auto kern = gemm_planes_kernel<BN, STAGES>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, kTcThreads, smem, st>>>(pa);
  return cudaGetLastError();
}


// ================================================================================================
// Variant 4: persistent, warp-specialised planes GEMM - the kernel every production GEMM runs.
//   warps 0-7  : two consumer warpgroups.  Plain GEMMs (GEN = 0, no FOLD) run them PING-PONG: warpgroup j % 2 owns
//                the whole j-th tile of the CTA (both 64-row halves, two accumulators) and the two alternate, so one
//                warpgroup's epilogue runs while the other issues its MMAs.  Per k-block a warpgroup waits for the
//                full stage, issues its 24 wgmma as two groups of 12 (K-steps 0-1, then 2-3, each alternating
//                between the two halves' accumulators), keeps one group in flight and hands a stage back to the
//                producers once both groups have retired.  Named barriers order the MMA phases: a warpgroup starts
//                a tile only after the other one has issued the previous tile's last k-block.  The generated-operand and FOLD kernels stay COOPERATIVE: each warpgroup owns 64 rows of
//                every tile and both run the epilogue together (their producers / fold leave no registers for a
//                second accumulator).  The plain kernels run cooperatively too when a split-K launch has at most
//                one unit per CTA (WsArgs::coop): ping-pong would leave warpgroup 1 idle.
//   producers  : GEN = 0: one elected thread arms the stage barrier and issues cp.async.bulk.tensor.2d (TMA) loads
//                of the four plane slices; its warpgroup gives up its registers to the ping-pong consumers.
//                GEN = 1 / 2: eight warps GENERATE the A tile in shared memory (CIN outer product / DIN attention
//                input) while B arrives by TMA.
// The producers run up to STAGES k-blocks ahead, across tile boundaries: the next tile's operands load while the
// consumers run the epilogue of the current one.
// Persistent: grid = min(#tiles, #SMs); tile = CTA id + j * #CTAs, N-tile fastest (neighbouring CTAs share the
// A rows through L2).  BN <= 128: an m64n128 accumulator is 64 registers per consumer thread; ping-pong consumers
// hold two, so those kernels move registers from the producer warpgroup to them with setmaxnreg.
// ================================================================================================
constexpr int kWsConsumerWarps = 8;
constexpr int kWsProducers = 4;   // warps: one issues the TMA loads, but setmaxnreg works per warpgroup

struct WsArgs {
  PlaneArgs p;
  int tiles_m, tiles_n;
  int64_t ntiles;
  int c_tma;          // the epilogue stores through shared memory with TMA (store_acc_tma) instead of store_acc:
                      // 1 = C (2-D map), 2 = split-K slices into the workspace (3-D map)
  int coop;           // plain kernels: the consumers run cooperatively instead of ping-pong
};
// bytes of one consumer warpgroup's epilogue staging buffer: 64 rows x one 64-column half of the tile, fp32
template <int BN>
__host__ __device__ constexpr int ws_staging_bytes() { return 64 * (BN < 64 ? BN : 64) * 4; }
// ---- TMA (cp.async.bulk.tensor) producer primitives --------------------------------------------------
// One elected thread arms the stage's mbarrier with the bytes that will land (expect_tx) and issues the
// tiled bulk copies; the hardware writes the 128-byte-swizzled rows itself (CU_TENSOR_MAP_SWIZZLE_128B is
// exactly the `chunk ^ (row & 7)` layout the wgmma descriptors above expect) and completes the barrier.
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int32_t c0, int32_t c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(src),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(src),
               "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void warpgroup_sync(int wg) {   // named barrier 1 + wg: the 128 threads of one warpgroup
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
}
// Ping-pong order of the two consumer warpgroups' MMA phases: named barrier 3 + wg is passed when warpgroup wg waits
// on it (128 threads) and the other warpgroup has arrived (128 threads).
__device__ __forceinline__ void mma_order_wait(int wg) { asm volatile("bar.sync %0, 256;" ::"r"(3 + wg) : "memory"); }
__device__ __forceinline__ void mma_order_arrive(int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(3 + wg) : "memory"); }
// Per-warpgroup register budgets (multiples of 8; all warps of the warpgroup execute them)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Epilogue through shared memory and TMA stores, for C = act(alpha acc + bias) (the same arithmetic as store_acc).
// The warpgroup's 64 x BN tile leaves in 64-column halves: the 128 threads write a half into the warpgroup's staging
// buffer as two 32-column x 64-row fp32 boxes in the 128-byte-swizzled layout (16-byte chunk index XOR row % 8: the
// four rows a half-warp writes hit two bank sets instead of one), then one thread stores the boxes with
// cp.async.bulk.tensor and the warpgroup returns to the MMAs.  The buffer is rewritten only after the previous
// store has read it.  TMA clips the boxes at m, but along a row only in 16-byte units, so the map covers the first
// n4 = n & ~3 columns and the last n - n4 columns of a row are stored from registers: padding columns of C past n
// stay untouched.
// The activation is a template parameter (ACT < 0: g.act at run time) and the checks that are uniform over the
// tile are taken outside the element loop, so the loop is straight-line code: with one warp per SM sub-partition
// the epilogue is bound by instruction latency, not by shared-memory or store bandwidth.
// Split-K slices (z >= 0) leave the same way: alpha acc only, stored into slice z of the workspace through a 3-D map
// {n, m, splits} that clips rows >= m inside the slice.  That map needs n % 4 == 0, so a slice has no tail columns.
template <int BN, int ACT>
__device__ __forceinline__ void store_acc_tma_act(const PlaneArgs& g, const float (&d)[BN / 2], const CUtensorMap* map,
                                                  uint32_t stg, int wg, int64_t row0, int64_t n0, int32_t z) {
  constexpr int HALF = BN < 64 ? BN : 64;
  const int t = threadIdx.x & 127, lane = t & 31, w = t >> 5;
  const int64_t n4 = g.n & ~(int64_t)3;
  const bool tail = n0 + BN > n4;       // the tile holds columns past the map (stored from registers)
  const float* bias = z < 0 ? g.bias : nullptr;
  const float alpha = g.alpha;
#pragma unroll
  for (int hf = 0; hf < BN / HALF; ++hf) {
    if (t == 0) bulk_wait_read();
    warpgroup_sync(wg);
#pragma unroll
    for (int i = hf * HALF / 8; i < (hf + 1) * HALF / 8; ++i) {
      const int col = 8 * i + 2 * (lane & 3) - hf * HALF;
      const int64_t gn = n0 + 8 * i + 2 * (lane & 3);
      const bool in0 = gn < g.n, in1 = gn + 1 < g.n;
      float b0 = 0.f, b1 = 0.f;
      if (bias) {
        if (in0) b0 = __ldg(bias + gn);
        if (in1) b1 = __ldg(bias + gn + 1);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = w * 16 + (lane >> 2) + 8 * h;
        float v0 = __fmul_rn(alpha, d[4 * i + 2 * h]), v1 = __fmul_rn(alpha, d[4 * i + 2 * h + 1]);
        if (bias) {
          if (in0) v0 = __fadd_rn(v0, b0);
          if (in1) v1 = __fadd_rn(v1, b1);
        }
        v0 = act_apply(v0, ACT < 0 ? g.act : ACT);
        v1 = act_apply(v1, ACT < 0 ? g.act : ACT);
        const uint32_t off = (col >> 5) * 8192 + r * 128 + ((((col & 31) >> 2) ^ (r & 7)) << 4) + (col & 3) * 4;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg + off), "f"(v0), "f"(v1) : "memory");
        if (tail && gn >= n4 && in0 && row0 + r < g.m) {     // (gn and n4 are even: the pair is all tail or none)
          float* cp = g.c + (row0 + r) * g.ldc + gn;
          cp[0] = v0;
          if (in1) cp[1] = v1;
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    warpgroup_sync(wg);
    if (t == 0 && row0 < g.m) {
#pragma unroll
      for (int b = 0; b < HALF / 32; ++b) {
        const int64_t c0 = n0 + hf * HALF + 32 * b;
        if (c0 >= n4) continue;
        if (z < 0) tma_store_2d(map, stg + b * 8192, (int32_t)c0, (int32_t)row0);
        else tma_store_3d(map, stg + b * 8192, (int32_t)c0, (int32_t)row0, z);
      }
      bulk_commit();
    }
  }
}
// z < 0: C = act(alpha acc + bias) through the 2-D C map; z >= 0: split-K slice z through the 3-D workspace map
template <int BN>
__device__ __forceinline__ void store_acc_tma(const PlaneArgs& g, const float (&d)[BN / 2], const CUtensorMap* map,
                                              uint32_t stg, int wg, int64_t row0, int64_t n0, int32_t z) {
  if (z >= 0 || g.act == B2CTR_ACT_NONE) store_acc_tma_act<BN, B2CTR_ACT_NONE>(g, d, map, stg, wg, row0, n0, z);
  else if (g.act == B2CTR_ACT_RELU) store_acc_tma_act<BN, B2CTR_ACT_RELU>(g, d, map, stg, wg, row0, n0, z);
  else store_acc_tma_act<BN, -1>(g, d, map, stg, wg, row0, n0, z);
}

// fp32 pair -> bf16 hi pair + bf16 lo pair (v = hi + lo up to 2^-17): two cvt.rn.bf16x2.f32 + four ALU ops
__device__ __forceinline__ void split_pair(float v0, float v1, uint32_t& h, uint32_t& l) {
  const __nv_bfloat162 hh = __floats2bfloat162_rn(v0, v1);        // .x = v0 in the low half
  h = *reinterpret_cast<const uint32_t*>(&hh);
  const float h0 = __uint_as_float(h << 16), h1 = __uint_as_float(h & 0xffff0000u);
  const __nv_bfloat162 ll = __floats2bfloat162_rn(v0 - h0, v1 - h1);
  l = *reinterpret_cast<const uint32_t*>(&ll);
}
__device__ __forceinline__ void store_chunk(const float (&v)[8], unsigned char* hi_row, unsigned char* lo_row, int off) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) split_pair(v[2 * e], v[2 * e + 1], h[e], l[e]);
  *reinterpret_cast<uint4*>(hi_row + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo_row + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

// Generated A operand, CIN: one producer thread = half a row r of the outer product per stage: 32 consecutive
// q = i*hp + j starting at q0 (a multiple of 32; hp is 32 or a multiple of 64, so the 32 columns share one i), split
// into bf16 hi/lo and stored as four 16-byte chunks [c0, c0+4) of the 128-byte-swizzled row `rr`.
// Two steps, so that the producer loop can issue the global loads of k-block kb + 1 before it multiplies / splits /
// stores k-block kb.
struct GenRegs {
  float4 x[8];         // 32 values of X_k
  float a;             // T0[r, i]
};
__device__ __forceinline__ void cin_load_half(const PlaneArgs& g, int64_t r, int q0, GenRegs& o) {
  const bool row_ok = r < g.cin_rows;
  const float* xk = g.cin_xk + r * g.cin_ldk;
  const int hp = g.cin_hp, h = g.cin_h;
  const int i = q0 / hp, j = q0 - i * hp;          // hp is 32 or a multiple of 64: the 32 columns share one i
  o.a = (row_ok && i < g.cin_m) ? __ldg(g.cin_t0 + r * g.cin_ld0 + i) : 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int jj = j + 8 * c;
    o.x[2 * c] = (row_ok && jj < h) ? __ldg(reinterpret_cast<const float4*>(xk + jj)) : make_float4(0.f, 0.f, 0.f, 0.f);
    o.x[2 * c + 1] = (row_ok && jj + 4 < h) ? __ldg(reinterpret_cast<const float4*>(xk + jj) + 1)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
// multiply / split / store the half row held in `io` (k-block kb) and refill each register pair with the operands
// of k-block kb + 1 as soon as it has been consumed: a rolling prefetch that costs no extra registers.
__device__ __forceinline__ void cin_emit_half(const PlaneArgs& g, GenRegs& io, int q0, unsigned char* hi_row,
                                              unsigned char* lo_row, int rr, int c0, bool has_next, int64_t r_next,
                                              int q0_next, bool reload_x) {
  const int hp = g.cin_hp, h = g.cin_h;
  const int j = q0 - (q0 / hp) * hp;
  const float a = io.a;
  const bool row_ok = has_next && r_next < g.cin_rows;
  const float* xk = g.cin_xk + r_next * g.cin_ldk;
  const int in_ = q0_next / hp, jn = q0_next - in_ * hp;
  if (has_next) io.a = (row_ok && in_ < g.cin_m) ? __ldg(g.cin_t0 + r_next * g.cin_ld0 + in_) : 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float v[8] = {a * io.x[2 * c].x, a * io.x[2 * c].y, a * io.x[2 * c].z, a * io.x[2 * c].w,
                  a * io.x[2 * c + 1].x, a * io.x[2 * c + 1].y, a * io.x[2 * c + 1].z, a * io.x[2 * c + 1].w};
    if (reload_x) {       // (the next k-block may need the same 32 values of X_k: they then stay where they are)
      const int jj = jn + 8 * c;
      io.x[2 * c] = (row_ok && jj < h) ? __ldg(reinterpret_cast<const float4*>(xk + jj)) : make_float4(0.f, 0.f, 0.f, 0.f);
      io.x[2 * c + 1] = (row_ok && jj + 4 < h) ? __ldg(reinterpret_cast<const float4*>(xk + jj) + 1)
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (h & 7) {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (j + 8 * c + e >= h) v[e] = 0.f;
    }
    store_chunk(v, hi_row, lo_row, ((c0 + c) ^ (rr & 7)) << 4);
  }
}

// DIN local-activation-unit input (deepctr/layers/core.py:96-101), generated the same way: row r = (b, t),
//   A[r, :] = [ q_b , k_bt , q_b - k_bt , q_b * k_bt ]   (4 segments of E columns; E % 8 == 0)
// cin_t0 = queries [B, ld0], cin_xk = keys (sample stride cin_ldk, row stride E), cin_m = T, cin_h = E.
// (generic E: not inlined - one copy instead of eight in the producer loop)
__device__ __noinline__ void att_generate_half(const PlaneArgs& g, int64_t r, int col0, unsigned char* hi_row,
                                                  unsigned char* lo_row, int rr, int c0) {
  const int T = g.cin_m, E = g.cin_h;
  const bool row_ok = r < g.cin_rows;
  const uint32_t bu = row_ok ? (uint32_t)r / (uint32_t)T : 0u;      // rows < 2^31 (checked on the host)
  const int64_t b = bu;
  const int t = row_ok ? (int)((uint32_t)r - bu * (uint32_t)T) : 0;
  const float* q = g.cin_t0 + b * g.cin_ld0;
  const float* k = g.cin_xk + b * g.cin_ldk + (int64_t)t * E;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int col = col0 + 8 * c;
    const int seg = col / E, e = col - seg * E;
    float v[8];
    if (row_ok && seg < 4) {
      float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;
      if (seg != 1) { a0 = __ldg(reinterpret_cast<const float4*>(q + e)); a1 = __ldg(reinterpret_cast<const float4*>(q + e) + 1); }
      if (seg != 0) { b0 = __ldg(reinterpret_cast<const float4*>(k + e)); b1 = __ldg(reinterpret_cast<const float4*>(k + e) + 1); }
      const float qa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float ka[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int jx = 0; jx < 8; ++jx)
        v[jx] = seg == 0 ? qa[jx] : seg == 1 ? ka[jx] : seg == 2 ? __fsub_rn(qa[jx], ka[jx]) : __fmul_rn(qa[jx], ka[jx]);
    } else {
#pragma unroll
      for (int jx = 0; jx < 8; ++jx) v[jx] = 0.f;
    }
    store_chunk(v, hi_row, lo_row, ((c0 + c) ^ (rr & 7)) << 4);
  }
}

// generated-operand kernels run 8 producer warps (two threads per generated row), the others 4
template <bool GENERATED>
struct WsLayout {
  static constexpr int kProducers = GENERATED ? 8 : kWsProducers;
  static constexpr int kThreads = (kWsConsumerWarps + kProducers) * 32;
};

// GEN: 0 = both operands from memory; 1 = A generated as the CIN outer product; 2 = A generated as the DIN
// attention input (one instantiation per generator: the code of the other one would only fill the instruction cache)
template <int BN, int STAGES, int GEN = 0, bool FOLD = false>
__global__ void __launch_bounds__(WsLayout<GEN != 0>::kThreads, 1)
    gemm_planes_ws_kernel(const __grid_constant__ WsArgs w, const __grid_constant__ CUtensorMap tm_ah,
                          const __grid_constant__ CUtensorMap tm_al, const __grid_constant__ CUtensorMap tm_bh,
                          const __grid_constant__ CUtensorMap tm_bl, const __grid_constant__ CUtensorMap tm_c) {
  static_assert(BN <= 128, "the consumer accumulator is BN / 2 registers per thread");
  constexpr bool PINGPONG = GEN == 0 && !FOLD;
  const PlaneArgs& g = w.p;
  constexpr int A_PLANE = kTM * 128;
  constexpr int B_PLANE = BN * 128;
  constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* tiles = align1024(smem_raw);
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t cta0 = blockIdx.x, nctas = gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      // TMA: one arrive.expect_tx; generated A: one arrival per generating thread of the stage + the TMA expect_tx
      // of the B planes
      mbar_init(&full_bar[s], GEN == 1 ? 1 + 256 : GEN == 2 ? 1 + 128 : 1);
      // a stage is released by every consumer warp (cooperative) or by the four warps of the tile's owner (ping-pong)
      mbar_init(&empty_bar[s], PINGPONG && !w.coop ? kWsConsumerWarps / 2 : kWsConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // tile -> coordinates (N tile fastest, then M, then the split-K slice)
  auto decode = [&](int64_t tile, int64_t& mt, int64_t& nt, int64_t& kbeg, int& nkb) {
    if constexpr (FOLD) {
      // a CTA owns whole ROW BLOCKS and walks all their N tiles in turn (its epilogue accumulates across
      // them): work item j of CTA c is (row block c + (j / tiles_n) * nctas, N tile j % tiles_n)
      const int64_t j = tile / nctas;
      nt = j % w.tiles_n;
      mt = tile % nctas + (j / w.tiles_n) * nctas;
      kbeg = 0;
      nkb = mt < w.tiles_m ? (int)(g.k_pad / kTK) : 0;
      return;
    }
    nt = tile % w.tiles_n;
    const int64_t rest = tile / w.tiles_n;
    mt = rest % w.tiles_m;
    const int64_t z = rest / w.tiles_m;
    kbeg = z * g.k_per_split;
    const int64_t kend = kbeg + g.k_per_split < g.k_pad ? kbeg + g.k_per_split : g.k_pad;
    nkb = kend > kbeg ? (int)((kend - kbeg) / kTK) : 0;
  };

  if (GEN != 0 && warp >= kWsConsumerWarps) {
    // ------------------------------------------------------------------------------ generating producers
    // 8 warps in TWO GROUPS of 128 threads; group g owns the stages with (stage counter & 1) == g and generates a
    // whole row (64 columns) per thread for them.  Two stages are therefore in production at any time: while one
    // group waits for its global loads (the producer is load-latency-bound: ncu source page, FMUL on the loaded
    // operands holds the stall samples), the other one multiplies / splits / stores.  B (filter / dY planes)
    // arrives by TMA, issued by thread 0 of the group that owns the stage.
    const int tid = threadIdx.x - kWsConsumerWarps * 32;
    const int grp = tid >> 7, t128 = tid & 127;
    if (t128 == 0) { tma_prefetch_desc(&tm_bh); tma_prefetch_desc(&tm_bl); }
    uint32_t it = 0;
    if constexpr (GEN == 1) {
      // CIN: 256 threads per stage (two per generated row), software-pipelined over the FLATTENED sequence of
      // k-blocks of all the tiles of this CTA: the operands of the next k-block (the next tile's first one included)
      // are requested while the current one is multiplied / split / stored, and stay in flight across the stage
      // hand-over.  The generator was load-latency-bound (ncu source page: the stall samples sit on the first use
      // of the loaded operands).
      const int half = tid & 1;
      const int atom = tid >> 7, rr = g.a_mn ? (tid & 127) >> 1 : tid >> 1;
      const int soff = (g.a_mn ? atom * 8192 : 0) + rr * 128;
      // (32-bit coordinates: rows, columns and tile counts of the generated-operand GEMMs fit 31 bits, checked on
      // the host; the state of two k-blocks stays in registers next to the prefetched operands)
      const int ntiles = (int)w.ntiles, stride = (int)nctas;
      auto dec = [&](int tile, int& m0, int& n0, int& kbeg, int& nkb) {
        int64_t mt, nt, kb64;
        decode(tile, mt, nt, kb64, nkb);
        m0 = (int)(mt * kTM);
        n0 = (int)(nt * BN);
        kbeg = (int)kb64;
      };
      int tile = (int)cta0, m0 = 0, n0 = 0, kbeg = 0, nkb = 0, kb = 0;
      for (; tile < ntiles; tile += stride) {            // first tile with work
        dec(tile, m0, n0, kbeg, nkb);
        if (nkb > 0) break;
      }
      // this thread's row and first column in the k-block at (m0, k0)
      auto row_of = [&](int m0_, int k0_) { return g.a_mn ? k0_ + rr : m0_ + rr; };
      auto col_of = [&](int m0_, int k0_) { return g.a_mn ? m0_ + atom * 64 + half * 32 : k0_ + half * 32; };
      GenRegs gr;
      if (tile < ntiles) cin_load_half(g, row_of(m0, kbeg), col_of(m0, kbeg), gr);     // (k_of(kbeg, 0, .) == kbeg)
      // CIN forward, hp = nj * 64: the k-blocks of a tile are walked j-block-major (all i for the first 64 columns of
      // X_k, then all i for the next 64 ...).  A thread's 32 values of X_k are then the same for m consecutive
      // k-blocks and stay in registers; only T0[r, i] is fetched per k-block.  (The B planes are fetched at the same
      // k0, and the order of the K accumulation is free.)
      const int nj = (!g.a_mn && g.splits == 1 && g.cin_hp >= 128) ? g.cin_hp / kTK : 1;
      auto k_of = [&](int kbeg_, int kb_, int nkb_) {
        if (nj == 1) return kbeg_ + kb_ * kTK;
        const int ni = nkb_ / nj;                      // = m (k_pad = m * hp)
        const int jb = kb_ / ni, i = kb_ - jb * ni;
        return (i * nj + jb) * kTK;
      };
      while (tile < ntiles) {
        const int k0 = k_of(kbeg, kb, nkb);
        // the k-block after this one
        int tile_n = tile, m0_n = m0, n0_n = n0, kbeg_n = kbeg, nkb_n = nkb, kb_n = kb + 1;
        if (kb_n >= nkb) {
          kb_n = 0;
          for (tile_n = tile + stride; tile_n < ntiles; tile_n += stride) {
            dec(tile_n, m0_n, n0_n, kbeg_n, nkb_n);
            if (nkb_n > 0) break;
          }
        }
        const bool has_next = tile_n < ntiles;
        const int k0_n = k_of(kbeg_n, kb_n, nkb_n);
        const int s = it % STAGES;
        mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
        unsigned char* stp = tiles + (size_t)s * STAGE;
        if (tid == 0) {
          uint64_t* bar = &full_bar[s];
          mbar_expect_tx(bar, (uint32_t)(2 * B_PLANE));
          const uint32_t st = smem_u32(stp);
          if (g.b_mn) {
#pragma unroll
            for (int j = 0; j < (BN >= 64 ? BN / 64 : 1); ++j) {
              tma_load_2d(st + 2 * A_PLANE + j * 8192, &tm_bh, n0 + 64 * j, k0, bar);
              tma_load_2d(st + 2 * A_PLANE + B_PLANE + j * 8192, &tm_bl, n0 + 64 * j, k0, bar);
            }
          } else {
            tma_load_2d(st + 2 * A_PLANE, &tm_bh, k0, n0, bar);
            tma_load_2d(st + 2 * A_PLANE + B_PLANE, &tm_bl, k0, n0, bar);
          }
        }
        const int r = row_of(m0, k0), r_n = row_of(m0_n, k0_n), q = col_of(m0, k0), q_n = col_of(m0_n, k0_n);
        cin_emit_half(g, gr, q, stp + soff, stp + A_PLANE + soff, rr, half * 4, has_next, r_n, q_n,
                      has_next && (r_n != r || q_n % g.cin_hp != q % g.cin_hp));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(&full_bar[s]);
        ++it;
        tile = tile_n; m0 = m0_n; n0 = n0_n; kbeg = kbeg_n; nkb = nkb_n; kb = kb_n;
      }
    } else
    for (int64_t tile = cta0; tile < w.ntiles; tile += nctas) {
      int64_t mt, nt, kbeg;
      int nkb;
      decode(tile, mt, nt, kbeg, nkb);
      const int64_t m0 = mt * kTM;
      const int32_t n0 = (int32_t)(nt * BN);
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        if ((int)(it & 1) != grp) continue;
        const int s = it % STAGES;
        mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
        unsigned char* stp = tiles + (size_t)s * STAGE;
        const int64_t k0 = kbeg + (int64_t)kb * kTK;
        if (t128 == 0) {
          uint64_t* bar = &full_bar[s];
          mbar_expect_tx(bar, (uint32_t)(2 * B_PLANE));
          const uint32_t st = smem_u32(stp);
          if (g.b_mn) {
#pragma unroll
            for (int j = 0; j < (BN >= 64 ? BN / 64 : 1); ++j) {
              tma_load_2d(st + 2 * A_PLANE + j * 8192, &tm_bh, n0 + 64 * j, (int32_t)k0, bar);
              tma_load_2d(st + 2 * A_PLANE + B_PLANE + j * 8192, &tm_bl, n0 + 64 * j, (int32_t)k0, bar);
            }
          } else {
            tma_load_2d(st + 2 * A_PLANE, &tm_bh, (int32_t)k0, n0, bar);
            tma_load_2d(st + 2 * A_PLANE + B_PLANE, &tm_bl, (int32_t)k0, n0, bar);
          }
        }
        if (g.a_mn) {      // A^T: M = q (two 64-wide atoms), K = r: thread -> (atom, k-row)
          const int atom = t128 >> 6, rr = t128 & 63;
          unsigned char* row = stp + atom * 8192 + rr * 128;
          att_generate_half(g, k0 + rr, (int)(m0 + atom * 64), row, row + A_PLANE, rr, 0);
          att_generate_half(g, k0 + rr, (int)(m0 + atom * 64 + 32), row, row + A_PLANE, rr, 4);
        } else {           // A: M = r, K = q: thread -> row
          unsigned char* row = stp + t128 * 128;
          att_generate_half(g, m0 + t128, (int)k0, row, row + A_PLANE, t128, 0);
          att_generate_half(g, m0 + t128, (int)(k0 + 32), row, row + A_PLANE, t128, 4);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(&full_bar[s]);
      }
    }
  } else if (warp >= kWsConsumerWarps) {
    // ------------------------------------------------------------------------------ TMA producer
    // one elected lane: wait for a free stage, arm its barrier with the stage bytes, issue the bulk tensor copies
    // of the four operand planes.  Data moves global -> swizzled shared memory inside the async proxy, where
    // wgmma reads it.
    if constexpr (PINGPONG) setmaxnreg_dec<56>();
    if (warp == kWsConsumerWarps && lane == 0) {
      tma_prefetch_desc(&tm_ah); tma_prefetch_desc(&tm_al); tma_prefetch_desc(&tm_bh); tma_prefetch_desc(&tm_bl);
      uint32_t it = 0;
      for (int64_t tile = cta0; tile < w.ntiles; tile += nctas) {
        int64_t mt, nt, kbeg;
        int nkb;
        decode(tile, mt, nt, kbeg, nkb);
        const int32_t m0 = (int32_t)(mt * kTM);
        const int32_t n0 = (int32_t)(nt * BN);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
          uint64_t* bar = &full_bar[s];
          mbar_expect_tx(bar, (uint32_t)STAGE);
          const uint32_t st = smem_u32(tiles + (size_t)s * STAGE);
          const int32_t k0 = (int32_t)(kbeg + (int64_t)kb * kTK);
          if (g.a_mn) {        // [k, m] planes: one 64(m) x 64(k) box per 64-wide atom
#pragma unroll
            for (int j = 0; j < kTM / 64; ++j) {
              tma_load_2d(st + j * 8192, &tm_ah, m0 + 64 * j, k0, bar);
              tma_load_2d(st + A_PLANE + j * 8192, &tm_al, m0 + 64 * j, k0, bar);
            }
          } else {             // [m, k] planes: one 64(k) x 128(m) box
            tma_load_2d(st, &tm_ah, k0, m0, bar);
            tma_load_2d(st + A_PLANE, &tm_al, k0, m0, bar);
          }
          if (g.b_mn) {        // (an MN-major B tile is at least one 64-wide atom: BN >= 64)
#pragma unroll
            for (int j = 0; j < (BN >= 64 ? BN / 64 : 1); ++j) {
              tma_load_2d(st + 2 * A_PLANE + j * 8192, &tm_bh, n0 + 64 * j, k0, bar);
              tma_load_2d(st + 2 * A_PLANE + B_PLANE + j * 8192, &tm_bl, n0 + 64 * j, k0, bar);
            }
          } else {
            tma_load_2d(st + 2 * A_PLANE, &tm_bh, k0, n0, bar);
            tma_load_2d(st + 2 * A_PLANE + B_PLANE, &tm_bl, k0, n0, bar);
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------------------ consumers
    const int wg = warp >> 2;
    // Ping-pong: warpgroup wg owns the tiles j (of this CTA) with j % 2 == wg and issues each k-block as two groups
    // of 12 wgmma over both 64-row halves (tile_kblock_half): every output element sees the same MMAs in the same
    // order as in the cooperative loop.  Both warpgroups count every k-block of the CTA (`it`), so the
    // stage ring is walked in the producers' order.  The order barrier also keeps a warpgroup from waiting on a
    // full barrier whose previous phase the other warpgroup has not consumed yet (parity waits see only one phase).
    auto pingpong = [&](auto ta, auto tb) {
      constexpr int TA = decltype(ta)::value, TB = decltype(tb)::value;
      const uint32_t stg = smem_u32(tiles + STAGES * STAGE + wg * ws_staging_bytes<BN>());
      uint32_t it = 0;
      float d0[BN / 2], d1[BN / 2];
      int64_t j = 0;
      for (int64_t tile = cta0; tile < w.ntiles; tile += nctas, ++j) {
        int64_t mt, nt, kbeg;
        int nkb;
        decode(tile, mt, nt, kbeg, nkb);
        if ((j & 1) != wg) {
          it += nkb;
          continue;
        }
        if (j > 0) mma_order_wait(wg);          // the other warpgroup has issued the last k-block of tile j - 1
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) d0[i] = d1[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&full_bar[s], (it / STAGES) & 1);
          const uint32_t st = smem_u32(tiles + (size_t)s * STAGE);
          tile_kblock_half<BN, TA, TB, 0>(d0, d1, st);
          wgmma_wait<1>();                      // the previous k-block has retired: release its stage
          if (prev >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
          }
          tile_kblock_half<BN, TA, TB, 2>(d0, d1, st);
          wgmma_wait<1>();
          prev = s;
        }
        if (tile + nctas < w.ntiles) mma_order_arrive(wg ^ 1);
        wgmma_wait<0>();
        fence_acc(d0);
        fence_acc(d1);
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        const int64_t row0 = mt * kTM;
        // (z is a constant -1 for plain outputs: a run-time z in their epilogue cost the forward and dgrad launches
        // several microseconds each)
        if (w.c_tma == 2) {
          const int32_t z = (int32_t)(tile / ((int64_t)w.tiles_n * w.tiles_m));
          store_acc_tma<BN>(g, d0, &tm_c, stg, wg, row0, nt * BN, z);
          store_acc_tma<BN>(g, d1, &tm_c, stg, wg, row0 + 64, nt * BN, z);
        } else if (w.c_tma) {
          store_acc_tma<BN>(g, d0, &tm_c, stg, wg, row0, nt * BN, -1);
          store_acc_tma<BN>(g, d1, &tm_c, stg, wg, row0 + 64, nt * BN, -1);
        } else {
          const int64_t z = tile / ((int64_t)w.tiles_n * w.tiles_m);
          store_acc<BN>(g, d0, row0, nt * BN, z);
          store_acc<BN>(g, d1, row0 + 64, nt * BN, z);
        }
      }
      if (w.c_tma && (threadIdx.x & 127) == 0) bulk_wait_all();   // the last stores have left the CTA
    };
    auto consume = [&](auto ta, auto tb) {
      uint32_t it = 0;
      float d[BN / 2];
      [[maybe_unused]] float dxk[FOLD ? BN / 2 : 1];      // FOLD: this thread's dXk partial sums, same layout as d
      for (int64_t tile = cta0; tile < w.ntiles; tile += nctas) {
        int64_t mt, nt, kbeg;
        int nkb;
        decode(tile, mt, nt, kbeg, nkb);
        if (FOLD && nkb == 0) continue;
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) d[j] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&full_bar[s], (it / STAGES) & 1);
          wg_kblock<BN, decltype(ta)::value, decltype(tb)::value>(d, smem_u32(tiles + (size_t)s * STAGE), wg);
          wgmma_wait<1>();                 // the group of the previous k-block has retired: release its stage
          if (prev >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
          }
          prev = s;
        }
        wgmma_wait<0>();
        fence_acc(d);
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        const int64_t row0 = mt * kTM + wg * 64;
        if constexpr (FOLD) {
          // CIN backward: the accumulator tile is dZ[r, q] (q = i*hp + j) = dY W'^T and is never stored - it is folded
          // onto the two factors of the outer product right here:
          //   dT0[r, i] += sum_j dZ[r, i*hp + j] * xk[r, j]      (quad shuffle + one red.add per row and hp columns)
          //   dXk[r, j] += sum_i dZ[r, i*hp + j] * t0[r, i]      (registers across the N tiles of the row block,
          //                                                       red.add once per row block)
          // BN % hp == 0, so a thread's columns keep their j from tile to tile.
          if (nt == 0) {
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) dxk[j] = 0.f;
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t gm = row0 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
            const bool row_ok = gm < g.m;
            const float* t0 = g.cin_t0 + (row_ok ? gm : 0) * g.cin_ld0;
            const float* xk = g.cin_xk + (row_ok ? gm : 0) * g.cin_ldk;
            float p = 0.f;
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
              const int c = 8 * i + 2 * (lane & 3);
              const int64_t q = nt * BN + c;
              const int ic = (int)(q / g.cin_hp), j = (int)(q - (int64_t)ic * g.cin_hp);
              const bool ok = row_ok && ic < g.cin_m;
              const float a = ok ? __ldg(t0 + ic) : 0.f;
              const float x0 = ok && j < g.cin_h ? __ldg(xk + j) : 0.f;
              const float x1 = ok && j + 1 < g.cin_h ? __ldg(xk + j + 1) : 0.f;
              const float d0 = d[4 * i + 2 * h], d1 = d[4 * i + 2 * h + 1];
              p += d0 * x0 + d1 * x1;
              dxk[4 * i + 2 * h] += d0 * a;
              dxk[4 * i + 2 * h + 1] += d1 * a;
              if ((8 * (i + 1)) % g.cin_hp == 0) {     // last 8 columns of the hp-wide group of output i (warp-uniform)
                p += __shfl_xor_sync(0xffffffffu, p, 1);
                p += __shfl_xor_sync(0xffffffffu, p, 2);
                if ((lane & 3) == 0 && ok) red_add_f1(g.fold_dt0 + gm * g.cin_ld0 + ic, p);
                p = 0.f;
              }
            }
            if (nt == w.tiles_n - 1 && row_ok) {
              float* dst = g.fold_dxk + gm * g.fold_ldx;
#pragma unroll
              for (int i = 0; i < BN / 8; ++i) {
                const int j = (8 * i + 2 * (lane & 3)) % g.cin_hp;
                if (j < g.cin_h) red_add_f1(dst + j, dxk[4 * i + 2 * h]);
                if (j + 1 < g.cin_h) red_add_f1(dst + j + 1, dxk[4 * i + 2 * h + 1]);
              }
            }
          }
        } else if (w.c_tma) {
          const uint32_t stg = smem_u32(tiles + STAGES * STAGE + wg * ws_staging_bytes<BN>());
          if (w.c_tma == 2)
            store_acc_tma<BN>(g, d, &tm_c, stg, wg, row0, nt * BN, (int32_t)(tile / ((int64_t)w.tiles_n * w.tiles_m)));
          else
            store_acc_tma<BN>(g, d, &tm_c, stg, wg, row0, nt * BN, -1);
        } else {
          const int64_t z = tile / ((int64_t)w.tiles_n * w.tiles_m);
          store_acc<BN>(g, d, row0, nt * BN, z);
        }
      }
      if (!FOLD && w.c_tma && (threadIdx.x & 127) == 0) bulk_wait_all();   // the last stores have left the CTA
    };
    // only the layouts a launch can ask for: the CIN fold reads both operands K-major, the generated-A kernels read
    // MN-major B planes, and an MN-major B tile is at least one 64-wide atom
    if constexpr (FOLD) consume(Major<0>{}, Major<0>{});
    else if constexpr (GEN != 0) {
      if (g.a_mn) consume(Major<1>{}, Major<1>{});
      else consume(Major<0>{}, Major<1>{});
    } else {
      setmaxnreg_inc<224>();       // two accumulators: 56 (producers) x 128 + 224 x 256 threads = 384 x 168 registers
      // w.coop (split-K launches with at most one unit per CTA): ping-pong would leave warpgroup 1 idle, so both
      // warpgroups take 64 rows of the unit, in variant 3's order
      auto run = [&](auto ta, auto tb) {
        if (w.coop) consume(ta, tb);
        else pingpong(ta, tb);
      };
      if constexpr (BN < 64) {
        if (g.a_mn) run(Major<1>{}, Major<0>{});
        else run(Major<0>{}, Major<0>{});
      } else {
        with_majorness(g.a_mn, g.b_mn, run);
      }
    }
  }
}

struct TmaMaps {
  CUtensorMap ah, al, bh, bl, c;
};

template <int BN, int STAGES, int GEN = 0, bool FOLD = false>
static cudaError_t launch_ws_impl(const WsArgs& wa, const TmaMaps& tm, cudaStream_t st) {
  constexpr size_t smem = (size_t)STAGES * (2 * kTM * 128 + 2 * BN * 128) + 2 * ws_staging_bytes<BN>() + 1024;
  static_assert(smem + 256 <= 227 * 1024, "stage ring + epilogue staging exceed shared memory");
  auto kern = gemm_planes_ws_kernel<BN, STAGES, GEN, FOLD>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int64_t nctas = wa.ntiles < kNumSMs ? wa.ntiles : kNumSMs;
  WsArgs wcopy = wa;
  if (FOLD) {      // CTAs own row blocks: ntiles = work-item slots of the round-robin over row blocks
    nctas = wa.tiles_m < kNumSMs ? wa.tiles_m : kNumSMs;
    wcopy.ntiles = ceil_div(wa.tiles_m, nctas) * wa.tiles_n * nctas;
  }
  kern<<<(unsigned)nctas, WsLayout<GEN != 0>::kThreads, smem, st>>>(wcopy, tm.ah, tm.al, tm.bh, tm.bl, tm.c);
  return cudaGetLastError();
}

// ---- tensor maps: cuTensorMapEncodeTiled resolved through the runtime's driver entry-point query ---------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tma_encoder() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
    else
      cudaGetLastError();
  }
  return fn;
}
// bf16 matrix [outer, inner] with `pitch` elements between rows; box = box_inner x box_outer, 128-byte swizzle,
// out-of-range box parts read as zero.
static bool tma_map_2d(CUtensorMap* m, const void* base, int64_t inner, int64_t outer, int64_t pitch,
                       int box_inner, int box_outer) {
  EncodeTiledFn enc = tma_encoder();
  if (!enc || ((uintptr_t)base & 15) || (pitch * 2) % 16 || box_inner * 2 > 128 || box_outer > 256) return false;
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// C tensor map for the TMA-store epilogue (store_acc_tma): fp32 [m, n & ~3] with ldc elements between rows, box
// 32 x 64 with 128-byte swizzle.  Only plain stores qualify: split-K slices go to the workspace, accumulate reads C,
// and TMA needs a 16-byte aligned base and row pitch.  Returns whether wa.c_tma may be set.
static bool tma_map_c(CUtensorMap* m, const PlaneArgs& p) {
  EncodeTiledFn enc = tma_encoder();
  if (!enc || p.splits > 1 || p.accumulate || !p.c || ((uintptr_t)p.c & 15) || p.ldc % 4 || p.ldc < p.n ||
      p.n < 4 || p.m >= (1ll << 31) || p.n >= (1ll << 31))
    return false;
  cuuint64_t dims[2] = {(cuuint64_t)(p.n & ~(int64_t)3), (cuuint64_t)p.m};
  cuuint64_t strides[1] = {(cuuint64_t)p.ldc * 4};
  cuuint32_t box[2] = {32, 64};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, p.c, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) ==
         CUDA_SUCCESS;
}
// Split-K workspace map for the same epilogue: fp32 [splits, m, n] (ws[z][m][n]), box 32 x 64 x 1.  The third
// dimension keeps TMA's row clipping at m inside each slice.  Rows must be whole 16-byte units (n % 4 == 0);
// otherwise the slices keep the register epilogue.  Returns whether wa.c_tma may be 2.
static bool tma_map_ws(CUtensorMap* m, const PlaneArgs& p) {
  EncodeTiledFn enc = tma_encoder();
  if (!enc || p.splits < 2 || !p.ws || ((uintptr_t)p.ws & 15) || p.n % 4 || p.m >= (1ll << 31) ||
      p.n >= (1ll << 31))
    return false;
  cuuint64_t dims[3] = {(cuuint64_t)p.n, (cuuint64_t)p.m, (cuuint64_t)p.splits};
  cuuint64_t strides[2] = {(cuuint64_t)p.n * 4, (cuuint64_t)(p.m * p.n) * 4};
  cuuint32_t box[3] = {32, 64, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, p.ws, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) ==
         CUDA_SUCCESS;
}

static inline int64_t round_up(int64_t v, int64_t q) { return (v + q - 1) / q * q; }
// Padded extent of caller planes: rows to 256 (largest N tile of a K-major B / M tile pair), columns to 128
// (M tile of an MN-major A, N tiles of an MN-major B); narrow matrices (<= 64 columns) pad to one 64-wide
// swizzle atom only - a 128-wide MN-major tile then runs into the next plane row, which only feeds output
// rows/columns >= m/n that are never stored.
static inline int planes_bn(int64_t n, int64_t k) {
  if (n <= 32) return 32;
  if (n <= 64) return 64;
  if (n <= 128 || k <= 4 * kTK) return 128;   // short K: prefer 128-wide tiles, 3 CTAs per SM
  return 256;
}

size_t gemm_bf16x3_workspace_bytes(const b2ctr_gemm_t* g) {
  size_t splitk = g->split_k > 1 ? (size_t)g->split_k * g->m * g->n * sizeof(float) : 0;
  const int64_t kp = round_up(g->k > 0 ? g->k : 1, kTK), mp = round_up(g->m, 2 * kTM), np = round_up(g->n, 256);
  return splitk + (size_t)(mp + np) * kp * 2 * sizeof(__nv_bfloat16) + 512;
}

// variant 0 / 4: the persistent kernel; variant 3: the non-persistent reference kernel
b2ctr_status_t gemm_bf16x3(const b2ctr_gemm_t* g, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  B2_REQUIRE(g->variant == 0 || g->variant == 3 || g->variant == 4, "gemm: variant must be 0, 3 or 4, got %d",
             g->variant);
  B2_REQUIRE(((uintptr_t)g->a_planes & 15) == 0 && ((uintptr_t)g->b_planes & 15) == 0,
             "gemm: a_planes / b_planes must be 16-byte aligned");
  const size_t need = gemm_bf16x3_workspace_bytes(g);
  if (!workspace || workspace_bytes < need) {
    set_error("gemm(bf16x3): needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int splits = g->split_k > 1 ? g->split_k : 1;
  const bool ws_kernel = g->variant != 3;
  int bn = ws_kernel ? (g->n <= 32 ? 32 : g->n <= 64 ? 64 : 128)
                     : planes_bn(g->n, g->k / (g->split_k > 1 ? g->split_k : 1));
  const int64_t kp = round_up(g->k > 0 ? g->k : 1, kTK), mp = round_up(g->m, 2 * kTM);
  unsigned char* w = (unsigned char*)workspace;
  float* ws = (float*)w;
  w += splits > 1 ? (size_t)splits * g->m * g->n * sizeof(float) : 0;
  w = (unsigned char*)(((uintptr_t)w + 255) & ~(uintptr_t)255);
  // Row-contiguous sources keep their layout (MN-major planes) and the wgmma descriptors do the transposition -
  // the same planes then serve every GEMM that reads the tensor (forward / dgrad / wgrad), which is what
  // caller-provided planes (g->a_planes / g->b_planes) exploit.  An MN-major B tile is at least one 64-wide atom:
  // under a 32-wide N tile a row-contiguous B goes through the transposing split into K-major planes instead.
  const bool a_kc = !g->trans_a, b_kc = g->trans_b != 0;
  const int64_t a_sr = g->trans_a ? g->k : g->m, a_sc = g->trans_a ? g->m : g->k;   // stored rows / cols
  const int64_t b_sr = g->trans_b ? g->n : g->k, b_sc = g->trans_b ? g->k : g->n;
  const bool a_given = g->a_planes != nullptr;
  const bool b_given = g->b_planes && (b_kc || bn >= 64);
  // an fp32 operand is read only when this call splits it (given planes are used whenever the tiling allows)
  B2_REQUIRE(a_given || g->a, "gemm: NULL A without its planes");
  B2_REQUIRE(b_given || g->b, "gemm: NULL B, and its planes are missing or unusable at N = %lld", (long long)g->n);
  if (b_given && !b_kc && planes_cols_pad(b_sc) % bn != 0) bn = planes_cols_pad(b_sc) == 64 ? 64 : 128;   // N tiles inside the pad
  const int64_t np = round_up(g->n, bn);
  const int a_mn = !a_kc;
  const int b_mn = !b_kc && bn >= 64;
  __nv_bfloat16 *a_hi, *a_lo, *b_hi, *b_lo;
  int64_t a_pitch, b_pitch;
  int64_t a_prows, b_prows;      // rows of the plane matrices as stored (TMA extents)
  auto split_k = [&](const float* p, int64_t ld, int64_t rows, int64_t cols, int64_t rows_pad, int64_t cols_pad,
                     __nv_bfloat16* hi, __nv_bfloat16* lo) {      // planes[r, c] = p[r*ld + c]
    const int vec = (ld % 4 == 0) && (((uintptr_t)p & 15) == 0);
    split_planes_kernel<<<grid_for(rows_pad * (cols_pad / 8), 256, 8), 256, 0, st>>>(p, ld, rows, cols, rows_pad,
                                                                                   cols_pad, hi, lo, vec);
  };
  auto split_t = [&](const float* p, int64_t ld, int64_t rows, int64_t rows_pad, __nv_bfloat16* hi,
                     __nv_bfloat16* lo) {                        // planes[r, k] = p[k*ld + r]
    dim3 grid((unsigned)ceil_div(rows_pad, 64), (unsigned)(kp / 64));
    split_planes_t_kernel<<<grid, 256, 0, st>>>(p, ld, rows, g->k, rows_pad, kp, hi, lo);
  };
  if (a_given) {
    const int64_t rp = round_up(a_sr, 256), cp = planes_cols_pad(a_sc);
    a_hi = (__nv_bfloat16*)g->a_planes; a_lo = a_hi + rp * cp; a_pitch = cp; a_prows = rp;
  } else {
    a_hi = (__nv_bfloat16*)w; a_lo = a_hi + mp * kp; w = (unsigned char*)(a_lo + mp * kp);
    a_pitch = a_mn ? mp : kp; a_prows = a_mn ? kp : mp;
    if (a_kc) split_k(g->a, g->lda, g->m, g->k, mp, kp, a_hi, a_lo);
    else split_k(g->a, g->lda, g->k, g->m, kp, mp, a_hi, a_lo);
    B2_CHECK_LAUNCH("b2ctr_gemm(bf16x3 split A)");
  }
  if (b_given) {
    const int64_t rp = round_up(b_sr, 256), cp = planes_cols_pad(b_sc);
    b_hi = (__nv_bfloat16*)g->b_planes; b_lo = b_hi + rp * cp; b_pitch = cp; b_prows = rp;
  } else {
    b_hi = (__nv_bfloat16*)w; b_lo = b_hi + np * kp;
    b_pitch = b_mn ? np : kp; b_prows = b_mn ? kp : np;
    if (b_kc) split_k(g->b, g->ldb, g->n, g->k, np, kp, b_hi, b_lo);
    else if (b_mn) split_k(g->b, g->ldb, g->k, g->n, kp, np, b_hi, b_lo);
    else split_t(g->b, g->ldb, g->n, np, b_hi, b_lo);
    B2_CHECK_LAUNCH("b2ctr_gemm(bf16x3 split B)");
  }
  PlaneArgs pa;
  pa.a_hi = a_hi; pa.a_lo = a_lo; pa.b_hi = b_hi; pa.b_lo = b_lo;
  pa.a_mn = a_mn; pa.b_mn = b_mn;
  pa.a_pitch = a_pitch; pa.b_pitch = b_pitch;
  pa.c = g->c; pa.bias = g->bias; pa.ws = ws;
  pa.m = g->m; pa.n = g->n; pa.k_pad = kp; pa.ldc = g->ldc;
  pa.k_per_split = ceil_div(ceil_div(kp, splits), kTK) * kTK;
  pa.alpha = g->alpha; pa.act = g->act; pa.accumulate = g->accumulate; pa.splits = splits;
  pa.cin_on = 0; pa.cin_t0 = pa.cin_xk = nullptr; pa.cin_ld0 = pa.cin_ldk = pa.cin_rows = 0; pa.cin_m = pa.cin_h = pa.cin_hp = 0;
  pa.fold_dt0 = pa.fold_dxk = nullptr; pa.fold_ldx = 0;
  cudaError_t e;
  const bool short_k = pa.k_per_split <= 4 * kTK;
  if (ws_kernel) {
    WsArgs wa;
    wa.p = pa;
    wa.tiles_m = (int)ceil_div(g->m, (int64_t)kTM);
    wa.tiles_n = (int)ceil_div(g->n, bn);
    wa.ntiles = (int64_t)wa.tiles_m * wa.tiles_n * splits;
    // TMA producers: four tiled tensor maps over the operand planes (box = one stage's slice of a plane)
    TmaMaps tm{};
    if (!(tma_map_2d(&tm.ah, a_hi, a_pitch, a_prows, a_pitch, 64, a_mn ? 64 : kTM) &&
          tma_map_2d(&tm.al, a_lo, a_pitch, a_prows, a_pitch, 64, a_mn ? 64 : kTM) &&
          tma_map_2d(&tm.bh, b_hi, b_pitch, b_prows, b_pitch, 64, b_mn ? 64 : bn) &&
          tma_map_2d(&tm.bl, b_lo, b_pitch, b_prows, b_pitch, 64, b_mn ? 64 : bn))) {
      set_error("b2ctr_gemm(bf16x3): cuTensorMapEncodeTiled unavailable (the kernel loads its operands by TMA)");
      return B2CTR_ERR_UNSUPPORTED;
    }
    wa.c_tma = tma_map_c(&tm.c, pa) ? 1 : tma_map_ws(&tm.c, pa) ? 2 : 0;
    // split-K with at most one unit per CTA (256 -> 128 and 128 -> 64 wgrads: 128 and 64 units): cooperative
    // consumers.  With more units (845 -> 256: 252 on 132 CTAs) ping-pong overlaps one unit's epilogue with the
    // next one's MMAs.
    wa.coop = splits > 1 && wa.ntiles <= kNumSMs;
    if (bn == 32) e = launch_ws_impl<32, 5>(wa, tm, st);
    else if (bn == 64) e = launch_ws_impl<64, 4>(wa, tm, st);
    else e = launch_ws_impl<128, 3>(wa, tm, st);
  } else if (bn == 32) e = short_k ? launch_planes<32, 1>(pa, st) : launch_planes<32, 4>(pa, st);
  else if (bn == 64) e = short_k ? launch_planes<64, 1>(pa, st) : launch_planes<64, 4>(pa, st);
  else if (bn == 128) e = short_k ? launch_planes<128, 1>(pa, st) : launch_planes<128, 3>(pa, st);
  else e = launch_planes<256, 2>(pa, st);
  if (e != cudaSuccess) {
    set_error("b2ctr_gemm(bf16x3 planes): CUDA launch failed: %s", cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  if (splits > 1) {
    // variant 3 keeps the scalar reduction: the reference the persistent path is compared against
    if (ws_kernel) splitk_reduce(pa, st);
    else tc_splitk_reduce_kernel<<<grid_for(g->m * g->n, 256, 4), 256, 0, st>>>(pa);
    B2_CHECK_LAUNCH("b2ctr_gemm(bf16x3 splitk_reduce)");
  }
  return B2CTR_OK;
}

// ================================================================================================
// CIN on the tensor cores without ever materialising the outer product (SURVEY.md 3.3 / 8a17).
// ================================================================================================
// planes of the PADDED filter W'[i*hp + j, n] = W[i*h + j, n] (j < h), zero rows for h <= j < hp
__global__ void __launch_bounds__(256)
    cin_filter_planes_kernel(const float* __restrict__ w, int m, int h, int hp, int64_t n, int64_t rows_pad,
                             int64_t cols_pad, __nv_bfloat16* hi, __nv_bfloat16* lo) {
  const int64_t chunks = cols_pad / 8;
  const int64_t total = rows_pad * chunks;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / chunks;
    const int64_t c0 = (t - r * chunks) * 8;
    const int i = (int)(r / hp), j = (int)(r - (int64_t)i * hp);
    const bool ok = i < m && j < h;
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float v0 = (ok && c0 + 2 * e < n) ? __ldg(w + ((int64_t)i * h + j) * n + c0 + 2 * e) : 0.f;
      const float v1 = (ok && c0 + 2 * e + 1 < n) ? __ldg(w + ((int64_t)i * h + j) * n + c0 + 2 * e + 1) : 0.f;
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v0), h1 = __float2bfloat16_rn(v1);
      hh[e] = pack_bf16(h0, h1);
      ll[e] = pack_bf16(__float2bfloat16_rn(v0 - __bfloat162float(h0)), __float2bfloat16_rn(v1 - __bfloat162float(h1)));
    }
    *reinterpret_cast<uint4*>(hi + r * cols_pad + c0) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    *reinterpret_cast<uint4*>(lo + r * cols_pad + c0) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
  }
}

b2ctr_status_t cin_filter_planes(const float* w, int m, int h, int hp, int64_t n, void* planes, cudaStream_t st) {
  const int64_t rp = round_up((int64_t)m * hp, 256), cp = planes_cols_pad(n);
  __nv_bfloat16* hi = (__nv_bfloat16*)planes;
  cin_filter_planes_kernel<<<grid_for(rp * (cp / 8), 256, 8), 256, 0, st>>>(w, m, h, hp, n, rp, cp, hi, hi + rp * cp);
  B2_CHECK_LAUNCH("b2ctr_cin_filter_planes");
  return B2CTR_OK;
}

// A GEMM whose A operand is generated by the producer warps (kind 1: CIN outer product, kind 2: DIN attention input)
struct GenSpec {
  int kind;
  const float* p0; int64_t ld0;
  const float* p1; int64_t ld1;
  int64_t rows;
  int m, h, hp;
  int64_t kq;            // columns of the generated matrix
};

static size_t gen_gemm_workspace_bytes(const GenSpec& sp, int mode, int64_t n, int split_k) {
  const int64_t M = mode == 0 ? sp.rows : sp.kq;
  return split_k > 1 ? (size_t)split_k * M * n * sizeof(float) + 256 : 0;
}

template <int GEN>
static cudaError_t launch_gen(const WsArgs& wa, const TmaMaps& tm, int bn, cudaStream_t st) {
  if (bn == 64) return launch_ws_impl<64, 4, GEN>(wa, tm, st);
  return launch_ws_impl<128, 3, GEN>(wa, tm, st);
}

// mode 0: c[rows, n] = act(A B + bias), B = planes of a [kq, n] row-major matrix; mode 1: c[kq, n] = A^T dY,
// dY given as the planes of a [rows, n] row-major matrix.
static b2ctr_status_t gen_gemm(const GenSpec& sp, int mode, int64_t n, const void* planes, float* c, int64_t ldc,
                               const float* bias, int act, int split_k, void* workspace, size_t workspace_bytes,
                               cudaStream_t st, const char* what) {
  B2_REQUIRE(sp.rows < (1ll << 31) && sp.kq < (1ll << 31), "%s: rows and generated width must fit 31 bits", what);
  const size_t need = gen_gemm_workspace_bytes(sp, mode, n, split_k);
  if (need && (!workspace || workspace_bytes < need)) {
    set_error("%s: needs %zu workspace bytes, got %zu", what, need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int splits = split_k > 1 ? split_k : 1;
  PlaneArgs pa;
  pa.a_hi = pa.a_lo = nullptr; pa.a_pitch = 0;
  pa.cin_on = sp.kind; pa.cin_t0 = sp.p0; pa.cin_xk = sp.p1; pa.cin_ld0 = sp.ld0; pa.cin_ldk = sp.ld1;
  pa.cin_rows = sp.rows; pa.cin_m = sp.m; pa.cin_h = sp.h; pa.cin_hp = sp.hp;
  pa.fold_dt0 = pa.fold_dxk = nullptr; pa.fold_ldx = 0;
  pa.b_mn = 1;      // both B operands are row-major matrices whose reduction dim is their row index
  pa.c = c; pa.bias = bias; pa.ws = (float*)workspace; pa.ldc = ldc;
  pa.alpha = 1.f; pa.act = act; pa.accumulate = 0; pa.splits = splits;
  pa.n = n;
  const int64_t cp = planes_cols_pad(n);
  int64_t b_prows;
  if (mode == 0) {
    pa.a_mn = 0; pa.m = sp.rows; pa.k_pad = round_up(sp.kq, kTK);
    b_prows = round_up(sp.kq, 256);
  } else {
    pa.a_mn = 1; pa.m = sp.kq; pa.k_pad = round_up(sp.rows, kTK);
    b_prows = round_up(sp.rows, 256);
  }
  const __nv_bfloat16* bp = (const __nv_bfloat16*)planes;
  pa.b_hi = bp; pa.b_lo = bp + b_prows * cp; pa.b_pitch = cp;
  pa.k_per_split = ceil_div(ceil_div(pa.k_pad, splits), kTK) * kTK;
  const int bn = n <= 64 ? 64 : 128;
  WsArgs wa;
  wa.p = pa;
  wa.tiles_m = (int)ceil_div(pa.m, (int64_t)kTM);
  wa.tiles_n = (int)ceil_div(n, bn);
  wa.ntiles = (int64_t)wa.tiles_m * wa.tiles_n * splits;
  TmaMaps tm{};
  if (!tma_map_2d(&tm.bh, pa.b_hi, cp, b_prows, cp, 64, 64) || !tma_map_2d(&tm.bl, pa.b_lo, cp, b_prows, cp, 64, 64)) {
    set_error("%s: cuTensorMapEncodeTiled unavailable (the kernel loads its B operand by TMA)", what);
    return B2CTR_ERR_UNSUPPORTED;
  }
  tm.ah = tm.bh; tm.al = tm.bl;
  wa.c_tma = tma_map_c(&tm.c, pa);
  wa.coop = 0;
  const cudaError_t e = sp.kind == 1 ? launch_gen<1>(wa, tm, bn, st) : launch_gen<2>(wa, tm, bn, st);
  if (e != cudaSuccess) {
    set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  if (splits > 1) {
    tc_splitk_reduce_kernel<<<grid_for(pa.m * n, 256, 4), 256, 0, st>>>(pa);
    B2_CHECK_LAUNCH("generated-operand gemm (splitk_reduce)");
  }
  return B2CTR_OK;
}

static GenSpec cin_spec(const b2ctr_cin_gemm_t* g) {
  GenSpec sp;
  sp.kind = 1; sp.p0 = g->t0; sp.ld0 = g->ld0; sp.p1 = g->xk; sp.ld1 = g->ldk; sp.rows = g->rows;
  sp.m = g->m; sp.h = g->h; sp.hp = g->hp; sp.kq = (int64_t)g->m * g->hp;
  return sp;
}
size_t cin_gemm_workspace_bytes(const b2ctr_cin_gemm_t* g) {
  return gen_gemm_workspace_bytes(cin_spec(g), g->mode, g->n, g->split_k);
}
b2ctr_status_t cin_gemm(const b2ctr_cin_gemm_t* g, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  B2_REQUIRE(g && g->t0 && g->xk && g->c && g->rows > 0 && g->m > 0 && g->h > 0 && g->n > 0, "cin_gemm: bad arguments");
  B2_REQUIRE(g->hp >= g->h && (g->hp == 32 || g->hp % 64 == 0), "cin_gemm: hp must be 32 or a multiple of 64 and >= h");
  B2_REQUIRE(g->ldk % 4 == 0 && ((uintptr_t)g->xk & 15) == 0 && g->ld0 >= g->m, "cin_gemm: xk rows must be 16-byte aligned");
  B2_REQUIRE(g->h % 4 == 0 || g->ldk >= g->hp, "cin_gemm: h must be a multiple of 4 unless the xk rows are padded to hp");
  B2_REQUIRE(g->mode == 0 ? g->w_planes != nullptr : g->dy_planes != nullptr, "cin_gemm: operand planes missing");
  return gen_gemm(cin_spec(g), g->mode, g->n, g->mode == 0 ? g->w_planes : g->dy_planes, g->c, g->ldc, g->bias, g->act,
                  g->split_k, workspace, workspace_bytes, st, "b2ctr_cin_gemm");
}

// CIN backward, data gradient: dZ = dY W'^T folded onto T0 and X_k inside the epilogue (FOLD kernel).
// dY given as K-major planes of [rows, n]; W' planes (b2ctr_cin_filter_planes) read K-major (rows = q).
b2ctr_status_t cin_fold(const b2ctr_cin_gemm_t* g, float* dt0, float* dxk, int64_t ldx, cudaStream_t st) {
  B2_REQUIRE(g && g->t0 && g->xk && g->w_planes && g->dy_planes && dt0 && dxk, "cin_fold: bad arguments");
  B2_REQUIRE(g->hp == 32 || g->hp == 64 || g->hp == 128, "cin_fold: hp must be 32, 64 or 128");
  B2_REQUIRE(g->ldk % 4 == 0 && ldx % 4 == 0 && ((uintptr_t)dxk & 15) == 0 && ((uintptr_t)g->xk & 15) == 0 &&
                 (g->h % 4 == 0 || (g->ldk >= g->hp && ldx >= g->hp)) && ldx >= g->h,
             "cin_fold: xk / dxk rows must be 16-byte aligned (and padded to hp when h is not a multiple of 4)");
  const int64_t kq = (int64_t)g->m * g->hp;
  PlaneArgs pa;
  const int64_t cpn = planes_cols_pad(g->n);
  const __nv_bfloat16* ap = (const __nv_bfloat16*)g->dy_planes;
  const int64_t a_prows = round_up(g->rows, 256);
  pa.a_hi = ap; pa.a_lo = ap + a_prows * cpn; pa.a_pitch = cpn; pa.a_mn = 0;
  const __nv_bfloat16* bp = (const __nv_bfloat16*)g->w_planes;
  const int64_t b_prows = round_up(kq, 256);
  pa.b_hi = bp; pa.b_lo = bp + b_prows * cpn; pa.b_pitch = cpn; pa.b_mn = 0;
  pa.c = nullptr; pa.bias = nullptr; pa.ws = nullptr; pa.ldc = 0;
  pa.m = g->rows; pa.n = kq; pa.k_pad = round_up(g->n, kTK);
  pa.k_per_split = pa.k_pad; pa.alpha = 1.f; pa.act = 0; pa.accumulate = 0; pa.splits = 1;
  pa.cin_on = 0; pa.cin_t0 = g->t0; pa.cin_xk = g->xk; pa.cin_ld0 = g->ld0; pa.cin_ldk = g->ldk; pa.cin_rows = g->rows;
  pa.cin_m = g->m; pa.cin_h = g->h; pa.cin_hp = g->hp;
  pa.fold_dt0 = dt0; pa.fold_dxk = dxk; pa.fold_ldx = ldx;
  constexpr int bn = 128;
  WsArgs wa;
  wa.p = pa;
  wa.tiles_m = (int)ceil_div(g->rows, (int64_t)kTM);
  wa.tiles_n = (int)ceil_div(kq, bn);
  wa.ntiles = (int64_t)wa.tiles_m * wa.tiles_n;
  TmaMaps tm{};
  if (!(tma_map_2d(&tm.ah, pa.a_hi, cpn, a_prows, cpn, 64, kTM) && tma_map_2d(&tm.al, pa.a_lo, cpn, a_prows, cpn, 64, kTM) &&
        tma_map_2d(&tm.bh, pa.b_hi, cpn, b_prows, cpn, 64, bn) && tma_map_2d(&tm.bl, pa.b_lo, cpn, b_prows, cpn, 64, bn))) {
    set_error("cin_fold: cuTensorMapEncodeTiled unavailable");
    return B2CTR_ERR_UNSUPPORTED;
  }
  wa.c_tma = 0;      // the fold epilogue never stores the accumulator tile
  wa.coop = 0;
  cudaError_t e = launch_ws_impl<128, 3, 0, true>(wa, tm, st);
  if (e != cudaSuccess) {
    set_error("b2ctr_cin_fold: CUDA launch failed: %s", cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  return B2CTR_OK;
}

static GenSpec att_spec(const b2ctr_att_gemm_t* g) {
  GenSpec sp;
  sp.kind = 2; sp.p0 = g->query; sp.ld0 = g->ldq; sp.p1 = g->keys; sp.ld1 = g->key_batch_stride;
  sp.rows = g->batch * g->maxlen; sp.m = g->maxlen; sp.h = g->dim; sp.hp = g->dim; sp.kq = 4 * (int64_t)g->dim;
  return sp;
}
size_t att_gemm_workspace_bytes(const b2ctr_att_gemm_t* g) {
  return gen_gemm_workspace_bytes(att_spec(g), g->mode, g->n, g->split_k);
}
b2ctr_status_t att_gemm(const b2ctr_att_gemm_t* g, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  B2_REQUIRE(g && g->query && g->keys && g->c && g->planes && g->batch > 0 && g->maxlen > 0 && g->n > 0,
             "att_gemm: bad arguments");
  B2_REQUIRE(g->dim > 0 && g->dim % 8 == 0, "att_gemm: the embedding size must be a multiple of 8");
  B2_REQUIRE(g->ldq % 4 == 0 && g->key_batch_stride % 4 == 0 && ((uintptr_t)g->query & 15) == 0 &&
                 ((uintptr_t)g->keys & 15) == 0, "att_gemm: query / keys rows must be 16-byte aligned");
  return gen_gemm(att_spec(g), g->mode, g->n, g->planes, g->c, g->ldc, g->bias, g->act, g->split_k, workspace,
                  workspace_bytes, st, "b2ctr_att_gemm");
}

size_t planes_bytes(int64_t rows, int64_t cols) {
  return (size_t)round_up(rows, 256) * planes_cols_pad(cols) * 2 * sizeof(__nv_bfloat16) + 256;
}
b2ctr_status_t split_planes(const float* src, int64_t ld, int64_t rows, int64_t cols, void* planes,
                            cudaStream_t st) {
  const int64_t rp = round_up(rows, 256), cp = planes_cols_pad(cols);
  __nv_bfloat16* hi = (__nv_bfloat16*)planes;
  const int vec = (ld % 4 == 0) && (((uintptr_t)src & 15) == 0);
  split_planes_kernel<<<grid_for(rp * (cp / 8), 256, 8), 256, 0, st>>>(src, ld, rows, cols, rp, cp, hi, hi + rp * cp,
                                                                      vec);
  B2_CHECK_LAUNCH("b2ctr_split_planes");
  return B2CTR_OK;
}

}  // namespace b2ctr

extern "C" {
size_t b2ctr_cin_filter_planes_bytes(int32_t m, int32_t hp, int64_t n) { return b2ctr::planes_bytes((int64_t)m * hp, n); }
b2ctr_status_t b2ctr_cin_filter_planes(const float* w, int32_t m, int32_t h, int32_t hp, int64_t n, void* planes,
                                       void* stream) {
  B2_REQUIRE(w && planes && m > 0 && h > 0 && hp >= h && n > 0, "cin_filter_planes: bad arguments");
  return b2ctr::cin_filter_planes(w, m, h, hp, n, planes, (cudaStream_t)stream);
}
size_t b2ctr_cin_gemm_workspace_bytes(const b2ctr_cin_gemm_t* g) { return g ? b2ctr::cin_gemm_workspace_bytes(g) : 0; }
b2ctr_status_t b2ctr_cin_gemm(const b2ctr_cin_gemm_t* g, void* workspace, size_t workspace_bytes, void* stream) {
  return b2ctr::cin_gemm(g, workspace, workspace_bytes, (cudaStream_t)stream);
}
b2ctr_status_t b2ctr_cin_fold(const b2ctr_cin_gemm_t* g, float* dt0, float* dxk, int64_t ldx, void* stream) {
  return b2ctr::cin_fold(g, dt0, dxk, ldx, (cudaStream_t)stream);
}
size_t b2ctr_att_gemm_workspace_bytes(const b2ctr_att_gemm_t* g) { return g ? b2ctr::att_gemm_workspace_bytes(g) : 0; }
b2ctr_status_t b2ctr_att_gemm(const b2ctr_att_gemm_t* g, void* workspace, size_t workspace_bytes, void* stream) {
  return b2ctr::att_gemm(g, workspace, workspace_bytes, (cudaStream_t)stream);
}
}
