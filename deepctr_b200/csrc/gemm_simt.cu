// gemm_simt.cu — exact-fp32 GEMM on the FFMA pipe with fused bias/activation epilogue.
//
// This is the B2CTR_GEMM_FP32 precision mode: bit-for-bit fp32 products and fp32 accumulation,
// used for parity runs and as the checker of the wgmma split-bf16 path (gemm_tc.cu).
// Replaces tf.tensordot/tf.matmul of deepctr/layers/core.py:193-195 (DNN), deepctr/layers/core.py:106
// (LocalActivationUnit), deepctr/layers/interaction.py:414-418 (CrossNet), :754-757 (InteractingLayer).
#include "common.cuh"

namespace b2ctr {

constexpr int kBK = 8;
constexpr int kThreads = 256;

struct GemmArgs {
  const float* a; const float* b; float* c; const float* bias; float* ws;
  int64_t m, n, k;
  int64_t sam, sak;  // A(m,k) = a[m*sam + k*sak]
  int64_t sbk, sbn;  // B(k,n) = b[k*sbk + n*sbn]
  int64_t ldc;
  int64_t k_per_split;
  float alpha;
  int act, accumulate, splits;
};

template <int BM, int BN, bool A_KCONTIG, bool B_NCONTIG>
__global__ void __launch_bounds__(kThreads) sgemm_kernel(const GemmArgs g) {
  constexpr int TM = BM / 16, TN = BN / 16;
  constexpr int APT = BM * kBK / kThreads, BPT = BN * kBK / kThreads;
  constexpr int PAD = 4;
  __shared__ __align__(16) float As[2][kBK][BM + PAD];
  __shared__ __align__(16) float Bs[2][kBK][BN + PAD];

  const int t = threadIdx.x;
  const int tx = t % 16, ty = t / 16;
  const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN;
  const int64_t kbeg = (int64_t)blockIdx.z * g.k_per_split;
  const int64_t kend = kbeg + g.k_per_split < g.k ? kbeg + g.k_per_split : g.k;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[APT], rb[BPT];
  auto load_tile = [&](int64_t k0) {
#pragma unroll
    for (int i = 0; i < APT; ++i) {
      const int l = t + i * kThreads;
      const int kk = A_KCONTIG ? l % kBK : l / BM;
      const int mm = A_KCONTIG ? l / kBK : l % BM;
      const int64_t gm = m0 + mm, gk = k0 + kk;
      ra[i] = (gm < g.m && gk < kend) ? g.a[gm * g.sam + gk * g.sak] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < BPT; ++i) {
      const int l = t + i * kThreads;
      const int kk = B_NCONTIG ? l / BN : l % kBK;
      const int nn = B_NCONTIG ? l % BN : l / kBK;
      const int64_t gn = n0 + nn, gk = k0 + kk;
      rb[i] = (gn < g.n && gk < kend) ? g.b[gk * g.sbk + gn * g.sbn] : 0.f;
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int i = 0; i < APT; ++i) {
      const int l = t + i * kThreads;
      const int kk = A_KCONTIG ? l % kBK : l / BM;
      const int mm = A_KCONTIG ? l / kBK : l % BM;
      As[buf][kk][mm] = ra[i];
    }
#pragma unroll
    for (int i = 0; i < BPT; ++i) {
      const int l = t + i * kThreads;
      const int kk = B_NCONTIG ? l / BN : l % kBK;
      const int nn = B_NCONTIG ? l % BN : l / kBK;
      Bs[buf][kk][nn] = rb[i];
    }
  };
  // thread-tile coordinates: groups of 4 contiguous elements, groups 64 apart (conflict-free float4)
  auto row_of = [&](int i) { return TM >= 4 ? (i / 4) * 64 + ty * 4 + (i % 4) : ty * TM + i; };
  auto col_of = [&](int j) { return TN >= 4 ? (j / 4) * 64 + tx * 4 + (j % 4) : tx * TN + j; };

  int buf = 0;
  if (kbeg < kend) {
    load_tile(kbeg);
    store_tile(0);
  }
  __syncthreads();
  for (int64_t k0 = kbeg; k0 < kend; k0 += kBK) {
    const bool has_next = k0 + kBK < kend;
    if (has_next) load_tile(k0 + kBK);
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      float av[TM], bv[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) av[i] = As[buf][kk][row_of(i)];
#pragma unroll
      for (int j = 0; j < TN; ++j) bv[j] = Bs[buf][kk][col_of(j)];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (has_next) store_tile(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t gm = m0 + row_of(i);
    if (gm >= g.m) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int64_t gn = n0 + col_of(j);
      if (gn >= g.n) continue;
      float v = g.alpha * acc[i][j];
      if (g.splits > 1) {
        g.ws[((int64_t)blockIdx.z * g.m + gm) * g.n + gn] = v;
      } else {
        if (g.accumulate) v += g.c[gm * g.ldc + gn];
        if (g.bias) v += g.bias[gn];
        g.c[gm * g.ldc + gn] = act_apply(v, g.act);
      }
    }
  }
}

// deterministic split-K reduction (ascending split order) + epilogue
__global__ void splitk_reduce_kernel(const GemmArgs g) {
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

// Few outputs, many slices (the [64, 1] / [13, 1] wgrads of the [*, 1] projections arrive in ~256 slices): one warp
// per output, lanes stride over the slices, fixed shuffle tree - deterministic, and 8 dependent loads per lane
// instead of 256 per thread (measured 25 us -> for a 64 x 256 reduction in the one-thread-per-output kernel).
__global__ void __launch_bounds__(256) splitk_reduce_small_kernel(const GemmArgs g) {
  const int64_t total = g.m * g.n;
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= total) return;
  float v = 0.f;
  for (int z = lane; z < g.splits; z += 32) v += g.ws[(int64_t)z * total + i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) {
    const int64_t gm = i / g.n, gn = i - gm * g.n;
    if (g.accumulate) v += g.c[gm * g.ldc + gn];
    if (g.bias) v += g.bias[gn];
    g.c[gm * g.ldc + gn] = act_apply(v, g.act);
  }
}
static void launch_splitk_reduce(const GemmArgs& ga, cudaStream_t st) {
  const int64_t total = ga.m * ga.n;
  if (total <= 4096 && ga.splits >= 16)
    splitk_reduce_small_kernel<<<(unsigned)ceil_div(total, 8), 256, 0, st>>>(ga);
  else
    splitk_reduce_kernel<<<grid_for(total, 256, 4), 256, 0, st>>>(ga);
}

// ---- skinny shapes -----------------------------------------------------------------------------
// The final [*, 1] projection of every CTR tower (and its dgrad) is a GEMV / outer product: HBM-bound, and a
// 128 x 32 tile kernel spends 97 % of its lanes on padding (measured 81 us for M = 65536, K = 64, N = 1).
//
// N <= 8, A row-major: LPR lanes share a row (float4 each per pass), partial dot products meet by shuffles.
template <int N>
__global__ void __launch_bounds__(256) skinny_n_kernel(const GemmArgs g, int lpr, int vec) {
  const int lane = threadIdx.x & 31;
  const int rows_per_warp = 32 / lpr;
  const int sub = lane / lpr, li = lane % lpr;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  if (vec && g.k <= (int64_t)lpr * 4) {
    // one 16-byte load per lane covers its share of a row: four row groups per iteration, their loads issued
    // back to back (the one-group loop below keeps a single load in flight per lane: 0.7 TB/s on [409600, 40]).
    // The last group may reach past k into the row's padding: those columns are replaced by zero rather than
    // multiplied by a zero weight, so that a NaN or Inf in the padding cannot reach the output.
    const int64_t k = (int64_t)li * 4;
    const bool kin = k < g.k;
    const bool in1 = k + 1 < g.k, in2 = k + 2 < g.k, in3 = k + 3 < g.k;
    float b[N][4];
#pragma unroll
    for (int n = 0; n < N; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        b[n][e] = (n < g.n && k + e < g.k) ? __ldg(g.b + (k + e) * g.sbk + n * g.sbn) : 0.f;
    const int64_t step = (int64_t)rows_per_warp * 4;
    for (int64_t r0 = warp * step; r0 < g.m; r0 += nwarps * step) {
      float4 a[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t r = r0 + u * rows_per_warp + sub;
        a[u] = (r < g.m && kin) ? __ldg(reinterpret_cast<const float4*>(g.a + r * g.sam + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
        a[u].y = in1 ? a[u].y : 0.f;
        a[u].z = in2 ? a[u].z : 0.f;
        a[u].w = in3 ? a[u].w : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t r = r0 + u * rows_per_warp + sub;
        float acc[N];
#pragma unroll
        for (int n = 0; n < N; ++n) {
          acc[n] = fmaf(a[u].w, b[n][3], fmaf(a[u].z, b[n][2], fmaf(a[u].y, b[n][1], a[u].x * b[n][0])));
          for (int o = lpr >> 1; o > 0; o >>= 1) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
        }
        if (r < g.m && li == 0) {
#pragma unroll
          for (int n = 0; n < N; ++n) {
            if (n < g.n) {
              float v = g.alpha * acc[n];
              if (g.accumulate) v += g.c[r * g.ldc + n];
              if (g.bias) v += g.bias[n];
              g.c[r * g.ldc + n] = act_apply(v, g.act);
            }
          }
        }
      }
    }
    return;
  }
  for (int64_t r0 = warp * rows_per_warp; r0 < g.m; r0 += nwarps * rows_per_warp) {
    const int64_t r = r0 + sub;
    float acc[N];
#pragma unroll
    for (int n = 0; n < N; ++n) acc[n] = 0.f;
    if (r < g.m) {
      const float* arow = g.a + r * g.sam;
      if (vec) {
        for (int64_t k = (int64_t)li * 4; k < g.k; k += (int64_t)lpr * 4) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(arow + k));
#pragma unroll
          for (int n = 0; n < N; ++n) {
            if (n < g.n) {
              const float* bp = g.b + k * g.sbk + n * g.sbn;
              acc[n] = fmaf(a.x, __ldg(bp), acc[n]);
              if (k + 1 < g.k) acc[n] = fmaf(a.y, __ldg(bp + g.sbk), acc[n]);
              if (k + 2 < g.k) acc[n] = fmaf(a.z, __ldg(bp + 2 * g.sbk), acc[n]);
              if (k + 3 < g.k) acc[n] = fmaf(a.w, __ldg(bp + 3 * g.sbk), acc[n]);
            }
          }
        }
      } else {
        for (int64_t k = li; k < g.k; k += lpr) {
          const float a = __ldg(arow + k);
#pragma unroll
          for (int n = 0; n < N; ++n)
            if (n < g.n) acc[n] = fmaf(a, __ldg(g.b + k * g.sbk + n * g.sbn), acc[n]);
        }
      }
    }
#pragma unroll
    for (int n = 0; n < N; ++n)
      for (int o = lpr >> 1; o > 0; o >>= 1) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
    if (r < g.m && li == 0) {
#pragma unroll
      for (int n = 0; n < N; ++n) {
        if (n < g.n) {
          float v = g.alpha * acc[n];
          if (g.accumulate) v += g.c[r * g.ldc + n];
          if (g.bias) v += g.bias[n];
          g.c[r * g.ldc + n] = act_apply(v, g.act);
        }
      }
    }
  }
}
// A stored [K, M] (wgrad of a skinny layer: C[m, n] = sum_k A[k, m] B(k, n), N <= 8, K = batch): a stream over
// the rows of A; thread = (column m, one of 4 k-lanes), 8 independent row loads in flight, k-lanes meet in
// shared memory.  One CTA per (64-column block, K slice); slices go through the split-K workspace.
template <int N, int COLS = 64>
__global__ void __launch_bounds__(256) skinny_tn_kernel(const GemmArgs g) {
  constexpr int KL = 256 / COLS;         // k-lanes: 4 for 64-column blocks, 16 for M <= 16 (the 13 dense features)
  __shared__ float red[KL][COLS][N];
  const int col = threadIdx.x % COLS, kl = threadIdx.x / COLS;
  const int64_t m = (int64_t)blockIdx.x * COLS + col;
  const int64_t kbeg = (int64_t)blockIdx.z * g.k_per_split;
  const int64_t kend = kbeg + g.k_per_split < g.k ? kbeg + g.k_per_split : g.k;
  float acc[N];
#pragma unroll
  for (int n = 0; n < N; ++n) acc[n] = 0.f;
  if (m < g.m) {
    int64_t k = kbeg + kl;
    for (; k + 7 * KL < kend; k += 8 * KL) {
      float a[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] = __ldg(g.a + (k + KL * u) * g.sak + m);
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int n = 0; n < N; ++n)
          if (n < g.n) acc[n] = fmaf(a[u], __ldg(g.b + (k + KL * u) * g.sbk + n * g.sbn), acc[n]);
    }
    for (; k < kend; k += KL) {
      const float a = __ldg(g.a + k * g.sak + m);
#pragma unroll
      for (int n = 0; n < N; ++n)
        if (n < g.n) acc[n] = fmaf(a, __ldg(g.b + k * g.sbk + n * g.sbn), acc[n]);
    }
  }
#pragma unroll
  for (int n = 0; n < N; ++n) red[kl][col][n] = acc[n];
  __syncthreads();
  if (kl == 0 && m < g.m) {
#pragma unroll
    for (int n = 0; n < N; ++n) {
      if (n < g.n) {
        float v = 0.f;
#pragma unroll
        for (int l = 0; l < KL; ++l) v += red[l][col][n];        // ascending k-lane order
        v *= g.alpha;
        if (g.splits > 1) {
          g.ws[((int64_t)blockIdx.z * g.m + m) * g.n + n] = v;
        } else {
          if (g.accumulate) v += g.c[m * g.ldc + n];
          if (g.bias) v += g.bias[n];
          g.c[m * g.ldc + n] = act_apply(v, g.act);
        }
      }
    }
  }
}
// The same stream with 16-byte loads (M % 4 == 0, aligned rows): thread = (4 consecutive columns, one of 16 k-lanes),
// 4 rows in flight per thread = 4x the bytes in flight of the scalar kernel.
template <int N>
__global__ void __launch_bounds__(256) skinny_tn_vec4_kernel(const GemmArgs g) {
  __shared__ float red[16][64][N];
  const int cq = threadIdx.x & 15, kl = threadIdx.x >> 4;
  const int64_t m = (int64_t)blockIdx.x * 64 + cq * 4;
  const int64_t kbeg = (int64_t)blockIdx.z * g.k_per_split;
  const int64_t kend = kbeg + g.k_per_split < g.k ? kbeg + g.k_per_split : g.k;
  float acc[N][4];
#pragma unroll
  for (int n = 0; n < N; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  if (m < g.m) {             // M % 4 == 0: the quad is inside the matrix
    int64_t k = kbeg + kl;
    for (; k + 48 < kend; k += 64) {
      float4 a[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) a[u] = __ldg(reinterpret_cast<const float4*>(g.a + (k + 16 * u) * g.sak + m));
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int n = 0; n < N; ++n)
          if (n < g.n) {
            const float b = __ldg(g.b + (k + 16 * u) * g.sbk + n * g.sbn);
            acc[n][0] = fmaf(a[u].x, b, acc[n][0]); acc[n][1] = fmaf(a[u].y, b, acc[n][1]);
            acc[n][2] = fmaf(a[u].z, b, acc[n][2]); acc[n][3] = fmaf(a[u].w, b, acc[n][3]);
          }
    }
    for (; k < kend; k += 16) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(g.a + k * g.sak + m));
#pragma unroll
      for (int n = 0; n < N; ++n)
        if (n < g.n) {
          const float b = __ldg(g.b + k * g.sbk + n * g.sbn);
          acc[n][0] = fmaf(a.x, b, acc[n][0]); acc[n][1] = fmaf(a.y, b, acc[n][1]);
          acc[n][2] = fmaf(a.z, b, acc[n][2]); acc[n][3] = fmaf(a.w, b, acc[n][3]);
        }
    }
  }
#pragma unroll
  for (int n = 0; n < N; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) red[kl][cq * 4 + e][n] = acc[n][e];
  __syncthreads();
  const int col = threadIdx.x & 63;
  const int64_t mc = (int64_t)blockIdx.x * 64 + col;
  if (threadIdx.x < 64 && mc < g.m) {
#pragma unroll
    for (int n = 0; n < N; ++n) {
      if (n < g.n) {
        float v = 0.f;
#pragma unroll
        for (int l = 0; l < 16; ++l) v += red[l][col][n];       // ascending k-lane order
        v *= g.alpha;
        if (g.splits > 1) {
          g.ws[((int64_t)blockIdx.z * g.m + mc) * g.n + n] = v;
        } else {
          if (g.accumulate) v += g.c[mc * g.ldc + n];
          if (g.bias) v += g.bias[n];
          g.c[mc * g.ldc + n] = act_apply(v, g.act);
        }
      }
    }
  }
}
// K <= 8, A row-major: C[m, n] = sum_k A[m,k] B(k,n) is an outer-product-shaped stream of writes
// (dgrad of a [*, 1] layer); thread = (row, 4 consecutive columns).
__global__ void __launch_bounds__(256) skinny_k_kernel(const GemmArgs g, int vec_c) {
  const int64_t chunks = (g.n + 3) / 4;
  const int64_t total = g.m * chunks;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / chunks;
    const int64_t n0 = (t - r * chunks) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < g.k; ++k) {
      const float a = __ldg(g.a + r * g.sam + k);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n0 + j < g.n) v[j] = fmaf(a, __ldg(g.b + k * g.sbk + (n0 + j) * g.sbn), v[j]);
    }
    float* cp = g.c + r * g.ldc + n0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (n0 + j < g.n) {
        float o = g.alpha * v[j];
        if (g.accumulate) o += cp[j];
        if (g.bias) o += g.bias[n0 + j];
        v[j] = act_apply(o, g.act);
      }
    }
    if (vec_c && n0 + 4 <= g.n) {
      *reinterpret_cast<float4*>(cp) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n0 + j < g.n) cp[j] = v[j];
    }
  }
}

template <int BM, int BN>
static void launch_cfg(const GemmArgs& ga, bool akc, bool bnc, cudaStream_t st) {
  dim3 grid((unsigned)ceil_div(ga.n, BN), (unsigned)ceil_div(ga.m, BM), (unsigned)ga.splits);
  if (akc && bnc) sgemm_kernel<BM, BN, true, true><<<grid, kThreads, 0, st>>>(ga);
  else if (akc && !bnc) sgemm_kernel<BM, BN, true, false><<<grid, kThreads, 0, st>>>(ga);
  else if (!akc && bnc) sgemm_kernel<BM, BN, false, true><<<grid, kThreads, 0, st>>>(ga);
  else sgemm_kernel<BM, BN, false, false><<<grid, kThreads, 0, st>>>(ga);
}

b2ctr_status_t gemm_fp32(const b2ctr_gemm_t* g, void* workspace, size_t workspace_bytes,
                         cudaStream_t st) {
  GemmArgs ga;
  ga.a = g->a; ga.b = g->b; ga.c = g->c; ga.bias = g->bias; ga.ws = (float*)workspace;
  ga.m = g->m; ga.n = g->n; ga.k = g->k;
  ga.sam = g->trans_a ? 1 : g->lda;  ga.sak = g->trans_a ? g->lda : 1;
  ga.sbk = g->trans_b ? 1 : g->ldb;  ga.sbn = g->trans_b ? g->ldb : 1;
  ga.ldc = g->ldc; ga.alpha = g->alpha; ga.act = g->act; ga.accumulate = g->accumulate;
  ga.splits = g->split_k > 1 ? g->split_k : 1;
  if (ga.splits > 1) {
    const size_t need = (size_t)ga.splits * g->m * g->n * sizeof(float);
    if (!workspace || workspace_bytes < need) {
      set_error("gemm: split_k=%d needs %zu workspace bytes, got %zu", ga.splits, need, workspace_bytes);
      return B2CTR_ERR_WORKSPACE;
    }
  }
  ga.k_per_split = ceil_div(ceil_div(g->k, ga.splits), kBK) * kBK;
  const bool akc = !g->trans_a, bnc = !g->trans_b;
  if (akc && ga.splits == 1 && g->n <= 8 && g->k >= 16) {
    int lpr = 1;
    while (lpr < 32 && lpr * 4 < g->k) lpr <<= 1;
    const int vec = (g->lda % 4 == 0) && ((reinterpret_cast<uintptr_t>(g->a) & 15) == 0);
    const int grid = grid_for(ceil_div(g->m, 32 / lpr), 8, 8);
    if (g->n <= 1) skinny_n_kernel<1><<<grid, 256, 0, st>>>(ga, lpr, vec);
    else if (g->n <= 2) skinny_n_kernel<2><<<grid, 256, 0, st>>>(ga, lpr, vec);
    else if (g->n <= 4) skinny_n_kernel<4><<<grid, 256, 0, st>>>(ga, lpr, vec);
    else skinny_n_kernel<8><<<grid, 256, 0, st>>>(ga, lpr, vec);
    B2_CHECK_LAUNCH("b2ctr_gemm(fp32 skinny-N)");
    return B2CTR_OK;
  }
  if (!akc && g->n <= 8 && g->k >= 64) {
    // sak = lda (A stored [K, M]); the K slices of split-K launches land in the workspace as usual
    dim3 grid((unsigned)ceil_div(g->m, 64), 1, (unsigned)ga.splits);
    if (g->m <= 16 && g->n <= 1) {         // a handful of columns (the dense features' [13, 1] kernel): 16 k-lanes
      skinny_tn_kernel<1, 16><<<grid, 256, 0, st>>>(ga);
      B2_CHECK_LAUNCH("b2ctr_gemm(fp32 skinny-TN)");
      if (ga.splits > 1) {
        launch_splitk_reduce(ga, st);
        B2_CHECK_LAUNCH("b2ctr_gemm(splitk_reduce)");
      }
      return B2CTR_OK;
    }
    const bool v4 = g->m % 4 == 0 && ga.sak % 4 == 0 && (reinterpret_cast<uintptr_t>(ga.a) & 15) == 0;
    if (v4 && g->n <= 1) skinny_tn_vec4_kernel<1><<<grid, 256, 0, st>>>(ga);
    else if (v4 && g->n <= 2) skinny_tn_vec4_kernel<2><<<grid, 256, 0, st>>>(ga);
    else if (g->n <= 1) skinny_tn_kernel<1><<<grid, 256, 0, st>>>(ga);
    else if (g->n <= 2) skinny_tn_kernel<2><<<grid, 256, 0, st>>>(ga);
    else if (g->n <= 4) skinny_tn_kernel<4><<<grid, 256, 0, st>>>(ga);
    else skinny_tn_kernel<8><<<grid, 256, 0, st>>>(ga);
    B2_CHECK_LAUNCH("b2ctr_gemm(fp32 skinny-TN)");
    if (ga.splits > 1) {
      launch_splitk_reduce(ga, st);
      B2_CHECK_LAUNCH("b2ctr_gemm(splitk_reduce)");
    }
    return B2CTR_OK;
  }
  if (akc && ga.splits == 1 && g->k <= 8 && g->n >= 16) {
    const int vec_c = (g->ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(g->c) & 15) == 0);
    skinny_k_kernel<<<grid_for(g->m * ceil_div(g->n, 4), 256, 8), 256, 0, st>>>(ga, vec_c);
    B2_CHECK_LAUNCH("b2ctr_gemm(fp32 skinny-K)");
    return B2CTR_OK;
  }
  if (g->n <= 32) launch_cfg<128, 32>(ga, akc, bnc, st);
  else if (g->n <= 64) launch_cfg<128, 64>(ga, akc, bnc, st);
  else launch_cfg<128, 128>(ga, akc, bnc, st);
  B2_CHECK_LAUNCH("b2ctr_gemm(fp32)");
  if (ga.splits > 1) {
    launch_splitk_reduce(ga, st);
    B2_CHECK_LAUNCH("b2ctr_gemm(splitk_reduce)");
  }
  return B2CTR_OK;
}

b2ctr_status_t gemm_bf16x3(const b2ctr_gemm_t* g, void* workspace, size_t workspace_bytes,
                           cudaStream_t st);  // gemm_tc.cu
size_t gemm_bf16x3_workspace_bytes(const b2ctr_gemm_t* g);
size_t planes_bytes(int64_t rows, int64_t cols);
b2ctr_status_t split_planes(const float* src, int64_t ld, int64_t rows, int64_t cols, void* planes,
                            cudaStream_t st);

}  // namespace b2ctr

using namespace b2ctr;

extern "C" {

size_t b2ctr_gemm_workspace_bytes(const b2ctr_gemm_t* g) {
  if (!g) return 0;
  if (g->precision == B2CTR_GEMM_BF16X3) return gemm_bf16x3_workspace_bytes(g);
  return g->split_k > 1 ? (size_t)g->split_k * g->m * g->n * sizeof(float) : 0;
}

size_t b2ctr_planes_bytes(int64_t rows, int64_t cols) { return planes_bytes(rows, cols); }

b2ctr_status_t b2ctr_split_planes(const float* src, int64_t ld, int64_t rows, int64_t cols, void* planes,
                                  void* stream) {
  B2_REQUIRE(src && planes && rows > 0 && cols > 0 && ld >= cols, "split_planes: bad arguments");
  B2_REQUIRE(((uintptr_t)planes & 15) == 0, "split_planes: planes must be 16-byte aligned");
  return split_planes(src, ld, rows, cols, planes, (cudaStream_t)stream);
}

b2ctr_status_t b2ctr_gemm(const b2ctr_gemm_t* g, void* workspace, size_t workspace_bytes,
                          void* stream) {
  B2_REQUIRE(g && g->c, "gemm: NULL descriptor or matrix pointer");
  // bf16x3 with caller planes: gemm_bf16x3 checks that an fp32 operand left NULL is not one it has to split
  const bool bf = g->precision == B2CTR_GEMM_BF16X3;
  B2_REQUIRE((g->a || (bf && g->a_planes)) && (g->b || (bf && g->b_planes)),
             "gemm: NULL A or B (allowed only in bf16x3 mode with the operand's planes)");
  B2_REQUIRE(g->m >= 0 && g->n >= 0 && g->k >= 0, "gemm: negative dimension");
  B2_REQUIRE(g->lda >= (g->trans_a ? g->m : g->k) && g->ldb >= (g->trans_b ? g->k : g->n) &&
                 g->ldc >= g->n,
             "gemm: leading dimension smaller than the row length");
  B2_REQUIRE(!(g->accumulate && g->act != B2CTR_ACT_NONE), "gemm: accumulate with activation");
  B2_REQUIRE(g->act >= B2CTR_ACT_NONE && g->act <= B2CTR_ACT_TANH, "gemm: bad activation");
  if (g->m == 0 || g->n == 0) return B2CTR_OK;
  if (g->precision == B2CTR_GEMM_BF16X3)
    return gemm_bf16x3(g, workspace, workspace_bytes, (cudaStream_t)stream);
  B2_REQUIRE(g->precision == B2CTR_GEMM_FP32, "gemm: unknown precision mode %d", g->precision);
  return gemm_fp32(g, workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
