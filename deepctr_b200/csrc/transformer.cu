// transformer.cu — the Transformer layer of BST (sm_90a): fused masked multi-head attention and
// LayerNormalization.
//
// Reference math restated (never copied): deepctr/layers/sequence.py:544-617 (scaled dot product, key mask,
// blinding, max-subtracted softmax, query mask, dropout, weighted sum, residual) and
// deepctr/layers/normalization.py:34-43.
//
// Attention: one CTA per (sample, head).  The head's Q / K / V slices are staged in shared memory (rows padded
// to DP + 1 floats, DP = d rounded up to 8 / 16 / 32 / 64, zero filled), one thread owns one query row (forward,
// backward dQ) or one key row (backward dK / dV).  The score row is consumed on the fly (online softmax in the
// forward, recomputed from the saved (max, sum) in the backward): no [T, T] tile exists anywhere.
#include "common.cuh"

namespace b2ctr {

constexpr float kMaskScore = -4294967295.f;  // -2^32 + 1 (rounds to -2^32 in fp32, as in TF)
constexpr int kMhaMaxT = 128;
constexpr int kMhaMaxD = 64;

struct MhaShape {
  int T, H, d, S;  // S = padded smem row pitch
};

__device__ __forceinline__ bool mha_valid(const int32_t* len, const uint8_t* mask, int64_t b, int t, int T) {
  if (len) return t < len[b];
  if (mask) return mask[b * T + t] != 0;
  return true;
}

// stage rows [b*T, b*T + T) of the head's column slice into s[t*S + c] (zero for c >= d)
template <int DP>
__device__ __forceinline__ void mha_stage(const float* __restrict__ src, int64_t ld, int64_t b, int h,
                                          const MhaShape& sh, float* s) {
  for (int idx = threadIdx.x; idx < sh.T * DP; idx += blockDim.x) {
    const int t = idx / DP, c = idx % DP;
    s[t * sh.S + c] = c < sh.d ? src[(b * sh.T + t) * ld + (int64_t)h * sh.d + c] : 0.f;
  }
}

// s[t*S + c] -> dst rows (+ optional residual)
__device__ __forceinline__ void mha_store(const float* s, float* __restrict__ dst, int64_t ld,
                                          const float* __restrict__ res, int64_t ldr, int64_t b, int h,
                                          const MhaShape& sh) {
  for (int idx = threadIdx.x; idx < sh.T * sh.d; idx += blockDim.x) {
    const int t = idx / sh.d, c = idx % sh.d;
    const int64_t row = b * sh.T + t;
    float v = s[t * sh.S + c];
    if (res) v += res[row * ldr + (int64_t)h * sh.d + c];
    dst[row * ld + (int64_t)h * sh.d + c] = v;
  }
}

struct MhaDrop {
  uint32_t thr;
  float keep_scale;
  uint64_t seed_mix;
  __device__ __forceinline__ float factor(uint64_t idx) const {
    if (thr == 0u) return 1.f;
    return mix32(seed_mix + idx) >= thr ? keep_scale : 0.f;
  }
};

__device__ __forceinline__ MhaDrop mha_drop(const b2ctr_mha_t& a) {
  MhaDrop d;
  d.thr = (uint32_t)((double)a.dropout_rate * 4294967296.0);
  d.keep_scale = 1.f / (1.f - a.dropout_rate);
  d.seed_mix = a.seed * 0x9E3779B97F4A7C15ULL;
  return d;
}

template <int DP>
__device__ __forceinline__ float mha_score(const float* qrow, const float* krow, float scale, bool valid) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < DP; ++c) s = fmaf(qrow[c], krow[c], s);
  return valid ? s * scale : kMaskScore;
}

template <int DP>
__global__ void __launch_bounds__(kMhaMaxT) mha_fwd_kernel(const b2ctr_mha_t a) {
  extern __shared__ float sm[];
  const MhaShape sh{a.T, a.heads, a.d, DP + 1};
  const int64_t b = blockIdx.x / sh.H;
  const int h = (int)(blockIdx.x % sh.H);
  float* qs = sm;
  float* ks = qs + sh.T * sh.S;
  float* vs = ks + sh.T * sh.S;
  float* qm = vs + sh.T * sh.S;
  float* km = qm + sh.T;
  mha_stage<DP>(a.q, a.ldq, b, h, sh, qs);
  mha_stage<DP>(a.k, a.ldk, b, h, sh, ks);
  mha_stage<DP>(a.v, a.ldv, b, h, sh, vs);
  for (int t = threadIdx.x; t < sh.T; t += blockDim.x) {
    qm[t] = mha_valid(a.qlen, a.qmask, b, t, sh.T) ? 1.f : 0.f;
    km[t] = mha_valid(a.klen, a.kmask, b, t, sh.T) ? 1.f : 0.f;
  }
  __syncthreads();
  const int i = threadIdx.x;
  if (i < sh.T) {
    const MhaDrop drop = mha_drop(a);
    const uint64_t base = (((uint64_t)h * a.batch + b) * sh.T + i) * sh.T;
    float qr[DP], acc[DP];
#pragma unroll
    for (int c = 0; c < DP; ++c) {
      qr[c] = qs[i * sh.S + c];
      acc[c] = 0.f;
    }
    float m = -INFINITY, l = 0.f;
    for (int j = 0; j < sh.T; ++j) {
      const float* kr = ks + j * sh.S;
      const float s = mha_score<DP>(qr, kr, a.scale, km[j] != 0.f && !(a.blinding && i == j));
      if (s > m) {  // online softmax: rescale what was accumulated against the old maximum
        const float corr = expf(m - s);
        l *= corr;
#pragma unroll
        for (int c = 0; c < DP; ++c) acc[c] *= corr;
        m = s;
      }
      const float p = expf(s - m);
      l += p;
      const float pd = p * drop.factor(base + j);
      const float* vr = vs + j * sh.S;
#pragma unroll
      for (int c = 0; c < DP; ++c) acc[c] = fmaf(pd, vr[c], acc[c]);
    }
    const float f = qm[i] / l;
    // only thread i ever reads row i of qs: it can take the output without a barrier
#pragma unroll
    for (int c = 0; c < DP; ++c) qs[i * sh.S + c] = acc[c] * f;
    float* st = a.stats + (((uint64_t)b * sh.H + h) * sh.T + i) * 2;
    st[0] = m;
    st[1] = l;
  }
  __syncthreads();
  mha_store(qs, a.out, a.ldo, a.res, a.ldr, b, h, sh);
}

template <int DP>
__global__ void __launch_bounds__(kMhaMaxT) mha_bwd_kernel(const b2ctr_mha_t a) {
  extern __shared__ float sm[];
  const MhaShape sh{a.T, a.heads, a.d, DP + 1};
  const int64_t b = blockIdx.x / sh.H;
  const int h = (int)(blockIdx.x % sh.H);
  float* qs = sm;
  float* ks = qs + sh.T * sh.S;
  float* vs = ks + sh.T * sh.S;
  float* gs = vs + sh.T * sh.S;   // dout
  float* os = gs + sh.T * sh.S;   // output staging
  float* qm = os + sh.T * sh.S;
  float* km = qm + sh.T;
  float* mrow = km + sh.T;
  float* lrow = mrow + sh.T;
  float* drow = lrow + sh.T;      // D_i = sum_j P_ij (dout_i . v_j)
  mha_stage<DP>(a.q, a.ldq, b, h, sh, qs);
  mha_stage<DP>(a.k, a.ldk, b, h, sh, ks);
  mha_stage<DP>(a.v, a.ldv, b, h, sh, vs);
  mha_stage<DP>(a.dout, a.lddo, b, h, sh, gs);
  for (int t = threadIdx.x; t < sh.T; t += blockDim.x) {
    qm[t] = mha_valid(a.qlen, a.qmask, b, t, sh.T) ? 1.f : 0.f;
    km[t] = mha_valid(a.klen, a.kmask, b, t, sh.T) ? 1.f : 0.f;
    const float* st = a.stats + (((uint64_t)b * sh.H + h) * sh.T + t) * 2;
    mrow[t] = st[0];
    lrow[t] = st[1];
  }
  __syncthreads();
  const MhaDrop drop = mha_drop(a);
  const uint64_t head_base = ((uint64_t)h * a.batch + b) * sh.T;
  const int tid = threadIdx.x;

  // ---- dQ: thread i owns query row i ------------------------------------------------------------
  if (tid < sh.T) {
    const int i = tid;
    const uint64_t base = (head_base + i) * sh.T;
    // q_i and dQ_i live in registers; dout_i is read from its (bank-conflict free) shared row, which keeps
    // the DP = 64 instantiation free of spills
    const float* gr = gs + i * sh.S;
    float qr[DP], dq[DP];
#pragma unroll
    for (int c = 0; c < DP; ++c) {
      qr[c] = qs[i * sh.S + c];
      dq[c] = 0.f;
    }
    const float mi = mrow[i], li = lrow[i], qmi = qm[i];
    float D = 0.f;
    for (int j = 0; j < sh.T; ++j) {
      const float s = mha_score<DP>(qr, ks + j * sh.S, a.scale, km[j] != 0.f && !(a.blinding && i == j));
      const float p = expf(s - mi) / li;
      float gv = 0.f;
      const float* vr = vs + j * sh.S;
#pragma unroll
      for (int c = 0; c < DP; ++c) gv = fmaf(gr[c], vr[c], gv);
      D = fmaf(p * qmi * drop.factor(base + j), gv, D);
    }
    for (int j = 0; j < sh.T; ++j) {
      const bool valid = km[j] != 0.f && !(a.blinding && i == j);
      if (!valid) continue;   // the masked scores are constants: no gradient reaches q or k through them
      const float* kr = ks + j * sh.S;
      const float s = mha_score<DP>(qr, kr, a.scale, true);
      const float p = expf(s - mi) / li;
      float gv = 0.f;
      const float* vr = vs + j * sh.S;
#pragma unroll
      for (int c = 0; c < DP; ++c) gv = fmaf(gr[c], vr[c], gv);
      const float ds = p * (gv * qmi * drop.factor(base + j) - D);
#pragma unroll
      for (int c = 0; c < DP; ++c) dq[c] = fmaf(ds, kr[c], dq[c]);
    }
    drow[i] = D;
#pragma unroll
    for (int c = 0; c < DP; ++c) os[i * sh.S + c] = dq[c] * a.scale;
  }
  __syncthreads();
  mha_store(os, a.dq, a.lddq, nullptr, 0, b, h, sh);

  // ---- dV: thread j owns key row j --------------------------------------------------------------
  float kr[DP], acc[DP];
  if (tid < sh.T) {
    const int j = tid;
#pragma unroll
    for (int c = 0; c < DP; ++c) {
      kr[c] = ks[j * sh.S + c];
      acc[c] = 0.f;
    }
    for (int i = 0; i < sh.T; ++i) {
      const float s = mha_score<DP>(qs + i * sh.S, kr, a.scale, km[j] != 0.f && !(a.blinding && i == j));
      const float P = expf(s - mrow[i]) / lrow[i] * qm[i] * drop.factor((head_base + i) * sh.T + j);
      const float* gr = gs + i * sh.S;
#pragma unroll
      for (int c = 0; c < DP; ++c) acc[c] = fmaf(P, gr[c], acc[c]);
    }
  }
  __syncthreads();   // os is free again once every thread has finished storing dQ
  if (tid < sh.T) {
#pragma unroll
    for (int c = 0; c < DP; ++c) os[tid * sh.S + c] = acc[c];
  }
  __syncthreads();
  mha_store(os, a.dv, a.lddv, nullptr, 0, b, h, sh);

  // ---- dK ---------------------------------------------------------------------------------------
  if (tid < sh.T) {
    const int j = tid;
    const float* vr = vs + j * sh.S;
#pragma unroll
    for (int c = 0; c < DP; ++c) acc[c] = 0.f;
    if (km[j] != 0.f) {
      for (int i = 0; i < sh.T; ++i) {
        if (a.blinding && i == j) continue;
        const float* qrow = qs + i * sh.S;
        const float s = mha_score<DP>(qrow, kr, a.scale, true);
        const float p = expf(s - mrow[i]) / lrow[i];
        const float* gr = gs + i * sh.S;
        float gv = 0.f;
#pragma unroll
        for (int c = 0; c < DP; ++c) gv = fmaf(gr[c], vr[c], gv);
        const float ds = p * (gv * qm[i] * drop.factor((head_base + i) * sh.T + j) - drow[i]);
#pragma unroll
        for (int c = 0; c < DP; ++c) acc[c] = fmaf(ds, qrow[c], acc[c]);
      }
    }
  }
  __syncthreads();
  if (tid < sh.T) {
#pragma unroll
    for (int c = 0; c < DP; ++c) os[tid * sh.S + c] = acc[c] * a.scale;
  }
  __syncthreads();
  mha_store(os, a.dk, a.lddk, nullptr, 0, b, h, sh);
}

static size_t mha_smem(int T, int DP, bool bwd) {
  const int S = DP + 1;
  return bwd ? (size_t)(5 * T * S + 5 * T) * sizeof(float) : (size_t)(3 * T * S + 2 * T) * sizeof(float);
}

template <int DP>
static cudaError_t mha_launch(const b2ctr_mha_t& a, bool bwd, cudaStream_t s) {
  const size_t smem = mha_smem(a.T, DP, bwd);
  const int threads = (a.T + 31) / 32 * 32;
  const unsigned grid = (unsigned)(a.batch * a.heads);
  if (bwd) {
    cudaError_t e = cudaFuncSetAttribute(mha_bwd_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    mha_bwd_kernel<DP><<<grid, threads, smem, s>>>(a);
  } else {
    cudaError_t e = cudaFuncSetAttribute(mha_fwd_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    mha_fwd_kernel<DP><<<grid, threads, smem, s>>>(a);
  }
  return cudaGetLastError();
}

static cudaError_t mha_dispatch(const b2ctr_mha_t& a, bool bwd, cudaStream_t s) {
  if (a.d <= 8) return mha_launch<8>(a, bwd, s);
  if (a.d <= 16) return mha_launch<16>(a, bwd, s);
  if (a.d <= 32) return mha_launch<32>(a, bwd, s);
  return mha_launch<64>(a, bwd, s);
}

static bool mha_args_ok(const b2ctr_mha_t* a, bool bwd) {
  if (!a) return false;
  if (a->batch < 0 || a->T < 1 || a->T > kMhaMaxT || a->d < 1 || a->d > kMhaMaxD || a->heads < 1) {
    set_error("mha: need 1 <= T <= %d, 1 <= d <= %d, heads >= 1 (got T=%d, d=%d, heads=%d)", kMhaMaxT, kMhaMaxD,
              a->T, a->d, a->heads);
    return false;
  }
  const int64_t w = (int64_t)a->heads * a->d;
  if (!a->q || !a->k || !a->v || !a->stats || a->ldq < w || a->ldk < w || a->ldv < w) {
    set_error("mha: null operand or row pitch below heads*d = %lld", (long long)w);
    return false;
  }
  if (!(a->dropout_rate >= 0.f && a->dropout_rate < 1.f)) {
    set_error("mha: dropout rate must be in [0, 1)");
    return false;
  }
  if (!bwd && (!a->out || a->ldo < w || (a->res && a->ldr < w))) {
    set_error("mha_fwd: null output or row pitch below heads*d");
    return false;
  }
  if (bwd && (!a->dout || !a->dq || !a->dk || !a->dv || a->lddo < w || a->lddq < w || a->lddk < w || a->lddv < w)) {
    set_error("mha_bwd: null gradient or row pitch below heads*d");
    return false;
  }
  return true;
}

// ---- LayerNormalization ---------------------------------------------------------------------------
// One warp per row, lane l owns columns l, l + 32, ...; the row is re-read from L1 for each pass.
constexpr int kLnWarps = 8;
constexpr int kLnMaxCols = 1024;

__device__ __forceinline__ float ln_x(const float* __restrict__ a, int64_t lda, const float* __restrict__ b,
                                      int64_t ldb, int64_t r, int c) {
  float x = a[r * lda + c];
  if (b) x += b[r * ldb + c];
  return x;
}

__global__ void __launch_bounds__(kLnWarps * 32) layernorm_fwd_kernel(const float* __restrict__ a, int64_t lda,
                                                                     const float* __restrict__ b, int64_t ldb,
                                                                     const float* __restrict__ gamma,
                                                                     const float* __restrict__ beta, float* y,
                                                                     int64_t ldy, float* stats, int64_t rows, int n,
                                                                     float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kLnWarps + (threadIdx.x >> 5);
  if (r >= rows) return;
  float s = 0.f;
  for (int c = lane; c < n; c += 32) s += ln_x(a, lda, b, ldb, r, c);
  const float mean = warp_sum(s) / (float)n;
  float v = 0.f;
  for (int c = lane; c < n; c += 32) {
    const float dlt = ln_x(a, lda, b, ldb, r, c) - mean;
    v = fmaf(dlt, dlt, v);
  }
  const float rstd = 1.f / sqrtf(warp_sum(v) / (float)n + eps);
  for (int c = lane; c < n; c += 32) {
    float o = (ln_x(a, lda, b, ldb, r, c) - mean) * rstd;
    if (gamma) o = __fmul_rn(o, gamma[c]);
    if (beta) o = __fadd_rn(o, beta[c]);
    y[r * ldy + c] = o;
  }
  if (lane == 0) {
    stats[2 * r] = mean;
    stats[2 * r + 1] = rstd;
  }
}

static int ln_bwd_blocks(int64_t rows) {
  const int64_t need = ceil_div(rows, kLnWarps);
  return (int)(need < 2 * kNumSMs ? (need < 1 ? 1 : need) : 2 * kNumSMs);
}

// dx per row; each warp keeps its (dgamma, dbeta) partial for its columns in registers and writes it to
// partial[global warp][0:2n]; the rows a warp visits depend only on (rows, grid), so the sums are reproducible
template <int NK>
__global__ void __launch_bounds__(kLnWarps * 32) layernorm_bwd_kernel(const float* __restrict__ a, int64_t lda,
                                                                     const float* __restrict__ b, int64_t ldb,
                                                                     const float* __restrict__ gamma,
                                                                     const float* __restrict__ stats,
                                                                     const float* __restrict__ dy, int64_t lddy,
                                                                     float* dx, int64_t lddx, float* partial,
                                                                     int64_t rows, int n) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float dg[NK], db[NK];
#pragma unroll
  for (int k = 0; k < NK; ++k) dg[k] = db[k] = 0.f;
  const float inv_n = 1.f / (float)n;
  for (int64_t r = (int64_t)blockIdx.x * kLnWarps + warp; r < rows; r += (int64_t)gridDim.x * kLnWarps) {
    const float mean = stats[2 * r], rstd = stats[2 * r + 1];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int c = lane + 32 * k;
      if (c < n) {
        const float xh = (ln_x(a, lda, b, ldb, r, c) - mean) * rstd;
        const float g = dy[r * lddy + c];
        const float gg = gamma ? g * gamma[c] : g;
        s1 += gg;
        s2 = fmaf(gg, xh, s2);
        dg[k] = fmaf(g, xh, dg[k]);
        db[k] += g;
      }
    }
    s1 = warp_sum(s1) * inv_n;
    s2 = warp_sum(s2) * inv_n;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const int c = lane + 32 * k;
      if (c < n) {
        const float xh = (ln_x(a, lda, b, ldb, r, c) - mean) * rstd;
        const float g = dy[r * lddy + c];
        const float gg = gamma ? g * gamma[c] : g;
        dx[r * lddx + c] = rstd * (gg - s1 - xh * s2);
      }
    }
  }
  float* pw = partial + ((int64_t)blockIdx.x * kLnWarps + warp) * 2 * n;
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    const int c = lane + 32 * k;
    if (c < n) {
      pw[c] = dg[k];
      pw[n + c] = db[k];
    }
  }
}

__global__ void layernorm_wsum_kernel(const float* __restrict__ partial, int nblk, int n, float* dgamma,
                                      float* dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 2 * n) return;
  float s = 0.f;
  for (int k = 0; k < nblk; ++k) s += partial[(int64_t)k * 2 * n + c];
  if (c < n) {
    if (dgamma) dgamma[c] = s;
  } else if (dbeta) {
    dbeta[c - n] = s;
  }
}

template <int NK>
static void ln_bwd_launch(int grid, cudaStream_t s, const float* a, int64_t lda, const float* b, int64_t ldb,
                          const float* gamma, const float* stats, const float* dy, int64_t lddy, float* dx,
                          int64_t lddx, float* partial, int64_t rows, int n) {
  layernorm_bwd_kernel<NK><<<grid, kLnWarps * 32, 0, s>>>(a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial,
                                                          rows, n);
}

}  // namespace b2ctr

using namespace b2ctr;
#define ST ((cudaStream_t)stream)

extern "C" {

b2ctr_status_t b2ctr_mha_fwd(const b2ctr_mha_t* a, void* stream) {
  if (!mha_args_ok(a, false)) return B2CTR_ERR_INVALID_ARG;
  if (a->batch == 0) return B2CTR_OK;
  cudaError_t e = mha_dispatch(*a, false, ST);
  if (e != cudaSuccess) {
    set_error("b2ctr_mha_fwd: %s", cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_mha_bwd(const b2ctr_mha_t* a, void* stream) {
  if (!mha_args_ok(a, true)) return B2CTR_ERR_INVALID_ARG;
  if (a->batch == 0) return B2CTR_OK;
  cudaError_t e = mha_dispatch(*a, true, ST);
  if (e != cudaSuccess) {
    set_error("b2ctr_mha_bwd: %s", cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_layernorm_fwd(const float* a, int64_t lda, const float* b, int64_t ldb, const float* gamma,
                                   const float* beta, float* y, int64_t ldy, float* stats, int64_t rows, int32_t n,
                                   float eps, void* stream) {
  B2_REQUIRE(a && y && stats && rows >= 0 && n >= 1 && n <= kLnMaxCols && lda >= n && ldy >= n &&
                 (!b || ldb >= n),
             "layernorm_fwd: bad arguments (need 1 <= n <= %d, pitches >= n)", kLnMaxCols);
  if (rows == 0) return B2CTR_OK;
  layernorm_fwd_kernel<<<(unsigned)ceil_div(rows, kLnWarps), kLnWarps * 32, 0, ST>>>(a, lda, b, ldb, gamma, beta, y,
                                                                                     ldy, stats, rows, n, eps);
  B2_CHECK_LAUNCH("b2ctr_layernorm_fwd");
  return B2CTR_OK;
}

size_t b2ctr_layernorm_bwd_workspace_bytes(int64_t rows, int32_t n) {
  return (size_t)ln_bwd_blocks(rows) * kLnWarps * 2 * (size_t)(n > 0 ? n : 0) * sizeof(float);
}

b2ctr_status_t b2ctr_layernorm_bwd(const float* a, int64_t lda, const float* b, int64_t ldb, const float* gamma,
                                   const float* stats, const float* dy, int64_t lddy, float* dx, int64_t lddx,
                                   float* dgamma, float* dbeta, int64_t rows, int32_t n, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  B2_REQUIRE(a && stats && dy && dx && rows >= 0 && n >= 1 && n <= kLnMaxCols && lda >= n && lddy >= n &&
                 lddx >= n && (!b || ldb >= n),
             "layernorm_bwd: bad arguments (need 1 <= n <= %d, pitches >= n)", kLnMaxCols);
  const size_t need = b2ctr_layernorm_bwd_workspace_bytes(rows, n);
  if (!workspace || workspace_bytes < need) {
    set_error("layernorm_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int grid = ln_bwd_blocks(rows);
  float* partial = (float*)workspace;
  if (rows == 0) {
    cudaMemsetAsync(partial, 0, need, ST);
  } else {
    const int nk = (n + 31) / 32;
    if (nk <= 1) ln_bwd_launch<1>(grid, ST, a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial, rows, n);
    else if (nk <= 2) ln_bwd_launch<2>(grid, ST, a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial, rows, n);
    else if (nk <= 4) ln_bwd_launch<4>(grid, ST, a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial, rows, n);
    else if (nk <= 8) ln_bwd_launch<8>(grid, ST, a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial, rows, n);
    else if (nk <= 16) ln_bwd_launch<16>(grid, ST, a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial, rows, n);
    else ln_bwd_launch<32>(grid, ST, a, lda, b, ldb, gamma, stats, dy, lddy, dx, lddx, partial, rows, n);
    B2_CHECK_LAUNCH("b2ctr_layernorm_bwd");
  }
  if (dgamma || dbeta) {
    layernorm_wsum_kernel<<<(unsigned)ceil_div(2 * n, 128), 128, 0, ST>>>(partial, grid * kLnWarps, n, dgamma,
                                                                          dbeta);
    B2_CHECK_LAUNCH("b2ctr_layernorm_bwd(sum)");
  }
  return B2CTR_OK;
}

}  // extern "C"
