// interaction.cu — CrossNet, CIN helpers, InteractingLayer attention core (sm_90a).
//
// Reference math restated (never copied): deepctr/layers/interaction.py:410-424 (CrossNet),
// :277-325 (CIN), :754-779 (InteractingLayer), :1113-1126 (SENETLayer), :1190-1209 (BilinearInteraction).  Pairwise reductions use warp shuffles; the dense
// contractions (CIN feature-map contraction, Q/K/V projections, CrossNet-matrix) go through b2ctr_gemm.
#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace b2ctr {

// ------------------------------------------------------------------------------------------------
// elementwise helpers shared by several layers
//   op 0: out = a*b        op 1: out = a*b + c       op 2: out = a + b*s (s scalar broadcast per row)
// ------------------------------------------------------------------------------------------------
__global__ void ewise_kernel(int op, const float* __restrict__ a, const float* __restrict__ b,
                             const float* __restrict__ c, float* out, int64_t n, int acc) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v = op == 0 ? a[i] * b[i] : a[i] * b[i] + c[i];
    out[i] = acc ? out[i] + v : v;
  }
}

// ------------------------------------------------------------------------------------------------
// CrossNet, vector parameterisation: one warp per sample.
//   s_b = <x_l[b], w>;  out[b] = x_0[b] * s_b + bias + x_l[b]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    cross_vector_fwd_kernel(const float* __restrict__ x0, int64_t ld0, const float* __restrict__ xl,
                            int64_t ldl, const float* __restrict__ w, const float* __restrict__ bias,
                            float* out, float* s_out, int64_t batch, int dim) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* p0 = x0 + b * ld0;
    const float* pl = xl + b * ldl;
    float s = 0.f;
    for (int j = lane; j < dim; j += 32) s += pl[j] * w[j];
    s = warp_sum(s);
    for (int j = lane; j < dim; j += 32) out[b * dim + j] = p0[j] * s + bias[j] + pl[j];
    if (lane == 0) s_out[b] = s;
  }
}
// dx0 = dout * s ; dxl = dout + w * ds ; ds_b = <dout[b], x0[b]>   (dw = xl^T ds, db = colsum(dout): GEMM / bias kernels)
__global__ void __launch_bounds__(256)
    cross_vector_bwd_kernel(const float* __restrict__ x0, int64_t ld0, const float* __restrict__ w,
                            const float* __restrict__ dout, const float* __restrict__ s, float* dx0,
                            float* dxl, float* ds_out, int64_t batch, int dim) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* p0 = x0 + b * ld0;
    const float* g = dout + b * dim;
    float ds = 0.f;
    for (int j = lane; j < dim; j += 32) ds += g[j] * p0[j];
    ds = warp_sum(ds);
    const float sb = s[b];
    for (int j = lane; j < dim; j += 32) {
      dx0[b * dim + j] = g[j] * sb;
      dxl[b * dim + j] = g[j] + w[j] * ds;
    }
    if (lane == 0) ds_out[b] = ds;
  }
}

// ------------------------------------------------------------------------------------------------
// CIN.  X0(b,i,d) = x0[b*s0b + i*s0i + d*s0d], Xk likewise.  A batch chunk's outer product
//   Z[(b,d), i*H + j] = X0(b,i,d) * Xk(b,j,d)
// is materialised for a chunk small enough to stay in the 50 MB L2 and contracted with the filter
// by b2ctr_gemm (tensor cores in BF16X3 mode); it never reaches HBM-sized buffers (DESIGN.md 4.3).
// ------------------------------------------------------------------------------------------------
struct CinView {
  const float* p;
  int64_t sb, si, sd;
};
__global__ void __launch_bounds__(256)
    cin_outer_fwd_kernel(CinView x0, CinView xk, float* z, int64_t nb, int m, int h, int d) {
  const int64_t kdim = (int64_t)m * h;
  const int64_t total = nb * d * kdim;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / kdim;
    const int q = (int)(t - row * kdim);
    const int64_t b = row / d;
    const int dd = (int)(row - b * d);
    const int i = q / h, j = q - i * h;
    z[t] = x0.p[b * x0.sb + i * x0.si + dd * x0.sd] * xk.p[b * xk.sb + j * xk.si + dd * xk.sd];
  }
}
// T0[(b,d), i] = X0(b,i,d) (i < m), zero up to ld0: the per-row factor table of the generated outer product
__global__ void __launch_bounds__(256)
    cin_t0_kernel(CinView x0, float* t0, int64_t ld0, int64_t nb, int m, int d) {
  const int64_t total = nb * d * ld0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / ld0;
    const int i = (int)(t - row * ld0);
    const int64_t b = row / d;
    const int dd = (int)(row - b * d);
    t0[t] = i < m ? x0.p[b * x0.sb + i * x0.si + dd * x0.sd] : 0.f;
  }
}
// dX0(b,i,d) (+)= dT0[(b,d), i]: the factor-table gradient back in the caller's [B, m, D] layout
__global__ void __launch_bounds__(256)
    cin_t0_bwd_kernel(const float* __restrict__ dt0, int64_t ld0, float* dx, int64_t gb, int64_t gi, int64_t gd,
                      int acc, int64_t nb, int m, int d) {
  const int64_t total = nb * d * m;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / m;
    const int i = (int)(t - row * m);
    const int64_t b = row / d;
    const int dd = (int)(row - b * d);
    float* o = dx + b * gb + i * gi + dd * gd;
    const float v = dt0[row * ld0 + i];
    *o = acc ? *o + v : v;
  }
}
__global__ void __launch_bounds__(256)
    cin_unpad_rows_kernel(const float* __restrict__ src, float* dst, int m, int h, int hp, int64_t n) {
  const int64_t total = (int64_t)m * h * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / n;
    const int64_t c = t - r * n;
    const int i = (int)(r / h), j = (int)(r - (int64_t)i * h);
    dst[t] = src[((int64_t)i * hp + j) * n + c];
  }
}

// dX0(b,i,d) (+)= sum_j dZ[(b,d),(i,j)] * Xk(b,j,d) ;  dXk(b,j,d) (+)= sum_i dZ[(b,d),(i,j)] * X0(b,i,d)
// one warp per (b,d) row: lanes stride j (coalesced reads of dZ), i walked sequentially.
__global__ void __launch_bounds__(256)
    cin_outer_bwd_kernel(const float* __restrict__ dz, CinView x0, CinView xk, float* dx0, int64_t g0b,
                         int64_t g0i, int64_t g0d, int acc0, float* dxk, int64_t gkb, int64_t gki,
                         int64_t gkd, int acck, int64_t nb, int m, int h, int d, int hp) {
  // dZ rows hold m groups of hp columns, of which the first h are used (hp = h: the dense layout)
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t rows = nb * d;
  const int64_t kdim = (int64_t)m * hp;
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += nw) {
    const int64_t b = row / d;
    const int dd = (int)(row - b * d);
    const float* g = dz + row * kdim;
    // dXk: each lane owns columns j = lane, lane+32, ...
    for (int j0 = 0; j0 < h; j0 += 32) {
      const int j = j0 + lane;
      float a = 0.f;
      if (j < h)
        for (int i = 0; i < m; ++i) a += g[i * hp + j] * x0.p[b * x0.sb + i * x0.si + dd * x0.sd];
      if (j < h && dxk) {
        float* o = dxk + b * gkb + j * gki + dd * gkd;
        *o = acck ? *o + a : a;
      }
    }
    __syncwarp();   // dx0 may alias dxk (layer 0: X_k is X_0): order the two phases within the warp
    if (dx0) {
      for (int i = 0; i < m; ++i) {
        float a = 0.f;
        for (int j = lane; j < h; j += 32) a += g[i * hp + j] * xk.p[b * xk.sb + j * xk.si + dd * xk.sd];
        a = warp_sum(a);
        if (lane == 0) {
          float* o = dx0 + b * g0b + i * g0i + dd * g0d;
          *o = acc0 ? *o + a : a;
        }
      }
    }
  }
}
// out[b, out_col + n] = sum_d y[(b,d), col0 + n]     (reduce_sum over D of the direct maps, :322-323)
__global__ void cin_sum_d_kernel(const float* __restrict__ y, int64_t ldy, int col0, int ncols, int d,
                                 float* out, int64_t ldo, int out_col, int64_t nb) {
  const int64_t total = nb * ncols;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = t / ncols;
    const int n = (int)(t - b * ncols);
    float s = 0.f;
    for (int dd = 0; dd < d; ++dd) s += y[(b * d + dd) * ldy + col0 + n];
    out[b * ldo + out_col + n] = s;
  }
}
// dy[(b,d), n] = (n in [col0, col0+ncols) ? dout[b, out_col + n - col0] : 0) + (dh ? dh[(b,d), n] over [0, hcols) : 0)
__global__ void cin_expand_grad_kernel(const float* __restrict__ dout, int64_t ldo, int out_col, int col0,
                                       int ncols, const float* __restrict__ dh, int64_t ldh, int hcols,
                                       float* dy, int64_t nfilt, int d, int64_t nb) {
  const int64_t total = nb * d * nfilt;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / nfilt;
    const int n = (int)(t - row * nfilt);
    const int64_t b = row / d;
    float v = 0.f;
    if (n >= col0 && n < col0 + ncols) v += dout[b * ldo + out_col + n - col0];
    if (dh && n < hcols) v += dh[row * ldh + n];
    dy[t] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// InteractingLayer attention core: one CTA per sample, thread (head, query-field) pairs.
//   S = Q_h K_h^T [/ sqrt(d)], P = softmax_rows(S), O = P V_h, out = relu(O + res)
// q/k/v/res/out: [B, F, H*D] contiguous.
// ------------------------------------------------------------------------------------------------
constexpr int kIntMaxF = 64;
// F*H*D bound of both entry points: the backward stages K, V, dK and dV (4 F*H*D floats) in 48 KB of shared memory
constexpr int kIntMaxFHD = 48 * 1024 / (4 * (int)sizeof(float));

__global__ void __launch_bounds__(128)
    interacting_fwd_kernel(const float* __restrict__ q, const float* __restrict__ k,
                           const float* __restrict__ v, const float* __restrict__ res, float* out, int F,
                           int H, int D, float scale) {
  extern __shared__ float sm[];
  const int HD = H * D;
  float* sk = sm;
  float* sv = sm + F * HD;
  const int64_t b = blockIdx.x;
  const float* kb = k + b * F * HD;
  const float* vb = v + b * F * HD;
  for (int i = threadIdx.x; i < F * HD; i += blockDim.x) { sk[i] = kb[i]; sv[i] = vb[i]; }
  __syncthreads();
  for (int r = threadIdx.x; r < F * H; r += blockDim.x) {
    const int h = r / F, i = r - h * F;
    const float* qi = q + (b * F + i) * HD + h * D;
    float sc[kIntMaxF];
    float mx = -INFINITY;
    for (int j = 0; j < F; ++j) {
      float s = 0.f;
      for (int e = 0; e < D; ++e) s += qi[e] * sk[j * HD + h * D + e];
      s *= scale;
      sc[j] = s;
      mx = fmaxf(mx, s);
    }
    float den = 0.f;
    for (int j = 0; j < F; ++j) { sc[j] = expf(sc[j] - mx); den += sc[j]; }
    const float inv = 1.f / den;
    for (int e = 0; e < D; ++e) {
      float o = 0.f;
      for (int j = 0; j < F; ++j) o += sc[j] * sv[j * HD + h * D + e];
      o *= inv;
      const int64_t oi = (b * F + i) * HD + h * D + e;
      if (res) o += res[oi];
      out[oi] = o > 0.f ? o : 0.f;
    }
  }
}
__global__ void __launch_bounds__(128)
    interacting_bwd_kernel(const float* __restrict__ q, const float* __restrict__ k,
                           const float* __restrict__ v, const float* __restrict__ out,
                           const float* __restrict__ dout, float* dq, float* dk, float* dv, float* dres,
                           int F, int H, int D, float scale) {
  extern __shared__ float sm[];
  const int HD = H * D;
  float* sk = sm;
  float* sv = sm + F * HD;
  float* sdk = sm + 2 * F * HD;
  float* sdv = sm + 3 * F * HD;
  const int64_t b = blockIdx.x;
  for (int i = threadIdx.x; i < F * HD; i += blockDim.x) {
    sk[i] = k[b * F * HD + i];
    sv[i] = v[b * F * HD + i];
    sdk[i] = 0.f;
    sdv[i] = 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.x; r < F * H; r += blockDim.x) {
    const int h = r / F, i = r - h * F;
    const int64_t base = (b * F + i) * HD + h * D;
    const float* qi = q + base;
    float p[kIntMaxF], dO[32];
    float mx = -INFINITY;
    for (int j = 0; j < F; ++j) {
      float s = 0.f;
      for (int e = 0; e < D; ++e) s += qi[e] * sk[j * HD + h * D + e];
      s *= scale;
      p[j] = s;
      mx = fmaxf(mx, s);
    }
    float den = 0.f;
    for (int j = 0; j < F; ++j) { p[j] = expf(p[j] - mx); den += p[j]; }
    const float inv = 1.f / den;
    for (int e = 0; e < D; ++e) {
      const float g = out[base + e] > 0.f ? dout[base + e] : 0.f;   // relu'
      dO[e] = g;
      if (dres) dres[base + e] = g;
    }
    // dP_j = <dO, V_j>;  dS_j = P_j (dP_j - sum_k P_k dP_k)
    float dot = 0.f;
    float dp[kIntMaxF];
    for (int j = 0; j < F; ++j) {
      p[j] *= inv;
      float a = 0.f;
      for (int e = 0; e < D; ++e) a += dO[e] * sv[j * HD + h * D + e];
      dp[j] = a;
      dot += p[j] * a;
    }
    float dqi[32];
    for (int e = 0; e < D; ++e) dqi[e] = 0.f;
    for (int j = 0; j < F; ++j) {
      const float ds = p[j] * (dp[j] - dot) * scale;
      for (int e = 0; e < D; ++e) {
        dqi[e] += ds * sk[j * HD + h * D + e];
        atomicAdd(&sdk[j * HD + h * D + e], ds * qi[e]);
        atomicAdd(&sdv[j * HD + h * D + e], p[j] * dO[e]);
      }
    }
    for (int e = 0; e < D; ++e) dq[base + e] = dqi[e];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < F * HD; i += blockDim.x) {
    dk[b * F * HD + i] = sdk[i];
    dv[b * F * HD + i] = sdv[i];
  }
}

// ------------------------------------------------------------------------------------------------
// BiInteractionPooling (deepctr/layers/interaction.py:196-201): one warp per sample, lanes over e.
//   out[b, e] = 0.5 * ((sum_f x)^2 - sum_f x^2);   dx[b, f, e] = g[b, e] * (S[b, e] - x[b, f, e])
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    bi_interaction_fwd_kernel(const float* __restrict__ x, int64_t ldx, int nfield, int dim, float* out,
                              int64_t ldo, int64_t batch) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* xr = x + b * ldx;
    for (int e = lane; e < dim; e += 32) {
      float s = 0.f, q = 0.f;
      for (int f = 0; f < nfield; ++f) {
        const float v = xr[f * dim + e];
        s += v;
        q += v * v;
      }
      out[b * ldo + e] = 0.5f * (s * s - q);
    }
  }
}
__global__ void __launch_bounds__(256)
    bi_interaction_bwd_kernel(const float* __restrict__ x, int64_t ldx, int nfield, int dim,
                              const float* __restrict__ g, int64_t ldg, float* dx, int64_t lddx, int64_t batch) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* xr = x + b * ldx;
    float* dr = dx + b * lddx;
    for (int e = lane; e < dim; e += 32) {
      const float ge = g[b * ldg + e];
      float s = 0.f;
      for (int f = 0; f < nfield; ++f) s += xr[f * dim + e];
      for (int f = 0; f < nfield; ++f) dr[f * dim + e] = ge * (s - xr[f * dim + e]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// AFMLayer attention pooling (deepctr/layers/interaction.py:122-141), the pairwise products generated on
// chip.  For the P = F(F-1)/2 pairs p = (i < j) of a sample, in itertools.combinations order:
//   prod_p = x_i * x_j  [E];  s_p = h . relu(W^T prod_p + bias);  alpha = softmax_p(s);  att = sum_p alpha_p prod_p
// One warp per sample, one lane per pair (lanes stride the pair list), the sample's [F, E] rows staged in
// shared memory with a padded pitch.  Neither prod [B,P,E] nor the hidden layer [B,P,A] ever exists.
// E and A are padded to the template sizes EP (4/8/16/32) and AP (1/2/4/8/16) with zero weights: a padded
// column of x / row of W / entry of bias and h contributes exactly 0 to every sum.
// Forward: online softmax per lane, merged across the warp; the per-sample state (max, sum) is saved.
// Backward: with sum_q alpha_q d alpha_q = <g, att>, ds_p = alpha_p (<g, prod_p> - <g, att>) needs one pass.
//   Lanes handle 32 pairs per round and park (prod, d prod, d t, ds*hidden) of the round in shared memory;
//   every output element then has ONE owner lane that adds the round's terms in a fixed order: dx[f, e] the
//   lane (e, f mod 32/EP), dW[e, a] the lane (e*AP + a) mod 32, dbias / dh lane a.  Per-CTA weight partials
//   are summed in a fixed order by afm_reduce_kernel: no float atomics, bit-identical from run to run.
// ------------------------------------------------------------------------------------------------
constexpr int kAfmWarps = 4;
constexpr int kAfmMaxF = 64;
constexpr int kAfmMaxE = 32;
constexpr int kAfmMaxA = 16;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// shared header of both AFM kernels: zero-padded W^T [AP][EP] (16-byte rows: float4 broadcast reads), bias [AP],
// h [AP] and the pair list (i << 8 | j)
template <int EP, int AP>
__device__ __forceinline__ int afm_load_header(float* sm, const float* __restrict__ W, const float* __restrict__ bias,
                                               const float* __restrict__ h, int F, int E, int A) {
  float* sW = sm;
  float* sb = sW + EP * AP;
  float* sh = sb + AP;
  int* spair = (int*)(sh + AP);
  for (int k = threadIdx.x; k < EP * AP; k += blockDim.x) {
    const int a = k / EP, e = k - a * EP;
    sW[k] = (e < E && a < A) ? W[e * A + a] : 0.f;
  }
  for (int a = threadIdx.x; a < AP; a += blockDim.x) {
    sb[a] = a < A ? bias[a] : 0.f;
    sh[a] = a < A ? h[a] : 0.f;
  }
  const int P = F * (F - 1) / 2;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    int i = 0, off = 0;
    while (off + (F - 1 - i) <= p) { off += F - 1 - i; ++i; }
    spair[p] = (i << 8) | (i + 1 + p - off);
  }
  return P;
}
template <int EP, int AP>
__host__ __device__ constexpr int afm_header_floats() { return EP * AP + 2 * AP + kAfmMaxF * (kAfmMaxF - 1) / 2; }

// <prod, W[:, a]> over the padded embedding axis (the a-loops stay rolled: unrolled, ptxas keeps all of W^T in
// registers and spills)
template <int EP>
__device__ __forceinline__ float afm_dot(const float (&pr)[EP], const float* __restrict__ wa) {
  float t = 0.f;
#pragma unroll
  for (int e = 0; e < EP; e += 4) {
    const float4 w = *reinterpret_cast<const float4*>(wa + e);
    t = fmaf(pr[e], w.x, t);
    t = fmaf(pr[e + 1], w.y, t);
    t = fmaf(pr[e + 2], w.z, t);
    t = fmaf(pr[e + 3], w.w, t);
  }
  return t;
}

// [F, E] rows of sample b -> padded [F, EP + 1] tile (columns >= E stay zero from the initial fill)
template <int EP>
__device__ __forceinline__ void afm_stage_x(float* sx, const float* __restrict__ xr, int F, int E, int lane) {
  constexpr int XP = EP + 1;
  for (int k = lane; k < F * E; k += 32) {
    const int f = k / E;
    sx[f * XP + (k - f * E)] = xr[k];
  }
}

template <int EP, int AP>
__global__ void __launch_bounds__(kAfmWarps * 32)
    afm_fwd_kernel(const float* __restrict__ x, int64_t ldx, int F, int E, int A, const float* __restrict__ W,
                   const float* __restrict__ bias, const float* __restrict__ h, float* att, int64_t ldo,
                   float* state, int64_t batch) {
  constexpr int XP = EP + 1;
  extern __shared__ float sm[];
  const int P = afm_load_header<EP, AP>(sm, W, bias, h, F, E, A);
  const float* sW = sm;
  const float* sb = sW + EP * AP;
  const float* sh = sb + AP;
  const int* spair = (const int*)(sh + AP);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sx = sm + afm_header_floats<EP, AP>() + warp * F * XP;
  for (int k = lane; k < F * XP; k += 32) sx[k] = 0.f;
  __syncthreads();
  const int64_t nw = (int64_t)gridDim.x * kAfmWarps;
  for (int64_t b = (int64_t)blockIdx.x * kAfmWarps + warp; b < batch; b += nw) {
    afm_stage_x<EP>(sx, x + b * ldx, F, E, lane);
    __syncwarp();
    float m = -INFINITY, l = 0.f, acc[EP];
#pragma unroll
    for (int e = 0; e < EP; ++e) acc[e] = 0.f;
    for (int p = lane; p < P; p += 32) {
      const int ij = spair[p];
      const float* xi = sx + (ij >> 8) * XP;
      const float* xj = sx + (ij & 255) * XP;
      float pr[EP];
#pragma unroll
      for (int e = 0; e < EP; ++e) pr[e] = xi[e] * xj[e];
      float s = 0.f;
#pragma unroll 1
      for (int a = 0; a < AP; ++a) {
        const float t = afm_dot<EP>(pr, sW + a * EP) + sb[a];
        s = fmaf(sh[a], fmaxf(t, 0.f), s);
      }
      if (s > m) {
        const float c = expf(m - s);     // m = -inf on the first pair: c = 0, acc and l are 0 anyway
        l *= c;
#pragma unroll
        for (int e = 0; e < EP; ++e) acc[e] *= c;
        m = s;
      }
      const float w = expf(s - m);
      l += w;
#pragma unroll
      for (int e = 0; e < EP; ++e) acc[e] = fmaf(w, pr[e], acc[e]);
    }
    const float M = warp_max(m);
    const float c = m == -INFINITY ? 0.f : expf(m - M);   // lanes without a pair (P < 32) contribute nothing
    const float L = warp_sum(l * c);
    const float inv = 1.f / L;
    float* o = att + b * ldo;
#pragma unroll
    for (int e = 0; e < EP; ++e) {
      const float v = warp_sum(acc[e] * c);
      if (lane == e && e < E) o[e] = v * inv;
    }
    if (lane == 0) {
      state[2 * b] = M;
      state[2 * b + 1] = L;
    }
    __syncwarp();   // sx is restaged for the next sample
  }
}

template <int EP, int AP>
__host__ __device__ constexpr int afm_bwd_warp_floats(int F) {
  return 2 * F * (EP + 1) + 2 * 32 * (EP + 1) + 2 * 32 * (AP + 1) + (EP + 1);
}

template <int EP, int AP>
__global__ void __launch_bounds__(kAfmWarps * 32)
    afm_bwd_kernel(const float* __restrict__ x, int64_t ldx, int F, int E, int A, const float* __restrict__ W,
                   const float* __restrict__ bias, const float* __restrict__ h, const float* __restrict__ g,
                   int64_t ldg, const float* __restrict__ att, int64_t lda, const float* __restrict__ state,
                   float* dx, int64_t lddx, float* partial, int64_t batch) {
  constexpr int XP = EP + 1;
  constexpr int RP = AP + 1;                           // odd pitch: lane-indexed rows hit distinct banks
  constexpr int NW = EP * AP + 2 * AP;                 // per-CTA partial: dW (padded), dbias, dh
  constexpr int R = (EP * AP + 31) / 32;               // dW entries owned per lane
  constexpr int G = 32 / EP;                           // lanes sharing one column e in the dx fold
  extern __shared__ float sm[];
  const int P = afm_load_header<EP, AP>(sm, W, bias, h, F, E, A);
  const float* sW = sm;
  const float* sb = sW + EP * AP;
  const float* sh = sb + AP;
  const int* spair = (const int*)(sh + AP);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sx = sm + afm_header_floats<EP, AP>() + warp * afm_bwd_warp_floats<EP, AP>(F);
  float* sdx = sx + F * XP;
  float* rp = sdx + F * XP;      // [32][XP] prod of the round's pairs
  float* rd = rp + 32 * XP;      // [32][XP] d prod
  float* rt = rd + 32 * XP;      // [32][RP] d t (pre-relu hidden)
  float* rh = rt + 32 * RP;      // [32][RP] ds * hidden
  float* sg = rh + 32 * RP;      // [XP] incoming gradient of the sample
  for (int k = lane; k < F * XP; k += 32) sx[k] = 0.f;
  for (int k = lane; k < XP; k += 32) sg[k] = 0.f;
  __syncthreads();
  const int ecol = lane % EP, grp = lane / EP;
  float accW[R];
#pragma unroll
  for (int r = 0; r < R; ++r) accW[r] = 0.f;
  float accB = 0.f, accH = 0.f;
  const int64_t nw = (int64_t)gridDim.x * kAfmWarps;
  for (int64_t b = (int64_t)blockIdx.x * kAfmWarps + warp; b < batch; b += nw) {
    afm_stage_x<EP>(sx, x + b * ldx, F, E, lane);
    for (int k = lane; k < F * XP; k += 32) sdx[k] = 0.f;
    float gatt = 0.f;
    if (lane < E) {
      const float ge = g[b * ldg + lane];
      sg[lane] = ge;
      gatt = ge * att[b * lda + lane];
    }
    gatt = warp_sum(gatt);
    const float M = state[2 * b], invL = 1.f / state[2 * b + 1];
    __syncwarp();
    for (int base = 0; base < P; base += 32) {
      const int p = base + lane;
      float pr[EP], dpr[EP];
      float* tl = rt + lane * RP;
      float* hl = rh + lane * RP;
      if (p < P) {
        const int ij = spair[p];
        const float* xi = sx + (ij >> 8) * XP;
        const float* xj = sx + (ij & 255) * XP;
#pragma unroll
        for (int e = 0; e < EP; ++e) pr[e] = xi[e] * xj[e];
        float s = 0.f, gp = 0.f;
#pragma unroll 1
        for (int a = 0; a < AP; ++a) {
          const float t = afm_dot<EP>(pr, sW + a * EP) + sb[a];
          tl[a] = t;                       // pre-activation, turned into its gradient below
          s = fmaf(sh[a], fmaxf(t, 0.f), s);
        }
#pragma unroll
        for (int e = 0; e < EP; ++e) gp = fmaf(sg[e], pr[e], gp);
        const float alpha = expf(s - M) * invL;
        const float ds = alpha * (gp - gatt);
#pragma unroll
        for (int e = 0; e < EP; ++e) dpr[e] = alpha * sg[e];
#pragma unroll 1
        for (int a = 0; a < AP; ++a) {
          const float t = tl[a];
          const float d = t > 0.f ? ds * sh[a] : 0.f;
          hl[a] = ds * fmaxf(t, 0.f);
          tl[a] = d;
          const float* wa = sW + a * EP;
#pragma unroll
          for (int e = 0; e < EP; e += 4) {
            const float4 w = *reinterpret_cast<const float4*>(wa + e);
            dpr[e] = fmaf(w.x, d, dpr[e]);
            dpr[e + 1] = fmaf(w.y, d, dpr[e + 1]);
            dpr[e + 2] = fmaf(w.z, d, dpr[e + 2]);
            dpr[e + 3] = fmaf(w.w, d, dpr[e + 3]);
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < EP; ++e) pr[e] = dpr[e] = 0.f;
        for (int a = 0; a < AP; ++a) tl[a] = hl[a] = 0.f;
      }
#pragma unroll
      for (int e = 0; e < EP; ++e) {
        rp[lane * XP + e] = pr[e];
        rd[lane * XP + e] = dpr[e];
      }
      __syncwarp();
      const int nq = min(32, P - base);
      for (int q = 0; q < nq; ++q) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int k = lane + 32 * r;
          if (k < EP * AP) accW[r] = fmaf(rp[q * XP + k / AP], rt[q * RP + k % AP], accW[r]);
        }
        if (lane < AP) {
          accB += rt[q * RP + lane];
          accH += rh[q * RP + lane];
        }
        const int ij = spair[base + q];
        const int i = ij >> 8, j = ij & 255;
        const float d = rd[q * XP + ecol];
        if (i % G == grp) sdx[i * XP + ecol] = fmaf(d, sx[j * XP + ecol], sdx[i * XP + ecol]);
        if (j % G == grp) sdx[j * XP + ecol] = fmaf(d, sx[i * XP + ecol], sdx[j * XP + ecol]);
      }
      __syncwarp();
    }
    float* dr = dx + b * lddx;
    for (int k = lane; k < F * E; k += 32) {
      const int f = k / E;
      dr[k] = sdx[f * XP + (k - f * E)];
    }
    __syncwarp();
  }
  // CTA partial: warps in a fixed order
  float* wp = sx + 2 * F * XP;   // this warp's rp region (>= NW floats)
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int k = lane + 32 * r;
    if (k < EP * AP) wp[k] = accW[r];
  }
  if (lane < AP) {
    wp[EP * AP + lane] = accB;
    wp[EP * AP + AP + lane] = accH;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < NW; k += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < kAfmWarps; ++w)
      s += (sm + afm_header_floats<EP, AP>() + w * afm_bwd_warp_floats<EP, AP>(F) + 2 * F * XP)[k];
    partial[(int64_t)blockIdx.x * NW + k] = s;
  }
}

// dW[e, a], dbias[a], dh[a] = sum over the CTA partials in ascending CTA order
__global__ void afm_reduce_kernel(const float* __restrict__ partial, int nblocks, int EP, int AP, int E, int A,
                                  float* dW, float* dbias, float* dh) {
  const int NW = EP * AP + 2 * AP;
  const int n = E * A + 2 * A;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    int src;
    float* dst;
    if (t < E * A) {
      const int e = t / A, a = t - e * A;
      src = e * AP + a;
      dst = dW + t;
    } else if (t < E * A + A) {
      src = EP * AP + (t - E * A);
      dst = dbias + (t - E * A);
    } else {
      src = EP * AP + AP + (t - E * A - A);
      dst = dh + (t - E * A - A);
    }
    float s = 0.f;
    for (int c = 0; c < nblocks; ++c) s += partial[(int64_t)c * NW + src];
    *dst = s;
  }
}

static inline int afm_pad_e(int E) { return E <= 4 ? 4 : E <= 8 ? 8 : E <= 16 ? 16 : 32; }
static inline int afm_pad_a(int A) { return A <= 1 ? 1 : A <= 2 ? 2 : A <= 4 ? 4 : A <= 8 ? 8 : 16; }
static inline int afm_bwd_blocks(int64_t batch) { return grid_for(batch, kAfmWarps, 4); }
static inline size_t afm_fwd_smem(int EP, int AP, int F) {
  return sizeof(float) * ((size_t)EP * AP + 2 * AP + kAfmMaxF * (kAfmMaxF - 1) / 2 + (size_t)kAfmWarps * F * (EP + 1));
}
static inline size_t afm_bwd_smem(int EP, int AP, int F) {
  const size_t warp = 2 * (size_t)F * (EP + 1) + 2 * 32 * (EP + 1) + 2 * 32 * (AP + 1) + (EP + 1);
  return sizeof(float) * ((size_t)EP * AP + 2 * AP + kAfmMaxF * (kAfmMaxF - 1) / 2 + kAfmWarps * warp);
}

// host-side launch of one (EP, AP) instantiation; afm_dispatch picks it at run time
struct AfmArgs {
  const float* x; int64_t ldx; int F, E, A;
  const float *W, *bias, *h;
  const float* g; int64_t ldg;
  float* att; int64_t lda;       // forward: output; backward: input
  float* state;                  // forward: output; backward: input
  float* dx; int64_t lddx;
  float* partial;
  int64_t batch;
};
struct AfmFwd {
  template <int EP, int AP>
  static cudaError_t run(const AfmArgs& a, cudaStream_t s) {
    const size_t smem = afm_fwd_smem(EP, AP, a.F);
    cudaError_t e = cudaFuncSetAttribute(afm_fwd_kernel<EP, AP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return e;
    afm_fwd_kernel<EP, AP><<<grid_for(a.batch, kAfmWarps, 8), kAfmWarps * 32, smem, s>>>(
        a.x, a.ldx, a.F, a.E, a.A, a.W, a.bias, a.h, a.att, a.lda, a.state, a.batch);
    return cudaSuccess;
  }
};
struct AfmBwd {
  template <int EP, int AP>
  static cudaError_t run(const AfmArgs& a, cudaStream_t s) {
    const size_t smem = afm_bwd_smem(EP, AP, a.F);
    cudaError_t e = cudaFuncSetAttribute(afm_bwd_kernel<EP, AP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return e;
    afm_bwd_kernel<EP, AP><<<afm_bwd_blocks(a.batch), kAfmWarps * 32, smem, s>>>(
        a.x, a.ldx, a.F, a.E, a.A, a.W, a.bias, a.h, a.g, a.ldg, a.att, a.lda, a.state, a.dx, a.lddx, a.partial,
        a.batch);
    return cudaSuccess;
  }
};
template <class Op, int EP>
cudaError_t afm_dispatch_a(int AP, const AfmArgs& a, cudaStream_t s) {
  switch (AP) {
    case 1: return Op::template run<EP, 1>(a, s);
    case 2: return Op::template run<EP, 2>(a, s);
    case 4: return Op::template run<EP, 4>(a, s);
    case 8: return Op::template run<EP, 8>(a, s);
    default: return Op::template run<EP, 16>(a, s);
  }
}
template <class Op>
cudaError_t afm_dispatch(int EP, int AP, const AfmArgs& a, cudaStream_t s) {
  switch (EP) {
    case 4: return afm_dispatch_a<Op, 4>(AP, a, s);
    case 8: return afm_dispatch_a<Op, 8>(AP, a, s);
    case 16: return afm_dispatch_a<Op, 16>(AP, a, s);
    default: return afm_dispatch_a<Op, 32>(AP, a, s);
  }
}

// ------------------------------------------------------------------------------------------------
// SENETLayer (deepctr/layers/interaction.py:1113-1126): one warp per sample, x [F, E] read in place.
//   Z = mean_e x;  A1 = relu(Z W1) [R];  A2 = relu(A1 W2) [F];  V = x * A2[:, None]
// Backward, with d2 = relu'(A2) . <dV_f, x_f>,  d1 = relu'(A1) . (W2 d2),  dZ = W1 d1:
//   dx = dV * A2 + dZ / E;   dW1 = Z^T d1,  dW2 = A1^T d2   (relu' is 0 at 0, as in TF)
// The weight gradients are summed per CTA in shared memory: the warps of a CTA take samples in lockstep rounds,
// park (Z, A1, d1, d2) of their sample, and every entry of dW1 / dW2 has ONE owner thread that adds the round's
// samples in warp order.  senet_reduce_kernel then sums the CTA partials in CTA order: bit-identical runs.
// ------------------------------------------------------------------------------------------------
constexpr int kSenetWarps = 8;
constexpr int kSenetMaxF = 64;
constexpr int kSenetVec = 6 * kSenetMaxF;     // per-warp vectors: z, a1, a2, d1, d2, dz

__global__ void __launch_bounds__(kSenetWarps * 32)
    senet_fwd_kernel(const float* __restrict__ x, int64_t ldx, int F, int E, int R, const float* __restrict__ W1,
                     const float* __restrict__ W2, float* v, int64_t ldv, float* saved, int64_t batch) {
  __shared__ float sm[kSenetWarps * kSenetVec];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sz = sm + warp * kSenetVec;
  float* sa1 = sz + kSenetMaxF;
  float* sa2 = sa1 + kSenetMaxF;
  const float inv_e = 1.f / (float)E;
  const int64_t nw = (int64_t)gridDim.x * kSenetWarps;
  for (int64_t b = (int64_t)blockIdx.x * kSenetWarps + warp; b < batch; b += nw) {
    const float* xr = x + b * ldx;
    for (int f = 0; f < F; ++f) {
      float s = 0.f;
      for (int e = lane; e < E; e += 32) s += xr[f * E + e];
      s = warp_sum(s);
      if (lane == 0) sz[f] = s * inv_e;
    }
    __syncwarp();
    float* sv = saved + b * (R + F);
    for (int r = lane; r < R; r += 32) {
      float t = 0.f;
      for (int f = 0; f < F; ++f) t = fmaf(sz[f], W1[f * R + r], t);
      t = fmaxf(t, 0.f);
      sa1[r] = t;
      sv[r] = t;
    }
    __syncwarp();
    for (int f = lane; f < F; f += 32) {
      float t = 0.f;
      for (int r = 0; r < R; ++r) t = fmaf(sa1[r], W2[r * F + f], t);
      t = fmaxf(t, 0.f);
      sa2[f] = t;
      sv[R + f] = t;
    }
    __syncwarp();
    float* vr = v + b * ldv;
    for (int k = lane; k < F * E; k += 32) vr[k] = xr[k] * sa2[k / E];
    __syncwarp();   // the vectors are rewritten for the next sample
  }
}

__global__ void __launch_bounds__(kSenetWarps * 32)
    senet_bwd_kernel(const float* __restrict__ g, int64_t ldg, const float* __restrict__ x, int64_t ldx, int F, int E,
                     int R, const float* __restrict__ W1, const float* __restrict__ W2,
                     const float* __restrict__ saved, float* dx, int64_t lddx, float* partial, int64_t batch) {
  __shared__ float sm[kSenetWarps * kSenetVec + 2 * kSenetMaxF * kSenetMaxF];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sz = sm + warp * kSenetVec;
  float* sa1 = sz + kSenetMaxF;
  float* sa2 = sa1 + kSenetMaxF;
  float* sd1 = sa2 + kSenetMaxF;
  float* sd2 = sd1 + kSenetMaxF;
  float* sdz = sd2 + kSenetMaxF;
  float* acc = sm + kSenetWarps * kSenetVec;     // [F*R] dW1, then [R*F] dW2; entry k owned by thread k % blockDim
  const int nacc = 2 * F * R;
  for (int k = threadIdx.x; k < nacc; k += blockDim.x) acc[k] = 0.f;
  const float inv_e = 1.f / (float)E;
  const int64_t step = (int64_t)gridDim.x * kSenetWarps;
  for (int64_t b0 = (int64_t)blockIdx.x * kSenetWarps; b0 < batch; b0 += step) {
    const int64_t b = b0 + warp;
    if (b < batch) {
      const float* xr = x + b * ldx;
      const float* gr = g + b * ldg;
      const float* sv = saved + b * (R + F);
      for (int f = 0; f < F; ++f) {
        float s = 0.f, d = 0.f;
        for (int e = lane; e < E; e += 32) {
          const float xv = xr[f * E + e];
          s += xv;
          d = fmaf(gr[f * E + e], xv, d);
        }
        s = warp_sum(s);
        d = warp_sum(d);
        if (lane == 0) {
          const float a2 = sv[R + f];
          sz[f] = s * inv_e;
          sa2[f] = a2;
          sd2[f] = a2 > 0.f ? d : 0.f;
        }
      }
      __syncwarp();
      for (int r = lane; r < R; r += 32) {
        float t = 0.f;
        for (int f = 0; f < F; ++f) t = fmaf(sd2[f], W2[r * F + f], t);
        const float a1 = sv[r];
        sa1[r] = a1;
        sd1[r] = a1 > 0.f ? t : 0.f;
      }
      __syncwarp();
      for (int f = lane; f < F; f += 32) {
        float t = 0.f;
        for (int r = 0; r < R; ++r) t = fmaf(sd1[r], W1[f * R + r], t);
        sdz[f] = t * inv_e;
      }
      __syncwarp();
      float* dr = dx + b * lddx;
      for (int k = lane; k < F * E; k += 32) {
        const int f = k / E;
        dr[k] = fmaf(gr[k], sa2[f], sdz[f]);
      }
    } else {
      for (int k = lane; k < kSenetMaxF; k += 32) sz[k] = sa1[k] = sd1[k] = sd2[k] = 0.f;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < nacc; k += blockDim.x) {
      float a = acc[k];
      if (k < F * R) {
        const int f = k / R, r = k - f * R;
        for (int w = 0; w < kSenetWarps; ++w) a = fmaf(sm[w * kSenetVec + f], sm[w * kSenetVec + 3 * kSenetMaxF + r], a);
      } else {
        const int q = k - F * R, r = q / F, f = q - r * F;
        for (int w = 0; w < kSenetWarps; ++w)
          a = fmaf(sm[w * kSenetVec + kSenetMaxF + r], sm[w * kSenetVec + 4 * kSenetMaxF + f], a);
      }
      acc[k] = a;
    }
    __syncthreads();
  }
  for (int k = threadIdx.x; k < nacc; k += blockDim.x) partial[(int64_t)blockIdx.x * nacc + k] = acc[k];
}

// out[k] = sum over the n CTA partials (pitch `pitch`) in ascending order
__global__ void ordered_sum_kernel(const float* __restrict__ partial, int64_t pitch, int n, int64_t count, float* out) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < n; ++c) s += partial[(int64_t)c * pitch + k];
    out[k] = s;
  }
}

static inline int senet_bwd_blocks(int64_t batch) { return grid_for(batch, kSenetWarps, 4); }

// ------------------------------------------------------------------------------------------------
// BilinearInteraction (deepctr/layers/interaction.py:1190-1209).  For the P = F(F-1)/2 pairs p = (i < j) in
// itertools.combinations order, with W_k(p) one of the stacked [E, E] weights (k = 0 'all', i 'each', p
// 'interaction'):
//   out_p = (x_i W_k) * x_j  [E]
// written to out[b*ldo + col0 + p*pitch + o]: a window of a wider buffer (the DNN input) is written in place.
// Backward from g_p (same addressing):
//   dx_i += W_k (g_p * x_j),   dx_j += g_p * (x_i W_k),   dW_k += x_i^T (g_p * x_j)
// Every kernel is a register-tiled [TS, EP] x [EP, EP] product on shared-memory tiles: 256 threads, each owning
// 4 samples x 4 columns, E padded with zeros to EP in {4, 8, 16, 32, 64} (TS = 4096 / EP samples per tile).
// * bilinear_fwd_kernel: CTA (pair, sample tile).  The pair index runs fastest so the CTAs that share a
//   sample tile find it in L2.
// * bilinear_dx_kernel: CTA (field, sample tile); the field's F-1 pairs are added in ascending partner order
//   into registers: one owner per (b, f, e), no atomics.
// * bilinear_dw_kernel: CTA (pair, batch chunk) -> partial[chunk][pair][E][E]; bilinear_dw_reduce_kernel adds,
//   for each weight, its pairs in ascending order and each pair's chunks in ascending order.
// ------------------------------------------------------------------------------------------------
constexpr int kBiThreads = 256;
constexpr int kBiMaxF = 64;
constexpr int kBiMaxE = 64;
constexpr int kBiDwSub = 64;      // samples staged per round of bilinear_dw_kernel

__host__ __device__ __forceinline__ int bi_pair_index(int F, int i, int j) { return i * (2 * F - i - 1) / 2 + (j - i - 1); }
__host__ __device__ __forceinline__ int bi_weight_index(int type, int i, int p) { return type == 0 ? 0 : type == 1 ? i : p; }
__device__ __forceinline__ void bi_pair_of(int F, int p, int& i, int& j) {
  int off = 0;
  i = 0;
  while (off + (F - 1 - i) <= p) { off += F - 1 - i; ++i; }
  j = i + 1 + p - off;
}

// M[r][c] = W[r][c] (or W[c][r] when trans) for a matrix of row stride ld, zero outside [E, E]
template <int EP>
__device__ __forceinline__ void bi_stage_w(float* M, const float* __restrict__ W, int E, bool trans, int64_t ld) {
  for (int k = threadIdx.x; k < EP * EP; k += blockDim.x) {
    const int r = k / EP, c = k - r * EP;
    M[k] = (r < E && c < E) ? (trans ? W[c * ld + r] : W[r * ld + c]) : 0.f;
  }
}
template <int EP>
__device__ __forceinline__ void bi_stage_w(float* M, const float* __restrict__ W, int E, bool trans) {
  bi_stage_w<EP>(M, W, E, trans, (int64_t)E);
}

// acc[r][c] += sum_k AT[k][s0 + r] * M[k][o0 + c]
template <int EP>
__device__ __forceinline__ void bi_tile_mm(const float* AT, int apitch, const float* M, int s0, int o0,
                                           float (&acc)[4][4]) {
#pragma unroll 4
  for (int k = 0; k < EP; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(AT + k * apitch + s0);
    const float4 m = *reinterpret_cast<const float4*>(M + k * EP + o0);
    const float av[4] = {a.x, a.y, a.z, a.w}, mv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(av[r], mv[c], acc[r][c]);
  }
}

template <int EP>
__host__ __device__ constexpr int bi_ts() { return 4096 / EP; }
template <int EP>
__host__ __device__ constexpr int bi_apitch() { return bi_ts<EP>() + 4; }
template <int EP>
__host__ __device__ constexpr int bi_smem_floats() { return EP * bi_apitch<EP>() + EP * EP; }

struct BiArgs {
  const float* x; int64_t ldx;
  int F, E, type;
  const float* W;
  float* out; int64_t ldo, col0, pitch;      // forward output / backward gradient window
  float* dx; int64_t lddx;
  float* partial; int nchunk;
  int64_t batch;
};

template <int EP>
__global__ void __launch_bounds__(kBiThreads) bilinear_fwd_kernel(const BiArgs a) {
  constexpr int TS = bi_ts<EP>(), AP = bi_apitch<EP>(), NOG = EP / 4;
  extern __shared__ __align__(16) float sm[];
  float* AT = sm;
  float* M = sm + EP * AP;
  const int F = a.F, E = a.E, p = blockIdx.x;
  int i, j;
  bi_pair_of(F, p, i, j);
  bi_stage_w<EP>(M, a.W + (int64_t)bi_weight_index(a.type, i, p) * E * E, E, false);
  const int o0 = (threadIdx.x % NOG) * 4, s0 = (threadIdx.x / NOG) * 4;
  const int64_t ntiles = (a.batch + TS - 1) / TS;
  for (int64_t t = blockIdx.y; t < ntiles; t += gridDim.y) {
    const int64_t b0 = t * TS;
    const int ns = (int)min((int64_t)TS, a.batch - b0);
    for (int k = threadIdx.x; k < TS * EP; k += blockDim.x) {
      const int s = k / EP, e = k - s * EP;
      AT[e * AP + s] = (s < ns && e < E) ? a.x[(b0 + s) * a.ldx + i * E + e] : 0.f;
    }
    __syncthreads();
    float acc[4][4] = {};
    bi_tile_mm<EP>(AT, AP, M, s0, o0, acc);
    if (o0 < E) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (s0 + r >= ns) break;
        const int64_t b = b0 + s0 + r;
        const float* xj = a.x + b * a.ldx + j * E + o0;
        float* o = a.out + b * a.ldo + a.col0 + (int64_t)p * a.pitch + o0;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (o0 + c < E) o[c] = acc[r][c] * xj[c];
      }
    }
    __syncthreads();   // AT is restaged for the next tile
  }
}

template <int EP>
__global__ void __launch_bounds__(kBiThreads) bilinear_dx_kernel(const BiArgs a) {
  constexpr int TS = bi_ts<EP>(), AP = bi_apitch<EP>(), NOG = EP / 4;
  extern __shared__ __align__(16) float sm[];
  float* AT = sm;
  float* M = sm + EP * AP;
  const int F = a.F, E = a.E, f = blockIdx.x;
  const int o0 = (threadIdx.x % NOG) * 4, s0 = (threadIdx.x / NOG) * 4;
  const int64_t ntiles = (a.batch + TS - 1) / TS;
  for (int64_t t = blockIdx.y; t < ntiles; t += gridDim.y) {
    const int64_t b0 = t * TS;
    const int ns = (int)min((int64_t)TS, a.batch - b0);
    float dacc[4][4] = {};
    for (int q = 0; q < F; ++q) {
      if (q == f) continue;
      const bool second = q < f;            // pair (q, f): f is the second field
      const int i = second ? q : f, j = second ? f : q;
      const int p = bi_pair_index(F, i, j);
      bi_stage_w<EP>(M, a.W + (int64_t)bi_weight_index(a.type, i, p) * E * E, E, !second);
      for (int k = threadIdx.x; k < TS * EP; k += blockDim.x) {
        const int s = k / EP, e = k - s * EP;
        float v = 0.f;
        if (s < ns && e < E) {
          const int64_t b = b0 + s;
          v = a.x[b * a.ldx + q * E + e];
          if (!second) v *= a.out[b * a.ldo + a.col0 + (int64_t)p * a.pitch + e];
        }
        AT[e * AP + s] = v;
      }
      __syncthreads();
      float acc[4][4] = {};
      bi_tile_mm<EP>(AT, AP, M, s0, o0, acc);
      if (second) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          if (s0 + r >= ns) break;
          const float* gp = a.out + (b0 + s0 + r) * a.ldo + a.col0 + (int64_t)p * a.pitch + o0;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (o0 + c < E) dacc[r][c] = fmaf(gp[c], acc[r][c], dacc[r][c]);
        }
      } else {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) dacc[r][c] += acc[r][c];
      }
      __syncthreads();   // AT and M are restaged for the next partner
    }
    if (o0 < E) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (s0 + r >= ns) break;
        float* d = a.dx + (b0 + s0 + r) * a.lddx + f * E + o0;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (o0 + c < E) d[c] = dacc[r][c];
      }
    }
  }
}

template <int EP>
__host__ __device__ constexpr int bi_dw_smem_floats() {
  return 2 * kBiDwSub * EP > (kBiThreads / ((EP / 4) * (EP / 4))) * EP * EP ? 2 * kBiDwSub * EP
                                                                          : (kBiThreads / ((EP / 4) * (EP / 4))) * EP * EP;
}

// kPairScalar: the gradient is one scalar per (sample, pair) at out[b*ldo + col0 + p] (FEFM, b2ctr_fefm_bwd)
// instead of an [E] vector per pair
template <int EP, bool kPairScalar = false>
__global__ void __launch_bounds__(kBiThreads) bilinear_dw_kernel(const BiArgs a) {
  constexpr int NOG = EP / 4, NT = NOG * NOG, G = kBiThreads / NT;
  extern __shared__ __align__(16) float sm[];
  float* XS = sm;                          // [kBiDwSub][EP]: x_i
  float* TT = sm + kBiDwSub * EP;          // [kBiDwSub][EP]: g_p * x_j
  const int F = a.F, E = a.E, p = blockIdx.x, c = blockIdx.y;
  int i, j;
  bi_pair_of(F, p, i, j);
  const int tl = threadIdx.x % NT, grp = threadIdx.x / NT;
  const int e0 = (tl / NOG) * 4, o0 = (tl % NOG) * 4;
  const int64_t per = (a.batch + a.nchunk - 1) / a.nchunk;
  const int64_t lo = (int64_t)c * per, hi = min(a.batch, lo + per);
  float acc[4][4] = {};
  for (int64_t b0 = lo; b0 < hi; b0 += kBiDwSub) {
    const int ns = (int)min((int64_t)kBiDwSub, hi - b0);
    for (int k = threadIdx.x; k < kBiDwSub * EP; k += blockDim.x) {
      const int s = k / EP, e = k - s * EP;
      float xv = 0.f, tv = 0.f;
      if (s < ns && e < E) {
        const int64_t b = b0 + s;
        xv = a.x[b * a.ldx + i * E + e];
        tv = a.out[b * a.ldo + a.col0 + (kPairScalar ? (int64_t)p : (int64_t)p * a.pitch + e)] *
             a.x[b * a.ldx + j * E + e];
      }
      XS[k] = xv;
      TT[k] = tv;
    }
    __syncthreads();
    for (int s = grp; s < ns; s += G) {
      const float4 xv = *reinterpret_cast<const float4*>(XS + s * EP + e0);
      const float4 tv = *reinterpret_cast<const float4*>(TT + s * EP + o0);
      const float av[4] = {xv.x, xv.y, xv.z, xv.w}, mv[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[r][q] = fmaf(av[r], mv[q], acc[r][q]);
    }
    __syncthreads();
  }
  // sample groups in a fixed order
  float* red = sm;                         // [G][EP*EP]
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) red[grp * EP * EP + (e0 + r) * EP + o0 + q] = acc[r][q];
  __syncthreads();
  float* dst = a.partial + ((int64_t)c * (F * (F - 1) / 2) + p) * E * E;
  for (int k = threadIdx.x; k < E * E; k += blockDim.x) {
    const int e = k / E, o = k - e * E;
    float s = 0.f;
    for (int g = 0; g < G; ++g) s += red[g * EP * EP + e * EP + o];
    dst[k] = s;
  }
}

// dW[k][e][o] = sum over the pairs of weight k (ascending) of the sum over their chunk partials (ascending)
__global__ void bilinear_dw_reduce_kernel(const float* __restrict__ partial, int F, int E, int type, int nchunk,
                                          float* dW, int64_t count) {
  const int P = F * (F - 1) / 2;
  const int ee = E * E;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(t / ee), q = (int)(t - (int64_t)k * ee);
    const int plo = type == 0 ? 0 : type == 1 ? bi_pair_index(F, k, k + 1) : k;
    const int phi = type == 0 ? P : type == 1 ? bi_pair_index(F, k, F - 1) + 1 : k + 1;
    float s = 0.f;
    for (int p = plo; p < phi; ++p)
      for (int c = 0; c < nchunk; ++c) s += partial[((int64_t)c * P + p) * ee + q];
    dW[t] = s;
  }
}

static inline int bi_pad_e(int E) { return E <= 4 ? 4 : E <= 8 ? 8 : E <= 16 ? 16 : E <= 32 ? 32 : 64; }
static inline int bi_num_weights(int type, int F) { return type == 0 ? 1 : type == 1 ? F - 1 : F * (F - 1) / 2; }
// batch chunks of the weight-gradient pass: about 8 CTAs per SM over all pairs, at least 64 samples a chunk
static inline int bi_dw_chunks(int F, int64_t batch) {
  const int64_t P = (int64_t)F * (F - 1) / 2;
  const int64_t want = ceil_div((int64_t)kNumSMs * 8, P);
  const int64_t most = ceil_div(batch, kBiDwSub);
  return (int)std::max<int64_t>(1, std::min(want, most));
}
static inline unsigned bi_tile_grid(int64_t batch, int TS) { return (unsigned)std::min<int64_t>(ceil_div(batch, TS), 65535); }

struct BiFwd {
  template <int EP>
  static cudaError_t run(const BiArgs& a, cudaStream_t s) {
    const size_t smem = sizeof(float) * bi_smem_floats<EP>();
    const dim3 grid(a.F * (a.F - 1) / 2, bi_tile_grid(a.batch, bi_ts<EP>()));
    bilinear_fwd_kernel<EP><<<grid, kBiThreads, smem, s>>>(a);
    return cudaSuccess;
  }
};
struct BiBwd {
  template <int EP>
  static cudaError_t run(const BiArgs& a, cudaStream_t s) {
    if (a.dx) {
      const size_t smem = sizeof(float) * bi_smem_floats<EP>();
      bilinear_dx_kernel<EP><<<dim3(a.F, bi_tile_grid(a.batch, bi_ts<EP>())), kBiThreads, smem, s>>>(a);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return e;
    }
    if (a.partial) {
      const size_t smem = sizeof(float) * bi_dw_smem_floats<EP>();   // <= 32 KB for every EP
      bilinear_dw_kernel<EP><<<dim3(a.F * (a.F - 1) / 2, a.nchunk), kBiThreads, smem, s>>>(a);
    }
    return cudaSuccess;
  }
};
template <class Op>
cudaError_t bi_dispatch(int EP, const BiArgs& a, cudaStream_t s) {
  switch (EP) {
    case 4: return Op::template run<4>(a, s);
    case 8: return Op::template run<8>(a, s);
    case 16: return Op::template run<16>(a, s);
    case 32: return Op::template run<32>(a, s);
    default: return Op::template run<64>(a, s);
  }
}

// ------------------------------------------------------------------------------------------------
// FwFMLayer (deepctr/layers/interaction.py:1395-1411): out[b] = sum_{i<j} r[i][j] <x_i, x_j>, upper triangle of the
// [F, F] strengths only.  One warp per sample, the sample's [F, E] staged in shared memory (row pitch E+1); lane e
// computes, for 4 first fields i0..i0+3 at a time, y_k = sum_j rt[j][i0+k] x_j[e] from one float4 of the
// transposed, zero-padded strengths rt [F][FQ] (rt[j][i] = r[i][j] for i < j, else 0), then adds x_{i0+k}[e] y_k.
// Backward from g [B, 1]:
//   dx_i = g * sum_{j != i} r[min(i,j)][max(i,j)] x_j   (same loop on the symmetric rt, partners ascending)
//   dR[i][j] = sum_b g_b <x_i, x_j> for i < j, 0 elsewhere.
// The CTA's warps take samples in lockstep rounds; every upper-triangle entry of dR has ONE owner thread that adds
// the round's samples in warp order into a per-CTA accumulator, written as a partial and summed over the CTAs in
// CTA order by fwfm_dr_reduce_kernel.  No atomics: bit-identical runs.
// ------------------------------------------------------------------------------------------------
constexpr int kFwWarps = 8;
constexpr int kFwMaxF = 64;
constexpr int kFwMaxE = 64;

__host__ __device__ __forceinline__ int fw_fq(int F) { return (F + 3) & ~3; }
static inline size_t fw_fwd_smem(int F, int E) {
  return sizeof(float) * ((size_t)F * fw_fq(F) + (size_t)kFwWarps * F * (E + 1));
}
static inline size_t fw_bwd_smem(int F, int E) {
  return fw_fwd_smem(F, E) + sizeof(float) * (kFwWarps + 2 * (size_t)(F * (F - 1) / 2));
}
static inline int fw_bwd_blocks(int64_t batch) { return grid_for(batch, kFwWarps, 4); }

// rt[j][i] = r[i][j] where i < j (sym: also r[j][i]'s mirror where i > j), 0 elsewhere and in the padding
__device__ __forceinline__ void fw_stage_r(float* rt, const float* __restrict__ r, int F, bool sym) {
  const int FQ = fw_fq(F);
  for (int k = threadIdx.x; k < F * FQ; k += blockDim.x) {
    const int j = k / FQ, i = k - j * FQ;
    rt[k] = (i < j) ? r[i * F + j] : (sym && i > j && i < F) ? r[j * F + i] : 0.f;
  }
}

// y[k] = sum_{j in [j0, F)} rt[j][i0+k] * sx[j][e]
__device__ __forceinline__ void fw_rows4(const float* rt, const float* sx, int F, int XP, int i0, int j0, int e,
                                         float (&y)[4]) {
  const int FQ = fw_fq(F);
  y[0] = y[1] = y[2] = y[3] = 0.f;
  for (int j = j0; j < F; ++j) {
    const float xj = sx[j * XP + e];
    const float4 rr = *reinterpret_cast<const float4*>(rt + j * FQ + i0);
    y[0] = fmaf(rr.x, xj, y[0]);
    y[1] = fmaf(rr.y, xj, y[1]);
    y[2] = fmaf(rr.z, xj, y[2]);
    y[3] = fmaf(rr.w, xj, y[3]);
  }
}

__device__ __forceinline__ void fw_stage_x(float* sx, const float* __restrict__ xr, int F, int E, int lane) {
  const int XP = E + 1;
  for (int k = lane; k < F * E; k += 32) {
    const int f = k / E;
    sx[f * XP + (k - f * E)] = xr[k];
  }
}

__global__ void __launch_bounds__(kFwWarps * 32)
    fwfm_fwd_kernel(const float* __restrict__ x, int64_t ldx, int F, int E, const float* __restrict__ r, float* out,
                    int64_t ldo, int64_t batch) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, XP = E + 1;
  float* rt = sm;
  float* sx = sm + F * fw_fq(F) + warp * F * XP;
  fw_stage_r(rt, r, F, false);
  __syncthreads();
  const int64_t nw = (int64_t)gridDim.x * kFwWarps;
  for (int64_t b = (int64_t)blockIdx.x * kFwWarps + warp; b < batch; b += nw) {
    fw_stage_x(sx, x + b * ldx, F, E, lane);
    __syncwarp();
    float acc = 0.f;
    for (int e = lane; e < E; e += 32) {
      for (int i0 = 0; i0 < F - 1; i0 += 4) {
        float y[4];
        fw_rows4(rt, sx, F, XP, i0, i0 + 1, e, y);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (i0 + k < F) acc = fmaf(sx[(i0 + k) * XP + e], y[k], acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) out[b * ldo] = acc;
    __syncwarp();   // sx is restaged for the next sample
  }
}

__global__ void __launch_bounds__(kFwWarps * 32)
    fwfm_bwd_kernel(const float* __restrict__ g, int64_t ldg, const float* __restrict__ x, int64_t ldx, int F, int E,
                    const float* __restrict__ r, float* dx, int64_t lddx, float* partial, int64_t batch) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, XP = E + 1;
  const int P = F * (F - 1) / 2;
  float* rt = sm;                                          // symmetric strengths [F][FQ]
  float* sxs = sm + F * fw_fq(F);                          // kFwWarps x [F][XP]
  float* sg = sxs + kFwWarps * F * XP;                     // [kFwWarps]: g of the round's samples
  float* acc = sg + kFwWarps;                              // [P]: this CTA's dR, entry k owned by thread k % blockDim
  int* pairs = reinterpret_cast<int*>(acc + P);            // [P]: (i << 8) | j
  float* sx = sxs + warp * F * XP;
  fw_stage_r(rt, r, F, true);
  for (int i = 0, k = 0; i < F; ++i)
    for (int j = i + 1; j < F; ++j, ++k)
      if (k % blockDim.x == threadIdx.x) {
        pairs[k] = (i << 8) | j;
        acc[k] = 0.f;
      }
  __syncthreads();
  const int64_t step = (int64_t)gridDim.x * kFwWarps;
  for (int64_t b0 = (int64_t)blockIdx.x * kFwWarps; b0 < batch; b0 += step) {
    const int64_t b = b0 + warp;
    if (b < batch) {
      fw_stage_x(sx, x + b * ldx, F, E, lane);
      const float gb = g[b * ldg];
      if (lane == 0) sg[warp] = gb;
      __syncwarp();
      if (dx) {
        float* dr = dx + b * lddx;
        for (int e = lane; e < E; e += 32) {
          for (int i0 = 0; i0 < F; i0 += 4) {
            float y[4];
            fw_rows4(rt, sx, F, XP, i0, 0, e, y);
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (i0 + k < F) dr[(i0 + k) * E + e] = gb * y[k];
          }
        }
      }
    }
    if (!partial) {
      __syncwarp();
      continue;
    }
    __syncthreads();
    const int nvalid = (int)min((int64_t)kFwWarps, batch - b0);
    for (int k = threadIdx.x; k < P; k += blockDim.x) {
      const int i = pairs[k] >> 8, j = pairs[k] & 255;
      float a = acc[k];
      for (int w = 0; w < nvalid; ++w) {
        const float* xi = sxs + w * F * XP + i * XP;
        const float* xj = sxs + w * F * XP + j * XP;
        float d = 0.f;
        for (int e = 0; e < E; ++e) d = fmaf(xi[e], xj[e], d);
        a = fmaf(sg[w], d, a);
      }
      acc[k] = a;
    }
    __syncthreads();   // the round's samples are restaged
  }
  if (partial)
    for (int k = threadIdx.x; k < P; k += blockDim.x) partial[(int64_t)blockIdx.x * P + k] = acc[k];
}

// dR[i][j] = sum over the n CTA partials (ascending) of entry p(i, j) for i < j; 0 on and below the diagonal
__global__ void fwfm_dr_reduce_kernel(const float* __restrict__ partial, int n, int F, float* dR) {
  const int P = F * (F - 1) / 2;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < F * F; t += gridDim.x * blockDim.x) {
    const int i = t / F, j = t - i * F;
    float s = 0.f;
    if (i < j) {
      const int p = bi_pair_index(F, i, j);
      for (int c = 0; c < n; ++c) s += partial[(int64_t)c * P + p];
    }
    dR[t] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// FEFMLayer (deepctr/layers/interaction.py:1478-1491).  With S_p = W_p + W_p^T (fefm_sym_kernel, once per step)
// for the P pairs p = (i < j) in itertools.combinations order:
//   out[b*ldo + col0 + p] = x_i S_p x_j^T
// Backward from g[b*ldg + gcol0 + p], read in place:
//   dx_f = sum_{q != f} g_p(f,q) x_q S_p      (S_p symmetric: the same form for either field of the pair)
//   dS_p = sum_b g_p x_i^T x_j,   dW_p = dS_p + dS_p^T
// The products are the register-tiled [TS, EP] x [EP, EP] shared-memory tiles of the bilinear kernels above.
// * fefm_fwd_kernel: CTA (first field i, sample tile).  x_i's tile is staged once; for every partner j > i the CTA
//   stages S_p, forms the [TS, E] product and dots each row with x_j in the epilogue (a reduction over the EP/4
//   threads of a row): no [B, E] intermediate reaches memory.  The field index runs fastest so the CTAs that
//   share a sample tile find its x_j rows in L2.
// * fefm_dx_kernel: CTA (field, sample tile); the rows of x_q are scaled by g_p as they are staged and the F-1
//   partners are accumulated into the same registers in ascending order: one owner per (b, f, e), no atomics.
// * dS: bilinear_dw_kernel<EP, true> partials per (pair, batch chunk); fefm_dw_reduce_kernel adds the chunks in
//   ascending order, for both dS_p and its transpose.
// kPnn: OutterProductLayer(kernel_type='mat') (deepctr/layers/interaction.py:881-911) on the same tiles.  Its score
// is out_p = sum_{k,l} x_j[k] K[k][p][l] x_i[l] = x_i M_p x_j^T with M_p[l][k] = K[k][p][l], not symmetric: M_p is
// staged transposed straight from the reference's [E, P, E] kernel (row stride P*E), and the dx kernel stages
// M_p^T for the first field of a pair (dx_i = g x_j M_p^T) and M_p for the second (dx_j = g x_i M_p).
// ------------------------------------------------------------------------------------------------
constexpr int kFeMaxF = 64;
constexpr int kFeMaxE = 64;

// M = M_p (FEFM: S_p, [P][E][E]; kPnn: K[:, p, :]^T, or K[:, p, :] when trans)
template <int EP, bool kPnn>
__device__ __forceinline__ void fe_stage_m(float* M, const float* __restrict__ W, int F, int E, int p, bool trans) {
  if (kPnn)
    bi_stage_w<EP>(M, W + (int64_t)p * E, E, !trans, (int64_t)(F * (F - 1) / 2) * E);
  else
    bi_stage_w<EP>(M, W + (int64_t)p * E * E, E, false);
}

__global__ void fefm_sym_kernel(const float* __restrict__ W, int E, float* S, int64_t count) {
  const int ee = E * E;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = t / ee;
    const int q = (int)(t - p * ee), r = q / E, c = q - r * E;
    S[t] = W[t] + W[p * ee + c * E + r];
  }
}

template <int EP, bool kPnn = false>
__global__ void __launch_bounds__(kBiThreads) fefm_fwd_kernel(const BiArgs a) {
  constexpr int TS = bi_ts<EP>(), AP = bi_apitch<EP>(), NOG = EP / 4;
  extern __shared__ __align__(16) float sm[];
  float* AT = sm;
  float* M = sm + EP * AP;
  const int F = a.F, E = a.E, i = blockIdx.x;
  const int o0 = (threadIdx.x % NOG) * 4, s0 = (threadIdx.x / NOG) * 4;
  const int64_t ntiles = (a.batch + TS - 1) / TS;
  for (int64_t t = blockIdx.y; t < ntiles; t += gridDim.y) {
    const int64_t b0 = t * TS;
    const int ns = (int)min((int64_t)TS, a.batch - b0);
    for (int k = threadIdx.x; k < TS * EP; k += blockDim.x) {
      const int s = k / EP, e = k - s * EP;
      AT[e * AP + s] = (s < ns && e < E) ? a.x[(b0 + s) * a.ldx + i * E + e] : 0.f;
    }
    for (int j = i + 1; j < F; ++j) {
      const int p = bi_pair_index(F, i, j);
      fe_stage_m<EP, kPnn>(M, a.W, F, E, p, false);
      __syncthreads();
      float acc[4][4] = {};
      bi_tile_mm<EP>(AT, AP, M, s0, o0, acc);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const bool live = s0 + r < ns;
        float v = 0.f;
        if (live) {
          const float* xj = a.x + (b0 + s0 + r) * a.ldx + j * E + o0;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (o0 + c < E) v = fmaf(acc[r][c], xj[c], v);
        }
#pragma unroll
        for (int off = NOG / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (live && o0 == 0) a.out[(b0 + s0 + r) * a.ldo + a.col0 + p] = v;
      }
      __syncthreads();   // M is restaged for the next partner, AT for the next tile
    }
  }
}

template <int EP, bool kPnn = false>
__global__ void __launch_bounds__(kBiThreads) fefm_dx_kernel(const BiArgs a) {
  constexpr int TS = bi_ts<EP>(), AP = bi_apitch<EP>(), NOG = EP / 4;
  extern __shared__ __align__(16) float sm[];
  float* AT = sm;
  float* M = sm + EP * AP;
  const int F = a.F, E = a.E, f = blockIdx.x;
  const int o0 = (threadIdx.x % NOG) * 4, s0 = (threadIdx.x / NOG) * 4;
  const int64_t ntiles = (a.batch + TS - 1) / TS;
  for (int64_t t = blockIdx.y; t < ntiles; t += gridDim.y) {
    const int64_t b0 = t * TS;
    const int ns = (int)min((int64_t)TS, a.batch - b0);
    float acc[4][4] = {};
    for (int q = 0; q < F; ++q) {
      if (q == f) continue;
      const int p = q < f ? bi_pair_index(F, q, f) : bi_pair_index(F, f, q);
      fe_stage_m<EP, kPnn>(M, a.W, F, E, p, q > f);
      for (int k = threadIdx.x; k < TS * EP; k += blockDim.x) {
        const int s = k / EP, e = k - s * EP;
        float v = 0.f;
        if (s < ns && e < E) {
          const int64_t b = b0 + s;
          v = a.out[b * a.ldo + a.col0 + p] * a.x[b * a.ldx + q * E + e];
        }
        AT[e * AP + s] = v;
      }
      __syncthreads();
      bi_tile_mm<EP>(AT, AP, M, s0, o0, acc);
      __syncthreads();   // AT and M are restaged for the next partner
    }
    if (o0 < E) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (s0 + r >= ns) break;
        float* d = a.dx + (b0 + s0 + r) * a.lddx + f * E + o0;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (o0 + c < E) d[c] = acc[r][c];
      }
    }
  }
}

// dW[p][e][o] = sum_c partial[c][p][e][o] + sum_c partial[c][p][o][e], chunks ascending
__global__ void fefm_dw_reduce_kernel(const float* __restrict__ partial, int P, int E, int nchunk, float* dW,
                                      int64_t count) {
  const int ee = E * E;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(t / ee), q = (int)(t - (int64_t)p * ee), e = q / E, o = q - e * E;
    float s = 0.f, st = 0.f;
    for (int c = 0; c < nchunk; ++c) {
      const float* part = partial + ((int64_t)c * P + p) * ee;
      s += part[e * E + o];
      st += part[o * E + e];
    }
    dW[t] = s + st;
  }
}

// pnn mat: dK[k][p][l] = sum_c partial[c][p][l][k] (bilinear_dw_kernel's x_i^T (g_p x_j)), chunks ascending; no
// transposed second term as FEFM has
__global__ void pnn_mat_dk_reduce_kernel(const float* __restrict__ partial, int P, int E, int nchunk, float* dK,
                                         int64_t count) {
  const int ee = E * E, pe = P * E;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(t / pe), q = (int)(t - (int64_t)k * pe), p = q / E, l = q - p * E;
    float s = 0.f;
    for (int c = 0; c < nchunk; ++c) s += partial[((int64_t)c * P + p) * ee + l * E + k];
    dK[t] = s;
  }
}

template <bool kPnn>
struct FeFwd {
  template <int EP>
  static cudaError_t run(const BiArgs& a, cudaStream_t s) {
    const size_t smem = sizeof(float) * bi_smem_floats<EP>();
    fefm_fwd_kernel<EP, kPnn><<<dim3(a.F - 1, bi_tile_grid(a.batch, bi_ts<EP>())), kBiThreads, smem, s>>>(a);
    return cudaSuccess;
  }
};
template <bool kPnn>
struct FeBwd {
  template <int EP>
  static cudaError_t run(const BiArgs& a, cudaStream_t s) {
    if (a.dx) {
      const size_t smem = sizeof(float) * bi_smem_floats<EP>();
      fefm_dx_kernel<EP, kPnn><<<dim3(a.F, bi_tile_grid(a.batch, bi_ts<EP>())), kBiThreads, smem, s>>>(a);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return e;
    }
    if (a.partial) {
      const size_t smem = sizeof(float) * bi_dw_smem_floats<EP>();
      bilinear_dw_kernel<EP, true><<<dim3(a.F * (a.F - 1) / 2, a.nchunk), kBiThreads, smem, s>>>(a);
    }
    return cudaSuccess;
  }
};

// ------------------------------------------------------------------------------------------------
// PNN's InnerProductLayer (deepctr/layers/interaction.py:655-678) and OutterProductLayer(kernel_type 'vec' / 'num')
// (:912-919).  For the P pairs p = (i < j) in itertools.combinations order, on x [B, F, E] read in place:
//   B2CTR_PNN_INNER        out[b*ldo + col0 + p]         = <x_i, x_j>
//   B2CTR_PNN_ELEMENTWISE  out[b*ldo + col0 + p*E + e]   = x_i[e] x_j[e]          (reduce_sum=False)
//   B2CTR_PNN_VEC          out[b*ldo + col0 + p]         = sum_e x_i[e] x_j[e] K[p][e]
//   B2CTR_PNN_NUM          out[b*ldo + col0 + p]         = K[p] <x_i, x_j>
// Both kernels are instantiated per mode.
// * pnn_inner_fwd_kernel: one warp per sample, its [F, E] staged in shared memory (row pitch E+1, so the lanes'
//   consecutive partners j hit distinct banks while the shared x_i is a broadcast); lane p owns pair p (or, for
//   the elementwise form, the flattened (p, e)) and writes it, so the row is stored coalesced.  'vec' stages K
//   once per CTA (pitch E+1) when it fits (kPnStageKMax).
// * pnn_inner_dx_kernel: one warp per sample, sample and pair gradient staged; lane (f, e) adds its F-1 partners
//   in ascending order, the pair index stepped rather than recomputed: dx_f[e] = sum_{q != f} g_p w_p[e] x_q[e].
//   One owner per element, no atomics.
// * pnn_inner_dk_kernel (vec / num): CTA (tile of kPnDkPer * 256 kernel entries, batch chunk); each thread keeps
//   its entries' sums over the chunk in registers and writes them as a partial, and ordered_sum_kernel adds the
//   chunks in ascending order.  Bit-identical from run to run.
// ------------------------------------------------------------------------------------------------
constexpr int kPnWarps = 8;
constexpr int kPnMaxF = 64;
constexpr int kPnMaxE = 64;
constexpr int kPnDkPer = 8;

// 'vec' forward: the kernel K [P, E] is staged once per CTA in shared memory (row pitch E+1: lane p reads row p
// conflict-free) when it takes at most this many floats; larger kernels are read through L1
constexpr int kPnStageKMax = 16384;

static inline bool pn_stage_k(int F, int E, int mode) {
  return mode == B2CTR_PNN_VEC && (int64_t)F * (F - 1) / 2 * (E + 1) <= kPnStageKMax;
}
static inline size_t pn_fwd_smem(int F, int E, int mode) {
  const size_t P = (size_t)F * (F - 1) / 2;
  return sizeof(int) * P + sizeof(float) * ((pn_stage_k(F, E, mode) ? P * (E + 1) : 0) +
                                            (size_t)kPnWarps * F * (E + 1));
}
static inline size_t pn_dx_smem(int F, int E) {
  return sizeof(float) * (size_t)kPnWarps * (F * (E + 1) + F * (F - 1) / 2);
}

// pairs[p] = (i << 8) | j, for the CTA
__device__ __forceinline__ void pn_stage_pairs(int* pairs, int F) {
  for (int i = 0, k = 0; i < F; ++i)
    for (int j = i + 1; j < F; ++j, ++k)
      if (k % blockDim.x == threadIdx.x) pairs[k] = (i << 8) | j;
}

template <int kMode>
__global__ void __launch_bounds__(kPnWarps * 32)
    pnn_inner_fwd_kernel(const float* __restrict__ x, int64_t ldx, int F, int E, const float* __restrict__ K,
                         bool stage_k, float* out, int64_t ldo, int64_t col0, int64_t batch) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, XP = E + 1, P = F * (F - 1) / 2;
  int* pairs = reinterpret_cast<int*>(sm);
  float* sk = sm + P;                                          // [P][XP] when stage_k
  float* sx = sk + (stage_k ? P * XP : 0) + warp * F * XP;
  pn_stage_pairs(pairs, F);
  if (kMode == B2CTR_PNN_VEC && stage_k)
    for (int k = threadIdx.x; k < P * E; k += blockDim.x) {
      const int p = k / E;
      sk[p * XP + (k - p * E)] = K[k];
    }
  __syncthreads();
  const int64_t nw = (int64_t)gridDim.x * kPnWarps;
  for (int64_t b = (int64_t)blockIdx.x * kPnWarps + warp; b < batch; b += nw) {
    fw_stage_x(sx, x + b * ldx, F, E, lane);
    __syncwarp();
    float* o = out + b * ldo + col0;
    if (kMode == B2CTR_PNN_ELEMENTWISE) {
      for (int k = lane; k < P * E; k += 32) {
        const int p = k / E, e = k - p * E, i = pairs[p] >> 8, j = pairs[p] & 255;
        o[k] = sx[i * XP + e] * sx[j * XP + e];
      }
    } else {
      for (int p = lane; p < P; p += 32) {
        const float* xi = sx + (pairs[p] >> 8) * XP;
        const float* xj = sx + (pairs[p] & 255) * XP;
        float acc = 0.f;
        if (kMode == B2CTR_PNN_VEC) {
          if (stage_k) {
            const float* kp = sk + p * XP;
            for (int e = 0; e < E; ++e) acc = fmaf(xi[e] * xj[e], kp[e], acc);
          } else {
            const float* kp = K + (int64_t)p * E;
            for (int e = 0; e < E; ++e) acc = fmaf(xi[e] * xj[e], __ldg(kp + e), acc);
          }
        } else {
          for (int e = 0; e < E; ++e) acc = fmaf(xi[e], xj[e], acc);
          if (kMode == B2CTR_PNN_NUM) acc *= __ldg(K + p);
        }
        o[p] = acc;
      }
    }
    __syncwarp();   // sx is restaged for the next sample
  }
}

// w_p[e] * x_q[e] for pair p, partner q
template <int kMode>
__device__ __forceinline__ float pn_dx_term(const float* gb, const float* sg, const float* __restrict__ K,
                                            const float* sx, int XP, int E, int p, int q, int e, float acc) {
  float w;
  if (kMode == B2CTR_PNN_ELEMENTWISE)
    w = gb[(int64_t)p * E + e];
  else if (kMode == B2CTR_PNN_VEC)
    w = sg[p] * __ldg(K + (int64_t)p * E + e);
  else
    w = sg[p];
  return fmaf(w, sx[q * XP + e], acc);
}

// launch bounds with a minimum of 4 CTAs per SM: without it ptxas spills the 'vec' instantiation
template <int kMode>
__global__ void __launch_bounds__(kPnWarps * 32, 4)
    pnn_inner_dx_kernel(const float* __restrict__ g, int64_t ldg, int64_t gcol0, const float* __restrict__ x,
                        int64_t ldx, int F, int E, const float* __restrict__ K, float* dx, int64_t lddx,
                        int64_t batch) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, XP = E + 1, P = F * (F - 1) / 2;
  float* sx = sm + warp * (F * XP + P);
  float* sg = sx + F * XP;                                     // [P]: g_p (times K[p] for num)
  const int64_t nw = (int64_t)gridDim.x * kPnWarps;
  for (int64_t b = (int64_t)blockIdx.x * kPnWarps + warp; b < batch; b += nw) {
    fw_stage_x(sx, x + b * ldx, F, E, lane);
    const float* gb = g + b * ldg + gcol0;
    if (kMode != B2CTR_PNN_ELEMENTWISE)
      for (int p = lane; p < P; p += 32) sg[p] = kMode == B2CTR_PNN_NUM ? gb[p] * __ldg(K + p) : gb[p];
    __syncwarp();
    float* d = dx + b * lddx;
    for (int k = lane; k < F * E; k += 32) {
      const int f = k / E, e = k - f * E;
      float acc = 0.f;
      // partners ascending: q < f in pairs (q, f), p(q+1, f) = p(q, f) + F - q - 2; then q > f in pairs (f, q),
      // consecutive from p(f, f+1)
      int p = f - 1;
      for (int q = 0; q < f; ++q) {
        acc = pn_dx_term<kMode>(gb, sg, K, sx, XP, E, p, q, e, acc);
        p += F - q - 2;
      }
      p = bi_pair_index(F, f, f + 1);
      for (int q = f + 1; q < F; ++q, ++p) acc = pn_dx_term<kMode>(gb, sg, K, sx, XP, E, p, q, e, acc);
      d[k] = acc;
    }
    __syncwarp();   // sx / sg are restaged for the next sample
  }
}

template <class Op>
cudaError_t pn_dispatch(int mode, Op op) {
  switch (mode) {
    case B2CTR_PNN_INNER: return op(std::integral_constant<int, B2CTR_PNN_INNER>());
    case B2CTR_PNN_ELEMENTWISE: return op(std::integral_constant<int, B2CTR_PNN_ELEMENTWISE>());
    case B2CTR_PNN_VEC: return op(std::integral_constant<int, B2CTR_PNN_VEC>());
    default: return op(std::integral_constant<int, B2CTR_PNN_NUM>());
  }
}

// vec: entry n = p*E + e, sum_b g_p x_i[e] x_j[e];  num: entry n = p, sum_b g_p <x_i, x_j>
__global__ void __launch_bounds__(256)
    pnn_inner_dk_kernel(const float* __restrict__ g, int64_t ldg, int64_t gcol0, const float* __restrict__ x,
                        int64_t ldx, int F, int E, int vec, float* partial, int nent, int nchunk, int64_t batch) {
  const int c = blockIdx.y;
  const int64_t per = (batch + nchunk - 1) / nchunk;
  const int64_t lo = (int64_t)c * per, hi = min(batch, lo + per);
  int pp[kPnDkPer], xi[kPnDkPer], xj[kPnDkPer];
  float acc[kPnDkPer];
#pragma unroll
  for (int m = 0; m < kPnDkPer; ++m) {
    const int n = blockIdx.x * (kPnDkPer * 256) + m * 256 + threadIdx.x;
    const int p = n < nent ? (vec ? n / E : n) : 0, e = vec && n < nent ? n - p * E : 0;
    int i, j;
    bi_pair_of(F, p, i, j);
    pp[m] = n < nent ? p : -1;
    xi[m] = i * E + e;
    xj[m] = j * E + e;
    acc[m] = 0.f;
  }
  for (int64_t b = lo; b < hi; ++b) {
    const float* xb = x + b * ldx;
    const float* gb = g + b * ldg + gcol0;
#pragma unroll
    for (int m = 0; m < kPnDkPer; ++m) {
      if (pp[m] < 0) continue;
      float t;
      if (vec) {
        t = xb[xi[m]] * xb[xj[m]];
      } else {
        t = 0.f;
        for (int e = 0; e < E; ++e) t = fmaf(xb[xi[m] + e], xb[xj[m] + e], t);
      }
      acc[m] = fmaf(gb[pp[m]], t, acc[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < kPnDkPer; ++m)
    if (pp[m] >= 0) partial[(int64_t)c * nent + blockIdx.x * (kPnDkPer * 256) + m * 256 + threadIdx.x] = acc[m];
}

static inline int pn_dk_entries(int F, int E, int mode) {
  const int P = F * (F - 1) / 2;
  return mode == B2CTR_PNN_VEC ? P * E : mode == B2CTR_PNN_NUM ? P : 0;
}
static inline int pn_dk_tiles(int nent) { return (int)ceil_div((int64_t)nent, kPnDkPer * 256); }
// batch chunks of the kernel-gradient pass: about 8 CTAs per SM over all entry tiles, at least 64 samples a chunk
static inline int pn_dk_chunks(int nent, int64_t batch) {
  const int64_t want = ceil_div((int64_t)kNumSMs * 8, pn_dk_tiles(nent));
  return (int)std::max<int64_t>(1, std::min(want, ceil_div(batch, 64)));
}

// ------------------------------------------------------------------------------------------------
// EDCN's BridgeModule + RegulationModule (deepctr/layers/interaction.py:1556-1565, core.py:307-315), the math of
// b2ctr_regulate_fwd / _bwd in include/b2ctr.h.  V = 4: every thread owns 4 consecutive columns of one field
// (dim % 4 == 0, 16-byte aligned windows); V = 1 the scalar path.
// * regulate_fwd_kernel: grid-stride over (sample, column group); the gates come from shared memory.
// * regulate_bwd_kernel: CTA (batch chunk, column tile of whole fields); R row lanes of G column groups each
//   (R * G <= 256).  A thread walks its chunk's rows in ascending order, writes dx / dh / dax / dah for its columns
//   (one owner per element) and keeps sum_b v * dy_k in registers; the CTA then adds its row lanes and each field's
//   columns in a fixed order into the per-(field, chunk) partial.  ordered_sum_kernel adds the chunks in order and
//   regulate_dg_kernel applies the softmax Jacobian.  Bit-identical from run to run.
// ------------------------------------------------------------------------------------------------
constexpr int kRegMaxF = 1024;
constexpr int kRegMaxE = 256;
constexpr int kRegThreads = 256;

// gates[f] = softmax_f(g[f] * it) by one warp; lanes stride over f and reduce with a fixed xor tree, so every CTA,
// the backward and the final step form bit-identical gates
__device__ __forceinline__ void reg_gates(const float* __restrict__ g, float it, int F, float* gates, int lane) {
  float m = -INFINITY;
  for (int f = lane; f < F; f += 32) m = fmaxf(m, g[f] * it);
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int f = lane; f < F; f += 32) s += expf(g[f] * it - m);
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  for (int f = lane; f < F; f += 32) gates[f] = expf(g[f] * it - m) / s;
}

__device__ __forceinline__ void reg_stage_gates(const b2ctr_regulate_t& a, float* sg) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0 && a.y0) reg_gates(a.g0, a.inv_tau0, a.nfield, sg, lane);
  if (warp == 1 && a.y1) reg_gates(a.g1, a.inv_tau1, a.nfield, sg + kRegMaxF, lane);
  __syncthreads();
}

template <int V>
__device__ __forceinline__ void reg_ld(const float* p, float (&r)[V]) {
  if constexpr (V == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    r[0] = t.x, r[1] = t.y, r[2] = t.z, r[3] = t.w;
  } else {
    r[0] = *p;
  }
}

template <int V>
__device__ __forceinline__ void reg_st(float* p, const float (&r)[V]) {
  if constexpr (V == 4)
    *reinterpret_cast<float4*>(p) = make_float4(r[0], r[1], r[2], r[3]);
  else
    *p = r[0];
}

// the operands of sample b at column c, and v
template <int V, int kMode>
__device__ __forceinline__ void reg_operands(const b2ctr_regulate_t& a, int64_t b, int c, float (&x)[V], float (&h)[V],
                                             float (&ax)[V], float (&ah)[V], float (&v)[V]) {
  reg_ld<V>(a.x + b * a.ldx + c, x);
  if (kMode != B2CTR_REGULATE_COPY) reg_ld<V>(a.h + b * a.ldh + c, h);
  if (kMode == B2CTR_REGULATE_ATTENTION) {
    reg_ld<V>(a.ax + b * a.ldax + c, ax);
    reg_ld<V>(a.ah + b * a.ldah + c, ah);
  }
#pragma unroll
  for (int q = 0; q < V; ++q) {
    if (kMode == B2CTR_REGULATE_COPY) v[q] = x[q];
    else if (kMode == B2CTR_REGULATE_ADD) v[q] = x[q] + h[q];
    else if (kMode == B2CTR_REGULATE_HADAMARD) v[q] = x[q] * h[q];
    else v[q] = fmaf(ax[q], x[q], ah[q] * h[q]);
  }
}

template <int V, int kMode>
__global__ void __launch_bounds__(kRegThreads) regulate_fwd_kernel(const b2ctr_regulate_t a) {
  __shared__ float sg[2 * kRegMaxF];
  reg_stage_gates(a, sg);
  const int E = a.dim, G = a.nfield * E / V;
  const int64_t total = a.batch * G;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / G;
    const int c = (int)(i - b * G) * V, f = c / E;
    float x[V], h[V], ax[V], ah[V], v[V], y[V];
    reg_operands<V, kMode>(a, b, c, x, h, ax, ah, v);
    if (a.u) reg_st<V>(a.u + b * a.ldu + a.ucol + c, v);
    if (a.y0) {
      const float gt = sg[f];
#pragma unroll
      for (int q = 0; q < V; ++q) y[q] = v[q] * gt;
      reg_st<V>(a.y0 + b * a.ldy0 + a.y0col + c, y);
    }
    if (a.y1) {
      const float gt = sg[kRegMaxF + f];
#pragma unroll
      for (int q = 0; q < V; ++q) y[q] = v[q] * gt;
      reg_st<V>(a.y1 + b * a.ldy1 + a.y1col + c, y);
    }
  }
}

template <int V, int kMode>
__global__ void __launch_bounds__(kRegThreads, 4)
    regulate_bwd_kernel(const b2ctr_regulate_t a, int W, int R, int nchunk, float* partial) {
  __shared__ float sg[2 * kRegMaxF];
  __shared__ float scol[2 * kRegThreads * V];
  reg_stage_gates(a, sg);
  const int F = a.nfield, E = a.dim, d = F * E, G = W / V;
  const int r = threadIdx.x / G, j = threadIdx.x - r * G, c0 = blockIdx.y * W, c = c0 + j * V;
  const bool active = r < R && c < d;
  const int64_t per = (a.batch + nchunk - 1) / nchunk, lo = (int64_t)blockIdx.x * per, hi = min(a.batch, lo + per);
  float acc0[V], acc1[V];
#pragma unroll
  for (int q = 0; q < V; ++q) acc0[q] = acc1[q] = 0.f;
  if (active) {
    const int f = c / E;
    const float gt0 = a.y0 ? sg[f] : 0.f, gt1 = a.y1 ? sg[kRegMaxF + f] : 0.f;
    for (int64_t b = lo + r; b < hi; b += R) {
      float x[V], h[V], ax[V], ah[V], v[V], dv[V], t[V];
      reg_operands<V, kMode>(a, b, c, x, h, ax, ah, v);
      if (a.u) {
        reg_ld<V>(a.u + b * a.ldu + a.ucol + c, dv);
      } else {
#pragma unroll
        for (int q = 0; q < V; ++q) dv[q] = 0.f;
      }
      if (a.y0) {
        reg_ld<V>(a.y0 + b * a.ldy0 + a.y0col + c, t);
#pragma unroll
        for (int q = 0; q < V; ++q) dv[q] = fmaf(gt0, t[q], dv[q]), acc0[q] = fmaf(v[q], t[q], acc0[q]);
      }
      if (a.y1) {
        reg_ld<V>(a.y1 + b * a.ldy1 + a.y1col + c, t);
#pragma unroll
        for (int q = 0; q < V; ++q) dv[q] = fmaf(gt1, t[q], dv[q]), acc1[q] = fmaf(v[q], t[q], acc1[q]);
      }
      if (a.dx) {
        float* p = a.dx + b * a.lddx + c;
#pragma unroll
        for (int q = 0; q < V; ++q)
          t[q] = kMode == B2CTR_REGULATE_HADAMARD ? dv[q] * h[q] : kMode == B2CTR_REGULATE_ATTENTION ? dv[q] * ax[q] : dv[q];
        if (a.dx_accumulate) {
          float o[V];
          reg_ld<V>(p, o);
#pragma unroll
          for (int q = 0; q < V; ++q) t[q] += o[q];
        }
        reg_st<V>(p, t);
      }
      if (kMode != B2CTR_REGULATE_COPY && a.dh) {
#pragma unroll
        for (int q = 0; q < V; ++q)
          t[q] = kMode == B2CTR_REGULATE_HADAMARD ? dv[q] * x[q]
                 : kMode == B2CTR_REGULATE_ATTENTION ? dv[q] * ah[q] : dv[q];
        reg_st<V>(a.dh + b * a.lddh + c, t);
      }
      if (kMode == B2CTR_REGULATE_ATTENTION && a.dax) {
#pragma unroll
        for (int q = 0; q < V; ++q) t[q] = dv[q] * x[q];
        reg_st<V>(a.dax + b * a.lddax + c, t);
      }
      if (kMode == B2CTR_REGULATE_ATTENTION && a.dah) {
#pragma unroll
        for (int q = 0; q < V; ++q) t[q] = dv[q] * h[q];
        reg_st<V>(a.dah + b * a.lddah + c, t);
      }
    }
  }
  if (!partial) return;
  float* s0 = scol;
  float* s1 = scol + kRegThreads * V;
  if (active) {
#pragma unroll
    for (int q = 0; q < V; ++q) s0[r * W + j * V + q] = acc0[q], s1[r * W + j * V + q] = acc1[q];
  }
  __syncthreads();
  // the tile holds whole fields: c0 and min(W, d - c0) are multiples of E
  const int nf = min(W, d - c0) / E;
  for (int k = threadIdx.x; k < 2 * nf; k += blockDim.x) {
    const int gate = k / nf, fl = k - gate * nf;
    const float* s = gate ? s1 : s0;
    float sum = 0.f;
    for (int rr = 0; rr < R; ++rr)
      for (int e = 0; e < E; ++e) sum += s[rr * W + fl * E + e];
    partial[(int64_t)blockIdx.x * 2 * F + gate * F + c0 / E + fl] = sum;
  }
}

// dg_k = inv_tau_k * gate_k * (s_k - <gate_k, s_k>), one warp per gate; s [2, F] the chunk-summed partials
__global__ void regulate_dg_kernel(const b2ctr_regulate_t a, const float* __restrict__ s) {
  __shared__ float sg[2 * kRegMaxF];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, F = a.nfield;
  float* dg = warp ? a.dg1 : a.dg0;
  if (!dg) return;
  const float* g = warp ? a.g1 : a.g0;
  const float it = warp ? a.inv_tau1 : a.inv_tau0;
  float* gates = sg + warp * kRegMaxF;
  const float* sk = s + warp * F;
  reg_gates(g, it, F, gates, lane);
  __syncwarp();
  float dot = 0.f;
  for (int f = lane; f < F; f += 32) dot = fmaf(gates[f], sk[f], dot);
  for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  for (int f = lane; f < F; f += 32) dg[f] = it * gates[f] * (sk[f] - dot);
}

// backward geometry: column tiles of whole fields (W columns, G = W / V groups), R = 256 / G row lanes, and batch
// chunks of at least 128 samples, about 8 CTAs per SM in all
static inline int reg_tile(int E, int V) { return (kRegThreads * V / E) * E; }
static inline int reg_chunks(int64_t batch) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(batch, 128), (int64_t)kNumSMs * 8));
}

template <class Op>
cudaError_t reg_dispatch(int mode, bool vec, Op op) {
  auto m = [&](auto v) -> cudaError_t {
    switch (mode) {
      case B2CTR_REGULATE_COPY: return op(v, std::integral_constant<int, B2CTR_REGULATE_COPY>());
      case B2CTR_REGULATE_ADD: return op(v, std::integral_constant<int, B2CTR_REGULATE_ADD>());
      case B2CTR_REGULATE_HADAMARD: return op(v, std::integral_constant<int, B2CTR_REGULATE_HADAMARD>());
      default: return op(v, std::integral_constant<int, B2CTR_REGULATE_ATTENTION>());
    }
  };
  return vec ? m(std::integral_constant<int, 4>()) : m(std::integral_constant<int, 1>());
}

// ------------------------------------------------------------------------------------------------
// CCPM's convolution stack (b2ctr_conv_stack_fwd / _bwd in include/b2ctr.h).  A CTA serves kConvCols = 32 columns
// (sample, e); each column gets kConvG threads, one per channel slot (G = the most channels of any map), so a thread
// (g, col) owns the channels c = g, g + G, ... of its column in every stage.  The maps live in shared memory,
// interleaved [element][column] so the 32 columns of a warp hit 32 banks.  Forward: two maps ping-pong.  Backward:
// every map is kept (k-max stages also keep their selected rows), then the gradient goes back through two more maps;
// the weight gradients of a tile are summed by one owner thread per weight over the tile's columns in column order
// and added to the CTA's running sum, which goes to the workspace as the CTA's partial.
// ------------------------------------------------------------------------------------------------
constexpr int kConvCols = 32;
constexpr size_t kConvSmemCap = 224 * 1024;

struct ConvStagePlan {
  int kind, width, pad, act, k;
  int rows_in, cin, rows_out, cout;
  int in_off, out_off, idx_off;  // map offsets (elements of one column; backward layout)
  int w_off, nw;                 // weights in shared memory: kernel [width, cin, cout] then bias [cout]
};
struct ConvPlan {
  int nstage, G, nw;           // channel slots per column, total weight floats
  int map_floats, max_map;     // backward: all maps of a column; the largest map
  int ga_off, gb_off;          // backward gradient maps
  int rows_out, cout;          // last map
  ConvStagePlan s[B2CTR_CONV_STACK_MAX_STAGES];
};

__device__ __forceinline__ float& cs_at(float* sm, int off, int i, int col) { return sm[(off + i) * kConvCols + col]; }

// forward of stage p from map `in` to map `out` (and the selected rows to `idx` when k-max and idx_off >= 0)
__device__ __forceinline__ void conv_stage_fwd(const ConvStagePlan& p, const float* sw, float* sm, int in, int out,
                                               int idx, int g, int G, int col) {
  if (p.kind == B2CTR_CONV_STAGE_CONV) {
    const float* K = sw + p.w_off;
    const float* bias = K + p.width * p.cin * p.cout;
    for (int co = g; co < p.cout; co += G) {
      for (int r = 0; r < p.rows_out; ++r) {
        float acc = bias[co];
        for (int t = 0; t < p.width; ++t) {
          const int rr = r + t - p.pad;
          if (rr < 0 || rr >= p.rows_in) continue;
          const float* kt = K + t * p.cin * p.cout + co;
          for (int ci = 0; ci < p.cin; ++ci) acc = fmaf(cs_at(sm, in, rr * p.cin + ci, col), kt[ci * p.cout], acc);
        }
        cs_at(sm, out, r * p.cout + co, col) = act_apply(acc, p.act);
      }
    }
  } else {
    const int C = p.cin;
    for (int c = g; c < C; c += G) {
      // the j-th pick is the largest value ordered after the (j-1)-th in (value descending, row ascending)
      float pv = 0.f;
      int pi = -1;
      for (int j = 0; j < p.k; ++j) {
        float bv = 0.f;
        int bi = -1;
        for (int r = 0; r < p.rows_in; ++r) {
          const float v = cs_at(sm, in, r * C + c, col);
          const bool after = pi < 0 || v < pv || (v == pv && r > pi);
          if (after && (bi < 0 || v > bv)) { bv = v; bi = r; }
        }
        pv = bv;
        pi = bi;
        cs_at(sm, out, j * C + c, col) = bi < 0 ? __int_as_float(0x7fc00000) : bv;   // only NaN rows left
        if (idx >= 0) cs_at(sm, idx, j * C + c, col) = __int_as_float(bi);
      }
    }
  }
}

__device__ __forceinline__ void conv_stage_weights(const b2ctr_conv_stack_t& a, const ConvPlan& P, float* sw) {
  for (int s = 0; s < P.nstage; ++s) {
    const ConvStagePlan& p = P.s[s];
    if (p.kind != B2CTR_CONV_STAGE_CONV) continue;
    const int nk = p.width * p.cin * p.cout;
    for (int i = threadIdx.x; i < p.nw; i += blockDim.x)
      sw[p.w_off + i] = i < nk ? a.stage[s].kernel[i] : (a.stage[s].bias ? a.stage[s].bias[i - nk] : 0.f);
  }
}

// the input map of a column into map 0
__device__ __forceinline__ void conv_load_input(const b2ctr_conv_stack_t& a, float* sm, int off, int64_t b, int e,
                                                bool valid, int g, int G, int col) {
  const int C = a.channels;
  const float* xp = a.x + b * a.ldx + a.xcol;
  for (int c = g; c < C; c += G)
    for (int r = 0; r < a.rows; ++r)
      cs_at(sm, off, r * C + c, col) = valid ? xp[((int64_t)r * a.dim + e) * C + c] : 0.f;
}

__global__ void conv_stack_fwd_kernel(const b2ctr_conv_stack_t a, const __grid_constant__ ConvPlan P) {
  extern __shared__ float smem[];
  float* sw = smem;
  float* sm = smem + P.nw;
  const int G = P.G, col = threadIdx.x % kConvCols, g = threadIdx.x / kConvCols;
  const int64_t ncol = a.batch * a.dim, cg = (int64_t)blockIdx.x * kConvCols + col;
  const bool valid = cg < ncol;
  const int64_t b = valid ? cg / a.dim : 0;
  const int e = valid ? (int)(cg % a.dim) : 0;
  conv_stage_weights(a, P, sw);
  int cur = 0, nxt = P.max_map;
  conv_load_input(a, sm, cur, b, e, valid, g, G, col);
  __syncthreads();
  for (int s = 0; s < P.nstage; ++s) {
    conv_stage_fwd(P.s[s], sw, sm, cur, nxt, -1, g, G, col);
    __syncthreads();
    const int t = cur;
    cur = nxt;
    nxt = t;
  }
  if (!valid) return;
  float* op = a.out + b * a.ldout + a.outcol;
  for (int c = g; c < P.cout; c += G)
    for (int r = 0; r < P.rows_out; ++r) op[((int64_t)r * a.dim + e) * P.cout + c] = cs_at(sm, cur, r * P.cout + c, col);
}

__global__ void conv_stack_bwd_kernel(const b2ctr_conv_stack_t a, const __grid_constant__ ConvPlan P,
                                      float* __restrict__ partial) {
  extern __shared__ float smem[];
  float* sw = smem;
  float* sacc = smem + P.nw;
  float* sm = smem + 2 * P.nw;
  const int G = P.G, col = threadIdx.x % kConvCols, g = threadIdx.x / kConvCols;
  const int64_t ncol = a.batch * a.dim;
  conv_stage_weights(a, P, sw);
  for (int i = threadIdx.x; i < P.nw; i += blockDim.x) sacc[i] = 0.f;
  for (int64_t tile = blockIdx.x; tile * kConvCols < ncol; tile += gridDim.x) {
    const int64_t cg = tile * kConvCols + col;
    const bool valid = cg < ncol;
    const int nvalid = (int)min((int64_t)kConvCols, ncol - tile * kConvCols);
    const int64_t b = valid ? cg / a.dim : 0;
    const int e = valid ? (int)(cg % a.dim) : 0;
    __syncthreads();  // the previous tile's maps are no longer read
    conv_load_input(a, sm, 0, b, e, valid, g, G, col);
    __syncthreads();
    for (int s = 0; s < P.nstage; ++s) {
      const ConvStagePlan& p = P.s[s];
      conv_stage_fwd(p, sw, sm, p.in_off, p.out_off, p.idx_off, g, G, col);
      __syncthreads();
    }
    // incoming gradient of the last map
    int gcur = P.ga_off, gnxt = P.gb_off;
    if (valid) {
      const float* dp = a.out + b * a.ldout + a.outcol;
      for (int c = g; c < P.cout; c += G)
        for (int r = 0; r < P.rows_out; ++r)
          cs_at(sm, gcur, r * P.cout + c, col) = dp[((int64_t)r * a.dim + e) * P.cout + c];
    } else {
      for (int c = g; c < P.cout; c += G)
        for (int r = 0; r < P.rows_out; ++r) cs_at(sm, gcur, r * P.cout + c, col) = 0.f;
    }
    __syncthreads();
    for (int s = P.nstage - 1; s >= 0; --s) {
      const ConvStagePlan& p = P.s[s];
      if (p.kind == B2CTR_CONV_STAGE_KMAX) {
        const int C = p.cin;
        for (int c = g; c < C; c += G) {
          for (int r = 0; r < p.rows_in; ++r) cs_at(sm, gnxt, r * C + c, col) = 0.f;
          for (int j = 0; j < p.k; ++j) {
            const int r = __float_as_int(cs_at(sm, p.idx_off, j * C + c, col));
            if (r >= 0) cs_at(sm, gnxt, r * C + c, col) = cs_at(sm, gcur, j * C + c, col);
          }
        }
        __syncthreads();
      } else {
        // dz = dy * act'(y), in place
        for (int co = g; co < p.cout; co += G)
          for (int r = 0; r < p.rows_out; ++r)
            cs_at(sm, gcur, r * p.cout + co, col) *= act_grad_from_out(cs_at(sm, p.out_off, r * p.cout + co, col), p.act);
        __syncthreads();
        const float* K = sw + p.w_off;
        if (s > 0 || a.dx) {
          for (int ci = g; ci < p.cin; ci += G) {
            for (int r = 0; r < p.rows_in; ++r) {
              float acc = 0.f;
              for (int t = 0; t < p.width; ++t) {
                const int ro = r - t + p.pad;
                if (ro < 0 || ro >= p.rows_out) continue;
                const float* kt = K + (t * p.cin + ci) * p.cout;
                for (int co = 0; co < p.cout; ++co) acc = fmaf(cs_at(sm, gcur, ro * p.cout + co, col), kt[co], acc);
              }
              cs_at(sm, gnxt, r * p.cin + ci, col) = acc;
            }
          }
        }
        // weight gradients of this tile: one owner per weight, columns in order
        const int nk = p.width * p.cin * p.cout;
        for (int w = threadIdx.x; w < p.nw; w += blockDim.x) {
          float acc = 0.f;
          if (w < nk) {
            const int co = w % p.cout, ci = (w / p.cout) % p.cin, t = w / (p.cout * p.cin);
            for (int c = 0; c < nvalid; ++c)
              for (int r = 0; r < p.rows_out; ++r) {
                const int rr = r + t - p.pad;
                if (rr < 0 || rr >= p.rows_in) continue;
                acc = fmaf(cs_at(sm, p.in_off, rr * p.cin + ci, c), cs_at(sm, gcur, r * p.cout + co, c), acc);
              }
          } else {
            const int co = w - nk;
            for (int c = 0; c < nvalid; ++c)
              for (int r = 0; r < p.rows_out; ++r) acc += cs_at(sm, gcur, r * p.cout + co, c);
          }
          sacc[p.w_off + w] += acc;
        }
        __syncthreads();
      }
      const int t = gcur;
      gcur = gnxt;
      gnxt = t;
    }
    if (valid && a.dx) {
      const int C = a.channels;
      float* dp = a.dx + b * a.lddx + a.dxcol;
      for (int c = g; c < C; c += G)
        for (int r = 0; r < a.rows; ++r) {
          const int64_t o = ((int64_t)r * a.dim + e) * C + c;
          const float v = cs_at(sm, gcur, r * C + c, col);
          dp[o] = a.dx_accumulate ? dp[o] + v : v;
        }
    }
  }
  __syncthreads();
  if (partial)
    for (int i = threadIdx.x; i < P.nw; i += blockDim.x) partial[(int64_t)blockIdx.x * P.nw + i] = sacc[i];
}

// ------------------------------------------------------------------------------------------------
// FLEN's FieldWiseBiInteraction (b2ctr_field_wise_bi_fwd / _bwd in include/b2ctr.h).  A CTA is R row lanes of
// Gc = dim / V column groups; thread (r, j) owns the V columns [j * V, j * V + V) of every row it visits, so each
// thread forms S_g and S_g^2 - Q_g of its columns in registers from the members of every group, read in place
// through the per-field columns (sorted by group on the host).  Arrays over groups are indexed by compile-time
// g < kFwbiMaxG only (unrolled, guarded by the runtime G), so they stay in registers.
// * fwbi_fwd_kernel: row blocks of R rows, grid-stride; writes only h.
// * fwbi_bwd_kernel: CTA = one batch chunk walked in ascending row order; dx has one owner per element; the
//   weight-gradient sums stay in registers, then the CTA adds its threads (and row lanes, for the biases) in a
//   fixed order into its partial.  ordered_sum_kernel adds the partials in CTA order: bit-identical from run to run.
// ------------------------------------------------------------------------------------------------
constexpr int kFwbiMaxG = B2CTR_FWBI_MAX_GROUPS;
constexpr int kFwbiMaxP = kFwbiMaxG * (kFwbiMaxG - 1) / 2;
constexpr int kFwbiMaxE = 256;
constexpr int kFwbiThreads = 256;

struct FwbiArgs {
  int F, G, E, dx_accumulate;
  int64_t batch;
  const float* x; int64_t ldx;
  const float* kmf; const float* kfm; const float* bmf; const float* bfm;
  float* out; int64_t ldout, outcol;
  float* dx; int64_t lddx;
  int start[kFwbiMaxG + 1];                  // the members of group g are cols[start[g] .. start[g + 1])
  int cols[B2CTR_FWBI_MAX_FIELDS];
};

// index of pair (g, h), g < h, in itertools.combinations(range(G), 2) order
__device__ __forceinline__ int fwbi_pair(int g, int h, int G) { return g * (2 * G - g - 1) / 2 + h - g - 1; }

__device__ __forceinline__ void fwbi_stage_weights(const FwbiArgs& a, float* skmf, float* skfm) {
  const int P = a.G * (a.G - 1) / 2;
  for (int i = threadIdx.x; i < P; i += blockDim.x) skmf[i] = a.kmf[i];
  for (int i = threadIdx.x; i < a.G; i += blockDim.x) skfm[i] = a.kfm[i];
  __syncthreads();
}

// S[g] = sum of the members of group g and, through fm(g, v, S_g^2 - Q_g), the FM term of each group, for the V
// columns at xr
template <int V, class Fm>
__device__ __forceinline__ void fwbi_sums(const FwbiArgs& a, const float* xr, float (&S)[kFwbiMaxG][V], Fm fm) {
#pragma unroll
  for (int g = 0; g < kFwbiMaxG; ++g) {
    float s[V], q[V];
#pragma unroll
    for (int v = 0; v < V; ++v) s[v] = q[v] = 0.f;
    if (g < a.G) {
      for (int i = a.start[g]; i < a.start[g + 1]; ++i) {
        float t[V];
        reg_ld<V>(xr + a.cols[i], t);
#pragma unroll
        for (int v = 0; v < V; ++v) s[v] += t[v], q[v] = fmaf(t[v], t[v], q[v]);
      }
#pragma unroll
      for (int v = 0; v < V; ++v) fm(g, v, fmaf(s[v], s[v], -q[v]));
    }
#pragma unroll
    for (int v = 0; v < V; ++v) S[g][v] = s[v];
  }
}

template <int V>
__global__ void __launch_bounds__(kFwbiThreads, 2) fwbi_fwd_kernel(const __grid_constant__ FwbiArgs a) {
  __shared__ float skmf[kFwbiMaxP], skfm[kFwbiMaxG];
  fwbi_stage_weights(a, skmf, skfm);
  const int Gc = a.E / V, R = kFwbiThreads / Gc, r = threadIdx.x / Gc, c = (threadIdx.x - r * Gc) * V;
  if (r >= R) return;
  float bm[V], bf[V];
#pragma unroll
  for (int v = 0; v < V; ++v) bm[v] = a.bmf ? a.bmf[c + v] : 0.f, bf[v] = a.bfm ? a.bfm[c + v] : 0.f;
  for (int64_t b = (int64_t)blockIdx.x * R + r; b < a.batch; b += (int64_t)gridDim.x * R) {
    float S[kFwbiMaxG][V], hmf[V], hfm[V];
#pragma unroll
    for (int v = 0; v < V; ++v) hmf[v] = hfm[v] = 0.f;
    fwbi_sums<V>(a, a.x + b * a.ldx + c, S, [&](int g, int v, float d) { hfm[v] = fmaf(d, skfm[g], hfm[v]); });
#pragma unroll
    for (int g = 0; g < kFwbiMaxG; ++g) {
#pragma unroll
      for (int h = g + 1; h < kFwbiMaxG; ++h) {
        if (h < a.G) {
          const float k = skmf[fwbi_pair(g, h, a.G)];
#pragma unroll
          for (int v = 0; v < V; ++v) hmf[v] = fmaf(S[g][v] * S[h][v], k, hmf[v]);
        }
      }
    }
    float y[V];
#pragma unroll
    for (int v = 0; v < V; ++v) y[v] = (hmf[v] + bm[v]) + (hfm[v] + bf[v]);
    reg_st<V>(a.out + b * a.ldout + a.outcol + c, y);
  }
}

template <int V>
__global__ void __launch_bounds__(kFwbiThreads, 2)
    fwbi_bwd_kernel(const __grid_constant__ FwbiArgs a, int nchunk, float* partial, int pitch) {
  __shared__ float skmf[kFwbiMaxP], skfm[kFwbiMaxG];
  __shared__ float sred[(kFwbiMaxP + kFwbiMaxG) * kFwbiThreads];
  __shared__ float sbias[kFwbiThreads * 4];
  fwbi_stage_weights(a, skmf, skfm);
  const int G = a.G, Gc = a.E / V, R = kFwbiThreads / Gc, r = threadIdx.x / Gc, c = (threadIdx.x - r * Gc) * V;
  const bool active = r < R;
  const int64_t per = (a.batch + nchunk - 1) / nchunk, lo = (int64_t)blockIdx.x * per, hi = min(a.batch, lo + per);
  float amf[kFwbiMaxP], afm[kFwbiMaxG], adb[V];
#pragma unroll
  for (int k = 0; k < kFwbiMaxP; ++k) amf[k] = 0.f;
#pragma unroll
  for (int g = 0; g < kFwbiMaxG; ++g) afm[g] = 0.f;
#pragma unroll
  for (int v = 0; v < V; ++v) adb[v] = 0.f;
  if (active) {
    for (int64_t b = lo + r; b < hi; b += R) {
      const float* xr = a.x + b * a.ldx + c;
      float S[kFwbiMaxG][V], dh[V];
      reg_ld<V>(a.out + b * a.ldout + a.outcol + c, dh);
      fwbi_sums<V>(a, xr, S, [&](int g, int v, float d) { afm[g] = fmaf(dh[v], d, afm[g]); });
#pragma unroll
      for (int v = 0; v < V; ++v) adb[v] += dh[v];
#pragma unroll
      for (int g = 0, k = 0; g < kFwbiMaxG; ++g) {
#pragma unroll
        for (int h = g + 1; h < kFwbiMaxG; ++h, ++k) {
#pragma unroll
          for (int v = 0; v < V; ++v) amf[k] = fmaf(dh[v], S[g][v] * S[h][v], amf[k]);
        }
      }
      if (!a.dx) continue;
#pragma unroll
      for (int g = 0; g < kFwbiMaxG; ++g) {
        if (g >= G) break;
        const float two_fm = 2.f * skfm[g];
        float t[V];
#pragma unroll
        for (int v = 0; v < V; ++v) t[v] = two_fm * S[g][v];
#pragma unroll
        for (int h = 0; h < kFwbiMaxG; ++h) {
          if (h != g && h < G) {
            const float k = skmf[h < g ? fwbi_pair(h, g, G) : fwbi_pair(g, h, G)];
#pragma unroll
            for (int v = 0; v < V; ++v) t[v] = fmaf(k, S[h][v], t[v]);
          }
        }
        for (int i = a.start[g]; i < a.start[g + 1]; ++i) {
          float xv[V], d[V];
          reg_ld<V>(xr + a.cols[i], xv);
#pragma unroll
          for (int v = 0; v < V; ++v) d[v] = dh[v] * (t[v] - two_fm * xv[v]);
          float* p = a.dx + b * a.lddx + a.cols[i] + c;
          if (a.dx_accumulate) {
            float o[V];
            reg_ld<V>(p, o);
#pragma unroll
            for (int v = 0; v < V; ++v) d[v] += o[v];
          }
          reg_st<V>(p, d);
        }
      }
    }
  }
  if (!partial) return;
  // the sums in combinations order, then the groups, then the columns: k-th entry of thread t at sred[k * 256 + t]
  const int P = G * (G - 1) / 2;
#pragma unroll
  for (int g = 0, k = 0; g < kFwbiMaxG; ++g) {
    if (g < G) sred[(P + g) * kFwbiThreads + threadIdx.x] = afm[g];
#pragma unroll
    for (int h = g + 1; h < kFwbiMaxG; ++h, ++k)
      if (h < G) sred[fwbi_pair(g, h, G) * kFwbiThreads + threadIdx.x] = amf[k];
  }
  if (active) {
#pragma unroll
    for (int v = 0; v < V; ++v) sbias[r * a.E + c + v] = adb[v];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < P + G + a.E; k += blockDim.x) {
    float s = 0.f;
    if (k < P + G) {
      for (int t = 0; t < kFwbiThreads; ++t) s += sred[k * kFwbiThreads + t];
    } else {
      for (int rr = 0; rr < R; ++rr) s += sbias[rr * a.E + k - P - G];
    }
    partial[(int64_t)blockIdx.x * pitch + k] = s;
  }
}

// backward batch chunks: at least 128 samples each, about 4 CTAs per SM in all
static inline int fwbi_chunks(int64_t batch) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(batch, 128), (int64_t)kNumSMs * 4));
}

}  // namespace b2ctr

using namespace b2ctr;
#define ST ((cudaStream_t)stream)

extern "C" {

b2ctr_status_t b2ctr_ewise(int32_t op, const float* a, const float* b, const float* c, float* out,
                           int64_t n, int32_t accumulate, void* stream) {
  B2_REQUIRE(a && b && out && (op == 0 || (op == 1 && c)), "ewise: bad arguments");
  if (n <= 0) return B2CTR_OK;
  ewise_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(op, a, b, c, out, n, accumulate);
  B2_CHECK_LAUNCH("b2ctr_ewise");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cross_vector_fwd(const float* x0, int64_t ld0, const float* xl, int64_t ldl,
                                      const float* w, const float* bias, float* out, float* s,
                                      int64_t batch, int32_t dim, void* stream) {
  B2_REQUIRE(x0 && xl && w && bias && out && s && dim > 0 && ld0 >= dim && ldl >= dim,
             "cross_vector_fwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  cross_vector_fwd_kernel<<<grid_for(batch, 8, 8), 256, 0, ST>>>(x0, ld0, xl, ldl, w, bias, out, s, batch, dim);
  B2_CHECK_LAUNCH("b2ctr_cross_vector_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cross_vector_bwd(const float* x0, int64_t ld0, const float* w, const float* dout,
                                      const float* s, float* dx0, float* dxl, float* ds, int64_t batch,
                                      int32_t dim, void* stream) {
  B2_REQUIRE(x0 && w && dout && s && dx0 && dxl && ds && dim > 0 && ld0 >= dim, "cross_vector_bwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  cross_vector_bwd_kernel<<<grid_for(batch, 8, 8), 256, 0, ST>>>(x0, ld0, w, dout, s, dx0, dxl, ds, batch, dim);
  B2_CHECK_LAUNCH("b2ctr_cross_vector_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_outer_fwd(const float* x0, int64_t s0b, int64_t s0i, int64_t s0d, const float* xk,
                                   int64_t skb, int64_t ski, int64_t skd, float* z, int64_t nb, int32_t m,
                                   int32_t h, int32_t d, void* stream) {
  B2_REQUIRE(x0 && xk && z && m > 0 && h > 0 && d > 0, "cin_outer_fwd: bad arguments");
  if (nb <= 0) return B2CTR_OK;
  CinView a{x0, s0b, s0i, s0d}, b{xk, skb, ski, skd};
  cin_outer_fwd_kernel<<<grid_for(nb * d * m * h, 256, 8), 256, 0, ST>>>(a, b, z, nb, m, h, d);
  B2_CHECK_LAUNCH("b2ctr_cin_outer_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_outer_bwd(const float* dz, const float* x0, int64_t s0b, int64_t s0i, int64_t s0d,
                                   const float* xk, int64_t skb, int64_t ski, int64_t skd, float* dx0,
                                   int64_t g0b, int64_t g0i, int64_t g0d, int32_t acc0, float* dxk,
                                   int64_t gkb, int64_t gki, int64_t gkd, int32_t acck, int64_t nb, int32_t m,
                                   int32_t h, int32_t d, int32_t hp, void* stream) {
  B2_REQUIRE(dz && x0 && xk && (dx0 || dxk) && m > 0 && h > 0 && d > 0, "cin_outer_bwd: bad arguments");
  if (hp <= 0) hp = h;
  B2_REQUIRE(hp >= h, "cin_outer_bwd: hp < h");
  if (nb <= 0) return B2CTR_OK;
  CinView a{x0, s0b, s0i, s0d}, b{xk, skb, ski, skd};
  cin_outer_bwd_kernel<<<grid_for(nb * d, 8, 8), 256, 0, ST>>>(dz, a, b, dx0, g0b, g0i, g0d, acc0, dxk, gkb,
                                                              gki, gkd, acck, nb, m, h, d, hp);
  B2_CHECK_LAUNCH("b2ctr_cin_outer_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_t0(const float* x0, int64_t s0b, int64_t s0i, int64_t s0d, float* t0, int64_t ld0,
                            int64_t nb, int32_t m, int32_t d, void* stream) {
  B2_REQUIRE(x0 && t0 && m > 0 && d > 0 && ld0 >= m, "cin_t0: bad arguments");
  if (nb <= 0) return B2CTR_OK;
  CinView a{x0, s0b, s0i, s0d};
  cin_t0_kernel<<<grid_for(nb * d * ld0, 256, 8), 256, 0, ST>>>(a, t0, ld0, nb, m, d);
  B2_CHECK_LAUNCH("b2ctr_cin_t0");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_t0_bwd(const float* dt0, int64_t ld0, float* dx, int64_t gb, int64_t gi, int64_t gd,
                                int32_t accumulate, int64_t nb, int32_t m, int32_t d, void* stream) {
  B2_REQUIRE(dt0 && dx && m > 0 && d > 0 && ld0 >= m, "cin_t0_bwd: bad arguments");
  if (nb <= 0) return B2CTR_OK;
  cin_t0_bwd_kernel<<<grid_for(nb * d * m, 256, 8), 256, 0, ST>>>(dt0, ld0, dx, gb, gi, gd, accumulate, nb, m, d);
  B2_CHECK_LAUNCH("b2ctr_cin_t0_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_unpad_rows(const float* src, float* dst, int32_t m, int32_t h, int32_t hp, int64_t n,
                                    void* stream) {
  B2_REQUIRE(src && dst && m > 0 && h > 0 && hp >= h && n > 0, "cin_unpad_rows: bad arguments");
  cin_unpad_rows_kernel<<<grid_for((int64_t)m * h * n, 256, 8), 256, 0, ST>>>(src, dst, m, h, hp, n);
  B2_CHECK_LAUNCH("b2ctr_cin_unpad_rows");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_sum_d(const float* y, int64_t ldy, int32_t col0, int32_t ncols, int32_t d, float* out,
                               int64_t ldo, int32_t out_col, int64_t nb, void* stream) {
  B2_REQUIRE(y && out && ncols > 0 && d > 0, "cin_sum_d: bad arguments");
  if (nb <= 0) return B2CTR_OK;
  cin_sum_d_kernel<<<grid_for(nb * ncols, 256, 8), 256, 0, ST>>>(y, ldy, col0, ncols, d, out, ldo, out_col, nb);
  B2_CHECK_LAUNCH("b2ctr_cin_sum_d");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_cin_expand_grad(const float* dout, int64_t ldo, int32_t out_col, int32_t col0,
                                     int32_t ncols, const float* dh, int64_t ldh, int32_t hcols, float* dy,
                                     int64_t nfilt, int32_t d, int64_t nb, void* stream) {
  B2_REQUIRE(dout && dy && nfilt > 0 && d > 0, "cin_expand_grad: bad arguments");
  if (nb <= 0) return B2CTR_OK;
  cin_expand_grad_kernel<<<grid_for(nb * d * nfilt, 256, 8), 256, 0, ST>>>(dout, ldo, out_col, col0, ncols, dh,
                                                                         ldh, hcols, dy, nfilt, d, nb);
  B2_CHECK_LAUNCH("b2ctr_cin_expand_grad");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_interacting_fwd(const float* q, const float* k, const float* v, const float* res,
                                     float* out, int64_t batch, int32_t nfield, int32_t heads, int32_t dhead,
                                     int32_t scaling, void* stream) {
  B2_REQUIRE(q && k && v && out, "interacting_fwd: NULL pointer");
  B2_REQUIRE(nfield > 0 && nfield <= kIntMaxF && heads > 0 && dhead > 0 && dhead <= 32,
             "interacting_fwd: needs field_size <= %d and att_embedding_size <= 32", kIntMaxF);
  B2_REQUIRE((int64_t)nfield * heads * dhead <= kIntMaxFHD,
             "interacting_fwd: field_size * head_num * att_embedding_size must be <= %d", kIntMaxFHD);
  if (batch <= 0) return B2CTR_OK;
  const size_t smem = (size_t)2 * nfield * heads * dhead * sizeof(float);
  const float scale = scaling ? 1.f / sqrtf((float)dhead) : 1.f;
  interacting_fwd_kernel<<<(unsigned)batch, 128, smem, ST>>>(q, k, v, res, out, nfield, heads, dhead, scale);
  B2_CHECK_LAUNCH("b2ctr_interacting_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_interacting_bwd(const float* q, const float* k, const float* v, const float* out,
                                     const float* dout, float* dq, float* dk, float* dv, float* dres,
                                     int64_t batch, int32_t nfield, int32_t heads, int32_t dhead,
                                     int32_t scaling, void* stream) {
  B2_REQUIRE(q && k && v && out && dout && dq && dk && dv, "interacting_bwd: NULL pointer");
  B2_REQUIRE(nfield > 0 && nfield <= kIntMaxF && heads > 0 && dhead > 0 && dhead <= 32,
             "interacting_bwd: needs field_size <= %d and att_embedding_size <= 32", kIntMaxF);
  B2_REQUIRE((int64_t)nfield * heads * dhead <= kIntMaxFHD,
             "interacting_bwd: field_size * head_num * att_embedding_size must be <= %d", kIntMaxFHD);
  if (batch <= 0) return B2CTR_OK;
  const size_t smem = (size_t)4 * nfield * heads * dhead * sizeof(float);
  const float scale = scaling ? 1.f / sqrtf((float)dhead) : 1.f;
  interacting_bwd_kernel<<<(unsigned)batch, 128, smem, ST>>>(q, k, v, out, dout, dq, dk, dv, dres, nfield,
                                                            heads, dhead, scale);
  B2_CHECK_LAUNCH("b2ctr_interacting_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_bi_interaction_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, float* out,
                                        int64_t ldo, int64_t batch, void* stream) {
  B2_REQUIRE(x && out && nfield > 0 && dim > 0 && ldx >= (int64_t)nfield * dim && ldo >= dim,
             "bi_interaction_fwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  bi_interaction_fwd_kernel<<<grid_for(batch, 8, 8), 256, 0, ST>>>(x, ldx, nfield, dim, out, ldo, batch);
  B2_CHECK_LAUNCH("b2ctr_bi_interaction_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_bi_interaction_bwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* g,
                                        int64_t ldg, float* dx, int64_t lddx, int64_t batch, void* stream) {
  B2_REQUIRE(x && g && dx && nfield > 0 && dim > 0 && ldg >= dim, "bi_interaction_bwd: bad arguments");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && lddx >= (int64_t)nfield * dim, "bi_interaction_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  bi_interaction_bwd_kernel<<<grid_for(batch, 8, 8), 256, 0, ST>>>(x, ldx, nfield, dim, g, ldg, dx, lddx, batch);
  B2_CHECK_LAUNCH("b2ctr_bi_interaction_bwd");
  return B2CTR_OK;
}

#define AFM_REQUIRE_SHAPE(what)                                                                             \
  B2_REQUIRE(nfield >= 2 && nfield <= kAfmMaxF && dim >= 1 && dim <= kAfmMaxE && factor >= 1 &&             \
                 factor <= kAfmMaxA,                                                                         \
             what ": needs 2 <= field count <= %d, 1 <= embedding_size <= %d and 1 <= attention_factor <= %d " \
                  "(got %d, %d, %d)",                                                                        \
             kAfmMaxF, kAfmMaxE, kAfmMaxA, nfield, dim, factor)

b2ctr_status_t b2ctr_afm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t factor,
                             const float* W, const float* bias, const float* h, float* att, int64_t ldo,
                             float* state, int64_t batch, void* stream) {
  B2_REQUIRE(x && W && bias && h && att && state, "afm_fwd: NULL pointer");
  AFM_REQUIRE_SHAPE("afm_fwd");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && ldo >= dim, "afm_fwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  AfmArgs a{x, ldx, nfield, dim, factor, W, bias, h, nullptr, 0, att, ldo, state, nullptr, 0, nullptr, batch};
  const cudaError_t err = afm_dispatch<AfmFwd>(afm_pad_e(dim), afm_pad_a(factor), a, ST);
  if (err != cudaSuccess) {
    set_error("afm_fwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_afm_fwd");
  return B2CTR_OK;
}

size_t b2ctr_afm_bwd_workspace_bytes(int32_t dim, int32_t factor, int64_t batch) {
  if (dim < 1 || factor < 1 || batch <= 0) return 0;
  const int EP = afm_pad_e(dim), AP = afm_pad_a(factor);
  return (size_t)afm_bwd_blocks(batch) * (size_t)(EP * AP + 2 * AP) * sizeof(float);
}

b2ctr_status_t b2ctr_afm_bwd(const float* g, int64_t ldg, const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                             int32_t factor, const float* W, const float* bias, const float* h, const float* state,
                             const float* att, int64_t lda, float* dx, int64_t lddx, float* dW, float* dbias,
                             float* dh, int64_t batch, void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(g && x && W && bias && h && state && att && dx && dW && dbias && dh, "afm_bwd: NULL pointer");
  AFM_REQUIRE_SHAPE("afm_bwd");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && lddx >= (int64_t)nfield * dim && ldg >= dim && lda >= dim,
             "afm_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  const size_t need = b2ctr_afm_bwd_workspace_bytes(dim, factor, batch);
  if (!workspace || workspace_bytes < need) {
    set_error("afm_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int EP = afm_pad_e(dim), AP = afm_pad_a(factor);
  float* partial = (float*)workspace;
  AfmArgs a{x, ldx, nfield, dim, factor, W, bias, h, g, ldg, const_cast<float*>(att), lda, const_cast<float*>(state),
            dx, lddx, partial, batch};
  const cudaError_t err = afm_dispatch<AfmBwd>(EP, AP, a, ST);
  if (err != cudaSuccess) {
    set_error("afm_bwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_afm_bwd");
  afm_reduce_kernel<<<(unsigned)ceil_div(dim * factor + 2 * factor, 128), 128, 0, ST>>>(
      partial, afm_bwd_blocks(batch), EP, AP, dim, factor, dW, dbias, dh);
  B2_CHECK_LAUNCH("b2ctr_afm_bwd(reduce)");
  return B2CTR_OK;
}

#define SENET_REQUIRE_SHAPE(what)                                                                         \
  B2_REQUIRE(nfield >= 2 && nfield <= kSenetMaxF && dim >= 1 && reduce >= 1 && reduce <= kSenetMaxF,       \
             what ": needs 2 <= field count <= %d, embedding_size >= 1 and 1 <= reduction size <= %d "        \
                  "(got %d, %d, %d)",                                                                      \
             kSenetMaxF, kSenetMaxF, nfield, dim, reduce)

b2ctr_status_t b2ctr_senet_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t reduce,
                               const float* W1, const float* W2, float* v, int64_t ldv, float* saved, int64_t batch,
                               void* stream) {
  B2_REQUIRE(x && W1 && W2 && v && saved, "senet_fwd: NULL pointer");
  SENET_REQUIRE_SHAPE("senet_fwd");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && ldv >= (int64_t)nfield * dim, "senet_fwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  senet_fwd_kernel<<<grid_for(batch, kSenetWarps, 8), kSenetWarps * 32, 0, ST>>>(x, ldx, nfield, dim, reduce, W1, W2,
                                                                                v, ldv, saved, batch);
  B2_CHECK_LAUNCH("b2ctr_senet_fwd");
  return B2CTR_OK;
}

size_t b2ctr_senet_bwd_workspace_bytes(int32_t nfield, int32_t reduce, int64_t batch) {
  if (nfield < 1 || reduce < 1 || batch <= 0) return 0;
  return (size_t)senet_bwd_blocks(batch) * 2 * (size_t)nfield * reduce * sizeof(float);
}

b2ctr_status_t b2ctr_senet_bwd(const float* g, int64_t ldg, const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                               int32_t reduce, const float* W1, const float* W2, const float* saved, float* dx,
                               int64_t lddx, float* dW1, float* dW2, int64_t batch, void* workspace,
                               size_t workspace_bytes, void* stream) {
  B2_REQUIRE(g && x && W1 && W2 && saved && dx && dW1 && dW2, "senet_bwd: NULL pointer");
  SENET_REQUIRE_SHAPE("senet_bwd");
  const int64_t w = (int64_t)nfield * dim;
  B2_REQUIRE(ldg >= w && ldx >= w && lddx >= w, "senet_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  const size_t need = b2ctr_senet_bwd_workspace_bytes(nfield, reduce, batch);
  if (!workspace || workspace_bytes < need) {
    set_error("senet_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  float* partial = (float*)workspace;
  const int nb = senet_bwd_blocks(batch);
  senet_bwd_kernel<<<nb, kSenetWarps * 32, 0, ST>>>(g, ldg, x, ldx, nfield, dim, reduce, W1, W2, saved, dx, lddx,
                                                   partial, batch);
  B2_CHECK_LAUNCH("b2ctr_senet_bwd");
  const int64_t fr = (int64_t)nfield * reduce;
  ordered_sum_kernel<<<(unsigned)ceil_div(fr, 128), 128, 0, ST>>>(partial, 2 * fr, nb, fr, dW1);
  ordered_sum_kernel<<<(unsigned)ceil_div(fr, 128), 128, 0, ST>>>(partial + fr, 2 * fr, nb, fr, dW2);
  B2_CHECK_LAUNCH("b2ctr_senet_bwd(reduce)");
  return B2CTR_OK;
}

#define BILINEAR_REQUIRE_SHAPE(what)                                                                          \
  B2_REQUIRE(nfield >= 2 && nfield <= kBiMaxF && dim >= 1 && dim <= kBiMaxE && type >= 0 && type <= 2,        \
             what ": needs 2 <= field count <= %d, 1 <= embedding_size <= %d and type 0 / 1 / 2 "               \
                  "(got %d, %d, %d)",                                                                         \
             kBiMaxF, kBiMaxE, nfield, dim, type)
#define BILINEAR_REQUIRE_WINDOW(what, ld, col0, pitch)                                                        \
  B2_REQUIRE(col0 >= 0 && pitch >= dim &&                                                                     \
                 ld >= col0 + (int64_t)(nfield * (nfield - 1) / 2 - 1) * pitch + dim,                         \
             what ": the pair window (col0 %lld, pitch %lld) does not fit a row of %lld",                     \
             (long long)col0, (long long)pitch, (long long)ld)

b2ctr_status_t b2ctr_bilinear_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t type,
                                  const float* W, float* out, int64_t ldo, int64_t col0, int64_t pitch, int64_t batch,
                                  void* stream) {
  B2_REQUIRE(x && W && out, "bilinear_fwd: NULL pointer");
  BILINEAR_REQUIRE_SHAPE("bilinear_fwd");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim, "bilinear_fwd: ldx too small");
  BILINEAR_REQUIRE_WINDOW("bilinear_fwd", ldo, col0, pitch);
  if (batch <= 0) return B2CTR_OK;
  BiArgs a{x, ldx, nfield, dim, type, W, out, ldo, col0, pitch, nullptr, 0, nullptr, 0, batch};
  const cudaError_t err = bi_dispatch<BiFwd>(bi_pad_e(dim), a, ST);
  if (err != cudaSuccess) {
    set_error("bilinear_fwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_bilinear_fwd");
  return B2CTR_OK;
}

size_t b2ctr_bilinear_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch) {
  if (nfield < 2 || dim < 1 || batch <= 0) return 0;
  return (size_t)bi_dw_chunks(nfield, batch) * (size_t)(nfield * (nfield - 1) / 2) * dim * dim * sizeof(float);
}

b2ctr_status_t b2ctr_bilinear_bwd(const float* g, int64_t ldg, int64_t gcol0, int64_t gpitch, const float* x,
                                  int64_t ldx, int32_t nfield, int32_t dim, int32_t type, const float* W, float* dx,
                                  int64_t lddx, float* dW, int64_t batch, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  B2_REQUIRE(g && x && W && (dx || dW), "bilinear_bwd: NULL pointer, or nothing to compute");
  BILINEAR_REQUIRE_SHAPE("bilinear_bwd");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && (!dx || lddx >= (int64_t)nfield * dim), "bilinear_bwd: ld too small");
  BILINEAR_REQUIRE_WINDOW("bilinear_bwd", ldg, gcol0, gpitch);
  if (batch <= 0) return B2CTR_OK;
  const size_t need = dW ? b2ctr_bilinear_bwd_workspace_bytes(nfield, dim, batch) : 0;
  if (dW && (!workspace || workspace_bytes < need)) {
    set_error("bilinear_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int nchunk = bi_dw_chunks(nfield, batch);
  BiArgs a{x, ldx, nfield, dim, type, W, const_cast<float*>(g), ldg, gcol0, gpitch, dx, lddx,
           dW ? (float*)workspace : nullptr, nchunk, batch};
  const cudaError_t err = bi_dispatch<BiBwd>(bi_pad_e(dim), a, ST);
  if (err != cudaSuccess) {
    set_error("bilinear_bwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_bilinear_bwd");
  if (dW) {
    const int64_t count = (int64_t)bi_num_weights(type, nfield) * dim * dim;
    bilinear_dw_reduce_kernel<<<grid_for(count, 256, 8), 256, 0, ST>>>((const float*)workspace, nfield, dim, type,
                                                                     nchunk, dW, count);
    B2_CHECK_LAUNCH("b2ctr_bilinear_bwd(reduce)");
  }
  return B2CTR_OK;
}

#define FWFM_REQUIRE_SHAPE(what)                                                                       \
  B2_REQUIRE(nfield >= 2 && nfield <= kFwMaxF && dim >= 1 && dim <= kFwMaxE,                            \
             what ": needs 2 <= field count <= %d and 1 <= embedding_size <= %d (got %d, %d)", kFwMaxF, \
             kFwMaxE, nfield, dim)

b2ctr_status_t b2ctr_fwfm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* r, float* out,
                              int64_t ldo, int64_t batch, void* stream) {
  FWFM_REQUIRE_SHAPE("fwfm_fwd");
  B2_REQUIRE(x && r && out, "fwfm_fwd: NULL pointer");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && ldo >= 1, "fwfm_fwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  // large F * E need more than the default 48 KB; the attribute belongs to the current device, so it is set per call
  const cudaError_t err = cudaFuncSetAttribute(fwfm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)fw_fwd_smem(nfield, dim));
  if (err != cudaSuccess) {
    set_error("fwfm_fwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  fwfm_fwd_kernel<<<grid_for(batch, kFwWarps, 8), kFwWarps * 32, fw_fwd_smem(nfield, dim), ST>>>(
      x, ldx, nfield, dim, r, out, ldo, batch);
  B2_CHECK_LAUNCH("b2ctr_fwfm_fwd");
  return B2CTR_OK;
}

size_t b2ctr_fwfm_bwd_workspace_bytes(int32_t nfield, int64_t batch) {
  if (nfield < 2 || batch <= 0) return 0;
  return (size_t)fw_bwd_blocks(batch) * (size_t)(nfield * (nfield - 1) / 2) * sizeof(float);
}

b2ctr_status_t b2ctr_fwfm_bwd(const float* g, int64_t ldg, const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                              const float* r, float* dx, int64_t lddx, float* dR, int64_t batch, void* workspace,
                              size_t workspace_bytes, void* stream) {
  FWFM_REQUIRE_SHAPE("fwfm_bwd");
  B2_REQUIRE(g && x && r && (dx || dR), "fwfm_bwd: NULL pointer, or nothing to compute");
  B2_REQUIRE(ldg >= 1 && ldx >= (int64_t)nfield * dim && (!dx || lddx >= (int64_t)nfield * dim),
             "fwfm_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  const size_t need = dR ? b2ctr_fwfm_bwd_workspace_bytes(nfield, batch) : 0;
  if (dR && (!workspace || workspace_bytes < need)) {
    set_error("fwfm_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const cudaError_t err = cudaFuncSetAttribute(fwfm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)fw_bwd_smem(nfield, dim));
  if (err != cudaSuccess) {
    set_error("fwfm_bwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  const int nb = fw_bwd_blocks(batch);
  float* partial = dR ? (float*)workspace : nullptr;
  fwfm_bwd_kernel<<<nb, kFwWarps * 32, fw_bwd_smem(nfield, dim), ST>>>(g, ldg, x, ldx, nfield, dim, r, dx, lddx,
                                                                     partial, batch);
  B2_CHECK_LAUNCH("b2ctr_fwfm_bwd");
  if (dR) {
    fwfm_dr_reduce_kernel<<<(unsigned)ceil_div((int64_t)nfield * nfield, 256), 256, 0, ST>>>(partial, nb, nfield, dR);
    B2_CHECK_LAUNCH("b2ctr_fwfm_bwd(reduce)");
  }
  return B2CTR_OK;
}

#define FEFM_REQUIRE_SHAPE(what)                                                                       \
  B2_REQUIRE(nfield >= 2 && nfield <= kFeMaxF && dim >= 1 && dim <= kFeMaxE,                            \
             what ": needs 2 <= field count <= %d and 1 <= embedding_size <= %d (got %d, %d)", kFeMaxF, \
             kFeMaxE, nfield, dim)

b2ctr_status_t b2ctr_fefm_sym(const float* W, int32_t npairs, int32_t dim, float* S, void* stream) {
  B2_REQUIRE(W && S && W != S, "fefm_sym: NULL or aliased pointer");
  B2_REQUIRE(npairs >= 1 && dim >= 1 && dim <= kFeMaxE, "fefm_sym: needs npairs >= 1 and 1 <= dim <= %d (got %d, %d)",
             kFeMaxE, npairs, dim);
  const int64_t count = (int64_t)npairs * dim * dim;
  fefm_sym_kernel<<<grid_for(count, 256, 8), 256, 0, ST>>>(W, dim, S, count);
  B2_CHECK_LAUNCH("b2ctr_fefm_sym");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_fefm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* S, float* out,
                              int64_t ldo, int64_t col0, int64_t batch, void* stream) {
  FEFM_REQUIRE_SHAPE("fefm_fwd");
  B2_REQUIRE(x && S && out, "fefm_fwd: NULL pointer");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim, "fefm_fwd: ldx too small");
  B2_REQUIRE(col0 >= 0 && ldo >= col0 + nfield * (nfield - 1) / 2,
             "fefm_fwd: the pair window (col0 %lld) does not fit a row of %lld", (long long)col0, (long long)ldo);
  if (batch <= 0) return B2CTR_OK;
  BiArgs a{x, ldx, nfield, dim, 2, S, out, ldo, col0, 1, nullptr, 0, nullptr, 0, batch};
  const cudaError_t err = bi_dispatch<FeFwd<false>>(bi_pad_e(dim), a, ST);
  if (err != cudaSuccess) {
    set_error("fefm_fwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_fefm_fwd");
  return B2CTR_OK;
}

size_t b2ctr_fefm_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch) {
  return b2ctr_bilinear_bwd_workspace_bytes(nfield, dim, batch);
}

b2ctr_status_t b2ctr_fefm_bwd(const float* g, int64_t ldg, int64_t gcol0, const float* x, int64_t ldx, int32_t nfield,
                              int32_t dim, const float* S, float* dx, int64_t lddx, float* dW, int64_t batch,
                              void* workspace, size_t workspace_bytes, void* stream) {
  FEFM_REQUIRE_SHAPE("fefm_bwd");
  B2_REQUIRE(g && x && S && (dx || dW), "fefm_bwd: NULL pointer, or nothing to compute");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && (!dx || lddx >= (int64_t)nfield * dim), "fefm_bwd: ld too small");
  B2_REQUIRE(gcol0 >= 0 && ldg >= gcol0 + nfield * (nfield - 1) / 2,
             "fefm_bwd: the pair window (col0 %lld) does not fit a row of %lld", (long long)gcol0, (long long)ldg);
  if (batch <= 0) return B2CTR_OK;
  const size_t need = dW ? b2ctr_fefm_bwd_workspace_bytes(nfield, dim, batch) : 0;
  if (dW && (!workspace || workspace_bytes < need)) {
    set_error("fefm_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int nchunk = bi_dw_chunks(nfield, batch);
  BiArgs a{x, ldx, nfield, dim, 2, S, const_cast<float*>(g), ldg, gcol0, 1, dx, lddx,
           dW ? (float*)workspace : nullptr, nchunk, batch};
  const cudaError_t err = bi_dispatch<FeBwd<false>>(bi_pad_e(dim), a, ST);
  if (err != cudaSuccess) {
    set_error("fefm_bwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_fefm_bwd");
  if (dW) {
    const int P = nfield * (nfield - 1) / 2;
    const int64_t count = (int64_t)P * dim * dim;
    fefm_dw_reduce_kernel<<<grid_for(count, 256, 8), 256, 0, ST>>>((const float*)workspace, P, dim, nchunk, dW, count);
    B2_CHECK_LAUNCH("b2ctr_fefm_bwd(reduce)");
  }
  return B2CTR_OK;
}

#define PNN_REQUIRE_SHAPE(what)                                                                        \
  B2_REQUIRE(nfield >= 2 && nfield <= kPnMaxF && dim >= 1 && dim <= kPnMaxE,                             \
             what ": needs 2 <= field count <= %d and 1 <= embedding_size <= %d (got %d, %d)", kPnMaxF, \
             kPnMaxE, nfield, dim)

static inline int64_t pn_out_cols(int nfield, int dim, int mode) {
  const int64_t P = (int64_t)nfield * (nfield - 1) / 2;
  return mode == B2CTR_PNN_ELEMENTWISE ? P * dim : P;
}

b2ctr_status_t b2ctr_pnn_inner_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t mode,
                                   const float* K, float* out, int64_t ldo, int64_t col0, int64_t batch,
                                   void* stream) {
  PNN_REQUIRE_SHAPE("pnn_inner_fwd");
  B2_REQUIRE(mode >= B2CTR_PNN_INNER && mode <= B2CTR_PNN_NUM, "pnn_inner_fwd: unknown mode %d", mode);
  B2_REQUIRE(x && out && (K || mode == B2CTR_PNN_INNER || mode == B2CTR_PNN_ELEMENTWISE),
             "pnn_inner_fwd: NULL pointer");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim, "pnn_inner_fwd: ldx too small");
  B2_REQUIRE(col0 >= 0 && ldo >= col0 + pn_out_cols(nfield, dim, mode),
             "pnn_inner_fwd: the pair window (col0 %lld) does not fit a row of %lld", (long long)col0,
             (long long)ldo);
  if (batch <= 0) return B2CTR_OK;
  const size_t smem = pn_fwd_smem(nfield, dim, mode);
  const bool stage_k = pn_stage_k(nfield, dim, mode);
  // large F * E need more than the default 48 KB; the attribute belongs to the current device, so it is set per call
  const cudaError_t err = pn_dispatch(mode, [&](auto m) {
    constexpr int kMode = decltype(m)::value;
    const cudaError_t e = cudaFuncSetAttribute(pnn_inner_fwd_kernel<kMode>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    pnn_inner_fwd_kernel<kMode><<<grid_for(batch, kPnWarps, 8), kPnWarps * 32, smem, ST>>>(
        x, ldx, nfield, dim, K, stage_k, out, ldo, col0, batch);
    return cudaSuccess;
  });
  if (err != cudaSuccess) {
    set_error("pnn_inner_fwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_pnn_inner_fwd");
  return B2CTR_OK;
}

size_t b2ctr_pnn_inner_bwd_workspace_bytes(int32_t nfield, int32_t dim, int32_t mode, int64_t batch) {
  if (nfield < 2 || dim < 1 || batch <= 0) return 0;
  const int nent = pn_dk_entries(nfield, dim, mode);
  if (nent == 0) return 0;
  return (size_t)pn_dk_chunks(nent, batch) * (size_t)nent * sizeof(float);
}

b2ctr_status_t b2ctr_pnn_inner_bwd(const float* g, int64_t ldg, int64_t gcol0, const float* x, int64_t ldx,
                                   int32_t nfield, int32_t dim, int32_t mode, const float* K, float* dx,
                                   int64_t lddx, float* dK, int64_t batch, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  PNN_REQUIRE_SHAPE("pnn_inner_bwd");
  B2_REQUIRE(mode >= B2CTR_PNN_INNER && mode <= B2CTR_PNN_NUM, "pnn_inner_bwd: unknown mode %d", mode);
  const bool weighted = mode == B2CTR_PNN_VEC || mode == B2CTR_PNN_NUM;
  B2_REQUIRE(g && x && (K || !weighted) && (dx || dK), "pnn_inner_bwd: NULL pointer, or nothing to compute");
  B2_REQUIRE(!dK || weighted, "pnn_inner_bwd: mode %d has no kernel weight", mode);
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && (!dx || lddx >= (int64_t)nfield * dim), "pnn_inner_bwd: ld too small");
  B2_REQUIRE(gcol0 >= 0 && ldg >= gcol0 + pn_out_cols(nfield, dim, mode),
             "pnn_inner_bwd: the pair window (col0 %lld) does not fit a row of %lld", (long long)gcol0,
             (long long)ldg);
  if (batch <= 0) return B2CTR_OK;
  const size_t need = dK ? b2ctr_pnn_inner_bwd_workspace_bytes(nfield, dim, mode, batch) : 0;
  if (dK && (!workspace || workspace_bytes < need)) {
    set_error("pnn_inner_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  if (dx) {
    const size_t smem = pn_dx_smem(nfield, dim);
    const cudaError_t err = pn_dispatch(mode, [&](auto m) {
      constexpr int kMode = decltype(m)::value;
      const cudaError_t e = cudaFuncSetAttribute(pnn_inner_dx_kernel<kMode>,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      pnn_inner_dx_kernel<kMode><<<grid_for(batch, kPnWarps, 8), kPnWarps * 32, smem, ST>>>(
          g, ldg, gcol0, x, ldx, nfield, dim, K, dx, lddx, batch);
      return cudaSuccess;
    });
    if (err != cudaSuccess) {
      set_error("pnn_inner_bwd: %s", cudaGetErrorString(err));
      return B2CTR_ERR_CUDA;
    }
    B2_CHECK_LAUNCH("b2ctr_pnn_inner_bwd(dx)");
  }
  if (dK) {
    const int nent = pn_dk_entries(nfield, dim, mode), nchunk = pn_dk_chunks(nent, batch);
    float* partial = (float*)workspace;
    pnn_inner_dk_kernel<<<dim3(pn_dk_tiles(nent), nchunk), 256, 0, ST>>>(
        g, ldg, gcol0, x, ldx, nfield, dim, mode == B2CTR_PNN_VEC, partial, nent, nchunk, batch);
    B2_CHECK_LAUNCH("b2ctr_pnn_inner_bwd(dK)");
    ordered_sum_kernel<<<grid_for(nent, 256, 8), 256, 0, ST>>>(partial, nent, nchunk, nent, dK);
    B2_CHECK_LAUNCH("b2ctr_pnn_inner_bwd(reduce)");
  }
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_pnn_outer_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* K,
                                   float* out, int64_t ldo, int64_t col0, int64_t batch, void* stream) {
  PNN_REQUIRE_SHAPE("pnn_outer_fwd");
  B2_REQUIRE(x && K && out, "pnn_outer_fwd: NULL pointer");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim, "pnn_outer_fwd: ldx too small");
  B2_REQUIRE(col0 >= 0 && ldo >= col0 + nfield * (nfield - 1) / 2,
             "pnn_outer_fwd: the pair window (col0 %lld) does not fit a row of %lld", (long long)col0, (long long)ldo);
  if (batch <= 0) return B2CTR_OK;
  BiArgs a{x, ldx, nfield, dim, 2, K, out, ldo, col0, 1, nullptr, 0, nullptr, 0, batch};
  const cudaError_t err = bi_dispatch<FeFwd<true>>(bi_pad_e(dim), a, ST);
  if (err != cudaSuccess) {
    set_error("pnn_outer_fwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_pnn_outer_fwd");
  return B2CTR_OK;
}

size_t b2ctr_pnn_outer_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch) {
  return b2ctr_bilinear_bwd_workspace_bytes(nfield, dim, batch);
}

b2ctr_status_t b2ctr_pnn_outer_bwd(const float* g, int64_t ldg, int64_t gcol0, const float* x, int64_t ldx,
                                   int32_t nfield, int32_t dim, const float* K, float* dx, int64_t lddx, float* dK,
                                   int64_t batch, void* workspace, size_t workspace_bytes, void* stream) {
  PNN_REQUIRE_SHAPE("pnn_outer_bwd");
  B2_REQUIRE(g && x && K && (dx || dK), "pnn_outer_bwd: NULL pointer, or nothing to compute");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && (!dx || lddx >= (int64_t)nfield * dim), "pnn_outer_bwd: ld too small");
  B2_REQUIRE(gcol0 >= 0 && ldg >= gcol0 + nfield * (nfield - 1) / 2,
             "pnn_outer_bwd: the pair window (col0 %lld) does not fit a row of %lld", (long long)gcol0,
             (long long)ldg);
  if (batch <= 0) return B2CTR_OK;
  const size_t need = dK ? b2ctr_pnn_outer_bwd_workspace_bytes(nfield, dim, batch) : 0;
  if (dK && (!workspace || workspace_bytes < need)) {
    set_error("pnn_outer_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const int nchunk = bi_dw_chunks(nfield, batch);
  BiArgs a{x, ldx, nfield, dim, 2, K, const_cast<float*>(g), ldg, gcol0, 1, dx, lddx,
           dK ? (float*)workspace : nullptr, nchunk, batch};
  const cudaError_t err = bi_dispatch<FeBwd<true>>(bi_pad_e(dim), a, ST);
  if (err != cudaSuccess) {
    set_error("pnn_outer_bwd: %s", cudaGetErrorString(err));
    return B2CTR_ERR_CUDA;
  }
  B2_CHECK_LAUNCH("b2ctr_pnn_outer_bwd");
  if (dK) {
    const int P = nfield * (nfield - 1) / 2;
    const int64_t count = (int64_t)P * dim * dim;
    pnn_mat_dk_reduce_kernel<<<grid_for(count, 256, 8), 256, 0, ST>>>((const float*)workspace, P, dim, nchunk, dK,
                                                                      count);
    B2_CHECK_LAUNCH("b2ctr_pnn_outer_bwd(reduce)");
  }
  return B2CTR_OK;
}

static bool reg_aligned(const float* p, int64_t ld, int64_t col) {
  return !p || (((uintptr_t)(p + col) & 15) == 0 && ld % 4 == 0);
}

// the checks the forward and the backward share: mode, limits, operands and the windows of u / y0 / y1
static b2ctr_status_t reg_check(const b2ctr_regulate_t* a, const char* what) {
  B2_REQUIRE(a, "%s: NULL descriptor", what);
  B2_REQUIRE(a->mode >= B2CTR_REGULATE_COPY && a->mode <= B2CTR_REGULATE_ATTENTION, "%s: unknown mode %d", what,
             a->mode);
  B2_REQUIRE(a->nfield >= 1 && a->nfield <= kRegMaxF && a->dim >= 1 && a->dim <= kRegMaxE,
             "%s: needs 1 <= field count <= %d and 1 <= embedding_size <= %d (got %d, %d)", what, kRegMaxF, kRegMaxE,
             a->nfield, a->dim);
  const int64_t d = (int64_t)a->nfield * a->dim;
  B2_REQUIRE(a->batch >= 0, "%s: negative batch", what);
  B2_REQUIRE(a->x && a->ldx >= d, "%s: x is NULL or its pitch is below %lld", what, (long long)d);
  B2_REQUIRE(a->mode == B2CTR_REGULATE_COPY || (a->h && a->ldh >= d), "%s: h is NULL or its pitch is too small",
             what);
  B2_REQUIRE(a->mode != B2CTR_REGULATE_ATTENTION || (a->ax && a->ah && a->ldax >= d && a->ldah >= d),
             "%s: attention weights NULL or their pitch too small", what);
  B2_REQUIRE((!a->y0 || a->g0) && (!a->y1 || a->g1), "%s: a gated output without its gate weight", what);
  B2_REQUIRE((!a->u || (a->ucol >= 0 && a->ldu >= a->ucol + d)) && (!a->y0 || (a->y0col >= 0 && a->ldy0 >= a->y0col + d)) &&
                 (!a->y1 || (a->y1col >= 0 && a->ldy1 >= a->y1col + d)),
             "%s: an output window does not fit its row", what);
  return B2CTR_OK;
}

static bool reg_vec(const b2ctr_regulate_t* a) {
  return a->dim % 4 == 0 && reg_aligned(a->x, a->ldx, 0) && reg_aligned(a->h, a->ldh, 0) &&
         reg_aligned(a->ax, a->ldax, 0) && reg_aligned(a->ah, a->ldah, 0) && reg_aligned(a->u, a->ldu, a->ucol) &&
         reg_aligned(a->y0, a->ldy0, a->y0col) && reg_aligned(a->y1, a->ldy1, a->y1col) &&
         reg_aligned(a->dx, a->lddx, 0) && reg_aligned(a->dh, a->lddh, 0) && reg_aligned(a->dax, a->lddax, 0) &&
         reg_aligned(a->dah, a->lddah, 0);
}

b2ctr_status_t b2ctr_regulate_fwd(const b2ctr_regulate_t* a, void* stream) {
  const b2ctr_status_t st = reg_check(a, "regulate_fwd");
  if (st != B2CTR_OK) return st;
  B2_REQUIRE(a->u || a->y0 || a->y1, "regulate_fwd: no output");
  if (a->batch == 0) return B2CTR_OK;
  const int64_t d = (int64_t)a->nfield * a->dim;
  const bool vec = reg_vec(a);
  reg_dispatch(a->mode, vec, [&](auto v, auto m) {
    constexpr int V = decltype(v)::value, kMode = decltype(m)::value;
    regulate_fwd_kernel<V, kMode><<<grid_for(a->batch * d / V, kRegThreads, 8), kRegThreads, 0, ST>>>(*a);
    return cudaSuccess;
  });
  B2_CHECK_LAUNCH("b2ctr_regulate_fwd");
  return B2CTR_OK;
}

size_t b2ctr_regulate_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch) {
  if (nfield < 1 || dim < 1 || batch <= 0) return 0;
  return (size_t)(reg_chunks(batch) + 1) * 2 * (size_t)nfield * sizeof(float);
}

b2ctr_status_t b2ctr_regulate_bwd(const b2ctr_regulate_t* a, void* workspace, size_t workspace_bytes, void* stream) {
  const b2ctr_status_t st = reg_check(a, "regulate_bwd");
  if (st != B2CTR_OK) return st;
  const bool want_dg = a->dg0 || a->dg1;
  B2_REQUIRE(a->dx || a->dh || a->dax || a->dah || want_dg, "regulate_bwd: nothing to compute");
  B2_REQUIRE((!a->dg0 || a->y0) && (!a->dg1 || a->y1), "regulate_bwd: a gate gradient without its incoming gradient");
  const int64_t d = (int64_t)a->nfield * a->dim;
  B2_REQUIRE((!a->dx || a->lddx >= d) && (!a->dh || a->lddh >= d) && (!a->dax || a->lddax >= d) &&
                 (!a->dah || a->lddah >= d),
             "regulate_bwd: a gradient pitch is below %lld", (long long)d);
  if (a->batch == 0) return B2CTR_OK;
  const size_t need = want_dg ? b2ctr_regulate_bwd_workspace_bytes(a->nfield, a->dim, a->batch) : 0;
  if (want_dg && (!workspace || workspace_bytes < need)) {
    set_error("regulate_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const bool vec = reg_vec(a);
  const int V = vec ? 4 : 1, W = reg_tile(a->dim, V), R = kRegThreads / (W / V), nchunk = reg_chunks(a->batch);
  const int ntile = (int)ceil_div(d, W);
  float* partial = want_dg ? (float*)workspace : nullptr;
  const b2ctr_regulate_t k = *a;
  reg_dispatch(a->mode, vec, [&](auto v, auto m) {
    constexpr int VV = decltype(v)::value, kMode = decltype(m)::value;
    regulate_bwd_kernel<VV, kMode><<<dim3(nchunk, ntile), kRegThreads, 0, ST>>>(k, W, R, nchunk, partial);
    return cudaSuccess;
  });
  B2_CHECK_LAUNCH("b2ctr_regulate_bwd");
  if (want_dg) {
    float* sums = partial + (int64_t)nchunk * 2 * a->nfield;
    ordered_sum_kernel<<<grid_for(2 * a->nfield, 256, 8), 256, 0, ST>>>(partial, 2 * a->nfield, nchunk,
                                                                         2 * a->nfield, sums);
    B2_CHECK_LAUNCH("b2ctr_regulate_bwd(reduce)");
    regulate_dg_kernel<<<1, 64, 0, ST>>>(k, sums);
    B2_CHECK_LAUNCH("b2ctr_regulate_bwd(gates)");
  }
  return B2CTR_OK;
}

// ---- CCPM's convolution stack ---------------------------------------------------------------------
static b2ctr_status_t conv_plan(const b2ctr_conv_stack_t* a, const char* what, ConvPlan* P) {
  B2_REQUIRE(a, "%s: NULL descriptor", what);
  B2_REQUIRE(a->struct_size == (int32_t)sizeof(b2ctr_conv_stack_t), "%s: struct_size %d, expected %d", what,
             a->struct_size, (int)sizeof(b2ctr_conv_stack_t));
  B2_REQUIRE(a->nstage >= 1 && a->nstage <= B2CTR_CONV_STACK_MAX_STAGES, "%s: needs 1 to %d stages (got %d)", what,
             B2CTR_CONV_STACK_MAX_STAGES, a->nstage);
  B2_REQUIRE(a->rows >= 1 && a->rows <= 64, "%s: needs 1 <= rows <= 64 (got %d)", what, a->rows);
  B2_REQUIRE(a->dim >= 1 && a->channels >= 1 && a->channels <= 16, "%s: needs dim >= 1 and 1 <= channels <= 16", what);
  B2_REQUIRE(a->batch >= 0, "%s: negative batch", what);
  const int64_t in_w = (int64_t)a->rows * a->dim * a->channels;
  B2_REQUIRE(a->x && a->xcol >= 0 && a->ldx >= a->xcol + in_w, "%s: x is NULL or its window does not fit its row", what);
  *P = ConvPlan{};
  P->nstage = a->nstage;
  int rows = a->rows, C = a->channels, off = rows * C, G = C, maxmap = rows * C, nw = 0;
  for (int s = 0; s < a->nstage; ++s) {
    const b2ctr_conv_stage_t& st = a->stage[s];
    ConvStagePlan& p = P->s[s];
    p.kind = st.kind;
    p.rows_in = rows;
    p.cin = C;
    p.in_off = s == 0 ? 0 : P->s[s - 1].out_off;
    p.idx_off = -1;
    if (st.kind == B2CTR_CONV_STAGE_CONV) {
      B2_REQUIRE(st.width >= 1 && st.width <= 32 && st.filters >= 1 && st.filters <= 16,
                 "%s: stage %d needs 1 <= width <= 32 and 1 <= filters <= 16 (got %d, %d)", what, s, st.width,
                 st.filters);
      B2_REQUIRE(st.act >= B2CTR_ACT_NONE && st.act <= B2CTR_ACT_TANH, "%s: stage %d: unknown activation %d", what, s,
                 st.act);
      B2_REQUIRE(st.kernel, "%s: stage %d: NULL kernel", what, s);
      p.width = st.width;
      p.pad = (st.width - 1) / 2;
      p.act = st.act;
      p.rows_out = rows;
      p.cout = st.filters;
      p.w_off = nw;
      p.nw = st.width * C * st.filters + st.filters;
      nw += p.nw;
      p.out_off = off;
      off += rows * st.filters;
      C = st.filters;
    } else {
      B2_REQUIRE(st.kind == B2CTR_CONV_STAGE_KMAX, "%s: stage %d: unknown kind %d", what, s, st.kind);
      B2_REQUIRE(st.k >= 1 && st.k <= rows, "%s: stage %d needs 1 <= k <= %d rows (got %d)", what, s, rows, st.k);
      p.k = st.k;
      p.rows_out = st.k;
      p.cout = C;
      p.out_off = off;
      p.idx_off = off + st.k * C;
      off += 2 * st.k * C;
      rows = st.k;
    }
    G = std::max(G, C);
    maxmap = std::max(maxmap, rows * C);
  }
  P->G = G;
  P->nw = nw;
  P->max_map = maxmap;
  P->ga_off = off;
  P->gb_off = off + maxmap;
  P->map_floats = off + 2 * maxmap;
  P->rows_out = rows;
  P->cout = C;
  const size_t smem = (2 * (size_t)nw + (size_t)kConvCols * P->map_floats) * sizeof(float);
  B2_REQUIRE(smem <= kConvSmemCap, "%s: the backward needs %zu bytes of shared memory, above the %zu limit", what, smem,
             kConvSmemCap);
  const int64_t out_w = (int64_t)rows * a->dim * C;
  B2_REQUIRE(a->out && a->outcol >= 0 && a->ldout >= a->outcol + out_w,
             "%s: out is NULL or its window does not fit its row", what);
  return B2CTR_OK;
}

static size_t conv_fwd_smem(const ConvPlan& P) { return ((size_t)P.nw + (size_t)kConvCols * 2 * P.max_map) * sizeof(float); }
static size_t conv_bwd_smem(const ConvPlan& P) { return (2 * (size_t)P.nw + (size_t)kConvCols * P.map_floats) * sizeof(float); }
static int conv_bwd_blocks(const b2ctr_conv_stack_t* a, const ConvPlan& P) {
  const int per_sm = std::max(1, (int)((228 * 1024) / (conv_bwd_smem(P) + 1024)));
  return grid_for(a->batch * a->dim, kConvCols, std::min(per_sm, 2048 / (kConvCols * P.G)));
}

b2ctr_status_t b2ctr_conv_stack_fwd(const b2ctr_conv_stack_t* a, void* stream) {
  ConvPlan P;
  const b2ctr_status_t st = conv_plan(a, "conv_stack_fwd", &P);
  if (st != B2CTR_OK) return st;
  if (a->batch == 0) return B2CTR_OK;
  const size_t smem = conv_fwd_smem(P);
  if (cudaFuncSetAttribute(conv_stack_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("conv_stack_fwd: cannot reserve %zu bytes of shared memory", smem);
    return B2CTR_ERR_CUDA;
  }
  const int64_t nblk = ceil_div(a->batch * a->dim, kConvCols);
  conv_stack_fwd_kernel<<<(unsigned)nblk, kConvCols * P.G, smem, ST>>>(*a, P);
  B2_CHECK_LAUNCH("b2ctr_conv_stack_fwd");
  return B2CTR_OK;
}

size_t b2ctr_conv_stack_bwd_workspace_bytes(const b2ctr_conv_stack_t* a) {
  ConvPlan P;
  if (conv_plan(a, "conv_stack_bwd_workspace_bytes", &P) != B2CTR_OK || a->batch <= 0) return 0;
  return (size_t)conv_bwd_blocks(a, P) * P.nw * sizeof(float);
}

b2ctr_status_t b2ctr_conv_stack_bwd(const b2ctr_conv_stack_t* a, void* workspace, size_t workspace_bytes, void* stream) {
  ConvPlan P;
  const b2ctr_status_t st = conv_plan(a, "conv_stack_bwd", &P);
  if (st != B2CTR_OK) return st;
  const int64_t in_w = (int64_t)a->rows * a->dim * a->channels;
  B2_REQUIRE(!a->dx || (a->dxcol >= 0 && a->lddx >= a->dxcol + in_w), "conv_stack_bwd: the dx window does not fit its row");
  bool want_dw = false;
  for (int s = 0; s < a->nstage; ++s)
    if (a->stage[s].kind == B2CTR_CONV_STAGE_CONV) want_dw = want_dw || a->stage[s].dkernel || a->stage[s].dbias;
  B2_REQUIRE(a->dx || want_dw, "conv_stack_bwd: nothing to compute");
  if (a->batch == 0) {
    // no column: the weight gradients are zero
    for (int s = 0; s < a->nstage; ++s) {
      const ConvStagePlan& p = P.s[s];
      if (p.kind != B2CTR_CONV_STAGE_CONV) continue;
      if (a->stage[s].dkernel) cudaMemsetAsync(a->stage[s].dkernel, 0, sizeof(float) * (p.nw - p.cout), ST);
      if (a->stage[s].dbias) cudaMemsetAsync(a->stage[s].dbias, 0, sizeof(float) * p.cout, ST);
    }
    return B2CTR_OK;
  }
  const int nblk = conv_bwd_blocks(a, P);
  const size_t need = want_dw ? (size_t)nblk * P.nw * sizeof(float) : 0;
  if (want_dw && (!workspace || workspace_bytes < need)) {
    set_error("conv_stack_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  const size_t smem = conv_bwd_smem(P);
  if (cudaFuncSetAttribute(conv_stack_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    set_error("conv_stack_bwd: cannot reserve %zu bytes of shared memory", smem);
    return B2CTR_ERR_CUDA;
  }
  float* partial = want_dw ? (float*)workspace : nullptr;
  conv_stack_bwd_kernel<<<nblk, kConvCols * P.G, smem, ST>>>(*a, P, partial);
  B2_CHECK_LAUNCH("b2ctr_conv_stack_bwd");
  for (int s = 0; s < a->nstage && want_dw; ++s) {
    const ConvStagePlan& p = P.s[s];
    if (p.kind != B2CTR_CONV_STAGE_CONV) continue;
    const int nk = p.nw - p.cout;
    if (a->stage[s].dkernel) {
      ordered_sum_kernel<<<grid_for(nk, 256, 8), 256, 0, ST>>>(partial + p.w_off, P.nw, nblk, nk, a->stage[s].dkernel);
      B2_CHECK_LAUNCH("b2ctr_conv_stack_bwd(dkernel)");
    }
    if (a->stage[s].dbias) {
      ordered_sum_kernel<<<1, 32, 0, ST>>>(partial + p.w_off + nk, P.nw, nblk, p.cout, a->stage[s].dbias);
      B2_CHECK_LAUNCH("b2ctr_conv_stack_bwd(dbias)");
    }
  }
  return B2CTR_OK;
}

// ---- FLEN's FieldWiseBiInteraction ----------------------------------------------------------------
static bool fwbi_aligned(const void* p, int64_t ld) { return !p || (((uintptr_t)p & 15) == 0 && ld % 4 == 0); }

// the checks the forward and the backward share, and the kernels' arguments (the fields sorted by group)
static b2ctr_status_t fwbi_args(const b2ctr_field_wise_bi_t* a, const char* what, FwbiArgs* k, bool* vec) {
  B2_REQUIRE(a, "%s: NULL descriptor", what);
  B2_REQUIRE(a->struct_size == (int32_t)sizeof(b2ctr_field_wise_bi_t), "%s: struct_size %d, expected %d", what,
             a->struct_size, (int)sizeof(b2ctr_field_wise_bi_t));
  B2_REQUIRE(a->ngroup >= 2 && a->ngroup <= kFwbiMaxG, "%s: needs 2 <= groups <= %d (got %d)", what, kFwbiMaxG,
             a->ngroup);
  B2_REQUIRE(a->nfield >= a->ngroup && a->nfield <= B2CTR_FWBI_MAX_FIELDS, "%s: needs groups <= fields <= %d (got %d)",
             what, B2CTR_FWBI_MAX_FIELDS, a->nfield);
  B2_REQUIRE(a->dim >= 1 && a->dim <= kFwbiMaxE, "%s: needs 1 <= embedding_size <= %d (got %d)", what, kFwbiMaxE,
             a->dim);
  B2_REQUIRE(a->batch >= 0, "%s: negative batch", what);
  B2_REQUIRE(a->x && a->ldx >= a->dim && a->ldx < ((int64_t)1 << 31), "%s: x is NULL or its pitch is out of range",
             what);
  B2_REQUIRE(a->kernel_mf && a->kernel_fm, "%s: NULL kernel_mf / kernel_fm", what);
  B2_REQUIRE(a->out && a->outcol >= 0 && a->ldout >= a->outcol + a->dim, "%s: out is NULL or its window does not fit",
             what);
  *k = FwbiArgs{};
  int count[kFwbiMaxG + 1] = {0};
  bool cols4 = true;
  for (int f = 0; f < a->nfield; ++f) {
    B2_REQUIRE(a->group[f] >= 0 && a->group[f] < a->ngroup, "%s: field %d: group %d outside [0, %d)", what, f,
               a->group[f], a->ngroup);
    B2_REQUIRE(a->col[f] >= 0 && a->col[f] + a->dim <= a->ldx, "%s: field %d: column %lld does not fit the row", what,
               f, (long long)a->col[f]);
    ++count[a->group[f] + 1];
    cols4 = cols4 && a->col[f] % 4 == 0;
  }
  for (int g = 0; g < a->ngroup; ++g) {
    B2_REQUIRE(count[g + 1] > 0, "%s: group %d has no field", what, g);
    k->start[g + 1] = k->start[g] + count[g + 1];
  }
  int fill[kFwbiMaxG];
  for (int g = 0; g < a->ngroup; ++g) fill[g] = k->start[g];
  for (int f = 0; f < a->nfield; ++f) k->cols[fill[a->group[f]]++] = (int)a->col[f];
  k->F = a->nfield, k->G = a->ngroup, k->E = a->dim, k->dx_accumulate = a->dx_accumulate != 0;
  k->batch = a->batch;
  k->x = a->x, k->ldx = a->ldx;
  k->kmf = a->kernel_mf, k->kfm = a->kernel_fm, k->bmf = a->bias_mf, k->bfm = a->bias_fm;
  k->out = a->out, k->ldout = a->ldout, k->outcol = a->outcol;
  k->dx = a->dx, k->lddx = a->lddx;
  *vec = a->dim % 4 == 0 && cols4 && fwbi_aligned(a->x, a->ldx) && fwbi_aligned(a->out + a->outcol, a->ldout) &&
         fwbi_aligned(a->dx, a->lddx);
  return B2CTR_OK;
}

static inline int fwbi_pitch(const b2ctr_field_wise_bi_t* a) {
  return a->ngroup * (a->ngroup - 1) / 2 + a->ngroup + a->dim;
}

b2ctr_status_t b2ctr_field_wise_bi_fwd(const b2ctr_field_wise_bi_t* a, void* stream) {
  FwbiArgs k;
  bool vec;
  const b2ctr_status_t st = fwbi_args(a, "field_wise_bi_fwd", &k, &vec);
  if (st != B2CTR_OK) return st;
  if (a->batch == 0) return B2CTR_OK;
  const int V = vec ? 4 : 1, R = kFwbiThreads / (a->dim / V);
  const int grid = grid_for(ceil_div(a->batch, R), 1, 8);
  if (vec)
    fwbi_fwd_kernel<4><<<grid, kFwbiThreads, 0, ST>>>(k);
  else
    fwbi_fwd_kernel<1><<<grid, kFwbiThreads, 0, ST>>>(k);
  B2_CHECK_LAUNCH("b2ctr_field_wise_bi_fwd");
  return B2CTR_OK;
}

size_t b2ctr_field_wise_bi_bwd_workspace_bytes(const b2ctr_field_wise_bi_t* a) {
  FwbiArgs k;
  bool vec;
  if (fwbi_args(a, "field_wise_bi_bwd_workspace_bytes", &k, &vec) != B2CTR_OK || a->batch <= 0) return 0;
  return (size_t)fwbi_chunks(a->batch) * fwbi_pitch(a) * sizeof(float);
}

b2ctr_status_t b2ctr_field_wise_bi_bwd(const b2ctr_field_wise_bi_t* a, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  FwbiArgs k;
  bool vec;
  const b2ctr_status_t st = fwbi_args(a, "field_wise_bi_bwd", &k, &vec);
  if (st != B2CTR_OK) return st;
  if (a->dx)
    for (int f = 0; f < a->nfield; ++f)
      B2_REQUIRE(a->col[f] + a->dim <= a->lddx, "field_wise_bi_bwd: field %d does not fit a row of dx", f);
  const int P = a->ngroup * (a->ngroup - 1) / 2;
  const bool want_dw = a->dkernel_mf || a->dkernel_fm || a->dbias_mf || a->dbias_fm;
  B2_REQUIRE(a->dx || want_dw, "field_wise_bi_bwd: nothing to compute");
  if (a->batch == 0) {
    // no sample: the weight gradients are zero
    if (a->dkernel_mf) cudaMemsetAsync(a->dkernel_mf, 0, sizeof(float) * P, ST);
    if (a->dkernel_fm) cudaMemsetAsync(a->dkernel_fm, 0, sizeof(float) * a->ngroup, ST);
    if (a->dbias_mf) cudaMemsetAsync(a->dbias_mf, 0, sizeof(float) * a->dim, ST);
    if (a->dbias_fm) cudaMemsetAsync(a->dbias_fm, 0, sizeof(float) * a->dim, ST);
    return B2CTR_OK;
  }
  const int nchunk = fwbi_chunks(a->batch), pitch = fwbi_pitch(a);
  const size_t need = want_dw ? (size_t)nchunk * pitch * sizeof(float) : 0;
  if (want_dw && (!workspace || workspace_bytes < need)) {
    set_error("field_wise_bi_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  float* partial = want_dw ? (float*)workspace : nullptr;
  if (vec)
    fwbi_bwd_kernel<4><<<nchunk, kFwbiThreads, 0, ST>>>(k, nchunk, partial, pitch);
  else
    fwbi_bwd_kernel<1><<<nchunk, kFwbiThreads, 0, ST>>>(k, nchunk, partial, pitch);
  B2_CHECK_LAUNCH("b2ctr_field_wise_bi_bwd");
  const struct { float* out; int off, count; } sums[4] = {
      {a->dkernel_mf, 0, P}, {a->dkernel_fm, P, a->ngroup}, {a->dbias_mf, P + a->ngroup, a->dim},
      {a->dbias_fm, P + a->ngroup, a->dim}};
  for (const auto& s : sums) {
    if (!s.out) continue;
    ordered_sum_kernel<<<grid_for(s.count, 256, 8), 256, 0, ST>>>(partial + s.off, pitch, nchunk, s.count, s.out);
    B2_CHECK_LAUNCH("b2ctr_field_wise_bi_bwd(reduce)");
  }
  return B2CTR_OK;
}

}  // extern "C"
