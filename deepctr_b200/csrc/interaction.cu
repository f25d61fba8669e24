// interaction.cu — CrossNet, CIN helpers, InteractingLayer attention core (sm_90a).
//
// Reference math restated (never copied): deepctr/layers/interaction.py:410-424 (CrossNet),
// :277-325 (CIN), :754-779 (InteractingLayer), :1113-1126 (SENETLayer), :1190-1209 (BilinearInteraction).  Pairwise reductions use warp shuffles; the dense
// contractions (CIN feature-map contraction, Q/K/V projections, CrossNet-matrix) go through b2ctr_gemm.
#include <algorithm>

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

// M[r][c] = W[r][c] (or W[c][r] when trans), zero outside [E, E]
template <int EP>
__device__ __forceinline__ void bi_stage_w(float* M, const float* __restrict__ W, int E, bool trans) {
  for (int k = threadIdx.x; k < EP * EP; k += blockDim.x) {
    const int r = k / EP, c = k - r * EP;
    M[k] = (r < E && c < E) ? (trans ? W[c * E + r] : W[r * E + c]) : 0.f;
  }
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

template <int EP>
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
        tv = a.out[b * a.ldo + a.col0 + (int64_t)p * a.pitch + e] * a.x[b * a.ldx + j * E + e];
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

}  // extern "C"
