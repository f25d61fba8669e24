// interaction.cu — CrossNet, CIN helpers, InteractingLayer attention core (sm_90a).
//
// Reference math restated (never copied): deepctr/layers/interaction.py:410-424 (CrossNet),
// :277-325 (CIN), :754-779 (InteractingLayer).  Pairwise reductions use warp shuffles; the dense
// contractions (CIN feature-map contraction, Q/K/V projections, CrossNet-matrix) go through b2ctr_gemm.
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
  if (batch <= 0) return B2CTR_OK;
  const size_t smem = (size_t)2 * nfield * heads * dhead * sizeof(float);
  B2_REQUIRE(smem <= 48 * 1024, "interacting_fwd: F*H*D too large for shared memory");
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
  if (batch <= 0) return B2CTR_OK;
  const size_t smem = (size_t)4 * nfield * heads * dhead * sizeof(float);
  B2_REQUIRE(smem <= 48 * 1024, "interacting_bwd: F*H*D too large for shared memory");
  const float scale = scaling ? 1.f / sqrtf((float)dhead) : 1.f;
  interacting_bwd_kernel<<<(unsigned)batch, 128, smem, ST>>>(q, k, v, out, dout, dq, dk, dv, dres, nfield,
                                                            heads, dhead, scale);
  B2_CHECK_LAUNCH("b2ctr_interacting_bwd");
  return B2CTR_OK;
}

}  // extern "C"
