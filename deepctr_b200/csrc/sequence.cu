// sequence.cu — DIN local-activation attention pieces, standalone sequence pooling / weighting,
// Dice / BatchNormalization statistics, dropout (sm_90a).
//
// Reference math restated (never copied): deepctr/layers/core.py:94-108 (LocalActivationUnit input),
// deepctr/layers/sequence.py:76-106, :155-183, :261-298, deepctr/layers/activation.py:59-64.
#include "common.cuh"

namespace b2ctr {

constexpr float kNegPad = -4294967295.f;  // -2^32 + 1 (rounds to -2^32 in fp32, as in TF)

// att_in[b,t,:] = [q, k, q-k, q*k]   (core.py:98-101); q is [B,1,E] broadcast over T
__global__ void din_att_input_fwd_kernel(const float* __restrict__ q, int64_t ldq,
                                         const float* __restrict__ k, int64_t ldk, float* out, int64_t batch,
                                         int T, int E) {
  const int64_t total = batch * T * E;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int e = (int)(i % E);
    const int64_t bt = i / E;
    const int64_t b = bt / T;
    const int t = (int)(bt - b * T);
    const float qv = q[b * ldq + e], kv = k[b * ldk + (int64_t)t * E + e];
    float* o = out + bt * 4 * E;
    o[e] = qv;
    o[E + e] = kv;
    o[2 * E + e] = qv - kv;
    o[3 * E + e] = qv * kv;
  }
}
// dk[b,t,e] = g2 - g3 + g4*q ;  dq[b,e] = sum_t (g1 + g3 + g4*k)   (one thread per (b,e), t sequential)
__global__ void din_att_input_bwd_kernel(const float* __restrict__ q, int64_t ldq,
                                         const float* __restrict__ k, int64_t ldk,
                                         const float* __restrict__ g, float* dq, float* dk, int64_t batch,
                                         int T, int E) {
  const int64_t total = batch * E;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / E;
    const int e = (int)(i - b * E);
    const float qv = q[b * ldq + e];
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {
      const float* gg = g + (b * T + t) * 4 * E;
      const float kv = k[b * ldk + (int64_t)t * E + e];
      acc += gg[e] + gg[2 * E + e] + gg[3 * E + e] * kv;
      dk[(b * T + t) * E + e] = gg[E + e] - gg[2 * E + e] + gg[3 * E + e] * qv;
    }
    dq[b * E + e] = acc;
  }
}

// masked (optionally soft-maxed) scores, then out[b,:] = sum_t w_t * keys[b,t,:]   (sequence.py:278-291)
// one warp per sample.  `w_out` [B,T] keeps the post-mask / post-softmax weights for the backward.
__global__ void __launch_bounds__(256)
    din_pool_fwd_kernel(const float* __restrict__ score, const float* __restrict__ keys, int64_t ldk,
                        const uint8_t* __restrict__ mask, float* w_out, float* out, int64_t batch, int T,
                        int E, int weight_norm, int return_score) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* s = score + b * T;
    const uint8_t* m = mask + b * T;
    float* w = w_out + b * T;
    if (weight_norm) {
      float mx = -INFINITY;
      for (int t = lane; t < T; t += 32) mx = fmaxf(mx, m[t] ? s[t] : kNegPad);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float den = 0.f;
      for (int t = lane; t < T; t += 32) den += expf((m[t] ? s[t] : kNegPad) - mx);
      den = warp_sum(den);
      for (int t = lane; t < T; t += 32) w[t] = expf((m[t] ? s[t] : kNegPad) - mx) / den;
    } else {
      for (int t = lane; t < T; t += 32) w[t] = m[t] ? s[t] : 0.f;
    }
    __syncwarp();
    if (return_score) {
      for (int t = lane; t < T; t += 32) out[b * T + t] = w[t];
    } else {
      for (int e = lane; e < E; e += 32) {
        float a = 0.f;
        for (int t = 0; t < T; ++t) a += w[t] * keys[b * ldk + (int64_t)t * E + e];
        out[b * E + e] = a;
      }
    }
  }
}
__global__ void __launch_bounds__(256)
    din_pool_bwd_kernel(const float* __restrict__ w, const float* __restrict__ keys, int64_t ldk,
                        const uint8_t* __restrict__ mask, const float* __restrict__ dout, float* dscore,
                        float* dkeys, int64_t batch, int T, int E, int weight_norm, int return_score) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* wb = w + b * T;
    const uint8_t* m = mask + b * T;
    float* ds = dscore + b * T;
    // dw_t
    if (return_score) {
      for (int t = lane; t < T; t += 32) ds[t] = dout[b * T + t];
    } else {
      for (int t = 0; t < T; ++t) {
        float a = 0.f;
        for (int e = lane; e < E; e += 32) {
          const float g = dout[b * E + e];
          a += g * keys[b * ldk + (int64_t)t * E + e];
          if (dkeys) dkeys[(b * T + t) * E + e] = wb[t] * g;
        }
        a = warp_sum(a);
        if (lane == 0) ds[t] = a;
      }
    }
    __syncwarp();
    if (weight_norm) {
      float dot = 0.f;
      for (int t = lane; t < T; t += 32) dot += wb[t] * ds[t];
      dot = warp_sum(dot);
      for (int t = lane; t < T; t += 32) ds[t] = m[t] ? wb[t] * (ds[t] - dot) : 0.f;
    } else {
      for (int t = lane; t < T; t += 32) ds[t] = m[t] ? ds[t] : 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Standalone SequencePoolingLayer / WeightedSequenceLayer on an arbitrary [B,T,E] tensor
// (same arithmetic order as the fused gather: ascending t, fp32, no fma contraction)
// mode: 1 sum, 2 mean, 3 max.  valid(b,t) = mask ? mask[b,t] != 0 : t < len[b];  L = len[b] or the valid count
// ------------------------------------------------------------------------------------------------
__global__ void seqpool_fwd_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask,
                                   const int32_t* __restrict__ len, float* out, int64_t batch, int T, int E,
                                   int mode) {
  const int64_t total = batch * E;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / E;
    const int e = (int)(i - b * E);
    float L = 0.f;
    if (mask) { int c = 0; for (int t = 0; t < T; ++t) c += mask[b * T + t] != 0; L = (float)c; }
    else L = (float)len[b];
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {
      const bool v = mask ? mask[b * T + t] != 0 : t < len[b];
      const float xv = x[(b * T + t) * E + e];
      if (mode == 3) {
        const float c = v ? xv : __fsub_rn(xv, 1e9f);
        acc = t == 0 ? c : fmaxf(acc, c);
      } else if (v) {
        acc = __fadd_rn(acc, xv);
      }
    }
    if (mode == 2) acc = __fdiv_rn(acc, __fadd_rn(L, 1e-8f));
    out[i] = acc;
  }
}
__global__ void seqpool_bwd_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask,
                                   const int32_t* __restrict__ len, const float* __restrict__ dout,
                                   float* dx, int64_t batch, int T, int E, int mode) {
  const int64_t total = batch * E;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / E;
    const int e = (int)(i - b * E);
    float L = 0.f;
    if (mask) { int c = 0; for (int t = 0; t < T; ++t) c += mask[b * T + t] != 0; L = (float)c; }
    else L = (float)len[b];
    float g = dout[i];
    if (mode == 2) g = g / (L + 1e-8f);
    if (mode == 3) {
      float mx = -INFINITY;
      int cnt = 0;
      for (int t = 0; t < T; ++t) {
        const bool v = mask ? mask[b * T + t] != 0 : t < len[b];
        const float xv = x[(b * T + t) * E + e];
        const float c = v ? xv : __fsub_rn(xv, 1e9f);
        if (c > mx) { mx = c; cnt = 1; } else if (c == mx) cnt++;
      }
      for (int t = 0; t < T; ++t) {
        const bool v = mask ? mask[b * T + t] != 0 : t < len[b];
        const float xv = x[(b * T + t) * E + e];
        const float c = v ? xv : __fsub_rn(xv, 1e9f);
        dx[(b * T + t) * E + e] = c == mx ? g / (float)cnt : 0.f;
      }
    } else {
      for (int t = 0; t < T; ++t) {
        const bool v = mask ? mask[b * T + t] != 0 : t < len[b];
        dx[(b * T + t) * E + e] = v ? g : 0.f;
      }
    }
  }
}
// wt[b,t] = normalise ? softmax_t(where(valid, w, -2^32+1)) : where(valid, w, 0)
__global__ void seqweight_kernel(const float* __restrict__ w, const uint8_t* __restrict__ mask,
                                 const int32_t* __restrict__ len, float* wt, int64_t batch, int T, int norm) {
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < batch;
       b += (int64_t)gridDim.x * blockDim.x) {
    float mx = -INFINITY;
    for (int t = 0; t < T; ++t) {
      const bool v = mask ? mask[b * T + t] != 0 : t < len[b];
      const float s = v ? w[b * T + t] : (norm ? kNegPad : 0.f);
      wt[b * T + t] = s;
      mx = fmaxf(mx, s);
    }
    if (norm) {
      float den = 0.f;
      for (int t = 0; t < T; ++t) den = __fadd_rn(den, expf(__fsub_rn(wt[b * T + t], mx)));
      for (int t = 0; t < T; ++t) wt[b * T + t] = __fdiv_rn(expf(__fsub_rn(wt[b * T + t], mx)), den);
    }
  }
}
// out[b,t,e] = x[b,t,e] * wt[b,t]   (dx = dout * wt: same kernel)
__global__ void seqscale_kernel(const float* __restrict__ x, const float* __restrict__ wt, float* out,
                                int64_t rows, int E) {
  const int64_t total = rows * E;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __fmul_rn(x[i], wt[i / E]);
}

// ------------------------------------------------------------------------------------------------
// Column statistics over [M, N] (BatchNormalization / Dice batch statistics): two deterministic passes.
//   stats[0:N] = mean, stats[N:2N] = biased variance
// ------------------------------------------------------------------------------------------------
constexpr int kStatRows = 512;
__global__ void colsum_partial_kernel(const float* __restrict__ x, int64_t ld, const float* __restrict__ mean,
                                      float* partial, int64_t m, int64_t n) {
  const int64_t r0 = (int64_t)blockIdx.x * kStatRows;
  const int64_t r1 = r0 + kStatRows < m ? r0 + kStatRows : m;
  for (int64_t c = threadIdx.x; c < n; c += blockDim.x) {
    float s = 0.f;
    if (mean) {
      const float mu = mean[c];
      for (int64_t r = r0; r < r1; ++r) { const float d = x[r * ld + c] - mu; s += d * d; }
    } else {
      for (int64_t r = r0; r < r1; ++r) s += x[r * ld + c];
    }
    partial[(int64_t)blockIdx.x * n + c] = s;
  }
}
__global__ void colsum_final_kernel(const float* __restrict__ partial, float* out, int64_t nblocks, int64_t n,
                                    float scale) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  float s = 0.f;
  for (int64_t b = 0; b < nblocks; ++b) s += partial[b * n + c];
  out[c] = s * scale;
}
// moving = moving * momentum + batch * (1 - momentum)   (Keras BatchNormalization update)
__global__ void moving_update_kernel(float* moving, const float* __restrict__ batch, float momentum, int64_t n) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n) moving[c] = moving[c] * momentum + batch[c] * (1.f - momentum);
}

// y = gamma * (x - mean) * rsqrt(var + eps) + beta   (gamma/beta may be NULL)
__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                const float* __restrict__ var, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float* y, int64_t m, int64_t n, float eps) {
  const int64_t total = m * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % n);
    float v = (x[i] - mean[c]) * rsqrtf(var[c] + eps);
    if (gamma) v *= gamma[c];
    if (beta) v += beta[c];
    y[i] = v;
  }
}
// Dice: p = sigmoid((x-mean)*rsqrt(var+eps)); y = alpha*(1-p)*x + p*x   (activation.py:59-64)
__global__ void dice_fwd_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                const float* __restrict__ var, const float* __restrict__ alpha, float* y,
                                int64_t m, int64_t n, float eps) {
  const int64_t total = m * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % n);
    const float xn = (x[i] - mean[c]) * rsqrtf(var[c] + eps);
    const float p = 1.f / (1.f + expf(-xn));
    y[i] = alpha[c] * (1.f - p) * x[i] + p * x[i];
  }
}
// Dice backward, pass 1: g = dL/dxn = dy * x * (1-alpha) * p * (1-p);  emits
//   dx_direct = dy * (alpha + (1-alpha) p),  g,  and per-block column partials of [g, g*xn, dy*x*(1-p)]:
//   block b's row of 3n partials at partial[b*3n ...], the layout colsum_final_kernel reduces over 3n columns
__global__ void dice_bwd1_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                 const float* __restrict__ var, const float* __restrict__ alpha,
                                 const float* __restrict__ dy, float* dx, float* g_out, float* partial,
                                 int64_t m, int64_t n, float eps) {
  const int64_t r0 = (int64_t)blockIdx.x * kStatRows;
  const int64_t r1 = r0 + kStatRows < m ? r0 + kStatRows : m;
  float* prow = partial + (int64_t)blockIdx.x * 3 * n;
  for (int64_t c = threadIdx.x; c < n; c += blockDim.x) {
    const float mu = mean[c], rs = rsqrtf(var[c] + eps), al = alpha[c];
    float sg = 0.f, sgx = 0.f, sa = 0.f;
    for (int64_t r = r0; r < r1; ++r) {
      const int64_t i = r * n + c;
      const float xv = x[i], xn = (xv - mu) * rs;
      const float p = 1.f / (1.f + expf(-xn));
      const float d = dy[i];
      const float g = d * xv * (1.f - al) * p * (1.f - p);
      dx[i] = d * (al + (1.f - al) * p);
      g_out[i] = g;
      sg += g;
      sgx += g * xn;
      sa += d * xv * (1.f - p);
    }
    prow[c] = sg;
    prow[n + c] = sgx;
    prow[2 * n + c] = sa;
  }
}
// pass 2: dx += rs * (g - [training] (mean_g + xn * mean_gxn))
__global__ void dice_bwd2_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                 const float* __restrict__ var, const float* __restrict__ g,
                                 const float* __restrict__ sums, float* dx, int64_t m, int64_t n, float eps,
                                 int training) {
  const int64_t total = m * n;
  const float invm = 1.f / (float)m;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % n);
    const float rs = rsqrtf(var[c] + eps);
    float v = g[i];
    if (training) {
      const float xn = (x[i] - mean[c]) * rs;
      v -= sums[c] * invm + xn * sums[n + c] * invm;
    }
    dx[i] += rs * v;
  }
}
// BatchNormalization backward (training: batch statistics; inference: constants)
//   dxn = dy * gamma;  dx = rs * (dxn - [training](mean(dxn) + xn * mean(dxn*xn)))
// pass 1 writes block b's column partials [dy, dy*xn] as one row of 2n at partial[b*2n ...]
__global__ void bn_bwd1_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                               const float* __restrict__ var, const float* __restrict__ dy, float* partial,
                               int64_t m, int64_t n, float eps) {
  const int64_t r0 = (int64_t)blockIdx.x * kStatRows;
  const int64_t r1 = r0 + kStatRows < m ? r0 + kStatRows : m;
  float* prow = partial + (int64_t)blockIdx.x * 2 * n;
  for (int64_t c = threadIdx.x; c < n; c += blockDim.x) {
    const float mu = mean[c], rs = rsqrtf(var[c] + eps);
    float sd = 0.f, sdx = 0.f;
    for (int64_t r = r0; r < r1; ++r) {
      const int64_t i = r * n + c;
      sd += dy[i];
      sdx += dy[i] * (x[i] - mu) * rs;
    }
    prow[c] = sd;
    prow[n + c] = sdx;
  }
}
__global__ void bn_bwd2_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                               const float* __restrict__ var, const float* __restrict__ gamma,
                               const float* __restrict__ dy, const float* __restrict__ sums, float* dx,
                               int64_t m, int64_t n, float eps, int training) {
  const int64_t total = m * n;
  const float invm = 1.f / (float)m;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % n);
    const float rs = rsqrtf(var[c] + eps);
    const float gm = gamma ? gamma[c] : 1.f;
    float v = dy[i];
    if (training) {
      const float xn = (x[i] - mean[c]) * rs;
      v -= sums[c] * invm + xn * sums[n + c] * invm;
    }
    dx[i] = gm * rs * v;
  }
}

// dropout: keep with prob 1-rate (counter-based hash of (seed, index), mix32 in common.cuh), scale by 1/(1-rate)
__global__ void dropout_kernel(const float* __restrict__ x, float* y, int64_t n, float rate, uint64_t seed) {
  const float keep_scale = 1.f / (1.f - rate);
  const uint32_t thr = (uint32_t)(rate * 4294967296.0);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    y[i] = mix32(seed * 0x9E3779B97F4A7C15ULL + (uint64_t)i) >= thr ? x[i] * keep_scale : 0.f;
}

}  // namespace b2ctr

using namespace b2ctr;
#define ST ((cudaStream_t)stream)

extern "C" {

b2ctr_status_t b2ctr_din_att_input_fwd(const float* q, int64_t ldq, const float* keys, int64_t ldk, float* out,
                                       int64_t batch, int32_t T, int32_t E, void* stream) {
  B2_REQUIRE(q && keys && out && T > 0 && E > 0, "din_att_input_fwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  din_att_input_fwd_kernel<<<grid_for(batch * T * E, 256, 8), 256, 0, ST>>>(q, ldq, keys, ldk, out, batch, T, E);
  B2_CHECK_LAUNCH("b2ctr_din_att_input_fwd");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_din_att_input_bwd(const float* q, int64_t ldq, const float* keys, int64_t ldk,
                                       const float* g, float* dq, float* dk, int64_t batch, int32_t T,
                                       int32_t E, void* stream) {
  B2_REQUIRE(q && keys && g && dq && dk && T > 0 && E > 0, "din_att_input_bwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  din_att_input_bwd_kernel<<<grid_for(batch * E, 256, 8), 256, 0, ST>>>(q, ldq, keys, ldk, g, dq, dk, batch, T, E);
  B2_CHECK_LAUNCH("b2ctr_din_att_input_bwd");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_din_pool_fwd(const float* score, const float* keys, int64_t ldk, const uint8_t* mask,
                                  float* w, float* out, int64_t batch, int32_t T, int32_t E,
                                  int32_t weight_norm, int32_t return_score, void* stream) {
  B2_REQUIRE(score && keys && mask && w && out && T > 0 && E > 0, "din_pool_fwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  din_pool_fwd_kernel<<<grid_for(batch, 8, 8), 256, 0, ST>>>(score, keys, ldk, mask, w, out, batch, T, E,
                                                            weight_norm, return_score);
  B2_CHECK_LAUNCH("b2ctr_din_pool_fwd");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_din_pool_bwd(const float* w, const float* keys, int64_t ldk, const uint8_t* mask,
                                  const float* dout, float* dscore, float* dkeys, int64_t batch, int32_t T,
                                  int32_t E, int32_t weight_norm, int32_t return_score, void* stream) {
  B2_REQUIRE(w && keys && mask && dout && dscore && T > 0 && E > 0, "din_pool_bwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  din_pool_bwd_kernel<<<grid_for(batch, 8, 8), 256, 0, ST>>>(w, keys, ldk, mask, dout, dscore, dkeys, batch, T,
                                                            E, weight_norm, return_score);
  B2_CHECK_LAUNCH("b2ctr_din_pool_bwd");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_seqpool_fwd(const float* x, const uint8_t* mask, const int32_t* len, float* out,
                                 int64_t batch, int32_t T, int32_t E, int32_t mode, void* stream) {
  B2_REQUIRE(x && out && (mask || len) && mode >= 1 && mode <= 3, "seqpool_fwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  seqpool_fwd_kernel<<<grid_for(batch * E, 256, 8), 256, 0, ST>>>(x, mask, len, out, batch, T, E, mode);
  B2_CHECK_LAUNCH("b2ctr_seqpool_fwd");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_seqpool_bwd(const float* x, const uint8_t* mask, const int32_t* len, const float* dout,
                                 float* dx, int64_t batch, int32_t T, int32_t E, int32_t mode, void* stream) {
  B2_REQUIRE(x && dout && dx && (mask || len) && mode >= 1 && mode <= 3, "seqpool_bwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  seqpool_bwd_kernel<<<grid_for(batch * E, 256, 8), 256, 0, ST>>>(x, mask, len, dout, dx, batch, T, E, mode);
  B2_CHECK_LAUNCH("b2ctr_seqpool_bwd");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_seqweight(const float* w, const uint8_t* mask, const int32_t* len, float* wt, int64_t batch,
                               int32_t T, int32_t normalize, void* stream) {
  B2_REQUIRE(w && wt && (mask || len), "seqweight: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  seqweight_kernel<<<grid_for(batch, 128, 8), 128, 0, ST>>>(w, mask, len, wt, batch, T, normalize);
  B2_CHECK_LAUNCH("b2ctr_seqweight");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_seqscale(const float* x, const float* wt, float* out, int64_t rows, int32_t E, void* stream) {
  B2_REQUIRE(x && wt && out && E > 0, "seqscale: bad arguments");
  if (rows <= 0) return B2CTR_OK;
  seqscale_kernel<<<grid_for(rows * E, 256, 8), 256, 0, ST>>>(x, wt, out, rows, E);
  B2_CHECK_LAUNCH("b2ctr_seqscale");
  return B2CTR_OK;
}

size_t b2ctr_colstats_workspace_bytes(int64_t m, int64_t n) {
  return (size_t)3 * ceil_div(m, kStatRows) * (size_t)n * sizeof(float) + (size_t)3 * n * sizeof(float);
}
/* stats[0:n] = column means, stats[n:2n] = biased variances of x[m,n] (ld) */
b2ctr_status_t b2ctr_colstats(const float* x, int64_t ld, int64_t m, int64_t n, float* stats, void* workspace,
                              size_t workspace_bytes, void* stream) {
  B2_REQUIRE(x && stats && m > 0 && n > 0 && ld >= n, "colstats: bad arguments");
  if (!workspace || workspace_bytes < b2ctr_colstats_workspace_bytes(m, n)) {
    set_error("colstats: workspace too small");
    return B2CTR_ERR_WORKSPACE;
  }
  const int64_t nb = ceil_div(m, kStatRows);
  float* partial = (float*)workspace;
  colsum_partial_kernel<<<(unsigned)nb, 256, 0, ST>>>(x, ld, nullptr, partial, m, n);
  B2_CHECK_LAUNCH("b2ctr_colstats(sum)");
  colsum_final_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, ST>>>(partial, stats, nb, n, 1.f / (float)m);
  B2_CHECK_LAUNCH("b2ctr_colstats(mean)");
  colsum_partial_kernel<<<(unsigned)nb, 256, 0, ST>>>(x, ld, stats, partial, m, n);
  B2_CHECK_LAUNCH("b2ctr_colstats(sq)");
  colsum_final_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, ST>>>(partial, stats + n, nb, n, 1.f / (float)m);
  B2_CHECK_LAUNCH("b2ctr_colstats(var)");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_moving_update(float* moving, const float* batch, float momentum, int64_t n, void* stream) {
  B2_REQUIRE(moving && batch, "moving_update: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  moving_update_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, ST>>>(moving, batch, momentum, n);
  B2_CHECK_LAUNCH("b2ctr_moving_update");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_bn_apply(const float* x, const float* mean, const float* var, const float* gamma,
                              const float* beta, float* y, int64_t m, int64_t n, float eps, void* stream) {
  B2_REQUIRE(x && mean && var && y, "bn_apply: NULL pointer");
  if (m <= 0 || n <= 0) return B2CTR_OK;
  bn_apply_kernel<<<grid_for(m * n, 256, 8), 256, 0, ST>>>(x, mean, var, gamma, beta, y, m, n, eps);
  B2_CHECK_LAUNCH("b2ctr_bn_apply");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_bn_bwd(const float* x, const float* mean, const float* var, const float* gamma,
                            const float* dy, float* dx, float* dgamma, float* dbeta, int64_t m, int64_t n,
                            float eps, int32_t training, void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(x && mean && var && dy && dx, "bn_bwd: NULL pointer");
  if (m <= 0 || n <= 0) return B2CTR_OK;
  if (!workspace || workspace_bytes < b2ctr_colstats_workspace_bytes(m, n)) {
    set_error("bn_bwd: workspace too small");
    return B2CTR_ERR_WORKSPACE;
  }
  const int64_t nb = ceil_div(m, kStatRows);
  float* partial = (float*)workspace;
  float* sums = partial + 3 * nb * n;
  bn_bwd1_kernel<<<(unsigned)nb, 256, 0, ST>>>(x, mean, var, dy, partial, m, n, eps);
  B2_CHECK_LAUNCH("b2ctr_bn_bwd(1)");
  colsum_final_kernel<<<(unsigned)ceil_div(2 * n, 128), 128, 0, ST>>>(partial, sums, nb, 2 * n, 1.f);
  B2_CHECK_LAUNCH("b2ctr_bn_bwd(sum)");
  // sums[0:n] = sum dy (= dbeta), sums[n:2n] = sum dy*xn (= dgamma); the dx formula needs them scaled by gamma
  if (dbeta) cudaMemcpyAsync(dbeta, sums, n * sizeof(float), cudaMemcpyDeviceToDevice, ST);
  if (dgamma) cudaMemcpyAsync(dgamma, sums + n, n * sizeof(float), cudaMemcpyDeviceToDevice, ST);
  bn_bwd2_kernel<<<grid_for(m * n, 256, 8), 256, 0, ST>>>(x, mean, var, gamma, dy, sums, dx, m, n, eps, training);
  B2_CHECK_LAUNCH("b2ctr_bn_bwd(2)");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_dice_fwd(const float* x, const float* mean, const float* var, const float* alpha, float* y,
                              int64_t m, int64_t n, float eps, void* stream) {
  B2_REQUIRE(x && mean && var && alpha && y, "dice_fwd: NULL pointer");
  if (m <= 0 || n <= 0) return B2CTR_OK;
  dice_fwd_kernel<<<grid_for(m * n, 256, 8), 256, 0, ST>>>(x, mean, var, alpha, y, m, n, eps);
  B2_CHECK_LAUNCH("b2ctr_dice_fwd");
  return B2CTR_OK;
}
size_t b2ctr_dice_bwd_workspace_bytes(int64_t m, int64_t n) {
  return b2ctr_colstats_workspace_bytes(m, n) + (size_t)m * n * sizeof(float);
}
b2ctr_status_t b2ctr_dice_bwd(const float* x, const float* mean, const float* var, const float* alpha,
                              const float* dy, float* dx, float* dalpha, int64_t m, int64_t n, float eps,
                              int32_t training, void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(x && mean && var && alpha && dy && dx && dalpha, "dice_bwd: NULL pointer");
  if (m <= 0 || n <= 0) return B2CTR_OK;
  if (!workspace || workspace_bytes < b2ctr_dice_bwd_workspace_bytes(m, n)) {
    set_error("dice_bwd: workspace too small");
    return B2CTR_ERR_WORKSPACE;
  }
  const int64_t nb = ceil_div(m, kStatRows);
  float* partial = (float*)workspace;
  float* sums = partial + 3 * nb * n;
  float* g = sums + 3 * n;
  dice_bwd1_kernel<<<(unsigned)nb, 256, 0, ST>>>(x, mean, var, alpha, dy, dx, g, partial, m, n, eps);
  B2_CHECK_LAUNCH("b2ctr_dice_bwd(1)");
  colsum_final_kernel<<<(unsigned)ceil_div(3 * n, 128), 128, 0, ST>>>(partial, sums, nb, 3 * n, 1.f);
  B2_CHECK_LAUNCH("b2ctr_dice_bwd(sum)");
  cudaMemcpyAsync(dalpha, sums + 2 * n, n * sizeof(float), cudaMemcpyDeviceToDevice, ST);
  dice_bwd2_kernel<<<grid_for(m * n, 256, 8), 256, 0, ST>>>(x, mean, var, g, sums, dx, m, n, eps, training);
  B2_CHECK_LAUNCH("b2ctr_dice_bwd(2)");
  return B2CTR_OK;
}
b2ctr_status_t b2ctr_dropout(const float* x, float* y, int64_t n, float rate, uint64_t seed, void* stream) {
  B2_REQUIRE(x && y && rate >= 0.f && rate < 1.f, "dropout: bad arguments");
  if (n <= 0) return B2CTR_OK;
  dropout_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(x, y, n, rate, seed);
  B2_CHECK_LAUNCH("b2ctr_dropout");
  return B2CTR_OK;
}

}  // extern "C"
