// elementwise.cu — activation backward + bias gradient, n-ary add, strided copies, FM operator,
// prediction head + loss, optimizers.  All HBM-bound: 128-bit accesses where alignment allows,
// grid-stride loops on grids that are whole multiples of the SM count.
#include <cuda_bf16.h>
#include "common.cuh"

namespace b2ctr {

// -------------------------------------------------------------------------------------------
// dz = dy * act'(y);  dbias = column sums of dz  (two deterministic passes: per-block partial
// sums over a fixed row range, then a fixed-order reduction over blocks)
// -------------------------------------------------------------------------------------------
constexpr int kBiasRowsPerBlock = 128;

// block = 8 warps; warp w owns rows r0 + w, r0 + w + 8, ...; lanes own 32 consecutive columns (coalesced);
// the 8 per-warp partials are combined through shared memory in a fixed order.
__global__ void __launch_bounds__(256)
    bias_act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* dz,
                        float* partial, int64_t m, int64_t n, int64_t ld, int act) {
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * kBiasRowsPerBlock;
  const int64_t r1 = r0 + kBiasRowsPerBlock < m ? r0 + kBiasRowsPerBlock : m;
  for (int64_t c0 = 0; c0 < n; c0 += 32) {
    const int64_t c = c0 + lane;
    float s = 0.f;
    if (c < n) {
      for (int64_t r = r0 + warp; r < r1; r += 8) {
        const int64_t o = r * ld + c;
        const float g = dy[o] * (act == B2CTR_ACT_NONE ? 1.f : act_grad_from_out(y[o], act));
        if (dz) dz[o] = g;
        s += g;
      }
    }
    if (partial) {
      red[warp][lane] = s;
      __syncthreads();
      if (warp == 0 && c < n) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += red[w][lane];
        partial[(int64_t)blockIdx.x * n + c] = t;
      }
      __syncthreads();
    }
  }
}
// float4 variant for n % 4 == 0 with (n/4) dividing 256: thread -> (row group, 4-column group); the
// row groups are combined through shared memory in a fixed order.
__global__ void __launch_bounds__(256)
    bias_act_bwd_vec4_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* dz,
                             float* partial, int64_t m, int64_t n, int64_t ld, int act,
                             __nv_bfloat16* pl_hi, __nv_bfloat16* pl_lo, int64_t pl_pitch) {
  __shared__ float4 red[256];
  const int cgs = (int)(n >> 2);              // column groups
  const int rgs = 256 / cgs;                  // row groups per pass
  const int cg = threadIdx.x % cgs, rg = threadIdx.x / cgs;
  const int64_t r0 = (int64_t)blockIdx.x * kBiasRowsPerBlock;
  const int64_t r1 = r0 + kBiasRowsPerBlock < m ? r0 + kBiasRowsPerBlock : m;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int64_t r = r0 + rg; r < r1; r += rgs) {
    const int64_t o = r * ld + cg * 4;
    float4 g = *reinterpret_cast<const float4*>(dy + o);
    if (act != B2CTR_ACT_NONE) {
      const float4 yy = *reinterpret_cast<const float4*>(y + o);
      g.x *= act_grad_from_out(yy.x, act); g.y *= act_grad_from_out(yy.y, act);
      g.z *= act_grad_from_out(yy.z, act); g.w *= act_grad_from_out(yy.w, act);
    }
    if (dz) *reinterpret_cast<float4*>(dz + o) = g;
    if (pl_hi) {     // bf16 hi/lo operand planes of dz for the dgrad / wgrad GEMMs (b2ctr_split_planes layout)
      const __nv_bfloat16 h0 = __float2bfloat16_rn(g.x), h1 = __float2bfloat16_rn(g.y);
      const __nv_bfloat16 h2 = __float2bfloat16_rn(g.z), h3 = __float2bfloat16_rn(g.w);
      uint2 h, l;
      h.x = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
      h.y = (uint32_t)__bfloat16_as_ushort(h2) | ((uint32_t)__bfloat16_as_ushort(h3) << 16);
      l.x = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(g.x - __bfloat162float(h0))) |
            ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(g.y - __bfloat162float(h1))) << 16);
      l.y = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(g.z - __bfloat162float(h2))) |
            ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(g.w - __bfloat162float(h3))) << 16);
      const int64_t po = r * pl_pitch + cg * 4;
      *reinterpret_cast<uint2*>(pl_hi + po) = h;
      *reinterpret_cast<uint2*>(pl_lo + po) = l;
    }
    s.x += g.x; s.y += g.y; s.z += g.z; s.w += g.w;
  }
  if (partial) {
    red[threadIdx.x] = s;
    __syncthreads();
    if (rg == 0) {
      float4 t = red[cg];
      for (int k = 1; k < rgs; ++k) {
        const float4 v = red[k * cgs + cg];
        t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
      }
      *reinterpret_cast<float4*>(partial + (int64_t)blockIdx.x * n + cg * 4) = t;
    }
  }
}
// one block per 8 columns; 32 row-lanes stride the partial blocks and meet in shared memory in a fixed order
// (deterministic).  8-column blocks keep >= 32 CTAs busy at n = 256 - with 32-column blocks the reduce of a
// 512-row partial matrix ran on 8 CTAs and cost 12 us per layer.
__global__ void __launch_bounds__(256)
    bias_reduce_kernel(const float* __restrict__ partial, float* dbias, int64_t nblocks, int64_t n) {
  __shared__ float red[32][9];
  const int col = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int64_t c = (int64_t)blockIdx.x * 8 + col;
  float s = 0.f;
  if (c < n)
    for (int64_t b = rl; b < nblocks; b += 32) s += partial[b * n + c];
  red[rl][col] = s;
  __syncthreads();
  if (rl == 0 && c < n) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 32; ++w) t += red[w][col];
    dbias[c] = t;
  }
}

__global__ void act_fwd_kernel(const float* __restrict__ x, float* y, int64_t n, int act) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    y[i] = act_apply(x[i], act);
}

struct AddN {
  const float* in[8];
  float scale[8];
  int nin;
};
__global__ void add_n_kernel(const AddN a, float* out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
#pragma unroll 1
    for (int j = 0; j < a.nin; ++j) s += a.in[j][i] * a.scale[j];
    out[i] = s;
  }
}
__global__ void axpy_kernel(const float* __restrict__ x, float* y, float alpha, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    y[i] += alpha * x[i];
}
__global__ void fill_kernel(float* dst, float v, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = v;
}
template <bool VEC4>
__global__ void copy2d_kernel(const float* __restrict__ src, int64_t lds, float* dst, int64_t ldd,
                              int64_t rows, int64_t cols, int acc) {
  const int64_t w = VEC4 ? cols / 4 : cols;
  const int64_t total = rows * w;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / w, c = i - r * w;
    if (VEC4) {
      float4 v = *reinterpret_cast<const float4*>(src + r * lds + c * 4);
      float4* d = reinterpret_cast<float4*>(dst + r * ldd + c * 4);
      if (acc) { float4 o = *d; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
      *d = v;
    } else {
      float v = src[r * lds + c];
      if (acc) v += dst[r * ldd + c];
      dst[r * ldd + c] = v;
    }
  }
}
__global__ void mask_nonzero_and_kernel(const void* ids, int dtype, int64_t n, uint8_t* io, int first) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t v = load_idx(ids, i, dtype) != 0;
    io[i] = first ? v : (uint8_t)(io[i] & v);
  }
}
__global__ void mask_from_len_kernel(const int32_t* len, int64_t batch, int maxlen, uint8_t* out) {
  const int64_t n = batch * maxlen;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int)(i % maxlen) < len[i / maxlen];
}
// Feeder: per-input contiguous host blocks [B, w_i] -> one row-major [B, total] pack on the device
struct PackCols {
  int64_t off[64];     // element offset of block i inside src
  int32_t width[64];
  int32_t col[64];     // first column of block i in dst
  int32_t nblk, total;
};
__global__ void pack_rows_kernel(const float* __restrict__ src, const PackCols pc, int64_t batch, float* dst,
                                 int64_t ld) {
  const int64_t n = batch * pc.total;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / pc.total;
    const int c = (int)(i - b * pc.total);
    int k = 0;
    while (k + 1 < pc.nblk && c >= pc.col[k + 1]) ++k;
    dst[b * ld + c] = src[pc.off[k] + b * pc.width[k] + (c - pc.col[k])];
  }
}
// one warp per row, lanes stride the columns; partials combined in a fixed shuffle tree
__global__ void rowsum_kernel(const float* __restrict__ x, int64_t ld, float* out, int64_t rows,
                              int64_t cols) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += nw) {
    float s = 0.f;
    for (int64_t c = lane; c < cols; c += 32) s += x[r * ld + c];
    s = warp_sum(s);
    if (lane == 0) out[r] = s;
  }
}

// -------------------------------------------------------------------------------------------
// FM (deepctr/layers/interaction.py:597-602): one warp per sample, lanes over the embedding
// axis, fields walked sequentially; pairwise reduction over e by warp shuffles.
// WEIGHTED: FM of (m ⊙ x) with per-sample field weights m [B, F] (IFM / DIFM), the product formed
// in registers.  With m == 1 every multiply by m is exact, so the result is the unweighted one bit for bit.
// -------------------------------------------------------------------------------------------
template <bool WEIGHTED>
__global__ void fm_fwd_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ m,
                              int64_t ldm, int nfield, int dim, float* out, int64_t batch) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* xr = x + b * ldx;
    const float* mr = WEIGHTED ? m + b * ldm : nullptr;
    float tot = 0.f;
    for (int e = lane; e < dim; e += 32) {
      float s = 0.f, q = 0.f;
      for (int f = 0; f < nfield; ++f) {
        float v = xr[f * dim + e];
        if (WEIGHTED) v *= mr[f];
        s += v;
        q += v * v;
      }
      tot += s * s - q;
    }
    tot = warp_sum(tot);
    if (lane == 0) out[b] = 0.5f * tot;
  }
}
// dx_f = g m_f (S - m_f x_f) with S = sum_f m_f x_f (m == 1 unweighted).  WEIGHTED also writes
// dm_f = g sum_e x_f (S - m_f x_f): per 32-column chunk a fixed shuffle tree, chunks added in order by lane 0,
// so dm is bit-identical from run to run.
template <bool WEIGHTED>
__global__ void fm_bwd_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ m,
                              int64_t ldm, int nfield, int dim, const float* __restrict__ dout, float* dx,
                              int64_t lddx, float* dm, int64_t lddm, int acc, int64_t batch) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nw) {
    const float* xr = x + b * ldx;
    const float* mr = WEIGHTED ? m + b * ldm : nullptr;
    float* dr = dx ? dx + b * lddx : nullptr;
    float* dmr = WEIGHTED && dm ? dm + b * lddm : nullptr;
    const float g = dout[b];
    for (int e0 = 0; e0 < dim; e0 += 32) {
      const int e = e0 + lane;
      const bool on = e < dim;
      float s = 0.f;
      if (on)
        for (int f = 0; f < nfield; ++f) s += WEIGHTED ? mr[f] * xr[f * dim + e] : xr[f * dim + e];
      for (int f = 0; f < nfield; ++f) {
        if (WEIGHTED) {
          const float mf = mr[f];
          const float xv = on ? xr[f * dim + e] : 0.f;
          const float r = s - mf * xv;
          if (on && dr) {
            const float v = g * mf * r;
            dr[f * dim + e] = acc ? dr[f * dim + e] + v : v;
          }
          if (dmr) {
            const float t = warp_sum(xv * r);
            if (lane == 0) dmr[f] = e0 == 0 ? t : dmr[f] + t;
          }
        } else if (on) {
          const float v = g * (s - xr[f * dim + e]);
          dr[f * dim + e] = acc ? dr[f * dim + e] + v : v;
        }
      }
    }
    if (dmr && lane == 0)
      for (int f = 0; f < nfield; ++f) dmr[f] *= g;
  }
}

// -------------------------------------------------------------------------------------------
// Field scale y[b,f,:] = x[b,f,:] * m[b,f] (the refine product of IFM / DIFM, feature_column.py:193-200,
// ifm.py:66-67) and its backward.  One group of W lanes (W = the power of two >= min(dim, 32)) per (b, f)
// row, lanes striding e; dm's row sum is a fixed shuffle tree inside the group (deterministic).
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float group_sum(float v, int width) {
  for (int o = width >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, width);
  return v;
}
__global__ void field_scale_fwd_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ m,
                                       int64_t ldm, int nfield, int dim, float* y, int64_t ldy, int64_t batch,
                                       int width) {
  const int sub = threadIdx.x & (width - 1);
  const int64_t groups = (int64_t)gridDim.x * (blockDim.x / width);
  const int64_t rows = batch * nfield;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / width; r < rows; r += groups) {
    const int64_t b = r / nfield;
    const int f = (int)(r - b * nfield);
    const float mf = m[b * ldm + f];
    const float* xr = x + b * ldx + (int64_t)f * dim;
    float* yr = y + b * ldy + (int64_t)f * dim;
    for (int e = sub; e < dim; e += width) yr[e] = xr[e] * mf;
  }
}
__global__ void field_scale_bwd_kernel(const float* __restrict__ dy, int64_t lddy, const float* __restrict__ x,
                                       int64_t ldx, const float* __restrict__ m, int64_t ldm, int nfield, int dim,
                                       float* dx, int64_t lddx, float* dm, int64_t lddm, int acc, int64_t batch,
                                       int width) {
  const int sub = threadIdx.x & (width - 1);
  const int64_t groups = (int64_t)gridDim.x * (blockDim.x / width);
  const int64_t rows = batch * nfield;
  // every group of a warp runs the same number of iterations (rows rounded up), so the shuffles stay converged
  const int64_t rows_pad = (rows + 32 / width - 1) / (32 / width) * (32 / width);
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / width; r < rows_pad; r += groups) {
    const bool on = r < rows;
    const int64_t b = on ? r / nfield : 0;
    const int f = on ? (int)(r - b * nfield) : 0;
    const float mf = on ? m[b * ldm + f] : 0.f;
    const float* dyr = dy + b * lddy + (int64_t)f * dim;
    const float* xr = x + b * ldx + (int64_t)f * dim;
    float t = 0.f;
    if (on)
      for (int e = sub; e < dim; e += width) {
        const float gv = dyr[e];
        if (dx) {
          float* p = dx + b * lddx + (int64_t)f * dim + e;
          const float v = gv * mf;
          *p = acc ? *p + v : v;
        }
        t += gv * xr[e];
      }
    t = group_sum(t, width);
    if (on && sub == 0 && dm) dm[b * lddm + f] = t;
  }
}

// -------------------------------------------------------------------------------------------
// y = scale * softmax(x) along the rows of a [B, C] window (layers/utils.py softmax; IFM's F * softmax(z)).
// One warp per row; the maximum is subtracted first.  Backward: dx = y (dy - sum_j y_j dy_j / scale).
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__global__ void softmax_rows_fwd_kernel(const float* __restrict__ x, int64_t ldx, float* y, int64_t ldy,
                                        int64_t rows, int cols, float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += nw) {
    const float* xr = x + r * ldx;
    float* yr = y + r * ldy;
    float mx = -INFINITY;
    for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, xr[c]);
    mx = warp_max(mx);
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) s += expf(xr[c] - mx);
    s = warp_sum(s);
    const float k = scale / s;
    for (int c = lane; c < cols; c += 32) yr[c] = expf(xr[c] - mx) * k;
  }
}
__global__ void softmax_rows_bwd_kernel(const float* __restrict__ y, int64_t ldy, const float* __restrict__ dy,
                                        int64_t lddy, float* dx, int64_t lddx, int64_t rows, int cols,
                                        float scale) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += nw) {
    const float* yr = y + r * ldy;
    const float* gr = dy + r * lddy;
    float* dr = dx + r * lddx;
    float d = 0.f;
    for (int c = lane; c < cols; c += 32) d += yr[c] * gr[c];
    d = warp_sum(d) / scale;
    for (int c = lane; c < cols; c += 32) dr[c] = yr[c] * (gr[c] - d);
  }
}

// -------------------------------------------------------------------------------------------
// PredictionLayer + loss (SURVEY.md App. C: Keras binary_crossentropy on probabilities)
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    predict_loss_kernel(const float* __restrict__ logit, const float* __restrict__ bias,
                        const float* __restrict__ labels, float* pred, float* dlogit, float* dbias,
                        float* loss_sum, int64_t batch, int task) {
  const float bz = bias ? bias[0] : 0.f;
  const float invb = 1.f / (float)batch;
  float lsum = 0.f, gsum = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < batch;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float z = logit[i] + bz;
    float p, l = 0.f, dz = 0.f;
    if (task == B2CTR_TASK_BINARY) {
      p = 1.f / (1.f + expf(-z));
      if (labels) {
        const float eps = 1e-7f, y = labels[i];
        const float pc = fminf(fmaxf(p, eps), 1.f - eps);
        l = -(y * logf(pc + eps) + (1.f - y) * logf(1.f - pc + eps));
        const float inside = (p >= eps && p <= 1.f - eps) ? 1.f : 0.f;
        const float dldp = -(y / (pc + eps) - (1.f - y) / (1.f - pc + eps)) * inside;
        dz = dldp * p * (1.f - p);
      }
    } else {
      p = z;
      if (labels) {
        const float d = p - labels[i];
        l = d * d;
        dz = 2.f * d;
      }
    }
    if (pred) pred[i] = p;
    dz *= invb;
    if (dlogit) dlogit[i] = dz;
    lsum += l;
    gsum += dz;
  }
  if (loss_sum || dbias) {
    __shared__ float sl[8], sg[8];
    lsum = warp_sum(lsum);
    gsum = warp_sum(gsum);
    if ((threadIdx.x & 31) == 0) { sl[threadIdx.x >> 5] = lsum; sg[threadIdx.x >> 5] = gsum; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float a = 0.f, c = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += sl[w]; c += sg[w]; }
      if (loss_sum) atomicAdd(loss_sum, a);
      if (dbias) atomicAdd(dbias, c);
    }
  }
}

// -------------------------------------------------------------------------------------------
// optimizers (dense weights; embedding rows use the fused scatter-update in embed.cu)
// -------------------------------------------------------------------------------------------
__global__ void sgd_kernel(float* w, const float* __restrict__ g, float lr, float l2, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    w[i] -= lr * (g[i] + 2.f * l2 * w[i]);
}
// every dense weight of a tower in ONE launch (blockIdx.y = tensor): the 9-14 per-weight launches of a step were
// 3 us each for a few kB of work
constexpr int kSgdMulti = 32;
struct SgdMulti {
  float* w[kSgdMulti];
  const float* g[kSgdMulti];
  int64_t n[kSgdMulti];
  float l2[kSgdMulti];
};
__global__ void sgd_multi_kernel(const __grid_constant__ SgdMulti p, float lr) {
  const int t = blockIdx.y;
  float* w = p.w[t];
  const float* __restrict__ g = p.g[t];
  const int64_t n = p.n[t];
  const float l2 = p.l2[t];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    w[i] -= lr * (g[i] + 2.f * l2 * w[i]);
}
__global__ void adam_kernel(float* w, const float* __restrict__ g, float* m, float* v, float lr_t,
                            float b1, float b2, float eps, float l2, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] + 2.f * l2 * w[i];
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    w[i] -= lr_t * mi / (sqrtf(vi) + eps);
  }
}
__global__ void adagrad_kernel(float* w, const float* __restrict__ g, float* acc, float lr, float eps,
                               float l2, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] + 2.f * l2 * w[i];
    const float a = acc[i] + gi * gi;
    acc[i] = a;
    w[i] -= lr * gi / (sqrtf(a) + eps);
  }
}

}  // namespace b2ctr

using namespace b2ctr;
#define ST ((cudaStream_t)stream)

extern "C" {

size_t b2ctr_bias_act_bwd_workspace_bytes(int64_t m, int64_t n) {
  return (size_t)ceil_div(m, kBiasRowsPerBlock) * (size_t)n * sizeof(float);
}

b2ctr_status_t b2ctr_bias_act_bwd(const float* dy, const float* y, float* dz, float* dbias, int64_t m,
                                  int64_t n, int64_t ld, int32_t act, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return b2ctr_bias_act_bwd_planes(dy, y, dz, dbias, nullptr, m, n, ld, act, workspace, workspace_bytes, stream);
}

b2ctr_status_t b2ctr_bias_act_bwd_planes(const float* dy, const float* y, float* dz, float* dbias, void* dz_planes,
                                         int64_t m, int64_t n, int64_t ld, int32_t act, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  B2_REQUIRE(dy && (dz || dbias || dz_planes), "bias_act_bwd: NULL dy, or nothing to compute");
  B2_REQUIRE(act == B2CTR_ACT_NONE || y, "bias_act_bwd: activation output y required");
  B2_REQUIRE(ld >= n, "bias_act_bwd: ld < n");
  if (m <= 0 || n <= 0) return B2CTR_OK;
  const int64_t nblocks = ceil_div(m, kBiasRowsPerBlock);
  if (dbias) {
    const size_t need = b2ctr_bias_act_bwd_workspace_bytes(m, n);
    if (!workspace || workspace_bytes < need) {
      set_error("bias_act_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
      return B2CTR_ERR_WORKSPACE;
    }
  }
  const bool vec = n % 4 == 0 && n / 4 <= 256 && 256 % (n / 4) == 0 && ld % 4 == 0 &&
                   ((uintptr_t)dy & 15) == 0 && (!y || ((uintptr_t)y & 15) == 0) &&
                   (!dz || ((uintptr_t)dz & 15) == 0);
  __nv_bfloat16 *pl_hi = nullptr, *pl_lo = nullptr;
  const int64_t pl_pitch = planes_cols_pad(n);
  if (dz_planes) {
    // the planes are written row by row for [0, m) x [0, n): no padding may exist
    B2_REQUIRE(vec && m % 256 == 0 && pl_pitch == n && ((uintptr_t)dz_planes & 15) == 0,
               "bias_act_bwd: dz_planes needs m %% 256 == 0, n in {64, 128k} and the vectorised layout");
    pl_hi = (__nv_bfloat16*)dz_planes;
    pl_lo = pl_hi + planes_rows_pad(m) * pl_pitch;
  }
  if (vec)
    bias_act_bwd_vec4_kernel<<<(unsigned)nblocks, 256, 0, ST>>>(dy, y, dz, dbias ? (float*)workspace : nullptr,
                                                               m, n, ld, act, pl_hi, pl_lo, pl_pitch);
  else
    bias_act_bwd_kernel<<<(unsigned)nblocks, 256, 0, ST>>>(dy, y, dz, dbias ? (float*)workspace : nullptr,
                                                          m, n, ld, act);
  B2_CHECK_LAUNCH("b2ctr_bias_act_bwd");
  if (dbias) {
    bias_reduce_kernel<<<(unsigned)ceil_div(n, 8), 256, 0, ST>>>((const float*)workspace, dbias,
                                                                 nblocks, n);
    B2_CHECK_LAUNCH("b2ctr_bias_act_bwd(reduce)");
  }
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_act_fwd(const float* x, float* y, int64_t n, int32_t act, void* stream) {
  B2_REQUIRE(x && y, "act_fwd: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  act_fwd_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(x, y, n, act);
  B2_CHECK_LAUNCH("b2ctr_act_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_add_n(const float* const* ins, const float* scales, int32_t nin, float* out,
                           int64_t n, void* stream) {
  B2_REQUIRE(ins && out && nin >= 1 && nin <= 8, "add_n: need 1..8 inputs");
  AddN a;
  a.nin = nin;
  for (int i = 0; i < nin; ++i) {
    B2_REQUIRE(ins[i], "add_n: input %d is NULL", i);
    a.in[i] = ins[i];
    a.scale[i] = scales ? scales[i] : 1.f;
  }
  if (n <= 0) return B2CTR_OK;
  add_n_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(a, out, n);
  B2_CHECK_LAUNCH("b2ctr_add_n");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_axpy(const float* x, float* y, float alpha, int64_t n, void* stream) {
  B2_REQUIRE(x && y, "axpy: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  axpy_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(x, y, alpha, n);
  B2_CHECK_LAUNCH("b2ctr_axpy");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_fill(float* dst, float value, int64_t n, void* stream) {
  B2_REQUIRE(dst, "fill: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  fill_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(dst, value, n);
  B2_CHECK_LAUNCH("b2ctr_fill");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_mask_nonzero_and(const void* ids, int32_t idx_dtype, int64_t n, uint8_t* inout,
                                      int32_t first, void* stream) {
  B2_REQUIRE(ids && inout, "mask_nonzero_and: NULL pointer");
  B2_REQUIRE(idx_dtype == B2CTR_IDX_I32 || idx_dtype == B2CTR_IDX_I64, "mask_nonzero_and: bad dtype");
  if (n <= 0) return B2CTR_OK;
  mask_nonzero_and_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(ids, idx_dtype, n, inout, first);
  B2_CHECK_LAUNCH("b2ctr_mask_nonzero_and");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_mask_from_len(const int32_t* len, int64_t batch, int32_t maxlen, uint8_t* out,
                                   void* stream) {
  B2_REQUIRE(len && out && maxlen > 0, "mask_from_len: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  mask_from_len_kernel<<<grid_for(batch * maxlen, 256, 8), 256, 0, ST>>>(len, batch, maxlen, out);
  B2_CHECK_LAUNCH("b2ctr_mask_from_len");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_copy2d(const float* src, int64_t ld_src, float* dst, int64_t ld_dst, int64_t rows,
                            int64_t cols, int32_t accumulate, void* stream) {
  B2_REQUIRE(src && dst, "copy2d: NULL pointer");
  B2_REQUIRE(ld_src >= cols && ld_dst >= cols, "copy2d: leading dimension < cols");
  if (rows <= 0 || cols <= 0) return B2CTR_OK;
  const bool v4 = cols % 4 == 0 && ld_src % 4 == 0 && ld_dst % 4 == 0 &&
                  ((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0;
  if (v4)
    copy2d_kernel<true><<<grid_for(rows * cols / 4, 256, 8), 256, 0, ST>>>(src, ld_src, dst, ld_dst,
                                                                          rows, cols, accumulate);
  else
    copy2d_kernel<false><<<grid_for(rows * cols, 256, 8), 256, 0, ST>>>(src, ld_src, dst, ld_dst, rows,
                                                                       cols, accumulate);
  B2_CHECK_LAUNCH("b2ctr_copy2d");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_pack_rows(const float* src, const int32_t* widths, int32_t nblk, int64_t batch, float* dst,
                               int64_t ld_dst, void* stream) {
  B2_REQUIRE(src && widths && dst && nblk >= 1 && nblk <= 64, "pack_rows: need 1..64 blocks");
  PackCols pc;
  int64_t off = 0;
  int col = 0;
  for (int i = 0; i < nblk; ++i) {
    B2_REQUIRE(widths[i] > 0, "pack_rows: width %d is not positive", i);
    pc.off[i] = off; pc.width[i] = widths[i]; pc.col[i] = col;
    off += (int64_t)widths[i] * batch;
    col += widths[i];
  }
  pc.nblk = nblk; pc.total = col;
  B2_REQUIRE(ld_dst >= col, "pack_rows: ld_dst < total width");
  if (batch <= 0) return B2CTR_OK;
  pack_rows_kernel<<<grid_for(batch * col, 256, 8), 256, 0, ST>>>(src, pc, batch, dst, ld_dst);
  B2_CHECK_LAUNCH("b2ctr_pack_rows");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_rowsum(const float* x, int64_t ld, float* out, int64_t rows, int64_t cols,
                            void* stream) {
  B2_REQUIRE(x && out && ld >= cols, "rowsum: bad arguments");
  if (rows <= 0) return B2CTR_OK;
  rowsum_kernel<<<grid_for(rows, 8, 8), 256, 0, ST>>>(x, ld, out, rows, cols);
  B2_CHECK_LAUNCH("b2ctr_rowsum");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_fm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, float* out,
                            int64_t batch, void* stream) {
  B2_REQUIRE(x && out && nfield > 0 && dim > 0 && ldx >= (int64_t)nfield * dim, "fm_fwd: bad arguments");
  if (batch <= 0) return B2CTR_OK;
  fm_fwd_kernel<false><<<grid_for(batch, 8, 8), 256, 0, ST>>>(x, ldx, nullptr, 0, nfield, dim, out, batch);
  B2_CHECK_LAUNCH("b2ctr_fm_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_fm_bwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* dout,
                            float* dx, int64_t lddx, int32_t accumulate, int64_t batch, void* stream) {
  B2_REQUIRE(x && dout && dx && nfield > 0 && dim > 0, "fm_bwd: bad arguments");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && lddx >= (int64_t)nfield * dim, "fm_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  fm_bwd_kernel<false><<<grid_for(batch, 8, 8), 256, 0, ST>>>(x, ldx, nullptr, 0, nfield, dim, dout, dx, lddx,
                                                             nullptr, 0, accumulate, batch);
  B2_CHECK_LAUNCH("b2ctr_fm_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_fm_weighted_fwd(const float* x, int64_t ldx, const float* m, int64_t ldm, int32_t nfield,
                                     int32_t dim, float* out, int64_t batch, void* stream) {
  B2_REQUIRE(x && m && out && nfield > 0 && dim > 0, "fm_weighted_fwd: bad arguments");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && ldm >= nfield, "fm_weighted_fwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  fm_fwd_kernel<true><<<grid_for(batch, 8, 8), 256, 0, ST>>>(x, ldx, m, ldm, nfield, dim, out, batch);
  B2_CHECK_LAUNCH("b2ctr_fm_weighted_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_fm_weighted_bwd(const float* x, int64_t ldx, const float* m, int64_t ldm, int32_t nfield,
                                     int32_t dim, const float* dout, float* dx, int64_t lddx, int32_t accumulate,
                                     float* dm, int64_t lddm, int64_t batch, void* stream) {
  B2_REQUIRE(x && m && dout && (dx || dm) && nfield > 0 && dim > 0, "fm_weighted_bwd: bad arguments");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && ldm >= nfield && (!dx || lddx >= (int64_t)nfield * dim) &&
                 (!dm || lddm >= nfield),
             "fm_weighted_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  fm_bwd_kernel<true><<<grid_for(batch, 8, 8), 256, 0, ST>>>(x, ldx, m, ldm, nfield, dim, dout, dx, lddx, dm,
                                                            lddm, accumulate, batch);
  B2_CHECK_LAUNCH("b2ctr_fm_weighted_bwd");
  return B2CTR_OK;
}

static int field_scale_width(int32_t dim) {
  int w = 1;
  while (w < dim && w < 32) w <<= 1;
  return w;
}

b2ctr_status_t b2ctr_field_scale_fwd(const float* x, int64_t ldx, const float* m, int64_t ldm, int32_t nfield,
                                     int32_t dim, float* y, int64_t ldy, int64_t batch, void* stream) {
  B2_REQUIRE(x && m && y && nfield > 0 && dim > 0, "field_scale_fwd: bad arguments");
  B2_REQUIRE(ldx >= (int64_t)nfield * dim && ldm >= nfield && ldy >= (int64_t)nfield * dim,
             "field_scale_fwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  const int w = field_scale_width(dim);
  field_scale_fwd_kernel<<<grid_for(batch * nfield, 256 / w, 8), 256, 0, ST>>>(x, ldx, m, ldm, nfield, dim, y, ldy,
                                                                               batch, w);
  B2_CHECK_LAUNCH("b2ctr_field_scale_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_field_scale_bwd(const float* dy, int64_t lddy, const float* x, int64_t ldx, const float* m,
                                     int64_t ldm, int32_t nfield, int32_t dim, float* dx, int64_t lddx,
                                     int32_t accumulate, float* dm, int64_t lddm, int64_t batch, void* stream) {
  B2_REQUIRE(dy && x && m && (dx || dm) && nfield > 0 && dim > 0, "field_scale_bwd: bad arguments");
  B2_REQUIRE(lddy >= (int64_t)nfield * dim && ldx >= (int64_t)nfield * dim && ldm >= nfield &&
                 (!dx || lddx >= (int64_t)nfield * dim) && (!dm || lddm >= nfield),
             "field_scale_bwd: ld too small");
  if (batch <= 0) return B2CTR_OK;
  const int w = field_scale_width(dim);
  field_scale_bwd_kernel<<<grid_for(batch * nfield, 256 / w, 8), 256, 0, ST>>>(
      dy, lddy, x, ldx, m, ldm, nfield, dim, dx, lddx, dm, lddm, accumulate, batch, w);
  B2_CHECK_LAUNCH("b2ctr_field_scale_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_softmax_rows_fwd(const float* x, int64_t ldx, float* y, int64_t ldy, int64_t rows,
                                      int32_t cols, float scale, void* stream) {
  B2_REQUIRE(x && y && cols > 0 && ldx >= cols && ldy >= cols && scale != 0.f, "softmax_rows_fwd: bad arguments");
  if (rows <= 0) return B2CTR_OK;
  softmax_rows_fwd_kernel<<<grid_for(rows, 8, 8), 256, 0, ST>>>(x, ldx, y, ldy, rows, cols, scale);
  B2_CHECK_LAUNCH("b2ctr_softmax_rows_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_softmax_rows_bwd(const float* y, int64_t ldy, const float* dy, int64_t lddy, float* dx,
                                      int64_t lddx, int64_t rows, int32_t cols, float scale, void* stream) {
  B2_REQUIRE(y && dy && dx && cols > 0 && ldy >= cols && lddy >= cols && lddx >= cols && scale != 0.f,
             "softmax_rows_bwd: bad arguments");
  if (rows <= 0) return B2CTR_OK;
  softmax_rows_bwd_kernel<<<grid_for(rows, 8, 8), 256, 0, ST>>>(y, ldy, dy, lddy, dx, lddx, rows, cols, scale);
  B2_CHECK_LAUNCH("b2ctr_softmax_rows_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_predict_loss(const float* logit, const float* bias, const float* labels,
                                  float* pred, float* dlogit, float* dbias, float* loss_sum,
                                  int64_t batch, int32_t task, void* stream) {
  B2_REQUIRE(logit, "predict_loss: NULL logit");
  B2_REQUIRE(task == B2CTR_TASK_BINARY || task == B2CTR_TASK_REGRESSION, "predict_loss: bad task");
  B2_REQUIRE(labels || (!dlogit && !loss_sum && !dbias), "predict_loss: labels required for loss/grad");
  if (batch <= 0) return B2CTR_OK;
  predict_loss_kernel<<<grid_for(batch, 256, 4), 256, 0, ST>>>(logit, bias, labels, pred, dlogit, dbias,
                                                              loss_sum, batch, task);
  B2_CHECK_LAUNCH("b2ctr_predict_loss");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_sgd_step(float* w, const float* g, float lr, float l2, int64_t n, void* stream) {
  B2_REQUIRE(w && g, "sgd_step: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  sgd_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(w, g, lr, l2, n);
  B2_CHECK_LAUNCH("b2ctr_sgd_step");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_sgd_step_multi(float* const* w, const float* const* g, const int64_t* n, const float* l2,
                                    int32_t count, float lr, void* stream) {
  B2_REQUIRE(w && g && n && l2 && count >= 0, "sgd_step_multi: NULL pointer");
  for (int32_t base = 0; base < count; base += kSgdMulti) {
    SgdMulti p;
    const int32_t c = count - base < kSgdMulti ? count - base : kSgdMulti;
    int64_t nmax = 0;
    for (int32_t i = 0; i < c; ++i) {
      B2_REQUIRE(w[base + i] && g[base + i] && n[base + i] >= 0, "sgd_step_multi: NULL tensor %d", base + i);
      p.w[i] = w[base + i]; p.g[i] = g[base + i]; p.n[i] = n[base + i]; p.l2[i] = l2[base + i];
      if (p.n[i] > nmax) nmax = p.n[i];
    }
    if (nmax == 0) continue;
    dim3 grid((unsigned)grid_for(nmax, 256, 8), (unsigned)c);
    sgd_multi_kernel<<<grid, 256, 0, ST>>>(p, lr);
    B2_CHECK_LAUNCH("b2ctr_sgd_step_multi");
  }
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_adam_step(float* w, const float* g, float* m, float* v, float lr, float beta1,
                               float beta2, float eps, float l2, int64_t step, int64_t n, void* stream) {
  B2_REQUIRE(w && g && m && v && step >= 1, "adam_step: NULL pointer or step < 1");
  if (n <= 0) return B2CTR_OK;
  // Keras: lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t)
  const double lr_t = (double)lr * sqrt(1.0 - pow((double)beta2, (double)step)) /
                      (1.0 - pow((double)beta1, (double)step));
  adam_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(w, g, m, v, (float)lr_t, beta1, beta2, eps, l2, n);
  B2_CHECK_LAUNCH("b2ctr_adam_step");
  return B2CTR_OK;
}

// Adam with the step count in device memory: nothing step-dependent is passed by value, so the launch can be
// part of a replayed CUDA graph (the counter is advanced once per step by b2ctr_counter_add).
__global__ void adam_dev_kernel(float* w, const float* __restrict__ g, float* m, float* v, float lr, float b1,
                                float b2, float eps, float l2, const int64_t* __restrict__ step, int64_t n) {
  const double t = (double)(*step);
  const float lr_t = (float)((double)lr * sqrt(1.0 - pow((double)b2, t)) / (1.0 - pow((double)b1, t)));
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] + 2.f * l2 * w[i];
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    w[i] -= lr_t * mi / (sqrtf(vi) + eps);
  }
}
__global__ void counter_add_kernel(int64_t* c, int64_t delta) { *c += delta; }

b2ctr_status_t b2ctr_adam_step_dev(float* w, const float* g, float* m, float* v, float lr, float beta1,
                                   float beta2, float eps, float l2, const int64_t* step_dev, int64_t n,
                                   void* stream) {
  B2_REQUIRE(w && g && m && v && step_dev, "adam_step_dev: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  adam_dev_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(w, g, m, v, lr, beta1, beta2, eps, l2, step_dev, n);
  B2_CHECK_LAUNCH("b2ctr_adam_step_dev");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_counter_add(int64_t* counter, int64_t delta, void* stream) {
  B2_REQUIRE(counter, "counter_add: NULL pointer");
  counter_add_kernel<<<1, 1, 0, ST>>>(counter, delta);
  B2_CHECK_LAUNCH("b2ctr_counter_add");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_adagrad_step(float* w, const float* g, float* acc, float lr, float eps, float l2,
                                  int64_t n, void* stream) {
  B2_REQUIRE(w && g && acc, "adagrad_step: NULL pointer");
  if (n <= 0) return B2CTR_OK;
  adagrad_kernel<<<grid_for(n, 256, 8), 256, 0, ST>>>(w, g, acc, lr, eps, l2, n);
  B2_CHECK_LAUNCH("b2ctr_adagrad_step");
  return B2CTR_OK;
}

}  // extern "C"
