// embed.cu — fused multi-table embedding gather / scatter-update for sm_90a.
//
// Reference semantics restated here (never copied): deepctr/inputs.py:101-158 (lookup + pooling
// dispatch), deepctr/layers/sequence.py:76-106 (SequencePoolingLayer), :155-183
// (WeightedSequenceLayer), deepctr/layers/utils.py:89-112 (Hash), deepctr/feature_column.py:171-233.
//
// HBM-bound integer/byte work: no tensor cores.  Design rules (DESIGN.md §3):
//   * one launch for all tables; descriptors travel by value in the kernel parameter block;
//   * 128-bit row accesses, rows never staged through L1 (ld.global.nc.L1::no_allocate);
//   * every lane keeps several independent 16 B loads in flight.  Little's law on an H100 SXM: 3.35 TB/s x ~0.8 us
//     of loaded HBM latency is ~2.7 MB in flight, i.e. ~20 KB per SM = ~1300 16 B loads; 32 warps x 32 lanes x
//     4-7 loads per lane covers it;
//   * row updates are REDG.E.ADD.F32x4 (the add executes in the L2 slice, no read by the SM);
//   * grids are whole multiples of the 132 SMs.
#include "common.cuh"

namespace b2ctr {

// ============================================================================================
// FarmHash Fingerprint64 (== farmhashna::Hash64) for byte strings of length <= 32; restated
// from the published algorithm (google/farmhash, farmhash.cc), not present under /root/reference
// (TensorFlow's tf.strings.to_hash_bucket_fast calls it; deepctr/layers/utils.py:103-107).
// ============================================================================================
namespace farm {
__host__ __device__ constexpr uint64_t k0() { return 0xc3a5c85c97cb3127ULL; }
__host__ __device__ constexpr uint64_t k1() { return 0xb492b66fbe98f273ULL; }
__host__ __device__ constexpr uint64_t k2() { return 0x9ae16a3b2f90404fULL; }
__device__ __forceinline__ uint64_t rot(uint64_t v, int s) { return (v >> s) | (v << (64 - s)); }
__device__ __forceinline__ uint64_t shift_mix(uint64_t v) { return v ^ (v >> 47); }
__device__ __forceinline__ uint64_t fetch64(const unsigned char* p) {
  uint64_t r = 0;
#pragma unroll
  for (int i = 7; i >= 0; --i) r = (r << 8) | p[i];
  return r;
}
__device__ __forceinline__ uint64_t fetch32(const unsigned char* p) {
  return (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t hash_len16(uint64_t u, uint64_t v, uint64_t mul) {
  uint64_t a = (u ^ v) * mul;
  a ^= (a >> 47);
  uint64_t b = (v ^ a) * mul;
  b ^= (b >> 47);
  b *= mul;
  return b;
}
__device__ uint64_t fingerprint64(const unsigned char* s, int len) {
  if (len <= 16) {
    if (len >= 8) {
      uint64_t mul = k2() + (uint64_t)len * 2;
      uint64_t a = fetch64(s) + k2();
      uint64_t b = fetch64(s + len - 8);
      uint64_t c = rot(b, 37) * mul + a;
      uint64_t d = (rot(a, 25) + b) * mul;
      return hash_len16(c, d, mul);
    }
    if (len >= 4) {
      uint64_t mul = k2() + (uint64_t)len * 2;
      uint64_t a = fetch32(s);
      return hash_len16((uint64_t)len + (a << 3), fetch32(s + len - 4), mul);
    }
    if (len > 0) {
      uint32_t a = s[0], b = s[len >> 1], c = s[len - 1];
      uint32_t y = a + (b << 8);
      uint32_t z = (uint32_t)len + (c << 2);
      return shift_mix((uint64_t)y * k2() ^ (uint64_t)z * k0()) * k2();
    }
    return k2();
  }
  // 17..32
  uint64_t mul = k2() + (uint64_t)len * 2;
  uint64_t a = fetch64(s) * k1();
  uint64_t b = fetch64(s + 8);
  uint64_t c = fetch64(s + len - 8) * mul;
  uint64_t d = fetch64(s + len - 16) * k2();
  return hash_len16(rot(a + b, 43) + rot(c, 30) + d, a + rot(b + k2(), 18) + c, mul);
}
// tf.as_string(int): decimal, '-' prefix for negatives.  Returns length (<= 20).
__device__ __forceinline__ int to_decimal(int64_t v, unsigned char* buf) {
  unsigned char tmp[20];
  int n = 0;
  bool neg = v < 0;
  uint64_t u = neg ? (uint64_t)(-(v + 1)) + 1ULL : (uint64_t)v;
  do {
    tmp[n++] = (unsigned char)('0' + (u % 10));
    u /= 10;
  } while (u);
  int len = 0;
  if (neg) buf[len++] = '-';
  while (n) buf[len++] = tmp[--n];
  return len;
}
__device__ __forceinline__ int64_t hash_bucket(int64_t id, int64_t num_buckets, bool mask_zero) {
  unsigned char buf[24];
  int len = to_decimal(id, buf);
  uint64_t nb = (uint64_t)(mask_zero ? num_buckets - 1 : num_buckets);
  uint64_t h = fingerprint64(buf, len) % nb;
  if (mask_zero) return id == 0 ? 0 : (int64_t)(h + 1);
  return (int64_t)h;
}
}  // namespace farm

__device__ __forceinline__ int64_t lookup_id(const b2ctr_feature_t& ft, int64_t off) {
  int64_t id = load_idx(ft.idx, off, ft.idx_dtype);
  if (ft.hash_mode != B2CTR_HASH_NONE)
    id = farm::hash_bucket(id, ft.vocab, ft.hash_mode == B2CTR_HASH_FARM_MASK_ZERO);
  return id;
}

// ============================================================================================
// Generic kernels: one sub-warp group of G lanes per (sample, feature) task.
// ============================================================================================
constexpr int kFeatChunk = 64;  // descriptors per launch (6 KB of kernel parameters)
struct FeatBlock {
  b2ctr_feature_t f[kFeatChunk];
  unsigned long long* oob;      // out-of-range id counter (common.cuh)
  int32_t nfeat;
};

template <int VEC>
struct VecT;
template <>
struct VecT<4> {
  using T = float4;
};
template <>
struct VecT<1> {
  using T = float;
};

template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::T vzero();
template <>
__device__ __forceinline__ float4 vzero<4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <>
__device__ __forceinline__ float vzero<1>() { return 0.f; }

__device__ __forceinline__ float4 vload(const float* p, float4*) { return ldg_stream_f4(p); }
__device__ __forceinline__ float vload(const float* p, float*) { return ldg_stream_f1(p); }
__device__ __forceinline__ void vstore(float* p, float4 v) { stg_stream_f4(p, v); }
__device__ __forceinline__ void vstore(float* p, float v) { *p = v; }
__device__ __forceinline__ void vred(float* p, float4 v) { red_add_f4(p, v); }
__device__ __forceinline__ void vred(float* p, float v) { red_add_f1(p, v); }

// fp32 ops with no FMA contraction so pooled sums are bit-exact against the oracle
__device__ __forceinline__ float4 vadd(float4 a, float4 b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z),
                     __fadd_rn(a.w, b.w));
}
__device__ __forceinline__ float vadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float4 vmuls(float4 a, float s) {
  return make_float4(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s), __fmul_rn(a.w, s));
}
__device__ __forceinline__ float vmuls(float a, float s) { return __fmul_rn(a, s); }
__device__ __forceinline__ bool vnonzero(float4 a) { return a.x != 0.f || a.y != 0.f || a.z != 0.f || a.w != 0.f; }
__device__ __forceinline__ bool vnonzero(float a) { return a != 0.f; }
__device__ __forceinline__ float4 vdivs(float4 a, float s) {
  return make_float4(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s), __fdiv_rn(a.w, s));
}
__device__ __forceinline__ float vdivs(float a, float s) { return __fdiv_rn(a, s); }
__device__ __forceinline__ float4 vsubs(float4 a, float s) {
  return make_float4(__fsub_rn(a.x, s), __fsub_rn(a.y, s), __fsub_rn(a.z, s), __fsub_rn(a.w, s));
}
__device__ __forceinline__ float vsubs(float a, float s) { return __fsub_rn(a, s); }
__device__ __forceinline__ float4 vmax(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ float vmax(float a, float b) { return fmaxf(a, b); }

// strides of the optional per-sample side inputs (0 = dense default)
__device__ __forceinline__ int64_t wld(const b2ctr_feature_t& ft) { return ft.weight_ld > 0 ? ft.weight_ld : ft.maxlen; }
__device__ __forceinline__ int64_t lstride(const b2ctr_feature_t& ft) { return ft.len_stride > 0 ? ft.len_stride : 1; }

struct SeqInfo {
  float L;      // float(valid length) as the reference computes it
  float wmax;   // softmax max
  float wsum;   // softmax denominator
};

// validity of position t given the (post-hash) id
__device__ __forceinline__ bool pos_valid(const b2ctr_feature_t& ft, int t, int64_t id, int len) {
  if (ft.mask_mode == B2CTR_MASK_LENGTH) return t < len;
  if (ft.mask_mode == B2CTR_MASK_ZERO_ID) return id != 0;
  return true;
}

// per-position weight after WeightedSequenceLayer (sequence.py:170-183); 1 if unweighted
__device__ __forceinline__ float pos_weight(const b2ctr_feature_t& ft, const SeqInfo& si, int64_t b,
                                            int t, bool valid) {
  if (ft.weight_mode == B2CTR_WEIGHT_NONE) return 1.f;
  float w = ft.weight[b * wld(ft) + t];
  if (ft.weight_mode == B2CTR_WEIGHT_RAW) return valid ? w : 0.f;
  float wt = valid ? w : -4294967295.f;  // -2^32+1 rounds to -2^32 in fp32, as in TF
  return __fdiv_rn(expf(__fsub_rn(wt, si.wmax)), si.wsum);
}

__device__ SeqInfo seq_info(const b2ctr_feature_t& ft, int64_t b) {
  SeqInfo si;
  si.L = 0.f;
  si.wmax = 0.f;
  si.wsum = 1.f;
  const int T = ft.maxlen;
  const int len = ft.mask_mode == B2CTR_MASK_LENGTH ? ft.len[b * lstride(ft)] : 0;
  if (ft.mask_mode == B2CTR_MASK_LENGTH) {
    si.L = (float)len;
  } else if (ft.mask_mode == B2CTR_MASK_ZERO_ID) {
    int c = 0;
    for (int t = 0; t < T; ++t) c += lookup_id(ft, b * ft.idx_stride + t) != 0;
    si.L = (float)c;
  } else {
    si.L = (float)T;
  }
  if (ft.weight_mode == B2CTR_WEIGHT_SOFTMAX) {
    float m = -INFINITY;
    for (int t = 0; t < T; ++t) {
      int64_t id = ft.mask_mode == B2CTR_MASK_ZERO_ID ? lookup_id(ft, b * ft.idx_stride + t) : 1;
      bool v = pos_valid(ft, t, id, len);
      float w = v ? ft.weight[b * wld(ft) + t] : -4294967295.f;
      m = fmaxf(m, w);
    }
    float s = 0.f;
    for (int t = 0; t < T; ++t) {
      int64_t id = ft.mask_mode == B2CTR_MASK_ZERO_ID ? lookup_id(ft, b * ft.idx_stride + t) : 1;
      bool v = pos_valid(ft, t, id, len);
      float w = v ? ft.weight[b * wld(ft) + t] : -4294967295.f;
      s = __fadd_rn(s, expf(__fsub_rn(w, m)));
    }
    si.wmax = m;
    si.wsum = s;
  }
  return si;
}

template <int G, int VEC>
__global__ void __launch_bounds__(256)
    embed_gather_generic_kernel(const __grid_constant__ FeatBlock fb, int64_t batch) {
  using V = typename VecT<VEC>::T;
  constexpr int kGroups = 256 / G;
  const int lane = threadIdx.x % G;
  const int64_t ntasks = batch * fb.nfeat;
  for (int64_t task = (int64_t)blockIdx.x * kGroups + threadIdx.x / G; task < ntasks;
       task += (int64_t)gridDim.x * kGroups) {
    const int64_t b = task / fb.nfeat;
    const b2ctr_feature_t& ft = fb.f[task - b * fb.nfeat];
    const int dim = ft.dim, T = ft.maxlen;
    float* out = ft.out + b * ft.out_ld + ft.out_col;
    const int64_t ibase = b * ft.idx_stride;

    if (ft.pool == B2CTR_POOL_NONE) {
      // plain lookup: T rows copied verbatim (padded positions read their real row; Keras masks later)
      for (int t = 0; t < T; ++t) {
        const int64_t id = lookup_id(ft, ibase + t);
        const bool ok = id_in_range(id, ft.vocab);       // out-of-range id: zero row (+ counted)
        if (!ok && lane == 0) note_oob(fb.oob);
        const float* row = ft.table + (ok ? id : 0) * dim;
        for (int e = lane * VEC; e < dim; e += G * VEC)
          vstore(out + (int64_t)t * dim + e, ok ? vload(row + e, (V*)nullptr) : vzero<VEC>());
      }
      continue;
    }

    const int len = ft.mask_mode == B2CTR_MASK_LENGTH ? ft.len[b * lstride(ft)] : 0;
    const SeqInfo si = seq_info(ft, b);
    for (int e = lane * VEC; e < dim; e += G * VEC) {
      V acc = vzero<VEC>();
      bool first = true;
      for (int t0 = 0; t0 < T; t0 += 4) {
        int64_t id[4];
        bool val[4];
        V x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int t = t0 + u;
          id[u] = t < T ? lookup_id(ft, ibase + t) : 0;
          val[u] = t < T && pos_valid(ft, t, id[u], len);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          // max pooling reads masked rows too (x - 1e9 competes, sequence.py:97-98)
          const bool need = t0 + u < T && (val[u] || ft.pool == B2CTR_POOL_MAX);
          const bool ok = id_in_range(id[u], ft.vocab);
          if (need && !ok && e == 0) note_oob(fb.oob);      // e == 0 <=> lane 0, first pass
          x[u] = (need && ok) ? vload(ft.table + id[u] * dim + e, (V*)nullptr) : vzero<VEC>();
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int t = t0 + u;
          if (t >= T) break;
          V v = x[u];
          if (ft.weight_mode != B2CTR_WEIGHT_NONE) v = vmuls(v, pos_weight(ft, si, b, t, val[u]));
          if (ft.pool == B2CTR_POOL_MAX) {
            if (!val[u]) v = vsubs(v, 1e9f);
            acc = first ? v : vmax(acc, v);
            first = false;
          } else if (val[u]) {
            acc = vadd(acc, v);  // ascending t, fp32, no fma: bit-exact segment sum
          }
        }
      }
      if (ft.pool == B2CTR_POOL_MEAN) acc = vdivs(acc, __fadd_rn(si.L, 1e-8f));
      vstore(out + e, acc);
    }
  }
}

template <int G, int VEC>
__global__ void __launch_bounds__(256)
    embed_scatter_generic_kernel(const __grid_constant__ FeatBlock fb, int64_t batch, float scale) {
  using V = typename VecT<VEC>::T;
  constexpr int kGroups = 256 / G;
  const int lane = threadIdx.x % G;
  const unsigned gmask = G >= 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << ((threadIdx.x & 31) / G * G));
  const int64_t ntasks = batch * fb.nfeat;
  for (int64_t task = (int64_t)blockIdx.x * kGroups + threadIdx.x / G; task < ntasks;
       task += (int64_t)gridDim.x * kGroups) {
    const int64_t b = task / fb.nfeat;
    const b2ctr_feature_t& ft = fb.f[task - b * fb.nfeat];
    const int dim = ft.dim, T = ft.maxlen;
    const float* gout = ft.out + b * ft.out_ld + ft.out_col;
    const int64_t ibase = b * ft.idx_stride;

    if (ft.pool == B2CTR_POOL_NONE) {
      for (int t = 0; t < T; ++t) {
        const int64_t id = lookup_id(ft, ibase + t);
        if (!id_in_range(id, ft.vocab)) continue;          // never write outside the table
        // an all-zero gradient row (every masked position of a behaviour sequence: half of a padded batch,
        // all of them aimed at row 0) changes nothing: skip its atomics
        bool nz = false;
        for (int e = lane * VEC; e < dim; e += G * VEC) nz |= vnonzero(vload(gout + (int64_t)t * dim + e, (V*)nullptr));
        if (__ballot_sync(gmask, nz) == 0u) continue;
        float* row = ft.table + id * dim;
        for (int e = lane * VEC; e < dim; e += G * VEC)
          vred(row + e, vmuls(vload(gout + (int64_t)t * dim + e, (V*)nullptr), scale));
      }
      continue;
    }
    const int len = ft.mask_mode == B2CTR_MASK_LENGTH ? ft.len[b * lstride(ft)] : 0;
    const SeqInfo si = seq_info(ft, b);
    for (int e = lane * VEC; e < dim; e += G * VEC) {
      V g = vmuls(vload(gout + e, (V*)nullptr), scale);
      if (ft.pool == B2CTR_POOL_MEAN) g = vdivs(g, __fadd_rn(si.L, 1e-8f));
      if (ft.pool == B2CTR_POOL_MAX) {
        // TF's max gradient: split evenly among the positions that attain the max
        float gv[VEC], mx[VEC];
        int cnt[VEC];
        {
          float tmp[VEC];
          *reinterpret_cast<V*>(tmp) = g;
#pragma unroll
          for (int i = 0; i < VEC; ++i) { gv[i] = tmp[i]; mx[i] = -INFINITY; cnt[i] = 0; }
        }
        for (int pass = 0; pass < 2; ++pass) {
          for (int t = 0; t < T; ++t) {
            const int64_t id = lookup_id(ft, ibase + t);
            const bool valid = pos_valid(ft, t, id, len);
            const bool ok = id_in_range(id, ft.vocab);
            V xv = ok ? vload((ft.src_table ? ft.src_table : ft.table) + id * dim + e, (V*)nullptr) : vzero<VEC>();
            const float w = pos_weight(ft, si, b, t, valid);
            if (ft.weight_mode != B2CTR_WEIGHT_NONE) xv = vmuls(xv, w);
            if (!valid) xv = vsubs(xv, 1e9f);
            float xs[VEC];
            *reinterpret_cast<V*>(xs) = xv;
            if (pass == 0) {
#pragma unroll
              for (int i = 0; i < VEC; ++i) {
                if (xs[i] > mx[i]) { mx[i] = xs[i]; cnt[i] = 1; }
                else if (xs[i] == mx[i]) cnt[i]++;
              }
            } else {
#pragma unroll
              for (int i = 0; i < VEC; ++i)
                if (xs[i] == mx[i] && ok) red_add_f1(ft.table + id * dim + e + i, gv[i] / (float)cnt[i] * w);
            }
          }
        }
        continue;
      }
      for (int t = 0; t < T; ++t) {
        const int64_t id = lookup_id(ft, ibase + t);
        const bool valid = pos_valid(ft, t, id, len);
        if (!valid || !id_in_range(id, ft.vocab)) continue;
        V gt = g;
        if (ft.weight_mode != B2CTR_WEIGHT_NONE) gt = vmuls(gt, pos_weight(ft, si, b, t, true));
        vred(ft.table + id * dim + e, gt);
      }
    }
  }
}

// ============================================================================================
// Criteo-shaped fast path: one warp per sample, F same-dim single-valued tables.
// ============================================================================================
constexpr int kUniMaxFeat = 64;
struct UniParams {
  float* table[kUniMaxFeat];
  float* lin[kUniMaxFeat];
  const void* idx[kUniMaxFeat];
  int64_t idx_stride[kUniMaxFeat];
  int64_t vocab[kUniMaxFeat];     // FULL vocabulary (also when the table is row-sharded): id validity
  unsigned long long* oob;
  const float* dense;
  float* x;
  float* linear;
  float* fm;
  int64_t ldx;
  int64_t dense_ld;
  int64_t x_cols;
  uint64_t fm_mask;
  int32_t nfeat;
  int32_t ndense;
  int32_t dim;
  int32_t idx_dtype;
  int32_t has_lin;
  int32_t store_grads;
  // row-sharded tables over peer mappings (world = 2^wshift shards): device arrays [nfeat * world]
  float* const* peer_tab;
  float* const* peer_lin;
  int32_t world;
  int32_t wshift;
  // FM sum vectors S[b, 0:dim] (gather: written, scatter: read instead of re-summing x), or NULL
  float* fm_sum;
  // gather only: bf16 hi/lo planes (b2ctr_split_planes layout) of x[:, 0:xp_cols], row pitch xp_pitch, or NULL
  __nv_bfloat16* xp_hi;
  __nv_bfloat16* xp_lo;
  int64_t xp_pitch;
  int64_t xp_rows_pad;
};

// hi = bf16_rn(v), lo = bf16_rn(v - hi): the values b2ctr_split_planes writes
__device__ __forceinline__ void store_planes4(const UniParams& p, int64_t off, float4 v) {
  const __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y);
  const __nv_bfloat16 h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
  uint2 h, l;
  h.x = pack_bf16(h0, h1);
  h.y = pack_bf16(h2, h3);
  l.x = pack_bf16(__float2bfloat16_rn(v.x - __bfloat162float(h0)), __float2bfloat16_rn(v.y - __bfloat162float(h1)));
  l.y = pack_bf16(__float2bfloat16_rn(v.z - __bfloat162float(h2)), __float2bfloat16_rn(v.w - __bfloat162float(h3)));
  *reinterpret_cast<uint2*>(p.xp_hi + off) = h;
  *reinterpret_cast<uint2*>(p.xp_lo + off) = l;
}

// peer (NVLink) accesses: no read-only / L2-policy qualifiers - the line lives in the owner's L2
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ld_peer_f1(const float* p) {
  float r;
  asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void red_peer_f4(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void red_peer_f1(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// shard pointer + local row of global row `id` of feature f
__device__ __forceinline__ float* shard_row(float* const* tabs, const UniParams& p, int f, int64_t id, int width) {
  const int64_t own = id & (int64_t)(p.world - 1);
  return tabs[(int64_t)f * p.world + own] + (id >> p.wshift) * width;
}

__device__ __forceinline__ int64_t uni_id(const UniParams& p, int f, int64_t b) {
  return load_idx(p.idx[f], b * p.idx_stride[f], p.idx_dtype);
}

// LPR = lanes per row (= dim/4); RPI = rows per warp iteration; each lane keeps U 16-byte loads in flight.
// Latency hiding (ncu, profiles/r1_embed_before.txt: 40 % DRAM, 35 % warps active): the id -> row -> store
// chain is broken by prefetching the NEXT sample's ids before the current rows are requested, and the
// register budget is capped at 64 (4 CTAs = 32 warps per SM).  EXTRA: the instantiation that may also store S
// (p.fm_sum) and X's bf16 planes (p.xp_hi); those stores need 80 registers, so it runs 3 CTAs = 24 warps per SM,
// which still keep 24 x 32 x 7 x 16 B = 86 KB of row loads in flight per SM, four times the ~20 KB the H100's HBM
// needs (see the top of this file), and it is launched as one wave of 132 x 3 CTAs.
template <int LPR, bool SHARD, bool EXTRA>
__global__ void __launch_bounds__(256, (SHARD || EXTRA) ? 3 : 4)
    gather_uniform_fwd_kernel(const __grid_constant__ UniParams p, int64_t batch) {
  constexpr int RPI = 32 / LPR;
  constexpr int U = 7;   // 7 x RPI(4) = 28 >= 26 Criteo fields in one pass at dim 32
  const int lane = threadIdx.x & 31;
  const int slot = lane / LPR, chunk = lane % LPR;
  const int F = p.nfeat, dim = p.dim;
  const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  // ids: lane l holds features l and l+32.  They are validated against the vocabulary HERE, once per lookup
  // (an id outside [0, V) becomes -1: zero row, counted), so the row loop only tests a sign.
  auto checked = [&](int f, int64_t bb) -> int64_t {       // f: this lane's feature (lane or lane + 32)
    if (bb >= batch || f >= F) return 0;
    const int64_t id = uni_id(p, f, bb);
    if (id_in_range(id, p.vocab[f])) return id;
    note_oob(p.oob);
    return -1;
  };
  int64_t id0 = checked(lane, b);
  int64_t id1 = checked(lane + 32, b);
  for (; b < batch; b += nwarps) {
    const int64_t bn = b + nwarps;
    const int64_t nid0 = checked(lane, bn);        // prefetch
    const int64_t nid1 = checked(lane + 32, bn);
    float* xrow = p.x + b * p.ldx;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    float q = 0.f;
    for (int f0 = 0; f0 < F; f0 += U * RPI) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int f = f0 + u * RPI + slot;
        const int fs = f < F ? f : 0;
        const int64_t ida = __shfl_sync(0xffffffffu, id0, fs & 31);
        const int64_t idb = __shfl_sync(0xffffffffu, id1, fs & 31);
        const int64_t id = fs < 32 ? ida : idb;
        if (f < F) {
          if (id < 0) {                                     // out of range (see above): zero row
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          } else if (SHARD) {
            v[u] = ld_peer_f4(shard_row(p.peer_tab, p, f, id, dim) + chunk * 4);
          } else {
            v[u] = ldg_stream_f4_pol(p.table[f] + id * dim + chunk * 4, pol_stream);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int f = f0 + u * RPI + slot;
        if (f < F) {
          stg_stream_f4_pol(xrow + (int64_t)f * dim + chunk * 4, v[u], pol_stream);
          if (EXTRA && p.xp_hi) store_planes4(p, b * p.xp_pitch + (int64_t)f * dim + chunk * 4, v[u]);
          if ((p.fm_mask >> f) & 1ull) {
            s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w;
            q += v[u].x * v[u].x + v[u].y * v[u].y + v[u].z * v[u].z + v[u].w * v[u].w;
          }
        }
      }
    }
    if (p.fm != nullptr) {
      // S_e: combine the RPI row slots (lanes that share `chunk`), then sum S_e^2 over e
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1) {
        s.x += __shfl_xor_sync(0xffffffffu, s.x, o);
        s.y += __shfl_xor_sync(0xffffffffu, s.y, o);
        s.z += __shfl_xor_sync(0xffffffffu, s.z, o);
        s.w += __shfl_xor_sync(0xffffffffu, s.w, o);
      }
      // S as the scatter needs it: ascending f per lane slot, then the xor tree above
      if (EXTRA && p.fm_sum != nullptr && slot == 0) *reinterpret_cast<float4*>(p.fm_sum + b * dim + chunk * 4) = s;
      float sq = slot == 0 ? (s.x * s.x + s.y * s.y + s.z * s.z + s.w * s.w) : 0.f;
      sq = warp_sum(sq);
      q = warp_sum(q);
      if (lane == 0) p.fm[b] = 0.5f * (sq - q);
    }
    if (p.linear != nullptr) {
      float l = 0.f;
      if (p.has_lin) {
        const bool ok0 = lane < F && id0 >= 0;
        const bool ok1 = lane + 32 < F && id1 >= 0;
        if (SHARD) {
          if (ok0) l += ld_peer_f1(shard_row(p.peer_lin, p, lane, id0, 1));
          if (ok1) l += ld_peer_f1(shard_row(p.peer_lin, p, lane + 32, id1, 1));
        } else {
          if (ok0) l += ldg_f1_pol(p.lin[lane] + id0, pol_keep);
          if (ok1) l += ldg_f1_pol(p.lin[lane + 32] + id1, pol_keep);
        }
      }
      l = warp_sum(l);
      if (lane == 0) p.linear[b] = l;
    }
    // dense passthrough + zero padding up to x_cols (so x is directly the K-padded GEMM operand)
    const int64_t c0 = (int64_t)F * dim;
    for (int64_t c = c0 + lane; c < p.x_cols; c += 32) {
      const int j = (int)(c - c0);
      xrow[c] = j < p.ndense ? p.dense[b * p.dense_ld + j] : 0.f;
    }
    if (EXTRA && p.xp_hi) {      // plane columns behind the embeddings: the dense features, then zeros up to the pitch
      for (int64_t c = c0 + lane; c < p.xp_pitch; c += 32) {
        const int j = (int)(c - c0);
        const float v = j < p.ndense ? p.dense[b * p.dense_ld + j] : 0.f;
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        p.xp_hi[b * p.xp_pitch + c] = h;
        p.xp_lo[b * p.xp_pitch + c] = __float2bfloat16_rn(v - __bfloat162float(h));
      }
    }
    id0 = nid0;
    id1 = nid1;
  }
  if (EXTRA && p.xp_hi) {        // plane rows [batch, rows_pad) are zero
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (int64_t r = b; r < p.xp_rows_pad; r += nwarps)
      for (int64_t c = lane * 8; c < p.xp_pitch; c += 256) {
        *reinterpret_cast<uint4*>(p.xp_hi + r * p.xp_pitch + c) = z;
        *reinterpret_cast<uint4*>(p.xp_lo + r * p.xp_pitch + c) = z;
      }
  }
}

// Backward: 4 dx + 4 x loads in flight per lane, reds issued as soon as a chunk's gradient is formed
// (fire-and-forget), ids re-broadcast by shuffle instead of being kept in registers.  With the gather's S
// (p.fm_sum) the first red of a sample waits only for its own dx and x rows, not for a pass over all F rows; X is
// still read once, for the x of the Jacobian.
template <int LPR, bool SHARD>
__global__ void __launch_bounds__(256, SHARD ? 2 : 3)
    scatter_uniform_bwd_kernel(const __grid_constant__ UniParams p, const float* __restrict__ dx,
                               const float* __restrict__ dfm, const float* __restrict__ dlinear,
                               float scale, float lin_scale, int64_t batch) {
  constexpr int RPI = 32 / LPR;
  constexpr int U = 4;
  const int lane = threadIdx.x & 31;
  const int slot = lane / LPR, chunk = lane % LPR;
  const int F = p.nfeat, dim = p.dim;
  const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  auto checked = [&](int f, int64_t bb) -> int64_t {       // -1: id outside the vocabulary, skipped
    if (bb >= batch || f >= F) return 0;
    const int64_t id = uni_id(p, f, bb);
    return id_in_range(id, p.vocab[f]) ? id : -1;
  };
  int64_t id0 = checked(lane, b);
  int64_t id1 = checked(lane + 32, b);
  for (; b < batch; b += nwarps) {
    const int64_t bn = b + nwarps;
    const int64_t nid0 = checked(lane, bn);
    const int64_t nid1 = checked(lane + 32, bn);
    const float* xrow = p.x + b * p.ldx;
    const float* dxrow = dx ? dx + b * p.ldx : nullptr;
    const float gfm = dfm ? dfm[b] : 0.f;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (dfm && p.fm_sum) {
      s = *reinterpret_cast<const float4*>(p.fm_sum + b * dim + chunk * 4);   // the gather's S
    } else if (dfm) {
      // no stored S: sum the FM rows of x in the gather's order (ascending f per lane slot, then the xor tree)
      for (int f0 = 0; f0 < F; f0 += U * RPI) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int f = f0 + u * RPI + slot;
          v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (f < F && ((p.fm_mask >> f) & 1ull))
            v[u] = *reinterpret_cast<const float4*>(xrow + (int64_t)f * dim + chunk * 4);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) { s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w; }
      }
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1) {
        s.x += __shfl_xor_sync(0xffffffffu, s.x, o);
        s.y += __shfl_xor_sync(0xffffffffu, s.y, o);
        s.z += __shfl_xor_sync(0xffffffffu, s.z, o);
        s.w += __shfl_xor_sync(0xffffffffu, s.w, o);
      }
    }
    for (int f0 = 0; f0 < F; f0 += U * RPI) {
      float4 g[U], xv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int f = f0 + u * RPI + slot;
        g[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        xv[u] = g[u];
        if (f < F) {
          const int64_t off = (int64_t)f * dim + chunk * 4;
          if (dxrow) g[u] = ldg_stream_f4_pol(dxrow + off, pol_stream);
          // x for the Jacobian: an L1 hit after the pre-pass, else (stored S) the one read of the row
          if (dfm && ((p.fm_mask >> f) & 1ull)) xv[u] = *reinterpret_cast<const float4*>(xrow + off);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int f = f0 + u * RPI + slot;
        const int fs = f < F ? f : 0;
        const int64_t ida = __shfl_sync(0xffffffffu, id0, fs & 31);
        const int64_t idb = __shfl_sync(0xffffffffu, id1, fs & 31);
        const int64_t id = fs < 32 ? ida : idb;
        if (f < F && id >= 0) {
          float4 r = g[u];
          if (dfm && ((p.fm_mask >> f) & 1ull)) {
            r.x += gfm * (s.x - xv[u].x);
            r.y += gfm * (s.y - xv[u].y);
            r.z += gfm * (s.z - xv[u].z);
            r.w += gfm * (s.w - xv[u].w);
          }
          r.x *= scale; r.y *= scale; r.z *= scale; r.w *= scale;
          if (SHARD) red_peer_f4(shard_row(p.peer_tab, p, f, id, dim) + chunk * 4, r);
          else if (p.store_grads) stg_stream_f4(p.table[f] + id * dim + chunk * 4, r);
          else red_add_f4_pol(p.table[f] + id * dim + chunk * 4, r, pol_stream);
        }
      }
    }
    if (dlinear && p.has_lin) {
      const float gl = dlinear[b] * lin_scale;
      const bool ok0 = lane < F && id0 >= 0;
      const bool ok1 = lane + 32 < F && id1 >= 0;
      if (SHARD) {
        if (ok0) red_peer_f1(shard_row(p.peer_lin, p, lane, id0, 1), gl);
        if (ok1) red_peer_f1(shard_row(p.peer_lin, p, lane + 32, id1, 1), gl);
      } else if (p.store_grads) {
        if (ok0) p.lin[lane][id0] = gl;
        if (ok1) p.lin[lane + 32][id1] = gl;
      } else {
        if (ok0) red_add_f1_pol(p.lin[lane] + id0, gl, pol_keep);
        if (ok1) red_add_f1_pol(p.lin[lane + 32] + id1, gl, pol_keep);
      }
    }
    id0 = nid0;
    id1 = nid1;
  }
}

// ============================================================================================
// Hash and table initialisation
// ============================================================================================
__global__ void hash64_kernel(const void* ids, int dtype, int64_t n, int64_t nb, int mask_zero,
                              int64_t* out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = farm::hash_bucket(load_idx(ids, i, dtype), nb, mask_zero != 0);
}

// Philox4x32-10 (Salmon et al. 2011), counter = element index / 4, key = seed.
__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}
__global__ void init_normal_kernel(float* dst, int64_t n, float mean, float std, uint64_t seed) {
  const int64_t nquads = (n + 3) / 4;
  for (int64_t qd = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; qd < nquads;
       qd += (int64_t)gridDim.x * blockDim.x) {
    uint32_t c[4] = {(uint32_t)qd, (uint32_t)(qd >> 32), 0u, 0u};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    float z[4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // Box-Muller on (0,1] uniforms
      const float u1 = ((float)c[2 * h] + 1.0f) * 2.3283064365386963e-10f;
      const float u2 = ((float)c[2 * h + 1] + 1.0f) * 2.3283064365386963e-10f;
      const float r = sqrtf(-2.f * logf(u1));
      float sn, cs;
      sincosf(6.283185307179586f * u2, &sn, &cs);
      z[2 * h] = r * cs;
      z[2 * h + 1] = r * sn;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (qd * 4 + i < n) dst[qd * 4 + i] = mean + std * z[i];
  }
}

// ============================================================================================
// host side
// ============================================================================================
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static b2ctr_status_t validate_feats(const b2ctr_feature_t* feats, int32_t nfeat, int64_t batch,
                                     bool* vec4, int* maxlanes) {
  B2_REQUIRE(feats != nullptr && nfeat > 0, "embed: feats is NULL or nfeat <= 0");
  B2_REQUIRE(batch >= 0, "embed: negative batch");
  *vec4 = true;
  *maxlanes = 1;
  for (int i = 0; i < nfeat; ++i) {
    const b2ctr_feature_t& f = feats[i];
    B2_REQUIRE(f.table && f.idx && f.out, "embed: feature %d has a NULL table/idx/out pointer", i);
    B2_REQUIRE(f.dim > 0 && f.maxlen > 0 && f.vocab > 0, "embed: feature %d bad dim/maxlen/vocab", i);
    B2_REQUIRE(f.idx_dtype == B2CTR_IDX_I32 || f.idx_dtype == B2CTR_IDX_I64,
               "embed: feature %d bad idx_dtype", i);
    B2_REQUIRE(f.pool >= B2CTR_POOL_NONE && f.pool <= B2CTR_POOL_MAX, "embed: feature %d bad pool", i);
    B2_REQUIRE(f.mask_mode >= 0 && f.mask_mode <= 2, "embed: feature %d bad mask_mode", i);
    B2_REQUIRE(f.mask_mode != B2CTR_MASK_LENGTH || f.len, "embed: feature %d needs len[]", i);
    B2_REQUIRE(f.weight_mode == B2CTR_WEIGHT_NONE || f.weight, "embed: feature %d needs weight[]", i);
    B2_REQUIRE(f.hash_mode >= 0 && f.hash_mode <= 2, "embed: feature %d bad hash_mode", i);
    B2_REQUIRE(f.hash_mode != B2CTR_HASH_FARM_MASK_ZERO || f.vocab >= 2,
               "embed: feature %d: mask_zero hashing needs >= 2 buckets", i);
    if (f.dim % 4 || f.out_col % 4 || f.out_ld % 4 || !aligned16(f.table) || !aligned16(f.out))
      *vec4 = false;
  }
  for (int i = 0; i < nfeat; ++i) {
    int lanes = *vec4 ? feats[i].dim / 4 : feats[i].dim;
    if (lanes > *maxlanes) *maxlanes = lanes;
  }
  return B2CTR_OK;
}

#define B2_DISPATCH_G(KERNEL, lanes, vec4, ...)                                          \
  do {                                                                                   \
    int g__ = 1;                                                                         \
    while (g__ < (lanes) && g__ < 32) g__ <<= 1;                                         \
    const int grid__ = grid_for(batch * fb.nfeat, 256 / g__, 8);                         \
    if (vec4) {                                                                          \
      switch (g__) {                                                                     \
        case 1: KERNEL<1, 4><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 2: KERNEL<2, 4><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 4: KERNEL<4, 4><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 8: KERNEL<8, 4><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 16: KERNEL<16, 4><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;              \
        default: KERNEL<32, 4><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;              \
      }                                                                                  \
    } else {                                                                             \
      switch (g__) {                                                                     \
        case 1: KERNEL<1, 1><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 2: KERNEL<2, 1><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 4: KERNEL<4, 1><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 8: KERNEL<8, 1><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;                \
        case 16: KERNEL<16, 1><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;              \
        default: KERNEL<32, 1><<<grid__, 256, 0, st>>>(__VA_ARGS__); break;              \
      }                                                                                  \
    }                                                                                    \
  } while (0)

static b2ctr_status_t fill_uni(const b2ctr_uniform_gather_t* g, UniParams* p) {
  B2_REQUIRE(g && g->feats && g->x, "uniform gather: NULL descriptor / feats / x");
  B2_REQUIRE(g->nfeat > 0 && g->nfeat <= kUniMaxFeat, "uniform gather: nfeat must be in [1,%d]",
             kUniMaxFeat);
  const int dim = g->feats[0].dim;
  B2_REQUIRE(dim == 4 || dim == 8 || dim == 16 || dim == 32 || dim == 64 || dim == 128,
             "uniform gather: dim must be one of 4,8,16,32,64,128 (got %d)", dim);
  B2_REQUIRE(g->ldx % 4 == 0 && g->ldx >= (int64_t)g->nfeat * dim + g->ndense,
             "uniform gather: ldx must be a multiple of 4 and >= F*dim+ndense");
  B2_REQUIRE(aligned16(g->x), "uniform gather: x must be 16-byte aligned");
  B2_REQUIRE(g->ndense == 0 || g->dense, "uniform gather: dense is NULL but ndense > 0");
  for (int f = 0; f < g->nfeat; ++f) {
    const b2ctr_feature_t& ft = g->feats[f];
    B2_REQUIRE(ft.dim == dim && ft.maxlen == 1 && ft.hash_mode == B2CTR_HASH_NONE,
               "uniform gather: feature %d is not a plain single-valued feature of dim %d", f, dim);
    B2_REQUIRE(ft.idx_dtype == g->feats[0].idx_dtype, "uniform gather: mixed idx dtypes");
    B2_REQUIRE(ft.idx && (g->world > 1 || (ft.table && aligned16(ft.table))),
               "uniform gather: feature %d bad pointers", f);
    p->table[f] = ft.table;
    p->vocab[f] = ft.vocab;
    p->idx[f] = ft.idx;
    p->idx_stride[f] = ft.idx_stride;
    p->lin[f] = (g->lin_tables && g->world <= 1) ? g->lin_tables[f] : nullptr;
    B2_REQUIRE(g->world > 1 || !g->lin_tables || p->lin[f], "uniform gather: lin_tables[%d] is NULL", f);
  }
  p->oob = oob_counter();
  p->world = g->world > 1 ? g->world : 1;
  p->wshift = 0;
  p->peer_tab = g->peer_tables;
  p->peer_lin = g->peer_lin_tables;
  if (g->world > 1) {
    B2_REQUIRE((g->world & (g->world - 1)) == 0, "uniform gather: world must be a power of two (got %d)", g->world);
    B2_REQUIRE(g->peer_tables, "uniform gather: world > 1 needs peer_tables");
    B2_REQUIRE(!(g->flags & B2CTR_UNIFORM_STORE_GRADS), "uniform gather: STORE_GRADS is not defined for sharded tables");
    while ((1 << p->wshift) < g->world) ++p->wshift;
  }
  p->dense = g->dense;
  p->x = g->x;
  p->linear = g->linear;
  p->fm = g->fm;
  p->ldx = g->ldx;
  p->dense_ld = g->dense_ld;
  p->x_cols = g->x_cols > 0 ? g->x_cols : g->ldx;
  B2_REQUIRE(p->x_cols <= g->ldx && p->x_cols >= (int64_t)g->nfeat * dim + g->ndense, "uniform gather: x_cols out of range");
  p->fm_mask = g->fm_mask[0];
  p->nfeat = g->nfeat;
  p->ndense = g->ndense;
  p->dim = dim;
  p->idx_dtype = g->feats[0].idx_dtype;
  p->has_lin = g->world > 1 ? (g->peer_lin_tables != nullptr) : (g->lin_tables != nullptr);
  p->store_grads = (g->flags & B2CTR_UNIFORM_STORE_GRADS) ? 1 : 0;
  p->fm_sum = nullptr;
  p->xp_hi = p->xp_lo = nullptr;
  p->xp_pitch = p->xp_rows_pad = 0;
  return B2CTR_OK;
}

template <bool SHARD, bool EXTRA>
static void launch_gather(const UniParams& p, int64_t batch, int grid, cudaStream_t st) {
  switch (p.dim / 4) {
    case 1: gather_uniform_fwd_kernel<1, SHARD, EXTRA><<<grid, 256, 0, st>>>(p, batch); break;
    case 2: gather_uniform_fwd_kernel<2, SHARD, EXTRA><<<grid, 256, 0, st>>>(p, batch); break;
    case 4: gather_uniform_fwd_kernel<4, SHARD, EXTRA><<<grid, 256, 0, st>>>(p, batch); break;
    case 8: gather_uniform_fwd_kernel<8, SHARD, EXTRA><<<grid, 256, 0, st>>>(p, batch); break;
    case 16: gather_uniform_fwd_kernel<16, SHARD, EXTRA><<<grid, 256, 0, st>>>(p, batch); break;
    default: gather_uniform_fwd_kernel<32, SHARD, EXTRA><<<grid, 256, 0, st>>>(p, batch); break;
  }
}


// ============================================================================================
// Field-aware pairwise products (ONN / NFFM, deepctr/models/onn.py:79-97): field a has one table per partner
// field b; pair p = (i, j), i < j, in itertools.combinations order, is  e_{i,(j)} * e_{j,(i)}.  One warp per
// sample: the lanes resolve (and hash) the F ids once into shared memory, then walk the P pairs, each lane reading
// its pair's two rows straight from their tables.  The [B, F(F-1), E] lookups are never written.
// A pre-pooled field (a VarLenSparseFeat bag) is read from `pooled`, which the generic gather filled.
// ============================================================================================
constexpr int kFfmMaxF = 64;
constexpr int kFfmWarps = 8;

struct FfmParams {
  b2ctr_ffm_field_t f[kFfmMaxF];
  float* const* tables;          // device [F*F]: field a's table for partner b at a*F + b
  float* out;                    // fwd: products; bwd: NULL
  const float* g;                // bwd: gradient of the products, fwd: NULL
  int64_t ld;                    // pitch of out / g
  unsigned long long* oob;
  int32_t F, E, reduce_sum, col;
};

template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::T vmul(typename VecT<VEC>::T a, typename VecT<VEC>::T b);
template <>
__device__ __forceinline__ float4 vmul<4>(float4 a, float4 b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
template <>
__device__ __forceinline__ float vmul<1>(float a, float b) { return a * b; }
__device__ __forceinline__ float vsum(float4 a) { return (a.x + a.y) + (a.z + a.w); }
__device__ __forceinline__ float vsum(float a) { return a; }
__device__ __forceinline__ float4 vbcast(float s, float4*) { return make_float4(s, s, s, s); }
__device__ __forceinline__ float vbcast(float s, float*) { return s; }

// field a's operand for partner c in sample b: a table row, a pooled row, or NULL (out-of-range id: a zero row)
__device__ __forceinline__ const float* ffm_row(const FfmParams& p, const int64_t* ids, int a, int c, int64_t b) {
  const b2ctr_ffm_field_t& fa = p.f[a];
  const int s = c - (c > a);
  if (fa.idx == nullptr) return fa.pooled + b * fa.pooled_ld + (int64_t)s * p.E;
  const int64_t id = ids[a];
  if (id < 0) return nullptr;
  return p.tables[a * p.F + c] + id * p.E;
}

// the row index of a single-valued field in sample b (hashed if the field hashes), -1 when out of range
__device__ __forceinline__ int64_t ffm_resolve_id(const b2ctr_ffm_field_t& f, int64_t b, unsigned long long* oob) {
  int64_t id = load_idx(f.idx, b * f.idx_stride, f.idx_dtype);
  if (f.hash_mode != B2CTR_HASH_NONE) id = farm::hash_bucket(id, f.vocab, f.hash_mode == B2CTR_HASH_FARM_MASK_ZERO);
  if (id_in_range(id, f.vocab)) return id;
  note_oob(oob);
  return -1;
}

// (min 4 blocks per SM: without that bound the 64-bit hash modulo makes ptxas spill around its call)
template <int VEC, bool BWD>
__global__ void __launch_bounds__(kFfmWarps * 32, 4) ffm_product_kernel(const __grid_constant__ FfmParams p,
                                                                     int64_t batch) {
  using V = typename VecT<VEC>::T;
  __shared__ uint16_t s_pair[kFfmMaxF * (kFfmMaxF - 1) / 2];
  __shared__ int64_t s_id[kFfmWarps][kFfmMaxF];
  const int F = p.F, E = p.E, P = F * (F - 1) / 2, nv = E / VEC;
  for (int i = 0, q = 0; i < F - 1; q += F - 1 - i, ++i)
    for (int k = threadIdx.x; k < F - 1 - i; k += blockDim.x) s_pair[q + k] = (uint16_t)((i << 8) | (i + 1 + k));
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int64_t* ids = s_id[warp];
  for (int64_t b = (int64_t)blockIdx.x * kFfmWarps + warp; b < batch; b += (int64_t)gridDim.x * kFfmWarps) {
    for (int a = lane; a < F; a += 32)
      if (p.f[a].idx != nullptr) ids[a] = ffm_resolve_id(p.f[a], b, BWD ? nullptr : p.oob);
    __syncwarp();
    for (int q = lane; q < P; q += 32) {
      const int i = s_pair[q] >> 8, j = s_pair[q] & 0xff;
      const float* ri = ffm_row(p, ids, i, j, b);
      const float* rj = ffm_row(p, ids, j, i, b);
      if (!BWD) {
        float* o = p.out + b * p.ld + p.col;
        float acc = 0.f;
        for (int c = 0; c < nv; ++c) {
          const V x = ri ? vload(ri + c * VEC, (V*)nullptr) : vzero<VEC>();
          const V y = rj ? vload(rj + c * VEC, (V*)nullptr) : vzero<VEC>();
          const V z = vmul<VEC>(x, y);
          if (p.reduce_sum) acc += vsum(z);
          else *reinterpret_cast<V*>(o + (int64_t)q * E + c * VEC) = z;
        }
        if (p.reduce_sum) o[q] = acc;
      } else {
        // d e_{i,(j)} = g_p * e_{j,(i)},  d e_{j,(i)} = g_p * e_{i,(j)}: one writer per element, no atomics
        const float* gr = p.g + b * p.ld + p.col;
        const b2ctr_ffm_field_t& fi = p.f[i];
        const b2ctr_ffm_field_t& fj = p.f[j];
        float* di = fi.grad + b * fi.grad_ld + (int64_t)(j - 1) * E;
        float* dj = fj.grad + b * fj.grad_ld + (int64_t)i * E;
        const float gs = p.reduce_sum ? gr[q] : 0.f;
        for (int c = 0; c < nv; ++c) {
          const V x = ri ? vload(ri + c * VEC, (V*)nullptr) : vzero<VEC>();
          const V y = rj ? vload(rj + c * VEC, (V*)nullptr) : vzero<VEC>();
          const V gv = p.reduce_sum ? vbcast(gs, (V*)nullptr)
                                    : *reinterpret_cast<const V*>(gr + (int64_t)q * E + c * VEC);
          *reinterpret_cast<V*>(di + c * VEC) = vmul<VEC>(gv, y);
          *reinterpret_cast<V*>(dj + c * VEC) = vmul<VEC>(gv, x);
        }
      }
    }
    __syncwarp();
  }
}

static b2ctr_status_t ffm_params(const b2ctr_ffm_field_t* fields, int32_t nfield, float* const* tables, int32_t dim,
                                 int32_t reduce_sum, int64_t ld, int32_t col, int64_t batch, bool bwd, FfmParams* p,
                                 bool* vec4) {
  B2_REQUIRE(nfield >= 2 && nfield <= kFfmMaxF, "ffm_product: the field count must be in [2, %d] (got %d)",
             kFfmMaxF, nfield);
  B2_REQUIRE(dim >= 1 && dim <= 64, "ffm_product: dim must be in [1, 64] (got %d)", dim);
  B2_REQUIRE(fields && tables && batch >= 0 && col >= 0, "ffm_product: NULL pointer or negative batch / column");
  B2_REQUIRE(reduce_sum == 0 || reduce_sum == 1, "ffm_product: reduce_sum must be 0 or 1");
  const int64_t P = (int64_t)nfield * (nfield - 1) / 2;
  B2_REQUIRE(ld >= col + P * (reduce_sum ? 1 : dim), "ffm_product: row pitch %lld too small for %lld products",
             (long long)ld, (long long)P);
  bool v4 = dim % 4 == 0 && ld % 4 == 0 && col % 4 == 0 && aligned16(tables);
  for (int a = 0; a < nfield; ++a) {
    const b2ctr_ffm_field_t& f = fields[a];
    B2_REQUIRE((f.idx != nullptr) != (f.pooled != nullptr), "ffm_product: field %d needs exactly one of ids and "
               "a pooled operand", a);
    if (f.idx) {
      B2_REQUIRE(f.idx_dtype == B2CTR_IDX_I32 || f.idx_dtype == B2CTR_IDX_I64, "ffm_product: field %d bad idx dtype", a);
      B2_REQUIRE(f.hash_mode >= B2CTR_HASH_NONE && f.hash_mode <= B2CTR_HASH_FARM_MASK_ZERO && f.vocab >= 1,
                 "ffm_product: field %d bad hash mode or vocabulary", a);
    } else {
      B2_REQUIRE(f.pooled_ld >= (int64_t)(nfield - 1) * dim, "ffm_product: field %d pooled pitch too small", a);
      v4 = v4 && f.pooled_ld % 4 == 0 && aligned16(f.pooled);
    }
    if (bwd) {
      B2_REQUIRE(f.grad && f.grad_ld >= (int64_t)(nfield - 1) * dim, "ffm_product: field %d needs a gradient "
                 "buffer of pitch >= (F-1)*dim", a);
      v4 = v4 && f.grad_ld % 4 == 0 && aligned16(f.grad);
    }
    p->f[a] = f;
  }
  p->tables = tables;
  p->ld = ld;
  p->oob = oob_counter();
  p->F = nfield;
  p->E = dim;
  p->reduce_sum = reduce_sum;
  p->col = col;
  *vec4 = v4;
  return B2CTR_OK;
}

}  // namespace b2ctr

using namespace b2ctr;

extern "C" {

b2ctr_status_t b2ctr_embed_gather_fwd(const b2ctr_feature_t* feats, int32_t nfeat, int64_t batch,
                                      void* stream) {
  bool vec4;
  int lanes;
  b2ctr_status_t s = validate_feats(feats, nfeat, batch, &vec4, &lanes);
  if (s != B2CTR_OK) return s;
  if (batch == 0) return B2CTR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  for (int base = 0; base < nfeat; base += kFeatChunk) {
    FeatBlock fb;
    fb.oob = oob_counter();
    fb.nfeat = nfeat - base < kFeatChunk ? nfeat - base : kFeatChunk;
    for (int i = 0; i < fb.nfeat; ++i) fb.f[i] = feats[base + i];
    B2_DISPATCH_G(embed_gather_generic_kernel, lanes, vec4, fb, batch);
    B2_CHECK_LAUNCH("b2ctr_embed_gather_fwd");
  }
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_embed_scatter_add(const b2ctr_feature_t* feats, int32_t nfeat, int64_t batch,
                                       float scale, void* stream) {
  bool vec4;
  int lanes;
  b2ctr_status_t s = validate_feats(feats, nfeat, batch, &vec4, &lanes);
  if (s != B2CTR_OK) return s;
  if (batch == 0) return B2CTR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  for (int base = 0; base < nfeat; base += kFeatChunk) {
    FeatBlock fb;
    fb.oob = nullptr;            // the forward pass already counted them
    fb.nfeat = nfeat - base < kFeatChunk ? nfeat - base : kFeatChunk;
    for (int i = 0; i < fb.nfeat; ++i) fb.f[i] = feats[base + i];
    B2_DISPATCH_G(embed_scatter_generic_kernel, lanes, vec4, fb, batch, scale);
    B2_CHECK_LAUNCH("b2ctr_embed_scatter_add");
  }
  return B2CTR_OK;
}

#define B2_DISPATCH_LPR1(KERNEL, SH, dim, ...)                                 \
  switch ((dim) / 4) {                                                         \
    case 1: KERNEL<1, SH><<<grid, 256, 0, st>>>(__VA_ARGS__); break;           \
    case 2: KERNEL<2, SH><<<grid, 256, 0, st>>>(__VA_ARGS__); break;           \
    case 4: KERNEL<4, SH><<<grid, 256, 0, st>>>(__VA_ARGS__); break;           \
    case 8: KERNEL<8, SH><<<grid, 256, 0, st>>>(__VA_ARGS__); break;           \
    case 16: KERNEL<16, SH><<<grid, 256, 0, st>>>(__VA_ARGS__); break;         \
    default: KERNEL<32, SH><<<grid, 256, 0, st>>>(__VA_ARGS__); break;         \
  }
#define B2_DISPATCH_LPR(KERNEL, dim, ...)                                      \
  if (p.world > 1) { B2_DISPATCH_LPR1(KERNEL, true, dim, __VA_ARGS__) }        \
  else { B2_DISPATCH_LPR1(KERNEL, false, dim, __VA_ARGS__) }

b2ctr_status_t b2ctr_embed_gather_uniform_fwd(const b2ctr_uniform_gather_t* g, int64_t batch,
                                              void* stream) {
  return b2ctr_embed_gather_uniform_fwd_ex(g, nullptr, nullptr, 0, batch, stream);
}

b2ctr_status_t b2ctr_embed_gather_uniform_fwd_ex(const b2ctr_uniform_gather_t* g, float* fm_sum, void* x_planes,
                                                 int64_t x_planes_cols, int64_t batch, void* stream) {
  UniParams p;
  b2ctr_status_t s = fill_uni(g, &p);
  if (s != B2CTR_OK) return s;
  B2_REQUIRE(!fm_sum || (g->fm && aligned16(fm_sum)), "uniform gather: fm_sum needs fm and 16-byte alignment");
  p.fm_sum = fm_sum;
  if (x_planes) {
    B2_REQUIRE(x_planes_cols >= (int64_t)g->nfeat * p.dim + g->ndense && x_planes_cols <= p.x_cols,
               "uniform gather: x_planes_cols must be in [F*dim + ndense, x_cols]");
    B2_REQUIRE(aligned16(x_planes), "uniform gather: x_planes must be 16-byte aligned");
    p.xp_pitch = planes_cols_pad(x_planes_cols);
    p.xp_rows_pad = planes_rows_pad(batch);
    p.xp_hi = (__nv_bfloat16*)x_planes;
    p.xp_lo = p.xp_hi + p.xp_rows_pad * p.xp_pitch;
  }
  if (batch <= 0) return B2CTR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (p.fm_sum || p.xp_hi) {      // one wave of the 3-CTA instantiation
    const int grid = grid_for(batch, 8, 3);
    if (p.world > 1) launch_gather<true, true>(p, batch, grid, st);
    else launch_gather<false, true>(p, batch, grid, st);
  } else {
    const int grid = grid_for(batch, 8, 8);
    if (p.world > 1) launch_gather<true, false>(p, batch, grid, st);
    else launch_gather<false, false>(p, batch, grid, st);
  }
  B2_CHECK_LAUNCH("b2ctr_embed_gather_uniform_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_embed_scatter_uniform_bwd(const b2ctr_uniform_gather_t* g, const float* dx,
                                               const float* dfm, const float* dlinear, float scale,
                                               float lin_scale, int64_t batch, void* stream) {
  return b2ctr_embed_scatter_uniform_bwd_ex(g, dx, dfm, nullptr, dlinear, scale, lin_scale, batch, stream);
}

b2ctr_status_t b2ctr_embed_scatter_uniform_bwd_ex(const b2ctr_uniform_gather_t* g, const float* dx,
                                                  const float* dfm, const float* fm_sum, const float* dlinear,
                                                  float scale, float lin_scale, int64_t batch, void* stream) {
  UniParams p;
  b2ctr_status_t s = fill_uni(g, &p);
  if (s != B2CTR_OK) return s;
  B2_REQUIRE(!dx || aligned16(dx), "uniform scatter: dx must be 16-byte aligned");
  B2_REQUIRE(!fm_sum || aligned16(fm_sum), "uniform scatter: fm_sum must be 16-byte aligned");
  p.fm_sum = const_cast<float*>(fm_sum);
  if (batch <= 0) return B2CTR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(batch, 8, 8);
  B2_DISPATCH_LPR(scatter_uniform_bwd_kernel, p.dim, p, dx, dfm, dlinear, scale, lin_scale, batch);
  B2_CHECK_LAUNCH("b2ctr_embed_scatter_uniform_bwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_hash64(const void* ids, int32_t idx_dtype, int64_t n, int64_t num_buckets,
                            int32_t mask_zero, int64_t* out, void* stream) {
  B2_REQUIRE(ids && out, "hash64: NULL pointer");
  B2_REQUIRE(idx_dtype == B2CTR_IDX_I32 || idx_dtype == B2CTR_IDX_I64, "hash64: bad idx_dtype");
  B2_REQUIRE(num_buckets >= (mask_zero ? 2 : 1), "hash64: num_buckets too small");
  if (n <= 0) return B2CTR_OK;
  hash64_kernel<<<grid_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(ids, idx_dtype, n, num_buckets,
                                                                      mask_zero, out);
  B2_CHECK_LAUNCH("b2ctr_hash64");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_init_normal(float* dst, int64_t n, float mean, float std, uint64_t seed,
                                 void* stream) {
  B2_REQUIRE(dst, "init_normal: NULL dst");
  if (n <= 0) return B2CTR_OK;
  init_normal_kernel<<<grid_for((n + 3) / 4, 256, 8), 256, 0, (cudaStream_t)stream>>>(dst, n, mean,
                                                                                     std, seed);
  B2_CHECK_LAUNCH("b2ctr_init_normal");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_ffm_product_fwd(const b2ctr_ffm_field_t* fields, int32_t nfield, float* const* tables,
                                     int32_t dim, int32_t reduce_sum, float* out, int64_t out_ld, int32_t out_col,
                                     int64_t batch, void* stream) {
  FfmParams p;
  bool v4;
  b2ctr_status_t s = ffm_params(fields, nfield, tables, dim, reduce_sum, out_ld, out_col, batch, false, &p, &v4);
  if (s != B2CTR_OK) return s;
  B2_REQUIRE(out, "ffm_product_fwd: NULL out");
  p.out = out;
  p.g = nullptr;
  v4 = v4 && aligned16(out);
  if (batch == 0) return B2CTR_OK;
  const int grid = grid_for(batch, kFfmWarps, 8);
  if (v4) ffm_product_kernel<4, false><<<grid, kFfmWarps * 32, 0, (cudaStream_t)stream>>>(p, batch);
  else ffm_product_kernel<1, false><<<grid, kFfmWarps * 32, 0, (cudaStream_t)stream>>>(p, batch);
  B2_CHECK_LAUNCH("b2ctr_ffm_product_fwd");
  return B2CTR_OK;
}

b2ctr_status_t b2ctr_ffm_product_bwd(const b2ctr_ffm_field_t* fields, int32_t nfield, float* const* tables,
                                     int32_t dim, int32_t reduce_sum, const float* g, int64_t g_ld, int32_t g_col,
                                     int64_t batch, void* stream) {
  FfmParams p;
  bool v4;
  b2ctr_status_t s = ffm_params(fields, nfield, tables, dim, reduce_sum, g_ld, g_col, batch, true, &p, &v4);
  if (s != B2CTR_OK) return s;
  B2_REQUIRE(g, "ffm_product_bwd: NULL gradient");
  p.out = nullptr;
  p.g = g;
  v4 = v4 && aligned16(g);
  if (batch == 0) return B2CTR_OK;
  const int grid = grid_for(batch, kFfmWarps, 8);
  if (v4) ffm_product_kernel<4, true><<<grid, kFfmWarps * 32, 0, (cudaStream_t)stream>>>(p, batch);
  else ffm_product_kernel<1, true><<<grid, kFfmWarps * 32, 0, (cudaStream_t)stream>>>(p, batch);
  B2_CHECK_LAUNCH("b2ctr_ffm_product_bwd");
  return B2CTR_OK;
}

}  // extern "C"
