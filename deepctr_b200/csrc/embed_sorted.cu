// embed_sorted.cu — DETERMINISTIC fused embedding update of the Criteo-shaped fast path (sm_90a).
//
// north_star asks for bit-exact segment sums; SURVEY.md section 7: "backward duplicate-index accumulation needs a
// sort + ordered segmented reduce, not float atomics".  b2ctr_embed_scatter_uniform_bwd (embed.cu) combines the
// gradient rows of duplicate ids with red.global.add: exact up to fp32 re-association, but in an order that
// changes from run to run.  This path instead
//   1. keys every (sample, feature) lookup with (feature << vbits | id)           [make_keys_kernel]
//   2. stably radix-sorts the keys (cub::DeviceRadixSort, CUDA toolkit)          -> runs of equal (feature, id),
//      inside a run in ascending sample order
//   3. gives every run to ONE warp, which sums the run's gradient rows in that order in fp32 (no FMA
//      contraction) and writes the row exactly once                               [apply_runs_kernel]
// -> run-to-run bit-identical, and the natural home of optimizers that need a per-row read-modify-write of
// state: row-wise SGD and Keras' Adagrad (whose sparse apply is lazy, i.e. touches only the rows of the batch:
// acc += g^2; w -= lr * g / (sqrt(acc) + eps)).  Gradient of row (b, f), as in embed.cu:
//   g = dx[b, f*dim : (f+1)*dim] + dfm[b] * (S_b - x[b, f*dim : ...]),   S_b = sum over the FM fields of x[b, f, :].
// HBM-bound integer / byte work: no tensor cores; 128-bit accesses; grids sized from the SM count.
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"

namespace b2ctr {
namespace {

constexpr int kMaxFeat = 64;
struct SortedParams {
  float* table[kMaxFeat];
  float* lin[kMaxFeat];
  float* acc[kMaxFeat];        // Adagrad accumulators (same shape as table) or NULL
  float* lin_acc[kMaxFeat];
  const void* idx[kMaxFeat];
  int64_t idx_stride[kMaxFeat];
  int64_t vocab[kMaxFeat];
  const float* x;              // forward activations [B, ldx]
  const float* dx;             // [B, ldx] or NULL
  const float* dfm;            // [B] or NULL
  const float* dlinear;        // [B] or NULL
  int64_t ldx;
  uint64_t fm_mask;
  int32_t nfeat, dim, idx_dtype, optimizer;
  int32_t shift;               // bits of the largest vocabulary: key = feature << shift | id
  float lr, lin_lr, eps;
};

__global__ void __launch_bounds__(256)
    make_keys_kernel(const __grid_constant__ SortedParams p, int64_t batch, uint64_t* keys, uint32_t* vals) {
  const int64_t total = batch * p.nfeat;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < total; n += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = n / p.nfeat;
    const int f = (int)(n - b * p.nfeat);
    const int64_t id = load_idx(p.idx[f], b * p.idx_stride[f], p.idx_dtype);
    // ids outside the vocabulary get the key of a feature that does not exist: they sort last and are skipped
    keys[n] = ((uint64_t)(id_in_range(id, p.vocab[f]) ? f : p.nfeat) << p.shift) | (id_in_range(id, p.vocab[f]) ? (uint64_t)id : 0ull);
    vals[n] = (uint32_t)n;
  }
}

// S[b, :] = sum over the FM fields of x[b, f, :]  (only when dfm is given)
__global__ void __launch_bounds__(256)
    fm_sum_kernel(const __grid_constant__ SortedParams p, int64_t batch, float* S) {
  const int64_t total = batch * p.dim;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = t / p.dim;
    const int e = (int)(t - b * p.dim);
    float s = 0.f;
    for (int f = 0; f < p.nfeat; ++f)
      if ((p.fm_mask >> f) & 1ull) s = __fadd_rn(s, p.x[b * p.ldx + (int64_t)f * p.dim + e]);
    S[t] = s;
  }
}

// one warp per sorted position; only the head of a run works: lanes = 4-float chunks of the row (dim <= 128)
__global__ void __launch_bounds__(256)
    apply_runs_kernel(const __grid_constant__ SortedParams p, int64_t total, const uint64_t* __restrict__ keys,
                      const uint32_t* __restrict__ vals, const float* __restrict__ S) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int chunks = p.dim >> 2;
  for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < total; i += nw) {
    const uint64_t key = keys[i];
    const int f = (int)(key >> p.shift);
    if (f >= p.nfeat || (i > 0 && keys[i - 1] == key)) continue;             // invalid id / not the head of a run
    const int64_t id = (int64_t)(key & ((1ull << p.shift) - 1));
    const bool fm_on = p.dfm != nullptr && ((p.fm_mask >> f) & 1ull);
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    float gl = 0.f;
    for (int64_t j = i; j < total && keys[j] == key; ++j) {                  // ascending sample order (stable sort)
      const int64_t b = (int64_t)(vals[j] / (uint32_t)p.nfeat);
      if (lane < chunks) {
        const int64_t off = b * p.ldx + (int64_t)f * p.dim + lane * 4;
        float4 r = p.dx ? *reinterpret_cast<const float4*>(p.dx + off) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (fm_on) {
          const float gf = p.dfm[b];
          const float4 xv = *reinterpret_cast<const float4*>(p.x + off);
          const float4 sv = *reinterpret_cast<const float4*>(S + b * p.dim + lane * 4);
          r.x = __fadd_rn(r.x, __fmul_rn(gf, __fsub_rn(sv.x, xv.x)));
          r.y = __fadd_rn(r.y, __fmul_rn(gf, __fsub_rn(sv.y, xv.y)));
          r.z = __fadd_rn(r.z, __fmul_rn(gf, __fsub_rn(sv.z, xv.z)));
          r.w = __fadd_rn(r.w, __fmul_rn(gf, __fsub_rn(sv.w, xv.w)));
        }
        g.x = __fadd_rn(g.x, r.x); g.y = __fadd_rn(g.y, r.y); g.z = __fadd_rn(g.z, r.z); g.w = __fadd_rn(g.w, r.w);
      }
      if (p.dlinear) gl = __fadd_rn(gl, p.dlinear[b]);
    }
    if (lane < chunks) {
      float* row = p.table[f] + id * p.dim + lane * 4;
      float4 w = *reinterpret_cast<float4*>(row);
      if (p.optimizer == 1) {          // Keras Adagrad: acc += g^2 ; w -= lr * g / (sqrt(acc) + eps)
        float* arow = p.acc[f] + id * p.dim + lane * 4;
        float4 a = *reinterpret_cast<float4*>(arow);
        a.x = __fadd_rn(a.x, __fmul_rn(g.x, g.x)); a.y = __fadd_rn(a.y, __fmul_rn(g.y, g.y));
        a.z = __fadd_rn(a.z, __fmul_rn(g.z, g.z)); a.w = __fadd_rn(a.w, __fmul_rn(g.w, g.w));
        *reinterpret_cast<float4*>(arow) = a;
        w.x -= p.lr * g.x / (sqrtf(a.x) + p.eps); w.y -= p.lr * g.y / (sqrtf(a.y) + p.eps);
        w.z -= p.lr * g.z / (sqrtf(a.z) + p.eps); w.w -= p.lr * g.w / (sqrtf(a.w) + p.eps);
      } else {
        w.x = __fsub_rn(w.x, __fmul_rn(p.lr, g.x)); w.y = __fsub_rn(w.y, __fmul_rn(p.lr, g.y));
        w.z = __fsub_rn(w.z, __fmul_rn(p.lr, g.z)); w.w = __fsub_rn(w.w, __fmul_rn(p.lr, g.w));
      }
      *reinterpret_cast<float4*>(row) = w;
    }
    if (lane == 0 && p.dlinear && p.lin[f]) {
      float* lw = p.lin[f] + id;
      if (p.optimizer == 1) {
        float* la = p.lin_acc[f] + id;
        const float a = __fadd_rn(*la, __fmul_rn(gl, gl));
        *la = a;
        *lw -= p.lin_lr * gl / (sqrtf(a) + p.eps);
      } else {
        *lw = __fsub_rn(*lw, __fmul_rn(p.lin_lr, gl));
      }
    }
  }
}

inline size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

size_t cub_temp_bytes(int64_t n, int end_bit) {
  size_t tmp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)n, 0, end_bit);
  return tmp;
}

}  // namespace
}  // namespace b2ctr

using namespace b2ctr;

extern "C" {

size_t b2ctr_embed_update_sorted_workspace_bytes(int32_t nfeat, int32_t dim, int64_t batch) {
  if (nfeat <= 0 || batch <= 0) return 0;
  const int64_t n = batch * nfeat;
  return 2 * align_up((size_t)n * 8) + 2 * align_up((size_t)n * 4) + align_up((size_t)batch * dim * 4) +
         align_up(cub_temp_bytes(n, 64)) + 256;      // (the sort uses fewer bits: 64 is an upper bound)
}

b2ctr_status_t b2ctr_embed_update_sorted(const b2ctr_uniform_gather_t* g, const float* dx, const float* dfm,
                                         const float* dlinear, int32_t optimizer, float lr, float lin_lr, float eps,
                                         float* const* acc_tables, float* const* lin_acc_tables, int64_t batch,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(g && g->feats && g->x, "embed_update_sorted: NULL descriptor / feats / x");
  B2_REQUIRE(g->nfeat > 0 && g->nfeat <= kMaxFeat, "embed_update_sorted: nfeat must be in [1,%d]", kMaxFeat);
  B2_REQUIRE(g->world <= 1, "embed_update_sorted: row-sharded tables are not supported (use the atomic path)");
  B2_REQUIRE(optimizer == 0 || optimizer == 1, "embed_update_sorted: optimizer must be 0 (sgd) or 1 (adagrad)");
  B2_REQUIRE(optimizer == 0 || acc_tables, "embed_update_sorted: adagrad needs accumulator tables");
  const int dim = g->feats[0].dim;
  B2_REQUIRE(dim % 4 == 0 && dim >= 4 && dim <= 128, "embed_update_sorted: dim must be a multiple of 4 in [4,128]");
  B2_REQUIRE(g->ldx % 4 == 0 && (!dx || ((uintptr_t)dx & 15) == 0) && ((uintptr_t)g->x & 15) == 0,
             "embed_update_sorted: x / dx must be 16-byte aligned with ldx % 4 == 0");
  B2_REQUIRE(batch * g->nfeat < (1ll << 32), "embed_update_sorted: batch * nfeat must fit 32 bits");
  if (batch <= 0) return B2CTR_OK;
  const size_t need = b2ctr_embed_update_sorted_workspace_bytes(g->nfeat, dim, batch);
  if (!workspace || workspace_bytes < need) {
    set_error("embed_update_sorted: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  SortedParams p;
  int64_t max_vocab = 1;
  for (int f = 0; f < g->nfeat; ++f) {
    const b2ctr_feature_t& ft = g->feats[f];
    B2_REQUIRE(ft.table && ft.idx && ft.dim == dim && ft.maxlen == 1 && ft.hash_mode == B2CTR_HASH_NONE &&
                   ft.idx_dtype == g->feats[0].idx_dtype && ((uintptr_t)ft.table & 15) == 0,
               "embed_update_sorted: feature %d is not a plain single-valued feature of dim %d", f, dim);
    B2_REQUIRE(ft.vocab < (1ll << 40), "embed_update_sorted: vocabulary of feature %d does not fit 40 bits", f);
    if (ft.vocab > max_vocab) max_vocab = ft.vocab;
    p.table[f] = ft.table; p.idx[f] = ft.idx; p.idx_stride[f] = ft.idx_stride; p.vocab[f] = ft.vocab;
    p.lin[f] = g->lin_tables ? g->lin_tables[f] : nullptr;
    p.acc[f] = acc_tables ? acc_tables[f] : nullptr;
    p.lin_acc[f] = lin_acc_tables ? lin_acc_tables[f] : nullptr;
    B2_REQUIRE(optimizer == 0 || (p.acc[f] && (!p.lin[f] || !dlinear || p.lin_acc[f])),
               "embed_update_sorted: adagrad accumulator of feature %d missing", f);
  }
  p.x = g->x; p.dx = dx; p.dfm = dfm; p.dlinear = g->lin_tables ? dlinear : nullptr; p.ldx = g->ldx;
  p.fm_mask = g->fm_mask[0]; p.nfeat = g->nfeat; p.dim = dim; p.idx_dtype = g->feats[0].idx_dtype;
  p.optimizer = optimizer; p.lr = lr; p.lin_lr = lin_lr; p.eps = eps;
  p.shift = 1;
  while ((1ll << p.shift) < max_vocab) ++p.shift;
  int fbits = 1;
  while ((1 << fbits) <= g->nfeat) ++fbits;          // values 0..nfeat (nfeat = the invalid bucket)
  const int end_bit = p.shift + fbits;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = batch * g->nfeat;
  unsigned char* w = (unsigned char*)workspace;
  uint64_t* k_in = (uint64_t*)w; w += align_up((size_t)n * 8);
  uint64_t* k_out = (uint64_t*)w; w += align_up((size_t)n * 8);
  uint32_t* v_in = (uint32_t*)w; w += align_up((size_t)n * 4);
  uint32_t* v_out = (uint32_t*)w; w += align_up((size_t)n * 4);
  float* S = (float*)w; w += align_up((size_t)batch * dim * 4);
  size_t tmp_bytes = cub_temp_bytes(n, end_bit);
  make_keys_kernel<<<grid_for(n, 256, 8), 256, 0, st>>>(p, batch, k_in, v_in);
  B2_CHECK_LAUNCH("b2ctr_embed_update_sorted(keys)");
  if (dfm) {
    fm_sum_kernel<<<grid_for(batch * dim, 256, 8), 256, 0, st>>>(p, batch, S);
    B2_CHECK_LAUNCH("b2ctr_embed_update_sorted(fm sums)");
  }
  cudaError_t e = cub::DeviceRadixSort::SortPairs(w, tmp_bytes, k_in, k_out, v_in, v_out, (int)n, 0, end_bit, st);
  if (e != cudaSuccess) {
    set_error("embed_update_sorted: cub::DeviceRadixSort failed: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  apply_runs_kernel<<<grid_for(n, 8, 8), 256, 0, st>>>(p, n, k_out, v_out, S);
  B2_CHECK_LAUNCH("b2ctr_embed_update_sorted(apply)");
  return B2CTR_OK;
}

}  // extern "C"
