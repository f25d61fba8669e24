/*
 * b2ctr.h — C-ABI of libb2ctr.so: the H100 (sm_90a) CTR forward/backward hot path.
 *
 * The reference (shenweichen/DeepCTR, pure Python over TensorFlow) has no FFI of its own
 * (SURVEY.md §8b).  Each entry point below is what a maintainer would bind in place of the
 * TensorFlow ops a `deepctr.layers` operator dispatches to; the reference interface it
 * replaces is cited as deepctr/<file>:<line> next to every declaration.
 *
 * Conventions
 *   - every function returns b2ctr_status_t (0 = OK, <0 = error); b2ctr_last_error() returns a
 *     thread-local message for the last non-zero status;
 *   - all data pointers are DEVICE pointers owned by the caller (they are never retained or
 *     freed); descriptor structs are HOST structs passed by pointer and copied by value into
 *     the launch (no hidden allocations, no hidden synchronisation);
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream;
 *   - tensors are dense row-major fp32 unless a leading dimension (`ld*`, in elements) is given;
 *   - no torch / python types anywhere in this header.
 */
#ifndef B2CTR_H_
#define B2CTR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define B2CTR_API
#else
#define B2CTR_API __attribute__((visibility("default")))
#endif

typedef int32_t b2ctr_status_t;
enum {
  B2CTR_OK = 0,
  B2CTR_ERR_INVALID_ARG = -1, /* bad shape / null pointer / unsupported combination -> ValueError */
  B2CTR_ERR_CUDA = -2,        /* launch or runtime failure -> RuntimeError */
  B2CTR_ERR_UNSUPPORTED = -3, /* valid request the library cannot serve (e.g. alignment) */
  B2CTR_ERR_WORKSPACE = -4    /* workspace missing or too small */
};

/* version / diagnostics -------------------------------------------------------------------- */
B2CTR_API int32_t b2ctr_abi_version(void);
B2CTR_API const char* b2ctr_last_error(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches evidence) */
B2CTR_API int64_t b2ctr_launch_count(void);
B2CTR_API void b2ctr_reset_launch_count(void);

/* Host-side input staging (no GPU work): copy n blocks src[i][0 .. nbytes[i]) to dst + dst_off[i] with a
 * persistent pool of `threads` helper threads (0 = pick from the core count, 1 = inline memcpy).  Replaces the
 * per-feature numpy -> tensor conversion of Keras' data adapter behind model.fit(model_input, y)
 * (reference examples/run_classification_criteo.py:48); the caller uploads dst with one cudaMemcpyAsync. */
/* One process per GPU: let kernels of the current device dereference memory of `peer_device` that was
 * mapped through CUDA IPC (cudaDeviceEnablePeerAccess; already-enabled is not an error). */
B2CTR_API b2ctr_status_t b2ctr_enable_peer_access(int32_t peer_device);

B2CTR_API b2ctr_status_t b2ctr_host_pack(const void* const* src, const int64_t* nbytes, const int64_t* dst_off,
                                         int32_t n, void* dst, int32_t threads);

/* ------------------------------------------------------------------------------------------ */
/* 1. Embedding gather / scatter-update                                                        */
/*    replaces: tf.keras.layers.Embedding call in deepctr/inputs.py:101-130 (embedding_lookup,  */
/*    varlen_embedding_lookup), the pooling of deepctr/inputs.py:133-158 +                      */
/*    deepctr/layers/sequence.py:41-197, the Hash op of deepctr/layers/utils.py:89-112, and     */
/*    the orchestration of deepctr/feature_column.py:213-233 (input_from_feature_columns).      */
/* ------------------------------------------------------------------------------------------ */

enum { B2CTR_IDX_I32 = 0, B2CTR_IDX_I64 = 1 };
enum { B2CTR_POOL_NONE = 0, /* emit the [T,dim] sequence, no pooling (DIN keys)      */
       B2CTR_POOL_SUM = 1, B2CTR_POOL_MEAN = 2, B2CTR_POOL_MAX = 3 };
enum { B2CTR_MASK_NONE = 0,   /* every position valid                                  */
       B2CTR_MASK_ZERO_ID = 1,/* Keras mask_zero: position valid iff id != 0, tested on the id AFTER hashing
                                 (the raw id only under B2CTR_HASH_FARM_MASK_ZERO, which keeps 0 as 0) */
       B2CTR_MASK_LENGTH = 2  /* tf.sequence_mask: position t valid iff t < len[b]     */ };
enum { B2CTR_HASH_NONE = 0,
       B2CTR_HASH_FARM = 1,          /* Fingerprint64(decimal(id)) % num_buckets                 */
       B2CTR_HASH_FARM_MASK_ZERO = 2 /* (Fingerprint64 % (num_buckets-1) + 1) * (id != 0)       */ };
enum { B2CTR_WEIGHT_NONE = 0, B2CTR_WEIGHT_RAW = 1, /* where(mask, w, 0)                        */
       B2CTR_WEIGHT_SOFTMAX = 2                     /* softmax_t(where(mask, w, -2^32+1))        */ };

/* One feature column bound to one table for one launch.  sizeof == 112. */
typedef struct b2ctr_feature {
  float* table;          /* [vocab, dim] fp32 rows (read in fwd, updated in bwd)                 */
  const void* idx;       /* ids: element (b, t) at idx[b*idx_stride + t]                          */
  const int32_t* len;    /* [B] valid lengths (mask_mode LENGTH), else NULL                       */
  const float* weight;   /* [B, maxlen] per-position weights (weight_mode != NONE), else NULL    */
  float* out;            /* fwd: destination; bwd: incoming gradient of the same layout          */
  int64_t vocab;         /* rows in table; also num_buckets for hashing                          */
  int64_t idx_stride;    /* elements between consecutive samples in idx                          */
  int64_t out_ld;        /* elements between consecutive samples in out                          */
  int32_t out_col;       /* first column of this feature inside out rows                         */
  int32_t dim;           /* embedding_dim                                                        */
  int32_t maxlen;        /* 1 for SparseFeat, T for VarLenSparseFeat                             */
  int32_t idx_dtype;     /* B2CTR_IDX_*                                                          */
  int32_t pool;          /* B2CTR_POOL_*                                                         */
  int32_t mask_mode;     /* B2CTR_MASK_*                                                         */
  int32_t hash_mode;     /* B2CTR_HASH_*                                                         */
  int32_t weight_mode;   /* B2CTR_WEIGHT_*                                                       */
  const float* src_table;/* scatter only: table holding the FORWARD rows when `table` is a separate
                            gradient buffer (needed by max pooling to re-find the arg-max); NULL = table */
  int32_t len_stride;   /* elements between consecutive samples in len (0 = 1)                   */
  int32_t weight_ld;    /* elements between consecutive samples in weight (0 = maxlen)            */
} b2ctr_feature_t;

#define B2CTR_MAX_FEATURES 128

/* Generic fused multi-table gather: any mix of single / pooled / sequence / hashed / weighted
 * features of any dim, one launch.  Pooled sums accumulate in ascending-t order in fp32
 * (bit-exact against oracle/seqpool, SURVEY.md App. A.3). */
B2CTR_API b2ctr_status_t b2ctr_embed_gather_fwd(const b2ctr_feature_t* feats, int32_t nfeat,
                                               int64_t batch, void* stream);

/* Generic scatter: table[id] += scale * d(out) routed through the pooling Jacobian.
 * scale = -lr gives fused SGD; scale = 1 with `table` pointing at a zeroed [vocab,dim] buffer
 * gives a dense gradient (for dense optimizers / l2 on the whole table, SURVEY.md App. C).
 * Duplicate ids are combined with fp32 atomics (vector red.global.add.v4.f32).            */
B2CTR_API b2ctr_status_t b2ctr_embed_scatter_add(const b2ctr_feature_t* feats, int32_t nfeat,
                                                int64_t batch, float scale, void* stream);
/* Max pooling re-finds its arg-max at the forward rows, so a POOL_MAX feature of the scatter above needs them in a
 * src_table other than `table` (B2CTR_ERR_INVALID_ARG otherwise, before any launch).  An update in place goes
 * through this call instead: it reads the forward rows from `table` (and writes no table), and writes every
 * position's share of the gradient `out`
 *   shares[b*shares_ld + c_f + t*dim + e] = out[b, e] / cnt * w_t   where position t attains the max of column e
 *                                           0                        elsewhere (and for out-of-range ids)
 * (cnt = number of positions attaining it, w_t the position weight or 1), c_f = sum over g < f of
 * maxlen_g * dim_g.  Feature f's block is then one B2CTR_POOL_NONE feature of b2ctr_embed_scatter_add (same ids and
 * hashing, out = shares, out_col = c_f), which skips the all-zero rows.  Every feature must be POOL_MAX. */
B2CTR_API b2ctr_status_t b2ctr_embed_max_pool_shares(const b2ctr_feature_t* feats, int32_t nfeat, int64_t batch,
                                                    float* shares, int64_t shares_ld, void* stream);

/* Criteo-shaped fast path (all features single-valued, same dim, dim % 4 == 0, dim <= 128):
 * one warp per sample gathers F rows with 128-bit loads into x[b, f*dim : (f+1)*dim], copies
 * `dense` into x[b, F*dim : F*dim+ndense], zero-fills up to ldx, and in the same pass emits
 *   linear[b] = sum_f lin_table_f[id_f]                 (get_linear_logit, feature_column.py:171-210)
 *   fm[b]     = 0.5 * sum_e((sum_f x)^2 - sum_f x^2)    (FM, layers/interaction.py:597-602)
 * over the features whose bit is set in fm_mask (bit f of fm_mask[f/64]).
 * feats[f].{table,idx,idx_stride,idx_dtype,vocab,dim} are used; lin_tables may be NULL. */
typedef struct b2ctr_uniform_gather {
  const b2ctr_feature_t* feats;
  float* const* lin_tables;     /* host array [nfeat] of device ptrs to [vocab] fp32, or NULL   */
  const float* dense;           /* [B, ndense] (ld = dense_ld) or NULL                          */
  float* x;                     /* [B, ldx] output / saved activations                          */
  float* linear;                /* [B] or NULL                                                  */
  float* fm;                    /* [B] or NULL                                                  */
  int64_t ldx;
  int64_t dense_ld;
  int64_t x_cols;               /* columns of x this call owns: [F*dim+ndense, x_cols) is zero-filled;
                                   0 means ldx (other features may live in x beyond x_cols)        */
  int32_t nfeat;
  int32_t ndense;
  uint64_t fm_mask[2];
  int32_t flags;                /* B2CTR_UNIFORM_* */
  int32_t world;                /* row shards per table (power of two); 0 / 1 = tables are whole         */
  /* world > 1 (row-sharded tables read / updated IN PLACE over NVLink peer mappings, one process per GPU):
   * row r of feature f lives at peer_tables[f * world + (r % world)] + (r / world) * dim.  Both arrays are
   * DEVICE arrays of device pointers (the owner's own shard included); feats[f].table / lin_tables are then
   * ignored.  Gathers are plain peer loads, the backward update is red.add at the owner's L2. */
  float* const* peer_tables;
  float* const* peer_lin_tables; /* [nfeat * world] or NULL */
} b2ctr_uniform_gather_t;
/* scatter_uniform_bwd: every (sample, feature) id is distinct (the ids are positions in a private row
 * buffer, as on the row-sharded path): write scale*g instead of accumulating, no zero-fill needed. */
#define B2CTR_UNIFORM_STORE_GRADS 1

B2CTR_API b2ctr_status_t b2ctr_embed_gather_uniform_fwd(const b2ctr_uniform_gather_t* g,
                                                       int64_t batch, void* stream);
/* The same gather, also writing (each optional, NULL = off):
 *   fm_sum   [batch, dim] fp32: S_b = sum over the fm_mask fields of x[b, f*dim:(f+1)*dim], the vector fm[b] is
 *            formed from (needs fm).  Handing it to b2ctr_embed_scatter_uniform_bwd_ex saves the scatter its own
 *            pass over x; it is summed in the order that scatter would use, so the update is the same bit for bit.
 *   x_planes b2ctr_planes_bytes(batch, x_planes_cols) bytes: the bf16 hi/lo planes of x[:, 0:x_planes_cols] in
 *            b2ctr_split_planes' layout and values (pad columns and pad rows zero), for a first GEMM that reads that
 *            window; F*dim + ndense <= x_planes_cols <= x_cols. */
B2CTR_API b2ctr_status_t b2ctr_embed_gather_uniform_fwd_ex(const b2ctr_uniform_gather_t* g, float* fm_sum,
                                                          void* x_planes, int64_t x_planes_cols, int64_t batch,
                                                          void* stream);

/* Backward of the above fused with the row update:
 *   g_row(b,f) = dx[b, f*dim:(f+1)*dim] + dfm[b] * (S_b - x[b, f*dim:...])   (FM Jacobian, App. A.6)
 *   table_f[id] += scale * g_row ;  lin_table_f[id] += lin_scale * dlinear[b]
 * dx, dfm, dlinear may each be NULL.  The dense columns of dx are not read: their gradient is the caller's.
 * Rows of duplicate ids are combined with red.global.add, in an order that changes from run to run. */
B2CTR_API b2ctr_status_t b2ctr_embed_scatter_uniform_bwd(const b2ctr_uniform_gather_t* g,
                                                        const float* dx, const float* dfm,
                                                        const float* dlinear, float scale,
                                                        float lin_scale, int64_t batch,
                                                        void* stream);
/* The same update with S_b read from fm_sum (written by b2ctr_embed_gather_uniform_fwd_ex) instead of summed
 * from x; fm_sum NULL = the call above. */
B2CTR_API b2ctr_status_t b2ctr_embed_scatter_uniform_bwd_ex(const b2ctr_uniform_gather_t* g,
                                                           const float* dx, const float* dfm,
                                                           const float* fm_sum, const float* dlinear,
                                                           float scale, float lin_scale, int64_t batch,
                                                           void* stream);

/* Ids outside [0, vocab) (b2ctr_feature_t.vocab = the FULL vocabulary_size, also for row-sharded tables):
 * every gather kernel returns a ZERO row for them and every update kernel skips them - no out-of-bounds
 * access in either direction (tf.keras.layers.Embedding on a GPU returns zeros, on a CPU it raises
 * InvalidArgument; deepctr/inputs.py:101-130 just calls it).  The kernels count such ids in a per-device
 * counter; this call reads (and optionally resets) it, synchronising `stream` - the host mirror raises
 * ValueError like TF-CPU when it is non-zero. */
B2CTR_API b2ctr_status_t b2ctr_embed_oob_count(int64_t* count, int32_t reset, void* stream);

/* Field-aware pairwise products (ONN / NFFM, deepctr/models/onn.py): field a owns one [vocab_a, dim] table per
 * partner field b != a.  Pair p = (i, j), i < j, in itertools.combinations order, is
 *   prod_p = e_{i,(j)} * e_{j,(i)}          e_{a,(b)} = field a's row in its table for partner b
 * written to out[b*out_ld + out_col + p*dim + e] (reduce_sum = 0) or its sum over e to out[b*out_ld + out_col + p]
 * (reduce_sum = 1).  One launch forms all P = F(F-1)/2 products from the tables; the F(F-1) looked-up rows are
 * never written.  A hashed field is hashed once per sample.  An id outside [0, vocab) reads a zero row and is
 * counted as for every other gather (b2ctr_embed_oob_count).
 *   tables: DEVICE array [F*F] of device pointers, field a's table for partner b at a*F + b (the diagonal is
 *           unused); it can stay at one address for the life of a model, so a captured step keeps it.
 *           When dim % 4 == 0, every table must be 16-byte aligned: the kernel takes its float4 path from the
 *           other operands' alignment and cannot see the pointers inside this device array.
 * A field is either single-valued (idx != NULL) or a pre-pooled operand (pooled != NULL: a VarLenSparseFeat bag
 * pooled per partner by b2ctr_embed_gather_fwd).  Partner b of field a has slot s = b - (b > a) in `pooled` and
 * `grad`, whose rows hold F-1 operands of dim floats.  2 <= F <= 64, 1 <= dim <= 64. */
typedef struct b2ctr_ffm_field {
  const void* idx;       /* single-valued: the id of sample b at idx[b*idx_stride]; NULL for a pooled field       */
  const float* pooled;   /* pooled: the operand for partner slot s at pooled[b*pooled_ld + s*dim]; else NULL     */
  float* grad;           /* bwd: d(operand) of partner slot s goes to grad[b*grad_ld + s*dim] (written, no add)  */
  int64_t idx_stride;
  int64_t vocab;         /* rows of each of the field's tables; also num_buckets for hashing                     */
  int64_t pooled_ld;
  int64_t grad_ld;
  int32_t idx_dtype;     /* B2CTR_IDX_*                                                                          */
  int32_t hash_mode;     /* B2CTR_HASH_*                                                                         */
} b2ctr_ffm_field_t;

B2CTR_API b2ctr_status_t b2ctr_ffm_product_fwd(const b2ctr_ffm_field_t* fields, int32_t nfield,
                                               float* const* tables, int32_t dim, int32_t reduce_sum, float* out,
                                               int64_t out_ld, int32_t out_col, int64_t batch, void* stream);
/* Gradient rows of every lookup at the tables' current (pre-step) values, given g = d(out) in the layout of the
 * forward's out:  d e_{i,(j)} = g_p * e_{j,(i)},  d e_{j,(i)} = g_p * e_{i,(j)}  (g_p broadcast over e when
 * reduce_sum).  Each element has one writer: the result is the same bit for bit from run to run.  The tables are
 * only read; the caller applies the rows with b2ctr_embed_scatter_add, one single-valued (or pooled) feature per
 * lookup, which also skips out-of-range ids. */
B2CTR_API b2ctr_status_t b2ctr_ffm_product_bwd(const b2ctr_ffm_field_t* fields, int32_t nfield,
                                               float* const* tables, int32_t dim, int32_t reduce_sum, const float* g,
                                               int64_t g_ld, int32_t g_col, int64_t batch, void* stream);

/* DETERMINISTIC fused update of the Criteo-shaped fast path (same descriptor and gradients as
 * b2ctr_embed_scatter_uniform_bwd; tables whole, world <= 1): the lookups are sorted by (table, id), the
 * gradient rows of all the lookups of one row are summed in ascending (sample, feature) order in fp32 and every
 * touched row is written ONCE - bit-identical from run to run, and the home of row-state optimizers:
 *   optimizer 0: w -= lr * g                       (row-wise SGD)
 *   optimizer 1: acc += g^2; w -= lr * g / (sqrt(acc) + eps)   (Keras Adagrad, whose sparse apply is lazy)
 * acc_tables / lin_acc_tables: host arrays [nfeat] of device pointers shaped like the tables (optimizer 1).
 * Features may share a table (a shared embedding_name); they must then share its linear table and
 * accumulators too, else the call fails with B2CTR_ERR_INVALID_ARG before any launch.
 * Uses cub::DeviceRadixSort from the CUDA toolkit for the key sort. */
B2CTR_API size_t b2ctr_embed_update_sorted_workspace_bytes(int32_t nfeat, int32_t dim, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_embed_update_sorted(const b2ctr_uniform_gather_t* g, const float* dx,
                                                  const float* dfm, const float* dlinear, int32_t optimizer,
                                                  float lr, float lin_lr, float eps, float* const* acc_tables,
                                                  float* const* lin_acc_tables, int64_t batch, void* workspace,
                                                  size_t workspace_bytes, void* stream);

/* Hash (deepctr/layers/utils.py:89-112): ids -> int64 buckets, FarmHash Fingerprint64 of the
 * decimal ASCII form.  mask_zero: 0 stays 0, others land in [1, num_buckets).               */
B2CTR_API b2ctr_status_t b2ctr_hash64(const void* ids, int32_t idx_dtype, int64_t n,
                                     int64_t num_buckets, int32_t mask_zero, int64_t* out,
                                     void* stream);

/* On-device table initialisation: table[i] = mean + std * N(0,1), Philox4x32-10 keyed by seed
 * (RandomNormal(0, 1e-4, seed=2020), deepctr/feature_column.py:46-47; needed because a
 * 26 x 100M x 128 table set cannot be initialised on the host, SURVEY.md §7). */
B2CTR_API b2ctr_status_t b2ctr_init_normal(float* dst, int64_t n, float mean, float std,
                                          uint64_t seed, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 2. Dense linear algebra: C = epilogue(op(A) @ op(B))                                        */
/*    replaces tf.tensordot / tf.matmul in deepctr/layers/core.py:193-195 (DNN), :106 (LAU),   */
/*    deepctr/layers/interaction.py:754-757 (InteractingLayer projections), :414-418 (CrossNet)*/
/* ------------------------------------------------------------------------------------------ */
enum { B2CTR_ACT_NONE = 0, B2CTR_ACT_RELU = 1, B2CTR_ACT_SIGMOID = 2, B2CTR_ACT_TANH = 3 };
enum { B2CTR_GEMM_FP32 = 0,  /* exact fp32 FFMA path (CUDA cores)                              */
       B2CTR_GEMM_BF16X3 = 1 /* wgmma tensor cores, 3-term split-bf16 (~2^-17 rel. error)      */ };

typedef struct b2ctr_gemm {
  const float* a; const float* b; float* c;
  const float* bias;       /* [N] added to every row, or NULL                                  */
  int64_t m, n, k;
  int64_t lda, ldb, ldc;   /* leading dims of the STORED matrices (row-major)                  */
  int32_t trans_a;         /* 0: A stored [M,K]; 1: A stored [K,M]                             */
  int32_t trans_b;         /* 0: B stored [K,N]; 1: B stored [N,K]                             */
  int32_t act;             /* B2CTR_ACT_* applied after bias                                   */
  int32_t accumulate;      /* 1: C += result (before act; act must be NONE)                    */
  int32_t precision;       /* B2CTR_GEMM_*                                                     */
  int32_t split_k;         /* >1: split the K loop over this many CTAs (needs workspace)       */
  float alpha;             /* scales op(A)@op(B)                                               */
  int32_t variant;         /* BF16X3 only: 0 default (persistent), 3 non-persistent reference kernel, 4 persistent */
  const void* a_planes;    /* optional: b2ctr_split_planes() of the STORED a / b matrix.  Lets one split */
  const void* b_planes;    /* serve every GEMM that reads the tensor (forward, dgrad, wgrad); BF16X3 only */
                           /* a / b may then be NULL unless the call must split that operand itself    */
                           /* (B with N <= 32 stored [K,N]): B2CTR_ERR_INVALID_ARG                    */
} b2ctr_gemm_t;

/* bf16 (hi, lo) planes of an fp32 matrix [rows, cols]: hi = bf16(x), lo = bf16(x - hi), zero padded to
 * [round_up(rows,256), cols <= 64 ? 64 : round_up(cols,128)]; the buffer holds the hi plane followed by the
 * lo plane (b2ctr_planes_bytes() includes the slack the tile loads need). */
B2CTR_API size_t b2ctr_planes_bytes(int64_t rows, int64_t cols);
B2CTR_API b2ctr_status_t b2ctr_split_planes(const float* src, int64_t ld, int64_t rows, int64_t cols,
                                           void* planes, void* stream);

B2CTR_API size_t b2ctr_gemm_workspace_bytes(const b2ctr_gemm_t* g);
B2CTR_API b2ctr_status_t b2ctr_gemm(const b2ctr_gemm_t* g, void* workspace, size_t workspace_bytes,
                                   void* stream);

/* A relu DNN tower's hidden layers after the first, fused.  widths[0..nlayers-1] are the widths of hidden layers
 * 0..L-1 (L = nlayers); y_i = relu(y_{i-1} W_i + b_i) for i = 1..L-1 in split-bf16 (hi*hi + hi*lo + lo*hi, fp32
 * accumulation), W_i = w[i-1] [widths[i-1], widths[i]] row-major, b_i = b[i-1].  All activations and gradients are
 * contiguous [batch, width] fp32.  b2ctr_mlp_relu_supported says whether a tower is supported (1) or not (0); the
 * other calls return B2CTR_ERR_INVALID_ARG for an unsupported one.
 * Forward: reads y0, writes planes[i] = b2ctr_split_planes of y_i for i = 0..L-2 (b2ctr_planes_bytes(batch,
 * widths[i]) bytes each) and y_last = y_{L-1}.
 * Backward: dy_last is the gradient of y_last; dz_{L-1} = dy_last * [y_last > 0], dz_{i-1} = (dz_i W_i^T) * [y_{i-1} > 0]
 * (y_0's mask from y0, the inner layers' from the forward's planes).  Writes dz_planes[i] = b2ctr_split_planes of dz_i
 * and dbias[i] = column sums of dz_i (per-CTA partials reduced in a fixed order: deterministic), i = 0..L-1. */
B2CTR_API int32_t b2ctr_mlp_relu_supported(const int32_t* widths, int32_t nlayers);
B2CTR_API b2ctr_status_t b2ctr_mlp_relu_fwd(const float* y0, const float* const* w, const float* const* b,
                                           void* const* planes, float* y_last, const int32_t* widths,
                                           int32_t nlayers, int64_t batch, void* stream);
B2CTR_API size_t b2ctr_mlp_relu_bwd_workspace_bytes(const int32_t* widths, int32_t nlayers);
B2CTR_API b2ctr_status_t b2ctr_mlp_relu_bwd(const float* dy_last, const float* y_last, const float* y0,
                                           void* const* planes, const float* const* w, void* const* dz_planes,
                                           float* const* dbias, const int32_t* widths, int32_t nlayers,
                                           int64_t batch, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 3. Elementwise / reductions                                                                 */
/* ------------------------------------------------------------------------------------------ */
/* dz = dy * act'(y) (y = activation OUTPUT), dbias[n] = sum_m dz[m,n] (deterministic two-pass)  */
B2CTR_API size_t b2ctr_bias_act_bwd_workspace_bytes(int64_t m, int64_t n);
B2CTR_API b2ctr_status_t b2ctr_bias_act_bwd(const float* dy, const float* y, float* dz,
                                           float* dbias, int64_t m, int64_t n, int64_t ld,
                                           int32_t act, void* workspace, size_t workspace_bytes,
                                           void* stream);
/* Same, and additionally the bf16 hi/lo operand planes of dz (b2ctr_split_planes layout) for the dgrad /
 * wgrad GEMMs that consume dz next - saves the separate split pass.  Requires m % 256 == 0 and
 * n == 64 or n % 128 == 0 (no padding inside the planes), n / 4 dividing 256. */
B2CTR_API b2ctr_status_t b2ctr_bias_act_bwd_planes(const float* dy, const float* y, float* dz, float* dbias,
                                                  void* dz_planes, int64_t m, int64_t n, int64_t ld,
                                                  int32_t act, void* workspace, size_t workspace_bytes,
                                                  void* stream);
/* y = act(x) elementwise over n contiguous elements */
B2CTR_API b2ctr_status_t b2ctr_act_fwd(const float* x, float* y, int64_t n, int32_t act,
                                      void* stream);
/* out[i] = sum_j in_j[i] * (scale_j), j < nin <= 8, in_j may alias out */
B2CTR_API b2ctr_status_t b2ctr_add_n(const float* const* ins, const float* scales, int32_t nin,
                                    float* out, int64_t n, void* stream);
/* y[i] += alpha * x[i] */
B2CTR_API b2ctr_status_t b2ctr_axpy(const float* x, float* y, float alpha, int64_t n, void* stream);
/* strided 2-D copy: dst[r*ld_dst + c] (+)= src[r*ld_src + c], r<rows, c<cols  (concat / slice)  */
B2CTR_API b2ctr_status_t b2ctr_copy2d(const float* src, int64_t ld_src, float* dst, int64_t ld_dst,
                                     int64_t rows, int64_t cols, int32_t accumulate, void* stream);
/* input staging: src holds nblk contiguous blocks, block i = [batch, widths[i]] row-major; dst[b, :] is
 * their row-wise concatenation (the dense-feature pack, deepctr/inputs.py:161-172 + layers/utils.py:336-346) */
B2CTR_API b2ctr_status_t b2ctr_pack_rows(const float* src, const int32_t* widths, int32_t nblk, int64_t batch,
                                        float* dst, int64_t ld_dst, void* stream);
/* out[r] = sum_c x[r*ld + c] (ascending c, fp32)   (Linear mode 0/2, layers/utils.py:160-171) */
B2CTR_API b2ctr_status_t b2ctr_rowsum(const float* x, int64_t ld, float* out, int64_t rows,
                                     int64_t cols, void* stream);
B2CTR_API b2ctr_status_t b2ctr_fill(float* dst, float value, int64_t n, void* stream);
/* Keras masks as uint8 [B,T]: inout[i] = (first ? 1 : inout[i]) & (ids[i] != 0)   (Embedding mask_zero,
 * AND-ed across concatenated features, deepctr/layers/utils.py:198-228) */
B2CTR_API b2ctr_status_t b2ctr_mask_nonzero_and(const void* ids, int32_t idx_dtype, int64_t n,
                                               uint8_t* inout, int32_t first, void* stream);
/* tf.sequence_mask: out[b,t] = t < len[b] */
B2CTR_API b2ctr_status_t b2ctr_mask_from_len(const int32_t* len, int64_t batch, int32_t maxlen,
                                            uint8_t* out, void* stream);

/* FM second-order term on [B,F,E] (deepctr/layers/interaction.py:588-604) and its Jacobian */
B2CTR_API b2ctr_status_t b2ctr_fm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                                     float* out, int64_t batch, void* stream);
B2CTR_API b2ctr_status_t b2ctr_fm_bwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                                     const float* dout, float* dx, int64_t lddx, int32_t accumulate,
                                     int64_t batch, void* stream);
/* FM of the field-weighted input m ⊙ x (IFM / DIFM: FM(refined embeddings), deepctr/models/ifm.py:66-68) without
 * writing m ⊙ x.  x [B, nfield, dim] (row pitch ldx), m [B, nfield] (row pitch ldm):
 *   out[b] = 1/2 sum_e [(sum_f m_bf x_bfe)^2 - sum_f m_bf^2 x_bfe^2]
 * Backward, with S_be = sum_f m_bf x_bfe:
 *   dx_bfe = g_b m_bf (S_be - m_bf x_bfe)       (pitch lddx; added to dx when accumulate; may be NULL)
 *   dm_bf  = g_b sum_e x_bfe (S_be - m_bf x_bfe) (pitch lddm, overwritten; may be NULL)
 * Same launch shape and limits as b2ctr_fm_fwd / _bwd; with m == 1 the results equal theirs bit for bit.  No float
 * atomics: bit-identical from run to run. */
B2CTR_API b2ctr_status_t b2ctr_fm_weighted_fwd(const float* x, int64_t ldx, const float* m, int64_t ldm,
                                              int32_t nfield, int32_t dim, float* out, int64_t batch, void* stream);
B2CTR_API b2ctr_status_t b2ctr_fm_weighted_bwd(const float* x, int64_t ldx, const float* m, int64_t ldm,
                                              int32_t nfield, int32_t dim, const float* dout, float* dx, int64_t lddx,
                                              int32_t accumulate, float* dm, int64_t lddm, int64_t batch,
                                              void* stream);
/* Materialised field scale (RefineWeight of get_linear_logit, feature_column.py:193-200, with dim = 1; the refine
 * product when its consumer is not FM):  y[b, f*dim + e] = x[b, f*dim + e] * m[b, f]   (pitches ldx, ldm, ldy).
 * Backward: dx = dy * m (pitch lddx; added when accumulate; may be NULL), dm[b, f] = sum_e dy x (pitch lddm,
 * overwritten; may be NULL), summed in a fixed order: bit-identical from run to run. */
B2CTR_API b2ctr_status_t b2ctr_field_scale_fwd(const float* x, int64_t ldx, const float* m, int64_t ldm,
                                              int32_t nfield, int32_t dim, float* y, int64_t ldy, int64_t batch,
                                              void* stream);
B2CTR_API b2ctr_status_t b2ctr_field_scale_bwd(const float* dy, int64_t lddy, const float* x, int64_t ldx,
                                              const float* m, int64_t ldm, int32_t nfield, int32_t dim, float* dx,
                                              int64_t lddx, int32_t accumulate, float* dm, int64_t lddm,
                                              int64_t batch, void* stream);
/* y = scale * softmax(x) along the rows of a [rows, cols] window (layers/utils.py softmax on the last axis; IFM
 * uses scale = F).  The row maximum is subtracted first.  Backward: dx = y * (dy - sum_j y_j dy_j / scale),
 * overwritten.  scale must not be 0. */
B2CTR_API b2ctr_status_t b2ctr_softmax_rows_fwd(const float* x, int64_t ldx, float* y, int64_t ldy, int64_t rows,
                                               int32_t cols, float scale, void* stream);
B2CTR_API b2ctr_status_t b2ctr_softmax_rows_bwd(const float* y, int64_t ldy, const float* dy, int64_t lddy,
                                               float* dx, int64_t lddx, int64_t rows, int32_t cols, float scale,
                                               void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 4. Prediction head, loss, optimizers                                                         */
/* ------------------------------------------------------------------------------------------ */
/* PredictionLayer (deepctr/layers/core.py:250-259) + Keras binary_crossentropy / mse
 * (SURVEY.md App. C) in one pass:
 *   z = logit[b] + (bias ? *bias : 0);  p = task==binary ? sigmoid(z) : z;  pred[b] = p
 *   loss_sum[0] += sum_b l(y_b, p_b)  (caller zeroes it; divide by B on the host side)
 *   dlogit[b] = (1/B) * dl/dz   (dlogit / labels / loss_sum may be NULL for inference)        */
enum { B2CTR_TASK_BINARY = 0, B2CTR_TASK_REGRESSION = 1 };
B2CTR_API b2ctr_status_t b2ctr_predict_loss(const float* logit, const float* bias,
                                           const float* labels, float* pred, float* dlogit,
                                           float* dbias, float* loss_sum, int64_t batch,
                                           int32_t task, void* stream);

B2CTR_API b2ctr_status_t b2ctr_sgd_step(float* w, const float* g, float lr, float l2, int64_t n,
                                       void* stream);
/* The same update for `count` tensors in one launch (host arrays of device pointers / sizes / l2 factors):
 * w[t][i] -= lr * (g[t][i] + 2 * l2[t] * w[t][i]).  A tower's 9-14 dense weights are a few kB each. */
B2CTR_API b2ctr_status_t b2ctr_sgd_step_multi(float* const* w, const float* const* g, const int64_t* n,
                                              const float* l2, int32_t count, float lr, void* stream);
/* Keras Adam (lr 1e-3, b1 .9, b2 .999, eps 1e-7): step counts from 1 */
B2CTR_API b2ctr_status_t b2ctr_adam_step(float* w, const float* g, float* m, float* v, float lr,
                                        float beta1, float beta2, float eps, float l2,
                                        int64_t step, int64_t n, void* stream);
/* Same update with the step count t read from device memory (>= 1 when the kernel runs): no step-dependent
 * by-value argument, so the launch can live in a replayed CUDA graph.  b2ctr_counter_add advances the counter
 * (once per training step, before the first b2ctr_adam_step_dev of the step). */
B2CTR_API b2ctr_status_t b2ctr_adam_step_dev(float* w, const float* g, float* m, float* v, float lr,
                                            float beta1, float beta2, float eps, float l2,
                                            const int64_t* step_dev, int64_t n, void* stream);
B2CTR_API b2ctr_status_t b2ctr_counter_add(int64_t* counter, int64_t delta, void* stream);
B2CTR_API b2ctr_status_t b2ctr_adagrad_step(float* w, const float* g, float* acc, float lr,
                                           float eps, float l2, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 5. Interaction operators                                                                     */
/* ------------------------------------------------------------------------------------------ */
/* out = a*b (op 0) or a*b + c (op 1), elementwise over n; accumulate: out += */
B2CTR_API b2ctr_status_t b2ctr_ewise(int32_t op, const float* a, const float* b, const float* c,
                                    float* out, int64_t n, int32_t accumulate, void* stream);

/* CrossNet 'vector' layer (deepctr/layers/interaction.py:413-416):
 *   s[b] = <xl[b], w>;  out[b] = x0[b]*s[b] + bias + xl[b]          (one warp per sample, shuffles)
 * backward: dx0 = dout*s, dxl = dout + w*ds, ds[b] = <dout[b], x0[b]>; dw = xl^T ds and
 * dbias = colsum(dout) are left to b2ctr_gemm / b2ctr_bias_act_bwd.                            */
B2CTR_API b2ctr_status_t b2ctr_cross_vector_fwd(const float* x0, int64_t ld0, const float* xl,
                                               int64_t ldl, const float* w, const float* bias,
                                               float* out, float* s, int64_t batch, int32_t dim,
                                               void* stream);
B2CTR_API b2ctr_status_t b2ctr_cross_vector_bwd(const float* x0, int64_t ld0, const float* w,
                                               const float* dout, const float* s, float* dx0,
                                               float* dxl, float* ds, int64_t batch, int32_t dim,
                                               void* stream);

/* CIN (deepctr/layers/interaction.py:277-325).  X(b,i,d) = x[b*sb + i*si + d*sd].
 * outer_fwd: z[(b,d), i*h + j] = X0(b,i,d) * Xk(b,j,d) for a batch chunk sized to stay in L2; the
 * contraction z @ filter runs through b2ctr_gemm.  outer_bwd folds d z back onto X0 / Xk.       */
B2CTR_API b2ctr_status_t b2ctr_cin_outer_fwd(const float* x0, int64_t s0b, int64_t s0i, int64_t s0d,
                                            const float* xk, int64_t skb, int64_t ski, int64_t skd,
                                            float* z, int64_t nb, int32_t m, int32_t h, int32_t d,
                                            void* stream);
B2CTR_API b2ctr_status_t b2ctr_cin_outer_bwd(const float* dz, const float* x0, int64_t s0b, int64_t s0i,
                                            int64_t s0d, const float* xk, int64_t skb, int64_t ski,
                                            int64_t skd, float* dx0, int64_t g0b, int64_t g0i,
                                            int64_t g0d, int32_t acc0, float* dxk, int64_t gkb,
                                            int64_t gki, int64_t gkd, int32_t acck, int64_t nb,
                                            int32_t m, int32_t h, int32_t d, int32_t hp, void* stream);
/* (hp: dZ rows hold m groups of hp columns of which the first h are used - the padded layout of
 *  b2ctr_cin_gemm; 0 or h = dense) */
/* out[b, out_col+n] = sum_d y[(b,d), col0+n]  (reduce_sum over D of the direct maps, :322-323) */
/* CIN filter contraction with the outer product GENERATED inside the GEMM producer (never stored):
 *   Z[r, i*hp + j] = t0[r, i] * xk[r, j]     r = b*D + d;  t0[r, i] = X0(b,i,d);  xk[r, j] = X_k(b,j,d), j < h
 * hp = h padded to 32 (h <= 32) or to a multiple of 64, so that a 64-deep k-block never straddles an i; the
 * filter is used in the matching padded layout W'[i*hp + j, n] (b2ctr_cin_filter_planes: bf16 hi/lo planes).
 *   mode 0:  c[rows, n]   = act(Z W' + bias)     (forward; deepctr/layers/interaction.py:291-306)
 *   mode 1:  c[m*hp, n]   = Z^T dY               (filter gradient; dY given as b2ctr_split_planes of [rows, n])
 * wgmma split-bf16 (BF16X3) arithmetic, TMA for the B operand, 128 producer threads generate A. */
typedef struct b2ctr_cin_gemm {
  const float* t0; int64_t ld0;      /* [rows, ld0], columns >= m are ignored                          */
  const float* xk; int64_t ldk;      /* [rows, ldk], 16-byte aligned rows (ldk % 4 == 0)                */
  int64_t rows;
  int32_t m, h, hp, n;
  const void* w_planes;              /* mode 0                                                         */
  const void* dy_planes;             /* mode 1                                                         */
  float* c; int64_t ldc;
  const float* bias;                 /* mode 0: [n] or NULL                                            */
  int32_t act, mode, split_k;
} b2ctr_cin_gemm_t;
B2CTR_API size_t b2ctr_cin_filter_planes_bytes(int32_t m, int32_t hp, int64_t n);
B2CTR_API b2ctr_status_t b2ctr_cin_filter_planes(const float* w, int32_t m, int32_t h, int32_t hp, int64_t n,
                                                void* planes, void* stream);
B2CTR_API size_t b2ctr_cin_gemm_workspace_bytes(const b2ctr_cin_gemm_t* g);
B2CTR_API b2ctr_status_t b2ctr_cin_gemm(const b2ctr_cin_gemm_t* g, void* workspace, size_t workspace_bytes,
                                       void* stream);
/* First layer of DIN's LocalActivationUnit (deepctr/layers/core.py:96-103) with its input
 *   A[(b,t), :] = [ q_b , k_bt , q_b - k_bt , q_b * k_bt ]     ([B*T, 4E]; the reference materialises it)
 * GENERATED inside the GEMM producer from the queries [B, E] and the keys [B, T, E]:
 *   mode 0:  c[B*T, n] = act(A W + bias), planes = b2ctr_split_planes of W [4E, n]
 *   mode 1:  c[4E, n]  = A^T dY,          planes = b2ctr_split_planes of dY [B*T, n]     (kernel gradient)  */
typedef struct b2ctr_att_gemm {
  const float* query; int64_t ldq;              /* [batch, ldq], first `dim` columns                         */
  const float* keys; int64_t key_batch_stride;  /* keys of sample b start at keys + b*key_batch_stride, rows of `dim` */
  int64_t batch; int32_t maxlen, dim, n;
  const void* planes;
  float* c; int64_t ldc;
  const float* bias; int32_t act, mode, split_k;
} b2ctr_att_gemm_t;
B2CTR_API size_t b2ctr_att_gemm_workspace_bytes(const b2ctr_att_gemm_t* g);
B2CTR_API b2ctr_status_t b2ctr_att_gemm(const b2ctr_att_gemm_t* g, void* workspace, size_t workspace_bytes,
                                       void* stream);
/* CIN backward, data gradient: dZ = dY W'^T (dy_planes: b2ctr_split_planes of dY [rows, n]; w_planes as in mode 0)
 * is formed tile by tile in registers and FOLDED onto the two factors inside the GEMM epilogue - it is never stored:
 *   dt0[r, i]  += sum_j dZ[r, i*hp + j] * xk[r, j]        dxk[r, j] += sum_i dZ[r, i*hp + j] * t0[r, i]
 * Both outputs are accumulated with red.add (zero them first; layer 0 passes dxk = dt0).  hp in {32, 64, 128};
 * c / ldc / bias / act / mode / split_k of the descriptor are ignored. */
B2CTR_API b2ctr_status_t b2ctr_cin_fold(const b2ctr_cin_gemm_t* g, float* dt0, float* dxk, int64_t ldx,
                                       void* stream);
/* dX0(b,i,d) (+)= dt0[(b*D + d), i] (dX0 given by its three strides). */
B2CTR_API b2ctr_status_t b2ctr_cin_t0_bwd(const float* dt0, int64_t ld0, float* dx, int64_t gb, int64_t gi,
                                         int64_t gd, int32_t accumulate, int64_t nb, int32_t m, int32_t d,
                                         void* stream);
/* t0[(b*D + d), i] = X0(b,i,d) for i < m, zero for m <= i < ld0 (X0 given by its three strides). */
B2CTR_API b2ctr_status_t b2ctr_cin_t0(const float* x0, int64_t s0b, int64_t s0i, int64_t s0d, float* t0,
                                     int64_t ld0, int64_t nb, int32_t m, int32_t d, void* stream);
/* dst[i*h + j, :] = src[i*hp + j, :] (j < h): the gradient of the padded filter back in W's layout. */
B2CTR_API b2ctr_status_t b2ctr_cin_unpad_rows(const float* src, float* dst, int32_t m, int32_t h, int32_t hp,
                                             int64_t n, void* stream);

B2CTR_API b2ctr_status_t b2ctr_cin_sum_d(const float* y, int64_t ldy, int32_t col0, int32_t ncols,
                                        int32_t d, float* out, int64_t ldo, int32_t out_col,
                                        int64_t nb, void* stream);
/* dy[(b,d), n] = [col0 <= n < col0+ncols] dout[b, out_col+n-col0] + [n < hcols] dh[(b,d), n] */
B2CTR_API b2ctr_status_t b2ctr_cin_expand_grad(const float* dout, int64_t ldo, int32_t out_col,
                                              int32_t col0, int32_t ncols, const float* dh,
                                              int64_t ldh, int32_t hcols, float* dy, int64_t nfilt,
                                              int32_t d, int64_t nb, void* stream);

/* InteractingLayer attention core (deepctr/layers/interaction.py:760-777) on projected
 * q/k/v[/res] of shape [B, F, heads*dhead]: out = relu(softmax(q_h k_h^T [/sqrt(d)]) v_h + res).
 * Both entry points accept the same shapes: F <= 64, dhead <= 32 and F*heads*dhead <= 3072 (the
 * backward keeps K, V, dK and dV of one sample in 48 KB of shared memory), so a forward that runs
 * always has a backward that runs. */
B2CTR_API b2ctr_status_t b2ctr_interacting_fwd(const float* q, const float* k, const float* v,
                                              const float* res, float* out, int64_t batch,
                                              int32_t nfield, int32_t heads, int32_t dhead,
                                              int32_t scaling, void* stream);
B2CTR_API b2ctr_status_t b2ctr_interacting_bwd(const float* q, const float* k, const float* v,
                                              const float* out, const float* dout, float* dq,
                                              float* dk, float* dv, float* dres, int64_t batch,
                                              int32_t nfield, int32_t heads, int32_t dhead,
                                              int32_t scaling, void* stream);

/* BiInteractionPooling (deepctr/layers/interaction.py:163-206) on x [B, nfield, dim] (row pitch ldx, so a
 * window of the fused gather's buffer is read in place):
 *   out[b*ldo + e] = 0.5 * ((sum_f x[b,f,e])^2 - sum_f x[b,f,e]^2)
 * backward: dx[b*lddx + f*dim + e] = g[b*ldg + e] * (S[b,e] - x[b,f,e]), S = sum_f x.  One warp per sample. */
B2CTR_API b2ctr_status_t b2ctr_bi_interaction_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                                                 float* out, int64_t ldo, int64_t batch, void* stream);
B2CTR_API b2ctr_status_t b2ctr_bi_interaction_bwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim,
                                                 const float* g, int64_t ldg, float* dx, int64_t lddx,
                                                 int64_t batch, void* stream);

/* AFMLayer attention pooling (deepctr/layers/interaction.py:116-143 up to the dropout) on x [B, nfield, dim]
 * (pitch ldx), W [dim, factor] (attention_W), bias [factor] (attention_b), h [factor] (projection_h):
 *   prod_p = x_i * x_j for the P = nfield(nfield-1)/2 pairs i < j
 *   alpha  = softmax_p(h . relu(W^T prod_p + bias));   att[b*ldo + e] = sum_p alpha_p prod_p[e]
 *   state[2b] = max_p s_p, state[2b+1] = sum_p exp(s_p - max)   (saved for the backward)
 * The pairwise products and the attention hidden layer are generated on chip and never written.
 * Limits: 2 <= nfield <= 64, 1 <= dim <= 32, 1 <= factor <= 16; anything else is B2CTR_ERR_INVALID_ARG. */
B2CTR_API b2ctr_status_t b2ctr_afm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t factor,
                                      const float* W, const float* bias, const float* h, float* att, int64_t ldo,
                                      float* state, int64_t batch, void* stream);
/* Backward from g = d att [B, dim] (pitch ldg), the forward's state and att (pitch lda):
 *   dx [B, nfield*dim] (pitch lddx, overwritten), dW [dim, factor], dbias [factor], dh [factor] (overwritten).
 * Weight gradients are summed per CTA into the workspace and reduced in a fixed order: no float atomics,
 * bit-identical from run to run. */
B2CTR_API size_t b2ctr_afm_bwd_workspace_bytes(int32_t dim, int32_t factor, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_afm_bwd(const float* g, int64_t ldg, const float* x, int64_t ldx, int32_t nfield,
                                      int32_t dim, int32_t factor, const float* W, const float* bias,
                                      const float* h, const float* state, const float* att, int64_t lda,
                                      float* dx, int64_t lddx, float* dW, float* dbias, float* dh, int64_t batch,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* SENETLayer (deepctr/layers/interaction.py:1067-1139) on x [B, nfield, dim] (row pitch ldx), W1 [nfield, reduce],
 * W2 [reduce, nfield]:
 *   Z = mean_e x;  A1 = relu(Z W1);  A2 = relu(A1 W2);  v[b*ldv + f*dim + e] = x[b,f,e] * A2[b,f]
 *   saved [B, reduce + nfield] = (A1, A2), kept for the backward.
 * Limits: 2 <= nfield <= 64, 1 <= reduce <= 64; anything else is B2CTR_ERR_INVALID_ARG. */
B2CTR_API b2ctr_status_t b2ctr_senet_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t reduce,
                                        const float* W1, const float* W2, float* v, int64_t ldv, float* saved,
                                        int64_t batch, void* stream);
/* Backward from g = dV (pitch ldg): dx = g * A2 + dZ / dim (pitch lddx, overwritten), dW1, dW2 (overwritten).
 * The gradient of relu at 0 is 0.  Weight gradients go through per-CTA partials in the workspace, summed in a
 * fixed order: bit-identical from run to run. */
B2CTR_API size_t b2ctr_senet_bwd_workspace_bytes(int32_t nfield, int32_t reduce, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_senet_bwd(const float* g, int64_t ldg, const float* x, int64_t ldx, int32_t nfield,
                                        int32_t dim, int32_t reduce, const float* W1, const float* W2,
                                        const float* saved, float* dx, int64_t lddx, float* dW1, float* dW2,
                                        int64_t batch, void* workspace, size_t workspace_bytes, void* stream);

/* BilinearInteraction (deepctr/layers/interaction.py:1142-1221) on x [B, nfield, dim] (row pitch ldx) and the
 * stacked weights W [nW, dim, dim]: type 0 'all' (nW = 1), 1 'each' (nW = nfield - 1, W_i for the pairs (i, j)),
 * 2 'interaction' (nW = P, one per pair).  For the P = nfield(nfield-1)/2 pairs p = (i < j) in
 * itertools.combinations order:
 *   out[b*ldo + col0 + p*pitch + o] = (x_i W_k)[o] * x_j[o]
 * so the output can be a window of a wider buffer (the first DNN layer's input); nothing else is written.
 * Limits: 2 <= nfield <= 64, 1 <= dim <= 64, pitch >= dim. */
B2CTR_API b2ctr_status_t b2ctr_bilinear_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t type,
                                           const float* W, float* out, int64_t ldo, int64_t col0, int64_t pitch,
                                           int64_t batch, void* stream);
/* Backward from g, addressed like the forward's output (ldg, gcol0, gpitch), read in place:
 *   dx [B, nfield*dim] (pitch lddx, overwritten; may be NULL), dW [nW, dim, dim] (overwritten; may be NULL).
 * Every dx element has one owner that adds its pairs in a fixed order; dW goes through ordered partials in the
 * workspace.  No float atomics: bit-identical from run to run. */
B2CTR_API size_t b2ctr_bilinear_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_bilinear_bwd(const float* g, int64_t ldg, int64_t gcol0, int64_t gpitch,
                                           const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t type,
                                           const float* W, float* dx, int64_t lddx, float* dW, int64_t batch,
                                           void* workspace, size_t workspace_bytes, void* stream);

/* FwFMLayer (deepctr/layers/interaction.py:1350-1425) on x [B, nfield, dim] (row pitch ldx) and the field-pair
 * strengths r [nfield, nfield], of which only the upper triangle i < j is read:
 *   out[b*ldo] = sum_{i<j} r[i][j] <x_i, x_j>
 * Limits: 2 <= nfield <= 64, 1 <= dim <= 64; anything else is B2CTR_ERR_INVALID_ARG. */
B2CTR_API b2ctr_status_t b2ctr_fwfm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* r,
                                       float* out, int64_t ldo, int64_t batch, void* stream);
/* Backward from g [B, 1] (pitch ldg):
 *   dx_i = g * sum_{j != i} r[min(i,j)][max(i,j)] x_j   (pitch lddx, overwritten; may be NULL)
 *   dR [nfield, nfield] (overwritten; may be NULL): sum_b g_b <x_i, x_j> for i < j, exactly 0 elsewhere.
 * Every dx element has one owner that adds its partners in ascending order; dR goes through per-CTA partials in
 * the workspace, summed in CTA order.  No float atomics: bit-identical from run to run. */
B2CTR_API size_t b2ctr_fwfm_bwd_workspace_bytes(int32_t nfield, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_fwfm_bwd(const float* g, int64_t ldg, const float* x, int64_t ldx, int32_t nfield,
                                       int32_t dim, const float* r, float* dx, int64_t lddx, float* dR, int64_t batch,
                                       void* workspace, size_t workspace_bytes, void* stream);

/* FEFMLayer (deepctr/layers/interaction.py:1428-1499).  b2ctr_fefm_sym builds S_p = W_p + W_p^T for the npairs
 * stacked [dim, dim] weights W (S must not alias W); the forward and backward take S.  For the
 * P = nfield(nfield-1)/2 pairs p = (i < j) in itertools.combinations order, on x [B, nfield, dim] (row pitch ldx):
 *   out[b*ldo + col0 + p] = x_i S_p x_j^T
 * so the scores can be a window of a wider buffer (the first DNN layer's input); nothing else is written.
 * Limits: 2 <= nfield <= 64, 1 <= dim <= 64. */
B2CTR_API b2ctr_status_t b2ctr_fefm_sym(const float* W, int32_t npairs, int32_t dim, float* S, void* stream);
B2CTR_API b2ctr_status_t b2ctr_fefm_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* S,
                                       float* out, int64_t ldo, int64_t col0, int64_t batch, void* stream);
/* Backward from g[b*ldg + gcol0 + p], read in place:
 *   dx_f = sum_{q != f} g_p(f,q) x_q S_p   (pitch lddx, overwritten; may be NULL)
 *   dW_p = dS_p + dS_p^T with dS_p = sum_b g_p x_i^T x_j   ([P, dim, dim], overwritten; may be NULL)
 * Every dx element has one owner that adds its partners in ascending order; dW goes through per-(pair, batch chunk)
 * partials in the workspace, reduced in a fixed order.  No float atomics: bit-identical from run to run. */
B2CTR_API size_t b2ctr_fefm_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_fefm_bwd(const float* g, int64_t ldg, int64_t gcol0, const float* x, int64_t ldx,
                                       int32_t nfield, int32_t dim, const float* S, float* dx, int64_t lddx, float* dW,
                                       int64_t batch, void* workspace, size_t workspace_bytes, void* stream);

/* PNN (deepctr/models/pnn.py).  For the P = nfield(nfield-1)/2 pairs p = (i < j) in itertools.combinations order,
 * on x [B, nfield, dim] (row pitch ldx), written to the column window out[b*ldo + col0 + ...] of a wider buffer:
 *   B2CTR_PNN_INNER        out[.. + p]         = <x_i, x_j>                 InnerProductLayer()
 *   B2CTR_PNN_ELEMENTWISE  out[.. + p*dim + e] = x_i[e] x_j[e]              InnerProductLayer(reduce_sum=False)
 *   B2CTR_PNN_VEC          out[.. + p]         = sum_e x_i[e] x_j[e] K[p][e]  OutterProductLayer('vec'), K [P, dim]
 *   B2CTR_PNN_NUM          out[.. + p]         = K[p] <x_i, x_j>            OutterProductLayer('num'), K [P, 1]
 * K is ignored (may be NULL) for the first two.  Limits: 2 <= nfield <= 64, 1 <= dim <= 64. */
enum { B2CTR_PNN_INNER = 0, B2CTR_PNN_ELEMENTWISE = 1, B2CTR_PNN_VEC = 2, B2CTR_PNN_NUM = 3 };
B2CTR_API b2ctr_status_t b2ctr_pnn_inner_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, int32_t mode,
                                            const float* K, float* out, int64_t ldo, int64_t col0, int64_t batch,
                                            void* stream);
/* Backward from g[b*ldg + gcol0 + ...] (addressed like the forward's output), read in place:
 *   dx_f[e] = sum_{q != f} g_p w_p[e] x_q[e]   (pitch lddx, overwritten; may be NULL)
 *   dK (vec / num only; may be NULL): sum_b g_p x_i[e] x_j[e]  /  sum_b g_p <x_i, x_j>
 * Every dx element has one owner that adds its partners in ascending order; dK goes through per-(entry tile,
 * batch chunk) partials in the workspace, summed in chunk order.  No float atomics: bit-identical from run to run. */
B2CTR_API size_t b2ctr_pnn_inner_bwd_workspace_bytes(int32_t nfield, int32_t dim, int32_t mode, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_pnn_inner_bwd(const float* g, int64_t ldg, int64_t gcol0, const float* x, int64_t ldx,
                                            int32_t nfield, int32_t dim, int32_t mode, const float* K, float* dx,
                                            int64_t lddx, float* dK, int64_t batch, void* workspace,
                                            size_t workspace_bytes, void* stream);

/* OutterProductLayer(kernel_type='mat') with the reference's kernel K [dim, P, dim], read in place:
 *   out[b*ldo + col0 + p] = sum_{k,l} x_j[k] K[k][p][l] x_i[l]
 * on the FEFM kernels' register-tiled products (no [B, dim] product reaches memory).  Backward from
 * g[b*ldg + gcol0 + p]:
 *   dx_i = g_p x_j K[:,p,:],   dx_j = g_p K[:,p,:] x_i   (pitch lddx, overwritten; may be NULL)
 *   dK[k][p][l] = sum_b g_p x_j[k] x_i[l]                ([dim, P, dim], overwritten; may be NULL)
 * Same ordering guarantees as b2ctr_fefm_bwd.  Limits: 2 <= nfield <= 64, 1 <= dim <= 64. */
B2CTR_API b2ctr_status_t b2ctr_pnn_outer_fwd(const float* x, int64_t ldx, int32_t nfield, int32_t dim, const float* K,
                                            float* out, int64_t ldo, int64_t col0, int64_t batch, void* stream);
B2CTR_API size_t b2ctr_pnn_outer_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_pnn_outer_bwd(const float* g, int64_t ldg, int64_t gcol0, const float* x, int64_t ldx,
                                            int32_t nfield, int32_t dim, const float* K, float* dx, int64_t lddx,
                                            float* dK, int64_t batch, void* workspace, size_t workspace_bytes,
                                            void* stream);

/* EDCN's BridgeModule (deepctr/layers/interaction.py:1502-1570) and RegulationModule (deepctr/layers/core.py:270-321)
 * in one pass over [B, nfield*dim].  Per element (b, f, e), from operands read in place through their own pitch:
 *   B2CTR_REGULATE_COPY       v = x                       (a RegulationModule on its own)
 *   B2CTR_REGULATE_ADD        v = x + h                   (bridge_type 'pointwise_addition')
 *   B2CTR_REGULATE_HADAMARD   v = x * h                   ('hadamard_product')
 *   B2CTR_REGULATE_ATTENTION  v = ax * x + ah * h         ('attention_pooling', ax / ah the two softmax DNNs)
 * and writes, each into the column window [col, col + nfield*dim) of a wider buffer and only where its pointer is
 * set: the bridge output u = v, and the gated outputs y_k = v * gate_k[f], gate_k = softmax_f(g_k * inv_tau_k)
 * (g_k the module's [1, nfield, 1] weight, inv_tau_k the reference's stored 1 / tau).  Every CTA forms the gates in
 * shared memory.  16-byte loads and stores when dim % 4 == 0 and every pointer and pitch allows, else a scalar path.
 * Backward (the same descriptor; u / y0 / y1 now address the incoming gradients du / dy0 / dy1, NULL = zero):
 * v is recomputed from the operands, dv = du + sum_k gate_k * dy_k, then by mode dx = dv (COPY, ADD) or dv * h
 * (HADAMARD) or dv * ax (ATTENTION), dh = dv (ADD) or dv * x (HADAMARD) or dv * ah, dax = dv * x, dah = dv * h.
 * dx is added to (dx_accumulate) or overwritten; dh / dax / dah are overwritten; any of them may be NULL.  dg_k
 * [nfield] = inv_tau_k * gate_k * (s_k - <gate_k, s_k>) with s_k[f] = sum_{b,e} v * dy_k: per-(field, batch
 * chunk) partials in the workspace, summed in chunk order, then the softmax Jacobian on the device.  Every element
 * has one owner, no float atomics: bit-identical from run to run.
 * Limits: 1 <= nfield <= 1024 (both gates in shared memory), 1 <= dim <= 256 (a field inside one backward column
 * tile), hence nfield*dim <= 262144; anything else is INVALID_ARG. */
enum { B2CTR_REGULATE_COPY = 0, B2CTR_REGULATE_ADD = 1, B2CTR_REGULATE_HADAMARD = 2, B2CTR_REGULATE_ATTENTION = 3 };
typedef struct b2ctr_regulate {
  int32_t mode, nfield, dim, dx_accumulate;
  int64_t batch;
  const float* x; int64_t ldx;
  const float* h; int64_t ldh;                   /* ADD, HADAMARD, ATTENTION */
  const float* ax; int64_t ldax;                 /* ATTENTION */
  const float* ah; int64_t ldah;                 /* ATTENTION */
  const float* g0; const float* g1;              /* [nfield] gate logits (a gate whose y is NULL is unused) */
  float inv_tau0, inv_tau1;
  float* u; int64_t ldu, ucol;                   /* forward outputs / backward incoming gradients */
  float* y0; int64_t ldy0, y0col;
  float* y1; int64_t ldy1, y1col;
  float* dx; int64_t lddx;                       /* backward outputs */
  float* dh; int64_t lddh;
  float* dax; int64_t lddax;
  float* dah; int64_t lddah;
  float* dg0; float* dg1;                        /* [nfield] */
} b2ctr_regulate_t;
B2CTR_API b2ctr_status_t b2ctr_regulate_fwd(const b2ctr_regulate_t* a, void* stream);
B2CTR_API size_t b2ctr_regulate_bwd_workspace_bytes(int32_t nfield, int32_t dim, int64_t batch);
B2CTR_API b2ctr_status_t b2ctr_regulate_bwd(const b2ctr_regulate_t* a, void* workspace, size_t workspace_bytes,
                                           void* stream);

/* CCPM's convolution stack (deepctr/models/ccpm.py:58-70) over a [B, rows, dim, channels] view, run per column.
 * Every stage keeps the embedding coordinate e apart, so each (sample, e) column is an independent 1-D signal over
 * the rows carrying C channels; the whole stack runs on chip per column and only the last map is written.  Stages:
 *   B2CTR_CONV_STAGE_CONV  Keras Conv2D with kernel (width, 1), strides (1, 1), padding 'same', channels_last:
 *                          out[r, co] = act(bias[co] + sum_{t, ci} in[r + t - pb, ci] * kernel[t, ci, co]), a
 *                          cross-correlation; rows outside [0, rows) read zero; pb = (width - 1) / 2 rows of padding
 *                          before and width - 1 - pb after (TF's 'same'; width may exceed rows).  kernel is Keras'
 *                          [width, 1, C_in, filters] as [width, C_in, filters]; bias [filters] or NULL.
 *   B2CTR_CONV_STAGE_KMAX  KMaxPooling(k) along the rows (deepctr/layers/sequence.py:818-874): per channel the k
 *                          largest values in descending order, equal values lower row first (tf.nn.top_k, sorted).
 * Element (r, e, c) of the input is x[b * ldx + xcol + (r * dim + e) * channels + c]; the last map [k, dim, C] is
 * written in Keras' Flatten order, (r * dim + e) * C + c from column outcol of a [B, ldout] buffer.
 * Backward (the same descriptor; `out` now addresses the incoming gradient): the forward is recomputed per column,
 * the gradient goes back through each k-max (to the selected rows only), activation and conv; dx is written (or
 * added, dx_accumulate) in x's layout from column dxcol of a [B, lddx] buffer (NULL: not wanted).  The weight
 * gradients dkernel / dbias (overwritten; NULL: not wanted) go through per-CTA partials in the workspace, each CTA
 * adding its columns in a fixed order, then summed in CTA order: no float atomics, bit-identical from run to run.
 * Nothing but the output is written by the forward, so the backward needs no saved state.
 * Limits: 1 <= nstage <= B2CTR_CONV_STACK_MAX_STAGES, 1 <= rows <= 64, 1 <= channels, filters <= 16,
 * 1 <= width <= 32, 1 <= k <= the rows it pools; and the backward's shared memory fits in 224 KB: 4 bytes times
 * 2 * W + 32 * (M + 2 * G), with W the conv weights and biases of all stages (kept with their gradient sums), M the
 * floats of every map of one column (the input, each conv output, each k-max output twice: values and rows) and G
 * the largest map (the gradient ping-pong).  Anything else is INVALID_ARG. */
enum { B2CTR_CONV_STAGE_CONV = 0, B2CTR_CONV_STAGE_KMAX = 1 };
#define B2CTR_CONV_STACK_MAX_STAGES 8
typedef struct b2ctr_conv_stage {
  int32_t kind, width, filters, act, k, reserved;  /* width / filters / act: CONV; k: KMAX */
  const float* kernel;                             /* [width, C_in, filters] */
  const float* bias;                               /* [filters] or NULL */
  float* dkernel; float* dbias;                    /* backward outputs or NULL */
} b2ctr_conv_stage_t;
typedef struct b2ctr_conv_stack {
  int32_t struct_size;                             /* sizeof(b2ctr_conv_stack_t) */
  int32_t nstage, rows, dim, channels, dx_accumulate;
  int64_t batch;
  const float* x; int64_t ldx, xcol;
  float* out; int64_t ldout, outcol;               /* forward output / backward incoming gradient */
  float* dx; int64_t lddx, dxcol;                  /* backward */
  b2ctr_conv_stage_t stage[B2CTR_CONV_STACK_MAX_STAGES];
} b2ctr_conv_stack_t;
B2CTR_API b2ctr_status_t b2ctr_conv_stack_fwd(const b2ctr_conv_stack_t* a, void* stream);
B2CTR_API size_t b2ctr_conv_stack_bwd_workspace_bytes(const b2ctr_conv_stack_t* a);
B2CTR_API b2ctr_status_t b2ctr_conv_stack_bwd(const b2ctr_conv_stack_t* a, void* workspace, size_t workspace_bytes,
                                             void* stream);

/* FLEN's FieldWiseBiInteraction (deepctr/layers/interaction.py:1224-1348) over G groups of fields read in place.
 * Field f (0 <= f < nfield) is the [dim] row at column col[f] of a [B, ldx] buffer and belongs to group
 * group[f]; the members of a group need not be adjacent.  Per sample and coordinate e, with
 * S_g = sum_{f in g} x_f and Q_g = sum_{f in g} x_f^2:
 *   h[e] = sum_{p = (g < h)} kernel_mf[p] * S_g * S_h + bias_mf  +  sum_g kernel_fm[g] * (S_g^2 - Q_g) + bias_fm
 * (pairs in itertools.combinations order, no 1/2 on the FM term, as in the reference).  S_g and Q_g live in
 * registers; only h is written, into the column window [outcol, outcol + dim) of a [B, ldout] buffer.
 * Backward (the same descriptor; `out` now addresses the incoming gradient dh): the forward is recomputed from x,
 *   dx_f = dh * (sum_{h != g} kernel_mf[p(g, h)] * S_h + 2 * kernel_fm[g] * (S_g - x_f))
 * written (or added, dx_accumulate) at column col[f] of a [B, lddx] buffer (NULL: not wanted), and
 *   dkernel_mf[p] = sum_{b, e} dh * S_g * S_h,  dkernel_fm[g] = sum_{b, e} dh * (S_g^2 - Q_g),
 *   dbias_mf = dbias_fm = sum_b dh,
 * each overwritten (NULL: not wanted), through per-CTA partials in the workspace summed in CTA order: no float
 * atomics, bit-identical from run to run.  The forward saves nothing.  bias_mf / bias_fm may be NULL (use_bias
 * False).  16-byte loads and stores when dim % 4 == 0 and every column, pitch and pointer allows, else a scalar
 * path.  Limits: 2 <= ngroup <= B2CTR_FWBI_MAX_GROUPS, every group non-empty, ngroup <= nfield <=
 * B2CTR_FWBI_MAX_FIELDS, 1 <= dim <= 256, 0 <= col[f] and col[f] + dim <= ldx < 2^31; anything else is INVALID_ARG. */
#define B2CTR_FWBI_MAX_FIELDS 256
#define B2CTR_FWBI_MAX_GROUPS 8
typedef struct b2ctr_field_wise_bi {
  int32_t struct_size;                             /* sizeof(b2ctr_field_wise_bi_t) */
  int32_t nfield, ngroup, dim, dx_accumulate, reserved;
  int64_t batch;
  const float* x; int64_t ldx;
  int64_t col[B2CTR_FWBI_MAX_FIELDS];              /* column of field f in a row of x (and of dx) */
  int32_t group[B2CTR_FWBI_MAX_FIELDS];            /* group of field f, 0 <= group < ngroup */
  const float* kernel_mf;                          /* [ngroup * (ngroup - 1) / 2] */
  const float* kernel_fm;                          /* [ngroup] */
  const float* bias_mf; const float* bias_fm;      /* [dim] or NULL */
  float* out; int64_t ldout, outcol;               /* forward output h / backward incoming gradient dh */
  float* dx; int64_t lddx;                         /* backward */
  float* dkernel_mf; float* dkernel_fm; float* dbias_mf; float* dbias_fm;
} b2ctr_field_wise_bi_t;
B2CTR_API b2ctr_status_t b2ctr_field_wise_bi_fwd(const b2ctr_field_wise_bi_t* a, void* stream);
B2CTR_API size_t b2ctr_field_wise_bi_bwd_workspace_bytes(const b2ctr_field_wise_bi_t* a);
B2CTR_API b2ctr_status_t b2ctr_field_wise_bi_bwd(const b2ctr_field_wise_bi_t* a, void* workspace,
                                                size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 6. Sequence operators (DIN, pooling, Dice / BatchNormalization, dropout)                     */
/* ------------------------------------------------------------------------------------------ */
/* LocalActivationUnit input (deepctr/layers/core.py:98-101): out[b,t] = [q, k, q-k, q*k] */
B2CTR_API b2ctr_status_t b2ctr_din_att_input_fwd(const float* q, int64_t ldq, const float* keys,
                                                int64_t ldk, float* out, int64_t batch, int32_t T,
                                                int32_t E, void* stream);
B2CTR_API b2ctr_status_t b2ctr_din_att_input_bwd(const float* q, int64_t ldq, const float* keys,
                                                int64_t ldk, const float* g, float* dq, float* dk,
                                                int64_t batch, int32_t T, int32_t E, void* stream);
/* AttentionSequencePoolingLayer tail (deepctr/layers/sequence.py:278-291): masked fill (0 or
 * -2^32+1 + softmax), then out = w @ keys (or the weights themselves when return_score).      */
B2CTR_API b2ctr_status_t b2ctr_din_pool_fwd(const float* score, const float* keys, int64_t ldk,
                                           const uint8_t* mask, float* w, float* out, int64_t batch,
                                           int32_t T, int32_t E, int32_t weight_norm,
                                           int32_t return_score, void* stream);
B2CTR_API b2ctr_status_t b2ctr_din_pool_bwd(const float* w, const float* keys, int64_t ldk,
                                           const uint8_t* mask, const float* dout, float* dscore,
                                           float* dkeys, int64_t batch, int32_t T, int32_t E,
                                           int32_t weight_norm, int32_t return_score, void* stream);
/* SequencePoolingLayer on a materialised [B,T,E] tensor (deepctr/layers/sequence.py:76-106);
 * mode = B2CTR_POOL_SUM/MEAN/MAX; validity from mask (uint8 [B,T], any non-zero byte is a valid
 * position, and mean divides by the number of valid positions) or len ([B]).                   */
B2CTR_API b2ctr_status_t b2ctr_seqpool_fwd(const float* x, const uint8_t* mask, const int32_t* len,
                                          float* out, int64_t batch, int32_t T, int32_t E,
                                          int32_t mode, void* stream);
B2CTR_API b2ctr_status_t b2ctr_seqpool_bwd(const float* x, const uint8_t* mask, const int32_t* len,
                                          const float* dout, float* dx, int64_t batch, int32_t T,
                                          int32_t E, int32_t mode, void* stream);
/* WeightedSequenceLayer (deepctr/layers/sequence.py:155-183): wt = masked [soft-maxed] weights;
 * seqscale: out[r, :] = x[r, :] * wt[r]                                                        */
B2CTR_API b2ctr_status_t b2ctr_seqweight(const float* w, const uint8_t* mask, const int32_t* len,
                                        float* wt, int64_t batch, int32_t T, int32_t normalize,
                                        void* stream);
B2CTR_API b2ctr_status_t b2ctr_seqscale(const float* x, const float* wt, float* out, int64_t rows,
                                       int32_t E, void* stream);
/* column mean / biased variance of x[m,n] -> stats[0:n], stats[n:2n] (deterministic two-pass) */
B2CTR_API size_t b2ctr_colstats_workspace_bytes(int64_t m, int64_t n);
B2CTR_API b2ctr_status_t b2ctr_colstats(const float* x, int64_t ld, int64_t m, int64_t n, float* stats,
                                       void* workspace, size_t workspace_bytes, void* stream);
B2CTR_API b2ctr_status_t b2ctr_moving_update(float* moving, const float* batch, float momentum,
                                            int64_t n, void* stream);
B2CTR_API b2ctr_status_t b2ctr_bn_apply(const float* x, const float* mean, const float* var,
                                       const float* gamma, const float* beta, float* y, int64_t m,
                                       int64_t n, float eps, void* stream);
B2CTR_API b2ctr_status_t b2ctr_bn_bwd(const float* x, const float* mean, const float* var,
                                     const float* gamma, const float* dy, float* dx, float* dgamma,
                                     float* dbeta, int64_t m, int64_t n, float eps, int32_t training,
                                     void* workspace, size_t workspace_bytes, void* stream);
/* Dice (deepctr/layers/activation.py:59-64): p = sigmoid(BN(x)); y = alpha*(1-p)*x + p*x */
B2CTR_API b2ctr_status_t b2ctr_dice_fwd(const float* x, const float* mean, const float* var,
                                       const float* alpha, float* y, int64_t m, int64_t n, float eps,
                                       void* stream);
B2CTR_API size_t b2ctr_dice_bwd_workspace_bytes(int64_t m, int64_t n);
B2CTR_API b2ctr_status_t b2ctr_dice_bwd(const float* x, const float* mean, const float* var,
                                       const float* alpha, const float* dy, float* dx, float* dalpha,
                                       int64_t m, int64_t n, float eps, int32_t training,
                                       void* workspace, size_t workspace_bytes, void* stream);
/* y = keep(seed, i) ? x / (1 - rate) : 0   (the backward applies the same call to dy) */
B2CTR_API b2ctr_status_t b2ctr_dropout(const float* x, float* y, int64_t n, float rate, uint64_t seed,
                                      void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 6b. Transformer layer of BST (deepctr/layers/sequence.py:431-651, layers/normalization.py:18-51) */
/* ------------------------------------------------------------------------------------------ */
/* Masked multi-head scaled-dot-product attention over [B, T, heads*d] (sequence.py:544-617).
 * Row r = b*T + t of Q / K / V starts at q + r*ldq (k + r*ldk, v + r*ldv); head h is columns [h*d, (h+1)*d).
 * For every (b, h, query i):
 *   s_j = scale * q_i . k_j;  s_j = -2^32 where key j is invalid, and on the diagonal j == i when blinding;
 *   p_j = softmax_j(s);  P_j = p_j * valid_q(i) * keep(i, j) / (1 - dropout_rate)
 *   out[r*ldo + h*d + c] = sum_j P_j v_j[c] (+ res[r*ldr + h*d + c] when res != NULL)
 * (a sample whose keys are all masked gets uniform 1/T weights before the query mask, as in the reference).
 * keep(i, j) is b2ctr_dropout's test on the element index ((h*B + b)*T + i)*T + j of the reference's
 * head-major [heads*B, T, T] layout; dropout_rate == 0 keeps everything.
 * Validity: t < qlen[b] (klen) when given, else qmask[b*T + t] != 0 (kmask) when given, else valid.
 * stats [B, heads, T, 2] = (max_j s_j, sum_j exp(s_j - max)) is all the backward needs: the [B, heads, T, T]
 * scores and probabilities never reach memory in either direction.
 * Backward: dq / dk / dv (pitches lddq / lddk / lddv, overwritten) from dout (pitch lddo); the residual's
 * gradient is dout itself.  One owner per element, terms added in a fixed order, no float atomics:
 * bit-identical from run to run.  Limits: 1 <= T <= 128, 1 <= d <= 64; anything else is INVALID_ARG. */
typedef struct b2ctr_mha {
  const float* q; int64_t ldq;
  const float* k; int64_t ldk;
  const float* v; int64_t ldv;
  const float* res; int64_t ldr;
  float* out; int64_t ldo;
  float* stats;
  const int32_t* qlen; const int32_t* klen;
  const uint8_t* qmask; const uint8_t* kmask;
  int64_t batch; int32_t T, heads, d;
  float scale; int32_t blinding; float dropout_rate; uint64_t seed;
  const float* dout; int64_t lddo;               /* backward only */
  float* dq; int64_t lddq;
  float* dk; int64_t lddk;
  float* dv; int64_t lddv;
} b2ctr_mha_t;
B2CTR_API b2ctr_status_t b2ctr_mha_fwd(const b2ctr_mha_t* a, void* stream);
B2CTR_API b2ctr_status_t b2ctr_mha_bwd(const b2ctr_mha_t* a, void* stream);

/* LayerNormalization (normalization.py:34-43) over the last axis of x = a (+ b), rows of n <= 1024 columns:
 *   mean = avg(x), var = avg((x - mean)^2), y = (x - mean) / sqrt(var + eps) * gamma + beta
 * gamma / beta may be NULL (scale / center off); b may be NULL.  stats [rows, 2] = (mean, 1/sqrt(var + eps)).
 * Backward: dx (pitch lddx, overwritten; the gradient of both summands), dgamma / dbeta [n] (overwritten, may be
 * NULL) through per-CTA partials in the workspace summed in CTA order: bit-identical from run to run. */
B2CTR_API b2ctr_status_t b2ctr_layernorm_fwd(const float* a, int64_t lda, const float* b, int64_t ldb,
                                            const float* gamma, const float* beta, float* y, int64_t ldy,
                                            float* stats, int64_t rows, int32_t n, float eps, void* stream);
B2CTR_API size_t b2ctr_layernorm_bwd_workspace_bytes(int64_t rows, int32_t n);
B2CTR_API b2ctr_status_t b2ctr_layernorm_bwd(const float* a, int64_t lda, const float* b, int64_t ldb,
                                            const float* gamma, const float* stats, const float* dy, int64_t lddy,
                                            float* dx, int64_t lddx, float* dgamma, float* dbeta, int64_t rows,
                                            int32_t n, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 7. Row-sharded embedding exchange (SURVEY.md 8e; new capability, no reference counterpart)     */
/*    row r of every table lives on rank r % world as local row r / world.                        */
/* ------------------------------------------------------------------------------------------ */
/* pass 1: counts[owner] += #lookups owned by `owner` (counts must be zero on entry);
 * slot[b*nfeat+f] = owner << 32 | rank-inside-the-owner's-bucket.  feats[f].{idx,idx_stride,idx_dtype}. */
B2CTR_API b2ctr_status_t b2ctr_shard_bucketize(const b2ctr_feature_t* feats, int32_t nfeat, int64_t batch,
                                              int32_t world, int32_t* counts, int64_t* slot, void* stream);
/* pass 2: keys grouped by owner (key = feature << 40 | local_row) and pos[b*nfeat+f] = index of that
 * lookup inside keys (= row of the answer in the buffer the owners send back).                    */
B2CTR_API b2ctr_status_t b2ctr_shard_fill(const b2ctr_feature_t* feats, int32_t nfeat, int64_t batch,
                                         int32_t world, const int32_t* counts, const int64_t* slot,
                                         int64_t* keys, int32_t* pos, void* stream);
/* owner: rows[i,:] = tables[f][row,:], lin_out[i] = lin_tables[f][row] for keys[i] = f << 40 | row */
B2CTR_API b2ctr_status_t b2ctr_shard_gather_rows(float* const* tables, float* const* lin_tables,
                                                int32_t nfeat, int32_t dim, const int64_t* keys, int64_t n,
                                                float* rows, float* lin_out, void* stream);
/* owner, backward: tables[f][row,:] += scale * grows[i,:]; lin_tables[f][row] += lin_scale * glin[i] */
B2CTR_API b2ctr_status_t b2ctr_shard_scatter_rows(float* const* tables, float* const* lin_tables,
                                                 int32_t nfeat, int32_t dim, const int64_t* keys, int64_t n,
                                                 const float* grows, const float* glin, float scale,
                                                 float lin_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2CTR_H_ */
