// tower.cu — the relu layers of a DNN tower after its first layer, as one fused forward and one fused backward
// kernel.  Both weight matrices (split into bf16 hi/lo) stay in shared memory, each warp owns 16 rows at a time,
// and one layer's mma.sync accumulators become the next layer's A fragments in registers: the intermediate
// activations and gradients only ever leave the SM as the bf16 operand planes the weight-gradient GEMMs read.
#include <cuda_bf16.h>
#include "common.cuh"

namespace b2ctr {
namespace {

typedef __nv_bfloat16 bf16;
constexpr int kTowerWarps = 8;
constexpr int kTowerThreads = kTowerWarps * 32;

__host__ __device__ constexpr int cols_pad(int w) { return w <= 64 ? 64 : (w + 127) / 128 * 128; }   // planes_cols_pad

struct TowerFwd {
  const float* y0;            // [batch, N0]
  const float* w1; const float* b1;
  const float* w2; const float* b2;
  bf16* p0; bf16* p1;         // planes of y0, of y1 (N2 > 0)
  float* ylast;               // [batch, N2 ? N2 : N1]
  int64_t batch, rows_pad;
};
struct TowerBwd {
  const float* dy;            // [batch, NL]: gradient of the last layer's output
  const float* ylast;         // [batch, NL]
  const float* y0;            // [batch, N0]
  const bf16* p1;             // planes of y1 (N2 > 0): its relu mask
  const float* w1; const float* w2;
  bf16* dz0; bf16* dz1; bf16* dz2;   // planes
  float* partial;             // [gridDim.x, N0 + N1 + N2]
  int64_t batch, rows_pad;
};

__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// hi = bf16_rn(v), lo = bf16_rn(v - hi) of two consecutive columns: the values b2ctr_split_planes writes
struct Split2 { uint32_t hi, lo; };
__device__ __forceinline__ Split2 split2(float x, float y) {
  const bf16 hx = __float2bfloat16_rn(x), hy = __float2bfloat16_rn(y);
  return {pack_bf16(hx, hy), pack_bf16(__float2bfloat16_rn(x - __bfloat162float(hx)),
                                       __float2bfloat16_rn(y - __bfloat162float(hy)))};
}

// relu(acc + b) with the add flushing denormals to zero: a positive result is then a normal number, whose bf16 hi
// part is nonzero.  So "hi plane element != 0" is exactly "y > 0", and the backward reads y's relu mask from its
// hi plane instead of an fp32 copy of y.
__device__ __forceinline__ float relu_bias(float acc, float b) {
  float v;
  asm("add.ftz.f32 %0, %1, %2;" : "=f"(v) : "f"(acc), "f"(b));
  return v > 0.f ? v : 0.f;
}

__device__ __forceinline__ float2 ld2(const float* p, bool ok) {
  return ok ? __ldg(reinterpret_cast<const float2*>(p)) : make_float2(0.f, 0.f);
}

// Stores a warp's [16 rows x 16 columns] block of one bf16 plane, columns c0 .. c0 + 15, rows ra (= r0 + g) and
// rb = ra + 8.  Lane (g, t) holds the column pairs 2t, 2t + 1 (a: row ra, b: row rb) and 8 + 2t, 9 + 2t (c: ra,
// d: rb).  A 4 x 4 transpose inside each lane quad gives lane t eight consecutive columns, so every store is 16 bytes
// and a warp's store fills whole 32-byte sectors: the 4-byte stores straight from the fragments cost the kernels
// about half their time.
__device__ __forceinline__ void st_chunk(bf16* plane, int64_t cp, int64_t ra, int c0, uint32_t a, uint32_t b,
                                         uint32_t c, uint32_t d, int t) {
  const int quad = threadIdx.x & 28;
  uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = (t - r) & 3, src = (t + r) & 3;          // send piece t of the quad lane that will ask for it
    const uint32_t send = i == 0 ? a : i == 1 ? c : i == 2 ? b : d;
    const uint32_t v = __shfl_sync(0xffffffffu, send, quad | src);
    o0 = src == 0 ? v : o0;
    o1 = src == 1 ? v : o1;
    o2 = src == 2 ? v : o2;
    o3 = src == 3 ? v : o3;
  }
  *reinterpret_cast<uint4*>(plane + (ra + (t >> 1) * 8) * cp + c0 + (t & 1) * 8) = make_uint4(o0, o1, o2, o3);
}

// acc[NT][4] += A[16 x 16 at k0] * B[k0 .. k0+16, NT*8 columns] in split-bf16 (hi*hi + hi*lo + lo*hi).
// B is stored n-major in shared memory, [n][P] with P = K + 8 (conflict-free fragment loads).
template <int NT, int P>
__device__ __forceinline__ void mma_k16(float (&acc)[NT][4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                        const bf16* sh, const bf16* sl, int k0, int g, int t) {
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int o = (j * 8 + g) * P + k0 + 2 * t;
    const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(sh + o), bh1 = *reinterpret_cast<const uint32_t*>(sh + o + 8);
    const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(sl + o), bl1 = *reinterpret_cast<const uint32_t*>(sl + o + 8);
    mma_bf16(acc[j], ah, bh0, bh1);
    mma_bf16(acc[j], ah, bl0, bl1);
    mma_bf16(acc[j], al, bh0, bh1);
  }
}

// W [K][N] row-major (fp32, global) -> shared hi/lo planes; transposed: [N][K + 8], else [K][N + 8]
template <int K, int N, bool kTrans>
__device__ __forceinline__ void stage_weight(const float* __restrict__ w, bf16* sh, bf16* sl) {
  for (int i = threadIdx.x; i < K * N; i += kTowerThreads) {
    const int k = i / N, n = i - k * N;
    const float v = __ldg(w + i);
    const bf16 h = __float2bfloat16_rn(v);
    const int o = kTrans ? n * (K + 8) + k : k * (N + 8) + n;
    sh[o] = h;
    sl[o] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

// pad columns [W, CP) of a warp's 16 plane rows are zero, as in b2ctr_split_planes
template <int W>
__device__ __forceinline__ void zero_pad_cols(bf16* hi, bf16* lo, int64_t r0, int lane) {
  constexpr int CP = cols_pad(W), V = (CP - W) / 8;
  if constexpr (V > 0) {
    for (int i = lane; i < 16 * V; i += 32) {
      const int64_t o = (r0 + i / V) * CP + W + (i % V) * 8;
      *reinterpret_cast<uint4*>(hi + o) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(lo + o) = make_uint4(0, 0, 0, 0);
    }
  }
}

// Column sums of a [16 x 8] accumulator tile (rows ra, rb of this thread: v[0..1], v[2..3]) into the warp's
// shared partial at column c: fixed shuffle order, one writer per column.
__device__ __forceinline__ void colsum_add(float* red, int c, float v0, float v1, int g) {
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    v0 += __shfl_xor_sync(0xffffffffu, v0, o);
    v1 += __shfl_xor_sync(0xffffffffu, v1, o);
  }
  if (g == 0) {
    red[c] += v0;
    red[c + 1] += v1;
  }
}

template <int N0, int N1, int N2>
constexpr size_t tower_smem_bytes(bool bwd) {
  return bwd ? ((size_t)N0 * (N1 + 8) + (size_t)N1 * (N2 + 8)) * 2 * sizeof(bf16) +
                   (size_t)kTowerWarps * (N0 + N1 + N2) * sizeof(float)
             : ((size_t)N1 * (N0 + 8) + (size_t)N2 * (N1 + 8)) * 2 * sizeof(bf16);
}

// y1 = relu(y0 W1 + b1) [, y2 = relu(y1 W2 + b2)]; writes the planes of y0 [and y1] and the last output in fp32
template <int N0, int N1, int N2>
__global__ void __launch_bounds__(kTowerThreads, 1) mlp_relu_fwd_kernel(const TowerFwd p) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int P1 = N0 + 8, P2 = N1 + 8, CP0 = cols_pad(N0), CP1 = cols_pad(N1);
  bf16* w1h = reinterpret_cast<bf16*>(smem);
  bf16* w1l = w1h + N1 * P1;
  bf16* w2h = w1l + N1 * P1;
  bf16* w2l = w2h + N2 * P2;
  stage_weight<N0, N1, true>(p.w1, w1h, w1l);
  if constexpr (N2 > 0) stage_weight<N1, N2, true>(p.w2, w2h, w2l);
  __syncthreads();

  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  bf16* p0l = p.p0 + p.rows_pad * CP0;
  const int64_t tiles = p.rows_pad / 16;
  for (int64_t tile = (int64_t)blockIdx.x * kTowerWarps + (threadIdx.x >> 5); tile < tiles;
       tile += (int64_t)gridDim.x * kTowerWarps) {
    const int64_t r0 = tile * 16, ra = r0 + g, rb = ra + 8;
    const bool va = ra < p.batch, vb = rb < p.batch;
    float acc1[N1 / 8][4];
#pragma unroll
    for (int j = 0; j < N1 / 8; ++j) acc1[j][0] = acc1[j][1] = acc1[j][2] = acc1[j][3] = 0.f;
#pragma unroll 4
    for (int kc = 0; kc < N0 / 16; ++kc) {
      const int c = kc * 16 + 2 * t;
      const float2 x0 = ld2(p.y0 + ra * N0 + c, va), x1 = ld2(p.y0 + rb * N0 + c, vb);
      const float2 x2 = ld2(p.y0 + ra * N0 + c + 8, va), x3 = ld2(p.y0 + rb * N0 + c + 8, vb);
      const Split2 s0 = split2(x0.x, x0.y), s1 = split2(x1.x, x1.y), s2 = split2(x2.x, x2.y), s3 = split2(x3.x, x3.y);
      const uint32_t ah[4] = {s0.hi, s1.hi, s2.hi, s3.hi}, al[4] = {s0.lo, s1.lo, s2.lo, s3.lo};
      st_chunk(p.p0, CP0, ra, kc * 16, s0.hi, s1.hi, s2.hi, s3.hi, t);
      st_chunk(p0l, CP0, ra, kc * 16, s0.lo, s1.lo, s2.lo, s3.lo, t);
      mma_k16<N1 / 8, P1>(acc1, ah, al, w1h, w1l, kc * 16, g, t);
    }
    zero_pad_cols<N0>(p.p0, p0l, r0, lane);

    if constexpr (N2 == 0) {
#pragma unroll
      for (int j = 0; j < N1 / 8; ++j) {
        const int c = j * 8 + 2 * t;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.b1 + c));
        if (va) *reinterpret_cast<float2*>(p.ylast + ra * N1 + c) =
                    make_float2(relu_bias(acc1[j][0], b.x), relu_bias(acc1[j][1], b.y));
        if (vb) *reinterpret_cast<float2*>(p.ylast + rb * N1 + c) =
                    make_float2(relu_bias(acc1[j][2], b.x), relu_bias(acc1[j][3], b.y));
      }
    } else {
      // y1 -> A fragments of layer 2 (the m16n8 accumulator layout of two adjacent column tiles is the m16k16 A
      // layout) and its planes; pad rows of the planes stay zero
      bf16* p1l = p.p1 + p.rows_pad * CP1;
      uint32_t a2h[N1 / 16][4], a2l[N1 / 16][4];
      Split2 pa, pb;                // the even column tile of the current 16-column chunk
#pragma unroll
      for (int j = 0; j < N1 / 8; ++j) {
        const int c = j * 8 + 2 * t;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.b1 + c));
        const Split2 sa = va ? split2(relu_bias(acc1[j][0], b.x), relu_bias(acc1[j][1], b.y)) : Split2{0u, 0u};
        const Split2 sb = vb ? split2(relu_bias(acc1[j][2], b.x), relu_bias(acc1[j][3], b.y)) : Split2{0u, 0u};
        a2h[j / 2][(j & 1) * 2] = sa.hi; a2h[j / 2][(j & 1) * 2 + 1] = sb.hi;
        a2l[j / 2][(j & 1) * 2] = sa.lo; a2l[j / 2][(j & 1) * 2 + 1] = sb.lo;
        if (j & 1) {
          st_chunk(p.p1, CP1, ra, (j / 2) * 16, pa.hi, pb.hi, sa.hi, sb.hi, t);
          st_chunk(p1l, CP1, ra, (j / 2) * 16, pa.lo, pb.lo, sa.lo, sb.lo, t);
        } else {
          pa = sa, pb = sb;
        }
      }
      zero_pad_cols<N1>(p.p1, p1l, r0, lane);
      float acc2[N2 / 8][4];
#pragma unroll
      for (int j = 0; j < N2 / 8; ++j) acc2[j][0] = acc2[j][1] = acc2[j][2] = acc2[j][3] = 0.f;
#pragma unroll
      for (int kc = 0; kc < N1 / 16; ++kc) mma_k16<N2 / 8, P2>(acc2, a2h[kc], a2l[kc], w2h, w2l, kc * 16, g, t);
#pragma unroll
      for (int j = 0; j < N2 / 8; ++j) {
        const int c = j * 8 + 2 * t;
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.b2 + c));
        if (va) *reinterpret_cast<float2*>(p.ylast + ra * N2 + c) =
                    make_float2(relu_bias(acc2[j][0], b.x), relu_bias(acc2[j][1], b.y));
        if (vb) *reinterpret_cast<float2*>(p.ylast + rb * N2 + c) =
                    make_float2(relu_bias(acc2[j][2], b.x), relu_bias(acc2[j][3], b.y));
      }
    }
  }
}

// dz_last = dy * [y_last > 0]; [dz1 = (dz2 W2^T) * [y1 > 0];]  dz0 = (dz1 W1^T) * [y0 > 0].  Writes the planes of every
// dz and per-CTA column sums of each (the bias gradients, reduced by tower_bias_reduce_kernel).
template <int N0, int N1, int N2>
__global__ void __launch_bounds__(kTowerThreads, 1) mlp_relu_bwd_kernel(const TowerBwd p) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int NL = N2 ? N2 : N1, NT = N0 + N1 + N2;
  constexpr int P1 = N1 + 8, P2 = N2 + 8, CP0 = cols_pad(N0), CP1 = cols_pad(N1), CPL = cols_pad(NL);
  constexpr int NC = 32;                     // dz0 is produced in column chunks of NC (registers)
  bf16* w1h = reinterpret_cast<bf16*>(smem);
  bf16* w1l = w1h + N0 * P1;
  bf16* w2h = w1l + N0 * P1;
  bf16* w2l = w2h + N1 * P2;
  float* red_all = reinterpret_cast<float*>(w2l + N1 * P2);
  stage_weight<N0, N1, false>(p.w1, w1h, w1l);
  if constexpr (N2 > 0) stage_weight<N1, N2, false>(p.w2, w2h, w2l);
  for (int i = threadIdx.x; i < kTowerWarps * NT; i += kTowerThreads) red_all[i] = 0.f;
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  float* red = red_all + warp * NT;     // columns: dz0 [0, N0), dz1 [N0, N0 + N1), dz2 [N0 + N1, NT)
  bf16* dzl = N2 ? p.dz2 : p.dz1;
  bf16* dzl_lo = dzl + p.rows_pad * CPL;
  bf16* dz0l = p.dz0 + p.rows_pad * CP0;
  const int64_t tiles = p.rows_pad / 16;
  for (int64_t tile = (int64_t)blockIdx.x * kTowerWarps + warp; tile < tiles; tile += (int64_t)gridDim.x * kTowerWarps) {
    const int64_t r0 = tile * 16, ra = r0 + g, rb = ra + 8;
    const bool va = ra < p.batch, vb = rb < p.batch;

    // last layer: dz from dy and the fp32 output, as A fragments of the next product
    uint32_t alh[NL / 16][4], all[NL / 16][4];
    Split2 pa, pb;                  // the even column tile of the current 16-column chunk
#pragma unroll
    for (int j = 0; j < NL / 8; ++j) {
      const int c = j * 8 + 2 * t;
      const float2 da = ld2(p.dy + ra * NL + c, va), db = ld2(p.dy + rb * NL + c, vb);
      const float2 ya = ld2(p.ylast + ra * NL + c, va), yb = ld2(p.ylast + rb * NL + c, vb);
      const float z0 = da.x * (ya.x > 0.f ? 1.f : 0.f), z1 = da.y * (ya.y > 0.f ? 1.f : 0.f);
      const float z2 = db.x * (yb.x > 0.f ? 1.f : 0.f), z3 = db.y * (yb.y > 0.f ? 1.f : 0.f);
      const Split2 sa = split2(z0, z1), sb = split2(z2, z3);
      alh[j / 2][(j & 1) * 2] = sa.hi; alh[j / 2][(j & 1) * 2 + 1] = sb.hi;
      all[j / 2][(j & 1) * 2] = sa.lo; all[j / 2][(j & 1) * 2 + 1] = sb.lo;
      if (j & 1) {
        st_chunk(dzl, CPL, ra, (j / 2) * 16, pa.hi, pb.hi, sa.hi, sb.hi, t);
        st_chunk(dzl_lo, CPL, ra, (j / 2) * 16, pa.lo, pb.lo, sa.lo, sb.lo, t);
      } else {
        pa = sa, pb = sb;
      }
      colsum_add(red, N0 + (N2 ? N1 : 0) + c, z0 + z2, z1 + z3, g);
    }
    zero_pad_cols<NL>(dzl, dzl_lo, r0, lane);

    // A fragments of dz1
    uint32_t a1h[N1 / 16][4], a1l[N1 / 16][4];
    if constexpr (N2 == 0) {
#pragma unroll
      for (int kc = 0; kc < N1 / 16; ++kc)
#pragma unroll
        for (int q = 0; q < 4; ++q) a1h[kc][q] = alh[kc][q], a1l[kc][q] = all[kc][q];
    } else {
      float acc[N1 / 8][4];
#pragma unroll
      for (int j = 0; j < N1 / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
      for (int kc = 0; kc < N2 / 16; ++kc) mma_k16<N1 / 8, P2>(acc, alh[kc], all[kc], w2h, w2l, kc * 16, g, t);
      const bf16* y1h = p.p1;
      bf16* dz1l = p.dz1 + p.rows_pad * CP1;
#pragma unroll
      for (int j = 0; j < N1 / 8; ++j) {
        const int c = j * 8 + 2 * t;
        // relu mask of y1 from its hi plane (see relu_bias); pad rows there are zero
        uint32_t ma, mb;              // volatile: loaded next to their use, not all hoisted over the chunk
        asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(ma) : "l"(y1h + ra * CP1 + c));
        asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(mb) : "l"(y1h + rb * CP1 + c));
        const float z0 = acc[j][0] * ((ma & 0xffffu) ? 1.f : 0.f), z1 = acc[j][1] * ((ma >> 16) ? 1.f : 0.f);
        const float z2 = acc[j][2] * ((mb & 0xffffu) ? 1.f : 0.f), z3 = acc[j][3] * ((mb >> 16) ? 1.f : 0.f);
        const Split2 sa = split2(z0, z1), sb = split2(z2, z3);
        a1h[j / 2][(j & 1) * 2] = sa.hi; a1h[j / 2][(j & 1) * 2 + 1] = sb.hi;
        a1l[j / 2][(j & 1) * 2] = sa.lo; a1l[j / 2][(j & 1) * 2 + 1] = sb.lo;
        if (j & 1) {
          st_chunk(p.dz1, CP1, ra, (j / 2) * 16, pa.hi, pb.hi, sa.hi, sb.hi, t);
          st_chunk(dz1l, CP1, ra, (j / 2) * 16, pa.lo, pb.lo, sa.lo, sb.lo, t);
        } else {
          pa = sa, pb = sb;
        }
        colsum_add(red, N0 + c, z0 + z2, z1 + z3, g);
      }
      zero_pad_cols<N1>(p.dz1, dz1l, r0, lane);
    }

    // dz0 = (dz1 W1^T) * [y0 > 0], NC columns at a time
#pragma unroll 1
    for (int n0 = 0; n0 < N0; n0 += NC) {
      float acc[NC / 8][4];
#pragma unroll
      for (int j = 0; j < NC / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
      for (int kc = 0; kc < N1 / 16; ++kc)
        mma_k16<NC / 8, P1>(acc, a1h[kc], a1l[kc], w1h + n0 * P1, w1l + n0 * P1, kc * 16, g, t);
#pragma unroll
      for (int j = 0; j < NC / 8; ++j) {
        const int c = n0 + j * 8 + 2 * t;
        const float2 ya = ld2(p.y0 + ra * N0 + c, va), yb = ld2(p.y0 + rb * N0 + c, vb);
        const float z0 = acc[j][0] * (ya.x > 0.f ? 1.f : 0.f), z1 = acc[j][1] * (ya.y > 0.f ? 1.f : 0.f);
        const float z2 = acc[j][2] * (yb.x > 0.f ? 1.f : 0.f), z3 = acc[j][3] * (yb.y > 0.f ? 1.f : 0.f);
        const Split2 sa = split2(z0, z1), sb = split2(z2, z3);
        if (j & 1) {
          st_chunk(p.dz0, CP0, ra, n0 + (j / 2) * 16, pa.hi, pb.hi, sa.hi, sb.hi, t);
          st_chunk(dz0l, CP0, ra, n0 + (j / 2) * 16, pa.lo, pb.lo, sa.lo, sb.lo, t);
        } else {
          pa = sa, pb = sb;
        }
        colsum_add(red, c, z0 + z2, z1 + z3, g);
      }
    }
    zero_pad_cols<N0>(p.dz0, dz0l, r0, lane);
  }

  __syncthreads();
  for (int c = threadIdx.x; c < NT; c += kTowerThreads) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kTowerWarps; ++w) s += red_all[w * NT + c];
    p.partial[(int64_t)blockIdx.x * NT + c] = s;
  }
}

// db_i[c] = sum of the CTAs' partials, in CTA order
__global__ void __launch_bounds__(128)
    tower_bias_reduce_kernel(const float* __restrict__ partial, int nblocks, int n0, int n1, int n2, float* db0,
                             float* db1, float* db2) {
  const int nt = n0 + n1 + n2, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nt) return;
  float s = 0.f;
  for (int b = 0; b < nblocks; ++b) s += partial[(int64_t)b * nt + c];
  if (c < n0) db0[c] = s;
  else if (c < n0 + n1) db1[c - n0] = s;
  else db2[c - n0 - n1] = s;
}

int tower_grid(int64_t rows_pad) {
  const int64_t need = ceil_div(rows_pad / 16, kTowerWarps);
  return (int)(need < kNumSMs ? need : kNumSMs);
}

template <typename Kern>
b2ctr_status_t launch_tower(Kern kern, size_t smem, int grid, cudaStream_t st, const void* args, const char* name) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    set_error("%s: cannot reserve %zu bytes of shared memory: %s", name, smem, cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  void* argv[] = {const_cast<void*>(args)};
  e = cudaLaunchKernel((const void*)kern, dim3(grid), dim3(kTowerThreads), argv, smem, st);
  if (e != cudaSuccess) {
    set_error("%s: CUDA launch failed: %s", name, cudaGetErrorString(e));
    return B2CTR_ERR_CUDA;
  }
  count_launch();
  return B2CTR_OK;
}

// The supported towers: (N0, N1, N2), N2 = 0 for two hidden layers.  Each one's A fragments and accumulators fit
// the registers of 8 warps per SM, and its weight planes fit shared memory.  Every width is at least 64: the
// split-K weight-gradient GEMM reads a dz narrower than 32 columns only in fp32, which these kernels never write.
#define B2_TOWERS(X) X(256, 128, 64) X(128, 128, 64) X(256, 128, 0) X(128, 64, 0)

bool tower_widths(const int32_t* widths, int32_t nlayers, int* n) {
  if (!widths || nlayers < 2 || nlayers > 3) return false;
  n[0] = widths[0];
  n[1] = widths[1];
  n[2] = nlayers == 3 ? widths[2] : 0;
#define B2_MATCH(a, b, c) if (n[0] == a && n[1] == b && n[2] == c) return true;
  B2_TOWERS(B2_MATCH)
#undef B2_MATCH
  return false;
}

}  // namespace
}  // namespace b2ctr

using namespace b2ctr;

extern "C" {

int32_t b2ctr_mlp_relu_supported(const int32_t* widths, int32_t nlayers) {
  int n[3];
  return tower_widths(widths, nlayers, n) ? 1 : 0;
}

b2ctr_status_t b2ctr_mlp_relu_fwd(const float* y0, const float* const* w, const float* const* b, void* const* planes,
                                  float* y_last, const int32_t* widths, int32_t nlayers, int64_t batch, void* stream) {
  int n[3];
  B2_REQUIRE(tower_widths(widths, nlayers, n), "mlp_relu_fwd: unsupported tower widths");
  B2_REQUIRE(y0 && w && b && planes && y_last && batch > 0, "mlp_relu_fwd: bad arguments");
  B2_REQUIRE(w[0] && b[0] && planes[0] && (n[2] == 0 || (w[1] && b[1] && planes[1])), "mlp_relu_fwd: NULL operand");
  TowerFwd p{y0, w[0], b[0], n[2] ? w[1] : nullptr, n[2] ? b[1] : nullptr, (bf16*)planes[0],
             n[2] ? (bf16*)planes[1] : nullptr, y_last, batch, planes_rows_pad(batch)};
  const int grid = tower_grid(p.rows_pad);
#define B2_FWD(a, b_, c)                                                                                     \
  if (n[0] == a && n[1] == b_ && n[2] == c)                                                                  \
    return launch_tower(mlp_relu_fwd_kernel<a, b_, c>, tower_smem_bytes<a, b_, c>(false), grid, (cudaStream_t)stream, \
                        &p, "b2ctr_mlp_relu_fwd");
  B2_TOWERS(B2_FWD)
#undef B2_FWD
  return B2CTR_ERR_INVALID_ARG;
}

size_t b2ctr_mlp_relu_bwd_workspace_bytes(const int32_t* widths, int32_t nlayers) {
  int n[3];
  if (!tower_widths(widths, nlayers, n)) return 0;
  return (size_t)kNumSMs * (n[0] + n[1] + n[2]) * sizeof(float);
}

b2ctr_status_t b2ctr_mlp_relu_bwd(const float* dy_last, const float* y_last, const float* y0, void* const* planes,
                                  const float* const* w, void* const* dz_planes, float* const* dbias,
                                  const int32_t* widths, int32_t nlayers, int64_t batch, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  int n[3];
  B2_REQUIRE(tower_widths(widths, nlayers, n), "mlp_relu_bwd: unsupported tower widths");
  B2_REQUIRE(dy_last && y_last && y0 && w && dz_planes && dbias && batch > 0, "mlp_relu_bwd: bad arguments");
  const int L = nlayers;
  for (int i = 0; i < L; ++i) B2_REQUIRE(dz_planes[i] && dbias[i], "mlp_relu_bwd: NULL output");
  B2_REQUIRE(w[0] && (n[2] == 0 || (w[1] && planes && planes[1])), "mlp_relu_bwd: NULL operand");
  const size_t need = b2ctr_mlp_relu_bwd_workspace_bytes(widths, nlayers);
  if (!workspace || workspace_bytes < need) {
    set_error("mlp_relu_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return B2CTR_ERR_WORKSPACE;
  }
  TowerBwd p{dy_last, y_last, y0, n[2] ? (const bf16*)planes[1] : nullptr, w[0], n[2] ? w[1] : nullptr,
             (bf16*)dz_planes[0], (bf16*)dz_planes[1], n[2] ? (bf16*)dz_planes[2] : nullptr, (float*)workspace,
             batch, planes_rows_pad(batch)};
  const int grid = tower_grid(p.rows_pad);
  b2ctr_status_t s = B2CTR_ERR_INVALID_ARG;
#define B2_BWD(a, b_, c)                                                                                     \
  if (n[0] == a && n[1] == b_ && n[2] == c)                                                                  \
    s = launch_tower(mlp_relu_bwd_kernel<a, b_, c>, tower_smem_bytes<a, b_, c>(true), grid, (cudaStream_t)stream, \
                     &p, "b2ctr_mlp_relu_bwd");
  B2_TOWERS(B2_BWD)
#undef B2_BWD
  if (s != B2CTR_OK) return s;
  const int nt = n[0] + n[1] + n[2];
  tower_bias_reduce_kernel<<<(unsigned)ceil_div(nt, 128), 128, 0, (cudaStream_t)stream>>>(
      (const float*)workspace, grid, n[0], n[1], n[2], dbias[0], dbias[1], n[2] ? dbias[2] : nullptr);
  B2_CHECK_LAUNCH("b2ctr_mlp_relu_bwd(reduce)");
  return B2CTR_OK;
}

}  // extern "C"
