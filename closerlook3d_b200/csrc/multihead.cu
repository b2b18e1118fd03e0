// multihead.cu -- the fused multi-shape part-segmentation head (sm_90a).
//
// Replaces the S heads of MultiPartSegHeadResNet (models/heads/segmentation_head.py:80-149), which the reference runs
// one after the other over every point of the batch:
//     y_s = W1_s x,  z_s = relu(BN_s(y_s)),  logits_s = W2_s z_s + b2_s        x (B,C,N), P = B*N points.
// The reference materialises y_s and z_s, (B,C,N) each, for every head (17 x 2 x 23 MB at PartNet's shape) and
// runs ~10 launches per head forward and backward.  Here nothing of size S*C*P reaches HBM:
//
//   forward  mh_prep     zero-padded (and transposed) copies of the weights, CE = padded width (16..128)
//            mh_moments  training: per-CTA sum(x - s) and sum (x - s)(x - s)^T with s = x[0,:,0] (a data point, so
//                        the shifted moments do not cancel catastrophically), reduced by cl3d_reduce_partials
//            mh_stats    one CTA per head: mean_s = W1_s xbar, var_s[c] = w_sc^T Cov w_sc (double), the running
//                        statistics update of nn.BatchNorm1d; eval: running statistics.  It folds BatchNorm into a
//                        scale/shift on y' = W1_s (x - ref): ref = xbar in training, s in eval, so the large common
//                        offset of x never enters a subtraction of two large numbers.
//            mh_fwd      tile of 128 points of x in shared memory; per head: y' (registers), z -> shared memory,
//                        logits -> HBM (coalesced along N).
//   backward mh_bwd_a    head-major (grid chunks x S): y' and z again, the ReLU mask bits (S*CE bits per point),
//                        gy = (W2^T dL) . mask, per-CTA partials of G = sum gy (x - ref)^T, sum gy, dW2, db2
//            mh_bwd_fin  one CTA per head: dgamma, dbeta, dW1 from G and the second moments (the BatchNorm
//                        batch-statistic terms are algebraic: dy = sc*gy - u0 - k*(y' + c0)), and k, u0
//            mh_bwd_mx   M = sum_s W1_s^T diag(k_s) W1_s, v0 = sum_s W1_s^T (u0_s + k_s c0_s)
//            mh_bwd_dx   tile-major: dx = sum_s W1_s^T (sc_s * gy_s) - M (x - ref) - v0, gy rebuilt from the mask
//                        bits (no recomputation of y), accumulated over the heads in registers, written once.
// Arithmetic is fp32 FFMA (register-blocked, 4 points x CE/8 rows per thread); reductions over points are per-CTA
// partials summed in a fixed order: no float atomics, repeat runs are bit-identical.
// x, the logits, d/dlogits and d/dx may be fp16 or bf16 (template parameter T of the kernels that touch them): they
// are widened exactly where they are loaded and rounded once where they are stored; everything else stays fp32.
#include <string.h>

#include "common.cuh"

namespace cl3d {

constexpr int kMhT = 128;        // points per tile
constexpr int kMhTS = kMhT + 4;  // shared-memory row stride (float4-aligned, staggers banks between rows)
constexpr int kMhThreads = 256;
constexpr int kMhMaxParts = CL3D_MHEAD_MAX_PARTS;

struct MhArgs {
  int S, C, NPT;
  int np[CL3D_MHEAD_MAX_HEADS];
  int off[CL3D_MHEAD_MAX_HEADS + 1];
  const void* g[CL3D_MHEAD_MAX_HEADS];  // d/dlogits in the boundary type T of the backward kernels
  float* rm[CL3D_MHEAD_MAX_HEADS];
  float* rv[CL3D_MHEAD_MAX_HEADS];
  long long* nbt[CL3D_MHEAD_MAX_HEADS];
};

template <int CE>
struct MhCfg {
  static constexpr int R = CE / 8;            // rows per warp in the row products
  static constexpr int MT = (CE + 15) / 16;   // micro-tile of the point-reduction products (16 x 16 threads)
  static constexpr int RS = 16 * MT;          // rows allocated for operands of the point-reduction products
  static constexpr int CW = (CE + 31) / 32;   // mask words per point and head
};

// save layout (floats): per head [mean | invstd | sc | sh | c0] (5C) | ref (C) | shift (C) | m1 (C) | M2 (C*C)
__host__ __device__ inline size_t mh_ref_off(int S, int C) { return (size_t)5 * S * C; }

// ---- boundary loads and stores ----------------------------------------------------------------------
// read-only element load, widened to fp32 (exact)
__device__ __forceinline__ float mh_ldg(const float* p) { return __ldg(p); }
__device__ __forceinline__ float mh_ldg(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float mh_ldg(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }

// o[0..3] = v0..v3, rounded once to the element type: one 16-byte store for fp32, one 8-byte store for 16 bits.
// o must be aligned to 4 elements (mh_vec_store).
template <typename P2>
__device__ __forceinline__ uint32_t mh_bits(P2 v) {
  uint32_t u;
  memcpy(&u, &v, sizeof(u));
  return u;
}
__device__ __forceinline__ void mh_store4(float* o, float v0, float v1, float v2, float v3) {
  *reinterpret_cast<float4*>(o) = make_float4(v0, v1, v2, v3);
}
__device__ __forceinline__ void mh_store4(__half* o, float v0, float v1, float v2, float v3) {
  *reinterpret_cast<uint2*>(o) = make_uint2(mh_bits(__floats2half2_rn(v0, v1)), mh_bits(__floats2half2_rn(v2, v3)));
}
__device__ __forceinline__ void mh_store4(__nv_bfloat16* o, float v0, float v1, float v2, float v3) {
  *reinterpret_cast<uint2*>(o) =
      make_uint2(mh_bits(__floats2bfloat162_rn(v0, v1)), mh_bits(__floats2bfloat162_rn(v2, v3)));
}
// Whether the rows of a (rows, N) output starting at `base` take mh_store4 at every point index n = 4i: N % 4 == 0
// puts every row start and every 4i at a multiple of 4 elements from `base`; a 16-bit base must then be 8-byte aligned
// (fp32 keeps its former rule, N % 4 alone, which assumes a 16-byte aligned buffer as torch allocates).  A row of odd
// N is only 2-byte aligned in 16 bits, so this depends on N and the address, never on the point index.
template <typename T>
__device__ __forceinline__ bool mh_vec_store(const T* base, int N) {
  return (N & 3) == 0 && (sizeof(T) == 4 || (reinterpret_cast<uintptr_t>(base) & 7) == 0);
}

// ---- tile loads ---------------------------------------------------------------------------------
// Xs[c][p] = x[b][c][n0+p] - ref[c] for c < C and valid points, 0 for points past N
template <typename T>
__device__ __forceinline__ void mh_load_x(float* Xs, const T* __restrict__ x, const float* ref, int C, int N, int b,
                                          int n0) {
  for (int e = threadIdx.x; e < C * kMhT; e += kMhThreads) {
    const int c = e / kMhT, p = e - c * kMhT, n = n0 + p;
    Xs[c * kMhTS + p] = n < N ? __fsub_rn(mh_ldg(x + ((size_t)b * C + c) * N + n), ref[c]) : 0.f;
  }
}
// Ls[j][p] = g[b][j][n0+p] for j < np, 0 for rows np..rows-1 and points past N
template <typename T>
__device__ __forceinline__ void mh_load_g(float* Ls, const T* __restrict__ g, int np, int rows, int N, int b, int n0) {
  for (int e = threadIdx.x; e < rows * kMhT; e += kMhThreads) {
    const int j = e / kMhT, p = e - j * kMhT, n = n0 + p;
    Ls[j * kMhTS + p] = (j < np && n < N) ? mh_ldg(g + ((size_t)b * np + j) * N + n) : 0.f;
  }
}

// ---- register-blocked products --------------------------------------------------------------------
// acc[r][q] += sum_{k<K} A[row_r][k] * Xs[k][4*lane+q],  row_r = r0 + r*rs (rows >= nr skipped, warp-uniform).
// A is a zero-padded global matrix (lda multiple of 4, 16-byte aligned): every lane reads the same float4, one
// broadcast transaction through L1.  K is a multiple of 4.
template <int R>
__device__ __forceinline__ void mh_gemm_rows(float (&acc)[R][4], const float* __restrict__ A, int lda, int r0, int rs,
                                             int nr, const float* Xs, int K) {
  const float* xp = Xs + 4 * (threadIdx.x & 31);
#pragma unroll 2
  for (int k = 0; k < K; k += 4) {
    const float4 x0 = *reinterpret_cast<const float4*>(xp + (k + 0) * kMhTS);
    const float4 x1 = *reinterpret_cast<const float4*>(xp + (k + 1) * kMhTS);
    const float4 x2 = *reinterpret_cast<const float4*>(xp + (k + 2) * kMhTS);
    const float4 x3 = *reinterpret_cast<const float4*>(xp + (k + 3) * kMhTS);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int row = r0 + r * rs;
      if (row < nr) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(A + (size_t)row * lda + k));
        acc[r][0] = fmaf(a.x, x0.x, acc[r][0]); acc[r][1] = fmaf(a.x, x0.y, acc[r][1]);
        acc[r][2] = fmaf(a.x, x0.z, acc[r][2]); acc[r][3] = fmaf(a.x, x0.w, acc[r][3]);
        acc[r][0] = fmaf(a.y, x1.x, acc[r][0]); acc[r][1] = fmaf(a.y, x1.y, acc[r][1]);
        acc[r][2] = fmaf(a.y, x1.z, acc[r][2]); acc[r][3] = fmaf(a.y, x1.w, acc[r][3]);
        acc[r][0] = fmaf(a.z, x2.x, acc[r][0]); acc[r][1] = fmaf(a.z, x2.y, acc[r][1]);
        acc[r][2] = fmaf(a.z, x2.z, acc[r][2]); acc[r][3] = fmaf(a.z, x2.w, acc[r][3]);
        acc[r][0] = fmaf(a.w, x3.x, acc[r][0]); acc[r][1] = fmaf(a.w, x3.y, acc[r][1]);
        acc[r][2] = fmaf(a.w, x3.z, acc[r][2]); acc[r][3] = fmaf(a.w, x3.w, acc[r][3]);
      }
    }
  }
}

// acc[i][j] += sum_{p<kMhT} U[ty+16i][p] * V[tx+16j][p]   (tx = tid & 15, ty = tid >> 4; both operands in shared
// memory with rows up to 16*MI / 16*MJ allocated)
template <int MI, int MJ>
__device__ __forceinline__ void mh_gemm_pts(float (&acc)[MI][MJ], const float* U, const float* V) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll 2
  for (int p = 0; p < kMhT; p += 4) {
    float4 u[MI], v[MJ];
#pragma unroll
    for (int i = 0; i < MI; ++i) u[i] = *reinterpret_cast<const float4*>(U + (ty + 16 * i) * kMhTS + p);
#pragma unroll
    for (int j = 0; j < MJ; ++j) v[j] = *reinterpret_cast<const float4*>(V + (tx + 16 * j) * kMhTS + p);
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
      for (int j = 0; j < MJ; ++j) {
        float a = acc[i][j];
        a = fmaf(u[i].x, v[j].x, a);
        a = fmaf(u[i].y, v[j].y, a);
        a = fmaf(u[i].z, v[j].z, a);
        a = fmaf(u[i].w, v[j].w, a);
        acc[i][j] = a;
      }
  }
}

// ---- kernels ---------------------------------------------------------------------------------------
// W1p[s] (CE,CE), W1tp[s] = W1p[s]^T, W2p[s] (64,CE), W2tp[s] = W2p[s]^T (CE,64); all zero-padded
__global__ void __launch_bounds__(256) mh_prep_kernel(MhArgs a, const float* __restrict__ w1,
                                                      const float* __restrict__ w2, int CE, float* __restrict__ W1p,
                                                      float* __restrict__ W1tp, float* __restrict__ W2p,
                                                      float* __restrict__ W2tp) {
  const int s = blockIdx.x, C = a.C, np = a.np[s];
  const float* w1s = w1 + (size_t)s * C * C;
  const float* w2s = w2 + (size_t)a.off[s] * C;
  for (int e = threadIdx.x; e < CE * CE; e += blockDim.x) {
    const int i = e / CE, j = e - i * CE;
    const float v = (i < C && j < C) ? w1s[i * C + j] : 0.f;
    W1p[(size_t)s * CE * CE + e] = v;
    W1tp[(size_t)s * CE * CE + j * CE + i] = v;
  }
  for (int e = threadIdx.x; e < kMhMaxParts * CE; e += blockDim.x) {
    const int i = e / CE, j = e - i * CE;
    const float v = (i < np && j < C) ? w2s[i * C + j] : 0.f;
    W2p[(size_t)s * kMhMaxParts * CE + e] = v;
    W2tp[(size_t)s * kMhMaxParts * CE + j * kMhMaxParts + i] = v;
  }
}

// training: per CTA, m1 = sum (x - s), M2 = sum (x - s)(x - s)^T over its tiles -> partial[blk] = [m1 (C) | M2 (C*C)]
template <int CE, typename T>
__global__ void __launch_bounds__(kMhThreads) mh_moments_kernel(const T* __restrict__ x, int B, int C, int N,
                                                                float* __restrict__ partial) {
  using Cf = MhCfg<CE>;
  extern __shared__ float4 mh_smem4[];
  float* Xs = reinterpret_cast<float*>(mh_smem4);
  __shared__ float s_shift[CL3D_MHEAD_MAX_CHANNELS];
  for (int e = threadIdx.x; e < Cf::RS * kMhTS; e += kMhThreads) Xs[e] = 0.f;
  if (threadIdx.x < C) s_shift[threadIdx.x] = load_f32(x + (size_t)threadIdx.x * N);
  float acc[Cf::MT][Cf::MT] = {};
  float m1 = 0.f;
  const int tpc = ceil_div(N, kMhT), ntiles = B * tpc;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    __syncthreads();
    mh_load_x(Xs, x, s_shift, C, N, t / tpc, (t % tpc) * kMhT);
    __syncthreads();
    mh_gemm_pts<Cf::MT, Cf::MT>(acc, Xs, Xs);
    if (threadIdx.x < C) {
      const float* row = Xs + threadIdx.x * kMhTS;
      float s = 0.f;
      for (int p = 0; p < kMhT; ++p) s += row[p];
      m1 += s;
    }
  }
  float* out = partial + (size_t)blockIdx.x * (C + C * C);
  if (threadIdx.x < C) out[threadIdx.x] = m1;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < Cf::MT; ++i)
#pragma unroll
    for (int j = 0; j < Cf::MT; ++j) {
      const int r = ty + 16 * i, c = tx + 16 * j;
      if (r < C && c < C) out[C + r * C + c] = acc[i][j];
    }
}

// one CTA per head: batch (training) or running (eval) statistics, running-statistics update, folded scale/shift
template <typename T>
__global__ void __launch_bounds__(128) mh_stats_kernel(MhArgs a, const T* __restrict__ x, int N,
                                                       const float* __restrict__ w1, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, float momentum,
                                                       int training, long long P, float* __restrict__ save) {
  const int s = blockIdx.x, c = threadIdx.x, C = a.C, S = a.S;
  float* ref = save + mh_ref_off(S, C);
  float* shift = ref + C;
  const float* m1 = shift + C;
  const float* M2 = m1 + C;
  __shared__ double s_ref[CL3D_MHEAD_MAX_CHANNELS], s_sh[CL3D_MHEAD_MAX_CHANNELS];
  const double dP = (double)P;
  if (c < C) {
    const float sh = load_f32(x + (size_t)c * N);
    const float r = training ? (float)((double)sh + (double)m1[c] / dP) : sh;
    s_ref[c] = (double)r;
    s_sh[c] = (double)sh;
    if (s == 0) {
      ref[c] = r;
      shift[c] = sh;
    }
  }
  long long nbt_new = 0;
  if (training && a.nbt[s]) nbt_new = *a.nbt[s] + 1;
  __syncthreads();
  if (c < C) {
    const float* w = w1 + ((size_t)s * C + c) * C;
    double mean, var, invstd;
    if (training) {
      double wm = 0.0, ws = 0.0, q = 0.0;
      for (int i = 0; i < C; ++i) {
        const double wi = (double)w[i];
        wm += wi * (double)m1[i];
        ws += wi * s_sh[i];
        double t = 0.0;
        for (int j = 0; j < C; ++j) t += (double)w[j] * (double)M2[(size_t)i * C + j];
        q += wi * t;
      }
      mean = ws + wm / dP;
      var = q / dP - (wm / dP) * (wm / dP);
      if (var < 0.0) var = 0.0;
      invstd = 1.0 / sqrt(var + (double)eps);
      const double m = momentum >= 0.f ? (double)momentum : 1.0 / (double)nbt_new;
      const double unbiased = dP > 1.0 ? var * dP / (dP - 1.0) : var;
      a.rm[s][c] = (float)((1.0 - m) * (double)a.rm[s][c] + m * mean);
      a.rv[s][c] = (float)((1.0 - m) * (double)a.rv[s][c] + m * unbiased);
    } else {
      mean = (double)a.rm[s][c];
      var = (double)a.rv[s][c];
      invstd = (double)(1.0f / sqrtf(a.rv[s][c] + eps));
    }
    double wr = 0.0;
    for (int j = 0; j < C; ++j) wr += (double)w[j] * s_ref[j];
    const double c0 = wr - mean;
    const double sc = (double)gamma[s * C + c] * invstd;
    float* hs = save + (size_t)s * 5 * C;
    hs[c] = (float)mean;
    hs[C + c] = (float)invstd;
    hs[2 * C + c] = (float)sc;
    hs[3 * C + c] = (float)((double)beta[s * C + c] + c0 * sc);
    hs[4 * C + c] = (float)c0;
  }
  __syncthreads();
  if (c == 0 && training && a.nbt[s]) *a.nbt[s] = nbt_new;
}

// logits of every head for a tile of 128 points
template <int CE, typename T>
__global__ void __launch_bounds__(kMhThreads) mh_fwd_kernel(MhArgs a, const T* __restrict__ x,
                                                            const float* __restrict__ W1p,
                                                            const float* __restrict__ W2p,
                                                            const float* __restrict__ b2,
                                                            const float* __restrict__ save, int B, int N,
                                                            T* __restrict__ logits) {
  using Cf = MhCfg<CE>;
  constexpr int R = Cf::R;
  extern __shared__ float4 mh_smem4[];
  float* Xs = reinterpret_cast<float*>(mh_smem4);
  float* Zs = Xs + CE * kMhTS;
  const int C = a.C, S = a.S, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* ref = save + mh_ref_off(S, C);
  for (int e = threadIdx.x; e < CE * kMhTS; e += kMhThreads) Xs[e] = 0.f;
  const int tpc = ceil_div(N, kMhT), ntiles = B * tpc;
  const bool vec = mh_vec_store(logits, N);  // head blocks start at B*N*off[s] elements: a multiple of 4 too
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int b = t / tpc, n0 = (t % tpc) * kMhT, n = n0 + 4 * lane;
    __syncthreads();
    mh_load_x(Xs, x, ref, C, N, b, n0);
    __syncthreads();
    for (int s = 0; s < S; ++s) {
      const float* hs = save + (size_t)s * 5 * C;
      float acc[R][4] = {};
      mh_gemm_rows<R>(acc, W1p + (size_t)s * CE * CE, CE, warp * R, 1, CE, Xs, CE);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int c = warp * R + r;
        const float sc = c < C ? hs[2 * C + c] : 0.f, sh = c < C ? hs[3 * C + c] : 0.f;
        float4 z;
        z.x = fmaxf(fmaf(acc[r][0], sc, sh), 0.f);
        z.y = fmaxf(fmaf(acc[r][1], sc, sh), 0.f);
        z.z = fmaxf(fmaf(acc[r][2], sc, sh), 0.f);
        z.w = fmaxf(fmaf(acc[r][3], sc, sh), 0.f);
        *reinterpret_cast<float4*>(Zs + c * kMhTS + 4 * lane) = z;
      }
      __syncthreads();
      const int np = a.np[s];
      float lo[8][4] = {};
      mh_gemm_rows<8>(lo, W2p + (size_t)s * kMhMaxParts * CE, CE, warp, 8, np, Zs, CE);
      T* out = logits + (size_t)B * N * a.off[s];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int j = warp + 8 * r;
        if (j < np) {
          const float bj = b2[a.off[s] + j];
          T* o = out + ((size_t)b * np + j) * N + n;
          if (vec) {
            if (n < N) mh_store4(o, lo[r][0] + bj, lo[r][1] + bj, lo[r][2] + bj, lo[r][3] + bj);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
              if (n + q < N) store_f32(o + q, lo[r][q] + bj);
          }
        }
      }
      __syncthreads();
    }
  }
}

// backward phase A, CTA (chunk, head): mask bits and per-CTA partials of G, sum gy, dW2, db2
// partial row layout: G (S,C,C) | sum gy (S,C) | dW2 (NPT,C) | db2 (NPT)
template <int CE, typename T>
__global__ void __launch_bounds__(kMhThreads) mh_bwd_a_kernel(MhArgs a, const T* __restrict__ x,
                                                              const float* __restrict__ W1p,
                                                              const float* __restrict__ W2tp,
                                                              const float* __restrict__ save, int B, int N,
                                                              float* __restrict__ partial, size_t LA,
                                                              uint32_t* __restrict__ mask) {
  using Cf = MhCfg<CE>;
  constexpr int R = Cf::R, MT = Cf::MT, RS = Cf::RS, CW = Cf::CW;
  const int s = blockIdx.y;
  const T* g = static_cast<const T*>(a.g[s]);
  if (!g) return;
  extern __shared__ float4 mh_smem4[];
  float* Xs = reinterpret_cast<float*>(mh_smem4);
  float* Ls = Xs + RS * kMhTS;
  float* Zs = Ls + kMhMaxParts * kMhTS;
  const int C = a.C, S = a.S, np = a.np[s], np4 = (np + 3) & ~3, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* ref = save + mh_ref_off(S, C);
  const float* hs = save + (size_t)s * 5 * C;
  const float* W1s = W1p + (size_t)s * CE * CE;
  const float* W2ts = W2tp + (size_t)s * kMhMaxParts * CE;
  for (int e = threadIdx.x; e < (2 * RS + kMhMaxParts) * kMhTS; e += kMhThreads) Xs[e] = 0.f;
  float sc[R], sh[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int c = warp * R + r;
    sc[r] = c < C ? hs[2 * C + c] : 0.f;
    sh[r] = c < C ? hs[3 * C + c] : 0.f;
  }
  float G[MT][MT] = {}, W2[4][MT] = {};
  float rsum = 0.f;
  const long long P = (long long)B * N;
  const int tpc = ceil_div(N, kMhT), ntiles = B * tpc;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int b = t / tpc, n0 = (t % tpc) * kMhT;
    __syncthreads();
    mh_load_x(Xs, x, ref, C, N, b, n0);
    mh_load_g(Ls, g, np, np, N, b, n0);
    __syncthreads();
    float acc[R][4] = {};
    mh_gemm_rows<R>(acc, W1s, CE, warp * R, 1, CE, Xs, CE);
    unsigned long long on = 0ull;  // bit r*4+q: z > 0
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float4 z;
      z.x = fmaxf(fmaf(acc[r][0], sc[r], sh[r]), 0.f);
      z.y = fmaxf(fmaf(acc[r][1], sc[r], sh[r]), 0.f);
      z.z = fmaxf(fmaf(acc[r][2], sc[r], sh[r]), 0.f);
      z.w = fmaxf(fmaf(acc[r][3], sc[r], sh[r]), 0.f);
      on |= (unsigned long long)((z.x > 0.f) | ((z.y > 0.f) << 1) | ((z.z > 0.f) << 2) | ((z.w > 0.f) << 3))
            << (4 * r);
      *reinterpret_cast<float4*>(Zs + (warp * R + r) * kMhTS + 4 * lane) = z;
    }
    __syncthreads();
    if (threadIdx.x < kMhT && n0 + (int)threadIdx.x < N) {
      const int p = threadIdx.x;
#pragma unroll
      for (int wd = 0; wd < CW; ++wd) {
        uint32_t word = 0u;
        for (int bit = 0; bit < 32; ++bit) {
          const int c = wd * 32 + bit;
          if (c < C && Zs[c * kMhTS + p] > 0.f) word |= 1u << bit;
        }
        mask[((size_t)s * CW + wd) * P + (size_t)b * N + n0 + p] = word;
      }
    }
    mh_gemm_pts<4, MT>(W2, Ls, Zs);
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
    mh_gemm_rows<R>(acc, W2ts, kMhMaxParts, warp * R, 1, CE, Ls, np4);
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float4 v;
      v.x = (on >> (4 * r + 0)) & 1ull ? acc[r][0] : 0.f;
      v.y = (on >> (4 * r + 1)) & 1ull ? acc[r][1] : 0.f;
      v.z = (on >> (4 * r + 2)) & 1ull ? acc[r][2] : 0.f;
      v.w = (on >> (4 * r + 3)) & 1ull ? acc[r][3] : 0.f;
      *reinterpret_cast<float4*>(Zs + (warp * R + r) * kMhTS + 4 * lane) = v;
    }
    __syncthreads();
    mh_gemm_pts<MT, MT>(G, Zs, Xs);
    const int tr = threadIdx.x;
    const float* row = tr < CE ? Zs + tr * kMhTS : (tr >= 128 && tr - 128 < np ? Ls + (tr - 128) * kMhTS : nullptr);
    if (row) {
      float v = 0.f;
      for (int p = 0; p < kMhT; ++p) v += row[p];
      rsum += v;
    }
  }
  float* out = partial + (size_t)blockIdx.x * LA;
  const size_t oW2 = (size_t)S * C * C + (size_t)S * C, oB2 = oW2 + (size_t)a.NPT * C;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < MT; ++j) {
      const int r = ty + 16 * i, c = tx + 16 * j;
      if (r < C && c < C) out[(size_t)s * C * C + r * C + c] = G[i][j];
    }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < MT; ++j) {
      const int r = ty + 16 * i, c = tx + 16 * j;
      if (r < np && c < C) out[oW2 + (size_t)(a.off[s] + r) * C + c] = W2[i][j];
    }
  if (threadIdx.x < C) out[(size_t)S * C * C + (size_t)s * C + threadIdx.x] = rsum;
  if (threadIdx.x >= 128 && threadIdx.x - 128 < np) out[oB2 + a.off[s] + threadIdx.x - 128] = rsum;
}

// one CTA per head: parameter gradients from the reduced partials; k = sc*invstd*mean(gy*xhat) and
// u = u0 + k*c0 (u0 = sc*mean(gy)) for the dx pass.  Training needs the second moments about ref:
// Q = M2 - m1 d^T - d m1^T + P d d^T, q1 = m1 - P d, d = ref - shift.
__global__ void __launch_bounds__(128) mh_bwd_fin_kernel(MhArgs a, const float* __restrict__ w1,
                                                         const float* __restrict__ save, const float* __restrict__ RA,
                                                         int training, long long P, float* __restrict__ gw1,
                                                         float* __restrict__ ggamma, float* __restrict__ gbeta,
                                                         float* __restrict__ gw2, float* __restrict__ gb2,
                                                         float* __restrict__ ku) {
  extern __shared__ float4 mh_smem4[];
  float* Q = reinterpret_cast<float*>(mh_smem4);
  __shared__ double s_q1[CL3D_MHEAD_MAX_CHANNELS];
  const int s = blockIdx.x, c = threadIdx.x, C = a.C, S = a.S, np = a.np[s], off = a.off[s];
  const size_t oW2 = (size_t)S * C * C + (size_t)S * C, oB2 = oW2 + (size_t)a.NPT * C;
  if (!a.g[s]) {
    for (int e = c; e < C * C; e += blockDim.x) gw1[(size_t)s * C * C + e] = 0.f;
    for (int e = c; e < np * C; e += blockDim.x) gw2[(size_t)off * C + e] = 0.f;
    if (c < np) gb2[off + c] = 0.f;
    if (c < C) {
      ggamma[s * C + c] = 0.f;
      gbeta[s * C + c] = 0.f;
      ku[(size_t)s * 2 * C + c] = 0.f;
      ku[(size_t)s * 2 * C + C + c] = 0.f;
    }
    return;
  }
  const float* ref = save + mh_ref_off(S, C);
  const float* shift = ref + C;
  const float* m1 = shift + C;
  const float* M2 = m1 + C;
  const double dP = (double)P;
  if (training) {
    for (int e = c; e < C * C; e += blockDim.x) {
      const int i = e / C, j = e - i * C;
      const double di = (double)ref[i] - (double)shift[i], dj = (double)ref[j] - (double)shift[j];
      Q[e] = (float)((double)M2[e] - (double)m1[i] * dj - di * (double)m1[j] + dP * di * dj);
    }
    if (c < C) s_q1[c] = (double)m1[c] - dP * ((double)ref[c] - (double)shift[c]);
  }
  __syncthreads();
  for (int e = c; e < np * C; e += blockDim.x) gw2[(size_t)off * C + e] = RA[oW2 + (size_t)off * C + e];
  if (c < np) gb2[off + c] = RA[oB2 + off + c];
  if (c >= C) return;
  const float* w = w1 + ((size_t)s * C + c) * C;
  const float* hs = save + (size_t)s * 5 * C;
  const double invstd = hs[C + c], sc = hs[2 * C + c], c0 = hs[4 * C + c];
  const float* Gr = RA + (size_t)s * C * C + (size_t)c * C;
  const double Sg = RA[(size_t)S * C * C + (size_t)s * C + c];
  double wG = 0.0;
  for (int j = 0; j < C; ++j) wG += (double)w[j] * (double)Gr[j];
  const double dgamma = invstd * (wG + c0 * Sg);
  ggamma[s * C + c] = (float)dgamma;
  gbeta[s * C + c] = (float)Sg;
  double k = 0.0, u0 = 0.0, wq1 = 0.0;
  if (training) {
    k = sc * invstd * dgamma / dP;
    u0 = sc * Sg / dP;
    for (int j = 0; j < C; ++j) wq1 += (double)w[j] * s_q1[j];
  }
  const double sumdy = sc * Sg - dP * u0 - k * (wq1 + dP * c0);
  float* gr = gw1 + ((size_t)s * C + c) * C;
  for (int j = 0; j < C; ++j) {
    double v = sc * (double)Gr[j] + sumdy * (double)ref[j];
    if (training) {
      double t = 0.0;
      for (int i = 0; i < C; ++i) t += (double)w[i] * (double)Q[i * C + j];
      v -= u0 * s_q1[j] + k * (t + c0 * s_q1[j]);
    }
    gr[j] = (float)v;
  }
  ku[(size_t)s * 2 * C + c] = (float)k;
  ku[(size_t)s * 2 * C + C + c] = (float)(u0 + k * c0);
}

// M = sum_s W1_s^T diag(k_s) W1_s (CE x CE, zero-padded), v0 = sum_s W1_s^T u_s; fixed order over s and c
__global__ void __launch_bounds__(128) mh_bwd_mx_kernel(MhArgs a, const float* __restrict__ w1,
                                                        const float* __restrict__ ku, int CE, float* __restrict__ Mp,
                                                        float* __restrict__ v0) {
  const int i = blockIdx.x, j = threadIdx.x, C = a.C;
  if (j >= CE) return;
  float m = 0.f, v = 0.f;
  if (i < C) {
    for (int s = 0; s < a.S; ++s) {
      if (!a.g[s]) continue;
      const float* ws = w1 + (size_t)s * C * C;
      const float* ks = ku + (size_t)s * 2 * C;
      for (int c = 0; c < C; ++c) {
        const float wi = ws[c * C + i];
        if (j < C) m = fmaf(wi * ks[c], ws[c * C + j], m);
        if (j == 0) v = fmaf(wi, ks[C + c], v);
      }
    }
  }
  Mp[i * CE + j] = m;
  if (j == 0) v0[i] = v;
}

// dx for a tile of 128 points, accumulated over the heads in registers
template <int CE, typename T>
__global__ void __launch_bounds__(kMhThreads) mh_bwd_dx_kernel(MhArgs a, const T* __restrict__ x,
                                                               const float* __restrict__ W1tp,
                                                               const float* __restrict__ W2tp,
                                                               const float* __restrict__ save,
                                                               const float* __restrict__ Mp,
                                                               const float* __restrict__ v0,
                                                               const uint32_t* __restrict__ mask, int training, int B,
                                                               int N, T* __restrict__ gx) {
  using Cf = MhCfg<CE>;
  constexpr int R = Cf::R, CW = Cf::CW;
  extern __shared__ float4 mh_smem4[];
  float* Us = reinterpret_cast<float*>(mh_smem4);
  float* Ls = Us + CE * kMhTS;
  uint32_t* Ms = reinterpret_cast<uint32_t*>(Ls + kMhMaxParts * kMhTS);
  const int C = a.C, S = a.S, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* ref = save + mh_ref_off(S, C);
  const long long P = (long long)B * N;
  for (int e = threadIdx.x; e < CE * kMhTS; e += kMhThreads) Us[e] = 0.f;
  const int tpc = ceil_div(N, kMhT), ntiles = B * tpc;
  const bool vec = mh_vec_store(gx, N);
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int b = t / tpc, n0 = (t % tpc) * kMhT, n = n0 + 4 * lane;
    float acc[R][4] = {};
    if (training) {
      __syncthreads();
      mh_load_x(Us, x, ref, C, N, b, n0);
      __syncthreads();
      mh_gemm_rows<R>(acc, Mp, CE, warp * R, 1, CE, Us, CE);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float vr = v0[warp * R + r];
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[r][q] = -acc[r][q] - vr;
      }
    }
    for (int s = 0; s < S; ++s) {
      const T* g = static_cast<const T*>(a.g[s]);
      if (!g) continue;
      const int np = a.np[s], np4 = (np + 3) & ~3;
      const float* hs = save + (size_t)s * 5 * C;
      __syncthreads();
      mh_load_g(Ls, g, np, np4, N, b, n0);
      if (threadIdx.x < kMhT) {
        const int p = threadIdx.x;
        const bool ok = n0 + p < N;
#pragma unroll
        for (int wd = 0; wd < CW; ++wd)
          Ms[wd * kMhT + p] = ok ? mask[((size_t)s * CW + wd) * P + (size_t)b * N + n0 + p] : 0u;
      }
      __syncthreads();
      float gy[R][4] = {};
      mh_gemm_rows<R>(gy, W2tp + (size_t)s * kMhMaxParts * CE, kMhMaxParts, warp * R, 1, CE, Ls, np4);
      __syncthreads();  // every warp is done reading Us (previous head's product) before it is overwritten
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int c = warp * R + r;
        const float sc = c < C ? hs[2 * C + c] : 0.f;
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t wbits = Ms[(c >> 5) * kMhT + 4 * lane + q];
          v[q] = (wbits >> (c & 31)) & 1u ? gy[r][q] * sc : 0.f;
        }
        *reinterpret_cast<float4*>(Us + c * kMhTS + 4 * lane) = make_float4(v[0], v[1], v[2], v[3]);
      }
      __syncthreads();
      mh_gemm_rows<R>(acc, W1tp + (size_t)s * CE * CE, CE, warp * R, 1, CE, Us, CE);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = warp * R + r;
      if (c < C) {
        T* o = gx + ((size_t)b * C + c) * N + n;
        if (vec) {
          if (n < N) mh_store4(o, acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (n + q < N) store_f32(o + q, acc[r][q]);
        }
      }
    }
  }
}

// ---- host side --------------------------------------------------------------------------------------
static int mh_width(int C) {
  const int Cp = padded_channels(C);
  const int widths[] = {16, 32, 48, 72, 96, 128};
  for (int w : widths)
    if (Cp <= w) return w;
  return 0;
}

static int mh_args(const cl3d_mhead_desc* d, MhArgs& a, int& CE, const char* who) {
  if (!d) {
    set_error("%s: desc_host is NULL", who);
    return CL3D_ERR_BAD_ARG;
  }
  if (d->S < 1 || d->C < 1) {
    set_error("%s: S and C must be >= 1", who);
    return CL3D_ERR_BAD_ARG;
  }
  if (d->S > CL3D_MHEAD_MAX_HEADS || padded_channels(d->C) > CL3D_MHEAD_MAX_CHANNELS) {
    set_error("%s: S = %d heads, C = %d channels: limits are 32 heads and 128 (padded) channels", who, d->S, d->C);
    return CL3D_ERR_UNSUPPORTED;
  }
  a = MhArgs{};
  a.S = d->S;
  a.C = d->C;
  a.off[0] = 0;
  for (int s = 0; s < d->S; ++s) {
    if (d->num_parts[s] < 1) {
      set_error("%s: num_parts[%d] = %d", who, s, d->num_parts[s]);
      return CL3D_ERR_BAD_ARG;
    }
    if (d->num_parts[s] > kMhMaxParts) {
      set_error("%s: num_parts[%d] = %d exceeds 64", who, s, d->num_parts[s]);
      return CL3D_ERR_UNSUPPORTED;
    }
    a.np[s] = d->num_parts[s];
    a.off[s + 1] = a.off[s] + a.np[s];
    a.g[s] = d->grad_logits[s];
    a.rm[s] = d->running_mean[s];
    a.rv[s] = d->running_var[s];
    a.nbt[s] = d->num_batches_tracked[s];
  }
  a.NPT = a.off[d->S];
  CE = mh_width(d->C);
  return CL3D_OK;
}

static int mh_tile_grid(int B, int N) {
  const int ntiles = B * ceil_div(N, kMhT);
  int g = 2 * sm_count();
  const int cap = persistent_grid_cap();
  g = g < cap ? g : cap;
  g = g < ntiles ? g : ntiles;
  return g < 1 ? 1 : g;
}
static int mh_chunks(int S, int B, int N) {
  const int ntiles = B * ceil_div(N, kMhT);
  int g = ceil_div(2 * sm_count(), S);
  const int cap = persistent_grid_cap();
  g = g < cap ? g : cap;
  g = g < ntiles ? g : ntiles;
  return g < 1 ? 1 : g;
}

static size_t mh_a64(size_t n) { return align_up(n, 64); }  // section sizes in floats, 256-byte aligned
static size_t mh_prep_floats(int S, int CE) { return mh_a64((size_t)S * CE * CE) * 2 + mh_a64((size_t)S * 64 * CE) * 2; }
static size_t mh_LA(const MhArgs& a) {
  return (size_t)a.S * a.C * a.C + (size_t)a.S * a.C + (size_t)a.NPT * a.C + a.NPT;
}

struct MhPrep {
  float *W1p, *W1tp, *W2p, *W2tp;
};
static MhPrep mh_prep_layout(float* base, int S, int CE) {
  MhPrep p;
  p.W1p = base;
  p.W1tp = p.W1p + mh_a64((size_t)S * CE * CE);
  p.W2p = p.W1tp + mh_a64((size_t)S * CE * CE);
  p.W2tp = p.W2p + mh_a64((size_t)S * 64 * CE);
  return p;
}

template <int CE, typename T>
static int mh_fwd_impl(const MhArgs& a, const T* x, int B, int N, const float* w1, const float* gamma,
                       const float* beta, const float* w2, const float* b2, float eps, float momentum, int training,
                       T* logits, float* save, float* ws, cudaStream_t st) {
  using Cf = MhCfg<CE>;
  const int S = a.S, C = a.C;
  const long long P = (long long)B * N;
  MhPrep pw = mh_prep_layout(ws, S, CE);
  mh_prep_kernel<<<S, 256, 0, st>>>(a, w1, w2, CE, pw.W1p, pw.W1tp, pw.W2p, pw.W2tp); CL3D_LAUNCHED(1);
  if (training) {
    float* partial = ws + mh_prep_floats(S, CE);
    const int g = mh_tile_grid(B, N);
    const size_t smem = (size_t)Cf::RS * kMhTS * sizeof(float);
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(mh_moments_kernel<CE, T>, seen);
    mh_moments_kernel<CE, T><<<g, kMhThreads, smem, st>>>(x, B, C, N, partial); CL3D_LAUNCHED(1);
    int rc = check_launch("mh_moments_kernel");
    if (rc) return rc;
    rc = cl3d_reduce_partials(partial, g, C + C * C, save + mh_ref_off(S, C) + 2 * C, st);
    if (rc) return rc;
  }
  mh_stats_kernel<T><<<S, 128, 0, st>>>(a, x, N, w1, gamma, beta, eps, momentum, training, P, save); CL3D_LAUNCHED(1);
  {
    const size_t smem = (size_t)2 * CE * kMhTS * sizeof(float);
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(mh_fwd_kernel<CE, T>, seen);
    mh_fwd_kernel<CE, T><<<mh_tile_grid(B, N), kMhThreads, smem, st>>>(a, x, pw.W1p, pw.W2p, b2, save, B, N, logits);
    CL3D_LAUNCHED(1);
  }
  return check_launch("mhead forward kernels");
}

struct MhBwdWs {
  MhPrep pw;
  float *partial, *RA, *ku, *Mp, *v0;
  uint32_t* mask;
  size_t LA;
  int chunks;
  size_t total;  // floats
};
static MhBwdWs mh_bwd_layout(const MhArgs& a, int CE, int B, int N, float* base) {
  MhBwdWs w;
  const long long P = (long long)B * N;
  w.LA = mh_LA(a);
  w.chunks = mh_chunks(a.S, B, N);
  w.pw = mh_prep_layout(base, a.S, CE);
  size_t o = mh_prep_floats(a.S, CE);
  w.partial = base + o; o += mh_a64((size_t)w.chunks * w.LA);
  w.RA = base + o; o += mh_a64(w.LA);
  w.ku = base + o; o += mh_a64((size_t)a.S * 2 * a.C);
  w.Mp = base + o; o += mh_a64((size_t)CE * CE);
  w.v0 = base + o; o += mh_a64(CE);
  w.mask = reinterpret_cast<uint32_t*>(base + o); o += mh_a64((size_t)a.S * ((CE + 31) / 32) * P);
  w.total = o;
  return w;
}

template <int CE, typename T>
static int mh_bwd_impl(const MhArgs& a, const T* x, int B, int N, const float* w1, const float* w2,
                       const float* save, int training, T* gx, float* gw1, float* ggamma, float* gbeta,
                       float* gw2, float* gb2, float* ws, cudaStream_t st) {
  using Cf = MhCfg<CE>;
  const int S = a.S, C = a.C;
  const long long P = (long long)B * N;
  MhBwdWs w = mh_bwd_layout(a, CE, B, N, ws);
  mh_prep_kernel<<<S, 256, 0, st>>>(a, w1, w2, CE, w.pw.W1p, w.pw.W1tp, w.pw.W2p, w.pw.W2tp); CL3D_LAUNCHED(1);
  {
    const size_t smem = (size_t)(2 * Cf::RS + kMhMaxParts) * kMhTS * sizeof(float);
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(mh_bwd_a_kernel<CE, T>, seen);
    mh_bwd_a_kernel<CE, T><<<dim3(w.chunks, S), kMhThreads, smem, st>>>(a, x, w.pw.W1p, w.pw.W2tp, save, B, N,
                                                                      w.partial, w.LA, w.mask);
    CL3D_LAUNCHED(1);
    const int rc = check_launch("mh_bwd_a_kernel");
    if (rc) return rc;
  }
  int rc = cl3d_reduce_partials(w.partial, w.chunks, (int)w.LA, w.RA, st);
  if (rc) return rc;
  {
    const size_t smem = training ? (size_t)C * C * sizeof(float) : 0;
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(mh_bwd_fin_kernel, seen);
    mh_bwd_fin_kernel<<<S, 128, smem, st>>>(a, w1, save, w.RA, training, P, gw1, ggamma, gbeta, gw2, gb2, w.ku);
    CL3D_LAUNCHED(1);
  }
  if (training) {
    mh_bwd_mx_kernel<<<CE, 128, 0, st>>>(a, w1, w.ku, CE, w.Mp, w.v0); CL3D_LAUNCHED(1);
  }
  {
    const size_t smem = (size_t)(CE + kMhMaxParts) * kMhTS * sizeof(float) + (size_t)Cf::CW * kMhT * sizeof(uint32_t);
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(mh_bwd_dx_kernel<CE, T>, seen);
    mh_bwd_dx_kernel<CE, T><<<mh_tile_grid(B, N), kMhThreads, smem, st>>>(a, x, w.pw.W1tp, w.pw.W2tp, save, w.Mp, w.v0,
                                                                        w.mask, training, B, N, gx);
    CL3D_LAUNCHED(1);
  }
  return check_launch("mhead backward kernels");
}

#define CL3D_MH_DISPATCH(CE, T, fn, ...)        \
  switch (CE) {                                 \
    case 16: return fn<16, T>(__VA_ARGS__);     \
    case 32: return fn<32, T>(__VA_ARGS__);     \
    case 48: return fn<48, T>(__VA_ARGS__);     \
    case 72: return fn<72, T>(__VA_ARGS__);     \
    case 96: return fn<96, T>(__VA_ARGS__);     \
    case 128: return fn<128, T>(__VA_ARGS__);   \
    default: return CL3D_ERR_UNSUPPORTED;       \
  }

}  // namespace cl3d

using namespace cl3d;

extern "C" size_t cl3d_mhead_save_floats(int S, int C) {
  return (size_t)5 * S * C + 3 * (size_t)C + (size_t)C * C;
}

extern "C" size_t cl3d_mhead_fwd_workspace_bytes(const cl3d_mhead_desc* desc_host, int B, int N) {
  MhArgs a;
  int CE = 0;
  if (mh_args(desc_host, a, CE, "cl3d_mhead_fwd_workspace_bytes") != CL3D_OK || B < 1 || N < 1) return 0;
  return (mh_prep_floats(a.S, CE) + (size_t)mh_tile_grid(B, N) * (a.C + (size_t)a.C * a.C)) * sizeof(float);
}

extern "C" size_t cl3d_mhead_bwd_workspace_bytes(const cl3d_mhead_desc* desc_host, int B, int N) {
  MhArgs a;
  int CE = 0;
  if (mh_args(desc_host, a, CE, "cl3d_mhead_bwd_workspace_bytes") != CL3D_OK || B < 1 || N < 1) return 0;
  return mh_bwd_layout(a, CE, B, N, nullptr).total * sizeof(float);
}

extern "C" int cl3d_mhead_fwd(const cl3d_mhead_desc* desc_host, const void* x, int dtype, int B, int N,
                              const float* w1, const float* gamma, const float* beta, const float* w2,
                              const float* b2, float eps, float momentum, int training, void* logits, float* save,
                              void* workspace, size_t workspace_bytes, cl3d_stream_t stream_) {
  MhArgs a;
  int CE = 0;
  const int rc = mh_args(desc_host, a, CE, "cl3d_mhead_fwd");
  if (rc != CL3D_OK) return rc;
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_mhead_fwd");
  CL3D_REQUIRE(x && w1 && gamma && beta && w2 && b2 && logits && save && workspace, "cl3d_mhead_fwd: null pointer");
  CL3D_REQUIRE(B >= 1 && N >= 1, "cl3d_mhead_fwd: bad sizes");
  for (int s = 0; s < a.S; ++s) {
    CL3D_REQUIRE(a.rm[s] && a.rv[s], "cl3d_mhead_fwd: head %d has no running statistics", s);
    CL3D_REQUIRE(!training || momentum >= 0.f || a.nbt[s], "cl3d_mhead_fwd: momentum=None needs num_batches_tracked");
  }
  if (workspace_bytes < cl3d_mhead_fwd_workspace_bytes(desc_host, B, N)) {
    set_error("cl3d_mhead_fwd: workspace too small");
    return CL3D_ERR_WORKSPACE;
  }
  float* ws = static_cast<float*>(workspace);
  cudaStream_t st = (cudaStream_t)stream_;
  return with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    CL3D_MH_DISPATCH(CE, T, mh_fwd_impl, a, static_cast<const T*>(x), B, N, w1, gamma, beta, w2, b2, eps, momentum,
                     training, static_cast<T*>(logits), save, ws, st)
  });
}

extern "C" int cl3d_mhead_bwd(const cl3d_mhead_desc* desc_host, const void* x, int dtype, int B, int N,
                              const float* w1, const float* w2, const float* save, int training, void* grad_x,
                              float* grad_w1, float* grad_gamma, float* grad_beta, float* grad_w2, float* grad_b2,
                              void* workspace, size_t workspace_bytes, cl3d_stream_t stream_) {
  MhArgs a;
  int CE = 0;
  const int rc = mh_args(desc_host, a, CE, "cl3d_mhead_bwd");
  if (rc != CL3D_OK) return rc;
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_mhead_bwd");
  CL3D_REQUIRE(x && w1 && w2 && save && grad_x && grad_w1 && grad_gamma && grad_beta && grad_w2 && grad_b2 &&
                   workspace,
               "cl3d_mhead_bwd: null pointer");
  CL3D_REQUIRE(B >= 1 && N >= 1, "cl3d_mhead_bwd: bad sizes");
  if (workspace_bytes < cl3d_mhead_bwd_workspace_bytes(desc_host, B, N)) {
    set_error("cl3d_mhead_bwd: workspace too small");
    return CL3D_ERR_WORKSPACE;
  }
  float* ws = static_cast<float*>(workspace);
  cudaStream_t st = (cudaStream_t)stream_;
  return with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    CL3D_MH_DISPATCH(CE, T, mh_bwd_impl, a, static_cast<const T*>(x), B, N, w1, w2, save, training,
                     static_cast<T*>(grad_x), grad_w1, grad_gamma, grad_beta, grad_w2, grad_b2, ws, st)
  });
}
