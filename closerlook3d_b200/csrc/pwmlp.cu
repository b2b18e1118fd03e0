// pwmlp.cu -- fused Point-wise MLP local aggregation (feature_type 'dp_fi_df', num_mlps 1, reduction max).
//
// Reference: /root/reference/pytorch/models/local_aggregation_operators.py:254-257 (conv + BatchNorm2d + ReLU),
// :288-303 (input assembly [dp; f_i; f_j - f_i], max over K).  With one conv layer W = [Wp | Wc | Wr]:
//     y[o,q,k] = Wp[o]·dp_k + Wc[o]·f_i + Wr[o]·(f_{j_k} - f_i),     f_i = f of slot 0 (nearest neighbour)
// and dp_k = (s_{j_k} - q)/r is a difference, so y separates into a per-QUERY and a per-POINT term:
//     y[o,q,k] = a'[q][o] + bv[j_k][o],   a'[q] = (Wc-Wr) f_{j_0} - Wp q/r,   bv[j] = Wr f_j + Wp s_j/r .
// Both positions are taken relative to the cloud's first support point o_b (q - o_b, s - o_b: the difference is
// unchanged), so the two terms that cancel stay of the size of the cloud's extent / r even for scenes far from the
// coordinate origin (S3DIS rooms: |xyz| / r ~ 300 would cost 2e-5 of dp in fp32).
// The per-point terms are ONE (B*N x (C+3)) x ((C+3) x 2*Cop) product over the augmented point-major matrix
// [f | s/r] (csrc/gemm.cu); the per-neighbour work that remains is a row gather with 6 instructions per
// element.  BatchNorm2d statistics over all B*M*K positions (padding slots included, as in the reference) are
// accumulated on the fly:  sum_k y = K a' + S,  sum_k y^2 = K a'^2 + 2 a' S + S2  with S = sum_k bv.
// The max over K commutes with the monotone BN + ReLU; which extremum is needed depends only on the sign of
// gamma, so the host folds sgn = sign(gamma) into the T rows of the product (t = sgn*bv) and the kernel tracks
// max_k t with its FIRST arg-max slot (max_pool2d's tie rule):  y_sel = a' + sgn*max_k t,
// out = relu(sc*y_sel + sh).
//
// backward (BatchNorm2d backward is dense over B*M*K:  dy = sc*[k==k*]*dz - c1 - c2*(y - mean)):
//   pwmlp_bwd_stats_kernel  sum dz, sum dz*yhat, and sc*dz written point-major     (elementwise + reduce)
//   pwmlp_bwd_dense_kernel  support-major over the all-slots CSR lists: the dense part of d/dbv needs only
//                           cnt_j and sum_e a'[q_e]  -> one row gather, 2 instructions per element, no atomics
//   pwmlp_bwd_query_kernel  thread per (query, 4 channels), no K loop: d/da' in closed form from the saved S,
//                           d/dA[j_0] as one red.global.add.v4.f32, the arg-max slot's sc*dz, d/dWp partials
#include <mutex>

#include "common.cuh"

namespace cl3d {

constexpr int kPWWarps = 8;
constexpr int kPWTile = 32;
constexpr int kPWMaxCI = 4;  // 128 output channels per CTA chunk
constexpr int kPWU = 8;      // neighbour rows in flight per lane

struct PwArgs {
  const float* ab_pm;        // (B,N,2*Cop): row = [A (Cop) | T (Cop)],  T = sgn * bv
  const float* wp;           // (Cout,3)
  const float* sgn;          // (Cout) +1 / -1
  const float* query_xyz;    // (B,M,3)
  const float* support_xyz;  // (B,N,3): row 0 of each cloud is the origin the separable terms are centred on
  const int* idx;            // (B,M,K)
  float* ysel;               // (B,Cout,M)
  float* aq;                 // (B,M,Cop) a'
  float* sq;                 // (B,M,Cop) S = sum_k bv
  unsigned char* karg;       // (B,M,Cop) first arg-max slot
  float* partial;            // fwd: (ntiles,2,Cout) ; bwd sparse: (ntiles,3,Cout) dWp partials
  // backward only
  const float* grad_out;     // (B,Cout,M)
  const float* out;          // (B,Cout,M)
  const float* stats;        // (2,Cout) mean, invstd
  const float* gamma;        // (Cout)
  const float* dgb;          // (2,Cout): sum dz*yhat, sum dz
  const int* csr_off;        // (B,N+1)   all-slots lists
  const int* csr_ent;        // (B,M*K)
  float* grad_ab_pm;         // (B,N,2*Cop)
  const float* dzs_pm;       // (B,M,Cop) sc*dz, point-major
  int B, N, M, K, Cout, Cop;
  float inv_radius, inv_count;
  int ntiles;
};

// =================================================================================================
// forward: statistics + selected extremum
// =================================================================================================
template <int CI>
__global__ void __launch_bounds__(kPWWarps * 32) pwmlp_fwd_kernel(const PwArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int chunkC = min(32 * CI, a.Cop - c0);
  int* s_idx = reinterpret_cast<int*>(smem) + (size_t)warp * a.K;                       // [warps][K]
  float* s_y = reinterpret_cast<float*>(smem + align_up((size_t)kPWWarps * a.K * 4, 16));  // [chunk][tile+1]
  float* s_red = s_y + (size_t)32 * CI * (kPWTile + 1);                                  // [warps][2][chunk]

  const int tiles_per_cloud = (a.M + kPWTile - 1) / kPWTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kPWTile;

  bool okc[CI];
  float wpx[CI], wpy[CI], wpz[CI], sg[CI], s1[CI], s2[CI];
#pragma unroll
  for (int i = 0; i < CI; ++i) {
    okc[i] = lane + 32 * i < chunkC;
    const int c = c0 + lane + 32 * i;
    const bool ok = c < a.Cout;
    wpx[i] = ok ? a.wp[c * 3 + 0] : 0.f;
    wpy[i] = ok ? a.wp[c * 3 + 1] : 0.f;
    wpz[i] = ok ? a.wp[c * 3 + 2] : 0.f;
    sg[i] = ok ? a.sgn[c] : 1.f;
    s1[i] = s2[i] = 0.f;
  }
  const float* ab = a.ab_pm + (size_t)b * a.N * 2 * a.Cop + c0 + lane;  // per-lane base pointer (A half)
  const float* tb = ab + a.Cop;                                           // T half
  const unsigned rstride = 2u * (unsigned)a.Cop;
  const float fK = (float)a.K;

  // neighbour indices of the NEXT query are fetched while the current one is processed (K <= 64: two per lane)
  const bool pre_ok = a.K <= 64;
  int pre0 = 0, pre1 = 0;
  if (pre_ok && q0 + warp < a.M) {
    const int* ip = a.idx + ((size_t)b * a.M + q0 + warp) * a.K;
    if (lane < a.K) pre0 = ip[lane];
    if (lane + 32 < a.K) pre1 = ip[lane + 32];
  }
  for (int ql = warp; ql < kPWTile; ql += kPWWarps) {
    const int q = q0 + ql;
    float ys[CI];
#pragma unroll
    for (int i = 0; i < CI; ++i) ys[i] = 0.f;
    if (q < a.M) {
      const size_t gq = (size_t)b * a.M + q;
      if (pre_ok) {
        if (lane < a.K) s_idx[lane] = (int)((unsigned)pre0 * rstride);
        if (lane + 32 < a.K) s_idx[lane + 32] = (int)((unsigned)pre1 * rstride);
        if (ql + kPWWarps < kPWTile && q + kPWWarps < a.M) {
          const int* ip = a.idx + (gq + kPWWarps) * a.K;
          if (lane < a.K) pre0 = ip[lane];
          if (lane + 32 < a.K) pre1 = ip[lane + 32];
        }
      } else {
        for (int k = lane; k < a.K; k += 32) s_idx[k] = (int)((unsigned)a.idx[gq * a.K + k] * rstride);  // row offsets
      }
      // a' = A[j_0] - Wp q/r      (slot 0 = nearest neighbour, reference :290)
      const float* org = a.support_xyz + (size_t)b * a.N * 3;
      const float qx = __fmul_rn(__fsub_rn(a.query_xyz[gq * 3 + 0], org[0]), a.inv_radius),
                  qy = __fmul_rn(__fsub_rn(a.query_xyz[gq * 3 + 1], org[1]), a.inv_radius),
                  qz = __fmul_rn(__fsub_rn(a.query_xyz[gq * 3 + 2], org[2]), a.inv_radius);
      __syncwarp();
      float ap[CI], S[CI], S2[CI], m[CI];
      int km[CI];
      {
        const float* arow = row_at(ab, (unsigned)s_idx[0]);
#pragma unroll
        for (int i = 0; i < CI; ++i) {
          ap[i] = __ldg(arow + 32 * i) - fmaf(wpz[i], qz, fmaf(wpy[i], qy, wpx[i] * qx));
          S[i] = S2[i] = 0.f;
          m[i] = -INFINITY;
          km[i] = 0;
        }
      }
      int k0 = 0;
      for (; k0 + kPWU <= a.K; k0 += kPWU) {
        float v[kPWU][CI];
#pragma unroll
        for (int u = 0; u < kPWU; ++u) {
          const float* row = row_at(tb, (unsigned)s_idx[k0 + u]);
#pragma unroll
          for (int i = 0; i < CI; ++i) v[u][i] = __ldg(row + 32 * i);  // lanes past the chunk read slack (unused)
        }
#pragma unroll
        for (int u = 0; u < kPWU; ++u)
#pragma unroll
          for (int i = 0; i < CI; ++i) {
            const float t = v[u][i];
            S[i] += t;
            S2[i] = fmaf(t, t, S2[i]);
            const bool gt = t > m[i];  // strict: the first occurrence keeps the slot, as max_pool2d
            m[i] = gt ? t : m[i];
            km[i] = gt ? (k0 + u) : km[i];
          }
      }
      for (; k0 < a.K; ++k0) {
        const float* row = row_at(tb, (unsigned)s_idx[k0]);
#pragma unroll
        for (int i = 0; i < CI; ++i) {
          const float t = __ldg(row + 32 * i);
          S[i] += t;
          S2[i] = fmaf(t, t, S2[i]);
          const bool gt = t > m[i];
          m[i] = gt ? t : m[i];
          km[i] = gt ? k0 : km[i];
        }
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < CI; ++i) {
        const float Sb = sg[i] * S[i];             // sum_k bv
        ys[i] = ap[i] + sg[i] * m[i];              // selected extremum of y
        s1[i] += fmaf(fK, ap[i], Sb);              // sum_k y
        s2[i] += fmaf(fK * ap[i], ap[i], fmaf(2.f * ap[i], Sb, S2[i]));  // sum_k y^2
        if (lane + 32 * i < chunkC) {
          const size_t o = gq * a.Cop + c0 + lane + 32 * i;
          a.aq[o] = ap[i];
          a.sq[o] = Sb;
          a.karg[o] = (unsigned char)km[i];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < CI; ++i) s_y[(size_t)(lane + 32 * i) * (kPWTile + 1) + ql] = ys[i];
  }
#pragma unroll
  for (int i = 0; i < CI; ++i) {
    s_red[((size_t)warp * 2 + 0) * 32 * CI + lane + 32 * i] = s1[i];
    s_red[((size_t)warp * 2 + 1) * 32 * CI + lane + 32 * i] = s2[i];
  }
  __syncthreads();
  const int q = q0 + lane;
  for (int cl = warp; cl < 32 * CI; cl += kPWWarps) {
    const int c = c0 + cl;
    if (c >= a.Cout) break;
    if (q < a.M) a.ysel[((size_t)b * a.Cout + c) * a.M + q] = s_y[(size_t)cl * (kPWTile + 1) + lane];
  }
  for (int cl = threadIdx.x; cl < 32 * CI; cl += blockDim.x) {
    const int c = c0 + cl;
    if (c >= a.Cout) continue;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int w = 0; w < kPWWarps; ++w) {
      t1 += s_red[((size_t)w * 2 + 0) * 32 * CI + cl];
      t2 += s_red[((size_t)w * 2 + 1) * 32 * CI + cl];
    }
    a.partial[((size_t)blockIdx.x * 2 + 0) * a.Cout + c] = t1;
    a.partial[((size_t)blockIdx.x * 2 + 1) * a.Cout + c] = t2;
  }
}

// out[b,o,q] = relu(sc*ysel + sh)
__global__ void __launch_bounds__(256) pwmlp_out_kernel(const float* __restrict__ ysel, const float* __restrict__ stats,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, int C, int M,
                                                        float* __restrict__ out) {
  const int row = blockIdx.x;
  const int c = row % C;
  const float mean = stats[c], sc = stats[C + c] * gamma[c], sh = beta[c];
  const float* src = ysel + (size_t)row * M;
  float* dst = out + (size_t)row * M;
  for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < M; i += gridDim.y * blockDim.x) {
    const float v = __fmaf_rn(__fsub_rn(src[i], mean), sc, sh);
    dst[i] = v > 0.f ? v : 0.f;
  }
}

// =================================================================================================
// backward
// =================================================================================================
__global__ void __launch_bounds__(256) pwmlp_bwd_stats_kernel(const float* __restrict__ grad_out,
                                                              const float* __restrict__ out,
                                                              const float* __restrict__ ysel,
                                                              const float* __restrict__ stats,
                                                              const float* __restrict__ gamma, int C, int Cop, int M,
                                                              float* __restrict__ partial,
                                                              float* __restrict__ dzs_pm /*(B,M,Cop): sc*dz*/) {
  extern __shared__ float s_tile[];  // [32][Cop + 1]
  const int tiles_per_cloud = (M + kPWTile - 1) / kPWTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kPWTile;
  const int q = q0 + (threadIdx.x & 31);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int c = warp; c < Cop; c += 8) {
    float dz = 0.f, dzy = 0.f, sc = 0.f;
    if (c < C && q < M) {
      const size_t o = ((size_t)b * C + c) * M + q;
      dz = out[o] > 0.f ? grad_out[o] : 0.f;
      dzy = dz * ((ysel[o] - stats[c]) * stats[C + c]);
      sc = stats[C + c] * gamma[c];
    }
    s_tile[(size_t)lane * (Cop + 1) + c] = sc * dz;
    if (c < C) {
      const float t1 = warp_sum(dz), t2 = warp_sum(dzy);
      if (lane == 0) {
        partial[((size_t)blockIdx.x * 2 + 0) * C + c] = t2;  // -> dgamma = sum dz*yhat
        partial[((size_t)blockIdx.x * 2 + 1) * C + c] = t1;  // -> dbeta  = sum dz
      }
    }
  }
  __syncthreads();
  const int nq = min(kPWTile, M - q0);
  float* dst = dzs_pm + ((size_t)b * M + q0) * Cop;
  for (int e = threadIdx.x; e < nq * Cop; e += blockDim.x) dst[e] = s_tile[(size_t)(e / Cop) * (Cop + 1) + e % Cop];
}

// Support-major pass over the all-slots CSR lists of point j (no float atomics): dense part of d/dbv
//   grad_T[j] = sgn * ( -cnt*c1 - c2*(sum_e a'[q_e] + cnt*(bv[j] - mean)) ),   grad_A[j] = 0
template <int CI>
__global__ void __launch_bounds__(kPWWarps * 32) pwmlp_bwd_dense_kernel(const PwArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int chunkC = min(32 * CI, a.Cop - c0);
  bool okc[CI];
  float c1[CI], c2[CI], mean[CI], sg[CI];
#pragma unroll
  for (int i = 0; i < CI; ++i) {
    okc[i] = lane + 32 * i < chunkC;
    const int c = c0 + lane + 32 * i;
    const bool ok = c < a.Cout;
    const float invstd = ok ? a.stats[a.Cout + c] : 0.f;
    const float sc = ok ? invstd * a.gamma[c] : 0.f;
    mean[i] = ok ? a.stats[c] : 0.f;
    c1[i] = ok ? sc * a.dgb[a.Cout + c] * a.inv_count : 0.f;
    c2[i] = ok ? sc * invstd * a.dgb[c] * a.inv_count : 0.f;
    sg[i] = ok ? a.sgn[c] : 1.f;
  }
  const int per_cloud = (a.N + kPWTile - 1) / kPWTile;
  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int b = tile / per_cloud;
    const int j0 = (tile % per_cloud) * kPWTile;
    const float* aq = a.aq + (size_t)b * a.M * a.Cop + c0 + lane;  // per-lane base pointer
    const int* off = a.csr_off + (size_t)b * (a.N + 1);
    const int* ent = a.csr_ent + (size_t)b * a.M * a.K;
    for (int jl = warp; jl < kPWTile; jl += kPWWarps) {
      const int j = j0 + jl;
      if (j >= a.N) continue;
      const int e0 = off[j], e1 = off[j + 1];
      float acc[CI];
#pragma unroll
      for (int i = 0; i < CI; ++i) acc[i] = 0.f;
      for (int eb = e0; eb < e1; eb += 32) {
        const int rows = min(32, e1 - eb);
        const unsigned myq = lane < rows ? (unsigned)(ent[eb + lane] / a.K) * (unsigned)a.Cop : 0u;  // row offset
        int r = 0;
        for (; r + kPWU <= rows; r += kPWU) {
          float v[kPWU][CI];
#pragma unroll
          for (int u = 0; u < kPWU; ++u) {
            const float* row = row_at(aq, __shfl_sync(0xffffffffu, myq, r + u));
#pragma unroll
            for (int i = 0; i < CI; ++i) v[u][i] = __ldg(row + 32 * i);  // lanes past the chunk read slack (unused)
          }
#pragma unroll
          for (int u = 0; u < kPWU; ++u)
#pragma unroll
            for (int i = 0; i < CI; ++i) acc[i] += v[u][i];
        }
        for (; r < rows; ++r) {
          const float* row = row_at(aq, __shfl_sync(0xffffffffu, myq, r));
#pragma unroll
          for (int i = 0; i < CI; ++i) acc[i] += __ldg(row + 32 * i);
        }
      }
      const float cnt = (float)(e1 - e0);
      const float* trow = a.ab_pm + ((size_t)b * a.N + j) * 2 * a.Cop + a.Cop + c0 + lane;
      float* grow = a.grad_ab_pm + ((size_t)b * a.N + j) * 2 * a.Cop;
#pragma unroll
      for (int i = 0; i < CI; ++i) {
        if (okc[i]) {
          const float bv = sg[i] * __ldg(trow + 32 * i);
          const float dbv = -cnt * c1[i] - c2[i] * (acc[i] + cnt * (bv - mean[i]));
          // grad_ab is zero-filled by the entry point; the query pass adds its arg-max hits to the same words
          // concurrently, so this is a reduction too (one per word: no contention)
          if (c0 + lane + 32 * i < a.Cout) atomicAdd(&grow[a.Cop + c0 + lane + 32 * i], sg[i] * dbv);
        }
      }
    }
  }
}

// Query-side pass, no K loop.  Thread (x, y): x = one group of 4 consecutive channels, y = a query lane; every
// thread walks kPWQPT queries so that d/dWp accumulates in registers (deterministic, no shared-memory atomics):
//   da'[q] = sum_k dy[q,k] = sc*dz - K*c1 - c2*(K*(a' - mean) + S)      (closed form from the saved S)
//   grad_A[j_0(q)] += da'      one 16-byte vector reduction (red.global.add.v4.f32) per (query, 4 channels)
//   grad_T[idx[q][k*]] += sgn*sc*dz  at the arg-max slot of each channel (scalar red.add, non-zero only)
//   d/dWp -= da' (x) q/r      per-CTA partial (gridDim.x, 3, Cout), reduced afterwards in a fixed order
// Layers wider than 4 * kPWQGroups channels split their channel groups over blockIdx.y (one slice per CTA).
constexpr int kPWQPT = 8;        // queries per thread
constexpr int kPWQGroups = 256;  // channel groups of 4 per CTA slice (= the block size when ny = 1)
__global__ void __launch_bounds__(256) pwmlp_bwd_query_kernel(const PwArgs a, long long nqueries /* B*M */) {
  extern __shared__ float s_dw[];  // [ny][3][Cop]
  const int ngroups = a.Cop >> 2;
  const int nx = ngroups < kPWQGroups ? ngroups : kPWQGroups, ny = blockDim.x / nx;
  const int x = blockIdx.y * nx + threadIdx.x % nx, y = threadIdx.x / nx;
  const bool active = x < ngroups;  // the last slice of a wide layer may be narrower than nx
  const int c4 = x * 4;
  float c1[4], c2[4], mean[4], sg[4], dw[3][4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int c = c4 + t;
    const bool ok = c < a.Cout;
    const float invstd = ok ? a.stats[a.Cout + c] : 0.f;
    const float sc = ok ? invstd * a.gamma[c] : 0.f;
    mean[t] = ok ? a.stats[c] : 0.f;
    c1[t] = ok ? sc * a.dgb[a.Cout + c] * a.inv_count : 0.f;
    c2[t] = ok ? sc * invstd * a.dgb[c] * a.inv_count : 0.f;
    sg[t] = ok ? a.sgn[c] : 1.f;
    dw[0][t] = dw[1][t] = dw[2][t] = 0.f;
  }
  const float fK = (float)a.K;
  {
    const long long qbase = (long long)blockIdx.x * ny * kPWQPT;
#pragma unroll 2
    for (int it = 0; it < kPWQPT; ++it) {
      const long long gq = qbase + (long long)it * ny + y;  // b*M + q
      if (gq >= nqueries || !active) break;
      const long long b = gq / a.M;
      const size_t o = (size_t)gq * a.Cop + c4;
      const float4 ap = *reinterpret_cast<const float4*>(a.aq + o);
      const float4 sb = *reinterpret_cast<const float4*>(a.sq + o);
      const float4 dz = *reinterpret_cast<const float4*>(a.dzs_pm + o);
      const uchar4 ks = *reinterpret_cast<const uchar4*>(a.karg + o);
      const int* irow = a.idx + gq * a.K;
      const int j0 = irow[0];
      const float* org = a.support_xyz + (size_t)b * a.N * 3;
      const float qx = __fmul_rn(__fsub_rn(a.query_xyz[gq * 3 + 0], org[0]), a.inv_radius),
                  qy = __fmul_rn(__fsub_rn(a.query_xyz[gq * 3 + 1], org[1]), a.inv_radius),
                  qz = __fmul_rn(__fsub_rn(a.query_xyz[gq * 3 + 2], org[2]), a.inv_radius);
      const float apv[4] = {ap.x, ap.y, ap.z, ap.w}, sbv[4] = {sb.x, sb.y, sb.z, sb.w}, dzv[4] = {dz.x, dz.y, dz.z, dz.w};
      const int ksv[4] = {ks.x, ks.y, ks.z, ks.w};
      float* gab = a.grad_ab_pm + (size_t)b * a.N * 2 * a.Cop;
      float da[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        da[t] = (c4 + t < a.Cout) ? dzv[t] - fK * c1[t] - c2[t] * fmaf(fK, apv[t] - mean[t], sbv[t]) : 0.f;
        if (dzv[t] != 0.f && c4 + t < a.Cout)
          atomicAdd(gab + (size_t)irow[ksv[t]] * 2 * a.Cop + a.Cop + c4 + t, sg[t] * dzv[t]);
        dw[0][t] = fmaf(-da[t], qx, dw[0][t]);
        dw[1][t] = fmaf(-da[t], qy, dw[1][t]);
        dw[2][t] = fmaf(-da[t], qz, dw[2][t]);
      }
      float* pa = gab + (size_t)j0 * 2 * a.Cop + c4;
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(pa), "f"(da[0]), "f"(da[1]), "f"(da[2]), "f"(da[3])
                   : "memory");
    }
    if (active)
#pragma unroll
      for (int s3 = 0; s3 < 3; ++s3)
#pragma unroll
        for (int t = 0; t < 4; ++t) s_dw[((size_t)y * 3 + s3) * a.Cop + c4 + t] = dw[s3][t];
  }
  __syncthreads();
  // this CTA's channels [cs0, cs0 + w)
  const int cs0 = blockIdx.y * nx * 4, w = min(nx * 4, a.Cout - cs0);
  for (int e = threadIdx.x; e < 3 * w; e += blockDim.x) {
    const int s3 = e / w, c = cs0 + e % w;
    float t = 0.f;
    for (int yy = 0; yy < ny; ++yy) t += s_dw[((size_t)yy * 3 + s3) * a.Cop + c];
    a.partial[((size_t)blockIdx.x * 3 + s3) * a.Cout + c] = t;
  }
}

// (B,C,N) features + (B,N,3) xyz -> (B,N,Cpa) rows [f | (xyz - xyz[b,0])*inv_r | 0...], Cpa = padded(C+3)
__global__ void __launch_bounds__(256) to_point_major_aug_kernel(const float* __restrict__ in, const float* __restrict__ xyz,
                                                                 int C, int N, int Cpa, float inv_r,
                                                                 float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  in += (size_t)b * C * N;
  xyz += (size_t)b * N * 3;
  out += (size_t)b * N * Cpa;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, n = n0 + tx;
    float v = 0.f;
    if (n < N) {
      if (c < C) v = in[(size_t)c * N + n];
      else if (c < C + 3) v = __fmul_rn(__fsub_rn(xyz[(size_t)n * 3 + (c - C)], xyz[c - C]), inv_r);
    }
    tile[r][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int n = n0 + r, c = c0 + tx;
    if (n < N && c < Cpa) out[(size_t)n * Cpa + c] = tile[tx][r];
  }
}

// W (Cout, 3+2C) = [Wp | Wc | Wr], gamma -> wcat (2*Cop, C+3), wp (Cout,3), sgn (Cout)   (see file header)
__global__ void pwmlp_prep_kernel(const float* __restrict__ W, const float* __restrict__ gamma, int C, int Cout, int Cop,
                                  int Cpa, float* __restrict__ wcat, float* __restrict__ wp, float* __restrict__ sgn) {
  const int row = blockIdx.x;  // 0 .. 2*Cop-1
  const bool trow = row >= Cop;
  const int o = trow ? row - Cop : row;
  const int W3 = 3 + 2 * C;
  for (int c = threadIdx.x; c < Cpa; c += blockDim.x) {  // rows padded to Cpa (zeros): float4-friendly
    float v = 0.f;
    if (o < Cout && c < C + 3) {
      const float sg = gamma[o] >= 0.f ? 1.f : -1.f;
      if (!trow) v = c < C ? W[(size_t)o * W3 + 3 + c] - W[(size_t)o * W3 + 3 + C + c] : 0.f;
      else v = sg * (c < C ? W[(size_t)o * W3 + 3 + C + c] : W[(size_t)o * W3 + (c - C)]);
      if (!trow && c < 3) wp[o * 3 + c] = W[(size_t)o * W3 + c];
      if (!trow && c == 0) sgn[o] = sg;
    }
    wcat[(size_t)row * Cpa + c] = v;
  }
}

// gwcat (2*Cop, C+3), grad_wp (3,Cout), sgn -> gW (Cout, 3+2C) = [dWp | dWc | dWr]
__global__ void pwmlp_wgrad_kernel(const float* __restrict__ gwcat, const float* __restrict__ grad_wp,
                                   const float* __restrict__ sgn, int C, int Cout, int Cop, int Cpa,
                                   float* __restrict__ gW) {
  const int o = blockIdx.x;
  const int W3 = 3 + 2 * C;
  const float sg = sgn[o];
  const float* gA = gwcat + (size_t)o * Cpa;
  const float* gT = gwcat + (size_t)(Cop + o) * Cpa;
  for (int c = threadIdx.x; c < W3; c += blockDim.x) {
    float v;
    if (c < 3) v = sg * gT[C + c] + grad_wp[(size_t)c * Cout + o];  // Wp: T rows' xyz columns + the a' part
    else if (c < 3 + C) v = gA[c - 3];                               // Wc
    else v = sg * gT[c - 3 - C] - gA[c - 3 - C];                     // Wr
    gW[(size_t)o * W3 + c] = v;
  }
}

static int pw_ci(int Cop) {
  int ci = ceil_div(Cop, 32);
  return ci > kPWMaxCI ? kPWMaxCI : ci;
}

template <int CI>
static int launch_pw_fwd(const PwArgs& a, cudaStream_t stream) {
  const size_t smem = align_up((size_t)kPWWarps * a.K * 4, 16) + (size_t)32 * CI * (kPWTile + 1) * 4 +
                      (size_t)kPWWarps * 2 * 32 * CI * 4;
  static std::atomic<unsigned long long> seen{0};
  allow_big_smem(pwmlp_fwd_kernel<CI>, seen);
  dim3 grid(a.ntiles, ceil_div(a.Cop, 32 * CI));
  pwmlp_fwd_kernel<CI><<<grid, kPWWarps * 32, smem, stream>>>(a);
  CL3D_LAUNCHED(1);
  return check_launch("pwmlp_fwd_kernel");
}
template <int CI>
static int launch_pw_bwd(const PwArgs& a, int ntiles_n, int gx, cudaStream_t stream) {
  PwArgs d = a;
  d.ntiles = ntiles_n;
  pwmlp_bwd_dense_kernel<CI><<<dim3(gx, ceil_div(a.Cop, 32 * CI)), kPWWarps * 32, 0, stream>>>(d);
  CL3D_LAUNCHED(1);
  return check_launch("pwmlp_bwd_dense_kernel");
}

static int pw_dense_grid(int ntiles_n) {
  int gx = persistent_grid_cap();
  return gx > ntiles_n ? ntiles_n : gx;
}
static int pw_query_grid(int B, int M, int Cop) {
  const int ny = 256 / (Cop / 4 < kPWQGroups ? Cop / 4 : kPWQGroups);  // queries per CTA row (pwmlp_bwd_query_kernel)
  return (int)(((long long)B * M + (long long)ny * kPWQPT - 1) / ((long long)ny * kPWQPT));
}

}  // namespace cl3d

using namespace cl3d;

extern "C" int cl3d_to_point_major_aug(const float* in_cn, const float* xyz, int B, int C, int N, float radius,
                                       float* out_nc, cl3d_stream_t stream_) {
  CL3D_REQUIRE(in_cn && xyz && out_nc && B >= 0 && C >= 1 && N >= 1, "cl3d_to_point_major_aug: bad arguments");
  if (B == 0) return CL3D_OK;
  const int Cpa = padded_channels(C + 3);
  dim3 grid(ceil_div(N, 32), ceil_div(Cpa, 32), B);
  to_point_major_aug_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>(in_cn, xyz, C, N, Cpa, 1.0f / radius, out_nc);
  CL3D_LAUNCHED(1);
  return check_launch("to_point_major_aug_kernel");
}

extern "C" int cl3d_pwmlp_prep_weights(const float* conv_weight, const float* gamma, int C, int Cout, float* wcat,
                                       float* wp, float* sgn, cl3d_stream_t stream_) {
  CL3D_REQUIRE(conv_weight && gamma && wcat && wp && sgn && C >= 1 && Cout >= 1, "cl3d_pwmlp_prep_weights: bad arguments");
  const int Cop = padded_channels(Cout);
  pwmlp_prep_kernel<<<2 * Cop, 128, 0, (cudaStream_t)stream_>>>(conv_weight, gamma, C, Cout, Cop,
                                                                padded_channels(C + 3), wcat, wp, sgn);
  CL3D_LAUNCHED(1);
  return check_launch("pwmlp_prep_kernel");
}

extern "C" int cl3d_pwmlp_weight_grad(const float* gwcat, const float* grad_wp, const float* sgn, int C, int Cout,
                                      float* grad_conv_weight, cl3d_stream_t stream_) {
  CL3D_REQUIRE(gwcat && grad_wp && sgn && grad_conv_weight && C >= 1 && Cout >= 1, "cl3d_pwmlp_weight_grad: bad arguments");
  pwmlp_wgrad_kernel<<<Cout, 128, 0, (cudaStream_t)stream_>>>(gwcat, grad_wp, sgn, C, Cout, padded_channels(Cout),
                                                              padded_channels(C + 3), grad_conv_weight);
  CL3D_LAUNCHED(1);
  return check_launch("pwmlp_wgrad_kernel");
}

extern "C" int cl3d_pwmlp_fwd_stats(const float* ab_pm, const float* wp, const float* sgn, const float* query_xyz,
                                    const float* support_xyz, const int* idx, int B, int N, int M, int K, int Cout,
                                    float radius, float* ysel,
                                    float* aq, float* sq, unsigned char* karg, float* bn_partial,
                                    cl3d_stream_t stream_) {
  CL3D_REQUIRE(ab_pm && wp && sgn && query_xyz && support_xyz && idx && ysel && aq && sq && karg && bn_partial,
               "cl3d_pwmlp_fwd_stats: null pointer");
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 1 && K >= 1 && K <= 255 && Cout >= 1, "cl3d_pwmlp_fwd_stats: bad sizes (K <= 255)");
  if (B == 0) return CL3D_OK;
  PwArgs a = {};
  a.ab_pm = ab_pm; a.wp = wp; a.sgn = sgn; a.query_xyz = query_xyz; a.support_xyz = support_xyz; a.idx = idx;
  a.ysel = ysel; a.aq = aq; a.sq = sq; a.karg = karg; a.partial = bn_partial;
  a.B = B; a.N = N; a.M = M; a.K = K; a.Cout = Cout; a.Cop = padded_channels(Cout);
  a.inv_radius = 1.0f / radius;
  a.ntiles = B * ceil_div(M, kPWTile);
  switch (pw_ci(a.Cop)) {
    case 1: return launch_pw_fwd<1>(a, (cudaStream_t)stream_);
    case 2: return launch_pw_fwd<2>(a, (cudaStream_t)stream_);
    case 3: return launch_pw_fwd<3>(a, (cudaStream_t)stream_);
    default: return launch_pw_fwd<4>(a, (cudaStream_t)stream_);
  }
}

extern "C" int cl3d_pwmlp_fwd_out(const float* ysel, const float* save_stats, const float* gamma, const float* beta,
                                  int B, int M, int Cout, float* out, cl3d_stream_t stream_) {
  CL3D_REQUIRE(ysel && save_stats && gamma && beta && out && B >= 0 && M >= 1 && Cout >= 1,
               "cl3d_pwmlp_fwd_out: bad arguments");
  if (B == 0) return CL3D_OK;
  int chunks = ceil_div(M, 1024);
  chunks = chunks < 1 ? 1 : (chunks > 65535 ? 65535 : chunks);
  pwmlp_out_kernel<<<dim3(B * Cout, chunks), 256, 0, (cudaStream_t)stream_>>>(ysel, save_stats, gamma, beta, Cout, M, out);
  CL3D_LAUNCHED(1);
  return check_launch("pwmlp_out_kernel");
}

extern "C" size_t cl3d_pwmlp_bwd_scratch_floats(int B, int N, int M, int Cout) {
  const int Cop = padded_channels(Cout);
  (void)N;
  const size_t ntm = (size_t)B * ceil_div(M, kPWTile), gq = (size_t)pw_query_grid(B, M, Cop);
  const size_t part = (ntm * 2 > gq * 3 ? ntm * 2 : gq * 3) * (size_t)Cout;
  return part + (size_t)B * M * Cop + 64;
}

// fork/join events of cl3d_pwmlp_bwd: a small per-device ring of event sets, so that several calls can be in
// flight (each call only orders its own streams; an event is reusable as soon as the waits on it are enqueued)
struct PwEvents {
  cudaEvent_t start, zeroed, stats, joined;
};
static PwEvents* pw_events() {
  constexpr int kDevs = 64, kRing = 16;
  static PwEvents ring[kDevs][kRing];
  static bool made[kDevs] = {};
  static unsigned next[kDevs] = {};
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kDevs) return nullptr;
  if (!made[dev]) {
    for (int i = 0; i < kRing; ++i) {
      cudaEvent_t* e[4] = {&ring[dev][i].start, &ring[dev][i].zeroed, &ring[dev][i].stats, &ring[dev][i].joined};
      for (auto p : e)
        if (cudaEventCreateWithFlags(p, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    }
    made[dev] = true;
  }
  return &ring[dev][next[dev]++ % kRing];
}

extern "C" int cl3d_pwmlp_bwd(const float* grad_out, const float* out, const float* ab_pm, const float* wp,
                              const float* sgn, const float* query_xyz, const float* support_xyz, const int* idx,
                              const int* csr_off, const int* csr_ent, const float* ysel, const float* aq, const float* sq,
                              const unsigned char* karg, const float* save_stats, const float* gamma, int B, int N,
                              int M, int K, int Cout, float radius, int training, float* scratch,
                              float* dgamma_dbeta, float* grad_ab_pm, float* grad_wp, cl3d_stream_t stream_,
                              cl3d_stream_t side_stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  // With a side stream the zero-fill of grad_ab and the latency-bound query pass run beside the statistics and
  // the support-major gather (fork/join with events: capturable into a CUDA graph); without one, in order.
  cudaStream_t side = side_stream_ ? (cudaStream_t)side_stream_ : stream;
  const bool forked = side != stream;
  PwEvents* ev = forked ? pw_events() : nullptr;
  if (forked && !ev) return CL3D_ERR_LAUNCH;
  CL3D_REQUIRE(grad_out && out && ab_pm && wp && sgn && query_xyz && support_xyz && idx && ysel && aq && sq &&
                   karg && save_stats && gamma && scratch && dgamma_dbeta && grad_ab_pm && grad_wp,
               "cl3d_pwmlp_bwd: null pointer");
  CL3D_REQUIRE(!training || (csr_off && csr_ent), "cl3d_pwmlp_bwd: training mode needs the all-slots CSR lists");
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 1 && K >= 1 && K <= 255 && Cout >= 1, "cl3d_pwmlp_bwd: bad sizes");
  if (B == 0) return CL3D_OK;
  const int ntiles = B * ceil_div(M, kPWTile);
  const int ntn = B * ceil_div(N, kPWTile);
  const int gx = pw_dense_grid(ntn);
  const int Cop = padded_channels(Cout);
  // scratch = [ partials (max(ntiles*2, gx*3) * Cout) | dzs_pm (B*M*Cop) ]
  const int gqy = pw_query_grid(B, M, Cop);
  const size_t part = ((size_t)ntiles * 2 > (size_t)gqy * 3 ? (size_t)ntiles * 2 : (size_t)gqy * 3) * (size_t)Cout;
  float* partial = scratch;
  float* dzs_pm = scratch + ((part + 63) / 64) * 64;
  const size_t smem_s = (size_t)kPWTile * (Cop + 1) * sizeof(float);
  static std::atomic<unsigned long long> seen_stats{0};
  allow_big_smem(pwmlp_bwd_stats_kernel, seen_stats);
  if (forked) {
    cudaEventRecord(ev->start, stream);
    cudaStreamWaitEvent(side, ev->start, 0);
  }
  cudaMemsetAsync(grad_ab_pm, 0, sizeof(float) * (size_t)B * N * 2 * Cop, side);
  if (forked) cudaEventRecord(ev->zeroed, side);
  pwmlp_bwd_stats_kernel<<<ntiles, 256, smem_s, stream>>>(grad_out, out, ysel, save_stats, gamma, Cout, Cop, M, partial,
                                                          dzs_pm);
  CL3D_LAUNCHED(1);
  int rc = cl3d_reduce_partials(partial, ntiles, 2 * Cout, dgamma_dbeta, stream_);  // (dgamma, dbeta)
  if (rc) return rc;
  if (forked) {
    cudaEventRecord(ev->stats, stream);
    cudaStreamWaitEvent(side, ev->stats, 0);   // the query pass needs (dgamma, dbeta) and sc*dz
    cudaStreamWaitEvent(stream, ev->zeroed, 0);  // the gather pass needs the zero-filled grad_ab
  }
  PwArgs a = {};
  a.ab_pm = ab_pm; a.wp = wp; a.sgn = sgn; a.query_xyz = query_xyz; a.support_xyz = support_xyz; a.idx = idx;
  a.ysel = const_cast<float*>(ysel); a.aq = const_cast<float*>(aq); a.sq = const_cast<float*>(sq);
  a.karg = const_cast<unsigned char*>(karg);
  a.partial = partial;
  a.grad_out = grad_out; a.out = out; a.stats = save_stats; a.gamma = gamma; a.dgb = dgamma_dbeta;
  a.csr_off = csr_off; a.csr_ent = csr_ent;
  a.grad_ab_pm = grad_ab_pm;
  a.dzs_pm = dzs_pm;
  a.B = B; a.N = N; a.M = M; a.K = K; a.Cout = Cout; a.Cop = Cop;
  a.inv_radius = 1.0f / radius;
  // eval mode (frozen BatchNorm): the batch-statistics terms c1, c2 vanish (inv_count = 0 zeroes them in the query
  // pass) and the dense support-major pass would add exact zeros, so it is not launched
  a.inv_count = training ? 1.0f / (float)((double)B * M * K) : 0.f;
  a.ntiles = ntiles;
  if (training) {
    switch (pw_ci(Cop)) {
      case 1: rc = launch_pw_bwd<1>(a, ntn, gx, stream); break;
      case 2: rc = launch_pw_bwd<2>(a, ntn, gx, stream); break;
      case 3: rc = launch_pw_bwd<3>(a, ntn, gx, stream); break;
      default: rc = launch_pw_bwd<4>(a, ntn, gx, stream); break;
    }
    if (rc) return rc;
  }
  const int nx = Cop / 4 < kPWQGroups ? Cop / 4 : kPWQGroups, ny = 256 / nx;
  pwmlp_bwd_query_kernel<<<dim3(gqy, ceil_div(Cop / 4, nx)), ny * nx, (size_t)ny * 3 * Cop * sizeof(float), side>>>(
      a, (long long)B * M);
  CL3D_LAUNCHED(1);
  rc = check_launch("pwmlp_bwd_query_kernel");
  if (rc) return rc;
  rc = cl3d_reduce_partials(partial, gqy, 3 * Cout, grad_wp, (cl3d_stream_t)side);
  if (forked) {
    cudaEventRecord(ev->joined, side);
    cudaStreamWaitEvent(stream, ev->joined, 0);
  }
  return rc;
}
