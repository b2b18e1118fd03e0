// gemm.cu -- fp32 GEMM with arbitrary element strides and optional split-K (sm_90a).
//
// Used for the per-point products of the fused PointWiseMLP (see pwmlp.cu): the reference's per-neighbour
// 1x1 conv over [dp; f_i; f_j - f_i] (/root/reference/pytorch/models/local_aggregation_operators.py:254-257,
// 288-295) becomes ONE per-point product (B*N x (C+3)) x ((C+3) x 2*Cout), plus its two gradients.
//
//   C[m][n] = sum_k A[m*sa_m + k*sa_k] * B[k*sb_k + n*sb_n]
//
// Two implementations behind cl3d_sgemm_algo:
//   CL3D_GEMM_TC3X (default): wgmma tensor cores, every operand split into two TF32 halves and three MMAs
//     per product (gemm_tc.cuh) -- fp32-level accuracy, within the 1e-5 parity bar (BASELINE.json north_star);
//   CL3D_GEMM_FFMA: the vectorised fp32 FMA kernel below (plain TF32/BF16 would break the parity bar).
//
// FFMA kernel: CTA tile 128 x (16*TN), k tile 16, 256 threads, 8 x TN outputs per thread (TN chosen from N so that skinny
// outputs waste few columns), operands transposed into shared memory as [k][m] / [k][n] (LDS.128 for the A
// fragment), next k tile prefetched into registers while the current one is multiplied.  With splitk > 1 the k
// range is divided among gridDim.z CTAs that write partial tiles, reduced afterwards in a fixed order.
#include "common.cuh"
#include "gemm_tc.cuh"

namespace cl3d {

constexpr int kBM = 128, kBK = 16;

template <int TN, bool VEC>
__global__ void __launch_bounds__(256) sgemm_tiled_kernel(const float* __restrict__ A, long long sa_m, long long sa_k,
                                                          const float* __restrict__ B, long long sb_k,
                                                          long long sb_n, int M, int N, int K, int k_per_split,
                                                          float* __restrict__ C, long long ldc,
                                                          float* __restrict__ partial) {
  constexpr int BN = 16 * TN;
  __shared__ __align__(16) float sA[kBK][kBM + 4];
  __shared__ __align__(16) float sB[kBK][BN + 4];
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split, kend = min(K, kbeg + k_per_split);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const bool a_k_fast = (sa_k == 1), b_k_fast = (sb_k == 1);
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  // VEC: every operand is read as float4 along its unit-stride dimension (host guarantees 16-byte alignment,
  // strides and extents that are multiples of 4, so a vector is entirely inside or entirely outside)
  constexpr int NVB = (BN * kBK / 4 + 255) / 256;  // float4 of the B tile per thread
  float ra[8], rb[VEC ? NVB * 4 : TN];

  auto load_tiles = [&](int k0) {
    if constexpr (VEC) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int e = threadIdx.x + 256 * r;  // 512 float4 of the A tile
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a_k_fast) {
          const int mm = e >> 2, kk = (e & 3) * 4;
          const int m = m0 + mm, k = k0 + kk;
          if (m < M && k < kend) v = __ldg(reinterpret_cast<const float4*>(A + m * sa_m + k));
        } else {
          const int kk = e >> 5, mm = (e & 31) * 4;
          const int m = m0 + mm, k = k0 + kk;
          if (m < M && k < kend) v = __ldg(reinterpret_cast<const float4*>(A + k * sa_k + m));
        }
        ra[r * 4 + 0] = v.x; ra[r * 4 + 1] = v.y; ra[r * 4 + 2] = v.z; ra[r * 4 + 3] = v.w;
      }
#pragma unroll
      for (int r = 0; r < NVB; ++r) {
        const int e = threadIdx.x + 256 * r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < BN * kBK / 4) {
          if (b_k_fast) {
            const int nn = e >> 2, kk = (e & 3) * 4;
            const int n = n0 + nn, k = k0 + kk;
            if (n < N && k < kend) v = __ldg(reinterpret_cast<const float4*>(B + n * sb_n + k));
          } else {
            const int kk = e / (BN / 4), nn = (e % (BN / 4)) * 4;
            const int n = n0 + nn, k = k0 + kk;
            if (n < N && k < kend) v = __ldg(reinterpret_cast<const float4*>(B + k * sb_k + n));
          }
        }
        rb[r * 4 + 0] = v.x; rb[r * 4 + 1] = v.y; rb[r * 4 + 2] = v.z; rb[r * 4 + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int e = threadIdx.x + 256 * r;
        const int mm = a_k_fast ? e / kBK : e % kBM, kk = a_k_fast ? e % kBK : e / kBM;
        const int m = m0 + mm, k = k0 + kk;
        ra[r] = (m < M && k < kend) ? __ldg(A + m * sa_m + k * sa_k) : 0.f;
      }
#pragma unroll
      for (int r = 0; r < TN; ++r) {
        const int e = threadIdx.x + 256 * r;
        const int nn = b_k_fast ? e / kBK : e % BN, kk = b_k_fast ? e % kBK : e / BN;
        const int n = n0 + nn, k = k0 + kk;
        rb[r] = (n < N && k < kend) ? __ldg(B + k * sb_k + n * sb_n) : 0.f;
      }
    }
  };
  auto store_tiles = [&]() {
    if constexpr (VEC) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int e = threadIdx.x + 256 * r;
        if (a_k_fast) {
          const int mm = e >> 2, kk = (e & 3) * 4;
#pragma unroll
          for (int t = 0; t < 4; ++t) sA[kk + t][mm] = ra[r * 4 + t];
        } else {
          const int kk = e >> 5, mm = (e & 31) * 4;
          *reinterpret_cast<float4*>(&sA[kk][mm]) = make_float4(ra[r * 4], ra[r * 4 + 1], ra[r * 4 + 2], ra[r * 4 + 3]);
        }
      }
#pragma unroll
      for (int r = 0; r < NVB; ++r) {
        const int e = threadIdx.x + 256 * r;
        if (e < BN * kBK / 4) {
          if (b_k_fast) {
            const int nn = e >> 2, kk = (e & 3) * 4;
#pragma unroll
            for (int t = 0; t < 4; ++t) sB[kk + t][nn] = rb[r * 4 + t];
          } else {
            const int kk = e / (BN / 4), nn = (e % (BN / 4)) * 4;
            *reinterpret_cast<float4*>(&sB[kk][nn]) = make_float4(rb[r * 4], rb[r * 4 + 1], rb[r * 4 + 2], rb[r * 4 + 3]);
          }
        }
      }
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int e = threadIdx.x + 256 * r;
        const int mm = a_k_fast ? e / kBK : e % kBM, kk = a_k_fast ? e % kBK : e / kBM;
        sA[kk][mm] = ra[r];
      }
#pragma unroll
      for (int r = 0; r < TN; ++r) {
        const int e = threadIdx.x + 256 * r;
        const int nn = b_k_fast ? e / kBK : e % BN, kk = b_k_fast ? e % kBK : e / BN;
        sB[kk][nn] = rb[r];
      }
    }
  };

  load_tiles(kbeg);
  for (int k0 = kbeg; k0 < kend; k0 += kBK) {
    store_tiles();
    __syncthreads();
    if (k0 + kBK < kend) load_tiles(k0 + kBK);  // prefetch the next k tile into registers
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&sA[kk][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&sA[kk][ty * 8 + 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[TN];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = sB[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 8 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n >= N) continue;
      if (partial)
        partial[(size_t)blockIdx.z * M * N + (size_t)m * N + n] = acc[i][j];
      else
        C[(size_t)m * ldc + n] = acc[i][j];
    }
  }
}

// Fixed-order split-K reduction: 32 outputs x 8 slices per CTA; slice j sums splits j, j+8, ... in double,
// the 8 slice sums are combined in a fixed order.  C[m*sc_m + n*sc_n] for the partial element (m, n).
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ partial, int splits, int M, int N,
                                                            float* __restrict__ C, long long sc_m, long long sc_n) {
  __shared__ double red[8][33];
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const long long e = (long long)blockIdx.x * 32 + lane;
  const size_t stride = (size_t)M * N;
  double a0 = 0.0, a1 = 0.0;
  if (e < (long long)stride) {
    int s = slice;
    for (; s + 8 < splits; s += 16) {
      a0 += (double)partial[(size_t)s * stride + e];
      a1 += (double)partial[(size_t)(s + 8) * stride + e];
    }
    if (s < splits) a0 += (double)partial[(size_t)s * stride + e];
  }
  red[slice][lane] = a0 + a1;
  __syncthreads();
  if (slice == 0 && e < (long long)stride) {
    double t = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += red[j][lane];
    C[(e / N) * sc_m + (e % N) * sc_n] = (float)t;
  }
}

template <int TN>
static void launch_sgemm(dim3 grid, cudaStream_t stream, const float* a, long long sa_m, long long sa_k, const float* b,
                         long long sb_k, long long sb_n, int M, int N, int K, int kps, float* c, long long ldc,
                         float* partial) {
  // float4 path: unit stride along one dimension of each operand, everything else a multiple of 4 floats
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool va = al16(a) && ((sa_k == 1 && sa_m % 4 == 0 && K % 4 == 0 && kps % 4 == 0) ||
                              (sa_m == 1 && sa_k % 4 == 0 && M % 4 == 0));
  const bool vb = al16(b) && ((sb_k == 1 && sb_n % 4 == 0 && K % 4 == 0 && kps % 4 == 0) ||
                              (sb_n == 1 && sb_k % 4 == 0 && N % 4 == 0));
  if (va && vb && (sa_k == 1 || sa_m == 1) && (sb_k == 1 || sb_n == 1))
    sgemm_tiled_kernel<TN, true><<<grid, 256, 0, stream>>>(a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial);
  else
    sgemm_tiled_kernel<TN, false><<<grid, 256, 0, stream>>>(a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial);
  CL3D_LAUNCHED(1);
}

}  // namespace cl3d

using namespace cl3d;

extern "C" size_t cl3d_sgemm_workspace_bytes(int M, int N, int splitk) {
  return splitk > 1 ? sizeof(float) * (size_t)splitk * M * N : 0;
}

static int sgemm_ffma(const float* a, long long sa_m, long long sa_k, const float* b, long long sb_k, long long sb_n,
                      int M, int N, int K, float* c, long long ldc, int splitk, float* partial, cudaStream_t stream) {
  int kps = ceil_div(K, splitk);
  kps = ceil_div(kps, kBK) * kBK;
  splitk = ceil_div(K, kps);
  if (splitk == 1) partial = nullptr;
  // columns per thread: spread N over the fewest 144-wide column tiles, then round each tile up to 16*TN
  const int nct = ceil_div(N, 144);
  int tn = ceil_div(ceil_div(N, nct), 16);
  if (tn < 1) tn = 1;
  if (tn > 9) tn = 9;
  dim3 grid(ceil_div(N, 16 * tn), ceil_div(M, kBM), splitk);
  switch (tn) {
    case 1: launch_sgemm<1>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 2: launch_sgemm<2>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 3: launch_sgemm<3>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 4: launch_sgemm<4>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 5: launch_sgemm<5>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 6: launch_sgemm<6>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 7: launch_sgemm<7>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    case 8: launch_sgemm<8>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
    default: launch_sgemm<9>(grid, stream, a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, kps, c, ldc, partial); break;
  }
  if (partial) {
    const long long total = (long long)M * N;
    splitk_reduce_kernel<<<(unsigned)((total + 31) / 32), 256, 0, stream>>>(partial, splitk, M, N, c, ldc, 1);
    CL3D_LAUNCHED(1);
  }
  return check_launch("sgemm_tiled_kernel");
}

// staged floats per k of one problem orientation: (#row tiles) x (#column tiles) x (128 + columns per tile)
static long long tc_cost(int M, int N) {
  const int nt = ceil_div(N, kTcMaxN);
  return (long long)ceil_div(M, kTcBM) * nt * (kTcBM + tc_tile_n(N));
}

static int sgemm_tc(const float* a, long long sa_m, long long sa_k, const float* b, long long sb_k, long long sb_n,
                    int M, int N, int K, float* c, long long ldc, int splitk, float* partial, cudaStream_t stream) {
  TcGemmArgs g{};
  // C^T = B^T A^T when that orientation stages fewer operand rows (e.g. a 144 x 80 weight gradient: one
  // 80(->128) x 144 tile instead of two 128 x 80 tiles)
  // (only for short M: a long M already fills the machine, and the transposed epilogue is the slower one)
  const bool swap = M <= 256 && tc_cost(N, M) < tc_cost(M, N);
  if (!swap) {
    g.A = a; g.sa_m = sa_m; g.sa_k = sa_k; g.B = b; g.sb_k = sb_k; g.sb_n = sb_n;
    g.M = M; g.N = N; g.sc_m = ldc; g.sc_n = 1;
  } else {
    g.A = b; g.sa_m = sb_n; g.sa_k = sb_k; g.B = a; g.sb_k = sa_k; g.sb_n = sa_m;
    g.M = N; g.N = M; g.sc_m = 1; g.sc_n = ldc;
  }
  g.K = K;
  int kps = ceil_div(K, splitk);
  kps = ceil_div(kps, kTcBK) * kTcBK;
  splitk = ceil_div(K, kps);
  g.k_per_split = kps;
  g.C = c;
  g.partial = splitk > 1 ? partial : nullptr;
  if (!tc_gemm_supported(g)) return 1;  // caller falls back to the FMA kernel
  tc_gemm_launch(g, splitk, stream);
  CL3D_LAUNCHED(1);
  if (g.partial) {
    const long long total = (long long)M * N;
    splitk_reduce_kernel<<<(unsigned)((total + 31) / 32), 256, 0, stream>>>(partial, splitk, g.M, g.N, c, g.sc_m,
                                                                             g.sc_n);
    CL3D_LAUNCHED(1);
  }
  return check_launch("gemm_tf32x3_kernel");
}

extern "C" int cl3d_sgemm_algo(const float* a, long long sa_m, long long sa_k, const float* b, long long sb_k,
                               long long sb_n, int M, int N, int K, float* c, long long ldc, int splitk,
                               void* workspace, size_t workspace_bytes, int algo, cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(a && b && c && M >= 1 && N >= 1 && K >= 1 && ldc >= N, "cl3d_sgemm: bad arguments");
  CL3D_REQUIRE(algo == CL3D_GEMM_AUTO || algo == CL3D_GEMM_FFMA || algo == CL3D_GEMM_TC3X, "cl3d_sgemm: bad algo");
  if (splitk < 1) splitk = 1;
  if (splitk > K) splitk = K;
  CL3D_REQUIRE(splitk <= 65535, "cl3d_sgemm: splitk too large");
  float* partial = nullptr;
  if (splitk > 1) {
    if (!workspace || workspace_bytes < cl3d_sgemm_workspace_bytes(M, N, splitk)) {
      set_error("cl3d_sgemm: split-K workspace too small");
      return CL3D_ERR_WORKSPACE;
    }
    partial = (float*)workspace;
  }
  // AUTO leaves un-split reductions longer than 512 to the FMA kernel; the tensor-core kernel bounds the
  // truncation of its accumulators by promoting them every 64 k (gemm_tc.cuh), so CL3D_GEMM_TC3X stays within
  // the fp32 bar there too.
  if (algo == CL3D_GEMM_AUTO && ceil_div(K, splitk) > 512) algo = CL3D_GEMM_FFMA;
  if (algo != CL3D_GEMM_FFMA) {
    const int rc = sgemm_tc(a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, c, ldc, splitk, partial, stream);
    if (rc <= 0) return rc;
    if (algo == CL3D_GEMM_TC3X) {
      set_error("cl3d_sgemm: operand extent exceeds the 32-bit offsets of the tensor-core kernel");
      return CL3D_ERR_UNSUPPORTED;
    }
  }
  return sgemm_ffma(a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, c, ldc, splitk, partial, stream);
}
