// pool.cu -- fused neighbourhood max-pool (the body of the reference's MaskedMaxPool,
//   /root/reference/pytorch/ops/pt_custom_ops/pt_utils.py:188-202: group_points -> F.max_pool2d over K)
// and its gradient, without the (B,C,M,K) tensor.  Also used by MaskedUpsample(mode='max').
//
// forward : warp per query, lane = channel, neighbour rows of the point-major feature matrix streamed with
//           coalesced loads; max over ALL K slots (the reference ignores masks here; cyclic padding duplicates
//           cannot change a max), first arg-max slot kept (max_pool2d's tie rule) for the backward.
// backward: grad_f[b, c, idx[b,q,arg]] += grad_out[b,c,q]  -- one fp32 red.add row per query into a zeroed
//           point-major buffer (the reference scatters K times as many atomics through group_points_grad); a CTA stages
//           the grad_out of its 32 queries in shared memory, 32 x (C + 1) floats, so a layer wider than the 227 KB
//           opt-in allows (C > 1815: the width x2 network's layer4 pool, C = 2304) runs as equal channel chunks of a
//           multiple of 32 over blockIdx.y; or, given the transposed lists of idx, the same sum gathered per support
//           point in list order (deterministic mode).
#include "common.cuh"

namespace cl3d {

constexpr int kPoolWarps = 8;
constexpr int kPoolTile = 32;
constexpr int kPoolU = 4;

template <int CI, typename T>
__global__ void __launch_bounds__(kPoolWarps * 32) gather_max_fwd_kernel(const float* __restrict__ feat_pm,
                                                                         const int* __restrict__ idx, int N, int M,
                                                                         int K, int C, int Cp, T* __restrict__ out,
                                                                         unsigned char* __restrict__ arg) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int chunkC = min(32 * CI, Cp - c0);
  unsigned* s_off = reinterpret_cast<unsigned*>(smem) + (size_t)warp * K;
  float* s_out = reinterpret_cast<float*>(smem + align_up((size_t)kPoolWarps * K * 4, 16));
  const int tiles_per_cloud = (M + kPoolTile - 1) / kPoolTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kPoolTile;
  const float* base = feat_pm + (size_t)b * N * Cp + c0 + lane;
  for (int ql = warp; ql < kPoolTile; ql += kPoolWarps) {
    const int q = q0 + ql;
    float m[CI];
    int km[CI];
#pragma unroll
    for (int i = 0; i < CI; ++i) { m[i] = -INFINITY; km[i] = 0; }
    if (q < M) {
      const size_t gq = (size_t)b * M + q;
      for (int k = lane; k < K; k += 32) s_off[k] = (unsigned)idx[gq * K + k] * (unsigned)Cp;
      __syncwarp();
      int k0 = 0;
      for (; k0 + kPoolU <= K; k0 += kPoolU) {
        float v[kPoolU][CI];
#pragma unroll
        for (int u = 0; u < kPoolU; ++u) {
          const float* row = base + s_off[k0 + u];
#pragma unroll
          for (int i = 0; i < CI; ++i) v[u][i] = __ldg(row + 32 * i);
        }
#pragma unroll
        for (int u = 0; u < kPoolU; ++u)
#pragma unroll
          for (int i = 0; i < CI; ++i) {
            const bool gt = v[u][i] > m[i];
            m[i] = gt ? v[u][i] : m[i];
            km[i] = gt ? k0 + u : km[i];
          }
      }
      for (; k0 < K; ++k0) {
        const float* row = base + s_off[k0];
#pragma unroll
        for (int i = 0; i < CI; ++i) {
          const float t = __ldg(row + 32 * i);
          const bool gt = t > m[i];
          m[i] = gt ? t : m[i];
          km[i] = gt ? k0 : km[i];
        }
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < CI; ++i)
        if (lane + 32 * i < chunkC) arg[gq * Cp + c0 + lane + 32 * i] = (unsigned char)km[i];
    }
#pragma unroll
    for (int i = 0; i < CI; ++i) s_out[(size_t)(lane + 32 * i) * (kPoolTile + 1) + ql] = m[i];
  }
  __syncthreads();
  const int q = q0 + lane;
  for (int cl = warp; cl < 32 * CI; cl += kPoolWarps) {
    const int c = c0 + cl;
    if (c >= C) break;
    if (q < M) store_f32(out + ((size_t)b * C + c) * M + q, s_out[(size_t)cl * (kPoolTile + 1) + lane]);
  }
}

// grad_pm[b, idx[b,q,arg[b,q,c]], c] += grad_out[b,c,q] for the channels c0 <= c < c0 + chunk of blockIdx.y
template <typename T>
__global__ void __launch_bounds__(256) gather_max_bwd_kernel(const T* __restrict__ grad_out,
                                                             const int* __restrict__ idx,
                                                             const unsigned char* __restrict__ arg, int N, int M, int K,
                                                             int C, int Cp, int chunk, float* __restrict__ grad_pm) {
  extern __shared__ float s_g[];  // [32 queries][Cc + 1]
  const int tiles_per_cloud = (M + 31) / 32;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * 32;
  const int c0 = blockIdx.y * chunk;
  const int Cc = min(chunk, C - c0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const T* g = grad_out + ((size_t)b * C + c0) * M + q0;
  for (int c = warp; c < Cc; c += 8)
    s_g[(size_t)lane * (Cc + 1) + c] = q0 + lane < M ? load_f32(g + (size_t)c * M + lane) : 0.f;
  __syncthreads();
  const unsigned char* a = arg + ((size_t)b * M + q0) * Cp + c0;
  const int* id = idx + ((size_t)b * M + q0) * K;
  float* gp = grad_pm + (size_t)b * N * Cp + c0;
  for (int ql = warp; ql < 32; ql += 8) {
    if (q0 + ql >= M) continue;
    for (int c = lane; c < Cc; c += 32) {
      const int j = id[ql * K + a[(size_t)ql * Cp + c]];
      atomicAdd(gp + (size_t)j * Cp + c, s_g[(size_t)ql * (Cc + 1) + c]);
    }
  }
}

// gather form over the transposed lists of idx (all K slots, cl3d_build_csr): one warp per support point j, lane =
// channel; grad_pm[b,j,c] = sum over the list's entries q*K + k with arg[b,q,c] == k of grad_out[b,c,q], in list
// order, so canonical lists give the same bits on every run.  Every row is written, padded channels with 0.
template <typename T>
__global__ void __launch_bounds__(256) gather_max_bwd_csr_kernel(const T* __restrict__ grad_out,
                                                                 const unsigned char* __restrict__ arg,
                                                                 const int* __restrict__ csr_off,
                                                                 const int* __restrict__ csr_ent, int B, int N, int M,
                                                                 int K, int C, int Cp, float* __restrict__ grad_pm) {
  const long long gw = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (gw >= (long long)B * N) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(gw / N), j = (int)(gw - (long long)b * N);
  const int o0 = csr_off[(size_t)b * (N + 1) + j], o1 = csr_off[(size_t)b * (N + 1) + j + 1];
  const int* ent = csr_ent + (size_t)b * M * K;
  const unsigned char* a = arg + (size_t)b * M * Cp;
  float* row = grad_pm + ((size_t)b * N + j) * Cp;
  for (int c = lane; c < Cp; c += 32) {
    float acc = 0.f;
    if (c < C) {
      const T* g = grad_out + ((size_t)b * C + c) * M;
      for (int p = o0; p < o1; ++p) {
        const int e = ent[p];
        const int q = e / K;
        if (a[(size_t)q * Cp + c] == e - q * K) acc += load_f32(g + q);
      }
    }
    row[c] = acc;
  }
}

template <int CI, typename T>
static int launch_pool_fwd(const float* feat_pm, const int* idx, int B, int N, int M, int K, int C, int Cp, T* out,
                           unsigned char* arg, cudaStream_t stream) {
  const size_t smem = align_up((size_t)kPoolWarps * K * 4, 16) + (size_t)32 * CI * (kPoolTile + 1) * 4;
  static std::atomic<unsigned long long> seen{0};
  allow_big_smem(gather_max_fwd_kernel<CI, T>, seen);
  dim3 grid(B * ceil_div(M, kPoolTile), ceil_div(Cp, 32 * CI));
  gather_max_fwd_kernel<CI, T><<<grid, kPoolWarps * 32, smem, stream>>>(feat_pm, idx, N, M, K, C, Cp, out, arg);
  CL3D_LAUNCHED(1);
  return check_launch("gather_max_fwd_kernel");
}

}  // namespace cl3d

using namespace cl3d;

extern "C" int cl3d_gather_max_fwd(const float* feat_pm, const int* idx, int B, int N, int M, int K, int C,
                                   void* out, int dtype, unsigned char* arg, cl3d_stream_t stream_) {
  CL3D_REQUIRE(feat_pm && idx && out && arg && B >= 0 && N >= 1 && M >= 1 && K >= 1 && K <= 255 && C >= 1,
               "cl3d_gather_max_fwd: bad arguments (K <= 255)");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_gather_max_fwd");
  if (B == 0) return CL3D_OK;
  const int Cp = padded_channels(C);
  int ci = ceil_div(Cp, 32);
  if (ci > 4) ci = 4;
  cudaStream_t s = (cudaStream_t)stream_;
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    T* o = static_cast<T*>(out);
    switch (ci) {
      case 1: return launch_pool_fwd<1>(feat_pm, idx, B, N, M, K, C, Cp, o, arg, s);
      case 2: return launch_pool_fwd<2>(feat_pm, idx, B, N, M, K, C, Cp, o, arg, s);
      case 3: return launch_pool_fwd<3>(feat_pm, idx, B, N, M, K, C, Cp, o, arg, s);
      default: return launch_pool_fwd<4>(feat_pm, idx, B, N, M, K, C, Cp, o, arg, s);
    }
  });
}

extern "C" int cl3d_gather_max_bwd(const void* grad_out, int dtype, const int* idx, const unsigned char* arg, int B,
                                   int N, int M, int K, int C, const int* csr_off, const int* csr_ent, float* grad_pm,
                                   cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(grad_out && idx && arg && grad_pm && B >= 0 && N >= 1 && M >= 1 && K >= 1 && C >= 1,
               "cl3d_gather_max_bwd: bad arguments");
  CL3D_REQUIRE(!csr_off == !csr_ent, "cl3d_gather_max_bwd: csr_off and csr_ent are both given or both NULL");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_gather_max_bwd");
  if (B == 0) return CL3D_OK;
  const int Cp = padded_channels(C);
  if (csr_off) {
    return with_dtype(dtype, [&](auto t) {
      using T = typename decltype(t)::type;
      const long long rows = (long long)B * N;
      gather_max_bwd_csr_kernel<T><<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(
          static_cast<const T*>(grad_out), arg, csr_off, csr_ent, B, N, M, K, C, Cp, grad_pm);
      CL3D_LAUNCHED(1);
      return check_launch("gather_max_bwd_csr_kernel");
    });
  }
  cudaMemsetAsync(grad_pm, 0, sizeof(float) * (size_t)B * N * Cp, stream);
  // all C channels in one CTA while its 32 x (C + 1) staged floats fit (C <= 1815), else the fewest equal chunks of a
  // multiple of 32 channels that do
  int chunk = C;
  if ((size_t)32 * (C + 1) * sizeof(float) > (size_t)kMaxDynSmem) {
    const int most = (kMaxDynSmem / (32 * (int)sizeof(float)) - 1) / 32 * 32;
    chunk = ceil_div(ceil_div(C, ceil_div(C, most)), 32) * 32;
  }
  const size_t smem = (size_t)32 * (chunk + 1) * sizeof(float);
  const dim3 grid(B * ceil_div(M, 32), ceil_div(C, chunk));
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(gather_max_bwd_kernel<T>, seen);
    gather_max_bwd_kernel<T><<<grid, 256, smem, stream>>>(static_cast<const T*>(grad_out), idx, arg, N, M, K, C, Cp,
                                                          chunk, grad_pm);
    CL3D_LAUNCHED(1);
    return check_launch("gather_max_bwd_kernel");
  });
}
