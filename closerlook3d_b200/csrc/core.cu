// core.cu -- error reporting, device queries, layout transposes, compatibility gather/scatter.
#include <stdarg.h>
#include <string.h>

#include <stdlib.h>

#include <type_traits>

#include "common.cuh"

namespace cl3d {

static thread_local char g_err[512] = "";
static long long g_launches = 0;
void count_launches(int n) { __atomic_fetch_add(&g_launches, (long long)n, __ATOMIC_RELAXED); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA error: %s", what, cudaGetErrorString(e));
    return CL3D_ERR_LAUNCH;
  }
  return CL3D_OK;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kNumSMsFallback;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kNumSMsFallback;
    cached[dev] = n;
  }
  return cached[dev];
}

// Grid size of the persistent (tile-loop) kernels: 4 CTAs per SM.  CL3D_TEST_MAX_GRID (read on every call, tests
// only) caps it so that small inputs run several tiles per CTA.
int persistent_grid_cap() {
  int cap = sm_count() * 4;
  const char* e = getenv("CL3D_TEST_MAX_GRID");
  if (e && *e) {
    const int v = atoi(e);
    if (v >= 1 && v < cap) cap = v;
  }
  return cap;
}

// ---------------------------------------------------------------------------------------------
// (B,C,N) channel-major -> (B,N,Cp) point-major, zero padded.  32x32 smem tile transpose; reads are
// coalesced along N, writes along C.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) to_point_major_kernel(const T* __restrict__ in, int C, int N, int Cp,
                                                             float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  in += (size_t)b * C * N;
  out += (size_t)b * N * Cp;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, n = n0 + tx;
    tile[r][tx] = (c < C && n < N) ? load_f32(in + (size_t)c * N + n) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int n = n0 + r, c = c0 + tx;
    if (n < N && c < Cp) out[(size_t)n * Cp + c] = tile[tx][r];
  }
}

template <typename T>
__global__ void __launch_bounds__(256) to_channel_major_kernel(const float* __restrict__ in, int C, int N, int Cp,
                                                               T* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int n0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  in += (size_t)b * N * Cp;
  out += (size_t)b * C * N;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int n = n0 + r, c = c0 + tx;
    tile[r][tx] = (n < N && c < C) ? in[(size_t)n * Cp + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, n = n0 + tx;
    if (c < C && n < N) store_f32(out + (size_t)c * N + n, tile[tx][r]);
  }
}

// ---------------------------------------------------------------------------------------------
// compatibility path: materialising gather (reference group_points_gpu.cu:13-33) and its gradient
// (:48-69).  One thread per (c, j) row of K outputs; the gradient is computed in gather form over a
// per-call scan of idx ... kept simple: these are NOT on the fused hot path.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) group_points_kernel(const T* __restrict__ points,
                                                           const int* __restrict__ idx, int C, int N, int M, int K,
                                                           T* __restrict__ out) {
  const int b = blockIdx.z, c = blockIdx.y;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * K) return;
  const T* p = points + ((size_t)b * C + c) * N;
  out[((size_t)b * C + c) * M * K + e] = p[idx[(size_t)b * M * K + e]];
}

// Deterministic scatter-add: one warp owns one (b, c) row of grad_points and walks all M*K entries in
// order, accumulating through shared-memory bins would need N floats; instead use fp32 atomics like the
// reference but on a zero-filled output.  (Order non-determinism matches the reference's own atomicAdd.)
template <typename T>
__global__ void __launch_bounds__(256) group_points_grad_kernel(const T* __restrict__ grad_out,
                                                                const int* __restrict__ idx, int C, int N, int M,
                                                                int K, float* __restrict__ grad_points) {
  const int b = blockIdx.z, c = blockIdx.y;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * K) return;
  float* gp = grad_points + ((size_t)b * C + c) * N;
  atomicAdd(gp + idx[(size_t)b * M * K + e], load_f32(grad_out + ((size_t)b * C + c) * M * K + e));
}

// gather form over the transposed lists of idx (all K slots): grad_points[b,c,j] = sum of grad_out[b,c,e] over the
// entries e = q*K + k of j's list, in list order, rounded once to T.  Canonical lists give the same bits every run.
template <typename T>
__global__ void __launch_bounds__(256) group_points_grad_csr_kernel(const T* __restrict__ grad_out,
                                                                    const int* __restrict__ csr_off,
                                                                    const int* __restrict__ csr_ent, int C, int N,
                                                                    int M, int K, T* __restrict__ grad_points) {
  const int b = blockIdx.z, c = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  const int o0 = csr_off[(size_t)b * (N + 1) + j], o1 = csr_off[(size_t)b * (N + 1) + j + 1];
  const int* ent = csr_ent + (size_t)b * M * K;
  const T* g = grad_out + ((size_t)b * C + c) * M * K;
  float acc = 0.f;
  for (int p = o0; p < o1; ++p) acc += load_f32(g + ent[p]);
  store_f32(grad_points + ((size_t)b * C + c) * N + j, acc);
}

// the 16-bit group_points gradient: fp32 accumulation buffer -> dtype, one rounding per element
template <typename T>
__global__ void __launch_bounds__(256) convert_kernel(const float* __restrict__ in, size_t n, T* __restrict__ out) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    store_f32(out + i, in[i]);
}

// out[p] = sum_t partial[t][p].  32 parameters x 32 tile-lanes per CTA; every tile-lane sums a fixed
// strided subset in double, then the 32 lanes are combined in a fixed order -> deterministic.
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const float* __restrict__ partial, int ntiles, int P,
                                                               float* __restrict__ out) {
  __shared__ double s_acc[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int p = blockIdx.x * 32 + tx;
  double acc = 0.0;
  if (p < P) {
    double b = 0.0, c = 0.0, d = 0.0;
    int t = ty;
    for (; t + 96 < ntiles; t += 128) {  // four independent load streams per thread
      acc += (double)partial[(size_t)t * P + p];
      b += (double)partial[(size_t)(t + 32) * P + p];
      c += (double)partial[(size_t)(t + 64) * P + p];
      d += (double)partial[(size_t)(t + 96) * P + p];
    }
    for (; t < ntiles; t += 32) acc += (double)partial[(size_t)t * P + p];
    acc = (acc + b) + (c + d);
  }
  s_acc[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && p < P) {
    double a = 0.0;
#pragma unroll
    for (int i = 0; i < 32; ++i) a += s_acc[i][tx];
    out[p] = (float)a;
  }
}

}  // namespace cl3d

using namespace cl3d;

extern "C" int cl3d_version(void) { return 106; }
extern "C" const char* cl3d_last_error(void) { return g_err; }
extern "C" int cl3d_padded_channels(int C) { return padded_channels(C); }
extern "C" int cl3d_sm_count(void) { return sm_count(); }
extern "C" long long cl3d_launch_count(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

extern "C" int cl3d_to_point_major(const void* in_cn, int dtype, int B, int C, int N, float* out_nc,
                                   cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(B >= 0 && C >= 1 && N >= 1 && in_cn && out_nc, "cl3d_to_point_major: bad arguments");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_to_point_major");
  if (B == 0) return CL3D_OK;
  const int Cp = padded_channels(C);
  dim3 grid(ceil_div(N, 32), ceil_div(Cp, 32), B);
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    to_point_major_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(in_cn), C, N, Cp, out_nc); CL3D_LAUNCHED(1);
    return check_launch("to_point_major_kernel");
  });
}

extern "C" int cl3d_to_channel_major(const float* in_nc, int B, int C, int N, void* out_cn, int dtype,
                                     cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(B >= 0 && C >= 1 && N >= 1 && in_nc && out_cn, "cl3d_to_channel_major: bad arguments");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_to_channel_major");
  if (B == 0) return CL3D_OK;
  const int Cp = padded_channels(C);
  dim3 grid(ceil_div(N, 32), ceil_div(C, 32), B);
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    to_channel_major_kernel<T><<<grid, 256, 0, stream>>>(in_nc, C, N, Cp, static_cast<T*>(out_cn)); CL3D_LAUNCHED(1);
    return check_launch("to_channel_major_kernel");
  });
}

extern "C" int cl3d_group_points(const void* points, int dtype, const int* idx, int B, int C, int N, int M, int K,
                                 void* out, cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(B >= 0 && C >= 1 && N >= 1 && M >= 0 && K >= 1 && points && idx && out, "cl3d_group_points: bad arguments");
  CL3D_REQUIRE(C <= 65535 && B <= 65535, "cl3d_group_points: C or B too large");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_group_points");
  if (B == 0 || M == 0) return CL3D_OK;
  const long long ents = (long long)M * K;
  dim3 grid((unsigned)((ents + 255) / 256), C, B);
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    group_points_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(points), idx, C, N, M, K, static_cast<T*>(out));
    CL3D_LAUNCHED(1);
    return check_launch("group_points_kernel");
  });
}

extern "C" int cl3d_group_points_grad(const void* grad_out, int dtype, const int* idx, int B, int C, int N, int M,
                                      int K, const int* csr_off, const int* csr_ent, void* grad_points, float* acc,
                                      cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(B >= 0 && C >= 1 && N >= 1 && M >= 0 && K >= 1 && grad_out && idx && grad_points,
               "cl3d_group_points_grad: bad arguments");
  CL3D_REQUIRE(C <= 65535 && B <= 65535, "cl3d_group_points_grad: C or B too large");
  CL3D_REQUIRE(!csr_off == !csr_ent, "cl3d_group_points_grad: csr_off and csr_ent are both given or both NULL");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_group_points_grad");
  CL3D_REQUIRE(dtype == CL3D_DTYPE_F32 || acc || csr_off,
               "cl3d_group_points_grad: a 16-bit gradient needs the fp32 buffer acc");
  if (B == 0) return CL3D_OK;
  if (csr_off) {
    return with_dtype(dtype, [&](auto t) {
      using T = typename decltype(t)::type;
      dim3 grid(ceil_div(N, 256), C, B);
      group_points_grad_csr_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(grad_out), csr_off, csr_ent, C,
                                                                N, M, K, static_cast<T*>(grad_points));
      CL3D_LAUNCHED(1);
      return check_launch("group_points_grad_csr_kernel");
    });
  }
  // no atomics on 16-bit types: a 16-bit gradient is accumulated in fp32 and converted once
  float* gp = dtype == CL3D_DTYPE_F32 ? static_cast<float*>(grad_points) : acc;
  const size_t n = (size_t)B * C * N;
  cudaMemsetAsync(gp, 0, sizeof(float) * n, stream);
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    if (M > 0) {
      const long long ents = (long long)M * K;
      dim3 grid((unsigned)((ents + 255) / 256), C, B);
      group_points_grad_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(grad_out), idx, C, N, M, K, gp);
      CL3D_LAUNCHED(1);
    }
    if constexpr (!std::is_same<T, float>::value) {
      const size_t blocks = (n + 255) / 256;
      convert_kernel<T><<<(unsigned)(blocks < 65535 ? blocks : 65535), 256, 0, stream>>>(gp, n, static_cast<T*>(grad_points));
      CL3D_LAUNCHED(1);
    }
    return check_launch("group_points_grad_kernel");
  });
}

extern "C" int cl3d_reduce_partials(const float* partial, int ntiles, int P, float* out, cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(ntiles >= 0 && P >= 1 && partial && out, "cl3d_reduce_partials: bad arguments");
  reduce_partials_kernel<<<ceil_div(P, 32), 1024, 0, stream>>>(partial, ntiles, P, out); CL3D_LAUNCHED(1);
  return check_launch("reduce_partials_kernel");
}
