// bn.cu -- the out_transform of PosPool / AdaptiveWeight / PseudoGrid: BatchNorm1d + ReLU on the
//          channel-major aggregated tensor (B,C,M), forward and backward (sm_90a).
//
// Replaces nn.Sequential(nn.BatchNorm1d(C, momentum), nn.ReLU(inplace=True)) of
//   /root/reference/pytorch/models/local_aggregation_operators.py:43-45,110 (and :166-168, :363-365).
// Batch statistics come from the per-tile moments the aggregation kernel already produced, so the
// forward costs one read + one write of (B,C,M); the backward is two passes (statistics, apply) and writes
// d(loss)/d(agg) directly in the point-major layout the gather-form aggregation backward consumes.
// PointWiseMLP's output relu(BN2d(ysel)) is the same forward over its selected extremum ysel (B,Cout,M).
#include <type_traits>

#include "common.cuh"

namespace cl3d {

// one tile's moments (store_bn_moments), or one rank's record (cl3d_bn_rank_moments), added to the sums of (x - shift)
// and (x - shift)^2: with g = centre - shift,
//   sum (x - shift) = d + n g,   sum (x - shift)^2 = q + 2 g d + n g^2
template <typename T>
__device__ __forceinline__ void bn_tile_add(const T* __restrict__ p, int C, double shift, double& a1, double& a2) {
  const double n = p[0], g = (double)p[C] - shift, d = p[2 * C], q = p[3 * C];
  a1 += fma(n, g, d);
  a2 += fma(g, fma(n, g, 2.0 * d), q);
}

// The tiles of a forward's partials merged in double about one shift per channel, tile 0's centre (a value of the
// channel, so the sums are of spread-sized terms and the variance never cancels against the mean), in a fixed order:
// deterministic.  One CTA of 1024 threads = 8 channels (one 32-byte sector of a partial row) x 128 tile slices, so the
// whole partial array is in flight at once (pure load latency).  Every thread calls it with tx = threadIdx.x & 7,
// ty = threadIdx.x >> 3 and c = blockIdx.x * 8 + tx; it returns the shift, and s1[0][tx], s2[0][tx] then hold channel
// c's sum (x - shift) and sum (x - shift)^2 (all zero when training = 0 or c >= C).
__device__ __forceinline__ double bn_merge_tiles(const float* __restrict__ partial, int ntiles, int C, int training,
                                                 int tx, int ty, int c, double (&s1)[128][9], double (&s2)[128][9]) {
  const size_t ts = (size_t)kBnRows * C;  // floats per tile
  const double shift = training && c < C ? (double)partial[C + c] : 0.0;
  double a1 = 0.0, a2 = 0.0;
  if (training && c < C) {
    const float* p = partial + c;
    double b1 = 0.0, b2 = 0.0, c1 = 0.0, c2 = 0.0, d1 = 0.0, d2 = 0.0;
    int t = ty;
    for (; t + 384 < ntiles; t += 512) {  // four independent load streams per thread
      bn_tile_add(p + (size_t)t * ts, C, shift, a1, a2);
      bn_tile_add(p + (size_t)(t + 128) * ts, C, shift, b1, b2);
      bn_tile_add(p + (size_t)(t + 256) * ts, C, shift, c1, c2);
      bn_tile_add(p + (size_t)(t + 384) * ts, C, shift, d1, d2);
    }
    for (; t < ntiles; t += 128) bn_tile_add(p + (size_t)t * ts, C, shift, a1, a2);
    a1 = (a1 + b1) + (c1 + d1);
    a2 = (a2 + b2) + (c2 + d2);
  }
  s1[ty][tx] = a1;
  s2[ty][tx] = a2;
  __syncthreads();
  // fixed-order tree over the 128 slices (deterministic)
  for (int h = 64; h >= 1; h >>= 1) {
    if (ty < h) {
      s1[ty][tx] += s1[ty + h][tx];
      s2[ty][tx] += s2[ty + h][tx];
    }
    __syncthreads();
  }
  return shift;
}

// batch mean / invstd of channel c from its merged sums about `shift`; running-stat update as nn.BatchNorm1d
// (unbiased variance over `count`)
__device__ __forceinline__ void bn_store_batch_stats(int c, int C, double count, double shift, double sum1, double sum2,
                                                     float eps, float momentum, float* __restrict__ running_mean,
                                                     float* __restrict__ running_var, float* __restrict__ save_stats) {
  const double dm = sum1 / count;  // mean - shift
  const double mean = shift + dm;
  double var = sum2 / count - dm * dm;
  if (var < 0.0) var = 0.0;
  save_stats[c] = (float)mean;
  save_stats[C + c] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean && running_var) {
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    running_mean[c] = (float)((1.0 - (double)momentum) * (double)running_mean[c] + (double)momentum * mean);
    running_var[c] = (float)((1.0 - (double)momentum) * (double)running_var[c] + (double)momentum * unbiased);
  }
}

// mean / invstd from the per-tile moments (training) or from the running statistics (eval)
__global__ void __launch_bounds__(1024) bn_finalize_kernel(const float* __restrict__ partial, int ntiles, int C,
                                                           double count, float eps, float momentum, int training,
                                                           float* __restrict__ running_mean,
                                                           float* __restrict__ running_var,
                                                           float* __restrict__ save_stats) {
  __shared__ double s1[128][9], s2[128][9];
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + tx;
  const double shift = bn_merge_tiles(partial, ntiles, C, training, tx, ty, c, s1, s2);
  if (ty == 0 && c < C) {
    if (training) {
      bn_store_batch_stats(c, C, count, shift, s1[0][tx], s2[0][tx], eps, momentum, running_mean, running_var,
                           save_stats);
    } else {
      save_stats[c] = running_mean[c];
      save_stats[C + c] = 1.0f / sqrtf(running_var[c] + eps);
    }
  }
}

// one rank's record (4,C) float64 for the cross-rank merge: count, centre (tile 0's), sum (x - centre),
// sum (x - centre)^2 -- the same merge as bn_finalize_kernel, stopped before the division
__global__ void __launch_bounds__(1024) bn_rank_moments_kernel(const float* __restrict__ partial, int ntiles, int C,
                                                               double count, double* __restrict__ record) {
  __shared__ double s1[128][9], s2[128][9];
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + tx;
  const double shift = bn_merge_tiles(partial, ntiles, C, 1, tx, ty, c, s1, s2);
  if (ty == 0 && c < C) {
    record[c] = count;
    record[C + c] = shift;
    record[2 * C + c] = s1[0][tx];
    record[3 * C + c] = s2[0][tx];
  }
}

// the W ranks' records (W,4,C) merged in rank order about rank 0's centre (bn_tile_add: every rank computes the same
// bits); the global count is their sum, written to *count_out for the backward
__global__ void __launch_bounds__(128) bn_finalize_ranks_kernel(const double* __restrict__ records, int W, int C,
                                                                float eps, float momentum,
                                                                float* __restrict__ running_mean,
                                                                float* __restrict__ running_var,
                                                                float* __restrict__ save_stats,
                                                                double* __restrict__ count_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double shift = records[C + c];
  double a1 = 0.0, a2 = 0.0, count = 0.0;
  for (int r = 0; r < W; ++r) {
    const double* p = records + (size_t)r * 4 * C + c;
    bn_tile_add(p, C, shift, a1, a2);
    count += p[0];
  }
  if (c == 0) *count_out = count;
  bn_store_batch_stats(c, C, count, shift, a1, a2, eps, momentum, running_mean, running_var, save_stats);
}

// out = sums * (1 / count): the batch-statistic means of the BatchNorm backward over a count held on the device, so
// that an apply pass taking a host scalar inv_count can run with inv_count = 1
__global__ void __launch_bounds__(256) bn_mean_terms_kernel(const float* __restrict__ sums, int n,
                                                            const double* __restrict__ count, float* __restrict__ out) {
  const float inv = 1.0f / (float)*count;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = sums[i] * inv;
}

int bn_mean_terms(const float* sums, int n, const double* count, float* out, cudaStream_t stream) {
  bn_mean_terms_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(sums, n, count, out);
  CL3D_LAUNCHED(1);
  return check_launch("bn_mean_terms_kernel");
}

// y = relu((x - mean) * invstd * gamma + beta), channel-major, float4 along M when aligned
template <typename T>
__global__ void __launch_bounds__(256) bn_relu_fwd_kernel(const float* __restrict__ x, const float* __restrict__ stats,
                                                          const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, int C, int M,
                                                          T* __restrict__ y) {
  const int row = blockIdx.x;  // b*C + c
  const int c = row % C;
  const float mean = stats[c], invstd = stats[C + c];
  const float sc = invstd * gamma[c], sh = beta[c];
  const float* xr = x + (size_t)row * M;
  T* yr = y + (size_t)row * M;
  for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < M; i += gridDim.y * blockDim.x) {
    const float v = bn_preact(xr[i], mean, sc, sh);
    store_f32(yr + i, v > 0.f ? v : 0.f);
  }
}

// Backward, tiles of 128 consecutive queries of one cloud: a warp owns a channel row segment (512 bytes, one
// float4 per lane when M % 4 == 0), so both passes stream (B,C,M) with full-width, page-friendly accesses.
constexpr int kBwdTile = 128;
constexpr int kBwdCh = 32;  // channels staged per shared-memory transpose round in the apply pass

// 16-bit rows (grad_y) are read element by element: they are only 2-byte aligned when M is odd
template <typename T>
__device__ __forceinline__ void load4(const T* __restrict__ p, int q, int M, bool vec, float (&v)[4]) {
  if (std::is_same<T, float>::value && vec && q + 3 < M) {
    const float4 t = *reinterpret_cast<const float4*>(p + q);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
#pragma unroll
    for (int t = 0; t < 4; ++t) v[t] = (q + t < M) ? load_f32(p + q + t) : 0.f;
  }
}

// pass 1: per tile and channel: sum(gy * xhat), sum(gy) -- rows (dgamma, dbeta) for cl3d_reduce_partials
template <typename T>
__global__ void __launch_bounds__(256) bn_relu_bwd_stats_kernel(const T* __restrict__ grad_y,
                                                                const float* __restrict__ x,
                                                                const float* __restrict__ stats,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, int C, int M,
                                                                float* __restrict__ partial) {
  const int tiles_per_cloud = (M + kBwdTile - 1) / kBwdTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = (blockIdx.x % tiles_per_cloud) * kBwdTile + lane * 4;
  const bool vec = (M & 3) == 0;
  for (int c = warp; c < C; c += 8) {
    const size_t row = ((size_t)b * C + c) * M;
    float xv[4], gv[4];
    load4(x + row, q, M, vec, xv);
    load4(grad_y + row, q, M, vec, gv);
    const float mean = stats[c], invstd = stats[C + c], sc = invstd * gamma[c], sh = beta[c];
    float gy = 0.f, gx = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (q + t < M) {
        const float g = bn_preact(xv[t], mean, sc, sh) > 0.f ? gv[t] : 0.f;
        gy += g;
        gx = fmaf(g, __fsub_rn(xv[t], mean) * invstd, gx);
      }
    }
    const float s1 = warp_sum(gy), s2 = warp_sum(gx);
    if (lane == 0) {
      partial[((size_t)blockIdx.x * 2 + 0) * C + c] = s2;
      partial[((size_t)blockIdx.x * 2 + 1) * C + c] = s1;
    }
  }
}

// pass 2: g = gamma*invstd*(gy - mean(gy) - xhat*mean(gy*xhat)) (training) or gamma*invstd*gy (eval), written
// point-major (B,M,Cp) through a shared-memory transpose, kBwdCh channels per round; padding channels = 0.
template <typename T>
__global__ void __launch_bounds__(256) bn_relu_bwd_apply_kernel(const T* __restrict__ grad_y,
                                                                const float* __restrict__ x,
                                                                const float* __restrict__ stats,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ beta,
                                                                const float* __restrict__ dgb, int C, int Cp, int M,
                                                                float inv_count, int training,
                                                                float* __restrict__ g_pm) {
  __shared__ float s_tile[kBwdTile][kBwdCh + 1];
  const int tiles_per_cloud = (M + kBwdTile - 1) / kBwdTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kBwdTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = q0 + lane * 4;
  const bool vec = (M & 3) == 0;
  const int nq = min(kBwdTile, M - q0);
  for (int cb = 0; cb < Cp; cb += kBwdCh) {
    for (int cl = warp; cl < kBwdCh; cl += 8) {
      const int c = cb + cl;
      float g[4] = {0.f, 0.f, 0.f, 0.f};
      if (c < C) {
        const size_t row = ((size_t)b * C + c) * M;
        float xv[4], gv[4];
        load4(x + row, q, M, vec, xv);
        load4(grad_y + row, q, M, vec, gv);
        const float mean = stats[c], invstd = stats[C + c], ga = gamma[c], sc = invstd * ga, sh = beta[c];
        const float mg = training ? dgb[C + c] * inv_count : 0.f, mgx = training ? dgb[c] * inv_count : 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float gy = bn_preact(xv[t], mean, sc, sh) > 0.f ? gv[t] : 0.f;
          g[t] = sc * (gy - mg - __fsub_rn(xv[t], mean) * invstd * mgx);
        }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) s_tile[lane * 4 + t][cl] = g[t];
    }
    __syncthreads();
    const int ncb = min(kBwdCh, Cp - cb);
    for (int e = threadIdx.x; e < nq * ncb; e += blockDim.x) {
      const int ql = e / ncb, cl = e % ncb;
      g_pm[((size_t)b * M + q0 + ql) * Cp + cb + cl] = s_tile[ql][cl];
    }
    __syncthreads();
  }
}

}  // namespace cl3d

using namespace cl3d;

extern "C" int cl3d_bn_finalize(const float* bn_partial, int ntiles, int C, long long count, float eps, float momentum,
                                int training, float* running_mean, float* running_var, float* save_stats,
                                cl3d_stream_t stream_) {
  CL3D_REQUIRE(C >= 1 && save_stats, "cl3d_bn_finalize: bad arguments");
  CL3D_REQUIRE(!training || (bn_partial && ntiles >= 1 && count >= 1), "cl3d_bn_finalize: training needs partial moments");
  CL3D_REQUIRE(training || (running_mean && running_var), "cl3d_bn_finalize: eval needs running statistics");
  bn_finalize_kernel<<<ceil_div(C, 8), 1024, 0, (cudaStream_t)stream_>>>(bn_partial, ntiles, C, (double)count, eps,
                                                                         momentum, training, running_mean,
                                                                         running_var, save_stats); CL3D_LAUNCHED(1);
  return check_launch("bn_finalize_kernel");
}

extern "C" int cl3d_bn_relu_fwd(const float* x, const float* save_stats, const float* gamma, const float* beta,
                                int B, int C, int M, void* y, int dtype, cl3d_stream_t stream_) {
  CL3D_REQUIRE(x && save_stats && gamma && beta && y && B >= 0 && C >= 1 && M >= 1, "cl3d_bn_relu_fwd: bad arguments");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_bn_relu_fwd");
  if (B == 0) return CL3D_OK;
  int chunks = ceil_div(M, 1024);
  chunks = chunks < 1 ? 1 : (chunks > 65535 ? 65535 : chunks);
  dim3 grid(B * C, chunks);
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    bn_relu_fwd_kernel<T><<<grid, 256, 0, (cudaStream_t)stream_>>>(x, save_stats, gamma, beta, C, M, static_cast<T*>(y));
    CL3D_LAUNCHED(1);
    return check_launch("bn_relu_fwd_kernel");
  });
}

extern "C" int cl3d_bn_rank_moments(const float* bn_partial, int ntiles, int C, long long count, double* record,
                                    cl3d_stream_t stream_) {
  CL3D_REQUIRE(bn_partial && record && ntiles >= 1 && C >= 1 && count >= 1, "cl3d_bn_rank_moments: bad arguments");
  bn_rank_moments_kernel<<<ceil_div(C, 8), 1024, 0, (cudaStream_t)stream_>>>(bn_partial, ntiles, C, (double)count,
                                                                             record);
  CL3D_LAUNCHED(1);
  return check_launch("bn_rank_moments_kernel");
}

extern "C" int cl3d_bn_finalize_ranks(const double* records, int W, int C, float eps, float momentum,
                                      float* running_mean, float* running_var, float* save_stats, double* count,
                                      cl3d_stream_t stream_) {
  CL3D_REQUIRE(records && save_stats && count && W >= 1 && C >= 1, "cl3d_bn_finalize_ranks: bad arguments");
  bn_finalize_ranks_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream_>>>(records, W, C, eps, momentum,
                                                                                running_mean, running_var, save_stats,
                                                                                count);
  CL3D_LAUNCHED(1);
  return check_launch("bn_finalize_ranks_kernel");
}

extern "C" int cl3d_bn_relu_bwd_stats(const void* grad_y, int dtype, const float* x, const float* save_stats,
                                      const float* gamma, const float* beta, int B, int C, int M, float* partial,
                                      float* dgamma_dbeta, cl3d_stream_t stream_) {
  CL3D_REQUIRE(grad_y && x && save_stats && gamma && beta && partial && dgamma_dbeta,
               "cl3d_bn_relu_bwd_stats: null pointer");
  CL3D_REQUIRE(B >= 0 && C >= 1 && M >= 1, "cl3d_bn_relu_bwd_stats: bad sizes");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_bn_relu_bwd_stats");
  if (B == 0) return CL3D_OK;
  const int ntiles = B * ceil_div(M, kBwdTile);  // <= cl3d_agg_num_tiles(B, M): the caller's partial buffer fits
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    bn_relu_bwd_stats_kernel<T><<<ntiles, 256, 0, (cudaStream_t)stream_>>>(static_cast<const T*>(grad_y), x, save_stats,
                                                                           gamma, beta, C, M, partial);
    CL3D_LAUNCHED(1);
    return cl3d_reduce_partials(partial, ntiles, 2 * C, dgamma_dbeta, stream_);  // (dgamma, dbeta)
  });
}

extern "C" int cl3d_bn_relu_bwd_apply(const void* grad_y, int dtype, const float* x, const float* save_stats,
                                      const float* gamma, const float* beta, int B, int C, int M, int training,
                                      const float* dgb_sums, const double* count, float* work, float* g_pm,
                                      cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(grad_y && x && save_stats && gamma && beta && dgb_sums && g_pm && (!count || work),
               "cl3d_bn_relu_bwd_apply: null pointer");
  CL3D_REQUIRE(B >= 0 && C >= 1 && M >= 1, "cl3d_bn_relu_bwd_apply: bad sizes");
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_bn_relu_bwd_apply");
  if (B == 0) return CL3D_OK;
  const int ntiles = B * ceil_div(M, kBwdTile);
  const int Cp = padded_channels(C);
  float inv_count = 1.0f / (float)((long long)B * M);
  const float* dgb = dgb_sums;
  if (count && training) {  // the means over the device-held count, then the same apply pass with inv_count = 1
    const int rc = bn_mean_terms(dgb_sums, 2 * C, count, work, stream);
    if (rc) return rc;
    dgb = work;
    inv_count = 1.0f;
  }
  return with_dtype(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    bn_relu_bwd_apply_kernel<T><<<ntiles, 256, 0, stream>>>(static_cast<const T*>(grad_y), x, save_stats, gamma, beta,
                                                            dgb, C, Cp, M, inv_count, training, g_pm);
    CL3D_LAUNCHED(1);
    return check_launch("bn_relu_bwd kernels");
  });
}

extern "C" int cl3d_bn_relu_bwd(const void* grad_y, int dtype, const float* x, const float* save_stats,
                                const float* gamma, const float* beta, int B, int C, int M, int training,
                                float* partial, float* dgamma_dbeta, float* g_pm, cl3d_stream_t stream_) {
  const int rc = cl3d_bn_relu_bwd_stats(grad_y, dtype, x, save_stats, gamma, beta, B, C, M, partial, dgamma_dbeta,
                                        stream_);
  if (rc) return rc;
  return cl3d_bn_relu_bwd_apply(grad_y, dtype, x, save_stats, gamma, beta, B, C, M, training, dgamma_dbeta, nullptr,
                                nullptr, g_pm, stream_);
}
