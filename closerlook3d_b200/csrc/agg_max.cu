// agg_max.cu -- fused local aggregation with MAX reduction for PosPool (xyz | sin_cos) and AdaptiveWeight (sm_90a).
//
// Replaces /root/reference/pytorch/models/local_aggregation_operators.py:87-91 (PosPool) and :199-203
// (AdaptiveWeight): F.max_pool2d over the nsample axis of the (B,C,npoint,nsample) product tensor, and its
// autograd backward (the gradient goes to the FIRST maximal slot of each (query, channel) window).
//
// No shipped cfg uses this reduction, so these kernels are the plain form of the design in agg.cu (warp per
// query / per support point, lane = channel, rows of the point-major matrices gathered with coalesced loads) --
// they exist so that no setting of the three families leaves the fused CUDA path.
//   forward : running maximum per (query, channel) in registers; the winning slot goes out as one byte per
//             (query, channel) in point-major order (B,M,Cp).  The ball query pads each list cyclically with its own
//             first entries (masked_ordered_ball_query_gpu.cu:85-93), so the maximum over the first `ncount` slots
//             with a strict comparison is max_pool2d's value AND its first arg-max over all nsample slots.
//   backward: gather form over the transposed lists like agg_bwd_kernel; an entry (query, slot) contributes iff
//             slot == winner[query][channel].
#include "agg_common.cuh"

namespace cl3d {

template <int FAM, int CI>
__global__ void __launch_bounds__(kAggWarps * 32) aggmax_fwd_kernel(const AggArgs a) {
  __shared__ float s_out[32 * CI * (kTile + 1)];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int tiles_per_cloud = (a.M + kTile - 1) / kTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kTile;

  LaneParams<FAM, CI> lp;
  load_lane_params<FAM, CI>(lp, a, c0, lane);
  const float* feat = a.feat_pm + (size_t)b * a.N * a.Cp + c0 + lane;  // per-lane base pointer
  const float* sxyz = a.support_xyz + (size_t)b * a.N * 3;

  for (int ql = warp; ql < kTile; ql += kAggWarps) {
    const int q = q0 + ql;
    float best[CI];
    int win[CI];
#pragma unroll
    for (int i = 0; i < CI; ++i) best[i] = 0.f, win[i] = 0;
    if (q < a.M) {
      const size_t gq = (size_t)b * a.M + q;
      const int nrows = a.ncount[gq];
      const float qx = a.query_xyz[gq * 3 + 0], qy = a.query_xyz[gq * 3 + 1], qz = a.query_xyz[gq * 3 + 2];
      for (int k0 = 0; k0 < nrows; k0 += 32) {
        const int rows = min(32, nrows - k0);
        float dx = 0.f, dy = 0.f, dz = 0.f;
        unsigned roff = 0;
        if (lane < rows) {  // relative position of slot k0+lane
          const int j = a.idx[gq * a.K + k0 + lane];
          const float3 d = rel_pos(a, sxyz[j * 3 + 0], sxyz[j * 3 + 1], sxyz[j * 3 + 2], qx, qy, qz);
          dx = d.x, dy = d.y, dz = d.z;
          roff = (unsigned)j * (unsigned)a.Cp;
        }
#pragma unroll 2
        for (int s = 0; s < rows; ++s) {
          float4 dp;
          dp.x = __shfl_sync(0xffffffffu, dx, s);
          dp.y = __shfl_sync(0xffffffffu, dy, s);
          dp.z = __shfl_sync(0xffffffffu, dz, s);
          dp.w = 0.f;
          const float* row = row_at(feat, __shfl_sync(0xffffffffu, roff, s));
          float v[CI];
#pragma unroll
          for (int i = 0; i < CI; ++i) v[i] = __ldg(row + 32 * i);  // lanes past the chunk read slack (unused)
#pragma unroll
          for (int i = 0; i < CI; ++i) {
            const float val = __fmul_rn(v[i], family_weight<FAM, CI>(lp, i, dp));
            if (k0 + s == 0 || val > best[i]) best[i] = val, win[i] = k0 + s;
          }
        }
      }
      unsigned char* wrow = a.arg_pm + gq * a.Cp + c0 + lane;
#pragma unroll
      for (int i = 0; i < CI; ++i)
        if (c0 + lane + 32 * i < a.Cp) wrow[32 * i] = (unsigned char)win[i];
    }
#pragma unroll
    for (int i = 0; i < CI; ++i) s_out[(size_t)(lane + 32 * i) * (kTile + 1) + ql] = best[i];
  }
  __syncthreads();
  store_fwd_tile<true>(a, s_out, 32 * CI, b, q0, [&](int r) { return c0 + r; });
}

template <int FAM, int CI, typename TO>
__global__ void __launch_bounds__(kAggWarps * 32) aggmax_bwd_kernel(const AggArgs a) {
  constexpr bool AW = FAM == CL3D_FAM_ADAPTIVE_DP;
  constexpr int NACC = AW ? 4 : 1;
  __shared__ float s_out[32 * CI][kTile + 1];
  __shared__ float s_red[NACC * 32 * CI];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int chunkC = min(32 * CI, a.Cp - c0);

  LaneParams<FAM, CI> lp;
  load_lane_params<FAM, CI>(lp, a, c0, lane);
  bool ok[CI];
#pragma unroll
  for (int i = 0; i < CI; ++i) ok[i] = lane + 32 * i < chunkC;
  float pacc[NACC][CI];  // AdaptiveWeight: d/d(Wx, Wy, Wz, bias) per owned channel over all points of this warp
#pragma unroll
  for (int s = 0; s < NACC; ++s)
#pragma unroll
    for (int i = 0; i < CI; ++i) pacc[s][i] = 0.f;

  const int tiles_per_cloud = (a.N + kTile - 1) / kTile;
  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int b = tile / tiles_per_cloud;
    const int j0 = (tile % tiles_per_cloud) * kTile;
    const float* gpm = a.g_pm + (size_t)b * a.M * a.Cp + c0 + lane;
    const unsigned char* wpm = a.arg_pm + (size_t)b * a.M * a.Cp + c0 + lane;
    const float* qxyz = a.query_xyz + (size_t)b * a.M * 3;
    const int* off = a.csr_off + (size_t)b * (a.N + 1);
    const int* ent = a.csr_ent + (size_t)b * a.M * a.K;

    for (int jl = warp; jl < kTile; jl += kAggWarps) {
      const int j = j0 + jl;
      float res[CI];
#pragma unroll
      for (int i = 0; i < CI; ++i) res[i] = 0.f;
      if (j < a.N) {
        const int e0 = off[j], e1 = off[j + 1];
        const float* sp = a.support_xyz + ((size_t)b * a.N + j) * 3;
        const float px = sp[0], py = sp[1], pz = sp[2];
        float acc[NACC][CI];
#pragma unroll
        for (int s = 0; s < NACC; ++s)
#pragma unroll
          for (int i = 0; i < CI; ++i) acc[s][i] = 0.f;
        for (int eb = e0; eb < e1; eb += 32) {
          const int rows = min(32, e1 - eb);
          float dx = 0.f, dy = 0.f, dz = 0.f;
          unsigned roff = 0;
          int slot = 0;
          if (lane < rows) {
            const int en = ent[eb + lane];
            const int q = en / a.K;
            slot = en - q * a.K;
            const float3 d = rel_pos(a, px, py, pz, qxyz[q * 3 + 0], qxyz[q * 3 + 1], qxyz[q * 3 + 2]);
            dx = d.x, dy = d.y, dz = d.z;
            roff = (unsigned)q * (unsigned)a.Cp;
          }
#pragma unroll 2
          for (int s = 0; s < rows; ++s) {
            float4 dp;
            dp.x = __shfl_sync(0xffffffffu, dx, s);
            dp.y = __shfl_sync(0xffffffffu, dy, s);
            dp.z = __shfl_sync(0xffffffffu, dz, s);
            dp.w = 0.f;
            const unsigned ro = __shfl_sync(0xffffffffu, roff, s);
            const int sl = __shfl_sync(0xffffffffu, slot, s);
            const float* row = row_at(gpm, ro);
            const unsigned char* wrow = wpm + ro;
#pragma unroll
            for (int i = 0; i < CI; ++i) {
              // the upstream gradient reaches this neighbour only where it won the maximum
              const float g = (ok[i] && (int)wrow[32 * i] == sl) ? __ldg(row + 32 * i) : 0.f;
              if constexpr (AW) {
                acc[0][i] = fmaf(g, dp.x, acc[0][i]);  // S_x, S_y, S_z, S_1 as in agg_bwd_kernel
                acc[1][i] = fmaf(g, dp.y, acc[1][i]);
                acc[2][i] = fmaf(g, dp.z, acc[2][i]);
                acc[3][i] += g;
              } else {
                acc[0][i] = fmaf(g, family_weight<FAM, CI>(lp, i, dp), acc[0][i]);
              }
            }
          }
        }
        if constexpr (AW) {
          const float* frow = a.feat_pm + ((size_t)b * a.N + j) * a.Cp + c0 + lane;
#pragma unroll
          for (int i = 0; i < CI; ++i) {
            const float f = ok[i] ? __ldg(frow + 32 * i) : 0.f;
            res[i] = fmaf(lp.c[i], acc[2][i], fmaf(lp.b[i], acc[1][i], fmaf(lp.a[i], acc[0][i], lp.d[i] * acc[3][i])));
#pragma unroll
            for (int s = 0; s < 4; ++s) pacc[s][i] = fmaf(f, acc[s][i], pacc[s][i]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < CI; ++i) res[i] = acc[0][i];
        }
      }
#pragma unroll
      for (int i = 0; i < CI; ++i) s_out[lane + 32 * i][jl] = res[i];
    }
    __syncthreads();
    const int j = j0 + lane;
    for (int cl = warp; cl < 32 * CI; cl += kAggWarps) {
      const int c = c0 + cl;
      if (c >= a.C) break;
      if (j < a.N) store_out<TO>(s_out[cl][lane], a, ((size_t)b * a.C + c) * a.N + j);
    }
    __syncthreads();
  }
  if constexpr (AW) aw_bwd_params<CI>(a, pacc, s_red, c0);
}

template <int FAM, int CI>
static int launch_max(const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream) {
  dim3 grid(grid_x, ceil_div(a.Cp, 32 * CI));
  if (!bwd)
    aggmax_fwd_kernel<FAM, CI><<<grid, kAggWarps * 32, 0, stream>>>(a);
  else
    with_dtype(a.out_dtype, [&](auto t) {
      aggmax_bwd_kernel<FAM, CI, typename decltype(t)::type><<<grid, kAggWarps * 32, 0, stream>>>(a);
      return CL3D_OK;
    });
  CL3D_LAUNCHED(1);
  return check_launch(bwd ? "aggmax_bwd_kernel" : "aggmax_fwd_kernel");
}

template <int FAM>
static int pick_max(const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream) {
  switch (ceil_div(a.Cp, 32)) {  // channels per lane; wider layers run as several chunks of 96 (blockIdx.y)
    case 1: return launch_max<FAM, 1>(a, bwd, grid_x, stream);
    case 2: return launch_max<FAM, 2>(a, bwd, grid_x, stream);
    default: return launch_max<FAM, 3>(a, bwd, grid_x, stream);
  }
}

int aggmax_launch(int family, const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream) {
  switch (family) {
    case CL3D_FAM_POSPOOL_XYZ: return pick_max<CL3D_FAM_POSPOOL_XYZ>(a, bwd, grid_x, stream);
    case CL3D_FAM_POSPOOL_SINCOS: return pick_max<CL3D_FAM_POSPOOL_SINCOS>(a, bwd, grid_x, stream);
    case CL3D_FAM_ADAPTIVE_DP: return pick_max<CL3D_FAM_ADAPTIVE_DP>(a, bwd, grid_x, stream);
  }
  set_error("cl3d_agg: max reduction exists for PosPool and AdaptiveWeight (family %d)", family);
  return CL3D_ERR_UNSUPPORTED;
}

}  // namespace cl3d
