// agg_common.cuh -- argument block, tile constants and the steps shared by the fused aggregation kernels
// (agg.cu, agg_max.cu, pg.cu).
#pragma once
#include <type_traits>

#include "common.cuh"

namespace cl3d {

constexpr int kAggWarps = 8;
constexpr int kTile = 32;   // queries (fwd) / support points (bwd) per CTA tile
constexpr int kMaxKP = 16;  // PseudoGrid kernel points (reference default 15)
constexpr int kMaxCI = 6;   // channel chunk = 32*CI <= 192 channels per CTA
constexpr int kSlots = 32;  // neighbour slots (fwd) / CSR entries (bwd) staged per round

struct AggArgs {
  const float* feat_pm;      // (B,N,Cp)   fwd: features; bwd: features (for parameter gradients)
  const float* g_pm;         // (B,M,Cp)   bwd only
  const float* query_xyz;    // (B,M,3)
  const float* support_xyz;  // (B,N,3)
  const int* idx;            // (B,M,K)    fwd only
  const int* ncount;         // (B,M)
  const int* csr_off;        // (B,N+1)    bwd only
  const int* csr_ent;        // (B,M*K)    bwd only
  const float* p0;           // family parameter 0 (see cl3d.h)
  const float* p1;           // family parameter 1
  float* out;                // fwd: agg (B,C,M); bwd: grad_feat (B,C,N)
  float* partial;            // fwd: bn partial (ntiles,2,C); bwd: param-grad partial (gridDim.x, P)
  int B, N, M, K, C, Cp;
  int reduction, normalize, shared, nkp, influence;
  float inv_radius, extent, inv_extent;
  int ntiles;
  int out_dtype;              // bwd: CL3D_DTYPE_* of `out` (the backward kernels' TO), fwd: CL3D_DTYPE_F32.  Sits in
                              // what was padding before arg_pm, so the block's layout and size are unchanged
  unsigned char* arg_pm;      // (B,M,Cp) max reduction only: winning neighbour slot per (query, channel)
};

// the channel-major store of the backward kernels: `out` holds elements of type TO (fp32 -> TO rounds once).
// The value comes first so that it is evaluated before the index, as in the assignment `a.out[i] = v`.
template <typename TO>
__device__ __forceinline__ void store_out(float v, const AggArgs& a, size_t i) {
  if constexpr (std::is_same<TO, float>::value) a.out[i] = v;
  else store_f32(reinterpret_cast<TO*>(a.out) + i, v);
}

// relative position of a neighbour, support - query (pt_utils.py:127-129), divided by the radius when normalising.
// torch's CUDA `tensor /= python_scalar` multiplies by the fp32 reciprocal; the 1e-5 parity bar depends on rounding
// exactly as it does.
__device__ __forceinline__ float3 rel_pos(const AggArgs& a, float sx, float sy, float sz, float qx, float qy, float qz) {
  float3 d = make_float3(__fsub_rn(sx, qx), __fsub_rn(sy, qy), __fsub_rn(sz, qz));
  if (a.normalize) {
    d.x = __fmul_rn(d.x, a.inv_radius);
    d.y = __fmul_rn(d.y, a.inv_radius);
    d.z = __fmul_rn(d.z, a.inv_radius);
  }
  return d;
}

// ---------------------------------------------------------------------------------------------
// one-warp-per-point kernels (agg.cu, agg_max.cu): a CTA handles a tile of kTile centre points, one warp per point,
// and collects its results in shared memory, s_out[row * (kTile + 1) + point], one row per owned channel.
// `channel(r)` maps tile row r to its channel.  ORDERED: channels ascend with r, and the first row at or past a.C ends
// the walk; otherwise a row mapped to a negative channel has none and is skipped.
// ---------------------------------------------------------------------------------------------

// forward: the tile channel-major into `out` (B,C,M) and each row's BatchNorm moments, one warp per row
template <bool ORDERED, typename RowChannel>
__device__ __forceinline__ void store_fwd_tile(const AggArgs& a, const float* s_out, int nrows, int b, int q0,
                                               RowChannel channel) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = q0 + lane;
  for (int r = warp; r < nrows; r += kAggWarps) {
    const int c = channel(r);
    if constexpr (ORDERED) {
      if (c >= a.C) break;
    } else if (c < 0) {
      continue;
    }
    float v = 0.f;
    if (q < a.M) {
      v = s_out[(size_t)r * (kTile + 1) + lane];
      a.out[((size_t)b * a.C + c) * a.M + q] = v;
    }
    if (a.partial) warp_bn_moments(a.partial, blockIdx.x, a.C, c, v, q < a.M);
  }
}

// backward: the tile of d/dfeatures channel-major into `out` (B,C,N)
template <typename TO, bool ORDERED, typename RowChannel>
__device__ __forceinline__ void store_bwd_tile(const AggArgs& a, const float* s_out, int nrows, int b, int j0,
                                               RowChannel channel) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = j0 + lane;
  for (int r = warp; r < nrows; r += kAggWarps) {
    const int c = channel(r);
    if constexpr (ORDERED) {
      if (c >= a.C) break;
    } else if (c < 0) {
      continue;
    }
    if (j < a.N) store_out<TO>(s_out[(size_t)r * (kTile + 1) + lane], a, ((size_t)b * a.C + c) * a.N + j);
  }
}

// backward: one entry en = q * K + slot of a support point's transposed list -- the query q, the relative position
// of the support point (px, py, pz) to it, and the element offset of q's row in the point-major matrices
struct BwdEntry {
  int q;
  float3 dp;
  unsigned roff;
};
__device__ __forceinline__ BwdEntry bwd_entry(const AggArgs& a, const float* qxyz, int en, float px, float py, float pz) {
  BwdEntry e;
  e.q = en / a.K;
  e.dp = rel_pos(a, px, py, pz, qxyz[e.q * 3 + 0], qxyz[e.q * 3 + 1], qxyz[e.q * 3 + 2]);
  e.roff = (unsigned)e.q * (unsigned)a.Cp;
  return e;
}

// this CTA's rows of the parameter-gradient partials (gridDim.x, ppc, C), from s_red[ppc][32*CI]; aw_bwd_params
// writes AdaptiveWeight's four rows per channel through it
template <int CI>
__device__ __forceinline__ void store_param_partial(const AggArgs& a, const float* s_red, int ppc, int c0) {
  for (int e = threadIdx.x; e < ppc * 32 * CI; e += blockDim.x) {
    const int s = e / (32 * CI), cl = e % (32 * CI);
    const int c = c0 + cl;
    if (c < a.C) a.partial[((size_t)blockIdx.x * ppc + s) * a.C + c] = s_red[e];
  }
}


// ---------------------------------------------------------------------------------------------
// family weights
// ---------------------------------------------------------------------------------------------
template <int FAM, int CI>
struct LaneParams {  // per-lane, per owned channel constants
  int axis[CI];      // XYZ / SINCOS: which coordinate
  float a[CI];       // SINCOS: dim_mat value ; ADAPTIVE: Wx
  float b[CI];       // ADAPTIVE: Wy
  float c[CI];       // ADAPTIVE: Wz
  float d[CI];       // ADAPTIVE: bias
  int is_cos[CI];
};

template <int FAM, int CI>
__device__ __forceinline__ void load_lane_params(LaneParams<FAM, CI>& lp, const AggArgs& a, int c0, int lane) {
#pragma unroll
  for (int i = 0; i < CI; ++i) {
    const int c = c0 + lane + 32 * i;
    lp.axis[i] = 0;
    lp.a[i] = 1.f;
    lp.b[i] = lp.c[i] = lp.d[i] = 0.f;
    lp.is_cos[i] = 0;
    if (c >= a.C) continue;
    if constexpr (FAM == CL3D_FAM_POSPOOL_XYZ) {
      lp.axis[i] = c % 3;  // view(B, C//3, 3, ...) : local_aggregation_operators.py:67
    } else if constexpr (FAM == CL3D_FAM_POSPOOL_SINCOS) {
      const int F = a.C / 6;  // channel = axis*2F + t ; t<F sin, t>=F cos  (:70-83)
      const int t = c % (2 * F);
      lp.axis[i] = c / (2 * F);
      lp.is_cos[i] = t >= F;
      lp.a[i] = a.p0[t % F];
    } else if constexpr (FAM == CL3D_FAM_ADAPTIVE_DP) {
      const int g = c / a.shared;  // :194-197 channel c uses weight row c // S
      lp.a[i] = a.p0[g * 3 + 0];
      lp.b[i] = a.p0[g * 3 + 1];
      lp.c[i] = a.p0[g * 3 + 2];
      lp.d[i] = a.p1[g];
    }
  }
}

// weight of channel slot i for relative position dp (float4: x,y,z,-)
template <int FAM, int CI>
__device__ __forceinline__ float family_weight(const LaneParams<FAM, CI>& lp, int i, const float4& dp) {
  if constexpr (FAM == CL3D_FAM_POSPOOL_XYZ) {
    return lp.axis[i] == 0 ? dp.x : (lp.axis[i] == 1 ? dp.y : dp.z);
  } else if constexpr (FAM == CL3D_FAM_POSPOOL_SINCOS) {
    const float p = lp.axis[i] == 0 ? dp.x : (lp.axis[i] == 1 ? dp.y : dp.z);
    const float arg = __fdiv_rn(__fmul_rn(100.f, p), lp.a[i]);  // torch.div(alpha * dp, dim_mat) :75-77
    return lp.is_cos[i] ? cosf(arg) : sinf(arg);
  } else if constexpr (FAM == CL3D_FAM_ADAPTIVE_DP) {
    return fmaf(lp.c[i], dp.z, fmaf(lp.b[i], dp.y, fmaf(lp.a[i], dp.x, lp.d[i])));  // 1x1 conv 3 -> C/S, bias
  } else {
    return 0.f;
  }
}

// AdaptiveWeight backward, end of the CTA: sum the warps' accumulators in a fixed order over the warps into
// s_red[4][32*CI] and write them as this CTA's rows of the (gridDim.x, 4, C) partials
template <int CI>
__device__ __forceinline__ void aw_bwd_params(const AggArgs& a, const float (&pacc)[4][CI], float* s_red, int c0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int w = 0; w < kAggWarps; ++w) {
    if (warp == w) {
#pragma unroll
      for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int i = 0; i < CI; ++i) {
          float* p = s_red + (size_t)s * 32 * CI + lane + 32 * i;
          *p = (w == 0) ? pacc[s][i] : (*p + pacc[s][i]);
        }
    }
    __syncthreads();
  }
  store_param_partial<CI>(a, s_red, 4, c0);
}


// pg.cu: PseudoGrid forward / backward (sum reduction); picks the tensor-core kernel where it serves the shape, the
// general one otherwise.  Forward: grid_x = a.ntiles; backward: grid_x = rows of a.partial the caller sums
int pg_launch(const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream);

// agg_max.cu: max reduction for PosPool (xyz | sin_cos) and AdaptiveWeight
int aggmax_launch(int family, const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream);

}  // namespace cl3d
