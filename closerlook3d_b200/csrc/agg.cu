// agg.cu -- fused local aggregation, forward and backward, for the per-(channel, neighbour)-weight families
//           PosPool(xyz | sin_cos) and AdaptiveWeight(dp) (sm_90a).
//
// Replaces, per LocalAggregation call of the reference
//   /root/reference/pytorch/ops/pt_custom_ops/pt_utils.py:121-144            (2x group_points, subtract, normalise)
//   /root/reference/pytorch/models/local_aggregation_operators.py:65-105      (PosPool transform + reduction)
//   .../local_aggregation_operators.py:188-217                                (AdaptiveWeight)
// none of which exists as a fused kernel there: the reference materialises (B,C,M,K) tensors ~10 times.
//
// Forward  (one warp per query, 32 consecutive queries per CTA):
//   lanes load the query's neighbour indices, gather the neighbours' xyz and build dp = (s - q) * (1/r) in
//   shared memory (32 slots per round); the warp then streams the neighbours' ROWS of the point-major
//   feature matrix with coalesced read-only loads (lane = channel, U rows in flight per lane), multiplies by
//   the family weight w_c(dp_k) and reduces over K in registers, so only the aggregated (B,C,M) tensor is
//   written -- transposed through shared memory into the reference's channel-major layout, together with
//   per-tile BatchNorm partial sums.
// Backward (gather form, one warp per SUPPORT point over its CSR list of (query, slot) references):
//   rows of d(loss)/d(agg) are streamed the same way; no float atomics on activations; parameter gradients
//   are accumulated per CTA and reduced afterwards in a fixed order.
//
// Staging the rows with one cp.async.bulk (TMA) per row makes the kernel issue-bound (about 11 warp-instructions
// per 288-byte row, plus the shared-memory load to read it back); plain coalesced loads do better here.
#include "agg_common.cuh"

namespace cl3d {

template <int FAM, bool BWD>
constexpr int num_acc() {
  return (BWD && FAM == CL3D_FAM_ADAPTIVE_DP) ? 4 : 1;
}

// floats of s_h per slot.  Only the first is used (the backward's scale), but at a stride of 1 or 2 the compiler
// schedules several backward kernels differently (agg_bwd_kernel<0, 4, *> grows from 648 to 768 instructions at 1);
// at 4 their code differs from a wider stride only in shared-memory offsets.
constexpr int kSlotH = 4;

// shared-memory carve-up (per CTA): per-warp slot arrays (dp + row index, backward scale) + output tile
struct SmemLayout {
  size_t dp_off, h_off, out_off, red_off, total;
};
__host__ __device__ inline SmemLayout smem_layout(int chunkC, int red_floats) {
  SmemLayout L;
  size_t o = 0;
  L.dp_off = o;
  o += (size_t)kAggWarps * kSlots * sizeof(float4);
  L.h_off = o;
  o += (size_t)kAggWarps * kSlots * kSlotH * sizeof(float);
  L.out_off = o;
  o += (size_t)chunkC * (kTile + 1) * sizeof(float);
  o = align_up(o, 16);
  L.red_off = o;
  o += (size_t)red_floats * sizeof(float);
  L.total = align_up(o, 16);
  return L;
}

// one staged slot: applies the family to the row values v[CI] of that slot; hk[0] is the backward's scale
template <int FAM, int CI, bool BWD, int NACC>
__device__ __forceinline__ void apply_slot(const float (&v)[CI], const float4& dp, const float* __restrict__ hk,
                                           const LaneParams<FAM, CI>& lp, float (&acc)[NACC][CI]) {
  if constexpr (BWD && FAM == CL3D_FAM_ADAPTIVE_DP) {
    const float sc = hk[0];  // 1/ncount (avg) or 1
#pragma unroll
    for (int i = 0; i < CI; ++i) {
      const float gs = v[i] * sc;
      acc[0][i] = fmaf(gs, dp.x, acc[0][i]);  // S_x, S_y, S_z, S_1
      acc[1][i] = fmaf(gs, dp.y, acc[1][i]);
      acc[2][i] = fmaf(gs, dp.z, acc[2][i]);
      acc[3][i] += gs;
    }
  } else if constexpr (BWD) {
    const float sc = hk[0];
#pragma unroll
    for (int i = 0; i < CI; ++i) acc[0][i] = fmaf(v[i] * sc, family_weight<FAM, CI>(lp, i, dp), acc[0][i]);
  } else {
#pragma unroll
    for (int i = 0; i < CI; ++i) acc[0][i] = fmaf(v[i], family_weight<FAM, CI>(lp, i, dp), acc[0][i]);
  }
}

// Consume n staged slots.  dp.w holds the row's ELEMENT OFFSET (row index * Cp) as a 32-bit unsigned, `lbase`
// is the per-lane base pointer (matrix + chunk offset + lane): one IMAD.WIDE per row, then the CI loads use
// immediate offsets (+32 floats each).  Lanes past the chunk read whatever follows (the next row, or the
// CL3D_PM_SLACK floats every point-major buffer carries after its last row); their results are never stored.
// Rows are loaded U = 4 at a time straight into registers (U*CI independent loads in flight per lane); these
// kernels need few registers, so many resident warps hide the latency.
template <int FAM, int CI, bool BWD, int NACC>
__device__ __forceinline__ void consume_slots(const float* __restrict__ lbase, const float4* __restrict__ s_dp,
                                              const float* __restrict__ s_h, int n, const LaneParams<FAM, CI>& lp,
                                              float (&acc)[NACC][CI]) {
  constexpr int U = 4;
  const int ng = n / U;
  for (int g = 0; g < ng; ++g) {
    float4 dp[U];
    float v[U][CI];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      dp[u] = s_dp[g * U + u];
      const float* row = lbase + __float_as_uint(dp[u].w);
#pragma unroll
      for (int i = 0; i < CI; ++i) v[u][i] = __ldg(row + 32 * i);  // lanes past the chunk read slack (unused)
    }
#pragma unroll
    for (int u = 0; u < U; ++u) apply_slot<FAM, CI, BWD, NACC>(v[u], dp[u], s_h + (size_t)(g * U + u), lp, acc);
  }
  for (int s = ng * U; s < n; ++s) {
    const float4 dp = s_dp[s];
    const float* row = lbase + __float_as_uint(dp.w);
    float v[CI];
#pragma unroll
    for (int i = 0; i < CI; ++i) v[i] = __ldg(row + 32 * i);
    apply_slot<FAM, CI, BWD, NACC>(v, dp, s_h + (size_t)s, lp, acc);
  }
}

// =================================================================================================
// forward
// =================================================================================================
template <int FAM, int CI>
__global__ void __launch_bounds__(kAggWarps * 32, 1) agg_fwd_kernel(const AggArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int chunkC = min(32 * CI, a.Cp - c0);  // multiple of 8
  const SmemLayout L = smem_layout(32 * CI, 0);
  float4* s_dp = reinterpret_cast<float4*>(smem + L.dp_off) + (size_t)warp * kSlots;
  float* s_h = reinterpret_cast<float*>(smem + L.h_off) + (size_t)warp * kSlots * kSlotH;
  float* s_out = reinterpret_cast<float*>(smem + L.out_off);

  const int tiles_per_cloud = (a.M + kTile - 1) / kTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kTile;

  LaneParams<FAM, CI> lp;
  load_lane_params<FAM, CI>(lp, a, c0, lane);
  constexpr int NACC = num_acc<FAM, false>();
  const float* feat = a.feat_pm + (size_t)b * a.N * a.Cp + c0 + lane;  // per-lane base pointer
  const float* sxyz = a.support_xyz + (size_t)b * a.N * 3;

  for (int ql = warp; ql < kTile; ql += kAggWarps) {
    const int q = q0 + ql;
    float res[CI];
#pragma unroll
    for (int i = 0; i < CI; ++i) res[i] = 0.f;
    if (q < a.M) {
      const size_t gq = (size_t)b * a.M + q;
      const int nrows = a.ncount[gq];
      const float qx = a.query_xyz[gq * 3 + 0], qy = a.query_xyz[gq * 3 + 1], qz = a.query_xyz[gq * 3 + 2];
      float acc[NACC][CI];
#pragma unroll
      for (int s = 0; s < NACC; ++s)
#pragma unroll
        for (int i = 0; i < CI; ++i) acc[s][i] = 0.f;
      for (int k0 = 0; k0 < nrows; k0 += kSlots) {
        const int rows = min(kSlots, nrows - k0);
        // ---- stage: indices, relative positions (pt_utils.py:127-129)
        if (lane < rows) {
          const int j = a.idx[gq * a.K + k0 + lane];
          const float3 d = rel_pos(a, sxyz[j * 3 + 0], sxyz[j * 3 + 1], sxyz[j * 3 + 2], qx, qy, qz);
          s_dp[lane] = make_float4(d.x, d.y, d.z, __uint_as_float((unsigned)j * (unsigned)a.Cp));
        }
        __syncwarp();
        consume_slots<FAM, CI, false, NACC>(feat, s_dp, s_h, rows, lp, acc);
        __syncwarp();  // slots are rewritten by the next round / query
      }
#pragma unroll
      for (int i = 0; i < CI; ++i)
        res[i] = a.reduction == CL3D_REDUCE_AVG ? __fdiv_rn(acc[0][i], (float)nrows) : acc[0][i];  // :96-98
    }
#pragma unroll
    for (int i = 0; i < CI; ++i) s_out[(size_t)(lane + 32 * i) * (kTile + 1) + ql] = res[i];
  }
  __syncthreads();
  store_fwd_tile<true>(a, s_out, 32 * CI, b, q0, [&](int r) { return c0 + r; });
}

// =================================================================================================
// backward (gather form over the CSR lists)
// =================================================================================================
template <int FAM>
__host__ __device__ constexpr int params_per_channel() {
  return FAM == CL3D_FAM_ADAPTIVE_DP ? 4 : 0;
}

template <int FAM, int CI, typename TO>
__global__ void __launch_bounds__(kAggWarps * 32, CI > 3 ? 2 : 3) agg_bwd_kernel(const AggArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * 32 * CI;
  const int chunkC = min(32 * CI, a.Cp - c0);
  constexpr int NACC = num_acc<FAM, true>();
  constexpr bool AW = FAM == CL3D_FAM_ADAPTIVE_DP;
  const SmemLayout L = smem_layout(32 * CI, params_per_channel<FAM>() * 32 * CI);
  float4* s_dp = reinterpret_cast<float4*>(smem + L.dp_off) + (size_t)warp * kSlots;
  float* s_h = reinterpret_cast<float*>(smem + L.h_off) + (size_t)warp * kSlots * kSlotH;
  float* s_out = reinterpret_cast<float*>(smem + L.out_off);
  float* s_red = reinterpret_cast<float*>(smem + L.red_off);

  LaneParams<FAM, CI> lp;
  load_lane_params<FAM, CI>(lp, a, c0, lane);
  bool ok[CI];
#pragma unroll
  for (int i = 0; i < CI; ++i) ok[i] = lane + 32 * i < chunkC;
  // AdaptiveWeight: per-lane parameter-gradient accumulators (x,y,z,bias) over all points this warp handles
  float pacc[AW ? 4 : 1][CI];
#pragma unroll
  for (int s = 0; s < (AW ? 4 : 1); ++s)
#pragma unroll
    for (int i = 0; i < CI; ++i) pacc[s][i] = 0.f;

  const int tiles_per_cloud = (a.N + kTile - 1) / kTile;
  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int b = tile / tiles_per_cloud;
    const int j0 = (tile % tiles_per_cloud) * kTile;
    const float* gpm = a.g_pm + (size_t)b * a.M * a.Cp + c0 + lane;  // per-lane base pointer
    const float* qxyz = a.query_xyz + (size_t)b * a.M * 3;
    const int* ncnt = a.ncount + (size_t)b * a.M;
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

        for (int eb = e0; eb < e1; eb += kSlots) {
          const int rows = min(kSlots, e1 - eb);
          if (lane < rows) {
            const BwdEntry e = bwd_entry(a, qxyz, ent[eb + lane], px, py, pz);
            s_dp[lane] = make_float4(e.dp.x, e.dp.y, e.dp.z, __uint_as_float(e.roff));
            s_h[lane] = a.reduction == CL3D_REDUCE_AVG ? __fdiv_rn(1.f, (float)ncnt[e.q]) : 1.f;
          }
          __syncwarp();
          consume_slots<FAM, CI, true, NACC>(gpm, s_dp, s_h, rows, lp, acc);
          __syncwarp();
        }
        // ---- epilogue: gradient w.r.t. this support point's features, parameter gradients
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
      for (int i = 0; i < CI; ++i) s_out[(size_t)(lane + 32 * i) * (kTile + 1) + jl] = res[i];
    }
    __syncthreads();
    store_bwd_tile<TO, true>(a, s_out, 32 * CI, b, j0, [&](int r) { return c0 + r; });
    __syncthreads();
  }
  // ---- CTA-level reduction of the parameter-gradient accumulators, fixed order over the warps
  if constexpr (AW) aw_bwd_params<CI>(a, pacc, s_red, c0);
}

// =================================================================================================
// PosPool sin_cos: pair ownership.  Channel c = axis*2F + t (t<F: sin, t>=F: cos of the SAME argument
// 100*dp_axis/dim_t, local_aggregation_operators.py:70-83), so a lane owns the PAIR (axis,t) = both channels
// and evaluates one division + one sincosf per (neighbour, pair) instead of a sinf AND a cosf per channel.
// Pair p = axis*F + t ; chunk of 32*PI pairs per CTA (blockIdx.y).
// =================================================================================================
template <int PI>
struct PairLane {
  unsigned osin[PI], ocos[PI];  // channel offsets inside a row
  float dim[PI], rdim[PI];
  int axis[PI];
};

template <int PI>
__device__ __forceinline__ void load_pair_lane(PairLane<PI>& pl, const AggArgs& a, int p0, int lane) {
  const int F = a.C / 6, npairs = 3 * F;
#pragma unroll
  for (int i = 0; i < PI; ++i) {
    int p = p0 + lane + 32 * i;
    if (p >= npairs) p = npairs - 1;  // duplicate work of a valid pair; its result is not written
    const int ax = p / F, t = p % F;
    pl.axis[i] = ax;
    pl.osin[i] = (unsigned)(ax * 2 * F + t);
    pl.ocos[i] = pl.osin[i] + (unsigned)F;
    pl.dim[i] = a.p0[t];
    pl.rdim[i] = __frcp_rn(pl.dim[i]);
  }
}

// sin and cos of x for |x| < ~1e4 (here |x| <= 100*|dp| ~ 1e2): Cody-Waite reduction by pi/2 in three steps,
// then the classic single-precision minimax polynomials on [-pi/4, pi/4]; ~1 ulp, branch-free, no slow path
// (the library sincosf inlines a Payne-Hanek path whose code size thrashed the instruction cache here).
__device__ __forceinline__ void sincos_small(float x, float& sn, float& cs) {
  const float j = rintf(x * 0.636619747f);
  float r = __fmaf_rn(j, -1.57079601e+00f, x);
  r = __fmaf_rn(j, -3.13916473e-07f, r);
  r = __fmaf_rn(j, -5.39030253e-15f, r);
  const int q = (int)j;
  const float r2 = r * r;
  float ps = __fmaf_rn(r2, -1.95152959e-4f, 8.33216087e-3f);
  ps = __fmaf_rn(ps, r2, -1.66666546e-1f);
  ps = __fmaf_rn(ps * r2, r, r);                      // sin(r)
  float pc = __fmaf_rn(r2, 2.44331571e-5f, -1.38873163e-3f);
  pc = __fmaf_rn(pc, r2, 4.16666457e-2f);
  pc = __fmaf_rn(pc, r2, -0.5f);
  pc = __fmaf_rn(pc, r2, 1.0f);                       // cos(r)
  const bool swap = q & 1;
  float s0 = swap ? pc : ps, c0 = swap ? ps : pc;
  sn = (q & 2) ? -s0 : s0;
  cs = ((q + 1) & 2) ? -c0 : c0;
}

// n / d, correctly rounded, with a precomputed correctly-rounded reciprocal: two residual corrections on the
// quotient (Markstein).  d >= 1 and |n| ~ 1e2 here: no overflow / denormals.  One ulp of the argument is
// 7.6e-6 rad at |arg| ~ 100, so the division has to be exact to stay inside the 1e-5 parity bar.
__device__ __forceinline__ float div_by(float n, float d, float rcp_d) {
  float q = n * rcp_d;
  q = __fmaf_rn(__fmaf_rn(-d, q, n), rcp_d, q);
  q = __fmaf_rn(__fmaf_rn(-d, q, n), rcp_d, q);
  return q;
}

// sin and cos of two arguments at once (the same wave length for two neighbour slots).  A polynomial version needs
// about 34 instructions per (neighbour, wave length) evaluation, most of them polynomial steps and quadrant swap /
// sign logic.  Here the argument is reduced EXACTLY (Cody-Waite with
// a three-term 2*pi, packed; the nearest integer by the magic-number add, no F2I / FRND) to r in [-pi, pi], where the
// hardware approximations are specified to 2^-21.4 (sin) / 2^-21.2 (cos) absolute error -- 4e-7, with the averaging over
// the K neighbours well inside the 1e-5 parity bar (measured in tests/test_local_aggregation_gpu.py) -- and cost one
// MUFU each: no polynomials, no quadrant logic.
__device__ __forceinline__ void sincos_small2(u64 x2, u64& sn2, u64& cs2) {
  const float kMagic = 12582912.f;  // 1.5 * 2^23
  const u64 t2 = fma2(x2, pack2(0.15915494309f, 0.15915494309f), pack2(kMagic, kMagic));   // x / (2 pi) + magic
  const u64 j2 = sub2(t2, pack2(kMagic, kMagic));                                         // nearest integer
  u64 r2v = fma2(j2, pack2(-6.28318548202514648e+00f, -6.28318548202514648e+00f), x2);    // 2 pi = hi + mid + lo
  r2v = fma2(j2, pack2(1.74845553146951715e-07f, 1.74845553146951715e-07f), r2v);
  r2v = fma2(j2, pack2(7.1054273576010019e-15f, 7.1054273576010019e-15f), r2v);
  float ra, rb;
  unpack2(r2v, ra, rb);
  sn2 = pack2(__sinf(ra), __sinf(rb));
  cs2 = pack2(__cosf(ra), __cosf(rb));
}

template <int PI, bool BWD>
__device__ __forceinline__ void consume_pairs(const float* __restrict__ base, const float4* __restrict__ s_dp,
                                              const float* __restrict__ s_h, int n, const PairLane<PI>& pl,
                                              float (&as)[PI], float (&ac)[PI]) {
  // neighbour slots two at a time: component 0 = even slot, component 1 = odd slot of the pair; each half keeps its
  // own partial sum (added at the end), every operation is a packed IEEE operation on both slots
  u64 as2[PI], ac2[PI], nd2[PI], rd2[PI];
#pragma unroll
  for (int i = 0; i < PI; ++i) {
    as2[i] = ac2[i] = 0ull;
    nd2[i] = pack2(-pl.dim[i], -pl.dim[i]);
    rd2[i] = pack2(pl.rdim[i], pl.rdim[i]);
  }
  const u64 hundred = pack2(100.f, 100.f);
  // The gathered values of slot pair s+2 are requested BEFORE the arithmetic of slot pair s (software pipeline, one
  // pair deep): a third of the stall samples sat on the accumulate FMAs waiting for loads that
  // had been issued ~45 instructions earlier -- an L2 hit takes several hundred cycles.
  auto gather = [&](int s0, u64 (&vs2)[PI], u64 (&vc2)[PI]) {
    const unsigned o0 = __float_as_uint(s_dp[s0].w), o1 = __float_as_uint(s_dp[s0 + 1].w);   // row element offsets
#pragma unroll
    for (int i = 0; i < PI; ++i) {  // one 32-bit add + one IMAD.WIDE per address (row_at)
      vs2[i] = pack2(__ldg(row_at(base, o0 + pl.osin[i])), __ldg(row_at(base, o1 + pl.osin[i])));
      vc2[i] = pack2(__ldg(row_at(base, o0 + pl.ocos[i])), __ldg(row_at(base, o1 + pl.ocos[i])));
    }
  };
  const int n2 = n & ~1;
  u64 vs2[PI], vc2[PI], nvs2[PI], nvc2[PI];
  if (n2 > 0) gather(0, vs2, vc2);
  int s = 0;
  for (; s < n2; s += 2) {
    if (s + 2 < n2) gather(s + 2, nvs2, nvc2);
    const float4 dp0 = s_dp[s], dp1 = s_dp[s + 1];
    u64 sc2 = 0ull;
    if constexpr (BWD) sc2 = pack2(s_h[s], s_h[s + 1]);
    const u64 px = mul2(pack2(dp0.x, dp1.x), hundred), py = mul2(pack2(dp0.y, dp1.y), hundred),
              pz = mul2(pack2(dp0.z, dp1.z), hundred);   // alpha * dp  (:75)
#pragma unroll
    for (int i = 0; i < PI; ++i) {
      const u64 n2v = pl.axis[i] == 0 ? px : (pl.axis[i] == 1 ? py : pz);
      // torch.div(alpha * dp, dim_mat): correctly rounded quotient, two Markstein corrections (see div_by)
      u64 q2 = mul2(n2v, rd2[i]);
      q2 = fma2(fma2(nd2[i], q2, n2v), rd2[i], q2);
      q2 = fma2(fma2(nd2[i], q2, n2v), rd2[i], q2);
      u64 sn2, cs2;
      sincos_small2(q2, sn2, cs2);
      as2[i] = fma2(BWD ? mul2(vs2[i], sc2) : vs2[i], sn2, as2[i]);
      ac2[i] = fma2(BWD ? mul2(vc2[i], sc2) : vc2[i], cs2, ac2[i]);
    }
#pragma unroll
    for (int i = 0; i < PI; ++i) {
      vs2[i] = nvs2[i];
      vc2[i] = nvc2[i];
    }
  }
#pragma unroll
  for (int i = 0; i < PI; ++i) {
    float a0, a1, c0, c1;
    unpack2(as2[i], a0, a1);
    unpack2(ac2[i], c0, c1);
    as[i] += a0 + a1;
    ac[i] += c0 + c1;
  }
  for (; s < n; ++s) {
    const float4 dp = s_dp[s];
    const float* row = base + __float_as_uint(dp.w);
    const float sc = BWD ? s_h[s] : 1.f;
#pragma unroll
    for (int i = 0; i < PI; ++i) {
      const float vs = __ldg(row + pl.osin[i]), vc = __ldg(row + pl.ocos[i]);
      const float pcomp = pl.axis[i] == 0 ? dp.x : (pl.axis[i] == 1 ? dp.y : dp.z);
      const float arg = div_by(__fmul_rn(100.f, pcomp), pl.dim[i], pl.rdim[i]);
      float sn, cs;
      sincos_small(arg, sn, cs);
      as[i] = fmaf(BWD ? vs * sc : vs, sn, as[i]);
      ac[i] = fmaf(BWD ? vc * sc : vc, cs, ac[i]);
    }
  }
}

// tile row r in [0, 2*32*PI): half h = r / (32*PI) (0 sin, 1 cos), pair p0 + r % (32*PI) -> channel or -1
__device__ __forceinline__ int pair_row_channel(int r, int p0, int pairs_per_cta, int F) {
  const int h = r / pairs_per_cta, p = p0 + r % pairs_per_cta;
  if (p >= 3 * F) return -1;
  return (p / F) * 2 * F + (p % F) + h * F;
}

template <int PI>
__global__ void __launch_bounds__(kAggWarps * 32, 3) sincos_fwd_kernel(const AggArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p0 = blockIdx.y * 32 * PI;
  const int F = a.C / 6;
  const SmemLayout L = smem_layout(2 * 32 * PI, 0);
  float4* s_dp = reinterpret_cast<float4*>(smem + L.dp_off) + (size_t)warp * kSlots;
  float* s_out = reinterpret_cast<float*>(smem + L.out_off);
  const int tiles_per_cloud = (a.M + kTile - 1) / kTile;
  const int b = blockIdx.x / tiles_per_cloud;
  const int q0 = (blockIdx.x % tiles_per_cloud) * kTile;
  PairLane<PI> pl;
  load_pair_lane<PI>(pl, a, p0, lane);
  const float* feat = a.feat_pm + (size_t)b * a.N * a.Cp;
  const float* sxyz = a.support_xyz + (size_t)b * a.N * 3;
  for (int ql = warp; ql < kTile; ql += kAggWarps) {
    const int q = q0 + ql;
    float rs[PI], rc[PI];
#pragma unroll
    for (int i = 0; i < PI; ++i) rs[i] = rc[i] = 0.f;
    if (q < a.M) {
      const size_t gq = (size_t)b * a.M + q;
      const int nrows = a.ncount[gq];
      const float qx = a.query_xyz[gq * 3 + 0], qy = a.query_xyz[gq * 3 + 1], qz = a.query_xyz[gq * 3 + 2];
      for (int k0 = 0; k0 < nrows; k0 += kSlots) {
        const int rows = min(kSlots, nrows - k0);
        if (lane < rows) {
          const int j = a.idx[gq * a.K + k0 + lane];
          const float3 dp = rel_pos(a, sxyz[j * 3 + 0], sxyz[j * 3 + 1], sxyz[j * 3 + 2], qx, qy, qz);
          s_dp[lane] = make_float4(dp.x, dp.y, dp.z, __uint_as_float((unsigned)j * (unsigned)a.Cp));
        }
        __syncwarp();
        consume_pairs<PI, false>(feat, s_dp, nullptr, rows, pl, rs, rc);
        __syncwarp();
      }
      if (a.reduction == CL3D_REDUCE_AVG) {
#pragma unroll
        for (int i = 0; i < PI; ++i) {
          rs[i] = __fdiv_rn(rs[i], (float)nrows);
          rc[i] = __fdiv_rn(rc[i], (float)nrows);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < PI; ++i) {
      s_out[(size_t)(lane + 32 * i) * (kTile + 1) + ql] = rs[i];
      s_out[(size_t)(32 * PI + lane + 32 * i) * (kTile + 1) + ql] = rc[i];
    }
  }
  __syncthreads();
  store_fwd_tile<false>(a, s_out, 2 * 32 * PI, b, q0, [&](int r) { return pair_row_channel(r, p0, 32 * PI, F); });
}

template <int PI, typename TO>
__global__ void __launch_bounds__(kAggWarps * 32, 3) sincos_bwd_kernel(const AggArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p0 = blockIdx.y * 32 * PI;
  const int F = a.C / 6;
  const SmemLayout L = smem_layout(2 * 32 * PI, 0);
  float4* s_dp = reinterpret_cast<float4*>(smem + L.dp_off) + (size_t)warp * kSlots;
  float* s_h = reinterpret_cast<float*>(smem + L.h_off) + (size_t)warp * kSlots * kSlotH;
  float* s_out = reinterpret_cast<float*>(smem + L.out_off);
  PairLane<PI> pl;
  load_pair_lane<PI>(pl, a, p0, lane);
  const int tiles_per_cloud = (a.N + kTile - 1) / kTile;
  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int b = tile / tiles_per_cloud;
    const int j0 = (tile % tiles_per_cloud) * kTile;
    const float* gpm = a.g_pm + (size_t)b * a.M * a.Cp;
    const float* qxyz = a.query_xyz + (size_t)b * a.M * 3;
    const int* ncnt = a.ncount + (size_t)b * a.M;
    const int* off = a.csr_off + (size_t)b * (a.N + 1);
    const int* ent = a.csr_ent + (size_t)b * a.M * a.K;
    for (int jl = warp; jl < kTile; jl += kAggWarps) {
      const int j = j0 + jl;
      float rs[PI], rc[PI];
#pragma unroll
      for (int i = 0; i < PI; ++i) rs[i] = rc[i] = 0.f;
      if (j < a.N) {
        const int e0 = off[j], e1 = off[j + 1];
        const float* sp = a.support_xyz + ((size_t)b * a.N + j) * 3;
        const float px = sp[0], py = sp[1], pz = sp[2];
        for (int eb = e0; eb < e1; eb += kSlots) {
          const int rows = min(kSlots, e1 - eb);
          if (lane < rows) {
            const BwdEntry e = bwd_entry(a, qxyz, ent[eb + lane], px, py, pz);
            s_dp[lane] = make_float4(e.dp.x, e.dp.y, e.dp.z, __uint_as_float(e.roff));
            s_h[lane] = a.reduction == CL3D_REDUCE_AVG ? __fdiv_rn(1.f, (float)ncnt[e.q]) : 1.f;
          }
          __syncwarp();
          consume_pairs<PI, true>(gpm, s_dp, s_h, rows, pl, rs, rc);
          __syncwarp();
        }
      }
#pragma unroll
      for (int i = 0; i < PI; ++i) {
        s_out[(size_t)(lane + 32 * i) * (kTile + 1) + jl] = rs[i];
        s_out[(size_t)(32 * PI + lane + 32 * i) * (kTile + 1) + jl] = rc[i];
      }
    }
    __syncthreads();
    store_bwd_tile<TO, false>(a, s_out, 2 * 32 * PI, b, j0, [&](int r) { return pair_row_channel(r, p0, 32 * PI, F); });
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------------------
template <int FAM, int CI>
static int launch_fwd(const AggArgs& a, cudaStream_t stream) {
  const int nchunks = ceil_div(a.Cp, 32 * CI);
  const SmemLayout L = smem_layout(32 * CI, 0);
  static std::atomic<unsigned long long> seen{0};
  allow_big_smem(agg_fwd_kernel<FAM, CI>, seen);
  dim3 grid(a.ntiles, nchunks);
  agg_fwd_kernel<FAM, CI><<<grid, kAggWarps * 32, L.total, stream>>>(a);
  CL3D_LAUNCHED(1);
  return check_launch("agg_fwd_kernel");
}

template <int FAM, int CI>
static int launch_bwd(const AggArgs& a, int grid_x, cudaStream_t stream) {
  const int nchunks = ceil_div(a.Cp, 32 * CI);
  const SmemLayout L = smem_layout(32 * CI, params_per_channel<FAM>() * 32 * CI);
  dim3 grid(grid_x, nchunks);
  return with_dtype(a.out_dtype, [&](auto t) {
    using TO = typename decltype(t)::type;
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(agg_bwd_kernel<FAM, CI, TO>, seen);
    agg_bwd_kernel<FAM, CI, TO><<<grid, kAggWarps * 32, L.total, stream>>>(a);
    CL3D_LAUNCHED(1);
    return check_launch("agg_bwd_kernel");
  });
}

static int pick_ci(int Cp) {
  const int ci = ceil_div(Cp, 32);
  return ci > kMaxCI ? kMaxCI : ci;
}

#define DISPATCH_CI(FN, FAM, ...)                          \
  switch (ci) {                                            \
    case 1: return FN<FAM, 1>(__VA_ARGS__);                \
    case 2: return FN<FAM, 2>(__VA_ARGS__);                \
    case 3: return FN<FAM, 3>(__VA_ARGS__);                \
    case 4: return FN<FAM, 4>(__VA_ARGS__);                \
    case 5: return FN<FAM, 5>(__VA_ARGS__);                \
    default: return FN<FAM, 6>(__VA_ARGS__);               \
  }

template <int PI>
static int launch_sincos(const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream) {
  const int npairs = a.C / 2;
  const SmemLayout L = smem_layout(2 * 32 * PI, 0);
  dim3 grid(grid_x, ceil_div(npairs, 32 * PI));
  if (!bwd) {
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(sincos_fwd_kernel<PI>, seen);
    sincos_fwd_kernel<PI><<<grid, kAggWarps * 32, L.total, stream>>>(a);
  } else {
    with_dtype(a.out_dtype, [&](auto t) {
      using TO = typename decltype(t)::type;
      static std::atomic<unsigned long long> seen{0};
      allow_big_smem(sincos_bwd_kernel<PI, TO>, seen);
      sincos_bwd_kernel<PI, TO><<<grid, kAggWarps * 32, L.total, stream>>>(a);
      return CL3D_OK;
    });
  }
  CL3D_LAUNCHED(1);
  return check_launch("sincos kernel");
}
static int dispatch_sincos(const AggArgs& a, bool bwd, int grid_x, cudaStream_t s) {
  int pi = ceil_div(a.C / 2, 32);
  if (pi > 3) pi = 3;
  switch (pi) {
    case 1: return launch_sincos<1>(a, bwd, grid_x, s);
    case 2: return launch_sincos<2>(a, bwd, grid_x, s);
    default: return launch_sincos<3>(a, bwd, grid_x, s);
  }
}

static int dispatch_fwd(int family, int ci, const AggArgs& a, cudaStream_t s) {
  switch (family) {
    case CL3D_FAM_POSPOOL_XYZ: DISPATCH_CI(launch_fwd, CL3D_FAM_POSPOOL_XYZ, a, s)
    case CL3D_FAM_POSPOOL_SINCOS: return dispatch_sincos(a, false, a.ntiles, s);
    case CL3D_FAM_ADAPTIVE_DP: DISPATCH_CI(launch_fwd, CL3D_FAM_ADAPTIVE_DP, a, s)
  }
  return CL3D_ERR_UNSUPPORTED;
}
static int dispatch_bwd(int family, int ci, const AggArgs& a, int gx, cudaStream_t s) {
  switch (family) {
    case CL3D_FAM_POSPOOL_XYZ: DISPATCH_CI(launch_bwd, CL3D_FAM_POSPOOL_XYZ, a, gx, s)
    case CL3D_FAM_POSPOOL_SINCOS: return dispatch_sincos(a, true, gx, s);
    case CL3D_FAM_ADAPTIVE_DP: DISPATCH_CI(launch_bwd, CL3D_FAM_ADAPTIVE_DP, a, gx, s)
  }
  return CL3D_ERR_UNSUPPORTED;
}

static int bwd_grid_x(int ntiles) {
  const int cap = persistent_grid_cap();
  return ntiles < cap ? (ntiles > 0 ? ntiles : 1) : cap;
}

}  // namespace cl3d

using namespace cl3d;

extern "C" int cl3d_agg_num_tiles(int B, int M) { return B * ceil_div(M, kTile); }

extern "C" int cl3d_agg_bwd_num_blocks(int B, int N) { return bwd_grid_x(B * ceil_div(N, kTile)); }

extern "C" int cl3d_agg_num_params(int family, int C, int shared, int nkp) {
  (void)shared;
  if (family == CL3D_FAM_ADAPTIVE_DP) return 4 * C;  // per-channel (x,y,z,bias); caller folds `shared` groups
  if (family == CL3D_FAM_PSEUDOGRID) return nkp * C;
  return 0;
}

static int check_common(int family, int reduction, int B, int N, int M, int K, int C, int shared, int nkp) {
  CL3D_REQUIRE(family >= 0 && family <= 3, "cl3d_agg: unknown family %d", family);
  CL3D_REQUIRE(reduction == CL3D_REDUCE_AVG || reduction == CL3D_REDUCE_SUM || reduction == CL3D_REDUCE_MAX,
               "cl3d_agg: unknown reduction %d", reduction);
  if (reduction == CL3D_REDUCE_MAX) {
    CL3D_REQUIRE(family != CL3D_FAM_PSEUDOGRID, "cl3d_agg: PseudoGrid sums over its neighbours (no max reduction)");
    CL3D_REQUIRE(K <= 256, "cl3d_agg: max reduction stores the winning slot in one byte (nsample %d > 256)", K);
  }
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 1 && K >= 1 && C >= 1, "cl3d_agg: bad sizes");
  if (family == CL3D_FAM_POSPOOL_XYZ) CL3D_REQUIRE(C % 3 == 0, "PosPool xyz needs C %% 3 == 0 (got %d)", C);
  if (family == CL3D_FAM_POSPOOL_SINCOS) CL3D_REQUIRE(C % 6 == 0, "PosPool sin_cos needs C %% 6 == 0 (got %d)", C);
  if (family == CL3D_FAM_ADAPTIVE_DP) CL3D_REQUIRE(shared >= 1 && C % shared == 0, "AdaptiveWeight: bad shared_channels");
  if (family == CL3D_FAM_PSEUDOGRID) CL3D_REQUIRE(nkp >= 1 && nkp <= kMaxKP, "PseudoGrid: 1..%d kernel points", kMaxKP);
  return CL3D_OK;
}

static void fill_common(AggArgs& a, int B, int N, int M, int K, int C, float radius, int reduction, int normalize,
                        int shared, int nkp, float extent, int influence) {
  a.B = B; a.N = N; a.M = M; a.K = K; a.C = C;
  a.Cp = padded_channels(C);
  a.reduction = reduction;
  a.normalize = normalize;
  a.shared = shared > 0 ? shared : 1;
  a.nkp = nkp;
  a.influence = influence;
  a.inv_radius = 1.0f / radius;
  a.extent = extent;
  a.inv_extent = 1.0f / extent;
}

extern "C" int cl3d_agg_fwd(int family, int reduction, const float* feat_pm, const float* query_xyz,
                            const float* support_xyz, const int* idx, const int* ncount, const float* p0,
                            const float* p1, int B, int N, int M, int K, int C, float radius, int normalize,
                            int shared, int nkp, float extent, int influence, float* agg, float* bn_partial,
                            unsigned char* arg_pm, cl3d_stream_t stream_) {
  int rc = check_common(family, reduction, B, N, M, K, C, shared, nkp);
  if (rc) return rc;
  CL3D_REQUIRE(feat_pm && query_xyz && support_xyz && idx && ncount && agg, "cl3d_agg_fwd: null pointer");
  CL3D_REQUIRE(reduction != CL3D_REDUCE_MAX || arg_pm, "cl3d_agg_fwd: max reduction needs the arg_pm buffer");
  if (B == 0) return CL3D_OK;
  AggArgs a = {};
  a.feat_pm = feat_pm;
  a.query_xyz = query_xyz;
  a.support_xyz = support_xyz;
  a.idx = idx;
  a.ncount = ncount;
  a.p0 = p0;
  a.p1 = p1;
  a.out = agg;
  a.partial = bn_partial;
  fill_common(a, B, N, M, K, C, radius, reduction, normalize, shared, nkp, extent, influence);
  a.ntiles = B * ceil_div(M, kTile);
  a.arg_pm = arg_pm;
  if (reduction == CL3D_REDUCE_MAX) return aggmax_launch(family, a, false, a.ntiles, (cudaStream_t)stream_);
  if (family == CL3D_FAM_PSEUDOGRID) return pg_launch(a, false, a.ntiles, (cudaStream_t)stream_);
  return dispatch_fwd(family, pick_ci(a.Cp), a, (cudaStream_t)stream_);
}

extern "C" int cl3d_agg_bwd(int family, int reduction, const float* g_pm, const float* feat_pm,
                            const float* query_xyz, const float* support_xyz, const int* ncount,
                            const int* csr_off, const int* csr_ent, const float* p0, const float* p1, int B, int N,
                            int M, int K, int C, float radius, int normalize, int shared, int nkp, float extent,
                            int influence, void* grad_feat, int dtype, float* grad_params_partial,
                            const unsigned char* arg_pm, cl3d_stream_t stream_) {
  int rc = check_common(family, reduction, B, N, M, K, C, shared, nkp);
  if (rc) return rc;
  CL3D_REQUIRE_DTYPE(dtype, "cl3d_agg_bwd");
  CL3D_REQUIRE(g_pm && query_xyz && support_xyz && ncount && csr_off && csr_ent && grad_feat,
               "cl3d_agg_bwd: null pointer");
  const bool has_params = family == CL3D_FAM_ADAPTIVE_DP || family == CL3D_FAM_PSEUDOGRID;
  CL3D_REQUIRE(!has_params || (feat_pm && grad_params_partial), "cl3d_agg_bwd: family needs feat_pm and a partial buffer");
  CL3D_REQUIRE(reduction != CL3D_REDUCE_MAX || arg_pm, "cl3d_agg_bwd: max reduction needs the forward's arg_pm");
  if (B == 0) return CL3D_OK;
  AggArgs a = {};
  a.feat_pm = feat_pm;
  a.g_pm = g_pm;
  a.query_xyz = query_xyz;
  a.support_xyz = support_xyz;
  a.ncount = ncount;
  a.csr_off = csr_off;
  a.csr_ent = csr_ent;
  a.p0 = p0;
  a.p1 = p1;
  a.out = static_cast<float*>(grad_feat);
  a.out_dtype = dtype;
  a.partial = grad_params_partial;
  fill_common(a, B, N, M, K, C, radius, reduction, normalize, shared, nkp, extent, influence);
  a.ntiles = B * ceil_div(N, kTile);
  a.arg_pm = const_cast<unsigned char*>(arg_pm);
  if (reduction == CL3D_REDUCE_MAX) return aggmax_launch(family, a, true, bwd_grid_x(a.ntiles), (cudaStream_t)stream_);
  if (family == CL3D_FAM_PSEUDOGRID) return pg_launch(a, true, bwd_grid_x(a.ntiles), (cudaStream_t)stream_);
  return dispatch_bwd(family, pick_ci(a.Cp), a, bwd_grid_x(a.ntiles), (cudaStream_t)stream_);
}
