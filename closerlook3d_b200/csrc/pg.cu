// pg.cu -- PseudoGrid (KPConv-like) local aggregation, forward and backward, second generation (sm_90a).
//
// Reference: /root/reference/pytorch/models/local_aggregation_operators.py:384-419
//     h[k',m]  = clamp(1 - |dp_m - K_k'| / extent, min 0)                (linear; 'constant': 1)
//     out[q,c] = sum_k' Wk[k',c] * sum_m h[k',m] * mask_m * f[j_m, c]
// evaluated in the "w-form"        out[q,c] = sum_m f[j_m,c] * w_c(dp_m),   w_c(dp) = sum_k' Wk[k',c] h(k',dp)
// which the backward shares:       d/df[j,c] = sum_e g[q_e,c] * w_c(s_j - q_e)        (e over the transposed lists)
//                                  d/dWk[k',c] = sum_e h(k', s_j - q_e) * f[j,c] * g[q_e,c].
// ONE kernel template serves both directions: centre point p (query / support point), a list of neighbour rows
// (features / upstream gradients).
//
// Why a second generation.  The first one (agg.cu) spends most of its forward instructions on influences (16 scalar
// IEEE square roots per neighbour) and on walking the (neighbour, kernel point) pairs at 15 instructions per pair (bit
// scan + two address computations + three 4-byte weight loads + three scalar FMAs), plus shuffle reductions of the
// BatchNorm partials; its backward keeps 16 accumulators per channel (127 registers).  Here:
//   * a lane owns 4 CONSECUTIVE channels: one 16-byte load per neighbour row / weight row, arithmetic in channel
//     pairs (FMAs with a scalar-broadcast h operand);
//   * staging compiles, per neighbour with any non-zero influence, a list of (h, weight-row byte offset) entries
//     -- 40 % of the neighbours have none and are dropped, the others ~3 of 15 -- so the pair loop is
//     {8-byte entry load, 16-byte weight load, 4 FFMA, branch}: 7 instructions instead of 15;
//   * influences are evaluated straight-line and packed (two kernel points per instruction), the square root with
//     the hardware approximation (2^-22 relative: h moves by < 3e-7, far inside the 1e-5 parity bar);
//   * BatchNorm partial sums are accumulated per lane in registers and combined once per tile;
//   * the backward uses the same one-accumulator w-form for d/df and adds d/dWk into a per-warp shared-memory
//     accumulator addressed by the entry's offset: ~64 registers instead of 127.
// One warp per centre point, 32 centre points per CTA tile; the backward is a persistent tile loop.
//
// Not shipped: kernel weights and d/dWk accumulators resident in registers with dense kernel-point quads (3x fewer
// shared-memory wavefronts, but at 128 / 168 registers too few warps per SM stay resident to hide the load latencies).
#include <stdlib.h>

#include "agg_common.cuh"

namespace cl3d {

constexpr int kPgWarps = 8;
constexpr int kPgTile = 32;  // centre points per CTA tile
// entries per staged neighbour + 1: rows of 17 float2 = 34 words put consecutive lanes' stores 2 banks apart (a
// stride of 16 entries = 32 words sent every lane's store to the same banks: up to 26-way conflicts)
constexpr int kEntStride = kMaxKP + 1;

// dynamic shared memory of the PG kernels:
//   s_kx, s_ky, s_kz  [8] u64      kernel points as packed pairs (k', k'+1), missing points = far away
//   s_wk             [16][CpR]     kernel weights (zero rows for missing kernel points)
//   per warp:  s_rec [32] uint2    {row element offset, number of entries} of the staged neighbours (compacted)
//              s_ent [32][17] float2  their entries {h, byte offset of the kernel point's weight row}
//   s_out            [CpR][kPgTile + 1]   output tile (transposed write-out)
//   s_bn             [warps][2][CpR]      forward: per-warp BatchNorm sums
//   bwd, per warp:   s_pacc [16][CpR]     d/dWk accumulator (same row layout as s_wk: one offset serves both)
struct PgSmem {
  size_t kp_off, wk_off, rec_off, ent_off, out_off, aux_off, total;
  int CpR;
};
__host__ __device__ inline PgSmem pg_smem(int Cp, bool bwd) {
  PgSmem L;
  L.CpR = (Cp + 3) / 4 * 4;
  size_t o = 0;
  L.kp_off = o;
  o += 3 * 8 * sizeof(u64);
  L.wk_off = o;
  o += (size_t)kMaxKP * L.CpR * sizeof(float);
  L.rec_off = o;
  o += (size_t)kPgWarps * 32 * sizeof(uint2);
  L.ent_off = o;
  o += (size_t)kPgWarps * 32 * kEntStride * sizeof(float2);
  L.out_off = o;
  o += (size_t)L.CpR * (kPgTile + 1) * sizeof(float);
  o = align_up(o, 16);
  L.aux_off = o;
  o += bwd ? (size_t)kPgWarps * kMaxKP * L.CpR * sizeof(float) : (size_t)kPgWarps * 2 * L.CpR * sizeof(float);
  L.total = align_up(o, 16);
  return L;
}

// Coordinates of point r from a packed (n,3) array with two requests instead of three: the 12 bytes start 8-byte
// aligned for even r (8 + 4) and end 8-byte aligned for odd r (4 + 8).  A scattered 4-byte load costs the L1 one
// wavefront per distinct line and instruction, and these kernels are bound by exactly that.
__device__ __forceinline__ void load_xyz(const float* __restrict__ xyz, int r, float& x, float& y, float& z) {
  const float* p = xyz + (size_t)r * 3;
  if (r & 1) {
    x = p[0];
    const float2 t = *reinterpret_cast<const float2*>(p + 1);
    y = t.x;
    z = t.y;
  } else {
    const float2 t = *reinterpret_cast<const float2*>(p);
    x = t.x;
    y = t.y;
    z = p[2];
  }
}

// All 32 lanes: lane `valid` holds one neighbour (relative position, row offset).  Evaluates its 16 influences
// (reference :385-398: sq = |dp - K|^2, h = clamp(1 - sqrt(sq)/extent, 0); 'constant': 1) two kernel points per
// instruction, and appends -- for neighbours with at least one non-zero influence, in lane order -- a record
// {row offset, n} and n entries {h, byte offset of Wk[k']} in ascending k'.  Returns the number of records.
__device__ __forceinline__ int pg_stage(uint2* __restrict__ s_rec, float2* __restrict__ s_ent, bool valid, float dx, float dy,
                                        float dz, unsigned row_off, const u64* __restrict__ s_kx,
                                        const u64* __restrict__ s_ky, const u64* __restrict__ s_kz, int nkp, int influence,
                                        float inv_extent, int row_bytes) {
  float h[kMaxKP];
  if (influence == 1) {  // 'constant'
#pragma unroll
    for (int kp = 0; kp < kMaxKP; ++kp) h[kp] = (valid && kp < nkp) ? 1.f : 0.f;
  } else {
    const u64 dxx = pack2(dx, dx), dyy = pack2(dy, dy), dzz = pack2(dz, dz);
    const u64 ninv = pack2(-inv_extent, -inv_extent), one = pack2(1.f, 1.f);
#pragma unroll
    for (int p = 0; p < kMaxKP / 2; ++p) {
      const u64 ex = sub2(dxx, s_kx[p]), ey = sub2(dyy, s_ky[p]), ez = sub2(dzz, s_kz[p]);
      const u64 sq2 = fma2(ez, ez, fma2(ey, ey, mul2(ex, ex)));
      float sq0, sq1;
      unpack2(sq2, sq0, sq1);
      float h0, h1;
      unpack2(fma2(pack2(sqrt_approx(sq0), sqrt_approx(sq1)), ninv, one), h0, h1);   // 1 - sqrt(sq) / extent
      h[2 * p] = valid ? fmaxf(h0, 0.f) : 0.f;   // a missing kernel point sits at 1e18: h < 0 -> 0
      h[2 * p + 1] = valid ? fmaxf(h1, 0.f) : 0.f;
    }
  }
  unsigned nz = 0;
#pragma unroll
  for (int kp = 0; kp < kMaxKP; ++kp) nz |= h[kp] > 0.f ? (1u << kp) : 0u;
  const unsigned m = __ballot_sync(0xffffffffu, nz != 0);
  if (nz != 0) {
    const int pos = __popc(m & ((1u << lane_id()) - 1u));
    s_rec[pos] = make_uint2(row_off, (unsigned)__popc(nz));
    float2* e = s_ent + (size_t)pos * kEntStride;
    int n = 0;
#pragma unroll
    for (int kp = 0; kp < kMaxKP; ++kp) {
      if (h[kp] > 0.f) e[n++] = make_float2(h[kp], __int_as_float(kp * row_bytes));
    }
  }
  return __popc(m);
}

// shared-memory accesses through 32-bit shared-window addresses (one add per access, no generic-pointer conversion)
__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_f4(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Consume n staged neighbours (warp-uniform control flow).
//   w    = sum over the neighbour's entries of h * Wk[k']        (ascending k')
//   acc += row * w
//   BWD: pacc[k'] += h * (fown * row)                            (d/dWk; lanes that own channels only)
// `rows` = per-lane base pointer of the gathered matrix (+ the lane's channel offset); `rec_a` / `ent_a` = shared
// addresses of the warp's record / entry lists; `wk_a` / `pacc_a` = the lane's shared address inside the weight /
// accumulator rows.  The next neighbour's row is requested before the current one is used.  The entry loop is kept
// rolled on purpose: 8 instructions per entry; unrolled by the compiler it grew a 70-instruction remainder ladder
// per neighbour.
template <bool BWD>
__device__ __forceinline__ void pg_consume(const float* __restrict__ rows, uint32_t rec_a, uint32_t ent_a, uint32_t wk_a,
                                           uint32_t pacc_a, const float4& fown, bool owner, int n, float4& acc) {
  if (n <= 0) return;
  float2 rec = lds_f2(rec_a);
  float4 row = __ldg(reinterpret_cast<const float4*>(row_at(rows, __float_as_uint(rec.x))));
#pragma unroll 1
  for (int s = 0; s < n; ++s) {
    const uint32_t e_end = ent_a + __float_as_uint(rec.y) * (uint32_t)sizeof(float2);
    const float4 v = row;
    if (s + 1 < n) {
      rec = lds_f2(rec_a + (uint32_t)(s + 1) * (uint32_t)sizeof(float2));
      row = __ldg(reinterpret_cast<const float4*>(row_at(rows, __float_as_uint(rec.x))));
    }
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (BWD) {
      fmul2(fown.x, fown.y, v.x, v.y, p.x, p.y);
      fmul2(fown.z, fown.w, v.z, v.w, p.z, p.w);
    }
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (uint32_t e = ent_a; e != e_end; e += (uint32_t)sizeof(float2)) {
      const float2 en = lds_f2(e);                       // {h, byte offset of the kernel point's rows}
      const uint32_t off = __float_as_uint(en.y);
      const float4 wk = lds_f4(wk_a + off);
      ffma2_bcast(en.x, wk.x, wk.y, w.x, w.y);
      ffma2_bcast(en.x, wk.z, wk.w, w.z, w.w);
      if constexpr (BWD) {
        if (owner) {  // lanes without channels shadow lane 0: they must not touch its accumulator words
          float4 t = lds_f4(pacc_a + off);
          ffma2_bcast(en.x, p.x, p.y, t.x, t.y);
          ffma2_bcast(en.x, p.z, p.w, t.z, t.w);
          sts_f4(pacc_a + off, t);
        }
      }
    }
    ffma2(v.x, v.y, w.x, w.y, acc.x, acc.y);
    ffma2(v.z, v.w, w.z, w.w, acc.z, acc.w);
    ent_a += (uint32_t)(kEntStride * sizeof(float2));
  }
}

// Layers wider than 128 channels run as gridDim.y channel chunks of equal width (a multiple of 4, <= 128): every
// chunk stages the influences again -- as the first generation does per 96 channels -- but keeps this kernel's
// cheaper pair loop.
__host__ __device__ inline int pg_num_chunks(int Cp) { return (Cp + 127) / 128; }
__host__ __device__ inline int pg_chunk_width(int Cp, int nchunks) { return ((Cp + nchunks - 1) / nchunks + 3) / 4 * 4; }

// kernel points (p0: (nkp,3)) and kernel weights (p1: (nkp,C), channels c0 .. c0+CpR) -> shared memory
__device__ __forceinline__ void pg_load_params(const AggArgs& a, const PgSmem& L, unsigned char* smem, int c0) {
  u64* s_kx = reinterpret_cast<u64*>(smem + L.kp_off);
  float* s_wk = reinterpret_cast<float*>(smem + L.wk_off);
  if (threadIdx.x < 3 * 8) {
    const int axis = threadIdx.x / 8, p = threadIdx.x % 8;
    // a missing kernel point sits far away: 1 - |dp - K| / extent < 0 -> h = 0
    const float k0 = 2 * p < a.nkp ? a.p0[(2 * p) * 3 + axis] : 1.0e18f;
    const float k1 = 2 * p + 1 < a.nkp ? a.p0[(2 * p + 1) * 3 + axis] : 1.0e18f;
    s_kx[axis * 8 + p] = pack2(k0, k1);
  }
  for (int e = threadIdx.x; e < kMaxKP * L.CpR; e += blockDim.x) {
    const int kp = e / L.CpR, c = e % L.CpR;
    s_wk[e] = (kp < a.nkp && c0 + c < a.C) ? a.p1[(size_t)kp * a.C + c0 + c] : 0.f;
  }
}

// =================================================================================================
//   BWD = false: centre = query q of cloud b, neighbour rows = feat_pm[idx[q][k]], k < ncount[q];
//                out[b,:,q] = acc ; per-tile BatchNorm partial sums.                         (one tile per CTA)
//   BWD = true : centre = support point j, neighbour rows = g_pm[q_e] over the transposed list of j;
//                out[b,:,j] = acc ; d/dWk accumulated per warp in shared memory.            (persistent tiles)
// =================================================================================================
template <bool BWD, bool CHUNKED>
__global__ void __launch_bounds__(kPgWarps * 32, BWD ? 3 : 4) pg2_kernel(const AggArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // CHUNKED = false (Cp <= 128, every BASELINE shape): one chunk, the constants below fold away
  const int W = CHUNKED ? pg_chunk_width(a.Cp, gridDim.y) : a.Cp;
  const int c0 = CHUNKED ? blockIdx.y * W : 0;     // this CTA's channel chunk
  const int Cw = CHUNKED ? min(W, a.Cp - c0) : a.Cp;  // its (padded) width, a multiple of 4
  const int Cv = CHUNKED ? min(Cw, a.C - c0) : a.C;   // real channels in it
  const PgSmem L = pg_smem(W, BWD);
  const u64* s_kx = reinterpret_cast<const u64*>(smem + L.kp_off);
  const u64* s_ky = s_kx + 8;
  const u64* s_kz = s_kx + 16;
  uint2* s_rec = reinterpret_cast<uint2*>(smem + L.rec_off) + (size_t)warp * 32;
  float2* s_ent = reinterpret_cast<float2*>(smem + L.ent_off) + (size_t)warp * 32 * kEntStride;
  float* s_out = reinterpret_cast<float*>(smem + L.out_off);
  float* s_aux = reinterpret_cast<float*>(smem + L.aux_off);
  pg_load_params(a, L, smem, c0);
  if constexpr (BWD)
    for (int e = threadIdx.x; e < kPgWarps * kMaxKP * L.CpR; e += blockDim.x) s_aux[e] = 0.f;
  __syncthreads();

  const int G = CHUNKED ? Cw / 4 : L.CpR / 4;   // lanes that own channels
  const bool owner = lane < G;
  const int cl = owner ? lane * 4 : 0;      // the others shadow lane 0 (their results are dropped)
  const int row_bytes = L.CpR * (int)sizeof(float);
  const int P = BWD ? a.N : a.M;            // centre points per cloud
  const int R = BWD ? a.M : a.N;            // rows of the gathered matrix per cloud
  const int tiles_per_cloud = (P + kPgTile - 1) / kPgTile;
  const uint32_t rec_a = smem_u32(s_rec), ent_a = smem_u32(s_ent);
  const uint32_t wk_a = smem_u32(smem + L.wk_off) + (uint32_t)cl * (uint32_t)sizeof(float);
  const uint32_t pacc_a = smem_u32(s_aux + (size_t)warp * kMaxKP * L.CpR + cl);

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int b = tile / tiles_per_cloud;
    const int p0 = (tile % tiles_per_cloud) * kPgTile;
    const float* rows = (BWD ? a.g_pm : a.feat_pm) + (size_t)b * R * a.Cp + c0 + cl;
    const float* cxyz = (BWD ? a.support_xyz : a.query_xyz) + (size_t)b * P * 3;   // centres
    const float* nxyz = (BWD ? a.query_xyz : a.support_xyz) + (size_t)b * R * 3;   // neighbours
    float4 bn1 = make_float4(0.f, 0.f, 0.f, 0.f), bn2 = bn1;                        // forward: sum, sum of squares

    for (int pl = warp; pl < kPgTile; pl += kPgWarps) {
      const int p = p0 + pl;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p < P) {
        const size_t gp = (size_t)b * P + p;
        int e0, e1;
        const int* list;
        if constexpr (BWD) {
          const int* off = a.csr_off + (size_t)b * (a.N + 1);
          e0 = off[p];
          e1 = off[p + 1];
          list = a.csr_ent + (size_t)b * a.M * a.K;
        } else {
          e0 = 0;
          e1 = a.ncount[gp];
          list = a.idx + gp * a.K;
        }
        const float cx = cxyz[p * 3 + 0], cy = cxyz[p * 3 + 1], cz = cxyz[p * 3 + 2];
        float4 fown = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (BWD)  // own features (d/dWk)
          fown = __ldg(reinterpret_cast<const float4*>(a.feat_pm + ((size_t)b * a.N + p) * a.Cp + c0 + cl));
        for (int eb = e0; eb < e1; eb += 32) {
          const bool valid = eb + lane < e1;
          float dx = 0.f, dy = 0.f, dz = 0.f;
          unsigned roff = 0;
          if (valid) {
            const int r = BWD ? list[eb + lane] / a.K : list[eb + lane];
            // relative position = support - query in both directions (pt_utils.py:127)
            float nx, ny, nz;
            load_xyz(nxyz, r, nx, ny, nz);
            if constexpr (BWD) {
              dx = __fsub_rn(cx, nx), dy = __fsub_rn(cy, ny), dz = __fsub_rn(cz, nz);
            } else {
              dx = __fsub_rn(nx, cx), dy = __fsub_rn(ny, cy), dz = __fsub_rn(nz, cz);
            }
            if (a.normalize) {
              dx = __fmul_rn(dx, a.inv_radius);
              dy = __fmul_rn(dy, a.inv_radius);
              dz = __fmul_rn(dz, a.inv_radius);
            }
            roff = (unsigned)r * (unsigned)a.Cp;
          }
          const int n = pg_stage(s_rec, s_ent, valid, dx, dy, dz, roff, s_kx, s_ky, s_kz, a.nkp, a.influence, a.inv_extent,
                                 row_bytes);
          __syncwarp();
          // Only the lanes that own channels walk the lists.  A shared-memory access is served per quarter warp: with
          // all 32 lanes active (the spare ones shadowing lane 0) a 16-byte weight / accumulator access took 4
          // wavefronts, with lanes 0..17 it takes 3 -- and this kernel is bound by exactly those wavefronts.
          if (owner) pg_consume<BWD>(rows, rec_a, ent_a, wk_a, pacc_a, fown, true, n, acc);
          __syncwarp();
        }
      }
      if constexpr (!BWD) {
        bn1.x += acc.x, bn1.y += acc.y, bn1.z += acc.z, bn1.w += acc.w;
        ffma2(acc.x, acc.y, acc.x, acc.y, bn2.x, bn2.y);
        ffma2(acc.z, acc.w, acc.z, acc.w, bn2.z, bn2.w);
      }
      if (owner) {
        s_out[(size_t)(cl + 0) * (kPgTile + 1) + pl] = acc.x;
        s_out[(size_t)(cl + 1) * (kPgTile + 1) + pl] = acc.y;
        s_out[(size_t)(cl + 2) * (kPgTile + 1) + pl] = acc.z;
        s_out[(size_t)(cl + 3) * (kPgTile + 1) + pl] = acc.w;
      }
    }
    if constexpr (!BWD) {
      if (owner && a.partial) {  // this warp's sums over its centre points of the tile
        *reinterpret_cast<float4*>(s_aux + ((size_t)warp * 2 + 0) * L.CpR + cl) = bn1;
        *reinterpret_cast<float4*>(s_aux + ((size_t)warp * 2 + 1) * L.CpR + cl) = bn2;
      }
    }
    __syncthreads();
    // ---- tile -> channel-major (B,C,P)
    const int p = p0 + lane;
    for (int c = warp; c < Cv; c += kPgWarps)
      if (p < P) a.out[((size_t)b * a.C + c0 + c) * P + p] = s_out[(size_t)c * (kPgTile + 1) + lane];
    if constexpr (!BWD) {
      if (a.partial) {  // BatchNorm partial sums of the tile: the warps' sums in a fixed order
        for (int e = threadIdx.x; e < 2 * Cv; e += blockDim.x) {
          const int s2 = e / Cv, c = e % Cv;
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < kPgWarps; ++w) t += s_aux[((size_t)w * 2 + s2) * L.CpR + c];
          a.partial[((size_t)tile * 2 + s2) * a.C + c0 + c] = t;
        }
      }
    }
    __syncthreads();
  }
  if constexpr (BWD) {
    // ---- d/dWk: sum the warps' accumulators in a fixed order -> one partial row per CTA: (gridDim.x, nkp, C)
    for (int e = threadIdx.x; e < a.nkp * Cv; e += blockDim.x) {
      const int kp = e / Cv, c = e % Cv;
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kPgWarps; ++w) t += s_aux[((size_t)w * kMaxKP + kp) * L.CpR + c];
      if constexpr (CHUNKED)
        a.partial[((size_t)blockIdx.x * a.nkp + kp) * a.C + c0 + c] = t;
      else
        a.partial[(size_t)blockIdx.x * a.nkp * a.C + e] = t;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
bool pg2_supported(const AggArgs& a) {
  if (getenv("CL3D_PG_V1")) return false;  // A/B switch: first-generation kernels (tests, profiling)
  return a.nkp >= 1 && a.nkp <= kMaxKP;
}

int pg2_launch_fwd(const AggArgs& a, cudaStream_t stream) {
  if (!pg2_supported(a)) return CL3D_ERR_UNSUPPORTED;

  const int nchunks = pg_num_chunks(a.Cp);
  const PgSmem L = pg_smem(pg_chunk_width(a.Cp, nchunks), false);
  static std::atomic<unsigned long long> seen{0};
  if (nchunks == 1) {
    allow_big_smem(pg2_kernel<false, false>, seen);
    pg2_kernel<false, false><<<a.ntiles, kPgWarps * 32, L.total, stream>>>(a);
  } else {
    static std::atomic<unsigned long long> seen_c{0};
    allow_big_smem(pg2_kernel<false, true>, seen_c);
    pg2_kernel<false, true><<<dim3(a.ntiles, nchunks), kPgWarps * 32, L.total, stream>>>(a);
  }
  CL3D_LAUNCHED(1);
  return check_launch("pg2_kernel<fwd>");
}

int pg2_launch_bwd(const AggArgs& a, int grid_x, cudaStream_t stream) {
  if (!pg2_supported(a)) return CL3D_ERR_UNSUPPORTED;

  const int nchunks = pg_num_chunks(a.Cp);
  const PgSmem L = pg_smem(pg_chunk_width(a.Cp, nchunks), true);
  static std::atomic<unsigned long long> seen{0};
  if (nchunks == 1) {
    allow_big_smem(pg2_kernel<true, false>, seen);
    pg2_kernel<true, false><<<grid_x, kPgWarps * 32, L.total, stream>>>(a);
  } else {
    static std::atomic<unsigned long long> seen_c{0};
    allow_big_smem(pg2_kernel<true, true>, seen_c);
    pg2_kernel<true, true><<<dim3(grid_x, nchunks), kPgWarps * 32, L.total, stream>>>(a);
  }
  CL3D_LAUNCHED(1);
  return check_launch("pg2_kernel<bwd>");
}

}  // namespace cl3d
