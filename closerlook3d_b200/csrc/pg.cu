// pg.cu -- PseudoGrid (KPConv-like) local aggregation (sm_90a): second generation (forward and backward, any width)
// and third generation (up to 128 channels: per-kernel-point sums on the tensor cores, see pg3_body).
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
// pg2_kernel.  Its instructions go to the influences (16 per neighbour) and to the walk over the (neighbour, kernel
// point) pairs, so both are kept short, and one accumulator per channel keeps the registers down:
//   * a lane owns 4 CONSECUTIVE channels: one 16-byte load per neighbour row / weight row, arithmetic in channel
//     pairs (FMAs with a scalar-broadcast h operand);
//   * staging compiles, per neighbour with any non-zero influence, a list of (h, weight-row byte offset) entries
//     -- 40 % of the neighbours have none and are dropped, the others ~3 of 15 -- so the pair loop is
//     {8-byte entry load, 16-byte weight load, 4 FFMA, branch}: 7 instructions per pair;
//   * influences are evaluated straight-line and packed (two kernel points per instruction), the square root with
//     the hardware approximation (2^-22 relative: h moves by < 3e-7, far inside the 1e-5 parity bar);
//   * BatchNorm partial moments are taken once per tile from the output tile in shared memory;
//   * the backward uses the same one-accumulator w-form for d/df and adds d/dWk into a per-warp shared-memory
//     accumulator addressed by the entry's offset (~64 registers; 16 register accumulators per channel took 127).
// One warp per centre point, 32 centre points per CTA tile; the backward is a persistent tile loop.
//
// Not shipped: kernel weights and d/dWk accumulators resident in registers with dense kernel-point quads on the FMA
// pipe (3x fewer shared-memory wavefronts, but at 128 / 168 registers too few warps per SM stay resident to hide the
// load latencies).  The third-generation backward below is that regrouping with the dense product given to the
// tensor cores and the rows staged by cp.async.
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
  if (bwd) o += (size_t)kPgWarps * kMaxKP * L.CpR * sizeof(float);
  L.total = align_up(o, 16);
  return L;
}

// true when the 12 bytes of a point's coordinates start 4 bytes past an 8-byte boundary (then they END on one).  The
// address decides, not the point's index: a cloud's rows start at b * n * 3 floats, which is only 4-byte aligned for
// odd b when the cloud size n is odd.
__device__ __forceinline__ bool xyz_odd(const float* p) { return (reinterpret_cast<uintptr_t>(p) & 4) != 0; }

// Coordinates of point r from a packed (n,3) array with two requests instead of three: 8 + 4 bytes when they start
// 8-byte aligned, 4 + 8 when they end so.  A scattered 4-byte load costs the L1 one wavefront per distinct line and
// instruction, and these kernels are bound by exactly that.
__device__ __forceinline__ void load_xyz(const float* __restrict__ xyz, int r, float& x, float& y, float& z) {
  const float* p = xyz + (size_t)r * 3;
  if (xyz_odd(p)) {
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

// The 16 influences of one neighbour at relative position (dx, dy, dz) (reference :385-398: sq = |dp - K|^2,
// h = clamp(1 - sqrt(sq)/extent, 0); 'constant': 1), two kernel points per instruction.  pg2_kernel and pg3_body
// both take their influences from here, so they agree bit for bit.
__device__ __forceinline__ void pg_influences(float (&h)[kMaxKP], bool valid, float dx, float dy, float dz,
                                              const u64* __restrict__ s_kx, const u64* __restrict__ s_ky,
                                              const u64* __restrict__ s_kz, int nkp, int influence, float inv_extent) {
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
}

// All 32 lanes: lane `valid` holds one neighbour (relative position, row offset).  Evaluates its influences and
// appends -- for neighbours with at least one non-zero influence, in lane order -- a record {row offset, n} and n
// entries {h, byte offset of Wk[k']} in ascending k'.  Returns the number of records.
__device__ __forceinline__ int pg_stage(uint2* __restrict__ s_rec, float2* __restrict__ s_ent, bool valid, float dx, float dy,
                                        float dz, unsigned row_off, const u64* __restrict__ s_kx,
                                        const u64* __restrict__ s_ky, const u64* __restrict__ s_kz, int nkp, int influence,
                                        float inv_extent, int row_bytes) {
  float h[kMaxKP];
  pg_influences(h, valid, dx, dy, dz, s_kx, s_ky, s_kz, nkp, influence, inv_extent);
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

// Layers wider than 128 channels (32 lanes of 4 channels) run as gridDim.y channel chunks of equal width (a multiple
// of 4, <= 128); every chunk stages the influences again.
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
//                out[b,:,q] = acc ; per-tile BatchNorm partial moments.                      (one tile per CTA)
//   BWD = true : centre = support point j, neighbour rows = g_pm[q_e] over the transposed list of j;
//                out[b,:,j] = acc ; d/dWk accumulated per warp in shared memory.            (persistent tiles)
// =================================================================================================
// (The backward's bound of 3 CTAs per SM sets its register budget; its shared memory -- 88 KB at 72 channels --
// lets 2 be resident.)
template <bool BWD, bool CHUNKED, typename TO>
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
            // the centre point is the support point in the backward, the query in the forward
            float nx, ny, nz;
            load_xyz(nxyz, r, nx, ny, nz);
            const float3 d = BWD ? rel_pos(a, cx, cy, cz, nx, ny, nz) : rel_pos(a, nx, ny, nz, cx, cy, cz);
            dx = d.x, dy = d.y, dz = d.z;
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
      if (owner) {
        s_out[(size_t)(cl + 0) * (kPgTile + 1) + pl] = acc.x;
        s_out[(size_t)(cl + 1) * (kPgTile + 1) + pl] = acc.y;
        s_out[(size_t)(cl + 2) * (kPgTile + 1) + pl] = acc.z;
        s_out[(size_t)(cl + 3) * (kPgTile + 1) + pl] = acc.w;
      }
    }
    __syncthreads();
    // ---- tile -> channel-major (B,C,P)
    const int p = p0 + lane;
    for (int c = warp; c < Cv; c += kPgWarps)
      if (p < P) store_out<TO>(s_out[(size_t)c * (kPgTile + 1) + lane], a, ((size_t)b * a.C + c0 + c) * P + p);
    if constexpr (!BWD) {
      if (a.partial)  // BatchNorm partial moments of the tile, from the output tile in query order
        for (int c = threadIdx.x; c < Cv; c += blockDim.x)
          row_bn_moments(a.partial, tile, a.C, c0 + c, s_out + (size_t)c * (kPgTile + 1), min(kPgTile, P - p0));
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

// =================================================================================================
// Third generation, both directions: per centre point the sums are regrouped per kernel point,
//     U[k',c]     = sum_e h(k', e) * row_e[c]                a (16 x S) x (S x C) product, S = surviving entries
//     out[p,c]    = sum_k' Wk[k',c] * U[k',c]                forward: agg (rows = features);  backward: d/df (rows = g)
//     d/dWk[k',c] += f[j,c] * U[k',c]                        backward only, in registers over the warp's centre points
// so the weight row and the d/dWk accumulator are touched once per (centre point, kernel point) in registers instead
// of once per entry in shared memory.  U is computed on the tensor cores (mma.sync m16n8k8, 3xTF32 as gemm_tc.cuh:
// every operand split into hi + lo TF32 halves, small terms first -- fp32 accuracy).  One warp per centre point:
//   * staging as pg2 (lane = list entry, pg_influences), ballot-compacted; a surviving entry writes its dense
//     h[16] row and its row offset into the warp's slot table, padded with zero rows to a multiple of 8 slots;
//   * the surviving rows go global -> shared with cp.async, 16 bytes per lane, all rows of the batch in flight at once
//     (pad slots alias the first row: 0 * finite);
//   * per 8 slots and 8 channels: 2 B-fragment loads, 3 MMAs into the 4 accumulators of the tile;
//   * epilogue in accumulator-fragment order; the sum over the 8 row groups of the warp by recursive halving;
//   * the next centre point's chain -- list range, the lane's list entry, its coordinates -- is loaded into registers
//     while the current one's rows are in flight, so a centre point starts with its influences.
// A CTA serves a chunk of 8 * NT <= 72 channels (gridDim.y chunks of equal width) and loops over 32-centre tiles.
// =================================================================================================
constexpr int kPg3MaxNT = 9;     // 8-channel MMA tiles per chunk
constexpr int kPg3Row = 72;      // words per staged row / weight row: == 8 (mod 32), B-fragment and Wk reads conflict-free
constexpr int kPg3HRow = 24;     // words per slot-table row {h[16], row offset, spare}: A-fragment reads conflict-free
// The spare words of the slot table carry the next centre point's coordinates (pg3_fetch): words 17..19 of row 0 its
// own, words 20..22 (even row r) or 21..23 (odd r) of row `lane` those of the lane's first list entry
constexpr int kPg3CentreW = 17, kPg3NbrW = 20;
constexpr int kPg3CtasPerSM = 2;

struct Pg3Smem {
  size_t kp_off, wk_off, h_off, rows_off, own_off, out_off, total;
};
__host__ __device__ inline Pg3Smem pg3_smem(bool bwd) {
  Pg3Smem L;
  size_t o = 0;
  L.kp_off = o;
  o += 3 * 8 * sizeof(u64);
  L.wk_off = o;
  o += (size_t)kMaxKP * kPg3Row * sizeof(float);
  L.h_off = o;    // per warp [32][kPg3HRow] (slot table, see kPg3CentreW)
  o += (size_t)kPgWarps * 32 * kPg3HRow * sizeof(float);
  L.rows_off = o;  // per warp [32][kPg3Row]; at the end of a backward CTA: the warp's d/dWk sums [16][kPg3Row]
  o += (size_t)kPgWarps * 32 * kPg3Row * sizeof(float);
  L.own_off = o;  // backward, per warp [kPg3Row]: the centre point's own feature row
  o += bwd ? (size_t)kPgWarps * kPg3Row * sizeof(float) : 0;
  L.out_off = o;
  o += (size_t)kPg3Row * (kPgTile + 1) * sizeof(float);
  L.total = align_up(o, 16);
  return L;
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
// D (16 x 8, fp32) += A (16 x 8, row) * B (8 x 8, col), TF32 operands
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// x = hi + lo, hi = x rounded to TF32 (the subtraction is exact); the tensor core ignores the low mantissa bits of lo
__device__ __forceinline__ void tf32_split(uint32_t x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(__uint_as_float(x)));
  lo = __float_as_uint(__uint_as_float(x) - __uint_as_float(hi));
}

// What a lane needs in registers to start a centre point: its list range and the row of its first list entry
// (e0 + lane < e1).  The coordinates travel through the slot table's spare words (kPg3CentreW, kPg3NbrW).
struct Pg3Next {
  int e0, e1, r;
};

// Issues the loads of centre point pl of `tile` (an empty list past the last tile or the end of the cloud): list range
// and entry into registers, the centre's and the entry's coordinates by cp.async into the slot table at h_a.  Always
// commits exactly one cp.async group, empty or not, so that the caller's wait_group 1 leaves only this one pending.
// Forward: centre = query, list = idx[q][0 .. ncount[q]); backward: centre = support point j, list = its transposed
// entries q * K + k.
template <bool BWD>
__device__ __forceinline__ Pg3Next pg3_fetch(const AggArgs& a, int tile, int pl, int tiles_per_cloud, uint32_t h_a,
                                             int lane) {
  Pg3Next n = {0, 0, 0};
  const int P = BWD ? a.N : a.M, R = BWD ? a.M : a.N;
  const int b = tile / tiles_per_cloud, p = (tile % tiles_per_cloud) * kPgTile + pl;
  if (tile >= a.ntiles || p >= P) {
    cp_async_commit();
    return n;
  }
  if (lane < 3)
    cp_async4(h_a + (kPg3CentreW + lane) * 4, (BWD ? a.support_xyz : a.query_xyz) + ((size_t)b * P + p) * 3 + lane);
  if constexpr (BWD) {
    const int* off = a.csr_off + (size_t)b * (a.N + 1);
    n.e0 = off[p];
    n.e1 = off[p + 1];
    if (n.e0 + lane < n.e1) n.r = a.csr_ent[(size_t)b * a.M * a.K + n.e0 + lane] / a.K;
  } else {
    const size_t gp = (size_t)b * a.M + p;
    n.e1 = a.ncount[gp];
    if (lane < n.e1) n.r = a.idx[gp * a.K + lane];
  }
  if (n.e0 + lane < n.e1) {  // 12 bytes in two requests, the 8-byte piece 8-byte aligned at both ends (as load_xyz)
    const float* q = (BWD ? a.query_xyz : a.support_xyz) + ((size_t)b * R + n.r) * 3;
    const uint32_t d = h_a + (uint32_t)(lane * kPg3HRow + kPg3NbrW + (n.r & 1)) * 4;
    if (xyz_odd(q) != (bool)(n.r & 1)) {  // odd cloud size, odd b: the source's alignment differs from the slot's
      cp_async4(d, q);
      cp_async4(d + 4, q + 1);
      cp_async4(d + 8, q + 2);
    } else if (n.r & 1) {
      cp_async4(d, q);
      cp_async8(d + 4, q + 1);
    } else {
      cp_async8(d, q);
      cp_async4(d + 8, q + 2);
    }
  }
  cp_async_commit();
  return n;
}

// Stages one batch of up to 32 list entries (lane = entry, relative position (dx, dy, dz), row offset roff) for the
// tensor cores: evaluates the influences, ballot-compacts the entries with a non-zero influence into the warp's slot
// table at h_a -- a dense h[16] row and the row offset per slot, padded with zero rows to a multiple of 8 slots --
// and issues the cp.async of their rows into rows_a (2 * NT 16-byte pieces per row, 32 pieces per instruction) as
// one committed group.  Returns the number of slots; 0 when no entry survived (nothing issued).
template <int NT>
__device__ __forceinline__ int pg3_stage(uint32_t h_a, uint32_t rows_a, const float* __restrict__ rows, bool valid, float dx,
                                         float dy, float dz, unsigned roff, const u64* __restrict__ s_kx,
                                         const u64* __restrict__ s_ky, const u64* __restrict__ s_kz, const AggArgs& a,
                                         int lane) {
  float h[kMaxKP];
  pg_influences(h, valid, dx, dy, dz, s_kx, s_ky, s_kz, a.nkp, a.influence, a.inv_extent);
  bool nz = false;
#pragma unroll
  for (int kp = 0; kp < kMaxKP; ++kp) nz |= h[kp] > 0.f;
  const unsigned m = __ballot_sync(0xffffffffu, nz);
  if (m == 0) return 0;
  const int n = __popc(m), n8 = (n + 7) & ~7;
  if (nz) {
    const uint32_t d = h_a + (uint32_t)__popc(m & ((1u << lane) - 1u)) * (kPg3HRow * 4);
#pragma unroll
    for (int q = 0; q < 4; ++q) sts_f4(d + 16 * q, make_float4(h[4 * q], h[4 * q + 1], h[4 * q + 2], h[4 * q + 3]));
    sts_u32(d + 64, roff);
  }
  const unsigned roff0 = __shfl_sync(0xffffffffu, roff, __ffs(m) - 1);
  if (lane >= n && lane < n8) {  // pad slots: zero influences, a valid row
    const uint32_t d = h_a + (uint32_t)lane * (kPg3HRow * 4);
#pragma unroll
    for (int q = 0; q < 4; ++q) sts_f4(d + 16 * q, make_float4(0.f, 0.f, 0.f, 0.f));
    sts_u32(d + 64, roff0);
  }
  __syncwarp();
  for (int id = lane; id < n8 * 2 * NT; id += 32) {
    const int slot = id / (2 * NT), part = id % (2 * NT);
    const unsigned ro = lds_u32(h_a + (uint32_t)slot * (kPg3HRow * 4) + 64);
    cp_async16(rows_a + (uint32_t)(slot * kPg3Row + part * 4) * 4, row_at(rows, ro + 4u * part));
  }
  cp_async_commit();
  return n8;
}

// U += h^T * rows over n8 staged slots (lane (g, t): A fragments from afrag_a, B fragments from bfrag_a)
template <int NT>
__device__ __forceinline__ void pg3_accumulate(float (&U)[NT][4], uint32_t afrag_a, uint32_t bfrag_a, int n8) {
  for (int s = 0; s < n8; s += 8) {
    uint32_t ah[4], al[4];
    const uint32_t aa = afrag_a + (uint32_t)s * (kPg3HRow * 4);
    tf32_split(lds_u32(aa), ah[0], al[0]);
    tf32_split(lds_u32(aa + 8 * 4), ah[1], al[1]);
    tf32_split(lds_u32(aa + 4 * kPg3HRow * 4), ah[2], al[2]);
    tf32_split(lds_u32(aa + 4 * kPg3HRow * 4 + 8 * 4), ah[3], al[3]);
    const uint32_t ba = bfrag_a + (uint32_t)s * (kPg3Row * 4);
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      uint32_t bh0, bl0, bh1, bl1;
      tf32_split(lds_u32(ba + 32 * i), bh0, bl0);
      tf32_split(lds_u32(ba + 32 * i + 4 * kPg3Row * 4), bh1, bl1);
      mma_tf32(U[i], al, bh0, bh1);
      mma_tf32(U[i], ah, bl0, bl1);
      mma_tf32(U[i], ah, bh0, bh1);
    }
  }
}

// Sums v[0 .. V) over the 8 row groups of the warp (lane bits 2, 3, 4) by recursive halving: per level, a lane keeps
// one half of its values and receives the partner's copy of that half, ceil(n / 2) shuffles for n values (17 for
// V = 18, where an xor all-reduce takes 3 V = 54).  Partners pair by lane xor 4, then 8, then 16 -- the order of an
// xor all-reduce with those offsets, so every sum is bit-identical to it.  On return s[j] is the sum of value
// pg3_sum_index<V>(lane, j) when that is >= 0.
template <int V>
__device__ __forceinline__ void pg3_sum_rowgroups(const float (&v)[V], float (&s)[(V + 7) / 8], int lane) {
  constexpr int H1 = (V + 1) / 2, H2 = (V + 3) / 4, H3 = (V + 7) / 8;
  const bool b2 = lane & 4, b3 = lane & 8, b4 = lane & 16;
  float w1[H1], w2[H2];
#pragma unroll
  for (int j = 0; j < H1; ++j) {
    const float lo = v[j], hi = H1 + j < V ? v[H1 + j] : 0.f;
    w1[j] = (b2 ? hi : lo) + __shfl_xor_sync(0xffffffffu, b2 ? lo : hi, 4);
  }
#pragma unroll
  for (int j = 0; j < H2; ++j) {
    const float lo = w1[j], hi = H2 + j < H1 ? w1[H2 + j] : 0.f;
    w2[j] = (b3 ? hi : lo) + __shfl_xor_sync(0xffffffffu, b3 ? lo : hi, 8);
  }
#pragma unroll
  for (int j = 0; j < H3; ++j) {
    const float lo = w2[j], hi = H3 + j < H2 ? w2[H3 + j] : 0.f;
    s[j] = (b4 ? hi : lo) + __shfl_xor_sync(0xffffffffu, b4 ? lo : hi, 16);
  }
}
template <int V>
__device__ __forceinline__ int pg3_sum_index(int lane, int j) {
  constexpr int H1 = (V + 1) / 2, H2 = (V + 3) / 4, H3 = (V + 7) / 8;
  const int r2 = (lane & 16 ? H3 : 0) + j;      // position among the level-2 values
  const int r1 = (lane & 8 ? H2 : 0) + r2;      // among the level-1 values
  const int r0 = (lane & 4 ? H1 : 0) + r1;      // among v
  return r2 < H2 && r1 < H1 && r0 < V ? r0 : -1;  // else a padding slot
}

// BWD = false: centre = query q of cloud b, rows = feat_pm[idx[q][k]], k < ncount[q]; out[b,:,q] = agg and per tile
//              the BatchNorm partial moments (store_bn_moments).
// BWD = true : centre = support point j, rows = g_pm[q_e] over the transposed list of j; out[b,:,j] = d/df and
//              d/dWk in registers -> one partial row per CTA.
template <bool BWD, int NT, typename TO>
__device__ __forceinline__ void pg3_body(const AggArgs& a, int partial_rows) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;  // MMA fragment coordinates
  constexpr int W = 8 * NT;               // channels of this CTA's chunk
  const int c0 = blockIdx.y * W;
  const int Cv = min(W, a.C - c0);  // real channels in it
  const Pg3Smem L = pg3_smem(BWD);
  const u64* s_kx = reinterpret_cast<const u64*>(smem + L.kp_off);
  const u64* s_ky = s_kx + 8;
  const u64* s_kz = s_kx + 16;
  float* s_out = reinterpret_cast<float*>(smem + L.out_off);
  {
    PgSmem P2 = {};
    P2.kp_off = L.kp_off, P2.wk_off = L.wk_off, P2.CpR = kPg3Row;
    pg_load_params(a, P2, smem, c0);
  }
  __syncthreads();

  const uint32_t h_a = smem_u32(smem + L.h_off) + (uint32_t)warp * 32 * kPg3HRow * 4;
  const uint32_t rows_a = smem_u32(smem + L.rows_off) + (uint32_t)warp * 32 * kPg3Row * 4;
  const uint32_t own_a = smem_u32(smem + L.own_off) + (uint32_t)warp * kPg3Row * 4;
  const uint32_t wk_a = smem_u32(smem + L.wk_off) + (uint32_t)(g * kPg3Row + 2 * t) * 4;
  const uint32_t afrag_a = h_a + (uint32_t)(t * kPg3HRow + g) * 4;
  const uint32_t bfrag_a = rows_a + (uint32_t)(t * kPg3Row + g) * 4;
  const int P = BWD ? a.N : a.M;  // centre points per cloud
  const int R = BWD ? a.M : a.N;  // rows of the gathered matrix per cloud
  const int tiles_per_cloud = (P + kPgTile - 1) / kPgTile;

  float dwk[BWD ? NT : 1][4];  // d/dWk of this warp's centre points, accumulator-fragment order
#pragma unroll
  for (int i = 0; i < (BWD ? NT : 1); ++i) dwk[i][0] = dwk[i][1] = dwk[i][2] = dwk[i][3] = 0.f;

  Pg3Next nxt = pg3_fetch<BWD>(a, blockIdx.x, warp, tiles_per_cloud, h_a, lane);
  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    const int b = tile / tiles_per_cloud;
    const int p0 = (tile % tiles_per_cloud) * kPgTile;
    const float* rows = (BWD ? a.g_pm : a.feat_pm) + (size_t)b * R * a.Cp + c0;
    const float* nxyz = (BWD ? a.query_xyz : a.support_xyz) + (size_t)b * R * 3;

    for (int pl = warp; pl < kPgTile; pl += kPgWarps) {
      const int p = p0 + pl;
      const Pg3Next cur = nxt;
      // the warp's next centre point: the next one of this tile, else its first one of the CTA's next tile
      const bool last = pl + kPgWarps >= kPgTile;
      const int ntile = last ? tile + gridDim.x : tile, npl = last ? warp : pl + kPgWarps;
      const int* list = BWD ? a.csr_ent + (size_t)b * a.M * a.K : a.idx + ((size_t)b * a.M + p) * a.K;
      float U[NT][4];
#pragma unroll
      for (int i = 0; i < NT; ++i) U[i][0] = U[i][1] = U[i][2] = U[i][3] = 0.f;
      bool any = false;
      cp_async_wait<0>();  // this centre point's coordinates (pg3_fetch)
      __syncwarp();
      float cx = 0.f, cy = 0.f, cz = 0.f;
      if (cur.e1 > cur.e0) {
        cx = __uint_as_float(lds_u32(h_a + kPg3CentreW * 4));
        cy = __uint_as_float(lds_u32(h_a + (kPg3CentreW + 1) * 4));
        cz = __uint_as_float(lds_u32(h_a + (kPg3CentreW + 2) * 4));
      }
      if constexpr (BWD)
        if (cur.e1 > cur.e0 && lane < 2 * NT)  // own features (d/dWk), waited for with the first batch of rows
          cp_async16(own_a + lane * 16, a.feat_pm + ((size_t)b * a.N + p) * a.Cp + c0 + lane * 4);
      for (int eb = cur.e0; eb < cur.e1; eb += 32) {
        const bool valid = eb + lane < cur.e1;
        int r = cur.r;
        float nx, ny, nz;
        if (valid) {
          if (eb == cur.e0) {
            const uint32_t q = h_a + (uint32_t)(lane * kPg3HRow + kPg3NbrW + (r & 1)) * 4;
            nx = __uint_as_float(lds_u32(q));
            ny = __uint_as_float(lds_u32(q + 4));
            nz = __uint_as_float(lds_u32(q + 8));
          } else {  // later batches (lists longer than 32)
            r = BWD ? list[eb + lane] / a.K : list[eb + lane];
            load_xyz(nxyz, r, nx, ny, nz);
          }
        }
        float dx = 0.f, dy = 0.f, dz = 0.f;
        unsigned roff = 0;
        if (valid) {
          // the centre point is the support point in the backward, the query in the forward
          const float3 d = BWD ? rel_pos(a, cx, cy, cz, nx, ny, nz) : rel_pos(a, nx, ny, nz, cx, cy, cz);
          dx = d.x, dy = d.y, dz = d.z;
          roff = (unsigned)r * (unsigned)a.Cp;
        }
        const int n8 = pg3_stage<NT>(h_a, rows_a, rows, valid, dx, dy, dz, roff, s_kx, s_ky, s_kz, a, lane);
        const bool last = eb + 32 >= cur.e1;
        if (last) nxt = pg3_fetch<BWD>(a, ntile, npl, tiles_per_cloud, h_a, lane);  // while the rows are in flight
        if (n8 == 0) continue;
        if (last)
          cp_async_wait<1>();  // the rows; the next centre point's coordinates may still be in flight
        else
          cp_async_wait<0>();
        __syncwarp();
        pg3_accumulate<NT>(U, afrag_a, bfrag_a, n8);
        any = true;
        __syncwarp();  // the slot table and the rows are overwritten by the next batch
      }
      if (cur.e1 <= cur.e0) nxt = pg3_fetch<BWD>(a, ntile, npl, tiles_per_cloud, h_a, lane);
      if constexpr (BWD) {
        cp_async_wait<0>();  // own row, when no batch had a surviving entry
        __syncwarp();
      }
      // ---- epilogue: lane (g, t) holds U[g][c], U[g][c+1], U[g+8][c], U[g+8][c+1] for c = 8i + 2t
      float v[2 * NT];
#pragma unroll
      for (int i = 0; i < 2 * NT; ++i) v[i] = 0.f;
      if (any) {
#pragma unroll
        for (int i = 0; i < NT; ++i) {
          const float2 w0 = lds_f2(wk_a + 32 * i), w1 = lds_f2(wk_a + 32 * i + 8 * kPg3Row * 4);
          v[2 * i] = fmaf(w1.x, U[i][2], w0.x * U[i][0]);
          v[2 * i + 1] = fmaf(w1.y, U[i][3], w0.y * U[i][1]);
          if constexpr (BWD) {
            const float2 f = lds_f2(own_a + (uint32_t)(8 * i + 2 * t) * 4);
            dwk[i][0] = fmaf(f.x, U[i][0], dwk[i][0]);
            dwk[i][1] = fmaf(f.y, U[i][1], dwk[i][1]);
            dwk[i][2] = fmaf(f.x, U[i][2], dwk[i][2]);
            dwk[i][3] = fmaf(f.y, U[i][3], dwk[i][3]);
          }
        }
      }
      float s[(2 * NT + 7) / 8];
      pg3_sum_rowgroups<2 * NT>(v, s, lane);
#pragma unroll
      for (int j = 0; j < (2 * NT + 7) / 8; ++j) {
        const int k = pg3_sum_index<2 * NT>(lane, j);  // value k = 2 i + (0: x, 1: y): channel 8 i + 2 t + (k & 1)
        if (k >= 0) s_out[(size_t)(8 * (k >> 1) + 2 * t + (k & 1)) * (kPgTile + 1) + pl] = s[j];
      }
      if constexpr (BWD) __syncwarp();  // the own row is overwritten by the next centre point
    }
    __syncthreads();
    // ---- tile -> channel-major (B,C,P)
    const int p = p0 + lane;
    for (int c = warp; c < Cv; c += kPgWarps)
      if (p < P) {
        // fp32: the plain assignment (through store_out the compiler schedules this kernel's loops differently)
        if constexpr (std::is_same<TO, float>::value) a.out[((size_t)b * a.C + c0 + c) * P + p] = s_out[(size_t)c * (kPgTile + 1) + lane];
        else store_out<TO>(s_out[(size_t)c * (kPgTile + 1) + lane], a, ((size_t)b * a.C + c0 + c) * P + p);
      }
    if constexpr (!BWD) {
      if (a.partial)  // BatchNorm partial moments of the tile, over its present queries in order
        for (int c = threadIdx.x; c < Cv; c += blockDim.x)
          row_bn_moments(a.partial, tile, a.C, c0 + c, s_out + (size_t)c * (kPgTile + 1), min(kPgTile, P - p0));
    }
    __syncthreads();
  }
  if constexpr (BWD) {
    // ---- d/dWk: the warps' sums in a fixed order -> one partial row per CTA: (gridDim.x, nkp, C); the rows of
    // `partial` beyond gridDim.x (the caller sums cl3d_agg_bwd_num_blocks rows) are zero-filled
    float* s_red = reinterpret_cast<float*>(smem + L.rows_off);
    constexpr int kRedWarp = 32 * kPg3Row;  // floats between the warps' regions
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      float* d = s_red + (size_t)warp * kRedWarp + g * kPg3Row + 8 * i + 2 * t;
      *reinterpret_cast<float2*>(d) = make_float2(dwk[i][0], dwk[i][1]);
      *reinterpret_cast<float2*>(d + 8 * kPg3Row) = make_float2(dwk[i][2], dwk[i][3]);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < a.nkp * Cv; e += blockDim.x) {
      const int kp = e / Cv, c = e % Cv;
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kPgWarps; ++w) s += s_red[(size_t)w * kRedWarp + kp * kPg3Row + c];
      a.partial[((size_t)blockIdx.x * a.nkp + kp) * a.C + c0 + c] = s;
      for (int row = gridDim.x + blockIdx.x; row < partial_rows; row += gridDim.x)
        a.partial[((size_t)row * a.nkp + kp) * a.C + c0 + c] = 0.f;
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(kPgWarps * 32, kPg3CtasPerSM) pg3_fwd_kernel(const AggArgs a) {
  pg3_body<false, NT, float>(a, 0);
}
template <int NT, typename TO>
__global__ void __launch_bounds__(kPgWarps * 32, kPg3CtasPerSM) pg3_bwd_kernel(const AggArgs a, int partial_rows) {
  pg3_body<true, NT, TO>(a, partial_rows);
}

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
// Third generation: up to 72 padded channels in one chunk, or two equal chunks up to 128.
// CL3D_PG_V2 forces the second generation in both directions (A/B measurements, tests).
static int pg3_num_chunks(int Cp) { return Cp <= 8 * kPg3MaxNT ? 1 : 2; }
static bool pg3_supported(const AggArgs& a) {
  if (getenv("CL3D_PG_V2") || a.Cp > 128) return false;
  return a.Cp % (8 * pg3_num_chunks(a.Cp)) == 0;
}
// The forward takes the third generation only up to 40 padded channels: measured on H100 (DESIGN.md 7.1) it beats
// pg2_kernel<false> at 36 channels but loses at 72 and 128, where its row staging at 2 CTAs per SM costs more than
// pg2's weight-row loads at 4.  That is one chunk, so the forward is instantiated for NT <= kPg3FwdMaxCp / 8 only.
constexpr int kPg3FwdMaxCp = 40;
static bool pg3_fwd_supported(const AggArgs& a) { return a.Cp <= kPg3FwdMaxCp && pg3_supported(a); }

template <bool BWD, int NT>
static void pg3_launch_nt(const AggArgs& a, dim3 grid, int partial_rows, cudaStream_t stream) {
  if constexpr (BWD) {
    with_dtype(a.out_dtype, [&](auto t) {
      using TO = typename decltype(t)::type;
      static std::atomic<unsigned long long> seen_b{0};
      allow_big_smem(pg3_bwd_kernel<NT, TO>, seen_b);
      pg3_bwd_kernel<NT, TO><<<grid, kPgWarps * 32, pg3_smem(true).total, stream>>>(a, partial_rows);
      return CL3D_OK;
    });
  } else {
    static std::atomic<unsigned long long> seen{0};
    allow_big_smem(pg3_fwd_kernel<NT>, seen);
    pg3_fwd_kernel<NT><<<grid, kPgWarps * 32, pg3_smem(false).total, stream>>>(a);
  }
}

// the instance for nt 8-channel tiles per chunk, NT_MAX for nt >= NT_MAX
template <bool BWD, int NT_MAX>
static void pg3_launch(int nt, const AggArgs& a, dim3 grid, int partial_rows, cudaStream_t stream) {
  if constexpr (NT_MAX > 1)
    if (nt < NT_MAX) return pg3_launch<BWD, NT_MAX - 1>(nt, a, grid, partial_rows, stream);
  pg3_launch_nt<BWD, NT_MAX>(a, grid, partial_rows, stream);
}

// one wave of resident CTAs looping over the 32-query tiles (CL3D_TEST_MAX_GRID caps it)
static int pg3_launch_fwd(const AggArgs& a, cudaStream_t stream) {
  const int gx = max(1, min(a.ntiles, min(kPg3CtasPerSM * sm_count(), persistent_grid_cap())));
  pg3_launch<false, kPg3FwdMaxCp / 8>(a.Cp / 8, a, dim3(gx, 1), 0, stream);
  CL3D_LAUNCHED(1);
  return check_launch("pg3_fwd_kernel");
}

// grid_x = rows of a.partial the caller sums; the kernel runs one wave of resident CTAs
static int pg3_launch_bwd(const AggArgs& a, int grid_x, cudaStream_t stream) {
  const int nchunks = pg3_num_chunks(a.Cp);
  const dim3 grid(min(grid_x, kPg3CtasPerSM * sm_count()), nchunks);
  pg3_launch<true, kPg3MaxNT>(a.Cp / (8 * nchunks), a, grid, grid_x, stream);
  CL3D_LAUNCHED(1);
  return check_launch("pg3_bwd_kernel");
}

static int pg2_launch_fwd(const AggArgs& a, int grid_x, cudaStream_t stream) {
  const int nchunks = pg_num_chunks(a.Cp);
  const PgSmem L = pg_smem(pg_chunk_width(a.Cp, nchunks), false);
  static std::atomic<unsigned long long> seen{0};
  if (nchunks == 1) {
    allow_big_smem(pg2_kernel<false, false, float>, seen);
    pg2_kernel<false, false, float><<<grid_x, kPgWarps * 32, L.total, stream>>>(a);
  } else {
    static std::atomic<unsigned long long> seen_c{0};
    allow_big_smem(pg2_kernel<false, true, float>, seen_c);
    pg2_kernel<false, true, float><<<dim3(grid_x, nchunks), kPgWarps * 32, L.total, stream>>>(a);
  }
  CL3D_LAUNCHED(1);
  return check_launch("pg2_kernel<fwd>");
}

static int pg2_launch_bwd(const AggArgs& a, int grid_x, cudaStream_t stream) {
  const int nchunks = pg_num_chunks(a.Cp);
  const PgSmem L = pg_smem(pg_chunk_width(a.Cp, nchunks), true);
  with_dtype(a.out_dtype, [&](auto t) {
    using TO = typename decltype(t)::type;
    static std::atomic<unsigned long long> seen{0};
    if (nchunks == 1) {
      allow_big_smem(pg2_kernel<true, false, TO>, seen);
      pg2_kernel<true, false, TO><<<grid_x, kPgWarps * 32, L.total, stream>>>(a);
    } else {
      static std::atomic<unsigned long long> seen_c{0};
      allow_big_smem(pg2_kernel<true, true, TO>, seen_c);
      pg2_kernel<true, true, TO><<<dim3(grid_x, nchunks), kPgWarps * 32, L.total, stream>>>(a);
    }
    return CL3D_OK;
  });
  CL3D_LAUNCHED(1);
  return check_launch("pg2_kernel<bwd>");
}

int pg_launch(const AggArgs& a, bool bwd, int grid_x, cudaStream_t stream) {
  if (bwd) return pg3_supported(a) ? pg3_launch_bwd(a, grid_x, stream) : pg2_launch_bwd(a, grid_x, stream);
  return pg3_fwd_supported(a) ? pg3_launch_fwd(a, stream) : pg2_launch_fwd(a, grid_x, stream);
}

}  // namespace cl3d
