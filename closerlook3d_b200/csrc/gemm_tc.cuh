// gemm_tc.cuh -- fp32-accurate GEMM on the Hopper tensor cores (wgmma, sm_90a): 3xTF32.
//
//   C[m][n] = sum_k A[m*sa_m + k*sa_k] * B[k*sb_k + n*sb_n]
//
// Every fp32 operand x is split on the fly into  hi = tf32(x)  and  lo = tf32(x - hi)  (round-to-nearest, the
// subtraction is exact), and the product is accumulated in fp32 registers as
//       lo_a*hi_b + hi_a*lo_b + hi_a*hi_b
// The dropped terms (lo*lo and the rounding of the two lo parts) are <= 3 * 2^-22 relative per product --
// the same order as one fp32 rounding -- so the result meets the fp32 1e-5 parity bar of the local
// aggregation path (BASELINE.json north_star) while the multiply-adds leave the FMA pipe.
//
// One CTA = one 128 x BN output tile (BN = N rounded up to 32, <= 160), two warpgroups (256 threads):
//   * all threads stage 16-wide k chunks: global (any element strides; float4 along k when possible) ->
//     registers -> hi/lo split -> shared memory in the canonical K-major no-swizzle GMMA layout
//       offset(row, k) = (k/4)*LBO + (row/8)*SBO + (row%8)*16 + (k%4)*4     [bytes]
//     i.e. a [k/4][row] array of float4 (padded), so the staging stores are conflict-free 16-byte writes;
//   * warpgroup w owns output rows [64w, 64w + 64): per chunk it issues, for each of the 2 k-steps and each
//     32-column slice of the tile, 3 wgmma.m64n32k8 (tf32) into its register accumulators;
//   * a 3-deep ring of stages with at most one wgmma group in flight per warpgroup keeps staging and MMA
//     overlapped (the next chunk is loaded into registers while the tensor core works);
//   * the tensor core accumulates with truncation (about half an ulp of bias per accumulation step), so its
//     accumulators only ever hold kTcPromote chunks (64 k, 24 accumulation steps): then they are added, rounded
//     to nearest, into a second set of fp32 registers and restarted from zero.  The error of a long reduction
//     then grows like an ordinary fp32 sum instead of linearly with k;
//   * the sums are staged through the (now idle) stage buffers and written to C / the split-K partial
//     tile row-contiguously.
// Rows of A / B beyond M / N are not zero-filled but clamped to the last valid row: a row only feeds its own
// output row / column, which is never stored.  Only the k tail is zero-filled.
// With gridDim.z > 1 the k range is divided among CTAs (split-K) and reduced afterwards in a fixed order.
#pragma once
#include <atomic>

#include "common.cuh"

namespace cl3d {

constexpr int kTcBM = 128, kTcBK = 16, kTcStages = 3, kTcThreads = 256, kTcSliceN = 32;
constexpr int kTcMaxN = 160;   // widest tile: two register sets of 80 accumulators per thread
constexpr int kTcPromote = 4;  // chunks per tensor-core accumulation window
// Shared-memory operand layout (canonical K-major, no swizzle): 8-row x 16-byte core matrices of 128 contiguous
// bytes, 8-row groups back to back (SBO = 128); LBO = distance between the 16-byte k columns = rows*16 + pad.
// The pad is chosen per staging mode so that a quarter warp's float4 stores hit 8 distinct 16-byte bank groups:
// LBO/16 == 2 (mod 8) for mode 1, == 1 (mod 8) for mode 2.
constexpr int kTcSbo = 128;
__host__ __device__ inline int tc_row_off(int r) { return r * 16; }

struct TcGemmArgs {
  const float* A; long long sa_m, sa_k;
  const float* B; long long sb_k, sb_n;
  int M, N, K, k_per_split;
  float* C; long long sc_m, sc_n;
  float* partial;  // split-K partial tiles [z][M][N] or nullptr
};

// cute/arch/mma_sm90_desc.hpp GmmaDescriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base_offset
// [49,52)=0, layout_type [62,64)=0 (no swizzle).  K-major, no swizzle: LBO = byte distance between the two
// 16-byte k columns of one MMA, SBO = distance between 8-row groups.
__device__ __forceinline__ uint64_t tc_smem_desc_hi(uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
__device__ __forceinline__ uint64_t tc_smem_desc(uint64_t hi, uint32_t saddr) { return hi | ((saddr >> 4) & 0x3FFFu); }

// D[64 x 32] += A[64 x 8] * B[8 x 32]^T, both operands tf32 from shared memory (K-major)
__device__ __forceinline__ void tc_wgmma_n32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db)
      : "memory");
}
__device__ __forceinline__ void tc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tc_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// round-to-nearest (ties away in magnitude) to the 10-bit TF32 mantissa: two integer ops
__device__ __forceinline__ float tf32_round(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}

__device__ __forceinline__ void tc_split_store(unsigned char* hi_base, unsigned char* lo_base, uint32_t off, float4 v) {
  float4 h, l;
  h.x = tf32_round(v.x); h.y = tf32_round(v.y); h.z = tf32_round(v.z); h.w = tf32_round(v.w);
  // |lo| <= 2^-11 |x| with either sign; the tensor core drops its low 13 mantissa bits (<= 2^-21 |x|, unbiased)
  l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
  *reinterpret_cast<float4*>(hi_base + off) = h;
  *reinterpret_cast<float4*>(lo_base + off) = l;
}

// one float4 = 4 consecutive k of one row.  VEC: a 16-byte load; else 4 loads `sk` elements apart.
template <bool VEC, bool FULL>
__device__ __forceinline__ float4 tc_load4(const float* __restrict__ p, int sk, int k, int kend) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if constexpr (VEC) {
    if (FULL || k < kend) v = __ldg(reinterpret_cast<const float4*>(p));
  } else {
    if (FULL || k + 0 < kend) v.x = __ldg(p);
    if (FULL || k + 1 < kend) v.y = __ldg(p + sk);
    if (FULL || k + 2 < kend) v.z = __ldg(p + 2 * sk);
    if (FULL || k + 3 < kend) v.w = __ldg(p + 3 * sk);
  }
  return v;
}

__host__ __device__ inline int tc_lbo(int rows, int mode = 1) { return rows * 16 + (mode == 2 ? 16 : 32); }
__host__ __device__ inline size_t tc_stage_bytes(int bn) { return 2 * 4 * (size_t)tc_lbo(kTcBM) + 2 * 4 * (size_t)tc_lbo(bn); }
__host__ inline size_t tc_smem_bytes(int bn) { return kTcStages * tc_stage_bytes(bn); }
__host__ inline int tc_tile_n(int N) { return N >= kTcMaxN ? kTcMaxN : ((N + kTcSliceN - 1) & ~(kTcSliceN - 1)); }

// WN = widest tile this instantiation serves (its accumulator registers); AV / BV: how the operand is read
// (staging modes below: 1 = float4 along k, 2 = float4 along the rows + register transpose, 0 = scalar).
template <int WN, int AV, int BV>
__global__ void __launch_bounds__(kTcThreads) gemm_tf32x3_kernel(const TcGemmArgs g) {
  extern __shared__ __align__(128) unsigned char tc_smem[];
  constexpr int NS = WN / kTcSliceN;                                // 32-column slices
  constexpr int NA = AV == 2 ? 4 : 2;                               // float4 registers of the A chunk per thread
  constexpr int NB = BV == 2 ? 4 : (WN * 4 + kTcThreads - 1) / kTcThreads;  // ... of the B chunk
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int m0 = blockIdx.y * kTcBM, n0 = blockIdx.x * kTcMaxN;
  const int bn = min(kTcMaxN, ((g.N - n0) + kTcSliceN - 1) & ~(kTcSliceN - 1));  // columns of this tile
  const int kbeg = blockIdx.z * g.k_per_split, kend = min(g.K, kbeg + g.k_per_split);
  const int nchunks = (kend - kbeg + kTcBK - 1) / kTcBK;
  const int lbo_a = tc_lbo(kTcBM, AV), lbo_b = tc_lbo(bn, BV);
  const uint32_t stage_bytes = (uint32_t)tc_stage_bytes(bn);

  // staging maps (fixed per thread), one float4 = 4 consecutive k of one row once it is in shared memory:
  //   mode 1 (k is the unit stride): 4 threads per row, each loads its float4 directly (64 contiguous bytes/row)
  //   mode 2 (row is the unit stride): a thread loads a 4 (k) x 4 (rows) block as four float4 along the rows
  //           (a warp reads 4 k-rows x 128 contiguous bytes per instruction) and transposes it in registers
  //   mode 0 (anything else): one row per thread, four scalar loads
  const int ska = (int)g.sa_k, skb = (int)g.sb_k;
  const int nb4 = bn * 4;
  const bool a_on = AV != 2 || tid < kTcBM;  // mode 2: 128 blocks of 4 x 4 cover the A chunk
  const bool b2_on = tid < bn;               // mode 2: bn blocks of 4 x 4 cover the B chunk
  uint32_t ga[2], sa[2], gb[NB], sb[NB];     // element offset in global memory, byte offset in the stage
  int cb2 = 0;
  if constexpr (AV == 2) {
    const int mg = tid >> 2 & 31, c = tid & 3;
    ga[0] = (uint32_t)((long long)min(m0 + 4 * mg, g.M - 4) + (long long)(4 * c) * g.sa_k);
    sa[0] = (uint32_t)(c * lbo_a + tc_row_off(4 * mg));
  } else {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int e = tid + kTcThreads * j;
      const int r = AV ? (e >> 2) : (e & (kTcBM - 1)), c = AV ? (e & 3) : (e >> 7);
      ga[j] = (uint32_t)((long long)min(m0 + r, g.M - 1) * g.sa_m + (long long)(4 * c) * g.sa_k);
      sa[j] = (uint32_t)(c * lbo_a + tc_row_off(r));
    }
  }
  if constexpr (BV == 2) {
    const int e = min(tid, bn - 1);
    const int mg = e >> 2, c = e & 3;
    cb2 = c;
    gb[0] = (uint32_t)((long long)min(n0 + 4 * mg, g.N - 4) + (long long)(4 * c) * g.sb_k);
    sb[0] = (uint32_t)(8 * lbo_a + c * lbo_b + tc_row_off(4 * mg));
  } else {
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int e = min(tid + kTcThreads * j, nb4 - 1);
      const int r = BV ? (e >> 2) : (e % bn), c = BV ? (e & 3) : (e / bn);
      gb[j] = (uint32_t)((long long)min(n0 + r, g.N - 1) * g.sb_n + (long long)(4 * c) * g.sb_k);
      sb[j] = (uint32_t)(8 * lbo_a + c * lbo_b + tc_row_off(r));
    }
  }
  const int ca = tid & 3, cb = tid & 3;  // k column (of 4), k tail only

  float4 ra[NA], rb[NB];
  auto load_chunk = [&](int k0) {
    const float* Ak = g.A + (long long)k0 * g.sa_k;
    const float* Bk = g.B + (long long)k0 * g.sb_k;
    const bool full_chunk = k0 + kTcBK <= kend;
    if constexpr (AV == 2) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        ra[kk] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a_on && (full_chunk || k0 + 4 * ca + kk < kend))
          ra[kk] = __ldg(reinterpret_cast<const float4*>(Ak + ga[0] + kk * ska));
      }
    } else if (full_chunk) {
#pragma unroll
      for (int j = 0; j < 2; ++j) ra[j] = tc_load4<AV == 1, true>(Ak + ga[j], ska, 0, 0);
    } else {
#pragma unroll
      for (int j = 0; j < 2; ++j)
        ra[j] = tc_load4<AV == 1, false>(Ak + ga[j], ska, k0 + 4 * (AV ? ca : (tid + kTcThreads * j) >> 7), kend);
    }
    if constexpr (BV == 2) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        rb[kk] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b2_on && (full_chunk || k0 + 4 * cb2 + kk < kend))
          rb[kk] = __ldg(reinterpret_cast<const float4*>(Bk + gb[0] + kk * skb));
      }
    } else if (full_chunk) {
#pragma unroll
      for (int j = 0; j < NB; ++j)
        if (tid + kTcThreads * j < nb4) rb[j] = tc_load4<BV == 1, true>(Bk + gb[j], skb, 0, 0);
    } else {
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const int e = tid + kTcThreads * j;
        if (e < nb4) rb[j] = tc_load4<BV == 1, false>(Bk + gb[j], skb, k0 + 4 * (BV ? cb : e / bn), kend);
      }
    }
  };
  auto store_chunk = [&](unsigned char* st) {
    unsigned char* lo_a = st + 4 * lbo_a;
    unsigned char* lo_b = st + 4 * lbo_b;
    if constexpr (AV == 2) {
      if (a_on) {
        tc_split_store(st, lo_a, sa[0], make_float4(ra[0].x, ra[1].x, ra[2].x, ra[3].x));
        tc_split_store(st, lo_a, sa[0] + 16, make_float4(ra[0].y, ra[1].y, ra[2].y, ra[3].y));
        tc_split_store(st, lo_a, sa[0] + 32, make_float4(ra[0].z, ra[1].z, ra[2].z, ra[3].z));
        tc_split_store(st, lo_a, sa[0] + 48, make_float4(ra[0].w, ra[1].w, ra[2].w, ra[3].w));
      }
    } else {
#pragma unroll
      for (int j = 0; j < 2; ++j) tc_split_store(st, lo_a, sa[j], ra[j]);
    }
    if constexpr (BV == 2) {
      if (b2_on) {
        tc_split_store(st, lo_b, sb[0], make_float4(rb[0].x, rb[1].x, rb[2].x, rb[3].x));
        tc_split_store(st, lo_b, sb[0] + 16, make_float4(rb[0].y, rb[1].y, rb[2].y, rb[3].y));
        tc_split_store(st, lo_b, sb[0] + 32, make_float4(rb[0].z, rb[1].z, rb[2].z, rb[3].z));
        tc_split_store(st, lo_b, sb[0] + 48, make_float4(rb[0].w, rb[1].w, rb[2].w, rb[3].w));
      }
    } else {
#pragma unroll
      for (int j = 0; j < NB; ++j)
        if (tid + kTcThreads * j < nb4) tc_split_store(st, lo_b, sb[j], rb[j]);
    }
  };

  float acc[NS][16], sum[NS][16];  // tensor-core window, rounded running sum
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[s][q] = sum[s][q] = 0.f;
  const uint64_t dhi_a = tc_smem_desc_hi((uint32_t)lbo_a, kTcSbo), dhi_b = tc_smem_desc_hi((uint32_t)lbo_b, kTcSbo);
  const int nslices = bn / kTcSliceN;

  load_chunk(kbeg);
  for (int i = 0; i < nchunks; ++i) {
    // Stage i % 3 was last read by the MMAs of chunk i - 3.  Each warpgroup waited for those at the end of
    // iteration i - 2, before the barrier of iteration i - 1 that every thread has passed.
    unsigned char* st = tc_smem + (size_t)(i % kTcStages) * stage_bytes;
    store_chunk(st);
    fence_proxy_async();  // generic-proxy writes -> visible to the tensor core (async proxy)
    __syncthreads();
    if (i + 1 < nchunks) load_chunk(kbeg + (i + 1) * kTcBK);  // in flight while the tensor core works
    const uint32_t a_hi = smem_u32(st) + (uint32_t)(wg * 64 / 8 * kTcSbo), a_lo = a_hi + 4 * lbo_a,
                   b_hi = smem_u32(st) + 8 * lbo_a, b_lo = b_hi + 4 * lbo_b;
    tc_wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTcBK / 8; ++kk) {
      const uint32_t oa = kk * 2 * lbo_a, ob = kk * 2 * lbo_b;
      const uint64_t dah = tc_smem_desc(dhi_a, a_hi + oa), dal = tc_smem_desc(dhi_a, a_lo + oa);
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        if (s < nslices) {  // uniform over the CTA
          const uint32_t os = ob + (uint32_t)(s * kTcSliceN / 8 * kTcSbo);
          const uint64_t dbh = tc_smem_desc(dhi_b, b_hi + os), dbl = tc_smem_desc(dhi_b, b_lo + os);
          tc_wgmma_n32(acc[s], dal, dbh);
          tc_wgmma_n32(acc[s], dah, dbl);
          tc_wgmma_n32(acc[s], dah, dbh);
        }
      }
    }
    tc_wgmma_commit();
    if ((i + 1) % kTcPromote == 0 || i + 1 == nchunks) {
      tc_wgmma_wait<0>();
#pragma unroll
      for (int s = 0; s < NS; ++s)
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          sum[s][q] = __fadd_rn(sum[s][q], acc[s][q]);
          acc[s][q] = 0.f;
        }
    } else {
      tc_wgmma_wait<1>();
    }
  }
  tc_wgmma_wait<0>();
  __syncthreads();  // every MMA of the CTA has read its operands: the stage buffers are free

  // epilogue.  Accumulator fragment of wgmma m64nN (per 8-column block j of a slice): warp w of the warpgroup
  // holds rows 16w + lane/4 (+8), columns 8j + 2*(lane%4) (+1).  The tile goes through a padded shared-memory
  // slab and is then written out row-contiguously so that the global stores are fully coalesced.
  const int ldp = bn + 4;  // (bn+4) % 32 is 4 or 20: the per-lane float4 rows below hit distinct banks
  float* ep = reinterpret_cast<float*>(tc_smem);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      if (s < nslices) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = s * kTcSliceN + 8 * j + c0;
          *reinterpret_cast<float2*>(ep + r0 * ldp + c) = make_float2(sum[s][4 * j], sum[s][4 * j + 1]);
          *reinterpret_cast<float2*>(ep + (r0 + 8) * ldp + c) = make_float2(sum[s][4 * j + 2], sum[s][4 * j + 3]);
        }
      }
    }
  }
  __syncthreads();
  {
    constexpr int RW = kTcBM / (kTcThreads / 32);  // rows per warp
    const int mw = m0 + warp * RW;       // first row of this warp
    const int rows = min(RW, g.M - mw);  // valid rows (<= 0: nothing to write)
    const int ncol = min(bn, g.N - n0);  // valid columns of this tile
    const float* ew = ep + (size_t)warp * RW * ldp;
    float* dst;
    long long sm, sn;
    if (g.partial) {
      dst = g.partial + ((size_t)blockIdx.z * g.M + mw) * g.N + n0;
      sm = g.N; sn = 1;
    } else {
      dst = g.C + (long long)mw * g.sc_m + (long long)n0 * g.sc_n;
      sm = g.sc_m; sn = g.sc_n;
    }
    const bool al = (reinterpret_cast<uintptr_t>(dst) & 15) == 0;
    if (rows > 0 && sn == 1 && sm == ncol && (ncol & 3) == 0 && al) {
      // the warp's rows are one contiguous range of the output: flat float4 copy, 4 vectors in flight
      int r = 0, c = 4 * lane;
      while (c >= ncol) { c -= ncol; ++r; }
      float4* d4 = reinterpret_cast<float4*>(dst) + lane;
      while (r < rows) {
        float4 v[4];
        bool ok[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ok[u] = r < rows;
          if (ok[u]) v[u] = *reinterpret_cast<const float4*>(ew + r * ldp + c);
          c += 128;
          while (c >= ncol) { c -= ncol; ++r; }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (ok[u]) d4[32 * u] = v[u];
        d4 += 128;
      }
    } else if (rows > 0 && sn == 1 && (sm & 3) == 0 && (ncol & 3) == 0 && al) {
      for (int c = 4 * lane; c < ncol; c += 128) {
        int r = 0;
        for (; r + 4 <= rows; r += 4) {
          float4 v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(ew + (r + u) * ldp + c);
#pragma unroll
          for (int u = 0; u < 4; ++u) *reinterpret_cast<float4*>(dst + (long long)(r + u) * sm + c) = v[u];
        }
        for (; r < rows; ++r)
          *reinterpret_cast<float4*>(dst + (long long)r * sm + c) = *reinterpret_cast<const float4*>(ew + r * ldp + c);
      }
    } else if (rows > 0 && sm == 1) {
      // transposed output (the row index is the unit-stride one): lane = row
      for (int c = 0; c < ncol; ++c)
        if (lane < rows) dst[lane + (long long)c * sn] = ew[lane * ldp + c];
    } else {
      for (int r = 0; r < rows; ++r)
        for (int c = lane; c < ncol; c += 32) dst[(long long)r * sm + (long long)c * sn] = ew[r * ldp + c];
    }
  }
}

// Host-side shape check: 32-bit element offsets inside the kernel.
inline bool tc_gemm_supported(const TcGemmArgs& g) {
  auto ext = [](long long r, long long sr, long long k, long long sk) { return (r - 1) * sr + (k - 1) * sk; };
  const long long lim = (1ll << 31) - 1;
  return g.sa_m >= 0 && g.sa_k >= 0 && g.sb_k >= 0 && g.sb_n >= 0 && ext(g.M, g.sa_m, g.K, g.sa_k) < lim &&
         ext(g.N, g.sb_n, g.K, g.sb_k) < lim && g.sa_k < (1 << 28) && g.sb_k < (1 << 28);
}

template <int WN, int AV, int BV>
inline void tc_gemm_launch_k(const TcGemmArgs& g, dim3 grid, size_t smem, cudaStream_t stream) {
  static std::atomic<unsigned long long> attr_set{0};
  if (first_call_on_device(attr_set))
    cudaFuncSetAttribute(gemm_tf32x3_kernel<WN, AV, BV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)tc_smem_bytes(WN));
  gemm_tf32x3_kernel<WN, AV, BV><<<grid, kTcThreads, smem, stream>>>(g);
}

template <int WN, int AV>
inline void tc_gemm_launch_b(const TcGemmArgs& g, int bv, dim3 grid, size_t smem, cudaStream_t stream) {
  if (bv == 1) tc_gemm_launch_k<WN, AV, 1>(g, grid, smem, stream);
  else if (bv == 2) tc_gemm_launch_k<WN, AV, 2>(g, grid, smem, stream);
  else tc_gemm_launch_k<WN, AV, 0>(g, grid, smem, stream);
}

template <int WN>
inline void tc_gemm_launch_nb(const TcGemmArgs& g, int av, int bv, dim3 grid, size_t smem, cudaStream_t stream) {
  if (av == 1) tc_gemm_launch_b<WN, 1>(g, bv, grid, smem, stream);
  else if (av == 2) tc_gemm_launch_b<WN, 2>(g, bv, grid, smem, stream);
  else tc_gemm_launch_b<WN, 0>(g, bv, grid, smem, stream);
}

// Launch.  k_per_split must be a multiple of kTcBK when splits > 1.
inline void tc_gemm_launch(const TcGemmArgs& g, int splits, cudaStream_t stream) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool kal = g.K % 4 == 0 && g.k_per_split % 4 == 0;
  const int av = (g.sa_k == 1 && al16(g.A) && g.sa_m % 4 == 0 && kal) ? 1
                 : (g.sa_m == 1 && al16(g.A) && g.sa_k % 4 == 0 && g.M % 4 == 0) ? 2 : 0;
  const int bv = (g.sb_k == 1 && al16(g.B) && g.sb_n % 4 == 0 && kal) ? 1
                 : (g.sb_n == 1 && al16(g.B) && g.sb_k % 4 == 0 && g.N % 4 == 0) ? 2 : 0;
  const int bn = tc_tile_n(g.N);
  const size_t smem = tc_smem_bytes(bn);
  dim3 grid((g.N + kTcMaxN - 1) / kTcMaxN, (g.M + kTcBM - 1) / kTcBM, splits);
  if (bn <= 96) tc_gemm_launch_nb<96>(g, av, bv, grid, smem, stream);
  else tc_gemm_launch_nb<kTcMaxN>(g, av, bv, grid, smem, stream);
}

}  // namespace cl3d
