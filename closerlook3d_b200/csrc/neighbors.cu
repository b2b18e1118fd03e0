// neighbors.cu -- neighbour search for the local-aggregation engine (sm_90a).
//
//   cl3d_ball_query_algo  bit-exact replacement of the reference's masked_ordered_ball_query
//                         (/root/reference/pytorch/ops/pt_custom_ops/_ext_src/src/masked_ordered_ball_query_gpu.cu:11-96)
//   cl3d_nearest_query    bit-exact replacement of masked_nearest_query (masked_nearest_query_gpu.cu:8-62)
//   cl3d_build_csr        transposed neighbour lists for the gather-form backward kernels (arrival order, or
//                         ascending entry order with `deterministic`)
//
// The reference scans ALL support points per query on B thread blocks.  Here the support cloud is binned
// into a uniform grid (cell edge >= radius, counting sort, points stored as float4 {x,y,z,index} in cell
// order so that the three x-adjacent cells of a row are ONE contiguous, coalesced range) and one warp per
// query walks the 9 rows of its 27 neighbouring cells.  The reference's result depends on index order
// (first 3K in-radius points by index, nearest-overwrite rule, stable sort by distance, cyclic padding);
// that rule is reproduced on the candidate set with 64-bit keys (d2 bits << 32 | index), which order
// exactly like the reference's stable sort because candidates are unique in index.
#include <limits.h>
#include <stdlib.h>

#include "common.cuh"

namespace cl3d {

struct GridParams {
  float ox, oy, oz, inv_h;
  int gx, gy, gz, ncells;
  int n_valid, pad0, pad1, pad2;
};

constexpr int kBQWarps = 8;           // warps per CTA in the query kernels
constexpr int kCandCap = 256;         // on-chip candidate list per warp (grid path); overflow -> exact brute force
constexpr int kBruteMaxN = 2048;      // below this the grid is not worth its extra launches

__host__ __device__ inline int cell_cap_for(int N) { return N * 4 > 4096 ? N * 4 : 4096; }

// ---------------------------------------------------------------------------------------------
// grid build
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int cell_coord(float x, float o, float inv_h, int g) {
  int c = (int)((x - o) * inv_h);
  return c < 0 ? 0 : (c >= g ? g - 1 : c);
}

// The whole grid build of a cloud is one CTA of 1024 threads: valid prefix (the reference stops at the first mask 0,
// masked_ordered_ball_query_gpu.cu:49-52), bounding box, grid dimensions, cell counts, exclusive scan, scatter into
// cell order.  The cell counters live in shared memory up to kFusedGridCells cells (every BASELINE cloud: 10^3 .. 15^3
// cells), so counting is shared-memory atomics; larger grids keep them in the cloud's slice of the workspace.
constexpr int kFusedGridCells = 12288;   // 48 KB of counters

__device__ __forceinline__ GridParams make_grid_params(int nv, const float (&mn)[3], const float (&mx)[3], float radius,
                                                       int cell_cap) {
  GridParams p;
  p.n_valid = nv;
  p.pad0 = p.pad1 = p.pad2 = 0;
  if (nv == 0) {
    p.ox = p.oy = p.oz = 0.f;
    p.inv_h = 1.f;
    p.gx = p.gy = p.gz = 1;
    p.ncells = 1;
    return p;
  }
  const float ex = mx[0] - mn[0], ey = mx[1] - mn[1], ez = mx[2] - mn[2];
  // cell edge strictly larger than the radius: two points closer than `radius` along an axis then land
  // in the same or adjacent cells even after fp32 rounding of the cell coordinate (< 512 per axis).
  float h = radius * 1.001f;
  if (!(h > 1e-20f)) h = 1e-20f;
  int gx = 1, gy = 1, gz = 1;
  for (int it = 0; it < 400; ++it) {  // bounded: non-finite coordinates fall back to a single cell
    const float fx = fminf(ex / h, 510.f), fy = fminf(ey / h, 510.f), fz = fminf(ez / h, 510.f);
    const int tx = (int)fx + 1, ty = (int)fy + 1, tz = (int)fz + 1;
    if ((long long)tx * ty * tz <= (long long)cell_cap && ex / h < 511.f && ey / h < 511.f && ez / h < 511.f) {
      gx = tx;
      gy = ty;
      gz = tz;
      break;
    }
    h *= 1.25f;
  }
  p.ox = mn[0];
  p.oy = mn[1];
  p.oz = mn[2];
  p.inv_h = 1.0f / h;
  p.gx = gx;
  p.gy = gy;
  p.gz = gz;
  p.ncells = gx * gy * gz;
  return p;
}

// Block-wide exclusive scan of one value per thread: returns the sum of the values of the threads before this one.
// Warp scan, then a scan of the warps' totals in s_warp[32].  Every thread of the block calls it.
__device__ __forceinline__ int block_exclusive_scan(int sum, int* s_warp) {
  int v = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) >= o) v += t;
  }
  if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    int w = threadIdx.x < (blockDim.x >> 5) ? s_warp[threadIdx.x] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (threadIdx.x >= o) w += t;
    }
    s_warp[threadIdx.x] = w;
  }
  __syncthreads();
  return v - sum + ((threadIdx.x >> 5) > 0 ? s_warp[(threadIdx.x >> 5) - 1] : 0);
}

__global__ void __launch_bounds__(1024) grid_build_fused_kernel(const float* __restrict__ xyz, const int* __restrict__ mask,
                                                                int N, float radius, int cell_cap,
                                                                GridParams* __restrict__ params,
                                                                int* __restrict__ cell_cnt, int* __restrict__ cell_start,
                                                                int2* __restrict__ cell_rank, float4* __restrict__ sorted) {
  extern __shared__ int s_cnt_smem[];  // kFusedGridCells counters, then reused as the cell starts
  const int b = blockIdx.x;
  xyz += (size_t)b * N * 3;
  mask += (size_t)b * N;
  cell_start += (size_t)b * (cell_cap + 1);
  cell_rank += (size_t)b * N;
  sorted += (size_t)b * N;
  __shared__ int s_first;
  __shared__ float s_red[6][32];
  __shared__ GridParams s_p;
  __shared__ int s_warp[32];
  // Every loop of this kernel is a per-thread strided loop over the cloud with one CTA per cloud: written with four
  // independent loads in flight per thread (a one-load-per-iteration loop exposes a full L2 latency per point; the
  // first version of this kernel took 38 us at N = 15000 for that reason alone).
  if (threadIdx.x == 0) s_first = N;
  __syncthreads();
  int first = N;
  {
    const int T = blockDim.x;
    int i = threadIdx.x;
    for (; i + 3 * T < N; i += 4 * T) {   // no early exit: the loads must not depend on each other
      const int m0 = mask[i], m1 = mask[i + T], m2 = mask[i + 2 * T], m3 = mask[i + 3 * T];
      if (m3 == 0) first = min(first, i + 3 * T);
      if (m2 == 0) first = min(first, i + 2 * T);
      if (m1 == 0) first = min(first, i + T);
      if (m0 == 0) first = min(first, i);
    }
    for (; i < N; i += T)
      if (mask[i] == 0) first = min(first, i);
  }
  if (first < N) atomicMin(&s_first, first);
  __syncthreads();
  const int nv = s_first;
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  {
    const int T = blockDim.x;
    int i = threadIdx.x;
    for (; i + 3 * T < nv; i += 4 * T) {
      float v[4][3];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int a = 0; a < 3; ++a) v[u][a] = xyz[(size_t)(i + u * T) * 3 + a];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          mn[a] = fminf(mn[a], v[u][a]);
          mx[a] = fmaxf(mx[a], v[u][a]);
        }
    }
    for (; i < nv; i += T) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float v = xyz[(size_t)i * 3 + a];
        mn[a] = fminf(mn[a], v);
        mx[a] = fmaxf(mx[a], v);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
    if ((threadIdx.x & 31) == 0) {
      s_red[a][threadIdx.x >> 5] = mn[a];
      s_red[3 + a][threadIdx.x >> 5] = mx[a];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float gmn[3], gmx[3];
    for (int a = 0; a < 3; ++a) {
      gmn[a] = s_red[a][0];
      gmx[a] = s_red[3 + a][0];
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
        gmn[a] = fminf(gmn[a], s_red[a][w]);
        gmx[a] = fmaxf(gmx[a], s_red[3 + a][w]);
      }
    }
    s_p = make_grid_params(nv, gmn, gmx, radius, cell_cap);
    params[b] = s_p;
  }
  __syncthreads();
  const GridParams p = s_p;
  // counters in shared memory when they fit (every BASELINE cloud), else in this cloud's slice of the global buffer
  int* s_cnt = p.ncells <= kFusedGridCells ? s_cnt_smem : cell_cnt + (size_t)b * cell_cap;
  for (int c = threadIdx.x; c < p.ncells; c += blockDim.x) s_cnt[c] = 0;
  __syncthreads();
  {
    const int T = blockDim.x;
    int i = threadIdx.x;
    for (; i + 3 * T < nv; i += 4 * T) {
      float v[4][3];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int a = 0; a < 3; ++a) v[u][a] = xyz[(size_t)(i + u * T) * 3 + a];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int cell = cell_coord(v[u][0], p.ox, p.inv_h, p.gx) +
                         p.gx * (cell_coord(v[u][1], p.oy, p.inv_h, p.gy) + p.gy * cell_coord(v[u][2], p.oz, p.inv_h, p.gz));
        cell_rank[i + u * T] = make_int2(cell, atomicAdd(&s_cnt[cell], 1));
      }
    }
    for (; i < nv; i += T) {
      const int cell = cell_coord(xyz[(size_t)i * 3 + 0], p.ox, p.inv_h, p.gx) +
                       p.gx * (cell_coord(xyz[(size_t)i * 3 + 1], p.oy, p.inv_h, p.gy) +
                               p.gy * cell_coord(xyz[(size_t)i * 3 + 2], p.oz, p.inv_h, p.gz));
      cell_rank[i] = make_int2(cell, atomicAdd(&s_cnt[cell], 1));
    }
  }
  __syncthreads();
  // exclusive scan of the counters, in place
  const int per = (p.ncells + blockDim.x - 1) / blockDim.x;
  const int lo = min((int)threadIdx.x * per, p.ncells), hi = min(lo + per, p.ncells);
  int sum = 0;
  for (int c = lo; c < hi; ++c) sum += s_cnt[c];
  int base = block_exclusive_scan(sum, s_warp);
  for (int c = lo; c < hi; ++c) {
    const int n = s_cnt[c];
    s_cnt[c] = base;
    cell_start[c] = base;
    base += n;
  }
  if (threadIdx.x == blockDim.x - 1) cell_start[p.ncells] = base;  // == n_valid
  __syncthreads();
  {
    const int T = blockDim.x;
    int i = threadIdx.x;
    for (; i + 3 * T < nv; i += 4 * T) {
      int2 cr[4];
      float v[4][3];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        cr[u] = cell_rank[i + u * T];
#pragma unroll
        for (int a = 0; a < 3; ++a) v[u][a] = xyz[(size_t)(i + u * T) * 3 + a];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        sorted[s_cnt[cr[u].x] + cr[u].y] = make_float4(v[u][0], v[u][1], v[u][2], __int_as_float(i + u * T));
    }
    for (; i < nv; i += T) {
      const int2 cr = cell_rank[i];
      sorted[s_cnt[cr.x] + cr.y] = make_float4(xyz[(size_t)i * 3 + 0], xyz[(size_t)i * 3 + 1], xyz[(size_t)i * 3 + 2],
                                               __int_as_float(i));
    }
  }
}

// The grid's workspace, one slice per cloud in each region.  grid_workspace(nullptr, ...) only sizes it.
struct GridWorkspace {
  int cap;               // cells per cloud at most
  GridParams* params;    // B
  int* cell_cnt;         // B x cap: the counters of grids above kFusedGridCells cells
  int* cell_start;       // B x (cap + 1)
  int2* cell_rank;       // B x N: cell id + arrival rank in the cell
  float4* sorted;        // B x N: {x, y, z, index} in cell order
  size_t bytes;
};

static GridWorkspace grid_workspace(void* base, int B, int N) {
  GridWorkspace g;
  g.cap = cell_cap_for(N);
  size_t off = 0;
  auto take = [&](size_t n) {
    void* p = base ? (unsigned char*)base + off : nullptr;
    off += align_up(n, 256);
    return p;
  };
  g.params = (GridParams*)take(sizeof(GridParams) * (size_t)B);
  g.cell_cnt = (int*)take(sizeof(int) * (size_t)B * g.cap);
  g.cell_start = (int*)take(sizeof(int) * (size_t)B * (g.cap + 1));
  g.cell_rank = (int2*)take(sizeof(int2) * (size_t)B * N);
  g.sorted = (float4*)take(sizeof(float4) * (size_t)B * N);
  g.bytes = off;
  return g;
}

// every cloud's valid supports into its cell grid, one CTA per cloud
static void build_grid(const float* support_xyz, const int* support_mask, int B, int N, float radius,
                       const GridWorkspace& g, cudaStream_t stream) {
  static std::atomic<unsigned long long> attr{0};
  allow_big_smem(grid_build_fused_kernel, attr);
  grid_build_fused_kernel<<<B, 1024, kFusedGridCells * sizeof(int), stream>>>(support_xyz, support_mask, N, radius,
                                                                              g.cap, g.params, g.cell_cnt, g.cell_start,
                                                                              g.cell_rank, g.sorted); CL3D_LAUNCHED(1);
}

// ---------------------------------------------------------------------------------------------
// per-query selection shared by the grid and brute-force paths
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ u64 make_key(float d2, int idx) {
  return ((u64)__float_as_uint(d2) << 32) | (unsigned)idx;  // d2 >= +0 -> bit pattern is monotone
}

// s_sorted[rank of L[i]] = index of L[i] for every rank < K.  A lane ranks E keys (i = base + e*32 + lane) per pass
// over the list, so each broadcast load serves E compares and the E counts are independent dependency chains.
template <int E>
__device__ __forceinline__ void rank_keys(const u64* L, int cnt, int* s_sorted, int K) {
  const int lane = lane_id();
  for (int base = 0; base < cnt; base += 32 * E) {
    u64 my[E];
    int rho[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int i = base + e * 32 + lane;
      my[e] = i < cnt ? L[i] : ~0ull;
      rho[e] = 0;
    }
#pragma unroll 4
    for (int j = 0; j < cnt; ++j) {
      const u64 v = L[j];
#pragma unroll
      for (int e = 0; e < E; ++e) rho[e] += (v < my[e]) ? 1 : 0;
    }
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (base + e * 32 + lane < cnt && rho[e] < K) s_sorted[rho[e]] = (int)(unsigned)(my[e] & 0xffffffffu);
  }
}

// L[0..cnt) holds the reference's candidate list (any order; unique indices).  Emits the first K of the list
// sorted by (d2, index) -- identical to the reference's stable sort of an index-ascending list
// (masked_ordered_ball_query_gpu.cu:77) -- then the cyclic padding (:83-86) and masks (:79-93).
// Selection by counting: the keys are unique, so a key's place in the sorted list is the number of smaller keys.  Each
// lane ranks the keys it holds against the whole list (broadcast shared-memory loads, cnt * ceil(cnt/32) compares
// per lane) and writes the ones that land below K -- one loop for every cnt <= 3K, no sorting network.
// csr_cnt (may be null): per-support-point reference counters of this cloud.  Every counted slot (k < ncount, or all K
// slots with csr_all) takes its rank inside the support point's transposed list right here (one int atomic per
// slot, K of them in flight per warp), so the list build that follows is a scan and an atomic-free scatter.
__device__ __forceinline__ void emit_query(const u64* L, int cnt, int* s_sorted, int K, int qm, int* __restrict__ idx_out,
                                           int* __restrict__ mask_out, int* __restrict__ ncount_out,
                                           int* __restrict__ csr_cnt = nullptr, int* __restrict__ rank_out = nullptr,
                                           int csr_all = 0) {
  const int lane = lane_id();
  if (cnt <= 32)
    rank_keys<1>(L, cnt, s_sorted, K);
  else
    rank_keys<2>(L, cnt, s_sorted, K);
  __syncwarp();
  const int ncnt = qm != 0 ? (cnt < K ? cnt : K) : K;
  for (int k = lane; k < K; k += 32) {
    int v = 0;
    if (cnt > 0) v = s_sorted[k < cnt ? k : (k % cnt)];
    idx_out[k] = v;
    if (mask_out) mask_out[k] = (k < cnt && qm != 0) ? 1 : 0;
    if (csr_cnt && (csr_all || k < ncnt)) rank_out[k] = atomicAdd(&csr_cnt[v], 1);
  }
  if (ncount_out && lane == 0) *ncount_out = ncnt;
  __syncwarp();
}

// Exact index-order scan of the reference (warp-cooperative): first 3K in-radius points in index order,
// global first-strict-minimum, overwrite rule (:45-75).  Returns cnt; list in L (capacity >= 3K).
template <typename LoadXYZ>
__device__ __forceinline__ int brute_force_collect(LoadXYZ load, int n_valid, float qx, float qy, float qz, float r2,
                                                   int cap3k, u64* L) {
  const int lane = lane_id();
  const unsigned lt = (1u << lane) - 1u;
  int T = 0;
  u64 best = ~0ull;
  for (int base = 0; base < n_valid; base += 32) {
    const int i = base + lane;
    bool in = false;
    u64 key = 0;
    if (i < n_valid) {
      float x, y, z;
      load(i, x, y, z);
      float d2 = ref_d2(qx, qy, qz, x, y, z);
      in = d2 < r2;
      key = make_key(d2, i);
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (in) {
      int pos = T + __popc(m & lt);
      if (pos < cap3k) L[pos] = key;
      best = key < best ? key : best;
    }
    T += __popc(m);
  }
  __syncwarp();
  if (T >= cap3k && cap3k > 0) {
    best = warp_min_u64(best);
    const u64 last = L[cap3k - 1];
    if ((unsigned)(best & 0xffffffffu) > (unsigned)(last & 0xffffffffu)) {
      __syncwarp();
      if (lane == 0) L[cap3k - 1] = best;
    }
    __syncwarp();
    return cap3k;
  }
  return T;
}

// ---------------------------------------------------------------------------------------------
// brute-force kernel for small clouds: the cloud lives in shared memory as float4, padded to a multiple of 32
// with far-away sentinels (and sentinels behind the valid prefix), so the scan loop has no bounds checks
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBQWarps * 32) ball_query_brute_kernel(
    const float* __restrict__ query_xyz, const float* __restrict__ support_xyz, const int* __restrict__ query_mask,
    const int* __restrict__ support_mask, int N, int M, float radius, int K, int queries_per_cta,
    int* __restrict__ idx, int* __restrict__ idx_mask, int* __restrict__ ncount, int* __restrict__ csr_cnt,
    int* __restrict__ csr_rank, int csr_all) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.y;
  const int cap3k = 3 * K;
  const int npad = (N + 31) & ~31;
  float4* s_pts = reinterpret_cast<float4*>(smem_raw);                               // npad points
  u64* s_list = reinterpret_cast<u64*>(smem_raw + (size_t)npad * 16);                // warps * 3K keys
  int* s_sorted = reinterpret_cast<int*>(s_list + (size_t)kBQWarps * cap3k);         // warps * K
  __shared__ int s_first;
  if (threadIdx.x == 0) s_first = N;
  __syncthreads();
  const int* sm = support_mask + (size_t)b * N;
  const float* sx = support_xyz + (size_t)b * N * 3;
  int first = N;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (sm[i] == 0) { first = i; break; }
  if (first < N) atomicMin(&s_first, first);
  __syncthreads();
  const int n_valid = s_first;
  for (int i = threadIdx.x; i < npad; i += blockDim.x)
    s_pts[i] = i < n_valid ? make_float4(sx[i * 3 + 0], sx[i * 3 + 1], sx[i * 3 + 2], 0.f)
                           : make_float4(1.0e18f, 1.0e18f, 1.0e18f, 0.f);  // never inside any ball
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  const float r2 = __fmul_rn(radius, radius);
  u64* L = s_list + (size_t)warp * cap3k;
  int* srt = s_sorted + (size_t)warp * K;
  const int q0 = blockIdx.x * queries_per_cta;
  const int q1 = min(q0 + queries_per_cta, M);
  for (int q = q0 + warp; q < q1; q += kBQWarps) {
    const float* qp = query_xyz + ((size_t)b * M + q) * 3;
    const float qx = qp[0], qy = qp[1], qz = qp[2];
    // index-order scan (:48-70): the first 3K in-radius points, in index order
    int T = 0;
    for (int base = 0; base < npad; base += 32) {
      const float4 p = s_pts[base + lane];
      const float d2 = ref_d2(qx, qy, qz, p.x, p.y, p.z);
      const bool in = d2 < r2;
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (in) {
        const int pos = T + __popc(m & lt);
        if (pos < cap3k) L[pos] = make_key(d2, base + lane);
      }
      T += __popc(m);
    }
    __syncwarp();
    int cnt = T;
    if (T >= cap3k) {
      // rare: more than 3K in the ball -> the global nearest may lie beyond the cut (:59-62,72-75)
      u64 best = ~0ull;
      for (int base = 0; base < npad; base += 32) {
        const float4 p = s_pts[base + lane];
        const float d2 = ref_d2(qx, qy, qz, p.x, p.y, p.z);
        if (d2 < r2) {
          const u64 key = make_key(d2, base + lane);
          best = key < best ? key : best;
        }
      }
      best = warp_min_u64(best);
      const u64 last = L[cap3k - 1];
      __syncwarp();
      if (lane == 0 && (unsigned)(best & 0xffffffffu) > (unsigned)(last & 0xffffffffu)) L[cap3k - 1] = best;
      __syncwarp();
      cnt = cap3k;
    }
    const size_t o = ((size_t)b * M + q);
    emit_query(L, cnt, srt, K, query_mask[o], idx + o * K, idx_mask ? idx_mask + o * K : nullptr,
               ncount ? ncount + o : nullptr, csr_cnt ? csr_cnt + (size_t)b * N : nullptr,
               csr_rank ? csr_rank + o * K : nullptr, csr_all);
  }
}

// ---------------------------------------------------------------------------------------------
// grid kernel: one warp per query, 9 contiguous cell-row ranges
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBQWarps * 32, 5) ball_query_grid_kernel(
    const float* __restrict__ query_xyz, const float* __restrict__ support_xyz, const int* __restrict__ query_mask,
    const GridParams* __restrict__ params, const int* __restrict__ cell_start, const float4* __restrict__ sorted,
    int B, int N, int M, float radius, int K, int cell_cap, int cell_order, int* __restrict__ idx,
    int* __restrict__ idx_mask, int* __restrict__ ncount, int* __restrict__ csr_cnt, int* __restrict__ csr_rank,
    int csr_all) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int cap3k = 3 * K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  u64* s_cand = reinterpret_cast<u64*>(smem_raw) + (size_t)warp * kCandCap;
  u64* s_keep = reinterpret_cast<u64*>(smem_raw) + (size_t)kBQWarps * kCandCap + (size_t)warp * cap3k;
  int* s_sorted = reinterpret_cast<int*>(reinterpret_cast<u64*>(smem_raw) + (size_t)kBQWarps * (kCandCap + cap3k)) +
                  (size_t)warp * K;
  const long long gw = (long long)blockIdx.x * kBQWarps + warp;
  if (gw >= (long long)B * M) return;
  const int b = (int)(gw / M);
  const GridParams p = params[b];
  const float4* pts = sorted + (size_t)b * N;
  // Query set == support set (cell_order): warp w takes the w-th valid point in cell order, so the warps of a CTA and
  // the CTAs resident beside it walk the same cells and find their candidates in L1.  The padded rows past the valid
  // prefix still get lists; they follow in index order.
  int q = (int)(gw - (long long)b * M);
  float qx, qy, qz;
  if (cell_order && q < p.n_valid) {
    const float4 c = pts[q];
    q = __float_as_int(c.w);
    qx = c.x;
    qy = c.y;
    qz = c.z;
  } else {
    const float* qp = query_xyz + ((size_t)b * M + q) * 3;
    qx = qp[0];
    qy = qp[1];
    qz = qp[2];
  }
  const size_t gq = (size_t)b * M + q;
  const float r2 = __fmul_rn(radius, radius);
  const unsigned lt = (1u << lane) - 1u;
  const int* cs = cell_start + (size_t)b * (cell_cap + 1);

  // query cell (may lie outside the support's bounding box)
  float fx = floorf((qx - p.ox) * p.inv_h), fy = floorf((qy - p.oy) * p.inv_h), fz = floorf((qz - p.oz) * p.inv_h);
  fx = fminf(fmaxf(fx, -2.f), (float)p.gx + 1.f);
  fy = fminf(fmaxf(fy, -2.f), (float)p.gy + 1.f);
  fz = fminf(fmaxf(fz, -2.f), (float)p.gz + 1.f);
  const int cx = (int)fx, cy = (int)fy, cz = (int)fz;
  const int x0 = max(cx - 1, 0), x1 = min(cx + 1, p.gx - 1);

  // The 9 (dz, dy) rows of the 27 cells: lane r < 9 loads row r's [start, end) -- all 18 loads in flight together --
  // and a 9-lane scan lays the rows end to end, so the candidates are one range [0, total) walked in full 32-lane
  // chunks.  Position i belongs to the last row whose offset is <= i (empty rows share their successor's offset).
  int st = 0, len = 0;
  if (lane < 9 && p.n_valid > 0 && x0 <= x1) {
    const int z = cz + lane / 3 - 1, y = cy + lane % 3 - 1;
    if (z >= 0 && z < p.gz && y >= 0 && y < p.gy) {
      const int row = p.gx * (y + p.gy * z);
      st = cs[row + x0];
      len = cs[row + x1 + 1] - st;
    }
  }
  int incl = len;
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 8);
  const int shift = st - (incl - len);  // row's source position minus its concatenated offset
  int roff[9];
#pragma unroll
  for (int r = 1; r < 9; ++r) roff[r] = __shfl_sync(0xffffffffu, incl - len, r);

  int T = 0;
  u64 best = ~0ull;
  for (int base = 0; base < total; base += 32) {
    const int i = base + lane;
    int row = 0;
#pragma unroll
    for (int r = 1; r < 9; ++r) row += i >= roff[r] ? 1 : 0;
    const int src = i + __shfl_sync(0xffffffffu, shift, row);
    bool in = false;
    u64 key = 0;
    if (i < total) {
      const float4 c = pts[src];
      const float d2 = ref_d2(qx, qy, qz, c.x, c.y, c.z);
      in = d2 < r2;
      key = make_key(d2, __float_as_int(c.w));
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (in) {
      const int pos = T + __popc(m & lt);
      if (pos < kCandCap) s_cand[pos] = key;
      best = key < best ? key : best;
    }
    T += __popc(m);
  }
  __syncwarp();
  const u64* list = s_cand;
  int cnt = T;
  if (T > kCandCap) {
    // neighbourhood does not fit on chip: exact index-order scan straight from global memory (rare)
    const float* sx = support_xyz + (size_t)b * N * 3;
    cnt = brute_force_collect(
        [&](int i, float& x, float& y, float& z) {
          x = sx[i * 3 + 0];
          y = sx[i * 3 + 1];
          z = sx[i * 3 + 2];
        },
        p.n_valid, qx, qy, qz, r2, cap3k, s_keep);
    list = s_keep;
  } else if (T > cap3k) {
    // more than 3K candidates: the reference keeps the 3K SMALLEST INDICES (it scans in index order, :64-68),
    // then overwrites the last kept one with the global nearest if that lies beyond it (:72-75).
    best = warp_min_u64(best);
    int kept = 0;  // warp-uniform running count
    for (int base = 0; base < T; base += 32) {
      const int i = base + lane;
      bool keep = false;
      u64 my = 0;
      if (i < T) {
        my = s_cand[i];
        const unsigned myidx = (unsigned)(my & 0xffffffffu);
        int r = 0;
        for (int j = 0; j < T; ++j) r += ((unsigned)(s_cand[j] & 0xffffffffu) < myidx) ? 1 : 0;
        keep = r < cap3k;
        if (r == cap3k - 1 && (unsigned)(best & 0xffffffffu) > myidx) my = best;  // overwrite rule
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) s_keep[kept + __popc(m & lt)] = my;
      kept += __popc(m);
    }
    __syncwarp();
    list = s_keep;
    cnt = cap3k;
  }
  emit_query(list, cnt, s_sorted, K, query_mask[gq], idx + gq * K, idx_mask ? idx_mask + gq * K : nullptr,
             ncount ? ncount + gq : nullptr, csr_cnt ? csr_cnt + (size_t)b * N : nullptr,
             csr_rank ? csr_rank + gq * K : nullptr, csr_all);
}

// ---------------------------------------------------------------------------------------------
// nearest query: thread per query, support tiles in shared memory, sequential in index order so the
// reference's first-strict-minimum tie rule holds (masked_nearest_query_gpu.cu:37-52)
// ---------------------------------------------------------------------------------------------
constexpr int kNNTile = 1024;
__global__ void __launch_bounds__(256) nearest_query_kernel(const float* __restrict__ query_xyz,
                                                            const float* __restrict__ support_xyz,
                                                            const int* __restrict__ query_mask,
                                                            const int* __restrict__ support_mask, int N, int M,
                                                            int* __restrict__ idx, int* __restrict__ idx_mask) {
  __shared__ float s_xyz[kNNTile * 3];
  __shared__ int s_first;
  const int b = blockIdx.y;
  const float* sx = support_xyz + (size_t)b * N * 3;
  const int* sm = support_mask + (size_t)b * N;
  if (threadIdx.x == 0) s_first = N;
  __syncthreads();
  int first = N;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (sm[i] == 0) { first = i; break; }
  if (first < N) atomicMin(&s_first, first);
  __syncthreads();
  const int n_valid = s_first;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (q < M) {
    const float* qp = query_xyz + ((size_t)b * M + q) * 3;
    qx = qp[0];
    qy = qp[1];
    qz = qp[2];
  }
  float min_d = 100.f;
  int min_i = -1;
  for (int t0 = 0; t0 < n_valid; t0 += kNNTile) {
    const int tn = min(kNNTile, n_valid - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < tn * 3; i += blockDim.x) s_xyz[i] = sx[(size_t)t0 * 3 + i];
    __syncthreads();
    if (q < M) {
#pragma unroll 4
      for (int i = 0; i < tn; ++i) {
        const float d2 = ref_d2(qx, qy, qz, s_xyz[i * 3], s_xyz[i * 3 + 1], s_xyz[i * 3 + 2]);
        if (d2 < min_d) {
          min_d = d2;
          min_i = t0 + i;
        }
      }
    }
  }
  if (q < M) {
    idx[(size_t)b * M + q] = min_i;
    idx_mask[(size_t)b * M + q] = query_mask[(size_t)b * M + q] == 0 ? 0 : 1;
  }
}

// ---------------------------------------------------------------------------------------------
// nearest query over the cell grid (clouds too large for the tile scan above): thread per query, the supports'
// cells visited in Chebyshev rings around the query's cell.  A point outside the (2r+1)^3 block is at least as far
// as the block's nearest face that is not the grid's own boundary, so the walk stops as soon as the best distance
// is below that bound; ties go to the smaller index, which is the reference's first strict minimum in index order
// (masked_nearest_query_gpu.cu:37-52), and its start value min_dist = 100 is kept (:35).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void nn_scan(const float4* __restrict__ sorted, int s, int e, float qx, float qy, float qz,
                                        float& best_d, int& best_i) {
  for (int t = s; t < e; ++t) {
    const float4 p = sorted[t];
    const float d2 = ref_d2(qx, qy, qz, p.x, p.y, p.z);
    const int i = __float_as_int(p.w);
    if (d2 < best_d || (d2 == best_d && i < best_i)) {
      best_d = d2;
      best_i = i;
    }
  }
}

__global__ void __launch_bounds__(256) nearest_query_grid_kernel(const float* __restrict__ query_xyz,
                                                                 const int* __restrict__ query_mask,
                                                                 const GridParams* __restrict__ params,
                                                                 const int* __restrict__ cell_start,
                                                                 const float4* __restrict__ sorted, int N, int M,
                                                                 int cell_cap, int* __restrict__ idx,
                                                                 int* __restrict__ idx_mask) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= M) return;
  const GridParams p = params[b];
  const int* cs = cell_start + (size_t)b * (cell_cap + 1);
  const float4* pts = sorted + (size_t)b * N;
  const float* qp = query_xyz + ((size_t)b * M + q) * 3;
  const float qx = qp[0], qy = qp[1], qz = qp[2];
  float best_d = 100.f;
  int best_i = -1;
  if (p.n_valid > 0) {
    const float h = 1.0f / p.inv_h;
    const int cx = cell_coord(qx, p.ox, p.inv_h, p.gx), cy = cell_coord(qy, p.oy, p.inv_h, p.gy),
              cz = cell_coord(qz, p.oz, p.inv_h, p.gz);
    const int rmax = max(max(max(cx, p.gx - 1 - cx), max(cy, p.gy - 1 - cy)), max(cz, p.gz - 1 - cz));
    for (int r = 0; r <= rmax; ++r) {
      const int x0 = max(cx - r, 0), x1 = min(cx + r, p.gx - 1);
      const int y0 = max(cy - r, 0), y1 = min(cy + r, p.gy - 1);
      const int z0 = max(cz - r, 0), z1 = min(cz + r, p.gz - 1);
      for (int z = z0; z <= z1; ++z)
        for (int y = y0; y <= y1; ++y) {
          const int base = p.gx * (y + p.gy * z);
          if (z - cz == r || cz - z == r || y - cy == r || cy - y == r) {
            // a row of the ring's shell: its cells are consecutive in the cell-sorted array
            nn_scan(pts, cs[base + x0], cs[base + x1 + 1], qx, qy, qz, best_d, best_i);
          } else {  // inner row: only the two end cells belong to ring r
            if (cx - r >= 0) nn_scan(pts, cs[base + cx - r], cs[base + cx - r + 1], qx, qy, qz, best_d, best_i);
            if (cx + r <= p.gx - 1) nn_scan(pts, cs[base + cx + r], cs[base + cx + r + 1], qx, qy, qz, best_d, best_i);
          }
        }
      // lower bound of the distance to any point outside the block; a face on the grid's boundary has nothing
      // behind it.  The margin covers the fp32 rounding of the cell coordinates (points) and of the faces.
      float bound = 3.0e38f;
      const float qa[3] = {qx, qy, qz}, oa[3] = {p.ox, p.oy, p.oz};
      const int ca[3] = {cx, cy, cz}, ga[3] = {p.gx, p.gy, p.gz};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (ca[a] - r > 0) {
          const float face = oa[a] + (float)(ca[a] - r) * h;
          bound = fminf(bound, (qa[a] - face) - (0.01f * h + 2e-6f * (fabsf(qa[a]) + fabsf(face))));
        }
        if (ca[a] + r < ga[a] - 1) {
          const float face = oa[a] + (float)(ca[a] + r + 1) * h;
          bound = fminf(bound, (face - qa[a]) - (0.01f * h + 2e-6f * (fabsf(qa[a]) + fabsf(face))));
        }
      }
      if (bound > 0.f) {
        if (best_i >= 0 && sqrtf(best_d) < bound) break;  // nothing outside can be nearer or tie
        if (bound > 10.01f) break;                        // nothing outside can beat the start value 100
      }
    }
  }
  idx[(size_t)b * M + q] = best_i;
  idx_mask[(size_t)b * M + q] = query_mask[(size_t)b * M + q] == 0 ? 0 : 1;
}

// ---------------------------------------------------------------------------------------------
// CSR ("who gathers me") build: count -> scan -> fill
// ---------------------------------------------------------------------------------------------
__global__ void csr_count_kernel(const int* __restrict__ idx, const int* __restrict__ ncount, int N, int M, int K,
                                 int* __restrict__ cnt) {
  const int b = blockIdx.y;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * K) return;
  const int q = (int)(e / K), k = (int)(e % K);
  if (k >= ncount[(size_t)b * M + q]) return;
  atomicAdd(&cnt[(size_t)b * N + idx[((size_t)b * M + q) * K + k]], 1);
}

__global__ void __launch_bounds__(1024) csr_scan_kernel(int N, const int* __restrict__ cnt, int* __restrict__ off,
                                                        int* __restrict__ cursor) {
  const int b = blockIdx.x;
  cnt += (size_t)b * N;
  if (cursor) cursor += (size_t)b * N;
  off += (size_t)b * (N + 1);
  __shared__ int s_warp[32];
  const int per = (N + blockDim.x - 1) / blockDim.x;
  const int lo = min(threadIdx.x * per, N), hi = min(lo + per, N);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += cnt[i];
  int base = block_exclusive_scan(sum, s_warp);
  for (int i = lo; i < hi; ++i) {
    off[i] = base;
    if (cursor) cursor[i] = base;
    base += cnt[i];
  }
  if (threadIdx.x == blockDim.x - 1) off[N] = base;
}

__global__ void csr_fill_kernel(const int* __restrict__ idx, const int* __restrict__ ncount, int N, int M, int K,
                                int* __restrict__ cursor, int* __restrict__ ent) {
  const int b = blockIdx.y;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * K) return;
  const int q = (int)(e / K), k = (int)(e % K);
  if (k >= ncount[(size_t)b * M + q]) return;
  const int j = idx[((size_t)b * M + q) * K + k];
  const int pos = atomicAdd(&cursor[(size_t)b * N + j], 1);
  ent[(size_t)b * M * K + pos] = (int)e;
}

// lists from ranks taken during the search: ent[off[j] + rank] = entry id  (no atomics)
__global__ void csr_place_kernel(const int* __restrict__ idx, const int* __restrict__ ncount,
                                 const int* __restrict__ rank, const int* __restrict__ off, int N, int M, int K,
                                 int csr_all, int* __restrict__ ent) {
  const int b = blockIdx.y;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * K) return;
  const int q = (int)(e / K), k = (int)(e % K);
  if (!csr_all && k >= ncount[(size_t)b * M + q]) return;
  const size_t g = (size_t)b * M * K + e;
  ent[(size_t)b * M * K + off[(size_t)b * (N + 1) + idx[g]] + rank[g]] = (int)e;
}

// ---------------------------------------------------------------------------------------------
// canonical list order (deterministic mode): the lists above are filled in atomic arrival order; these two passes
// rewrite each list from a scratch copy in ascending entry order q*K + k, the order a serial fill would give.
// Entries of a list are unique, so an entry's place is the number of smaller entries in its list.
// ---------------------------------------------------------------------------------------------
constexpr int kCanonWarpMax = 1024;  // longest list one warp ranks (len^2/32 compares per lane); longer: grid pass
constexpr int kCanonTile = 2048;     // list tile the grid pass stages in shared memory

// one warp per list; lists longer than kCanonWarpMax are queued for csr_canon_long_kernel
__global__ void __launch_bounds__(256) csr_canon_warp_kernel(const int* __restrict__ off, const int* __restrict__ src,
                                                             int B, int N, int M, int K, int* __restrict__ ent,
                                                             int* __restrict__ long_cnt, int* __restrict__ long_list) {
  const long long gw = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (gw >= (long long)B * N) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(gw / N), j = (int)(gw - (long long)b * N);
  const int o0 = off[(size_t)b * (N + 1) + j];
  const int len = off[(size_t)b * (N + 1) + j + 1] - o0;
  if (len > kCanonWarpMax) {
    if (lane == 0) long_list[atomicAdd(long_cnt, 1)] = (int)gw;
    return;
  }
  const int* s = src + (size_t)b * M * K + o0;
  int* d = ent + (size_t)b * M * K + o0;
  if (len <= 32) {  // the common case: one entry per lane, ranked against the others through shuffles
    const int v = lane < len ? s[lane] : INT_MAX;
    int r = 0;
    for (int t = 0; t < len; ++t) r += __shfl_sync(0xffffffffu, v, t) < v ? 1 : 0;
    if (lane < len) d[r] = v;
    return;
  }
  for (int base = 0; base < len; base += 64) {
    const int i0 = base + lane, i1 = base + 32 + lane;
    const int v0 = i0 < len ? s[i0] : INT_MAX, v1 = i1 < len ? s[i1] : INT_MAX;
    int r0 = 0, r1 = 0;
#pragma unroll 4
    for (int t = 0; t < len; ++t) {
      const int v = s[t];
      r0 += v < v0 ? 1 : 0;
      r1 += v < v1 ? 1 : 0;
    }
    if (i0 < len) d[r0] = v0;
    if (i1 < len) d[r1] = v1;
  }
}

// the queued long lists (coincident points, or isolated and padded queries filling all K slots with one point), one
// at a time with every thread of the grid: thread t ranks entries t, t + T, ... against the list staged in tiles
__global__ void __launch_bounds__(256) csr_canon_long_kernel(const int* __restrict__ off, const int* __restrict__ src,
                                                             int N, int M, int K, int* __restrict__ ent,
                                                             const int* __restrict__ long_cnt,
                                                             const int* __restrict__ long_list) {
  __shared__ int s_t[kCanonTile];
  const int nl = *long_cnt;
  const int T = gridDim.x * blockDim.x;
  for (int l = 0; l < nl; ++l) {
    const int gw = long_list[l];
    const int b = gw / N, j = gw - b * N;
    const int o0 = off[(size_t)b * (N + 1) + j];
    const int len = off[(size_t)b * (N + 1) + j + 1] - o0;
    const int* s = src + (size_t)b * M * K + o0;
    int* d = ent + (size_t)b * M * K + o0;
    for (int base = blockIdx.x * blockDim.x; base < len; base += T) {  // CTA-uniform bounds
      const int i = base + threadIdx.x;
      const int v = i < len ? s[i] : INT_MAX;
      int r = 0;
      for (int t0 = 0; t0 < len; t0 += kCanonTile) {
        const int n = min(kCanonTile, len - t0);
        __syncthreads();
        for (int t = threadIdx.x; t < n; t += blockDim.x) s_t[t] = s[t0 + t];
        __syncthreads();
#pragma unroll 8
        for (int t = 0; t < n; ++t) r += s_t[t] < v ? 1 : 0;
      }
      if (i < len) d[r] = v;
    }
  }
}

// scratch of the canonical pass behind a caller's workspace: the arrival-order copy, the long-list queue, its count
static size_t canon_workspace_bytes(int B, int N, int M, int K) {
  const size_t b = (size_t)(B > 0 ? B : 1);
  return align_up(sizeof(int) * b * (size_t)(M > 0 ? M : 1) * (size_t)K, 256) +
         align_up(sizeof(int) * b * (size_t)N, 256) + 256;
}

struct CanonScratch {
  int* src;
  int* long_list;
  int* long_cnt;
};

static CanonScratch canon_scratch(void* w, int B, int N, int M, int K) {
  CanonScratch c;
  c.src = (int*)w;
  c.long_list = (int*)((unsigned char*)w + align_up(sizeof(int) * (size_t)B * (size_t)M * (size_t)K, 256));
  c.long_cnt = (int*)((unsigned char*)c.long_list + align_up(sizeof(int) * (size_t)B * (size_t)N, 256));
  return c;
}

// the lists in c.src (arrival order) -> ent (ascending entries); sizes only, so a captured graph replays it
static void canon_lists(const int* off, const CanonScratch& c, int B, int N, int M, int K, int* ent,
                        cudaStream_t stream) {
  cudaMemsetAsync(c.long_cnt, 0, sizeof(int), stream);
  const long long lists = (long long)B * N;
  csr_canon_warp_kernel<<<(unsigned)((lists + 7) / 8), 256, 0, stream>>>(off, c.src, B, N, M, K, ent, c.long_cnt,
                                                                         c.long_list); CL3D_LAUNCHED(1);
  csr_canon_long_kernel<<<2 * sm_count(), 256, 0, stream>>>(off, c.src, N, M, K, ent, c.long_cnt, c.long_list);
  CL3D_LAUNCHED(1);
}

}  // namespace cl3d

// =================================================================================================
// C ABI
// =================================================================================================
using namespace cl3d;

extern "C" size_t cl3d_ball_query_workspace_bytes(int B, int N, int M, int K) {
  (void)M;
  (void)K;
  if (B <= 0 || N <= 0) return 256;
  return grid_workspace(nullptr, B, N).bytes;
}

static int ball_query_impl(const float* query_xyz, const float* support_xyz, const int* query_mask,
                           const int* support_mask, int B, int N, int M, float radius, int K, int* idx,
                           int* idx_mask, int* ncount, void* workspace, size_t workspace_bytes, int algo,
                           int* csr_cnt, int* csr_rank, int csr_all, cudaStream_t stream);

extern "C" int cl3d_ball_query_algo(const float* query_xyz, const float* support_xyz, const int* query_mask,
                                    const int* support_mask, int B, int N, int M, float radius, int K, int* idx,
                                    int* idx_mask, int* ncount, void* workspace, size_t workspace_bytes, int algo,
                                    cl3d_stream_t stream_) {
  return ball_query_impl(query_xyz, support_xyz, query_mask, support_mask, B, N, M, radius, K, idx, idx_mask, ncount,
                         workspace, workspace_bytes, algo, nullptr, nullptr, 0, (cudaStream_t)stream_);
}

extern "C" size_t cl3d_ball_query_csr_workspace_bytes(int B, int N, int M, int K, int deterministic) {
  return cl3d_ball_query_workspace_bytes(B, N, M, K) + align_up(sizeof(int) * (size_t)(B > 0 ? B : 1) * (size_t)N, 256) +
         align_up(sizeof(int) * (size_t)(B > 0 ? B : 1) * (size_t)(M > 0 ? M : 1) * (size_t)K, 256) +
         (deterministic ? canon_workspace_bytes(B, N, M, K) : 0);
}

extern "C" int cl3d_ball_query_csr(const float* query_xyz, const float* support_xyz, const int* query_mask,
                                   const int* support_mask, int B, int N, int M, float radius, int K, int* idx,
                                   int* idx_mask, int* ncount, int all_slots, int* csr_off, int* csr_ent,
                                   void* workspace, size_t workspace_bytes, int algo, int phases, int deterministic,
                                   cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(phases >= 1 && phases <= 3, "cl3d_ball_query_csr: phases is a mask of 1 (search) | 2 (lists)");
  CL3D_REQUIRE(csr_off && csr_ent && ncount, "cl3d_ball_query_csr: null pointer");
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 0 && K >= 1, "cl3d_ball_query_csr: bad sizes");
  if (workspace_bytes < cl3d_ball_query_csr_workspace_bytes(B, N, M, K, deterministic) || !workspace) {
    set_error("cl3d_ball_query_csr: workspace too small");
    return CL3D_ERR_WORKSPACE;
  }
  if (B == 0) return CL3D_OK;
  const size_t bq = cl3d_ball_query_workspace_bytes(B, N, M, K);
  int* cnt = (int*)((unsigned char*)workspace + bq);
  int* rank = (int*)((unsigned char*)cnt + align_up(sizeof(int) * (size_t)B * N, 256));
  if (phases & 1) {
    cudaMemsetAsync(cnt, 0, sizeof(int) * (size_t)B * N, stream);
    if (M > 0) {
      int rc = ball_query_impl(query_xyz, support_xyz, query_mask, support_mask, B, N, M, radius, K, idx, idx_mask,
                               ncount, workspace, bq, algo, cnt, rank, all_slots ? 1 : 0, stream);
      if (rc) return rc;
    }
  }
  if (!(phases & 2)) return check_launch("ball query (ranked)");
  csr_scan_kernel<<<B, 1024, 0, stream>>>(N, cnt, csr_off, nullptr); CL3D_LAUNCHED(1);
  const long long ents = (long long)M * K;
  if (ents > 0) {
    const CanonScratch c =
        canon_scratch((unsigned char*)rank + align_up(sizeof(int) * (size_t)B * M * K, 256), B, N, M, K);
    csr_place_kernel<<<dim3((unsigned)((ents + 255) / 256), B), 256, 0, stream>>>(
        idx, ncount, rank, csr_off, N, M, K, all_slots ? 1 : 0, deterministic ? c.src : csr_ent); CL3D_LAUNCHED(1);
    if (deterministic) canon_lists(csr_off, c, B, N, M, K, csr_ent, stream);
  }
  return check_launch("ball query + transposed lists");
}

static int ball_query_impl(const float* query_xyz, const float* support_xyz, const int* query_mask,
                           const int* support_mask, int B, int N, int M, float radius, int K, int* idx,
                           int* idx_mask, int* ncount, void* workspace, size_t workspace_bytes, int algo,
                           int* csr_cnt, int* csr_rank, int csr_all, cudaStream_t stream) {
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 0 && K >= 1, "cl3d_ball_query: bad sizes B=%d N=%d M=%d K=%d", B, N, M, K);
  CL3D_REQUIRE(K <= 256, "cl3d_ball_query: nsample %d > 256 unsupported", K);
  CL3D_REQUIRE(query_xyz && support_xyz && query_mask && support_mask && idx, "cl3d_ball_query: null pointer");
  if (B == 0 || M == 0) return CL3D_OK;
  const int cap3k = 3 * K;
  CL3D_REQUIRE(algo != CL3D_BQ_BRUTE || N <= 8192, "cl3d_ball_query: brute-force path limited to N <= 8192");
  const bool brute = algo == CL3D_BQ_BRUTE || (algo == CL3D_BQ_AUTO && N <= kBruteMaxN);
  if (brute) {
    size_t smem = (size_t)((N + 31) & ~31) * 16 + (size_t)kBQWarps * cap3k * 8 + (size_t)kBQWarps * K * 4;
    // queries per CTA: 64 (8 per warp) amortises the cloud load; fewer when that would leave SMs idle
    int qpc = 64;
    while (qpc > 8 && (long long)B * ceil_div(M, qpc) < 6LL * sm_count()) qpc >>= 1;
    static std::atomic<unsigned long long> attr_brute{0};
    if (first_call_on_device(attr_brute))
      cudaFuncSetAttribute(ball_query_brute_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    dim3 grid(ceil_div(M, qpc), B);
    ball_query_brute_kernel<<<grid, kBQWarps * 32, smem, stream>>>(query_xyz, support_xyz, query_mask, support_mask,
                                                                   N, M, radius, K, qpc, idx, idx_mask, ncount, csr_cnt,
                                                                   csr_rank, csr_all); CL3D_LAUNCHED(1);
    return check_launch("ball_query_brute_kernel");
  }
  if (workspace_bytes < cl3d_ball_query_workspace_bytes(B, N, M, K) || !workspace) {
    set_error("cl3d_ball_query: workspace too small (%zu < %zu)", workspace_bytes,
              cl3d_ball_query_workspace_bytes(B, N, M, K));
    return CL3D_ERR_WORKSPACE;
  }
  const GridWorkspace g = grid_workspace(workspace, B, N);
  build_grid(support_xyz, support_mask, B, N, radius, g, stream);
  size_t smem = (size_t)kBQWarps * (kCandCap + cap3k) * 8 + (size_t)kBQWarps * K * 4;
  static std::atomic<unsigned long long> attr_grid{0};
  if (first_call_on_device(attr_grid))
    cudaFuncSetAttribute(ball_query_grid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
  const long long total = (long long)B * M;
  // the same points and mask as query and support (every non-strided layer): walk the queries in cell order
  const int cell_order = query_xyz == support_xyz && query_mask == support_mask && M == N;
  ball_query_grid_kernel<<<(unsigned)((total + kBQWarps - 1) / kBQWarps), kBQWarps * 32, smem, stream>>>(
      query_xyz, support_xyz, query_mask, g.params, g.cell_start, g.sorted, B, N, M, radius, K, g.cap, cell_order, idx,
      idx_mask, ncount, csr_cnt, csr_rank, csr_all); CL3D_LAUNCHED(1);
  return check_launch("ball_query_grid_kernel");
}

extern "C" size_t cl3d_nearest_query_workspace_bytes(int B, int N, int M) {
  if (N <= kBruteMaxN) return 0;  // the tile scan needs none
  return cl3d_ball_query_workspace_bytes(B, N, M, 1);
}

extern "C" int cl3d_nearest_query(const float* query_xyz, const float* support_xyz, const int* query_mask,
                                  const int* support_mask, int B, int N, int M, int* idx, int* idx_mask,
                                  void* workspace, size_t workspace_bytes, cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 0, "cl3d_nearest_query: bad sizes");
  CL3D_REQUIRE(query_xyz && support_xyz && query_mask && support_mask && idx && idx_mask,
               "cl3d_nearest_query: null pointer");
  if (B == 0 || M == 0) return CL3D_OK;
  const bool grid = N > kBruteMaxN && workspace && !getenv("CL3D_NN_BRUTE");
  if (!grid) {  // every support against every query, tiles in shared memory
    nearest_query_kernel<<<dim3(ceil_div(M, 256), B), 256, 0, stream>>>(query_xyz, support_xyz, query_mask,
                                                                        support_mask, N, M, idx, idx_mask); CL3D_LAUNCHED(1);
    return check_launch("nearest_query_kernel");
  }
  if (workspace_bytes < cl3d_nearest_query_workspace_bytes(B, N, M)) {
    set_error("cl3d_nearest_query: workspace too small (%zu < %zu)", workspace_bytes,
              cl3d_nearest_query_workspace_bytes(B, N, M));
    return CL3D_ERR_WORKSPACE;
  }
  // no radius here: the build picks the smallest cell edge whose grid fits the cell budget (4 cells per point)
  const GridWorkspace g = grid_workspace(workspace, B, N);
  build_grid(support_xyz, support_mask, B, N, 0.f, g, stream);
  nearest_query_grid_kernel<<<dim3(ceil_div(M, 256), B), 256, 0, stream>>>(query_xyz, query_mask, g.params, g.cell_start,
                                                                           g.sorted, N, M, g.cap, idx, idx_mask); CL3D_LAUNCHED(1);
  return check_launch("nearest_query_grid_kernel");
}

extern "C" size_t cl3d_csr_workspace_bytes(int B, int N, int M, int K, int deterministic) {
  return align_up(sizeof(int) * (size_t)(B > 0 ? B : 1) * (size_t)(N > 0 ? N : 1), 256) * 2 +
         (deterministic ? canon_workspace_bytes(B, N > 0 ? N : 1, M, K) : 0);
}

extern "C" int cl3d_build_csr(const int* idx, const int* ncount, int B, int N, int M, int K, int* csr_off,
                              int* csr_ent, void* workspace, size_t workspace_bytes, int deterministic,
                              cl3d_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  CL3D_REQUIRE(B >= 0 && N >= 1 && M >= 0 && K >= 1, "cl3d_build_csr: bad sizes");
  CL3D_REQUIRE(idx && ncount && csr_off && csr_ent, "cl3d_build_csr: null pointer");
  if (workspace_bytes < cl3d_csr_workspace_bytes(B, N, M, K, deterministic) || !workspace) {
    set_error("cl3d_build_csr: workspace too small");
    return CL3D_ERR_WORKSPACE;
  }
  if (B == 0) return CL3D_OK;
  int* cnt = (int*)workspace;
  int* cursor = (int*)((unsigned char*)workspace + align_up(sizeof(int) * (size_t)B * N, 256));
  cudaMemsetAsync(cnt, 0, sizeof(int) * (size_t)B * N, stream);
  const long long ents = (long long)M * K;
  if (ents > 0) {
    csr_count_kernel<<<dim3((unsigned)((ents + 255) / 256), B), 256, 0, stream>>>(idx, ncount, N, M, K, cnt); CL3D_LAUNCHED(1);
  }
  csr_scan_kernel<<<B, 1024, 0, stream>>>(N, cnt, csr_off, cursor); CL3D_LAUNCHED(1);
  if (ents > 0) {
    const CanonScratch c = canon_scratch((unsigned char*)cursor + align_up(sizeof(int) * (size_t)B * N, 256), B, N, M, K);
    csr_fill_kernel<<<dim3((unsigned)((ents + 255) / 256), B), 256, 0, stream>>>(
        idx, ncount, N, M, K, cursor, deterministic ? c.src : csr_ent); CL3D_LAUNCHED(1);
    if (deterministic) canon_lists(csr_off, c, B, N, M, K, csr_ent, stream);
  }
  return check_launch("csr kernels");
}
