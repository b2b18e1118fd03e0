// common.cuh -- shared device/host helpers for libcl3d (sm_90a only).
#pragma once
#include <atomic>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/cl3d.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libcl3d is written for sm_90a (Hopper) only"
#endif

namespace cl3d {

constexpr int kWarp = 32;
constexpr int kNumSMsFallback = 132;

// ---------------------------------------------------------------------------------------------
// error reporting (thread-local message, integer return codes; never exit())
// ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define CL3D_REQUIRE(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      ::cl3d::set_error(__VA_ARGS__);      \
      return CL3D_ERR_BAD_ARG;             \
    }                                      \
  } while (0)

// true exactly once per CUDA device (host side; for per-device one-time settings such as
// cudaFuncAttributeMaxDynamicSharedMemorySize, which is a per-device attribute)
inline bool first_call_on_device(std::atomic<unsigned long long>& seen) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return true;
  const unsigned long long bit = 1ull << (dev & 63);
  return (seen.fetch_or(bit) & bit) == 0;
}
// Opt a kernel into the full dynamic shared-memory carve-out (227 KB) ONCE per device instead of calling
// cudaFuncSetAttribute on every launch.  `seen` must be a static per kernel instantiation.
constexpr int kMaxDynSmem = 227 * 1024;
template <typename K>
inline void allow_big_smem(K kernel, std::atomic<unsigned long long>& seen) {
  if (first_call_on_device(seen)) {
    // the 227 KB limit covers static + dynamic shared memory of the block
    cudaFuncAttributes fa;
    int stat = 0;
    if (cudaFuncGetAttributes(&fa, kernel) == cudaSuccess) stat = (int)fa.sharedSizeBytes;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem - stat) != cudaSuccess)
      cudaGetLastError();  // reported by the launch that follows if the kernel really needs it
  }
}
// ---------------------------------------------------------------------------------------------
// element type of a channel-major tensor at the layout boundary (CL3D_DTYPE_*).  Everything inside stays fp32:
// a 16-bit value is widened exactly on load, an fp32 result is rounded once (to nearest even) on store.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_f32(const float* p) { return *p; }
__device__ __forceinline__ float load_f32(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ float load_f32(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void store_f32(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_f32(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void store_f32(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

inline bool valid_dtype(int dtype) {
  return dtype == CL3D_DTYPE_F32 || dtype == CL3D_DTYPE_F16 || dtype == CL3D_DTYPE_BF16;
}
template <typename T>
struct TypeTag {
  using type = T;
};
// Calls fn(TypeTag<T>{}) with the element type of `dtype` (checked by the entry point with valid_dtype).
template <typename F>
inline int with_dtype(int dtype, F&& fn) {
  switch (dtype) {
    case CL3D_DTYPE_F16: return fn(TypeTag<__half>{});
    case CL3D_DTYPE_BF16: return fn(TypeTag<__nv_bfloat16>{});
    default: return fn(TypeTag<float>{});
  }
}
#define CL3D_REQUIRE_DTYPE(dt, what) CL3D_REQUIRE(::cl3d::valid_dtype(dt), "%s: unknown dtype code %d", what, dt)

__host__ __device__ inline int padded_channels(int C) { return (C + 7) & ~7; }
__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int sm_count();
int persistent_grid_cap();  // 4 x SMs (test hook: CL3D_TEST_MAX_GRID)

// number of kernels this library has launched in this process (bench.py reports it as gpu_launches)
void count_launches(int n);
#define CL3D_LAUNCHED(n) ::cl3d::count_launches(n)

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// The reference's squared distance, bit-exact: nvcc contracts the source expression of
// masked_ordered_ball_query_gpu.cu:56-57 / masked_nearest_query_gpu.cu:47-48 to
//   t = dy*dy; t = fma(dx,dx,t); t = fma(dz,dz,t)   with d = query - support   (checked in SASS).
__device__ __forceinline__ float ref_d2(float qx, float qy, float qz, float x, float y, float z) {
  float dx = __fsub_rn(qx, x), dy = __fsub_rn(qy, y), dz = __fsub_rn(qz, z);
  float t = __fmul_rn(dy, dy);
  t = __fmaf_rn(dx, dx, t);
  t = __fmaf_rn(dz, dz, t);
  return t;
}

// base + elem_off floats as ONE instruction (IMAD.WIDE.U32): the compiler otherwise rebuilds the 64-bit address
// of a gathered row from two partial bases with four instructions (measured in the PointWiseMLP gather loops)
__device__ __forceinline__ const float* row_at(const float* base, unsigned elem_off) {
  unsigned long long r;
  asm("mad.wide.u32 %0, %1, 4, %2;" : "=l"(r) : "r"(elem_off), "l"(base));
  return reinterpret_cast<const float*>(r);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- BatchNorm forward partials: (ntiles, kBnRows, C), one row group per tile, tiles of one cloud contiguous.
// Per tile and channel: [0] n, the number of values; [1] c, a centre near the tile's values; [2] sum (x - c);
// [3] sum (x - c)^2.  The sums are of small, spread-sized terms, so a channel whose mean dwarfs its spread keeps its
// variance: a raw fp32 sum of squares loses (mean/std)^2 * 2^-24 of it, a raw fp32 tile sum ~ 2^-24 * |mean| of the
// tile mean, and both cancel in the finalize.  cl3d_bn_finalize merges the tiles in double.
constexpr int kBnRows = CL3D_BN_PARTIAL_ROWS;
// out[i] = sums[i] * (1 / *count) for the BatchNorm backward's apply passes when the count is held on the device
// (cross-rank statistics): they then run with inv_count = 1 (bn.cu)
int bn_mean_terms(const float* sums, int n, const double* count, float* out, cudaStream_t stream);

__device__ __forceinline__ void store_bn_moments(float* partial, size_t tile, int C, int c, float n, float ctr,
                                                 float d, float q) {
  float* p = partial + tile * kBnRows * C + c;
  p[0] = n;
  p[C] = ctr;
  p[2 * C] = d;
  p[3 * C] = q;
}

// BatchNorm pre-activation (x - mean) * sc + sh with sc = invstd * gamma, sh = beta, rounded exactly as written.  Every
// ReLU forward and every backward that recomputes the ReLU decision takes it from here, so they agree bit for bit (the
// backward cannot decide from the output: a 16-bit output may round a small positive value to zero).
__device__ __forceinline__ float bn_preact(float x, float mean, float sc, float sh) {
  return __fmaf_rn(__fsub_rn(x, mean), sc, sh);
}

// one tile row held one value per lane (queries q0 + lane, present where q < M; lane 0 always is), centred about its
// fp32 mean (a centre at one of the values would make sum (x - c)^2 cancel when that value is an outlier, e.g. a
// padded query); absent lanes count nothing
__device__ __forceinline__ void warp_bn_moments(float* partial, size_t tile, int C, int c, float v, bool present) {
  const int n = __popc(__ballot_sync(0xffffffffu, present));
  const float ctr = __fdividef(warp_sum(present ? v : 0.f), (float)n);  // any centre near the values will do
  const float e = present ? __fsub_rn(v, ctr) : 0.f;
  const float d = warp_sum(e), q = warp_sum(e * e);
  if ((threadIdx.x & 31) == 0) store_bn_moments(partial, tile, C, c, (float)n, ctr, d, q);
}

// one tile row of n >= 1 values in shared memory, in order, centred about its fp32 mean
__device__ __forceinline__ void row_bn_moments(float* partial, size_t tile, int C, int c, const float* row, int n) {
  float s = 0.f;
  for (int i = 0; i < n; ++i) s += row[i];
  const float ctr = __fdividef(s, (float)n);
  float d = 0.f, q = 0.f;
  for (int i = 0; i < n; ++i) {
    const float e = __fsub_rn(row[i], ctr);
    d += e;
    q = fmaf(e, e, q);
  }
  store_bn_moments(partial, tile, C, c, (float)n, ctr, d, q);
}
__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o);
    v = t < v ? t : v;
  }
  return v;
}

// ---- fp32 pairs.  Hopper has no packed fp32x2 instructions, so each pair operation is two IEEE-rounded scalar
// operations (__fmaf_rn / __fmul_rn / ... are never contracted or reassociated by the compiler); the results are
// the same bits a packed instruction gives.  A pair travels as one 64-bit value (lo = .x, hi = .y).
typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) {
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(u64 v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {  // a - b, component-wise (exactly rounded like __fsub_rn)
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}

__device__ __forceinline__ float sqrt_approx(float x) {  // MUFU: 2^-22 relative, sqrt(0) = 0
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ u64 fma2_bcast(float h, u64 b, u64 c) {  // (h, h) * b + c ; h is a scalar-broadcast operand
  float b0, b1, c0, c1;
  unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(__fmaf_rn(h, b0, c0), __fmaf_rn(h, b1, c1));
}

// The same operations on plain float operands.
//   (cx, cy) += (h, h) * (bx, by)
__device__ __forceinline__ void ffma2_bcast(float h, float bx, float by, float& cx, float& cy) {
  cx = __fmaf_rn(h, bx, cx);
  cy = __fmaf_rn(h, by, cy);
}
//   (cx, cy) += (ax, ay) * (bx, by)
__device__ __forceinline__ void ffma2(float ax, float ay, float bx, float by, float& cx, float& cy) {
  cx = __fmaf_rn(ax, bx, cx);
  cy = __fmaf_rn(ay, by, cy);
}
//   (cx, cy) = (ax, ay) * (bx, by)
__device__ __forceinline__ void fmul2(float ax, float ay, float bx, float by, float& cx, float& cy) {
  cx = __fmul_rn(ax, bx);
  cy = __fmul_rn(ay, by);
}
// ---- mbarrier helpers (producer/consumer rings of the wgmma GEMM, gemm_tc.cuh) ----------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// ---- cp.async (non-bulk): 16 bytes per lane global -> shared without passing through registers; completion per
// thread by commit_group / wait_group, no mbarrier.  `dst` is a shared-window address, both sides 16-byte aligned.
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {  // until at most N of this thread's groups are pending
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
}  // namespace cl3d
