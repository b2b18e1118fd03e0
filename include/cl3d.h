/*
 * cl3d.h -- C ABI of the H100-native local-aggregation engine (libcl3d.so, sm_90a).
 *
 * This is the drop-in boundary for the hot path of zeliu98/CloserLook3D (SURVEY.md section 8b).  It replaces
 * the reference's pybind module `pt_custom_ops._ext`
 *     /root/reference/pytorch/ops/pt_custom_ops/_ext_src/src/bindings.cpp:6-15
 * (group_points, group_points_grad, masked_ordered_ball_query, masked_grid_subsampling, masked_nearest_query)
 * and adds one fused forward and one fused backward per local-aggregation family, which together replace
 * the chain  MaskedQueryAndGroup -> elementwise torch ops -> reduction -> BN/ReLU  of
 *     /root/reference/pytorch/models/local_aggregation_operators.py:47-112,170-224,274-316,368-426
 *     /root/reference/pytorch/ops/pt_custom_ops/pt_utils.py:114-144
 *
 * Conventions (they differ from the reference on purpose, see SURVEY.md 8b "Ownership"/"Error conventions"):
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless its name ends in _host;
 *   - all outputs and all scratch memory are CALLER-allocated (torch allocates, passes data_ptr());
 *     nothing is retained or freed by the library; `*_workspace_bytes` tells how much scratch to pass;
 *   - every entry point takes the CUDA stream to launch on (a cudaStream_t passed as void*), is
 *     asynchronous, never synchronises and never calls exit();
 *   - return value: 0 = ok, negative = error code below; cl3d_last_error() gives a message
 *     (the reference prints and exit(-1)s: cuda_utils.h:35-44);
 *   - tensors are contiguous; float = fp32, int = int32, shapes in the reference's notation:
 *     B clouds, N support points, M query points, K = nsample, C channels.
 *   - "point-major" (B,N,Cp) buffers are this library's internal feature layout: row stride
 *     Cp = cl3d_padded_channels(C) floats (multiple of 8 -> rows are 32-byte sectors, 16-byte aligned
 *     for bulk async copies); the reference's layout is channel-major (B,C,N).
 */
#ifndef CL3D_H_
#define CL3D_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CL3D_OK 0
#define CL3D_ERR_BAD_ARG (-1)
#define CL3D_ERR_WORKSPACE (-2)
#define CL3D_ERR_LAUNCH (-3)
#define CL3D_ERR_UNSUPPORTED (-4)

/* reduction over the K neighbour slots (local_aggregation_operators.py:87-105) */
#define CL3D_REDUCE_AVG 0
#define CL3D_REDUCE_SUM 1
#define CL3D_REDUCE_MAX 2

/* family selector of the fused aggregation kernels */
#define CL3D_FAM_POSPOOL_XYZ 0    /* PosPool, position_embedding='xyz'      (:65-69)  */
#define CL3D_FAM_POSPOOL_SINCOS 1 /* PosPool, position_embedding='sin_cos'  (:70-83)  */
#define CL3D_FAM_ADAPTIVE_DP 2    /* AdaptiveWeight, weight_type='dp', num_mlps=1 (:188-197) */
#define CL3D_FAM_PSEUDOGRID 3     /* PseudoGrid, linear / constant influence, sum (:368-419) */

/* Element type of a channel-major feature tensor: an entry point that reads or writes one takes it as `int dtype`
 * beside the pointer it describes (`const void*` / `void*`).  Only the tensors that cross the channel-major <->
 * point-major boundary take it; inside, every buffer and every operation stays fp32.  A 16-bit input is widened
 * exactly; an fp32 result is rounded once, to nearest even, where it is stored.  Unknown codes: CL3D_ERR_BAD_ARG. */
#define CL3D_DTYPE_F32 0
#define CL3D_DTYPE_F16 1
#define CL3D_DTYPE_BF16 2

typedef void* cl3d_stream_t; /* cudaStream_t */

int cl3d_version(void);
const char* cl3d_last_error(void);
int cl3d_padded_channels(int C);
/* Every point-major buffer the gather kernels read (feat_pm, g_pm, ab_pm, aq) must be followed by
 * CL3D_PM_SLACK readable floats: lanes past a row's channel chunk load without a predicate and discard. */
#define CL3D_PM_SLACK 256
/* number of SMs of the current device (grid sizing); negative on error */
int cl3d_sm_count(void);
/* kernels launched by this library in this process so far (for bench.py's gpu_launches) */
long long cl3d_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Neighbour search.  Replaces _ext.masked_ordered_ball_query (masked_ordered_ball_query.cpp:13-59,
 * kernel masked_ordered_ball_query_gpu.cu:11-96): bit-exact idx / idx_mask.
 *   idx       (B,M,K) int32  out
 *   idx_mask  (B,M,K) int32  out, may be NULL (the fused kernels only need ncount)
 *   ncount    (B,M)   int32  out, may be NULL: number of slots that count in avg/sum reductions
 *                     = query_mask ? min(cnt,K) : K   (prefix of the K slots;  feature_mask of
 *                     local_aggregation_operators.py:92 is exactly  k < ncount)
 * Implementation: uniform grid hash over the support cloud (cell edge >= radius), warp per query walking
 * the 27 neighbouring cells; brute force (warp per query, index order) for small clouds and as the exact
 * fallback when a neighbourhood overflows the on-chip candidate list.
 * ---------------------------------------------------------------------------------------------- */
size_t cl3d_ball_query_workspace_bytes(int B, int N, int M, int K);
/* algo: CL3D_BQ_AUTO picks brute force for N <= 2048 and the grid otherwise; BRUTE / GRID force one (tests,
 * benchmarks) */
#define CL3D_BQ_AUTO 0
#define CL3D_BQ_BRUTE 1
#define CL3D_BQ_GRID 2
int cl3d_ball_query_algo(const float* query_xyz, const float* support_xyz, const int* query_mask,
                         const int* support_mask, int B, int N, int M, float radius, int K, int* idx,
                         int* idx_mask, int* ncount, void* workspace, size_t workspace_bytes, int algo,
                         cl3d_stream_t stream);

/* Replaces _ext.masked_nearest_query (masked_nearest_query_gpu.cu:8-62). idx, idx_mask: (B,M) int32.
 * N <= 2048: every support against every query from shared-memory tiles.  Larger clouds: the supports are binned
 * into the cell grid of the ball query (cell edge chosen from the cell budget) and each query walks rings of cells
 * until nothing outside can be nearer; same result bit for bit, including the reference's tie rule (first minimum
 * in index order) and its start value min_dist = 100.  workspace: cl3d_nearest_query_workspace_bytes (0 for small
 * clouds); workspace == NULL always takes the tile scan. */
size_t cl3d_nearest_query_workspace_bytes(int B, int N, int M);
int cl3d_nearest_query(const float* query_xyz, const float* support_xyz, const int* query_mask,
                       const int* support_mask, int B, int N, int M, int* idx, int* idx_mask,
                       void* workspace, size_t workspace_bytes, cl3d_stream_t stream);

/* Search AND transposed lists in one call (what a forward that will be differentiated needs): every counted slot
 * takes its rank inside its support point's list during the search's emit phase (int atomics), so the list build is
 * a scan plus an atomic-free scatter instead of count + scan + atomic fill.  all_slots = 0: lists over the counted
 * slots k < ncount (avg / sum families); 1: over all K slots (PointWiseMLP: BatchNorm2d sees every slot).
 * csr_off (B,N+1), csr_ent (B,M*K) as cl3d_build_csr, with the same list order rule (`deterministic`).
 * phases: 1 = the search (idx / idx_mask / ncount final, ranks left in the workspace), 2 = the lists from those ranks,
 * 3 = both.  A caller that overlaps the list build with the forward kernels issues phase 1, records its "search done"
 * event, then issues phase 2 with the same workspace (and the same `deterministic`). */
size_t cl3d_ball_query_csr_workspace_bytes(int B, int N, int M, int K, int deterministic);
int cl3d_ball_query_csr(const float* query_xyz, const float* support_xyz, const int* query_mask,
                        const int* support_mask, int B, int N, int M, float radius, int K, int* idx, int* idx_mask,
                        int* ncount, int all_slots, int* csr_off, int* csr_ent, void* workspace,
                        size_t workspace_bytes, int algo, int phases, int deterministic, cl3d_stream_t stream);

/* Transposed neighbour lists ("who gathers me"), used by the gather-form backward kernels:
 *   csr_off (B,N+1) int32  out: entries of support point j of cloud b are csr_ent[b][off[j]..off[j+1])
 *   csr_ent (B,M*K) int32  out: q*K + k for every counted slot (k < ncount[q]) with idx[q][k] == j
 * List order: deterministic = 0: atomic arrival order, which varies from run to run.  deterministic = 1: ascending
 * q*K + k (the order of a serial fill), the same bits on every run; the workspace query takes the same flag (the
 * canonical pass needs B*M*K + B*N ints more). */
size_t cl3d_csr_workspace_bytes(int B, int N, int M, int K, int deterministic);
int cl3d_build_csr(const int* idx, const int* ncount, int B, int N, int M, int K, int* csr_off,
                   int* csr_ent, void* workspace, size_t workspace_bytes, int deterministic, cl3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Compatibility gather / scatter (the reference's materialising path; kept for the non-fused module API).
 * Replace _ext.group_points / _ext.group_points_grad (group_points_gpu.cu:13-33,48-69).
 * ---------------------------------------------------------------------------------------------- */
/* points / out and grad_out / grad_points in `dtype`.
 * grad_points (B,C,N) is fully overwritten.  csr_off / csr_ent NULL: zero-filled first, then contributions are added
 * with fp32 atomics, so the summation order -- like the reference's group_points_grad_gpu.cu:48-69 -- is not
 * deterministic (tolerance parity); a 16-bit gradient is accumulated into `acc` (B*C*N floats of caller scratch; may
 * be NULL for CL3D_DTYPE_F32, which accumulates in grad_points) and converted once.  csr_off / csr_ent given (the
 * cl3d_build_csr lists of idx over all K slots): each element is the fp32 sum over its list in list order, rounded
 * once to `dtype`; `acc` is not used.  With canonical lists the result is the same bits on every run. */
int cl3d_group_points(const void* points /*(B,C,N)*/, int dtype, const int* idx /*(B,M,K)*/, int B, int C, int N,
                      int M, int K, void* out /*(B,C,M,K)*/, cl3d_stream_t stream);
int cl3d_group_points_grad(const void* grad_out /*(B,C,M,K)*/, int dtype, const int* idx, int B, int C, int N,
                           int M, int K, const int* csr_off, const int* csr_ent, void* grad_points, float* acc,
                           cl3d_stream_t stream);

/* Replaces _ext.masked_grid_subsampling (masked_grid_subsampling_gpu.cu:11-153).
 * sub_xyz (B,m,3) f32, sub_mask (B,m) i32. */
size_t cl3d_grid_subsample_workspace_bytes(int B, int n, int m);
int cl3d_grid_subsample(const float* points, const int* mask, int B, int n, int m, float sampleDl,
                        float* sub_xyz, int* sub_mask, void* workspace, size_t workspace_bytes,
                        cl3d_stream_t stream);

/* Fused neighbourhood max-pool (body of MaskedMaxPool, pt_utils.py:195-201) and its gradient.
 *   feat_pm (B,N,Cp) point-major (+CL3D_PM_SLACK); out (B,C,M); arg (B,M,Cp) uint8 first arg-max slot (K <= 255)
 *   bwd: grad_pm (B,N,Cp) point-major.  csr_off / csr_ent NULL: zero-filled by the call then accumulated (one red.add
 *   row per query; summation order varies from run to run).  Given (the cl3d_build_csr lists of idx over all K
 *   slots): every row gathered from its list in list order, padded channels 0; canonical lists -> the same bits.
 *   out / grad_out in `dtype` (the maximum of exactly widened values is exact); feat_pm, grad_pm fp32. */
int cl3d_gather_max_fwd(const float* feat_pm, const int* idx, int B, int N, int M, int K, int C, void* out,
                        int dtype, unsigned char* arg, cl3d_stream_t stream);
int cl3d_gather_max_bwd(const void* grad_out, int dtype, const int* idx, const unsigned char* arg, int B, int N,
                        int M, int K, int C, const int* csr_off, const int* csr_ent, float* grad_pm,
                        cl3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Layout: channel-major (B,C,N) <-> point-major (B,N,Cp), Cp = cl3d_padded_channels(C), pad = 0.
 * The channel-major side in `dtype`; the point-major side fp32.
 * ---------------------------------------------------------------------------------------------- */
int cl3d_to_point_major(const void* in_cn, int dtype, int B, int C, int N, float* out_nc, cl3d_stream_t stream);
int cl3d_to_channel_major(const float* in_nc, int B, int C, int N, void* out_cn, int dtype, cl3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused aggregation, families PosPool(xyz|sin_cos) / AdaptiveWeight(dp) / PseudoGrid.
 *
 * forward:  agg[b,c,q] = reduce_k  w_c(dp_k) * f[b, idx[b,q,k], c]      (never materialises (B,C,M,K))
 *   feat_pm   (B,N,Cp) point-major support features
 *   p0, p1    family parameters, fp32 (NULL when unused):
 *               POSPOOL_XYZ    : -
 *               POSPOOL_SINCOS : p0 = dim_mat (C/6)   [torch.pow(1000, arange(F)/F), passed in for bit parity]
 *               ADAPTIVE_DP    : p0 = W (C/S,3), p1 = b (C/S); `shared` = S
 *               PSEUDOGRID     : p0 = K_points (nkp,3), p1 = kernel_weights (nkp,C); `extent`;
 *                                `influence` 0 = linear, 1 = constant
 *   normalize : 1 -> dp /= radius (pt_utils.py:128-129; PosPool/AdaptiveWeight), 0 -> raw (PseudoGrid)
 *   agg       (B,C,M) channel-major out (pre-BN)
 *   bn_partial (ntiles, CL3D_BN_PARTIAL_ROWS, C) out: per-tile moments of agg for the out_transform BN (see
 *               cl3d_bn_finalize); ntiles = cl3d_agg_num_tiles(B,M), the tiles of one cloud contiguous.  May be NULL.
 * backward (gather form over the CSR lists; no float atomics on activations):
 *   g_pm      (B,M,Cp) point-major d(loss)/d(agg)
 *   grad_feat (B,C,N) channel-major out in `dtype`, fully written (by each backward kernel's own channel-major store)
 *   grad_params_partial (nblocks, P) out: per-CTA partial parameter gradients, nblocks =
 *               cl3d_agg_bwd_num_blocks(B,N), P = cl3d_agg_num_params(...) laid out (slot, C) with
 *               slot = {x,y,z,bias} (ADAPTIVE_DP, per channel: the caller folds `shared` groups) or the
 *               kernel point (PSEUDOGRID); reduce with cl3d_reduce_partials.
 * reduction = CL3D_REDUCE_MAX (PosPool, AdaptiveWeight; local_aggregation_operators.py:87-91,199-203 --
 *   F.max_pool2d over nsample and its autograd backward): arg_pm (B,M,Cp) bytes receives the winning slot of
 *   every (query, channel) in the forward and is read by the backward; nsample <= 256.  Pass NULL for avg / sum.
 *   PseudoGrid is a sum by construction (CL3D_ERR_BAD_ARG for max).
 * ---------------------------------------------------------------------------------------------- */
int cl3d_agg_num_tiles(int B, int M);
int cl3d_agg_bwd_num_blocks(int B, int N);
int cl3d_agg_num_params(int family, int C, int shared, int nkp);
int cl3d_agg_fwd(int family, int reduction, const float* feat_pm, const float* query_xyz,
                 const float* support_xyz, const int* idx, const int* ncount, const float* p0,
                 const float* p1, int B, int N, int M, int K, int C, float radius, int normalize,
                 int shared, int nkp, float extent, int influence, float* agg, float* bn_partial,
                 unsigned char* arg_pm, cl3d_stream_t stream);
int cl3d_agg_bwd(int family, int reduction, const float* g_pm, const float* feat_pm,
                 const float* query_xyz, const float* support_xyz, const int* ncount,
                 const int* csr_off, const int* csr_ent, const float* p0, const float* p1, int B, int N,
                 int M, int K, int C, float radius, int normalize, int shared, int nkp, float extent,
                 int influence, void* grad_feat, int dtype, float* grad_params_partial,
                 const unsigned char* arg_pm, cl3d_stream_t stream);
/* out[p] = sum_t partial[t][p]  (fixed order -> deterministic given the partials) */
int cl3d_reduce_partials(const float* partial, int ntiles, int P, float* out, cl3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * out_transform = BatchNorm1d + ReLU (local_aggregation_operators.py:43-45,110), channel-major (B,C,M).
 *   bn_finalize: from the per-tile partials -> batch mean / invstd (save_stats (2,C)), updates running
 *                stats with `momentum` (unbiased variance, as nn.BatchNorm1d) when training.  A forward's
 *                partials hold, per tile and channel, CL3D_BN_PARTIAL_ROWS rows: n (number of values), c (a
 *                centre near the tile's values), sum (x - c), sum (x - c)^2.  The tiles are merged in
 *                double, so a channel whose mean dwarfs its spread keeps its variance.
 *   bn_relu_fwd: y = relu((x-mean)*invstd*gamma + beta); in eval mode pass stats made from running stats.
 *   bn_relu_bwd: per-tile partial rows (sum gy*xhat, sum gy) reduced as cl3d_reduce_partials into dgamma_dbeta, then
 *                the apply pass writes d(loss)/d(agg) POINT-MAJOR (B,M,Cp) ready for cl3d_agg_bwd.
 *   y written / grad_y read in `dtype`; x, the statistics, partials, dgamma_dbeta and g_pm fp32.
 * ---------------------------------------------------------------------------------------------- */
#define CL3D_BN_PARTIAL_ROWS 4
int cl3d_bn_finalize(const float* bn_partial /*(ntiles,CL3D_BN_PARTIAL_ROWS,C)*/, int ntiles, int C, long long count, float eps,
                     float momentum, int training, float* running_mean, float* running_var,
                     float* save_stats /*(2,C): mean, invstd*/, cl3d_stream_t stream);
int cl3d_bn_relu_fwd(const float* x, const float* save_stats, const float* gamma, const float* beta,
                     int B, int C, int M, void* y, int dtype, cl3d_stream_t stream);
int cl3d_bn_relu_bwd(const void* grad_y, int dtype, const float* x, const float* save_stats, const float* gamma,
                     const float* beta, int B, int C, int M, int training, float* partial /*(ntiles,2,C)*/,
                     float* dgamma_dbeta /*(2,C)*/, float* g_pm /*(B,M,Cp)*/, cl3d_stream_t stream);
/* cl3d_bn_relu_bwd is its two halves in sequence:
 *   bwd_stats: the statistics pass and its reduction -> dgamma_dbeta (2,C) = this call's (sum gy*xhat, sum gy).
 *   bwd_apply: the apply pass with dgb_sums (2,C) = (sum gy*xhat, sum gy) over the whole batch and their count:
 *              count = NULL -> B*M; else a device float64 (cl3d_bn_finalize_ranks' count), and work (2,C) floats
 *              receives the means.  Between the halves a caller may exchange and add the sums of several ranks.
 * Cross-rank statistics (SyncBatchNorm).  Each rank of W turns its forward partials into a (4,C) float64 record
 * (count, centre, sum (x - centre), sum (x - centre)^2: counts beyond 2^24 stay exact), the W records are gathered in
 * rank order, and every rank merges them in that order about rank 0's centre: the same merge as cl3d_bn_finalize,
 * so all ranks get the same bits.  bn_finalize_ranks (training only) writes save_stats, updates the running statistics
 * with the global count (running_* may be NULL) and stores that count in *count (one float64). */
int cl3d_bn_relu_bwd_stats(const void* grad_y, int dtype, const float* x, const float* save_stats, const float* gamma,
                           const float* beta, int B, int C, int M, float* partial /*(ntiles,2,C)*/,
                           float* dgamma_dbeta /*(2,C)*/, cl3d_stream_t stream);
int cl3d_bn_relu_bwd_apply(const void* grad_y, int dtype, const float* x, const float* save_stats, const float* gamma,
                           const float* beta, int B, int C, int M, int training, const float* dgb_sums /*(2,C)*/,
                           const double* count, float* work /*(2,C)*/, float* g_pm /*(B,M,Cp)*/, cl3d_stream_t stream);
int cl3d_bn_rank_moments(const float* bn_partial /*(ntiles,CL3D_BN_PARTIAL_ROWS,C)*/, int ntiles, int C, long long count,
                         double* record /*(4,C)*/, cl3d_stream_t stream);
int cl3d_bn_finalize_ranks(const double* records /*(W,4,C)*/, int W, int C, float eps, float momentum,
                           float* running_mean, float* running_var, float* save_stats /*(2,C)*/, double* count,
                           cl3d_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused PointWiseMLP (feature_type='dp_fi_df', num_mlps=1, reduction='max';
 * local_aggregation_operators.py:254-257,288-303).  The per-neighbour 1x1 conv over [dp; f_i; f_j-f_i] is
 * refactored into two per-point products  A = f (Wc-Wr)^T,  Bv = f Wr^T  plus a gather-add, so only
 * (B,N,Cout)-sized tensors exist; BatchNorm2d statistics over all B*M*K positions are accumulated on the
 * fly and the max over K is taken through the monotone BN+ReLU as relu(a*(a>=0?max:min)+b).
 * See DESIGN.md for the kernel list; entry points are declared in the PWMLP section below.
 * ---------------------------------------------------------------------------------------------- */
/* fp32 GEMM with element strides and optional split-K (gemm.cu, gemm_tc.cuh):
 *   C[m][n] = sum_k A[m*sa_m + k*sa_k] * B[k*sb_k + n*sb_n],  C row stride ldc.
 * splitk > 1 divides k among CTAs (fixed-order reduction); workspace = cl3d_sgemm_workspace_bytes.
 * algo: CL3D_GEMM_TC3X = wgmma tensor cores with the 3xTF32 operand split (fp32-level accuracy, the default
 * behind CL3D_GEMM_AUTO), CL3D_GEMM_FFMA = fp32 FMA pipe. */
#define CL3D_GEMM_AUTO 0
#define CL3D_GEMM_FFMA 1
#define CL3D_GEMM_TC3X 2
size_t cl3d_sgemm_workspace_bytes(int M, int N, int splitk);
int cl3d_sgemm_algo(const float* a, long long sa_m, long long sa_k, const float* b, long long sb_k,
                    long long sb_n, int M, int N, int K, float* c, long long ldc, int splitk, void* workspace,
                    size_t workspace_bytes, int algo, cl3d_stream_t stream);

/* Fused PointWiseMLP (pwmlp.cu).  Cop = cl3d_padded_channels(Cout), Cpa = cl3d_padded_channels(C+3).
 *   cl3d_to_point_major_aug : (B,C,N) features in `dtype` + (B,N,3) xyz -> (B,N,Cpa) fp32 rows
 *                             [f | (xyz - o_b)/r | 0], o_b = xyz[b,0]
 *                             (support_xyz of fwd_stats / bwd supplies the same origin for the query term)
 *   ab_pm (B,N,2*Cop)       : row = [A | T],  A = (Wc-Wr) f,  T = sgn*(Wr f + Wp s/r)   (one cl3d_sgemm_algo)
 *   wp (Cout,3), sgn (Cout) : conv weight columns 0..2; sign(gamma) as +-1.0
 * fwd_stats : ysel (B,Cout,M) selected extremum of y; aq, sq (B,M,Cop) a' and sum_k bv; karg (B,M,Cop) uint8
 *             first arg-max slot (K <= 255); bn_partial (cl3d_agg_num_tiles(B,M), CL3D_BN_PARTIAL_ROWS, Cout) -> cl3d_bn_finalize
 *             with count = B*M*K.
 * output    : out (B,Cout,M) = relu(sc*ysel + sh) in `dtype` is cl3d_bn_relu_fwd(ysel, save_stats, gamma, beta, B, Cout,
 *             M, out, dtype, stream).
 * bwd       : grad_out (B,Cout,M) in `dtype`.  The ReLU decision is recomputed from ysel, save_stats, gamma and beta
 *             with the forward's expression (bit-identical to the forward's fp32 decision; a 16-bit output may have
 *             rounded a small positive value to zero, so the stored output cannot decide).
 *             csr_off/csr_ent = cl3d_build_csr over ALL K slots (ncount = K); scratch =
 *             cl3d_pwmlp_bwd_scratch_floats(...) floats; dgamma_dbeta (2,Cout); grad_ab_pm (B,N,2*Cop) fully
 *             written (zero-filled, then the support-major pass and the query pass add their parts with fp32
 *             red.add); side_stream (may be NULL): the zero-fill and the query pass run on it beside the other
 *             two passes, forked from and joined back into `stream` with events (CUDA-graph capturable);
 *             grad_wp (3,Cout) = the -sum da' (x) q/r part of d/dWp (the rest comes out of the weight-gradient
 *             product).  training = 0: BatchNorm2d in eval mode (save_stats = running statistics): its backward
 *             has no batch-statistics terms, dy = sc*dz at the arg-max slot only (csr lists may then be NULL).
 *             deterministic = 1: no atomics.  The query pass stores d/da' point-major in the scratch, and one
 *             support-major pass over the (canonical, cl3d_build_csr deterministic = 1) all-slots lists stores every
 *             grad_ab_pm row once, summed in list order; lists are then required in eval mode too, the side stream
 *             is not used, and the scratch query takes the same flag (B*M*Cop floats more). */
size_t cl3d_pwmlp_bwd_scratch_floats(int B, int N, int M, int Cout, int deterministic);
/* conv weight (Cout, 3+2C) = [Wp|Wc|Wr] + BN gamma -> wcat (2*Cop, Cpa) (rows zero-padded to Cpa), wp (Cout,3),
 * sgn (Cout); and back: d/dwcat (2*Cop, Cpa) + grad_wp (3,Cout) -> d/d(conv weight) (Cout, 3+2C). */
int cl3d_pwmlp_prep_weights(const float* conv_weight, const float* gamma, int C, int Cout, float* wcat,
                            float* wp, float* sgn, cl3d_stream_t stream);
int cl3d_pwmlp_weight_grad(const float* gwcat, const float* grad_wp, const float* sgn, int C, int Cout,
                           float* grad_conv_weight, cl3d_stream_t stream);
int cl3d_to_point_major_aug(const void* in_cn, int dtype, const float* xyz, int B, int C, int N, float radius,
                            float* out_nc, cl3d_stream_t stream);
int cl3d_pwmlp_fwd_stats(const float* ab_pm, const float* wp, const float* sgn, const float* query_xyz,
                         const float* support_xyz, const int* idx, int B, int N, int M, int K, int Cout,
                         float radius, float* ysel,
                         float* aq, float* sq, unsigned char* karg, float* bn_partial, cl3d_stream_t stream);
int cl3d_pwmlp_bwd(const void* grad_out, int dtype, const float* beta, const float* ab_pm, const float* wp,
                   const float* sgn, const float* query_xyz, const float* support_xyz, const int* idx,
                   const int* csr_off, const int* csr_ent, const float* ysel, const float* aq, const float* sq,
                   const unsigned char* karg, const float* save_stats, const float* gamma, int B, int N,
                   int M, int K, int Cout, float radius, int training, int deterministic, float* scratch,
                   float* dgamma_dbeta, float* grad_ab_pm, float* grad_wp, cl3d_stream_t stream,
                   cl3d_stream_t side_stream);
/* cl3d_pwmlp_bwd is its two halves in sequence (the unsplit call also overlaps the zero-fill with the first):
 *   bwd_stats: the statistics pass (sc*dz into the scratch) and its reduction -> dgamma_dbeta (2,Cout) = this call's
 *              (sum dz*yhat, sum dz).  Only grad_out, beta, ysel, save_stats and gamma are read.
 *   bwd_apply: the dense, query and (deterministic) gather passes with dgb_sums (2,Cout) over the whole batch and
 *              their count: NULL -> B*M*K, else a device float64 (cl3d_bn_finalize_ranks' count).  The same scratch,
 *              after bwd_stats on it. */
int cl3d_pwmlp_bwd_stats(const void* grad_out, int dtype, const float* beta, const float* ysel, const float* save_stats,
                         const float* gamma, int B, int M, int Cout, float* scratch, float* dgamma_dbeta,
                         cl3d_stream_t stream);
int cl3d_pwmlp_bwd_apply(const void* grad_out, int dtype, const float* beta, const float* ab_pm, const float* wp,
                         const float* sgn, const float* query_xyz, const float* support_xyz, const int* idx,
                         const int* csr_off, const int* csr_ent, const float* ysel, const float* aq, const float* sq,
                         const unsigned char* karg, const float* save_stats, const float* gamma, int B, int N,
                         int M, int K, int Cout, float radius, int training, int deterministic, float* scratch,
                         const float* dgb_sums, const double* count, float* grad_ab_pm, float* grad_wp,
                         cl3d_stream_t stream, cl3d_stream_t side_stream);

/* ------------------------------------------------------------------------------------------------
 * Fused multi-shape part-segmentation head (multihead.cu).  Replaces the S per-shape heads of
 * MultiPartSegHeadResNet (models/heads/segmentation_head.py:80-149), each
 *     Conv1d(C,C,no bias) -> BatchNorm1d(C) -> ReLU -> Conv1d(C, num_parts[s]) + bias,
 * all run over every point of x (B,C,N) channel-major.  Nothing of size S*C*B*N is materialised: BatchNorm
 * statistics of every head follow from the channel means and one centred C x C second-moment matrix of x.
 * Semantics of nn.BatchNorm1d in both modes (training: biased variance normalises, running statistics take the
 * unbiased one, num_batches_tracked += 1, momentum < 0 means momentum=None; eval: running statistics).
 *   desc_host    : host struct below (copied into kernel arguments: no device upload, CUDA-graph capturable)
 *   w1 (S,C,C), gamma (S,C), beta (S,C), w2 (sum num_parts, C), b2 (sum num_parts): the heads' parameters
 *                 concatenated over s
 *   logits       : concatenation over s of contiguous (B, num_parts[s], N) blocks
 *   save         : cl3d_mhead_save_floats(S,C) floats written by fwd, read by bwd
 *   bwd          : desc_host->grad_logits[s] = d(loss)/d(logits of head s), (B,num_parts[s],N) contiguous, or NULL
 *                  (counts as zero); grad_x (B,C,N) and every parameter gradient are fully written (no float atomics,
 *                  fixed-order reductions: repeat runs are bit-identical).
 *   dtype        : CL3D_DTYPE_* of x, logits, every grad_logits[s] and grad_x.  Parameters, running statistics, save
 *                  and the parameter gradients are fp32 whatever it is; a 16-bit run computes exactly the fp32 head on
 *                  the widened x and d/dlogits and rounds logits and grad_x once.  The workspace sizes do not depend
 *                  on it.
 * Limits: padded C <= 128, num_parts[s] <= 64, S <= 32; otherwise CL3D_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
#define CL3D_MHEAD_MAX_HEADS 32
#define CL3D_MHEAD_MAX_PARTS 64
#define CL3D_MHEAD_MAX_CHANNELS 128
typedef struct cl3d_mhead_desc {
  int S;                                              /* number of heads (shape categories) */
  int C;                                              /* channels of x */
  int num_parts[CL3D_MHEAD_MAX_HEADS];                /* output channels of head s */
  float* running_mean[CL3D_MHEAD_MAX_HEADS];          /* (C) per head: read in eval, updated in training */
  float* running_var[CL3D_MHEAD_MAX_HEADS];
  long long* num_batches_tracked[CL3D_MHEAD_MAX_HEADS]; /* per head, += 1 in training; may be NULL if momentum >= 0 */
  const void* grad_logits[CL3D_MHEAD_MAX_HEADS];      /* backward only, in `dtype`, see above */
} cl3d_mhead_desc;
size_t cl3d_mhead_save_floats(int S, int C);
size_t cl3d_mhead_fwd_workspace_bytes(const cl3d_mhead_desc* desc_host, int B, int N);
size_t cl3d_mhead_bwd_workspace_bytes(const cl3d_mhead_desc* desc_host, int B, int N);
int cl3d_mhead_fwd(const cl3d_mhead_desc* desc_host, const void* x, int dtype, int B, int N, const float* w1,
                   const float* gamma, const float* beta, const float* w2, const float* b2, float eps,
                   float momentum, int training, void* logits, float* save, void* workspace,
                   size_t workspace_bytes, cl3d_stream_t stream);
int cl3d_mhead_bwd(const cl3d_mhead_desc* desc_host, const void* x, int dtype, int B, int N, const float* w1,
                   const float* w2, const float* save, int training, void* grad_x, float* grad_w1,
                   float* grad_gamma, float* grad_beta, float* grad_w2, float* grad_b2, void* workspace,
                   size_t workspace_bytes, cl3d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CL3D_H_ */
