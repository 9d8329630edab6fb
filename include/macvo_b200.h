/*
 * macvo_b200.h — C ABI of the H100 (sm_90a) hot path for MAC-VO.
 *
 * MAC-VO's plugin boundary is a Python class registry (SURVEY.md §8b), not an FFI; this header is
 * the thin C layer BELOW the plugin classes (`mac-vo_b200/plugins.py`). Every entry point takes raw
 * device pointers + sizes + a CUDA stream, enqueues work on that stream (CUDA-graph capturable
 * unless noted) and returns 0 on success, a negative MACVO_E_* code for bad arguments or a positive
 * cudaError_t. No ownership is transferred: all buffers are allocated by the caller (PyTorch on the
 * Python side) and must outlive the stream work. `stream` is a `cudaStream_t` passed as `void*` so
 * the header needs no CUDA include.
 *
 * Each function cites the reference interface (file:line under the MAC-VO tree) it replaces.
 */
#ifndef MACVO_B200_H
#define MACVO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MACVO_OK 0
#define MACVO_E_ARG (-1)        /* null pointer / non-positive size / unsupported shape            */
#define MACVO_E_WORKSPACE (-2)  /* workspace too small (query the *_workspace_bytes function)      */
#define MACVO_E_UNSUPPORTED (-3)/* mode not available for these shapes on this device              */
#define MACVO_E_DRIVER (-4)     /* driver entry point (cuTensorMapEncodeTiled) could not be loaded */

/* library identification: "macvo_b200 <version> sm_90a" */
const char* macvo_b200_version(void);

/* ------------------------------------------------------------------------------------------------
 * (a3) all-pairs correlation volume — replaces MemoryEncoder.corr
 *      Module/Network/FlowFormer/core/encoder.py:256-275 (torch.bmm of the two feature maps).
 *
 *   corr[b, i, j] = sum_d fmap1[b, d, i] * fmap2[b, d, j]        (no 1/sqrt(d) scaling)
 *
 * fmap1/fmap2: (batch, dim, n) row-major fp32 — exactly the NCHW output of `channel_convertor`
 * viewed as (B, D, H1*W1). corr: (batch, n, n) row-major fp32 == the contiguous
 * (B, 1, H1, W1, H1, W1) tensor the cost perceiver and the decoder view.
 *
 * mode: MACVO_CORR_SIMT      fp32 FFMA shared-memory tiled kernel (reference-accuracy baseline)
 *       MACVO_CORR_TC_3XF16  wgmma (tensor core) kernel: each fp32 operand is split into
 *                            fp16 hi + lo; hi*hi + hi*lo + lo*hi accumulated in fp32
 *                            (~2^-22 relative product error: fp32-class accuracy)
 *       MACVO_CORR_TC_1XF16  wgmma, operands rounded to fp16 once (MACVO_Fast: fp16 encoder)
 * The tensor-core modes need dim % 64 == 0 and n % 8 == 0 and a workspace of
 * macvo_corr_workspace_bytes() bytes (device memory, 1024-byte aligned).
 */
#define MACVO_CORR_SIMT 0
#define MACVO_CORR_TC_3XF16 1
#define MACVO_CORR_TC_1XF16 2
#define MACVO_CORR_TC_TF32 3   /* wgmma tf32, ONE pass straight over the fp32 K-major (channels_last) features: no
                                * operand pre-pass, no workspace; operands truncated to TF32 by the tensor core (10-bit
                                * mantissa) = what the reference's own torch.matmul does for this product once its frontend
                                * has set allow_tf32 (Frontend.py:275-277). Requires MACVO_CORR_KMAJOR_INPUT. */
/* OR-ed into `mode` (tensor-core modes only): fmap1 / fmap2 are given K-major, (batch, n, dim) row-major — the memory of
 * a channels_last (B, D, H1, W1) tensor, which is what cuDNN's NHWC `channel_convertor` produces — so the operand
 * pre-pass is an elementwise fp16 split instead of a transpose. */
#define MACVO_CORR_KMAJOR_INPUT 16
size_t macvo_corr_workspace_bytes(int batch, int dim, int n, int mode);
int macvo_corr_build(const float* fmap1, const float* fmap2, float* corr, int batch, int dim, int n, int mode,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (a5) 9x9 bilinear window lookup — replaces MemoryDecoder.encode_flow_token
 *      Module/Network/FlowFormer/core/decoder.py:141-153 (+ bilinear_sampler core/utils.py:26-34,
 *      the `delta` buffer decoder.py:124-129; grid_sample align_corners=True, zeros padding).
 *
 * cost_maps: (batch*h1*w1, h2, w2) fp32 (one map per query pixel), coords: (batch, 2, h1, w1) fp32
 * [x, y] in cost-map pixels, out: (batch, 81, h1, w1) fp32; out channel i*9+j samples at
 * (x + i - 4, y + j - 4)  — the reference's transposed window (first axis steps in x).
 */
int macvo_corr_lookup(const float* cost_maps, const float* coords, float* out, int batch, int h1, int w1, int h2,
                      int w2, void* stream);

/* same lookup with the output as (batch*h1*w1, 81) pixels-major rows (NHWC view of the map above) */
int macvo_corr_lookup_rows(const float* cost_maps, const float* coords, float* out, int batch, int h1, int w1, int h2,
                           int w2, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (a7)+(a8 scoring) fused dense post-processing of one `estimate_pair` + keypoint scoring —
 *      replaces FlowFormerCovFrontend.inference_2_depth / inference_2_match
 *      (Module/Frontend/Frontend.py:184-200), disparity_to_depth / disparity_to_depth_cov
 *      (Module/Frontend/StereoDepth.py:271-282), IMatcher.Output.from_partial_cov
 *      (Module/Frontend/Matching.py:29-40) and the quality / NMS part of
 *      CovAwareSelector_NoDepth.select_point (Module/KeypointSelector.py:368-379).
 *
 * est_flow, est_cov: (2, 2, h, w) fp32 network output; slot 0 = stereo pair (t2), slot 1 = temporal.
 * Outputs (any may be NULL to skip): depth, disparity, depth_cov (h*w fp32 each),
 * depth_mask (h*w uint8, 1 where flow_x <= 0; only written if non-NULL), flow_cov (3, h, w) fp32
 * = cat(est_cov[1], 0). bl_fx = baseline*fx and bl_fx_sq = (baseline*fx)^2 evaluated in double by
 * the caller exactly like the reference's Python floats.
 * Scoring (if score != NULL): quality = cov_uu + cov_vv - 2 cov_uv of `score_cov` (3, h, w) —
 * pass flow_cov to fuse, or any (3,h,w) map for a standalone selector — written to `score->quality`;
 * `score->nms` (h*w uint8) = quality == min over the ksize x ksize window and no NaN in it;
 * NMS survivors' quality values are appended (unordered) to score->cand_vals, count in *score->n_cand
 * (caller zeroes it). All pointers device memory.
 * est_cov == NULL with est_flow set: a frontend without covariance (FlowFormerDepth.estimate,
 * Module/Frontend/StereoDepth.py:122-128: disparity = |flow_x| of slot 0, depth = (bl*fx) * disparity.reciprocal(),
 * StereoDepth.py:270-272). Only depth and / or disparity are written, with the arithmetic above; depth_cov,
 * depth_mask, flow_cov and score must be NULL (MACVO_E_ARG otherwise).
 */
typedef struct {
    const float* score_cov; /* (3,h,w) or NULL = use the freshly written flow_cov */
    float* quality;         /* h*w */
    uint8_t* nms;           /* h*w */
    float* cand_vals;       /* capacity h*w */
    int* n_cand;            /* 1 */
    int ksize;              /* odd, <= 15 */
    /* depth-aware variant (CovAwareSelector.select_point, Module/KeypointSelector.py:260-334); all NULL for the
     * NoDepth variant: quality = (depth_cov0 + depth_cov1) * (uu + vv - 2 uv); `flow_quality` receives the
     * second factor, cand_vals its values at the NMS survivors and cand_vals2 depth_cov0 there. */
    const float* depth_cov0; /* (h,w) */
    const float* depth_cov1; /* (h,w) */
    float* flow_quality;     /* h*w */
    float* cand_vals2;       /* capacity h*w */
} macvo_score_t;
int macvo_dense_postproc(const float* est_flow, const float* est_cov, int h, int w, double bl_fx, double bl_fx_sq,
                         float* depth, float* disparity, float* depth_cov, uint8_t* depth_mask, float* flow_cov,
                         const macvo_score_t* score, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (a8) candidate selection — the rest of CovAwareSelector_NoDepth.select_point
 *      (Module/KeypointSelector.py:381-400): threshold = min(max_match_cov, 1.5 * lower-median of
 *      the NMS survivors), mask = nms & border & quality < threshold [& extra_mask], then the
 *      row-major ordered list of candidates (== torch.nonzero order).
 * cand_idx: capacity h*w int32 (linear pixel index row*w+col, ascending); *n_out: number written;
 * *thresh_out: the fp32 threshold; *status: 0 ok, 1 = no NMS survivor (torch.median of an empty tensor is NaN,
 * python's min(max_match_cov, nan) keeps max_match_cov, and the candidate list is simply empty).
 * workspace: macvo_select_workspace_bytes(h, w) bytes.
 */
size_t macvo_select_workspace_bytes(int h, int w);
int macvo_select_candidates(const float* quality, const uint8_t* nms, const float* cand_vals, const int* n_cand,
                            const uint8_t* extra_mask, int h, int w, int mask_width, double max_match_cov,
                            int* cand_idx, int* n_out, float* thresh_out, int* status, void* workspace,
                            size_t workspace_bytes, void* stream);

/* (a8') CovAwareSelector.select_point candidates (Module/KeypointSelector.py:292-330): mask = nms & border
 *      & depth0 < max_depth & depth1 < max_depth & depth_cov0 < min(max_depth_cov, 1.5 nanmedian(depth_cov0[nms]))
 *      & flow_quality < min(max_match_cov, 1.5 nanmedian(flow_quality[nms])) [& mask_a & mask_b].
 *      thresh_out[0] = depth-cov threshold, thresh_out[1] = flow threshold. */
int macvo_select_candidates_depth(const float* flow_quality, const float* depth0, const float* depth1,
                                  const float* depth_cov0, const uint8_t* nms, const float* cand_flow_quality,
                                  const float* cand_depth_cov0, const int* n_cand, const uint8_t* mask_a,
                                  const uint8_t* mask_b, int h, int w, int mask_width, double max_depth,
                                  double max_depth_cov, double max_match_cov, int* cand_idx, int* n_out,
                                  float* thresh_out, int* status, void* workspace, size_t workspace_bytes,
                                  void* stream);

/* (a8'') MappingPointSelector.select_point candidates (Module/KeypointSelector.py:87-97):
 *      depth < max_depth & depth_cov < max_depth_cov & border, row-major ordered. */
int macvo_select_mapping_candidates(const float* depth, const float* depth_cov, int h, int w, int mask_width,
                                    float max_depth, float max_depth_cov, int* cand_idx, int* n_out,
                                    void* workspace, size_t workspace_bytes, void* stream);

/* pixels[k] = (u, v) = (cand_idx[perm[k]] % w, cand_idx[perm[k]] / w) as int64 — the
 * `selected_points[perm][..., 2:].roll(1)` gather (KeypointSelector.py:404-405). */
int macvo_gather_pixels(const int* cand_idx, const int64_t* perm, int k, int w, int64_t* pixels_uv, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (a9) IFrontend.retrieve_pixels (Module/Frontend/Frontend.py:104-118): out[c, k] =
 *      map[0, c, (long) v_k, (long) u_k]. kp is (k, 2) [u, v], int64 (kp_is_int64 = 1) or fp32.
 */
int macvo_retrieve_pixels(const void* kp, int kp_is_int64, int k, const float* map, int channels, int h, int w,
                          float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (a10)+(a11) observation covariance — replaces MatchCovariance.estimate
 *      (Module/Covariance/Project2to3.py:124-182), gaussain_full_kernels (Utility/Math.py:44-63),
 *      Covariance_2to3_full (Project2to3.py:377-424); optionally pixel2point_NED (Utility/Point.py:15).
 *
 * kp (k,2) [u,v] int64 or fp32; depth (h,w) fp32; flow_cov (k,3) fp32 [uu, vv, uv], CLAMPED IN
 * PLACE to >= min_flow_cov^2 on its first two columns (reference side effect), or NULL = use
 * match_cov_default; element (i, c) is read / written at flow_cov[i * row_stride + c * col_stride] (in elements), so the
 * transposed view Odometry/MACVO.py:231-232 passes is clamped in the caller's own storage. depth_var (k) fp32 or NULL:
 * with flow_cov == NULL it replaces the Gaussian-weighted patch variance (Project2to3.py:163-171). out_cov (k,3,3) float64 (NED order z,x,y); out_point (k,3) fp32 NED point of
 * the CENTRE pixel depth (may be NULL); *status != 0 if a patch leaves the image (reference raises).
 */
int macvo_match_covariance(const void* kp, int kp_is_int64, int k, const float* depth, int h, int w, float* flow_cov,
                           long long flow_cov_row_stride, long long flow_cov_col_stride, const float* depth_var,
                           float fx, float fy, float cx, float cy, int kernel_size, float min_flow_cov,
                           float min_depth_cov, float match_cov_default, double* out_cov, float* out_point,
                           int* status, void* stream);
/* GaussianMixtureCovariance.estimate (Project2to3.py:194-272, gaussian_mixture_mean_var Utility/Math.py:66-93): the
 * arguments of macvo_match_covariance, plus depth_cov (h,w) fp32, the stereo network's per-pixel depth variance
 * (depth_est.cov, required: the reference asserts it). The same Gaussian weights p over the patch; p < 1e-3 becomes 0
 * (NaN stays NaN) and the rest is renormalised; mean = sum p d (the depth of the projection), variance =
 * (sum p (depth_cov + d^2) - mean^2) / 2, replaced by depth_var when flow_cov is NULL and depth_var is given. The
 * variance is NOT clamped (the reference never reads min_depth_cov, so there is no such argument): fp32 cancellation
 * can leave it slightly negative. A NaN depth or variance tap anywhere in the patch makes the matrix NaN. */
int macvo_gaussian_mixture_covariance(const void* kp, int kp_is_int64, int k, const float* depth, const float* depth_cov,
                                      int h, int w, float* flow_cov, long long flow_cov_row_stride,
                                      long long flow_cov_col_stride, const float* depth_var, float fx, float fy, float cx,
                                      float cy, int kernel_size, float min_flow_cov, float match_cov_default,
                                      double* out_cov, float* out_point, int* status, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (a14)+(a15) two-frame pose-graph optimisation — replaces TwoFrame_PGO._optimize
 *      (Module/Optimization/TwoFramePGO/Optimizer.py:82-102) = LM_analytic.step loop
 *      (Module/Optimization/PyposeOptimizers.py:160-194) over Analytic_ReprojDisp_TwoFramePGO
 *      (Module/Optimization/TwoFramePGO/Graphs.py:121-148, 201-230) with Huber(0.1) + FastTriggs,
 *      PINV, TrustRegion(radius 1e3), StopOnPlateau(10, patience 2, 1e-5).
 *
 * One persistent launch runs the whole LM loop on the device (a cluster of `cluster` CTAs, 1..8;
 * 0 = choose from k). Inputs fp64 (the reference promotes its fp32 buffers with .to(torch.double)):
 * pos_Tw (k,3), kp2_uv (k,2), kp2_disp (k), uv_cov (k,3) [uu,vv,uv], disp_cov (k);
 * intr = {fx, fy, cx, cy, baseline}; pose_io (7) [t, q_xyzw]: initial pose in, optimised pose out.
 * stats (8 doubles, may be NULL): {steps, loss evaluations, final loss, initial loss, last reject count,
 * final damping, 0, 0}.
 */
typedef struct {
    int max_steps;      /* 10   */
    int patience;       /* 2    */
    int max_reject;     /* 16   */
    int cluster;        /* 0 = auto */
    double decreasing;  /* 1e-5 */
    double huber_delta; /* 0.1  */
    double radius;      /* 1e3  */
    double diag_min;    /* 1e-6 */
    double diag_max;    /* 1e32 */
} macvo_pgo_params_t;
int macvo_pgo_solve(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp, const double* uv_cov,
                    const double* disp_cov, int k, const double* intr, double* pose_io,
                    const macvo_pgo_params_t* params, double* stats, void* stream);

/* The other graph types of TwoFrame_PGO (TwoFramePGO/Optimizer.py:51-68, analytic Jacobians Graphs.py:151-198):
 *   MACVO_PGO_DISP   (0) reprojection + disparity  (= macvo_pgo_solve)
 *   MACVO_PGO_REPROJ (1) reprojection only: kp2_disp / disp_cov unused (may be NULL)
 *   MACVO_PGO_ICP    (2) r = T p_c - p_w with p_c = pc_obs (k,3) [pixel2point_NED(pixel2_uv, pixel2_d), camera frame], block
 *                        covariance R obs_cov R^T + pts_cov ((k,3,3) float64 each: obs2_covTc, cov_Tw), re-inverted at every
 *                        linearisation like the reference's driver loop; kp2_uv / kp2_disp / uv_cov / disp_cov unused. */
#define MACVO_PGO_DISP 0
#define MACVO_PGO_REPROJ 1
#define MACVO_PGO_ICP 2
int macvo_pgo_solve_graph(int graph_type, const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                          const double* uv_cov, const double* disp_cov, const double* pc_obs, const double* obs_cov,
                          const double* pts_cov, int k, const double* intr, double* pose_io,
                          const macvo_pgo_params_t* params, double* stats, void* stream);

/* Same solve with the residual-block count read on the DEVICE (k = min(*k_dev, k_capacity)), so that the
 * observation kernel's survivor count never visits the host; fewer than min_k blocks ("lost track",
 * Odometry/MACVO.py:300-305: the optimiser is not started) leaves pose_io untouched and sets stats[6] = 1.
 * stats[7] = 1 when a rank-deficient covariance block received its pseudo-inverse weight. */
int macvo_pgo_solve_counted(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp, const double* uv_cov,
                            const double* disp_cov, int k_capacity, const int* k_dev, int min_k, const double* intr,
                            double* pose_io, const macvo_pgo_params_t* params, double* stats, void* stream,
                            int graph_type, const double* pc_obs, const double* obs_cov, const double* pts_cov);
/* graph_type / pc_obs / obs_cov / pts_cov as in macvo_pgo_solve_graph (0 / NULL: "disp", as before); for MACVO_PGO_ICP
 * they are the points_Tc / obs2_covTc / cov_Tw sections of an extended macvo_observe_pack buffer. */

/* Multi-GPU solve (BASELINE config 4; SURVEY.md §8e): the K residual blocks are sharded across `world` ranks (one process
 * per GPU), every rank launches this with ITS shard and the same pose_io / params; the all-reduce of the 55-double
 * accumulator happens INSIDE the persistent kernel through peer memory (stores into every rank's exchange buffer over
 * NVLink + system-scope release / acquire flags, summed in rank order -> identical bits on every rank), once per
 * evaluation; no NCCL call and no host round trip inside the LM loop. exchange_bufs: HOST array of `world` device
 * pointers, entry r = rank r's exchange buffer (macvo_pgo_exchange_bytes(world) bytes, zero-initialised, allocated with
 * macvo_p2p_alloc and mapped into this process with macvo_p2p_open; entry `rank` = this rank's own allocation).
 * All ranks must launch the same sequence of solves. A peer that never arrives traps after ~3 s instead of hanging. */
size_t macvo_pgo_exchange_bytes(int world);
int macvo_p2p_alloc(size_t bytes, void** dev_ptr, unsigned char* ipc_handle64);       /* cudaMalloc + zero + cudaIpcGetMemHandle */
int macvo_p2p_open(const unsigned char* ipc_handle64, void** peer_ptr);               /* cudaIpcOpenMemHandle (peer access) */
int macvo_p2p_close(void* peer_ptr);
int macvo_p2p_free(void* dev_ptr);
/* k_total_dev (optional device int, the same value on every rank): only the first *k_total_dev blocks of the GLOBAL
 * array are valid and this rank's k_shard blocks start at global index k_offset -> it uses
 * clamp(*k_total_dev - k_offset, 0, k_shard) of them; fewer than min_k valid blocks in total: every rank skips. */
int macvo_pgo_solve_sharded(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp, const double* uv_cov,
                            const double* disp_cov, int k_shard, const int* k_total_dev, int k_offset, int min_k,
                            const double* intr, double* pose_io, const macvo_pgo_params_t* params, double* stats,
                            void* const* exchange_bufs, int world, int rank, void* stream);

/* One evaluation of the packed normal-equation accumulator for a SHARD of residual blocks
 * (multi-GPU: each rank reduces its blocks, ranks all-reduce the 55 doubles, SURVEY.md §8e):
 * acc = [A upper 6x6 (21) | b (6) | G = Js^T Js upper (21) | h = Js^T Rs (6) | robust loss (1)].
 */
#define MACVO_PGO_ACC 55
#define MACVO_PGO_MAX_RANKS 8
int macvo_pgo_accumulate(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp, const double* uv_cov,
                         const double* disp_cov, int k, const double* intr, const double* pose, double huber_delta,
                         double* acc, void* stream);
/* The same accumulator for any graph type (graph_type and the icp columns as in macvo_pgo_solve_graph), reduced over a
 * cluster of `cluster` CTAs (1..8; 0 = choose from k as the solve does). singular_flag (one device double, may be NULL)
 * is set to 1 when a covariance block lost an eigenvalue to the pseudo-inverse, like stats[7] of the solve; it is never
 * cleared. macvo_pgo_accumulate = graph type MACVO_PGO_DISP, cluster 1, no flag. */
int macvo_pgo_accumulate_graph(int graph_type, const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                               const double* uv_cov, const double* disp_cov, const double* pc_obs, const double* obs_cov,
                               const double* pts_cov, int k, const double* intr, const double* pose, double huber_delta,
                               int cluster, double* acc, double* singular_flag, void* stream);

/* ---- frontend "next" rows (SURVEY.md §8f-1/2): memory-bound layers of the cost perceiver ----------------
 * fp32 only; replace the torch ops of Module/Network/FlowFormer/core/encoder.py:12-55 (PatchEmbed conv1 + pad),
 * the nn.LayerNorm calls of core/attention.py / core/twins.py / core/Twins/svt_large.py, and their
 * softmax(q k^T / sqrt(d)) v products (core/attention.py:6-29, core/twins.py:103-114,173-183).
 */
/* y = LayerNorm(x) over the last dim; x, y (rows, channels) contiguous; channels in {64, 128, 256, 512}. */
int macvo_layer_norm(const float* x, const float* weight, const float* bias, float* y, long long rows,
                     int channels, float eps, void* stream);
/* sum_out = x + resid; y = LayerNorm(sum_out) in one pass (channels in {128, 256, 512}); sum_out may alias x or resid. */
int macvo_add_layer_norm(const float* x, const float* resid, const float* weight, const float* bias, float* sum_out,
                         float* y, long long rows, int channels, float eps, void* stream);
/* Transformer MLP with residual, TF32 tensor cores (sm_90a): out = resid + w2 GELU_erf(w1 xn + b1) + b2, row-wise.
 * xn, resid, out (rows, channels) contiguous; w1 (hidden, channels), b1 (hidden), w2 (channels, hidden), b2 (channels);
 * channels == 128, hidden in {128, 512} (else MACVO_E_UNSUPPORTED); every pointer 16-byte aligned; out may not alias xn.
 * xn and the hidden activation (which never leaves the SM) are rounded to tf32, nearest-even, as cuBLAS rounds TF32 GEMM
 * operands; w1 / w2 are truncated by the MMA, so pass them pre-rounded the same way to compute what cuBLAS TF32 computes. */
int macvo_mlp_tc(const float* xn, const float* resid, const float* w1, const float* b1, const float* w2, const float* b2,
                 float* out, int rows, int channels, int hidden, void* stream);
/* PatchEmbed token head in one TF32 tensor-core kernel:
 *     out[r] = LayerNorm(w2 relu(w0 x[r] + term[r % period]) + b2; ln_w, ln_b, eps)
 * x (rows, in_channels), out (rows, channels) contiguous; w0 (channels, in_channels), term (period, channels),
 * w2 (channels, channels), b2 / ln_w / ln_b (channels); in_channels == 64, channels == 128 (else MACVO_E_UNSUPPORTED);
 * every pointer 16-byte aligned; out may not alias x. x and the hidden activation are rounded to tf32, nearest-even, as
 * cuBLAS rounds TF32 GEMM operands; pass w0 / w2 pre-rounded the same way to compute what the cuBLAS TF32 GEMMs, the
 * bias + ReLU pass and macvo_layer_norm compute, bit for bit. */
int macvo_patch_tokens_tc(const float* x, const float* w0, const float* term, const float* w2, const float* b2,
                          const float* ln_w, const float* ln_b, float* out, long long rows, int in_channels, int channels,
                          int period, float eps, void* stream);
/* maps (n_maps, 1, h, w) -> out (n_maps, ho, wo, 16) [NHWC], ho = ceil8(h)/2, wo = ceil8(w)/2:
 * ReLU(conv2d(zero-pad to multiples of 8, weight (16,1,6,6), stride 2, padding 2) + bias).
 * allow_tf32 bit 0: TF32 tensor-core implicit GEMM (what cuDNN does for the reference under cudnn.allow_tf32), else fp32 FMA.
 * allow_tf32 bit 1 (needs bit 0): write the result space-to-depth, i.e. as the NHWC tensor (n_maps, ho/2, wo/2, 64) whose channel
 *   block (y & 1) * 2 + (x & 1) holds pixel (y, x): PatchEmbed's next 6x6 / stride-2 convolution over 16 channels becomes a
 *   3x3 / stride-1 convolution over 64 channels (same arithmetic, full K blocks for the implicit GEMM). */
int macvo_patch_embed_conv1(const float* maps, const float* weight, const float* bias, float* out,
                            long long n_maps, int h, int w, int allow_tf32, void* stream);
/* in place x[r, :] = relu(x[r, :] + term[r % period, :]); x (rows, channels), term (period, channels), channels % 4 == 0
 * (PatchEmbed.ffn_with_coord.0 with its position input folded into a per-position bias, encoder.py:40-52) */
int macvo_add_rows_relu(float* x, const float* term, long long rows, int period, int channels, void* stream);
/* out = softmax(q k^T / sqrt(head_dim)) v per (batch, head); q (batch | 1, nq, heads, head_dim),
 * k, v (batch, nk, heads, head_dim), out (batch, nq, heads, head_dim); head_dim in {16, 32};
 * q_broadcast != 0: one query set shared by every batch element. head_dim 8 only for nq <= 8, heads == 8.
 * allow_tf32 != 0: products with nq >= 16 run on the tensor cores in TF32 (fp32 accumulate, fp32 softmax), the
 * precision the reference runs its attention bmm's at (Frontend.py:275-277); 0 = fp32 FMA throughout. */
int macvo_small_attention(const float* q, const float* k, const float* v, float* out, int batch, int nq, int nk,
                          int heads, int head_dim, int q_broadcast, int allow_tf32, void* stream);

/* extended form: row strides ldq / ldk / ldv in floats (0 = heads*head_dim, must be multiples of 4) so a fused [q|k|v]
 * projection output is consumed in place, and optional additive terms q_add (add_period, nq, heads*head_dim) /
 * k_add (add_period, nk, heads*head_dim) added to q / k on load, batch b using slice b % add_period — the
 * context + position half of the vertical attention's projections (core/twins.py:46-66, 120-150). */
int macvo_small_attention_ex(const float* q, const float* k, const float* v, float* out, int batch, int nq, int nk,
                             int heads, int head_dim, int q_broadcast, int allow_tf32, int ldq, int ldk, int ldv,
                             const float* q_add, const float* k_add, int add_period, void* stream);

/* Perceiver input layer, fused (core/encoder.py:150-191): 8 shared latent queries x 8 heads (head_dim 16) attend to
 * the nk token rows of every cost map WITHOUT materialising K and V:  tokens (n_maps, nk, 128) fp32;
 * ut (64, 128) = rows h*8+i of Wk[h]^T q[i,h] / sqrt(16); wv (128,128), bv (128) = the value projection;
 * out (n_maps, 8, 128) = softmax(...) V in the layout of `MultiHeadAttention`'s output. TF32 tensor cores. */
int macvo_latent_pool(const float* tokens, const float* ut, const float* wv, const float* bv, float* out,
                      long long n_maps, int nk, void* stream);

/* ---- decoder iteration glue (SURVEY.md §8f-2): SepConvGRU state kept in NHWC [h | x] buffers ---------------
 * Module/Network/FlowFormer/core/gru.py:22-43 (SepConvGRU), gma.py:84-130, covhead.py:95-131. fp32, pixels-major.
 * A GRU input buffer is (pixels, 512): channels 0..127 = h (or r*h), 128..255 = inp, 256..383 = motion features,
 * 384..511 = motion features + gamma * aggregated motion features.
 */
/* writes channels 256..511 of up to four buffers (NULL entries after buf0 are skipped) */
int macvo_gru_input(const float* mf, const float* agg, const float* gamma, float* buf0, float* buf1, float* buf2,
                    float* buf3, long long pixels, void* stream);
/* zr (pixels,256) = conv([h|x]) pre-activation, bias (256, may be NULL) is added first;
 * z_out (pixels,128) = sigmoid(zr[:, :128]); rhx[:, :128] = sigmoid(zr[:, 128:]) * hx[:, :128] */
int macvo_gru_gates(const float* zr, const float* bias, const float* hx, float* z_out, float* rhx, long long pixels,
                    void* stream);
/* hx[:, :128] <- (1 - z) * hx[:, :128] + z * tanh(q + bias); bias (128) may be NULL; optional dense copy (pixels,128) */
int macvo_gru_blend(const float* q, const float* bias, const float* z, float* hx, float* h_dense, long long pixels,
                    void* stream);
/* ---- decoder convolutions on wgmma (csrc/conv_tc.cu): 3x3 (padding 1) / 1x1 convolutions of the motion encoder, the GMA value
 * projection, the flow head and the covariance head (core/gru.py:6-14,45-64, gma.py:84-130, FlowFormerCov/covhead.py:20-58) as
 * implicit GEMMs over fp16 pixel rows in "layout U" (csrc/rows_layout.cuh): image b, pixel (y, x) lives at row
 * 2 + (b (H + 4) + y + 2)(W + 4) + x + 2 of a zero-initialised buffer of macvo_rows_count(batch, H, W, 0) rows; the kernels only
 * write pixel rows, so the padding stays zero.
 *   in_rows   (rows, in_channels) fp16, in_channels % 64 == 0; in_dense = 1 (ksize 1 only): plain (pixels, in_channels) rows
 *   weights   (n_pad, ksize^2 * in_channels) fp16, K index = (ky * ksize + kx) * in_channels + c; n_pad % 32 == 0, rows >= n_valid
 *             zero; bias (n_pad) fp32 or NULL; relu != 0 applies max(., 0)
 *   out16     optional fp16 rows [.., out16_offset + n] with row pitch out16_pitch (elements): layout U rows, or dense pixel rows when
 *             out16_dense; out32: optional fp32 dense pixel rows, or — out32_planes != 0 — a (batch, n_valid, H, W) fp32 map to
 *             which the result is ADDED in place (the decoder's `coords1 = coords1 + delta_flow`, covhead.py:133-134).
 *             Only columns n < n_valid are stored. */
size_t macvo_rows_count(int batch, int height, int width, int vertical);
int macvo_conv_tc(const void* in_rows, int in_channels, int in_dense, const void* weights, const float* bias, int n_pad,
                  int n_valid, int ksize, int relu, int batch, int height, int width, void* out16, int out16_pitch,
                  int out16_offset, int out16_dense, float* out32, int out32_pitch, int out32_offset, int out32_planes,
                  void* stream);
/* the motion encoder's 7x7 convolution of the 2-channel flow as a GEMM operand (gru.py:50,57): rows (pixels, 128) fp16 dense,
 * column (ky * 7 + kx) * 2 + c = (coords1 - coords0)[c, y + ky - 3, x + kx - 3], zero outside / beyond column 98; also writes the
 * flow into channels 126, 127 of the motion-feature rows (mf32: (pixels, 128) fp32 dense, mf16_rows: layout U, 128 ch; may be NULL) */
int macvo_flow_im2col(const float* coords1, const float* coords0, void* rows, float* mf32, void* mf16_rows, int batch,
                      int height, int width, void* stream);

/* ---- SepConvGRU on wgmma (csrc/gru_conv_tc.cu): the 1x5 / 5x1 gate convolutions of gru.py:22-43 as implicit GEMMs with the
 * gate math in the epilogue, for one recurrent unit (flow or covariance — covhead.py:95-131) per launch.
 * Operands are fp16 PADDED pixel rows: pass `vertical` = 0 (1x5) uses layout U (above), `vertical` = 1 (5x1) stores pixel
 * (b, y, x) at row 2 + (b W + x)(H + 4) + y + 2; all other rows must be zero (allocate
 * macvo_gru_tc_operand_rows(...) zeroed rows once; the kernels only ever write pixel rows).
 *   h_rows      (rows, 128) fp16: stage 0: h, stage 1: r*h          x_rows (rows, 384) fp16: [inp | mf | mf + gamma agg]
 *   weights     (N, 5*512) fp16, K index = tap * 512 + channel of cat[h, x]; N = 256 (z | r) for stage 0, 128 (q) for stage 1
 *   bias (N) fp32;  h_master, z (pixels, 128) fp32 in dense pixel order (the recurrent state stays fp32)
 *   out_rows    (rows', 128) fp16: stage 0 writes r*h rows of THIS pass's layout, stage 1 writes the new h in the OTHER
 *   pass's layout (the next pass's input) and updates h_master in place.
 * stage 0: z = sigmoid(conv + b)[:128] -> z;  r*h -> out_rows.     stage 1: h <- (1 - z) h + z tanh(conv + b). */
size_t macvo_gru_tc_operand_rows(int batch, int height, int width, int vertical);
int macvo_gru_tc_stage(int stage, int vertical, int batch, int height, int width, const void* h_rows, const void* x_rows,
                       const void* weights, const float* bias, float* h_master, float* z, void* out_rows, void* stream);
/* fp32 dense pixel rows src (pixels, src_pitch)[:, :channels] -> fp16 operand rows dst[:, dst_offset : dst_offset + channels] */
int macvo_gru_tc_pack(const float* src, int src_pitch, int channels, void* dst, int dst_channels, int dst_offset, int batch,
                      int height, int width, int vertical, void* stream);
/* per iteration: x channels [128, 384) = [mf | mf + gamma * agg] of both layouts (gma.py:84-130) */
int macvo_gru_tc_pack_motion(const float* mf, const float* agg, const float* gamma, void* x_rows_h, void* x_rows_v, int batch,
                             int height, int width, void* stream);
/* GMA attention matrix (gma.py:39-82): out (rows, cols) fp16 = softmax over each row of the fp32 scores; cols % 4 == 0, <= 8192.
 * Replaces softmax (fp32 read + write) + cast to fp16: the row is read once. Used when TF32 matmuls are allowed (the matrix is
 * then kept in fp16 for the per-iteration aggregation GEMM). */
int macvo_softmax_rows_f16(const float* scores, void* out, long long rows, int cols, void* stream);
/* convex 8x upsampling (core/decoder.py:131-139): flow (batch, 2, H, W) fp32 planes, mask_nhwc (batch, H, W, 576) fp32 logits
 * (channel k*64 + i*8 + j; a channels_last convolution output), out (batch, 2, 8H, 8W):
 * out[n, c, 8y+i, 8x+j] = sum_k softmax_k(scale * mask[.., k*64 + i*8 + j]) * 8 * flow[n, c, y + k/3 - 1, x + k%3 - 1] (zero outside) */
int macvo_convex_upsample(const float* flow, const float* mask_nhwc, float* out, float scale, int batch, int height, int width,
                          void* stream);

/* ------------------------------------------------------------------------------------------------
 * (f3) observation building + sanity filter + MatchObs packing on the device — replaces the host code of
 *      Odometry/MACVO.py:198-270 (flow lookup, filterPointsInRange, retrieve_pixels x9, ObsCovModel.estimate x2,
 *      pixel2point_NED, MatchObs.init), CovarianceSanityFilter.filter (Module/OutlierFilter.py:91-100) and the
 *      point registration SE3.Act(prev_pose, pos0_Tc) (MACVO.py:279-283) for the two-frame pose graph.
 *
 * kp0_uv (k,2) int64 selected keypoints; flow (2,h,w), match_cov (3,h,w) of the frame0->frame1 match; depth0 of
 * frame 0; depth1 / disparity1 / disp_unc1 of frame 1 (all (h,w) fp32 device). intr0 / intr1: HOST {fx,fy,cx,cy}.
 * prev_pose (7) float64 device [t, q_xyzw]; next_pose (7) receives the static-motion-model prediction (prev pose
 * rounded to fp32, what the map stores). packed: macvo_observe_packed_doubles(capacity) float64, layout with c = capacity:
 *   [0,3c) pos_Tw | [3c,5c) pixel2_uv | [5c,6c) pixel2_disp | [6c,9c) pixel2_uv_cov | [9c,10c) pixel2_disp_cov
 *   [10c,19c) obs1_covTc | [19c,28c) obs2_covTc | [28c,30c) pixel1_uv | [30c,31c) pixel1_d | [31c,31c+4) n_obs, n_inbound, k, status
 * (the first five sections are exactly the arrays macvo_pgo_solve_counted reads). *n_obs = survivors (device int).
 * *status (zeroed by the caller) is a bitmask, OR-ed by every observation that meets a condition:
 *   bit 0 (1): a covariance patch crossed the bottom or right image edge (the reference raises IndexError; those
 *              rows' covariances are unspecified). Patches crossing the top / left edge wrap like python indices.
 *              Never set with the NoCovariance model (ext->cov_model == MACVO_COV_IDENTITY), which reads no patch.
 *   bit 1 (2): a keypoint kp0 lies outside the image; its row is dropped and not counted in n_inbound.
 */
/* CovarianceSanityFilter.filter (Module/OutlierFilter.py:91-100) on device-resident (k,3,3) float64 covariances:
 * good[i] = 1 iff neither matrix of observation i holds a NaN / Inf. */
int macvo_cov_sanity_filter(const double* obs1_cov, const double* obs2_cov, int k, uint8_t* good, void* stream);
/* Optional extension of macvo_observe_pack (HOST struct; NULL = sanity filter only, the layout above): the other two
 * observation filters of FilterCompose (Module/OutlierFilter.py:106-141) and the columns of the "icp" pose graph.
 * Per in-bound row the kernel also gathers pixel2_d = depth1 at the truncated kp1, pixel1_d_cov = depth_cov0 at kp0 and
 * pixel2_d_cov = depth_cov1 at kp1 (-1, the reference's placeholder, where the map is NULL). fp32 throughout:
 *   simple_depth  drop a row when d < min_depth or d > max_depth on either frame (NaN depth passes);
 *   front_of_cam  keep a row when d - 2 sqrt(d_cov) > 0 on both frames (NaN / negative d_cov drops it), unless ANY
 *                 in-bound row has pixel1_d_cov == -1: then this filter passes every row;
 *   icp           also pack pixel2_d, pixel1_d_cov, pixel2_d_cov, points_Tc = pixel2point_NED(pixel2_uv, pixel2_d, K1)
 *                 (fp32, widened) and cov_Tw = R obs1_covTc R^T (float64; R = rotation matrix of prev_pose rounded to
 *                 fp32, computed in fp32, widened) for the kept rows, AFTER the header (every offset above stays):
 *   [31c+4,32c+4) pixel2_d | [32c+4,33c+4) pixel1_d_cov | [33c+4,34c+4) pixel2_d_cov | [34c+4,37c+4) points_Tc (c,3)
 *   [37c+4,46c+4) cov_Tw (c,3,3)        -> `packed` must hold macvo_observe_packed_doubles(capacity, 1) = 46c + 4 doubles.
 * macvo_observe_packed_doubles(capacity, 0) = 31c + 4.
 *
 * The covariance model (Module/Covariance/Project2to3.py:48-57, 194-272, 281-323); all zero = MatchCovariance without
 * modifiers, exactly the behaviour above:
 *   cov_model     MACVO_COV_MATCH, MACVO_COV_IDENTITY (NoCovariance: no depth taps, the uv-covariance columns hold the
 *                 network's values unclamped, status bit 0 is never set, both 3x3 covariances are the identity), or
 *                 MACVO_COV_GAUSSIAN_MIXTURE (GaussianMixtureCovariance, see macvo_gaussian_mixture_covariance: depth_cov0
 *                 / depth_cov1 are the variance maps of frame 0 / 1 and must both be given, else MACVO_E_ARG; its
 *                 covariances can be NaN, which the sanity filter drops);
 *   cov_ops[0..n_cov_ops)  modifiers in the order they apply (innermost wrapper first), in float64 on the widened fp32
 *                 covariances, BEFORE the sanity filter, the obs1_covTc / obs2_covTc columns and cov_Tw (see macvo_cov_modify).
 * Setting only these fields (no filter, icp 0) keeps the 31c + 4 layout and applies the sanity filter alone. */
#define MACVO_COV_MATCH 0
#define MACVO_COV_IDENTITY 1
#define MACVO_COV_GAUSSIAN_MIXTURE 2
#define MACVO_COV_DIAGONALIZE 1
#define MACVO_COV_NORMALIZE 2
#define MACVO_COV_MAX_OPS 2
typedef struct {
    const float* depth_cov0; /* (h,w) device, or NULL */
    const float* depth_cov1; /* (h,w) device, or NULL */
    int simple_depth;
    float min_depth, max_depth;
    int front_of_cam;
    int icp;
    int cov_model;
    int cov_ops[MACVO_COV_MAX_OPS];
    int n_cov_ops;
} macvo_observe_ext_t;
/* The covariance modifiers on device (k,3,3) float64 matrices, in place, applied in the order of the HOST array ops[0..n_ops):
 *   MACVO_COV_DIAGONALIZE  Modifier_Diagonalize: the six off-diagonal entries become 0 (a NaN / Inf there disappears);
 *   MACVO_COV_NORMALIZE    Modifier_Normalize: each matrix divided by ITS OWN determinant, from a 3x3 LU with partial
 *                          pivoting (largest |a|, first on ties; multipliers by division; det = sign u00 u11 u22), each
 *                          element divided (round-to-nearest) — det 0 gives +-Inf / NaN, a negative det flips the sign.
 * n_ops <= MACVO_COV_MAX_OPS. The same routine runs inside macvo_observe_pack. */
int macvo_cov_modify(double* cov, int k, const int* ops, int n_ops, void* stream);
size_t macvo_observe_workspace_bytes(int capacity);
size_t macvo_observe_packed_doubles(int capacity, int extended);
int macvo_observe_pack(const int64_t* kp0_uv, int k, int capacity, const float* flow, const float* match_cov,
                       const float* depth0, const float* depth1, const float* disparity1, const float* disp_unc1,
                       int h, int w, int edge_width, const float* intr0, const float* intr1, int kernel_size,
                       float min_flow_cov, float min_depth_cov, float match_cov_default, const double* prev_pose,
                       double* next_pose, double* packed, int* n_obs, int* status, void* workspace,
                       size_t workspace_bytes, void* stream, const macvo_observe_ext_t* ext);
/* match_cov == NULL && disp_unc1 == NULL: the frontend gives no covariance maps (FrontendCompose of FlowFormerDepth +
 * FlowFormerMatcher, the Vanilla ablation; Odometry/MACVO.py:212-264 with kp*_sigma_dd, kp1_sigma_disparity and
 * kp1_sigma_uv None). Passing only one of the two as NULL is MACVO_E_ARG.
 *   - pixel2_uv_cov (all 3 columns) and pixel2_disp_cov hold -1, MatchObs' placeholder (MACVO.py:250-264); so do the
 *     icp columns pixel1_d_cov / pixel2_d_cov when ext->depth_cov0 / depth_cov1 are NULL, as above.
 *   - MACVO_COV_MATCH: MatchCovariance.estimate with flow_cov None for kp1 (Project2to3.py:128-135): its 2x2 flow
 *     covariance is match_cov_default * [1, 1, 0] WITHOUT the min_flow_cov^2 clamp; kp0 keeps the clamped default.
 *   - MACVO_COV_IDENTITY: unchanged (identity covariances).
 *   - MACVO_COV_GAUSSIAN_MIXTURE: kp1's flow covariance as for MACVO_COV_MATCH, and its variance is depth_cov1 at kp1
 *     (Project2to3.py:254-255: no flow_cov, a depth_cov given). */

/* ------------------------------------------------------------------------------------------------
 * (f2) decoder token path of one refinement iteration as one kernel — replaces flow_token_encoder (decoder.py:112-116),
 *      CrossAttentionLayer (decoder.py:20-76: LayerNorm + sine position embedding, q projection, 8-head attention of each
 *      pixel's query to its 8 cost-memory tokens, output projection, FFN) and the motion encoder's input concat
 *      (gru.py:53-54).  cost_forward (P,81) pixels-major lookup rows; coords (B,2,n1); key / value (P,8,64) (the k / v
 *      projections of the cost memory, computed once per frame); weight_blob: macvo_decoder_token_blob_floats() floats =
 *      [W0^T (81x64) | W2^T (64x64) | Wq^T (64x64) | Wproj^T (128x64) | F0^T (64x64) | F3^T (64x64) | b0 | b2 | ln1.w |
 *      ln1.b | bq | bproj | ln2.w | ln2.b | bf0 | bf3 | freq(16)].  out (P,160) = [cost_global (64) | cost_forward (81) | 0].
 */
size_t macvo_decoder_token_blob_floats(void);
int macvo_decoder_token(const float* cost_forward, const float* coords, const float* key, const float* value,
                        const float* weight_blob, float* out, int batch, int n1, float eps, void* stream);
/* same, writing fp16 "layout U" rows (see macvo_conv_tc; 192 channels per row, [0,160) = [g | cost_forward | 0]) */
int macvo_decoder_token_rows(const float* cost_forward, const float* coords, const float* key, const float* value,
                             const float* weight_blob, void* out16_rows, int batch, int height, int width, float eps,
                             void* stream);

/* ------------------------------------------------------------------------------------------------
 * (f4) trajectory post-process at terminate(): MotionInterpolate.elaborate_map (Module/MapProcessor.py:52-79) with
 *      interpolate_pose / NormalizeQuat (Utility/Math.py:96-135). poses (F,7) fp32 [t, q_xyzw] updated in place
 *      (row 0 untouched), need_interp (F) bytes; *n_interp (optional) = number of interpolated relative motions.
 */
size_t macvo_motion_interpolate_workspace_bytes(int num_frames);
int macvo_motion_interpolate(float* poses, const uint8_t* need_interp, int num_frames, int* n_interp, void* workspace,
                             size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (f5) TartanMotionNet pose network (VOFlowRes config 1, Module/Network/TartanVOStereo/FlowPoseNet.py:45-165).
 *
 * macvo_posenet_input: flow (2,H,W) + depth (1,H,W) fp32 (H >= 112, W >= 160) -> channels 0..2 of the (5,112,160) network
 *      input `out` (channels 3..4, the intrinsics layer, are left untouched): TartanStereoVOMotion.inference
 *      (StereoVO_Interface.py:158-194) — centre crop, bilinear align_corners resize, flow x 0.05, normalised disparity.
 * macvo_posenet_conv: y = epilogue(conv(x, W) + bias [+ resid]) for x (cin,hi,wi), y (cout,ho,wo); epilogue = ReLU when
 *      `relu`. w_packed (16-byte aligned) holds W (cout,cin,k,k) as per-CTA slabs [cout/co_tile][8][co_tile][cin/8*k*k];
 *      cin % 8 == 0, cout % co_tile == 0, co_tile * cin/8 * k*k % 4 == 0. Deterministic (no atomics).
 * macvo_posenet_head: fc1_out (256) = [trans 128 | rot 128] after ReLU; head_blob (macvo_posenet_head_floats()) =
 *      [fc2 trans W (32x128) | b | fc2 rot W | b | fc3 trans W (3x32) | b | fc3 rot W | b | pose_norm (6)];
 *      motion (6) fp32 = cat(trans, rot) * pose_norm; next_pose (7) float64 = prev_pose (rounded to fp32) @ se3(motion).Exp()
 *      in fp32 ([t, q_xyzw]).
 */
int macvo_posenet_input(const float* flow, const float* depth, int height, int width, double bl_fx, float* out, void* stream);
int macvo_posenet_conv(const float* x, int cin, int hi, int wi, const float* w_packed, const float* bias, int cout, int ksize,
                       int stride, int pad, int co_tile, const float* resid, int relu, float* y, void* stream);
size_t macvo_posenet_head_floats(void);
int macvo_posenet_head(const float* fc1_out, const float* head_blob, const double* prev_pose, float* motion,
                       double* next_pose, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (f6) TartanVOMatcher's PWC-Net (PWCDCNet_Adapted, Module/Network/PWCNet/pwc/pwc_model_tartanvo.py:64-297): warp +
 *      correlation + LeakyReLU(0.1) of one pyramid level — replaces warp() (:176-212), FunctionCorrelation and the
 *      leakyRELU after it (:230-232, 259-260), i.e. the cupy kernels of correlation.py:35-102, 277-318.
 * f1, f2 (batch, channels, H, W) fp32; flow (batch, 2, H, W) fp32, or NULL = no warp (level 6).
 * g = f2 when flow is NULL, else g[c,y,x] = grid_sample(f2, (x + s*flow_x, y + s*flow_y))[c] * m(y,x) (s = flow_scale,
 *      bilinear, zeros padding, align_corners=True; m = the same sampling of ones, 0 where < 0.9999, 1 where > 0). Tap
 *      positions, weights and m are computed in fp32 in the reference's order; a non-finite position or one beyond
 *      +-2^24 has no in-bounds tap (sample 0, m 0).
 * out (batch, out_channels, H, W) fp32: channels [out_offset, out_offset + 81) only are written,
 *      out[out_offset + (dy+4)*9 + (dx+4), y, x] = LeakyReLU_0.1((1/C) sum_c f1[c,y,x] g[c,y+dy,x+dx]), g = 0 outside the image.
 * MACVO_E_ARG (nothing launched): a NULL f1 / f2 / out, a size <= 0, out_offset < 0 or out_offset + 81 > out_channels.
 */
int macvo_pwc_warp_corr(const float* f1, const float* f2, const float* flow, float flow_scale,
                        int batch, int channels, int height, int width,
                        float* out, int out_channels, int out_offset, void* stream);

/* ------------------------------------------------------------------------------------------------
 * (f7) TartanVODepth's full-resolution heads and depth conversion (StereoCovNet(exp=False, decoder="hourglass"),
 *      Module/Network/StereoCov/{StereoNet,decoder,network}.py): for the disparity head (xd) and, when xc is not NULL, the
 *      covariance head (xc), with K = [x | cat0] (64 + 64 channels):
 *      out = conv_c13(relu(conv_c12(relu(deconv_c11(K))))) (+ relu on the covariance head), then disp = out_d / 0.02,
 *      depth = (1 / disp) * bf, var = bf2 * ((out_c / disp^2) / disp^2), all fp32 with IEEE division.
 * xd, xc, cat0 (1, 64, h2, w2) fp32 contiguous; w11_* (4 chunks, 4 phases, 4 taps, 64, 32) fp32, tf32-rounded
 *      (stereonet.arrange_head); small_* b11 (64) | w12 (16 x 64) | b12 (16) | w13 (16) | b13 (1) fp32.
 * depth, var (height, width) fp32: only [margin_y, margin_y + 2 h2) x [margin_x, margin_x + 2 w2) is written; var is
 *      not touched when xc is NULL. Runs the deconvolution on TF32 tensor cores (the caller decides that TF32 is allowed).
 * MACVO_E_ARG (nothing launched): a NULL xd / cat0 / w11_d / small_d / depth, xc without w11_c / small_c / var, a size
 *      <= 0, a negative margin, a crop beyond the frame, or a weight blob not 16-byte aligned.
 */
int macvo_stereo_head(const float* xd, const float* xc, const float* cat0, int h2, int w2, const float* w11_d,
                      const float* small_d, const float* w11_c, const float* small_c, float bf, float bf2, int margin_y,
                      int margin_x, int height, int width, float* depth, float* var, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MACVO_B200_H */
