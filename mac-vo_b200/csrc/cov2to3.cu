// (a10)+(a11) per-keypoint observation covariance: 31x31 Gaussian-weighted depth statistics and the
// closed-form 2D -> 3D covariance projection. One warp per keypoint.
//
// match_cov_kernel replaces MatchCovariance.estimate (Module/Covariance/Project2to3.py:124-182), gaussain_full_kernels
// (Utility/Math.py:44-63), Covariance_2to3_full (Project2to3.py:377-424), create_3x3_matrix (:426-434,
// which assembles the result on the CPU through 9 implicit device->host copies) and pixel2point_NED
// (Utility/Point.py:15-17). Given a depth-variance map, the same kernel replaces GaussianMixtureCovariance.estimate
// (Project2to3.py:194-272) and gaussian_mixture_mean_var (Utility/Math.py:66-93) the same way. Reference quirks kept (SURVEY.md §7.3): in-place clamp
// of the caller's flow_cov (through its strides: the caller's tensor may be a transposed view); the kernel axis weighted
// by sigma_uu runs along image ROWS of the depth patch; the depth_cov argument replaces the patch variance only when
// no flow_cov is given.
//
// L2-gather bound: K * (961*4 + 20) B in (twice the taps for the mixture), K * 72 B out (2 MB at K=512, 16 MB at K=4096).
// fp32 arithmetic like the reference, result widened to fp64 at the end (`.double()`).
#include "cov2to3.cuh"

namespace {

// flow_cov[..., :2].clamp_(min=min_flow_cov**2) in the caller's storage, or match_cov_default * [1, 1, 0]
__device__ __forceinline__ void flow_cov_of(float* __restrict__ flow_cov, long long fc_row, long long fc_col, int warp,
                                            int lane, float min_flow_var, float match_cov_default, float& suu, float& svv,
                                            float& suv) {
    if (flow_cov) {
        // element (i, c) of the caller's (K,3) view lives at i * fc_row + c * fc_col: MAC-VO passes the transposed
        // view `retrieve_pixels(...).T` (Odometry/MACVO.py:231-232), and the clamp below must land in THAT storage
        float* fc = flow_cov + (long long)warp * fc_row;
        const float a = fc[0], b = fc[fc_col];
        suu = (a != a) ? a : fmaxf(a, min_flow_var);             // clamp_(min=min_flow_cov**2); NaN stays NaN
        svv = (b != b) ? b : fmaxf(b, min_flow_var);
        suv = fc[2 * fc_col];
        __syncwarp();
        if (lane == 0) { fc[0] = suu; fc[fc_col] = svv; }
    } else {
        suu = svv = match_cov_default;
        suv = 0.f;
    }
}

// lane 0: the (3,3) float64 covariance and, when asked, pixel2point_NED with the CENTRE pixel's depth (Odometry/MACVO.py:209,239)
__device__ __forceinline__ void store_result(const float s6[6], float u, float v, long long ul, long long vl,
                                             const float* __restrict__ depth, int h, int w, const macvo::CovParams& P,
                                             int warp, double* __restrict__ out_cov, float* __restrict__ out_point) {
    macvo::store_cov9(out_cov + 9LL * warp, s6);
    if (out_point) {
        const long long yy = vl < 0 ? vl + h : vl, xx = ul < 0 ? ul + w : ul;
        const float d = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? depth[yy * w + xx] : CUDART_NAN_F;
        const float du = __fsub_rn(u, P.cx), dv = __fsub_rn(v, P.cy);
        out_point[3 * warp] = d;
        out_point[3 * warp + 1] = __fmul_rn(__fdiv_rn(du, P.fx), d);
        out_point[3 * warp + 2] = __fmul_rn(__fdiv_rn(dv, P.fy), d);
    }
}

// One kernel serves both models: depth_cov (the per-pixel depth variance map) selects GaussianMixtureCovariance, NULL
// MatchCovariance. The choice is uniform across the launch, so the branch never diverges.
template <typename KP>
__global__ void __launch_bounds__(128)
match_cov_kernel(const KP* __restrict__ kp, int k, const float* __restrict__ depth, const float* __restrict__ depth_cov,
                 int h, int w, float* __restrict__ flow_cov, long long fc_row, long long fc_col,
                 const float* __restrict__ depth_var, macvo::CovParams P, float min_flow_var, float match_cov_default,
                 double* __restrict__ out_cov, float* __restrict__ out_point, int* __restrict__ status) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= k) return;
    const KP ku = kp[2 * warp], kv = kp[2 * warp + 1];
    const float u = (float)ku, v = (float)kv;                   // value used in the closed form
    const long long ul = (long long)ku, vl = (long long)kv;     // .long(): truncation, used for indexing
    float suu, svv, suv;
    flow_cov_of(flow_cov, fc_row, fc_col, warp, lane, min_flow_var, match_cov_default, suu, svv, suv);
    const bool override_var = flow_cov == nullptr && depth_var != nullptr;
    const float dvar = override_var ? depth_var[warp] : 0.f;
    float s6[6];
    const bool oob = depth_cov
        ? macvo::mixture_cov_warp(u, v, ul, vl, depth, depth_cov, h, w, suu, svv, suv, override_var, dvar, P, lane, s6)
        : macvo::match_cov_warp(u, v, ul, vl, depth, h, w, suu, svv, suv, override_var, dvar, P, lane, s6);
    if (oob && lane == 0) atomicExch(status, 1);
    if (lane == 0) store_result(s6, u, v, ul, vl, depth, h, w, P, warp, out_cov, out_point);
}

int launch_cov(const void* kp, int kp_is_int64, int k, const float* depth, const float* depth_cov, int h, int w,
               float* flow_cov, long long rs, long long cs, const float* depth_var, float fx, float fy, float cx, float cy,
               int kernel_size, float min_flow_cov, float min_depth_cov, float match_cov_default, double* out_cov,
               float* out_point, int* status, void* stream) {
    if (k < 0 || h <= 0 || w <= 0 || kernel_size < 1 || (kernel_size & 1) == 0 || kernel_size > 31) return MACVO_E_ARG;
    if (k == 0) return MACVO_OK;
    if (!kp || !depth || !out_cov || !status) return MACVO_E_ARG;
    if (flow_cov && (rs == 0 || cs == 0)) return MACVO_E_ARG;
    const float min_flow_var = min_flow_cov * min_flow_cov;
    const macvo::CovParams P{fx, fy, cx, cy, kernel_size, min_depth_cov};
    const int blocks = ceil_div(k * 32, 128);
    cudaStream_t st = as_stream(stream);
    if (kp_is_int64)
        match_cov_kernel<int64_t><<<blocks, 128, 0, st>>>(static_cast<const int64_t*>(kp), k, depth, depth_cov, h, w,
                                                         flow_cov, rs, cs, depth_var, P, min_flow_var, match_cov_default,
                                                         out_cov, out_point, status);
    else
        match_cov_kernel<float><<<blocks, 128, 0, st>>>(static_cast<const float*>(kp), k, depth, depth_cov, h, w, flow_cov,
                                                       rs, cs, depth_var, P, min_flow_var, match_cov_default, out_cov,
                                                       out_point, status);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

}  // namespace

extern "C" int macvo_match_covariance(const void* kp, int kp_is_int64, int k, const float* depth, int h, int w,
                                      float* flow_cov, long long flow_cov_row_stride, long long flow_cov_col_stride,
                                      const float* depth_var, float fx, float fy, float cx, float cy, int kernel_size,
                                      float min_flow_cov, float min_depth_cov, float match_cov_default,
                                      double* out_cov, float* out_point, int* status, void* stream) {
    return launch_cov(kp, kp_is_int64, k, depth, nullptr, h, w, flow_cov, flow_cov_row_stride,
                      flow_cov_col_stride, depth_var, fx, fy, cx, cy, kernel_size, min_flow_cov, min_depth_cov,
                      match_cov_default, out_cov, out_point, status, stream);
}

extern "C" int macvo_gaussian_mixture_covariance(const void* kp, int kp_is_int64, int k, const float* depth,
                                                 const float* depth_cov, int h, int w, float* flow_cov,
                                                 long long flow_cov_row_stride, long long flow_cov_col_stride,
                                                 const float* depth_var, float fx, float fy, float cx, float cy,
                                                 int kernel_size, float min_flow_cov, float match_cov_default,
                                                 double* out_cov, float* out_point, int* status, void* stream) {
    if (k > 0 && !depth_cov) return MACVO_E_ARG;       // the reference asserts depth_est.cov is not None
    return launch_cov(kp, kp_is_int64, k, depth, depth_cov, h, w, flow_cov, flow_cov_row_stride,
                      flow_cov_col_stride, depth_var, fx, fy, cx, cy, kernel_size, min_flow_cov, 0.f, match_cov_default,
                      out_cov, out_point, status, stream);
}
