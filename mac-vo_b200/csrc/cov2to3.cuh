// Warp-level observation-covariance routines shared by match_cov_kernel (cov2to3.cu) and the fused
// observation kernel (observe.cu). See cov2to3.cu for the reference lines they follow.
#pragma once
#include "common.cuh"
#include <math_constants.h>

namespace macvo {

constexpr int COV_MAX_PER_LANE = 31;   // kernel_size <= 31 -> <= 961 taps -> <= 31 per lane

struct CovParams {
    float fx, fy, cx, cy;
    int ksize;
    float min_depth_cov;
};

// gaussain_full_kernels' per-keypoint constants: the 2x2 inverse (the reference uses pinverse: identical for the
// non-singular matrices of this path) and the normalisation 2 pi sqrt(det)
struct Gauss2 {
    float i00, i11, i01, norm_c;
};

__device__ __forceinline__ Gauss2 gauss2(float suu, float svv, float suv) {
    const float det = __fsub_rn(__fmul_rn(suu, svv), __fmul_rn(suv, suv));
    const float idet = __frcp_rn(det);
    return Gauss2{__fmul_rn(svv, idet), __fmul_rn(suu, idet), -__fmul_rn(suv, idet), __fmul_rn(2.f * CUDART_PI_F, sqrtf(det))};
}

// unnormalised weight of tap (a, b): exp(-0.5 * [xa, yb] inv [xa, yb]^T) / (2 pi sqrt(det)). a runs along the kernel's
// x-axis (sigma_uu), which the reference pairs with the image ROW offset
__device__ __forceinline__ float gauss_tap(const Gauss2& g, int a, int b, int half) {
    const float xa = (float)(a - half), yb = (float)(b - half);
    const float quad = __fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(xa, xa), g.i00), __fmul_rn(__fmul_rn(2.f * xa, yb), g.i01)),
                                 __fmul_rn(__fmul_rn(yb, yb), g.i11));
    return __fdiv_rn(expf(-0.5f * quad), g.norm_c);
}

// pixel offset of tap (a, b) around (ul, vl) with python index semantics: a negative index wraps; -1 past the bottom /
// right edge (the reference raises IndexError there)
__device__ __forceinline__ long long tap_pixel(long long ul, long long vl, int a, int b, int half, int h, int w) {
    long long yy = vl + (a - half), xx = ul + (b - half);
    if (yy < 0) yy += h;
    if (xx < 0) xx += w;
    return (yy < 0 || yy >= h || xx < 0 || xx >= w) ? -1 : yy * w + xx;
}

// Covariance_2to3_full (Project2to3.py:377-424): s = [zz, xz, yz, xx, xy, yy] (NED order) of depth d, variance var
__device__ __forceinline__ void project_cov6(float u, float v, float d, float var, float suu, float svv, float suv,
                                             const CovParams& P, float s6[6]) {
    const float fx = P.fx, fy = P.fy;
    const float du = __fsub_rn(u, P.cx), dv = __fsub_rn(v, P.cy);
    const float d2 = __fmul_rn(d, d);
    s6[3] = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(du, du), var), __fmul_rn(d2, suu)),
                                __fmul_rn(suu, var)), __fmul_rn(fx, fx));                          // xx
    s6[5] = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(dv, dv), var), __fmul_rn(d2, svv)),
                                __fmul_rn(svv, var)), __fmul_rn(fy, fy));                          // yy
    s6[0] = var;                                                                                   // zz
    s6[4] = __fdiv_rn(__fadd_rn(__fmul_rn(__fmul_rn(du, dv), var),
                                __fmul_rn(__fadd_rn(d2, var), suv)), __fmul_rn(fx, fy));           // xy
    s6[1] = __fdiv_rn(__fmul_rn(var, du), fx);                                                     // xz
    s6[2] = __fdiv_rn(__fmul_rn(var, dv), fy);                                                     // yz
}

// MatchCovariance: one warp, Gaussian-weighted depth mean and variance around (ul, vl) + the 2D -> 3D projection.
// (suu, svv, suv) already clamped by the caller; override_var selects `wvar_depth = depth_cov`.
// Lane 0 receives the 6 unique entries s = [zz, xz, yz, xx, xy, yy] (NED order) in fp32; returns the warp-uniform
// out-of-image flag.
__device__ __forceinline__ bool match_cov_warp(float u, float v, long long ul, long long vl,
                                               const float* __restrict__ depth, int h, int w, float suu, float svv,
                                               float suv, bool override_var, float depth_var, const CovParams& P,
                                               int lane, float s6[6]) {
    const Gauss2 g = gauss2(suu, svv, suv);
    const int ksize = P.ksize, half = ksize / 2, taps = ksize * ksize;

    float z[COV_MAX_PER_LANE], pv[COV_MAX_PER_LANE];
    float zsum = 0.f;
    bool oob = false;
#pragma unroll
    for (int t = 0; t < COV_MAX_PER_LANE; ++t) {
        const int e = lane + 32 * t;
        z[t] = 0.f; pv[t] = 0.f;
        if (e < taps) {
            const int a = e / ksize, b = e - a * ksize;
            z[t] = gauss_tap(g, a, b, half);
            const long long p = tap_pixel(ul, vl, a, b, half, h, w);
            if (p < 0) oob = true;
            else pv[t] = __ldg(depth + p);
            zsum += z[t];
        }
    }
    zsum = warp_sum(zsum);
    float wavg = 0.f;
#pragma unroll
    for (int t = 0; t < COV_MAX_PER_LANE; ++t) {
        z[t] = __fdiv_rn(z[t], zsum);                               // normalised weights
        wavg = fmaf(z[t], pv[t], wavg);
    }
    wavg = warp_sum(wavg);
    float wvar = 0.f;
#pragma unroll
    for (int t = 0; t < COV_MAX_PER_LANE; ++t) {
        const float dd = pv[t] - wavg;
        wvar = fmaf(z[t], dd * dd, wvar);
    }
    wvar = warp_sum(wvar);
    // `wvar_depth = depth_cov` when no flow covariance is given but a per-keypoint depth variance is (Project2to3.py:163-171)
    if (override_var) wvar = depth_var;
    wvar = (wvar != wvar) ? wvar : fmaxf(wvar, P.min_depth_cov);        // clamp(min=...) keeps NaN
    oob = __any_sync(0xffffffffu, oob);
    project_cov6(u, v, wavg, wvar, suu, svv, suv, P, s6);
    return oob;
}

constexpr float MIXTURE_PROB_THRESHOLD = 1e-3f;   // gaussian_mixture_mean_var's prob_threshold (Utility/Math.py:66)

// GaussianMixtureCovariance (Project2to3.py:194-272): every tap is a Gaussian N(depth, depth_cov) weighted by the same
// filter as match_cov_warp; gaussian_mixture_mean_var (Utility/Math.py:66-93) drops weights below 1e-3 (NaN stays),
// renormalises, and takes mean = sum p d, var = (sum p (v + d^2) - mean^2) / 2 — the `/ 2` and the missing clamp on
// the variance (min_depth_cov is never read) are the reference's. Only the weights stay in registers: the depth and
// variance taps are read in the accumulation pass. Same result layout and out-of-image flag as match_cov_warp.
__device__ __forceinline__ bool mixture_cov_warp(float u, float v, long long ul, long long vl,
                                                 const float* __restrict__ depth, const float* __restrict__ dvar, int h,
                                                 int w, float suu, float svv, float suv, bool override_var,
                                                 float depth_var, const CovParams& P, int lane, float s6[6]) {
    const Gauss2 g = gauss2(suu, svv, suv);
    const int ksize = P.ksize, half = ksize / 2, taps = ksize * ksize;

    float z[COV_MAX_PER_LANE];
    float zsum = 0.f;
#pragma unroll
    for (int t = 0; t < COV_MAX_PER_LANE; ++t) {
        const int e = lane + 32 * t;
        z[t] = 0.f;
        if (e < taps) {
            const int a = e / ksize, b = e - a * ksize;
            z[t] = gauss_tap(g, a, b, half);
            zsum += z[t];
        }
    }
    zsum = warp_sum(zsum);
    float psum = 0.f;
#pragma unroll
    for (int t = 0; t < COV_MAX_PER_LANE; ++t) {
        const float p = __fdiv_rn(z[t], zsum);                      // gaussain_full_kernels' normalised weight
        z[t] = p < MIXTURE_PROB_THRESHOLD ? 0.f : p;
        psum += z[t];
    }
    psum = warp_sum(psum);
    float mean = 0.f, m2 = 0.f;
    bool oob = false;
#pragma unroll
    for (int t = 0; t < COV_MAX_PER_LANE; ++t) {
        const int e = lane + 32 * t;
        if (e < taps) {
            const int a = e / ksize, b = e - a * ksize;
            const long long pix = tap_pixel(ul, vl, a, b, half, h, w);
            float d = 0.f, var = 0.f;
            if (pix < 0) oob = true;
            else { d = __ldg(depth + pix); var = __ldg(dvar + pix); }
            const float p = __fdiv_rn(z[t], psum);                  // renormalised
            mean = fmaf(p, d, mean);
            m2 = fmaf(p, __fadd_rn(var, __fmul_rn(d, d)), m2);
        }
    }
    mean = warp_sum(mean);
    m2 = warp_sum(m2);
    float wvar = __fmul_rn(__fsub_rn(m2, __fmul_rn(mean, mean)), 0.5f);
    // `wvar_depth = depth_cov` when no flow covariance is given but a per-keypoint depth variance is (Project2to3.py:254-255)
    if (override_var) wvar = depth_var;
    oob = __any_sync(0xffffffffu, oob);
    project_cov6(u, v, mean, wvar, suu, svv, suv, P, s6);
    return oob;
}

// (K,3,3) float64 NED layout [[zz, xz, yz], [xz, xx, xy], [yz, xy, yy]]
__device__ __forceinline__ void store_cov9(double* o, const float s6[6]) {
    o[0] = s6[0]; o[1] = s6[1]; o[2] = s6[2];
    o[3] = s6[1]; o[4] = s6[3]; o[5] = s6[4];
    o[6] = s6[2]; o[7] = s6[4]; o[8] = s6[5];
}

}  // namespace macvo
