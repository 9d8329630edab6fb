// (f3) Observation building + outlier filter + MatchObs packing on the device.
//
// Replaces, for the two-frame pose graph, the per-frame host code between keypoint selection and the optimiser in
// Odometry/MACVO.py:198-270 (flow lookup, in-bound filter `filterPointsInRange`, nine `retrieve_pixels` gathers, two
// `ObsCovModel.estimate` calls, `pixel2point_NED`, `MatchObs.init`), the CovarianceSanityFilter
// (Module/OutlierFilter.py:91-100) and the point registration `pp.SE3.Act(prev_pose, pos0_Tc)` (:279-283), which the
// reference runs as ~14 device->host copies plus CPU tensor code per frame.
//
//   observe_kernel   one warp per selected keypoint: every gather, both 31x31 covariance estimates, the NaN / Inf
//                    sanity test and the world point, written to slot i of an uncompacted record table;
//   pack_kernel      one CTA: order-preserving compaction of the surviving records into (a) the float64
//                    structure-of-arrays the LM kernel reads (pgo.cu) and (b) the MatchObs columns the map wants,
//                    all inside ONE buffer so that a single asynchronous device->host copy ships a frame's
//                    observations; the survivor count stays on the device (pgo_lm_kernel reads it there).
//
// With a macvo_observe_ext_t another covariance model replaces MatchCovariance: NoCovariance (identity, no depth taps),
// GaussianMixtureCovariance (mixture_cov_warp on the depth and depth-covariance maps) and the Diagonalize / Normalize
// modifiers (cov_modify9, shared with macvo_cov_modify).
//
// Arithmetic: fp32 in the reference's operation order (explicit round-to-nearest intrinsics, no contraction), widened
// to fp64 exactly where the reference calls `.double()`.
#include "cov2to3.cuh"

namespace {

struct ObserveArgs {
    const int64_t* kp0;            // (k,2) [u,v] selected keypoints on frame 0
    int k;
    const float* flow;             // (2,h,w) match flow frame0 -> frame1
    const float* match_cov;        // (3,h,w) [uu, vv, uv], or nullptr with disp_unc1: a frontend without covariance
    const float* depth0;           // (h,w)
    const float* depth1;           // (h,w)
    const float* disparity1;       // (h,w)
    const float* disp_unc1;        // (h,w) or nullptr
    int h, w, edge;
    macvo::CovParams P0, P1;       // intrinsics of frame 0 / frame 1 + covariance-model parameters
    float min_flow_var, match_cov_default;
    const double* prev_pose;       // (7) [t, q_xyzw] optimised pose of frame 0 (device, float64)
    double* next_pose;             // (7) receives the motion-model prediction for frame 1 (= prev pose, fp32-rounded)
    // macvo_observe_ext_t (ext == 0: none of this is read or written)
    int ext, simple_depth, front_of_cam;
    float min_depth, max_depth;
    const float* depth_cov0;       // (h,w) or nullptr (-1 placeholder)
    const float* depth_cov1;
    float* rex;                    // (k, REX) extension records
    int identity;                  // NoCovariance: no depth taps, raw uv covariances, identity 3x3 covariances
    int mixture;                   // GaussianMixtureCovariance: depth_cov0 / depth_cov1 are the variance patches
    int n_ops, op0, op1;           // covariance modifiers, op0 first
    double* rcov;                  // (k, RCOV) modified covariances (n_ops > 0 only)
};

// record slot (floats): 0 keep | 1,2 kp1 uv | 3 depth0 | 4 disp1 | 5 disp_unc1 | 6..8 uv cov (clamped) | 9..11 pos_Tw |
//                       12..17 cov0 (6 unique) | 18..23 cov1 (6 unique) | 24 inbound
constexpr int REC = 25;
// extension record (ext only): 0 pixel2_d | 1 pixel1_d_cov | 2 pixel2_d_cov | 3 LikelyFrontOfCam verdict | 4..6 points_Tc
constexpr int REX = 7;
// modified-covariance record (float64, only with modifiers): 0..8 cov0 (3,3) | 9..17 cov1 (3,3).
// A modified covariance is float64 and no longer fits the fp32 record. observe_kernel, which needs it for the keep decision
// anyway, stores it here and pack_kernel copies it: recomputing the LU in pack_kernel (1024 threads, so at most 64
// registers) spills, and the keep decision and the packed values are then the same numbers by construction.
constexpr int RCOV = 18;
static_assert((REC + REX) % 2 == 0, "the float64 records after the fp32 ones must stay 8-byte aligned");

__device__ __forceinline__ bool bad6(const float* s) {
    bool b = false;
#pragma unroll
    for (int i = 0; i < 6; ++i) b |= !isfinite(s[i]);
    return b;
}

__device__ __forceinline__ bool bad9(const double* m) {
    bool b = false;
#pragma unroll
    for (int i = 0; i < 9; ++i) b |= !isfinite(m[i]);
    return b;
}

// torch.det of a 3x3 float64 matrix as an LU factorisation with partial pivoting: pivot = largest |a| of the column (the
// first on ties; a NaN is never preferred), multipliers by division (a zero pivot leaves its column unscaled, like LAPACK's
// getrf, and the trailing update still runs); det = sign * u00 * u11 * u22 (the product of the diagonal, then the sign)
// CPU torch.det hands the row-major matrix to column-major LAPACK, so it factors the TRANSPOSE (det A^T = det A); so does
// this routine, which makes the NaN / Inf / signed-zero class of the result agree with it, not only its value
__device__ __forceinline__ double det3_lu(const double* m) {
    double a[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) a[e] = m[3 * (e % 3) + e / 3];
    double sign = 1.0;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        int p = j;
        double best = fabs(a[3 * j + j]);
#pragma unroll
        for (int i = j + 1; i < 3; ++i)
            if (fabs(a[3 * i + j]) > best) { best = fabs(a[3 * i + j]); p = i; }
        if (p != j) sign = -sign;
#pragma unroll
        for (int i = j + 1; i < 3; ++i)             // row swap with constant indices only: the matrix stays in registers
            if (p == i) {
#pragma unroll
                for (int c = j; c < 3; ++c) { const double t = a[3 * j + c]; a[3 * j + c] = a[3 * i + c]; a[3 * i + c] = t; }
            }
        const double piv = a[3 * j + j];
#pragma unroll
        for (int i = j + 1; i < 3; ++i) {
            const double l = piv != 0.0 ? __ddiv_rn(a[3 * i + j], piv) : a[3 * i + j];
#pragma unroll
            for (int c = j + 1; c < 3; ++c) a[3 * i + c] = __dsub_rn(a[3 * i + c], __dmul_rn(l, a[3 * j + c]));
        }
    }
    return __dmul_rn(__dmul_rn(__dmul_rn(a[0], a[4]), a[8]), sign);
}

// The covariance modifiers (Project2to3.py:281-323) on one (3,3) float64 matrix, ops[0] first (the innermost wrapper).
// observe_kernel (keep decision), pack_kernel (the packed columns, cov_Tw) and macvo_cov_modify all call this one routine.
__device__ __forceinline__ void cov_modify9(double* m, int n_ops, int op0, int op1) {
    for (int o = 0; o < n_ops; ++o) {
        const int op = o == 0 ? op0 : op1;
        if (op == MACVO_COV_DIAGONALIZE) {
            m[1] = m[2] = m[3] = m[5] = m[6] = m[7] = 0.0;
        } else {                                                     // MACVO_COV_NORMALIZE: covs /= det(covs)
            const double det = det3_lu(m);
#pragma unroll
            for (int e = 0; e < 9; ++e) m[e] = __ddiv_rn(m[e], det);
        }
    }
}

// the base model's six fp32 entries, widened, then the modifiers
__device__ __forceinline__ void modified_cov9(double* m, const float* s6, int n_ops, int op0, int op1) {
    macvo::store_cov9(m, s6);
    cov_modify9(m, n_ops, op0, op1);
}

__global__ void __launch_bounds__(128)
observe_kernel(ObserveArgs A, float* __restrict__ rec, int* __restrict__ status) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x < 7) {
        // StaticMotionModel.predict: est_pose = previous pose; the map stores poses in fp32 (Module/Map: FrameNode "pose")
        A.next_pose[threadIdx.x] = (double)(float)A.prev_pose[threadIdx.x];
    }
    if (i >= A.k) return;
    const long long u0 = A.kp0[2 * i], v0 = A.kp0[2 * i + 1];
    const int hw = A.h * A.w;
    float* r = rec + (long long)i * REC;
    const bool in0 = u0 >= 0 && u0 < A.w && v0 >= 0 && v0 < A.h;
    if (!in0) {                                  // cannot happen for selector output; keep the table defined
        if (lane == 0) { r[0] = 0.f; r[24] = 0.f; atomicOr(status, 2); }
        return;
    }
    const int p0 = (int)(v0 * A.w + u0);
    // kp1 = kp0 + flow[kp0]   (int64 + fp32 -> fp32)
    const float u1 = __fadd_rn((float)u0, A.flow[p0]);
    const float v1 = __fadd_rn((float)v0, A.flow[hw + p0]);
    // filterPointsInRange: strict inequalities against python ints
    const bool inb = (u1 < (float)(A.w - A.edge)) && (u1 > (float)A.edge) && (v1 < (float)(A.h - A.edge)) && (v1 > (float)A.edge);
    if (!inb) {
        if (lane == 0) { r[0] = 0.f; r[24] = 0.f; }
        return;
    }
    const long long ul1 = (long long)u1, vl1 = (long long)v1;         // .long(): truncation
    const int p1 = (int)(vl1 * A.w + ul1);                            // inside the image: edge > 0
    const float d0 = A.depth0[p0];
    // no covariance maps (MACVO.py:250-264): MatchObs holds the -1 placeholder in pixel2_uv_cov and pixel2_disp_cov
    const bool no_cov = A.match_cov == nullptr;
    const float disp1 = A.disparity1[p1], dunc1 = no_cov ? -1.f : A.disp_unc1[p1];
    float c0[6], c1[6];
    const float a = no_cov ? -1.f : A.match_cov[p0], b = no_cov ? -1.f : A.match_cov[hw + p0];
    const float suv = no_cov ? -1.f : A.match_cov[2 * hw + p0];
    float suu, svv;
    bool oob = false;
    if (A.identity) {
        // NoCovariance.estimate (Project2to3.py:52-54): identity, no patch read, flow_cov left as the network gave it
        if (lane != 0) return;
        suu = a; svv = b;
#pragma unroll
        for (int e = 0; e < 6; ++e) c0[e] = c1[e] = (e == 0 || e == 3 || e == 5) ? 1.f : 0.f;
    } else {
        // the covariance estimate of one frame's keypoint: MatchCovariance, or GaussianMixtureCovariance on that frame's
        // depth-covariance map
        auto estimate = [&](float u, float v, long long ul, long long vl, const float* depth, const float* dvar, float su,
                            float sv, float suv_, bool override_var, float depth_var, const macvo::CovParams& P, float* s6) {
            return A.mixture ? macvo::mixture_cov_warp(u, v, ul, vl, depth, dvar, A.h, A.w, su, sv, suv_, override_var,
                                                       depth_var, P, lane, s6)
                             : macvo::match_cov_warp(u, v, ul, vl, depth, A.h, A.w, su, sv, suv_, false, 0.f, P, lane, s6);
        };
        // frame-0 keypoints: constant quantisation covariance, clamped like any flow_cov (Project2to3.py:130-133)
        const float s0 = fmaxf(A.match_cov_default, A.min_flow_var);
        oob = estimate((float)u0, (float)v0, u0, v0, A.depth0, A.depth_cov0, s0, s0, 0.f, false, 0.f, A.P0, c0);
        if (no_cov) {
            // frame-1 keypoints without a network covariance: the model's own default, NOT clamped
            // (Project2to3.py:128-135, 212-218); the packed column keeps the placeholder. The mixture then takes kp1's
            // depth_cov as its variance (Project2to3.py:254-255)
            const float s1 = A.match_cov_default;
            oob |= estimate(u1, v1, ul1, vl1, A.depth1, A.depth_cov1, s1, s1, 0.f, true, A.mixture ? A.depth_cov1[p1] : 0.f,
                            A.P1, c1);
            suu = svv = -1.f;
        } else {
            // frame-1 keypoints: the network's match covariance at the source pixel, clamped in place
            suu = (a != a) ? a : fmaxf(a, A.min_flow_var);
            svv = (b != b) ? b : fmaxf(b, A.min_flow_var);
            oob |= estimate(u1, v1, ul1, vl1, A.depth1, A.depth_cov1, suu, svv, suv, false, 0.f, A.P1, c1);
        }
        if (lane != 0) return;
    }
    if (oob) atomicOr(status, 1);                // status is a bitmask: both conditions may occur in one call
    // CovarianceSanityFilter: drop observations with NaN / Inf covariance on either frame, after the modifiers
    bool keep;
    if (A.n_ops == 0) {
        keep = !(bad6(c0) || bad6(c1));
    } else {
        double m[9];
        double* w = A.rcov + (long long)i * RCOV;
        modified_cov9(m, c0, A.n_ops, A.op0, A.op1);
        keep = !bad9(m);
#pragma unroll
        for (int e = 0; e < 9; ++e) w[e] = m[e];
        modified_cov9(m, c1, A.n_ops, A.op0, A.op1);
        keep &= !bad9(m);
#pragma unroll
        for (int e = 0; e < 9; ++e) w[9 + e] = m[e];
    }
    if (A.ext) {
        // Module/OutlierFilter.py:106-141 in fp32 on the MatchObs columns (MACVO.py:205-248 gathers)
        const float d1 = A.depth1[p1];
        const float dc0 = A.depth_cov0 ? A.depth_cov0[p0] : -1.f, dc1 = A.depth_cov1 ? A.depth_cov1[p1] : -1.f;
        // SimpleDepthFilter: ordered comparisons are false for NaN, so a NaN depth passes
        if (A.simple_depth)
            keep &= !(d0 < A.min_depth || d0 > A.max_depth || d1 < A.min_depth || d1 > A.max_depth);
        // LikelyFrontOfCamFilter: d - sqrt(d_cov) * 2 > 0 on both frames; pack_kernel applies it unless a placeholder
        // pixel1_d_cov == -1 exists among the in-bound rows
        const bool front = __fsub_rn(d0, __fmul_rn(__fsqrt_rn(dc0), 2.f)) > 0.f &&
                           __fsub_rn(d1, __fmul_rn(__fsqrt_rn(dc1), 2.f)) > 0.f;
        float* x = A.rex + (long long)i * REX;
        x[0] = d1; x[1] = dc0; x[2] = dc1; x[3] = front ? 1.f : 0.f;
        // ICP_TwoframePGO's points_Tc = pixel2point_NED(pixel2_uv, pixel2_d, K1) (Graphs.py:49-51)
        x[4] = d1;
        x[5] = __fmul_rn(__fdiv_rn(__fsub_rn(u1, A.P1.cx), A.P1.fx), d1);
        x[6] = __fmul_rn(__fdiv_rn(__fsub_rn(v1, A.P1.cy), A.P1.fy), d1);
    }
    // pixel2point_NED (Utility/Point.py:15-17): [d, (u - cx) / fx * d, (v - cy) / fy * d]
    const float px = d0;
    const float py = __fmul_rn(__fdiv_rn(__fsub_rn((float)u0, A.P0.cx), A.P0.fx), d0);
    const float pz = __fmul_rn(__fdiv_rn(__fsub_rn((float)v0, A.P0.cy), A.P0.fy), d0);
    // SE3.Act in fp32: p + w * (2 q_v x p) + q_v x (2 q_v x p) + t
    const float tx = (float)A.prev_pose[0], ty = (float)A.prev_pose[1], tz = (float)A.prev_pose[2];
    const float qx = (float)A.prev_pose[3], qy = (float)A.prev_pose[4], qz = (float)A.prev_pose[5], qw = (float)A.prev_pose[6];
    const float ax = __fmul_rn(2.f, __fsub_rn(__fmul_rn(qy, pz), __fmul_rn(qz, py)));
    const float ay = __fmul_rn(2.f, __fsub_rn(__fmul_rn(qz, px), __fmul_rn(qx, pz)));
    const float az = __fmul_rn(2.f, __fsub_rn(__fmul_rn(qx, py), __fmul_rn(qy, px)));
    const float bx = __fsub_rn(__fmul_rn(qy, az), __fmul_rn(qz, ay));
    const float by = __fsub_rn(__fmul_rn(qz, ax), __fmul_rn(qx, az));
    const float bz = __fsub_rn(__fmul_rn(qx, ay), __fmul_rn(qy, ax));
    r[0] = keep ? 1.f : 0.f;
    r[1] = u1; r[2] = v1; r[3] = d0; r[4] = disp1; r[5] = dunc1;
    r[6] = suu; r[7] = svv; r[8] = suv;
    r[9] = __fadd_rn(__fadd_rn(__fadd_rn(px, __fmul_rn(qw, ax)), bx), tx);
    r[10] = __fadd_rn(__fadd_rn(__fadd_rn(py, __fmul_rn(qw, ay)), by), ty);
    r[11] = __fadd_rn(__fadd_rn(__fadd_rn(pz, __fmul_rn(qw, az)), bz), tz);
#pragma unroll
    for (int e = 0; e < 6; ++e) { r[12 + e] = c0[e]; r[18 + e] = c1[e]; }
    r[24] = 1.f;
}

struct PackExt {
    int on, front_of_cam, icp;
    const float* rex;
    const double* prev_pose;
    const double* rcov;            // observe_kernel's modified covariances, or nullptr (no modifier)
};

// packed float64 buffer, sections sized by the CAPACITY cap (fixed pointers for the LM kernel):
//   [0,3c) pos_Tw | [3c,5c) kp2 uv | [5c,6c) kp2 disp | [6c,9c) uv cov | [9c,10c) disp cov          <- pgo.cu inputs
//   [10c,19c) obs1_covTc (c,3,3) | [19c,28c) obs2_covTc (c,3,3) | [28c,30c) pixel1_uv | [30c,31c) pixel1_d
//   [31c,31c+4) header: n_obs, n_inbound, k, status
// with the icp extension, after the header (E = 31c+4):
//   [E,E+c) pixel2_d | [E+c,E+2c) pixel1_d_cov | [E+2c,E+3c) pixel2_d_cov | [E+3c,E+6c) points_Tc | [E+6c,E+15c) cov_Tw
__global__ void __launch_bounds__(1024)
pack_kernel(const float* __restrict__ rec, const int64_t* __restrict__ kp0, int k, int cap, double* __restrict__ out,
            int* __restrict__ n_obs, const int* __restrict__ status, PackExt X) {
    __shared__ int s_warp[32];
    __shared__ int s_base, s_inb;
    __shared__ double s_R[9];
    if (threadIdx.x == 0) { s_base = 0; s_inb = 0; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long c = cap;
    bool front_all = false;
    if (X.on) {
        if (X.icp && threadIdx.x == 0) {
            // pp.SE3(fp32 pose).rotation().matrix() in fp32, then .to(torch.float64) (MACVO.py:274-275)
            const float qx = (float)X.prev_pose[3], qy = (float)X.prev_pose[4], qz = (float)X.prev_pose[5],
                        qw = (float)X.prev_pose[6];
            const float xx = __fmul_rn(qx, qx), yy = __fmul_rn(qy, qy), zz = __fmul_rn(qz, qz);
            const float xy = __fmul_rn(qx, qy), xz = __fmul_rn(qx, qz), yz = __fmul_rn(qy, qz);
            const float xw = __fmul_rn(qx, qw), yw = __fmul_rn(qy, qw), zw = __fmul_rn(qz, qw);
            s_R[0] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(yy, zz)));
            s_R[1] = __fmul_rn(2.f, __fsub_rn(xy, zw));
            s_R[2] = __fmul_rn(2.f, __fadd_rn(xz, yw));
            s_R[3] = __fmul_rn(2.f, __fadd_rn(xy, zw));
            s_R[4] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, zz)));
            s_R[5] = __fmul_rn(2.f, __fsub_rn(yz, xw));
            s_R[6] = __fmul_rn(2.f, __fsub_rn(xz, yw));
            s_R[7] = __fmul_rn(2.f, __fadd_rn(yz, xw));
            s_R[8] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, yy)));
        }
        // LikelyFrontOfCamFilter passes every row when any in-bound row holds the -1 placeholder (OutlierFilter.py:130-133)
        int ph = 0;
        if (X.front_of_cam)
            for (int i = threadIdx.x; i < k; i += 1024)
                ph |= rec[(long long)i * REC + 24] != 0.f && X.rex[(long long)i * REX + 1] == -1.f;
        front_all = __syncthreads_or(ph) != 0 || !X.front_of_cam;
    }
    __syncthreads();
    for (int start = 0; start < k; start += 1024) {
        const int i = start + threadIdx.x;
        const float* r = rec + (long long)i * REC;
        const float* x = X.rex + (long long)i * REX;
        const bool keep = i < k && r[0] != 0.f && (!X.on || front_all || x[3] != 0.f);
        const bool inb = i < k && r[24] != 0.f;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        const unsigned bal_in = __ballot_sync(0xffffffffu, inb);
        if (lane == 0) { s_warp[warp] = __popc(bal); if (bal_in) atomicAdd(&s_inb, __popc(bal_in)); }
        __syncthreads();
        int off = 0, tot = 0;
        for (int wv = 0; wv < 32; ++wv) { if (wv < warp) off += s_warp[wv]; tot += s_warp[wv]; }
        const int j = s_base + off + __popc(bal & ((1u << lane) - 1));
        if (keep && j < cap) {
            out[3 * j] = r[9]; out[3 * j + 1] = r[10]; out[3 * j + 2] = r[11];
            out[3 * c + 2 * j] = r[1]; out[3 * c + 2 * j + 1] = r[2];
            out[5 * c + j] = r[4];
            out[6 * c + 3 * j] = r[6]; out[6 * c + 3 * j + 1] = r[7]; out[6 * c + 3 * j + 2] = r[8];
            out[9 * c + j] = r[5];
            if (!X.rcov) {
                macvo::store_cov9(out + 10 * c + 9LL * j, r + 12);
                macvo::store_cov9(out + 19 * c + 9LL * j, r + 18);
            } else {
                const double* m = X.rcov + (long long)i * RCOV;
#pragma unroll
                for (int e = 0; e < 9; ++e) { out[10 * c + 9LL * j + e] = m[e]; out[19 * c + 9LL * j + e] = m[9 + e]; }
            }
            out[28 * c + 2 * j] = (double)kp0[2 * i]; out[28 * c + 2 * j + 1] = (double)kp0[2 * i + 1];
            out[30 * c + j] = r[3];
            if (X.icp) {
                double* e = out + 31 * c + 4;
                e[j] = x[0]; e[c + j] = x[1]; e[2 * c + j] = x[2];
                e[3 * c + 3 * j] = x[4]; e[3 * c + 3 * j + 1] = x[5]; e[3 * c + 3 * j + 2] = x[6];
                // cov_Tw = R obs1_covTc R^T in float64 (torch.bmm(torch.bmm(R, cov), R^T), MACVO.py:280)
                double C[9], RC[9];                                 // obs1_covTc as packed above (modifiers applied)
                if (!X.rcov) {
                    macvo::store_cov9(C, r + 12);
                } else {
#pragma unroll
                    for (int e = 0; e < 9; ++e) C[e] = X.rcov[(long long)i * RCOV + e];
                }
#pragma unroll
                for (int a = 0; a < 3; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b)
                        RC[3 * a + b] = s_R[3 * a] * C[b] + s_R[3 * a + 1] * C[3 + b] + s_R[3 * a + 2] * C[6 + b];
                double* o = e + 6 * c + 9LL * j;
#pragma unroll
                for (int a = 0; a < 3; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b)
                        o[3 * a + b] = RC[3 * a] * s_R[3 * b] + RC[3 * a + 1] * s_R[3 * b + 1] + RC[3 * a + 2] * s_R[3 * b + 2];
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) s_base += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int n = min(s_base, cap);
        *n_obs = n;
        out[31 * c] = n; out[31 * c + 1] = s_inb; out[31 * c + 2] = k; out[31 * c + 3] = *status;
    }
}

// CovarianceSanityFilter.filter (Module/OutlierFilter.py:91-100) for device-resident covariances: one thread per observation
__global__ void cov_sanity_kernel(const double* __restrict__ c1, const double* __restrict__ c2, int k, uint8_t* __restrict__ good) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    bool ok = true;
#pragma unroll
    for (int e = 0; e < 9; ++e) ok &= isfinite(c1[9LL * i + e]) && isfinite(c2[9LL * i + e]);
    good[i] = ok ? 1 : 0;
}

// macvo_cov_modify: one thread per (3,3) matrix, in place
__global__ void cov_modify_kernel(double* __restrict__ cov, int k, int n_ops, int op0, int op1) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    double m[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) m[e] = cov[9LL * i + e];
    cov_modify9(m, n_ops, op0, op1);
#pragma unroll
    for (int e = 0; e < 9; ++e) cov[9LL * i + e] = m[e];
}

bool valid_cov_ops(const int* ops, int n_ops) {
    if (n_ops < 0 || n_ops > MACVO_COV_MAX_OPS || (n_ops > 0 && !ops)) return false;
    for (int o = 0; o < n_ops; ++o)
        if (ops[o] != MACVO_COV_DIAGONALIZE && ops[o] != MACVO_COV_NORMALIZE) return false;
    return true;
}

}  // namespace

extern "C" int macvo_cov_modify(double* cov, int k, const int* ops, int n_ops, void* stream) {
    if (k < 0 || !valid_cov_ops(ops, n_ops)) return MACVO_E_ARG;
    if (k == 0 || n_ops == 0) return MACVO_OK;
    if (!cov) return MACVO_E_ARG;
    cov_modify_kernel<<<ceil_div(k, 256), 256, 0, as_stream(stream)>>>(cov, k, n_ops, ops[0], n_ops > 1 ? ops[1] : 0);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_cov_sanity_filter(const double* obs1_cov, const double* obs2_cov, int k, uint8_t* good, void* stream) {
    if (k < 0) return MACVO_E_ARG;
    if (k == 0) return MACVO_OK;
    if (!obs1_cov || !obs2_cov || !good) return MACVO_E_ARG;
    cov_sanity_kernel<<<ceil_div(k, 256), 256, 0, as_stream(stream)>>>(obs1_cov, obs2_cov, k, good);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" size_t macvo_observe_workspace_bytes(int capacity) {
    // the fp32 records, then the float64 modified covariances
    return (size_t)capacity * ((REC + REX) * sizeof(float) + RCOV * sizeof(double));
}

extern "C" size_t macvo_observe_packed_doubles(int capacity, int extended) {
    return (size_t)(extended ? 46 : 31) * capacity + 4;
}

extern "C" int macvo_observe_pack(const int64_t* kp0_uv, int k, int capacity, const float* flow, const float* match_cov,
                                  const float* depth0, const float* depth1, const float* disparity1,
                                  const float* disp_unc1, int h, int w, int edge_width, const float* intr0,
                                  const float* intr1, int kernel_size, float min_flow_cov, float min_depth_cov,
                                  float match_cov_default, const double* prev_pose, double* next_pose, double* packed,
                                  int* n_obs, int* status, void* workspace, size_t workspace_bytes, void* stream,
                                  const macvo_observe_ext_t* ext) {
    if (k < 0 || capacity < 1 || k > capacity || h <= 0 || w <= 0 || edge_width <= 0 || kernel_size < 1 ||
        (kernel_size & 1) == 0 || kernel_size > 31)
        return MACVO_E_ARG;
    // match_cov and disp_unc1 are NULL together (a frontend without covariance) or not at all
    if (!match_cov != !disp_unc1) return MACVO_E_ARG;
    if (!flow || !depth0 || !depth1 || !disparity1 || !intr0 || !intr1 || !prev_pose ||
        !next_pose || !packed || !n_obs || !status || !workspace || (k > 0 && !kp0_uv))
        return MACVO_E_ARG;
    if (workspace_bytes < macvo_observe_workspace_bytes(capacity)) return MACVO_E_WORKSPACE;
    if (ext && ext->simple_depth && !(ext->min_depth <= ext->max_depth)) return MACVO_E_ARG;
    if (ext && ((ext->cov_model != MACVO_COV_MATCH && ext->cov_model != MACVO_COV_IDENTITY &&
                 ext->cov_model != MACVO_COV_GAUSSIAN_MIXTURE) ||
                !valid_cov_ops(ext->cov_ops, ext->n_cov_ops)))
        return MACVO_E_ARG;
    // GaussianMixtureCovariance asserts depth_est.cov is not None (Project2to3.py:206)
    if (ext && ext->cov_model == MACVO_COV_GAUSSIAN_MIXTURE && (!ext->depth_cov0 || !ext->depth_cov1)) return MACVO_E_ARG;
    ObserveArgs A;
    A.kp0 = kp0_uv; A.k = k; A.flow = flow; A.match_cov = match_cov; A.depth0 = depth0; A.depth1 = depth1;
    A.disparity1 = disparity1; A.disp_unc1 = disp_unc1; A.h = h; A.w = w; A.edge = edge_width;
    A.P0 = macvo::CovParams{intr0[0], intr0[1], intr0[2], intr0[3], kernel_size, min_depth_cov};   // HOST {fx, fy, cx, cy}
    A.P1 = macvo::CovParams{intr1[0], intr1[1], intr1[2], intr1[3], kernel_size, min_depth_cov};
    A.min_flow_var = min_flow_cov * min_flow_cov;
    A.match_cov_default = match_cov_default;
    A.prev_pose = prev_pose; A.next_pose = next_pose;
    float* rec = static_cast<float*>(workspace);
    A.ext = ext != nullptr;
    A.simple_depth = ext && ext->simple_depth; A.front_of_cam = ext && ext->front_of_cam;
    A.min_depth = ext ? ext->min_depth : 0.f; A.max_depth = ext ? ext->max_depth : 0.f;
    A.depth_cov0 = ext ? ext->depth_cov0 : nullptr; A.depth_cov1 = ext ? ext->depth_cov1 : nullptr;
    A.rex = rec + (size_t)capacity * REC;
    A.identity = ext && ext->cov_model == MACVO_COV_IDENTITY;
    A.mixture = ext && ext->cov_model == MACVO_COV_GAUSSIAN_MIXTURE;
    A.n_ops = ext ? ext->n_cov_ops : 0;
    A.op0 = A.n_ops > 0 ? ext->cov_ops[0] : 0;
    A.op1 = A.n_ops > 1 ? ext->cov_ops[1] : 0;
    A.rcov = reinterpret_cast<double*>(A.rex + (size_t)capacity * REX);
    PackExt X{A.ext, A.front_of_cam, ext && ext->icp, A.rex, prev_pose, A.n_ops > 0 ? A.rcov : nullptr};
    cudaStream_t st = as_stream(stream);
    observe_kernel<<<max(1, ceil_div(k * 32, 128)), 128, 0, st>>>(A, rec, status);
    MACVO_LAUNCH_CHECK();
    pack_kernel<<<1, 1024, 0, st>>>(rec, kp0_uv, k, capacity, packed, n_obs, status, X);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
