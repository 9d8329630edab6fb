// (a14)+(a15) covariance-weighted two-frame pose-graph optimisation, fp64, fully on the device.
//
// Replaces TwoFrame_PGO._optimize (Module/Optimization/TwoFramePGO/Optimizer.py:82-102): the LM_analytic
// step loop (Module/Optimization/PyposeOptimizers.py:160-194) over Analytic_ReprojDisp_TwoFramePGO
// (Module/Optimization/TwoFramePGO/Graphs.py:121-148 residual / covariance, :201-230 Jacobian) with
// pypose's Huber(0.1) kernel, FastTriggs corrector, PINV solver, TrustRegion(radius=1e3) strategy and
// StopOnPlateau(steps=10, patience=2, decreasing=1e-5) scheduler. The reference builds a dense
// 3K x 3K block-diagonal weight every step (1.2 GB at K = 4096) on the CPU; here every residual block keeps
// its own 3x3 information matrix and the whole loop is ONE persistent launch.
//
// Kernel shape (north_star: "warp-per-residual-block kernel with a tree reduction into the 6x6 system"):
//   * a thread-block cluster of 1..8 CTAs x 8 warps; residual block k is owned by global warp k % nwarps;
//   * linearisation: the warp evaluates r (3), J (3x6, the reference's 7th column is identically zero),
//     W = Sigma^-1, the FastTriggs scale s, stages s*J, W*s*J, s*r in shared memory, then lane e
//     accumulates entry e of the packed system  [A = Js^T W Js (21) | b = -Js^T W Rs (6) |
//     G = Js^T Js (21) | h = Js^T Rs (6) | robust loss (1)]  (55 entries, 2 per lane) in registers;
//   * reduction: fixed-order tree — per-warp registers -> shared memory -> per-CTA partial -> distributed
//     shared memory of the cluster -> every CTA sums the partials in rank order, so all CTAs hold the
//     same bits and run the (tiny) 6x6 solve / trust-region / accept-reject logic redundantly;
//   * loss-only evaluations use one LANE per residual block.
// Latency bound (80*K bytes per evaluation, SURVEY.md §8d): what matters is zero host round trips.
#include "common.cuh"
#include <cooperative_groups.h>
#include <math_constants.h>
#include <cstring>

namespace cg = cooperative_groups;

namespace {

constexpr int NACC = MACVO_PGO_ACC;      // 55
constexpr int WARPS = 8, THREADS = WARPS * 32;

struct Intr { double fx, fy, cx, cy, bl; };

struct Pose {            // SE3 as rotation matrix (row-major) + translation, derived from [t, q_xyzw]
    double R[9], t[3];
};

__device__ __forceinline__ void pose_from_vec(const double* p, Pose& o) {
    const double x = p[3], y = p[4], z = p[5], w = p[6];
    o.R[0] = 1 - 2 * (y * y + z * z); o.R[1] = 2 * (x * y - z * w);     o.R[2] = 2 * (x * z + y * w);
    o.R[3] = 2 * (x * y + z * w);     o.R[4] = 1 - 2 * (x * x + z * z); o.R[5] = 2 * (y * z - x * w);
    o.R[6] = 2 * (x * z - y * w);     o.R[7] = 2 * (y * z + x * w);     o.R[8] = 1 - 2 * (x * x + y * y);
    o.t[0] = p[0]; o.t[1] = p[1]; o.t[2] = p[2];
}

// p_c = T^-1 p_w = R^T (p_w - t)
__device__ __forceinline__ void to_camera(const Pose& T, const double* pw, double* pc) {
    const double d0 = pw[0] - T.t[0], d1 = pw[1] - T.t[1], d2 = pw[2] - T.t[2];
    pc[0] = T.R[0] * d0 + T.R[3] * d1 + T.R[6] * d2;
    pc[1] = T.R[1] * d0 + T.R[4] * d1 + T.R[7] * d2;
    pc[2] = T.R[2] * d0 + T.R[5] * d1 + T.R[8] * d2;
}

// r = [fx y/x + cx - u, fy z/x + cy - v, fx bl / x - disp]   (NED camera frame: x forward)
__device__ __forceinline__ void residual3(const Intr& K, const double* pc, double u, double v, double disp, double* r) {
    const double ix = 1.0 / pc[0];
    r[0] = K.fx * pc[1] * ix + K.cx - u;
    r[1] = K.fy * pc[2] * ix + K.cy - v;
    r[2] = ix * (K.fx * K.bl) - disp;
}

__device__ __forceinline__ double huber(double x, double delta) {        // on the SQUARED norm
    const double s = sqrt(x);
    return s < delta ? x : 2.0 * delta * s - delta * delta;
}

// torch.pinverse / np.linalg.pinv keep the singular values above this fraction of the largest one
constexpr double PINV_RCOND = 1e-15;

// one Jacobi rotation of the symmetric 3x3 `a` that zeroes a[p][q] (r is the third index); v accumulates the rotations
__device__ __forceinline__ void jacobi_rotate(double (&a)[3][3], double (&v)[3][3], int p, int q, int r) {
    const double apq = a[p][q];
    if (apq == 0.0) return;
    const double g = 100.0 * fabs(apq), app = a[p][p], aqq = a[q][q], h = aqq - app;
    if (fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) { a[p][q] = a[q][p] = 0.0; return; }   // below rounding
    double t;
    if (fabs(h) + g == fabs(h)) t = apq / h;
    else {
        const double th = 0.5 * h / apq;
        t = 1.0 / (fabs(th) + sqrt(th * th + 1.0));
        if (th < 0.0) t = -t;
    }
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
    a[p][p] = app - t * apq; a[q][q] = aqq + t * apq; a[p][q] = a[q][p] = 0.0;
    const double arp = a[r][p], arq = a[r][q];
    a[r][p] = a[p][r] = arp - s * (arq + arp * tau);
    a[r][q] = a[q][r] = arq + s * (arp - arq * tau);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double vp = v[i][p], vq = v[i][q];
        v[i][p] = vp - s * (vq + vp * tau);
        v[i][q] = vq + s * (vp - vq * tau);
    }
}

// Moore-Penrose inverse of the symmetric 3x3 [[m00 m01 m02] [. m11 m12] [. . m22]] by cyclic Jacobi: sum of v v^T / lambda
// over the eigenvalues with |lambda| > PINV_RCOND * max |lambda| (torch.pinverse of a symmetric matrix). Returns true when an
// eigenvalue was dropped.
__device__ bool sym3_pinv(double m00, double m01, double m02, double m11, double m12, double m22,
                          double& w00, double& w01, double& w02, double& w11, double& w12, double& w22) {
    double a[3][3] = {{m00, m01, m02}, {m01, m11, m12}, {m02, m12, m22}};
    double v[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    for (int sweep = 0; sweep < 32 && (a[0][1] != 0.0 || a[0][2] != 0.0 || a[1][2] != 0.0); ++sweep) {
        jacobi_rotate(a, v, 0, 1, 2);
        jacobi_rotate(a, v, 0, 2, 1);
        jacobi_rotate(a, v, 1, 2, 0);
    }
    const double lmax = fmax(fabs(a[0][0]), fmax(fabs(a[1][1]), fabs(a[2][2])));
    w00 = w01 = w02 = w11 = w12 = w22 = 0.0;
    bool dropped = false;
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const double l = a[e][e];
        if (!(fabs(l) > PINV_RCOND * lmax)) { dropped = true; continue; }
        const double il = 1.0 / l, x = v[0][e], y = v[1][e], z = v[2][e];
        w00 += x * x * il; w01 += x * y * il; w02 += x * z * il;
        w11 += y * y * il; w12 += y * z * il; w22 += z * z * il;
    }
    return dropped;
}

__device__ __forceinline__ int tri_index(int e, int& i, int& j) {        // upper-triangular (i <= j) of a 6x6, row-major
    int row = 0, rem = e;
    while (rem >= 6 - row) { rem -= 6 - row; ++row; }
    i = row; j = row + rem;
    return 0;
}

struct Shared {
    double part[NACC];             // this CTA's partial (read by the other CTAs of the cluster through DSMEM)
    double warp_acc[WARPS][NACC];
    double total[NACC];
    double sJ[WARPS][18], sWJ[WARPS][18], sR[WARPS][3], sWR[WARPS][3];
    double pose[7], trial[7];
    double Rm[9];                  // rotation matrix of the linearisation pose (dynamic indexing)
    int flag_inner, flag_cont;
    unsigned long long round;      // next cross-GPU exchange round (identical in every CTA and every rank)
};

// fixed-order reduction of per-lane accumulators (entry e lives in lane e%32, slot e/32) to Shared::total
__device__ void reduce_all(Shared& S, cg::cluster_group& cluster, double acc0, double acc1, int warp, int lane) {
    S.warp_acc[warp][lane] = acc0;
    if (lane + 32 < NACC) S.warp_acc[warp][lane + 32] = acc1;
    __syncthreads();
    if (threadIdx.x < NACC) {
        double s = 0.0;
#pragma unroll
        for (int wv = 0; wv < WARPS; ++wv) s += S.warp_acc[wv][threadIdx.x];
        S.part[threadIdx.x] = s;
    }
    cluster.sync();
    if (threadIdx.x < NACC) {
        double s = 0.0;
        const unsigned nr = cluster.num_blocks();
        for (unsigned r = 0; r < nr; ++r) s += cluster.map_shared_rank(&S.part[0], r)[threadIdx.x];
        S.total[threadIdx.x] = s;
    }
    cluster.sync();     // partials may be overwritten only after every CTA has read them
}

// exchange buffer of one rank (in ITS OWN memory; peers write into it):
//   [0, 2 * R * 56)                    data[parity][src rank][56]  partial accumulators (55 used)
//   [2 * R * 56, 2 * R * 56 + 2 * R)   flag[parity][src rank]      round number (as a double-sized u64) the slot holds
constexpr int XSLOT = 56;
//   [.., + 1)                          next round number (persists across launches; every rank runs the same number of rounds)
__host__ __device__ constexpr size_t xbuf_doubles(int world) { return (size_t)2 * world * XSLOT + 2 * world + 1; }

struct Problem;
__device__ void exchange_ranks(const Problem& P, Shared& S, cg::cluster_group& cluster);

struct Problem {
    const double *pos, *uv, *disp, *uvcov, *dcov;
    // graph type (TwoFramePGO/Optimizer.py:51-68): 0 "disp" reprojection + disparity (Graphs.py:121-148), 1 "reproj"
    // reprojection only (:76-118), 2 "icp" point alignment (:33-73) with pc_obs (k,3) = pixel2point_NED(pixel2_uv, pixel2_d),
    // obs_cov / pts_cov (k,3,3) = obs2_covTc / cov_Tw: covariance R Sigma_obs R^T + Sigma_pts, re-inverted at every linearisation
    int gtype;
    const double *pc_obs, *obs_cov, *pts_cov;
    int k;
    const int* k_dev;          // optional device-side block count (<= k): the observation kernel's survivor count
    int k_offset;              // sharded + k_dev: this rank owns global blocks [k_offset, k_offset + k) of the *k_dev valid ones
    int min_k;                 // fewer (global) blocks than this: leave the pose untouched (Odometry/MACVO.py:300-305)
    double* singular_flag;     // stats + 7 or nullptr
    // multi-GPU (residual blocks sharded across ranks, one process per GPU): every rank's exchange buffer, mapped into
    // this process through CUDA IPC (peer memory over NVLink / NVSwitch); xbuf[rank] is this GPU's own buffer
    double* xbuf[MACVO_PGO_MAX_RANKS];
    int world, rank;

    Intr K;
    double delta;
};

// full linearisation at `posevec`: warp-per-residual-block
__device__ void accumulate_full(const Problem& P, const double* posevec, Shared& S, cg::cluster_group& cluster,
                                int gwarp, int nwarps, int warp, int lane) {
    Pose T;
    pose_from_vec(posevec, T);
    if (threadIdx.x == 0) {
        S.Rm[0] = T.R[0]; S.Rm[1] = T.R[1]; S.Rm[2] = T.R[2]; S.Rm[3] = T.R[3]; S.Rm[4] = T.R[4];
        S.Rm[5] = T.R[5]; S.Rm[6] = T.R[6]; S.Rm[7] = T.R[7]; S.Rm[8] = T.R[8];
    }
    __syncthreads();
    double acc0 = 0.0, acc1 = 0.0;
    // which packed entries does this lane own?  slot0: e = lane (0..31), slot1: e = lane + 32 (32..54)
    int e0 = lane, e1 = lane + 32;
    int i0 = 0, j0 = 0, i1 = 0, j1 = 0, kind0, kind1;
    auto classify = [](int e, int& i, int& j) -> int {      // 0: A  1: b  2: G  3: h  4: loss  5: none
        if (e < 21) { tri_index(e, i, j); return 0; }
        if (e < 27) { i = e - 21; j = 0; return 1; }
        if (e < 48) { tri_index(e - 27, i, j); return 2; }
        if (e < 54) { i = e - 48; j = 0; return 3; }
        if (e == 54) return 4;
        return 5;
    };
    kind0 = classify(e0, i0, j0);
    kind1 = classify(e1, i1, j1);

    for (int k = gwarp; k < P.k; k += nwarps) {
        double r[3];
        const int ja = lane / 6, jc = lane - ja * 6;     // lanes 0..17 own (row ja, column jc) of the 3x6 Jacobian
        double j0v = 0.0, j1v = 0.0, j2v = 0.0;          // column jc of J (rows 0..2)
        double w00, w01, w02 = 0.0, w11, w12 = 0.0, w22; // symmetric information matrix of the block
        bool singular = false;
        if (P.gtype == 2) {
            // ---- icp: r = T p_c - p_w,  J = [I | -[T p_c]x],  W = pinv(R Sigma_obs R^T + Sigma_pts) ----
            const double* p = P.pc_obs + 3 * k;
            const double* pw = P.pos + 3 * k;
            double q[3];
            for (int a = 0; a < 3; ++a) q[a] = S.Rm[3 * a] * p[0] + S.Rm[3 * a + 1] * p[1] + S.Rm[3 * a + 2] * p[2] + T.t[a];
            r[0] = q[0] - pw[0]; r[1] = q[1] - pw[1]; r[2] = q[2] - pw[2];
            if (lane < 18) {
                if (jc < 3) { j0v = jc == 0; j1v = jc == 1; j2v = jc == 2; }
                else if (jc == 3) { j0v = 0.0; j1v = -q[2]; j2v = q[1]; }       // -[q]x columns
                else if (jc == 4) { j0v = q[2]; j1v = 0.0; j2v = -q[0]; }
                else { j0v = -q[1]; j1v = q[0]; j2v = 0.0; }
            }
            const double* So = P.obs_cov + 9LL * k;
            const double* Sp = P.pts_cov + 9LL * k;
            double RS[9], M[9];
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) RS[3 * i + j] = S.Rm[3 * i] * So[j] + S.Rm[3 * i + 1] * So[3 + j] + S.Rm[3 * i + 2] * So[6 + j];
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j)
                    M[3 * i + j] = RS[3 * i] * S.Rm[3 * j] + RS[3 * i + 1] * S.Rm[3 * j + 1] + RS[3 * i + 2] * S.Rm[3 * j + 2] + Sp[3 * i + j];
            // torch.pinverse of the (symmetrised) 3x3. A positive-definite block takes the cofactor inverse while that is
            // accurate: det rounds to within a few eps * tr^3, so det >= 1e-6 tr^3 keeps it to ~1e-12 relative (and, as
            // lambda_min >= 4 det / tr^2 and lambda_max <= tr, far above pinv's cutoff). MAC-VO's 2D->3D covariances are
            // long thin ellipsoids along the viewing ray (det / tr^3 ~ 1 / condition^2 ~ 1e-15), where the cofactor
            // inverse is off by 1e-4; those get the Jacobi eigen-decomposition (as accurate as pinv's SVD). An eigenvalue
            // pinv drops is flagged; a non-finite block keeps zero weight (flagged).
            const double m00 = M[0], m01 = 0.5 * (M[1] + M[3]), m02 = 0.5 * (M[2] + M[6]), m11 = M[4], m12 = 0.5 * (M[5] + M[7]), m22 = M[8];
            const double c00 = m11 * m22 - m12 * m12, c01 = m02 * m12 - m01 * m22, c02 = m01 * m12 - m02 * m11;
            const double c22 = m00 * m11 - m01 * m01;
            const double det = m00 * c00 + m01 * c01 + m02 * c02, tr = m00 + m11 + m22;
            if (!isfinite(det) || !isfinite(tr)) { w00 = w01 = w02 = w11 = w12 = w22 = 0.0; singular = true; }
            else if (m00 > 0.0 && c22 > 0.0 && det >= 1e-6 * tr * tr * tr) {      // Sylvester: positive definite
                const double id = 1.0 / det;
                w00 = c00 * id; w01 = c01 * id; w02 = c02 * id;
                w11 = (m00 * m22 - m02 * m02) * id; w12 = (m01 * m02 - m00 * m12) * id; w22 = c22 * id;
            } else singular = sym3_pinv(m00, m01, m02, m11, m12, m22, w00, w01, w02, w11, w12, w22);
        } else {
            double pc[3];
            to_camera(T, P.pos + 3 * k, pc);
            residual3(P.K, pc, P.uv[2 * k], P.uv[2 * k + 1], P.gtype == 0 ? P.disp[k] : 0.0, r);
            const double x = pc[0], y = pc[1], z = pc[2], ix = 1.0 / x, ix2 = ix * ix;
            // J_p = [-R^T | R^T [p_w]x]  (3x6);  J = [J_h J_p ; (-bl fx / x^2) J_p[0,:]]
            const double* pw = P.pos + 3 * k;
            double jp0 = 0.0, jp1 = 0.0, jp2 = 0.0;                                   // J_p[0..2][jc]
            if (lane < 18) {
                if (jc < 3) {                                                          // -R^T: (R^T)[a][c] = R[c][a]
                    jp0 = -S.Rm[3 * jc + 0]; jp1 = -S.Rm[3 * jc + 1]; jp2 = -S.Rm[3 * jc + 2];
                } else {                                                               // R^T [p_w]x
                    const int m = jc - 3, n1 = (m + 1) % 3, n2 = (m + 2) % 3;
                    const double p1 = pw[n2], p2 = pw[n1];
                    jp0 = S.Rm[3 * n1 + 0] * p1 - S.Rm[3 * n2 + 0] * p2;
                    jp1 = S.Rm[3 * n1 + 1] * p1 - S.Rm[3 * n2 + 1] * p2;
                    jp2 = S.Rm[3 * n1 + 2] * p1 - S.Rm[3 * n2 + 2] * p2;
                }
            }
            const double h00 = -P.K.fx * y * ix2, h01 = P.K.fx * ix, h10 = -P.K.fy * z * ix2, h12 = P.K.fy * ix;
            const double hd = P.gtype == 0 ? -(P.K.bl * P.K.fx) * ix2 : 0.0;     // reproj: no disparity row
            if (P.gtype == 1) r[2] = 0.0;
            j0v = h00 * jp0 + h01 * jp1;
            j1v = h10 * jp0 + h12 * jp2;
            j2v = hd * jp0;
            // information matrix of the block: inverse of [[a, c, 0], [c, b, 0], [0, 0, e]]
            const double ca = P.uvcov[3 * k], cb = P.uvcov[3 * k + 1], cc = P.uvcov[3 * k + 2], ce = P.gtype == 0 ? P.dcov[k] : 1.0;
            // the reference takes torch.pinverse of every covariance block (Optimizer.py:96-99): the inverse when every
            // eigenvalue of the block ("disp": the 3x3 diag(pixel 2x2, e); "reproj": the 2x2) exceeds PINV_RCOND times the
            // largest one; otherwise the dropped directions get zero weight (rank-1 pixel block M: M / trace(M)^2) instead
            // of a huge or inf / NaN one, and the block is reported in stats[7]
            // |det| / lbig is the smallest |eigenvalue| of the pixel block, lbig its largest; the row-sum bound
            // lbig <= |a| + |b| + |c| settles the common well-conditioned block without a square root or a division
            const double det = ca * cb - cc * cc, bnd = fabs(ca) + fabs(cb) + fabs(cc);
            const double e_abs = P.gtype == 0 && isfinite(ce) ? fabs(ce) : 0.0;
            double lbig = -1.0;
            auto largest = [&]() {
                if (lbig < 0.0) { const double hd2 = 0.5 * (ca - cb); lbig = fabs(0.5 * (ca + cb)) + sqrt(hd2 * hd2 + cc * cc); }
                return lbig;
            };
            const bool full = fabs(det) > PINV_RCOND * fmax(bnd, e_abs) * bnd ||
                              (largest() > 0.0 && fabs(det) / largest() > PINV_RCOND * fmax(largest(), e_abs));
            if (!isfinite(det) || !isfinite(bnd)) { w00 = w11 = w01 = 0.0; singular = true; }
            else if (full) {
                const double idet = 1.0 / det;
                w00 = cb * idet; w11 = ca * idet; w01 = -cc * idet;
            } else {
                const double tr = ca + cb, itr2 = largest() > PINV_RCOND * e_abs ? 1.0 / (tr * tr) : 0.0;
                w00 = ca * itr2; w11 = cb * itr2; w01 = cc * itr2;
                singular = true;
            }
            if (P.gtype == 1) w22 = 1.0;                                             // reproj: no third residual
            else if (isfinite(ce) && ce != 0.0 &&                                    // a non-finite pixel block leaves e alone
                     (!isfinite(bnd) || e_abs > PINV_RCOND * bnd || e_abs > PINV_RCOND * largest())) w22 = 1.0 / ce;
            else { w22 = 0.0; singular = true; }
        }
        const double nrm2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
        const double sn = sqrt(nrm2);
        const double s = sn < P.delta ? 1.0 : sqrt(P.delta / sn);              // FastTriggs: sqrt(rho'(|r|^2))
        if (singular && lane == 0 && P.singular_flag) *P.singular_flag = 1.0;
        if (lane < 18) {
            const int a = ja;
            S.sJ[warp][lane] = (a == 0 ? j0v : (a == 1 ? j1v : j2v)) * s;
            // (W Js)[a][c]
            S.sWJ[warp][lane] = (a == 0 ? (w00 * j0v + w01 * j1v + w02 * j2v)
                                        : (a == 1 ? (w01 * j0v + w11 * j1v + w12 * j2v) : (w02 * j0v + w12 * j1v + w22 * j2v))) * s;
        } else if (lane < 21) {
            const int a = lane - 18;
            S.sR[warp][a] = r[a] * s;
            S.sWR[warp][a] = (a == 0 ? (w00 * r[0] + w01 * r[1] + w02 * r[2])
                                     : (a == 1 ? (w01 * r[0] + w11 * r[1] + w12 * r[2]) : (w02 * r[0] + w12 * r[1] + w22 * r[2]))) * s;
        }
        __syncwarp();
        auto entry = [&](int kind, int i, int j) -> double {
            const double* J = S.sJ[warp];
            const double* WJ = S.sWJ[warp];
            switch (kind) {
                case 0: return J[i] * WJ[j] + J[6 + i] * WJ[6 + j] + J[12 + i] * WJ[12 + j];
                case 1: return -(J[i] * S.sWR[warp][0] + J[6 + i] * S.sWR[warp][1] + J[12 + i] * S.sWR[warp][2]);
                case 2: return J[i] * J[j] + J[6 + i] * J[6 + j] + J[12 + i] * J[12 + j];
                case 3: return J[i] * S.sR[warp][0] + J[6 + i] * S.sR[warp][1] + J[12 + i] * S.sR[warp][2];
                case 4: return huber(nrm2, P.delta);
                default: return 0.0;
            }
        };
        acc0 += entry(kind0, i0, j0);
        acc1 += entry(kind1, i1, j1);
        __syncwarp();
    }
    reduce_all(S, cluster, acc0, acc1, warp, lane);
    if (P.world > 1) exchange_ranks(P, S, cluster);
}

// robust loss only: lane-per-residual-block
__device__ double evaluate_loss(const Problem& P, const double* posevec, Shared& S, cg::cluster_group& cluster,
                                int gthread, int nthreads, int warp, int lane) {
    Pose T;
    pose_from_vec(posevec, T);
    double acc = 0.0;
    for (int k = gthread; k < P.k; k += nthreads) {
        double pc[3], r[3];
        if (P.gtype == 2) {
            const double* p = P.pc_obs + 3 * k;
            for (int a = 0; a < 3; ++a)
                r[a] = T.R[3 * a] * p[0] + T.R[3 * a + 1] * p[1] + T.R[3 * a + 2] * p[2] + T.t[a] - P.pos[3 * k + a];
        } else {
            to_camera(T, P.pos + 3 * k, pc);
            residual3(P.K, pc, P.uv[2 * k], P.uv[2 * k + 1], P.gtype == 0 ? P.disp[k] : 0.0, r);
            if (P.gtype == 1) r[2] = 0.0;
        }
        acc += huber(r[0] * r[0] + r[1] * r[1] + r[2] * r[2], P.delta);
    }
    acc = warp_sum(acc);                     // butterfly: every lane holds the same bits
    reduce_all(S, cluster, 0.0, lane == 22 ? acc : 0.0, warp, lane);   // packed entry 54 = lane 22, slot 1
    if (P.world > 1) exchange_ranks(P, S, cluster);
    return 0.0;
}

// All-reduce of the 55-double accumulator ACROSS GPUS inside the persistent kernel, over peer memory (the compute step and
// its collective are one launch; no NCCL call, no host round trip per evaluation):
//   CTA 0 of every rank's cluster stores its rank-local total into slot [parity][my rank] of EVERY rank's exchange buffer
//   (plain st.global to IPC-mapped peer memory -> NVLink), fences at system scope, then releases one flag per peer holding
//   the round number; it then spins (bounded) on the `world` flags of its own buffer, and every rank sums the partials in
//   rank order -> identical bits everywhere, so the redundant accept / reject logic cannot diverge between GPUs.
//   Two parities: a rank can run at most one round ahead of the slowest peer (it needs that peer's next partial to go on).
__device__ void exchange_ranks(const Problem& P, Shared& S, cg::cluster_group& cluster) {
    const unsigned long long round = S.round;          // stable: the caller's reduction ended with a cluster-wide sync
    const int parity = (int)(round & 1ull);
    const unsigned crank = cluster.block_rank();
    if (crank == 0) {
        const int W = P.world;
        if (threadIdx.x < NACC) {
            const double v = S.total[threadIdx.x];
            for (int p = 0; p < W; ++p)
                asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(P.xbuf[p] + ((size_t)parity * W + P.rank) * XSLOT + threadIdx.x), "d"(v) : "memory");
        }
        __threadfence_system();
        __syncthreads();
        if ((int)threadIdx.x < W) {
            unsigned long long* peer_flag = reinterpret_cast<unsigned long long*>(P.xbuf[threadIdx.x] + (size_t)2 * W * XSLOT) + parity * W + P.rank;
            asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(peer_flag), "l"(round + 1) : "memory");
            const unsigned long long* my_flag = reinterpret_cast<const unsigned long long*>(P.xbuf[P.rank] + (size_t)2 * W * XSLOT) + parity * W + threadIdx.x;
            const long long t0 = clock64();
            unsigned long long seen;
            do {
                asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(my_flag) : "memory");
                if (seen != round + 1 && clock64() - t0 > 6000000000LL) __trap();     // ~3 s: a lost peer must not hang the GPU
            } while (seen != round + 1);
        }
        __syncthreads();
        if (threadIdx.x < NACC) {
            double s = 0.0;
            for (int p = 0; p < W; ++p) {
                double v;
                asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(P.xbuf[P.rank] + ((size_t)parity * W + p) * XSLOT + threadIdx.x) : "memory");
                s += v;
            }
            S.total[threadIdx.x] = s;
        }
    }
    cluster.sync();
    if (crank != 0 && threadIdx.x < NACC) S.total[threadIdx.x] = cluster.map_shared_rank(&S.total[0], 0)[threadIdx.x];
    if (threadIdx.x == 0) S.round = round + 1;
    cluster.sync();
}

// ---- small dense algebra (thread 0 of each CTA) --------------------------------------------------------
__device__ void so3_exp(const double* phi, double* q) {
    const double t2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
    const double th = sqrt(t2);
    double imag, real;
    if (th > 2.220446049250313e-16) { imag = sin(0.5 * th) / th; real = cos(0.5 * th); }
    else { imag = 0.5 - t2 / 48 + t2 * t2 / 3840; real = 1 - t2 / 8 + t2 * t2 / 384; }
    q[0] = phi[0] * imag; q[1] = phi[1] * imag; q[2] = phi[2] * imag; q[3] = real;
}

__device__ void se3_exp(const double* xi, double* out) {      // out = [t, q]
    const double* phi = xi + 3;
    const double t2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
    const double th = sqrt(t2);
    double c1, c2;
    if (th > 2.220446049250313e-16) { c1 = (1 - cos(th)) / t2; c2 = (th - sin(th)) / (t2 * th); }
    else { c1 = 0.5 - t2 / 24 + t2 * t2 / 720; c2 = 1.0 / 6 - t2 / 120 + t2 * t2 / 5040; }
    // J_l tau = tau + c1 (phi x tau) + c2 (phi x (phi x tau))
    const double* tau = xi;
    const double a0 = phi[1] * tau[2] - phi[2] * tau[1], a1 = phi[2] * tau[0] - phi[0] * tau[2],
                 a2 = phi[0] * tau[1] - phi[1] * tau[0];
    const double b0 = phi[1] * a2 - phi[2] * a1, b1 = phi[2] * a0 - phi[0] * a2, b2 = phi[0] * a1 - phi[1] * a0;
    out[0] = tau[0] + c1 * a0 + c2 * b0;
    out[1] = tau[1] + c1 * a1 + c2 * b1;
    out[2] = tau[2] + c1 * a2 + c2 * b2;
    so3_exp(phi, out + 3);
}

__device__ void quat_rot(const double* q, const double* p, double* o) {
    const double uv0 = 2 * (q[1] * p[2] - q[2] * p[1]), uv1 = 2 * (q[2] * p[0] - q[0] * p[2]),
                 uv2 = 2 * (q[0] * p[1] - q[1] * p[0]);
    o[0] = p[0] + q[3] * uv0 + (q[1] * uv2 - q[2] * uv1);
    o[1] = p[1] + q[3] * uv1 + (q[2] * uv0 - q[0] * uv2);
    o[2] = p[2] + q[3] * uv2 + (q[0] * uv1 - q[1] * uv0);
}

// pose <- Exp(step[:6]) * pose   (pypose left retraction)
__device__ void retract(const double* pose, const double* step, double* out) {
    double e[7], rt[3];
    se3_exp(step, e);
    quat_rot(e + 3, pose, rt);
    const double ax = e[3], ay = e[4], az = e[5], aw = e[6], bx = pose[3], by = pose[4], bz = pose[5], bw = pose[6];
    out[0] = rt[0] + e[0]; out[1] = rt[1] + e[1]; out[2] = rt[2] + e[2];
    out[3] = aw * bx + ax * bw + ay * bz - az * by;
    out[4] = aw * by - ax * bz + ay * bw + az * bx;
    out[5] = aw * bz + ax * by - ay * bx + az * bw;
    out[6] = aw * bw - ax * bx - ay * by - az * bz;
}

// solve the SPD-after-damping 6x6 system by Gaussian elimination with partial pivoting (PINV stand-in:
// identical for the full-rank systems of this path; the dead 7th row/col of the reference solves to 0)
__device__ bool solve6(const double* Afull, const double* b, double* x) {
    double M[6][7];
    for (int i = 0; i < 6; ++i) {
        for (int j = 0; j < 6; ++j) M[i][j] = Afull[i * 6 + j];
        M[i][6] = b[i];
    }
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        double best = fabs(M[c][c]);
        for (int r = c + 1; r < 6; ++r)
            if (fabs(M[r][c]) > best) { best = fabs(M[r][c]); piv = r; }
        if (!(best > 0.0)) return false;
        if (piv != c)
            for (int j = c; j < 7; ++j) { const double t = M[c][j]; M[c][j] = M[piv][j]; M[piv][j] = t; }
        const double inv = 1.0 / M[c][c];
        for (int r = c + 1; r < 6; ++r) {
            const double f = M[r][c] * inv;
            for (int j = c; j < 7; ++j) M[r][j] -= f * M[c][j];
        }
    }
    for (int i = 5; i >= 0; --i) {
        double s = M[i][6];
        for (int j = i + 1; j < 6; ++j) s -= M[i][j] * x[j];
        x[i] = s / M[i][i];
    }
    return true;
}

__global__ void __launch_bounds__(THREADS)
pgo_lm_kernel(Problem P, double* __restrict__ pose_io, macvo_pgo_params_t prm, double* __restrict__ stats) {
    __shared__ Shared S;
    cg::cluster_group cluster = cg::this_cluster();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = (int)cluster.block_rank(), nblk = (int)cluster.num_blocks();
    const int gwarp = rank * WARPS + warp, nwarps = nblk * WARPS;
    const int gthread = rank * THREADS + threadIdx.x, nthreads = nblk * THREADS;

    if (threadIdx.x < 7) S.pose[threadIdx.x] = pose_io[threadIdx.x];
    if (threadIdx.x == 0)
        S.round = P.world > 1 ? *reinterpret_cast<const unsigned long long*>(P.xbuf[P.rank] + xbuf_doubles(P.world) - 1) : 0ull;
    int k_total = P.k;
    if (P.k_dev != nullptr) {
        k_total = max(*P.k_dev, 0);                                   // same value on every rank (broadcast with the data)
        P.k = min(P.k, max(k_total - P.k_offset, 0));
    }
    if (k_total < P.min_k) {    // lost track: every CTA of the cluster (and every rank) takes this branch together
        if (rank == 0 && threadIdx.x == 0 && stats) {
            for (int i = 0; i < 6; ++i) stats[i] = 0.0;
            stats[6] = 1.0;                                       // skipped
        }
        return;
    }
    __syncthreads();

    // optimiser / scheduler state, replicated identically in thread 0 of every CTA
    double damping = 1.0 / prm.radius, down = 0.5;
    const double TR_MIN = 1e-3, TR_MAX = 1e5, HIGH = 0.5, LOW = 1e-3, UP = 2.0, DOWN = 0.5, FACTOR = 0.5;
    double loss = 0.0, last = 0.0, first_loss = 0.0;
    bool have_loss = false;
    int steps = 0, patience_count = 0, reject_count = 0, evals = 0;
    double A[36], bvec[6], G[36], hvec[6], D[6];

    bool cont = true;
    while (cont) {
        accumulate_full(P, S.pose, S, cluster, gwarp, nwarps, warp, lane);      // S.total valid in all threads
        if (threadIdx.x == 0) {
            int e = 0;
            for (int i = 0; i < 6; ++i)
                for (int j = i; j < 6; ++j, ++e) {
                    A[i * 6 + j] = A[j * 6 + i] = S.total[e];
                    G[i * 6 + j] = G[j * 6 + i] = S.total[27 + e];
                }
            for (int i = 0; i < 6; ++i) { bvec[i] = S.total[21 + i]; hvec[i] = S.total[48 + i]; }
            if (!have_loss) { loss = S.total[54]; first_loss = loss; have_loss = true; }
            last = loss;
            reject_count = 0;
            for (int i = 0; i < 6; ++i) A[i * 6 + i] = fmin(fmax(A[i * 6 + i], prm.diag_min), prm.diag_max);
        }
        // inner accept / reject loop: `while self.last <= self.loss`
        bool inner = true;
        while (inner) {
            if (threadIdx.x == 0) {
                for (int i = 0; i < 6; ++i) A[i * 6 + i] += A[i * 6 + i] * damping;
                const bool ok = solve6(A, bvec, D);
                if (!ok) for (int i = 0; i < 6; ++i) D[i] = 0.0;
                retract(S.pose, D, S.trial);
            }
            __syncthreads();
            evaluate_loss(P, S.trial, S, cluster, gthread, nthreads, warp, lane);
            if (threadIdx.x == 0) {
                loss = S.total[54];
                ++evals;
                // TrustRegion.update: quality = (last - loss) / -((J D)^T (2 R + J D))
                double dh = 0.0, dGd = 0.0;
                for (int i = 0; i < 6; ++i) {
                    dh += D[i] * hvec[i];
                    double gi = 0.0;
                    for (int j = 0; j < 6; ++j) gi += G[i * 6 + j] * D[j];
                    dGd += D[i] * gi;
                }
                const double quality = (last - loss) / -(2.0 * dh + dGd);
                double radius = 1.0 / damping;
                if (quality > HIGH) { radius *= UP; down = DOWN; }
                else if (quality > LOW) { down = DOWN; }
                else { radius *= down; down *= FACTOR; }
                down = fmax(TR_MIN, fmin(down, TR_MAX));
                radius = fmax(TR_MIN, fmin(radius, TR_MAX));
                damping = 1.0 / radius;
                int flag;
                if (last < loss && reject_count < prm.max_reject) {   // reject: undo the step with Exp(-D)
                    double nD[6], back[7];
                    for (int i = 0; i < 6; ++i) nD[i] = -D[i];
                    retract(S.trial, nD, back);
                    for (int i = 0; i < 7; ++i) S.pose[i] = back[i];
                    loss = last;
                    ++reject_count;
                    flag = 1;                                          // `while last <= loss` holds: try again
                } else {
                    for (int i = 0; i < 7; ++i) S.pose[i] = S.trial[i];
                    flag = 0;
                }
                S.flag_inner = flag;
            }
            __syncthreads();
            inner = S.flag_inner != 0;
        }
        if (threadIdx.x == 0) {
            // StopOnPlateau.step
            ++steps;
            bool c = steps < prm.max_steps;
            patience_count = (last - loss) < prm.decreasing ? patience_count + 1 : 0;
            if (patience_count >= prm.patience) c = false;
            if (reject_count >= prm.max_reject) c = false;
            S.flag_cont = c ? 1 : 0;
        }
        __syncthreads();
        cont = S.flag_cont != 0;
    }
    if (rank == 0 && threadIdx.x == 0) {
        for (int i = 0; i < 7; ++i) pose_io[i] = S.pose[i];
        if (stats) {
            stats[0] = steps; stats[1] = evals; stats[2] = loss; stats[3] = first_loss;
            stats[4] = reject_count; stats[5] = damping; stats[6] = 0;      // stats[7]: singular-block flag (set above)
        }
    }
    if (P.world > 1 && rank == 0 && threadIdx.x == 0)
        *reinterpret_cast<unsigned long long*>(P.xbuf[P.rank] + xbuf_doubles(P.world) - 1) = S.round;
    cluster.sync();     // no CTA may exit while a peer can still read its shared memory
}

__global__ void __launch_bounds__(THREADS)
pgo_accumulate_kernel(Problem P, const double* __restrict__ pose, double* __restrict__ acc_out) {
    __shared__ Shared S;
    cg::cluster_group cluster = cg::this_cluster();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = (int)cluster.block_rank();
    if (threadIdx.x < 7) S.pose[threadIdx.x] = pose[threadIdx.x];
    __syncthreads();
    accumulate_full(P, S.pose, S, cluster, rank * WARPS + warp, (int)cluster.num_blocks() * WARPS, warp, lane);
    if (rank == 0 && threadIdx.x < NACC) acc_out[threadIdx.x] = S.total[threadIdx.x];
}

// CTAs per cluster: the given 1..8, or (0) chosen from the block count
int cluster_size(int cluster, int k) {
    if (cluster <= 0) cluster = k >= 2048 ? 8 : (k >= 768 ? 4 : (k >= 256 ? 2 : 1));
    return cluster > 8 ? 8 : cluster;
}

int launch_cluster(const void* fn, int cluster, void** args, cudaStream_t st) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cluster);
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MACVO_CUDA_TRY(cudaLaunchKernelExC(&cfg, fn, args));
    return MACVO_OK;
}

}  // namespace

struct GraphExtra { int gtype; const double *pc_obs, *obs_cov, *pts_cov; };

static int pgo_solve_impl(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                          const double* uv_cov, const double* disp_cov, int k, const int* k_dev, int min_k,
                          const double* intr, double* pose_io, const macvo_pgo_params_t* params, double* stats,
                          void* stream, void* const* peer_bufs = nullptr, int world = 1, int rank = 0, int k_offset = 0,
                          GraphExtra gx = GraphExtra{0, nullptr, nullptr, nullptr}) {
    if (k < 0 || !intr || !pose_io || !params || gx.gtype < 0 || gx.gtype > 2) return MACVO_E_ARG;
    if (k > 0 && !pos_Tw) return MACVO_E_ARG;
    if (k > 0 && gx.gtype == 0 && (!kp2_uv || !kp2_disp || !uv_cov || !disp_cov)) return MACVO_E_ARG;
    if (k > 0 && gx.gtype == 1 && (!kp2_uv || !uv_cov)) return MACVO_E_ARG;
    if (k > 0 && gx.gtype == 2 && (!gx.pc_obs || !gx.obs_cov || !gx.pts_cov)) return MACVO_E_ARG;
    macvo_pgo_params_t prm = *params;
    if (prm.max_steps < 1 || prm.radius <= 0 || prm.huber_delta <= 0) return MACVO_E_ARG;
    const int cluster = cluster_size(prm.cluster, k);
    Problem P;
    P.pos = pos_Tw; P.uv = kp2_uv; P.disp = kp2_disp; P.uvcov = uv_cov; P.dcov = disp_cov; P.k = k;
    P.k_dev = k_dev; P.k_offset = k_offset; P.min_k = min_k; P.singular_flag = stats ? stats + 7 : nullptr;
    P.gtype = gx.gtype; P.pc_obs = gx.pc_obs; P.obs_cov = gx.obs_cov; P.pts_cov = gx.pts_cov;
    P.world = 1; P.rank = 0;
    if (peer_bufs != nullptr) {
        if (world < 2 || world > MACVO_PGO_MAX_RANKS || rank < 0 || rank >= world) return MACVO_E_ARG;
        P.world = world; P.rank = rank;
        for (int r = 0; r < world; ++r) {
            if (!peer_bufs[r]) return MACVO_E_ARG;
            P.xbuf[r] = static_cast<double*>(peer_bufs[r]);
        }
    }
    // intr is HOST memory: {fx, fy, cx, cy, baseline}
    P.K.fx = intr[0]; P.K.fy = intr[1]; P.K.cx = intr[2]; P.K.cy = intr[3]; P.K.bl = intr[4];
    P.delta = prm.huber_delta;
    void* args[] = {&P, &pose_io, &prm, &stats};
    return launch_cluster(reinterpret_cast<const void*>(&pgo_lm_kernel), cluster, args, as_stream(stream));
}

extern "C" int macvo_pgo_solve(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                               const double* uv_cov, const double* disp_cov, int k, const double* intr,
                               double* pose_io, const macvo_pgo_params_t* params, double* stats, void* stream) {
    return pgo_solve_impl(pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov, k, nullptr, 0, intr, pose_io, params, stats, stream);
}

extern "C" int macvo_pgo_solve_graph(int graph_type, const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                                     const double* uv_cov, const double* disp_cov, const double* pc_obs,
                                     const double* obs_cov, const double* pts_cov, int k, const double* intr,
                                     double* pose_io, const macvo_pgo_params_t* params, double* stats, void* stream) {
    return pgo_solve_impl(pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov, k, nullptr, 0, intr, pose_io, params, stats, stream,
                          nullptr, 1, 0, 0, GraphExtra{graph_type, pc_obs, obs_cov, pts_cov});
}

extern "C" int macvo_pgo_solve_counted(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                                       const double* uv_cov, const double* disp_cov, int k_capacity, const int* k_dev,
                                       int min_k, const double* intr, double* pose_io,
                                       const macvo_pgo_params_t* params, double* stats, void* stream, int graph_type,
                                       const double* pc_obs, const double* obs_cov, const double* pts_cov) {
    if (!k_dev || min_k < 0) return MACVO_E_ARG;
    // every graph type's loops run over P.k = min(*k_dev, k_capacity): no block at or past the survivor count is read
    return pgo_solve_impl(pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov, k_capacity, k_dev, min_k, intr, pose_io, params,
                          stats, stream, nullptr, 1, 0, 0, GraphExtra{graph_type, pc_obs, obs_cov, pts_cov});
}

// ---- multi-GPU: sharded residual blocks, all-reduce fused into the persistent kernel over peer memory ---------------------
extern "C" size_t macvo_pgo_exchange_bytes(int world) {
    return world >= 1 && world <= MACVO_PGO_MAX_RANKS ? xbuf_doubles(world) * sizeof(double) : 0;
}

extern "C" int macvo_p2p_alloc(size_t bytes, void** dev_ptr, unsigned char* ipc_handle64) {
    if (!dev_ptr || !ipc_handle64 || bytes == 0) return MACVO_E_ARG;
    void* p = nullptr;
    MACVO_CUDA_TRY(cudaMalloc(&p, bytes));
    MACVO_CUDA_TRY(cudaMemset(p, 0, bytes));
    MACVO_CUDA_TRY(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    MACVO_CUDA_TRY(cudaIpcGetMemHandle(&h, p));
    static_assert(sizeof(h) == 64, "CUDA IPC handle size");
    memcpy(ipc_handle64, &h, 64);
    *dev_ptr = p;
    return MACVO_OK;
}

extern "C" int macvo_p2p_open(const unsigned char* ipc_handle64, void** peer_ptr) {
    if (!ipc_handle64 || !peer_ptr) return MACVO_E_ARG;
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle64, 64);
    MACVO_CUDA_TRY(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return MACVO_OK;
}

extern "C" int macvo_p2p_close(void* peer_ptr) {
    if (peer_ptr) MACVO_CUDA_TRY(cudaIpcCloseMemHandle(peer_ptr));
    return MACVO_OK;
}

extern "C" int macvo_p2p_free(void* dev_ptr) {
    if (dev_ptr) MACVO_CUDA_TRY(cudaFree(dev_ptr));
    return MACVO_OK;
}

extern "C" int macvo_pgo_solve_sharded(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                                       const double* uv_cov, const double* disp_cov, int k_shard, const int* k_total_dev,
                                       int k_offset, int min_k, const double* intr, double* pose_io,
                                       const macvo_pgo_params_t* params, double* stats, void* const* exchange_bufs,
                                       int world, int rank, void* stream) {
    if (!exchange_bufs || k_offset < 0 || min_k < 0) return MACVO_E_ARG;
    return pgo_solve_impl(pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov, k_shard, k_total_dev, min_k, intr, pose_io, params, stats,
                          stream, exchange_bufs, world, rank, k_offset);
}

extern "C" int macvo_pgo_accumulate_graph(int graph_type, const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                                          const double* uv_cov, const double* disp_cov, const double* pc_obs,
                                          const double* obs_cov, const double* pts_cov, int k, const double* intr,
                                          const double* pose, double huber_delta, int cluster, double* acc,
                                          double* singular_flag, void* stream) {
    if (k < 0 || !intr || !pose || !acc || graph_type < 0 || graph_type > 2 || cluster < 0 || cluster > 8) return MACVO_E_ARG;
    if (k > 0 && !pos_Tw) return MACVO_E_ARG;
    if (k > 0 && graph_type == 0 && (!kp2_uv || !kp2_disp || !uv_cov || !disp_cov)) return MACVO_E_ARG;
    if (k > 0 && graph_type == 1 && (!kp2_uv || !uv_cov)) return MACVO_E_ARG;
    if (k > 0 && graph_type == 2 && (!pc_obs || !obs_cov || !pts_cov)) return MACVO_E_ARG;
    Problem P;
    P.pos = pos_Tw; P.uv = kp2_uv; P.disp = kp2_disp; P.uvcov = uv_cov; P.dcov = disp_cov; P.k = k;
    P.k_dev = nullptr; P.k_offset = 0; P.min_k = 0; P.singular_flag = singular_flag; P.world = 1; P.rank = 0;
    P.gtype = graph_type; P.pc_obs = pc_obs; P.obs_cov = obs_cov; P.pts_cov = pts_cov;
    P.K.fx = intr[0]; P.K.fy = intr[1]; P.K.cx = intr[2]; P.K.cy = intr[3]; P.K.bl = intr[4];
    P.delta = huber_delta;
    void* args[] = {&P, &pose, &acc};
    return launch_cluster(reinterpret_cast<const void*>(&pgo_accumulate_kernel), cluster_size(cluster, k), args,
                          as_stream(stream));
}

extern "C" int macvo_pgo_accumulate(const double* pos_Tw, const double* kp2_uv, const double* kp2_disp,
                                    const double* uv_cov, const double* disp_cov, int k, const double* intr,
                                    const double* pose, double huber_delta, double* acc, void* stream) {
    return macvo_pgo_accumulate_graph(MACVO_PGO_DISP, pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov, nullptr, nullptr, nullptr, k,
                                      intr, pose, huber_delta, 1, acc, nullptr, stream);
}
