// (f5) TartanVO pose network of TartanMotionNet (Module/MotionModel.py:89-116): VOFlowRes(config=1, stereo, down_scale,
// intrinsic) (Module/Network/TartanVOStereo/FlowPoseNet.py:45-165) fed by TartanStereoVOMotion.inference
// (StereoVO_Interface.py:158-194).
//
//   posenet_input_kernel   full-resolution flow (2,H,W) + depth (1,H,W) -> channels 0..2 of the 5 x 112 x 160 network
//                          input: centre crop, bilinear align_corners=True resize (ATen's index / lambda arithmetic),
//                          flow x 0.05, depth -> normalised disparity with the reference's nan_to_num / clamp order.
//   posenet_conv_kernel    every convolution whose output is 7 x 10 pixels or smaller (layer3..layer5, downsamples
//                          included) and fc1 (both heads, run as a 1 x 1 convolution of the flattened 256 x 2 x 3 map).
//                          These layers are weight-streaming GEMVs: 6..70 output pixels against K = 1152..2304, 13.8 M
//                          of the network's 15.1 M parameters. Grid = (8 K-splits) x (cout / co_tile output-channel
//                          tiles) = 256 CTAs, one thread-block cluster of 8 per tile; each CTA streams ONE contiguous
//                          weight slab (packed at construction: [tile][split][co_tile][cin/8 * k * k]) exactly once,
//                          multiplies it with its 1/8 of the input channels (zero-padded copy in shared memory), and the
//                          cluster sums the 8 partials over DSMEM in rank order (deterministic: no atomics), adds bias,
//                          optional residual, optional ReLU — BasicBlock.forward (FlowPoseNet.py:35-43) in one launch.
//   posenet_head_kernel    one CTA: fc2 + ReLU and fc3 of both heads, x pose_norm, then the prediction
//                          next = prev (fp32) @ se3(motion).Exp() (pypose conventions, fp32), widened to float64.
//
// fp32 operands, fp32 accumulation.
#include "common.cuh"

#include <cfloat>
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace {

constexpr int PN_H = 112, PN_W = 160, PN_HW = PN_H * PN_W;
constexpr int SPLIT = 8;          // K split = cluster size
constexpr int CONV_NT = 256;
constexpr int PB = 10;            // output pixels per warp task (register block)
constexpr int HEAD_NT = 256;
constexpr float FLOW_NORM = 0.05f;                          // TartanStereoVONetInterface.flow_norm
constexpr float STEREO_NORM = 0.02f;                        // StereoVONet stereoNormFactor
constexpr float DEPTH_DIV = (float)(0.02 * 0.25);           // float(stereoNormFactor * poseDepthNormFactor)

struct Crop {
    int y0, x0, h, w;      // crop window inside the full map
    float sy, sx;          // align_corners=True source scales (in - 1) / (out - 1)
};

// ATen upsample_bilinear2d (align_corners=True): real = scale * dst; index = min(floor(real), in - 1);
// lambda = clamp(real - index, 0, 1); the second tap is index + 1 unless index is the last row / column
__device__ __forceinline__ void taps(float scale, int dst, int in_size, int& i0, int& i1, float& l0, float& l1) {
    const float real = __fmul_rn(scale, (float)dst);
    const int i = min((int)floorf(real), in_size - 1);
    const float lam = fminf(fmaxf(__fsub_rn(real, (float)i), 0.f), 1.f);
    i0 = i;
    i1 = i + (i < in_size - 1 ? 1 : 0);
    l1 = lam;
    l0 = __fsub_rn(1.f, lam);
}

__device__ __forceinline__ float bilinear(const float* m, int W, const Crop& c, int y0, int y1, int x0, int x1, float hy0,
                                          float hy1, float wx0, float wx1) {
    const float* r0 = m + (long long)(c.y0 + y0) * W + c.x0;
    const float* r1 = m + (long long)(c.y0 + y1) * W + c.x0;
    const float t0 = __fadd_rn(__fmul_rn(r0[x0], wx0), __fmul_rn(r0[x1], wx1));
    const float t1 = __fadd_rn(__fmul_rn(r1[x0], wx0), __fmul_rn(r1[x1], wx1));
    return __fadd_rn(__fmul_rn(t0, hy0), __fmul_rn(t1, hy1));
}

__global__ void __launch_bounds__(256)
posenet_input_kernel(const float* __restrict__ flow, const float* __restrict__ depth, int H, int W, Crop c, float bl_fx,
                     float* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= PN_HW) return;
    const int oy = idx / PN_W, ox = idx - oy * PN_W;
    int y0, y1, x0, x1;
    float hy0, hy1, wx0, wx1;
    taps(c.sy, oy, c.h, y0, y1, hy0, hy1);
    taps(c.sx, ox, c.w, x0, x1, wx0, wx1);
    const long long hw = (long long)H * W;
    // flow: resize, then x flow_norm
    out[idx] = __fmul_rn(bilinear(flow, W, c, y0, y1, x0, x1, hy0, hy1, wx0, wx1), FLOW_NORM);
    out[PN_HW + idx] = __fmul_rn(bilinear(flow + hw, W, c, y0, y1, x0, x1, hy0, hy1, wx0, wx1), FLOW_NORM);
    // depth: stereo = (bl fx) / d  (python scalar / tensor = reciprocal(d) * scalar), x stereoNormFactor,
    // nan_to_num(nan=0, +-inf -> +-FLT_MAX), clamp(min=0), / (bl fx), / float(0.02 * 0.25)
    const float d = bilinear(depth, W, c, y0, y1, x0, x1, hy0, hy1, wx0, wx1);
    float s = __fmul_rn(__fmul_rn(__frcp_rn(d), bl_fx), STEREO_NORM);
    if (isnan(s)) s = 0.f;
    else if (isinf(s)) s = s > 0.f ? FLT_MAX : -FLT_MAX;
    s = s < 0.f ? 0.f : s;
    out[2 * PN_HW + idx] = __fdiv_rn(__fdiv_rn(s, bl_fx), DEPTH_DIV);
}

struct ConvArgs {
    const float* x;        // (cin, hi, wi)
    const float* w;        // packed slabs [tile][split][co_tile][cin/8 * ks * ks]
    const float* bias;     // (cout)
    const float* resid;    // (cout, ho, wo) or null
    float* y;              // (cout, ho, wo)
    int cin, hi, wi, cout, ho, wo, ks, stride, pad, co_tile, relu;
};

__global__ void __cluster_dims__(SPLIT, 1, 1) __launch_bounds__(CONV_NT)
posenet_conv_kernel(ConvArgs a) {
    extern __shared__ __align__(16) float sm[];
    cg::cluster_group cluster = cg::this_cluster();
    const int split = blockIdx.x, tile = blockIdx.y;          // gridDim.x == SPLIT: split == cluster rank
    const int cps = a.cin / SPLIT, kk = a.ks * a.ks, kc = cps * kk;
    const int hp = a.hi + 2 * a.pad, wp = a.wi + 2 * a.pad, hwp = hp * wp;
    const int P = a.ho * a.wo, nout = a.co_tile * P;
    float* ws = sm;                                            // co_tile * kc weights
    float* xs = ws + a.co_tile * kc;                           // cps * hwp zero-padded input channels
    float* part = xs + cps * hwp;                              // nout partial sums (read by the cluster)
    int* ktab = reinterpret_cast<int*>(part + nout);           // kc: offset of tap k inside xs
    int* ptab = ktab + kc;                                     // P: offset of output pixel p's window origin

    // the weight slab: contiguous, 16-byte aligned, read once -> streaming loads that bypass L1
    const float4* wsrc = reinterpret_cast<const float4*>(a.w + ((size_t)tile * SPLIT + split) * a.co_tile * kc);
    const int n4 = a.co_tile * kc / 4;
    for (int i = threadIdx.x; i < n4; i += CONV_NT) reinterpret_cast<float4*>(ws)[i] = __ldcs(wsrc + i);
    const float* xsrc = a.x + (size_t)split * cps * a.hi * a.wi;
    for (int i = threadIdx.x; i < cps * hwp; i += CONV_NT) {
        const int ci = i / hwp, r = i - ci * hwp, yy = r / wp - a.pad, xx = r % wp - a.pad;
        xs[i] = (yy >= 0 && yy < a.hi && xx >= 0 && xx < a.wi) ? xsrc[(ci * a.hi + yy) * a.wi + xx] : 0.f;
    }
    for (int k = threadIdx.x; k < kc; k += CONV_NT) {
        const int ci = k / kk, r = k - ci * kk, ky = r / a.ks, kx = r - ky * a.ks;
        ktab[k] = ci * hwp + ky * wp + kx;
    }
    for (int p = threadIdx.x; p < P; p += CONV_NT) {
        const int oy = p / a.wo, ox = p - oy * a.wo;
        ptab[p] = oy * a.stride * wp + ox * a.stride;
    }
    __syncthreads();

    // warp task = (output channel, block of PB pixels); lanes stride over K; fixed-order shuffle reduction
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pblocks = (P + PB - 1) / PB, ntask = a.co_tile * pblocks;
    for (int task = warp; task < ntask; task += CONV_NT / 32) {
        const int co = task / pblocks, p0 = (task - co * pblocks) * PB;
        const int np = min(PB, P - p0);
        int po[PB];
#pragma unroll
        for (int j = 0; j < PB; ++j) po[j] = ptab[p0 + min(j, np - 1)];
        float acc[PB];
#pragma unroll
        for (int j = 0; j < PB; ++j) acc[j] = 0.f;
        const float* wr = ws + co * kc;
        for (int k = lane; k < kc; k += 32) {
            const float wv = wr[k];
            const float* xk = xs + ktab[k];
#pragma unroll
            for (int j = 0; j < PB; ++j) acc[j] = fmaf(wv, xk[po[j]], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < PB; ++j) {
            float v = acc[j];
#pragma unroll
            for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == 0 && j < np) part[co * P + p0 + j] = v;
        }
    }
    cluster.sync();
    // CTA `split` finishes outputs split, split + 8 * 256, ...: partials summed in rank order, then the fused epilogue
    for (int o = split * CONV_NT + threadIdx.x; o < nout; o += SPLIT * CONV_NT) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < SPLIT; ++r) s += cluster.map_shared_rank(part, r)[o];
        const int co = o / P, p = o - co * P, gco = tile * a.co_tile + co;
        s += a.bias[gco];
        const size_t gi = (size_t)gco * P + p;
        if (a.resid) s += a.resid[gi];
        if (a.relu) s = fmaxf(s, 0.f);
        a.y[gi] = s;
    }
    cluster.sync();     // no CTA may leave while another still reads its partials
}

size_t conv_smem_bytes(int cin, int hi, int wi, int ho, int wo, int ks, int pad, int co_tile) {
    const int cps = cin / SPLIT, kc = cps * ks * ks, hwp = (hi + 2 * pad) * (wi + 2 * pad), P = ho * wo;
    return sizeof(float) * ((size_t)co_tile * kc + (size_t)cps * hwp + (size_t)co_tile * P) + sizeof(int) * ((size_t)kc + P);
}

// ---- head ---------------------------------------------------------------------------------------------------------------
// blob layout (floats): fc2 trans W (32x128) | b (32) | fc2 rot W | b | fc3 trans W (3x32) | b (3) | fc3 rot W | b | pose_norm (6)
constexpr int FC1 = 128, FC2 = 32, FC3 = 3;
constexpr int OFF_W2T = 0, OFF_B2T = OFF_W2T + FC2 * FC1, OFF_W2R = OFF_B2T + FC2, OFF_B2R = OFF_W2R + FC2 * FC1;
constexpr int OFF_W3T = OFF_B2R + FC2, OFF_B3T = OFF_W3T + FC3 * FC2, OFF_W3R = OFF_B3T + FC3, OFF_B3R = OFF_W3R + FC3 * FC2;
constexpr int OFF_NORM = OFF_B3R + FC3, HEAD_FLOATS = OFF_NORM + 6;

__device__ __forceinline__ void cross3(const float* a, const float* b, float* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// R(q) p = p + w (2 v x p) + v x (2 v x p)   (pypose / oracle shim order)
__device__ __forceinline__ void qrot(const float* q, const float* p, float* o) {
    float uv[3], c[3];
    cross3(q, p, uv);
    for (int i = 0; i < 3; ++i) uv[i] *= 2.f;
    cross3(q, uv, c);
    for (int i = 0; i < 3; ++i) o[i] = p[i] + q[3] * uv[i] + c[i];
}

__global__ void __launch_bounds__(HEAD_NT)
posenet_head_kernel(const float* __restrict__ h1, const float* __restrict__ blob, const double* __restrict__ prev,
                    float* __restrict__ motion_out, double* __restrict__ next_pose) {
    __shared__ float x2[2 * FC2];
    __shared__ float mot[6];
    const int t = threadIdx.x;
    if (t < 2 * FC2) {                                   // fc2 + ReLU, trans rows 0..31, rot rows 32..63
        const int head = t / FC2, r = t - head * FC2;
        const float* W = blob + (head ? OFF_W2R : OFF_W2T) + r * FC1;
        const float* x = h1 + head * FC1;
        float s = 0.f;
        for (int k = 0; k < FC1; ++k) s = fmaf(W[k], x[k], s);
        x2[t] = fmaxf(s + blob[(head ? OFF_B2R : OFF_B2T) + r], 0.f);
    }
    __syncthreads();
    if (t < 6) {                                         // fc3; pose = cat(trans, rot) * pose_norm
        const int head = t / FC3, r = t - head * FC3;
        const float* W = blob + (head ? OFF_W3R : OFF_W3T) + r * FC2;
        float s = 0.f;
        for (int k = 0; k < FC2; ++k) s = fmaf(W[k], x2[head * FC2 + k], s);
        const float m = (s + blob[(head ? OFF_B3R : OFF_B3T) + r]) * blob[OFF_NORM + t];
        mot[t] = m;
        motion_out[t] = m;
    }
    __syncthreads();
    if (t != 0) return;
    // se3(motion).Exp(): q = [phi sin(th/2)/th, cos(th/2)], t = Jl(phi) tau   (series below fp32 eps, as pypose)
    const float* tau = mot;
    const float* phi = mot + 3;
    const float th = sqrtf(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
    const float t2 = th * th, t4 = t2 * t2;
    const bool small = th <= FLT_EPSILON;
    const float sf = small ? 1.f : th;
    const float imag = small ? 0.5f - t2 / 48.f + t4 / 3840.f : sinf(0.5f * sf) / sf;
    const float real = small ? 1.f - t2 / 8.f + t4 / 384.f : cosf(0.5f * th);
    const float c1 = small ? 0.5f - t2 / 24.f + t4 / 720.f : (1.f - cosf(sf)) / (sf * sf);
    const float c2 = small ? 1.f / 6.f - t2 / 120.f + t4 / 5040.f : (sf - sinf(sf)) / (sf * sf * sf);
    float kt[3], kkt[3], te[3], qe[4];
    cross3(phi, tau, kt);                                // K tau = phi x tau
    cross3(phi, kt, kkt);                                // K^2 tau
    for (int i = 0; i < 3; ++i) te[i] = tau[i] + c1 * kt[i] + c2 * kkt[i];
    for (int i = 0; i < 3; ++i) qe[i] = phi[i] * imag;
    qe[3] = real;
    // prev @ Exp: t = R(qp) te + tp, q = qp * qe
    float tp[3], qp[4], rt[3];
    for (int i = 0; i < 3; ++i) tp[i] = (float)prev[i];
    for (int i = 0; i < 4; ++i) qp[i] = (float)prev[3 + i];
    qrot(qp, te, rt);
    const float ax = qp[0], ay = qp[1], az = qp[2], aw = qp[3], bx = qe[0], by = qe[1], bz = qe[2], bw = qe[3];
    const float q[4] = {aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                        aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz};
    for (int i = 0; i < 3; ++i) next_pose[i] = (double)(rt[i] + tp[i]);
    for (int i = 0; i < 4; ++i) next_pose[3 + i] = (double)q[i];
}

}  // namespace

extern "C" int macvo_posenet_input(const float* flow, const float* depth, int height, int width, double bl_fx, float* out,
                                   void* stream) {
    if (!flow || !depth || !out || height < PN_H || width < PN_W) return MACVO_E_ARG;
    // TartanStereoVOMotion.cropAndResize: crop to (112 s, 160 s), s = min(H // 112, W // 160), by centerCropTo
    // (Utility/Utils.py:67-72), which keeps size - 2 * ((size - target) // 2): one extra row / column for an odd margin
    const int s = min(height / PN_H, width / PN_W);
    const int my = (height - PN_H * s) / 2, mx = (width - PN_W * s) / 2;
    Crop c;
    c.y0 = my;
    c.x0 = mx;
    c.h = height - 2 * my;
    c.w = width - 2 * mx;
    c.sy = (float)(c.h - 1) / (float)(PN_H - 1);
    c.sx = (float)(c.w - 1) / (float)(PN_W - 1);
    posenet_input_kernel<<<ceil_div(PN_HW, 256), 256, 0, as_stream(stream)>>>(flow, depth, height, width, c, (float)bl_fx, out);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_posenet_conv(const float* x, int cin, int hi, int wi, const float* w_packed, const float* bias, int cout,
                                  int ksize, int stride, int pad, int co_tile, const float* resid, int relu, float* y,
                                  void* stream) {
    if (!x || !w_packed || !bias || !y || cin <= 0 || cin % SPLIT || hi <= 0 || wi <= 0 || cout <= 0 || ksize <= 0 ||
        stride <= 0 || pad < 0 || co_tile <= 0 || cout % co_tile)
        return MACVO_E_ARG;
    if ((reinterpret_cast<uintptr_t>(w_packed) & 15) || (co_tile * (cin / SPLIT) * ksize * ksize) % 4) return MACVO_E_ARG;
    const int ho = (hi + 2 * pad - ksize) / stride + 1, wo = (wi + 2 * pad - ksize) / stride + 1;
    if (ho <= 0 || wo <= 0) return MACVO_E_ARG;
    const size_t smem = conv_smem_bytes(cin, hi, wi, ho, wo, ksize, pad, co_tile);
    if (smem > 200 * 1024) return MACVO_E_UNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(posenet_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    ConvArgs a{x, w_packed, bias, resid, y, cin, hi, wi, cout, ho, wo, ksize, stride, pad, co_tile, relu ? 1 : 0};
    posenet_conv_kernel<<<dim3(SPLIT, cout / co_tile), CONV_NT, smem, as_stream(stream)>>>(a);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" size_t macvo_posenet_head_floats(void) { return HEAD_FLOATS; }

extern "C" int macvo_posenet_head(const float* fc1_out, const float* head_blob, const double* prev_pose, float* motion,
                                  double* next_pose, void* stream) {
    if (!fc1_out || !head_blob || !prev_pose || !motion || !next_pose) return MACVO_E_ARG;
    posenet_head_kernel<<<1, HEAD_NT, 0, as_stream(stream)>>>(fc1_out, head_blob, prev_pose, motion, next_pose);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
