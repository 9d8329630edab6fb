// PWC-Net's warp + 81-displacement cost volume + LeakyReLU(0.1) for one pyramid level (TartanVO's PWCDCNet_Adapted,
// pwc_model_tartanvo.py:176-212, 230-232, 259-260, and its correlation kernel, correlation.py:35-102, 277-318).
//
// One CTA per 8 x 32 output tile. Before the channel loop the CTA computes, once, the bilinear taps of every position of the
// tile plus its 4-pixel halo (16 x 40 positions): tap weights, in-bounds flags and the warp mask, in fp32 and in the order
// torch's warp() / grid_sample take them. Then, for each chunk of 8 channels, it stages the *warped* f2 values of the halo
// tile in shared memory (each warped value is computed once, not once per displacement) and every thread — one output pixel —
// adds f1[c, y, x] * g[c, y + dy, x + dx] into its 81 fp32 accumulators. The epilogue divides by C, applies LeakyReLU(0.1)
// and stores 81 coalesced planes at channel offset `out_offset` of `out`.
#include "common.cuh"

#include <math.h>

namespace {

constexpr int kTileH = 8, kTileW = 32, kHalo = 4;
constexpr int kHaloH = kTileH + 2 * kHalo, kHaloW = kTileW + 2 * kHalo;   // 16 x 40
constexpr int kPos = kHaloH * kHaloW;                                        // 640 staged positions
constexpr int kChunk = 8;                                                    // channels per staging round
constexpr int kThreads = kTileH * kTileW;
constexpr int kDisp = 81;

// tap flags: which of nw / ne / sw / se lies inside f2; kDirect = no warp (g = f2 at that pixel)
constexpr unsigned kNW = 1u, kNE = 2u, kSW = 4u, kSE = 8u, kDirect = 16u;

__global__ void __launch_bounds__(kThreads)
pwc_warp_corr_kernel(const float* __restrict__ f1, const float* __restrict__ f2, const float* __restrict__ flow,
                     float flow_scale, int C, int H, int W, float* __restrict__ out, int out_channels, int out_offset) {
    __shared__ float s_w[4][kPos];          // nw, ne, sw, se weights
    __shared__ float s_m[kPos];             // warp mask (0 / 1); 0 for positions outside the image
    __shared__ int s_base[kPos];            // f2 plane offset of the nw tap (or of the pixel itself when kDirect)
    __shared__ unsigned char s_flags[kPos];
    __shared__ float s_g[kChunk][kPos];

    const int tid = threadIdx.x;
    const int tx = tid % kTileW, ty = tid / kTileW;
    const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
    const int b = blockIdx.z;
    const size_t plane = (size_t)H * W;

    // ---- taps of the halo tile (channel independent) ----
    for (int p = tid; p < kPos; p += kThreads) {
        const int gy = y0 - kHalo + p / kHaloW, gx = x0 - kHalo + p % kHaloW;
        float w0 = 0.f, w1 = 0.f, w2 = 0.f, w3 = 0.f, m = 0.f;
        int base = 0;
        unsigned flags = 0;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            if (flow == nullptr) {
                flags = kDirect;
                base = gy * W + gx;
                m = 1.f;
            } else {
                const float* fl = flow + (size_t)b * 2 * plane + (size_t)gy * W + gx;
                // warp(): vgrid = grid + flo, then 2 * v / max(W - 1, 1) - 1 (fp32 tensor ops, no contraction)
                const float vx = __fadd_rn((float)gx, __fmul_rn(flow_scale, fl[0]));
                const float vy = __fadd_rn((float)gy, __fmul_rn(flow_scale, fl[plane]));
                const float nx = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, vx), (float)max(W - 1, 1)), 1.f);
                const float ny = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, vy), (float)max(H - 1, 1)), 1.f);
                // grid_sample, align_corners=True: ((g + 1) / 2) * (size - 1)
                const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(nx, 1.f), 2.f), (float)(W - 1));
                const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(ny, 1.f), 2.f), (float)(H - 1));
                // in-bounds decisions in floating point, before any integer conversion; non-finite or |pos| > 2^24: no tap
                const float lim = 16777216.f;
                if (fabsf(ix) <= lim && fabsf(iy) <= lim) {          // false for NaN and +-inf
                    const float xw = floorf(ix), yn = floorf(iy);
                    const float xe = xw + 1.f, ys = yn + 1.f;          // exact below 2^24
                    const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1);
                    const bool inxw = xw >= 0.f && xw <= Wm1, inxe = xe >= 0.f && xe <= Wm1;
                    const bool inyn = yn >= 0.f && yn <= Hm1, inys = ys >= 0.f && ys <= Hm1;
                    // torch's nw / ne / sw / se weights
                    w0 = __fmul_rn(__fsub_rn(xe, ix), __fsub_rn(ys, iy));
                    w1 = __fmul_rn(__fsub_rn(ix, xw), __fsub_rn(ys, iy));
                    w2 = __fmul_rn(__fsub_rn(xe, ix), __fsub_rn(iy, yn));
                    w3 = __fmul_rn(__fsub_rn(ix, xw), __fsub_rn(iy, yn));
                    flags = (inxw && inyn ? kNW : 0u) | (inxe && inyn ? kNE : 0u) | (inxw && inys ? kSW : 0u)
                          | (inxe && inys ? kSE : 0u);
                    // the mask: the same sampling of a ones tensor, summed in nw / ne / sw / se order
                    float s = 0.f;
                    if (flags & kNW) s = __fadd_rn(s, w0);
                    if (flags & kNE) s = __fadd_rn(s, w1);
                    if (flags & kSW) s = __fadd_rn(s, w2);
                    if (flags & kSE) s = __fadd_rn(s, w3);
                    m = s < 0.9999f ? 0.f : (s > 0.f ? 1.f : s);
                    if (flags) base = (int)yn * W + (int)xw;       // yn in [-1, H-1], xw in [-1, W-1]; read via in-bounds taps only
                }
            }
        }
        s_w[0][p] = w0; s_w[1][p] = w1; s_w[2][p] = w2; s_w[3][p] = w3;
        s_m[p] = m;
        s_base[p] = base;
        s_flags[p] = (unsigned char)flags;
    }

    const int y = y0 + ty, x = x0 + tx;
    const bool live = y < H && x < W;
    float acc[kDisp];
#pragma unroll
    for (int k = 0; k < kDisp; ++k) acc[k] = 0.f;

    const float* f1b = f1 + (size_t)b * C * plane;
    const float* f2b = f2 + (size_t)b * C * plane;
    for (int c0 = 0; c0 < C; c0 += kChunk) {
        const int nc = min(kChunk, C - c0);
        __syncthreads();                                        // taps ready / previous chunk consumed
        for (int i = tid; i < nc * kPos; i += kThreads) {
            const int cc = i / kPos, p = i % kPos;
            const unsigned fl = s_flags[p];
            const float* src = f2b + (size_t)(c0 + cc) * plane + s_base[p];
            float g;
            if (fl & kDirect) {
                g = src[0];
            } else {
                float v = 0.f;
                if (fl & kNW) v = fmaf(src[0], s_w[0][p], v);
                if (fl & kNE) v = fmaf(src[1], s_w[1][p], v);
                if (fl & kSW) v = fmaf(src[W], s_w[2][p], v);
                if (fl & kSE) v = fmaf(src[W + 1], s_w[3][p], v);
                g = v * s_m[p];                                 // multiply, not select: NaN * 0 stays NaN
            }
            s_g[cc][p] = g;
        }
        __syncthreads();
        for (int cc = 0; cc < nc; ++cc) {
            const float a = live ? f1b[(size_t)(c0 + cc) * plane + (size_t)y * W + x] : 0.f;
            const float* row = &s_g[cc][ty * kHaloW + tx];
#pragma unroll
            for (int dy = 0; dy < 9; ++dy) {
#pragma unroll
                for (int dx = 0; dx < 9; ++dx) acc[dy * 9 + dx] = fmaf(a, row[dy * kHaloW + dx], acc[dy * 9 + dx]);
            }
        }
    }

    if (!live) return;
    float* o = out + ((size_t)b * out_channels + out_offset) * plane + (size_t)y * W + x;
    const float inv = (float)C;
#pragma unroll
    for (int k = 0; k < kDisp; ++k) {
        const float v = acc[k] / inv;                           // the reference divides the channel sum by C
        o[(size_t)k * plane] = v > 0.f ? v : v * 0.1f;
    }
}

}  // namespace

extern "C" int macvo_pwc_warp_corr(const float* f1, const float* f2, const float* flow, float flow_scale, int batch,
                                   int channels, int height, int width, float* out, int out_channels, int out_offset,
                                   void* stream) {
    if (!f1 || !f2 || !out) return MACVO_E_ARG;
    if (batch <= 0 || channels <= 0 || height <= 0 || width <= 0 || out_channels <= 0) return MACVO_E_ARG;
    if (out_offset < 0 || out_offset > out_channels - kDisp) return MACVO_E_ARG;
    if ((long long)height * width > (1ll << 30) || batch > 65535 || ceil_div(height, kTileH) > 65535) return MACVO_E_ARG;
    dim3 grid(ceil_div(width, kTileW), ceil_div(height, kTileH), batch);
    pwc_warp_corr_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(f1, f2, flow, flow_scale, channels, height, width, out,
                                                                    out_channels, out_offset);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
