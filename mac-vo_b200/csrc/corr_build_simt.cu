// (a3) all-pairs correlation volume, fp32 CUDA-core baseline (MACVO_CORR_SIMT).
//
// Replaces MemoryEncoder.corr (Module/Network/FlowFormer/core/encoder.py:256-275):
//   corr[b, i, j] = sum_d f1[b, d, i] * f2[b, d, j],   f1, f2: (B, D, N) row-major (NCHW feature maps).
// Both operands arrive "MN-major" (token index contiguous), i.e. C = F1^T F2, so global loads are
// coalesced along the token axis for both tiles. 128x128 output tile per CTA, 8x8 per thread, K-step 16.
// This kernel is the reference-accuracy arm: true fp32 FMA accumulation, any N and D. It is
// compute-bound (~116 flop/B, SURVEY.md §7.3); the roofline kernel is corr_build_tc.cu (wgmma).
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 16, TH = 256;

__global__ void __launch_bounds__(TH)
corr_simt_kernel(const float* __restrict__ f1, const float* __restrict__ f2, float* __restrict__ corr, int dim, int n) {
    __shared__ __align__(16) float As[2][BK][BM];
    __shared__ __align__(16) float Bs[2][BK][BN];
    const int b = blockIdx.z;
    const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
    const float* A = f1 + (long long)b * dim * n;
    const float* Bm = f2 + (long long)b * dim * n;
    float* C = corr + (long long)b * n * n;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;

    float acc[8][8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;

    // loader mapping: 2048 floats per operand tile, 8 per thread: row = tid / 16, 8 consecutive tokens
    const int lr = tid >> 4, lc = (tid & 15) * 8;
    auto load_tile = [&](int buf, int k0) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            int d = k0 + lr, i = i0 + lc + e, j = j0 + lc + e;
            As[buf][lr][lc + e] = (d < dim && i < n) ? __ldg(A + (long long)d * n + i) : 0.f;
            Bs[buf][lr][lc + e] = (d < dim && j < n) ? __ldg(Bm + (long long)d * n + j) : 0.f;
        }
    };

    const int nk = ceil_div(dim, BK);
    load_tile(0, 0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int cur = kt & 1;
        if (kt + 1 < nk) load_tile(cur ^ 1, (kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[8], bb[8];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w; bb[4] = b1.x; bb[5] = b1.y; bb[6] = b1.z; bb[7] = b1.w;
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(a[r], bb[c], acc[r][c]);
        }
        __syncthreads();
    }

#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int i = i0 + (r < 4 ? ty * 4 + r : 64 + ty * 4 + (r - 4));
        if (i >= n) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = j0 + h * 64 + tx * 4;
            float* dst = C + (long long)i * n + j;
            if (j + 3 < n && ((n & 3) == 0)) {
                *reinterpret_cast<float4*>(dst) = make_float4(acc[r][h * 4], acc[r][h * 4 + 1], acc[r][h * 4 + 2], acc[r][h * 4 + 3]);
            } else {
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (j + c < n) dst[c] = acc[r][h * 4 + c];
            }
        }
    }
}

}  // namespace

int macvo_corr_build_simt(const float* f1, const float* f2, float* corr, int batch, int dim, int n, cudaStream_t st) {
    dim3 grid(ceil_div(n, BN), ceil_div(n, BM), batch);
    corr_simt_kernel<<<grid, TH, 0, st>>>(f1, f2, corr, dim, n);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
