// LayerNorm of one C = 32 * VPL channel row held by a warp, shared by the warp-per-row LayerNorm (nn_kernels.cu) and the
// PatchEmbed token head (patch_tokens_tc.cu) so that both compute the same bits: lane owns the float4 chunks lane + 32 i of
// the row, as v[4 i .. 4 i + 3]; on return v holds the normalised values at the same positions.
#pragma once
#include "common.cuh"

template <int VPL>
__device__ __forceinline__ void layer_norm_row(float (&v)[VPL], const float* __restrict__ w, const float* __restrict__ b,
                                               float eps, int lane) {
    constexpr int C = 32 * VPL;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i) s += (v[4 * i] + v[4 * i + 1]) + (v[4 * i + 2] + v[4 * i + 3]);
    const float mean = warp_sum(s) * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) { const float d = v[i] - mean; q = fmaf(d, d, q); }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + eps);
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i) {
        const int c = (lane + 32 * i) * 4;
        const float4 ww = *reinterpret_cast<const float4*>(w + c), bb = *reinterpret_cast<const float4*>(b + c);
        v[4 * i] = (v[4 * i] - mean) * rstd * ww.x + bb.x;
        v[4 * i + 1] = (v[4 * i + 1] - mean) * rstd * ww.y + bb.y;
        v[4 * i + 2] = (v[4 * i + 2] - mean) * rstd * ww.z + bb.z;
        v[4 * i + 3] = (v[4 * i + 3] - mean) * rstd * ww.w + bb.w;
    }
}
