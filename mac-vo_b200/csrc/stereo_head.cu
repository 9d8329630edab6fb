// TartanVODepth's two full-resolution heads and the depth conversion on the Hopper tensor cores (wgmma tf32), sm_90a:
//
//     per head:  out = conv_c13( relu( conv_c12( relu( deconv_c11( [x | cat0] ) ) ) ) )   (+ ReLU on the covariance head)
//     then:      disp = out_d / 0.02, depth = (1 / disp) * bf, var = bf^2 * ((out_c / disp^2) / disp^2)
//
// StereoNet.py:190-195, decoder.py:65-74 and StereoCovNet.inference (network.py:63-73). Unfused these are, per head, a
// torch.cat at half resolution, a 64-channel full-resolution deconvolution written to and read back from HBM, two 1x1
// convolutions and a string of elementwise passes. Here the three 64-channel half-resolution maps are read once and only
// depth and variance are written.
//
//   * deconv_c11 (k 4, s 2, p 1) as four dense GEMMs, one per output phase (py, px): output row 2m + py takes input rows
//     m + dy at kernel row py + 1 - 2 dy, dy in {0, -1} (py = 0) or {+1, 0} (py = 1); columns alike. K = 2 x 2 taps x 128
//     channels = 512, N = 64, M = the CTA's 8 x 8 half-resolution pixels. wgmma m64n64k8 tf32, both operands K-major
//     SWIZZLE_128B in shared memory, accumulators for all four phases in registers (4 x 32 per thread).
//   * K is walked 32 channels at a time ([x | cat0] in the reference's channel order). The chunk's 10 x 10 halo is staged
//     three times, shifted by dx = -1, 0, +1, as 80 K-major rows (halo row, column): the A operand of tap (dy, dx) is then
//     the dx copy from halo row 1 + dy on, a 1024-byte aligned start. Inputs are rounded to tf32 (nearest-even) on staging;
//     the weights are rounded once at load (ops.round_tf32) and arranged as (chunk, phase, tap, out, in % 32) blocks, which
//     stream through two 32 KB cp.async buffers.
//   * conv_c12 (64 -> 16) and conv_c13 (16 -> 1) run in FP32 FMA on the accumulator fragments: a pixel's 64 channels sit in
//     the 4 lanes of a quad, 2 shuffles reduce each of the 16 dot products. They are 2 % of the head's FLOPs; in registers
//     they need no second shared-memory staging.
//   * Epilogue in fp32 with IEEE division and reciprocal, in torch's operation order on the device (tensor / scalar is a
//     multiplication by the scalar's fp32 reciprocal; scalar / tensor is reciprocal() * scalar). Only the crop region of the
//     frame-sized outputs is written.
// No atomics; every output bit is a function of the inputs alone.
#include "tc_common.cuh"

namespace {

constexpr int SH_TILE = 8;                                   // 8 x 8 half-resolution pixels per CTA
constexpr int SH_THREADS = 128;                              // one warpgroup
constexpr int HALO = SH_TILE + 2;
constexpr int HALO_COPY = HALO * SH_TILE * 128;              // 10 x 8 rows x 128 B = 10 KB
constexpr int HALO_BYTES = 3 * HALO_COPY;
constexpr int W_TAP = 64 * 128;                              // 64 out x 32 in x 4 B
constexpr int W_BLOCK = 4 * W_TAP;                           // one (chunk, phase): 4 taps, 32 KB
constexpr int OFF_HALO = 2 * W_BLOCK, OFF_OUT = OFF_HALO + HALO_BYTES;
constexpr int SH_SMEM = OFF_OUT + 2 * 4 * 64 * 4 + 1024;    // + alignment slack
static_assert(HALO_COPY % 1024 == 0 && W_TAP % 1024 == 0, "swizzle atoms stay aligned");

constexpr uint32_t SW128_HI = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t sw128_lo(uint32_t a) { return ((a & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint64_t sw128(uint32_t lo) { return ((uint64_t)SW128_HI << 32) | lo; }

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
// ReLU as torch's: NaN passes through
__device__ __forceinline__ float relu(float v) { return v < 0.f ? 0.f : v; }

// block g of the weight stream (head g / 16, chunk (g % 16) / 4, phase g % 4) -> buffer g & 1
__device__ __forceinline__ void load_weights(uint32_t dst, const float* w11, int block) {
    const float* src = w11 + (long long)(block & 15) * (W_BLOCK / 4);
#pragma unroll
    for (int u = 0; u < W_BLOCK / 16 / SH_THREADS; ++u) {
        const int q = u * SH_THREADS + threadIdx.x, row = q >> 3, c16 = q & 7;
        cp_async16(dst + row * 128 + ((c16 ^ (row & 7)) << 4), src + q * 4);
    }
}

__global__ void __launch_bounds__(SH_THREADS, 2)
stereo_head_kernel(const float* __restrict__ xd, const float* __restrict__ xc, const float* __restrict__ cat0, int h2,
                   int w2, const float* __restrict__ w11_d, const float* __restrict__ small_d,
                   const float* __restrict__ w11_c, const float* __restrict__ small_c, float bf, float bf2, int my, int mx,
                   int H, int W, float* __restrict__ depth, float* __restrict__ var) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t s_base = smem_u32(smem), s_halo = s_base + OFF_HALO;
    float* out_s = reinterpret_cast<float*>(smem + OFF_OUT);    // [head][phase][pixel of the tile]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int y0 = blockIdx.y * SH_TILE, x0 = blockIdx.x * SH_TILE;
    const long long plane = (long long)h2 * w2;
    const int heads = xc ? 2 : 1, blocks = 16 * heads;
    const int fr = warp * 16 + (lane >> 2), fc = 2 * (lane & 3);     // fragment row / column base (wgmma_ops.cuh)
    float acc[4][32];

    load_weights(s_base, w11_d, 0);
    cp_async_commit();
    for (int head = 0; head < heads; ++head) {
        const float* x = head ? xc : xd;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
            for (int ph = 0; ph < 4; ++ph) {
                const int g = head * 16 + kc * 4 + ph;
                if (g + 1 < blocks) load_weights(s_base + ((g + 1) & 1) * W_BLOCK, (g + 1) < 16 ? w11_d : w11_c, g + 1);
                cp_async_commit();
                if (ph == 0) {
                    // the chunk's 32 channels of the 10 x 10 halo, tf32-rounded, into the three dx-shifted copies
                    const float* src = (kc < 2 ? x + kc * 32 * plane : cat0 + (kc - 2) * 32 * plane);
                    for (int e = tid; e < 32 * HALO * HALO; e += SH_THREADS) {
                        const int c = e / (HALO * HALO), hr = (e / HALO) % HALO, hc = e % HALO;
                        const int y = y0 - 1 + hr, xx = x0 - 1 + hc;
                        const float v = (y >= 0 && y < h2 && xx >= 0 && xx < w2) ? __ldg(src + c * plane + (long long)y * w2 + xx) : 0.f;
                        const uint32_t t = to_tf32(v);
#pragma unroll
                        for (int s = 0; s < 3; ++s) {
                            const int j = hc - s;
                            if (j >= 0 && j < SH_TILE) {
                                const int row = hr * SH_TILE + j;
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(s_halo + s * HALO_COPY + row * 128 +
                                                                             ((((c >> 2) ^ (row & 7))) << 4) + (c & 3) * 4),
                                             "r"(t) : "memory");
                            }
                        }
                    }
                }
                cp_async_wait1();                                  // this thread's copies of block g have landed
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncthreads();
                const uint32_t wb = s_base + (g & 1) * W_BLOCK;
                const int py = ph >> 1, px = ph & 1;
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 4; ++tap) {
                    const int ty = tap >> 1, tx = tap & 1;
                    const int dy = py == 0 ? -ty : 1 - ty, dx = px == 0 ? -tx : 1 - tx;
                    uint32_t ad = sw128_lo(s_halo + (dx + 1) * HALO_COPY + (dy + 1) * SH_TILE * 128);
                    uint32_t bd = sw128_lo(wb + tap * W_TAP);
                    asm volatile("" : "+r"(ad), "+r"(bd));
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        Wgmma<64>::tf32(acc[ph], sw128(ad + 2 * k), sw128(bd + 2 * k), (kc | tap | k) != 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_acc(acc[ph]);
                __syncthreads();                                   // buffer g & 1 and the halo may be refilled
            }
        }

        // + b11, ReLU, conv_c12 (quad-reduced dot products), ReLU, conv_c13 (+ ReLU on the covariance head), per pixel
        const float* sm = head ? small_c : small_d;
        const float *b11 = sm, *w12 = sm + 64, *b12 = sm + 64 + 1024, *w13 = b12 + 16;
        const float b13 = __ldg(w13 + 16);
#pragma unroll
        for (int ph = 0; ph < 4; ++ph) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float h[16];
#pragma unroll
                for (int q = 0; q < 16; ++q) {
                    const int i = (q >> 1) * 4 + half * 2 + (q & 1), c = 8 * (i >> 2) + fc + (i & 1);
                    h[q] = relu(acc[ph][i] + __ldg(b11 + c));
                }
                float o = b13;
#pragma unroll 4
                for (int j = 0; j < 16; ++j) {
                    float s = 0.f;
#pragma unroll
                    for (int q = 0; q < 16; ++q) {
                        const int i = (q >> 1) * 4 + half * 2 + (q & 1), c = 8 * (i >> 2) + fc + (i & 1);
                        s = fmaf(__ldg(w12 + j * 64 + c), h[q], s);
                    }
                    s += __shfl_xor_sync(0xffffffffu, s, 1);
                    s += __shfl_xor_sync(0xffffffffu, s, 2);
                    o = fmaf(__ldg(w13 + j), relu(s + __ldg(b12 + j)), o);
                }
                if ((lane & 3) == 0) out_s[(head * 4 + ph) * 64 + fr + 8 * half] = head ? relu(o) : o;
            }
        }
    }
    __syncthreads();

    // depth and variance of the tile's 4 x 64 output pixels, written at the crop offset of the frame
    for (int e = tid; e < 4 * 64; e += SH_THREADS) {
        const int ph = e >> 6, r = e & 63, m = y0 + (r >> 3), n = x0 + (r & 7);
        if (m >= h2 || n >= w2) continue;
        const long long o = (long long)(my + 2 * m + (ph >> 1)) * W + mx + 2 * n + (ph & 1);
        const float disp = __fmul_rn(out_s[ph * 64 + r], 1.0f / 0.02f);
        depth[o] = __fmul_rn(__frcp_rn(disp), bf);
        if (heads == 2) {
            const float d2 = __fmul_rn(disp, disp);
            var[o] = __fmul_rn(bf2, __fdiv_rn(__fdiv_rn(out_s[(4 + ph) * 64 + r], d2), d2));
        }
    }
}

}  // namespace

int macvo_stereo_head(const float* xd, const float* xc, const float* cat0, int h2, int w2, const float* w11_d,
                      const float* small_d, const float* w11_c, const float* small_c, float bf, float bf2, int margin_y,
                      int margin_x, int height, int width, float* depth, float* var, void* stream) {
    if (!xd || !cat0 || !w11_d || !small_d || !depth || h2 <= 0 || w2 <= 0 || margin_y < 0 || margin_x < 0) return MACVO_E_ARG;
    if (xc && (!w11_c || !small_c || !var)) return MACVO_E_ARG;
    if ((long long)margin_y + 2LL * h2 > height || (long long)margin_x + 2LL * w2 > width) return MACVO_E_ARG;
    for (const void* p : {(const void*)w11_d, (const void*)w11_c})
        if (reinterpret_cast<uintptr_t>(p) & 15) return MACVO_E_ARG;
    // the attribute belongs to the current device, so it is set on every launch (host-only, allowed under graph capture)
    MACVO_CUDA_TRY(cudaFuncSetAttribute(stereo_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM));
    const dim3 grid(ceil_div(w2, SH_TILE), ceil_div(h2, SH_TILE));
    stereo_head_kernel<<<grid, SH_THREADS, SH_SMEM, as_stream(stream)>>>(xd, xc, cat0, h2, w2, w11_d, small_d, w11_c,
                                                                        small_c, bf, bf2, margin_y, margin_x, height,
                                                                        width, depth, var);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
