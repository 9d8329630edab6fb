// Frontend "next" row (SURVEY.md §8f-2): the elementwise glue of one MemoryDecoder refinement iteration
// (Module/Network/FlowFormer/core/gru.py:22-43 SepConvGRU, gma.py:84-130 Aggregate, covhead.py:95-131),
// fused so that the recurrent state lives in NHWC [h | x] buffers the cuDNN convolutions read in place:
//
//   gru_input   x = [inp | mf | mf + gamma * agg] written into the x-part (channels 128..511) of the 4 GRU input
//               buffers ([h|x] and [r*h|x] for the flow GRU and for the covariance GRU) — replaces 2 torch.cat
//               + mul + add per iteration and 8 torch.cat per GRU pass
//   gru_gates   z = sigmoid(zr[:, :128]);  [r*h | x] buffer <- sigmoid(zr[:, 128:]) * h
//   gru_blend   h <- (1 - z) * h + z * tanh(q), written to the [h|x] buffer and to a dense (P,128) copy
//
// All tensors fp32, pixels-major (P = B*H*W rows). Exact same arithmetic as the torch ops, one rounding each
// (sigmoid = 1 / (1 + exp(-x)) and tanhf at ATen's fp32 accuracy), parity in tests/test_gpu_nn_kernels.py.
#include "common.cuh"
#include <cuda_fp16.h>

namespace {

constexpr int HID = 128;          // hidden channels of SepConvGRU
constexpr int GRU_IN = 512;       // [h (128) | x (384)]

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__global__ void __launch_bounds__(256)
gru_input_kernel(const float* __restrict__ mf, const float* __restrict__ agg, const float* __restrict__ gamma,
                 float* __restrict__ b0, float* __restrict__ b1, float* __restrict__ b2, float* __restrict__ b3,
                 long long pixels) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // one float4 of one pixel's 128 channels
    if (e >= pixels * (HID / 4)) return;
    const long long p = e / (HID / 4);
    const int c = (int)(e % (HID / 4)) * 4;
    const float g = __ldg(gamma);
    const float4 m = *reinterpret_cast<const float4*>(mf + p * HID + c);
    const float4 a = *reinterpret_cast<const float4*>(agg + p * HID + c);
    const float4 s = make_float4(fmaf(g, a.x, m.x), fmaf(g, a.y, m.y), fmaf(g, a.z, m.z), fmaf(g, a.w, m.w));
    float* bufs[4] = {b0, b1, b2, b3};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (!bufs[i]) continue;
        *reinterpret_cast<float4*>(bufs[i] + p * GRU_IN + 2 * HID + c) = m;
        *reinterpret_cast<float4*>(bufs[i] + p * GRU_IN + 3 * HID + c) = s;
    }
}

__global__ void __launch_bounds__(256)
gru_gates_kernel(const float* __restrict__ zr, const float* __restrict__ bias, const float* __restrict__ hx,
                 float* __restrict__ z_out, float* __restrict__ rhx, long long pixels) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= pixels * (HID / 4)) return;
    const long long p = e / (HID / 4);
    const int c = (int)(e % (HID / 4)) * 4;
    float4 zz = *reinterpret_cast<const float4*>(zr + p * 2 * HID + c);
    float4 rr = *reinterpret_cast<const float4*>(zr + p * 2 * HID + HID + c);
    if (bias) {                                                     // conv bias folded in (conv launched without one)
        const float4 bz = *reinterpret_cast<const float4*>(bias + c), br = *reinterpret_cast<const float4*>(bias + HID + c);
        zz = make_float4(zz.x + bz.x, zz.y + bz.y, zz.z + bz.z, zz.w + bz.w);
        rr = make_float4(rr.x + br.x, rr.y + br.y, rr.z + br.z, rr.w + br.w);
    }
    const float4 h = *reinterpret_cast<const float4*>(hx + p * GRU_IN + c);
    *reinterpret_cast<float4*>(z_out + p * HID + c) =
        make_float4(sigmoidf_(zz.x), sigmoidf_(zz.y), sigmoidf_(zz.z), sigmoidf_(zz.w));
    *reinterpret_cast<float4*>(rhx + p * GRU_IN + c) =
        make_float4(sigmoidf_(rr.x) * h.x, sigmoidf_(rr.y) * h.y, sigmoidf_(rr.z) * h.z, sigmoidf_(rr.w) * h.w);
}

__global__ void __launch_bounds__(256)
gru_blend_kernel(const float* __restrict__ q, const float* __restrict__ bias, const float* __restrict__ z,
                 float* __restrict__ hx, float* __restrict__ h_dense, long long pixels) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= pixels * (HID / 4)) return;
    const long long p = e / (HID / 4);
    const int c = (int)(e % (HID / 4)) * 4;
    float4 qq = *reinterpret_cast<const float4*>(q + p * HID + c);
    if (bias) {
        const float4 bq = *reinterpret_cast<const float4*>(bias + c);
        qq = make_float4(qq.x + bq.x, qq.y + bq.y, qq.z + bq.z, qq.w + bq.w);
    }
    const float4 zz = *reinterpret_cast<const float4*>(z + p * HID + c);
    const float4 h = *reinterpret_cast<const float4*>(hx + p * GRU_IN + c);
    float4 o;                                    // (1 - z) * h + z * tanh(q), same association as gru.py:33,41
    o.x = (1.f - zz.x) * h.x + zz.x * tanhf(qq.x);
    o.y = (1.f - zz.y) * h.y + zz.y * tanhf(qq.y);
    o.z = (1.f - zz.z) * h.z + zz.z * tanhf(qq.z);
    o.w = (1.f - zz.w) * h.w + zz.w * tanhf(qq.w);
    *reinterpret_cast<float4*>(hx + p * GRU_IN + c) = o;
    if (h_dense) *reinterpret_cast<float4*>(h_dense + p * HID + c) = o;
}

inline unsigned grid_for(long long pixels) { return (unsigned)((pixels * (HID / 4) + 255) / 256); }

}  // namespace

extern "C" int macvo_gru_input(const float* mf, const float* agg, const float* gamma, float* buf0, float* buf1,
                               float* buf2, float* buf3, long long pixels, void* stream) {
    if (!mf || !agg || !gamma || !buf0 || pixels < 0) return MACVO_E_ARG;
    if (pixels == 0) return MACVO_OK;
    gru_input_kernel<<<grid_for(pixels), 256, 0, as_stream(stream)>>>(mf, agg, gamma, buf0, buf1, buf2, buf3, pixels);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_gru_gates(const float* zr, const float* bias, const float* hx, float* z_out, float* rhx,
                               long long pixels, void* stream) {
    if (!zr || !hx || !z_out || !rhx || pixels < 0) return MACVO_E_ARG;
    if (pixels == 0) return MACVO_OK;
    gru_gates_kernel<<<grid_for(pixels), 256, 0, as_stream(stream)>>>(zr, bias, hx, z_out, rhx, pixels);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_gru_blend(const float* q, const float* bias, const float* z, float* hx, float* h_dense,
                               long long pixels, void* stream) {
    if (!q || !z || !hx || pixels < 0) return MACVO_E_ARG;
    if (pixels == 0) return MACVO_OK;
    gru_blend_kernel<<<grid_for(pixels), 256, 0, as_stream(stream)>>>(q, bias, z, hx, h_dense, pixels);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

// ---- GMA attention matrix (gma.py:39-82): row softmax of the (B N) x N similarity scores, written as fp16 ------------------------
// The N x N matrix (184 MB fp32 at 640x480) is re-read by every iteration's aggregation GEMM, so under TF32 it is kept in fp16
// (values in [0, 1]); torch needed softmax (read + write fp32) + a cast (read fp32, write fp16) for that. One CTA per row: the row
// is read ONCE into registers, max / sum are block reductions, the normalised row is written as fp16.
namespace {
constexpr int SM_THREADS = 256, SM_MAX_V4 = 8;                    // up to 256 * 8 * 4 = 8192 columns per row

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float t = __shfl_xor_sync(0xffffffffu, v, o);
        v = is_max ? fmaxf(v, t) : v + t;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();                                               // `red` may still be read from the previous reduction
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = red[0];
#pragma unroll
    for (int w = 1; w < SM_THREADS / 32; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
    return r;
}

__global__ void __launch_bounds__(SM_THREADS)
softmax_rows_f16_kernel(const float* __restrict__ x, __half* __restrict__ out, int cols) {
    __shared__ float red[SM_THREADS / 32];
    const float4* row = reinterpret_cast<const float4*>(x + (long long)blockIdx.x * cols);
    const int quads = cols >> 2;
    float4 v[SM_MAX_V4];
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < SM_MAX_V4; ++i) {
        const int q = threadIdx.x + i * SM_THREADS;
        if (q < quads) {
            v[i] = __ldg(row + q);
            m = fmaxf(fmaxf(m, fmaxf(v[i].x, v[i].y)), fmaxf(v[i].z, v[i].w));
        }
    }
    m = block_reduce(m, true, red);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < SM_MAX_V4; ++i) {
        const int q = threadIdx.x + i * SM_THREADS;
        if (q < quads) {
            v[i].x = expf(v[i].x - m); v[i].y = expf(v[i].y - m); v[i].z = expf(v[i].z - m); v[i].w = expf(v[i].w - m);
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    }
    s = block_reduce(s, false, red);
    const float inv = 1.f / s;
    uint2* o = reinterpret_cast<uint2*>(out + (long long)blockIdx.x * cols);
#pragma unroll
    for (int i = 0; i < SM_MAX_V4; ++i) {
        const int q = threadIdx.x + i * SM_THREADS;
        if (q < quads) {
            __half2 h[2] = {__floats2half2_rn(v[i].x * inv, v[i].y * inv), __floats2half2_rn(v[i].z * inv, v[i].w * inv)};
            o[q] = *reinterpret_cast<uint2*>(h);
        }
    }
}
}  // namespace

extern "C" int macvo_softmax_rows_f16(const float* scores, void* out, long long rows, int cols, void* stream) {
    if (!scores || !out || rows < 0 || cols <= 0 || cols % 4 || cols > SM_THREADS * SM_MAX_V4 * 4) return MACVO_E_ARG;
    if (rows == 0) return MACVO_OK;
    softmax_rows_f16_kernel<<<(unsigned)rows, SM_THREADS, 0, as_stream(stream)>>>(scores, static_cast<__half*>(out), cols);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

// ---- convex upsampling (core/decoder.py:131-139, `upsample_flow`): 8x, softmax over the 9 neighbours ---------------------------
//   out[n, c, 8y + i, 8x + j] = sum_k softmax_k(scale * mask[n, k*64 + i*8 + j, y, x]) * 8 * flow[n, c, y + k/3 - 1, x + k%3 - 1]
// (zero outside). mask: channels_last (N, 576, H, W) = 576 contiguous logits per pixel; one warp per pixel, two sub-pixels per lane.
// Replaces scale, reshape, softmax, unfold, multiply, sum, permute + copy (10 launches over a 22 MB tensor) per map.
namespace {
__global__ void __launch_bounds__(256)
convex_upsample_kernel(const float* __restrict__ flow, const float* __restrict__ mask, float* __restrict__ out, float scale, int batch,
                       int height, int width) {
    const int lane = threadIdx.x & 31;
    const long long pix = (long long)blockIdx.x * 8 + (threadIdx.x >> 5), hw = (long long)height * width;
    if (pix >= (long long)batch * hw) return;
    const int n = (int)(pix / hw), y = (int)((pix - n * hw) / width), x = (int)(pix - n * hw - (long long)y * width);
    float f0[9], f1[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
        const bool in = yy >= 0 && yy < height && xx >= 0 && xx < width;
        f0[k] = in ? 8.f * __ldg(flow + ((long long)n * 2 + 0) * hw + (long long)yy * width + xx) : 0.f;
        f1[k] = in ? 8.f * __ldg(flow + ((long long)n * 2 + 1) * hw + (long long)yy * width + xx) : 0.f;
    }
    const float* m = mask + pix * 576;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int sub = lane + 32 * s, i = sub >> 3, j = sub & 7;          // sub-pixel (i, j) of the 8 x 8 block
        float l[9], mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < 9; ++k) { l[k] = scale * __ldg(m + k * 64 + sub); mx = fmaxf(mx, l[k]); }
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) { l[k] = expf(l[k] - mx); sum += l[k]; }
        float o0 = 0.f, o1 = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) { const float w = l[k] / sum; o0 += w * f0[k]; o1 += w * f1[k]; }
        const long long row = (long long)(8 * y + i) * (8 * width) + 8 * x + j, plane = 64 * hw;
        out[((long long)n * 2 + 0) * plane + row] = o0;
        out[((long long)n * 2 + 1) * plane + row] = o1;
    }
}
}  // namespace

extern "C" int macvo_convex_upsample(const float* flow, const float* mask_nhwc, float* out, float scale, int batch, int height,
                                     int width, void* stream) {
    if (!flow || !mask_nhwc || !out || batch <= 0 || height <= 0 || width <= 0) return MACVO_E_ARG;
    const long long pixels = (long long)batch * height * width;
    convex_upsample_kernel<<<(unsigned)((pixels + 7) / 8), 256, 0, as_stream(stream)>>>(flow, mask_nhwc, out, scale, batch, height, width);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
