// Frontend "next" row (SURVEY.md §8f-2): the per-pixel token path of one MemoryDecoder refinement iteration as ONE
// kernel. Replaces, per iteration, 17 launches (two token-MLP GEMMs + GELU, the LayerNorm + sine-embedding kernel, the
// query projection, the single-query cross attention, concat, output projection, residual adds, LayerNorm, two FFN
// GEMMs + GELU, the 145-channel concat in front of the motion encoder):
//
//   query  = flow_token_encoder(cost_forward)            1x1 conv 81->64, GELU, 1x1 conv 64->64      decoder.py:112-116
//   q      = Wq (LayerNorm(query) + sine(coords1)) + bq                                              decoder.py:56-66
//   a      = softmax_j(q_h . k_jh / sqrt(8)) v_jh         8 heads x 8 cost-memory tokens of THIS pixel attention.py:6-29
//   g      = query + Wp [a | query] + bp ;  g += FFN(LayerNorm(g))                                   decoder.py:67-76
//   out    = [g (64) | cost_forward (81) | 0 (15)]        the motion encoder's `cat([cost_global, cost_forward])`
//                                                         (gru.py:53-54), zero padded to 160 channels so that convc1
//                                                         is an aligned GEMM
//
// Everything is per pixel, so a CTA owns 64 pixels end to end: activations stay in shared memory in a channel-major
// [c][pixel] layout, the six weight matrices (transposed, 119 KB) sit in shared memory for the whole tile, each stage
// is a register-tiled fp32 FMA GEMM (4 pixels x 4 outputs per thread, two LDS.128 per 16 FMA). fp32 throughout in BOTH
// precision modes (the chain it replaces ran TF32 tensor-core GEMMs under allow_tf32): 0.6 GFLOP per call, HBM/L2
// traffic = the lookup rows (3.1 MB), the keys / values (39 MB) and the output rows (6.1 MB) at 640x480.
#include "common.cuh"
#include "rows_layout.cuh"
#include <cuda_fp16.h>

namespace {

// TP pixels per CTA (template parameter: 64 or 72 — the host picks the one that needs fewer waves of one-CTA-per-SM blocks:
// e.g. 9000 pixels on 132 SMs: 141 tiles of 64 = TWO waves, 125 tiles of 72 = one), LD = TP + 4 row stride of the
// [channel][pixel] activation buffers (16-B aligned rows), 4 threads per pixel.
constexpr int C = 64, CF = 81, OUTC = 160;
// weight blob (floats): transposed matrices [K][64], then 10 vectors of 64, then 16 frequencies
constexpr int W_FTE0 = 0, W_FTE2 = W_FTE0 + CF * C, W_Q = W_FTE2 + C * C, W_PROJ = W_Q + C * C,
              W_FFN0 = W_PROJ + 2 * C * C, W_FFN3 = W_FFN0 + C * C, W_END = W_FFN3 + C * C;
constexpr int V_BFTE0 = W_END, V_BFTE2 = V_BFTE0 + C, V_LN1W = V_BFTE2 + C, V_LN1B = V_LN1W + C, V_BQ = V_LN1B + C,
              V_BPROJ = V_BQ + C, V_LN2W = V_BPROJ + C, V_LN2B = V_LN2W + C, V_BFFN0 = V_LN2B + C, V_BFFN3 = V_BFFN0 + C,
              V_FREQ = V_BFFN3 + C, BLOB = V_FREQ + 16;
template <int TP> struct Lay {
    static constexpr int LD = TP + 4, NT = 4 * TP;
    static constexpr int S_X0 = BLOB, S_CAT = S_X0 + CF * LD, S_A = S_CAT + 2 * C * LD, S_END = S_A + C * LD;
    static_assert(BLOB % 4 == 0 && S_X0 % 4 == 0 && S_CAT % 4 == 0 && S_A % 4 == 0, "float4 alignment");
    static_assert(S_END * 4 <= 227 * 1024, "shared memory budget");
};

// acc[o][p] += sum_k WT[k][4 og + o] * X[k][4 pg + p]
template <int K, int LD>
__device__ __forceinline__ void gemm_tile(const float* __restrict__ WT, const float* __restrict__ X, int og, int pg,
                                          float (&acc)[4][4]) {
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
        const float4 w = *reinterpret_cast<const float4*>(WT + k * C + 4 * og);
        const float4 x = *reinterpret_cast<const float4*>(X + k * LD + 4 * pg);
        acc[0][0] = fmaf(w.x, x.x, acc[0][0]); acc[0][1] = fmaf(w.x, x.y, acc[0][1]);
        acc[0][2] = fmaf(w.x, x.z, acc[0][2]); acc[0][3] = fmaf(w.x, x.w, acc[0][3]);
        acc[1][0] = fmaf(w.y, x.x, acc[1][0]); acc[1][1] = fmaf(w.y, x.y, acc[1][1]);
        acc[1][2] = fmaf(w.y, x.z, acc[1][2]); acc[1][3] = fmaf(w.y, x.w, acc[1][3]);
        acc[2][0] = fmaf(w.z, x.x, acc[2][0]); acc[2][1] = fmaf(w.z, x.y, acc[2][1]);
        acc[2][2] = fmaf(w.z, x.z, acc[2][2]); acc[2][3] = fmaf(w.z, x.w, acc[2][3]);
        acc[3][0] = fmaf(w.w, x.x, acc[3][0]); acc[3][1] = fmaf(w.w, x.y, acc[3][1]);
        acc[3][2] = fmaf(w.w, x.z, acc[3][2]); acc[3][3] = fmaf(w.w, x.w, acc[3][3]);
    }
}

enum Epi { EPI_BIAS, EPI_GELU, EPI_RESID };

// Y[4 og + o][4 pg + p] = epi(acc + bias [+ R])
template <int EPI, int LD>
__device__ __forceinline__ void store_tile(float* __restrict__ Y, const float* __restrict__ bias,
                                           const float* __restrict__ R, int og, int pg, float (&acc)[4][4]) {
#pragma unroll
    for (int o = 0; o < 4; ++o) {
        const float b = bias[4 * og + o];
        float4 v = make_float4(acc[o][0] + b, acc[o][1] + b, acc[o][2] + b, acc[o][3] + b);
        if (EPI == EPI_GELU) v = make_float4(gelu_erf(v.x), gelu_erf(v.y), gelu_erf(v.z), gelu_erf(v.w));
        if (EPI == EPI_RESID) {
            const float4 r = *reinterpret_cast<const float4*>(R + (4 * og + o) * LD + 4 * pg);
            v = make_float4(r.x + v.x, r.y + v.y, r.z + v.z, r.w + v.w);
        }
        *reinterpret_cast<float4*>(Y + (4 * og + o) * LD + 4 * pg) = v;
    }
}

__device__ __forceinline__ void zero(float (&acc)[4][4]) {
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[o][p] = 0.f;
}

// LayerNorm over the 64 channels of each pixel column of X, optional sine embedding added; 4 threads per pixel.
template <int LD>
__device__ __forceinline__ void layer_norm_cols(const float* __restrict__ X, float* __restrict__ Y,
                                                const float* __restrict__ w, const float* __restrict__ b, float eps,
                                                int px, int quarter, bool add_sine, float coord,
                                                const float* __restrict__ freq) {
    float v[16];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) { v[i] = X[(16 * quarter + i) * LD + px]; s += v[i]; }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    const float mean = s * (1.f / 64);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) { v[i] -= mean; q = fmaf(v[i], v[i], q); }
    q += __shfl_xor_sync(0xffffffffu, q, 1);
    q += __shfl_xor_sync(0xffffffffu, q, 2);
    const float rstd = rsqrtf(q * (1.f / 64) + eps);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int c = 16 * quarter + i;
        float y = v[i] * rstd * w[c] + b[c];
        if (add_sine) {   // LinearPositionEmbeddingSine, dim 64: [sin x f | cos x f | sin y f | cos y f]  (attention.py:71-101)
            const float a = __fmul_rn(coord, freq[i]);
            y = __fadd_rn(y, (quarter & 1) ? cosf(a) : sinf(a));
        }
        Y[c * LD + px] = y;
    }
}

template <int TP>
__global__ void __launch_bounds__(4 * TP, 1)
decoder_token_kernel(const float* __restrict__ cf, const float* __restrict__ coords, const float* __restrict__ key,
                     const float* __restrict__ value, const float* __restrict__ blob, float* __restrict__ out,
                     long long pixels, int n1, float eps, __half* __restrict__ out16, int height, int width) {
    extern __shared__ __align__(16) float sm[];
    using L = Lay<TP>;
    constexpr int LD = L::LD, NT = L::NT, S_X0 = L::S_X0, S_CAT = L::S_CAT, S_A = L::S_A;
    const int tid = threadIdx.x;
    const long long p0 = (long long)blockIdx.x * TP;
    const int valid = (int)min((long long)TP, pixels - p0);

    float* X0 = sm + S_X0;        // cost_forward tile, [81][LD]
    float* CAT = sm + S_CAT;      // rows 0..63: q -> a -> LN(g);  rows 64..127: query -> FFN hidden
    float* A = sm + S_A;          // token hidden -> q_in -> g
    // ---- asynchronous fill: with one 8-warp CTA per SM every synchronous load round trip is exposed, so
    //   * the 119 KB weight blob arrives by ONE bulk copy (TMA engine) signalled on an mbarrier,
    //   * the (64 x 81) lookup rows are staged with 16-byte cp.async into the (still unused) CAT buffer and transposed
    //     shared -> shared afterwards,
    //   * this tile's keys / values (256 KB, needed ~10 us later) are pulled into L2 with prefetch hints.
    __shared__ __align__(8) unsigned long long s_bar;
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&s_bar);
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(BLOB * 4) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"((uint32_t)__cvta_generic_to_shared(sm)), "l"(blob), "r"(BLOB * 4), "r"(bar) : "memory");
    }
    const float* cft = cf + p0 * CF;
    const int nfl = valid * CF;                                        // contiguous floats of this tile's lookup rows
    {
        const uint32_t stage = (uint32_t)__cvta_generic_to_shared(CAT);
        for (int e = tid; e < nfl / 4; e += NT)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(stage + 16 * e), "l"(cft + 4 * e) : "memory");
        for (int e = (nfl / 4) * 4 + tid; e < nfl; e += NT) CAT[e] = __ldg(cft + e);
        asm volatile("cp.async.commit_group;" ::: "memory");
        const char* kb = reinterpret_cast<const char*>(key + p0 * 8 * C);
        const char* vb = reinterpret_cast<const char*>(value + p0 * 8 * C);
        for (int l = tid; l < valid * 16; l += NT) {                   // 8 tokens x 64 floats = 2 KB = 16 lines per pixel
            asm volatile("prefetch.global.L2 [%0];" ::"l"(kb + 128 * l));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(vb + 128 * l));
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    for (int e = tid; e < TP * CF; e += NT) {                          // staged rows -> channel-major [k][pixel]
        const int px = e / CF, k = e - px * CF;
        X0[k * LD + px] = px < valid ? CAT[e] : 0.f;
    }
    {   // weights landed?
        uint32_t ok = 0;
        while (!ok)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(ok) : "r"(bar) : "memory");
    }
    __syncthreads();

    const int og = tid & 15, pg = tid >> 4;            // GEMM micro-tile owner
    const int px = tid >> 2, quarter = tid & 3;        // per-pixel stages: 4 threads per pixel
    float acc[4][4];

    // token MLP: hidden = GELU(W0 cf + b0) -> A ; query = W2 hidden + b2 -> CAT[64..]
    zero(acc);
    gemm_tile<CF, LD>(sm + W_FTE0, X0, og, pg, acc);
    store_tile<EPI_GELU, LD>(A, sm + V_BFTE0, nullptr, og, pg, acc);
    __syncthreads();
    zero(acc);
    gemm_tile<C, LD>(sm + W_FTE2, A, og, pg, acc);
    store_tile<EPI_BIAS, LD>(CAT + C * LD, sm + V_BFTE2, nullptr, og, pg, acc);
    __syncthreads();

    // q_in = LayerNorm(query) + sine(coords1) -> A
    {
        const long long p = p0 + px;
        float coord = 0.f;
        if (px < valid) {
            const long long bi = p / n1, pi = p - bi * n1;
            coord = coords[(bi * 2 + (quarter >> 1)) * n1 + pi];        // quarters 0,1 embed x; 2,3 embed y
        }
        layer_norm_cols<LD>(CAT + C * LD, A, sm + V_LN1W, sm + V_LN1B, eps, px, quarter, true, coord, sm + V_FREQ);
    }
    __syncthreads();
    // q = Wq q_in + bq -> CAT[0..63]
    zero(acc);
    gemm_tile<C, LD>(sm + W_Q, A, og, pg, acc);
    store_tile<EPI_BIAS, LD>(CAT, sm + V_BQ, nullptr, og, pg, acc);
    __syncthreads();

    // cross attention of this pixel's query to its own 8 cost-memory tokens; this thread: heads 2*quarter, 2*quarter+1
    {
        float qv[16], av[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) { qv[i] = CAT[(16 * quarter + i) * LD + px] * 0.35355339059327376f; av[i] = 0.f; }
        if (px < valid) {
            const float* kp = key + ((p0 + px) * 8) * C + 16 * quarter;
            const float* vp = value + ((p0 + px) * 8) * C + 16 * quarter;
            float s0[8], s1[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 k0 = __ldg(reinterpret_cast<const float4*>(kp + j * C));
                const float4 k1 = __ldg(reinterpret_cast<const float4*>(kp + j * C + 4));
                const float4 k2 = __ldg(reinterpret_cast<const float4*>(kp + j * C + 8));
                const float4 k3 = __ldg(reinterpret_cast<const float4*>(kp + j * C + 12));
                s0[j] = qv[0] * k0.x + qv[1] * k0.y + qv[2] * k0.z + qv[3] * k0.w + qv[4] * k1.x + qv[5] * k1.y + qv[6] * k1.z + qv[7] * k1.w;
                s1[j] = qv[8] * k2.x + qv[9] * k2.y + qv[10] * k2.z + qv[11] * k2.w + qv[12] * k3.x + qv[13] * k3.y + qv[14] * k3.z + qv[15] * k3.w;
            }
            float m0 = s0[0], m1 = s1[0];
#pragma unroll
            for (int j = 1; j < 8; ++j) { m0 = fmaxf(m0, s0[j]); m1 = fmaxf(m1, s1[j]); }
            float d0 = 0.f, d1 = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) { s0[j] = expf(s0[j] - m0); d0 += s0[j]; s1[j] = expf(s1[j] - m1); d1 += s1[j]; }
            const float i0 = 1.f / d0, i1 = 1.f / d1;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float w0 = s0[j] * i0, w1 = s1[j] * i1;
                const float4 v0 = __ldg(reinterpret_cast<const float4*>(vp + j * C));
                const float4 v1 = __ldg(reinterpret_cast<const float4*>(vp + j * C + 4));
                const float4 v2 = __ldg(reinterpret_cast<const float4*>(vp + j * C + 8));
                const float4 v3 = __ldg(reinterpret_cast<const float4*>(vp + j * C + 12));
                av[0] = fmaf(w0, v0.x, av[0]); av[1] = fmaf(w0, v0.y, av[1]); av[2] = fmaf(w0, v0.z, av[2]); av[3] = fmaf(w0, v0.w, av[3]);
                av[4] = fmaf(w0, v1.x, av[4]); av[5] = fmaf(w0, v1.y, av[5]); av[6] = fmaf(w0, v1.z, av[6]); av[7] = fmaf(w0, v1.w, av[7]);
                av[8] = fmaf(w1, v2.x, av[8]); av[9] = fmaf(w1, v2.y, av[9]); av[10] = fmaf(w1, v2.z, av[10]); av[11] = fmaf(w1, v2.w, av[11]);
                av[12] = fmaf(w1, v3.x, av[12]); av[13] = fmaf(w1, v3.y, av[13]); av[14] = fmaf(w1, v3.z, av[14]); av[15] = fmaf(w1, v3.w, av[15]);
            }
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) CAT[(16 * quarter + i) * LD + px] = av[i];     // in place: same cells this thread read
    }
    __syncthreads();

    // g = query + Wp [a | query] + bp -> A
    zero(acc);
    gemm_tile<2 * C, LD>(sm + W_PROJ, CAT, og, pg, acc);
    store_tile<EPI_RESID, LD>(A, sm + V_BPROJ, CAT + C * LD, og, pg, acc);
    __syncthreads();
    // LN(g) -> CAT[0..63];  hidden = GELU(F0 LN(g) + b) -> CAT[64..];  g += F3 hidden + b (in place)
    layer_norm_cols<LD>(A, CAT, sm + V_LN2W, sm + V_LN2B, eps, px, quarter, false, 0.f, nullptr);
    __syncthreads();
    zero(acc);
    gemm_tile<C, LD>(sm + W_FFN0, CAT, og, pg, acc);
    store_tile<EPI_GELU, LD>(CAT + C * LD, sm + V_BFFN0, nullptr, og, pg, acc);
    __syncthreads();
    zero(acc);
    gemm_tile<C, LD>(sm + W_FFN3, CAT + C * LD, og, pg, acc);
    store_tile<EPI_RESID, LD>(A, sm + V_BFFN3, A, og, pg, acc);
    __syncthreads();

    if (out16 != nullptr) {
        // fp16 layout-U rows (csrc/rows_layout.cuh, 192 channels per row) for the tensor-core motion encoder: 2 channels per thread
        for (int e = tid; e < valid * (OUTC / 2); e += NT) {
            const int r = e / (OUTC / 2), c = 2 * (e - r * (OUTC / 2));
            auto val = [&](int ch) { return ch < C ? A[ch * LD + r] : (ch < C + CF ? X0[(ch - C) * LD + r] : 0.f); };
            const long long p = p0 + r;
            const int x = (int)(p % width), y = (int)((p / width) % height), b = (int)(p / ((long long)width * height));
            *reinterpret_cast<__half2*>(out16 + macvo_rows::urow(b, y, x, height, width) * 192 + c) = __floats2half2_rn(val(c), val(c + 1));
        }
        return;
    }
    // out rows [g | cost_forward | 0]: coalesced (consecutive threads -> consecutive floats of the (P,160) matrix)
    float* ot = out + p0 * OUTC;
    for (int e = tid; e < valid * OUTC; e += NT) {
        const int r = e / OUTC, c = e - r * OUTC;
        ot[e] = c < C ? A[c * LD + r] : (c < C + CF ? X0[(c - C) * LD + r] : 0.f);
    }
}

}  // namespace

extern "C" size_t macvo_decoder_token_blob_floats(void) { return BLOB; }

template <int TP>
static int launch_token(const float* cf, const float* coords, const float* key, const float* value, const float* blob,
                        float* out, long long pixels, int n1, float eps, cudaStream_t st, __half* out16 = nullptr, int height = 0,
                        int width = 0) {
    constexpr int smem = Lay<TP>::S_END * 4;
    MACVO_CUDA_TRY(cudaFuncSetAttribute(decoder_token_kernel<TP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    decoder_token_kernel<TP><<<(unsigned)((pixels + TP - 1) / TP), 4 * TP, smem, st>>>(cf, coords, key, value, blob, out, pixels, n1, eps, out16, height, width);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_decoder_token(const float* cost_forward, const float* coords, const float* key, const float* value,
                                   const float* weight_blob, float* out, int batch, int n1, float eps, void* stream) {
    if (!cost_forward || !coords || !key || !value || !weight_blob || !out || batch <= 0 || n1 <= 0) return MACVO_E_ARG;
    const long long pixels = (long long)batch * n1;
    int dev = 0, sms = 132;
    MACVO_CUDA_TRY(cudaGetDevice(&dev));
    MACVO_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    // one CTA per SM: cost ~ waves x pixels-per-tile
    auto cost = [&](int tp) { const long long tiles = (pixels + tp - 1) / tp; return ((tiles + sms - 1) / sms) * tp; };
    cudaStream_t st = as_stream(stream);
    return cost(72) < cost(64) ? launch_token<72>(cost_forward, coords, key, value, weight_blob, out, pixels, n1, eps, st)
                               : launch_token<64>(cost_forward, coords, key, value, weight_blob, out, pixels, n1, eps, st);
}

/* same, writing fp16 layout-U rows (rows, 192): channels [0,160) = [g | cost_forward | 0], the tensor-core motion encoder's input */
extern "C" int macvo_decoder_token_rows(const float* cost_forward, const float* coords, const float* key, const float* value,
                                        const float* weight_blob, void* out16_rows, int batch, int height, int width, float eps,
                                        void* stream) {
    if (!cost_forward || !coords || !key || !value || !weight_blob || !out16_rows || batch <= 0 || height <= 0 || width <= 0) return MACVO_E_ARG;
    const int n1 = height * width;
    const long long pixels = (long long)batch * n1;
    int dev = 0, sms = 132;
    MACVO_CUDA_TRY(cudaGetDevice(&dev));
    MACVO_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    auto cost = [&](int tp) { const long long tiles = (pixels + tp - 1) / tp; return ((tiles + sms - 1) / sms) * tp; };
    cudaStream_t st = as_stream(stream);
    __half* o = static_cast<__half*>(out16_rows);
    return cost(72) < cost(64) ? launch_token<72>(cost_forward, coords, key, value, weight_blob, nullptr, pixels, n1, eps, st, o, height, width)
                               : launch_token<64>(cost_forward, coords, key, value, weight_blob, nullptr, pixels, n1, eps, st, o, height, width);
}
