// (a3) all-pairs correlation volume on the Hopper tensor cores (wgmma, TMA, mbarrier), sm_90a.
//
// Replaces MemoryEncoder.corr (Module/Network/FlowFormer/core/encoder.py:256-275; one cuBLAS bmm in the
// reference):  corr[b, i, j] = sum_d f1[b, d, i] * f2[b, d, j],  output (B, N, N) fp32 — 184 MB per
// 640x480 `estimate_pair`, write-dominated: the roofline is HBM write bandwidth PROVIDED the K = 256
// contraction runs on tensor cores (116 flop/B; SURVEY.md §7.3).
//
// fp32-class accuracy on fp16 tensor cores (MACVO_CORR_TC_3XF16): every operand is scaled by 2^6 and split
//     x = hi + lo,  hi = fp16(x),  lo = fp16(x - hi)          (|x - hi - lo| <~ 2^-22 |x|)
// and  hi*hi + hi*lo + lo*hi  is accumulated in fp32 registers, rescaled by 2^-12 in the epilogue (the
// power-of-two scale keeps `lo` out of the fp16 subnormal range for |x| > 4e-3; fp16(x * 64) stays finite
// for |x| < 1023). MACVO_CORR_TC_1XF16 keeps only hi*hi, unscaled (exact for the MACVO_Fast configuration
// whose encoder already emits fp16 features). MACVO_CORR_TC_TF32 runs one wgmma kind tf32 pass straight over
// the fp32 K-major features (no pre-pass, no workspace).
//
//   * both operands are pre-split by one small pre-pass into K-major fp16 hi/lo and streamed by TMA
//     (SWIZZLE_128B, 64-wide K slices) through a ring of mbarrier-guarded stages: one stage = one 64-channel
//     k-block of the 128 query rows (A) and the 128 key rows (B), hi and lo.
//   * 288 threads: warps 0..7 = two consumer warpgroups, each owning 64 query rows of the 128 x 128 output tile
//     (m64n128k16 wgmma, 64 fp32 accumulators per thread); warp 8 = TMA producer.
//   * Persistent: CTA c takes tiles c, c + grid, ...; the producer runs up to a whole ring ahead, so the next
//     tile's operands stream in while the consumers write the previous tile (K = 256 is so short that the
//     output stores, not the MMAs, are the critical path). M/N edges: TMA zero fill on load, row guards on store.
#include "tc_common.cuh"
#include <cuda_fp16.h>

namespace {

constexpr int BLOCK_M = 128, BLOCK_N = 128, BLOCK_K = 64;
constexpr int SUB_BYTES = 128 * 128;                         // 16 KB: 128 rows x 128 B (64 fp16 | 32 fp32)
constexpr float SPLIT_SCALE = 64.f;       // 2^6 on both operands
constexpr float SPLIT_UNSCALE = 1.f / 4096.f;

// PASSES 3: fp16 hi*hi + hi*lo + lo*hi (fp32-class)    1: fp16 hi*hi    2: ONE tf32 pass over the fp32 K-major features,
// whose 64-channel k-block is two 32-channel (128 B) sub-tiles per operand
template <int PASSES> struct CorrCfg {
    static constexpr int SUBS = PASSES == 1 ? 1 : 2;         // sub-tiles per operand and k-block
    static constexpr int STAGE_BYTES = 2 * SUBS * SUB_BYTES; // [A sub-tiles | B sub-tiles]
    static constexpr int STAGES = PASSES == 1 ? 6 : 3;
    static constexpr int SMEM = STAGES * STAGE_BYTES + 256 + 1024;   // + barriers + alignment slack
};

// ---- kernel 1: operand pre-pass: fp32 (B, D, N) -> fp16 hi / lo (B, N, D), scaled (both maps, one launch) ----
__global__ void __launch_bounds__(256)
split_transpose_kernel(const float* __restrict__ f1, const float* __restrict__ f2, __half* __restrict__ a_hi,
                       __half* __restrict__ a_lo, __half* __restrict__ b_hi, __half* __restrict__ b_lo, int batch,
                       int dim, int n, float scale) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // let the main kernel's prologue start early (PDL)
    __shared__ float tile[64][33];                                   // [d][token]
    const bool second = (int)blockIdx.z >= batch;
    const int b = second ? blockIdx.z - batch : blockIdx.z;
    const int d0 = blockIdx.y * 64, n0 = blockIdx.x * 32;
    const float* s = (second ? f2 : f1) + (long long)b * dim * n;
    __half* hi = second ? b_hi : a_hi;
    __half* lo = second ? b_lo : a_lo;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
#pragma unroll
    for (int r = ty; r < 64; r += 8) {
        const int d = d0 + r, t = n0 + tx;
        tile[r][tx] = (d < dim && t < n) ? s[(long long)d * n + t] * scale : 0.f;
    }
    __syncthreads();
    // write: token-major rows, 64 consecutive d per row -> lanes cover d pairs (half2, 128 B per warp row)
#pragma unroll
    for (int r = ty; r < 32; r += 8) {
        const int t = n0 + r, d = d0 + 2 * tx;
        if (t < n) {
            const float x0 = tile[2 * tx][r], x1 = tile[2 * tx + 1][r];
            const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
            const long long o = ((long long)b * n + t) * dim + d;
            *reinterpret_cast<__half2*>(hi + o) = __halves2half2(h0, h1);
            if (lo) {
                const __half l0 = __float2half_rn(x0 - __half2float(h0)), l1 = __float2half_rn(x1 - __half2float(h1));
                *reinterpret_cast<__half2*>(lo + o) = __halves2half2(l0, l1);
            }
        }
    }
}

// K-major input (channels_last features, (B, N, D) rows): the pre-pass is a pure elementwise split, no transpose.
// One thread per 4 consecutive d of one token; blockIdx.y selects the map (f1 -> A operands, f2 -> B operands).
constexpr int SPLIT_ILP = 4;       // float4 loads in flight per thread (the pre-pass is latency bound: 20 MB in, 20 MB out)
__global__ void __launch_bounds__(256)
split_kmajor_kernel(const float* __restrict__ f1, const float* __restrict__ f2, __half* __restrict__ a_hi,
                    __half* __restrict__ a_lo, __half* __restrict__ b_hi, __half* __restrict__ b_lo, long long quads,
                    float scale) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // let the main kernel's prologue start early (PDL)
    const bool second = blockIdx.y != 0;
    const float4* src = reinterpret_cast<const float4*>(second ? f2 : f1);
    __half* hi = second ? b_hi : a_hi;
    __half* lo = second ? b_lo : a_lo;
    const long long e0 = (long long)blockIdx.x * (256 * SPLIT_ILP) + threadIdx.x;
    float4 x[SPLIT_ILP];
#pragma unroll
    for (int u = 0; u < SPLIT_ILP; ++u) {
        const long long e = e0 + u * 256;
        x[u] = e < quads ? __ldg(src + e) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < SPLIT_ILP; ++u) {
        const long long e = e0 + u * 256;
        if (e >= quads) continue;
        const float v[4] = {x[u].x * scale, x[u].y * scale, x[u].z * scale, x[u].w * scale};
        __half h[4], l[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { h[i] = __float2half_rn(v[i]); l[i] = __float2half_rn(v[i] - __half2float(h[i])); }
        __half2 hh[2] = {__halves2half2(h[0], h[1]), __halves2half2(h[2], h[3])};
        *reinterpret_cast<uint2*>(hi + 4 * e) = *reinterpret_cast<uint2*>(hh);
        if (lo) {
            __half2 ll[2] = {__halves2half2(l[0], l[1]), __halves2half2(l[2], l[3])};
            *reinterpret_cast<uint2*>(lo + 4 * e) = *reinterpret_cast<uint2*>(ll);
        }
    }
}

// ---- kernel 2 -----------------------------------------------------------------------------------------------
template <int PASSES>
__global__ void __launch_bounds__(TC_THREADS, 1)
corr_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
               float* __restrict__ corr, int batch, int n, int dim) {
    using C = CorrCfg<PASSES>;
    constexpr bool TF32 = PASSES == 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t bar_full = smem_u32(smem + C::STAGES * C::STAGE_BYTES), bar_empty = bar_full + 8 * C::STAGES;
    const int warp = threadIdx.x >> 5;
    const int mt = ceil_div(n, BLOCK_M), nt = ceil_div(n, BLOCK_N), kblocks = dim / BLOCK_K;
    const int tiles = batch * mt * nt;

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2); }
        fence_barrier_init();
        prefetch_tmap(&map_a_hi); prefetch_tmap(&map_b_hi);
    }
    __syncthreads();

    if (warp == TC_PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            // programmatic dependent launch: the set-up above overlapped the tail of the operand pre-pass
            asm volatile("griddepcontrol.wait;" ::: "memory");
            int stage = 0; uint32_t phase = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                const int b = t / (mt * nt), rem = t - b * mt * nt, m0 = (rem / nt) * BLOCK_M, n0 = (rem % nt) * BLOCK_N;
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                    const uint32_t full = bar_full + 8 * stage, sa = smem_u32(smem + stage * C::STAGE_BYTES);
                    const uint32_t sb = sa + C::SUBS * SUB_BYTES;
                    mbar_expect_tx(full, C::STAGE_BYTES);
                    if (TF32) {
                        tma_load_3d(sa, &map_a_hi, full, kb * BLOCK_K, m0, b);
                        tma_load_3d(sa + SUB_BYTES, &map_a_hi, full, kb * BLOCK_K + 32, m0, b);
                        tma_load_3d(sb, &map_b_hi, full, kb * BLOCK_K, n0, b);
                        tma_load_3d(sb + SUB_BYTES, &map_b_hi, full, kb * BLOCK_K + 32, n0, b);
                    } else {
                        tma_load_3d(sa, &map_a_hi, full, kb * BLOCK_K, m0, b);
                        tma_load_3d(sb, &map_b_hi, full, kb * BLOCK_K, n0, b);
                        if (PASSES == 3) {
                            tma_load_3d(sa + SUB_BYTES, &map_a_lo, full, kb * BLOCK_K, m0, b);
                            tma_load_3d(sb + SUB_BYTES, &map_b_lo, full, kb * BLOCK_K, n0, b);
                        }
                    }
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumers: wgmma over this warpgroup's 64 rows, then the stores =====================
        const int wg = warp >> 2, lane = threadIdx.x & 31;
        const float unscale = PASSES == 3 ? SPLIT_UNSCALE : 1.f;
        float acc[BLOCK_N / 2];
        int stage = 0; uint32_t phase = 0;
        for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
            const int b = t / (mt * nt), rem = t - b * mt * nt, m0 = (rem / nt) * BLOCK_M, n0 = (rem % nt) * BLOCK_N;
            for (int kb = 0; kb < kblocks; ++kb) {
                mbar_wait(bar_full + 8 * stage, phase);
                const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES) + wg * 64 * 128, sb = sa - wg * 64 * 128 + C::SUBS * SUB_BYTES;
                const uint64_t a0 = make_kmajor_sw128_desc(sa), a1 = make_kmajor_sw128_desc(sa + SUB_BYTES);
                const uint64_t b0 = make_kmajor_sw128_desc(sb), b1 = make_kmajor_sw128_desc(sb + SUB_BYTES);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {                        // 32 B of the 128-byte row per step: 16 fp16 | 8 fp32
                    const uint32_t first = (kb | k) != 0;
                    if (TF32) {              // channels kb*64 + [8k, 8k+8) from the first sub-tile, + 32 from the second
                        Wgmma<BLOCK_N>::tf32(acc, a0 + 2 * k, b0 + 2 * k, first);
                        Wgmma<BLOCK_N>::tf32(acc, a1 + 2 * k, b1 + 2 * k, 1u);
                    } else if (PASSES == 3) {   // small cross terms first, the dominant hi*hi product last
                        Wgmma<BLOCK_N>::f16(acc, a1 + 2 * k, b0 + 2 * k, first);
                        Wgmma<BLOCK_N>::f16(acc, a0 + 2 * k, b1 + 2 * k, 1u);
                        Wgmma<BLOCK_N>::f16(acc, a0 + 2 * k, b0 + 2 * k, 1u);
                    } else {
                        Wgmma<BLOCK_N>::f16(acc, a0 + 2 * k, b0 + 2 * k, first);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_acc(acc);
                if ((threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * stage);   // this warpgroup is done with the stage
                if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
            }
            // fragment -> rows: 4 lanes cover 8 consecutive columns (32 B) of a row; the volume is written once, streaming stores
            const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = n0 + 2 * (lane & 3);
            float* base = corr + (long long)b * n * n;
#pragma unroll
            for (int i = 0; i < BLOCK_N / 2; i += 2) {
                const int r = r0 + 8 * ((i >> 1) & 1), c = c0 + 8 * (i >> 2);
                if (r < n && c < n)                                          // n % 8 == 0: c < n implies c + 1 < n
                    __stcs(reinterpret_cast<float2*>(base + (long long)r * n + c), make_float2(acc[i] * unscale, acc[i + 1] * unscale));
            }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------------
size_t operand_bytes(int batch, int dim, int n) { return ((size_t)batch * n * dim * 2 + 1023) / 1024 * 1024; }

template <int PASSES>
int launch_main(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                float* m_out, int batch, int n, int dim, int ctas, cudaStream_t st) {
    // the attribute belongs to the current device, so it is set on every launch (host-only, allowed under graph capture)
    MACVO_CUDA_TRY(cudaFuncSetAttribute(corr_tc_kernel<PASSES>, cudaFuncAttributeMaxDynamicSharedMemorySize, CorrCfg<PASSES>::SMEM));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctas);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = CorrCfg<PASSES>::SMEM;
    cfg.stream = st;
    // programmatic dependent launch on the operand pre-pass
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MACVO_CUDA_TRY(cudaLaunchKernelEx(&cfg, corr_tc_kernel<PASSES>, a_hi, a_lo, b_hi, b_lo, m_out, batch, n, dim));
    return MACVO_OK;
}

}  // namespace

size_t macvo_corr_tc_workspace_bytes(int batch, int dim, int n, int passes) {
    return operand_bytes(batch, dim, n) * (passes == 3 ? 4 : 2);
}

int macvo_corr_build_tc(const float* f1, const float* f2, float* corr, int batch, int dim, int n, int passes, int kmajor,
                        void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (dim % BLOCK_K != 0 || n % 8 != 0) return MACVO_E_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(corr) & 31) return MACVO_E_ARG;
    int dev = 0, sms = 0;
    MACVO_CUDA_TRY(cudaGetDevice(&dev));
    MACVO_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long tiles = (long long)batch * ceil_div(n, BLOCK_M) * ceil_div(n, BLOCK_N);
    const int ctas = (int)(tiles < sms ? tiles : sms);                 // one persistent CTA per SM (the ring fills shared memory)
    if (passes == 2) {
        // tf32: TMA reads the fp32 (B, N, D) features themselves, 32 channels (128 B) per swizzled row
        if (!kmajor || (reinterpret_cast<uintptr_t>(f1) & 15) || (reinterpret_cast<uintptr_t>(f2) & 15)) return MACVO_E_ARG;
        CUtensorMap m_a, m_b;
        bool ok = make_map_3d(&m_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(f1), dim, n, batch, 32, BLOCK_M);
        ok = ok && make_map_3d(&m_b, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(f2), dim, n, batch, 32, BLOCK_N);
        if (!ok) return MACVO_E_DRIVER;
        return launch_main<2>(m_a, m_a, m_b, m_b, corr, batch, n, dim, ctas, st);
    }
    if (!workspace || workspace_bytes < macvo_corr_tc_workspace_bytes(batch, dim, n, passes)) return MACVO_E_WORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace) & 1023) return MACVO_E_ARG;
    const size_t ob = operand_bytes(batch, dim, n);
    char* ws = static_cast<char*>(workspace);
    __half* a_hi = reinterpret_cast<__half*>(ws);
    __half* b_hi = reinterpret_cast<__half*>(ws + ob);
    __half* a_lo = passes == 3 ? reinterpret_cast<__half*>(ws + 2 * ob) : nullptr;
    __half* b_lo = passes == 3 ? reinterpret_cast<__half*>(ws + 3 * ob) : nullptr;

    // one launch splits both feature maps: blockIdx.z in [0, batch) -> f1, [batch, 2 batch) -> f2
    if (kmajor) {
        const long long quads = (long long)batch * n * dim / 4;
        dim3 kgrid((unsigned)((quads + 256 * SPLIT_ILP - 1) / (256 * SPLIT_ILP)), 2);
        split_kmajor_kernel<<<kgrid, 256, 0, st>>>(f1, f2, a_hi, a_lo, b_hi, b_lo, quads, passes == 3 ? SPLIT_SCALE : 1.f);
    } else {
        dim3 pgrid(ceil_div(n, 32), ceil_div(dim, 64), 2 * batch);
        split_transpose_kernel<<<pgrid, 256, 0, st>>>(f1, f2, a_hi, a_lo, b_hi, b_lo, batch, dim, n,
                                                      passes == 3 ? SPLIT_SCALE : 1.f);
    }
    MACVO_LAUNCH_CHECK();

    CUtensorMap m_a_hi, m_a_lo, m_b_hi, m_b_lo;
    bool ok = make_map_3d(&m_a_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, a_hi, dim, n, batch, BLOCK_K, BLOCK_M);
    ok = ok && make_map_3d(&m_b_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, b_hi, dim, n, batch, BLOCK_K, BLOCK_N);
    ok = ok && make_map_3d(&m_a_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, passes == 3 ? a_lo : a_hi, dim, n, batch, BLOCK_K, BLOCK_M);
    ok = ok && make_map_3d(&m_b_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, passes == 3 ? b_lo : b_hi, dim, n, batch, BLOCK_K, BLOCK_N);
    if (!ok) return MACVO_E_DRIVER;

    return passes == 3 ? launch_main<3>(m_a_hi, m_a_lo, m_b_hi, m_b_lo, corr, batch, n, dim, ctas, st)
                       : launch_main<1>(m_a_hi, m_a_lo, m_b_hi, m_b_lo, corr, batch, n, dim, ctas, st);
}
