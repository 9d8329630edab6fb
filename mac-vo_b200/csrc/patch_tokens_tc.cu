// PatchEmbed's token head on the Hopper tensor cores (wgmma tf32, TMA, mbarrier), sm_90a:
//
//     out = LayerNorm( W2 relu(W0a x + term[row % period]) + b2 )      x (rows, 64), out (rows, 128) fp32;  W0a (128, 64),
//                                                                       W2 (128, 128), term (period, 128)
//
// ffn_with_coord.0 (its position half and both biases folded into `term`), ReLU, ffn_with_coord.2 and the PatchEmbed norm
// (encoder.py:40-55). Unfused, these are four passes over the largest activation of the frame (9600 maps x 80 tokens at
// 640x480): the 128-wide hidden and pre-norm tensors go through HBM five times. Here x is read once and out written once.
//
//   * Persistent CTAs (one per SM) walk the 128-row tiles. W0a (32 KB) and W2 (64 KB) stay resident in shared memory; x tiles
//     (two 32-channel SWIZZLE_128B sub-tiles, 32 KB) stream through a 2-slot TMA ring, so the next tile lands while this one
//     is computed and stored. Warpgroups 0 and 1 own 64 rows of each tile; warp 8 is the TMA producer.
//   * x is rounded to tf32 (nearest-even) in shared memory. GEMM1 (m64n128k8, K = 64) -> + term, ReLU, tf32 rounding ->
//     the warpgroup's 64 x 128 K-major hidden tile -> GEMM2 (m64n128k8, K = 128) -> + b2. The operand rounding, the K order
//     and the bias add are those of the cuBLAS TF32 GEMMs this replaces (as in mlp_tc.cu), so the bits are the same.
//   * LayerNorm: the 64 x 128 pre-norm rows are staged in the hidden tile's space and normalised warp-per-row by
//     layer_norm_row (the function the warp-per-row LayerNorm kernel calls), then streamed out as whole 512-byte rows.
//     Rows >= `rows`: TMA zero fill on load, masked on store. No atomics: the output bits repeat from launch to launch.
#include "tc_common.cuh"
#include "layer_norm_row.cuh"

namespace {

constexpr int PT_IN = 64, PT_C = 128, PT_ROWS = 128;
constexpr int X_SUB = PT_ROWS * 128;                        // 16 KB: 128 rows x 32 channels
constexpr int X_BYTES = 2 * X_SUB;                          // 32 KB per ring slot
constexpr int W0_SUB = PT_C * 128;                          // 16 KB: 128 output rows x 32 input channels
constexpr int W0_BYTES = 2 * W0_SUB;
constexpr int W2_SUB = PT_C * 128;
constexpr int W2_BYTES = 4 * W2_SUB;                        // 64 KB
constexpr int HID_SUB = 64 * 128;                           // 8 KB: 64 rows x 32 hidden
constexpr int HID_WG_BYTES = 4 * HID_SUB;                   // 32 KB per warpgroup; later its 64 pre-norm rows (512 B each)
constexpr int OFF_W2 = W0_BYTES, OFF_X = OFF_W2 + W2_BYTES, OFF_HID = OFF_X + 2 * X_BYTES;
constexpr int OFF_BAR = OFF_HID + 2 * HID_WG_BYTES;
constexpr int PT_SMEM = OFF_BAR + 64 + 1024;                // + barriers + alignment slack
static_assert(PT_SMEM <= 227 * 1024, "shared memory budget");
static_assert(PT_ROWS * PT_C * 4 == 2 * HID_WG_BYTES, "the pre-norm rows reuse the hidden tiles");

// see mlp_tc.cu: a K-major SWIZZLE_128B descriptor as a constant high word and a 32-bit low word
constexpr uint32_t SW128_DESC_HI = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t sw128_lo(uint32_t smem_addr) { return ((smem_addr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint64_t sw128_desc(uint32_t lo) { return ((uint64_t)SW128_DESC_HI << 32) | lo; }

// fp32 -> tf32, round to nearest, ties to even, as cuBLAS's TF32 GEMMs round their operands (the MMA would truncate)
__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void wg_sync(int wg) {
    if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
    else asm volatile("bar.sync 3, 128;" ::: "memory");
}

__global__ void __launch_bounds__(TC_THREADS, 1)
patch_tokens_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w0,
                       const __grid_constant__ CUtensorMap map_w2, const float* __restrict__ term, const float* __restrict__ b2,
                       const float* __restrict__ ln_w, const float* __restrict__ ln_b, float* __restrict__ out, int rows,
                       int period, float eps) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t s_base = smem_u32(smem);
    // barriers: w_full | x_full[2] | x_empty[2]
    const uint32_t bar_w = s_base + OFF_BAR, bar_xf = bar_w + 8, bar_xe = bar_xf + 16;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles = ceil_div(rows, PT_ROWS);

    if (threadIdx.x == 0) {
        mbar_init(bar_w, 1);
        for (int s = 0; s < 2; ++s) { mbar_init(bar_xf + 8 * s, 1); mbar_init(bar_xe + 8 * s, 2); }
        fence_barrier_init();
        prefetch_tmap(&map_x); prefetch_tmap(&map_w0); prefetch_tmap(&map_w2);
    }
    __syncthreads();

    if (warp == TC_PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            mbar_expect_tx(bar_w, W0_BYTES + W2_BYTES);
            for (int kc = 0; kc < 2; ++kc) tma_load_2d(s_base + kc * W0_SUB, &map_w0, bar_w, 32 * kc, 0);
            for (int kc = 0; kc < 4; ++kc) tma_load_2d(s_base + OFF_W2 + kc * W2_SUB, &map_w2, bar_w, 32 * kc, 0);
            int it = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x, ++it) {
                const int s = it & 1;
                mbar_wait(bar_xe + 8 * s, ((it >> 1) & 1) ^ 1);
                mbar_expect_tx(bar_xf + 8 * s, X_BYTES);
                for (int kc = 0; kc < 2; ++kc) tma_load_2d(s_base + OFF_X + s * X_BYTES + kc * X_SUB, &map_x, bar_xf + 8 * s, 32 * kc, t * PT_ROWS);
            }
        }
        return;
    }

    // ===================== consumers =====================
    const int wg = warp >> 2, t128 = threadIdx.x & 127;
    const bool leader = t128 == 0;
    const uint32_t hid = s_base + OFF_HID + wg * HID_WG_BYTES;
    const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);   // fragment row / column base (wgmma_ops.cuh)
    float acc[64];

    mbar_wait(bar_w, 0);
    int it = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x, ++it) {
        const int s = it & 1;
        const uint32_t xs = s_base + OFF_X + s * X_BYTES;
        mbar_wait(bar_xf + 8 * s, (it >> 1) & 1);
        // round this warpgroup's 64 x rows to tf32 in place (2 sub-tiles x 8 KB; the swizzle does not matter elementwise)
#pragma unroll
        for (int kc = 0; kc < 2; ++kc) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t a = xs + kc * X_SUB + wg * 64 * 128 + (u * 128 + t128) * 16;
                const float4 v = lds128(a);
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(to_tf32(v.x)), "r"(to_tf32(v.y)),
                             "r"(to_tf32(v.z)), "r"(to_tf32(v.w)) : "memory");
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        wg_sync(wg);        // the rounded rows are complete, and every warp has read the previous tile's pre-norm rows

        // GEMM1: acc = x (64 x 64) W0a^T
        {
            uint32_t xd = sw128_lo(xs + wg * 64 * 128), wd = sw128_lo(s_base);
            asm volatile("" : "+r"(xd), "+r"(wd));
            wgmma_fence();
#pragma unroll
            for (int kc = 0; kc < 2; ++kc) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    Wgmma<128>::tf32(acc, sw128_desc(xd + (kc * X_SUB >> 4) + 2 * k), sw128_desc(wd + (kc * W0_SUB >> 4) + 2 * k),
                                     (kc | k) != 0);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_acc(acc);
        }
        if (leader) mbar_arrive(bar_xe + 8 * s);

        // + term[row % period], ReLU, tf32 rounding -> K-major SWIZZLE_128B hidden tile (16-byte chunk c of row r at c ^ (r & 7))
        {
            const int row0 = t * PT_ROWS + wg * 64 + fr;
            const float* tr0 = term + (long long)(row0 % period) * PT_C;
            const float* tr1 = term + (long long)((row0 + 8) % period) * PT_C;
#pragma unroll
            for (int i = 0; i < 64; i += 2) {
                const int r = fr + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + fc;
                const float2 tt = __ldg(reinterpret_cast<const float2*>(((i >> 1) & 1 ? tr1 : tr0) + c));
                const uint32_t v0 = to_tf32(fmaxf(acc[i] + tt.x, 0.f)), v1 = to_tf32(fmaxf(acc[i + 1] + tt.y, 0.f));
                const int cc = c & 31;
                const uint32_t addr = hid + (c >> 5) * HID_SUB + r * 128 + ((((cc >> 2) ^ (r & 7))) << 4) + (cc & 3) * 4;
                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v0), "r"(v1) : "memory");
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> wgmma operand reads
        wg_sync(wg);

        // GEMM2: acc = hidden (64 x 128) W2^T
        {
            uint32_t hd = sw128_lo(hid), wd = sw128_lo(s_base + OFF_W2);
            asm volatile("" : "+r"(hd), "+r"(wd));
            wgmma_fence();
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    Wgmma<128>::tf32(acc, sw128_desc(hd + (kc * HID_SUB >> 4) + 2 * k), sw128_desc(wd + (kc * W2_SUB >> 4) + 2 * k),
                                     (kc | k) != 0);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_acc(acc);
        }

        // + b2, staged as 64 rows of 512 B over the hidden tile for the row-wise LayerNorm; a warp's staged rows overlay
        // hidden rows that the other warps' share of GEMM2 reads, so the whole warpgroup retires GEMM2 first
        wg_sync(wg);
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(b2 + 8 * (i >> 2) + fc));
            acc[i] = acc[i] + bb.x;
            acc[i + 1] = acc[i + 1] + bb.y;
        }
        stage_acc_rows<128>(hid, PT_C * 4, acc, 0);
        wg_sync(wg);

        // LayerNorm: warp w normalises rows 16 w .. 16 w + 15 of the warpgroup's 64, lane <-> float4 chunk as layer_norm_kernel<4>
        const int wrow0 = t * PT_ROWS + wg * 64 + (warp & 3) * 16;
#pragma unroll 2
        for (int j = 0; j < 16; ++j) {
            const int r = (warp & 3) * 16 + j;
            const float4 x4 = lds128(hid + r * (PT_C * 4) + ((lane ^ (r & 7)) << 4));
            float v[4] = {x4.x, x4.y, x4.z, x4.w};
            layer_norm_row<4>(v, ln_w, ln_b, eps, lane);
            if (wrow0 + j < rows)
                __stcs(reinterpret_cast<float4*>(out + (long long)(wrow0 + j) * PT_C) + lane, make_float4(v[0], v[1], v[2], v[3]));
        }
    }
}

}  // namespace

int macvo_patch_tokens_tc(const float* x, const float* w0, const float* term, const float* w2, const float* b2,
                          const float* ln_w, const float* ln_b, float* out, long long rows, int in_channels, int channels,
                          int period, float eps, void* stream) {
    if (!x || !w0 || !term || !w2 || !b2 || !ln_w || !ln_b || !out || rows < 0 || period <= 0) return MACVO_E_ARG;
    if (in_channels != PT_IN || channels != PT_C || rows > (long long)INT32_MAX - PT_ROWS) return MACVO_E_UNSUPPORTED;
    for (const void* p : {(const void*)x, (const void*)w0, (const void*)term, (const void*)w2, (const void*)b2,
                          (const void*)ln_w, (const void*)ln_b, (const void*)out})
        if (reinterpret_cast<uintptr_t>(p) & 15) return MACVO_E_ARG;
    if (rows == 0) return MACVO_OK;
    CUtensorMap m_x, m_w0, m_w2;
    bool ok = make_map_2d(&m_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x, PT_IN, (uint64_t)rows, PT_IN * 4, 32, PT_ROWS);
    ok = ok && make_map_2d(&m_w0, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, w0, PT_IN, PT_C, PT_IN * 4, 32, PT_C);
    ok = ok && make_map_2d(&m_w2, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, w2, PT_C, PT_C, PT_C * 4, 32, PT_C);
    if (!ok) return MACVO_E_DRIVER;
    // the SM count and the attribute belong to the current device: both are taken on every launch (host-only calls)
    int dev = 0, sms = 0;
    MACVO_CUDA_TRY(cudaGetDevice(&dev));
    MACVO_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    MACVO_CUDA_TRY(cudaFuncSetAttribute(patch_tokens_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PT_SMEM));
    const int tiles = ceil_div((int)rows, PT_ROWS);
    patch_tokens_tc_kernel<<<tiles < sms ? tiles : sms, TC_THREADS, PT_SMEM, as_stream(stream)>>>(
        m_x, m_w0, m_w2, term, b2, ln_w, ln_b, out, (int)rows, period, eps);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
