// Transformer MLP with residual on the Hopper tensor cores (wgmma tf32, TMA, mbarrier), sm_90a:
//
//     out = resid + W2 GELU_erf(W1 xn + b1) + b2          xn, resid, out: (M, 128) fp32 rows;  W1 (Hd, 128), W2 (128, Hd)
//
// The Twins-SVT / cost-perceiver MLPs (`x + fc2(gelu(fc1(xn)))`, Hd = 512 or 128). Unfused, the 4x-wide hidden activation
// goes through HBM four times (fc1 writes it, GELU reads and writes it, fc2 reads it); here it never leaves the SM.
//
//   * CTA = 128 rows: warpgroups 0 and 1 own 64 rows each, as in tc_common.cuh, and warp 8 is the TMA producer (its
//     warpgroup gives its registers to the consumers). The 128 x 128 xn tile stays resident (four 32-channel
//     SWIZZLE_128B sub-tiles, 64 KB).
//   * xn is rounded to tf32 in shared memory once per tile. The hidden dimension is walked in chunks of 64. Chunk j:
//     GEMM1 (m64n64k8, K = 128) -> +b1, GELU, tf32 rounding ->
//     the warpgroup's 64 x 64 K-major hidden tile in shared memory -> GEMM2 (m64n128k8, K = 64) accumulates the 64 x 128
//     output in registers. W1 chunks (64 x 128) and W2 chunks (128 x 64) stream from L2 through two 2-slot rings with
//     separate barriers, so chunk j+1's W1 can land while chunk j-1's W2 is still being read.
//   * GEMM1 of chunk j+1 is issued before the GELU of chunk j (two hidden accumulators): the erf work, which costs about as
//     many issue slots as the chunk's MMAs, overlaps the tensor cores instead of alternating with them.
//   * Epilogue straight from the accumulator fragment: + b2 + resid, float2 stores (4 lanes cover 32 contiguous bytes of a
//     row, so every sector is written whole). Rows >= M: TMA zero fill on load, masked on store. No atomics: the output
//     bits repeat from launch to launch.
#include "tc_common.cuh"

namespace {

constexpr int MLP_C = 128, MLP_ROWS = 128, MLP_CHUNK = 64;
constexpr int XN_BYTES = MLP_ROWS * MLP_C * 4;              // 64 KB: 4 sub-tiles of 128 rows x 32 channels
constexpr int XN_SUB = MLP_ROWS * 128;                      // 16 KB
constexpr int W1_BYTES = MLP_CHUNK * MLP_C * 4;             // 32 KB: 4 sub-tiles of 64 hidden rows x 32 channels
constexpr int W1_SUB = MLP_CHUNK * 128;                     // 8 KB
constexpr int W2_BYTES = MLP_C * MLP_CHUNK * 4;             // 32 KB: 2 sub-tiles of 128 output rows x 32 hidden
constexpr int W2_SUB = MLP_C * 128;                         // 16 KB
constexpr int HID_WG_BYTES = 64 * MLP_CHUNK * 4;            // 16 KB per warpgroup: 2 sub-tiles of 64 rows x 32 hidden
constexpr int HID_SUB = 64 * 128;                           // 8 KB
constexpr int OFF_W1 = XN_BYTES, OFF_W2 = OFF_W1 + 2 * W1_BYTES, OFF_HID = OFF_W2 + 2 * W2_BYTES;
constexpr int OFF_BAR = OFF_HID + 2 * HID_WG_BYTES;
constexpr int MLP_SMEM = OFF_BAR + 128 + 1024;              // + barriers + alignment slack
static_assert(MLP_SMEM <= 227 * 1024, "shared memory budget");

// make_kmajor_sw128_desc split into a constant high word and a low word (start address >> 4 | LBO): operand offsets are
// 32-bit adds, so the compiler keeps one register per hoisted descriptor instead of two (and does not spill them)
constexpr uint32_t SW128_DESC_HI = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t sw128_lo(uint32_t smem_addr) { return ((smem_addr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint64_t sw128_desc(uint32_t lo) { return ((uint64_t)SW128_DESC_HI << 32) | lo; }

// fp32 -> tf32, round to nearest, ties to even: how cuBLAS's TF32 GEMMs round their fp32 operands, so that the fused MLP
// computes the same values as the fc1 / GELU / fc2 sequence it replaces (the MMA itself would truncate)
__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// 128 output + 2 x 32 hidden accumulators per consumer thread do not fit the 168 registers a 288- or 384-thread CTA starts
// with: the producer is a whole warpgroup (warp 8 issues, 9..11 idle) so that it can hand registers to the consumers.
constexpr int MLP_THREADS = TC_CONSUMER_THREADS + 128;

__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w1,
              const __grid_constant__ CUtensorMap map_w2, const float* __restrict__ b1, const float* __restrict__ b2,
              const float* __restrict__ resid, float* __restrict__ out, int m, int hd) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t s_base = smem_u32(smem);
    // barriers: x_full | w1_full[2] | w1_empty[2] | w2_full[2] | w2_empty[2]
    const uint32_t bar_x = s_base + OFF_BAR, bar_w1f = bar_x + 8, bar_w1e = bar_w1f + 16, bar_w2f = bar_w1e + 16,
                   bar_w2e = bar_w2f + 16;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * MLP_ROWS, chunks = hd / MLP_CHUNK;

    if (threadIdx.x == 0) {
        mbar_init(bar_x, 1);
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar_w1f + 8 * s, 1); mbar_init(bar_w1e + 8 * s, 2);
            mbar_init(bar_w2f + 8 * s, 1); mbar_init(bar_w2e + 8 * s, 2);
        }
        fence_barrier_init();
        prefetch_tmap(&map_x); prefetch_tmap(&map_w1); prefetch_tmap(&map_w2);
    }
    __syncthreads();

    if (warp >= TC_PRODUCER_WARP) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == TC_PRODUCER_WARP && elect_one()) {
            mbar_expect_tx(bar_x, XN_BYTES);
            for (int kc = 0; kc < 4; ++kc) tma_load_2d(s_base + kc * XN_SUB, &map_x, bar_x, 32 * kc, m0);
            for (int j = 0; j < chunks; ++j) {
                const int s = j & 1;
                const uint32_t parity = ((j >> 1) & 1) ^ 1;
                mbar_wait(bar_w1e + 8 * s, parity);
                mbar_expect_tx(bar_w1f + 8 * s, W1_BYTES);
                for (int kc = 0; kc < 4; ++kc)
                    tma_load_2d(s_base + OFF_W1 + s * W1_BYTES + kc * W1_SUB, &map_w1, bar_w1f + 8 * s, 32 * kc, j * MLP_CHUNK);
                mbar_wait(bar_w2e + 8 * s, parity);
                mbar_expect_tx(bar_w2f + 8 * s, W2_BYTES);
                for (int h = 0; h < 2; ++h)
                    tma_load_2d(s_base + OFF_W2 + s * W2_BYTES + h * W2_SUB, &map_w2, bar_w2f + 8 * s, j * MLP_CHUNK + 32 * h, 0);
            }
        }
        return;
    }

    // ===================== consumers =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint32_t hid = s_base + OFF_HID + wg * HID_WG_BYTES;
    // descriptor low words: this warpgroup's 64 rows of xn sub-tile 0, its hidden tile
    const uint32_t xa = sw128_lo(s_base) + (wg * 64 * 128 >> 4), hid_d = sw128_lo(hid);
    const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);   // fragment row / column base (wgmma_ops.cuh)
    float acc[64], h0[32], h1[32];

    // GEMM1 of chunk j into h: the warpgroup's 64 rows x 64 hidden units, K = 128
    auto gemm1 = [&](float (&h)[32], int j) {
        const int s = j & 1;
        mbar_wait(bar_w1f + 8 * s, (j >> 1) & 1);
        uint32_t xd = xa;
        asm volatile("" : "+r"(xd));         // opaque: descriptors are two adds away, not 32 hoisted (spilled) registers
        const uint32_t wb = xd - (wg * 64 * 128 >> 4) + ((OFF_W1 + s * W1_BYTES) >> 4);
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                Wgmma<64>::tf32(h, sw128_desc(xd + (kc * XN_SUB >> 4) + 2 * k), sw128_desc(wb + (kc * W1_SUB >> 4) + 2 * k), (kc | k) != 0);
        }
        wgmma_commit();
    };

    // chunk j: h holds GEMM1(j), hn receives GEMM1(j+1)
    auto chunk = [&](float (&h)[32], float (&hn)[32], int j) {
        if (j + 1 < chunks) {
            gemm1(hn, j + 1);
            wgmma_wait<1>();                 // GEMM1(j) and GEMM2(j-1) retired; GEMM1(j+1) keeps running
        } else {
            wgmma_wait<0>();
        }
        fence_acc(h);
        fence_acc(acc);
        if (leader) {
            mbar_arrive(bar_w1e + 8 * (j & 1));
            if (j > 0) mbar_arrive(bar_w2e + 8 * ((j - 1) & 1));
        }
        // + b1, GELU, tf32 rounding -> K-major SWIZZLE_128B hidden tile (16-byte chunk c of row r at c ^ (r & 7))
        const float* bj = b1 + j * MLP_CHUNK;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int r = fr + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + fc;
            const float2 bb = __ldg(reinterpret_cast<const float2*>(bj + c));
            const uint32_t v0 = to_tf32(gelu_erf(h[i] + bb.x)), v1 = to_tf32(gelu_erf(h[i + 1] + bb.y));
            const int cc = c & 31;
            const uint32_t addr = hid + (c >> 5) * HID_SUB + r * 128 + ((((cc >> 2) ^ (r & 7))) << 4) + (cc & 3) * 4;
            asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v0), "r"(v1) : "memory");
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> wgmma operand reads
        if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");     // this warpgroup's hidden tile is complete
        else asm volatile("bar.sync 3, 128;" ::: "memory");
        // GEMM2 of chunk j: acc += hidden (64 x 64) W2[:, chunk]^T
        const int s = j & 1;
        mbar_wait(bar_w2f + 8 * s, (j >> 1) & 1);
        uint32_t hd_ = hid_d;
        asm volatile("" : "+r"(hd_));
        const uint32_t wb = hd_ - ((OFF_HID + wg * HID_WG_BYTES) >> 4) + ((OFF_W2 + s * W2_BYTES) >> 4);
        wgmma_fence();
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                Wgmma<128>::tf32(acc, sw128_desc(hd_ + (hh * HID_SUB >> 4) + 2 * k), sw128_desc(wb + (hh * W2_SUB >> 4) + 2 * k),
                                 (j | hh | k) != 0);
        }
        wgmma_commit();
    };

    mbar_wait(bar_x, 0);
    {   // round this warpgroup's 64 xn rows to tf32 in place (4 sub-tiles x 8 KB; the swizzle does not matter elementwise)
        const int t = threadIdx.x & 127;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t a = s_base + kc * XN_SUB + wg * 64 * 128 + (u * 128 + t) * 16;
                const float4 v = lds128(a);
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(to_tf32(v.x)), "r"(to_tf32(v.y)),
                             "r"(to_tf32(v.z)), "r"(to_tf32(v.w)) : "memory");
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
        else asm volatile("bar.sync 3, 128;" ::: "memory");
    }
    gemm1(h0, 0);
    for (int j = 0; j < chunks; j += 2) {    // chunks is even (Hd in {128, 512}): the accumulators alternate statically
        chunk(h0, h1, j);
        chunk(h1, h0, j + 1);
    }
    wgmma_wait<0>();
    fence_acc(acc);

    // out = resid + (acc + b2)
    const int row0 = m0 + wg * 64 + fr;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int r = row0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + fc;
        if (r < m) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(b2 + c));
            const float2 x = __ldg(reinterpret_cast<const float2*>(resid + (long long)r * MLP_C + c));
            *reinterpret_cast<float2*>(out + (long long)r * MLP_C + c) = make_float2(x.x + (acc[i] + bb.x), x.y + (acc[i + 1] + bb.y));
        }
    }
}

}  // namespace

int macvo_mlp_tc(const float* xn, const float* resid, const float* w1, const float* b1, const float* w2, const float* b2,
                 float* out, int rows, int channels, int hidden, void* stream) {
    if (!xn || !resid || !w1 || !b1 || !w2 || !b2 || !out || rows <= 0) return MACVO_E_ARG;
    if (channels != MLP_C || (hidden != 128 && hidden != 512)) return MACVO_E_UNSUPPORTED;
    for (const void* p : {(const void*)xn, (const void*)resid, (const void*)w1, (const void*)b1, (const void*)w2,
                          (const void*)b2, (const void*)out})
        if (reinterpret_cast<uintptr_t>(p) & 15) return MACVO_E_ARG;
    CUtensorMap m_x, m_w1, m_w2;
    bool ok = make_map_2d(&m_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, xn, MLP_C, rows, MLP_C * 4, 32, MLP_ROWS);
    ok = ok && make_map_2d(&m_w1, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, w1, MLP_C, hidden, MLP_C * 4, 32, MLP_CHUNK);
    ok = ok && make_map_2d(&m_w2, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, w2, hidden, MLP_C, (uint64_t)hidden * 4, 32, MLP_C);
    if (!ok) return MACVO_E_DRIVER;
    // the attribute belongs to the current device, so it is set on every launch (host-only, allowed under graph capture)
    MACVO_CUDA_TRY(cudaFuncSetAttribute(mlp_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MLP_SMEM));
    mlp_tc_kernel<<<ceil_div(rows, MLP_ROWS), MLP_THREADS, MLP_SMEM, as_stream(stream)>>>(m_x, m_w1, m_w2, b1, b2, resid, out,
                                                                                          rows, hidden);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
