// (f2) The decoder's 3x3 / 1x1 convolutions (motion encoder, GMA value projection, flow head, covariance head:
// Module/Network/FlowFormer/core/gru.py:45-64,6-14, gma.py:84-130, FlowFormerCov/covhead.py:20-58) as wgmma implicit GEMMs.
//
//   out[pixel, n] = act( bias[n] + sum_{tap, c} in[pixel + offset(tap), c] * w[n, tap, c] )
//
// rows = pixels, fp16 operands (11-bit significand >= TF32's 10), fp32 accumulation in registers. Activations live in layout U
// (csrc/rows_layout.cuh: one fp16 row per pixel, 2 zero pixels around every image), so a 3x3 tap is a row offset and a
// tile is any 128 consecutive rows: per 64-channel block and tap, TMA loads the 128 shifted input rows and the tap's filter
// rows into one ring slot (rows outside the buffer are zero filled). A 1x1 convolution may also read plain dense pixel rows.
//
// One CTA per (128-pixel tile, slice of N output channels): warps 0..7 = two consumer warpgroups (m64nNk16 wgmma, one
// MMA group kept in flight), warp 8 = TMA producer. Epilogue: accumulators -> XOR-swizzled smem transpose in the idle
// operand ring -> bias / ReLU -> row-contiguous global stores as fp16 rows for the next convolution and / or fp32 dense rows.
// Launched with programmatic stream serialization: the filters of the first ring slots are in flight before
// `griddepcontrol.wait` lets the input rows be touched.
#include "tc_common.cuh"
#include "rows_layout.cuh"
#include <cuda_fp16.h>

namespace {

constexpr int TILE_M = macvo_rows::TILE_M, BLOCK_K = 64;
constexpr int A_BYTES = TILE_M * 128;                          // 16 KB: 128 rows x 64 fp16
constexpr int SMEM_MAX = 200 * 1024;

struct ConvArgs {
    int taps, kblocks;            // 1 | 9 ; input channels / 64
    int slots;                    // ring depth
    int in_dense;                 // A rows are dense pixel rows (1x1 only) instead of layout U
    int batch, height, width, wp; // wp = width + 4
    int m_rows;                   // rows to cover: pixels (dense) or padded pixels (layout U)
    int relu, n_valid;            // columns >= n_valid are computed (zero filters) but never stored
    const float* bias;            // (grid.y * N) or NULL
    __half* out16; int out16_pitch, out16_off, out16_dense;
    float* out32; int out32_pitch, out32_off;
    int out32_planes;             // 1: out32 is a (batch, n_valid, H, W) map and the result is ADDED to it (coords += delta)
};

// N = output channels per CTA (multiple of 32, <= 256); grid.y slices the padded output channels
template <int N>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, ConvArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    // ring of `slots` slots: [A tile 16 KB | the tap's N filter rows]
    constexpr int SLOT_BYTES = A_BYTES + N * 128;
    const uint32_t bar_full = smem_u32(smem + a.slots * SLOT_BYTES), bar_empty = bar_full + 8 * a.slots;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x, slice = blockIdx.y;
    const int steps = a.kblocks * a.taps;

    if (threadIdx.x == 0) {
        for (int s = 0; s < a.slots; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2); }
        fence_barrier_init();
        prefetch_tmap(&map_a); prefetch_tmap(&map_w);
    }
    __syncthreads();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    if (warp == TC_PRODUCER_WARP) {
        // ===================== TMA producer =====================
        // steps run over (64-channel block, tap), taps fastest; all indices are running counters
        if (elect_one()) {
            const int c_in = a.kblocks * BLOCK_K;
            const int base_row = a.in_dense ? tile * TILE_M : macvo_rows::GUARD + tile * TILE_M;
            auto issue_w = [&](int sl, int kb_, int tap_) {                 // filters of one step -> slot sl (after the A tile)
                const uint32_t full = bar_full + 8 * sl;
                mbar_expect_tx(full, SLOT_BYTES);                          // A + filters
                tma_load_2d(smem_u32(smem + sl * SLOT_BYTES + A_BYTES), &map_w, full, tap_ * c_in + kb_ * BLOCK_K, slice * N);
            };
            auto issue_a = [&](int sl, int kb_, int tap_) {                 // tap (dy, dx) = row offset (dy - 1) wp + dx - 1
                const int off = a.taps == 9 ? (tap_ / 3 - 1) * a.wp + tap_ % 3 - 1 : 0;
                tma_load_2d(smem_u32(smem + sl * SLOT_BYTES), &map_a, bar_full + 8 * sl, kb_ * BLOCK_K, base_row + off);
            };
            auto advance = [&](int& kb_, int& tap_) { if (++tap_ == a.taps) { tap_ = 0; ++kb_; } };
            // the filters of the first `slots` steps do not depend on the previous kernel: in flight before the wait
            const int pre = steps < a.slots ? steps : a.slots;
            { int k2 = 0, t2 = 0; for (int g = 0; g < pre; ++g) { issue_w(g, k2, t2); advance(k2, t2); } }
            asm volatile("griddepcontrol.wait;" ::: "memory");
            int slot = 0, kb = 0, tap = 0;
            uint32_t phase = 0;
            for (int g = 0; g < steps; ++g) {
                if (g >= pre) {
                    mbar_wait(bar_empty + 8 * slot, phase ^ 1);
                    issue_w(slot, kb, tap);
                }
                issue_a(slot, kb, tap);
                advance(kb, tap);
                if (++slot == a.slots) { slot = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===================== consumers: MMAs =====================
    const int wg = warp >> 2;
    float acc[N / 2];
    {
        int slot = 0, prev = 0; uint32_t phase = 0;
        for (int g = 0; g < steps; ++g) {
            mbar_wait(bar_full + 8 * slot, phase);
            const uint32_t sa = smem_u32(smem + slot * SLOT_BYTES);
            const uint64_t da = make_kmajor_sw128_desc(sa + wg * 64 * 128), db = make_kmajor_sw128_desc(sa + A_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / 16; ++k) Wgmma<N>::f16(acc, da + 2 * k, db + 2 * k, (g | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();                                       // the previous step's MMAs retired: release its slot
            if (g > 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * prev);
            prev = slot;
            if (++slot == a.slots) { slot = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
    }

    // ===================== epilogue =====================
    // rows of 4 N bytes, 16-byte chunks XOR-swizzled by the row: conflict-free both ways; warp (quarter, half) then finishes
    // rows [32 quarter + 16 half, +16): one full row per instruction, 4 columns per lane
    const int pitch = N * 4;
    consumers_sync();                                              // every MMA of both warpgroups read its operands
    stage_acc_rows<N>(smem_u32(smem) + wg * 64 * pitch, pitch, acc, 0);
    const int quarter = warp & 3, half = warp >> 2;
    const int m = quarter * 32 + lane;
    const int r_in = tile * TILE_M + m;                           // dense pixel | padded pixel of this accumulator row
    bool valid = r_in < a.m_rows;
    int dense = 0, urow = 0;
    if (valid) {
        int b, y, x;
        if (a.in_dense) {
            x = r_in % a.width; y = (r_in / a.width) % a.height; b = r_in / (a.width * a.height);
        } else {
            const int line = r_in / a.wp;
            x = r_in - line * a.wp - 2;
            b = line / (a.height + 4);
            y = line - b * (a.height + 4) - 2;
            valid = x >= 0 && x < a.width && y >= 0 && y < a.height;
        }
        if (valid) {
            dense = (b * a.height + y) * a.width + x;
            urow = (int)macvo_rows::urow(b, y, x, a.height, a.width);
        }
    }
    const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
    const uint32_t stage_q = smem_u32(smem) + quarter * 32 * pitch;
    asm volatile("griddepcontrol.wait;" ::: "memory");            // nothing of the previous kernel is overwritten before it finished
    consumers_sync();                                              // all rows staged
    // (every lane runs every iteration — the shuffles below need the whole warp; lanes past the slice only skip the stores)
    for (int cg = 0; cg * 128 < N; ++cg) {
        const int col = cg * 128 + 4 * lane, gcol = slice * N + col;
        const bool lane_on = col < N;
        float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a.bias && lane_on) bb = __ldg(reinterpret_cast<const float4*>(a.bias + gcol));
        const int nv = lane_on ? a.n_valid - gcol : 0;       // valid columns among this lane's 4
#pragma unroll 4
        for (int i = 0; i < 16; ++i) {
            const int rr = half * 16 + i;
            const long long d = __shfl_sync(0xffffffffu, dense, rr), ur = __shfl_sync(0xffffffffu, urow, rr);
            if (!((vmask >> rr) & 1u) || nv <= 0) continue;
            float4 v = lds128(stage_q + rr * pitch + (((col >> 2) ^ (rr & 7)) << 4));
            v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w;
            if (a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            if (a.out32 && a.out32_planes) {
                const long long hw = (long long)a.height * a.width, img = d / hw;
                float* o = a.out32 + (img * a.n_valid + gcol) * hw + (d - img * hw);
                o[0] += v.x; if (nv > 1) o[hw] += v.y; if (nv > 2) o[2 * hw] += v.z; if (nv > 3) o[3 * hw] += v.w;
            } else if (a.out32) {
                float* o = a.out32 + d * a.out32_pitch + a.out32_off + gcol;
                if (nv >= 4 && ((a.out32_pitch | a.out32_off) & 3) == 0) *reinterpret_cast<float4*>(o) = v;
                else { o[0] = v.x; if (nv > 1) o[1] = v.y; if (nv > 2) o[2] = v.z; if (nv > 3) o[3] = v.w; }
            }
            if (a.out16) {
                // saturate instead of overflowing to inf (activations here are O(10); this is a guard, not a code path)
                const float lim = 65504.f;
                __half2 h2[2] = {__floats2half2_rn(fminf(fmaxf(v.x, -lim), lim), fminf(fmaxf(v.y, -lim), lim)),
                                 __floats2half2_rn(fminf(fmaxf(v.z, -lim), lim), fminf(fmaxf(v.w, -lim), lim))};
                __half* o = a.out16 + (a.out16_dense ? d : ur) * a.out16_pitch + a.out16_off + gcol;
                if (nv >= 4) *reinterpret_cast<uint2*>(o) = *reinterpret_cast<uint2*>(h2);
                else { o[0] = __low2half(h2[0]); if (nv > 1) o[1] = __high2half(h2[0]); if (nv > 2) o[2] = __low2half(h2[1]); }
            }
        }
    }
}

// 7x7 neighbourhood of the 2-channel flow as GEMM rows (the motion encoder's convf1, gru.py:50,57, becomes a 1x1 convolution):
// rows (pixels, 128) fp16, column (ky * 7 + kx) * 2 + c = flow[c, y + ky - 3, x + kx - 3] (zero outside), columns 98.. = 0.
// Also drops the flow itself into channels 126, 127 of the motion-feature rows (`cat([out, flow])`, gru.py:63).
__global__ void __launch_bounds__(256)
flow_im2col_kernel(const float* __restrict__ coords1, const float* __restrict__ coords0, __half* __restrict__ rows,
                   float* __restrict__ mf32, __half* __restrict__ mf16, int batch, int height, int width) {
    const int per = 32;                                            // 32 threads per pixel, 4 columns each
    const long long total = (long long)batch * height * width * per;
    const long long hw = (long long)height * width;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long p = e / per;
        const int q = (int)(e - p * per);
        const int x = (int)(p % width), y = (int)((p / width) % height), b = (int)(p / hw);
        const float* c1 = coords1 + (long long)b * 2 * hw;
        const float* c0 = coords0 + (long long)b * 2 * hw;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = 4 * q + j, tap = col >> 1, c = col & 1;
            const int yy = y + tap / 7 - 3, xx = x + tap % 7 - 3;
            v[j] = (col < 98 && yy >= 0 && yy < height && xx >= 0 && xx < width)
                       ? c1[c * hw + (long long)yy * width + xx] - c0[c * hw + (long long)yy * width + xx] : 0.f;
        }
        __half2 o[2] = {__floats2half2_rn(v[0], v[1]), __floats2half2_rn(v[2], v[3])};
        *reinterpret_cast<uint2*>(rows + p * 128 + 4 * q) = *reinterpret_cast<uint2*>(o);
        if (q == 0) {
            const float fx = c1[(long long)y * width + x] - c0[(long long)y * width + x];
            const float fy = c1[hw + (long long)y * width + x] - c0[hw + (long long)y * width + x];
            if (mf32) { mf32[p * 128 + 126] = fx; mf32[p * 128 + 127] = fy; }
            if (mf16) *reinterpret_cast<__half2*>(mf16 + macvo_rows::urow(b, y, x, height, width) * 128 + 126) = __floats2half2_rn(fx, fy);
        }
    }
}

template <int N>
int launch_conv(const CUtensorMap& map_a, const CUtensorMap& map_w, const ConvArgs& a, int tiles, int slices, int smem_bytes,
                cudaStream_t stream) {
    // the attribute belongs to the current device, so it is set on every launch (host-only, allowed under graph capture)
    MACVO_CUDA_TRY(cudaFuncSetAttribute(conv_tc_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(tiles, slices);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 1;
    MACVO_CUDA_TRY(cudaLaunchKernelEx(&cfg, conv_tc_kernel<N>, map_a, map_w, a));
    return MACVO_OK;
}

}  // namespace

extern "C" size_t macvo_rows_count(int batch, int height, int width, int vertical) {
    if (batch <= 0 || height <= 0 || width <= 0) return 0;
    return (size_t)macvo_rows::alloc_rows(batch, height, width, vertical);
}

extern "C" int macvo_conv_tc(const void* in_rows, int in_channels, int in_dense, const void* weights, const float* bias, int n_pad,
                             int n_valid, int ksize, int relu, int batch, int height, int width, void* out16, int out16_pitch,
                             int out16_offset, int out16_dense, float* out32, int out32_pitch, int out32_offset, int out32_planes,
                             void* stream) {
    if (!in_rows || !weights || batch <= 0 || height <= 0 || width <= 0 || in_channels <= 0 || in_channels % BLOCK_K ||
        n_pad <= 0 || n_pad % 32 || n_valid <= 0 || n_valid > n_pad || (ksize != 1 && ksize != 3) || (in_dense && ksize != 1) ||
        (!out16 && !out32) || (out16 && (out16_pitch % 4 || out16_offset % 4)))
        return MACVO_E_ARG;
    ConvArgs a = {};
    a.taps = ksize * ksize;
    a.kblocks = in_channels / BLOCK_K;
    a.in_dense = in_dense;
    a.batch = batch; a.height = height; a.width = width; a.wp = width + 4;
    a.m_rows = in_dense ? batch * height * width : macvo_rows::padded_pixels(batch, height, width, 0);
    const int tiles = (a.m_rows + TILE_M - 1) / TILE_M;
    int dev = 0, sms = 0;
    MACVO_CUDA_TRY(cudaGetDevice(&dev));
    MACVO_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    // slices of output channels: as many CTAs as fit one wave of the SMs, every slice a multiple of 32 columns (<= 256)
    int slices = 1;
    for (int s = 1; s <= 8; ++s)
        if (n_pad % (32 * s) == 0 && n_pad / s <= 256 && (tiles * s <= sms || n_pad / slices > 256)) slices = s;
    const int n_cta = n_pad / slices;
    if (n_cta > 256) return MACVO_E_UNSUPPORTED;
    const int slot_bytes = A_BYTES + n_cta * 128;
    a.slots = (SMEM_MAX - 2048) / slot_bytes;
    if (a.slots > 8) a.slots = 8;
    if (a.slots < 2 || a.slots * slot_bytes < TILE_M * n_cta * 4) return MACVO_E_UNSUPPORTED;    // epilogue staging reuses the ring
    const int smem_bytes = a.slots * slot_bytes + 512 + 1024;
    a.relu = relu; a.n_valid = n_valid; a.bias = bias;
    a.out16 = static_cast<__half*>(out16); a.out16_pitch = out16_pitch; a.out16_off = out16_offset; a.out16_dense = out16_dense;
    a.out32 = out32; a.out32_pitch = out32_pitch; a.out32_off = out32_offset; a.out32_planes = out32_planes;
    CUtensorMap map_a, map_w;
    const uint64_t in_rows_total = in_dense ? (uint64_t)a.m_rows : (uint64_t)macvo_rows::alloc_rows(batch, height, width, 0);
    if (!make_map_2d(&map_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, in_rows, in_channels, in_rows_total, (uint64_t)in_channels * 2, BLOCK_K, TILE_M))
        return MACVO_E_DRIVER;
    // filters (n_pad, taps * C): box = 64 channels of one tap x the slice's n_cta rows
    const uint64_t kk = (uint64_t)a.taps * in_channels;
    if (!make_map_2d(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, weights, kk, n_pad, kk * 2, BLOCK_K, n_cta)) return MACVO_E_DRIVER;
    cudaStream_t st = as_stream(stream);
    switch (n_cta) {
        case 32: return launch_conv<32>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        case 64: return launch_conv<64>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        case 96: return launch_conv<96>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        case 128: return launch_conv<128>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        case 160: return launch_conv<160>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        case 192: return launch_conv<192>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        case 224: return launch_conv<224>(map_a, map_w, a, tiles, slices, smem_bytes, st);
        default: return launch_conv<256>(map_a, map_w, a, tiles, slices, smem_bytes, st);
    }
}

extern "C" int macvo_flow_im2col(const float* coords1, const float* coords0, void* rows, float* mf32, void* mf16_rows, int batch,
                                 int height, int width, void* stream) {
    if (!coords1 || !coords0 || !rows || batch <= 0 || height <= 0 || width <= 0) return MACVO_E_ARG;
    const long long total = (long long)batch * height * width * 32;
    const int blocks = (int)((total + 255) / 256 < 132 * 8 ? (total + 255) / 256 : 132 * 8);
    flow_im2col_kernel<<<blocks, 256, 0, as_stream(stream)>>>(coords1, coords0, static_cast<__half*>(rows), mf32,
                                                              static_cast<__half*>(mf16_rows), batch, height, width);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
