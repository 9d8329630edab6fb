// (f2) SepConvGRU on the Hopper tensor cores (wgmma): the 1x5 / 5x1 gate convolutions of the decoder's two recurrent units
// (flow + covariance) as implicit GEMMs with the gate math in the epilogue. Replaces, per refinement iteration and pass,
//   zr = conv(cat[h, x]) ; z, r = sigmoid(zr) ; q = tanh(conv(cat[r*h, x])) ; h = (1-z) h + z q
// (Module/Network/FlowFormer/core/gru.py:22-43, update blocks covhead.py:95-131) — 8 cuDNN convolutions + 8 glue launches per
// unit and iteration before, 4 launches now (stage 0: z|r, stage 1: q + blend, for each of the two passes).
//
// GEMM view of one stage: rows = pixels (M), columns = output channels (N = 256 for z|r, 128 for q), K = 5 taps x 512
// channels. Operands are fp16 (11-bit significand >= TF32's 10; the recurrent state itself stays fp32 in `h_master`, only
// the convolution INPUTS are rounded, like TF32 does on the fly), accumulation fp32 in registers.
//
// Layout (csrc/rows_layout.cuh): each pass sees the image as independent LINES along the convolution axis (rows of layout U
// for 1x5, columns = layout V for 5x1), every line with 2 zero pixels of padding at both ends. A tile is 128
// consecutive padded pixels; tap t of output pixel p reads pixel p + t - 2, so the A operand of (channel block, tap t) is the
// 128 rows starting t rows after the tile's first halo pixel, loaded by TMA into its own swizzle-aligned ring slot together
// with the tap's weight rows.
// The x part of the input (384 of the 512 channels: context | motion features | aggregated motion) is identical for both
// units and both stages: it lives in one buffer per layout; the h / r*h part is a separate 128-channel buffer per unit.
//
// One launch per unit, one CTA per 128-pixel tile: warps 0..7 = two consumer warpgroups (m64nNk16 wgmma), warp 8 = TMA producer.
#include "tc_common.cuh"
#include "rows_layout.cuh"
#include <cuda_fp16.h>

namespace {

constexpr int HID = 128, XCH = 384, CIN = HID + XCH, TAPS = 5;
constexpr int TILE_M = macvo_rows::TILE_M, BLOCK_K = 64, KBLOCKS = CIN / BLOCK_K;     // 8 channel blocks: 2 from h, 6 from x
constexpr int A_BYTES = TILE_M * 128;                                                // 16 KB
constexpr int GUARD = macvo_rows::GUARD;                                             // leading zero rows of every operand buffer

template <int N> struct Cfg {
    static constexpr int SLOT_BYTES = A_BYTES + N * 128;                             // A rows of one tap + its N weight rows
    static constexpr int SLOTS = N == 256 ? 4 : 6;
    static constexpr int SMEM = SLOTS * SLOT_BYTES + 512 + 1024;
    static_assert(SLOTS * SLOT_BYTES >= TILE_M * N * 4, "the epilogue stages the accumulators in the operand ring");
};

// MUFU-based gate functions (ex2 + rcp): absolute error ~1e-7, far below the fp16 rounding of the convolution operands
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 1.f - __fdividef(2.f, 1.f + __expf(2.f * x)); }

struct Unit {                    // one recurrent unit (flow / covariance)
    const float* bias;           // (N)
    float* h_master;             // (P, 128) fp32 recurrent state, dense pixel order
    float* z;                    // (P, 128) fp32 update gate: written by stage 0, read by stage 1
    __half* out;                 // stage 0: r*h rows of THIS pass's layout | stage 1: h rows of the OTHER pass's layout
};
struct Geometry {
    int batch, height, width, vertical;
    int lines, len, lp;          // lines of `len` pixels, padded pitch lp = len + 4
    int m_pad, tiles;            // padded pixels, 128-pixel tiles
};

// STAGE 0: N = 256 (z | r)   STAGE 1: N = 128 (q, then the blend)
template <int STAGE>
__global__ void __launch_bounds__(TC_THREADS, 1)
gru_conv_tc_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_x,
                   const __grid_constant__ CUtensorMap map_w, Unit u, Geometry g) {
    constexpr int N = STAGE == 0 ? 256 : 128;
    using C = Cfg<N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const uint32_t bar_full = smem_u32(smem + C::SLOTS * C::SLOT_BYTES), bar_empty = bar_full + 8 * C::SLOTS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;                                          // this CTA's 128 padded pixels

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::SLOTS; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2); }
        fence_barrier_init();
        prefetch_tmap(&map_h); prefetch_tmap(&map_x); prefetch_tmap(&map_w);
    }
    __syncthreads();
    // Programmatic dependent launch: the next stage may start as soon as every CTA of this one got here. Its weights and the x
    // part of its input (6 of the 8 channel blocks) do not depend on this stage, so the K loop runs the x blocks FIRST and only
    // the h / r*h blocks (and the epilogue's reads of h_master / z) wait for the previous stage (`griddepcontrol.wait`).
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    if (warp == TC_PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            int slot = 0; uint32_t phase = 0;
            for (int it = 0; it < KBLOCKS; ++it) {
                const int kb = (it + HID / BLOCK_K) % KBLOCKS;                 // 2, 3, ..., 7, 0, 1
                if (kb == 0) asm volatile("griddepcontrol.wait;" ::: "memory");
                for (int t = 0; t < TAPS; ++t) {
                    mbar_wait(bar_empty + 8 * slot, phase ^ 1);
                    const uint32_t full = bar_full + 8 * slot, sa = smem_u32(smem + slot * C::SLOT_BYTES);
                    mbar_expect_tx(full, C::SLOT_BYTES);
                    if (kb < HID / BLOCK_K) tma_load_2d(sa, &map_h, full, kb * BLOCK_K, tile * TILE_M + t);
                    else tma_load_2d(sa, &map_x, full, kb * BLOCK_K - HID, tile * TILE_M + t);
                    tma_load_2d(sa + A_BYTES, &map_w, full, t * CIN + kb * BLOCK_K, 0);
                    if (++slot == C::SLOTS) { slot = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== consumers: MMAs (one group in flight) =====================
    const int wg = warp >> 2;
    float acc[N / 2];
    {
        int slot = 0, prev = 0; uint32_t phase = 0;
        for (int s = 0; s < KBLOCKS * TAPS; ++s) {
            mbar_wait(bar_full + 8 * slot, phase);
            const uint32_t sa = smem_u32(smem + slot * C::SLOT_BYTES);
            const uint64_t da = make_kmajor_sw128_desc(sa + wg * 64 * 128), db = make_kmajor_sw128_desc(sa + A_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BLOCK_K / 16; ++k) Wgmma<N>::f16(acc, da + 2 * k, db + 2 * k, (s | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            if (s > 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * prev);
            prev = slot;
            if (++slot == C::SLOTS) { slot = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
    }

    // ===================== epilogue: accumulators -> smem transpose -> gate math -> coalesced global ==============
    // The accumulator fragment holds scattered (row, column pair) elements; each warpgroup stages its 64 rows through the (now idle)
    // operand ring as rows of N floats, 16-byte chunks XOR-swizzled by the row -> conflict-free reads, and global memory is
    // then accessed one full pixel row (512 B) per warp instruction. Warp (quarter, half) owns rows [32 quarter, +32).
    consumers_sync();                                                     // every MMA of both warpgroups read its operands
    stage_acc_rows<N>(smem_u32(smem) + wg * 64 * (N * 4), N * 4, acc, 0);
    const int quarter = warp & 3, half = warp >> 2;
    const int m = quarter * 32 + lane;
    const int pp = tile * TILE_M + m;                                 // padded pixel of this accumulator row
    const int line = pp / g.lp, pos = pp - line * g.lp - 2;
    int dense = 0, other = 0;                                         // dense pixel index | operand row in the other pass's layout
    bool valid = pp < g.m_pad && pos >= 0 && pos < g.len;
    if (valid) {
        int b, y, x;
        if (!g.vertical) { b = line / (g.height + 4); y = line - b * (g.height + 4) - 2; x = pos; valid = y >= 0 && y < g.height; }
        else { b = line / g.width; x = line - b * g.width; y = pos; }
        if (valid) {
            dense = (b * g.height + y) * g.width + x;
            other = (int)(!g.vertical ? macvo_rows::vrow(b, y, x, g.height, g.width) : macvo_rows::urow(b, y, x, g.height, g.width));
        }
    }
    const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
    const uint32_t stage_q = smem_u32(smem) + quarter * (32 * N * 4);   // this quarter's 32 rows x N fp32
    // the state rows this warp needs (h for r*h | h and z for the blend) were written by the PREVIOUS stage
    asm volatile("griddepcontrol.wait;" ::: "memory");
    constexpr int ROWS = STAGE == 0 ? 32 : 16;                        // rows finished by this warp
    const int row0 = STAGE == 0 ? 0 : half * 16;
    float4 hh[ROWS], zz[STAGE == 0 ? 1 : ROWS];
    if (STAGE == 1 || half == 1) {
#pragma unroll
        for (int i = 0; i < ROWS; ++i) {
            const long long d = __shfl_sync(0xffffffffu, dense, row0 + i);          // invalid rows carry 0: a harmless read
            hh[i] = *reinterpret_cast<const float4*>(u.h_master + d * HID + 4 * lane);
            if (STAGE == 1) zz[i] = *reinterpret_cast<const float4*>(u.z + d * HID + 4 * lane);
        }
    }
    consumers_sync();                                                     // all rows staged
    if (STAGE == 0) {
        // half 0: z columns [0, 128) -> z buffer      half 1: r columns [128, 256) -> r * h operand rows (this layout)
        const float4 bb = __ldg(reinterpret_cast<const float4*>(u.bias + half * 128 + 4 * lane));
#pragma unroll
        for (int rr = 0; rr < 32; ++rr) {
            const long long d = __shfl_sync(0xffffffffu, dense, rr);
            if (!((vmask >> rr) & 1u)) continue;
            const int c16 = half * 32 + lane;
            const float4 v = lds128(stage_q + rr * (N * 4) + ((c16 ^ (rr & 7)) << 4));
            float4 o;
            o.x = sigmoid_fast(v.x + bb.x); o.y = sigmoid_fast(v.y + bb.y); o.z = sigmoid_fast(v.z + bb.z); o.w = sigmoid_fast(v.w + bb.w);
            if (half == 0) {
                *reinterpret_cast<float4*>(u.z + d * HID + 4 * lane) = o;
            } else {
                __half2 h2[2] = {__floats2half2_rn(o.x * hh[rr].x, o.y * hh[rr].y), __floats2half2_rn(o.z * hh[rr].z, o.w * hh[rr].w)};
                const long long orow = (long long)GUARD + tile * TILE_M + quarter * 32 + rr;
                *reinterpret_cast<uint2*>(u.out + orow * HID + 4 * lane) = *reinterpret_cast<uint2*>(h2);
            }
        }
    } else {
        // h <- (1 - z) h + z tanh(q + bias)   (same association as gru.py:33,41); warp `half` finishes rows [16 half, +16)
        const float4 bb = __ldg(reinterpret_cast<const float4*>(u.bias + 4 * lane));
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int rr = row0 + i;
            const long long d = __shfl_sync(0xffffffffu, dense, rr);
            const long long orow = __shfl_sync(0xffffffffu, other, rr);
            if (!((vmask >> rr) & 1u)) continue;
            const float4 v = lds128(stage_q + rr * (N * 4) + ((lane ^ (rr & 7)) << 4));
            const float4 h4 = hh[i], z4 = zz[STAGE == 0 ? 0 : i];
            float4 n;
            n.x = (1.f - z4.x) * h4.x + z4.x * tanh_fast(v.x + bb.x);
            n.y = (1.f - z4.y) * h4.y + z4.y * tanh_fast(v.y + bb.y);
            n.z = (1.f - z4.z) * h4.z + z4.z * tanh_fast(v.z + bb.z);
            n.w = (1.f - z4.w) * h4.w + z4.w * tanh_fast(v.w + bb.w);
            *reinterpret_cast<float4*>(u.h_master + d * HID + 4 * lane) = n;
            __half2 h2[2] = {__floats2half2_rn(n.x, n.y), __floats2half2_rn(n.z, n.w)};
            *reinterpret_cast<uint2*>(u.out + orow * HID + 4 * lane) = *reinterpret_cast<uint2*>(h2);
        }
    }
}

// fp32 pixel rows (dense order) -> fp16 operand rows of one layout (pad rows are never written: they stay zero)
__global__ void __launch_bounds__(256)
pack_rows_kernel(const float* __restrict__ src, int src_pitch, int channels, __half* __restrict__ dst, int dst_pitch, int dst_offset,
                 int batch, int height, int width, int vertical) {
    const int quads = channels >> 2;
    const long long total = (long long)batch * height * width * quads;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long p = e / quads;
        const int q = (int)(e - p * quads);
        const int x = (int)(p % width), y = (int)((p / width) % height), b = (int)(p / ((long long)width * height));
        const long long row = !vertical ? macvo_rows::urow(b, y, x, height, width) : macvo_rows::vrow(b, y, x, height, width);
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + p * src_pitch + 4 * q));
        __half2 o[2] = {__floats2half2_rn(v.x, v.y), __floats2half2_rn(v.z, v.w)};
        *reinterpret_cast<uint2*>(dst + row * dst_pitch + dst_offset + 4 * q) = *reinterpret_cast<uint2*>(o);
    }
}

// per iteration: x channels [128, 384) = [mf | mf + gamma * agg] of BOTH layouts (gma.py:84-130 aggregation, covhead.py:118-121)
__global__ void __launch_bounds__(256)
pack_motion_kernel(const float* __restrict__ mf, const float* __restrict__ agg, const float* __restrict__ gamma,
                   __half* __restrict__ x_h, __half* __restrict__ x_v, int batch, int height, int width) {
    const long long total = (long long)batch * height * width * (HID / 4);
    const float gm = __ldg(gamma);
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long p = e / (HID / 4);
        const int q = (int)(e - p * (HID / 4));
        const int x = (int)(p % width), y = (int)((p / width) % height), b = (int)(p / ((long long)width * height));
        const long long rh = macvo_rows::urow(b, y, x, height, width), rv = macvo_rows::vrow(b, y, x, height, width);
        const float4 m = __ldg(reinterpret_cast<const float4*>(mf + p * HID + 4 * q));
        const float4 a = __ldg(reinterpret_cast<const float4*>(agg + p * HID + 4 * q));
        __half2 o[2] = {__floats2half2_rn(m.x, m.y), __floats2half2_rn(m.z, m.w)};
        __half2 s[2] = {__floats2half2_rn(m.x + gm * a.x, m.y + gm * a.y), __floats2half2_rn(m.z + gm * a.z, m.w + gm * a.w)};
        *reinterpret_cast<uint2*>(x_h + rh * XCH + HID + 4 * q) = *reinterpret_cast<uint2*>(o);
        *reinterpret_cast<uint2*>(x_h + rh * XCH + 2 * HID + 4 * q) = *reinterpret_cast<uint2*>(s);
        *reinterpret_cast<uint2*>(x_v + rv * XCH + HID + 4 * q) = *reinterpret_cast<uint2*>(o);
        *reinterpret_cast<uint2*>(x_v + rv * XCH + 2 * HID + 4 * q) = *reinterpret_cast<uint2*>(s);
    }
}

Geometry make_geometry(int batch, int height, int width, int vertical) {
    Geometry g;
    g.batch = batch; g.height = height; g.width = width; g.vertical = vertical;
    g.lines = vertical ? batch * width : batch * (height + 4);
    g.len = vertical ? height : width;
    g.lp = g.len + 4;
    g.m_pad = g.lines * g.lp;
    g.tiles = (g.m_pad + TILE_M - 1) / TILE_M;
    return g;
}
size_t operand_rows(const Geometry& g) { return (size_t)macvo_rows::alloc_rows(g.batch, g.height, g.width, g.vertical); }

// A operand: (rows, channels) fp16, box = 128 rows x 64 channels; tap t of tile i starts at row 128 i + t (operand row = padded
// pixel + GUARD, so that row is padded pixel 128 i + t - 2, the tap's input of the tile's first pixel)
bool make_map_a(CUtensorMap* map, const void* base, int channels, const Geometry& g) {
    return make_map_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, channels, operand_rows(g), (uint64_t)channels * 2, BLOCK_K, TILE_M);
}

template <int STAGE>
int launch_stage(const CUtensorMap* maps, Unit u, const Geometry& g, cudaStream_t stream) {
    constexpr int N = STAGE == 0 ? 256 : 128;
    // the attribute belongs to the current device, so it is set on every launch (host-only, allowed under graph capture)
    MACVO_CUDA_TRY(cudaFuncSetAttribute(gru_conv_tc_kernel<STAGE>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<N>::SMEM));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(g.tiles);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = Cfg<N>::SMEM;
    cfg.stream = stream;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 1;
    MACVO_CUDA_TRY(cudaLaunchKernelEx(&cfg, gru_conv_tc_kernel<STAGE>, maps[0], maps[1], maps[2], u, g));
    return MACVO_OK;
}

}  // namespace

extern "C" size_t macvo_gru_tc_operand_rows(int batch, int height, int width, int vertical) {
    if (batch <= 0 || height <= 0 || width <= 0) return 0;
    return operand_rows(make_geometry(batch, height, width, vertical));
}

extern "C" int macvo_gru_tc_pack(const float* src, int src_pitch, int channels, void* dst, int dst_channels, int dst_offset,
                                 int batch, int height, int width, int vertical, void* stream) {
    if (!src || !dst || batch <= 0 || height <= 0 || width <= 0 || channels <= 0 || channels % 4 || dst_offset % 4 ||
        src_pitch < channels || src_pitch % 4 || dst_offset + channels > dst_channels)
        return MACVO_E_ARG;
    const long long total = (long long)batch * height * width * (channels / 4);
    const int blocks = (int)((total + 255) / 256 < 132 * 8 ? (total + 255) / 256 : 132 * 8);
    pack_rows_kernel<<<blocks, 256, 0, as_stream(stream)>>>(src, src_pitch, channels, static_cast<__half*>(dst), dst_channels, dst_offset,
                                                            batch, height, width, vertical);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_gru_tc_pack_motion(const float* mf, const float* agg, const float* gamma, void* x_rows_h, void* x_rows_v,
                                        int batch, int height, int width, void* stream) {
    if (!mf || !agg || !gamma || !x_rows_h || !x_rows_v || batch <= 0 || height <= 0 || width <= 0) return MACVO_E_ARG;
    const long long total = (long long)batch * height * width * (HID / 4);
    const int blocks = (int)((total + 255) / 256 < 132 * 8 ? (total + 255) / 256 : 132 * 8);
    pack_motion_kernel<<<blocks, 256, 0, as_stream(stream)>>>(mf, agg, gamma, static_cast<__half*>(x_rows_h), static_cast<__half*>(x_rows_v),
                                                              batch, height, width);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_gru_tc_stage(int stage, int vertical, int batch, int height, int width, const void* h_rows, const void* x_rows,
                                  const void* weights, const float* bias, float* h_master, float* z, void* out_rows, void* stream) {
    if ((stage != 0 && stage != 1) || batch <= 0 || height <= 0 || width <= 0 || !h_rows || !x_rows || !weights || !bias ||
        !h_master || !z || !out_rows)
        return MACVO_E_ARG;
    const Geometry g = make_geometry(batch, height, width, vertical);
    const int n = stage == 0 ? 256 : 128;
    CUtensorMap maps[3];                                                  // h | x | weights
    if (!make_map_a(&maps[0], h_rows, HID, g) || !make_map_a(&maps[1], x_rows, XCH, g) ||
        !make_map_2d(&maps[2], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, weights, (uint64_t)TAPS * CIN, n, (uint64_t)TAPS * CIN * 2, BLOCK_K, n))
        return MACVO_E_UNSUPPORTED;
    Unit u;
    u.bias = bias; u.h_master = h_master; u.z = z; u.out = static_cast<__half*>(out_rows);
    return stage == 0 ? launch_stage<0>(maps, u, g, as_stream(stream)) : launch_stage<1>(maps, u, g, as_stream(stream));
}
