// wgmma / TMA / mbarrier PTX wrappers and host-side tensor-map helpers shared by the sm_90a tensor-core kernels
// (corr_build_tc.cu: correlation volume; conv_tc.cu: decoder convolutions; gru_conv_tc.cu: SepConvGRU gates).
//
// All three share one CTA shape: warps 0..7 are two consumer warpgroups that issue wgmma (each owns 64 rows of the 128-row
// tile, fp32 accumulators in registers), warp 8 is the TMA producer feeding an mbarrier-guarded shared-memory ring.
// Descriptor bit layouts follow the PTX ISA (wgmma matrix descriptor) and the public CUTLASS / CuTe GmmaDescriptor.
#pragma once
#include "common.cuh"
#include "wgmma_ops.cuh"
#include <cuda.h>
#include <mutex>

namespace {

constexpr int TC_CONSUMER_THREADS = 256;                   // two warpgroups
constexpr int TC_THREADS = TC_CONSUMER_THREADS + 32;       // + the producer warp
constexpr int TC_PRODUCER_WARP = 8;

// ---- PTX wrappers ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must surface as a launch failure, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();          // ~2 s
    }
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .b32 r;\n\t.reg .pred p;\n\t"
        "elect.sync r|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// the two consumer warpgroups only (the producer warp never joins): named barrier 1
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMER_THREADS) : "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// explicit shared-space vector accesses for the epilogue transposes (the generic path compiles to LD.E / ST.E)
__device__ __forceinline__ void sts64(uint32_t addr, float a, float b) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps the compiler from touching accumulator registers across wgmma issue / wait points
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (wgmma):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (unused for swizzled K-major) | [32,46) SBO >> 4 | [62,64) layout = 1 (128B)
// rows are 128 B apart, 8-row groups (one swizzle atom) 1024 B apart; the tile base is 1024-byte aligned. The K slice of step
// k inside the 128-byte row starts k x 32 B further (16 fp16 | 8 fp32), i.e. descriptor + 2 k.
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// Stage a warpgroup's m64nN accumulator fragment as fp32 rows of `pitch` bytes with the 16-byte chunk c of row r stored at
// chunk c ^ (r & 7) (the layout the epilogues read back with lds128). `base` is the warpgroup's row 0.
template <int N>
__device__ __forceinline__ void stage_acc_rows(uint32_t base, int pitch, const float (&d)[N / 2], int col0) {
    const int lane = threadIdx.x & 31, wr = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int i = 0; i < N / 2; i += 2) {
        const int r = wr + 8 * ((i >> 1) & 1), c = col0 + 8 * (i >> 2) + 2 * (lane & 3);
        sts64(base + r * pitch + (((c >> 2) ^ (r & 7)) << 4) + (c & 3) * 4, d[i], d[i + 1]);
    }
}

// ---- host side: tensor maps ------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

// 3-D tensor map over a (batch, rows, inner) row-major array; box = (1, box_rows, box_inner), 128B swizzle
bool make_map_3d(CUtensorMap* map, CUtensorMapDataType dt, int elem_bytes, void* base, uint64_t inner, uint64_t rows,
                 uint64_t batch, uint32_t box_inner, uint32_t box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return false;
    cuuint64_t dims[3] = {inner, rows, batch};
    cuuint64_t strides[2] = {inner * elem_bytes, inner * rows * elem_bytes};
    cuuint32_t box[3] = {box_inner, box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    return enc(map, dt, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}


// 2-D tensor map over a (rows, inner) row-major array with an arbitrary row pitch; box = (box_rows, box_inner), 128B swizzle.
// Out-of-range box rows (negative or >= rows) are zero filled by the TMA unit: that IS the convolution's zero padding.
inline bool make_map_2d(CUtensorMap* map, CUtensorMapDataType dt, int elem_bytes, const void* base, uint64_t inner, uint64_t rows,
                        uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return false;
    cuuint64_t dims[2] = {inner, rows};
    cuuint64_t strides[1] = {row_pitch_bytes};
    cuuint32_t box[2] = {box_inner, box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace
