// Frontend "next" rows (SURVEY.md §8f-1/2): the memory-bound glue of the FlowFormerCov cost perceiver that
// cuDNN / ATen run far below HBM speed at these shapes (SURVEY.md §8f):
//
//   layer_norm          (9600*80, 128) fp32: ATen 1136 us for 786 MB of traffic      -> warp-per-row kernel
//   patch_embed_conv1   1 -> 16 ch, 6x6 stride 2 over 9600 cost maps: cuDNN 3636 us  -> direct conv, map in smem,
//                       fused zero padding (F.pad to a multiple of 8) + bias + ReLU, NHWC output
//   small_attention     head_dim 16 / 32, <= 512 keys, fp32: SDPA (mem-efficient sm80 kernel) 0.3 - 2.8 ms per call
//                       -> K, V of one (batch, head) staged in shared memory, one query per thread, online softmax
//
// They replace torch ops inside the network (Module/Network/FlowFormer/core/encoder.py:12-55 PatchEmbed,
// core/attention.py:6-29, core/twins.py:103-114,173-183, core/Twins/svt_large.py:111-114,161-164); numerics:
// fp32 throughout, exact erf-free ops only, parity vs torch fp32 in tests/test_gpu_nn_kernels.py.
#include "common.cuh"
#include "layer_norm_row.cuh"
#include <math_constants.h>

namespace {

// float2 multiply-add / multiply, one correctly rounded FMA / FMUL per component (sm_90 has no paired FFMA2 instruction)
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// ---- LayerNorm over the last dimension, one warp per row, C = 32 * VPL --------------------------------
template <int VPL>
__global__ void __launch_bounds__(256)
layer_norm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                  float* __restrict__ y, long long rows, float eps, const float* __restrict__ resid = nullptr,
                  float* __restrict__ sum_out = nullptr) {
    constexpr int C = 32 * VPL;
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* xr = x + row * C;
    float v[VPL];
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i) {                           // lane owns float4 chunks lane + 32 i
        float4 t = *reinterpret_cast<const float4*>(xr + (lane + 32 * i) * 4);
        if (resid) {   // fused residual: LN(x + r), the sum written out as the new residual stream (one pass instead of add + LN)
            const float4 r = *reinterpret_cast<const float4*>(resid + row * C + (lane + 32 * i) * 4);
            t = make_float4(t.x + r.x, t.y + r.y, t.z + r.z, t.w + r.w);
            *reinterpret_cast<float4*>(sum_out + row * C + (lane + 32 * i) * 4) = t;
        }
        v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
    layer_norm_row<VPL>(v, w, b, eps, lane);
    float* yr = y + row * C;
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i)
        *reinterpret_cast<float4*>(yr + (lane + 32 * i) * 4) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
}

// C = 64: two channels per lane
__global__ void __launch_bounds__(256)
layer_norm64_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                    float* __restrict__ y, long long rows, float eps) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float2 t = *reinterpret_cast<const float2*>(x + row * 64 + lane * 2);
    const float mean = warp_sum(t.x + t.y) * (1.f / 64);
    const float d0 = t.x - mean, d1 = t.y - mean;
    const float rstd = rsqrtf(warp_sum(fmaf(d0, d0, d1 * d1)) * (1.f / 64) + eps);
    const float2 ww = *reinterpret_cast<const float2*>(w + lane * 2), bb = *reinterpret_cast<const float2*>(b + lane * 2);
    *reinterpret_cast<float2*>(y + row * 64 + lane * 2) = make_float2(d0 * rstd * ww.x + bb.x, d1 * rstd * ww.y + bb.y);
}

// x[r, :] = relu(x[r, :] + term[r % period, :]) in place: PatchEmbed's ffn_with_coord.0 after the position half of its
// input has been folded into a per-patch-position bias (encoder.py:40-52); channels % 4 == 0.
__global__ void __launch_bounds__(256)
add_rows_relu_kernel(float* __restrict__ x, const float* __restrict__ term, long long rows, int period, int c4) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * c4) return;
    const long long r = e / c4;
    const int c = (int)(e % c4);
    float4 v = reinterpret_cast<float4*>(x)[e];
    const float4 t = __ldg(reinterpret_cast<const float4*>(term) + (r % period) * c4 + c);
    v.x = fmaxf(v.x + t.x, 0.f); v.y = fmaxf(v.y + t.y, 0.f); v.z = fmaxf(v.z + t.z, 0.f); v.w = fmaxf(v.w + t.w, 0.f);
    reinterpret_cast<float4*>(x)[e] = v;
}

// ---- PatchEmbed conv1: (M,1,H,W) -> ReLU(conv 6x6 s2 p2, 16 ch) as (M, Ho, Wo, 16) NHWC -----------------
// The reference first zero-pads H, W up to multiples of 8 (encoder.py:35-38); here out-of-range taps simply
// read 0. One CTA per cost map: the whole map (<= 96 x 160 fp32) sits in shared memory.
constexpr int PE_C = 16, PE_K = 6;
// filter taps [tap][channel] + bias in constant memory: with the tap loops fully unrolled every FFMA takes its weight
// as a constant-bank operand — no shared-memory traffic for the 576 weights (the first version was LSU-bound on them)
__constant__ float c_pe_w[PE_K * PE_K * PE_C + PE_C];
__device__ float g_pe_pack[PE_K * PE_K * PE_C + PE_C];       // staging for the repacked filter

__global__ void pe_pack_weights_kernel(const float* __restrict__ wgt, const float* __restrict__ bias, float* __restrict__ packed) {
    const int e = threadIdx.x + blockIdx.x * blockDim.x;
    if (e < PE_C * 36) { const int c = e / 36, t = e % 36; packed[t * PE_C + c] = wgt[e]; }      // (16,1,6,6) -> [tap][ch]
    else if (e < PE_C * 36 + PE_C) packed[e] = bias[e - PE_C * 36];
}

__global__ void __launch_bounds__(320)
patch_conv1_kernel(const float* __restrict__ maps, float* __restrict__ out, int h, int w, int ho, int wo) {
    extern __shared__ float sm[];
    float* s_map = sm;                                   // (2 ho + 4) x (2 wo + 4): 2-pixel zero frame on the top / left
    const int hp = 2 * ho + 4, wp = 2 * wo + 4;          // covers every tap of every output
    const float* src = maps + (long long)blockIdx.x * h * w;
    for (int e = threadIdx.x; e < hp * wp; e += blockDim.x) {
        const int y = e / wp - 2, x = e % wp - 2;
        s_map[e] = (y >= 0 && y < h && x >= 0 && x < w) ? __ldg(src + y * w + x) : 0.f;
    }
    __syncthreads();
    float* dst = out + (long long)blockIdx.x * ho * wo * PE_C;
    const int wo2 = wo >> 1;                                          // wo is a multiple of 4
    for (int p = threadIdx.x; p < ho * wo2; p += blockDim.x) {        // two horizontally adjacent outputs per thread
        const int oy = p / wo2, ox = (p % wo2) * 2;
        float a0[PE_C], a1[PE_C];
#pragma unroll
        for (int c = 0; c < PE_C; ++c) a0[c] = a1[c] = c_pe_w[PE_K * PE_K * PE_C + c];
        const float* base = s_map + (2 * oy) * wp + 2 * ox;           // tap (ky,kx) reads input (2oy-2+ky, 2ox-2+kx)
#pragma unroll
        for (int ky = 0; ky < PE_K; ++ky) {
            float x[8];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 t = *reinterpret_cast<const float2*>(base + ky * wp + 2 * e);
                x[2 * e] = t.x; x[2 * e + 1] = t.y;
            }
#pragma unroll
            for (int kx = 0; kx < PE_K; ++kx)
#pragma unroll
                for (int c = 0; c < PE_C; ++c) {
                    const float wv = c_pe_w[(ky * PE_K + kx) * PE_C + c];
                    a0[c] = fmaf(x[kx], wv, a0[c]);
                    a1[c] = fmaf(x[kx + 2], wv, a1[c]);
                }
        }
        float4* o = reinterpret_cast<float4*>(dst + ((long long)oy * wo + ox) * PE_C);   // 2 x 16 channels = 128 B
#pragma unroll
        for (int c4 = 0; c4 < PE_C / 4; ++c4) {
            o[c4] = make_float4(fmaxf(a0[4 * c4], 0.f), fmaxf(a0[4 * c4 + 1], 0.f), fmaxf(a0[4 * c4 + 2], 0.f), fmaxf(a0[4 * c4 + 3], 0.f));
            o[4 + c4] = make_float4(fmaxf(a1[4 * c4], 0.f), fmaxf(a1[4 * c4 + 1], 0.f), fmaxf(a1[4 * c4 + 2], 0.f), fmaxf(a1[4 * c4 + 3], 0.f));
        }
    }
}

// ---- small-head attention: softmax(q k^T / sqrt(D)) v, fp32, K/V of one (batch, head) in shared memory ----
// layouts: q (B or 1, Nq, H, D), k/v (B, Nk, H, D), out (B, Nq, H, D)  — i.e. the (tokens, heads*dim) matrices the
// linear layers produce, no permutes. q_bstride == 0 broadcasts one query set over the batch.
// optional operand layout + additive position terms of the shared-K/V kernels:
//   row strides (floats) of q / k / v so that a fused [q|k|v] projection output can be consumed in place, and
//   q_add (period, nq, heads*D), k_add (period, nk, heads*D) added to q / k on load, batch b using slice b % period
//   (the position / context half of a projection whose input was cat([x, context]) + position encoding).
struct AttnExtra {
    int ldq, ldk, ldv, period;
    const float* q_add;
    const float* k_add;
};

constexpr int ATT_CHUNK = 4;     // keys per online-softmax update (one rescale of the accumulator per chunk)

template <int D>
__global__ void __launch_bounds__(128)
attn_shared_kv_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                      float* __restrict__ out, int nq, int nk, int heads, long long q_bstride, float scale, AttnExtra ex) {
    extern __shared__ float sm[];
    const int nkp = (nk + ATT_CHUNK - 1) / ATT_CHUNK * ATT_CHUNK;
    float* sk = sm;                 // [nkp][D], rows >= nk zero
    float* sv = sm + nkp * D;
    const int b = blockIdx.z, hd = blockIdx.y;
    const float* kadd = ex.k_add ? ex.k_add + ((long long)(b % ex.period) * nk * heads + hd) * D : nullptr;
    for (int e = threadIdx.x; e < nkp * (D / 4); e += blockDim.x) {
        const int j = e / (D / 4), c = e % (D / 4);
        float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
        if (j < nk) {
            kk = *reinterpret_cast<const float4*>(k + ((long long)b * nk + j) * ex.ldk + hd * D + c * 4);
            vv = *reinterpret_cast<const float4*>(v + ((long long)b * nk + j) * ex.ldv + hd * D + c * 4);
            if (kadd) {
                const float4 t = *reinterpret_cast<const float4*>(kadd + (long long)j * heads * D + c * 4);
                kk.x += t.x; kk.y += t.y; kk.z += t.z; kk.w += t.w;
            }
        }
        *reinterpret_cast<float4*>(sk + j * D + c * 4) = kk;
        *reinterpret_cast<float4*>(sv + j * D + c * 4) = vv;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    float2 qr[D / 2], acc[D / 2];
    const float* qp = q + (long long)b * q_bstride + (long long)i * ex.ldq + hd * D;
    const float* qa = ex.q_add ? ex.q_add + (((long long)(b % ex.period) * nq + i) * heads + hd) * D : nullptr;
#pragma unroll
    for (int c = 0; c < D / 4; ++c) {
        float4 t = *reinterpret_cast<const float4*>(qp + 4 * c);
        if (qa) { const float4 u = *reinterpret_cast<const float4*>(qa + 4 * c); t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w; }
        qr[2 * c] = make_float2(t.x * scale, t.y * scale);
        qr[2 * c + 1] = make_float2(t.z * scale, t.w * scale);
    }
#pragma unroll
    for (int c = 0; c < D / 2; ++c) acc[c] = make_float2(0.f, 0.f);
    float m = -CUDART_INF_F, l = 0.f;
    for (int j0 = 0; j0 < nkp; j0 += ATT_CHUNK) {
        float s[ATT_CHUNK];
#pragma unroll
        for (int u = 0; u < ATT_CHUNK; ++u) {
            const float4* kj = reinterpret_cast<const float4*>(sk + (j0 + u) * D);
            float2 t = make_float2(0.f, 0.f);
#pragma unroll
            for (int c = 0; c < D / 4; ++c) {
                const float4 kk = kj[c];
                t = ffma2_rn(qr[2 * c], make_float2(kk.x, kk.y), t);
                t = ffma2_rn(qr[2 * c + 1], make_float2(kk.z, kk.w), t);
            }
            s[u] = (j0 + u < nk) ? t.x + t.y : -CUDART_INF_F;
        }
        float mn = m;
#pragma unroll
        for (int u = 0; u < ATT_CHUNK; ++u) mn = fmaxf(mn, s[u]);
        const float corr = __expf(m - mn);
        m = mn;
        l *= corr;
        const float2 c2 = make_float2(corr, corr);
#pragma unroll
        for (int c = 0; c < D / 2; ++c) acc[c] = fmul2_rn(acc[c], c2);
#pragma unroll
        for (int u = 0; u < ATT_CHUNK; ++u) {
            const float p = __expf(s[u] - mn);
            l += p;
            const float2 p2 = make_float2(p, p);
            const float4* vj = reinterpret_cast<const float4*>(sv + (j0 + u) * D);
#pragma unroll
            for (int c = 0; c < D / 4; ++c) {
                const float4 vv = vj[c];
                acc[2 * c] = ffma2_rn(p2, make_float2(vv.x, vv.y), acc[2 * c]);
                acc[2 * c + 1] = ffma2_rn(p2, make_float2(vv.z, vv.w), acc[2 * c + 1]);
            }
        }
    }
    const float inv = 1.f / l;
    float* op = out + (((long long)b * nq + i) * heads + hd) * D;
#pragma unroll
    for (int c = 0; c < D / 4; ++c)
        *reinterpret_cast<float4*>(op + 4 * c) = make_float4(acc[2 * c].x * inv, acc[2 * c].y * inv, acc[2 * c + 1].x * inv,
                                                             acc[2 * c + 1].y * inv);
}

// ---- tensor-core variant (TF32 mma.sync m16n8k8, fp32 accumulate): used when the caller allows TF32 matmuls, like
// the reference frontend does for its attention bmm's (Frontend.py:275-277). One warp = 16 queries; K, V of the
// (batch, head) in shared memory (tf32-rounded, row stride D + 4 -> conflict-free fragment loads); flash-style online
// softmax over blocks of 32 keys. The P tile comes out of the QK^T mma in the accumulator layout (columns 2t, 2t+1)
// and is fed straight back as the A operand of the PV mma by declaring A-column t <-> key 2t, t+4 <-> key 2t+1 and
// loading V's B fragment with the same key permutation: no shuffles, no shared-memory round trip.
__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float ex2f(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Shared-memory fragment layouts (both conflict-free for 128-bit loads, one LDS.128 feeds two mma B operands):
//   K row j (stride STK = 16 mod 32 words):  word (ks/2)*16 + t*4 + (ks%2)*2 + h  holds K[j][ks*8 + t + 4h]
//     -> lane (g,t) reads uint4 at row (key g), word (ks/2)*16 + t*4 = {b0,b1 of k-step ks, b0,b1 of k-step ks+1}
//   V block of 8 keys kb8, column pair-tile ndp: word (((ndp*nkb8 + kb8)*8 + g)*4 + t)*4 + (key&1)*2 + (nd&1)
//     holds V[kb8*8 + 2t + (key&1)][(2 ndp + (nd&1))*8 + g]  -> uint4 = {b0(nd even), b0(nd odd), b1(nd even), b1(nd odd)}
template <int D>
__global__ void __launch_bounds__(256)
attn_tc_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
               float* __restrict__ out, int nq, int nk, int heads, long long q_bstride, float scale, AttnExtra ex) {
    extern __shared__ float sm[];
    constexpr int KS = D / 8, STK = (D / 32) * 32 + 16, NVH = D / 16;
    const int nkp = (nk + 31) / 32 * 32, nkb8 = nkp / 8;
    uint32_t* sk = reinterpret_cast<uint32_t*>(sm);      // [nkp][STK]
    uint32_t* sv = sk + nkp * STK;                       // [NVH][nkb8][8][4][4]
    const int b = blockIdx.z, hd = blockIdx.y;
    const float* kadd = ex.k_add ? ex.k_add + ((long long)(b % ex.period) * nk * heads + hd) * D : nullptr;
    constexpr int FILL_U = 4;                                        // row loads in flight per thread
    for (int e0 = threadIdx.x; e0 < nkp * (D / 4); e0 += blockDim.x * FILL_U) {
        float4 kb_[FILL_U], vb_[FILL_U];
#pragma unroll
        for (int u = 0; u < FILL_U; ++u) {
            const int e = e0 + u * blockDim.x, j = e / (D / 4), c = (e % (D / 4)) * 4;
            kb_[u] = vb_[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j < nk) {
                kb_[u] = *reinterpret_cast<const float4*>(k + ((long long)b * nk + j) * ex.ldk + hd * D + c);
                vb_[u] = *reinterpret_cast<const float4*>(v + ((long long)b * nk + j) * ex.ldv + hd * D + c);
                if (kadd) {
                    const float4 w = *reinterpret_cast<const float4*>(kadd + (long long)j * heads * D + c);
                    kb_[u].x += w.x; kb_[u].y += w.y; kb_[u].z += w.z; kb_[u].w += w.w;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < FILL_U; ++u) {
            const int e = e0 + u * blockDim.x, j = e / (D / 4), c = (e % (D / 4)) * 4;
            if (j < nkp) {
                const int ks = c >> 3, h = (c >> 2) & 1;                       // c..c+3 -> t = 0..3 of (k-step ks, half h)
                uint32_t* kd = sk + j * STK + (ks >> 1) * 16 + (ks & 1) * 2 + h;
                kd[0] = to_tf32(kb_[u].x); kd[4] = to_tf32(kb_[u].y); kd[8] = to_tf32(kb_[u].z); kd[12] = to_tf32(kb_[u].w);
                const int nd = c >> 3, g0 = c & 7;                             // c..c+3 -> g = g0..g0+3 of column tile nd
                uint32_t* vd = sv + ((((nd >> 1) * nkb8 + (j >> 3)) * 8 + g0) * 4 + ((j & 7) >> 1)) * 4 + (j & 1) * 2 + (nd & 1);
                vd[0] = to_tf32(vb_[u].x); vd[16] = to_tf32(vb_[u].y); vd[32] = to_tf32(vb_[u].z); vd[48] = to_tf32(vb_[u].w);
            }
        }
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int q0 = (blockIdx.x * (blockDim.x >> 5) + warp) * 16;
    if (q0 >= nq) return;
    const int r0 = q0 + g, r1 = q0 + g + 8;
    const float* qb = q + (long long)b * q_bstride + (long long)hd * D;
    const int c0r = min(r0, nq - 1), c1r = min(r1, nq - 1);
    const float* q0p = qb + (long long)c0r * ex.ldq;
    const float* q1p = qb + (long long)c1r * ex.ldq;
    const float* qa = ex.q_add ? ex.q_add + ((long long)(b % ex.period) * nq * heads + hd) * D : nullptr;
    const float sl2 = scale * 1.4426950408889634f;                  // scores in log2 units: p = 2^(s - m)
    uint32_t a[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        float x0 = q0p[ks * 8 + t], x1 = q1p[ks * 8 + t], x2 = q0p[ks * 8 + t + 4], x3 = q1p[ks * 8 + t + 4];
        if (qa) {
            const float* a0p = qa + (long long)c0r * heads * D + ks * 8 + t;
            const float* a1p = qa + (long long)c1r * heads * D + ks * 8 + t;
            x0 += a0p[0]; x1 += a1p[0]; x2 += a0p[4]; x3 += a1p[4];
        }
        a[ks][0] = to_tf32(x0 * sl2);
        a[ks][1] = to_tf32(x1 * sl2);
        a[ks][2] = to_tf32(x2 * sl2);
        a[ks][3] = to_tf32(x3 * sl2);
    }
    float acc[KS][4];
#pragma unroll
    for (int nd = 0; nd < KS; ++nd) acc[nd][0] = acc[nd][1] = acc[nd][2] = acc[nd][3] = 0.f;
    float m0 = -CUDART_INF_F, m1 = -CUDART_INF_F, l0 = 0.f, l1 = 0.f;
    const uint32_t* kbase = sk + g * STK + t * 4;
    const uint32_t* vbase = sv + (g * 4 + t) * 4;
    for (int kb = 0; kb < nkp; kb += 32) {
        float s[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            const uint32_t* kr = kbase + (kb + nt * 8) * STK;
#pragma unroll
            for (int kp = 0; kp < KS / 2; ++kp) {
                const uint4 kq = *reinterpret_cast<const uint4*>(kr + kp * 16);
                mma_tf32(s[nt], a[2 * kp], kq.x, kq.y);
                mma_tf32(s[nt], a[2 * kp + 1], kq.z, kq.w);
            }
        }
        if (kb + 32 > nk) {                                  // ragged tail: keys >= nk do not take part
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int key = kb + nt * 8 + 2 * t;
                if (key >= nk) s[nt][0] = s[nt][2] = -CUDART_INF_F;
                if (key + 1 >= nk) s[nt][1] = s[nt][3] = -CUDART_INF_F;
            }
        }
        float x0 = s[0][0], x1 = s[0][2];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            x0 = fmaxf(x0, fmaxf(s[nt][0], s[nt][1]));
            x1 = fmaxf(x1, fmaxf(s[nt][2], s[nt][3]));
        }
        x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
        const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);
        const float c0 = ex2f(m0 - n0), c1 = ex2f(m1 - n1);
        m0 = n0; m1 = n1;
        l0 *= c0; l1 *= c1;
#pragma unroll
        for (int nd = 0; nd < KS; ++nd) { acc[nd][0] *= c0; acc[nd][1] *= c0; acc[nd][2] *= c1; acc[nd][3] *= c1; }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const float p00 = ex2f(s[nt][0] - n0), p01 = ex2f(s[nt][1] - n0);
            const float p10 = ex2f(s[nt][2] - n1), p11 = ex2f(s[nt][3] - n1);
            l0 += p00 + p01; l1 += p10 + p11;
            const uint32_t pa[4] = {to_tf32(p00), to_tf32(p10), to_tf32(p01), to_tf32(p11)};   // A cols t <-> key 2t, t+4 <-> 2t+1
            const uint32_t* vr = vbase + ((kb >> 3) + nt) * 128;
#pragma unroll
            for (int ndp = 0; ndp < NVH; ++ndp) {
                const uint4 vq = *reinterpret_cast<const uint4*>(vr + ndp * nkb8 * 128);
                mma_tf32(acc[2 * ndp], pa, vq.x, vq.z);
                mma_tf32(acc[2 * ndp + 1], pa, vq.y, vq.w);
            }
        }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    float* ob = out + ((long long)b * nq * heads + hd) * D;
#pragma unroll
    for (int nd = 0; nd < KS; ++nd) {
        if (r0 < nq) *reinterpret_cast<float2*>(ob + (long long)r0 * heads * D + nd * 8 + 2 * t) = make_float2(acc[nd][0] * i0, acc[nd][1] * i0);
        if (r1 < nq) *reinterpret_cast<float2*>(ob + (long long)r1 * heads * D + nd * 8 + 2 * t) = make_float2(acc[nd][2] * i1, acc[nd][3] * i1);
    }
}

// ---- PatchEmbed conv1 on the tensor cores (TF32 mma.sync implicit GEMM), used when the caller allows TF32 convolutions
// like cuDNN does for the reference (torch.backends.cudnn.allow_tf32): per cost map M = ho*wo output positions,
// N = 16 channels, K = 36 taps (padded to 40). The A fragment is gathered straight from the map in shared memory
// (neighbouring lanes read overlapping pixels -> broadcasts, no conflicts); the 16 x 40 filter lives in 20 registers.
__global__ void __launch_bounds__(256)
patch_conv1_tc_kernel(const float* __restrict__ maps, const float* __restrict__ wgt, const float* __restrict__ bias,
                      float* __restrict__ out, int h, int w, int ho, int wo, int s2d) {
    extern __shared__ float sm[];
    uint32_t* s_map = reinterpret_cast<uint32_t*>(sm);   // tf32 map with a 2-pixel zero frame on the top / left, (2ho+4) x (2wo+4)
    const int hp = 2 * ho + 4, wp = 2 * wo + 4;
    const float* src = maps + (long long)blockIdx.x * h * w;
    for (int e = threadIdx.x; e < hp * wp; e += blockDim.x) {
        const int y = e / wp - 2, x = e % wp - 2;
        s_map[e] = (y >= 0 && y < h && x >= 0 && x < w) ? to_tf32(__ldg(src + y * w + x)) : 0u;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    // B fragments: b0 = W[tap = 8 ks + t][c = 8 nt + g], b1 = W[tap + 4][c]; wgt is (16, 1, 6, 6) = [c][tap]
    uint32_t bw[5][2][2];
    int toff[5][2];                                      // smem offset of tap (ky, kx) relative to the window origin
#pragma unroll
    for (int ks = 0; ks < 5; ++ks)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int tap = ks * 8 + t + 4 * hh;
            toff[ks][hh] = tap < 36 ? (tap / 6) * wp + tap % 6 : 0;
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) bw[ks][nt][hh] = tap < 36 ? to_tf32(__ldg(wgt + (nt * 8 + g) * 36 + tap)) : 0u;
        }
    const float2 bia0 = make_float2(__ldg(bias + 2 * t), __ldg(bias + 2 * t + 1));
    const float2 bia1 = make_float2(__ldg(bias + 8 + 2 * t), __ldg(bias + 8 + 2 * t + 1));
    __syncthreads();
    float* dst = out + (long long)blockIdx.x * ho * wo * PE_C;
    const int npos = ho * wo;
    for (int p0 = warp * 16; p0 < npos; p0 += (blockDim.x >> 5) * 16) {
        const int pa = min(p0 + g, npos - 1), pb = min(p0 + g + 8, npos - 1);
        const uint32_t* wa = s_map + (2 * (pa / wo)) * wp + 2 * (pa % wo);      // window origin of position pa
        const uint32_t* wb = s_map + (2 * (pb / wo)) * wp + 2 * (pb % wo);
        float c0[4] = {bia0.x, bia0.y, bia0.x, bia0.y}, c1[4] = {bia1.x, bia1.y, bia1.x, bia1.y};
#pragma unroll
        for (int ks = 0; ks < 5; ++ks) {
            const uint32_t a[4] = {wa[toff[ks][0]], wb[toff[ks][0]], wa[toff[ks][1]], wb[toff[ks][1]]};
            mma_tf32(c0, a, bw[ks][0][0], bw[ks][0][1]);
            mma_tf32(c1, a, bw[ks][1][0], bw[ks][1][1]);
        }
        // output position -> row offset (in units of 16 channels). s2d: the NHWC tensor is written space-to-depth, i.e. as the
        // (ho/2, wo/2, 4 x 16) tensor whose channel block (y & 1) * 2 + (x & 1) holds pixel (y, x): the following 6x6 / stride-2
        // convolution over 16 channels is then a 3x3 / stride-1 convolution over 64 channels — the same arithmetic with full
        // 32-channel K blocks for the implicit GEMM instead of half-empty ones (PatchEmbed proj.2, encoder.py:24-27)
        auto row_of = [&](int p) -> long long {
            if (!s2d) return p;
            const int y = p / wo, x = p - y * wo;
            return ((long long)(y >> 1) * (wo >> 1) + (x >> 1)) * 4 + ((y & 1) * 2 + (x & 1));
        };
        if (p0 + g < npos) {
            float* o = dst + row_of(p0 + g) * PE_C;
            *reinterpret_cast<float2*>(o + 2 * t) = make_float2(fmaxf(c0[0], 0.f), fmaxf(c0[1], 0.f));
            *reinterpret_cast<float2*>(o + 8 + 2 * t) = make_float2(fmaxf(c1[0], 0.f), fmaxf(c1[1], 0.f));
        }
        if (p0 + g + 8 < npos) {
            float* o = dst + row_of(p0 + g + 8) * PE_C;
            *reinterpret_cast<float2*>(o + 2 * t) = make_float2(fmaxf(c0[2], 0.f), fmaxf(c0[3], 0.f));
            *reinterpret_cast<float2*>(o + 8 + 2 * t) = make_float2(fmaxf(c1[2], 0.f), fmaxf(c1[3], 0.f));
        }
    }
}

// ---- perceiver input layer, fused (core/encoder.py:150-191, attention.py:32-68) ---------------------------------------
// 8 learned latents cross-attend to the 80 patch tokens of every cost map. With q shared by all maps, linearity gives
//     score[i,h,j] = q[i,h] . (Wk[h] t_j + bk[h]) = (Wk[h]^T q[i,h]) . t_j + const     (const drops out of the softmax)
//     out[i,h]     = sum_j p_j (Wv[h] t_j + bv[h]) = Wv[h] (sum_j p_j t_j) + bv[h]
// so neither K nor V (2 x 393 MB at 640x480, plus their two GEMMs) is ever materialised: one CTA per cost map runs a
// 64-"query" (row = h*8+i of U^T = Wk^T q, pre-scaled), 128-dim attention whose keys AND values are the token rows,
// then projects the pooled tokens with Wv. TF32 mma.sync, fp32 softmax/accumulate; tokens are read exactly once.
constexpr int LP_D = 128, LP_HEADS = 8, LP_HD = 16;   // 64 score rows = 8 heads x 8 latents
__global__ void __launch_bounds__(128)
latent_pool_kernel(const float* __restrict__ tokens, const float* __restrict__ ut, const float* __restrict__ wv,
                   const float* __restrict__ bv, float* __restrict__ out, int nk) {
    extern __shared__ float sm[];
    constexpr int ST = LP_D + 4, KS = LP_D / 8;
    const int nkp = (nk + 31) / 32 * 32;
    uint32_t* st = reinterpret_cast<uint32_t*>(sm);                  // [nkp][ST] tf32 tokens, rows >= nk zero
    const long long b = blockIdx.x;
    const float* tb = tokens + b * nk * LP_D;
    constexpr int FILL_U = 8;                                        // loads in flight per thread (the fill is latency bound)
    for (int e0 = threadIdx.x; e0 < nkp * (LP_D / 4); e0 += blockDim.x * FILL_U) {
        float4 buf[FILL_U];
#pragma unroll
        for (int u = 0; u < FILL_U; ++u) {
            const int e = e0 + u * blockDim.x, j = e / (LP_D / 4), c = (e % (LP_D / 4)) * 4;
            buf[u] = (j < nk) ? __ldg(reinterpret_cast<const float4*>(tb + (long long)j * LP_D + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < FILL_U; ++u) {
            const int e = e0 + u * blockDim.x, j = e / (LP_D / 4), c = (e % (LP_D / 4)) * 4;
            if (j < nkp)
                *reinterpret_cast<uint4*>(st + j * ST + c) = make_uint4(to_tf32(buf[u].x), to_tf32(buf[u].y), to_tf32(buf[u].z), to_tf32(buf[u].w));
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int r0 = warp * 16 + g, r1 = r0 + 8;                        // rows of U^T: head 2*warp (i = g) and head 2*warp+1
    uint32_t a[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        a[ks][0] = to_tf32(__ldg(ut + r0 * LP_D + ks * 8 + t));
        a[ks][1] = to_tf32(__ldg(ut + r1 * LP_D + ks * 8 + t));
        a[ks][2] = to_tf32(__ldg(ut + r0 * LP_D + ks * 8 + t + 4));
        a[ks][3] = to_tf32(__ldg(ut + r1 * LP_D + ks * 8 + t + 4));
    }
    __syncthreads();
    float acc[KS][4];
#pragma unroll
    for (int nd = 0; nd < KS; ++nd) acc[nd][0] = acc[nd][1] = acc[nd][2] = acc[nd][3] = 0.f;
    float m0 = -CUDART_INF_F, m1 = -CUDART_INF_F, l0 = 0.f, l1 = 0.f;
    for (int kb = 0; kb < nkp; kb += 32) {
        float s[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            const uint32_t* kr = st + (kb + nt * 8 + g) * ST + t;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) mma_tf32(s[nt], a[ks], kr[ks * 8], kr[ks * 8 + 4]);
        }
        if (kb + 32 > nk) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int key = kb + nt * 8 + 2 * t;
                if (key >= nk) s[nt][0] = s[nt][2] = -CUDART_INF_F;
                if (key + 1 >= nk) s[nt][1] = s[nt][3] = -CUDART_INF_F;
            }
        }
        float x0 = s[0][0], x1 = s[0][2];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            x0 = fmaxf(x0, fmaxf(s[nt][0], s[nt][1]));
            x1 = fmaxf(x1, fmaxf(s[nt][2], s[nt][3]));
        }
        x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
        const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);
        const float c0 = __expf(m0 - n0), c1 = __expf(m1 - n1);
        m0 = n0; m1 = n1;
        l0 *= c0; l1 *= c1;
#pragma unroll
        for (int nd = 0; nd < KS; ++nd) { acc[nd][0] *= c0; acc[nd][1] *= c0; acc[nd][2] *= c1; acc[nd][3] *= c1; }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const float p00 = __expf(s[nt][0] - n0), p01 = __expf(s[nt][1] - n0);
            const float p10 = __expf(s[nt][2] - n1), p11 = __expf(s[nt][3] - n1);
            l0 += p00 + p01; l1 += p10 + p11;
            const uint32_t pa[4] = {to_tf32(p00), to_tf32(p10), to_tf32(p01), to_tf32(p11)};
            const uint32_t* vr = st + (kb + nt * 8 + 2 * t) * ST + g;
#pragma unroll
            for (int nd = 0; nd < KS; ++nd) mma_tf32(acc[nd], pa, vr[nd * 8], vr[ST + nd * 8]);
        }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    // pooled tokens z (16 rows x 128) sit in the accumulator layout (row g / g+8, channels 8 nd + 2t, +1). Output
    // projection out = Wv[h] z + bv[h]: rows g belong to head h0 = 2*warp, rows g+8 to h1 = h0 + 1, so two mma chains run
    // over the same A fragments (channel permutation trick: A col t <-> channel 2t, t+4 <-> 2t+1), one per head's weights.
    const int h0 = 2 * warp, h1 = h0 + 1;
    float o0[2][4], o1[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) { o0[nt][0] = o0[nt][1] = o0[nt][2] = o0[nt][3] = 0.f; o1[nt][0] = o1[nt][1] = o1[nt][2] = o1[nt][3] = 0.f; }
#pragma unroll
    for (int nd = 0; nd < KS; ++nd) {
        const uint32_t za[4] = {to_tf32(acc[nd][0] * i0), to_tf32(acc[nd][2] * i1), to_tf32(acc[nd][1] * i0), to_tf32(acc[nd][3] * i1)};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {                       // B[k = channel][n = d] = Wv[h*16 + nt*8 + g][8 nd + 2t (+1)]
            const float* w0 = wv + (long long)(h0 * LP_HD + nt * 8 + g) * LP_D + nd * 8 + 2 * t;
            const float* w1 = wv + (long long)(h1 * LP_HD + nt * 8 + g) * LP_D + nd * 8 + 2 * t;
            mma_tf32(o0[nt], za, to_tf32(__ldg(w0)), to_tf32(__ldg(w0 + 1)));
            mma_tf32(o1[nt], za, to_tf32(__ldg(w1)), to_tf32(__ldg(w1 + 1)));
        }
    }
    // o0: rows g (latent i = g) of head h0 in c0,c1; o1: rows g+8 (latent i = g) of head h1 in c2,c3
    float* ob = out + (b * 8 + g) * (LP_HEADS * LP_HD);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
        const int d = nt * 8 + 2 * t;
        *reinterpret_cast<float2*>(ob + h0 * LP_HD + d) = make_float2(o0[nt][0] + __ldg(bv + h0 * LP_HD + d), o0[nt][1] + __ldg(bv + h0 * LP_HD + d + 1));
        *reinterpret_cast<float2*>(ob + h1 * LP_HD + d) = make_float2(o1[nt][2] + __ldg(bv + h1 * LP_HD + d), o1[nt][3] + __ldg(bv + h1 * LP_HD + d + 1));
    }
}

// few queries per batch element (perceiver input layer: 8 latent queries x 8 heads vs 80 keys per cost map; latent
// self-attention 8 x 8; decoder cross-attention 1 x 8): ONE WARP per batch element, lane = slot * 8 + head, each lane
// owns queries slot and slot + 4. K/V rows stream straight from global memory: the 8 head segments of a key are one
// coalesced 512 B row, the 4 slots read identical addresses (one transaction) — the kernel is a pure HBM stream.
constexpr int FQ_HEADS = 8, FQ_SLOTS = 4, FQ_QPT = 2;
template <int FQ_D>
__global__ void __launch_bounds__(128)
attn_few_queries_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                        float* __restrict__ out, long long batch, int nq, int nk, long long q_bstride, float scale) {
    const long long b = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (b >= batch) return;
    const int lane = threadIdx.x & 31, hd = lane & 7, slot = lane >> 3;
    constexpr int C = FQ_HEADS * FQ_D;
    float2 qr[FQ_QPT][FQ_D / 2], acc[FQ_QPT][FQ_D / 2];
    float m[FQ_QPT], l[FQ_QPT];
#pragma unroll
    for (int t = 0; t < FQ_QPT; ++t) {
        const int i = min(slot + FQ_SLOTS * t, nq - 1);
        const float* qp = q + b * q_bstride + ((long long)i * FQ_HEADS + hd) * FQ_D;
#pragma unroll
        for (int c = 0; c < FQ_D / 4; ++c) {
            const float4 x = *reinterpret_cast<const float4*>(qp + 4 * c);
            qr[t][2 * c] = make_float2(x.x * scale, x.y * scale);
            qr[t][2 * c + 1] = make_float2(x.z * scale, x.w * scale);
        }
#pragma unroll
        for (int c = 0; c < FQ_D / 2; ++c) acc[t][c] = make_float2(0.f, 0.f);
        m[t] = -CUDART_INF_F; l[t] = 0.f;
    }
    const float4* kp = reinterpret_cast<const float4*>(k + b * nk * C + hd * FQ_D);
    const float4* vp = reinterpret_cast<const float4*>(v + b * nk * C + hd * FQ_D);
#pragma unroll 2
    for (int j = 0; j < nk; ++j) {
        float4 kk[FQ_D / 4], vv[FQ_D / 4];
#pragma unroll
        for (int c = 0; c < FQ_D / 4; ++c) { kk[c] = __ldg(kp + j * (C / 4) + c); vv[c] = __ldg(vp + j * (C / 4) + c); }
#pragma unroll
        for (int t = 0; t < FQ_QPT; ++t) {
            float2 sx = make_float2(0.f, 0.f);
#pragma unroll
            for (int c = 0; c < FQ_D / 4; ++c) {
                sx = ffma2_rn(qr[t][2 * c], make_float2(kk[c].x, kk[c].y), sx);
                sx = ffma2_rn(qr[t][2 * c + 1], make_float2(kk[c].z, kk[c].w), sx);
            }
            const float s = sx.x + sx.y;
            const float mn = fmaxf(m[t], s);
            const float corr = __expf(m[t] - mn), p = __expf(s - mn);
            m[t] = mn;
            l[t] = l[t] * corr + p;
            const float2 c2 = make_float2(corr, corr), p2 = make_float2(p, p);
#pragma unroll
            for (int c = 0; c < FQ_D / 4; ++c) {
                acc[t][2 * c] = ffma2_rn(p2, make_float2(vv[c].x, vv[c].y), fmul2_rn(acc[t][2 * c], c2));
                acc[t][2 * c + 1] = ffma2_rn(p2, make_float2(vv[c].z, vv[c].w), fmul2_rn(acc[t][2 * c + 1], c2));
            }
        }
    }
#pragma unroll
    for (int t = 0; t < FQ_QPT; ++t) {
        const int i = slot + FQ_SLOTS * t;
        if (i >= nq) continue;
        const float inv = 1.f / l[t];
        float* op = out + ((b * nq + i) * FQ_HEADS + hd) * FQ_D;
#pragma unroll
        for (int c = 0; c < FQ_D / 4; ++c)
            *reinterpret_cast<float4*>(op + 4 * c) = make_float4(acc[t][2 * c].x * inv, acc[t][2 * c].y * inv,
                                                                 acc[t][2 * c + 1].x * inv, acc[t][2 * c + 1].y * inv);
    }
}

// one query per batch element (decoder cross-attention: each pixel's query vs its 8 cost-memory tokens,
// decoder.py:56-76): one thread per (batch element, head); the 8 heads of a key row are one coalesced segment.
template <int D>
__global__ void __launch_bounds__(256)
attn_single_query_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                         float* __restrict__ out, long long batch, int nk, int heads, float scale) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= batch * heads) return;
    const long long b = e / heads;
    const int hd = (int)(e % heads), C = heads * D;
    float qr[D], acc[D];
#pragma unroll
    for (int c = 0; c < D; c += 4) {
        const float4 t = *reinterpret_cast<const float4*>(q + b * C + hd * D + c);
        qr[c] = t.x * scale; qr[c + 1] = t.y * scale; qr[c + 2] = t.z * scale; qr[c + 3] = t.w * scale;
        acc[c] = acc[c + 1] = acc[c + 2] = acc[c + 3] = 0.f;
    }
    float m = -CUDART_INF_F, l = 0.f;
    const float* kp = k + b * nk * C + hd * D;
    const float* vp = v + b * nk * C + hd * D;
#pragma unroll 4
    for (int j = 0; j < nk; ++j) {
        float kk[D], vv[D];
#pragma unroll
        for (int c = 0; c < D; c += 4) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(kp + (long long)j * C + c));
            const float4 u = __ldg(reinterpret_cast<const float4*>(vp + (long long)j * C + c));
            kk[c] = t.x; kk[c + 1] = t.y; kk[c + 2] = t.z; kk[c + 3] = t.w;
            vv[c] = u.x; vv[c + 1] = u.y; vv[c + 2] = u.z; vv[c + 3] = u.w;
        }
        float sc = 0.f;
#pragma unroll
        for (int c = 0; c < D; ++c) sc = fmaf(qr[c], kk[c], sc);
        const float mn = fmaxf(m, sc);
        const float corr = __expf(m - mn), p = __expf(sc - mn);
        m = mn;
        l = l * corr + p;
#pragma unroll
        for (int c = 0; c < D; ++c) acc[c] = fmaf(p, vv[c], acc[c] * corr);
    }
    const float inv = 1.f / l;
#pragma unroll
    for (int c = 0; c < D; c += 4)
        *reinterpret_cast<float4*>(out + b * C + hd * D + c) = make_float4(acc[c] * inv, acc[c + 1] * inv, acc[c + 2] * inv, acc[c + 3] * inv);
}

}  // namespace

extern "C" int macvo_layer_norm(const float* x, const float* weight, const float* bias, float* y, long long rows,
                                int channels, float eps, void* stream) {
    if (!x || !weight || !bias || !y || rows < 0) return MACVO_E_ARG;
    if (rows == 0) return MACVO_OK;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    cudaStream_t st = as_stream(stream);
    switch (channels) {
        case 64: layer_norm64_kernel<<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps); break;
        case 128: layer_norm_kernel<4><<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps); break;
        case 256: layer_norm_kernel<8><<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps); break;
        case 512: layer_norm_kernel<16><<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps); break;
        default: return MACVO_E_UNSUPPORTED;
    }
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

// sum_out = x + resid;  y = LayerNorm(sum_out)   (the residual-add that precedes every norm2 of the transformer blocks)
extern "C" int macvo_add_layer_norm(const float* x, const float* resid, const float* weight, const float* bias, float* sum_out,
                                    float* y, long long rows, int channels, float eps, void* stream) {
    if (!x || !resid || !weight || !bias || !sum_out || !y || rows < 0) return MACVO_E_ARG;
    if (rows == 0) return MACVO_OK;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    cudaStream_t st = as_stream(stream);
    switch (channels) {
        case 128: layer_norm_kernel<4><<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps, resid, sum_out); break;
        case 256: layer_norm_kernel<8><<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps, resid, sum_out); break;
        case 512: layer_norm_kernel<16><<<grid, 256, 0, st>>>(x, weight, bias, y, rows, eps, resid, sum_out); break;
        default: return MACVO_E_UNSUPPORTED;
    }
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_patch_embed_conv1(const float* maps, const float* weight, const float* bias, float* out,
                                       long long n_maps, int h, int w, int allow_tf32, void* stream) {
    if (!maps || !weight || !bias || !out || n_maps < 0 || h <= 0 || w <= 0) return MACVO_E_ARG;
    if (n_maps == 0) return MACVO_OK;
    const int hp8 = (h + 7) / 8 * 8, wp8 = (w + 7) / 8 * 8;
    const int ho = hp8 / 2, wo = wp8 / 2;
    const size_t smem = (size_t)(2 * ho + 4) * (2 * wo + 4) * sizeof(float);
    if (smem > 200 * 1024) return MACVO_E_UNSUPPORTED;
    cudaStream_t st = as_stream(stream);
    if ((allow_tf32 & 2) && !(allow_tf32 & 1)) return MACVO_E_UNSUPPORTED;      // space-to-depth output: tensor-core variant only
    if (allow_tf32 & 1) {
        MACVO_CUDA_TRY(cudaFuncSetAttribute(patch_conv1_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        patch_conv1_tc_kernel<<<(unsigned)n_maps, 256, smem, st>>>(maps, weight, bias, out, h, w, ho, wo, (allow_tf32 >> 1) & 1);
        MACVO_LAUNCH_CHECK();
        return MACVO_OK;
    }
    // weights -> constant bank (a 2.4 KB device-to-device copy node; stays valid under CUDA-graph replay)
    float* packed = nullptr;
    MACVO_CUDA_TRY(cudaGetSymbolAddress(reinterpret_cast<void**>(&packed), g_pe_pack));
    pe_pack_weights_kernel<<<3, 256, 0, st>>>(weight, bias, packed);
    MACVO_LAUNCH_CHECK();
    MACVO_CUDA_TRY(cudaMemcpyToSymbolAsync(c_pe_w, packed, sizeof(float) * (PE_K * PE_K * PE_C + PE_C), 0,
                                           cudaMemcpyDeviceToDevice, st));
    MACVO_CUDA_TRY(cudaFuncSetAttribute(patch_conv1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int items = ho * (wo / 2);
    patch_conv1_kernel<<<(unsigned)n_maps, items % 320 == 0 ? 320 : 256, smem, st>>>(maps, out, h, w, ho, wo);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_small_attention_ex(const float* q, const float* k, const float* v, float* out, int batch, int nq,
                                        int nk, int heads, int head_dim, int q_broadcast, int allow_tf32, int ldq, int ldk,
                                        int ldv, const float* q_add, const float* k_add, int add_period, void* stream) {
    if (!q || !k || !v || !out || batch <= 0 || nq <= 0 || nk <= 0 || heads <= 0) return MACVO_E_ARG;
    if (head_dim != 8 && head_dim != 16 && head_dim != 32) return MACVO_E_UNSUPPORTED;
    const int c = heads * head_dim;
    AttnExtra ex{ldq > 0 ? ldq : c, ldk > 0 ? ldk : c, ldv > 0 ? ldv : c, add_period > 0 ? add_period : 1, q_add, k_add};
    const bool plain = ex.ldq == c && ex.ldk == c && ex.ldv == c && !q_add && !k_add;
    if ((ex.ldq | ex.ldk | ex.ldv) & 3) return MACVO_E_ARG;
    cudaStream_t st = as_stream(stream);
    const float scale = 1.f / sqrtf((float)head_dim);
    const long long qbs = q_broadcast ? 0 : (long long)nq * ex.ldq;
    if (plain && nq == 1 && !q_broadcast && head_dim <= 16) {
        const unsigned grid = (unsigned)(((long long)batch * heads + 255) / 256);
        if (head_dim == 16) attn_single_query_kernel<16><<<grid, 256, 0, st>>>(q, k, v, out, batch, nk, heads, scale);
        else attn_single_query_kernel<8><<<grid, 256, 0, st>>>(q, k, v, out, batch, nk, heads, scale);
    } else if (plain && nq <= FQ_SLOTS * FQ_QPT && heads == FQ_HEADS && head_dim <= 16) {
        const unsigned grid = (unsigned)((batch + 3) / 4);
        if (head_dim == 16) attn_few_queries_kernel<16><<<grid, 128, 0, st>>>(q, k, v, out, batch, nq, nk, qbs, scale);
        else attn_few_queries_kernel<8><<<grid, 128, 0, st>>>(q, k, v, out, batch, nq, nk, qbs, scale);
    } else if (head_dim == 8) {
        return MACVO_E_UNSUPPORTED;
    } else if (allow_tf32 && nq >= 16) {
        const size_t smem = (size_t)((nk + 31) / 32 * 32) * ((head_dim / 32) * 32 + 16 + head_dim) * sizeof(float);
        if (smem > 200 * 1024) return MACVO_E_UNSUPPORTED;
        const int warps = nq > 64 ? 8 : 4;
        dim3 grid(ceil_div(nq, 16 * warps), heads, batch);
        if (head_dim == 16) {
            MACVO_CUDA_TRY(cudaFuncSetAttribute(attn_tc_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attn_tc_kernel<16><<<grid, 32 * warps, smem, st>>>(q, k, v, out, nq, nk, heads, qbs, scale, ex);
        } else {
            MACVO_CUDA_TRY(cudaFuncSetAttribute(attn_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attn_tc_kernel<32><<<grid, 32 * warps, smem, st>>>(q, k, v, out, nq, nk, heads, qbs, scale, ex);
        }
    } else {
        const size_t smem = (size_t)2 * ((nk + ATT_CHUNK - 1) / ATT_CHUNK * ATT_CHUNK) * head_dim * sizeof(float);
        if (smem > 200 * 1024) return MACVO_E_UNSUPPORTED;
        dim3 grid(ceil_div(nq, 128), heads, batch);
        if (head_dim == 16) {
            MACVO_CUDA_TRY(cudaFuncSetAttribute(attn_shared_kv_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attn_shared_kv_kernel<16><<<grid, 128, smem, st>>>(q, k, v, out, nq, nk, heads, qbs, scale, ex);
        } else {
            MACVO_CUDA_TRY(cudaFuncSetAttribute(attn_shared_kv_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attn_shared_kv_kernel<32><<<grid, 128, smem, st>>>(q, k, v, out, nq, nk, heads, qbs, scale, ex);
        }
    }
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_small_attention(const float* q, const float* k, const float* v, float* out, int batch, int nq,
                                     int nk, int heads, int head_dim, int q_broadcast, int allow_tf32, void* stream) {
    return macvo_small_attention_ex(q, k, v, out, batch, nq, nk, heads, head_dim, q_broadcast, allow_tf32, 0, 0, 0, nullptr,
                                    nullptr, 0, stream);
}

extern "C" int macvo_add_rows_relu(float* x, const float* term, long long rows, int period, int channels, void* stream) {
    if (!x || !term || rows < 0 || period <= 0 || channels <= 0 || (channels & 3)) return MACVO_E_ARG;
    if (rows == 0) return MACVO_OK;
    const long long n = rows * (channels / 4);
    add_rows_relu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(x, term, rows, period, channels / 4);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_latent_pool(const float* tokens, const float* ut, const float* wv, const float* bv, float* out,
                                 long long n_maps, int nk, void* stream) {
    if (!tokens || !ut || !wv || !bv || !out || n_maps < 0 || nk <= 0) return MACVO_E_ARG;
    if (n_maps == 0) return MACVO_OK;
    const size_t smem = (size_t)((nk + 31) / 32 * 32) * (LP_D + 4) * sizeof(float);
    if (smem > 200 * 1024) return MACVO_E_UNSUPPORTED;
    MACVO_CUDA_TRY(cudaFuncSetAttribute(latent_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    latent_pool_kernel<<<(unsigned)n_maps, 128, smem, as_stream(stream)>>>(tokens, ut, wv, bv, out, nk);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
