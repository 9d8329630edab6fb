// (a7) dense post-processing of the network output fused with (a8) keypoint scoring, plus the
// candidate selection that follows (median threshold, masks, row-major ordered compaction).
//
// Replaces, bit-exactly (fp32 compares / int64 indices must equal the reference's):
//   FlowFormerCovFrontend.inference_2_depth / inference_2_match   Module/Frontend/Frontend.py:184-200
//   disparity_to_depth / disparity_to_depth_cov                    Module/Frontend/StereoDepth.py:271-282
//   IMatcher.Output.from_partial_cov                               Module/Frontend/Matching.py:29-40
//   CovAwareSelector_NoDepth.select_point                          Module/KeypointSelector.py:362-407
//   MappingPointSelector.select_point                              Module/KeypointSelector.py:87-100
//
// All arithmetic uses explicit round-to-nearest intrinsics in the reference's operation order (no FMA
// contraction), so every fp32 map equals the reference's eager CPU result bit for bit.
// HBM streaming: ~25 MB per 640x480 frame (SURVEY.md §8d) in ONE coalesced pass.
#include "common.cuh"
#include <math_constants.h>

namespace {

constexpr int TX = 32, TY = 8, MAXR = 7;   // tile, max NMS radius (ksize <= 15)

__global__ void __launch_bounds__(TX * TY)
dense_score_kernel(const float* __restrict__ est_flow, const float* __restrict__ est_cov, int h, int w, float bl_fx,
                   float bl_fx_sq, float* __restrict__ depth, float* __restrict__ disparity,
                   float* __restrict__ depth_cov, uint8_t* __restrict__ depth_mask, float* __restrict__ flow_cov,
                   const float* __restrict__ score_cov, float* __restrict__ quality, uint8_t* __restrict__ nms,
                   float* __restrict__ cand_vals, int* __restrict__ n_cand, int radius,
                   const float* __restrict__ dcov0, const float* __restrict__ dcov1, float* __restrict__ flow_quality,
                   float* __restrict__ cand_vals2) {
    __shared__ float tile[TY + 2 * MAXR][TX + 2 * MAXR + 1];
    const int hw = h * w;
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    const bool inside = x < w && y < h;
    const int p = y * w + x;

    // ---- (a7) slot 0: disparity -> depth, depth covariance ------------------------------------
    // (est_cov == nullptr: a frontend without covariance, FlowFormerDepth.estimate, StereoDepth.py:122-128 -- depth and
    // disparity only)
    if (inside && est_flow != nullptr) {
        const float fxv = est_flow[p];                       // est_flow[0, 0]
        const float disp = fabsf(fxv);
        if (disparity) disparity[p] = disp;
        if (depth) depth[p] = __fmul_rn(bl_fx, __frcp_rn(disp));
        if (depth_cov) {
            const float dcv = est_cov[p];                    // est_cov[0, 0]  (disparity variance)
            const float d2 = __fmul_rn(disp, disp);
            const float err2 = __fmul_rn(dcv, __frcp_rn(d2));
            depth_cov[p] = __fmul_rn(bl_fx_sq, __fdiv_rn(err2, d2));
        }
        if (depth_mask) depth_mask[p] = fxv <= 0.f ? 1 : 0;
    }
    // ---- slot 1: match covariance, padded to 3 channels with zeros -----------------------------
    float cuu = 0.f, cvv = 0.f, cuv = 0.f;
    if (inside && (score_cov || est_cov)) {
        if (score_cov) {
            cuu = score_cov[p]; cvv = score_cov[hw + p]; cuv = score_cov[2 * hw + p];
        } else {
            cuu = est_cov[2 * hw + p]; cvv = est_cov[3 * hw + p];       // est_cov[1, 0], est_cov[1, 1]
        }
        if (flow_cov) { flow_cov[p] = cuu; flow_cov[hw + p] = cvv; flow_cov[2 * hw + p] = 0.f; }
    }
    if (quality == nullptr) return;

    // ---- (a8) quality = uu + vv - 2 uv, NMS = (q == window min) & no NaN in the window ----------
    // Halo cells recompute q from global memory; outside the image they hold +inf (max_pool2d pads -inf on -q).
    auto q_at = [&](int yy, int xx) -> float {
        if (xx < 0 || xx >= w || yy < 0 || yy >= h) return CUDART_INF_F;
        const int pp = yy * w + xx;
        float a, b2, c;
        if (score_cov) { a = score_cov[pp]; b2 = score_cov[hw + pp]; c = score_cov[2 * hw + pp]; }
        else { a = est_cov[2 * hw + pp]; b2 = est_cov[3 * hw + pp]; c = 0.f; }
        const float fq = __fsub_rn(__fadd_rn(a, b2), __fmul_rn(2.f, c));
        // depth-aware selector: quality = (depth_cov0 + depth_cov1) * flow quality (KeypointSelector.py:276-279)
        return dcov0 ? __fmul_rn(__fadd_rn(dcov0[pp], dcov1[pp]), fq) : fq;
    };
    const int tw = TX + 2 * radius, th = TY + 2 * radius;
    for (int e = threadIdx.y * TX + threadIdx.x; e < tw * th; e += TX * TY) {
        const int ry = e / tw, rx = e - ry * tw;
        tile[ry][rx] = q_at(y0 + ry - radius, x0 + rx - radius);
    }
    __syncthreads();
    if (!inside) return;
    const float q = tile[threadIdx.y + radius][threadIdx.x + radius];
    float m = CUDART_INF_F;
    bool has_nan = false;
    for (int dy = 0; dy <= 2 * radius; ++dy)
        for (int dx = 0; dx <= 2 * radius; ++dx) {
            const float v = tile[threadIdx.y + dy][threadIdx.x + dx];
            has_nan |= (v != v);
            m = fminf(m, v);                                   // fminf ignores NaN; tracked separately
        }
    const bool is_nms = !has_nan && (q == m);
    quality[p] = q;
    nms[p] = is_nms ? 1 : 0;
    float fq_here = q, dc0_here = 0.f;
    if (dcov0) {
        fq_here = __fsub_rn(__fadd_rn(cuu, cvv), __fmul_rn(2.f, cuv));
        dc0_here = dcov0[p];
        flow_quality[p] = fq_here;
    }
    if (is_nms) {   // warp-aggregated append (order irrelevant: only the median of the set is used)
        const unsigned mask = __activemask();
        const int lane = (threadIdx.y * TX + threadIdx.x) & 31;
        const int leader = __ffs(mask) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(n_cand, __popc(mask));
        base = __shfl_sync(mask, base, leader);
        const int slot = base + __popc(mask & ((1u << lane) - 1));
        cand_vals[slot] = fq_here;
        if (dcov0) cand_vals2[slot] = dc0_here;
    }
}

// order-preserving key for fp32 compare via unsigned ints
__device__ __forceinline__ unsigned f2key(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Lower median (torch.median: sorted[(n-1)/2]) of cand_vals[0..n) by 4x8-bit radix select; one CTA.
__global__ void __launch_bounds__(1024)
median_threshold_kernel(const float* __restrict__ vals, const int* __restrict__ n_ptr, double max_match_cov,
                        float* __restrict__ thresh_out, int* __restrict__ status) {
    __shared__ unsigned hist[256];
    __shared__ unsigned s_prefix, s_k;
    const int n = *n_ptr;
    if (n <= 0) {   // torch.median([]) = nan; python min(max, nan * 1.5) keeps max
        if (threadIdx.x == 0) { *status = 1; *thresh_out = (float)max_match_cov; }
        return;
    }
    if (threadIdx.x == 0) { s_prefix = 0; s_k = (unsigned)((n - 1) / 2); *status = 0; }
    __syncthreads();
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        if (threadIdx.x < 256) hist[threadIdx.x] = 0;
        __syncthreads();
        const unsigned prefix = s_prefix;
        const unsigned himask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned key = f2key(vals[i]);
            if ((key & himask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned k = s_k, cum = 0;
            int d = 0;
            for (; d < 256; ++d) {
                if (cum + hist[d] > k) break;
                cum += hist[d];
            }
            s_k = k - cum;
            s_prefix = prefix | ((unsigned)d << shift);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float med = key2f(s_prefix);
        // python: min(max_match_cov, median.item() * 1.5) in double, then compared as an fp32 scalar
        const double t = fmin(max_match_cov, (double)med * 1.5);
        *thresh_out = (float)t;
    }
}

constexpr int CHUNK = 1024;   // pixels per compaction block

// MODE 0: cov-aware (nms & border & q < thr & extra)   1: mapping (depth & depth_cov & border)
// MODE 2: depth-aware cov selector: a = flow quality, b2 = depth_cov0, c/d = depth0/depth1 (< lim_a), thr[0] = depth-cov
//         threshold, thr[1] = flow threshold, extra / extra2 = optional validity masks
template <int MODE>
__global__ void __launch_bounds__(256)
flag_count_kernel(const float* __restrict__ a, const float* __restrict__ b2, const uint8_t* __restrict__ nms,
                  const uint8_t* __restrict__ extra, const float* __restrict__ thr_ptr, float lim_a, float lim_b,
                  int h, int w, int mask_width, uint8_t* __restrict__ flags, int* __restrict__ block_counts,
                  const float* __restrict__ c = nullptr, const float* __restrict__ d = nullptr,
                  const uint8_t* __restrict__ extra2 = nullptr) {
    __shared__ int s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const int hw = h * w;
    const float thr = MODE == 0 ? *thr_ptr : (MODE == 2 ? thr_ptr[1] : 0.f);
    const float thr_dc = MODE == 2 ? thr_ptr[0] : 0.f;
    int local = 0;
    for (int e = threadIdx.x; e < CHUNK; e += 256) {
        const int p = blockIdx.x * CHUNK + e;
        if (p >= hw) break;
        const int y = p / w, x = p - y * w;
        // reference border slice [mw:-mw]: with mw == 0 the slice is empty (nothing selectable)
        const bool border = mask_width > 0 && x >= mask_width && x < w - mask_width && y >= mask_width && y < h - mask_width;
        bool f;
        if (MODE == 0) f = border && nms[p] && (a[p] < thr) && (extra == nullptr || extra[p]);
        else if (MODE == 1) f = border && (a[p] < lim_a) && (b2[p] < lim_b);
        else f = border && nms[p] && (c[p] < lim_a) && (d[p] < lim_a) && (b2[p] < thr_dc) && (a[p] < thr) &&
                 (extra == nullptr || extra[p]) && (extra2 == nullptr || extra2[p]);
        flags[p] = f ? 1 : 0;
        local += f ? 1 : 0;
    }
    local = warp_sum(local);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(&s_cnt, local);
    __syncthreads();
    if (threadIdx.x == 0) block_counts[blockIdx.x] = s_cnt;
}

// ordered write: block offset = sum of earlier block counts (<= a few hundred blocks), then an in-block
// ordered scan in row-major pixel order.
__global__ void __launch_bounds__(256)
ordered_write_kernel(const uint8_t* __restrict__ flags, const int* __restrict__ block_counts, int nblocks, int hw,
                     int* __restrict__ cand_idx, int* __restrict__ n_out) {
    __shared__ int s_red[8];
    __shared__ int s_base, s_warp_off[8];
    int part = 0;
    for (int i = threadIdx.x; i < nblocks; i += 256) {
        if (i < (int)blockIdx.x) part += block_counts[i];
    }
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int i = 0; i < 8; ++i) s += s_red[i];
        s_base = s;
        if (blockIdx.x == nblocks - 1) *n_out = s + block_counts[blockIdx.x];
    }
    __syncthreads();
    int base = s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = 0; r < CHUNK / 256; ++r) {
        const int p = blockIdx.x * CHUNK + r * 256 + threadIdx.x;
        const bool f = p < hw && flags[p];
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_warp_off[warp] = __popc(bal);
        __syncthreads();
        int off = 0, tot = 0;
        for (int i = 0; i < 8; ++i) {
            if (i < warp) off += s_warp_off[i];
            tot += s_warp_off[i];
        }
        if (f) cand_idx[base + off + __popc(bal & ((1u << lane) - 1))] = p;
        base += tot;
        __syncthreads();
    }
}

__global__ void gather_pixels_kernel(const int* __restrict__ cand_idx, const int64_t* __restrict__ perm, int k, int w,
                                     int64_t* __restrict__ uv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const int p = cand_idx[perm[i]];
    uv[2 * i] = p % w;
    uv[2 * i + 1] = p / w;
}

template <typename KP>
__global__ void retrieve_pixels_kernel(const KP* __restrict__ kp, int k, const float* __restrict__ map, int channels,
                                       int h, int w, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    long long u = (long long)kp[2 * i], v = (long long)kp[2 * i + 1];   // .long(): truncation toward zero
    if (u < 0) u += w;                                                   // python-style negative index
    if (v < 0) v += h;
    const bool ok = u >= 0 && u < w && v >= 0 && v < h;
    for (int c = 0; c < channels; ++c)
        out[(long long)c * k + i] = ok ? map[((long long)c * h + v) * w + u] : CUDART_NAN_F;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

extern "C" int macvo_dense_postproc(const float* est_flow, const float* est_cov, int h, int w, double bl_fx,
                                    double bl_fx_sq, float* depth, float* disparity, float* depth_cov,
                                    uint8_t* depth_mask, float* flow_cov, const macvo_score_t* score, void* stream) {
    if (h <= 0 || w <= 0) return MACVO_E_ARG;
    if (!est_cov && est_flow) {
        // no covariance maps: depth / disparity of slot 0 only (FlowFormerDepth.estimate)
        if (depth_cov || depth_mask || flow_cov || score || !(depth || disparity)) return MACVO_E_ARG;
    } else if (!est_cov && !(score && score->score_cov)) {
        return MACVO_E_ARG;
    }
    if ((depth || disparity || depth_cov || depth_mask) && !est_flow) return MACVO_E_ARG;
    int radius = 0;
    const float* score_cov = nullptr;
    float* quality = nullptr; uint8_t* nms = nullptr; float* cand = nullptr; int* ncand = nullptr;
    const float *dc0 = nullptr, *dc1 = nullptr; float *fq = nullptr, *cand2 = nullptr;
    if (score) {
        if (!score->quality || !score->nms || !score->cand_vals || !score->n_cand) return MACVO_E_ARG;
        if (score->ksize < 1 || (score->ksize & 1) == 0 || score->ksize > 2 * MAXR + 1) return MACVO_E_ARG;
        radius = score->ksize / 2;
        score_cov = score->score_cov; quality = score->quality; nms = score->nms;
        cand = score->cand_vals; ncand = score->n_cand;
        if (score->depth_cov0 || score->depth_cov1) {
            if (!score->depth_cov0 || !score->depth_cov1 || !score->flow_quality || !score->cand_vals2) return MACVO_E_ARG;
            dc0 = score->depth_cov0; dc1 = score->depth_cov1; fq = score->flow_quality; cand2 = score->cand_vals2;
        }
    }
    dim3 grid(ceil_div(w, TX), ceil_div(h, TY)), block(TX, TY);
    dense_score_kernel<<<grid, block, 0, as_stream(stream)>>>(
        (depth || disparity || depth_cov || depth_mask) ? est_flow : nullptr, est_cov, h, w, (float)bl_fx,
        (float)bl_fx_sq, depth, disparity, depth_cov, depth_mask, flow_cov, score_cov, quality, nms, cand, ncand, radius,
        dc0, dc1, fq, cand2);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" size_t macvo_select_workspace_bytes(int h, int w) {
    const size_t hw = (size_t)h * w;
    return align_up(hw, 256) + align_up((hw / CHUNK + 2) * sizeof(int), 256);
}

static int run_compaction(const uint8_t* flags, int* block_counts, int nblocks, int hw, int* cand_idx, int* n_out,
                          cudaStream_t st) {
    ordered_write_kernel<<<nblocks, 256, 0, st>>>(flags, block_counts, nblocks, hw, cand_idx, n_out);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_select_candidates(const float* quality, const uint8_t* nms, const float* cand_vals,
                                       const int* n_cand, const uint8_t* extra_mask, int h, int w, int mask_width,
                                       double max_match_cov, int* cand_idx, int* n_out, float* thresh_out, int* status,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    if (!quality || !nms || !cand_vals || !n_cand || !cand_idx || !n_out || !thresh_out || !status || !workspace ||
        h <= 0 || w <= 0 || mask_width < 0)
        return MACVO_E_ARG;
    if (workspace_bytes < macvo_select_workspace_bytes(h, w)) return MACVO_E_WORKSPACE;
    cudaStream_t st = as_stream(stream);
    const int hw = h * w, nblocks = ceil_div(hw, CHUNK);
    uint8_t* flags = static_cast<uint8_t*>(workspace);
    int* block_counts = reinterpret_cast<int*>(static_cast<char*>(workspace) + align_up((size_t)hw, 256));
    median_threshold_kernel<<<1, 1024, 0, st>>>(cand_vals, n_cand, max_match_cov, thresh_out, status);
    MACVO_LAUNCH_CHECK();
    flag_count_kernel<0><<<nblocks, 256, 0, st>>>(quality, nullptr, nms, extra_mask, thresh_out, 0.f, 0.f, h, w,
                                                  mask_width, flags, block_counts);
    MACVO_LAUNCH_CHECK();
    return run_compaction(flags, block_counts, nblocks, hw, cand_idx, n_out, st);
}

extern "C" int macvo_select_candidates_depth(const float* flow_quality, const float* depth0, const float* depth1,
                                             const float* depth_cov0, const uint8_t* nms, const float* cand_fq,
                                             const float* cand_dc0, const int* n_cand, const uint8_t* mask_a,
                                             const uint8_t* mask_b, int h, int w, int mask_width, double max_depth,
                                             double max_depth_cov, double max_match_cov, int* cand_idx, int* n_out,
                                             float* thresh_out, int* status, void* workspace, size_t workspace_bytes,
                                             void* stream) {
    if (!flow_quality || !depth0 || !depth1 || !depth_cov0 || !nms || !cand_fq || !cand_dc0 || !n_cand || !cand_idx ||
        !n_out || !thresh_out || !status || !workspace || h <= 0 || w <= 0 || mask_width < 0)
        return MACVO_E_ARG;
    if (workspace_bytes < macvo_select_workspace_bytes(h, w)) return MACVO_E_WORKSPACE;
    cudaStream_t st = as_stream(stream);
    const int hw = h * w, nblocks = ceil_div(hw, CHUNK);
    uint8_t* flags = static_cast<uint8_t*>(workspace);
    int* block_counts = reinterpret_cast<int*>(static_cast<char*>(workspace) + align_up((size_t)hw, 256));
    median_threshold_kernel<<<1, 1024, 0, st>>>(cand_dc0, n_cand, max_depth_cov, thresh_out, status);
    MACVO_LAUNCH_CHECK();
    median_threshold_kernel<<<1, 1024, 0, st>>>(cand_fq, n_cand, max_match_cov, thresh_out + 1, status);
    MACVO_LAUNCH_CHECK();
    flag_count_kernel<2><<<nblocks, 256, 0, st>>>(flow_quality, depth_cov0, nms, mask_a, thresh_out, (float)max_depth, 0.f,
                                                  h, w, mask_width, flags, block_counts, depth0, depth1, mask_b);
    MACVO_LAUNCH_CHECK();
    return run_compaction(flags, block_counts, nblocks, hw, cand_idx, n_out, st);
}

extern "C" int macvo_select_mapping_candidates(const float* depth, const float* depth_cov, int h, int w, int mask_width,
                                               float max_depth, float max_depth_cov, int* cand_idx, int* n_out,
                                               void* workspace, size_t workspace_bytes, void* stream) {
    if (!depth || !depth_cov || !cand_idx || !n_out || !workspace || h <= 0 || w <= 0 || mask_width < 0)
        return MACVO_E_ARG;
    if (workspace_bytes < macvo_select_workspace_bytes(h, w)) return MACVO_E_WORKSPACE;
    cudaStream_t st = as_stream(stream);
    const int hw = h * w, nblocks = ceil_div(hw, CHUNK);
    uint8_t* flags = static_cast<uint8_t*>(workspace);
    int* block_counts = reinterpret_cast<int*>(static_cast<char*>(workspace) + align_up((size_t)hw, 256));
    flag_count_kernel<1><<<nblocks, 256, 0, st>>>(depth, depth_cov, nullptr, nullptr, nullptr, max_depth,
                                                  max_depth_cov, h, w, mask_width, flags, block_counts);
    MACVO_LAUNCH_CHECK();
    return run_compaction(flags, block_counts, nblocks, hw, cand_idx, n_out, st);
}

extern "C" int macvo_gather_pixels(const int* cand_idx, const int64_t* perm, int k, int w, int64_t* pixels_uv,
                                   void* stream) {
    if (k < 0 || w <= 0) return MACVO_E_ARG;
    if (k == 0) return MACVO_OK;
    if (!cand_idx || !perm || !pixels_uv) return MACVO_E_ARG;
    gather_pixels_kernel<<<ceil_div(k, 256), 256, 0, as_stream(stream)>>>(cand_idx, perm, k, w, pixels_uv);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}

extern "C" int macvo_retrieve_pixels(const void* kp, int kp_is_int64, int k, const float* map, int channels, int h,
                                     int w, float* out, void* stream) {
    if (k < 0 || channels <= 0 || h <= 0 || w <= 0) return MACVO_E_ARG;
    if (k == 0) return MACVO_OK;
    if (!kp || !map || !out) return MACVO_E_ARG;
    if (kp_is_int64)
        retrieve_pixels_kernel<int64_t><<<ceil_div(k, 256), 256, 0, as_stream(stream)>>>(
            static_cast<const int64_t*>(kp), k, map, channels, h, w, out);
    else
        retrieve_pixels_kernel<float><<<ceil_div(k, 256), 256, 0, as_stream(stream)>>>(
            static_cast<const float*>(kp), k, map, channels, h, w, out);
    MACVO_LAUNCH_CHECK();
    return MACVO_OK;
}
