"""TEST INFRASTRUCTURE — CPU oracle for the frontend operators of MAC-VO's hot path.

Plain torch-CPU restatements (the reference itself is torch on CPU; using the same primitive
library keeps the oracle bit-faithful where the reference is) of:

* `corr_volume`     <- MemoryEncoder.corr              Module/Network/FlowFormer/core/encoder.py:256-275
* `window_lookup`   <- MemoryDecoder.encode_flow_token Module/Network/FlowFormer/core/decoder.py:141-153
                       + bilinear_sampler              Module/Network/FlowFormer/core/utils.py:26-34
                       + the `delta` buffer            Module/Network/FlowFormer/core/decoder.py:124-129
* `window_lookup_loops` — the same operator written with explicit per-tap arithmetic
                       (ATen's CPU grid_sampler, align_corners=True, zeros padding) for small cases
* `dense_postproc`  <- FlowFormerCovFrontend.inference_2_depth / inference_2_match
                                                       Module/Frontend/Frontend.py:184-200
                       disparity_to_depth[_cov]        Module/Frontend/StereoDepth.py:271-282
                       IMatcher.Output.from_partial_cov Module/Frontend/Matching.py:29-40
* `retrieve_pixels` <- IFrontend.retrieve_pixels       Module/Frontend/Frontend.py:104-118

PINNED by `tests/golden/*.pt` (generated from the reference itself by tests/golden/make_golden.py).
Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def corr_volume(fmap1: Tensor, fmap2: Tensor) -> Tensor:
    """C[b,0,i,j] = sum_d f1[b,d,i] f2[b,d,j]; (B,D,H,W) x2 -> (B,1,H,W,H,W). No 1/sqrt(d) scaling."""
    B, D, H, W = fmap1.shape
    a = fmap1.reshape(B, D, H * W).transpose(1, 2)          # (B, N, D) view, like the reference permute
    b = fmap2.reshape(B, D, H * W)
    return torch.bmm(a, b).view(B, 1, H, W, H, W)


def window_lookup(cost_maps: Tensor, coords: Tensor) -> Tensor:
    """cost_maps (B*H1*W1, 1, H2, W2), coords (B, 2, H1, W1) [x, y] -> (B, 81, H1, W1).

    Window index (i, j) samples at (x + (i-4), y + (j-4)): the reference builds `delta` as (dy, dx)
    but adds it to (x, y), so the FIRST window axis steps in x. Output channel = i*9 + j.
    """
    B, _, H1, W1 = coords.shape
    r = torch.linspace(-4, 4, 9, dtype=coords.dtype, device=coords.device)
    delta = torch.stack(torch.meshgrid(r, r, indexing="ij"), dim=-1).view(1, 9, 9, 2)
    c = coords.permute(0, 2, 3, 1).reshape(B * H1 * W1, 1, 1, 2) + delta
    H2, W2 = cost_maps.shape[-2:]
    gx = 2 * c[..., 0] / (W2 - 1) - 1
    gy = 2 * c[..., 1] / (H2 - 1) - 1
    out = F.grid_sample(cost_maps, torch.stack([gx, gy], dim=-1), align_corners=True)
    return out.view(B, H1, W1, 81).permute(0, 3, 1, 2)


def window_lookup_loops(cost_maps: Tensor, coords: Tensor) -> Tensor:
    """Same operator with the per-tap arithmetic spelled out (vectorised over queries).

    Follows ATen's CPU grid_sampler_2d (align_corners=True): ix = (gx + 1) * ((W-1)/2);
    taps nw/ne/sw/se weighted by (1-wx)(1-wy) ..., out-of-range taps contribute 0.
    """
    B, _, H1, W1 = coords.shape
    Q = B * H1 * W1
    H2, W2 = cost_maps.shape[-2:]
    maps = cost_maps.reshape(Q, H2 * W2)
    cx = coords[:, 0].reshape(Q)
    cy = coords[:, 1].reshape(Q)
    out = torch.zeros(Q, 81, dtype=cost_maps.dtype)
    for i in range(9):
        for j in range(9):
            gx = 2 * (cx + (i - 4)) / (W2 - 1) - 1
            gy = 2 * (cy + (j - 4)) / (H2 - 1) - 1
            ix = (gx + 1) * ((W2 - 1) / 2)
            iy = (gy + 1) * ((H2 - 1) / 2)
            x0, y0 = ix.floor(), iy.floor()
            wx, wy = ix - x0, iy - y0
            acc = torch.zeros(Q, dtype=cost_maps.dtype)
            for dy, dx, w in ((0, 0, (1 - wy) * (1 - wx)), (0, 1, (1 - wy) * wx),
                              (1, 0, wy * (1 - wx)), (1, 1, wy * wx)):
                xi, yi = (x0 + dx).long(), (y0 + dy).long()
                ok = (xi >= 0) & (xi < W2) & (yi >= 0) & (yi < H2)
                idx = (yi.clamp(0, H2 - 1) * W2 + xi.clamp(0, W2 - 1))
                val = maps.gather(1, idx.view(Q, 1)).view(Q)
                acc = acc + torch.where(ok, val * w, torch.zeros_like(val))
            out[:, i * 9 + j] = acc
    return out.view(B, H1, W1, 81).permute(0, 3, 1, 2).contiguous()


def dense_postproc(est_flow: Tensor, est_cov: Tensor, baseline: float, fx: float,
                   enforce_positive_disparity: bool = False) -> dict[str, Tensor | None]:
    """One `estimate_pair` worth of dense maps from the network output (Frontend.py:184-200, 291-299).

    est_flow / est_cov: (2, 2, H, W) fp32; slot 0 = stereo pair of frame t2, slot 1 = temporal pair.
    """
    f0, c0 = est_flow[0:1], est_cov[0:1]
    disparity, disparity_cov = f0[:, :1].abs(), c0[:, :1]
    depth = (baseline * fx) * disparity.reciprocal()
    d2 = disparity.square()
    err2 = disparity_cov * d2.reciprocal()
    depth_cov = ((baseline * fx) ** 2) * (err2 / d2)
    mask = (f0[:, :1] <= 0) if enforce_positive_disparity else None
    f1, c1 = est_flow[1:2], est_cov[1:2]
    B, C, H, W = c1.shape
    match_cov = torch.cat([c1, torch.zeros((B, 1, H, W)).to(c1)], dim=1)
    return {"depth": depth, "disparity": disparity, "depth_cov": depth_cov,
            "disparity_uncertainty": disparity_cov, "depth_mask": mask,
            "flow": f1, "flow_cov": match_cov}


def retrieve_pixels(pixel_uv: Tensor, scalar_map: Tensor | None) -> Tensor | None:
    """(K,2) [u,v] + (B,C,H,W) -> (C,K): values of batch 0 at (v.long(), u.long())."""
    if scalar_map is None:
        return None
    return scalar_map[0, ..., pixel_uv[..., 1].long(), pixel_uv[..., 0].long()]


def filter_points_in_range(pts: Tensor, u_range: tuple[int, int], v_range: tuple[int, int]) -> Tensor:
    """Strict-inequality in-bound test (Utility/Point.py:5-13)."""
    return ((pts[..., 0] < u_range[1]) & (pts[..., 0] > u_range[0])
            & (pts[..., 1] < v_range[1]) & (pts[..., 1] > v_range[0]))
