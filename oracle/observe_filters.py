"""TEST INFRASTRUCTURE — CPU oracle for the extended `macvo_observe_pack` (csrc/observe.cu with a `macvo_observe_ext_t`):
the rest of Paper_Reproduce.yaml's FilterCompose and the columns of its "icp" graph, on top of `oracle.observe.observe_pack`
(observation building, CovarianceSanityFilter, point registration), which it calls unchanged.

  SimpleDepthFilter / LikelyFrontOfCamFilter      Module/OutlierFilter.py:103-141 on the MatchObs columns pixel1_d,
                                                  pixel2_d (depth1 at the truncated kp1), pixel1_d_cov, pixel2_d_cov;
                                                  the -1 placeholder is looked for among ALL in-bound rows
  points_Tc                                       ICP_TwoframePGO (Graphs.py:49-51): pixel2point_NED(pixel2_uv, pixel2_d, K1)
  cov_Tw                                          MACVO.py:274-280: bmm(bmm(R, obs1_covTc), R^T), R = pypose matrix() of the
                                                  fp32 previous pose (computed in fp32), widened

PINNED by tests/golden/observe_icp_*.pt (tests/golden/make_golden_observe_icp.py, the reference functions themselves).
Only tests/ may import this module.
"""
from __future__ import annotations

import torch

from . import covariance as ocov
from . import frontend as ofe
from .observe import _k_matrix, observe_pack as observe_pack_sanity

Tensor = torch.Tensor
ROWS = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
        "pixel1_uv", "pixel1_d", "pos_Tc")


def quat_matrix_f32(q: Tensor) -> Tensor:
    """pypose SO3 `matrix()` of q = [x,y,z,w] in fp32"""
    x, y, z, w = q.float().unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], dim=-1),
        torch.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], dim=-1),
        torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], dim=-1),
    ], dim=-2)


def observe_pack(kp0: Tensor, flow: Tensor, match_cov: Tensor, depth0: Tensor, depth1: Tensor, disparity1: Tensor,
                 disp_unc1: Tensor, edge_width: int, intr0, intr1, prev_pose: Tensor, kernel_size: int = 31,
                 min_flow_cov: float = 0.25, min_depth_cov: float = 0.05, match_cov_default: float = 0.25,
                 depth_cov0: Tensor | None = None, depth_cov1: Tensor | None = None,
                 depth_range: tuple[float, float] | None = None, front_of_cam: bool = False, icp: bool = False) -> dict:
    """`oracle.observe.observe_pack`'s arguments and result, with the extension applied: depth_range = (min_depth,
    max_depth) runs SimpleDepthFilter, front_of_cam LikelyFrontOfCamFilter; depth_cov0 / depth_cov1 (1,1,H,W) or None (the
    -1 placeholder). icp adds the kept rows' pixel2_d, pixel1_d_cov, pixel2_d_cov (fp32), points_Tc (float64 of fp32)
    and cov_Tw (float64)."""
    out = observe_pack_sanity(kp0, flow, match_cov, depth0, depth1, disparity1, disp_unc1, edge_width, intr0, intr1,
                              prev_pose, kernel_size, min_flow_cov, min_depth_cov, match_cov_default)
    H, W = flow.shape[-2:]
    # the in-bound rows, as the base oracle finds them (kp0 inside the image, kp1 strictly inside the edge band)
    u0, v0 = kp0[:, 0], kp0[:, 1]
    idx0 = torch.nonzero((u0 >= 0) & (u0 < W) & (v0 >= 0) & (v0 < H)).reshape(-1)
    kp1_a = kp0[idx0] + ofe.retrieve_pixels(kp0[idx0], flow).T
    inb = ofe.filter_points_in_range(kp1_a, (edge_width, W - edge_width), (edge_width, H - edge_width))
    rows, kp0_i, kp1_i = idx0[inb], kp0[idx0][inb], kp1_a[inb]
    n = rows.numel()
    d0 = ofe.retrieve_pixels(kp0_i, depth0).squeeze(0)
    d1 = ofe.retrieve_pixels(kp1_i, depth1).squeeze(0)
    gather = lambda kp, m: torch.full((n,), -1.0) if m is None else ofe.retrieve_pixels(kp, m).squeeze(0)
    dc0, dc1 = gather(kp0_i, depth_cov0), gather(kp1_i, depth_cov1)
    ok = torch.ones(n, dtype=torch.bool)
    if depth_range is not None:
        lo, hi = depth_range
        ok &= ~((d0 < lo) | (d0 > hi) | (d1 < lo) | (d1 > hi))
    if front_of_cam and not bool((dc0 == -1).any()):
        ok &= ((d0 - (dc0.sqrt() * 2)) > 0.) & ((d1 - (dc1.sqrt() * 2)) > 0.)
    extra = torch.ones(kp0.shape[0], dtype=torch.bool)
    extra[rows] = ok
    keep = out["keep"] & extra
    kept_before = torch.nonzero(out["keep"]).reshape(-1)
    sel = extra[kept_before]                              # which of the sanity filter's survivors the chain keeps
    out = dict(out, keep=keep, n_obs=int(sel.sum()), **{k: out[k][sel] for k in ROWS})
    if icp:
        at = torch.zeros(kp0.shape[0], dtype=torch.long)
        at[rows] = torch.arange(n)
        i = at[keep]                                      # in-bound index of every kept row, in order
        R = quat_matrix_f32(prev_pose[3:7]).repeat((out["n_obs"], 1, 1)).to(torch.float64)
        out.update(pixel2_d=d1[i], pixel1_d_cov=dc0[i], pixel2_d_cov=dc1[i],
                   points_Tc=ocov.pixel2point_ned(kp1_i[i], d1[i], _k_matrix(intr1)).double(),
                   cov_Tw=torch.bmm(torch.bmm(R, out["obs1_covTc"]), R.transpose(1, 2)))
    return out
