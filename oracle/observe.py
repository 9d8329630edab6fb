"""TEST INFRASTRUCTURE — CPU oracle for `macvo_observe_pack` (csrc/observe.cu): observation building, the covariance
sanity filter and the point registration of the two-frame pose graph.

Restates Odometry/MACVO.py:198-283 (one frame pair, no map bookkeeping) from the oracle pieces already pinned:
  kp1 = kp0 + flow[kp0], filterPointsInRange     oracle.frontend.retrieve_pixels / filter_points_in_range
  ObsCovModel.estimate x2                         oracle.covariance.match_covariance (clamps kp1's flow covariance in
                                                  place: that clamped copy is MatchObs' pixel2_uv_cov)
  pixel2point_NED                                 oracle.covariance.pixel2point_ned
  CovarianceSanityFilter.filter                   Module/OutlierFilter.py:91-100
  pp.SE3_type.Act(prev_pose, pos0_Tc)             fp32, in the operation order csrc/observe.cu documents

Where the reference produces no result, the behaviour is defined here (DESIGN.md §2):
  * a non-finite 2x2 flow covariance (after the clamp): the reference's CPU `pinverse` raises; the row is dropped and
    `match_covariance` is not called on it;
  * a covariance window crossing the top / left edge wraps like python indices, in the reference and on the device;
  * a window crossing the bottom / right edge: the reference raises IndexError; status bit 0 (1) is set and the row's
    covariances and keep flag are unspecified (`unspecified` mask);
  * kp0 outside the image: status bit 1 (2); the row is dropped and not counted in n_inbound.

PINNED by tests/golden/observe_*.pt (generated from the reference functions by tests/golden/make_golden_observe.py).
Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module.
"""
from __future__ import annotations

import torch

from . import covariance as ocov
from . import frontend as ofe

Tensor = torch.Tensor


def se3_act_f32(pose: Tensor, p: Tensor) -> Tensor:
    """SE3.Act in fp32: p + w (2 q_v x p) + q_v x (2 q_v x p) + t, each operation rounded once, in the kernel's order"""
    t, q = pose[:3].float(), pose[3:7].float()
    qx, qy, qz, qw = q.unbind(0)
    px, py, pz = p.float().unbind(-1)
    ax = 2.0 * (qy * pz - qz * py)
    ay = 2.0 * (qz * px - qx * pz)
    az = 2.0 * (qx * py - qy * px)
    bx = qy * az - qz * ay
    by = qz * ax - qx * az
    bz = qx * ay - qy * ax
    return torch.stack([((px + qw * ax) + bx) + t[0], ((py + qw * ay) + by) + t[1], ((pz + qw * az) + bz) + t[2]], -1)


def _window_leaves(kp_long: Tensor, H: int, W: int, half: int) -> Tensor:
    """the window kp +- half reaches past the bottom / right edge (or wraps past the top / left one twice)"""
    u, v = kp_long[:, 0], kp_long[:, 1]
    return (u + half >= W) | (v + half >= H) | (u - half < -W) | (v - half < -H)


def _k_matrix(intr) -> Tensor:
    fx, fy, cx, cy = intr
    return torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32)


def observe_pack(kp0: Tensor, flow: Tensor, match_cov: Tensor, depth0: Tensor, depth1: Tensor, disparity1: Tensor,
                 disp_unc1: Tensor, edge_width: int, intr0, intr1, prev_pose: Tensor, kernel_size: int = 31,
                 min_flow_cov: float = 0.25, min_depth_cov: float = 0.05, match_cov_default: float = 0.25) -> dict:
    """kp0 (k,2) int64; flow (1,2,H,W); match_cov (1,3,H,W); the other maps (1,1,H,W) fp32; intr (fx, fy, cx, cy);
    prev_pose (7,) [t, q_xyzw]. Returns what the packed buffer holds: the kept rows in their original order
    (pos_Tw .. pixel1_d), n_obs, n_inbound, k, status, next_pose; plus `keep` (k,) bool, `unspecified` (k,) bool
    (rows whose window left the image), `pos_Tc` (n_obs,3) fp32 camera-frame points of the kept rows."""
    H, W = flow.shape[-2:]
    k = kp0.shape[0]
    status = 0
    u0, v0 = kp0[:, 0], kp0[:, 1]
    in0 = (u0 >= 0) & (u0 < W) & (v0 >= 0) & (v0 < H)
    if not bool(in0.all()):
        status |= 2
    idx0 = torch.nonzero(in0).reshape(-1)
    kp0_a = kp0[idx0]
    kp1_a = kp0_a + ofe.retrieve_pixels(kp0_a, flow).T                                   # int64 + fp32 -> fp32
    inb = ofe.filter_points_in_range(kp1_a, (edge_width, W - edge_width), (edge_width, H - edge_width))
    rows = idx0[inb]
    kp0_i, kp1_i = kp0_a[inb], kp1_a[inb]
    n = rows.numel()

    d0 = ofe.retrieve_pixels(kp0_i, depth0).squeeze(0)
    disp1 = ofe.retrieve_pixels(kp1_i, disparity1)
    dunc1 = ofe.retrieve_pixels(kp1_i, disp_unc1)
    kp0_sigma_uv = torch.ones((n, 3)) * match_cov_default
    kp0_sigma_uv[..., 2] = 0.0
    kp1_sigma_uv = ofe.retrieve_pixels(kp0_i, match_cov).T
    kp1_sigma_uv[..., :2].clamp_(min=min_flow_cov ** 2)          # what ObsCovModel.estimate does in place (idempotent)

    half = kernel_size // 2
    leaves = _window_leaves(kp0_i, H, W, half) | _window_leaves(kp1_i.long(), H, W, half)
    if bool(leaves.any()):
        status |= 1
    finite2 = torch.isfinite(kp1_sigma_uv).all(-1)
    ev = finite2 & ~leaves
    cov0 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
    cov1 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
    if bool(ev.any()):
        cov0[ev] = ocov.match_covariance(kp0_i[ev], depth0, kp0_sigma_uv[ev], *intr0, kernel_size, min_flow_cov,
                                         min_depth_cov, match_cov_default)
        cov1[ev] = ocov.match_covariance(kp1_i[ev], depth1, kp1_sigma_uv[ev], *intr1, kernel_size, min_flow_cov,
                                         min_depth_cov, match_cov_default)
    bad = (cov0.isnan().any(dim=(-1, -2)) | cov0.isinf().any(dim=(-1, -2))
           | cov1.isnan().any(dim=(-1, -2)) | cov1.isinf().any(dim=(-1, -2)))
    keep_i = ~bad & ev

    pos0_Tc = ocov.pixel2point_ned(kp0_i, d0, _k_matrix(intr0))
    pos_Tw = se3_act_f32(prev_pose, pos0_Tc)
    keep = torch.zeros(k, dtype=torch.bool)
    keep[rows[keep_i]] = True
    unspecified = torch.zeros(k, dtype=torch.bool)
    unspecified[rows[leaves]] = True
    return {
        "pos_Tw": pos_Tw[keep_i], "pixel2_uv": kp1_i[keep_i], "pixel2_disp": disp1.T[keep_i].reshape(-1),
        "pixel2_uv_cov": kp1_sigma_uv[keep_i], "pixel2_disp_cov": dunc1.T[keep_i].reshape(-1),
        "obs1_covTc": cov0[keep_i], "obs2_covTc": cov1[keep_i], "pixel1_uv": kp0_i[keep_i], "pixel1_d": d0[keep_i],
        "n_obs": int(keep_i.sum()), "n_inbound": n, "k": k, "status": status,
        "next_pose": prev_pose.double().float().double(),
        "keep": keep, "unspecified": unspecified, "pos_Tc": pos0_Tc[keep_i],
    }
