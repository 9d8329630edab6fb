"""Inputs and the CPU stand-in of the Vanilla ablation's covariance-free frontend (B200_FlowFormerFrontend) and of
`macvo_observe_pack` with NULL covariance maps.

`observe_pack_no_cov` restates Odometry/MACVO.py:198-283 for a frontend whose depth / match outputs carry no covariance
(FlowFormerDepth + FlowFormerMatcher): kp*_sigma_dd, kp1_sigma_disparity and kp1_sigma_uv are None, so MatchObs holds -1 in
pixel1/2_d_cov, pixel2_disp_cov and pixel2_uv_cov (:250-264), and `ObsCovModel.estimate(frame1, kp1, depth1, None, None)`
runs MatchCovariance with its own unclamped default flow covariance (Project2to3.py:128-135). It is built from the oracle
pieces the other fixtures pin (oracle.covariance.match_covariance, oracle.ablation), which take the None maps as the
reference does."""
from __future__ import annotations

import torch

from oracle import ablation as oab
from oracle import covariance as ocov
from oracle import frontend as ofe
from oracle.observe import _k_matrix, _window_leaves, se3_act_f32
from tests.golden import cases

PLAIN_CASES = {"small": (96, 128), "odd": (100, 130)}
FX, BASELINE = 320.0, 0.25


def plain_frontend_inputs(H: int, W: int):
    """(t1.L, t2.L, t2.R), each (1,3,H,W) in [0, 1]"""
    l2, r2 = cases.net_inputs(1, H, W, seed=2000)
    t1l, _ = cases.net_inputs(1, H, W, seed=2101)
    return t1l, l2, r2


def observe_pack_no_cov(kp0, flow, depth0, depth1, disparity1, edge_width: int, intr0, intr1, prev_pose,
                        kernel_size: int = 31, min_flow_cov: float = 0.25, min_depth_cov: float = 0.05,
                        match_cov_default: float = 0.25, cov_model: str = "match", depth_range=None, icp: bool = False) -> dict:
    """what macvo_observe_pack packs with match_cov = disp_unc1 = NULL (and depth_cov0 / depth_cov1 NULL)"""
    H, W = flow.shape[-2:]
    k = kp0.shape[0]
    u0, v0 = kp0[:, 0], kp0[:, 1]
    assert bool(((u0 >= 0) & (u0 < W) & (v0 >= 0) & (v0 < H)).all())
    kp1_a = kp0 + ofe.retrieve_pixels(kp0, flow).T
    inb = ofe.filter_points_in_range(kp1_a, (edge_width, W - edge_width), (edge_width, H - edge_width))
    rows = torch.nonzero(inb).reshape(-1)
    kp0_i, kp1_i = kp0[inb], kp1_a[inb]
    n = rows.numel()
    d0 = ofe.retrieve_pixels(kp0_i, depth0).squeeze(0)
    d1 = ofe.retrieve_pixels(kp1_i, depth1).squeeze(0)
    disp1 = ofe.retrieve_pixels(kp1_i, disparity1).T.reshape(-1)
    placeholder = torch.full((n,), -1.0)
    status = 0
    if cov_model == "identity":
        cov0, cov1 = oab.no_covariance(n), oab.no_covariance(n)
        ev = torch.ones(n, dtype=torch.bool)
        leaves = torch.zeros(n, dtype=torch.bool)
    else:
        kp0_sigma_uv = torch.ones((n, 3)) * match_cov_default
        kp0_sigma_uv[..., 2] = 0.0
        half = kernel_size // 2
        leaves = _window_leaves(kp0_i, H, W, half) | _window_leaves(kp1_i.long(), H, W, half)
        if bool(leaves.any()):
            status |= 1
        ev = ~leaves
        cov0 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
        cov1 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
        if bool(ev.any()):
            # kp0: the clamped default (a flow covariance is passed); kp1: flow_cov None -> the unclamped default
            cov0[ev] = ocov.match_covariance(kp0_i[ev], depth0, kp0_sigma_uv[ev], *intr0, kernel_size, min_flow_cov,
                                             min_depth_cov, match_cov_default)
            cov1[ev] = ocov.match_covariance(kp1_i[ev], depth1, None, *intr1, kernel_size, min_flow_cov,
                                             min_depth_cov, match_cov_default)
    bad = (~torch.isfinite(cov0)).any(dim=(-1, -2)) | (~torch.isfinite(cov1)).any(dim=(-1, -2))
    ok = ~bad & ev
    if depth_range is not None:
        lo, hi = depth_range
        ok &= ~((d0 < lo) | (d0 > hi) | (d1 < lo) | (d1 > hi))
    pos0_Tc = ocov.pixel2point_ned(kp0_i, d0, _k_matrix(intr0))
    keep = torch.zeros(k, dtype=torch.bool)
    keep[rows[ok]] = True
    out = {"pos_Tw": se3_act_f32(prev_pose, pos0_Tc)[ok], "pixel2_uv": kp1_i[ok], "pixel2_disp": disp1[ok],
           "pixel2_uv_cov": torch.full((int(ok.sum()), 3), -1.0), "pixel2_disp_cov": placeholder[ok],
           "obs1_covTc": cov0[ok], "obs2_covTc": cov1[ok], "pixel1_uv": kp0_i[ok], "pixel1_d": d0[ok],
           "n_obs": int(ok.sum()), "n_inbound": n, "k": k, "status": status, "keep": keep,
           "next_pose": prev_pose.double().float().double()}
    if icp:
        R = oab.ofil.quat_matrix_f32(prev_pose[3:7]).repeat((out["n_obs"], 1, 1)).to(torch.float64)
        out.update(pixel2_d=d1[ok], pixel1_d_cov=placeholder[ok], pixel2_d_cov=placeholder[ok],
                   points_Tc=ocov.pixel2point_ned(kp1_i[ok], d1[ok], _k_matrix(intr1)).double(),
                   cov_Tw=torch.bmm(torch.bmm(R, out["obs1_covTc"]), R.transpose(1, 2)))
    return out
