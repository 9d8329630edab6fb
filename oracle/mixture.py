"""TEST INFRASTRUCTURE — CPU oracle for MAC-VO's GaussianMixtureCovariance (csrc/cov2to3.cu `match_cov_kernel` given a
depth-variance map, and `macvo_observe_pack` with cov_model MACVO_COV_GAUSSIAN_MIXTURE).

  gaussian_mixture_covariance  <- GaussianMixtureCovariance.estimate   Module/Covariance/Project2to3.py:194-272
                                  gaussian_mixture_mean_var             Utility/Math.py:66-93
  mixture_bound                   the per-entry scale S of the device tolerance |device - reference| <= 1e-5 S
  observe_pack                 <- Odometry/MACVO.py:198-283 with GaussianMixtureCovariance as ObsCovModel (depth_cov0 /
                                  depth_cov1 are depth_est.cov of the two frames), then the modifiers, as
                                  oracle.ablation.observe_pack does for the other models

Reference quirks kept: the in-place clamp of the caller's flow_cov; the kernel axis weighted by sigma_uu runs along image
rows; weights below 1e-3 dropped (NaN stays) and the rest renormalised; the mixture variance halved and never clamped
(min_depth_cov is never read); `depth_cov` replaces the variance only when no flow_cov is given.

PINNED by tests/golden/mixture_*.pt (tests/golden/make_golden_mixture.py, the reference class itself).
Only tests/ may import this module.
"""
from __future__ import annotations

import torch

from . import ablation as oab
from . import covariance as ocov
from . import frontend as ofe
from . import observe_filters as ofil
from .observe import _k_matrix, _window_leaves, se3_act_f32

Tensor = torch.Tensor
PROB_THRESHOLD = 1e-3


def _flow_cov(n: int, flow_cov: Tensor | None, min_flow_cov: float, match_cov_default: float) -> Tensor:
    if flow_cov is not None:
        flow_cov[..., :2].clamp_(min=min_flow_cov ** 2)          # in place on the caller's tensor
        return flow_cov
    flow_cov = torch.ones((n, 3), dtype=torch.float) * match_cov_default
    flow_cov[..., 2] = 0.0
    return flow_cov


def _patches(kp: Tensor, maps: list[Tensor], kernel_size: int) -> list[Tensor]:
    """per map the (n, k*k) taps around each keypoint, in the filter weights' order (python index semantics)"""
    n, half = kp.size(0), kernel_size // 2
    kp_long = kp.long()
    off = torch.arange(-half, half + 1, dtype=torch.long)
    uu, vv = torch.meshgrid(off, off, indexing="ij")
    all_u = kp_long[:, 0].unsqueeze(-1) + uu.reshape(1, -1)
    all_v = kp_long[:, 1].unsqueeze(-1) + vv.reshape(1, -1)
    return [m[..., all_v, all_u].view(n, kernel_size, kernel_size).permute(0, 2, 1).flatten(1) for m in maps]


def filter_weights(flow_cov: Tensor, kernel_size: int) -> Tensor:
    """gaussain_full_kernels of the (n,3) [uu, vv, uv] flow covariances, flattened to (n, k*k)"""
    n = flow_cov.size(0)
    cov2 = torch.empty((n, 2, 2))
    cov2[:, 0, 0], cov2[:, 0, 1], cov2[:, 1, 0], cov2[:, 1, 1] = flow_cov[:, 0], flow_cov[:, 2], flow_cov[:, 2], flow_cov[:, 1]
    return ocov.gaussian_full_kernels(cov2, kernel_size).flatten(1)


def mixture_mean_var(means: Tensor, variances: Tensor, prob: Tensor, threshold: float = PROB_THRESHOLD):
    prob = prob.clone()
    prob[prob < threshold] = 0.
    prob = prob / prob.sum(dim=1, keepdim=True)
    mean = (means * prob).sum(dim=1)
    var = ((variances + means.square()) * prob).sum(dim=1) - mean.square()
    return mean, var / 2


def _project(u: Tensor, v: Tensor, d: Tensor, var: Tensor, fc: Tensor, fx, fy, cx, cy) -> Tensor:
    var_u, var_v, var_uv = fc[..., 0], fc[..., 1], fc[..., 2]
    s_xx = (((u - cx).square() * var) + (d.square() * var_u) + (var_u * var)) / (fx ** 2)
    s_yy = (((v - cy).square() * var) + (d.square() * var_v) + (var_v * var)) / (fy ** 2)
    s_xy = (((u - cx) * (v - cy) * var) + (d.square() + var) * var_uv) / (fx * fy)
    s_xz = (var * (u - cx)) / fx
    s_yz = (var * (v - cy)) / fy
    rows = [[var, s_xz, s_yz], [s_xz, s_xx, s_xy], [s_yz, s_xy, s_yy]]
    mat = torch.empty((u.shape[0], 3, 3))            # create_3x3_matrix: fp32
    for i in range(3):
        for j in range(3):
            mat[..., i, j] = rows[i][j]
    return mat


def gaussian_mixture_covariance(kp: Tensor, depth_map: Tensor, depth_cov_map: Tensor, flow_cov: Tensor | None, fx: float,
                                fy: float, cx: float, cy: float, kernel_size: int = 31, min_flow_cov: float = 0.25,
                                match_cov_default: float = 0.25, depth_cov: Tensor | None = None,
                                threshold: float = PROB_THRESHOLD) -> Tensor:
    """kp (K,2) int64 or fp32 [u,v]; depth_map / depth_cov_map (1,1,H,W); flow_cov (K,3) or None -> (K,3,3) float64.
    `threshold` 0 gives the mixture without the reference's pruning of small weights."""
    n = kp.size(0)
    has_flow_cov = flow_cov is not None
    fc = _flow_cov(n, flow_cov, min_flow_cov, match_cov_default)
    filt = filter_weights(fc, kernel_size)
    d, v = _patches(kp, [depth_map, depth_cov_map], kernel_size)
    mean, var = mixture_mean_var(d, v, filt, threshold)
    if not has_flow_cov and depth_cov is not None:
        var = depth_cov
    return _project(kp[..., 0], kp[..., 1], mean, var, fc, fx, fy, cx, cy).double()


def mixture_bound(kp: Tensor, depth_map: Tensor, depth_cov_map: Tensor, flow_cov: Tensor | None, fx: float, fy: float,
                  cx: float, cy: float, kernel_size: int = 31, min_flow_cov: float = 0.25, match_cov_default: float = 0.25,
                  depth_cov: Tensor | None = None) -> Tensor:
    """(K,3,3) float64 scale S per entry: the covariance recomputed in float64 with every term in absolute value and the
    variance replaced by the mixture's second moment M2 = 1/2 sum p (v + d^2) (or |depth_cov| where it overrides). The
    variance E[x^2] - mean^2 cancels, so fp32 evaluations in another order part by a few ulps of M2, not of the result."""
    n = kp.size(0)
    has_flow_cov = flow_cov is not None
    fc = _flow_cov(n, None if flow_cov is None else flow_cov.clone(), min_flow_cov, match_cov_default)
    filt = filter_weights(fc, kernel_size).double()
    d, v = _patches(kp, [depth_map.double(), depth_cov_map.double()], kernel_size)
    filt[filt < PROB_THRESHOLD] = 0.
    p = filt / filt.sum(dim=1, keepdim=True)
    mean = (d * p).sum(dim=1)
    m2 = ((v.abs() + d.square()) * p).sum(dim=1) / 2
    if not has_flow_cov and depth_cov is not None:
        m2 = depth_cov.double().abs()
    u, vv = kp[..., 0].double(), kp[..., 1].double()
    return _abs_project(u, vv, mean, m2, fc.double(), fx, fy, cx, cy)


def _abs_project(u: Tensor, v: Tensor, d: Tensor, var: Tensor, fc: Tensor, fx, fy, cx, cy) -> Tensor:
    """Covariance_2to3_full's entries with every term in absolute value, float64"""
    du, dv = (u - cx).abs(), (v - cy).abs()
    suu, svv, suv = fc[..., 0].abs(), fc[..., 1].abs(), fc[..., 2].abs()
    d2 = d.square()
    s_xx = (du.square() * var + d2 * suu + suu * var) / fx ** 2
    s_yy = (dv.square() * var + d2 * svv + svv * var) / fy ** 2
    s_xy = (du * dv * var + (d2 + var) * suv) / abs(fx * fy)
    s_xz, s_yz = var * du / abs(fx), var * dv / abs(fy)
    rows = [[var, s_xz, s_yz], [s_xz, s_xx, s_xy], [s_yz, s_xy, s_yy]]
    mat = torch.empty((u.shape[0], 3, 3), dtype=torch.float64)
    for i in range(3):
        for j in range(3):
            mat[..., i, j] = rows[i][j]
    return mat


def observe_pack(kp0: Tensor, flow: Tensor, match_cov: Tensor, depth0: Tensor, depth1: Tensor, disparity1: Tensor,
                 disp_unc1: Tensor, edge_width: int, intr0, intr1, prev_pose: Tensor, kernel_size: int = 31,
                 min_flow_cov: float = 0.25, min_depth_cov: float = 0.05, match_cov_default: float = 0.25,
                 depth_cov0: Tensor | None = None, depth_cov1: Tensor | None = None,
                 depth_range: tuple[float, float] | None = None, front_of_cam: bool = False, icp: bool = False,
                 cov_model: str = "mixture", cov_ops=()) -> dict:
    """oracle.ablation.observe_pack's arguments and result for cov_model "mixture" (any other model goes there), plus
    "bound0" / "bound1": `mixture_bound` of the kept rows' covariances before the modifiers"""
    if cov_model != "mixture":
        return oab.observe_pack(kp0, flow, match_cov, depth0, depth1, disparity1, disp_unc1, edge_width, intr0, intr1,
                                prev_pose, kernel_size, min_flow_cov, min_depth_cov, match_cov_default, depth_cov0,
                                depth_cov1, depth_range, front_of_cam, icp, cov_model, cov_ops)
    assert depth_cov0 is not None and depth_cov1 is not None, "GaussianMixtureCovariance needs depth_est.cov"
    H, W = flow.shape[-2:]
    k = kp0.shape[0]
    status = 0
    u0, v0 = kp0[:, 0], kp0[:, 1]
    in0 = (u0 >= 0) & (u0 < W) & (v0 >= 0) & (v0 < H)
    if not bool(in0.all()):
        status |= 2
    idx0 = torch.nonzero(in0).reshape(-1)
    kp1_a = kp0[idx0] + ofe.retrieve_pixels(kp0[idx0], flow).T
    inb = ofe.filter_points_in_range(kp1_a, (edge_width, W - edge_width), (edge_width, H - edge_width))
    rows, kp0_i, kp1_i = idx0[inb], kp0[idx0][inb], kp1_a[inb]
    n = rows.numel()
    d0 = ofe.retrieve_pixels(kp0_i, depth0).squeeze(0)
    d1 = ofe.retrieve_pixels(kp1_i, depth1).squeeze(0)
    disp1 = ofe.retrieve_pixels(kp1_i, disparity1).T.reshape(-1)
    dunc1 = ofe.retrieve_pixels(kp1_i, disp_unc1).T.reshape(-1)
    dc0 = ofe.retrieve_pixels(kp0_i, depth_cov0).squeeze(0)
    dc1 = ofe.retrieve_pixels(kp1_i, depth_cov1).squeeze(0)
    uv_cov = ofe.retrieve_pixels(kp0_i, match_cov).T
    kp0_sigma_uv = torch.ones((n, 3)) * match_cov_default
    kp0_sigma_uv[..., 2] = 0.0
    uv_cov[..., :2].clamp_(min=min_flow_cov ** 2)
    half = kernel_size // 2
    leaves = _window_leaves(kp0_i, H, W, half) | _window_leaves(kp1_i.long(), H, W, half)
    if bool(leaves.any()):
        status |= 1
    ev = torch.isfinite(uv_cov).all(-1) & ~leaves
    cov0 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
    cov1 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
    bound0, bound1 = cov0.clone(), cov1.clone()
    args = (kernel_size, min_flow_cov, match_cov_default)
    if bool(ev.any()):
        cov0[ev] = gaussian_mixture_covariance(kp0_i[ev], depth0, depth_cov0, kp0_sigma_uv[ev], *intr0, *args)
        cov1[ev] = gaussian_mixture_covariance(kp1_i[ev], depth1, depth_cov1, uv_cov[ev].clone(), *intr1, *args)
        bound0[ev] = mixture_bound(kp0_i[ev], depth0, depth_cov0, kp0_sigma_uv[ev], *intr0, *args)
        bound1[ev] = mixture_bound(kp1_i[ev], depth1, depth_cov1, uv_cov[ev], *intr1, *args)
    cov0, cov1 = oab.modify(cov0, cov_ops), oab.modify(cov1, cov_ops)
    bad = (~torch.isfinite(cov0)).any(dim=(-1, -2)) | (~torch.isfinite(cov1)).any(dim=(-1, -2))
    ok = ~bad & ev
    if depth_range is not None:
        lo, hi = depth_range
        ok &= ~((d0 < lo) | (d0 > hi) | (d1 < lo) | (d1 > hi))
    if front_of_cam and not bool((dc0 == -1).any()):
        ok &= ((d0 - (dc0.sqrt() * 2)) > 0.) & ((d1 - (dc1.sqrt() * 2)) > 0.)
    pos0_Tc = ocov.pixel2point_ned(kp0_i, d0, _k_matrix(intr0))
    pos_Tw = se3_act_f32(prev_pose, pos0_Tc)
    keep = torch.zeros(k, dtype=torch.bool)
    keep[rows[ok]] = True
    unspecified = torch.zeros(k, dtype=torch.bool)
    unspecified[rows[leaves]] = True
    out = {
        "pos_Tw": pos_Tw[ok], "pixel2_uv": kp1_i[ok], "pixel2_disp": disp1[ok], "pixel2_uv_cov": uv_cov[ok],
        "pixel2_disp_cov": dunc1[ok], "obs1_covTc": cov0[ok], "obs2_covTc": cov1[ok], "pixel1_uv": kp0_i[ok],
        "pixel1_d": d0[ok], "n_obs": int(ok.sum()), "n_inbound": n, "k": k, "status": status,
        "next_pose": prev_pose.double().float().double(), "keep": keep, "unspecified": unspecified, "pos_Tc": pos0_Tc[ok],
        "bound0": bound0[ok], "bound1": bound1[ok],
    }
    if icp:
        R = ofil.quat_matrix_f32(prev_pose[3:7]).repeat((out["n_obs"], 1, 1)).to(torch.float64)
        out.update(pixel2_d=d1[ok], pixel1_d_cov=dc0[ok], pixel2_d_cov=dc1[ok],
                   points_Tc=ocov.pixel2point_ned(kp1_i[ok], d1[ok], _k_matrix(intr1)).double(),
                   cov_Tw=torch.bmm(torch.bmm(R, out["obs1_covTc"]), R.transpose(1, 2)))
    return out
