"""TEST INFRASTRUCTURE — CPU oracle for the back ends of MAC-VO's ablation configs (Config/Experiment/MACVO/Ablation_Study):
the covariance models NoCovariance / Modifier_Diagonalize / Modifier_Normalize, `macvo_observe_pack` with a covariance
spec (csrc/observe.cu, `macvo_observe_ext_t.cov_model / cov_ops`) and RandomSelector.

  no_covariance                <- NoCovariance.estimate              Module/Covariance/Project2to3.py:48-57
  diagonalize                  <- Modifier_Diagonalize.estimate      Project2to3.py:281-302
  normalize                    <- Modifier_Normalize.estimate        Project2to3.py:305-323 (CPU float64 torch.det, literally)
  observe_pack                 <- Odometry/MACVO.py:198-283 with the covariance model applied where ObsCovModel.estimate is
                                  called: under NoCovariance `flow_cov` is not clamped (pixel2_uv_cov holds the network's
                                  values), no depth patch is read (no status bit 0, no unspecified rows) and a non-finite 2x2
                                  flow covariance drops nothing; the modifiers act before the sanity filter and cov_Tw
  random_selector              <- RandomSelector.select_point        Module/KeypointSelector.py:103-118

With cov_model "match" and no modifier `observe_pack` is `oracle.observe_filters.observe_pack`.
PINNED by tests/golden/ablation_*.pt (tests/golden/make_golden_ablation.py, the reference classes themselves).
Only tests/ may import this module.
"""
from __future__ import annotations

import torch

from . import covariance as ocov
from . import frontend as ofe
from . import observe_filters as ofil
from .observe import _k_matrix, _window_leaves, se3_act_f32

Tensor = torch.Tensor
OFF_DIAGONAL = [(i, j) for i in range(3) for j in range(3) if i != j]


def no_covariance(n: int) -> Tensor:
    return torch.eye(3).unsqueeze(0).repeat(n, 1, 1).double()


def diagonalize(covs: Tensor) -> Tensor:
    covs = covs.clone()
    for i, j in OFF_DIAGONAL:
        covs[..., i, j] = 0.
    return covs


def normalize(covs: Tensor) -> Tensor:
    covs = covs.clone()
    covs /= torch.det(covs).unsqueeze(-1).unsqueeze(-1)
    return covs


def modify(covs: Tensor, ops) -> Tensor:
    """the modifiers `ops` ("diagonalize" / "normalize"), innermost wrapper first"""
    for op in ops:
        covs = {"diagonalize": diagonalize, "normalize": normalize}[op](covs)
    return covs


def observe_pack(kp0: Tensor, flow: Tensor, match_cov: Tensor, depth0: Tensor, depth1: Tensor, disparity1: Tensor,
                 disp_unc1: Tensor, edge_width: int, intr0, intr1, prev_pose: Tensor, kernel_size: int = 31,
                 min_flow_cov: float = 0.25, min_depth_cov: float = 0.05, match_cov_default: float = 0.25,
                 depth_cov0: Tensor | None = None, depth_cov1: Tensor | None = None,
                 depth_range: tuple[float, float] | None = None, front_of_cam: bool = False, icp: bool = False,
                 cov_model: str = "match", cov_ops=()) -> dict:
    """`oracle.observe_filters.observe_pack`'s arguments and result, with the covariance model `cov_model` ("match" |
    "identity") and the modifiers `cov_ops` applied to both observation covariances"""
    if cov_model == "match" and not cov_ops:
        return ofil.observe_pack(kp0, flow, match_cov, depth0, depth1, disparity1, disp_unc1, edge_width, intr0, intr1,
                                 prev_pose, kernel_size, min_flow_cov, min_depth_cov, match_cov_default, depth_cov0,
                                 depth_cov1, depth_range, front_of_cam, icp)
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
    gather = lambda kp, m: torch.full((n,), -1.0) if m is None else ofe.retrieve_pixels(kp, m).squeeze(0)
    dc0, dc1 = gather(kp0_i, depth_cov0), gather(kp1_i, depth_cov1)
    uv_cov = ofe.retrieve_pixels(kp0_i, match_cov).T
    leaves = torch.zeros(n, dtype=torch.bool)
    if cov_model == "identity":
        cov0, cov1 = no_covariance(n), no_covariance(n)
        ev = torch.ones(n, dtype=torch.bool)
    else:
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
        if bool(ev.any()):
            cov0[ev] = ocov.match_covariance(kp0_i[ev], depth0, kp0_sigma_uv[ev], *intr0, kernel_size, min_flow_cov,
                                             min_depth_cov, match_cov_default)
            cov1[ev] = ocov.match_covariance(kp1_i[ev], depth1, uv_cov[ev].clone(), *intr1, kernel_size, min_flow_cov,
                                             min_depth_cov, match_cov_default)
    cov0, cov1 = modify(cov0, cov_ops), modify(cov1, cov_ops)
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
    }
    if icp:
        R = ofil.quat_matrix_f32(prev_pose[3:7]).repeat((out["n_obs"], 1, 1)).to(torch.float64)
        out.update(pixel2_d=d1[ok], pixel1_d_cov=dc0[ok], pixel2_d_cov=dc1[ok],
                   points_Tc=ocov.pixel2point_ned(kp1_i[ok], d1[ok], _k_matrix(intr1)).double(),
                   cov_Tw=torch.bmm(torch.bmm(R, out["obs1_covTc"]), R.transpose(1, 2)))
    return out


def random_selector(height: int, width: int, num_point: int, mask_width: int, device="cpu",
                    generator: torch.Generator | None = None) -> Tensor:
    """(num_point, 2) int64 (u, v): the reference's two `torch.randint` calls (rows, then columns)"""
    h = torch.randint(mask_width, height - mask_width, (num_point, 1), device=device, generator=generator)
    w = torch.randint(mask_width, width - mask_width, (num_point, 1), device=device, generator=generator)
    return torch.cat([w, h], dim=1)
