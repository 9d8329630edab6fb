"""Seeded inputs of the outlier-filter fixtures (tests/golden/filters_*.pt, tests/golden/observe_icp_*.pt) and of the device
tests of the extended `macvo_observe_pack` (tests/test_fused_paper_reproduce.py). Built, like observe_cases.py, from exactly
rounded operations only (randn / rand scaled by powers of two, +, -, *, table look-ups, avg_pool2d), so that every torch
build regenerates the same bits; each fixture stores the sha256 of its inputs.

Filter bundles: the MatchObs columns SimpleDepthFilter / LikelyFrontOfCamFilter / CovarianceSanityFilter read
(pixel1_d, pixel2_d, pixel1_d_cov, pixel2_d_cov (N,1) fp32; obs1_covTc, obs2_covTc (N,3,3) float64), with NaN / +-Inf /
negative / zero depths, depths at min_depth / max_depth and one fp32 ulp either side, negative and NaN d_cov, and one bundle
holding a -1 placeholder.

ICP cases: an observe_cases.py case plus depth covariance maps, planted so that each filter removes some rows but not all."""
from __future__ import annotations

import torch

from tests.golden import observe_cases as oc
from tests.golden.cases import _lognormal_like, sha

Tensor = torch.Tensor
NAN, INF = float("nan"), float("inf")
MIN_DEPTH = 4.0
MAX_DEPTH = 26.0
# the "auto" bundle: max_depth = fx * baseline of this camera (python floats from fp32 tensors, as StereoData gives them)
AUTO_FX, AUTO_BASELINE = 322.5, 0.0625


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def _ulps(x: float) -> list[float]:
    f = torch.tensor(x, dtype=torch.float32)
    return [float(f), float(torch.nextafter(f, torch.tensor(INF))), float(torch.nextafter(f, torch.tensor(-INF)))]


def auto_max_depth() -> float:
    return float(torch.tensor([AUTO_FX], dtype=torch.float32).item() * torch.tensor([AUTO_BASELINE]).item())


# name -> (rows, seed, max_depth config value, placeholder)
BUNDLES = {"random": (600, 80, MAX_DEPTH, False), "auto": (300, 81, "auto", False), "placeholder": (200, 82, MAX_DEPTH, True)}


def filter_bundle(name: str) -> dict:
    """-> {"data": {column: tensor}, "min_depth", "max_depth" (config value, may be "auto")}"""
    n, seed, max_depth, placeholder = BUNDLES[name]
    g = torch.Generator().manual_seed(seed)
    hi = auto_max_depth() if max_depth == "auto" else max_depth
    d = lambda: (torch.rand(n, 1, generator=g) * 32.0).float()
    dc = lambda: _lognormal_like((n, 1), g, 4.0)
    cols = {"pixel1_d": d(), "pixel2_d": d(), "pixel1_d_cov": dc(), "pixel2_d_cov": dc()}
    cov = lambda: torch.randn(n, 3, 3, generator=g, dtype=torch.float64) * 0.125
    c1, c2 = cov(), cov()
    specials = ([NAN, INF, -INF, -1.0, 0.0] + _ulps(MIN_DEPTH) + _ulps(hi)
                + [_f32(hi) * 2.0, MIN_DEPTH * 0.5])
    i = 0
    for col in ("pixel1_d", "pixel2_d"):
        for v in specials:
            cols[col][i, 0] = v
            i += 1
    for col in ("pixel1_d_cov", "pixel2_d_cov"):
        for v in (NAN, -0.25, INF, 0.0, -INF):
            cols[col][i, 0] = v
            i += 1
    # d - 2 sqrt(d_cov) == 0 exactly: dropped (strict inequality)
    cols["pixel1_d"][i, 0], cols["pixel1_d_cov"][i, 0] = 8.0, 16.0
    i += 1
    c1[i, 1, 2] = NAN
    c2[i + 1, 0, 0] = INF
    if placeholder:
        cols["pixel1_d_cov"][n - 3, 0] = -1.0
    return {"data": {**cols, "obs1_covTc": c1, "obs2_covTc": c2}, "min_depth": MIN_DEPTH, "max_depth": max_depth}


def bundle_sha(b: dict) -> str:
    return sha(*b["data"].values())


# ---- observe_pack with the Paper_Reproduce filter chain and the icp columns ----------------------------------------------
ICP_CASES = {"basic": "basic", "nonfinite": "nonfinite", "chunks": "chunks", "placeholder": "basic"}


def icp_inputs(name: str) -> dict:
    """observe_cases.observe_inputs(base) + depth_cov0 / depth_cov1 (1,1,H,W) fp32 and the filter settings; specials at
    the keypoints of the first rows: depth at min / max and an ulp either side on either frame, NaN / -Inf / negative
    depth, NaN and negative d_cov. "placeholder": one in-bound row's depth_cov0 is -1."""
    c = oc.observe_inputs(ICP_CASES[name])
    H, W = c["H"], c["W"]
    g = torch.Generator().manual_seed(90 + list(ICP_CASES).index(name))
    c["depth_cov0"] = _lognormal_like((1, 1, H, W), g, 4.0)
    c["depth_cov1"] = _lognormal_like((1, 1, H, W), g, 4.0)
    c["min_depth"], c["max_depth"] = MIN_DEPTH, MAX_DEPTH
    flow = c["flow"]
    rows = [r for r in range(c["kp0"].shape[0]) if r % 7 == 5][:40]       # away from the planted rows of observe_cases
    specials = [("depth0", v) for v in _ulps(MIN_DEPTH) + _ulps(MAX_DEPTH) + [NAN, -INF, -2.0]]
    specials += [("depth1", v) for v in _ulps(MIN_DEPTH) + _ulps(MAX_DEPTH) + [NAN, -2.0]]
    specials += [("depth_cov0", NAN), ("depth_cov0", -0.5), ("depth_cov1", NAN), ("depth_cov1", -0.5)]
    for r, (m, v) in zip(rows, specials):
        u, vv = c["kp0"][r].tolist()
        flow[0, 0, vv, u], flow[0, 1, vv, u] = 0.5, 0.25       # kp1 truncates to kp0's pixel
        c[m][0, 0, vv, u] = v
    if name == "placeholder":
        u, vv = c["kp0"][rows[-1]].tolist()
        flow[0, 0, vv, u], flow[0, 1, vv, u] = 0.5, 0.25
        c["depth_cov0"][0, 0, vv, u] = -1.0
    return c


def icp_sha(c: dict) -> str:
    return sha(c["flow"], c["match_cov"], c["depth0"], c["depth1"], c["disparity1"], c["disp_unc1"], c["kp0"],
               torch.tensor(c["intr0"] + c["intr1"]), c["prev_pose"], c["depth_cov0"], c["depth_cov1"],
               torch.tensor([c["min_depth"], c["max_depth"]]))


def ext_kwargs(c: dict) -> dict:
    """the oracle's filter / icp keyword arguments for case `c` (the Paper_Reproduce chain)"""
    return {"depth_cov0": c["depth_cov0"], "depth_cov1": c["depth_cov1"], "depth_range": (c["min_depth"], c["max_depth"]),
            "front_of_cam": True, "icp": True}


def icp_solve_inputs(k: int, seed: int) -> dict:
    """observe_cases.solve_inputs (a known small rigid motion, ~35 % of the rows dropped) whose depth1 at the truncated kp1 is
    the true camera-frame depth plus noise, so that the icp graph has a well-posed minimum; small depth covariances"""
    import numpy as np
    from oracle import pgo as opgo
    c = oc.solve_inputs(k, seed)
    H, W = c["H"], c["W"]
    g = torch.Generator().manual_seed(seed + 1)
    kp0 = c["kp0"]
    fx0, fy0, cx0, cy0 = c["intr0"]
    u0, v0 = kp0[:, 0].double().numpy(), kp0[:, 1].double().numpy()
    d0 = c["depth0"][0, 0, kp0[:, 1], kp0[:, 0]].double().numpy()
    pts_w = opgo.se3_act(c["prev_pose"].numpy(), np.stack([d0, (u0 - cx0) / fx0 * d0, (v0 - cy0) / fy0 * d0], -1))
    pc = opgo.se3_act(opgo.se3_inv(c["truth"].numpy()), pts_w)
    kp1 = kp0.float() + c["flow"][0, :, kp0[:, 1], kp0[:, 0]].T
    inside = (kp1[:, 0] >= 0) & (kp1[:, 0] < W) & (kp1[:, 1] >= 0) & (kp1[:, 1] < H)
    p1 = kp1[inside].long()
    noise = torch.randn(int(inside.sum()), generator=g, dtype=torch.float64) * 0.01
    c["depth1"][0, 0, p1[:, 1], p1[:, 0]] = (torch.tensor(pc[inside.numpy(), 0]) + noise).float()
    c["depth_cov0"] = _lognormal_like((1, 1, H, W), g, 2.0 ** -6)
    c["depth_cov1"] = _lognormal_like((1, 1, H, W), g, 2.0 ** -6)
    c["min_depth"], c["max_depth"] = MIN_DEPTH, MAX_DEPTH
    return c


def dense_frame_maps(H: int, W: int, seed: int) -> dict:
    """one frame's dense maps for the end-to-end tests: flow (1,2,H,W) |.| < 2 px, match_cov [uu, vv, uv], smooth depth0 /
    depth1 over [2, 28] m, scaled by 1/4 in the left third of the image (there SimpleDepthFilter drops part of the rows),
    depth covariances log-uniform over [2^-2, 2^5) (so that d - 2 sqrt(d_cov) <= 0 for part of the near pixels),
    disparity and its uncertainty"""
    g = torch.Generator().manual_seed(seed)
    m = oc.dense_maps(H, W, g, flow_scale=0.5)
    for k in ("depth0", "depth1"):
        m[k][..., : W // 3] *= 0.25
    m["depth_cov0"] = _lognormal_like((1, 1, H, W), g, 2.0)
    m["depth_cov1"] = _lognormal_like((1, 1, H, W), g, 2.0)
    return m
