"""Seeded inputs of the GaussianMixtureCovariance fixtures (tests/golden/mixture_*.pt, tests/golden/make_golden_mixture.py)
and of their device tests (tests/test_mixture_covariance.py); each fixture stores the sha256 of its inputs.

Standalone cases (one `GaussianMixtureCovariance.estimate` call each): name -> (kernel_size, keypoint dtype, flow mode,
variant). Flow modes: "flow" = a (K,3) flow covariance, part of it below min_flow_cov^2 (clamped in place); "none" = no
flow covariance (match_cov_default * [1, 1, 0]); "override" = no flow covariance and a per-keypoint depth_cov, which
replaces the mixture variance. Variants: "nan" plants a NaN depth tap and a NaN variance tap; "wrap" moves keypoints
next to the top / left edge, where python indexing wraps the patch; "narrow" uses flow variances of 1/16 .. 1/4, where
the 1e-3 weight threshold drops most of a 7x7 patch.

No keypoint has a reference filter weight within 1e-5 relative of the 1e-3 threshold (`drop_threshold_ties`; the generator
checks the reference's own weights again), so no comparison depends on how a weight rounds next to it.

Observe cases: ablation_cases' "planted" and "nonfinite" (the Paper_Reproduce filter chain, the icp columns) under the
mixture model, plain and under each modifier (MODELS)."""
from __future__ import annotations

import torch

from oracle import mixture as omix
from tests.golden import ablation_cases as ac
from tests.golden.cases import _lognormal_like, sha

Tensor = torch.Tensor
H, W, K = 72, 96, 48
INTR = (96.0, 92.0, 47.5, 35.5)
ARGS = dict(min_flow_cov=0.25, match_cov_default=0.25)
TIE_RTOL = 1e-5

CASES = {
    "k31_long_flow": (31, torch.int64, "flow", None),
    "k31_float_none": (31, torch.float32, "none", None),
    "k29_long_override": (29, torch.int64, "override", None),
    "k15_float_flow": (15, torch.float32, "flow", None),
    "k7_long_none": (7, torch.int64, "none", None),
    "k3_float_flow": (3, torch.float32, "flow", None),
    "k1_long_flow": (1, torch.int64, "flow", None),
    "k31_float_nan": (31, torch.float32, "flow", "nan"),
    "k7_long_wrap": (7, torch.int64, "flow", "wrap"),
    "k7_float_narrow": (7, torch.float32, "flow", "narrow"),
}
NAN_ROWS = (0, 1)            # "nan": row 0 sees a NaN depth tap, row 1 a NaN variance tap

# observe models: name -> (cov_model, cov_ops innermost first, the reference config of cov.obs)
MODELS = {"mixture": ("mixture", []), "mixture_diag": ("mixture", ["diagonalize"]),
          "mixture_norm": ("mixture", ["normalize"])}
OBSERVE_CASES = ("planted", "nonfinite")
REF_ARGS = dict(kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)   # README's YAML


def model_config(name: str, prefix: str = "", device: str | None = None):
    """cov.obs of a config that selects the model (prefix "B200_" for the plugins, which also take `device`)"""
    from types import SimpleNamespace as NS
    base = NS(type=prefix + "GaussianMixtureCovariance", args=NS(**REF_ARGS, **({"device": device} if device else {})))
    ops = MODELS[name][1]
    for op in ops:
        base = NS(type=prefix + {"diagonalize": "Modifier_Diagonalize", "normalize": "Modifier_Normalize"}[op], args=base)
    return base


def _flow_cov(n: int, g: torch.Generator, narrow: bool) -> Tensor:
    if narrow:
        suu = 0.0625 + torch.rand(n, generator=g) * 0.1875
        svv = 0.0625 + torch.rand(n, generator=g) * 0.1875
        return torch.stack([suu, svv, torch.zeros(n)], dim=1)
    suu = _lognormal_like((n,), g, 0.125)
    svv = _lognormal_like((n,), g, 0.125)
    rho = (torch.rand(n, generator=g) - 0.5) * 1.5
    return torch.stack([suu, svv, rho * (suu * svv).sqrt()], dim=1)


def threshold_ties(flow_cov: Tensor | None, n: int, kernel_size: int, min_flow_cov: float = 0.25,
                   match_cov_default: float = 0.25) -> Tensor:
    """(n,) bool: a filter weight of the row lies within TIE_RTOL relative of the 1e-3 threshold"""
    fc = omix._flow_cov(n, None if flow_cov is None else flow_cov.clone(), min_flow_cov, match_cov_default)
    p = omix.filter_weights(fc, kernel_size)
    return ((p - omix.PROB_THRESHOLD).abs() <= TIE_RTOL * omix.PROB_THRESHOLD).any(dim=1)


def inputs(case: str, seed: int = 700) -> dict:
    ks, dtype, mode, variant = CASES[case]
    g = torch.Generator().manual_seed(seed + list(CASES).index(case))
    half = ks // 2
    depth = _lognormal_like((1, 1, H, W), g, 2.0)
    dcov = _lognormal_like((1, 1, H, W), g, 0.25)
    n = 2 * K
    lo_u, lo_v = (0, 0) if variant == "wrap" else (half, half)
    u = torch.randint(lo_u, W - half, (n,), generator=g)
    v = torch.randint(lo_v, H - half, (n,), generator=g)
    if variant == "wrap":
        u[: n // 2] = torch.randint(0, max(half, 1), (n // 2,), generator=g)
        v[n // 4: 3 * n // 4] = torch.randint(0, max(half, 1), (n // 2,), generator=g)
    kp = torch.stack([u, v], dim=1)
    if dtype == torch.float32:        # fractions of 1/8: exact in fp32, truncated by .long()
        kp = kp.float() + torch.randint(0, 8, (n, 2), generator=g).float() * 0.125
    flow_cov = _flow_cov(n, g, variant == "narrow") if mode == "flow" else None
    depth_cov = _lognormal_like((n,), g, 0.5) if mode == "override" else None
    keep = ~threshold_ties(flow_cov, n, ks)
    keep = torch.nonzero(keep).reshape(-1)[:K]
    assert keep.numel() == K, f"{case}: too many threshold ties"
    c = {"case": case, "kernel_size": ks, "depth": depth, "depth_cov_map": dcov, "kp": kp[keep].contiguous(),
         "flow_cov": None if flow_cov is None else flow_cov[keep].contiguous(),
         "depth_cov": None if depth_cov is None else depth_cov[keep].contiguous(), "intr": INTR, **ARGS}
    if variant == "nan":
        for r, name in zip(NAN_ROWS, ("depth", "depth_cov_map")):
            uu, vv = c["kp"][r].long().tolist()
            c[name] = c[name].clone()
            c[name][0, 0, vv + min(1, half), uu] = float("nan")
    return c


def input_sha(c: dict) -> str:
    return sha(c["depth"], c["depth_cov_map"], c["kp"], c["flow_cov"], c["depth_cov"])


def oracle_call(c: dict, flow_cov: Tensor | None = None, **kw) -> dict:
    """keyword arguments of oracle.mixture.gaussian_mixture_covariance / mixture_bound for case `c` (flow_cov: the tensor to
    clamp in place, default a copy of the case's)"""
    fc = flow_cov if flow_cov is not None else (None if c["flow_cov"] is None else c["flow_cov"].clone())
    fx, fy, cx, cy = c["intr"]
    return dict(kp=c["kp"], depth_map=c["depth"], depth_cov_map=c["depth_cov_map"], flow_cov=fc, fx=fx, fy=fy, cx=cx,
                cy=cy, kernel_size=c["kernel_size"], depth_cov=c["depth_cov"], **ARGS, **kw)


def observe_inputs(case: str) -> dict:
    return ac.observe_inputs(case)


def ext_kwargs(c: dict, model: str) -> dict:
    cov_model, cov_ops = MODELS[model]
    return dict(ac.fc.ext_kwargs(c), cov_model=cov_model, cov_ops=cov_ops)
