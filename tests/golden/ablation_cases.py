"""Seeded inputs of the ablation back-end fixtures (tests/golden/ablation_*.pt, tests/golden/make_golden_ablation.py) and of
their device tests (tests/test_ablation_backends.py). Exactly rounded operations only (filter_cases.py / observe_cases.py
inputs, constants that are powers of two or small integers, randn scaled by powers of two); each fixture stores the sha256
of its inputs.

Covariance models (Config/Experiment/MACVO/Ablation_Study): name -> (macvo_observe_ext_t cov_model, modifiers innermost
first, the reference config of cov.obs).

Observe cases: "nonfinite" of filter_cases.py; "planted" = its "basic" case plus rows with an indefinite flow covariance
(sigma_uv = 2^30 over unit variances, at a depth of 2^50 m: the construction under which sigma_xy alone would overflow
fp32; and sigma_uv = 4, a plainly indefinite one); "boundary" = observe_cases' "boundary" (windows wrapping past the top /
left edge) plus three rows whose kp0 window crosses the bottom / right edge: only NoCovariance can run it. The depth 2^50 is written over a 31x31 patch, so that its neighbours'
windows see it too.

Modifier set: (K,3,3) float64 — an exact-zero row (det exactly 0), negative dets, NaN / +-Inf on and off the diagonal,
SPD matrices scaled by 2^+-365 (about 1e+-110: det overflow / underflow) and random SPD matrices."""
from __future__ import annotations

from types import SimpleNamespace as NS

import torch

from tests.golden import filter_cases as fc
from tests.golden import observe_cases as oc
from tests.golden.cases import _lognormal_like, sha

Tensor = torch.Tensor
NAN, INF = float("nan"), float("inf")
MATCH_ARGS = dict(kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)


def _match(prefix: str, device: str) -> NS:
    return NS(type=prefix + "MatchCovariance", args=NS(device=device, **MATCH_ARGS))


def model_config(name: str, prefix: str = "", device: str = "cpu") -> NS:
    """cov.obs of the ablation YAMLs (prefix "B200_" for the plugins)"""
    m = _match(prefix, device)
    wrap = lambda t, inner: NS(type=prefix + t, args=inner)
    return {"nocov": NS(type=prefix + "NoCovariance", args=None),
            "diag": wrap("Modifier_Diagonalize", m),
            "norm": wrap("Modifier_Normalize", m),
            "normdiag": wrap("Modifier_Normalize", wrap("Modifier_Diagonalize", m)),
            "diagnorm": wrap("Modifier_Diagonalize", wrap("Modifier_Normalize", m))}[name]


# name -> (cov_model, cov_ops)
MODELS = {"nocov": ("identity", []), "diag": ("match", ["diagonalize"]), "norm": ("match", ["normalize"]),
          "normdiag": ("match", ["diagonalize", "normalize"]), "diagnorm": ("match", ["normalize", "diagonalize"])}
CASES = ("planted", "nonfinite", "boundary")
PLANTED = (3, 14, 25)        # rows of the "planted" case: huge indefinite, huge indefinite (depth 2^50), plainly indefinite


def case_models(case: str) -> list[str]:
    """the reference raises IndexError for a MatchCovariance window past the bottom / right edge"""
    return ["nocov"] if case == "boundary" else list(MODELS)


def observe_inputs(case: str) -> dict:
    if case == "nonfinite":
        return fc.icp_inputs(case)
    if case == "boundary":
        c = oc.observe_inputs("boundary")
        g = torch.Generator().manual_seed(97)
        c["depth_cov0"] = _lognormal_like((1, 1, c["H"], c["W"]), g, 4.0)
        c["depth_cov1"] = _lognormal_like((1, 1, c["H"], c["W"]), g, 4.0)
        c["min_depth"], c["max_depth"] = fc.MIN_DEPTH, fc.MAX_DEPTH
        W, H = c["W"], c["H"]
        for r, (u, v, fu, fv) in enumerate(((W - 5, H - 5, -40.0, -40.0), (W - 10, 100, -40.0, 0.0), (100, H - 8, 0.0, -40.0))):
            c["kp0"][r] = torch.tensor([u, v])         # kp0's window crosses the right / bottom edge, kp1 lies in range
            c["flow"][0, 0, v, u], c["flow"][0, 1, v, u] = fu, fv
        return c
    c = fc.icp_inputs("basic")
    for r, (suv, depth) in zip(PLANTED, ((2.0 ** 30, None), (2.0 ** 30, 2.0 ** 50), (4.0, None))):
        u, v = c["kp0"][r].tolist()
        c["flow"][0, 0, v, u], c["flow"][0, 1, v, u] = 0.5, 0.25          # kp1 truncates to kp0's pixel
        c["match_cov"][0, :, v, u] = torch.tensor([1.0, 1.0, suv])
        if depth is not None:
            c["depth1"][0, 0, v - 15:v + 16, u - 15:u + 16] = depth
    return c


def input_sha(c: dict) -> str:
    return fc.icp_sha(c)


def ext_kwargs(c: dict, model: str) -> dict:
    cov_model, cov_ops = MODELS[model]
    return dict(fc.ext_kwargs(c), cov_model=cov_model, cov_ops=cov_ops)


def modifier_set(n_random: int = 64, seed: int = 120) -> Tensor:
    g = torch.Generator().manual_seed(seed)

    def spd(n):      # dyadic entries with few bits: the product and the sum are exact in any summation order
        a = torch.randint(-16, 17, (n, 3, 3), generator=g).double() * 0.0625
        return a @ a.transpose(1, 2) + torch.eye(3, dtype=torch.float64)
    rows = []
    z = spd(1)[0]
    z[1] = 0.0                                                   # exact-zero row: det exactly 0
    rows.append(z)
    z = spd(1)[0]
    z[:, 2] = 0.0                                                # exact-zero column
    rows.append(z)
    for m in spd(2):                                             # indefinite: negative det
        m[0, 1] = m[1, 0] = 4.0
        rows.append(m)
    rows.append(-spd(1)[0])                                      # negative definite: negative det
    for val in (NAN, INF, -INF):
        for i, j in ((0, 0), (1, 1), (0, 1), (2, 0), (1, 2)):
            m = spd(1)[0]
            m[i, j] = val
            rows.append(m)
    for m, s in zip(spd(4), (2.0 ** 365, 2.0 ** -365, 2.0 ** 340, 2.0 ** -340)):
        rows.append(m * s)                                       # det overflow / underflow (or not quite)
    rows += list(spd(n_random))
    return torch.stack(rows)
