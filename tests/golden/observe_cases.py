"""Seeded inputs of the observation-building fixtures (tests/golden/observe_*.pt) and of the device tests of
`macvo_observe_pack` (tests/test_observe.py), built from exactly rounded operations only (randn / rand scaled by powers of
two, +, -, *, table look-ups, avg_pool2d as in `cases.cov_inputs`), so that every torch build regenerates the same bits;
each fixture stores the sha256 of its inputs.

A case is a dict: the dense maps flow (1,2,H,W), match_cov (1,3,H,W) [uu, vv, uv], depth0, depth1, disparity1,
disp_unc1 (1,1,H,W); kp0 (k,2) int64 [u, v]; intr0 / intr1 (fx, fy, cx, cy); prev_pose (7,) float64 [t, q_xyzw]; the
scalars edge_width, kernel_size, min_flow_cov, min_depth_cov, match_cov_default."""
from __future__ import annotations

import numpy as np
import torch

from tests.golden.cases import _lognormal_like, sha  # noqa: F401  (sha re-exported for the tests)

Tensor = torch.Tensor
NAN, INF = float("nan"), float("inf")

# name -> (H, W, k, kernel_size, seed)
CASES = {
    "basic": (160, 224, 700, 31, 31),
    "chunks": (160, 224, 2500, 31, 32),
    "boundary": (160, 224, 300, 31, 33),
    "nonfinite": (160, 224, 300, 31, 34),
    **{f"ksize{ks}": (160, 224, 200, ks, 40 + ks) for ks in (1, 3, 7, 15, 29, 31)},
}
INTR0 = (320.0, 310.5, 111.25, 79.75)            # cx != cy, non-integer, fx != fy
INTR1 = (322.5, 309.0, 112.5, 80.25)             # intr0 != intr1
PREV_POSE = torch.tensor([0.5, -1.25, 2.0, 0.2, 0.4, 0.4, 0.8], dtype=torch.float64)   # unit quaternion (1,2,2,4)/5
# rows of the "chunks" case whose match covariance is NaN: warp edges, the whole last warp of chunk 0, both sides of
# every 1024-record boundary, a strided run inside chunk 1 and the last row
CHUNK_DROPS = sorted({0, 31, 32, 63, *range(992, 1024), 1024, 1025, 2047, 2048, 2049, *range(1500, 1700, 7), 2499})


def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def dense_maps(H: int, W: int, g: torch.Generator, flow_scale: float = 2.0) -> dict:
    """flow N(0, flow_scale^2); uu, vv log-uniform over [2^-5, 4) (the 0.25^2 clamp is active on part of them), |uv| <=
    2^-6 (positive definite); locally smooth depth; positive disparity and uncertainty"""
    flow = torch.randn(1, 2, H, W, generator=g) * flow_scale
    uv = (torch.rand(1, 1, H, W, generator=g) - 0.5) * 2.0 ** -5
    match_cov = torch.cat([_lognormal_like((1, 2, H, W), g, 0.25), uv], dim=1)

    def depth():
        d = 2.0 + 28.0 * torch.rand(1, 1, H, W, generator=g)
        d = torch.nn.functional.avg_pool2d(d, 9, stride=1, padding=4)
        return d + torch.randn(1, 1, H, W, generator=g) * 0.0625
    depth0, depth1 = depth(), depth()
    return {"flow": flow, "match_cov": match_cov, "depth0": depth0, "depth1": depth1,
            "disparity1": _lognormal_like((1, 1, H, W), g, 4.0), "disp_unc1": _lognormal_like((1, 1, H, W), g, 0.125)}


def unique_pixels(H: int, W: int, k: int, margin: int, g: torch.Generator) -> Tensor:
    """k distinct pixels [u, v] (int64) at least `margin` from every image edge, in random order"""
    nc, nr = W - 2 * margin, H - 2 * margin
    idx = torch.randperm(nr * nc, generator=g)[:k]
    return torch.stack([margin + idx % nc, margin + idx // nc], dim=-1)


def _scalars(kernel_size: int, edge_width: int = 32, clamp_default: bool = False) -> dict:
    if not clamp_default:       # MACVO_Performant's covariance settings
        return {"edge_width": edge_width, "kernel_size": kernel_size, "min_flow_cov": 0.25, "min_depth_cov": 0.05,
                "match_cov_default": 0.25}
    # min_flow_cov^2 = 0.09 > match_cov_default: frame 0's constant covariance is clamped too
    return {"edge_width": edge_width, "kernel_size": kernel_size, "min_flow_cov": 0.3, "min_depth_cov": 0.05,
            "match_cov_default": 0.0625}


def _ulp_targets(lo: int, hi: int) -> list[tuple[float, bool]]:
    """(coordinate, in range) for lo and hi exactly, one fp32 ulp inside and one outside each (strict inequalities)"""
    f = lambda x: torch.tensor(float(x), dtype=torch.float32)
    up, dn = torch.tensor(INF), torch.tensor(-INF)
    return [(float(f(lo)), False), (float(torch.nextafter(f(lo), up)), True), (float(torch.nextafter(f(lo), dn)), False),
            (float(f(hi)), False), (float(torch.nextafter(f(hi), dn)), True), (float(torch.nextafter(f(hi), up)), False)]


def _set_flow(c: dict, i: int, fu: float, fv: float) -> None:
    u, v = c["kp0"][i].tolist()
    c["flow"][0, 0, v, u], c["flow"][0, 1, v, u] = fu, fv


def boundary_rows(c: dict) -> list[tuple[int, str, float, bool]]:
    """flows that put kp1 on u = edge, w - edge, v = edge, h - edge, an ulp either side, or make it NaN.
    -> (row, axis, target, expected in range); the other coordinate lands in the middle of the image."""
    H, W, e = c["H"], c["W"], c["edge_width"]
    rows, i = [], 3
    for axis, lo, hi in (("u", e, W - e), ("v", e, H - e)):
        for j, (target, inside) in enumerate(_ulp_targets(lo, hi)):
            # a keypoint 4 px from the target: the flow target - kp0 is exact in fp32, and so is kp0 + flow; one
            # keypoint per row (3 px apart along the other axis), so that every row has its own flow
            base = int(round(target))
            kp = [W // 2 + 3 * j, H // 2 + 3 * j]
            kp[0 if axis == "u" else 1] = base + (4 if base == lo else -4)
            c["kp0"][i] = torch.tensor(kp)
            d = torch.tensor(target, dtype=torch.float32) - float(kp[0 if axis == "u" else 1])
            fu, fv = (float(d), 0.25) if axis == "u" else (0.25, float(d))
            _set_flow(c, i, fu, fv)
            got = torch.tensor(float(kp[0 if axis == "u" else 1]), dtype=torch.float32) + d
            assert float(got) == target, "boundary flow must land exactly on its target"
            rows.append((i, axis, target, inside))
            i += 7
    for fu, fv in ((NAN, 0.25), (0.25, NAN), (INF, 0.25), (0.25, -INF)):
        _set_flow(c, i, fu, fv)
        rows.append((i, "nan" if fu != fu or fv != fv else "inf", NAN, False))
        i += 7
    return rows


# (row offset, map, value, where) of the "nonfinite" case; "centre" = at the keypoint, "window" = 5 rows up, 7 columns
# right of it. The flow of these rows is (0.5, 0.25), so that kp1 truncates to the same pixel as kp0.
DEPTH_SPECIALS = [(m, v, w) for m in ("depth0", "depth1") for v in (NAN, INF, -INF, 0.0, -2.0, 2.0 ** 100)
                  for w in ("centre", "window")]
# (uu, vv, uv) at kp0: NaN / Inf entries, singular (uu vv == uv^2, also after the clamp), indefinite; -Inf on the
# diagonal is clamped to min_flow_cov^2 (kept), on the off-diagonal it is not (dropped)
COV_SPECIALS = [(NAN, 1.0, 0.0), (1.0, NAN, 0.0), (1.0, 1.0, NAN), (INF, 1.0, 0.0), (1.0, INF, 0.0), (1.0, 1.0, INF),
                (-INF, 1.0, 0.0), (1.0, 1.0, -INF), (1.0, 4.0, 2.0), (0.25, 0.25, 0.25), (0.01, 0.0625, 0.0625),
                (1.0, 1.0, 2.0), (0.5, 0.125, -1.0)]


def nonfinite_rows(c: dict) -> dict:
    """plant the specials at keypoints 12 px apart: the depth specials in two bands at v = 40 and 54, the covariance and
    pass-through specials at v = 100 and 116, out of reach of every planted depth (windows are +-15 px), so that each of
    these rows is dropped or kept for its own special alone; -> {kind: [rows]}"""
    out: dict = {"depth": [], "cov": [], "disp_nan": [], "unc_inf": []}
    i = 2

    def place(u: int, v: int) -> tuple[int, int, int]:
        nonlocal i
        c["kp0"][i] = torch.tensor([u, v])
        _set_flow(c, i, 0.5, 0.25)
        row, i = i, i + 5
        return row, u, v
    for j, (m, val, where) in enumerate(DEPTH_SPECIALS):
        row, u, v = place(40 + 12 * (j % 12), 40 + 14 * (j // 12))
        if where == "centre":
            c[m][0, 0, v, u] = val
        else:
            c[m][0, 0, v - 5, u + 7] = val
        out["depth"].append(row)
    for j, (uu, vv, uv) in enumerate(COV_SPECIALS):
        row, u, v = place(40 + 12 * j, 100)
        c["match_cov"][0, :, v, u] = torch.tensor([uu, vv, uv])
        out["cov"].append(row)
    for key, m, val, (u, v) in (("disp_nan", "disparity1", NAN, (60, 116)), ("unc_inf", "disp_unc1", INF, (150, 116))):
        row, u, v = place(u, v)
        c[m][0, 0, v, u] = val
        out[key].append(row)
    return out


def observe_inputs(name: str) -> dict:
    H, W, k, ks, seed = CASES[name]
    g = _gen(seed)
    c = {"H": H, "W": W, **dense_maps(H, W, g), **_scalars(ks, clamp_default=name.startswith("ksize"))}
    c["kp0"] = unique_pixels(H, W, k, 32, g)
    c["intr0"], c["intr1"], c["prev_pose"] = INTR0, INTR1, PREV_POSE.clone()
    if name == "chunks":
        rows = torch.tensor(CHUNK_DROPS)
        c["match_cov"][0, 0, c["kp0"][rows, 1], c["kp0"][rows, 0]] = NAN
        c["flow"] = c["flow"] * 0.125          # nearly every row in range: the kept rows follow the chosen drops
    elif name == "boundary":
        c["rows"] = boundary_rows(c)
    elif name == "nonfinite":
        c["rows"] = nonfinite_rows(c)
    return c


def input_sha(c: dict) -> str:
    return sha(c["flow"], c["match_cov"], c["depth0"], c["depth1"], c["disparity1"], c["disp_unc1"], c["kp0"],
               torch.tensor(c["intr0"] + c["intr1"]), c["prev_pose"])


def oracle_args(c: dict) -> tuple:
    """positional + keyword arguments of oracle.observe.observe_pack / macvo_b200.ops.observe_pack (maps in the same order)"""
    return ((c["kp0"], c["flow"], c["match_cov"], c["depth0"], c["depth1"], c["disparity1"], c["disp_unc1"],
             c["edge_width"], c["intr0"], c["intr1"], c["prev_pose"]),
            {k: c[k] for k in ("kernel_size", "min_flow_cov", "min_depth_cov", "match_cov_default")})


# ---- device tests that need no fixture ------------------------------------------------------------------------------------
def compaction_inputs(k: int, seed: int = 50) -> dict:
    """k in-range keypoints with finite maps on a 160 x 224 frame (|flow| <= 2^-3, kernel_size 3): a row is dropped exactly
    where the test puts NaN into its match covariance"""
    H, W = 160, 224
    g = _gen(seed)
    c = {"H": H, "W": W, **dense_maps(H, W, g, 1.0), **_scalars(3)}
    c["flow"] = (torch.rand(1, 2, H, W, generator=g) - 0.5) * 0.25
    c["kp0"] = unique_pixels(H, W, k, 34, g)
    c["intr0"], c["intr1"], c["prev_pose"] = INTR0, INTR1, PREV_POSE.clone()
    return c


def drop_rows(c: dict, rows) -> dict:
    """a copy of case `c` whose match covariance is NaN at the keypoints of `rows`"""
    c = dict(c)
    c["match_cov"] = c["match_cov"].clone()
    rows = torch.as_tensor(rows, dtype=torch.long)
    if rows.numel():
        c["match_cov"][0, 1, c["kp0"][rows, 1], c["kp0"][rows, 0]] = NAN
    return c


def solve_inputs(k: int, seed: int, drop: float = 0.35) -> dict:
    """a 480 x 640 frame pair (the bench shape) whose flow and disparity follow a known small rigid motion plus noise, so
    that the LM has a well-posed minimum; about `drop` of the rows get a NaN match covariance"""
    from oracle import pgo as opgo
    H, W = 480, 640
    g = _gen(seed)
    c = {"H": H, "W": W, **dense_maps(H, W, g), **_scalars(31)}
    d = 3.0 + 12.0 * torch.rand(1, 1, H, W, generator=g)
    c["depth0"] = torch.nn.functional.avg_pool2d(d, 9, stride=1, padding=4)
    c["kp0"] = kp0 = unique_pixels(H, W, k, 48, g)
    c["intr0"], c["intr1"] = (320.0, 318.0, 319.5, 239.5), (321.0, 319.0, 320.5, 240.5)
    c["prev_pose"] = prev = torch.tensor([0.1, -0.05, 0.2, 0.0, 0.0, 0.0, 1.0], dtype=torch.float64)
    c["baseline"] = 0.25
    rng = np.random.default_rng(seed)
    fx0, fy0, cx0, cy0 = c["intr0"]
    fx1, fy1, cx1, cy1 = c["intr1"]
    u0, v0 = kp0[:, 0].double().numpy(), kp0[:, 1].double().numpy()
    d0 = c["depth0"][0, 0, kp0[:, 1], kp0[:, 0]].double().numpy()
    pts_w = opgo.se3_act(prev.numpy(), np.stack([d0, (u0 - cx0) / fx0 * d0, (v0 - cy0) / fy0 * d0], -1))
    truth = opgo.se3_mul(prev.numpy(), opgo.se3_exp(np.array([0.04, -0.02, 0.01, 0.01, -0.015, 0.02])))
    pc = opgo.se3_act(opgo.se3_inv(truth), pts_w)
    u1 = fx1 * pc[:, 1] / pc[:, 0] + cx1 + rng.normal(size=k) * 0.3
    v1 = fy1 * pc[:, 2] / pc[:, 0] + cy1 + rng.normal(size=k) * 0.3
    c["flow"][0, 0, kp0[:, 1], kp0[:, 0]] = torch.tensor(u1 - u0, dtype=torch.float32)
    c["flow"][0, 1, kp0[:, 1], kp0[:, 0]] = torch.tensor(v1 - v0, dtype=torch.float32)
    kp1 = kp0.float() + c["flow"][0, :, kp0[:, 1], kp0[:, 0]].T
    inside = (kp1[:, 0] >= 0) & (kp1[:, 0] < W) & (kp1[:, 1] >= 0) & (kp1[:, 1] < H)
    p1 = kp1[inside].long()
    disp = fx1 * c["baseline"] / pc[inside.numpy(), 0] + rng.normal(size=int(inside.sum())) * 0.05
    c["disparity1"][0, 0, p1[:, 1], p1[:, 0]] = torch.tensor(disp, dtype=torch.float32)
    c["truth"] = torch.tensor(truth)
    rows = torch.nonzero(torch.rand(k, generator=g) < drop).reshape(-1)
    return drop_rows(c, rows)
