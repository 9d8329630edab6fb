"""Seeded synthetic inputs shared by tests/golden/make_golden.py (reference side)
and the parity tests (oracle / CUDA side). SURVEY.md §8(d) shapes.

Only CPU torch generators and EXACTLY ROUNDED operations (+, -, *, round, table look-ups) are used -> identical bits
wherever the same torch build runs. No transcendental functions: round 1's generators used `torch.exp(torch.randn(..))`
and on the 128-thread GPU hosts MKL's vectorised `vsExp` returned 1-ulp different values in ~5 % of fresh processes
(sha256 of the generated tensor differed run to run while the randn-only tensors never did), which surfaced as a
"flaky" bit-exactness test of the dense post-processing kernel: the kernel had simply been fed inputs that differed from
the ones the golden file was generated with (DESIGN.md §5). Every golden file now also records the sha256 of its inputs.
"""
from __future__ import annotations

import numpy as np
import torch

Tensor = torch.Tensor


def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


_POW2 = torch.tensor([0.125, 0.25, 0.5, 1.0, 2.0, 4.0, 8.0])


def _lognormal_like(shape, g: torch.Generator, scale: float = 1.0) -> Tensor:
    """positive, heavy-tailed (log-uniform over 2^-3 .. 2^4) values built from exact operations only:
    (1 + U[0,1)) * 2^k, k uniform in {-3..3}; multiplying by a power of two is exact in fp32."""
    mant = 1.0 + torch.rand(shape, generator=g)
    k = torch.randint(0, _POW2.numel(), shape, generator=g)
    return mant * _POW2[k] * scale


def sha(*tensors) -> str:
    """sha256 over the raw bytes of the given tensors (None skipped): stored in the golden files, checked by the tests"""
    import hashlib
    h = hashlib.sha256()
    for t in tensors:
        if t is not None:
            h.update(t.contiguous().numpy().tobytes())
    return h.hexdigest()


# ---- correlation volume -------------------------------------------------------------------------
CORR_CASES = {"tiny": (2, 5, 7), "small": (2, 12, 16), "ragged": (1, 9, 13), "clip": (1, 30, 40)}


def corr_inputs(B: int, H1: int, W1: int, D: int = 256, seed: int = 2) -> tuple[Tensor, Tensor]:
    g = _gen(seed + 17 * H1 + W1)
    return torch.randn(B, D, H1, W1, generator=g) * 0.5, torch.randn(B, D, H1, W1, generator=g) * 0.5


def corr_sample_index(N: int) -> tuple[Tensor, Tensor]:
    rows = torch.unique(torch.linspace(0, N - 1, min(N, 48)).long())
    cols = torch.unique(torch.linspace(0, N - 1, min(N, 64)).long())
    return rows, cols


# ---- window lookup --------------------------------------------------------------------------------
LOOKUP_CASES = {"tiny": (1, 5, 7), "small": (2, 12, 16)}


def lookup_inputs(B: int, H1: int, W1: int, seed: int = 3) -> tuple[Tensor, Tensor]:
    g = _gen(seed + 17 * H1 + W1)
    cost_maps = torch.randn(B * H1 * W1, 1, H1, W1, generator=g)
    ys, xs = torch.meshgrid(torch.arange(H1, dtype=torch.float32), torch.arange(W1, dtype=torch.float32), indexing="ij")
    grid = torch.stack([xs, ys], 0).unsqueeze(0).repeat(B, 1, 1, 1)
    coords = grid + torch.randn(B, 2, H1, W1, generator=g) * 3.0       # includes out-of-range targets
    coords[:, :, 0, 0] = -20.0                                          # a fully out-of-range window
    coords[:, 0, 0, 1], coords[:, 1, 0, 1] = float(W1 - 1), float(H1 - 1)  # exact corner
    coords[:, :, 1, 0] = 2.0                                            # exact integer coordinates
    return cost_maps, coords


# ---- network --------------------------------------------------------------------------------------
NET_CASES = {"small": (2, 96, 128), "odd": (1, 100, 130)}


def net_inputs(B: int, H: int, W: int, seed: int = 1000) -> tuple[Tensor, Tensor]:
    g = _gen(seed + H + W)
    base = torch.rand(B, 3, H + 8, W + 8, generator=g)
    base = torch.nn.functional.avg_pool2d(base, 5, stride=1, padding=2)
    return base[..., 4:-4, 4:-4].contiguous(), base[..., 3:-5, 6:-2].contiguous()


# ---- dense post-processing -------------------------------------------------------------------------
DENSE_CASES = {"small": (64, 96)}


def dense_inputs(H: int, W: int, seed: int = 4) -> tuple[Tensor, Tensor]:
    g = _gen(seed + H + W)
    flow = torch.randn(2, 2, H, W, generator=g) * 3.0
    flow[0, 0] = -(torch.rand(H, W, generator=g) * 30 + 1)              # stereo slot: disparity 1..31 px
    flow[0, 0, 0, :4] = torch.tensor([0.0, 1e-3, 2.5, -1e-4])           # zero / tiny / positive disparity
    cov = _lognormal_like((2, 2, H, W), g)
    return flow, cov


# ---- selectors --------------------------------------------------------------------------------------
SELECTOR_RNG_SEED = 5
SELECTOR_CASES = {
    "small": (160, 224, 64, "plain"),
    "cfgA_512": (480, 640, 512, "plain"),
    "cfgA_2048": (480, 640, 2048, "plain"),
    "ties": (160, 224, 4096, "ties"),
    "nan": (160, 224, 128, "nan"),
    "masked": (160, 224, 128, "masked"),
    "flat": (96, 128, 50, "flat"),
}


def selector_inputs(H: int, W: int, variant: str, seed: int = 4) -> tuple[Tensor, Tensor]:
    g = _gen(seed + H + W + sum(map(ord, variant)))
    flow = torch.randn(2, 2, H, W, generator=g) * 3.0
    flow[0, 0] = -(torch.rand(H, W, generator=g) * 30 + 1)
    cov = _lognormal_like((2, 2, H, W), g)
    if variant == "ties":      # quantised -> many equal minima inside one NMS window, equal medians
        cov = (cov * 4).round() / 4 + 0.25
    elif variant == "nan":
        idx = torch.randint(0, H * W, (200,), generator=g)
        cov[1, 0].view(-1)[idx] = float("nan")
        cov[1, 1].view(-1)[idx[:50] + 1] = float("inf")
    elif variant == "flat":    # constant quality: every pixel is its window minimum
        cov = torch.full_like(cov, 0.75)
    return flow, cov


SELECTOR_DEPTH_CASES = {"depth_small": (160, 224, 64, "plain"), "depth_cfgA": (480, 640, 512, "plain"),
                        "depth_masked": (160, 224, 128, "masked"), "depth_nan": (160, 224, 128, "nan")}


def selector_depth_inputs(H: int, W: int, variant: str):
    """two `estimate_pair`-like network outputs (previous / current frame) for the depth-aware selector"""
    f0, c0 = selector_inputs(H, W, variant, seed=14)
    f1, c1 = selector_inputs(H, W, variant, seed=4)
    return (f0, c0), (f1, c1)


def selector_match_mask(H: int, W: int, seed: int = 7) -> Tensor:
    return torch.rand(1, 1, H, W, generator=_gen(seed + H + W)) > 0.3


# ---- covariance model ---------------------------------------------------------------------------------
COV_CASES = {
    "int_default": (160, 224, 96, "int_default"),
    "float_cov": (160, 224, 96, "float_cov"),
    "float_fullcov": (160, 224, 96, "float_fullcov"),
    "none": (160, 224, 32, "none"),
    "cfgA_512": (480, 640, 512, "float_cov"),
}


def cov_inputs(H: int, W: int, K: int, kind: str, seed: int = 8):
    g = _gen(seed + H + W + K + sum(map(ord, kind)))
    depth = 2.0 + 28.0 * torch.rand(1, 1, H, W, generator=g)
    depth = torch.nn.functional.avg_pool2d(depth, 9, stride=1, padding=4)          # locally smooth, like a depth map
    depth = depth + 0.05 * torch.randn(1, 1, H, W, generator=g)
    u = torch.randint(33, W - 33, (K,), generator=g)
    v = torch.randint(33, H - 33, (K,), generator=g)
    if kind == "int_default":
        kp = torch.stack([u, v], dim=-1)                                            # int64, like kp0_uv
        flow_cov = torch.ones(K, 3) * 0.25
        flow_cov[:, 2] = 0.0
    elif kind == "none":
        kp = torch.stack([u, v], dim=-1)
        flow_cov = None
    else:
        kp = torch.stack([u, v], dim=-1).float() + torch.rand(K, 2, generator=g)   # fp32, like kp1_uv
        su = _lognormal_like((K,), g, 0.5)
        sv = _lognormal_like((K,), g, 0.5)
        su[:4] = torch.tensor([0.01, 0.0625, 40.0, 1e-4])                           # exercises the clamp
        suv = torch.zeros(K)
        if kind == "float_fullcov":
            suv = (torch.rand(K, generator=g) - 0.5) * 0.2
        flow_cov = torch.stack([su, sv, suv], dim=-1)
    return kp, depth, flow_cov


# ---- two-frame pose-graph optimisation -------------------------------------------------------------------
PGO_CASES = {"k64": (64, 6), "k512": (512, 6), "k200_far": (200, 9), "k12": (12, 3)}


def pgo_inputs(K: int, seed: int) -> dict:
    """SURVEY.md §8(d): NED points x~U(2,30), y,z~U(-.6x,.6x); true pose Exp([.05,-.02,.01,.01,-.02,.015]);
    observations = projection + N(0, Sigma_i), 5 % gross outliers; init = identity. fp32 like the map stores."""
    from oracle import pgo as opgo
    rng = np.random.default_rng(seed * 7919 + K)
    x = rng.uniform(2, 30, K)
    pts = np.stack([x, rng.uniform(-0.6, 0.6, K) * x, rng.uniform(-0.6, 0.6, K) * x], -1)
    true_pose = opgo.se3_exp(np.array([0.05, -0.02, 0.01, 0.01, -0.02, 0.015]) * (3.0 if seed == 9 else 1.0))
    fx = fy = 320.0
    cx, cy, bl = 320.0, 240.0, 0.25
    pc = opgo.se3_act(opgo.se3_inv(true_pose), pts)
    uv = np.stack([fx * pc[:, 1] / pc[:, 0] + cx, fy * pc[:, 2] / pc[:, 0] + cy], -1)
    disp = fx * bl / pc[:, 0]
    suu, svv = rng.uniform(0.0625, 4, K), rng.uniform(0.0625, 4, K)
    sdd = rng.uniform(0.01, 1, K)
    uv = uv + rng.normal(size=(K, 2)) * np.sqrt(np.stack([suu, svv], -1)) * 0.3
    disp = disp + rng.normal(size=K) * np.sqrt(sdd) * 0.1
    out = rng.uniform(size=K) < 0.05
    uv[out] += rng.uniform(5, 30, (int(out.sum()), 2))
    f32 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)
    return {
        "pos_Tw": f32(pts), "kp2_uv": f32(uv), "kp2_disp": f32(disp),
        "uv_cov": f32(np.stack([suu, svv, np.zeros(K)], -1)), "disp_cov": f32(sdd),
        "K": torch.tensor([[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]), "baseline": bl,
        "init_pose": torch.tensor([0., 0., 0., 0., 0., 0., 1.]),
        "true_pose": torch.tensor(true_pose),
    }


PGO_TYPE_CASES = {"icp_k64": ("icp", 64, 6), "icp_k512": ("icp", 512, 6), "icp_far": ("icp", 200, 9),
                  "reproj_k64": ("reproj", 64, 6), "reproj_k512": ("reproj", 512, 6), "reproj_far": ("reproj", 200, 9)}


def pgo_inputs_typed(graph_type: str, K: int, seed: int) -> dict:
    """`pgo_inputs` + what the icp graph reads (Graphs.py:46-55): pixel2_d, obs2_covTc, cov_Tw (float64 SPD blocks)"""
    from oracle import pgo as opgo
    c = pgo_inputs(K, seed)
    rng = np.random.default_rng(seed * 104729 + K + len(graph_type))
    pc = opgo.se3_act(opgo.se3_inv(c["true_pose"].numpy()), c["pos_Tw"].double().numpy())
    c["kp2_d"] = torch.tensor(pc[:, 0] * (1 + rng.normal(size=K) * 0.01), dtype=torch.float32)

    def spd(scale):
        a = rng.normal(size=(K, 3, 3)) * scale
        return torch.tensor(a @ a.transpose(0, 2, 1) + np.eye(3) * scale * scale * 0.5)
    c["obs_cov"], c["pts_cov"] = spd(0.2), spd(0.1)
    c["graph_type"] = graph_type
    return c


def pgo_graph(c: dict):
    """cases dict -> oracle.pgo.GraphData (fp32 values promoted to fp64, like `.to(torch.double)`)."""
    from oracle import pgo as opgo
    K = c["K"].double().numpy()
    return opgo.GraphData(
        pos_Tw=c["pos_Tw"].double().numpy(), kp2_uv=c["kp2_uv"].double().numpy(), kp2_disp=c["kp2_disp"].double().numpy(),
        uv_cov=c["uv_cov"].double().numpy(), disp_cov=c["disp_cov"].double().numpy(),
        fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]), cy=float(K[1, 2]),
        baseline=float(torch.tensor([c["baseline"]]).double().item()),
        init_pose=c["init_pose"].double().numpy(), **_typed_fields(c))


def _typed_fields(c: dict) -> dict:
    gt = c.get("graph_type", "disp")
    if gt != "icp":
        return {"graph_type": gt}
    from oracle import covariance as ocov
    pc = ocov.pixel2point_ned(c["kp2_uv"], c["kp2_d"], c["K"])           # fp32 like the registered buffer, then .double()
    return {"graph_type": gt, "pc_obs": pc.double().numpy(), "obs_cov": c["obs_cov"].double().numpy(),
            "pts_cov": c["pts_cov"].double().numpy()}


# ---- 640x480 / depth-12 network parity ladder (BASELINE configs[1] shape) -------------------------------------------
CFGA = (480, 640)


def cfgA_inputs() -> tuple[Tensor, Tensor]:
    """the `estimate_pair` batch of the bench sequence's first step: [t2.L, t1.L] vs [t2.R, t2.L] (Frontend.py:284-285)"""
    from macvo_b200 import synthetic
    fr = synthetic.make_sequence(2, *CFGA)
    return torch.cat([fr[1].imageL, fr[0].imageL]), torch.cat([fr[1].imageR, fr[1].imageL])


def cfgA_sample(name: str, t: Tensor) -> Tensor:
    """fixed strided samples of the per-stage tensors (keeps the fixture < 2 MB; same indices on both sides)"""
    if name in ("flow", "cov"):                 # (2,2,480,640) full-resolution outputs: stride 5, phase 2 (all 8x8 phases hit)
        return t[..., 2::5, 2::5]
    if name in ("feats", "context"):            # (B,256,60,80)
        return t[:, ::8, ::4, ::5]
    if name == "corr_rows":                     # (B, N/97, N) rows already strided by the tap
        return t[:, ::5, ::7]
    if name == "cost_memory":                   # (B*N, 8, 128)
        return t[::37, :, ::4]
    if name in ("flow_iter", "cov_iter"):       # (2,2,60,80) per iteration
        return t[..., ::2, ::2]
    raise KeyError(name)


# ---- trajectory post-process (MotionInterpolate) ----------------------------------------------------------------------
MOTION_CASES = {"f40": (40, 3, (1, 5, 6, 7, 15, 22, 23, 37, 38)), "f600": (600, 4, tuple(range(10, 590, 7)) + (300, 301, 302, 303)),
                "f5": (5, 5, (1, 2, 3)), "f3": (3, 6, (1,))}


def motion_inputs(F: int, seed: int, flagged: tuple) -> tuple[Tensor, Tensor]:
    """a random-walk trajectory (F,7) fp32 [t, q_xyzw] and the need_interp flags"""
    from oracle import pgo as opgo
    rng = np.random.default_rng(seed)
    poses = [np.array([0.3, -0.2, 0.1, 0, 0, 0, 1.0])]
    for _ in range(F - 1):
        step = np.concatenate([rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.05, 0.05, 3)])
        poses.append(opgo.se3_mul(poses[-1], opgo.se3_exp(step)))
    need = np.zeros(F, dtype=bool)
    need[list(flagged)] = True
    return torch.tensor(np.stack(poses), dtype=torch.float32), torch.tensor(need)


def golden_input_shas() -> dict:
    """file name -> sha256 of the inputs each golden file was generated from (recomputed on THIS host)"""
    out = {}
    for name, (B, H1, W1) in CORR_CASES.items():
        out[f"corr_{name}.pt"] = sha(*corr_inputs(B, H1, W1))
    for name, (B, H1, W1) in LOOKUP_CASES.items():
        out[f"lookup_{name}.pt"] = sha(*lookup_inputs(B, H1, W1))
    for name, (B, H, W) in NET_CASES.items():
        out[f"net_{name}.pt"] = sha(*net_inputs(B, H, W))
    out["net_fast_small.pt"] = sha(*net_inputs(*NET_CASES["small"]))
    for name, (H, W) in DENSE_CASES.items():
        for epd in (0, 1):
            out[f"dense_{name}_{epd}.pt"] = sha(*dense_inputs(H, W))
    for name, (H, W, _, variant) in SELECTOR_CASES.items():
        out[f"selector_{name}.pt"] = sha(*selector_inputs(H, W, variant))
    for name, (H, W, _, variant) in SELECTOR_DEPTH_CASES.items():
        (f0, c0), (f1, c1) = selector_depth_inputs(H, W, variant)
        out[f"selector_{name}.pt"] = sha(f0, c0, f1, c1)
    for name, (H, W, K, kind) in COV_CASES.items():
        out[f"covariance_{name}.pt"] = sha(*cov_inputs(H, W, K, kind))
    for name, (K, seed) in PGO_CASES.items():
        c = pgo_inputs(K, seed)
        out[f"pgo_{name}.pt"] = sha(*[c[k] for k in ("pos_Tw", "kp2_uv", "kp2_disp", "uv_cov", "disp_cov")])
    for name, (gt, K, seed) in PGO_TYPE_CASES.items():
        c = pgo_inputs_typed(gt, K, seed)
        out[f"pgo_{name}.pt"] = sha(*[c[k] for k in ("pos_Tw", "kp2_uv", "kp2_disp", "uv_cov", "disp_cov", "kp2_d", "obs_cov", "pts_cov")])
    for name, (F, seed, flagged) in MOTION_CASES.items():
        p, n = motion_inputs(F, seed, flagged)
        out[f"motion_{name}.pt"] = sha(p, n.to(torch.uint8))
    return out
