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
# "ragged": not a multiple of the 32x8 tile in x or y, nor of the 1024-pixel chunk (75*102 % 1024 = 482). The per-pixel
# arithmetic does not depend on the frame size, so a small ragged shape stands in for the dataset frames here.
DENSE_CASES = {"small": (64, 96), "ragged": (75, 102)}


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
    # the shipped dataset frame sizes (EuRoC 752x480, KITTI 1241x376 and 1226x370) and a small shape ragged on all three
    # counts: W % 32, H % 8 and H*W % 1024 are all non-zero except where noted (EuRoC: H % 8 = 0, KITTI: H % 8 = 0)
    "euroc": (480, 752, 512, "plain"),
    "kitti": (376, 1241, 512, "plain"),
    "kitti00": (370, 1226, 512, "plain"),
    "kitti00_nan": (370, 1226, 128, "nan"),
    "ragged": (75, 102, 64, "plain"),
    "ragged_ties": (75, 102, 4096, "ties"),
}
# `mask_width` of the selectors (border excluded from selection); 32 unless listed. At the dataset sizes the last partial
# 1024-pixel chunk lies inside the last image row, which no mask width >= 1 lets through; the small ragged cases use 2
# so that selectable candidates fall into their last partial chunk (rows 70-74 of 75).
_SELECTOR_MASK_WIDTH = {"ragged": 2, "ragged_ties": 2, "depth_ragged": 2, "depth_ragged_ties": 2}


def selector_mask_width(name: str) -> int:
    return _SELECTOR_MASK_WIDTH.get(name, 32)


def _is_ragged(H: int, W: int) -> bool:
    return W % 32 != 0 or H % 8 != 0 or (H * W) % 1024 != 0


def selector_plantings(H: int, W: int) -> dict:
    """Pixels `selector_inputs` plants into a shape that does not fill the 32x8 scoring tiles / 1024-pixel compaction
    chunks (flat row-major indices, (y, x) = divmod(p, W)):
      edge_min    (H-1, W-1): the strict minimum of its 7x7 NMS window, which crosses the right and bottom edges;
      nan         (H-1, W-9): a NaN flow covariance in the last partial chunk, outside edge_min's window;
      candidates  pixels of row H-3 in the last partial chunk: strict window minima, below every unplanted quality and
                  with depth 2.5 / depth covariance 7.6e-4 (selectable by all three selectors for mask_width <= 2).
                  Empty where the last partial chunk does not reach row H-3 (the dataset sizes)."""
    chunk0 = (H * W) // 1024 * 1024
    cands = [(H - 3) * W + x for x in (8, W // 2, W - 20) if (H - 3) * W + x >= chunk0]
    return {"edge_min": H * W - 1, "nan": H * W - 9, "candidates": cands, "last_chunk": chunk0}


def _plant_ragged_edges(flow: Tensor, cov: Tensor, H: int, W: int) -> None:
    pl = selector_plantings(H, W)
    low = 2.0 ** -6                              # flow quality uu + vv = 2^-5 < 0.25, the least unplanted value
    for p in [pl["edge_min"]] + pl["candidates"]:
        y, x = divmod(p, W)
        cov[1, 0, y, x] = cov[1, 1, y, x] = low
        flow[0, 0, y, x] = -32.0                 # disparity 32 (> the 1..31 of the rest): depth 2.5, depth cov 6400/8 / 32^4
        cov[0, 0, y, x] = 0.125
    cov[1, 0].view(-1)[pl["nan"]] = float("nan")
    # the plantings hold on the inputs themselves, not by assumption
    q = cov[1, 0] + cov[1, 1]                    # flow quality uu + vv - 2 * 0 (the padded uv channel)
    dcov = cov[0, 0] / flow[0, 0] ** 4           # depth covariance / (baseline * fx)^2
    unplanted = torch.ones(H * W, dtype=torch.bool)
    unplanted[[pl["edge_min"]] + pl["candidates"]] = False
    assert pl["last_chunk"] < pl["nan"] < H * W and q.view(-1)[pl["nan"]].isnan()
    for p in [pl["edge_min"]] + pl["candidates"]:
        y, x = divmod(p, W)
        win = q[max(y - 3, 0):y + 4, max(x - 3, 0):x + 4]
        assert not win.isnan().any() and int((win <= q[y, x]).sum()) == 1, (y, x)
        assert q[y, x] < q.view(-1)[unplanted].nan_to_num(float("inf")).min()
        assert dcov[y, x] < dcov.view(-1)[unplanted].min()           # also the least depth covariance (depth-aware)
        assert p >= pl["last_chunk"]
    y, x = divmod(pl["edge_min"], W)
    assert y + 3 >= H and x + 3 >= W                                    # window crosses the bottom and right edges
    for p in pl["candidates"]:
        y, x = divmod(p, W)
        assert 2 <= x < W - 2 and 2 <= y < H - 2                        # inside a mask_width-2 border


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
    if _is_ragged(H, W):
        _plant_ragged_edges(flow, cov, H, W)
    return flow, cov


SELECTOR_DEPTH_CASES = {"depth_small": (160, 224, 64, "plain"), "depth_cfgA": (480, 640, 512, "plain"),
                        "depth_masked": (160, 224, 128, "masked"), "depth_nan": (160, 224, 128, "nan"),
                        "depth_euroc": (480, 752, 512, "plain"), "depth_kitti": (376, 1241, 512, "plain"),
                        "depth_kitti00": (370, 1226, 512, "plain"), "depth_kitti00_nan": (370, 1226, 128, "nan"),
                        "depth_ragged": (75, 102, 64, "plain"), "depth_ragged_ties": (75, 102, 4096, "ties")}


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


# focal length -> image size (W, H) of the MAC-VO-shaped icp inputs: TartanAir 640x480, KITTI 1241x376, a 1280x720 camera
PGO_MACVO_CAMERAS = {320.0: (640, 480), 718.0: (1241, 376), 1000.0: (1280, 720)}


def project2to3_cov(u, v, d, depth_var, var_u, var_v, var_uv, fx, fy, cx, cy) -> np.ndarray:
    """(K,3,3) float64 camera-frame (NED) covariance of a back-projected pixel: the Project2to3 formula of
    oracle.covariance.match_covariance, evaluated in float64"""
    s_xx = ((u - cx) ** 2 * depth_var + d ** 2 * var_u + var_u * depth_var) / fx ** 2
    s_yy = ((v - cy) ** 2 * depth_var + d ** 2 * var_v + var_v * depth_var) / fy ** 2
    s_xy = ((u - cx) * (v - cy) * depth_var + (d ** 2 + depth_var) * var_uv) / (fx * fy)
    s_xz, s_yz = depth_var * (u - cx) / fx, depth_var * (v - cy) / fy
    rows = [[depth_var, s_xz, s_yz], [s_xz, s_xx, s_xy], [s_yz, s_xy, s_yy]]
    return np.stack([np.stack(r, -1) for r in rows], -2)


def pgo_inputs_macvo(K: int, seed: int, fx: float) -> dict:
    """icp inputs whose covariances look like MAC-VO's: obs_cov / pts_cov are the Project2to3 covariances of the same point
    seen in frame 2 and in frame 1 (= world), long thin ellipsoids along the viewing ray. Pixels cover the image and a
    quarter sit within 1.5 % of a corner; depth 1 - 80 m and depth variance 0.05 - 1e5 log-uniform; flow variance at the
    0.0625 clamp for half the pixels, up to 25 for the rest, a quarter correlated in u / v. Layout as `pgo_inputs_typed`."""
    from oracle import pgo as opgo
    rng = np.random.default_rng(seed * 15485863 + K + int(fx))
    W, H = PGO_MACVO_CAMERAS[fx]
    fy, cx, cy = fx, W / 2.0, H / 2.0
    true_pose = opgo.se3_exp(np.array([0.15, -0.05, 0.05, 0.02, -0.03, 0.02]))
    u, v = rng.uniform(0, W - 1, K), rng.uniform(0, H - 1, K)
    corner = rng.uniform(size=K) < 0.25
    n = int(corner.sum())
    u[corner] = np.where(rng.uniform(size=n) < 0.5, 0.0, W - 1) + rng.uniform(-0.015, 0.015, n) * W
    v[corner] = np.where(rng.uniform(size=n) < 0.5, 0.0, H - 1) + rng.uniform(-0.015, 0.015, n) * H
    u, v = np.clip(u, 0, W - 1), np.clip(v, 0, H - 1)
    d2 = np.exp(rng.uniform(np.log(1.0), np.log(80.0), K))
    pc2 = np.stack([d2, (u - cx) / fx * d2, (v - cy) / fy * d2], -1)            # frame-2 camera, NED (x forward)
    pw = opgo.se3_act(true_pose, pc2)                                            # frame 1 = world
    u1, v1 = fx * pw[:, 1] / pw[:, 0] + cx, fy * pw[:, 2] / pw[:, 0] + cy

    def flow_var():
        vu, vv = np.full(K, 0.0625), np.full(K, 0.0625)
        above = rng.uniform(size=K) < 0.5
        vu[above] = np.exp(rng.uniform(np.log(0.0625), np.log(25.0), int(above.sum())))
        vv[above] = np.exp(rng.uniform(np.log(0.0625), np.log(25.0), int(above.sum())))
        rho = np.where(rng.uniform(size=K) < 0.25, rng.uniform(-0.5, 0.5, K), 0.0)
        return vu, vv, rho * np.sqrt(vu * vv)

    depth_var = lambda: np.exp(rng.uniform(np.log(0.05), np.log(1e5), K))
    obs_cov = project2to3_cov(u, v, d2, depth_var(), *flow_var(), fx, fy, cx, cy)
    pts_cov = project2to3_cov(u1, v1, pw[:, 0], depth_var(), *flow_var(), fx, fy, cx, cy)
    # observations: 1 % depth noise, 0.3 px pixel noise, 5 % gross outliers
    kp2_uv = np.stack([u, v], -1) + rng.normal(size=(K, 2)) * 0.3
    kp2_d = d2 * (1 + rng.normal(size=K) * 0.01)
    out = rng.uniform(size=K) < 0.05
    kp2_uv[out] += rng.uniform(5, 30, (int(out.sum()), 2))
    f32 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)
    return {
        "pos_Tw": f32(pw), "kp2_uv": f32(kp2_uv), "kp2_disp": f32(fx * 0.25 / kp2_d), "uv_cov": f32(np.tile([0.0625, 0.0625, 0.0], (K, 1))),
        "disp_cov": f32(np.full(K, 0.1)), "K": torch.tensor([[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]), "baseline": 0.25,
        "init_pose": torch.tensor([0., 0., 0., 0., 0., 0., 1.]), "true_pose": torch.tensor(true_pose),
        "kp2_d": f32(kp2_d), "obs_cov": torch.tensor(obs_cov), "pts_cov": torch.tensor(pts_cov), "graph_type": "icp",
    }


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


# ---- sharpened checkpoint -----------------------------------------------------------------------------------------------
# `synthetic_state_dict(0)` draws every weight from U(+-1/sqrt(fan_in)): its attention logits have a std of 0.02 - 0.6
# and every softmax of the frontend is close to uniform, so the network's output is close to the mean of the values and
# an error in how the network calls its attention kernels (scale, key / value pairing, position terms) shrinks by one to
# two orders of magnitude before it reaches the flow. The sharpened checkpoint multiplies the query and key projections
# (weight and bias rows) of every softmax family by a power of two, which is exact in fp32 and under tf32 / fp16
# rounding. Gains per family: (query gain, key gain); the mask families scale the 576-channel logit convolution itself.
# Chosen by tests/golden/make_golden_sharp.py::calibrate for a median logit std in [2, 4] per family (float64, 640x480,
# decoder_depth 3); the GRU gates are not scaled (saturated gates only lower the sensitivity and raise the fp32 noise).
SHARP_GAINS = {"svt_local": (8.0, 4.0), "svt_global": (8.0, 4.0), "perceiver_input": (8.0, 4.0), "latent": (4.0, 2.0),
               "vert_local": (4.0, 4.0), "vert_global": (4.0, 2.0), "cross_attend": (2.0, 2.0), "gma": (16.0, 8.0),
               "mask_flow": 64.0, "mask_cov": 64.0}
# the median logit std every family of the sharpened checkpoint reaches (make_golden_sharp.py asserts it per fixture)
SHARP_TARGET = (2.0, 4.0)


def sharp_rows() -> dict[str, list[tuple[int, int, str, int]]]:
    """checkpoint key -> [(first row, end row, family, 0 = query gain / 1 = key gain), ...] of every scaled tensor"""
    out: dict[str, list[tuple[int, int, str, int]]] = {}

    def add(key: str, lo: int, hi: int, fam: str, which: int) -> None:
        for t in ("weight", "bias"):
            out.setdefault(f"{key}.{t}", []).append((lo, hi, fam, which))
    for enc in ("memory_encoder.feat_encoder", "context_encoder"):
        for s, C in enumerate((128, 256)):
            b = f"{enc}.svt.blocks.{s}."
            add(b + "0.attn.qkv", 0, C, "svt_local", 0)                  # rows [q | k | v]
            add(b + "0.attn.qkv", C, 2 * C, "svt_local", 1)
            add(b + "1.attn.q", 0, C, "svt_global", 0)
            add(b + "1.attn.kv", 0, C, "svt_global", 1)                   # rows [k | v]
    c = "memory_encoder.cost_perceiver_encoder."
    layers = [(c + "input_layer.", "perceiver_input")] + [(c + f"encoder_layers.{i}.", "latent") for i in range(3)]
    for i in range(3):
        layers += [(c + f"vertical_encoder_layers.{i}.local_block.attn.", "vert_local"),
                   (c + f"vertical_encoder_layers.{i}.global_block.attn.", "vert_global")]
    layers += [("memory_decoder.decoder_layer.cross_attend.", "cross_attend")]
    for p, fam in layers:
        add(p + "q", 0, 128 if fam != "cross_attend" else 64, fam, 0)
        add(p + "k", 0, 128 if fam != "cross_attend" else 64, fam, 1)
    out["memory_decoder.att.to_qk.weight"] = [(0, 128, "gma", 0), (128, 256, "gma", 1)]    # no bias
    for p, fam in (("memory_decoder.update_block.", "mask_flow"), ("memory_decoder.cov_update.", "mask_cov")):
        add(p + "mask.2", 0, 576, fam, 0)
    return out


def sharp_gain(gains: dict, fam: str, which: int) -> float:
    g = gains[fam]
    return float(g) if not isinstance(g, tuple) else float(g[which])


def sharp_state_dict(gains: dict | None = None) -> dict[str, Tensor]:
    """`synthetic_state_dict(0)` with the query / key rows of every softmax family times its power-of-two gain
    (`SHARP_GAINS`, or `gains` during calibration)"""
    from macvo_b200.flowformer_cov import synthetic_state_dict
    gains = SHARP_GAINS if gains is None else gains
    sd = synthetic_state_dict(0)
    for key, rows in sharp_rows().items():
        t = sd[key].clone()
        for lo, hi, fam, which in rows:
            t[lo:hi] *= sharp_gain(gains, fam, which)
        sd[key] = t
    return sd


def ladder_state_dict(weights: str) -> dict[str, Tensor]:
    """the checkpoint a parity fixture records in its `weights` entry: "synthetic:<seed>" or "sharp:0" """
    kind, seed = weights.split(":")
    if kind == "synthetic":
        from macvo_b200.flowformer_cov import synthetic_state_dict
        return synthetic_state_dict(int(seed))
    if kind == "sharp" and seed == "0":
        return sharp_state_dict()
    raise ValueError(f"unknown weights {weights!r}")


# ---- depth-12 network parity ladder: 640x480 (BASELINE configs[1] shape) and the shipped dataset frame sizes ----------
# (H, W) of the frame. cfgA and TartanAir share 640x480; EuRoC is 752x480 (1/8 grid 60x94); KITTI is 1241x376 (padded
# to 1248x376, 1/8 grid 47x156) and 1226x370 for sequences 00-02 (padded to 1232x376, 1/8 grid 47x154). The sharp cases
# run the sharpened checkpoint (`LADDER_WEIGHTS`) on the cfgA and kitti00 frames.
LADDER_CASES = {"cfgA": (480, 640), "euroc": (480, 752), "kitti": (376, 1241), "kitti00": (370, 1226),
                "sharp": (480, 640), "sharp_kitti00": (370, 1226)}
LADDER_WEIGHTS = {"sharp": "sharp:0", "sharp_kitti00": "sharp:0"}       # every other case: "synthetic:0"
# strided samples of each stage, the same indices on both sides of the comparison: full-resolution pixel stride (phase
# 2; 5 and 21 are coprime with 8, so every 8x8 upsampling phase is sampled), feature (channel, row, column) strides,
# correlation (tapped row, column) strides, cost-memory (row, channel) strides and the 1/8-grid iterate stride. Coarser at
# the dataset sizes, so that each of their fixtures stays under 0.5 MB.
_DATASET_SAMPLE = {"px": 21, "feat": (32, 8, 14), "corr": (10, 35), "mem": (388, 8), "iter": 6}
_LADDER_SAMPLES = {"cfgA": {"px": 5, "feat": (8, 4, 5), "corr": (5, 7), "mem": (37, 4), "iter": 2},
                   "euroc": _DATASET_SAMPLE, "kitti": _DATASET_SAMPLE, "kitti00": _DATASET_SAMPLE,
                   "sharp": _DATASET_SAMPLE, "sharp_kitti00": _DATASET_SAMPLE}


def ladder_inputs(case: str = "cfgA") -> tuple[Tensor, Tensor]:
    """the `estimate_pair` batch of the bench sequence's first step: [t2.L, t1.L] vs [t2.R, t2.L] (Frontend.py:284-285)"""
    from macvo_b200 import synthetic
    fr = synthetic.make_sequence(2, *LADDER_CASES[case])
    return torch.cat([fr[1].imageL, fr[0].imageL]), torch.cat([fr[1].imageR, fr[1].imageL])


def ladder_sample(case: str, name: str, t: Tensor) -> Tensor:
    """fixed strided samples of the per-stage tensors (`_LADDER_SAMPLES`)"""
    s = _LADDER_SAMPLES[case]
    if name in ("flow", "cov"):                 # (2,2,H,W) full-resolution outputs
        return t[..., 2::s["px"], 2::s["px"]]
    if name in ("feats", "context"):            # (B,256,H1,W1)
        c, r, w = s["feat"]
        return t[:, ::c, ::r, ::w]
    if name == "corr_rows":                     # (B, N/97, N) rows already strided by the tap
        r, w = s["corr"]
        return t[:, ::r, ::w]
    if name == "cost_memory":                   # (B*N, 8, 128)
        r, c = s["mem"]
        return t[::r, :, ::c]
    if name in ("flow_iter", "cov_iter"):       # (2,2,H1,W1) per iteration
        return t[..., ::s["iter"], ::s["iter"]]
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
