"""The odometry tail `bench.py` times, pinned to the CPU oracle chain: `FusedTwoFrameOdometry` over the B200 plugins as
`build_gpu_pipeline` and `run_sharded` build them (the frontend's own fused post-processing and keypoint scores, TF32 and
matmul precision "medium" as the frontend sets them, CUDA graph, frames software-pipelined with `next_frame`), against
`TwoFrameOdometry` over the `oracle.pipeline_cpu` plugins under precision "highest".

Both drivers get the same raw network output from `BankNet`, a stand-in for FlowFormerCovNet that returns precomputed
(flow, cov) maps: each side then runs its own dense post-processing (`ops.dense_postproc` with fused scoring on the GPU,
`oracle.frontend.dense_postproc` on the CPU). The maps come from a known scene — a smooth depth surface seen by three
cameras with small planted motions — with NaN / inf depth pixels, flow that lands keypoints exactly on the in-bound
border, and exact ties in the flow quality planted in. Network numerics are tests/test_gpu_parity_ladder.py's."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

# the three workloads of bench.py: its CONFIGS "performant" / "fast" (build_gpu_pipeline) and SHARDED (run_sharded on one GPU)
WORKLOADS = {
    "performant": dict(H=480, W=640, enc_dtype="fp32", dec_dtype="fp32", num_point=200, kernel_size=7),
    "fast": dict(H=480, W=640, enc_dtype="fp16", dec_dtype="bf16", num_point=2048, kernel_size=7),
    "sharded": dict(H=720, W=1280, enc_dtype="fp32", dec_dtype="fp32", num_point=4096, kernel_size=3),
}
MODES = ("eager", "graph", "graph_prefetch")
ORDER = (0, 1, 2, 1, 0, 1, 2)       # ping-pong over three frames: initialize(frames[0]), then six pairs, both directions
BASELINE = 0.25
SEED = 5                            # torch.manual_seed of both drivers (bench.py's)


@pytest.fixture(autouse=True)
def _restore_precision_flags():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev[:2]
        torch.set_float32_matmul_precision(prev[2])


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    yield ops
    _DATA.clear(), _ORACLE.clear(), _GPU.clear()
    if _WORKER:
        _WORKER.pop().shutdown(wait=True)


# The GPU drivers run in one spawned worker process for the whole module. Run in the pytest process, the torch.profiler
# session around one whole frame (the first pair of each eager run) made the short launch probes of
# tests/kernel_inventory.py in later modules miss their first kernels on an H100; the worker keeps that state out of them.
_WORKER: list = []


def _worker():
    if not _WORKER:
        import multiprocessing as mp
        from concurrent.futures import ProcessPoolExecutor
        _WORKER.append(ProcessPoolExecutor(max_workers=1, mp_context=mp.get_context("spawn")))
    return _WORKER[0]


# ---- the scene ------------------------------------------------------------------------------------------------------
def _rot(q: np.ndarray) -> torch.Tensor:
    from oracle import pgo as opgo
    return torch.tensor(opgo.quat_matrix(q), dtype=torch.float64)


def _act(pose: np.ndarray, p: torch.Tensor) -> torch.Tensor:
    """pose (7,) [t, q_xyzw] applied to (..., 3) float64 points"""
    return p @ _rot(pose[3:]).T + torch.tensor(pose[:3], dtype=torch.float64)


def _planted_poses() -> list[np.ndarray]:
    """camera-to-world poses of frames 0, 1, 2 (pypose layout, the frame-0 camera is the world; NED: x forward)"""
    from oracle import pgo as opgo
    p1 = opgo.se3_exp(np.array([0.06, 0.015, -0.01, 0.004, -0.006, 0.003]))
    p2 = opgo.se3_mul(p1, opgo.se3_exp(np.array([0.05, -0.02, 0.012, -0.003, 0.005, -0.004])))
    return [np.array([0., 0., 0., 0., 0., 0., 1.]), p1, p2]


class Scene:
    """Pixel grids and the planted camera of an H x W TartanAir-shape frame (synthetic.camera)."""

    def __init__(self, H: int, W: int):
        self.H, self.W = H, W
        self.f = 320.0 * W / 640.0
        self.cx, self.cy = W / 2.0, H / 2.0
        self.bf = BASELINE * self.f
        v, u = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
        self.u, self.v = u, v

    def backproject(self, u, v, d):
        return torch.stack([d, (u - self.cx) / self.f * d, (v - self.cy) / self.f * d], dim=-1)

    def project(self, p):
        return self.f * p[..., 1] / p[..., 0] + self.cx, self.f * p[..., 2] / p[..., 0] + self.cy, p[..., 0]

    def sample(self, d0: torch.Tensor, u, v):
        """bilinear d0(u, v), clamped to the image"""
        g = torch.stack([2 * u / (self.W - 1) - 1, 2 * v / (self.H - 1) - 1], dim=-1)[None]
        return torch.nn.functional.grid_sample(d0[None, None], g, align_corners=True, padding_mode="border")[0, 0]

    def depth_seen_from(self, d0: torch.Tensor, pose: np.ndarray) -> torch.Tensor:
        """depth map of the camera at `pose` looking at the surface that camera 0 sees as d0: per pixel p, the surface point
        whose projection is p, found by fixed-point iteration (the motions are a few pixels)"""
        from oracle import pgo as opgo
        inv = opgo.se3_inv(pose)
        qu, qv = self.u.clone(), self.v.clone()
        for _ in range(12):
            pc = _act(inv, self.backproject(qu, qv, self.sample(d0, qu, qv)))
            pu, pv, z = self.project(pc)
            qu, qv = qu + (self.u - pu), qv + (self.v - pv)
        return z


def _lognormal(shape, g: torch.Generator, scale: float) -> torch.Tensor:
    """positive covariances, log-uniform over 2^-3 .. 2^4 (cases.dense_inputs' distribution)"""
    from tests.golden import cases
    return cases._lognormal_like(shape, g, scale)


def make_bank(H: int, W: int, seed: int = 11):
    """-> (stereo_flow (3,2,H,W), stereo_cov, pair_flow (9,2,H,W) indexed by 3 * t1 + t2, pair_cov, planted poses).

    slot-0 (stereo) maps of frame t: flow x = -bf / depth_t, the disparity variance log-normal; slot-1 (temporal) maps of the
    pair t1 -> t2: the projection of depth_t1 through pose_t2^-1 pose_t1, plus 0.05 px noise, log-normal covariances.
    Planted: disparity 0 (inf depth) and NaN disparity pixels, whose 31 x 31 depth patch poisons nearby keypoints'
    covariances (the sanity filter drops those); temporal flow that puts kp1 exactly on, just inside and just outside the
    32-pixel in-bound border; flow quality quantised to multiples of 1/4 in a band and constant in a block (exact ties in
    the NMS windows and in the median); a few NaN / inf flow covariances (NMS windows with a NaN)."""
    g = torch.Generator().manual_seed(seed + H + W)
    sc = Scene(H, W)
    coarse = torch.rand(1, 1, H // 40 + 2, W // 40 + 2, generator=g, dtype=torch.float64)
    smooth = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bicubic", align_corners=True)[0, 0].clamp(0, 1)
    d0 = 2.5 + 10.0 * smooth                                             # metres; near parts pass the 5 m mapping gate
    poses = _planted_poses()
    depth = [d0] + [sc.depth_seen_from(d0, p) for p in poses[1:]]
    n_bad = max(4, H * W // 20000)

    stereo_flow = torch.zeros(3, 2, H, W)
    stereo_cov = torch.zeros(3, 2, H, W)
    for t in range(3):
        fx = -sc.bf / depth[t] + 0.01 * torch.randn(H, W, generator=g, dtype=torch.float64)
        stereo_flow[t, 0] = fx.float()
        stereo_flow[t, 1] = (0.05 * torch.randn(H, W, generator=g)).float()
        flat = stereo_flow[t, 0].view(-1)
        idx = torch.randint(0, H * W, (2 * n_bad,), generator=g)
        flat[idx[:n_bad]] = 0.0                                          # disparity 0: depth inf
        flat[idx[n_bad:]] = float("nan")
        stereo_cov[t] = _lognormal((2, H, W), g, 1.0 / 16)

    pair_flow = torch.full((9, 2, H, W), float("nan"))
    pair_cov = torch.full((9, 2, H, W), float("nan"))
    e = 32                                                               # the driver's edgewidth
    step = torch.tensor([0.0, 0.5, -0.5])
    for t1, t2 in ((0, 1), (1, 2), (2, 1), (1, 0)):
        pc = _act(_rel(poses[t1], poses[t2]), sc.backproject(sc.u, sc.v, depth[t1]))
        pu, pv, _ = sc.project(pc)
        fl = torch.stack([pu - sc.u, pv - sc.v]) + 0.05 * torch.randn(2, H, W, generator=g, dtype=torch.float64)
        fl = fl.float()
        # kp1 = kp0 + flow exactly on (dropped), 0.5 px inside (kept) and 0.5 px outside (dropped) the strict in-bound test
        jitter = step[torch.arange(H) % 3].view(H, 1)
        xs, ys = torch.arange(W, dtype=torch.float32), torch.arange(H, dtype=torch.float32).view(H, 1)
        fl[0, :, e:2 * e] = (e - xs[e:2 * e]) + jitter
        fl[0, :, W - 2 * e:W - e] = (W - e - xs[W - 2 * e:W - e]) - jitter
        jitter_c = step[torch.arange(W) % 3].view(1, W)
        fl[1, e:2 * e, :] = (e - ys[e:2 * e]) + jitter_c
        fl[1, H - 2 * e:H - e, :] = (H - e - ys[H - 2 * e:H - e]) - jitter_c
        cov = _lognormal((2, H, W), g, 1.0)
        band = slice(H // 2, H // 2 + 48)
        cov[:, band] = (cov[:, band] * 4).round() / 4 + 0.25             # equal minima inside one NMS window
        cov[:, H // 3:H // 3 + 40, W // 3:W // 3 + 40] = 0.75            # a constant block: every pixel is its window minimum
        idx = torch.randint(0, H * W, (n_bad,), generator=g)
        cov[0].view(-1)[idx] = float("nan")
        cov[1].view(-1)[idx[: n_bad // 2] + 1] = float("inf")
        pair_flow[3 * t1 + t2], pair_cov[3 * t1 + t2] = fl, cov
    return stereo_flow, stereo_cov, pair_flow, pair_cov, poses


def _rel(pose1: np.ndarray, pose2: np.ndarray) -> np.ndarray:
    """camera-1-to-camera-2 transform: pose2^-1 pose1"""
    from oracle import pgo as opgo
    return opgo.se3_mul(opgo.se3_inv(pose2), pose1)


class BankNet:
    """Stand-in for FlowFormerCovNet.inference: the raw (flow, cov) of a precomputed bank, in the network's layout.

    A frame's tag is pixel (0, 0, 0) of its images (a small integer, exact in fp32). Rows are picked by index_select on the
    tags read from the input on its own device, so the call has no host synchronisation (it is captured in the frontend's
    CUDA graph) and both devices return the same bits. Batch 2 ([t2.L, t1.L] vs [t2.R, t2.L], estimate_pair): slot 0 = the
    stereo maps of t2, slot 1 = the flow t1 -> t2. Batch 1 (estimate_depth): the stereo maps."""

    def __init__(self, stereo_flow, stereo_cov, pair_flow, pair_cov):
        self.n = stereo_flow.shape[0]
        self.banks = {"cpu": (stereo_flow, stereo_cov, pair_flow, pair_cov)}

    def to(self, device: str) -> "BankNet":
        bank = tuple(t.to(device) for t in self.banks["cpu"])
        self.banks[str(bank[0].device)] = bank
        return self

    def inference(self, A: torch.Tensor, B: torch.Tensor, shared=None):
        sf, sc, pf, pc = self.banks[str(A.device)]
        ta, tb = A[:, 0, 0, 0].long(), B[:, 0, 0, 0].long()
        stereo = ta[:1]
        if A.shape[0] == 1:
            return sf.index_select(0, stereo), sc.index_select(0, stereo)
        pair = ta[1:2] * self.n + tb[1:2]
        return (torch.cat([sf.index_select(0, stereo), pf.index_select(0, pair)]),
                torch.cat([sc.index_select(0, stereo), pc.index_select(0, pair)]))


def make_frames(H: int, W: int, pin: bool):
    from macvo_b200 import synthetic
    from macvo_b200.interfaces import StereoData
    K, bl = synthetic.camera(H, W)
    frames = []
    for t in range(3):
        img = torch.full((1, 3, H, W), 0.5)
        img[0, 0, 0, 0] = float(t)
        left, right = img, img.clone()
        if pin:
            left, right = left.pin_memory(), right.pin_memory()
        frames.append(StereoData(T_BS=None, K=K.clone(), baseline=torch.tensor([bl]), time_ns=[t], height=H, width=W,
                                 imageL=left, imageR=right))
    return frames


_DATA: dict = {}


def workload_data(name: str, pin: bool = False):
    """(frames, BankNet, planted poses) of a workload, built once per process (pinned images in the GPU worker)"""
    if name not in _DATA:
        w = WORKLOADS[name]
        sf, sc, pf, pc, poses = make_bank(w["H"], w["W"])
        _DATA[name] = (make_frames(w["H"], w["W"], pin=pin), BankNet(sf, sc, pf, pc), poses)
    return _DATA[name]


def bank_sha(name: str) -> str:
    from tests.golden import cases
    return cases.sha(*workload_data(name)[1].banks["cpu"])


# ---- the CPU oracle chain --------------------------------------------------------------------------------------------
def run_oracle(name: str) -> dict:
    """TwoFrameOdometry over the pc.Cpu* plugins on the bank, precision "highest" (bench.run_cpu pins it): per frame the
    FrameResult, the oracle's own mapping points and their covariances / points from oracle.covariance; the trajectory."""
    from macvo_b200.flowformer_cov import synthetic_state_dict
    from macvo_b200.pipeline import TwoFrameOdometry
    from oracle import covariance as ocov
    from oracle import pipeline_cpu as pc
    w = WORKLOADS[name]
    frames, net, _ = workload_data(name)
    maps = []

    class RecordingMapSelector(pc.CpuMapSelector):
        def select_point(self, frame, numPoint, depth0, depth1, match):
            uv = super().select_point(frame, numPoint, depth0, depth1, match)
            maps.append((frame, depth0.depth, uv))
            return uv

    fe = pc.CpuFrontend(synthetic_state_dict(0), decoder_depth=1)
    fe.net = net
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        odo = TwoFrameOdometry(fe, pc.CpuSelector(kernel_size=w["kernel_size"]), pc.CpuCovariance(), pc.CpuPGO(),
                               num_point=w["num_point"], map_selector=RecordingMapSelector(), keep_debug=True)
        torch.manual_seed(SEED)
        odo.initialize(frames[ORDER[0]])
        results = [odo.run_pair(frames[t]) for t in ORDER[1:]]
        poses = odo.finish()
        map_ref = []
        for frame, depth0, uv in maps:
            cov = ocov.match_covariance(uv, depth0, None, frame.fx, frame.fy, frame.cx, frame.cy, 31, 0.25, 0.05, 0.25)
            d = depth0[0, 0, uv[:, 1], uv[:, 0]]
            pt = ocov.pixel2point_ned(uv.float(), d, frame.frame_K)
            map_ref.append((uv, cov, pt))
    finally:
        torch.set_float32_matmul_precision(prev)
    return {"results": results, "maps": map_ref, "poses": poses}


_ORACLE: dict = {}


def oracle(name: str) -> dict:
    if name not in _ORACLE:
        _ORACLE[name] = run_oracle(name)
    return _ORACLE[name]


# ---- the GPU driver as bench.py builds it ---------------------------------------------------------------------------
class _RecordingOps:
    """the driver's `ops` module with `sample_from_counts` recorded: the drawn keypoints and mapping points of each frame"""

    def __init__(self, ops):
        self._ops, self.picks = ops, []

    def __getattr__(self, name):
        return getattr(self._ops, name)

    def sample_from_counts(self, reqs):
        out = self._ops.sample_from_counts(reqs)
        self.picks.append(out)
        return out


def build_fused(name: str, cuda_graph: bool):
    """bench.build_gpu_pipeline / run_sharded with the plugin configs copied, and the network replaced by the bank"""
    from macvo_b200 import plugins as P
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    w = WORKLOADS[name]
    _, net, _ = workload_data(name)
    fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype=w["enc_dtype"], dec_dtype=w["dec_dtype"],
                                         decoder_depth=12, enforce_positive_disparity=False, cuda_graph=cuda_graph))
    fe.net = net.to(DEV)
    sel = P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=w["kernel_size"], mask_width=32, max_match_cov=100.0))
    msel = P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32))
    cov = P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25))
    pgo = P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False))
    odo = FusedTwoFrameOdometry(fe, sel, cov, pgo, num_point=w["num_point"], map_selector=msel, solver=None)
    odo.ops = _RecordingOps(odo.ops)
    return odo


def run_gpu(name: str, mode: str) -> dict:
    """one workload in one driving mode, in the GPU worker; the first pair of the eager run is launched under torch.profiler"""
    from macvo_b200 import build, ops
    from tests.kernel_inventory import launched
    build.build(verbose=False)
    ops.load_library()
    frames, _, _ = workload_data(name, pin=True)
    odo = build_fused(name, cuda_graph=mode != "eager")
    # the process flags the frontend left: the tail runs in them, as in bench.py
    assert torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32
    assert torch.get_float32_matmul_precision() == "medium"
    seq = [frames[t] for t in ORDER[1:]]
    torch.manual_seed(SEED)
    odo.initialize(frames[ORDER[0]])
    out = {"frames": [], "kernels": None, "bank_sha": bank_sha(name)}
    for i, f in enumerate(seq):
        nxt = seq[i + 1] if mode == "graph_prefetch" and i + 1 < len(seq) else None     # the last frame sequential
        if i == 0 and mode == "eager":
            n0 = odo.frame_no
            out["kernels"] = launched(lambda: odo.run_pair(f, next_frame=nxt))
            assert odo.frame_no == n0 + 1, "the profiled pair ran more than once"
        else:
            odo.run_pair(f, next_frame=nxt)
        o = odo.observations()
        o["map_uv"] = odo.ops.picks[-1][1].cpu()
        o["pose"] = odo.latest_pose()
        out["frames"].append(o)
    out["poses"] = odo.finish()
    return out


_GPU: dict = {}


def gpu_run(name: str, mode: str) -> dict:
    if (name, mode) not in _GPU:
        got = _worker().submit(run_gpu, name, mode).result()
        assert got["bank_sha"] == bank_sha(name), "the worker's bank differs from the oracle's"
        _GPU[(name, mode)] = got
    return _GPU[(name, mode)]


def _rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    """max over (K,3,3) matrices of |a - b| / max|b| of the matrix; inf unless the same matrices are non-finite (a mapping
    point's depth patch may hold a planted inf / NaN depth: no sanity filter runs on mapping points)"""
    fin = torch.isfinite(b).all(dim=(1, 2))
    if not torch.equal(torch.isfinite(a).all(dim=(1, 2)), fin):
        return float("inf")
    a, b = a[fin], b[fin]
    if b.numel() == 0:
        return 0.0
    return ((a - b).abs() / b.abs().amax(dim=(1, 2), keepdim=True)).amax().item()


def _same_bits(x, y) -> bool:
    """equal values, NaN where the other has NaN"""
    if not isinstance(x, torch.Tensor):
        return x == y
    return x.dtype == y.dtype and x.shape == y.shape and bool((x == y).logical_or(x.isnan() & y.isnan()).all())


# ---- the tests -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(WORKLOADS))
def test_bench_tail_matches_cpu_oracle(lib, name, mode):
    """Per frame: counts, keypoints and kp1 bit-exact, observation covariances 1e-5 of each matrix' scale, world points
    1e-6, mapping points bit-exact with covariances 1e-5 and points 1e-6; the trajectory 1e-5 rel / 1e-6 abs."""
    ref = oracle(name)
    got = gpu_run(name, mode)
    for i, (o, b, (map_uv, map_cov, map_pt)) in enumerate(zip(got["frames"], ref["results"], ref["maps"])):
        where = (name, mode, i)
        keep = b.extras["keep"]
        assert o["status"] == 0, where
        assert (o["num_kp"], o["num_obs"]) == (b.num_kp, b.num_obs), where
        assert b.num_obs < b.num_kp, "the planted non-finite depths must drop keypoints"
        assert torch.equal(o["pixel1_uv"].long(), b.kp0_uv[keep]), where                 # selection is integer / compare only
        assert torch.equal(o["pixel2_uv"].float(), b.kp1_uv[keep]), where                # one fp32 add, same operands
        # 31 x 31 fp32 Gaussian-weighted sums in a different order (warp reduction vs torch): ~1e-6 of the scale
        for col, ref_cov in (("obs1_covTc", b.extras["pos0_cov"][keep]), ("obs2_covTc", b.extras["pos1_cov"][keep])):
            assert _rel_err(o[col], ref_cov) < 1e-5, (where, col, _rel_err(o[col], ref_cov))
        # fp32 transform by the previous frame's pose, each side's own float64 LM result rounded to fp32 (the chain tests' 1e-6)
        torch.testing.assert_close(o["pos_Tw"].float(), b.extras["pos_Tw"], rtol=1e-6, atol=1e-6)
        assert b.map_points == len(map_uv) > 0 and o["map_cov"].shape[0] == b.map_points, where
        assert torch.equal(o["map_uv"], map_uv), where
        assert _rel_err(o["map_cov"], map_cov) < 1e-5, (where, _rel_err(o["map_cov"], map_cov))   # as obs covariances
        # pixel2point_NED: two fp32 roundings per coordinate in both
        torch.testing.assert_close(o["map_pos_Tc"], map_pt, rtol=1e-6, atol=1e-6)
    # the LM in float64 on both sides from bit-equal inputs up to the covariance rounding above; the chain tests' bound
    np.testing.assert_allclose(got["poses"].numpy(), ref["poses"].numpy(), rtol=1e-5, atol=1e-6)
    for o, p in zip(got["frames"], got["poses"][1:]):
        assert torch.equal(o["pose"].float(), p)                                          # latest_pose == the trajectory row


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_driving_modes_agree_bit_for_bit(lib, name):
    """eager, CUDA-graph and CUDA-graph + next_frame prefetch run the same kernels on the same maps: identical bits"""
    runs = [gpu_run(name, m) for m in MODES]
    base = runs[0]
    for mode, r in zip(MODES[1:], runs[1:]):
        assert torch.equal(r["poses"], base["poses"]), (name, mode)
        for i, (x, y) in enumerate(zip(base["frames"], r["frames"])):
            assert x.keys() == y.keys()
            for k, v in x.items():
                assert _same_bits(v, y[k]), (name, mode, i, k)


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_selector_score_source(lib, name):
    """The frontend's dense pass scores keypoints with its 7 x 7 NMS window; the selector takes those scores through the
    `_b200_score` token when its own kernel_size is 7 (performant, fast) and scores the map again with `score_only` when it
    is 3 (sharded). Counted in the kernels one eager pair launched: one dense_score_kernel (the frontend's) or two."""
    names = gpu_run(name, "eager")["kernels"]
    want = 2 if WORKLOADS[name]["kernel_size"] != 7 else 1
    assert names.count("dense_score_kernel") == want, (name, sorted(set(names)))
    assert names.count("flag_count_kernel<0>") == 1 and names.count("pgo_lm_kernel") == 1, sorted(set(names))


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_workload_recovers_planted_motion(lib, name):
    """The bank is a real two-view problem: the oracle's chained poses land near the planted ones (a check on the
    workload, not a tolerance on the kernels: 0.05 px flow noise, planted outliers and the Huber LM leave ~mm errors)."""
    from oracle import pgo as opgo
    _, _, planted = workload_data(name)
    poses = oracle(name)["poses"].double().numpy()
    for est, t in zip(poses, ORDER):
        err = opgo.se3_mul(opgo.se3_inv(planted[t]), est)
        assert np.linalg.norm(err[:3]) < 1e-2, (name, t, err)                     # 1 cm of a 5-10 cm motion
        assert 2 * np.arccos(min(1.0, abs(err[6]))) < 2e-3, (name, t, err)           # 0.1 degree
