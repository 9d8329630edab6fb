"""The Paper_Reproduce back end (CovAwareSelector, FilterCompose(CovarianceSanityFilter, SimpleDepthFilter,
LikelyFrontOfCamFilter), TwoFrame_PGO graph_type icp, TartanMotionNet) on the fused device path.

CPU: the filter inputs regenerate bit for bit; the B200 filter plugins equal the reference's masks
(tests/golden/filters_*.pt, tests/golden/make_golden_filters.py); the extended oracle (oracle/observe_filters.py) equals the
reference chain (tests/golden/observe_icp_*.pt, tests/golden/make_golden_observe_icp.py) and `TwoFrameOdometry` with the CPU
plugins.
GPU: the extended `macvo_observe_pack` against the oracle; the counted icp solve against oracle.pgo.lm_solve; the
CovAwareSelector split; the fused driver against `TwoFrameOdometry`. Tolerances:
  keep mask, counts, gathers (pixel2_d, pixel1_d_cov, pixel2_d_cov), points_Tc: bit-exact
  cov_Tw: 1e-12 relative to each matrix's largest entry, against R obs1_covTc R^T of the kernel's own obs1_covTc
  the other columns as tests/test_observe.py
"""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import frontend as ofe
from oracle import observe as oobs
from oracle import observe_filters as ofil
from oracle import pgo as opgo
from tests.golden import filter_cases as fc
from tests.golden import observe_cases as oc

DEV = "cuda"
NAN = float("nan")
ROWS = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
        "pixel1_uv", "pixel1_d")
EXT = ("pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc", "cov_Tw")
EXACT = ("pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "pixel1_uv", "pixel1_d",
         "pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc")


def _bits(got: torch.Tensor, ref: torch.Tensor, what: str) -> None:
    torch.testing.assert_close(got, ref, rtol=0, atol=0, equal_nan=True, msg=lambda m: f"{what}: {m}")


def _oracle(c: dict) -> dict:
    args, kw = oc.oracle_args(c)
    return ofil.observe_pack(*args, **kw, **fc.ext_kwargs(c))


def _cov_tw(prev_pose: torch.Tensor, obs1: torch.Tensor) -> torch.Tensor:
    R = ofil.quat_matrix_f32(prev_pose[3:7]).double().expand(obs1.shape[0], 3, 3)
    return torch.bmm(torch.bmm(R, obs1), R.transpose(1, 2))


def _filters(P, max_depth=fc.MAX_DEPTH):
    return P.B200_FilterCompose(NS(filter_args=[
        NS(type="B200_CovarianceSanityFilter", args=None),
        NS(type="B200_SimpleDepthFilter", args=NS(min_depth=fc.MIN_DEPTH, max_depth=max_depth)),
        NS(type="B200_LikelyFrontOfCamFilter", args=None)]))


@pytest.fixture(scope="module")
def plugins_cpu():
    from macvo_b200 import plugins
    return plugins


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(fc.BUNDLES))
def test_filter_inputs_reproduce(golden, name):
    assert fc.bundle_sha(fc.filter_bundle(name)) == golden(f"filters_{name}.pt")["input_sha"]


@pytest.mark.parametrize("name", list(fc.ICP_CASES))
def test_icp_inputs_reproduce(golden, name):
    assert fc.icp_sha(fc.icp_inputs(name)) == golden(f"observe_icp_{name}.pt")["input_sha"]


@pytest.mark.parametrize("name", list(fc.BUNDLES))
def test_filter_plugins_match_reference_masks(plugins_cpu, golden, name):
    """each B200 filter and the composed chain give the reference's mask, bit for bit, on the CPU bundle MACVO.py passes"""
    g = golden(f"filters_{name}.pt")
    b = fc.filter_bundle(name)
    from macvo_b200.pipeline import MatchBundle
    bundle = MatchBundle(b["data"])
    meta = NS(fx=float(torch.tensor([fc.AUTO_FX]).item()), frame_baseline=float(torch.tensor([fc.AUTO_BASELINE]).item()))
    P = plugins_cpu
    sd = P.B200_SimpleDepthFilter(NS(min_depth=b["min_depth"], max_depth=b["max_depth"]))
    sd.set_meta(meta)
    comp = _filters(P, b["max_depth"])
    comp.set_meta(meta)
    got = {"sanity": P.B200_CovarianceSanityFilter(NS()).filter(bundle, torch.device("cpu")),
           "simple_depth": sd.filter(bundle, torch.device("cpu")),
           "front_of_cam": P.B200_LikelyFrontOfCamFilter(NS()).filter(bundle, torch.device("cpu")),
           "compose": comp.filter(bundle, torch.device("cpu"))}
    for k, mask in got.items():
        assert mask.dtype == torch.bool and torch.equal(mask, g[k]), k
    assert 0 < int(g["compose"].sum()) < len(bundle)
    assert comp.required_keys == {"obs1_covTc", "obs2_covTc", "pixel1_d", "pixel2_d", "pixel1_d_cov", "pixel2_d_cov"}


def test_filter_conversion(plugins_cpu):
    """the fused driver's conversion: the chain's settings, fp32 thresholds, `auto` resolved by set_meta; a chain without
    the sanity filter or with a filter the device cannot run raises"""
    P = plugins_cpu
    comp = _filters(P, "auto")
    with pytest.raises(ValueError):
        P.observe_ext(comp)
    comp.set_meta(NS(fx=128.0, frame_baseline=0.25))
    assert P.observe_ext(comp) == {"simple_depth": True, "min_depth": fc.MIN_DEPTH, "max_depth": 32.0, "front_of_cam": True}
    assert P.observe_ext(P.B200_CovarianceSanityFilter(NS())) == {}
    assert P.observe_ext(None) is None
    with pytest.raises(ValueError):
        P.observe_ext(P.B200_LikelyFrontOfCamFilter(NS()))

    class Foreign(P.IObservationFilter):
        required_keys = set()

        def filter(self, values, device):
            return torch.ones(len(values), dtype=torch.bool)
    chain = P.B200_FilterCompose(NS(filter_args=[NS(type="B200_CovarianceSanityFilter", args=None),
                                                 NS(type="Foreign", args=None)]))
    with pytest.raises(ValueError):
        P.observe_ext(chain)


@pytest.mark.parametrize("name", list(fc.ICP_CASES))
def test_extended_oracle_matches_reference_chain(golden, name):
    """keep mask, counts, gathers and points_Tc bit-exact; cov_Tw 1e-12 relative; the default columns unchanged"""
    g = golden(f"observe_icp_{name}.pt")
    c = fc.icp_inputs(name)
    ref = _oracle(c)
    assert torch.equal(ref["keep"], g["keep"])
    assert (ref["n_obs"], ref["n_inbound"], ref["k"]) == (g["n_obs"], g["n_inbound"], g["k"])
    for k in ("pixel1_uv", "pixel2_uv", "pixel1_d", "pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc",
              "obs1_covTc", "obs2_covTc"):
        assert ref[k].dtype == g[k].dtype, k
        _bits(ref[k], g[k], k)
    err = ((ref["cov_Tw"] - g["cov_Tw"]).abs() / g["cov_Tw"].abs().amax(dim=(-1, -2), keepdim=True)).max().item()
    assert err <= 1e-12, err
    args, kw = oc.oracle_args(c)
    plain = oobs.observe_pack(*args, **kw)
    assert not any(k in plain for k in EXT)
    if name == "placeholder":        # the -1 placeholder switches LikelyFrontOfCamFilter off for the whole frame
        no_front = ofil.observe_pack(*args, **kw, **dict(fc.ext_kwargs(c), front_of_cam=False))
        assert torch.equal(no_front["keep"], ref["keep"])
    elif name != "nonfinite":       # there the sanity filter already drops the planted depth rows
        for drop in ("depth_range", "front_of_cam"):
            off = dict(fc.ext_kwargs(c), **{drop: None if drop == "depth_range" else False})
            assert int(ofil.observe_pack(*args, **kw, **off)["n_obs"]) > ref["n_obs"] > 0, drop


def test_extended_oracle_matches_plugin_api_driver(plugins_cpu):
    """TwoFrameOdometry with the CPU plugins, the B200 filter chain and an icp optimiser on one frame pair: the filtered
    rows and the icp inputs equal the extended oracle's"""
    from macvo_b200.pipeline import TwoFrameOdometry
    from oracle.pipeline_cpu import CpuCovariance
    c = fc.icp_inputs("basic")
    ref = _oracle(c)

    class Frontend:
        retrieve_pixels = staticmethod(lambda uv, m, interpolate=False: ofe.retrieve_pixels(uv, m))

        def estimate_depth(self, frame):
            return NS(depth=c["depth0"], cov=c["depth_cov0"], disparity=None, disparity_uncertainty=None)

        def estimate_pair(self, f0, f1):
            return (NS(depth=c["depth1"], cov=c["depth_cov1"], disparity=c["disparity1"], disparity_uncertainty=c["disp_unc1"]),
                    NS(flow=c["flow"], cov=c["match_cov"].clone(), mask=None))

    class Selector:
        def select_point(self, *a):
            return c["kp0"].clone()

    class Capture:
        context = {"graph_type": "icp"}

        def start_optimize(self, inp):
            self.inp = inp

    def frame(intr):
        fx, fy, cx, cy = intr
        return NS(width=c["W"], height=c["H"], fx=fx, fy=fy, cx=cx, cy=cy, frame_baseline=0.25,
                  frame_K=torch.tensor([[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]))
    opt = Capture()
    odo = TwoFrameOdometry(Frontend(), Selector(), CpuCovariance(c["kernel_size"], c["min_flow_cov"], c["min_depth_cov"],
                                                                 c["match_cov_default"]),
                           opt, num_point=c["kp0"].shape[0], edgewidth=c["edge_width"],
                           match_cov_default=c["match_cov_default"], mapping=False, min_num_point=1, keep_debug=True,
                           outlier_filter=_filters(plugins_cpu))
    odo.initialize(frame(c["intr0"]))
    odo.poses = [c["prev_pose"].float()]
    res = odo.run_pair(frame(c["intr1"]))
    assert (res.num_kp, res.num_obs) == (ref["n_inbound"], ref["n_obs"])
    keep = res.extras["keep"]
    _bits(res.kp0_uv[keep], ref["pixel1_uv"], "pixel1_uv")
    _bits(opt.inp.kp2_uv, ref["pixel2_uv"], "pixel2_uv")
    _bits(opt.inp.kp2_d.reshape(-1), ref["pixel2_d"], "pixel2_d")
    _bits(opt.inp.obs_cov, ref["obs2_covTc"], "obs2_covTc")
    _bits(opt.inp.pts_cov, ref["cov_Tw"], "cov_Tw")
    torch.testing.assert_close(opt.inp.pos_Tw, ref["pos_Tw"], rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from macvo_b200 import build, ops as _ops
    build.build(verbose=False)
    _ops.load_library()
    return _ops


def _ext(c: dict) -> dict:
    return {"depth_cov0": c["depth_cov0"].to(DEV), "depth_cov1": c["depth_cov1"].to(DEV), "simple_depth": True,
            "min_depth": c["min_depth"], "max_depth": c["max_depth"], "front_of_cam": True, "icp": True}


def _observe(ops, c: dict, buf):
    args, kw = oc.oracle_args(c)
    kp0, maps, (ew, i0, i1, prev) = args[0], args[1:7], args[7:]
    buf.packed.fill_(NAN)
    next_pose = torch.full((7,), NAN, dtype=torch.float64, device=DEV)
    ops.observe_pack(buf, kp0.to(DEV), *(m.to(DEV) for m in maps), ew, i0, i1, prev.to(DEV), next_pose, ext=_ext(c), **kw)
    torch.cuda.synchronize()
    return next_pose.cpu()


def _assert_matches(buf, next_pose, ref: dict, prev_pose: torch.Tensor) -> dict:
    n = ref["n_obs"]
    assert buf.section("header").cpu().tolist() == [n, ref["n_inbound"], ref["k"], ref["status"]]
    assert int(buf.n_obs.item()) == n and torch.equal(next_pose, ref["next_pose"])
    got = {k: buf.section(k)[:n].cpu() for k in ROWS + EXT}
    for k in EXACT:
        _bits(got[k], ref[k].double(), k)
    for k in ("obs1_covTc", "obs2_covTc"):
        err = ((got[k] - ref[k]).abs() / ref[k].abs().amax(dim=(-1, -2), keepdim=True)).max().item() if n else 0.0
        assert err <= 1e-5, (k, err)
    torch.testing.assert_close(got["pos_Tw"], ref["pos_Tw"].double(), rtol=1e-6, atol=1e-6)
    want = _cov_tw(prev_pose, got["obs1_covTc"])
    assert torch.isfinite(got["cov_Tw"]).all()
    if n:
        err = ((got["cov_Tw"] - want).abs() / want.abs().amax(dim=(-1, -2), keepdim=True)).max().item()
        assert err <= 1e-12, err
    # nothing is written past n_obs in any section, old or new
    for k in ROWS + EXT:
        tail = buf.section(k)[n:].cpu()
        _bits(tail, torch.full_like(tail, NAN), f"{k}[{n}:]")
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(fc.ICP_CASES))
def test_extended_observe_pack_matches_oracle(ops, name):
    """every case (filter edge rows, non-finite inputs, 2500 rows across 1024-record chunks, the -1 placeholder) on a
    NaN-poisoned buffer one row larger than needed"""
    c = fc.icp_inputs(name)
    ref = _oracle(c)
    buf = ops.ObservationBuffers(c["kp0"].shape[0] + 1, DEV, extended=True)
    assert buf.n_doubles == 46 * buf.capacity + 4
    nxt = _observe(ops, c, buf)
    _assert_matches(buf, nxt, ref, c["prev_pose"])


@pytest.mark.gpu
def test_filters_without_icp_columns(ops):
    """the filter chain on a plain buffer: same rows as the oracle, the plain layout; icp on a plain buffer is refused"""
    c = fc.icp_inputs("basic")
    args, kw = oc.oracle_args(c)
    ref = ofil.observe_pack(*args, **kw, **dict(fc.ext_kwargs(c), icp=False))
    buf = ops.ObservationBuffers(c["kp0"].shape[0], DEV)
    kp0, maps, (ew, i0, i1, prev) = args[0], args[1:7], args[7:]
    nxt = torch.empty((7,), dtype=torch.float64, device=DEV)
    ops.observe_pack(buf, kp0.to(DEV), *(m.to(DEV) for m in maps), ew, i0, i1, prev.to(DEV), nxt,
                     ext=dict(_ext(c), icp=False), **kw)
    n = int(buf.n_obs.item())
    assert n == ref["n_obs"] and buf.n_doubles == 31 * buf.capacity + 4
    _bits(buf.section("pixel1_uv")[:n].cpu(), ref["pixel1_uv"].double(), "pixel1_uv")
    with pytest.raises(ops.MacvoB200Error):
        ops.observe_pack(buf, kp0.to(DEV), *(m.to(DEV) for m in maps), ew, i0, i1, prev.to(DEV), nxt, ext=_ext(c), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [512, 2048])
def test_counted_icp_solve(ops, cap):
    """the counted LM with graph type icp on the kernel's own rows: pose within 1e-8 of oracle.pgo.lm_solve, same steps and
    evaluations for cluster sizes 0 (auto), 1, 2, 4; min_k above n_obs leaves the pose untouched"""
    c = fc.icp_solve_inputs(cap, seed=170 + cap)
    ref = _oracle(c)
    assert 0.4 * cap < ref["n_obs"] < 0.8 * cap
    buf = ops.ObservationBuffers(cap, DEV, extended=True)
    init = _observe(ops, c, buf)
    got = _assert_matches(buf, init, ref, c["prev_pose"])
    n = int(buf.n_obs.item())
    fx, fy, cx, cy = c["intr1"]
    bl = float(torch.tensor(c["baseline"], dtype=torch.float32))
    graph = opgo.GraphData(pos_Tw=got["pos_Tw"].numpy(), kp2_uv=got["pixel2_uv"].numpy(),
                           kp2_disp=got["pixel2_disp"].numpy(), uv_cov=got["pixel2_uv_cov"].numpy(),
                           disp_cov=got["pixel2_disp_cov"].numpy(), fx=fx, fy=fy, cx=cx, cy=cy, baseline=bl,
                           init_pose=init.numpy(), graph_type="icp", pc_obs=got["points_Tc"].numpy(),
                           obs_cov=got["obs2_covTc"].numpy(), pts_cov=got["cov_Tw"].numpy())
    trace = opgo.LMTrace()
    pose_ref = opgo.lm_solve(graph, trace=trace)
    truth = c["truth"].numpy()
    assert np.linalg.norm(pose_ref[:3] - truth[:3]) < 0.5 * np.linalg.norm(init.numpy()[:3] - truth[:3])
    for cluster in (0, 1, 2, 4):
        pose = init.to(DEV)
        stats = torch.zeros(8, dtype=torch.float64, device=DEV)
        ops.pgo_solve_counted(buf, (fx, fy, cx, cy, bl), pose, stats, min_k=10, cluster=cluster, graph_type="icp")
        p, s = pose.cpu().numpy(), stats.cpu().numpy()
        assert np.isfinite(p).all(), f"cluster {cluster}: a row past n_obs was read"
        np.testing.assert_allclose(p, pose_ref, rtol=1e-8, atol=1e-8, err_msg=f"cluster {cluster}")
        assert (int(s[0]), int(s[1]), s[6]) == (trace.steps, trace.evaluations, 0.0), f"cluster {cluster}"
    pose = init.to(DEV)
    stats = torch.zeros(8, dtype=torch.float64, device=DEV)
    ops.pgo_solve_counted(buf, (fx, fy, cx, cy, bl), pose, stats, min_k=n + 1, graph_type="icp")
    assert torch.equal(pose.cpu(), init) and stats[6].item() == 1.0
    with pytest.raises(ops.MacvoB200Error):
        ops.pgo_solve_counted(ops.ObservationBuffers(cap, DEV), (fx, fy, cx, cy, bl), pose, stats, graph_type="icp")


@pytest.mark.gpu
def test_selector_enqueue_then_sample_equals_select_point(ops):
    """B200_CovAwareSelector: enqueue_candidates + sample_candidates equals select_point bit for bit from the same randperm
    state; `max_depth: auto` resolved on the first call"""
    from macvo_b200 import plugins as P
    H, W = 192, 256
    maps = fc.dense_frame_maps(H, W, seed=7)
    depth0 = NS(depth=maps["depth0"].to(DEV), cov=maps["depth_cov0"].to(DEV), mask=None)
    depth1 = NS(depth=maps["depth1"].to(DEV), cov=maps["depth_cov1"].to(DEV), mask=None)
    match = NS(flow=maps["flow"].to(DEV), cov=maps["match_cov"].to(DEV), mask=None)
    frame = NS(fx=128.0, frame_baseline=0.25)
    cfg = lambda: NS(device=DEV, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0, max_match_cov=100.0)
    a, b = P.B200_CovAwareSelector(cfg()), P.B200_CovAwareSelector(cfg())
    torch.manual_seed(11)
    want = a.select_point(frame, 200, depth0, depth1, match).cpu()
    torch.manual_seed(11)
    with torch.inference_mode():           # the candidate list is an inference tensor, as in the fused driver
        got = ops.sample_candidates(b.enqueue_candidates(frame, depth0, depth1, match), 200).cpu()
    assert a.config.max_depth == b.config.max_depth == 32.0
    assert 0 < want.shape[0] and torch.equal(got, want)


def _paper_backend(P, cls, frontend, **kw):
    return cls(frontend,
               P.B200_CovAwareSelector(NS(device=DEV, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0,
                                          max_match_cov=100.0)),
               P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05,
                                         min_flow_cov=0.25)),
               P.B200_TwoFrame_PGO(NS(graph_type="icp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
               num_point=200, mapping=False, motion_model=P.B200_TartanMotionNet(NS(weight="synthetic", device=DEV)),
               outlier_filter=P.B200_FilterCompose(NS(filter_args=[
                   NS(type="B200_CovarianceSanityFilter", args=None),
                   NS(type="B200_SimpleDepthFilter", args=NS(min_depth=fc.MIN_DEPTH, max_depth="auto")),
                   NS(type="B200_LikelyFrontOfCamFilter", args=None)])),
               keep_debug=True, **kw)


class _MapFrontend:
    """stand-in frontend: seeded dense maps per frame (fc.dense_frame_maps), on the device; the depth maps and depth
    covariances are crafted so that every filter of the chain removes some rows but not all"""

    def __init__(self, frames):
        self.frames = frames
        from macvo_b200 import plugins as P
        self.retrieve_pixels = staticmethod(P.B200_FlowFormerCovFrontend.retrieve_pixels)

    def _depth(self, frame):
        index = next(i for i, f in enumerate(self.frames) if f is frame)
        m = fc.dense_frame_maps(frame.height, frame.width, seed=300 + index)
        return m, NS(depth=m["depth1"].to(DEV), cov=m["depth_cov1"].to(DEV), disparity=m["disparity1"].to(DEV),
                     disparity_uncertainty=m["disp_unc1"].to(DEV), mask=None)

    def estimate_depth(self, frame):
        return self._depth(frame)[1]

    def estimate_pair(self, f0, f1):
        m, d = self._depth(f1)
        return d, NS(flow=m["flow"].to(DEV), cov=m["match_cov"].to(DEV), mask=None)


@pytest.mark.gpu
def test_fused_paper_reproduce_equals_plugin_api_path(ops):
    """the fused driver (one host sync per frame) against TwoFrameOdometry with the same plugins, Paper_Reproduce back end
    and the synthetic B200_TartanMotionNet: keypoints bit-exact, equal counts, poses 1e-6 / 1e-5; every filter removes rows;
    pipelined runs bit-identical to sequential ones"""
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    frames = synthetic.make_sequence(6, 192, 256)
    a = _paper_backend(P, TwoFrameOdometry, _MapFrontend(frames))
    torch.manual_seed(5)
    a.initialize(frames[0])
    ra = [a.run_pair(f) for f in frames[1:]]
    pa = a.finish()
    runs = []
    for pipelined in (False, True):
        b = _paper_backend(P, FusedTwoFrameOdometry, _MapFrontend(frames))
        torch.manual_seed(5)
        b.initialize(frames[0])
        obs = []
        for i in range(1, len(frames)):
            nxt = frames[i + 1] if pipelined and i + 1 < len(frames) and i != 3 else None
            b.run_pair(frames[i], next_frame=nxt)
            obs.append(b.observations())
        runs.append((obs, b.finish()))
    (oa, pb), (ob, pc) = runs
    assert torch.equal(pb, pc)
    for x, y in zip(oa, ob):
        assert x["num_obs"] == y["num_obs"]
        for k in ROWS + EXT:
            assert torch.equal(x[k], y[k]), k
    for o, r in zip(oa, ra):
        keep = r.extras["keep"].cpu()
        assert o["num_kp"] == r.num_kp and o["num_obs"] == r.num_obs
        assert r.num_obs < r.num_kp and r.num_obs >= 10
        assert torch.equal(o["pixel1_uv"].long(), r.kp0_uv.cpu()[keep]), "keypoints must be bit-exact"
        assert torch.equal(o["pixel2_d"].float(), r.extras["kp1_d"].cpu()[keep])
    np.testing.assert_allclose(pb.numpy(), pa.numpy(), rtol=1e-5, atol=1e-6)
    # on every frame pair each depth filter removes rows and leaves some (the sanity filter keeps all on finite maps)
    for i, r in enumerate(ra, start=1):
        m0 = fc.dense_frame_maps(192, 256, seed=300 + i - 1)
        m1 = fc.dense_frame_maps(192, 256, seed=300 + i)
        kp0, kp1 = r.kp0_uv.cpu(), r.kp1_uv.cpu()
        d0, d1 = ofe.retrieve_pixels(kp0, m0["depth1"])[0], ofe.retrieve_pixels(kp1, m1["depth1"])[0]
        c0, c1 = ofe.retrieve_pixels(kp0, m0["depth_cov1"])[0], ofe.retrieve_pixels(kp1, m1["depth_cov1"])[0]
        depth_ok = ~((d0 < fc.MIN_DEPTH) | (d0 > 32.0) | (d1 < fc.MIN_DEPTH) | (d1 > 32.0))
        front_ok = ((d0 - c0.sqrt() * 2) > 0) & ((d1 - c1.sqrt() * 2) > 0)
        for what, ok in (("SimpleDepthFilter", depth_ok), ("LikelyFrontOfCamFilter", front_ok)):
            assert 0 < int(ok.sum()) < ok.numel(), (i, what)
        assert torch.equal(r.extras["keep"].cpu(), depth_ok & front_ok), i


@pytest.mark.gpu
def test_fused_driver_refuses_custom_solver_with_icp(ops):
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    frames = synthetic.make_sequence(2, 192, 256)
    with pytest.raises(ValueError):
        _paper_backend(P, FusedTwoFrameOdometry, _MapFrontend(frames), solver=lambda *a: None)
