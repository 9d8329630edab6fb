"""B200_GaussianMixtureCovariance (GaussianMixtureCovariance, Module/Covariance/Project2to3.py:194-272): the standalone
kernel, macvo_observe_pack with cov_model "mixture", the plugin and the fused driver.

CPU: the fixture inputs regenerate bit for bit; oracle/mixture.py equals the reference class (tests/golden/mixture_*.pt,
tests/golden/make_golden_mixture.py); config handling; the plugin under the real Odometry/MACVO.py with tests/mock_ops.py
and the op answered by the oracle.
GPU: the kernel and observe_pack against the fixtures; the fused driver against TwoFrameOdometry.

Tolerance of a device covariance: per entry |device - reference| <= 1e-5 S, S = the entry recomputed in float64 with every
term in absolute value and the variance replaced by the mixture's second moment (oracle.mixture.mixture_bound). The
variance E[x^2] - mean^2 cancels: fp32 sums in another order differ by a few ulps of the second moment, which can be a
large part of the variance itself. NaN where the reference has NaN. Keep masks, counts and gathers: bit-exact.
"""
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import ablation as oab
from oracle import mixture as omix
from tests.golden import mixture_cases as mc
from tests.golden import observe_cases as oc
from tests.golden import refharness

DEV = "cuda"
NAN = float("nan")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
        "pixel1_uv", "pixel1_d")
EXACT = ("pixel2_uv", "pixel2_uv_cov", "pixel1_uv", "pixel2_d", "points_Tc")


def _bits(got, ref, what):
    torch.testing.assert_close(got, ref, rtol=0, atol=0, equal_nan=True, msg=lambda m: f"{what}: {m}")


def _within(got, ref, bound, what, rtol=1e-5):
    """same NaN pattern; |got - ref| <= rtol * bound where the reference is finite"""
    assert torch.equal(got.isnan(), ref.isnan()), f"{what}: NaN pattern differs"
    f = torch.isfinite(ref)
    if bool(f.any()):
        diff = (got - ref).abs()
        err = torch.where(diff == 0, 0.0, diff / bound)[f]           # (S is 0 where the entry is exactly 0)
        worst = err.max().item()
        assert worst <= rtol, f"{what}: {worst:.3g} of S (limit {rtol})"


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
def test_mixture_inputs_reproduce(golden):
    g = golden("mixture_standalone.pt")
    for case in mc.CASES:
        assert mc.input_sha(mc.inputs(case)) == g[case]["input_sha"], case
    for case in mc.OBSERVE_CASES:
        assert mc.ac.input_sha(mc.observe_inputs(case)) == golden(f"mixture_observe_{case}.pt")["input_sha"], case


@pytest.mark.parametrize("case", list(mc.CASES))
def test_oracle_matches_reference(golden, case):
    """the oracle's covariances, in-place clamp and bound S equal the reference fixture bit for bit"""
    g = golden("mixture_standalone.pt")[case]
    c = mc.inputs(case)
    kw = mc.oracle_call(c)
    _bits(omix.gaussian_mixture_covariance(**kw), g["cov"], case)
    if c["flow_cov"] is not None:
        _bits(kw["flow_cov"], g["flow_cov_clamped"], f"{case} clamped flow_cov")
        assert (kw["flow_cov"][:, :2] >= 0.0625).all()
        assert mc.CASES[case][3] == "narrow" or not torch.equal(kw["flow_cov"], c["flow_cov"]), "nothing was clamped"
    _bits(omix.mixture_bound(**mc.oracle_call(c)), g["bound"], f"{case} bound")
    if case == "k31_float_nan":
        assert all(bool(g["cov"][r].isnan().all()) for r in mc.NAN_ROWS)


@pytest.mark.parametrize("case", mc.OBSERVE_CASES)
def test_oracle_matches_reference_observe(golden, case):
    """keep mask, counts and gathers bit-exact; covariances bit-exact (Normalize: 1e-14 relative); bounds bit-exact"""
    g = golden(f"mixture_observe_{case}.pt")
    c = mc.observe_inputs(case)
    args, kw = oc.oracle_args(c)
    for model in mc.MODELS:
        ref, r = omix.observe_pack(*args, **kw, **mc.ext_kwargs(c, model)), g[model]
        assert torch.equal(ref["keep"], r["keep"]), model
        assert (ref["n_obs"], ref["n_inbound"], ref["k"]) == (r["n_obs"], g["n_inbound"], g["k"]), model
        for k in EXACT:
            _bits(ref[k].float() if k == "points_Tc" else ref[k], r[k], f"{model} {k}")
        for k in ("obs1_covTc", "obs2_covTc"):
            if model == "mixture_norm":
                torch.testing.assert_close(ref[k], r[k], rtol=1e-14, atol=0, equal_nan=True)
            else:
                _bits(ref[k], r[k], f"{model} {k}")
        _bits(ref["bound0"], r["bound0"], f"{model} bound0")
        _bits(ref["bound1"], r["bound1"], f"{model} bound1")
        err = ((ref["cov_Tw"] - r["cov_Tw"]).abs() / r["cov_Tw"].abs().amax(dim=(-1, -2), keepdim=True)).max().item()
        assert err <= 1e-12, (model, err)


def test_mixture_configs_validate():
    """the README's YAML with and without `device`, wrapped by either modifier; kernel_size 33, an even kernel_size and an
    unknown key are rejected; cov_spec names the model "mixture" with its kernel parameters"""
    from macvo_b200 import plugins as P
    for model in mc.MODELS:
        P.ICovariance2to3.is_valid_config(mc.model_config(model, "B200_"))
        P.ICovariance2to3.is_valid_config(mc.model_config(model, "B200_", DEV))
    for bad in (dict(kernel_size=33), dict(kernel_size=8), dict(extra=1), dict(device="cpu")):
        cfg = NS(type="B200_GaussianMixtureCovariance", args=NS(**dict(mc.REF_ARGS, **bad)))
        with pytest.raises((AssertionError, KeyError, ValueError)):
            P.ICovariance2to3.is_valid_config(cfg)
    with pytest.raises(KeyError):
        P.ICovariance2to3.is_valid_config(NS(type="B200_GaussianMixtureCovariance",
                                             args=NS(**{k: v for k, v in mc.REF_ARGS.items() if k != "min_depth_cov"})))
    P._require_cuda, keep = (lambda d, w: torch.device(d)), P._require_cuda
    try:
        for model, (_, ops) in mc.MODELS.items():
            cfg = mc.model_config(model, "B200_")
            base, got_ops, params = P.cov_spec(P.ICovariance2to3.instantiate(cfg.type, cfg.args))
            assert base.COV_MODEL == "mixture" and got_ops == ops, model
            assert params == {k: mc.REF_ARGS[k] for k in ("kernel_size", "min_flow_cov", "min_depth_cov")}
            assert base.device == torch.device("cuda")
    finally:
        P._require_cuda = keep


MACVO_CODE = r'''
import sys, os, torch
sys.path.insert(0, %r)
os.environ["TORCHDYNAMO_DISABLE"] = "1"
from tests.golden import refharness
refharness.install()
from types import SimpleNamespace as NS
import Module
from Odometry.MACVO import MACVO
from DataLoader import StereoFrame, StereoData
import pypose as pp
import macvo_b200.plugins as P
from macvo_b200 import synthetic
from macvo_b200.flowformer_cov import synthetic_state_dict
from tests.golden import mixture_cases as mc
torch.cuda.current_stream = lambda *a, **k: None
torch.save(synthetic_state_dict(0), sys.argv[1])
model = sys.argv[2]

def config(b200):
    t = (lambda n: "B200_" + n) if b200 else (lambda n: n)
    fe_args = NS(device="cpu", weight="synthetic:0" if b200 else sys.argv[1], enc_dtype="fp32", dec_dtype="fp32",
                 decoder_depth=4, enforce_positive_disparity=False)
    if b200:
        fe_args.cuda_graph = False
    return NS(Odometry=NS(name="t", args=NS(device="cpu", edgewidth=32, num_point=64, match_cov_default=0.25, profile=False, mapping=True),
        cov=NS(obs=mc.model_config(model, "B200_" if b200 else "", "cpu" if b200 else None)),
        keypoint=NS(type=t("CovAwareSelector_NoDepth"), args=NS(device="cpu", kernel_size=7, mask_width=32, max_match_cov=100.0)),
        mappoint=NS(type=t("MappingPointSelector"), args=(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32) if b200 else
                                                           NS(device="cpu", max_depth=5.0, max_depth_cov=0.005, mask_width=32))),
        frontend=NS(type=t("FlowFormerCovFrontend"), args=fe_args),
        motion=NS(type="StaticMotionModel", args=NS()), outlier=NS(type=t("CovarianceSanityFilter"), args=NS()),
        postprocess=NS(type=t("MotionInterpolate"), args=(NS(device="cpu") if b200 else NS())), keyframe=NS(type="AllKeyframe", args=NS()),
        optimizer=NS(type=t("TwoFrame_PGO"), args=NS(device="cpu", vectorize=True, parallel=False, graph_type="icp", autodiff=False))))

def run(b200):
    odo = MACVO[StereoFrame].from_config(config(b200))
    torch.set_float32_matmul_precision("highest")
    torch.manual_seed(5)
    for i, f in enumerate(synthetic.make_sequence(4, 192, 256)):
        sd = StereoData(T_BS=pp.identity_SE3(1), K=f.K, baseline=f.baseline, time_ns=f.time_ns, height=f.height,
                        width=f.width, imageL=f.imageL, imageR=f.imageR)
        odo.run(StereoFrame(idx=[i], time_ns=f.time_ns, stereo=sd))
    odo.terminate()
    m = odo.get_map()
    return (m.frames.data["pose"].tensor.clone(), len(m.match), len(m.points), m.match.data["pixel2_uv_cov"].tensor.clone(),
            m.match.data["obs2_covTc"].tensor.clone(), len(m.map_points), m.map_points.data["cov_Tw"].tensor.clone())

ref = run(False)
from tests import mock_ops
from oracle import ablation as oab
from oracle import mixture as omix
mock_ops.install()
calls = []

match = P.ops.match_covariance

def covariance(kp, depth_map, flow_cov, fx, fy, cx, cy, kernel_size=31, min_flow_cov=0.25, min_depth_cov=0.05,
               match_cov_default=0.25, want_point=False, depth_cov=None, out_cov=None, depth_cov_map=None):
    if depth_cov_map is None:
        return match(kp, depth_map, flow_cov, fx, fy, cx, cy, kernel_size, min_flow_cov, min_depth_cov, match_cov_default,
                     want_point, depth_cov, out_cov)
    calls.append(kp.shape[0])
    cov = omix.gaussian_mixture_covariance(kp, depth_map, depth_cov_map, flow_cov, fx, fy, cx, cy, kernel_size, min_flow_cov,
                                           match_cov_default, depth_cov=depth_cov)
    return cov, None, torch.zeros(1, dtype=torch.int32)
P.ops.match_covariance = covariance
P.ops.cov_modify = lambda cov, ops: cov.copy_(oab.modify(cov, ops))
got = run(True)
assert calls, "the B200 model did not reach the mixture op"
assert got[1] == ref[1] and got[2] == ref[2] and got[5] == ref[5] and got[1] > 100, (got[1:3], got[5], ref[1:3], ref[5])
assert torch.isfinite(got[0]).all()
torch.testing.assert_close(got[0], ref[0], rtol=1e-4, atol=1e-4)
# the B200 frontend's maps differ from the reference network's in the last bits, so everything downstream does too
torch.testing.assert_close(got[3], ref[3], rtol=1e-4, atol=1e-6)
assert (got[3][:, :2] >= 0.0625).all(), "pixel2_uv_cov must be clamped in place"
torch.testing.assert_close(got[4], ref[4], rtol=1e-3, atol=1e-9, equal_nan=True)
torch.testing.assert_close(got[6], ref[6], rtol=1e-3, atol=1e-9, equal_nan=True)
if model == "mixture_diag":
    assert (got[4][:, [0, 0, 1, 1, 2, 2], [1, 2, 0, 2, 0, 1]] == 0).all()
print("MIXTURE-MACVO-OK", got[1], got[2], got[5])
''' % REPO


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
@pytest.mark.parametrize("model", ["mixture", "mixture_diag"])
def test_b200_mixture_under_the_real_macvo(tmp_path, model):
    """the plain and the Diagonalize-wrapped B200 model through the real MACVO.run (icp graph, mapping on), the op answered
    by the oracle: the same observation and map-point counts as the reference classes, poses within 1e-4, pixel2_uv_cov
    clamped in place; the observation and map covariances within 1e-3 relative (the B200 frontend's maps, which feed
    them, differ from the reference network's by ~1e-5)"""
    r = subprocess.run([sys.executable, "-c", MACVO_CODE, str(tmp_path / "w.pth"), model], capture_output=True, text=True,
                       timeout=900, env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "MIXTURE-MACVO-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]


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


def _device_call(ops, c, flow_cov="copy", want_point=False):
    fc = c["flow_cov"].to(DEV) if (flow_cov == "copy" and c["flow_cov"] is not None) else (None if flow_cov == "copy" else flow_cov)
    fx, fy, cx, cy = c["intr"]
    out = ops.match_covariance(c["kp"].to(DEV), c["depth"].to(DEV), fc, fx, fy, cx, cy, kernel_size=c["kernel_size"],
                               want_point=want_point, depth_cov=None if c["depth_cov"] is None else c["depth_cov"].to(DEV),
                               depth_cov_map=c["depth_cov_map"].to(DEV), **mc.ARGS)
    return out, fc


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(mc.CASES))
def test_mixture_kernel_matches_reference(ops, golden, case):
    """every fixture case within 1e-5 S, the variant of the keypoint dtype proven by expect_variants; the flow covariance
    clamped in place like the reference's; the centre-pixel points as match_covariance gives them"""
    from tests.kernel_inventory import expect_variants
    g = golden("mixture_standalone.pt")[case]
    c = mc.inputs(case)
    # match_cov_kernel serves both models: a depth-variance map selects the mixture
    variant = "match_cov_kernel<long>" if c["kp"].dtype == torch.int64 else "match_cov_kernel<float>"
    (cov, pt, status), fc = expect_variants(lambda: _device_call(ops, c, want_point=True), variant)
    assert int(status.item()) == 0
    _within(cov.cpu(), g["cov"], g["bound"], case)
    if fc is not None:
        _bits(fc.cpu(), g["flow_cov_clamped"], f"{case} clamped flow_cov")
    fx, fy, cx, cy = c["intr"]
    _, pt_match, _ = ops.match_covariance(c["kp"].to(DEV), c["depth"].to(DEV), None, fx, fy, cx, cy, kernel_size=1,
                                          want_point=True)
    _bits(pt.cpu(), pt_match.cpu(), f"{case} points")


@pytest.mark.gpu
def test_mixture_threshold_applies(ops, golden):
    """narrow flow covariances: the 1e-3 threshold drops most of the patch; the kernel agrees with the thresholded
    reference and differs from the unthresholded mixture by more than the bound"""
    case = "k7_float_narrow"
    g = golden("mixture_standalone.pt")[case]
    c = mc.inputs(case)
    (cov, _, _), _ = _device_call(ops, c)
    cov = cov.cpu()
    _within(cov, g["cov"], g["bound"], case)
    plain = omix.gaussian_mixture_covariance(**mc.oracle_call(c, threshold=0.0))
    assert ((cov - plain).abs() / g["bound"]).amax().item() > 1e-3


@pytest.mark.gpu
def test_mixture_quirks(ops, golden):
    """the clamp lands in a transposed caller view; depth_cov replaces the variance without flow_cov; a NaN variance tap
    gives a NaN matrix; a patch past the bottom / right edge sets status bit 0 and the plugin raises IndexError"""
    from macvo_b200 import plugins as P
    c = mc.inputs("k31_long_flow")
    g = golden("mixture_standalone.pt")["k31_long_flow"]
    store = c["flow_cov"].T.contiguous().to(DEV)              # (3,K) storage, handed over as its (K,3) transposed view
    (cov, _, _), _ = _device_call(ops, c, flow_cov=store.T)
    _bits(store.T.cpu(), g["flow_cov_clamped"], "clamp through the transposed view")
    _within(cov.cpu(), g["cov"], g["bound"], "transposed view")

    c = mc.inputs("k29_long_override")
    (cov, _, _), _ = _device_call(ops, c)
    _bits(cov[:, 0, 0].cpu(), c["depth_cov"].double(), "zz = depth_cov")

    c = mc.inputs("k31_float_nan")
    (cov, _, _), _ = _device_call(ops, c)
    for r in mc.NAN_ROWS:
        assert bool(cov[r].isnan().all()), r

    c = mc.inputs("k7_long_none")
    kp = c["kp"].clone()
    kp[3] = torch.tensor([mc.W - 2, 10])                        # right edge
    kp[5] = torch.tensor([10, mc.H - 1])                        # bottom edge
    fx, fy, cx, cy = c["intr"]
    _, _, status = ops.match_covariance(kp.to(DEV), c["depth"].to(DEV), None, fx, fy, cx, cy, kernel_size=7,
                                       depth_cov_map=c["depth_cov_map"].to(DEV))
    assert int(status.item()) & 1 == 1
    model = P.B200_GaussianMixtureCovariance(NS(device=DEV, **dict(mc.REF_ARGS, kernel_size=7)))
    frame = NS(fx=fx, fy=fy, cx=cx, cy=cy)
    depth_est = NS(depth=c["depth"].to(DEV), cov=c["depth_cov_map"].to(DEV))
    with pytest.raises(IndexError):
        model.estimate(frame, kp.to(DEV), depth_est, None, None)
    out = model.estimate(frame, c["kp"].to(DEV), depth_est, None, None)
    assert out.device.type == "cpu" and out.dtype == torch.float64
    with pytest.raises(ValueError, match="depth covariance"):
        model.estimate(frame, c["kp"].to(DEV), NS(depth=depth_est.depth, cov=None), None, None)
    with pytest.raises(ops.MacvoB200Error, match="depth_cov_map"):       # one value per pixel
        ops.match_covariance(c["kp"].to(DEV), c["depth"].to(DEV), None, fx, fy, cx, cy, depth_cov_map=torch.ones(mc.K, device=DEV))


def _observe(ops, c, buf, ext):
    args, kw = oc.oracle_args(c)
    kp0, maps, (ew, i0, i1, prev) = args[0], args[1:7], args[7:]
    buf.packed.fill_(NAN)
    nxt = torch.full((7,), NAN, dtype=torch.float64, device=DEV)
    ops.observe_pack(buf, kp0.to(DEV), *(m.to(DEV) for m in maps), ew, i0, i1, prev.to(DEV), nxt, ext=ext, **kw)
    torch.cuda.synchronize()
    return nxt.cpu()


def _ext(c, model):
    cov_model, cov_ops = mc.MODELS[model]
    return {"depth_cov0": c["depth_cov0"].to(DEV), "depth_cov1": c["depth_cov1"].to(DEV), "simple_depth": True,
            "min_depth": c["min_depth"], "max_depth": c["max_depth"], "front_of_cam": True, "icp": True,
            "cov_model": cov_model, "cov_ops": cov_ops}


@pytest.mark.gpu
@pytest.mark.parametrize("case", mc.OBSERVE_CASES)
def test_observe_pack_mixture_matches_reference(ops, golden, case):
    """the mixture model with the Paper_Reproduce filter chain and the icp columns, plain and under each modifier: the
    fixture's kept rows and counts, its gathered columns bit-exact, the covariances within 1e-5 S (the modifiers: on the
    kernel's own mixture rows, Diagonalize bit-exact, Normalize 1e-14 x the condition number), cov_Tw = R obs1_covTc R^T"""
    from tests.test_ablation_backends import _device_rtol, _det_close
    g = golden(f"mixture_observe_{case}.pt")
    c = mc.observe_inputs(case)
    buf = ops.ObservationBuffers(c["kp0"].shape[0] + 1, DEV, extended=True)
    plain = None
    for model in mc.MODELS:
        r = g[model]
        nxt = _observe(ops, c, buf, _ext(c, model))
        n = r["n_obs"]
        hdr = buf.section("header").cpu().tolist()
        assert hdr[:3] == [n, g["n_inbound"], g["k"]] and hdr[3] == 0, (model, hdr)
        got = {k: buf.section(k)[:n].cpu() for k in ROWS + ("pixel2_d", "points_Tc", "cov_Tw")}
        for k in EXACT:
            _bits(got[k], r[k].double(), f"{model} {k}")
        if model == "mixture":
            plain = got
            _within(got["obs1_covTc"], r["obs1_covTc"], r["bound0"], f"{case} obs1_covTc")
            _within(got["obs2_covTc"], r["obs2_covTc"], r["bound1"], f"{case} obs2_covTc")
        else:
            for k in ("obs1_covTc", "obs2_covTc"):
                want = oab.modify(plain[k], mc.MODELS[model][1])
                if model == "mixture_diag":
                    _bits(got[k], want, f"{model} {k}")
                else:
                    _det_close(got[k], want, f"{model} {k}", _device_rtol(plain[k], "norm"))
        R = oab.ofil.quat_matrix_f32(nxt[3:7].float()).double().expand(n, 3, 3)
        want = torch.bmm(torch.bmm(R, got["obs1_covTc"]), R.transpose(1, 2))
        err = ((got["cov_Tw"] - want).abs() / want.abs().amax(dim=(-1, -2), keepdim=True)).max().item()
        assert err <= 1e-12, (model, err)
    ext = _ext(c, "mixture")
    ext["depth_cov1"] = None
    with pytest.raises(ops.MacvoB200Error, match="depth_cov"):
        _observe(ops, c, buf, ext)


class _MapFrontend:
    """seeded dense maps per frame (filter_cases.dense_frame_maps), uploaded once"""
    provide_cov = (True, True)

    def __init__(self, frames):
        from macvo_b200 import plugins as P
        from tests.golden import filter_cases as fc
        self.retrieve_pixels = staticmethod(P.B200_FlowFormerCovFrontend.retrieve_pixels)
        self.maps = []
        for i, f in enumerate(frames):
            m = fc.dense_frame_maps(f.height, f.width, seed=300 + i)
            self.maps.append((f, NS(depth=m["depth1"].to(DEV), cov=m["depth_cov1"].to(DEV), disparity=m["disparity1"].to(DEV),
                                    disparity_uncertainty=m["disp_unc1"].to(DEV), mask=None),
                              NS(flow=m["flow"].to(DEV), cov=m["match_cov"].to(DEV), mask=None)))

    def _get(self, frame):
        return next(x for x in self.maps if x[0] is frame)

    def estimate_depth(self, frame):
        return self._get(frame)[1]

    def estimate_pair(self, f0, f1):
        _, d, m = self._get(f1)
        return d, NS(flow=m.flow, cov=m.cov.clone(), mask=None)


def _driver(P, cls, frontend, model, **kw):
    from tests.golden import filter_cases as fc
    cfg = mc.model_config(model, "B200_", DEV)
    return cls(frontend,
               P.B200_CovAwareSelector(NS(device=DEV, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0,
                                          max_match_cov=100.0)),
               P.ICovariance2to3.instantiate(cfg.type, cfg.args),
               P.B200_TwoFrame_PGO(NS(graph_type="icp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
               num_point=200, mapping=True,
               map_selector=P.B200_MappingPointSelector(NS(max_depth=1e4, max_depth_cov=1e4, mask_width=32)),
               outlier_filter=P.B200_FilterCompose(NS(filter_args=[
                   NS(type="B200_CovarianceSanityFilter", args=None),
                   NS(type="B200_SimpleDepthFilter", args=NS(min_depth=fc.MIN_DEPTH, max_depth="auto")),
                   NS(type="B200_LikelyFrontOfCamFilter", args=None)])),
               keep_debug=True, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(mc.MODELS))
def test_fused_mixture_equals_plugin_api_path(ops, model):
    """the fused driver with mapping on against TwoFrameOdometry with the same plugins: keypoints bit-exact, equal counts,
    poses 1e-5, map covariances equal (the same kernel on the same inputs); pipelined runs bit-identical to sequential ones;
    one host wait per frame"""
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    frames = synthetic.make_sequence(6, 192, 256)
    a = _driver(P, TwoFrameOdometry, _MapFrontend(frames), model)
    est, map_covs = a.cov_model.estimate, []

    def recording(*args):
        out = est(*args)
        map_covs.append(out)
        return out
    a.cov_model.estimate = recording
    torch.manual_seed(5)
    a.initialize(frames[0])
    ra = [a.run_pair(f) for f in frames[1:]]
    pa = a.finish()
    runs = []
    for pipelined in (False, True):
        b = _driver(P, FusedTwoFrameOdometry, _MapFrontend(frames), model)
        torch.manual_seed(5)
        b.initialize(frames[0])
        obs = []
        for i in range(1, len(frames)):
            nxt = frames[i + 1] if pipelined and i + 1 < len(frames) and i != 3 else None
            b.run_pair(frames[i], next_frame=nxt)
            obs.append(b.observations())
        runs.append((obs, b.finish(), b.host_waits))
    (oa, pb, wa), (ob, pc, wb) = runs
    assert torch.equal(pb, pc)
    assert wa == wb == [1] * (len(frames) - 1)
    for x, y in zip(oa, ob):
        assert x["num_obs"] == y["num_obs"]
        for k in ROWS + ("map_cov", "map_pos_Tc"):
            assert torch.equal(x[k], y[k]), k
    for i, (o, r) in enumerate(zip(oa, ra)):
        keep = r.extras["keep"].cpu()
        assert o["num_kp"] == r.num_kp and o["num_obs"] == r.num_obs and r.num_obs >= 10
        assert torch.equal(o["pixel1_uv"].long(), r.kp0_uv.cpu()[keep]), "keypoints must be bit-exact"
        assert r.map_points == o["map_cov"].shape[0] > 0
        torch.testing.assert_close(o["map_cov"], map_covs[3 * i + 2], rtol=0, atol=0, equal_nan=True)
    np.testing.assert_allclose(pb.numpy(), pa.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_fused_mixture_refuses_a_frontend_without_depth_covariance(ops):
    from macvo_b200 import plugins as P
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    fe = P.B200_FlowFormerFrontend(NS(device=DEV, weight="synthetic:0", enc_dtype="fp32", dec_dtype="fp32", decoder_depth=4,
                                      enforce_positive_disparity=False, cuda_graph=False))
    with pytest.raises(ValueError, match="depth covariance"):
        _driver(P, FusedTwoFrameOdometry, fe, "mixture")
