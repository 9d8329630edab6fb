"""The back ends of the ablation configs (Config/Experiment/MACVO/Ablation_Study: CovDiag, ScaleNorm, NormDiag, CovKP, CovOpt):
B200_NoCovariance, B200_Modifier_Diagonalize / _Normalize, B200_RandomSelector, in the plugins and the fused driver.

CPU: the fixture inputs regenerate bit for bit; oracle/ablation.py equals the reference classes (tests/golden/ablation_*.pt,
tests/golden/make_golden_ablation.py); RandomSelector's draws; config handling; the plugins under the real Odometry/MACVO.py
with tests/mock_ops.py.
GPU: macvo_cov_modify and the extended macvo_observe_pack against the oracle; the counted icp solve; the fused driver against
TwoFrameOdometry. Tolerances:
  keep mask, counts, gathers, Diagonalize / NoCovariance covariances: bit-exact
  anything divided by a determinant: identical finite / NaN / +-Inf / zero pattern and sign; 1e-14 relative per element on
  the CPU (torch.det on both sides), 1e-14 times each matrix's condition number on the device (an LU of the same
  transposed matrix, other rounding)
"""
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import ablation as oab
from oracle import pgo as opgo
from tests.golden import ablation_cases as ac
from tests.golden import filter_cases as fc
from tests.golden import observe_cases as oc
from tests.golden import refharness

DEV = "cuda"
NAN = float("nan")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
        "pixel1_uv", "pixel1_d")
EXT = ("pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc", "cov_Tw")
EXACT = ("pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "pixel1_uv", "pixel1_d",
         "pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc")


def _bits(got, ref, what):
    torch.testing.assert_close(got, ref, rtol=0, atol=0, equal_nan=True, msg=lambda m: f"{what}: {m}")


def _classes(t: torch.Tensor) -> torch.Tensor:
    """0 finite non-zero, 1 zero, 2 NaN, 3 +Inf, 4 -Inf, times the sign bit of finite values"""
    c = torch.zeros_like(t, dtype=torch.int64)
    c[t == 0] = 1
    c[t.isnan()] = 2
    c[t == float("inf")] = 3
    c[t == -float("inf")] = 4
    return c * 2 + (torch.signbit(t) & torch.isfinite(t) & (t != 0)).long()


def _det_close(got, ref, what, rtol=1e-14):
    """same IEEE class and sign per element, finite values within rtol relative (a float, or one per matrix)"""
    assert torch.equal(_classes(got), _classes(ref)), what
    f = torch.isfinite(ref) & (ref != 0)
    if bool(f.any()):
        tol = torch.as_tensor(rtol, dtype=torch.float64).reshape(-1, 1, 1).expand_as(ref)
        err = (got - ref).abs() / ref.abs()
        worst = (err / tol)[f].max().item()
        assert worst <= 1.0, (what, err[f].max().item())


def _covs(got, ref, model, what, rtol=1e-14):
    if "norm" in model:
        _det_close(got, ref, what, rtol)
    else:
        _bits(got, ref, what)


def _device_rtol(inputs: torch.Tensor, model: str) -> torch.Tensor:
    """1e-14 times the condition number of each matrix the determinant is taken of: the device LU and CPU LAPACK round
    differently, and a determinant's relative error grows with the conditioning (up to 4e-12 measured on the observation
    covariances, which are far from isotropic)"""
    ops_ = ac.MODELS[model][1]
    m = oab.modify(inputs, ops_[:ops_.index("normalize")]) if "normalize" in ops_ else inputs
    ok = torch.isfinite(m).all(dim=(-1, -2))
    kappa = torch.ones(m.shape[0], dtype=torch.float64)
    if bool(ok.any()):
        kappa[ok] = torch.linalg.cond(m[ok]).nan_to_num(1.0, 1.0, 1.0)
    return 1e-14 * kappa.clamp(min=1.0)


def _oracle(c, model):
    args, kw = oc.oracle_args(c)
    return oab.observe_pack(*args, **kw, **ac.ext_kwargs(c, model))


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ac.CASES)
def test_ablation_inputs_reproduce(golden, case):
    assert ac.input_sha(ac.observe_inputs(case)) == golden(f"ablation_observe_{case}.pt")["input_sha"]


def test_modifier_inputs_reproduce(golden):
    assert ac.sha(ac.modifier_set()) == golden("ablation_modifiers.pt")["input_sha"]


@pytest.mark.parametrize("model", [m for m in ac.MODELS if m != "nocov"])
def test_oracle_modifiers_match_reference(golden, model):
    g = golden("ablation_modifiers.pt")
    got = oab.modify(g["input"], ac.MODELS[model][1])
    _covs(got, g[model], model, model)
    if model == "diag":          # a NaN / Inf off the diagonal disappears
        assert torch.isfinite(got).all(dim=(-1, -2)).sum() > torch.isfinite(g["input"]).all(dim=(-1, -2)).sum()


@pytest.mark.parametrize("case", ac.CASES)
def test_oracle_matches_reference_observe(golden, case):
    """keep mask, counts, gathers bit-exact; Diagonalize / NoCovariance covariances bit-identical, Normalize 1e-14; cov_Tw
    1e-12 relative; pixel2_uv_cov unclamped under NoCovariance"""
    g = golden(f"ablation_observe_{case}.pt")
    c = ac.observe_inputs(case)
    for model in ac.case_models(case):
        ref, r = _oracle(c, model), g[model]
        assert torch.equal(ref["keep"], r["keep"]), model
        assert (ref["n_obs"], ref["n_inbound"], ref["k"]) == (r["n_obs"], g["n_inbound"], g["k"]), model
        for k in ("pixel1_uv", "pixel2_uv", "pixel2_uv_cov", "pixel2_d", "points_Tc"):
            _bits(ref[k].float() if k == "points_Tc" else ref[k], r[k], f"{model} {k}")
        for k in ("obs1_covTc", "obs2_covTc"):
            _covs(ref[k], r[k], model, f"{model} {k}")
        if "cov_Tw" in r:
            err = ((ref["cov_Tw"] - r["cov_Tw"]).abs() / r["cov_Tw"].abs().amax(dim=(-1, -2), keepdim=True)).max().item()
            assert err <= 1e-12, (model, err)
        if model == "nocov":
            assert ref["status"] & 1 == 0 and not ref["unspecified"].any()
            assert (ref["pixel2_uv_cov"][:, :2] < 0.0625).any(), "NoCovariance must not clamp the flow covariance"
    if case == "planted":            # an indefinite flow covariance gives all-NaN Gaussian weights in the reference
        rows = {r for r in ac.PLANTED}
        for r in rows:
            assert g["planted_match"][r].isnan().all()
            assert not any(g[m]["sanity_keep"][r] for m in ac.MODELS if m != "nocov")
            assert g["nocov"]["sanity_keep"][r]          # (the depth filters may still drop it)


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_random_selector_matches_reference():
    code = r'''
import sys, torch
sys.path.insert(0, %r)
from tests.golden import refharness
refharness.install()
from types import SimpleNamespace as NS
from Module.KeypointSelector import RandomSelector
from oracle.ablation import random_selector
frame = NS(height=192, width=256)
torch.manual_seed(3)
ref = RandomSelector(NS(mask_width=32, device="cpu")).select_point(frame, 200, None, None, None)
torch.manual_seed(3)
got = random_selector(192, 256, 200, 32)
assert got.dtype == torch.int64 and got.shape == (200, 2) and torch.equal(got, ref)
assert (got[:, 0] >= 32).all() and (got[:, 0] < 224).all() and (got[:, 1] >= 32).all() and (got[:, 1] < 160).all()
print("RANDOM-OK")
''' % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "RANDOM-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_ablation_configs_validate():
    """cov.obs and keypoint of the five ablation YAMLs with B200_ names pass is_valid_config; a nested non-B200 model is
    rejected with a ValueError that names it"""
    from macvo_b200 import plugins as P
    for model in ac.MODELS:
        P.ICovariance2to3.is_valid_config(ac.model_config(model, "B200_", DEV))
    P.IKeypointSelector.is_valid_config(NS(type="B200_RandomSelector", args=NS(mask_width=32, device=DEV)))
    for t in ("MatchCovariance", "Foreign"):
        for wrapper in ("B200_Modifier_Diagonalize", "B200_Modifier_Normalize"):
            cfg = NS(type=wrapper, args=NS(type=t, args=NS(device=DEV, **ac.MATCH_ARGS)))
            with pytest.raises(ValueError, match=t):
                P.ICovariance2to3.is_valid_config(cfg)
            with pytest.raises(ValueError, match=t):
                P.ICovariance2to3.instantiate(cfg.type, cfg.args)
    P._require_cuda, keep = (lambda d, w: torch.device(d)), P._require_cuda
    try:
        for model, (cov_model, ops) in ac.MODELS.items():
            cfg = ac.model_config(model, "B200_", DEV)
            base, got_ops, params = P.cov_spec(P.ICovariance2to3.instantiate(cfg.type, cfg.args))
            assert got_ops == ops and (params is None) == (cov_model == "identity"), model
            assert params is None or params == {k: ac.MATCH_ARGS[k] for k in ("kernel_size", "min_flow_cov", "min_depth_cov")}
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
from tests.golden import ablation_cases as ac
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
        cov=NS(obs=ac.model_config(model, "B200_" if b200 else "", "cpu")),
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
            m.match.data["obs2_covTc"].tensor.clone())

ref = run(False)
from tests import mock_ops
from oracle import ablation as oab
mock_ops.install()
P.ops.cov_modify = lambda cov, ops: cov.copy_(oab.modify(cov, ops))
got = run(True)
assert got[1] == ref[1] and got[2] == ref[2] and got[1] > 100, (got[1:3], ref[1:3])
assert torch.isfinite(got[0]).all()
# Normalize makes each information matrix scale with det^2: on these synthetic frames the icp problem is poorly
# conditioned, and the two LM implementations (pypose's, oracle.pgo's stand-in for the kernel) part by ~2e-3 on one frame
tol = 5e-3 if model == "norm" else 1e-4
torch.testing.assert_close(got[0], ref[0], rtol=tol, atol=tol)
torch.testing.assert_close(got[3], ref[3], rtol=1e-4, atol=1e-6)
if model == "nocov":
    assert (got[3][:, :2] < 0.0625).any(), "NoCovariance: pixel2_uv_cov must hold the unclamped network values"
    assert torch.equal(got[4], torch.eye(3, dtype=torch.float64).expand_as(got[4]))
else:
    assert (got[3][:, :2] >= 0.0625).all()
    torch.testing.assert_close(got[4], ref[4], rtol=1e-3, atol=1e-9)
if model == "diag":
    assert (got[4][:, [0, 0, 1, 1, 2, 2], [1, 2, 0, 2, 0, 1]] == 0).all()
print("ABLATION-MACVO-OK", got[1], got[2])
''' % REPO


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
@pytest.mark.parametrize("model", ["diag", "norm", "nocov"])
def test_b200_covariance_models_under_the_real_macvo(tmp_path, model):
    """CovDiag-, ScaleNorm- and CovKP-shaped back ends (icp graph) through the real MACVO.run: same observation counts as
    the reference classes, poses within 1e-4, pixel2_uv_cov unclamped under NoCovariance"""
    r = subprocess.run([sys.executable, "-c", MACVO_CODE, str(tmp_path / "w.pth"), model], capture_output=True, text=True,
                       timeout=900, env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "ABLATION-MACVO-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]


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


@pytest.mark.gpu
@pytest.mark.parametrize("model", [m for m in ac.MODELS if m != "nocov"])
def test_cov_modify_matches_oracle(ops, model):
    """the adversarial set (zero row, negative det, NaN / +-Inf, det overflow / underflow) and 4096 random SPD matrices"""
    for covs in (ac.modifier_set(), ac.modifier_set(n_random=4096, seed=121)):
        want = oab.modify(covs, ac.MODELS[model][1])
        got = ops.cov_modify(covs.to(DEV).contiguous(), ac.MODELS[model][1]).cpu()
        _covs(got, want, model, model, _device_rtol(covs, model))
    with pytest.raises(ops.MacvoB200Error):
        ops.cov_modify(covs.to(DEV), ["transpose"])


def _observe(ops, c, buf, ext):
    args, kw = oc.oracle_args(c)
    kp0, maps, (ew, i0, i1, prev) = args[0], args[1:7], args[7:]
    buf.packed.fill_(NAN)
    nxt = torch.full((7,), NAN, dtype=torch.float64, device=DEV)
    ops.observe_pack(buf, kp0.to(DEV), *(m.to(DEV) for m in maps), ew, i0, i1, prev.to(DEV), nxt, ext=ext, **kw)
    torch.cuda.synchronize()
    return nxt.cpu()


def _device_ext(c, model, filters=True):
    cov_model, cov_ops = ac.MODELS[model]
    if not filters:
        return {"cov_model": cov_model, "cov_ops": cov_ops}
    return {"depth_cov0": c["depth_cov0"].to(DEV), "depth_cov1": c["depth_cov1"].to(DEV), "simple_depth": True,
            "min_depth": c["min_depth"], "max_depth": c["max_depth"], "front_of_cam": True, "icp": True,
            "cov_model": cov_model, "cov_ops": cov_ops}


def _assert_matches(buf, nxt, ref, model, ext=True, want_cov=None):
    n = ref["n_obs"]
    unspec = ref["unspecified"].any()
    hdr = buf.section("header").cpu().tolist()
    assert hdr[:3] == [n, ref["n_inbound"], ref["k"]] and hdr[3] == ref["status"], (model, hdr)
    assert torch.equal(nxt, ref["next_pose"])
    names = ROWS + (EXT if ext else ())
    got = {k: buf.section(k)[:n].cpu() for k in names}
    for k in EXACT:
        if k in got and not unspec:
            _bits(got[k], ref[k].double(), f"{model} {k}")
    for k in ("obs1_covTc", "obs2_covTc"):
        if model == "nocov":
            _bits(got[k], ref[k], f"{model} {k}")
        elif want_cov is False:        # (not compared)
            continue
        elif want_cov is not None:     # the modifiers on the kernel's own MatchCovariance output
            _covs(got[k], want_cov[k][0], model, f"{model} {k}", want_cov[k][1])
        else:       # the fp32 covariance kernel itself: 1e-5 of each matrix's largest entry (tests/test_observe.py)
            assert torch.equal(_classes(got[k]) // 2, _classes(ref[k]) // 2), (model, k)
            f = torch.isfinite(ref[k])
            scale = ref[k].abs().nan_to_num(0, 0, 0).amax(dim=(-1, -2), keepdim=True).expand_as(ref[k])
            if bool(f.any()):
                assert ((got[k] - ref[k]).abs()[f] / scale[f]).max().item() <= 1e-5, (model, k)
    torch.testing.assert_close(got["pos_Tw"], ref["pos_Tw"].double(), rtol=1e-6, atol=1e-6, equal_nan=True)
    if ext:
        R = oab.ofil.quat_matrix_f32(torch.tensor(ref["next_pose"][3:7])).double().expand(n, 3, 3)
        want = torch.bmm(torch.bmm(R, got["obs1_covTc"]), R.transpose(1, 2))
        f = torch.isfinite(want).all(dim=(-1, -2))
        if bool(f.any()):
            err = ((got["cov_Tw"] - want).abs() / want.abs().amax(dim=(-1, -2), keepdim=True))[f].max().item()
            assert err <= 1e-12, (model, err)
    for k in names:
        tail = buf.section(k)[n:].cpu()
        _bits(tail, torch.full_like(tail, NAN), f"{model} {k}[{n}:]")
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", ac.CASES)
def test_observe_pack_covariance_models_match_oracle(ops, case):
    """each covariance spec with the Paper_Reproduce filter chain and the icp columns, on every fixture case; status bit 0
    never set under NoCovariance; the planted indefinite rows dropped under every MatchCovariance-based model, kept under
    NoCovariance"""
    c = ac.observe_inputs(case)
    buf = ops.ObservationBuffers(c["kp0"].shape[0] + 1, DEV, extended=True)
    base = None
    if case != "boundary":           # the kernel's own MatchCovariance rows, which the modifiers act on
        ext = dict(_device_ext(c, "diag"), cov_model="match", cov_ops=[])
        _observe(ops, c, buf, ext)
        base_keep = oab.observe_pack(*oc.oracle_args(c)[0], **oc.oracle_args(c)[1], **dict(ac.ext_kwargs(c, "diag"),
                                                                                              cov_ops=[]))["keep"]
        n = int(base_keep.sum())
        base = (base_keep, {k: buf.section(k)[:n].cpu().clone() for k in ("obs1_covTc", "obs2_covTc")})
    for model in ac.case_models(case):
        ref = _oracle(c, model)
        nxt = _observe(ops, c, buf, _device_ext(c, model))
        want_cov = None
        if model != "nocov":
            base_keep, bc = base
            assert not bool((ref["keep"] & ~base_keep).any()), model
            sel = ref["keep"][base_keep]
            want_cov = {k: (oab.modify(v[sel], ac.MODELS[model][1]), _device_rtol(v[sel], model)) for k, v in bc.items()}
        got = _assert_matches(buf, nxt, ref, model, want_cov=want_cov)
        if model == "nocov":
            assert int(buf.section("header")[3].item()) & 1 == 0
            _bits(got["pixel2_uv_cov"], ref["pixel2_uv_cov"].double(), "unclamped uv cov")
        if case == "planted" and model != "nocov":
            assert not any(bool(ref["keep"][r]) for r in ac.PLANTED), model
    if case == "boundary":           # MatchCovariance there: status bit 0, as before
        _observe(ops, c, buf, _device_ext(c, "diag"))
        assert int(buf.section("header")[3].item()) & 1 == 1


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(ac.MODELS))
def test_covariance_fields_alone_keep_the_plain_layout(ops, model):
    """an ext with only the covariance fields: the 31c+4 layout, the sanity filter alone"""
    c = ac.observe_inputs("nonfinite")
    args, kw = oc.oracle_args(c)
    ref = oab.observe_pack(*args, **kw, cov_model=ac.MODELS[model][0], cov_ops=ac.MODELS[model][1])
    buf = ops.ObservationBuffers(c["kp0"].shape[0], DEV)
    assert buf.n_doubles == 31 * buf.capacity + 4
    plain = ops.ObservationBuffers(c["kp0"].shape[0], DEV)
    _observe(ops, c, plain, None)
    want_cov = None
    if model != "nocov":
        base_keep = oab.observe_pack(*args, **kw)["keep"]
        assert not bool((ref["keep"] & ~base_keep).any())
        sel = ref["keep"][base_keep]
        n = int(base_keep.sum())
        base = {k: plain.section(k)[:n].cpu()[sel] for k in ("obs1_covTc", "obs2_covTc")}
        want_cov = {k: (oab.modify(v, ac.MODELS[model][1]), _device_rtol(v, model)) for k, v in base.items()}
    nxt = _observe(ops, c, buf, _device_ext(c, model, filters=False))
    _assert_matches(buf, nxt, ref, model, ext=False, want_cov=want_cov)
    # the default spec through the same ext keeps today's bits
    _observe(ops, c, buf, {"cov_model": "match", "cov_ops": []})
    _bits(buf.packed.cpu(), plain.packed.cpu(), "match spec vs no ext")


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["nocov", "norm"])
def test_counted_icp_solve_ablation(ops, model):
    """the counted LM (graph icp) on the kernel's rows under NoCovariance and Normalize: pose within 1e-8 of
    oracle.pgo.lm_solve, same steps and evaluations"""
    c = fc.icp_solve_inputs(512, seed=682)
    ref = _oracle(c, model)
    assert ref["n_obs"] > 100
    buf = ops.ObservationBuffers(512, DEV, extended=True)
    init = _observe(ops, c, buf, _device_ext(c, model))
    got = _assert_matches(buf, init, ref, model, want_cov=False)      # (the covariances: test_observe_pack_covariance_...)
    fx, fy, cx, cy = c["intr1"]
    bl = float(torch.tensor(c["baseline"], dtype=torch.float32))
    graph = opgo.GraphData(pos_Tw=got["pos_Tw"].numpy(), kp2_uv=got["pixel2_uv"].numpy(),
                           kp2_disp=got["pixel2_disp"].numpy(), uv_cov=got["pixel2_uv_cov"].numpy(),
                           disp_cov=got["pixel2_disp_cov"].numpy(), fx=fx, fy=fy, cx=cx, cy=cy, baseline=bl,
                           init_pose=init.numpy(), graph_type="icp", pc_obs=got["points_Tc"].numpy(),
                           obs_cov=got["obs2_covTc"].numpy(), pts_cov=got["cov_Tw"].numpy())
    trace = opgo.LMTrace()
    pose_ref = opgo.lm_solve(graph, trace=trace)
    pose = init.to(DEV)
    stats = torch.zeros(8, dtype=torch.float64, device=DEV)
    ops.pgo_solve_counted(buf, (fx, fy, cx, cy, bl), pose, stats, min_k=10, graph_type="icp")
    p, s = pose.cpu().numpy(), stats.cpu().numpy()
    np.testing.assert_allclose(p, pose_ref, rtol=1e-8, atol=1e-8)
    assert (int(s[0]), int(s[1]), s[6]) == (trace.steps, trace.evaluations, 0.0)


BACKENDS = {"CovDiag": ("diag", False), "ScaleNorm": ("norm", False), "NormDiag": ("normdiag", False),
            "CovKP": ("nocov", False), "CovOpt": (None, True)}


def _backend(P, cls, frontend, name, motion=True, **kw):
    model, random = BACKENDS[name]
    cov_cfg = ac.model_config(model, "B200_", DEV) if model else NS(type="B200_MatchCovariance", args=NS(device=DEV, **ac.MATCH_ARGS))
    sel = (P.B200_RandomSelector(NS(mask_width=32, device=DEV)) if random else
           P.B200_CovAwareSelector(NS(device=DEV, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0,
                                      max_match_cov=100.0)))
    return cls(frontend, sel, P.ICovariance2to3.instantiate(cov_cfg.type, cov_cfg.args),
               P.B200_TwoFrame_PGO(NS(graph_type="icp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
               num_point=200, mapping=False,
               motion_model=P.B200_TartanMotionNet(NS(weight="synthetic", device=DEV)) if motion else None,
               outlier_filter=P.B200_FilterCompose(NS(filter_args=[
                   NS(type="B200_CovarianceSanityFilter", args=None),
                   NS(type="B200_SimpleDepthFilter", args=NS(min_depth=fc.MIN_DEPTH, max_depth="auto")),
                   NS(type="B200_LikelyFrontOfCamFilter", args=None)])),
               keep_debug=True, **kw)


class _MapFrontend:
    """seeded dense maps per frame (fc.dense_frame_maps), uploaded once: a frame's outputs are device tensors already"""

    def __init__(self, frames):
        from macvo_b200 import plugins as P
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
        return d, NS(flow=m.flow, cov=m.cov.clone(), mask=None)     # MatchCovariance clamps its gather, not the map


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BACKENDS))
def test_fused_ablation_equals_plugin_api_path(ops, name):
    """the fused driver against TwoFrameOdometry with the same plugins: keypoints bit-exact (CovOpt: the same CUDA-generator
    draws), equal counts, poses 1e-6 / 1e-5, pipelined runs bit-identical to sequential ones"""
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    frames = synthetic.make_sequence(6, 192, 256)
    a = _backend(P, TwoFrameOdometry, _MapFrontend(frames), name)
    torch.manual_seed(5)
    a.initialize(frames[0])
    ra = [a.run_pair(f) for f in frames[1:]]
    pa = a.finish()
    runs = []
    for pipelined in (False, True):
        b = _backend(P, FusedTwoFrameOdometry, _MapFrontend(frames), name)
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
    assert wa == wb == [0 if name == "CovOpt" else 1] * (len(frames) - 1)
    for x, y in zip(oa, ob):
        assert x["num_obs"] == y["num_obs"]
        for k in ROWS + EXT:
            assert torch.equal(x[k], y[k]), k
    for o, r in zip(oa, ra):
        keep = r.extras["keep"].cpu()
        assert o["num_kp"] == r.num_kp and o["num_obs"] == r.num_obs
        assert r.num_obs >= 10, name
        assert torch.equal(o["pixel1_uv"].long(), r.kp0_uv.cpu()[keep]), "keypoints must be bit-exact"
        if name == "CovKP":
            assert torch.equal(o["obs2_covTc"], torch.eye(3, dtype=torch.float64).expand_as(o["obs2_covTc"]))
    np.testing.assert_allclose(pb.numpy(), pa.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_covopt_fused_frame_has_no_host_wait(ops):
    """CovOpt with mapping off: 0 host waits per frame, and run_pair passes under torch's sync debug mode "error"; the
    keypoints are the reference's two randint draws from the device generator"""
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    frames = synthetic.make_sequence(5, 192, 256)
    b = _backend(P, FusedTwoFrameOdometry, _MapFrontend(frames), "CovOpt")
    torch.manual_seed(9)
    b.initialize(frames[0])
    b.run_pair(frames[1])                                # first frame: the motion model captures its CUDA graph
    torch.cuda.synchronize()
    state = torch.cuda.get_rng_state()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(2, len(frames)):
            b.run_pair(frames[i], next_frame=frames[i + 1] if i + 1 < len(frames) else None)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert b.host_waits == [0] * (len(frames) - 1)
    b.finish()
    torch.cuda.set_rng_state(state)
    for _ in range(2, len(frames)):
        want = oab.random_selector(192, 256, 200, 32, device=DEV)
    assert torch.equal(b.last.kp0_uv.cpu(), want.cpu())
    assert b.observations()["num_selected"] == 200
