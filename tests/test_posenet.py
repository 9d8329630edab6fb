"""B200_TartanMotionNet: the TartanVO pose network (input builder, macvo_posenet_conv, head / composition kernel), its
plugin and its place in the drivers, against the oracle (oracle/posenet.py) and the reference fixtures
(tests/golden/posenet_*.pt, written by tests/golden/make_golden_posenet.py from the MAC-VO tree itself)."""
import os
import tempfile
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.golden import posenet_cases

DEV = "cuda"
CASES = list(posenet_cases.CASES)


def _case(golden, name):
    return golden(f"posenet_{name}.pt"), posenet_cases.posenet_inputs(name)


def _deviation(got: torch.Tensor, ref: torch.Tensor) -> float:
    """max |got - ref| over ref's scale; NaN where the reference has NaN (a zero-depth tap reaches the network as +inf,
    as in the reference) is required, not measured"""
    got, ref = got.double().cpu(), ref.double().cpu()
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), (got, ref)
    fin = ~torch.isnan(ref)
    if not fin.any():
        return 0.0
    return ((got[fin] - ref[fin]).abs().max() / ref[fin].abs().max()).item()


def _oracle_input(c):
    from oracle import posenet as opn
    return opn.network_input(c["flow"], c["depth"], c["H"], c["W"], c["fx"], c["fy"], c["cx"], c["cy"], c["baseline"])


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_fixture_inputs_reproduce(golden, name):
    g, c = _case(golden, name)
    assert posenet_cases.sha(c["flow"], c["depth"]) == g["input_sha"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_fixture(golden, name):
    """input builder bit for bit (same CPU torch operations as the reference), the network + composition within fp32
    reassociation noise (the oracle evaluates the two fc1 heads / block sums in its own order)"""
    from macvo_b200.posenet import synthetic_posenet_state_dict
    from oracle import posenet as opn
    g, c = _case(golden, name)
    inp = _oracle_input(c)
    assert torch.equal(torch.nan_to_num(inp, posinf=1.0), torch.nan_to_num(g["net_input"], posinf=1.0))
    assert torch.equal(torch.isinf(inp), torch.isinf(g["net_input"]))
    motion = opn.motion(opn.forward(synthetic_posenet_state_dict(g["seed"]), inp)["pose"])
    assert _deviation(motion, g["motion"]) <= 1e-5
    nxt = opn.compose(c["prev_pose"], g["motion"])
    torch.testing.assert_close(nxt, g["next_pose"], rtol=0, atol=1e-6, equal_nan=True)


def test_synthetic_weights_give_a_live_network():
    """finite, non-zero motion that follows the flow: 25 residual blocks neither blow up nor die under ReLU"""
    from macvo_b200.posenet import synthetic_posenet_state_dict
    from oracle import posenet as opn
    sd = synthetic_posenet_state_dict(0)
    c = posenet_cases.posenet_inputs("480x640")
    out = opn.forward(sd, _oracle_input(c))
    m0 = opn.motion(out["pose"])
    assert torch.isfinite(m0).all() and m0.abs().min() > 0
    assert (out["fc1"] > 0).float().mean() > 0.1
    c["flow"] = c["flow"] + 3.0
    m1 = opn.motion(opn.forward(sd, _oracle_input(c))["pose"])
    assert (m1 - m0).abs().max() > 1e-3 * m0.abs().max()


def test_config_validation():
    from macvo_b200 import plugins as P
    cls = P.B200_TartanMotionNet
    cls.is_valid_config(NS(weight="synthetic:0", device="cuda"))
    with pytest.raises(Exception):
        cls.is_valid_config(NS(weight="synthetic:0", device="cuda", noise_std=0.1))     # unknown key
    with pytest.raises(Exception):
        cls.is_valid_config(NS(weight="synthetic:0", device="cpu"))
    with pytest.raises(ValueError):
        cls(NS(weight="synthetic:0", device="cpu"))
    from macvo_b200.posenet import synthetic_posenet_state_dict
    sd = {"module.flowPoseNet." + k: v for k, v in synthetic_posenet_state_dict(0).items()}
    sd["module.flowNet.conv1.weight"] = torch.zeros(1)                                 # other StereoVONet parts: ignored
    del sd["module.flowPoseNet.layer4.3.conv2.bias"]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "posenet.pkl")
        torch.save(sd, path)
        with pytest.raises(KeyError, match="layer4.3.conv2.bias"):
            cls(NS(weight=path, device="cuda:0"))


def test_checkpoint_keeps_only_pose_network_tensors():
    from macvo_b200.posenet import load_checkpoint, synthetic_posenet_state_dict
    ref = synthetic_posenet_state_dict(3)
    sd = {"module.flowPoseNet." + k: v for k, v in ref.items()}
    sd["module.flowNet.conv1.weight"] = torch.zeros(1)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "posenet.pkl")
        torch.save(sd, path)
        got = load_checkpoint(path)
    assert set(got) == set(ref) and all(torch.equal(got[k], ref[k]) for k in ref)


def test_posenet_symbols_exported():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    import ctypes
    lib = ctypes.CDLL(build.LIB_PATH)
    for name in ("macvo_posenet_input", "macvo_posenet_conv", "macvo_posenet_head", "macvo_posenet_head_floats"):
        assert name in ops.EXPORTS and hasattr(lib, name)
    assert ops.posenet_head_floats() == 2 * (32 * 128 + 32) + 2 * (3 * 32 + 3) + 6


def test_weight_slabs_are_contiguous_per_cta():
    from macvo_b200 import ops
    w = torch.randn(256, 128, 3, 3)
    packed, ct = ops.pack_posenet_conv(w)
    kc = 128 // 8 * 9
    tile, split = 5, 3
    slab = packed[(tile * 8 + split) * ct * kc:(tile * 8 + split + 1) * ct * kc].reshape(ct, kc)
    ref = w[tile * ct:(tile + 1) * ct].reshape(ct, 128 * 9)[:, split * kc:(split + 1) * kc]
    assert ct == 8 and torch.equal(slab, ref)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    return ops


def _strict_fp32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")


def _frame(c):
    K = torch.tensor([[[c["fx"], 0.0, c["cx"]], [0.0, c["fy"], c["cy"]], [0.0, 0.0, 1.0]]])
    return NS(height=c["H"], width=c["W"], fx=c["fx"], fy=c["fy"], cx=c["cx"], cy=c["cy"], frame_baseline=c["baseline"], K=K)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_input_builder_matches_reference(lib, golden, name):
    """channels 0..2 from macvo_posenet_input and channels 3..4 from the plugin's intrinsics layer vs the reference's network
    input: within 1e-6 of each channel's scale; positions the reference maps to 0 / inf (non-finite, zero, negative depth
    taps) exactly"""
    from macvo_b200 import posenet
    g, c = _case(golden, name)
    ref = g["net_input"][0]
    out = torch.full((1, 5, 112, 160), float("nan"), device=DEV)
    lib.posenet_input(c["flow"].to(DEV), c["depth"].to(DEV), c["baseline"] * c["fx"], out)
    out[:, 3:5] = posenet.intrinsic_layer(c["H"], c["W"], c["fx"], c["fy"], c["cx"], c["cy"], DEV)
    got = out[0].cpu()
    for ch in range(5):
        r, o = ref[ch], got[ch]
        exact = ~torch.isfinite(r) | (r == 0)
        assert torch.equal(o[exact], r[exact]), f"channel {ch}: special positions differ"
        fin = ~exact
        scale = r[fin].abs().max().item()
        err = (o[fin] - r[fin]).abs().max().item()
        assert err <= 1e-6 * scale, f"channel {ch}: {err / scale:.3g} of its scale"
    if name == "nonfinite":
        assert (ref[2] == 0).sum() > 0        # NaN / -inf / negative taps -> 0
    if name == "zerodepth":
        assert torch.isinf(ref[2]).sum() >= 4  # a zero bilinear depth overflows back to +inf after the final division


def _conv_shapes():
    """(cin, hi, wi, cout, k, stride, pad) of every distinct macvo_posenet_conv layer of the network (+ fc1)"""
    return [(128, 14, 20, 128, 3, 2, 1), (128, 14, 20, 128, 1, 2, 0), (128, 7, 10, 128, 3, 1, 1),
            (128, 7, 10, 256, 3, 2, 1), (128, 7, 10, 256, 1, 2, 0), (256, 4, 5, 256, 3, 1, 1),
            (256, 4, 5, 256, 3, 2, 1), (256, 4, 5, 256, 1, 2, 0), (256, 2, 3, 256, 3, 1, 1), (1536, 1, 1, 256, 1, 1, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", _conv_shapes(), ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("epilogue", ["bias", "relu", "resid_relu", "resid"])
def test_gpu_posenet_conv_matches_float64(lib, shape, epilogue):
    cin, hi, wi, cout, k, stride, pad = shape
    g = torch.Generator().manual_seed(cin + hi + cout + k + stride)
    x = torch.randn(1, cin, hi, wi, generator=g).relu()
    w = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=pad)
    resid = torch.randn(ref.shape, generator=g) if "resid" in epilogue else None
    if resid is not None:
        ref = ref + resid.double()
    if "relu" in epilogue:
        ref = ref.relu()
    packed, ct = lib.pack_posenet_conv(w)
    run = lambda: lib.posenet_conv(x.to(DEV), packed.to(DEV), ct, b.to(DEV), k, stride, pad,
                                   resid=resid.to(DEV) if resid is not None else None, relu="relu" in epilogue)
    y1, y2 = run(), run()
    assert torch.equal(y1, y2), "not bit-identical across launches"
    scale = ref.abs().max().item()
    err = (y1.double().cpu() - ref).abs().max().item()
    assert err <= 1e-6 * scale, f"{err / scale:.3g} of the output scale"


@pytest.mark.gpu
def test_gpu_head_matches_shim(lib):
    """fc2 / fc3 / pose_norm and prev @ se3(motion).Exp() on the device vs float64 evaluation with the pypose shim"""
    from macvo_b200.posenet import PoseNet, synthetic_posenet_state_dict
    from oracle import posenet as opn
    sd = synthetic_posenet_state_dict(1)
    net = PoseNet(sd, DEV)
    g = torch.Generator().manual_seed(7)
    prev = posenet_cases.PREV_POSE.double()
    for scale in (1.0, 30.0, 1e-4):          # small- and large-angle Exp branches around the typical motion
        fc1 = (torch.randn(256, generator=g) * scale).relu()
        motion = torch.empty(6, device=DEV)
        nxt = torch.empty(7, dtype=torch.float64, device=DEV)
        lib.posenet_head(fc1.to(DEV), net.head_blob, prev.to(DEV), motion, nxt)
        sd64 = {k: v.double() for k, v in sd.items()}
        m_ref = []
        for i, head in enumerate(("trans", "rot")):
            h = F.relu(F.linear(fc1.double()[128 * i:128 * (i + 1)], sd64[f"voflow_{head}.1.0.weight"], sd64[f"voflow_{head}.1.0.bias"]))
            m_ref.append(F.linear(h, sd64[f"voflow_{head}.2.weight"], sd64[f"voflow_{head}.2.bias"]))
        m_ref = opn.motion(torch.cat(m_ref))
        mscale = max(m_ref.abs().max().item(), 1e-30)
        assert (motion.cpu().double() - m_ref).abs().max().item() <= 1e-6 * mscale
        n_ref = opn.compose(prev.float().double(), motion.cpu().double())
        assert (nxt.cpu() - n_ref).abs().max().item() <= 1e-6


def _plugin(P, seed=0):
    return P.B200_TartanMotionNet(NS(weight=f"synthetic:{seed}", device=DEV))


@pytest.fixture(scope="module")
def P(lib):
    from macvo_b200 import plugins
    return plugins


def _pose(p):
    return (p.tensor() if hasattr(p, "ltype") else p).reshape(-1).cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("name", [n for n in CASES if n != "zerodepth"])   # +inf input: see DESIGN.md §2.2.1
def test_gpu_plugin_motion_matches_reference(P, golden, name, tf32):
    """the plugin's motion vs the reference fixture: strict fp32 within 1e-5 relative; with TF32 cuDNN convolutions in
    firstconv .. layer2 (as the frontend leaves the process) at about 1.5x the largest deviation measured (DESIGN.md §2)"""
    g, c = _case(golden, name)
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        mm = _plugin(P)
        first = _pose(mm.predict(_frame(c), None, None))
        assert torch.equal(first, torch.tensor([0., 0., 0., 0., 0., 0., 1.]))
        mm.update(c["prev_pose"].to(DEV))
        nxt = _pose(mm.predict(_frame(c), c["flow"].to(DEV), c["depth"].to(DEV)))
    finally:
        _strict_fp32()
    rel = _deviation(mm.motion, g["motion"])
    print(f"posenet {name} tf32={tf32}: motion deviation {rel:.3g} of its scale")
    assert rel <= (TF32_MOTION_TOL if tf32 else 1e-5), rel
    torch.testing.assert_close(nxt.double(), g["next_pose"].double(), rtol=0, atol=TF32_MOTION_TOL if tf32 else 1e-5,
                               equal_nan=True)


TF32_MOTION_TOL = 2e-4      # measured on an H100 80GB HBM3 (400 W): at most 1.23e-4 of the motion scale


@pytest.mark.gpu
def test_gpu_graph_replay_equals_first_call_and_guards_its_inputs(P):
    _strict_fp32()
    c = posenet_cases.posenet_inputs("480x640")
    fr = _frame(c)
    mm = _plugin(P)
    fl, dp = c["flow"].to(DEV), c["depth"].to(DEV)
    first = mm.enqueue(fr, fl, dp).clone()
    again = mm.enqueue(fr, fl, dp).clone()
    assert torch.equal(first, again)
    other = mm.enqueue(fr, fl + 1.0, dp).clone()
    assert not torch.equal(first, other)
    assert torch.equal(mm.enqueue(fr, fl, dp), first)
    # eager evaluation of the same network (no graph)
    inp = mm._static["inp"].clone()
    assert torch.equal(mm.net.body(inp), first)
    with pytest.raises(AssertionError):
        mm.enqueue(fr, fl[..., :-8], dp[..., :-8])
    fr2 = _frame(dict(c, fx=c["fx"] + 1.0))
    with pytest.raises(AssertionError):
        mm.enqueue(fr2, fl, dp)


@pytest.mark.gpu
def test_gpu_fused_driver_with_motion_model(P):
    """FusedTwoFrameOdometry(motion_model=...) vs TwoFrameOdometry with the same motion model class: equal observation
    counts, poses within 1e-6 absolute / 1e-5 relative (as test_gpu_pipeline.py's fused-vs-plugin check; measured 6.6e-6
    relative); the LM's initial pose in the fused tail is the motion model's prediction (TwoFrameOdometry's pose_init), not
    the previous pose; software-pipelined runs bit-identical to sequential ones"""
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    _strict_fp32()
    frames = synthetic.make_sequence(6, 192, 256, pin=True)

    def build(cls):
        fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp32", dec_dtype="fp32",
                                             decoder_depth=4, enforce_positive_disparity=False, cuda_graph=False))
        return cls(fe, P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=7, mask_width=32, max_match_cov=100.0)),
                   P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05,
                                             min_flow_cov=0.25)),
                   P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
                   num_point=64, map_selector=P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)),
                   keep_debug=True, motion_model=_plugin(P))

    a = build(TwoFrameOdometry)
    _strict_fp32()
    torch.manual_seed(5)
    a.initialize(frames[0])
    ra = [a.run_pair(f) for f in frames[1:]]
    pa = a.finish()
    runs = []
    for pipelined in (False, True):
        b = build(FusedTwoFrameOdometry)
        _strict_fp32()
        torch.manual_seed(5)
        b.initialize(frames[0])
        obs, inits = [], []
        for i in range(1, len(frames)):
            nxt = frames[i + 1] if pipelined and i + 1 < len(frames) and i != 3 else None
            inits.append(b.run_pair(frames[i], next_frame=nxt).extras["pose_init"])
            obs.append(b.observations())
        runs.append((obs, b.finish(), torch.stack([p.cpu() for p in inits])))
    (ob, pb, ib), (oc, pc, ic) = runs
    ia = torch.stack([x.pose_init for x in ra]).double()
    np.testing.assert_allclose(ib.numpy(), ia.numpy(), rtol=1e-5, atol=1e-6)
    assert (ib - pb[:-1].double()).abs().max(dim=1).values.min() > 1e-3     # every frame's LM started from a prediction
    assert torch.equal(ib, ic)
    for o, x in zip(ob, ra):
        assert o["num_obs"] == x.num_obs
    np.testing.assert_allclose(pb.numpy(), pa.numpy(), rtol=1e-5, atol=1e-6)
    assert not torch.equal(pa[1], pa[0])
    assert torch.equal(pb, pc)
    for x, y in zip(ob, oc):
        assert x["num_obs"] == y["num_obs"]
        for k in ("pixel1_uv", "pixel2_uv", "pos_Tw", "obs1_covTc", "obs2_covTc"):
            assert torch.equal(x[k], y[k]), k


# ---------------------------------------------------------------------------------------------------------------------------
# under the real Odometry/MACVO.py (CPU; needs a MAC-VO tree)
# ---------------------------------------------------------------------------------------------------------------------------
MACVO_CODE = r'''
import sys, os, torch
sys.path.insert(0, %r)
os.environ["TORCHDYNAMO_DISABLE"] = "1"
from tests.golden import refharness
refharness.install()
sys.modules["cupy"] = refharness._StubModule("cupy")    # PWC-Net's correlation module imports cupy; never run here
from types import SimpleNamespace as NS
import torch.nn.functional as F
import Module
from Odometry.MACVO import MACVO
from DataLoader import StereoFrame, StereoData
import pypose as pp
import macvo_b200.plugins as P
from macvo_b200 import ops, synthetic
from macvo_b200.flowformer_cov import synthetic_state_dict
from macvo_b200.posenet import synthetic_posenet_state_dict
from Module.Network.TartanVOStereo.StereoVO import StereoVONet
from oracle import keypoint as okp, posenet as opn
torch.cuda.current_stream = lambda *a, **k: None     # TwoFrame_PGO._optimize only hands it to an inactive Timer (Optimizer.py:83)
torch.save(synthetic_state_dict(0), sys.argv[1])
# one TartanVO checkpoint for both sides: the whole StereoVONet (the reference loads it strictly), pose network synthetic
full = StereoVONet(flowNormFactor=1.0, stereoNormFactor=0.02, poseDepthNormFactor=0.25).state_dict()
full.update({"flowPoseNet." + k: v for k, v in synthetic_posenet_state_dict(0).items()})
torch.save({"module." + k: v for k, v in full.items()}, sys.argv[2])

def config(b200):
    t = (lambda n: "B200_" + n) if b200 else (lambda n: n)
    fe_args = NS(device="cpu", weight="synthetic:0" if b200 else sys.argv[1], enc_dtype="fp32", dec_dtype="fp32",
                 decoder_depth=4, enforce_positive_disparity=False)
    if b200:
        fe_args.cuda_graph = False
    outlier = NS(type="FilterCompose", args=NS(filter_args=[NS(type="CovarianceSanityFilter", args=NS()),
                 NS(type="SimpleDepthFilter", args=NS(min_depth=0.05, max_depth="auto")),
                 NS(type="LikelyFrontOfCamFilter", args=NS())]))
    return NS(Odometry=NS(name="t", args=NS(device="cpu", edgewidth=32, num_point=64, match_cov_default=0.25, profile=False, mapping=False),
        cov=NS(obs=NS(type=t("MatchCovariance"), args=NS(device="cpu", kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25))),
        keypoint=NS(type=t("CovAwareSelector"), args=NS(device="cpu", kernel_size=7, mask_width=32, max_depth="auto",
                                                        max_depth_cov=250.0, max_match_cov=100.0)),
        mappoint=NS(type=t("MappingPointSelector"), args=(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32) if b200 else
                                                           NS(device="cpu", max_depth=5.0, max_depth_cov=0.005, mask_width=32))),
        frontend=NS(type=t("FlowFormerCovFrontend"), args=fe_args),
        motion=NS(type=t("TartanMotionNet"), args=NS(weight=sys.argv[2], device="cpu")), outlier=outlier,
        postprocess=NS(type=t("MotionInterpolate"), args=(NS(device="cpu") if b200 else NS())), keyframe=NS(type="AllKeyframe", args=NS()),
        optimizer=NS(type=t("TwoFrame_PGO"), args=NS(device="cpu", vectorize=True, parallel=False, graph_type="icp", autodiff=False))))

predictions = []
def run(b200):
    cfg = config(b200)
    odo = MACVO[StereoFrame].from_config(cfg)
    assert type(odo.MotionEstimator).__name__ == ("B200_TartanMotionNet" if b200 else "TartanMotionNet")
    pred = odo.MotionEstimator.predict
    def spy(*a, **k):
        p = pred(*a, **k)
        predictions.append(p.tensor().clone())
        return p
    odo.MotionEstimator.predict = spy
    torch.set_float32_matmul_precision("highest")
    torch.manual_seed(5)
    for i, f in enumerate(synthetic.make_sequence(4, 192, 256)):
        sd = StereoData(T_BS=pp.identity_SE3(1), K=f.K, baseline=f.baseline, time_ns=f.time_ns, height=f.height,
                        width=f.width, imageL=f.imageL, imageR=f.imageR)
        odo.run(StereoFrame(idx=[i], time_ns=f.time_ns, stereo=sd))
    odo.terminate()
    m = odo.get_map()
    return m.frames.data["pose"].tensor.clone(), len(m.match), len(m.points)

ref = run(False)
ref_pred = torch.stack(predictions); predictions.clear()

from tests import mock_ops
mock_ops.install()
# the motion model's C-ABI calls, answered by the oracle; the CUDA graph becomes a plain re-run
P.B200_TartanMotionNet._capture = lambda self, run: run
ops.posenet_input = lambda flow, depth, bl_fx, out: out[:, :3].copy_(opn.flow_depth_channels(flow, depth, bl_fx))
def posenet_conv(x, packed, co_tile, bias, k, stride, pad, resid=None, relu=False, out=None):
    cin, cout = x.shape[-3], bias.numel()
    w = packed.reshape(cout // co_tile, 8, co_tile, -1).permute(0, 2, 1, 3).reshape(cout, cin, k, k)
    y = F.conv2d(x.reshape(1, cin, *x.shape[-2:]), w, bias, stride=stride, padding=pad)
    y = y + resid.reshape(y.shape) if resid is not None else y
    return y.relu() if relu else y
ops.posenet_conv = posenet_conv
def posenet_head(fc1, blob, prev_pose, motion, next_pose):
    o, m = 0, []
    take = lambda n: blob[o:o + n]
    parts = {}
    for name, n in (("w2t", 4096), ("b2t", 32), ("w2r", 4096), ("b2r", 32), ("w3t", 96), ("b3t", 3), ("w3r", 96), ("b3r", 3), ("norm", 6)):
        parts[name] = blob[o:o + n]; o += n
    for i, h in enumerate("tr"):
        y = F.relu(F.linear(fc1[128 * i:128 * (i + 1)], parts["w2" + h].reshape(32, 128), parts["b2" + h]))
        m.append(F.linear(y, parts["w3" + h].reshape(3, 32), parts["b3" + h]))
    motion.copy_(torch.cat(m) * parts["norm"])
    next_pose.copy_(opn.compose(prev_pose.float(), motion).double())
ops.posenet_head = posenet_head
def score_depth_aware(match_cov, dcov0, dcov1, score):
    score.mock = (match_cov, dcov0, dcov1)
ops.score_depth_aware = score_depth_aware
def select_candidates_depth(score, d0, d1, dcov0, mw, md, mdc, mmc, m0, m1, out):
    out.req = ("depth", score.mock, d0, d1, score.ksize, mw, md, mdc, mmc, m0, m1)
ops.select_candidates_depth = select_candidates_depth
_sample = ops.sample_candidates
def sample_candidates(cand, num):
    if cand.req[0] != "depth":
        return _sample(cand, num)
    _, (mc, c0, c1), d0, d1, ks, mw, md, mdc, mmc, m0, m1 = cand.req
    return okp.cov_aware_select(mc, d0, c0, d1, c1, num, ks, mw, md, mdc, mmc, m0, m1)
ops.sample_candidates = sample_candidates

got = run(True)
got_pred = torch.stack(predictions)
# (with the synthetic frontend weights LikelyFrontOfCamFilter rejects every observation on both sides, so the poses are the
# motion model's chained predictions; the icp LM under MACVO.py is covered by test_macvo_integration.py)
assert got[1] == ref[1] and got[2] == ref[2], (got[1:3], ref[1:3])
assert torch.isfinite(got[0]).all()
torch.testing.assert_close(got_pred, ref_pred, rtol=1e-4, atol=1e-4)      # identity, then 3 predictions
assert (ref_pred[1:, :3] - ref[0][:3, :3]).abs().max() > 1e-3             # the predictions are not the previous poses
torch.testing.assert_close(got[0], ref[0], rtol=1e-4, atol=1e-4)          # poses of all 4 frames
print("MACVO-MOTION-OK", got[1], got[2])
''' % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _reference_tree() -> bool:
    from tests.golden import refharness
    return refharness.available()


@pytest.mark.skipif(not _reference_tree(), reason="MAC-VO reference tree not present")
def test_motion_model_under_the_real_macvo(tmp_path):
    """Paper_Reproduce-shaped config (CovAwareSelector, FilterCompose of the reference's three filters, icp graph) through the
    REAL Odometry/MACVO.py for 4 frames: B200_TartanMotionNet found by name in the registry, fed StereoFrames, updated with
    pp.SE3 map poses and unsqueezed like MACVO.py:160,193-194 — its C-ABI calls answered by the CPU oracle — against the
    reference TartanMotionNet (cupy stubbed, the same checkpoint): same observation counts, predictions and poses within 1e-4"""
    import subprocess
    import sys
    r = subprocess.run([sys.executable, "-c", MACVO_CODE, str(tmp_path / "fe.pth"), str(tmp_path / "tartanvo.pkl")],
                       capture_output=True, text=True, timeout=900, env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "MACVO-MOTION-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]
