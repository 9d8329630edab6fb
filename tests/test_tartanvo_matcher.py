"""B200_TartanVOMatcher on the CPU: the PWC-Net oracle (oracle/pwc.py) against the reference fixtures
(tests/golden/tartanvo_flow_*.pt, written by tests/golden/make_golden_tartanvo_flow.py from the MAC-VO tree itself), the
synthetic weights, checkpoint and config handling, registration, and the plugin's host logic with an oracle stand-in for
macvo_pwc_warp_corr."""
import os
import subprocess
import sys
import tempfile
from types import SimpleNamespace as NS

import pytest
import torch

from tests.golden import refharness, tartanvo_cases

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = list(tartanvo_cases.CASES)


def _sd(seed=0):
    from macvo_b200.pwcnet import synthetic_pwc_state_dict
    return synthetic_pwc_state_dict(seed)


@pytest.mark.parametrize("name", CASES)
def test_fixture_inputs_reproduce(golden, name):
    g = golden(f"tartanvo_flow_{name}.pt")
    f1, f2 = tartanvo_cases.frames(name)
    assert tartanvo_cases.sha(f1.imageL, f2.imageL) == g["input_sha"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_fixture(golden, name):
    """the oracle's network (same CPU torch operations as the reference, correlation restated identically) reproduces the
    reference's flow2; for `small` also the matcher's (flow, mask) and the cost volumes of levels 6..4, the latter through
    the kernel's fp32 tap rule (oracle.pwc.warp_corr) instead of torch's grid_sample"""
    from oracle import pwc as opwc
    g = golden(f"tartanvo_flow_{name}.pt")
    f1, f2 = tartanvo_cases.frames(name)
    flow, mask, res = opwc.match(_sd(g["seed"]), f1.imageL, f2.imageL)
    scale = g["flow2"].abs().max().item()
    assert (res["flow2"] - g["flow2"]).abs().max().item() <= 1e-6 * scale
    if name != "small":
        return
    assert torch.equal(mask, g["mask"]) and mask.shape == (1, 1, 192, 256)
    assert torch.equal(torch.isnan(flow), torch.isnan(g["flow"]))
    assert (flow - g["flow"]).nan_to_num().abs().max().item() <= 1e-6 * scale / 0.05
    for lv in g["levels"]:
        got = opwc.warp_corr(lv["f1"], lv["f2"], lv["flow"], 1.0)
        ref = lv["corr"]
        assert (got - ref).abs().max().item() <= 1e-5 * max(ref.abs().max().item(), 1e-6), lv["level"]


def test_mask_rule_at_the_fixture_shapes():
    """True on [ph:-ph, pw:-pw] of the (h64, w64) crop — all False when a margin is 0 (TartanAir's 480x640)"""
    from oracle import pwc as opwc
    for name, (H, W) in tartanvo_cases.CASES.items():
        (ph, pw), (h64, w64) = opwc.crop_margins(H, W)
        m = torch.zeros((h64, w64), dtype=torch.bool)
        m[ph:-ph, pw:-pw] = True
        expect = (h64 - 2 * ph) * (w64 - 2 * pw) if ph and pw else 0
        assert int(m.sum()) == expect, name
    assert opwc.crop_margins(480, 640) == ((16, 0), (448, 640))


def test_synthetic_weights_give_a_live_network():
    """every warp level keeps strictly between 50 % and 100 % of its samples, with fractional offsets; flow2 is not near
    zero and every cost volume has positive and negative entries"""
    from oracle import pwc as opwc
    f1, f2 = tartanvo_cases.frames("small")
    _, _, res = opwc.match(_sd(0), f1.imageL, f2.imageL)
    for level, uf in res["up_flow"].items():
        *_, m = opwc.warp_fp32_taps(uf, 1.0)
        kept = m.mean().item()
        assert 0.5 < kept < 1.0, (level, kept)
        frac = (uf - uf.round()).abs()
        assert (frac > 0.05).float().mean() > 0.5, level
        assert uf.abs().mean() > 0.1, level
    for level, cv in res["corr"].items():
        assert 0.0 < (cv > 0).float().mean() < 1.0, level
    assert res["flow2"].abs().mean() > 0.05 and torch.isfinite(res["flow2"]).all()


def test_state_dict_shapes_match_the_reference_module():
    if not refharness.available():
        pytest.skip("MAC-VO reference tree not present")
    code = r'''
import sys
sys.path.insert(0, %r)
from tests.golden import refharness
refharness.install()
sys.modules["cupy"] = refharness._StubModule("cupy")
from Module.Network.PWCNet.pwc.pwc_model_tartanvo import PWCDCNet_Adapted
from macvo_b200.pwcnet import state_dict_shapes
ref = {k: tuple(v.shape) for k, v in PWCDCNet_Adapted(md=4, uncertainty=False).state_dict().items()}
assert ref == state_dict_shapes(), set(ref) ^ set(state_dict_shapes())
print("SHAPES-OK")
''' % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "SHAPES-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_config_validation():
    from macvo_b200 import plugins as P
    cls = P.B200_TartanVOMatcher
    cls.is_valid_config(NS(weight="synthetic:0", device="cuda"))
    cls.is_valid_config(NS(weight="synthetic:0", device="cuda:0", cuda_graph=False))
    with pytest.raises(Exception):
        cls.is_valid_config(NS(weight="synthetic:0", device="cuda", enc_dtype="fp32"))     # unknown key
    with pytest.raises(Exception):
        cls.is_valid_config(NS(weight="synthetic:0", device="cuda", cuda_graph="yes"))
    with pytest.raises(Exception):
        cls.is_valid_config(NS(weight="synthetic:0", device="cpu"))
    with pytest.raises(ValueError):
        cls(NS(weight="synthetic:0", device="cpu"))
    assert P.PLUGINS["matcher_tartanvo"] is cls


def _checkpoint(path, flow_sd, pose_sd=None, extra=None):
    sd = {"module.flowNet." + k: v for k, v in flow_sd.items()}
    if pose_sd is not None:
        sd.update({"module.flowPoseNet." + k: v for k, v in pose_sd.items()})
    sd.update(extra or {})
    torch.save(sd, path)


def test_checkpoint_reads_only_the_flownet_tensors():
    from macvo_b200.pwcnet import load_checkpoint
    ref = _sd(3)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tartanvo.pkl")
        _checkpoint(path, ref, extra={"module.stereoNet.x": torch.zeros(1), "flowNet.conv1a.0.weight": torch.zeros(1),
                                      "module.flowNet.unused": torch.zeros(1)})
        got = load_checkpoint(path)
    assert set(got) == set(ref) and all(torch.equal(got[k], ref[k]) for k in ref)


def test_checkpoint_missing_or_misshapen_tensor_raises():
    from macvo_b200.pwcnet import load_checkpoint
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tartanvo.pkl")
        sd = _sd(0)
        del sd["conv4_2.0.bias"]
        _checkpoint(path, sd)
        with pytest.raises(KeyError, match="conv4_2.0.bias"):
            load_checkpoint(path)
        sd = _sd(0)
        sd["upfeat5.weight"] = sd["upfeat5.weight"][:, :1]
        _checkpoint(path, sd)
        with pytest.raises(ValueError, match="upfeat5.weight"):
            load_checkpoint(path)


def test_one_checkpoint_serves_both_tartanvo_plugins():
    """a StereoVONet-style file with module.flowNet.* and module.flowPoseNet.*: each loader takes its own half"""
    from macvo_b200 import posenet, pwcnet
    fsd, psd = _sd(1), posenet.synthetic_posenet_state_dict(2)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "MACVO_posenet.pkl")
        _checkpoint(path, fsd, psd)
        got_f, got_p = pwcnet.load_checkpoint(path), posenet.load_checkpoint(path)
    assert all(torch.equal(got_f[k], fsd[k]) for k in fsd) and set(got_f) == set(fsd)
    assert all(torch.equal(got_p[k], psd[k]) for k in psd) and set(got_p) == set(psd)


def test_symbol_exported():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    import ctypes
    assert "macvo_pwc_warp_corr" in ops.EXPORTS and hasattr(ctypes.CDLL(build.LIB_PATH), "macvo_pwc_warp_corr")


@pytest.fixture
def cpu_plugin(monkeypatch):
    """the plugin's host logic on the CPU: macvo_pwc_warp_corr answered by the oracle, no CUDA graph"""
    from macvo_b200 import ops, plugins
    from oracle import pwc as opwc

    def warp_corr(f1, f2, flow, scale, out, out_offset):
        out[:, out_offset:out_offset + 81] = opwc.warp_corr(f1, f2, flow, scale)
        return out
    monkeypatch.setattr(ops, "pwc_warp_corr", warp_corr)
    monkeypatch.setattr(plugins, "_require_cuda", lambda device, who: torch.device(device))
    return lambda: plugins.B200_TartanVOMatcher(NS(weight="synthetic:0", device="cpu", cuda_graph=False))


def test_plugin_host_logic_matches_the_reference_fixture(golden, cpu_plugin):
    """crop, raw images, flow2 / 0.05, nearest x4, NaN padding, the mask quirk and the errors, with an oracle stand-in for
    the kernel (the GPU tests pin the kernel to the oracle)"""
    g = golden("tartanvo_flow_small.pt")
    m = cpu_plugin()
    assert m.provide_cov is False
    f1, f2 = tartanvo_cases.frames("small")
    out = m.estimate(f1, f2)
    assert out.flow.dtype == torch.float32 and out.flow.shape == (1, 2, 200, 264) and out.cov is None
    assert torch.equal(out.mask, g["mask"])
    assert torch.equal(torch.isnan(out.flow), torch.isnan(g["flow"]))
    scale = g["flow"].nan_to_num().abs().max().item()
    assert (out.flow - g["flow"]).nan_to_num().abs().max().item() <= 1e-5 * scale
    two = NS(**dict(vars(f1), imageL=torch.cat([f1.imageL, f1.imageL])))
    with pytest.raises(AssertionError):
        m.estimate(two, f2)
    odd = tartanvo_cases.frame(f1.imageL[..., :199, :])       # 199 - 192 = 7: odd margin
    with pytest.raises(AssertionError, match="even padding"):
        m.estimate(odd, odd)


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_registers_into_macvo_imatcher():
    code = r'''
import sys
sys.path.insert(0, %r)
from tests.golden import refharness
refharness.install()
from types import SimpleNamespace as NS
from Module import IMatcher
import macvo_b200.plugins as P
assert P._REF
assert IMatcher.get_class("B200_TartanVOMatcher") is P.B200_TartanVOMatcher
assert issubclass(P.B200_TartanVOMatcher, IMatcher)
IMatcher.is_valid_config(NS(type="B200_TartanVOMatcher", args=NS(weight="./Model/MACVO_posenet.pkl", device="cuda")))
try:
    IMatcher.is_valid_config(NS(type="B200_TartanVOMatcher", args=NS(weight="w", device="cuda", extra=1)))
    raise SystemExit("excess key accepted")
except KeyError:
    pass
print("MATCHER-REGISTERED-OK")
''' % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "MATCHER-REGISTERED-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
BASELINE_CODE = r'''
import sys, os, torch
sys.path.insert(0, %r)
os.environ["TORCHDYNAMO_DISABLE"] = "1"
from tests.golden import make_golden_tartanvo_flow as gen, refharness
gen.write_checkpoint(sys.argv[1])                       # StereoVONet: synthetic flowNet and flowPoseNet (seed 0)
matcher_ref, _ = gen.reference_matcher(sys.argv[1])     # installs the generator's substitutions (cupy, correlation, .cuda)
from types import SimpleNamespace as NS
import Module
import pypose as pp
from DataLoader import StereoFrame, StereoData
from Module.Network.StereoCov import StereoCovNet
from Utility.Config import build_dynamic_config
from Odometry.BaselineTartanVO import TartanVO
from macvo_b200 import ops, plugins as P, synthetic
from oracle import pwc as opwc
from Module.MapProcessor import IMapProcessor
class Naive(IMapProcessor):
    """BaselineTartanVO.py:22 instantiates an IMapProcessor named "Naive" that the MAC-VO tree does not define; with
    keyframe_freq 1 no frame needs interpolation, so the stand-in leaves the map as it is (the same on both sides)"""
    def elaborate_map(self, frames):
        return frames, torch.zeros((0,), dtype=torch.long)
    @classmethod
    def is_valid_config(cls, config):
        return None
from Module.MotionModel import TartanMotionNet
_predict = TartanMotionNet.predict
def predict(self, frame, flow, depth):
    """BaselineTartanVO.run pushes predict's first pose, pp.identity_SE3() of shape (7,), into a (1, ...) FrameNode; the
    leading dimension MACVO.py adds itself (MACVO.py:160) is added here, identically for both runs"""
    pose = _predict(self, frame, flow, depth)
    return pose.unsqueeze(0) if pose.dim() == 1 else pose
TartanMotionNet.predict = predict
torch.manual_seed(4321)
cfg_sc, _ = build_dynamic_config({"exp": False, "decoder": "hourglass"})
torch.save({"module." + k: v for k, v in StereoCovNet(cfg_sc).state_dict().items()}, sys.argv[2])

def config(b200):
    match = (NS(type="B200_TartanVOMatcher", args=NS(weight=sys.argv[1], device="cpu", cuda_graph=False)) if b200 else
             NS(type="TartanVOMatcher", args=NS(weight=sys.argv[1], device="cpu")))
    return NS(name="TartanVOStereo", depth=NS(type="TartanVODepth", args=NS(weight=sys.argv[2], device="cpu", cov_mode="Est")),
              match=match, tartanvo=NS(weight=sys.argv[1], device="cpu"),
              keyframe=NS(type="UniformKeyframe", args=NS(keyframe_freq=1)))

H, W = 264, 328      # the reference StereoCovNet's 64x64 pooling needs a crop of at least 256 rows; margins 4 / 4
flows = []
def run(b200):
    cfg = config(b200)
    if b200:    # the driver's validator, with the device the plugin requires (this CPU run then bypasses _require_cuda)
        TartanVO.is_valid_config(NS(**dict(vars(cfg), match=NS(type=cfg.match.type, args=NS(**dict(vars(cfg.match.args), device="cuda"))))))
    else:
        TartanVO.is_valid_config(cfg)
    odo = TartanVO.from_config(cfg, None)
    assert type(odo.match_estimator).__name__ == ("B200_TartanVOMatcher" if b200 else "TartanVOMatcher")
    est = odo.match_estimator.estimate
    def spy(*a, **k):
        out = est(*a, **k)
        flows.append((out.flow.clone(), out.mask.clone()))
        return out
    odo.match_estimator.estimate = spy
    torch.manual_seed(5)
    for i, f in enumerate(synthetic.make_sequence(4, H, W)):
        sd = StereoData(T_BS=pp.identity_SE3(1), K=f.K, baseline=f.baseline, time_ns=f.time_ns, height=f.height,
                        width=f.width, imageL=f.imageL, imageR=f.imageR)
        odo.run(StereoFrame(idx=[i], time_ns=f.time_ns, stereo=sd))
    odo.terminate()
    return odo.get_map().frames.data["pose"].tensor.clone()

ref = run(False)
ref_flows = list(flows); flows.clear()
# the plugin's one C-ABI call answered by the oracle, on the CPU
P._require_cuda = lambda device, who: torch.device(device)
def warp_corr(f1, f2, flow, scale, out, out_offset):
    out[:, out_offset:out_offset + 81] = opwc.warp_corr(f1, f2, flow, scale)
    return out
ops.pwc_warp_corr = warp_corr
got = run(True)
assert len(flows) == len(ref_flows) == 3
for (fg, mg), (fr, mr) in zip(flows, ref_flows):
    assert fg.shape == fr.shape == (1, 2, H, W) and torch.equal(torch.isnan(fg), torch.isnan(fr))
    assert torch.equal(mg, mr) and mg.shape == (1, 1, 256, 320) and mg.any()
    scale = fr.nan_to_num().abs().max()
    assert (fg - fr).nan_to_num().abs().max() <= 1e-5 * scale, ((fg - fr).nan_to_num().abs().max(), scale)
assert torch.isfinite(got).all() and got.shape == (4, 7)
assert (ref[1:, :3] - ref[:1, :3]).abs().max() > 1e-4, ref       # the trajectory moves
torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-5)
print("TARTANVO-BASELINE-OK", (got - ref).abs().max().item())
''' % REPO


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_matcher_under_the_real_tartanvo_baseline(tmp_path):
    """Odometry/BaselineTartanVO.TartanVO.from_config on a TartanVOStereo.yaml-shaped config (match.type:
    B200_TartanVOMatcher, found through the IMatcher registry; depth TartanVODepth and the hard-wired TartanMotionNet from the
    reference with synthetic weights) over 4 frames of 264x328 on the CPU (the smallest such size: at 200x264 the
    reference's own StereoCovNet fails, its 64x64 average pooling meeting a 48-row feature map), the plugin's macvo_pwc_warp_corr answered by the
    oracle, against the same run through the reference TartanVOMatcher patched as in make_golden_tartanvo_flow.py. Both runs
    get the same two repairs of the driver: a stand-in for the "Naive" map processor it names but the tree lacks, and the
    leading dimension on the motion model's first (identity) pose that its FrameNode needs. Compared: the matcher outputs (flow within 1e-5 of its scale, NaN pattern and mask exactly) and the trajectory within 1e-4"""
    r = subprocess.run([sys.executable, "-c", BASELINE_CODE, str(tmp_path / "tartanvo.pkl"), str(tmp_path / "depth.pth")],
                       capture_output=True, text=True, timeout=900, env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "TARTANVO-BASELINE-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]
