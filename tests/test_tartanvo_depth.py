"""B200_TartanVODepth on the CPU: the StereoCovNet oracle (oracle/stereo.py) against the reference fixtures
(tests/golden/tartanvo_depth_*.pt, written by tests/golden/make_golden_tartanvo_depth.py from the MAC-VO tree itself), the
synthetic weights, checkpoint and config handling, registration, the plugin's torch-op path and errors, and the plugin under
the real Odometry/BaselineTartanVO.py."""
import os
import subprocess
import sys
import tempfile
from types import SimpleNamespace as NS

import pytest
import torch

from tests.golden import make_golden_tartanvo_depth as gen, refharness, tartanvo_cases

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = list(gen.CASES)


def _sd(seed=0):
    from macvo_b200.stereonet import synthetic_stereo_state_dict
    return synthetic_stereo_state_dict(seed)


def _close(got, ref, rel):
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    fin = torch.isfinite(ref)
    scale = ref[fin].abs().max().item()
    err = (got.double() - ref.double())[fin].abs().max().item()
    assert err <= rel * scale, (err, scale)


@pytest.mark.parametrize("name", CASES)
def test_fixture_inputs_reproduce(golden, name):
    g = golden(f"tartanvo_depth_{name}.pt")
    f = gen.frame(name)
    assert tartanvo_cases.sha(f.imageL, f.imageR) == g["input_sha"]
    assert g["bf"] == f.frame_baseline * f.fx == 80.0


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_fixture(golden, name):
    """the float64 oracle against the reference's fp32 CPU run: depth and variance within 1e-3 of their scale (the fp32
    rounding of the reference through ~60 layers), NaN border identical"""
    from oracle import stereo as ost
    g = golden(f"tartanvo_depth_{name}.pt")
    f = gen.frame(name)
    depth, cov = ost.estimate(_sd(g["seed"]), f.imageL, f.imageR, g["bf"])
    s = g["stride"]
    _close(depth[..., ::s, ::s], g["depth"], 1e-3)
    _close(cov[..., ::s, ::s], g["cov"], 1e-3)


def test_oracle_head_matches_the_reference_head(golden):
    """oracle.stereo.head (deconv_c11 written as four output phases) from the reference's own head inputs reproduces the
    reference's depth and variance on the pixels the stored window determines"""
    from oracle import stereo as ost
    g = golden("tartanvo_depth_small.pt")["head"]
    d, v = ost.head(_sd(0), g["xd"].double(), g["xc"].double(), g["cat0"].double(), 80.0)
    h, w = g["depth"].shape[-2:]
    _close(d[..., :h, :w], g["depth"], 1e-5)
    _close(v[..., :h, :w], g["cov"], 1e-4)


def test_synthetic_weights_give_a_live_network(golden):
    """disparity mostly positive and a few to a few tens of pixels; the covariance head positive on most pixels"""
    from oracle import stereo as ost
    for name in ("small", "euroc"):
        g = golden(f"tartanvo_depth_{name}.pt")
        fin = torch.isfinite(g["depth"])
        disp = 80.0 / g["depth"][fin]
        assert (disp > 0).float().mean() > 0.95 and 2.0 < disp.median() < 40.0, name
        assert (g["cov"][fin] > 0).float().mean() > 0.9, name
    head = golden("tartanvo_depth_small.pt")["head"]
    assert head["xd"].abs().mean() > 0.01 and head["xc"].abs().mean() > 0.01 and ost.MEAN == (0.485, 0.456, 0.406)


def test_state_dict_shapes_match_the_reference_module():
    if not refharness.available():
        pytest.skip("MAC-VO reference tree not present")
    code = r'''
import sys
sys.path.insert(0, %r)
from tests.golden import refharness
refharness.install()
from Utility.Config import build_dynamic_config
from Module.Network.StereoCov import StereoCovNet
from macvo_b200.stereonet import state_dict_shapes
cfg, _ = build_dynamic_config({"exp": False, "decoder": "hourglass"})
ref = {k: tuple(v.shape) for k, v in StereoCovNet(cfg).state_dict().items()}
assert ref == state_dict_shapes(), set(ref) ^ set(state_dict_shapes())
print("SHAPES-OK")
''' % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "SHAPES-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_checkpoint_strips_module_prefix_and_reads_batchnorm_statistics():
    from macvo_b200.stereonet import load_checkpoint
    ref = _sd(3)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "depth.pth")
        torch.save({"module." + k: v for k, v in ref.items()}, path)
        got = load_checkpoint(path)
        torch.save(ref, path)                                   # without the prefix as well
        got2 = load_checkpoint(path)
    assert set(got) == set(ref) and all(torch.equal(got[k], ref[k]) and torch.equal(got2[k], ref[k]) for k in ref)
    assert any(k.endswith("running_var") for k in got)


def test_checkpoint_missing_or_misshapen_tensor_raises():
    from macvo_b200.stereonet import load_checkpoint
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "depth.pth")
        sd = _sd(0)
        del sd["feature.stereo.feature_extraction.layer2.0.downsample.1.running_mean"]
        torch.save(sd, path)
        with pytest.raises(KeyError, match="layer2.0.downsample.1.running_mean"):
            load_checkpoint(path)
        sd = _sd(0)
        sd["decoder.deconv_c11.weight"] = sd["decoder.deconv_c11.weight"][:, :32]
        torch.save(sd, path)
        with pytest.raises(ValueError, match="decoder.deconv_c11.weight"):
            load_checkpoint(path)


def test_batchnorm_fold_matches_eval_batchnorm():
    import torch.nn.functional as F
    from macvo_b200.stereonet import fold_batchnorm
    sd = _sd(1)
    fd = fold_batchnorm(sd)
    p = "feature.stereo.feature_extraction.layer3.0.downsample"
    assert f"{p}.weight" in fd and f"{p}.0.weight" not in fd and f"{p}.1.running_var" not in fd
    x = torch.randn(1, 64, 8, 8, dtype=torch.float64)
    ref = F.batch_norm(F.conv2d(x, sd[f"{p}.0.weight"].double()), sd[f"{p}.1.running_mean"].double(),
                       sd[f"{p}.1.running_var"].double(), sd[f"{p}.1.weight"].double(), sd[f"{p}.1.bias"].double(),
                       False, 0.0, 1e-5)
    got = F.conv2d(x, fd[f"{p}.weight"].double(), fd[f"{p}.bias"].double())
    assert (got - ref).abs().max() <= 1e-5 * ref.abs().max()


def test_arranged_head_weights_are_the_phase_taps():
    """arrange_head's blocks applied as the kernel applies them equal F.conv_transpose2d (float64, unrounded weights)"""
    import torch.nn.functional as F
    from macvo_b200 import stereonet
    g = torch.Generator().manual_seed(2)
    w = torch.randn(128, 64, 4, 4, generator=g)
    k = torch.randn(1, 128, 5, 7, generator=g, dtype=torch.float64)
    blocks = stereonet.arrange_head(w).double()                       # (kc, phase, tap, 64, 32)
    ref = F.conv_transpose2d(k, w.double(), stride=2, padding=1)
    kp = F.pad(k, (1, 1, 1, 1))
    for py in (0, 1):
        for px in (0, 1):
            acc = torch.zeros(1, 64, 5, 7, dtype=torch.float64)
            for ty, (dy, _) in enumerate(stereonet.head_taps(py)):
                for tx, (dx, _) in enumerate(stereonet.head_taps(px)):
                    bt = blocks[:, 2 * py + px, 2 * ty + tx].permute(1, 0, 2).reshape(64, 128)
                    acc += torch.einsum("bchw,oc->bohw", kp[:, :, 1 + dy:6 + dy, 1 + dx:8 + dx], bt)
            assert (acc - ref[:, :, py::2, px::2]).abs().max() <= 2e-3 * ref.abs().max()     # tf32-rounded weights


def test_config_validation():
    from macvo_b200 import plugins as P
    cls = P.B200_TartanVODepth
    cls.is_valid_config(NS(weight="synthetic:0", device="cuda", cov_mode="Est"))
    cls.is_valid_config(NS(weight="x.pth", device="cuda:0", cov_mode="None", cuda_graph=False))
    for bad in (NS(weight="w", device="cuda", cov_mode="Est", enc_dtype="fp32"), NS(weight="w", device="cuda"),
                NS(weight="w", device="cuda", cov_mode="GT"), NS(weight="w", device="cuda", cov_mode="Est", cuda_graph=1),
                NS(weight="w", device="cpu", cov_mode="Est")):
        with pytest.raises(Exception):
            cls.is_valid_config(bad)
    with pytest.raises(ValueError):
        cls(NS(weight="synthetic:0", device="cpu", cov_mode="Est"))
    assert P.PLUGINS["depth_tartanvo"] is cls


def test_symbol_exported():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    import ctypes
    assert "macvo_stereo_head" in ops.EXPORTS and hasattr(ctypes.CDLL(build.LIB_PATH), "macvo_stereo_head")


@pytest.fixture
def cpu_plugin(monkeypatch):
    """the plugin's host logic and torch-op head path on the CPU, no CUDA graph"""
    from macvo_b200 import plugins
    monkeypatch.setattr(plugins, "_require_cuda", lambda device, who: torch.device(device))
    return lambda mode="Est": plugins.B200_TartanVODepth(NS(weight="synthetic:0", device="cpu", cov_mode=mode,
                                                            cuda_graph=False))


def test_plugin_torch_path_matches_the_reference_fixture(golden, cpu_plugin):
    g = golden("tartanvo_depth_small.pt")
    m = cpu_plugin()
    assert m.provide_cov is True
    out = m.estimate(gen.frame("small"))
    assert out.depth.shape == out.cov.shape == (1, 1, 264, 328) and out.depth.dtype == torch.float32
    s = g["stride"]
    _close(out.depth[..., ::s, ::s], g["depth"], 1e-4)
    _close(out.cov[..., ::s, ::s], g["cov"], 1e-4)
    none = cpu_plugin("None")
    assert none.provide_cov is False
    o2 = none.estimate(gen.frame("small"))
    assert o2.cov is None and torch.equal(o2.depth.nan_to_num(7.0), out.depth.nan_to_num(7.0))


def test_plugin_errors(cpu_plugin):
    m = cpu_plugin()
    f = gen.frame("small")
    small = tartanvo_cases.frame(f.imageL[..., :255, :])
    small.imageR = f.imageR[..., :255, :]
    with pytest.raises(ValueError, match="64x64 average pooling at 1/4 resolution"):
        m.estimate(small)
    odd = tartanvo_cases.frame(f.imageL[..., :263, :])                # 263 - 256 = 7: odd margin
    odd.imageR = f.imageR[..., :263, :]
    with pytest.raises(AssertionError, match="even padding"):
        m.estimate(odd)
    two = NS(**dict(vars(f), imageL=torch.cat([f.imageL, f.imageL]), imageR=torch.cat([f.imageR, f.imageR])))
    with pytest.raises(AssertionError):
        m.estimate(two)


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_registers_into_macvo_istereodepth():
    code = r'''
import sys
sys.path.insert(0, %r)
from tests.golden import refharness
refharness.install()
from types import SimpleNamespace as NS
from Module import IStereoDepth
import macvo_b200.plugins as P
assert P._REF
assert IStereoDepth.get_class("B200_TartanVODepth") is P.B200_TartanVODepth
IStereoDepth.is_valid_config(NS(type="B200_TartanVODepth", args=NS(weight="./Model/TartanVO_depth_cov.pth", device="cuda", cov_mode="Est")))
try:
    IStereoDepth.is_valid_config(NS(type="B200_TartanVODepth", args=NS(weight="w", device="cuda", cov_mode="Est", extra=1)))
    raise SystemExit("excess key accepted")
except KeyError:
    pass
print("DEPTH-REGISTERED-OK")
''' % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "DEPTH-REGISTERED-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_depth_and_matcher_under_the_real_tartanvo_baseline(tmp_path):
    """Odometry/BaselineTartanVO.TartanVO on a TartanVOStereo.yaml-shaped config with depth: B200_TartanVODepth and match:
    B200_TartanVOMatcher (torch-op head path and the matcher's kernel answered by the oracle, on the CPU) against the same run
    with the reference TartanVODepth and TartanVOMatcher, with the driver repairs of
    test_tartanvo_matcher.test_matcher_under_the_real_tartanvo_baseline; the depth outputs (99 % of pixels within 1e-3 relative) and the
    trajectories agree"""
    from tests import test_tartanvo_matcher as tm
    code = tm.BASELINE_CODE
    # both plugins instead of the matcher alone; the depth network with the synthetic StereoCovNet weights
    code = code.replace('torch.save({"module." + k: v for k, v in StereoCovNet(cfg_sc).state_dict().items()}, sys.argv[2])',
                        'from tests.golden import make_golden_tartanvo_depth as dgen\ndgen.write_checkpoint(sys.argv[2])')
    code = code.replace('depth=NS(type="TartanVODepth", args=NS(weight=sys.argv[2], device="cpu", cov_mode="Est"))',
                        'depth=(NS(type="B200_TartanVODepth", args=NS(weight=sys.argv[2], device="cpu", cov_mode="Est", '
                        'cuda_graph=False)) if b200 else NS(type="TartanVODepth", args=NS(weight=sys.argv[2], device="cpu", '
                        'cov_mode="Est")))')
    code = code.replace('TartanVO.is_valid_config(NS(**dict(vars(cfg), match=NS(type=cfg.match.type, args=NS(**dict(vars(cfg.match.args), device="cuda"))))))',
                        'TartanVO.is_valid_config(NS(**dict(vars(cfg), match=NS(type=cfg.match.type, args=NS(**dict(vars(cfg.match.args), device="cuda"))), '
                        'depth=NS(type=cfg.depth.type, args=NS(**dict(vars(cfg.depth.args), device="cuda"))))))')
    code = code.replace('''    est = odo.match_estimator.estimate''', '''    assert type(odo.depth_estimator).__name__ == ("B200_TartanVODepth" if b200 else "TartanVODepth")
    dest = odo.depth_estimator.estimate
    def dspy(*a, **k):
        out = dest(*a, **k)
        depths.append((out.depth.clone(), out.cov.clone()))
        return out
    odo.depth_estimator.estimate = dspy
    est = odo.match_estimator.estimate''')
    code = code.replace("flows = []\n", "flows = []\ndepths = []\n")
    code = code.replace("ref_flows = list(flows); flows.clear()", "ref_flows = list(flows); flows.clear()\nref_depths = list(depths); depths.clear()")
    code = code.replace('print("TARTANVO-BASELINE-OK"', '''assert len(depths) == len(ref_depths) > 0
for (dg, cg), (dr, cr) in zip(depths, ref_depths):
    for a, b in ((dg, dr), (cg, cr)):
        assert a.shape == b.shape == (1, 1, H, W) and torch.equal(torch.isnan(a), torch.isnan(b))
        fin = torch.isfinite(b)
        rel = ((a - b)[fin].abs() / b[fin].abs().clamp_min(1e-12)).double()
        # near-zero disparities amplify the fp32 rounding (folded BatchNorm, op order): 99 % within 1e-3 relative
        assert rel.quantile(0.99) <= 1e-3, (rel.quantile(0.99), rel.max())
print("TARTANVO-BASELINE-OK"''')
    assert code.count("B200_TartanVODepth") >= 2 and "depths.append" in code
    r = subprocess.run([sys.executable, "-c", code, str(tmp_path / "tartanvo.pkl"), str(tmp_path / "depth.pth")],
                       capture_output=True, text=True, timeout=900, env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "TARTANVO-BASELINE-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]
