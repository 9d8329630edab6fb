"""The five B200 plugin classes driven by the REAL, unmodified `Odometry/MACVO.py` (needs a MAC-VO
tree, see tests/golden/refharness; skipped elsewhere). YAML-shaped config -> `MACVO.from_config` -> registry -> 4 frames of `MACVO.run`
(`initialize`, `run_pair`, `get_graph_data` -> `B200_TwoFrame_PGO._optimize(GraphInput)` -> `write_graph_data`,
mapping branch) -> `terminate` (MotionInterpolate). No GPU here: every C-ABI call is answered by the CPU oracle
(tests/mock_ops.py), so what this pins is the plugin HOST logic under MAC-VO's exact call pattern — the transposed
`flow_cov` view of MACVO.py:231-232, (K,1) disparities, the `pp.SE3` initial motion, CPU float64 covariances — and the
result is compared with the same sequence through MAC-VO's own reference classes (CPU): same number of observations,
same poses."""
import os
import subprocess
import sys

import pytest

from tests.golden import refharness

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CODE = r'''
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
torch.cuda.current_stream = lambda *a, **k: None     # TwoFrame_PGO._optimize only hands it to an inactive Timer (Optimizer.py:83)
torch.save(synthetic_state_dict(0), sys.argv[1])

def config(b200):
    t = (lambda n: "B200_" + n) if b200 else (lambda n: n)
    fe_args = NS(device="cpu", weight="synthetic:0" if b200 else sys.argv[1], enc_dtype="fp32", dec_dtype="fp32",
                 decoder_depth=4, enforce_positive_disparity=False)
    if b200:
        fe_args.cuda_graph = False
    return NS(Odometry=NS(name="t", args=NS(device="cpu", edgewidth=32, num_point=64, match_cov_default=0.25, profile=False, mapping=True),
        cov=NS(obs=NS(type=t("MatchCovariance"), args=NS(device="cpu", kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25))),
        keypoint=NS(type=t("CovAwareSelector_NoDepth"), args=NS(device="cpu", kernel_size=7, mask_width=32, max_match_cov=100.0)),
        mappoint=NS(type=t("MappingPointSelector"), args=(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32) if b200 else
                                                           NS(device="cpu", max_depth=5.0, max_depth_cov=0.005, mask_width=32))),
        frontend=NS(type=t("FlowFormerCovFrontend"), args=fe_args),
        motion=NS(type="StaticMotionModel", args=NS()), outlier=NS(type=t("CovarianceSanityFilter"), args=NS()),
        postprocess=NS(type=t("MotionInterpolate"), args=(NS(device="cpu") if b200 else NS())), keyframe=NS(type="AllKeyframe", args=NS()),
        optimizer=NS(type=t("TwoFrame_PGO"), args=NS(device="cpu", vectorize=True, parallel=False, graph_type=sys.argv[2], autodiff=False))))

def run(b200):
    cfg = config(b200)
    odo = MACVO[StereoFrame].from_config(cfg)
    torch.set_float32_matmul_precision("highest")     # the B200 frontend switches to "medium" like the reference CUDA frontend
    torch.manual_seed(5)
    for i, f in enumerate(synthetic.make_sequence(4, 192, 256)):
        sd = StereoData(T_BS=pp.identity_SE3(1), K=f.K, baseline=f.baseline, time_ns=f.time_ns, height=f.height,
                        width=f.width, imageL=f.imageL, imageR=f.imageR)
        odo.run(StereoFrame(idx=[i], time_ns=f.time_ns, stereo=sd))
    odo.terminate()
    m = odo.get_map()
    return m.frames.data["pose"].tensor.clone(), len(m.match), len(m.points), m.match.data["pixel2_uv_cov"].tensor.clone(), \
        m.match.data["obs2_covTc"].tensor.clone()

ref = run(False)
from tests import mock_ops
mock_ops.install()
got = run(True)
assert got[1] == ref[1] and got[2] == ref[2] and got[1] > 100, (got[1:3], ref[1:3])
assert torch.isfinite(got[0]).all()
torch.testing.assert_close(got[0], ref[0], rtol=1e-4, atol=1e-4)          # poses of all 4 frames
torch.testing.assert_close(got[3], ref[3], rtol=1e-4, atol=1e-6)          # pixel2_uv_cov: the in-place clamp reached the map
torch.testing.assert_close(got[4], ref[4], rtol=1e-3, atol=1e-9)
assert (got[3][:, :2] >= 0.0625).all()
print("MACVO-INTEGRATION-OK", got[1], got[2])
''' % REPO


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
@pytest.mark.parametrize("graph_type", ["disp", "icp", "reproj"])
def test_b200_plugins_under_the_real_macvo_run_pair(tmp_path, graph_type):
    """`disp` is MACVO_Performant / Fast, `icp` Paper_Reproduce.yaml:108; each through the real GraphInput -> plugin adapter"""
    r = subprocess.run([sys.executable, "-c", CODE, str(tmp_path / "w.pth"), graph_type], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "MACVO-INTEGRATION-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]
