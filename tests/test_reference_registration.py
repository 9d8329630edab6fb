"""Drop-in check against the REAL MAC-VO tree (skipped where no MAC-VO tree is found, see tests/golden/refharness):
importing `macvo_b200.plugins` with MAC-VO importable registers the B200 classes in MAC-VO's own registries,
`Module.I<X>.instantiate` finds them by name and `is_valid_config` accepts the INTEGRATION.md YAML args.
Runs in a subprocess so that the reference import does not leak into the other tests."""
import os
import subprocess
import sys

import pytest

from tests.golden import refharness

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CODE = r'''
import sys
sys.path.insert(0, %r)
from tests.golden import refharness
refharness.install()
from types import SimpleNamespace as NS
import Module
import macvo_b200.plugins as P
assert P._REF, "plugins did not detect the MAC-VO tree"
from Module import IFrontend, IKeypointSelector, ICovariance2to3, IOptimizer
assert IFrontend.get_class("B200_FlowFormerCovFrontend") is P.B200_FlowFormerCovFrontend
assert IKeypointSelector.get_class("B200_CovAwareSelector_NoDepth") is P.B200_CovAwareSelector_NoDepth
assert IKeypointSelector.get_class("B200_MappingPointSelector") is P.B200_MappingPointSelector
assert ICovariance2to3.get_class("B200_MatchCovariance") is P.B200_MatchCovariance
assert IOptimizer.get_class("B200_TwoFrame_PGO") is P.B200_TwoFrame_PGO
from Module.Optimization.TwoFramePGO.Optimizer import TwoFrame_PGO
assert issubclass(P.B200_TwoFrame_PGO, TwoFrame_PGO)
# the interface-level validators MACVO.is_valid_config calls (Odometry/MACVO.py:137-156)
IFrontend.is_valid_config(NS(type="B200_FlowFormerCovFrontend", args=NS(device="cuda", weight="./Model/MACVO_FrontendCov.pth",
    enc_dtype="fp32", dec_dtype="fp32", decoder_depth=12, enforce_positive_disparity=False, cuda_graph=True)))
IKeypointSelector.is_valid_config(NS(type="B200_CovAwareSelector_NoDepth", args=NS(device="cuda", kernel_size=7, mask_width=32, max_match_cov=100.0)))
IKeypointSelector.is_valid_config(NS(type="B200_MappingPointSelector", args=NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)))
ICovariance2to3.is_valid_config(NS(type="B200_MatchCovariance", args=NS(device="cuda", kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)))
IOptimizer.is_valid_config(NS(type="B200_TwoFrame_PGO", args=NS(device="cuda", vectorize=True, parallel=False, graph_type="disp", autodiff=False)))
try:
    IKeypointSelector.is_valid_config(NS(type="B200_CovAwareSelector_NoDepth", args=NS(device="cuda", kernel_size=7, mask_width=32, max_match_cov=100.0, extra=1)))
    raise SystemExit("excess key accepted")
except KeyError:
    pass
try:
    P.B200_MatchCovariance(NS(device="cpu", kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25))
    raise SystemExit("cpu device accepted")
except ValueError:
    pass
print("REGISTERED-OK")
''' % REPO


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_plugins_register_into_macvo_registry():
    r = subprocess.run([sys.executable, "-c", CODE], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "REGISTERED-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_local_interfaces_registry_and_config_spec():
    from types import SimpleNamespace as NS
    from macvo_b200 import interfaces as I
    from macvo_b200 import plugins as P
    if not P._REF:
        assert I.IFrontend.get_class("B200_FlowFormerCovFrontend") is P.B200_FlowFormerCovFrontend
        I.IKeypointSelector.is_valid_config(NS(type="B200_MappingPointSelector",
                                               args=NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)))
        with pytest.raises(KeyError):
            P.B200_MappingPointSelector.is_valid_config(NS(max_depth=5.0, max_depth_cov=0.005))
        with pytest.raises(KeyError):
            I.IFrontend.get_class("NoSuchFrontend")
    with pytest.raises(ValueError):
        P.B200_CovAwareSelector_NoDepth(NS(device="cpu", kernel_size=7, mask_width=32, max_match_cov=100.0))
