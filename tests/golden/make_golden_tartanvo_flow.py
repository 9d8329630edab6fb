"""Generate tests/golden/tartanvo_flow_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_tartanvo_flow.py

For each case of tests/golden/tartanvo_cases.py the unmodified TartanVOMatcher.forward (Matching.py:213-223) ->
TartanStereoVOMatch.inference (StereoVO_Interface.py:124-151) -> StereoVONet.forward_flow (StereoVO.py:26-28) runs on the
CPU, with the synthetic PWC-Net weights (macvo_b200.pwcnet.synthetic_pwc_state_dict(0)) loaded by the reference's own
loadWeight from a temporary .pkl of `module.`-prefixed keys (the rest of StereoVONet keeps its initialisation).

The only substitutions, each needed because the reference's correlation is a cupy CUDA kernel:
  * `cupy` is a stub module (correlation.py imports it at module level);
  * `FunctionCorrelation` in pwc_model_tartanvo's namespace is oracle.pwc.correlation;
  * `torch.Tensor.cuda` is the identity (TartanStereoVOMatch.inference and warp() call `.cuda()`).

Stored: flow2 at 1/4 resolution, the inputs' sha256 and, for `small`, the matcher's (flow, mask) output and the per-level
LeakyReLU'd cost volumes of levels 6..4 with their inputs (f1, f2, up_flow * scale)."""
import os
import sys
import tempfile
from types import SimpleNamespace

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import refharness, tartanvo_cases  # noqa: E402

SEED = 0


def reference_matcher(weight_path: str):
    """TartanVOMatcher on the CPU with the three substitutions of the module docstring; returns (matcher, level log)"""
    refharness.install()
    sys.modules["cupy"] = refharness._StubModule("cupy")
    torch.Tensor.cuda = lambda self, *a, **k: self
    import Module.Network.PWCNet.pwc.pwc_model_tartanvo as pm
    from Module.Frontend.Matching import TartanVOMatcher
    from oracle import pwc as opwc
    log = []

    def correlation(tenFirst, tenSecond):
        log.append((tenFirst.clone(), tenSecond.clone()))
        return opwc.correlation(tenFirst, tenSecond)
    pm.FunctionCorrelation = correlation
    return TartanVOMatcher(SimpleNamespace(weight=weight_path, device="cpu")), log


def write_checkpoint(path: str, seed: int = SEED) -> None:
    """a whole-StereoVONet checkpoint (the reference loads it strictly) whose flowNet is the synthetic PWC-Net"""
    refharness.install()
    sys.modules.setdefault("cupy", refharness._StubModule("cupy"))
    from Module.Network.TartanVOStereo.StereoVO import StereoVONet
    from macvo_b200.pwcnet import synthetic_pwc_state_dict
    torch.manual_seed(1234)
    full = StereoVONet(flowNormFactor=1.0, stereoNormFactor=0.02, poseDepthNormFactor=0.25).state_dict()
    full.update({"flowNet." + k: v for k, v in synthetic_pwc_state_dict(seed).items()})
    torch.save({"module." + k: v for k, v in full.items()}, path)


def main() -> None:
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tartanvo.pkl")
        write_checkpoint(path)
        matcher, log = reference_matcher(path)
    from oracle import pwc as opwc
    flow_net = matcher.model.model.flowNet
    seen = {}
    flow_net.register_forward_hook(lambda m, a, o: seen.__setitem__("flow2", o[0][0].clone()))
    warps = []
    orig_warp = flow_net.warp
    flow_net.warp = lambda x, flo: (warps.append((x.clone(), flo.clone())), orig_warp(x, flo))[1]
    for name in tartanvo_cases.CASES:
        f1, f2 = tartanvo_cases.frames(name)
        log.clear()
        warps.clear()
        with torch.inference_mode():
            out = matcher.estimate(f1, f2)
        res = {"case": name, "seed": SEED, "input_sha": tartanvo_cases.sha(f1.imageL, f2.imageL), "flow2": seen["flow2"]}
        if name == "small":
            res.update(flow=out.flow.clone(), mask=out.mask.clone())
            # levels 6..4 (3 and 2 would take the file past 1 MB): f1, the unwarped f2, the warp's flow (up_flow * scale;
            # None at level 6) and the cost volume the network continues with (LeakyReLU'd)
            res["levels"] = [{"level": 6 - i, "f1": a, "f2": warps[i - 1][0] if i else b,
                              "flow": warps[i - 1][1] if i else None,
                              "corr": torch.nn.functional.leaky_relu(opwc.correlation(a, b), 0.1)}
                             for i, (a, b) in enumerate(log[:3])]
        path = os.path.join(REPO, "tests", "golden", f"tartanvo_flow_{name}.pt")
        torch.save(res, path)
        print(f"wrote {path}: flow2 {tuple(res['flow2'].shape)} |flow2| max {res['flow2'].abs().max().item():.4g}")


if __name__ == "__main__":
    main()
