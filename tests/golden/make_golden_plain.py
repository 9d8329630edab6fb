"""Generate tests/golden/frontend_plain_{small,odd}.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_plain.py

The Vanilla ablation's frontend, FrontendCompose(FlowFormerDepth, FlowFormerMatcher) (Module/Frontend/Frontend.py:131-155,
StereoDepth.py:99-135, Matching.py:120-154), instantiated from its YAML shape and loaded from a temporary `.pth` of the plain
synthetic weights (`synthetic_state_dict(0, covariance=False)`). Stored per case: `estimate_pair(t1, t2)` (depth, disparity,
flow) and `estimate_depth(t2)` (depth, disparity), plus the reference FlowFormerCov's flow on the same two image pairs and
the same weights (its covariance decoder added), which is asserted to lie within 1e-6 of the plain flow's scale: the
covariance branch does not feed back into the flow. The inputs come from the exactly rounded generators of
tests/golden/cases.py (`plain_cases.plain_frontend_inputs`); their sha256 is stored."""
import os
import sys
import tempfile
from types import SimpleNamespace as NS

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import cases, refharness  # noqa: E402
from tests.golden.plain_cases import BASELINE, FX, PLAIN_CASES, plain_frontend_inputs  # noqa: E402


def main() -> None:
    refharness.install()
    torch.set_num_threads(8)
    torch.set_float32_matmul_precision("highest")
    import Module  # noqa: F401  (registers every plugin class)
    from DataLoader import StereoData
    from Module.Frontend.Frontend import IFrontend
    from Module.Network.FlowFormer.configs.submission import get_cfg
    from Module.Network.FlowFormerCov import build_flowformer as build_cov
    from macvo_b200.flowformer_cov import synthetic_state_dict

    def frame(L, R, H, W):
        return StereoData(T_BS=None, K=torch.tensor([[[FX, 0., W / 2], [0., FX, H / 2], [0., 0., 1.]]]),
                          baseline=torch.tensor([BASELINE]), time_ns=[0], height=H, width=W, imageL=L, imageR=R)

    cov_net = build_cov(get_cfg(), torch.float32, torch.float32).eval()
    cov_net.load_state_dict(synthetic_state_dict(0))
    with tempfile.TemporaryDirectory() as tmp:
        weight = os.path.join(tmp, "flowformer_plain_synthetic.pth")
        torch.save(synthetic_state_dict(0, covariance=False), weight)
        args = NS(device="cpu", weight=weight)
        fe = IFrontend.instantiate("FrontendCompose", NS(depth=NS(type="FlowFormerDepth", args=args),
                                                         match=NS(type="FlowFormerMatcher", args=args)))
        for name, (H, W) in PLAIN_CASES.items():
            t1l, l2, r2 = plain_frontend_inputs(H, W)
            f1, f2 = frame(t1l, t1l, H, W), frame(l2, r2, H, W)
            depth, match = fe.estimate_pair(f1, f2)
            d_only = fe.estimate_depth(f2)
            assert depth.cov is None and depth.mask is None and depth.disparity_uncertainty is None and match.cov is None
            assert fe.provide_cov == (False, False)
            cov_stereo, _ = cov_net.inference(l2, r2)
            cov_match, _ = cov_net.inference(t1l, l2)
            scale = match.flow.abs().mean().item()
            assert (cov_match - match.flow).abs().max().item() <= 1e-6 * scale
            assert (cov_stereo[:, :1].abs() - depth.disparity).abs().max().item() <= 1e-6 * depth.disparity.abs().mean().item()
            out = {"shape": (H, W), "fx": FX, "baseline": BASELINE, "input_sha": cases.sha(t1l, l2, r2),
                   "pair": {"depth": depth.depth, "disparity": depth.disparity, "flow": match.flow},
                   "depth": {"depth": d_only.depth, "disparity": d_only.disparity},
                   "cov_flow": {"stereo": cov_stereo, "match": cov_match}}
            path = os.path.join(HERE, f"frontend_plain_{name}.pt")
            torch.save(out, path)
            print(f"wrote {path}: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()
