"""Generate tests/golden/tartanvo_depth_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_tartanvo_depth.py

For each case of CASES the unmodified TartanVODepth.estimate (StereoDepth.py:211-221) -> StereoCovNet.inference
(network.py:63-73) runs on the CPU, with the synthetic weights (macvo_b200.stereonet.synthetic_stereo_state_dict(0)) saved
as a `module.`-prefixed .pth and loaded by the reference's own load_ddp_state_dict. The one substitution: `torch.Tensor.cuda`
is the identity (StereoFeature.forward calls `.cuda()`), as in make_golden_tartanvo_flow.py.

Stored per case: depth and cov sampled every STRIDE-th row and column of the frame (STRIDE is odd, so all four output phases
of the deconvolution are sampled, and the NaN border too), the inputs' sha256 and baseline * fx. For `small` also the head
kernel's inputs on the top-left WINDOW of the half-resolution maps (xd, xc: the conv_c10 outputs of both decoders; cat0) and
the reference's depth and cov on the crop pixels those inputs fully determine (rows and columns < 2 * WINDOW - 2)."""
import os
import sys
import tempfile
from types import SimpleNamespace

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import plain_cases, refharness, tartanvo_cases  # noqa: E402

SEED = 0
STRIDE = 5
WINDOW = (16, 24)
CASES = {
    "small": (264, 328),         # near the 256 x 256 minimum crop; margins 4 / 4
    "tartanair": (480, 640),     # width margin 0
    "kitti": (376, 780),         # crop 320 x 768; margins 28 / 6
    "euroc": (480, 752),         # crop 448 x 704; margins 16 / 24
}


def frame(name: str) -> SimpleNamespace:
    """a stereo frame (the Vanilla fixtures' t2.L / t2.R texture pair) with baseline 0.25 and fx 320: bf = 80"""
    H, W = CASES[name]
    _, left, right = plain_cases.plain_frontend_inputs(H, W)
    f = tartanvo_cases.frame(left)
    f.imageR = right
    return f


def write_checkpoint(path: str, seed: int = SEED) -> None:
    from macvo_b200.stereonet import synthetic_stereo_state_dict
    torch.save({"module." + k: v for k, v in synthetic_stereo_state_dict(seed).items()}, path)


def reference_depth(weight_path: str, cov_mode: str = "Est"):
    """TartanVODepth on the CPU with `.cuda()` the identity"""
    refharness.install()
    torch.Tensor.cuda = lambda self, *a, **k: self
    from Module.Frontend.StereoDepth import TartanVODepth
    return TartanVODepth(SimpleNamespace(weight=weight_path, device="cpu", cov_mode=cov_mode))


def main() -> None:
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "TartanVO_depth_cov.pth")
        write_checkpoint(path)
        est = reference_depth(path)
    model = est.model
    seen = {}
    model.feature.stereo.conv_c10.register_forward_hook(lambda m, a, o: seen.__setitem__("xd", o.clone()))
    model.decoder.conv_c10.register_forward_hook(lambda m, a, o: seen.__setitem__("xc", o.clone()))
    model.feature.stereo.conv_c1.register_forward_hook(lambda m, a, o: seen.__setitem__("cat0", o.clone()))
    for name in CASES:
        f = frame(name)
        with torch.inference_mode():
            out = est.estimate(f)
        res = {"case": name, "seed": SEED, "stride": STRIDE, "bf": f.frame_baseline * f.fx,
               "input_sha": tartanvo_cases.sha(f.imageL, f.imageR),
               "depth": out.depth[..., ::STRIDE, ::STRIDE].clone(), "cov": out.cov[..., ::STRIDE, ::STRIDE].clone()}
        if name == "small":
            wy, wx = WINDOW
            H, W = CASES[name]
            my, mx = (H - H // 64 * 64) // 2, (W - W // 64 * 64) // 2
            res["head"] = {k: seen[k][..., :wy, :wx].clone() for k in ("xd", "xc", "cat0")}
            res["head"]["depth"] = out.depth[..., my:my + 2 * wy - 2, mx:mx + 2 * wx - 2].clone()
            res["head"]["cov"] = out.cov[..., my:my + 2 * wy - 2, mx:mx + 2 * wx - 2].clone()
        path = os.path.join(REPO, "tests", "golden", f"tartanvo_depth_{name}.pt")
        torch.save(res, path)
        dep = res["depth"][torch.isfinite(res["depth"])]
        print(f"wrote {path}: depth {tuple(out.depth.shape)} median {dep.median().item():.4g}")


if __name__ == "__main__":
    main()
