"""Generate tests/golden/tartanvo_vo_*.pt by running the MAC-VO tree's TartanVO baseline driver itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_tartanvo_vo.py

For each case of CASES the unmodified Odometry/BaselineTartanVO.TartanVO is built by its own `from_config` from a
TartanVOStereo.yaml-shaped Odometry section (TartanVOMatcher, TartanVODepth with cov_mode Est, the hard-wired
TartanMotionNet, UniformKeyframe), fed frame by frame through `run`, then `terminate` and `get_map`. Weights: the synthetic
PWC-Net and pose network (macvo_b200.pwcnet / posenet synthetic_*_state_dict(0)) in one StereoVONet checkpoint, and the
synthetic StereoCovNet (macvo_b200.stereonet.synthetic_stereo_state_dict(0)).

Substitutions, as in make_golden_tartanvo_flow.py: `cupy` is a stub module, `FunctionCorrelation` is
oracle.pwc.correlation and `torch.Tensor.cuda` is the identity. The driver's two defects are repaired exactly as
tests/test_tartanvo_matcher.py::BASELINE_CODE repairs them: a "Naive" IMapProcessor that leaves the map as it is, and the
leading dimension on the motion model's first (identity) pose.

Frames (FRAMES): frame t is the window at (2t, 3t) of a larger image pair of the Vanilla fixtures' generator
(tests/golden/cases.net_inputs), so consecutive frames move by (2, 3) pixels; fx = fy = 320, c = the image centre,
baseline 0.25, T_BS the identity, time_ns = 10^8 t.

Stored per case: the inputs' sha256, the map's pose (F,7), need_interp, T_BS and time_ns, and per keyframe after the first
its motion (the se3 of TartanStereoVOMotion.inference) and every STRIDE-th row and column of its flow and depth."""
import os
import sys
import tempfile
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import cases, tartanvo_cases  # noqa: E402

SEED = 0
STRIDE = 7
CASES = {                       # name: (H, W, frames, keyframe_freq)
    "small_f1": (264, 328, 8, 1),
    "small_f3": (264, 328, 8, 3),
    "tartanair": (480, 640, 4, 1),
    "kitti": (376, 780, 3, 1),
}


def frames(name: str) -> list:
    """[(left, right)] (1,3,H,W) in [0, 1]: windows of one image pair moving by (2, 3) pixels per frame"""
    H, W, n, _ = CASES[name]
    left, right = cases.net_inputs(1, H + 2 * n, W + 3 * n, seed=3000)
    return [(left[..., 2 * t:2 * t + H, 3 * t:3 * t + W].contiguous(),
             right[..., 2 * t:2 * t + H, 3 * t:3 * t + W].contiguous()) for t in range(n)]


def camera(H: int, W: int) -> tuple[torch.Tensor, float]:
    return torch.tensor([[[320.0, 0.0, W / 2], [0.0, 320.0, H / 2], [0.0, 0.0, 1.0]]]), 0.25


def sha(name: str) -> str:
    return tartanvo_cases.sha(*[im for pair in frames(name) for im in pair])


def write_checkpoints(vo_path: str, depth_path: str) -> None:
    """a whole-StereoVONet checkpoint with the synthetic flowNet and flowPoseNet, and the synthetic StereoCovNet"""
    from tests.golden import make_golden_tartanvo_depth as gdepth, make_golden_tartanvo_flow as gflow
    from macvo_b200.posenet import synthetic_posenet_state_dict
    gflow.write_checkpoint(vo_path, SEED)
    sd = torch.load(vo_path, weights_only=True)
    sd.update({"module.flowPoseNet." + k: v for k, v in synthetic_posenet_state_dict(SEED).items()})
    torch.save(sd, vo_path)
    gdepth.write_checkpoint(depth_path, SEED)


def reference_driver(vo_path: str, depth_path: str, freq: int):
    """BaselineTartanVO.TartanVO.from_config on the CPU, with the substitutions and repairs of the module docstring"""
    from tests.golden import make_golden_tartanvo_flow as gflow
    gflow.reference_matcher(vo_path)                # installs the cupy stub, the correlation and the .cuda identity
    from Module.MapProcessor import IMapProcessor
    from Module.MotionModel import TartanMotionNet
    from Odometry.BaselineTartanVO import TartanVO
    if not any(c.__name__ == "Naive" for c in IMapProcessor.__subclasses__()):
        class Naive(IMapProcessor):
            """the map processor BaselineTartanVO.py:22 names and MAC-VO lacks: leaves the map as it is"""
            def elaborate_map(self, frames):
                return frames, torch.zeros((0,), dtype=torch.long)

            @classmethod
            def is_valid_config(cls, config):
                return None
    if not getattr(TartanMotionNet.predict, "_repaired", False):
        _predict = TartanMotionNet.predict

        def predict(self, frame, flow, depth):
            """the leading dimension the first (identity) pose needs in its FrameNode"""
            pose = _predict(self, frame, flow, depth)
            return pose.unsqueeze(0) if pose.dim() == 1 else pose
        predict._repaired = True
        TartanMotionNet.predict = predict
    cfg = NS(name="TartanVOStereo",
             depth=NS(type="TartanVODepth", args=NS(weight=depth_path, device="cpu", cov_mode="Est")),
             match=NS(type="TartanVOMatcher", args=NS(weight=vo_path, device="cpu")),
             tartanvo=NS(weight=vo_path, device="cpu"),
             keyframe=NS(type="UniformKeyframe", args=NS(keyframe_freq=freq)))
    TartanVO.is_valid_config(cfg)
    return TartanVO.from_config(cfg, None)


def run_case(name: str, vo_path: str, depth_path: str) -> dict:
    import pypose as pp
    from DataLoader import StereoData, StereoFrame
    H, W, n, freq = CASES[name]
    odo = reference_driver(vo_path, depth_path, freq)
    log = {"motion": [], "flow": [], "depth": []}
    inference = odo.tartanvo.model.inference

    def spy(frame, flow, depth):
        m = inference(frame, flow, depth)
        log["motion"].append(m.clone().reshape(-1))
        log["flow"].append(flow[..., ::STRIDE, ::STRIDE].clone())
        log["depth"].append(depth[..., ::STRIDE, ::STRIDE].clone())
        return m
    odo.tartanvo.model.inference = spy
    K, bl = camera(H, W)
    for t, (left, right) in enumerate(frames(name)):
        sd = StereoData(T_BS=pp.identity_SE3(1), K=K.clone(), baseline=torch.tensor([bl]), time_ns=[t * 100_000_000],
                        height=H, width=W, imageL=left, imageR=right)
        odo.run(StereoFrame(idx=[t], time_ns=[t * 100_000_000], stereo=sd))
    odo.terminate()
    data = odo.get_map().frames.data
    col = lambda k: data[k].tensor.clone()
    return {"case": name, "seed": SEED, "stride": STRIDE, "H": H, "W": W, "frames": n, "keyframe_freq": freq,
            "input_sha": sha(name), "pose": col("pose"), "need_interp": col("need_interp"), "T_BS": col("T_BS"),
            "time_ns": col("time_ns"), "motion": torch.stack(log["motion"]) if log["motion"] else torch.zeros((0, 6)),
            "flow": log["flow"], "depth": log["depth"]}


def main() -> None:
    with tempfile.TemporaryDirectory() as d:
        vo_path, depth_path = os.path.join(d, "tartanvo.pkl"), os.path.join(d, "depth.pth")
        write_checkpoints(vo_path, depth_path)
        for name in CASES:
            with torch.inference_mode():
                res = run_case(name, vo_path, depth_path)
            path = os.path.join(REPO, "tests", "golden", f"tartanvo_vo_{name}.pt")
            torch.save(res, path)
            print(f"wrote {path}: pose {res['pose'].tolist()}")


if __name__ == "__main__":
    main()
