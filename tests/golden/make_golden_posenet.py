"""Generate tests/golden/posenet_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_posenet.py

For each case of tests/golden/posenet_cases.py: FlowPoseNet.VOFlowRes(config=1, stereo=True, down_scale=True,
intrinsic=True) with the synthetic weights (macvo_b200.posenet.synthetic_posenet_state_dict(0)), driven by the unmodified
TartanStereoVOMotion.inference (StereoVO_Interface.py:158-194) — the object is built without its __init__, so neither
PWC-Net nor cupy is needed — and TartanMotionNet.predict's composition (MotionModel.py:101-112) on the pypose shim.
Stored: the network input the reference built, its motion, the prior and predicted poses, the inputs' sha256."""
import os
import sys
from types import SimpleNamespace

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import posenet_cases, refharness  # noqa: E402

SEED = 0


def main() -> None:
    refharness.install()
    import pypose as pp
    from Module.Network.TartanVOStereo.FlowPoseNet import VOFlowRes
    from Module.Network.TartanVOStereo.StereoVO_Interface import TartanStereoVOMotion
    from Module.MotionModel import TartanMotionNet
    from macvo_b200.posenet import synthetic_posenet_state_dict
    net = VOFlowRes(config=1, stereo=True, down_scale=True, intrinsic=True)
    net.load_state_dict(synthetic_posenet_state_dict(SEED))
    net.eval()
    seen = {}
    net.register_forward_pre_hook(lambda m, args: seen.__setitem__("input", args[0].clone()))
    motion_net = TartanStereoVOMotion.__new__(TartanStereoVOMotion)
    motion_net.device = "cpu"
    motion_net.model = SimpleNamespace(flowPoseNet=net, stereoNormFactor=0.02, poseDepthNormFactor=0.25)
    motion_net.pose_norm = torch.tensor([0.13, 0.13, 0.13, 0.013, 0.013, 0.013], dtype=torch.float)
    motion_net.flow_norm = 0.05
    for name in posenet_cases.CASES:
        c = posenet_cases.posenet_inputs(name)
        K = torch.tensor([[[c["fx"], 0.0, c["cx"]], [0.0, c["fy"], c["cy"]], [0.0, 0.0, 1.0]]])
        meta = SimpleNamespace(height=c["H"], width=c["W"], fx=c["fx"], fy=c["fy"], cx=c["cx"], cy=c["cy"],
                               frame_baseline=c["baseline"], K=K)
        frame = SimpleNamespace(stereo=meta)
        model = TartanMotionNet.__new__(TartanMotionNet)
        model.config = SimpleNamespace(device="cpu", weight="synthetic")
        model.model = motion_net
        model.prev_pose = pp.SE3(c["prev_pose"])
        with torch.inference_mode():
            motion = motion_net.inference(frame, c["flow"], c["depth"]).clone()
            nxt = model.predict(frame, c["flow"], c["depth"])
        out = {"case": name, "seed": SEED, "input_sha": posenet_cases.sha(c["flow"], c["depth"]),
               "net_input": seen["input"], "motion": motion, "prev_pose": c["prev_pose"],
               "next_pose": nxt.tensor().clone() if hasattr(nxt, "tensor") else nxt.clone()}
        path = os.path.join(REPO, "tests", "golden", f"posenet_{name}.pt")
        torch.save(out, path)
        print(f"wrote {path}: motion {motion.tolist()}")


if __name__ == "__main__":
    main()
