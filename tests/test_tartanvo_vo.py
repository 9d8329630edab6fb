"""The TartanVO baseline's driver on the CPU: the oracle chain (oracle/pwc.py, oracle/stereo.py, oracle/posenet.py in
BaselineTartanVO.run's order) against the reference trajectories (tests/golden/tartanvo_vo_*.pt, written by
tests/golden/make_golden_tartanvo_vo.py from the MAC-VO tree's own driver), B200_TartanVO's config validation, and, where
the MAC-VO tree is present, B200_TartanVO.receive_frames' output files against the reference driver's."""
import os
import subprocess
import sys
from types import SimpleNamespace as NS

import pytest
import torch

from tests.golden import make_golden_tartanvo_vo as gen, refharness

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", list(gen.CASES))
def test_fixture_inputs_reproduce(golden, name):
    assert gen.sha(name) == golden(f"tartanvo_vo_{name}.pt")["input_sha"]


def oracle_trajectory(name: str):
    """UniformKeyframe, the matcher on consecutive keyframes, the depth of the current one, the pose network's motion
    composed onto the previous fp32 pose: (poses (F,7), need_interp (F,), motions)"""
    from macvo_b200 import posenet, pwcnet, stereonet
    from oracle import posenet as opn, pwc as opwc, stereo as ost
    psd, ssd = pwcnet.synthetic_pwc_state_dict(gen.SEED), stereonet.synthetic_stereo_state_dict(gen.SEED)
    qsd = posenet.synthetic_posenet_state_dict(gen.SEED)
    H, W, _, freq = gen.CASES[name]
    K, bl = gen.camera(H, W)
    fx, fy, cx, cy = (K[0, 0, 0].item(), K[0, 1, 1].item(), K[0, 0, 2].item(), K[0, 1, 2].item())
    pose = torch.tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    poses, interp, motions, prev_left = [], [], [], None
    for t, (left, right) in enumerate(gen.frames(name)):
        if t % freq:
            poses.append(poses[-1])
            interp.append(True)
            continue
        if prev_left is not None:
            flow, _, _ = opwc.match(psd, prev_left, left)
            depth, _ = ost.estimate(ssd, left, right, bl * fx, dtype=torch.float32)
            x = opn.network_input(flow, depth, H, W, fx, fy, cx, cy, bl)
            m = opn.motion(opn.forward(qsd, x)["pose"])
            motions.append(m)
            pose = opn.compose(pose, m).float()
        poses.append(pose)
        interp.append(False)
        prev_left = left
    return torch.stack(poses), torch.tensor(interp), motions


@pytest.mark.parametrize("name", list(gen.CASES))
def test_oracle_chain_reproduces_the_reference_trajectory(golden, name):
    """bit for bit, NaN positions included: at 376x780 (KITTI after Preprocess.yaml) the pose network's crop (rows
    20..355) reaches past the matcher's (rows 28..347) into its NaN padding, and the reference's trajectory is NaN from
    the second keyframe on"""
    g = golden(f"tartanvo_vo_{name}.pt")
    poses, interp, motions = oracle_trajectory(name)
    bits = lambda t: t.contiguous().view(torch.int32)
    assert torch.equal(interp, g["need_interp"])
    assert torch.equal(torch.isnan(poses), torch.isnan(g["pose"]))
    assert torch.equal(bits(poses.nan_to_num()), bits(g["pose"].nan_to_num()))
    assert len(motions) == g["motion"].shape[0]
    for m, r in zip(motions, g["motion"]):
        assert torch.equal(bits(m.nan_to_num()), bits(r.nan_to_num())) and torch.equal(m.isnan(), r.isnan())
    if name == "kitti":
        assert torch.isnan(g["pose"][1:]).all() and torch.isnan(g["motion"]).all()
    else:
        assert torch.isfinite(g["pose"]).all() and (g["pose"][-1, :3] - g["pose"][0, :3]).abs().max() > 1e-3
    H, W, n, freq = gen.CASES[name]
    assert g["T_BS"].shape == (n, 7) and g["time_ns"].tolist() == [t * 100_000_000 for t in range(n)]


def _section(**over):
    sec = dict(name="TartanVOStereo",
               depth=NS(type="B200_TartanVODepth", args=NS(weight="./Model/TartanVO_depth_cov.pth", device="cuda",
                                                           cov_mode="Est")),
               match=NS(type="B200_TartanVOMatcher", args=NS(weight="./Model/MACVO_posenet.pkl", device="cuda")),
               tartanvo=NS(weight="./Model/MACVO_posenet.pkl", device="cuda"),
               keyframe=NS(type="UniformKeyframe", args=NS(keyframe_freq=1)))
    sec.update(over)
    return NS(**sec)


def test_config_validation():
    from macvo_b200 import plugins as P
    cls = P.B200_TartanVO
    cls.is_valid_config(_section())
    cls.is_valid_config(_section(keyframe=NS(type="AllKeyframe", args=NS())))
    cls.is_valid_config(_section(depth=NS(type="B200_TartanVODepth", args=NS(weight="w", device="cuda", cov_mode="None",
                                                                            cuda_graph=False))))
    with pytest.raises(ValueError, match="B200_TartanVOMatcher"):
        cls.is_valid_config(_section(match=NS(type="TartanVOMatcher", args=NS(weight="w", device="cuda"))))
    with pytest.raises(ValueError, match="B200_TartanVODepth"):
        cls.is_valid_config(_section(depth=NS(type="TartanVODepth", args=NS(weight="w", device="cuda", cov_mode="Est"))))
    with pytest.raises(KeyError):
        cls.is_valid_config(_section(optimizer=NS(type="TwoFrame_PGO", args=NS())))
    with pytest.raises(KeyError):
        cls.is_valid_config(_section(tartanvo=NS(weight="w", device="cuda", extra=1)))
    with pytest.raises(Exception):
        cls.is_valid_config(_section(tartanvo=NS(weight="w", device="cpu")))
    with pytest.raises(Exception):
        cls.is_valid_config(_section(keyframe=NS(type="UniformKeyframe", args=NS(keyframe_freq=0))))
    with pytest.raises(ValueError, match="UniformKeyframe or AllKeyframe"):
        cls.is_valid_config(_section(keyframe=NS(type="NoKeyframe", args=NS())))
    assert P.PLUGINS["odometry_tartanvo"] is cls


RECEIVE_CODE = r'''
import sys, os, tempfile, torch, numpy as np
sys.path.insert(0, %r)
os.environ["TORCHDYNAMO_DISABLE"] = "1"
from types import SimpleNamespace as NS
from tests.golden import make_golden_tartanvo_vo as gen, refharness
refharness.install()
import pypose as pp
from DataLoader import StereoData, StereoFrame
from macvo_b200 import plugins as P, pipeline
assert P._IOdometry is not object

class Sandbox:
    def __init__(self, d): self.d = d
    def path(self, name): return os.path.join(self.d, name)

name = "small_f3"
H, W, n, freq = gen.CASES[name]
K, bl = gen.camera(H, W)
seq = [StereoFrame(idx=[t], time_ns=[t * 100_000_000], stereo=StereoData(
           T_BS=pp.identity_SE3(1), K=K.clone(), baseline=torch.tensor([bl]), time_ns=[t * 100_000_000], height=H,
           width=W, imageL=l, imageR=r)) for t, (l, r) in enumerate(gen.frames(name))]
with tempfile.TemporaryDirectory() as d:
    gen.write_checkpoints(os.path.join(d, "vo.pkl"), os.path.join(d, "depth.pth"))
    ref_odo = gen.reference_driver(os.path.join(d, "vo.pkl"), os.path.join(d, "depth.pth"), freq)
    os.makedirs(os.path.join(d, "ref")); os.makedirs(os.path.join(d, "b200"))
    ref_odo.receive_frames(seq, Sandbox(os.path.join(d, "ref")))
    ref_pose = ref_odo.get_map().frames.data["pose"].tensor.clone()

    class Replay:
        """FusedTartanVO's bookkeeping (keyframes, T_BS, need_interp) with the reference's poses instead of the device"""
        def __init__(self, *a, **k):
            self.inner = pipeline.FusedTartanVO.__new__(pipeline.FusedTartanVO)
            self.inner.keyframe_freq, self.inner.frames, self.inner.host_waits = freq, [], []
            self.frames = self.inner.frames
        def run(self, frame):
            k = frame.frame_idx %% freq == 0
            prev = self.frames[-1] if self.frames else None
            self.frames.append({"K": frame.stereo.K, "baseline": frame.stereo.baseline, "time_ns": frame.stereo.time_ns,
                                "T_BS": frame.stereo.T_BS if k else prev["T_BS"], "need_interp": not k})
        def finish(self):
            return ref_pose.clone(), torch.tensor([f["need_interp"] for f in self.frames])
    pipeline.FusedTartanVO = Replay
    cfg = NS(name="TartanVOStereo",
             depth=NS(type="B200_TartanVODepth", args=NS(weight="synthetic:0", device="cuda", cov_mode="Est")),
             match=NS(type="B200_TartanVOMatcher", args=NS(weight="synthetic:0", device="cuda")),
             tartanvo=NS(weight="synthetic:0", device="cuda"),
             keyframe=NS(type="UniformKeyframe", args=NS(keyframe_freq=freq)))
    P.B200_TartanVO.is_valid_config(cfg)
    odo = P.B200_TartanVO.__new__(P.B200_TartanVO)
    P._IOdometry.__init__(odo)
    odo.fused, odo._map = Replay(), None
    odo.receive_frames(seq, Sandbox(os.path.join(d, "b200")))
    for f in ("poses.npy",):
        a, b = np.load(os.path.join(d, "ref", f)), np.load(os.path.join(d, "b200", f))
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), (f, a, b)
    a, b = np.load(os.path.join(d, "ref", "tensor_map.npz")), np.load(os.path.join(d, "b200", "tensor_map.npz"))
    assert sorted(a.files) == sorted(b.files), set(a.files) ^ set(b.files)
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, (k, a[k].dtype, b[k].dtype, a[k].shape, b[k].shape)
        if k.startswith("frames/"):
            assert np.array_equal(a[k], b[k]), k
print("RECEIVE-FRAMES-OK", len(a.files))
''' % REPO


@pytest.mark.skipif(not refharness.available(), reason="MAC-VO reference tree not present")
def test_receive_frames_writes_what_the_reference_driver_writes():
    """IOdometry.receive_frames over B200_TartanVO (its FusedTartanVO replaced by a fake that replays the reference's poses)
    writes the same poses.npy and the same tensor_map.npz keys, dtypes and shapes (and frame columns) as over the
    reference driver with its two repairs, on the small keyframe_freq 3 case"""
    r = subprocess.run([sys.executable, "-c", RECEIVE_CODE], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, TORCHDYNAMO_DISABLE="1"))
    assert "RECEIVE-FRAMES-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-3500:]
