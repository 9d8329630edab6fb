"""pipeline.FusedTartanVO and plugins.B200_TartanVO on the H100: the fused driver's trajectory against the three B200
plugins driven in BaselineTartanVO.run's order (bit for bit), graph replay against the eager path, keyframe handling, no
host synchronisation per frame, and the errors."""
from types import SimpleNamespace as NS

import pytest
import torch

DEV = "cuda"
pytestmark = pytest.mark.gpu
SHAPES = {"tartanair": (480, 640), "kitti": (376, 780), "euroc": (480, 752)}


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    return ops


@pytest.fixture(autouse=True)
def _restore_precision_flags():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev[:2]
        torch.set_float32_matmul_precision(prev[2])


def _set_flags(strict: bool) -> None:
    if strict:
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        torch.set_float32_matmul_precision("highest")
    else:                                                   # torch's defaults
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = True


def _plugins(cov_mode: str, cuda_graph: bool = True):
    from macvo_b200 import plugins as P
    return (P.B200_TartanVOMatcher(NS(weight="synthetic:0", device=DEV, cuda_graph=cuda_graph)),
            P.B200_TartanVODepth(NS(weight="synthetic:0", device=DEV, cov_mode=cov_mode, cuda_graph=cuda_graph)),
            P.B200_TartanMotionNet(NS(weight="synthetic:0", device=DEV)))


def _frames(n: int, H: int, W: int, pin: bool = False, seed: int = 1000):
    """StereoFrames of the synthetic sequence, each with its own T_BS and time"""
    from macvo_b200 import synthetic
    from macvo_b200.interfaces import StereoFrame
    out = []
    for i, sd in enumerate(synthetic.make_sequence(n, H, W, seed=seed, pin=pin)):
        sd.T_BS = torch.tensor([[0.01 * i, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]])
        out.append(StereoFrame(idx=[i], time_ns=sd.time_ns, stereo=sd))
    return out


def _fused(frames, freq: int, cuda_graph: bool = True):
    from macvo_b200.pipeline import FusedTartanVO
    vo = FusedTartanVO(*_plugins("None", cuda_graph), keyframe_freq=freq, cuda_graph=cuda_graph)
    for f in frames:
        vo.run(f)
    return vo, *vo.finish()


def _plugin_sequence(frames, freq: int):
    """B200_TartanVOMatcher.estimate, B200_TartanVODepth.estimate (Est) and B200_TartanMotionNet.predict / update in
    BaselineTartanVO.run's order (Odometry/BaselineTartanVO.py:35-60)"""
    matcher, depth, motion = _plugins("Est")
    poses, interp, prev = [], [], None
    for f in frames:
        if f.frame_idx % freq:
            poses.append(poses[-1])
            interp.append(True)
            continue
        flow = matcher.estimate(prev.stereo, f.stereo).flow if prev is not None else None
        est_depth = depth.estimate(f.stereo)
        pose = motion.predict(f, flow, est_depth.depth)
        poses.append(motion._tensor(pose).cpu())
        interp.append(False)
        motion.update(pose)
        prev = f
    return torch.stack(poses), torch.tensor(interp)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("strict", [False, True], ids=["default", "strict"])
@pytest.mark.parametrize("freq", [1, 3])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_fused_matches_plugin_sequence(lib, shape, freq, strict):
    """the same trajectory, bit for bit (NaN positions included), as the plugins driven one by one"""
    _set_flags(strict)
    frames = _frames(7, *SHAPES[shape])
    ref, ref_interp = _plugin_sequence(frames, freq)
    vo, got, interp = _fused(frames, freq)
    assert got.shape == (7, 7) and got.dtype == torch.float32
    assert torch.equal(interp, ref_interp)
    assert torch.equal(_bits(got), _bits(ref)), (shape, freq, strict, got, ref)
    assert vo.num_keyframes == len(range(0, 7, freq))
    # at 376x780 the pose crop reads the matcher's NaN border; macvo_posenet_conv's ReLU (fmaxf) maps the NaN it meets to 0,
    # so the device poses stay finite where the reference's are NaN (INTEGRATION.md, tests/golden/tartanvo_vo_kitti.pt)
    assert torch.isfinite(got).all() and (got[freq:, :3] - got[0, :3]).abs().max() > 1e-4


# measured deviation from the reference trajectory (tests/golden/tartanvo_vo_*.pt), max over all pose elements, on one H100
# 80GB HBM3 at 700 W; asserted at about 1.5x (DESIGN.md §2.2.4)
# (strict fp32: 3.0e-7 / 6.0e-8 / 2.6e-8 for small_f1 / small_f3 / tartanair; default flags: 1.08e-5 / 4.1e-6 / 8.9e-6)
FIXTURE_BOUND = {"strict": 4.5e-7, "default": 1.6e-5}


@pytest.mark.parametrize("strict", [False, True], ids=["default", "strict"])
@pytest.mark.parametrize("name", ["small_f1", "small_f3", "tartanair", "kitti"])
def test_fused_matches_reference_fixture(lib, golden, name, strict):
    from macvo_b200.interfaces import StereoData, StereoFrame
    from tests.golden import make_golden_tartanvo_vo as gen
    _set_flags(strict)
    g = golden(f"tartanvo_vo_{name}.pt")
    H, W, n, freq = gen.CASES[name]
    K, bl = gen.camera(H, W)
    frames = [StereoFrame(idx=[t], time_ns=[t * 100_000_000], stereo=StereoData(
        T_BS=torch.tensor([[0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]]), K=K.clone(), baseline=torch.tensor([bl]),
        time_ns=[t * 100_000_000], height=H, width=W, imageL=left, imageR=right))
        for t, (left, right) in enumerate(gen.frames(name))]
    _, got, interp = _fused(frames, freq)
    assert torch.equal(interp, g["need_interp"])
    ref = g["pose"]
    if name == "kitti":     # the reference is NaN from the second keyframe on; the device is not (see above)
        assert torch.isnan(ref[1:]).all() and torch.equal(got[0], ref[0]) and torch.isfinite(got).all()
        return
    err = (got - ref).abs().max().item()
    print(f"[fixture] {name} {'strict' if strict else 'default'} max |pose - reference| = {err:.3e}")
    assert err <= FIXTURE_BOUND["strict" if strict else "default"], err


@pytest.mark.parametrize("strict", [False, True], ids=["default", "strict"])
def test_graph_replay_matches_eager(lib, strict):
    _set_flags(strict)
    frames = _frames(5, 480, 752)
    _, graphed, _ = _fused(frames, 1, cuda_graph=True)
    _, eager, _ = _fused(frames, 1, cuda_graph=False)
    assert torch.equal(_bits(graphed), _bits(eager))


def test_no_host_synchronisation_per_frame(lib):
    """after the first two keyframes (set-up and graph capture), 10 frames from pinned memory run with every
    synchronising CUDA call an error; the host never waits"""
    frames = _frames(12, 480, 640, pin=True)
    from macvo_b200.pipeline import FusedTartanVO
    vo = FusedTartanVO(*_plugins("None"), keyframe_freq=1)
    vo.run(frames[0])
    vo.run(frames[1])
    torch.cuda.set_sync_debug_mode("error")
    try:
        for f in frames[2:]:
            vo.run(f)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert vo.host_waits == [0] * 12
    got, _ = vo.finish()
    _, ref, _ = _fused(_frames(12, 480, 640), 1)
    assert torch.equal(_bits(got), _bits(ref))


def test_pageable_frames_go_through_staging(lib):
    """frames in pageable memory give the same trajectory as pinned ones"""
    _, pinned, _ = _fused(_frames(6, 480, 640, pin=True), 1)
    vo, pageable, _ = _fused(_frames(6, 480, 640), 1)
    assert vo._staging is not None and len(vo.host_waits) == 6
    assert torch.equal(_bits(pinned), _bits(pageable))


def test_keyframes_carry_pose_and_T_BS(lib):
    """keyframe_freq 3: a non-keyframe has the previous pose and T_BS with need_interp True, and the matcher sees
    consecutive keyframes' left images"""
    frames = _frames(8, 480, 640)
    from macvo_b200.pipeline import FusedTartanVO
    vo = FusedTartanVO(*_plugins("None", cuda_graph=False), keyframe_freq=3, cuda_graph=False)
    seen = []
    run = vo.matcher._run

    def spy(images, flow_out, margin, crop):
        seen.append(images.cpu())
        return run(images, flow_out, margin, crop)
    vo.matcher._run = spy
    for f in frames:
        vo.run(f)
    poses, interp = vo.finish()
    assert interp.tolist() == [False, True, True, False, True, True, False, True]
    for i in range(8):
        k = i - i % 3
        assert torch.equal(poses[i], poses[k])
        assert torch.equal(vo.frames[i]["T_BS"], frames[k].stereo.T_BS)
        assert vo.frames[i]["time_ns"] == frames[i].stereo.time_ns
    assert len(seen) == 2
    for images, (a, b) in zip(seen, ((0, 3), (3, 6))):
        assert torch.equal(images[0:1], frames[a].stereo.imageL) and torch.equal(images[1:2], frames[b].stereo.imageL)
    assert not torch.equal(poses[3], poses[0])


def test_errors(lib):
    from macvo_b200.pipeline import FusedTartanVO
    with pytest.raises(ValueError, match="cov_mode"):
        FusedTartanVO(*_plugins("Est"))
    frames = _frames(2, 480, 640)
    vo = FusedTartanVO(*_plugins("None"))
    for f in frames:
        vo.run(f)
    other = _frames(3, 480, 752)[2]
    with pytest.raises(AssertionError, match="image shape changed"):
        vo.run(other)
    moved = _frames(3, 480, 640)[2]
    moved.stereo.baseline = torch.tensor([0.5])
    with pytest.raises(AssertionError, match="baseline \\* fx changed"):
        vo.run(moved)


def test_drop_in_builds_the_map(lib):
    """B200_TartanVO from a TartanVOStereo.yaml-shaped section (cov_mode Est is accepted, the decoder is not run): the
    map's columns and the fused trajectory"""
    from macvo_b200 import plugins as P
    cfg = NS(name="TartanVOStereo",
             depth=NS(type="B200_TartanVODepth", args=NS(weight="synthetic:0", device=DEV, cov_mode="Est")),
             match=NS(type="B200_TartanVOMatcher", args=NS(weight="synthetic:0", device=DEV)),
             tartanvo=NS(weight="synthetic:0", device=DEV),
             keyframe=NS(type="UniformKeyframe", args=NS(keyframe_freq=2)))
    odo = P.B200_TartanVO.from_config(cfg, None)
    assert not odo.fused.depth.est_cov
    frames = _frames(5, 480, 640)
    for f in frames:
        odo.run(f)
    odo.terminate()
    data = odo.get_map().frames.data
    col = lambda k: data[k].tensor
    _, ref, ref_interp = _fused(frames, 2)
    assert torch.equal(_bits(col("pose")), _bits(ref)) and torch.equal(col("need_interp"), ref_interp)
    assert col("K").shape == (5, 3, 3) and col("baseline").shape == (5,) and col("time_ns").dtype == torch.long
    assert col("T_BS").shape == (5, 7) and torch.equal(col("T_BS")[3], frames[2].stereo.T_BS[0])
    assert col("time_ns").tolist() == [f.stereo.time_ns[0] for f in frames]
