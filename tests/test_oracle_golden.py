"""The CPU oracle (oracle/) pinned against fixtures produced by the reference itself
(tests/golden/make_golden.py). No GPU, no MAC-VO tree needed."""
import numpy as np
import pytest
import torch

from oracle import covariance as ocov
from oracle import frontend as ofe
from oracle import keypoint as okp
from oracle import pgo as opgo
from tests.golden import cases


@pytest.mark.parametrize("name", list(cases.CORR_CASES))
def test_corr_volume(golden, name):
    g = golden(f"corr_{name}.pt")
    B, H1, W1 = g["shape"]
    f1, f2 = cases.corr_inputs(B, H1, W1)
    out = ofe.corr_volume(f1, f2)
    assert out.shape == (B, 1, H1, W1, H1, W1)
    rows, cols = cases.corr_sample_index(H1 * W1)
    sample = out.reshape(B, H1 * W1, H1 * W1)[:, rows][:, :, cols]
    assert torch.equal(sample, g["sample"])                         # same torch.bmm -> bit-identical
    assert out.double().sum() == g["sum"]


@pytest.mark.parametrize("name", list(cases.LOOKUP_CASES))
def test_window_lookup(golden, name):
    g = golden(f"lookup_{name}.pt")
    B, H1, W1 = g["shape"]
    cost_maps, coords = cases.lookup_inputs(B, H1, W1)
    keep = coords.clone()
    out = ofe.window_lookup(cost_maps, coords)
    assert torch.equal(coords, keep)                                # the oracle must not mutate its input
    assert torch.equal(out, g["out"])
    loops = ofe.window_lookup_loops(cost_maps, coords)
    torch.testing.assert_close(loops, g["out"], rtol=1e-5, atol=1e-5)


def test_window_lookup_axis_quirk():
    """x-ramp cost map: window axis 0 (the slow output-channel axis) steps in x (SURVEY.md §7.3)."""
    H1, W1 = 10, 10
    ramp = torch.arange(W1, dtype=torch.float32).view(1, 1, 1, W1).expand(H1 * W1, 1, H1, W1).contiguous()
    coords = torch.full((1, 2, H1, W1), 4.0)
    out = ofe.window_lookup(ramp, coords)[0, :, 0, 0].view(9, 9)
    assert torch.allclose(out[:, 0], torch.arange(0., 9.), atol=1e-5)   # i -> x offset
    assert torch.allclose(out[4, :], torch.full((9,), 4.0), atol=1e-5)  # j -> y offset (no change on an x-ramp)


@pytest.mark.parametrize("epd", [0, 1])
def test_dense_postproc(golden, epd):
    g = golden(f"dense_small_{epd}.pt")
    H, W = g["shape"]
    flow, cov = cases.dense_inputs(H, W)
    out = ofe.dense_postproc(flow, cov, torch.tensor([0.25]).item(), torch.tensor(320.0).item(), bool(epd))
    for k in ("depth", "disparity", "depth_cov", "disparity_uncertainty", "flow", "flow_cov"):
        assert torch.equal(out[k].nan_to_num(123.0), g[k].nan_to_num(123.0)), k
    if epd:
        assert torch.equal(out["depth_mask"], g["depth_mask"])
    else:
        assert out["depth_mask"] is None and g["depth_mask"] is None


@pytest.mark.parametrize("name", list(cases.SELECTOR_CASES))
def test_selectors_bit_exact(golden, name):
    g = golden(f"selector_{name}.pt")
    H, W = g["shape"]
    flow, cov = cases.selector_inputs(H, W, g["variant"])
    d = ofe.dense_postproc(flow, cov, 0.25, 320.0)
    mm = cases.selector_match_mask(H, W) if g["variant"] == "masked" else None
    torch.manual_seed(cases.SELECTOR_RNG_SEED)
    kp = okp.cov_aware_select_nodepth(d["flow_cov"], g["num"], 7, 32, 100.0, mm)
    mp = okp.mapping_select(d["depth"], d["depth_cov"], 2000, 5.0, 0.005, 32)
    assert kp.dtype == torch.int64 and torch.equal(kp, g["kp"])
    assert torch.equal(mp, g["map_kp"])


def _depth_selector_inputs(g):
    H, W = g["shape"]
    (f0, c0), (f1, c1) = cases.selector_depth_inputs(H, W, g["variant"])
    d0 = ofe.dense_postproc(f0, c0, 0.25, 320.0, g["variant"] == "masked")
    d1 = ofe.dense_postproc(f1, c1, 0.25, 320.0)
    m0 = ~d0["depth_mask"] if g["variant"] == "masked" else None
    mm = cases.selector_match_mask(H, W) if g["variant"] == "masked" else None
    return d0, d1, m0, mm


@pytest.mark.parametrize("name", list(cases.SELECTOR_DEPTH_CASES))
def test_depth_aware_selector_bit_exact(golden, name):
    g = golden(f"selector_{name}.pt")
    d0, d1, m0, mm = _depth_selector_inputs(g)
    torch.manual_seed(cases.SELECTOR_RNG_SEED)
    kp = okp.cov_aware_select(d1["flow_cov"], d0["depth"], d0["depth_cov"], d1["depth"], d1["depth_cov"], g["num"],
                              7, 32, 320.0 * 0.25, 250.0, 100.0, m0, mm)
    assert torch.equal(kp, g["kp"])


def test_selector_empty_nms_set_gives_no_keypoints():
    """torch.median([]) is nan and python's min(max, nan) keeps max: the reference returns 0 keypoints, no error"""
    cov = torch.full((1, 3, 96, 128), float("nan"))
    assert okp.cov_aware_select_nodepth(cov, 10).shape == (0, 2)


@pytest.mark.parametrize("name", list(cases.COV_CASES))
def test_match_covariance(golden, name):
    g = golden(f"covariance_{name}.pt")
    H, W, K = g["shape"]
    kp, depth, flow_cov = cases.cov_inputs(H, W, K, g["kind"])
    out = ocov.match_covariance(kp, depth, flow_cov, 320.0, 320.0, W / 2, H / 2)
    assert out.dtype == torch.float64 and out.shape == (K, 3, 3)
    assert torch.equal(out, g["out"])
    if flow_cov is not None:                                        # in-place clamp of the caller's tensor
        assert torch.equal(flow_cov, g["flow_cov_after"])
        assert flow_cov[:, :2].min() >= 0.0625


@pytest.mark.parametrize("name", list(cases.PGO_CASES))
def test_pgo_against_reference_lm(golden, name):
    """numpy restatement vs the reference's LM_analytic + Analytic_ReprojDisp_TwoFramePGO run on the
    pypose shim (same control flow => same accept/reject sequence; fp64 rounding only)."""
    g = golden(f"pgo_{name}.pt")
    c = cases.pgo_inputs(g["K"], g["seed"])
    pose = opgo.lm_solve(cases.pgo_graph(c))
    ref = g["pose"].double().numpy()
    np.testing.assert_allclose(pose, ref, rtol=1e-9, atol=1e-10)
    # and it actually solves the problem: close to the generating pose
    true = c["true_pose"].numpy()
    assert np.abs(pose[:3] - true[:3]).max() < 0.05 and np.abs(pose[3:] - true[3:]).max() < 0.01


def test_pgo_jacobian_finite_difference():
    c = cases.pgo_inputs(64, 6)
    g = cases.pgo_graph(c)
    pose = opgo.se3_exp(np.array([0.3, -0.1, 0.2, 0.05, -0.04, 0.03]))
    r0, pc = opgo.residual(g, pose)
    J = opgo.jacobian(g, pose, pc)
    assert np.all(J[:, :, 6] == 0)
    for k in range(6):
        e = np.zeros(7)
        e[k] = 1e-6
        rp, _ = opgo.residual(g, opgo.retract(pose, e))
        rm, _ = opgo.residual(g, opgo.retract(pose, -e))
        np.testing.assert_allclose((rp - rm) / 2e-6, J[:, :, k], rtol=2e-5, atol=2e-5)


def test_se3_group_identities():
    rng = np.random.default_rng(0)
    for _ in range(5):
        a, b = opgo.se3_exp(rng.normal(size=6) * 0.5), opgo.se3_exp(rng.normal(size=6) * 0.5)
        p = rng.normal(size=(4, 3))
        np.testing.assert_allclose(opgo.se3_act(opgo.se3_mul(a, b), p), opgo.se3_act(a, opgo.se3_act(b, p)), atol=1e-12)
        np.testing.assert_allclose(opgo.se3_act(opgo.se3_inv(a), opgo.se3_act(a, p)), p, atol=1e-12)
        np.testing.assert_allclose(opgo.quat_matrix(a[3:]) @ p[0], opgo.quat_rot(a[3:], p[0]), atol=1e-12)
    np.testing.assert_allclose(opgo.se3_exp(np.zeros(6)), [0, 0, 0, 0, 0, 0, 1])


# ---- network class on the CPU vs the reference network's golden outputs ----------------------------------------------
@pytest.mark.parametrize("name", list(cases.NET_CASES))
def test_network_class_cpu_matches_reference_golden(golden, name):
    """`FlowFormerCovNet` (the functional re-implementation every CPU leg and the GPU path share) on the CPU with the
    oracle's correlation / lookup vs the REFERENCE network's fp32 output (net_*.pt, flownet.py:37-44): both are fp32
    MKL runs of the same arithmetic in different association order -> 1e-5 of the output scale (measured: flow 1.9e-5
    absolute on a scale of 19.5 = 1e-6 relative, covariance 1.5e-5 relative)."""
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    from oracle import frontend as ofe
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        g = golden(f"net_{name}.pt")
        B, H, W = g["shape"]
        img1, img2 = cases.net_inputs(B, H, W)
        net = FlowFormerCovNet(synthetic_state_dict(0), "cpu", corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup)
        flow, cov = net.inference(img1, img2)
    finally:
        torch.set_float32_matmul_precision(prev)
    scale = g["flow"].abs().mean().item()
    assert (flow - g["flow"]).abs().max().item() <= 1e-5 * scale, (flow - g["flow"]).abs().max().item() / scale
    assert ((cov - g["cov"]).abs() / g["cov"].abs()).max().item() <= 1e-4


def test_cfgA_fixture_records_the_fp32_noise_floor(golden):
    """net_cfgA.pt (640x480, depth 12): the reference's own fp32 run sits 2.6e-6 (flow, relative to the mean flow) and
    1.4e-4 (covariance, relative) from exact arithmetic — north_star's 1e-4 is below what fp32 itself delivers for the
    covariance; the GPU bounds (tests/test_gpu_parity_ladder.py) are stated as multiples of this floor."""
    g = golden("net_cfgA.pt")
    f = g["floor"]
    assert f["flow_abs_max"] / f["flow_scale"] < 5e-6 and 5e-5 < f["cov_rel_max"] < 5e-4
    assert f["class_fp32_vs_ref32_flow_abs_max"] / f["flow_scale"] < 5e-6
    assert len(g["truth"]["flow_iter"]) == 12 and g["truth"]["flow"].dtype == torch.float64


def test_golden_inputs_reproduce_bit_for_bit(golden):
    """Every fixture records the sha256 of the seeded inputs it was generated from; the generators (tests/golden/cases.py)
    use exactly rounded operations only, so this host must regenerate the same bits. Regression test of the round-1
    "flaky" dense post-processing test: its inputs came from `torch.exp` (MKL VML), which is not run-to-run reproducible
    on the GPU hosts."""
    for name, digest in cases.golden_input_shas().items():
        assert golden(name)["input_sha"] == digest, f"{name}: inputs generated on this host differ from the fixture's"


@pytest.mark.parametrize("name", list(cases.MOTION_CASES))
def test_motion_interpolate_oracle_matches_reference(golden, name):
    """oracle/map_processor.py vs the reference's MotionInterpolate.elaborate_map (MapProcessor.py:52-79) executed on the
    pypose shim: incl. runs of consecutive lost frames, flags inside the protected first / last two motions, F = 3 and 5."""
    from oracle import map_processor as omp
    g = golden(f"motion_{name}.pt")
    poses, need = cases.motion_inputs(g["F"], g["seed"], g["flagged"])
    out, idx = omp.motion_interpolate(poses.numpy(), need.numpy())
    np.testing.assert_allclose(out, g["out"].numpy(), rtol=0, atol=2e-6 * max(1.0, float(g["out"].abs().max())))
    assert idx.tolist() == g["interp_idx"].tolist()
    flagged_motion = [i - 1 for i in g["flagged"] if 2 <= i - 1 < g["F"] - 3]
    assert idx.tolist() == sorted(flagged_motion)


@pytest.mark.parametrize("name", list(cases.PGO_TYPE_CASES))
def test_pgo_other_graph_types_against_reference_lm(golden, name):
    """graph types "icp" (Paper_Reproduce.yaml; pose-dependent covariance R Sigma_obs R^T + Sigma_pts re-inverted before every
    step) and "reproj" vs the reference's LM_analytic + Analytic_ICP_TwoframePGO / Analytic_Reproj_TwoFramePGO on the shim"""
    g = golden(f"pgo_{name}.pt")
    c = cases.pgo_inputs_typed(g["graph_type"], g["K"], g["seed"])
    pose = opgo.lm_solve(cases.pgo_graph(c))
    np.testing.assert_allclose(pose, g["pose"].double().numpy(), rtol=1e-8, atol=1e-9)
    true = c["true_pose"].numpy()
    assert np.abs(pose[:3] - true[:3]).max() < 0.1 and np.abs(pose[3:] - true[3:]).max() < 0.02
