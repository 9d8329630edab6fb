"""The two-frame pose-graph kernel (csrc/pgo.cu) for every graph type ("disp", "reproj", "icp") against the float64 oracle
(oracle.pgo, pinned to the reference's LM by the pgo_* goldens):

  * the 55 packed normal-equation entries at every block count where the warp-per-block split and the cluster reduction
    change shape (one warp, warp tails, the automatic cluster thresholds at 256 / 768 / 2048), every cluster size, at the
    identity and at a pose 0.1 rad / 0.3 m away;
  * icp blocks shaped like MAC-VO's 2D->3D covariances (long thin ellipsoids along the viewing ray, condition up to ~5e7),
    whose weight must be torch.pinverse's: the normal equations, the full LM solve and its accept / reject sequence;
  * the pixel blocks of "disp" / "reproj" through a condition sweep 1e6 .. 1e16, against the exact pseudo-inverse;
  * rank-deficient and non-finite icp blocks;
  * the loss-only evaluation (lane per block) behind stats[2].

Tolerances: normal equations 1e-10 of each section's largest entry (1e-8 for the MAC-VO-shaped icp blocks, whose pinv is
itself only that well determined at condition 5e7); pose 1e-8 like tests/test_gpu_kernels.py; loss 1e-12.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import pgo as opgo
from tests.golden import cases

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRAPH_TYPES = ("disp", "reproj", "icp")
IDENTITY = np.array([0., 0., 0., 0., 0., 0., 1.])
FAR = opgo.se3_exp(np.array([0.2, -0.15, 0.15, 0.06, -0.05, 0.06]))       # ~0.3 m, ~0.1 rad
SECTIONS = {"A": slice(0, 21), "b": slice(21, 27), "G": slice(27, 48), "h": slice(48, 54), "loss": slice(54, 55)}


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from macvo_b200 import build, ops as _ops
    build.build(verbose=False)
    _ops.load_library()
    return _ops


def _intr(g):
    return (g.fx, g.fy, g.cx, g.cy, g.baseline)


def _columns(g) -> dict:
    """the graph's float64 columns on the device, exactly the values the oracle reads"""
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)
    return dict(kp2_uv=t(g.kp2_uv), kp2_disp=t(g.kp2_disp), uv_cov=t(g.uv_cov), disp_cov=t(g.disp_cov), pc_obs=t(g.pc_obs),
                obs_cov=t(g.obs_cov), pts_cov=t(g.pts_cov))


def _accumulate(ops, g, pose, cluster):
    col = _columns(g)
    flag = torch.zeros(1, dtype=torch.float64, device=DEV)
    acc = ops.pgo_accumulate(torch.from_numpy(g.pos_Tw).to(DEV), col.pop("kp2_uv"), col.pop("kp2_disp"), col.pop("uv_cov"),
                             col.pop("disp_cov"), _intr(g), torch.from_numpy(pose).to(DEV), graph_type=g.graph_type,
                             cluster=cluster, singular_flag=flag, **col)
    return acc.cpu().numpy(), flag.item()


def _solve(ops, g, cluster):
    pose, stats = ops.pgo_solve_graph(g.graph_type, torch.from_numpy(g.pos_Tw).to(DEV), _intr(g),
                                      torch.from_numpy(g.init_pose).to(DEV), cluster=cluster, **_columns(g))
    return pose.cpu().numpy(), stats.cpu().numpy()


def _pinv_weights(g, pose):
    return np.stack([np.linalg.pinv(c, rcond=1e-15) for c in g.cov_blocks(pose)])


def _assert_packed(acc, ref, rtol, what=""):
    """every section of the packed accumulator within rtol of its largest reference entry"""
    for name, s in SECTIONS.items():
        scale = max(np.abs(ref[s]).max(), 1e-300)
        err = np.abs(acc[s] - ref[s]).max()
        assert err <= rtol * scale, f"{what} {name}: max error {err:.3e} = {err / scale:.2e} of {scale:.3e}"


def _full_rank_by_pinv(blocks) -> bool:
    s = np.linalg.svd(blocks, compute_uv=False)
    return bool((s[:, -1] > 1e-15 * s[:, 0]).all())


# ---- normal equations, every graph type ---------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 7, 8, 255, 256, 257, 4096])
@pytest.mark.parametrize("graph_type", GRAPH_TYPES)
def test_normal_equations_every_graph_type(ops, graph_type, K):
    """one warp (1 .. 8 blocks), warp tails (255, 257), the automatic cluster sizes (256 -> 2, 4096 -> 8) and every
    explicit one: the same 55 entries as oracle.pgo.accumulate_packed"""
    g = cases.pgo_graph(cases.pgo_inputs_typed(graph_type, K, 6))
    for pose in (IDENTITY, FAR):
        ref = opgo.accumulate_packed(g, pose)
        for cluster in (0, 1, 2, 3, 8):
            acc, flag = _accumulate(ops, g, pose, cluster)
            _assert_packed(acc, ref, 1e-10, f"{graph_type} K={K} cluster={cluster}")
            assert flag == 0.0


def test_normal_equations_independent_of_cluster_size(ops):
    """the reduction runs in a fixed order per cluster size; the sums of different sizes agree to rounding"""
    g = cases.pgo_graph(cases.pgo_inputs_typed("icp", 4096, 6))
    accs = [_accumulate(ops, g, FAR, cluster)[0] for cluster in range(1, 9)]
    for a in accs[1:]:
        _assert_packed(a, accs[0], 1e-12)
    again, _ = _accumulate(ops, g, FAR, 5)
    assert np.array_equal(again, accs[4]), "same cluster size, same bits"


# ---- MAC-VO-shaped icp covariances --------------------------------------------------------------------------------------
MACVO_FX = sorted(cases.PGO_MACVO_CAMERAS)


@pytest.mark.parametrize("fx", MACVO_FX)
def test_icp_macvo_covariances_normal_equations(ops, fx):
    """Project2to3 covariances of the same point in two frames: every block is full rank by pinv's cutoff (condition
    < 1e9), so the weight is its inverse and nothing is flagged, also for the blocks whose det / (m00 m11 m22) < 1e-13"""
    g = cases.pgo_graph(cases.pgo_inputs_macvo(2048, 1, fx))
    for pose in (IDENTITY, FAR):
        assert _full_rank_by_pinv(g.cov_blocks(pose))
        ref = opgo.accumulate_packed(g, pose, W=_pinv_weights(g, pose))
        for cluster in (1, 3, 8):
            acc, flag = _accumulate(ops, g, pose, cluster)
            _assert_packed(acc, ref, 1e-8, f"fx={fx} cluster={cluster}")
            assert flag == 0.0


@pytest.mark.parametrize("fx", MACVO_FX)
def test_icp_macvo_covariances_solve(ops, fx):
    """the full LM solve at the MAC-VO-shaped blocks: pose 1e-8 against oracle.pgo.lm_solve, the same number of steps and
    loss evaluations, no block flagged, for every cluster size"""
    g = cases.pgo_graph(cases.pgo_inputs_macvo(2048, 1, fx))
    trace = opgo.LMTrace()
    ref = opgo.lm_solve(g, trace=trace)
    for cluster in range(1, 9):
        pose, s = _solve(ops, g, cluster)
        np.testing.assert_allclose(pose, ref, rtol=1e-8, atol=1e-9, err_msg=f"cluster {cluster}")
        assert (int(s[0]), int(s[1])) == (trace.steps, trace.evaluations), f"cluster {cluster}"
        assert s[7] == 0.0


# ---- pixel blocks of "disp" / "reproj": condition sweep -----------------------------------------------------------------
def _exact_pinv2(a: float, b: float, c: float):
    """Moore-Penrose inverse of [[a, c], [c, b]] in exact rational arithmetic, for a full-rank or an exactly rank-1 block"""
    a, b, c = Fraction(a), Fraction(b), Fraction(c)
    det = a * b - c * c
    if det != 0:
        return [float(b / det), float(a / det), float(-c / det)]
    tr2 = (a + b) ** 2
    return [float(a / tr2), float(b / tr2), float(c / tr2)]


def _pixel_sweep_blocks():
    """(uu, vv, uv, full rank by pinv): axis-aligned blocks of condition 1e6 .. 1e16 (their pseudo-inverse is exact in
    float64), and rotated ones with small-integer entries scaled by a power of two, so that uu * vv - uv^2 is exact:
    [[p^2, pq - 1], [pq - 1, q^2]] (condition ~(p^2 + q^2)^2 / 2pq, 1e6 .. 1e8) and the exactly rank-1 [[p^2, pq], [pq, q^2]]"""
    out = []
    for cond in (1e6, 1e8, 1e10, 1e12, 1e14, 3e14, 3e15, 1e16, 1e18):
        out.append((4.0, 4.0 / cond, 0.0, cond < 1e15))
        out.append((4.0 / cond, 4.0, 0.0, cond < 1e15))
    s = 2.0 ** -22
    for p, q in ((700, 700), (2236, 2237), (7071, 7072), (5000, 9000)):
        out.append((p * p * s, q * q * s, (p * q - 1) * s, True))
        out.append((q * q * s, p * p * s, -(p * q - 1) * s, True))
        out.append((p * p * s, q * q * s, p * q * s, False))
    return out


@pytest.mark.parametrize("graph_type", ["disp", "reproj"])
def test_pixel_covariance_condition_sweep(ops, graph_type):
    """every pixel block gets torch.pinverse's weight: the inverse while the small eigenvalue is above 1e-15 of the
    largest of the block (disp: of the 3x3 with the disparity variance), the rank-1 weight below, flagged only then"""
    sweep = _pixel_sweep_blocks()
    c = cases.pgo_inputs_typed(graph_type, 2 * len(sweep), 6)
    g = cases.pgo_graph(c)
    W = np.zeros((g.pos_Tw.shape[0], 3, 3))
    for i in range(g.pos_Tw.shape[0]):
        uu, vv, uv, _ = sweep[i % len(sweep)]
        g.uv_cov[i] = (uu, vv, uv)
        e = g.disp_cov[i] if graph_type == "disp" else 1.0
        if uv == 0.0:                                 # diagonal: keep each variance above 1e-15 of the largest
            big = max(uu, vv, e)
            W[i] = np.diag([1 / x if x > 1e-15 * big else 0.0 for x in (uu, vv, e)])
        else:
            w00, w11, w01 = _exact_pinv2(uu, vv, uv)
            W[i] = [[w00, w01, 0.0], [w01, w11, 0.0], [0.0, 0.0, 1 / e]]
    for pose in (IDENTITY, FAR):
        ref = opgo.accumulate_packed(g, pose, W=W)
        for cluster in (1, 2):
            acc, flag = _accumulate(ops, g, pose, cluster)
            _assert_packed(acc, ref, 1e-10, f"{graph_type} cluster={cluster}")
            assert flag == 1.0
    # only the full-rank blocks: nothing is flagged
    keep = np.array([sweep[i % len(sweep)][3] for i in range(g.pos_Tw.shape[0])])
    sub = cases.pgo_graph(c)
    for name in ("pos_Tw", "kp2_uv", "kp2_disp", "uv_cov", "disp_cov"):
        setattr(sub, name, np.ascontiguousarray(getattr(g, name)[keep]))
    acc, flag = _accumulate(ops, sub, FAR, 1)
    _assert_packed(acc, opgo.accumulate_packed(sub, FAR, W=W[keep]), 1e-10, graph_type)
    assert flag == 0.0


# ---- degenerate icp blocks ----------------------------------------------------------------------------------------------
def _degenerate_icp(K=64):
    """icp blocks whose R obs_cov R^T + pts_cov has rank 2 (both ways of making it), rank 1 and 0; integer vectors so the
    products are exact at the identity"""
    c = cases.pgo_inputs_typed("icp", K, 6)
    g = cases.pgo_graph(c)
    a, b = np.array([3.0, -1.0, 2.0]) / 8, np.array([1.0, 4.0, -2.0]) / 8
    z = np.zeros((3, 3))
    for k, (so, sp) in {3: (np.outer(a, a) + np.outer(b, b), z), 11: (np.outer(a, a), np.outer(b, b)),
                        5: (z, np.outer(a, a)), 19: (np.outer(b, b), z), 9: (z, z)}.items():
        g.obs_cov[k], g.pts_cov[k] = so, sp
    return g


def test_icp_rank_deficient_blocks_take_pseudo_inverse_weight(ops):
    """rank-2, rank-1 and zero blocks: the Moore-Penrose weight of np.linalg.pinv(rcond=1e-15), flagged, in the normal
    equations and through the solve"""
    g = _degenerate_icp()
    for pose in (IDENTITY, FAR):
        ref = opgo.accumulate_packed(g, pose)
        for cluster in (1, 2):
            acc, flag = _accumulate(ops, g, pose, cluster)
            _assert_packed(acc, ref, 1e-10, f"cluster={cluster}")
            assert flag == 1.0
    trace = opgo.LMTrace()
    ref = opgo.lm_solve(g, trace=trace)
    for cluster in (1, 2, 8):
        pose, s = _solve(ops, g, cluster)
        np.testing.assert_allclose(pose, ref, rtol=1e-8, atol=1e-9)
        assert (int(s[0]), int(s[1])) == (trace.steps, trace.evaluations)
        assert s[7] == 1.0


def test_icp_non_finite_block_keeps_zero_weight(ops):
    """a NaN / inf covariance (the sanity filter removes those upstream) contributes no weight and sets the flag; its
    residual still enters G, h and the loss"""
    g = cases.pgo_graph(cases.pgo_inputs_typed("icp", 64, 6))
    g.obs_cov[13][1, 1] = np.nan
    g.pts_cov[17][0, 2] = g.pts_cov[17][2, 0] = np.inf
    bad = {13, 17}
    for pose in (IDENTITY, FAR):
        W = np.stack([np.zeros((3, 3)) if k in bad else np.linalg.pinv(cb, rcond=1e-15)
                      for k, cb in enumerate(g.cov_blocks(pose))])
        acc, flag = _accumulate(ops, g, pose, 1)
        _assert_packed(acc, opgo.accumulate_packed(g, pose, W=W), 1e-10)
        assert flag == 1.0


# ---- loss-only evaluation -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph_type", GRAPH_TYPES)
def test_loss_only_path(ops, graph_type):
    """stats[2] is the lane-per-block loss evaluation at the returned pose: oracle.pgo.robust_loss there to 1e-12"""
    graphs = [cases.pgo_graph(cases.pgo_inputs_typed(graph_type, K, 6)) for K in (7, 257, 4096)]
    if graph_type == "icp":
        graphs.append(cases.pgo_graph(cases.pgo_inputs_macvo(2048, 1, 1000.0)))
    for g in graphs:
        for cluster in (1, 3, 8):
            pose, s = _solve(ops, g, cluster)
            np.testing.assert_allclose(s[2], opgo.robust_loss(g, pose, 0.1), rtol=1e-12)
