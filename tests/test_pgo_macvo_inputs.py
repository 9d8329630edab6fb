"""No-GPU check that the MAC-VO-shaped icp inputs (tests/golden/cases.py, pgo_inputs_macvo) are what
tests/test_gpu_pgo_graphs.py relies on: Project2to3 covariance blocks that correlate their axes so strongly that
det / (m00 m11 m22) < 1e-13 (a test of that ratio takes them for singular), yet are far from singular for
torch.pinverse (condition < 1e9, pinv == inv to 1e-8)."""
import numpy as np
import pytest

from oracle import pgo as opgo
from tests.golden import cases


@pytest.mark.parametrize("fx", sorted(cases.PGO_MACVO_CAMERAS))
def test_macvo_icp_blocks_are_ill_correlated_but_full_rank(fx):
    g = cases.pgo_graph(cases.pgo_inputs_macvo(2048, 1, fx))
    for pose in (g.init_pose, opgo.se3_exp(np.array([0.2, -0.15, 0.15, 0.06, -0.05, 0.06]))):
        blocks = g.cov_blocks(pose)
        cond = np.linalg.cond(blocks)
        assert cond.max() < 1e9 and np.quantile(cond, 0.5) > 1e4, "long thin ellipsoids, full rank by pinv's 1e-15 cutoff"
        inv = np.linalg.inv(blocks)
        pinv = np.stack([np.linalg.pinv(b, rcond=1e-15) for b in blocks])
        err = np.abs(pinv - inv).max(axis=(1, 2)) / np.abs(inv).max(axis=(1, 2))
        assert err.max() < 1e-8
        ratio = np.linalg.det(blocks) / np.abs(blocks[:, 0, 0] * blocks[:, 1, 1] * blocks[:, 2, 2])
        if fx == 1000.0:     # the long focal length reaches the band at the image corners
            assert (ratio < 1e-13).sum() >= 3, np.sort(ratio)[:5]
        assert ratio.min() < 1e-12


def test_macvo_icp_inputs_are_seeded():
    a, b = cases.pgo_inputs_macvo(64, 2, 718.0), cases.pgo_inputs_macvo(64, 2, 718.0)
    assert all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in a if k != "graph_type")
    assert not np.array_equal(a["obs_cov"], cases.pgo_inputs_macvo(64, 3, 718.0)["obs_cov"])
