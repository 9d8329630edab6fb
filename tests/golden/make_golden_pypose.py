"""Generate tests/golden/pypose_jacobian.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_pypose.py

The two-frame graph Analytic_ReprojDisp_TwoFramePGO (Module/Optimization/TwoFramePGO/Graphs.py:121-148, 201-230) on the
seeded K = 48 case of tests/golden/cases.py at a pose far from identity: its residual `forward()` and its analytic
`build_jacobian()`. tests/test_pypose_conventions.py checks the oracle's residual and the pypose shim's update rule
against these two arrays."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tests.golden import cases, refharness  # noqa: E402

K = 48
START_XI = np.array([0.3, -0.1, 0.2, 0.25, -0.2, 0.15])          # se3 vector of the linearisation pose


def main() -> None:
    refharness.install()
    import pypose as pp
    from Module.Map import MatchObs, PointNode
    from Module.Optimization.TwoFramePGO.Graphs import Analytic_ReprojDisp_TwoFramePGO, GraphInput
    from oracle import pgo as opgo
    c = cases.pgo_inputs(K, 6)
    obs = MatchObs.init({
        "pixel1_uv": torch.zeros(K, 2), "pixel2_uv": c["kp2_uv"], "pixel1_d": torch.zeros(K, 1), "pixel2_d": torch.zeros(K, 1),
        "pixel1_disp": torch.zeros(K, 1), "pixel2_disp": c["kp2_disp"].unsqueeze(-1),
        "pixel1_disp_cov": torch.zeros(K, 1), "pixel2_disp_cov": c["disp_cov"].unsqueeze(-1),
        "pixel1_d_cov": torch.zeros(K, 1), "pixel2_d_cov": torch.zeros(K, 1),
        "pixel1_uv_cov": torch.zeros(K, 3), "pixel2_uv_cov": c["uv_cov"],
        "obs1_covTc": torch.zeros(K, 3, 3, dtype=torch.double), "obs2_covTc": torch.zeros(K, 3, 3, dtype=torch.double)})
    pts = PointNode.init({"pos_Tw": c["pos_Tw"], "cov_Tw": torch.zeros(K, 3, 3, dtype=torch.double),
                          "color": torch.zeros(K, 3, dtype=torch.uint8)})
    start = torch.tensor(opgo.se3_exp(START_XI), dtype=torch.float32)
    gi = GraphInput(torch.tensor([1]), torch.tensor([0]), pp.SE3(start.unsqueeze(0)), torch.tensor([c["baseline"]]), obs, pts,
                    c["K"], torch.zeros(K, dtype=torch.long), "cpu")
    graph = Analytic_ReprojDisp_TwoFramePGO(gi).to(dtype=torch.double)
    with torch.no_grad():
        out = {"K": K, "start": start, "residual": graph.forward().clone().reshape(K, 3),
               "jacobian": graph.build_jacobian().reshape(K, 3, 7).clone(),
               "pose": graph.pose2opt.detach().clone().reshape(7)}
    path = os.path.join(REPO, "tests", "golden", "pypose_jacobian.pt")
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
