"""Generate tests/golden/observe_icp_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_observe_icp.py

For each case of tests/golden/filter_cases.py (an observe_cases.py case plus depth covariance maps), the calls of
Odometry/MACVO.py:198-283 as tests/golden/make_golden_observe.py makes them, plus the gathers the Paper_Reproduce back end
reads (kp1_d, kp0_sigma_dd, kp1_sigma_dd), the reference FilterCompose(CovarianceSanityFilter, SimpleDepthFilter,
LikelyFrontOfCamFilter) on the MatchObs columns, the point registration `cov_Tw = bmm(bmm(R, pos0_covTc), R^T)` with R the
rotation matrix of the fp32 previous pose (pypose shim), and the reference ICP_TwoframePGO constructor, whose registered
buffers `points_Tc` and `pts_covTw` are stored. Rows whose (clamped) 2x2 flow covariance is not finite are taken out of the
covariance estimate, where the reference's pinverse would raise; their covariances are NaN, so the sanity filter drops them.
Stored: the keep mask, the counts, the kept rows' columns and the inputs' sha256."""
import os
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import filter_cases as fc, refharness  # noqa: E402


class Bundle:
    def __init__(self, data):
        self.data = data

    def __len__(self):
        return next(iter(self.data.values())).shape[0]


def main() -> None:
    refharness.install()
    import pypose as pp
    from DataLoader import StereoData
    from Module.Covariance.Project2to3 import MatchCovariance
    from Module.Frontend.Frontend import IFrontend
    from Module.Frontend.StereoDepth import IStereoDepth
    from Module.OutlierFilter import FilterCompose
    from Module.Optimization.TwoFramePGO.Graphs import GraphInput, ICP_TwoframePGO
    from Utility.Point import filterPointsInRange, pixel2point_NED

    def stereo(c, intr):
        fx, fy, cx, cy = intr
        return StereoData(T_BS=None, K=torch.tensor([[[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]]),
                          baseline=torch.tensor([0.25]), time_ns=[0], height=c["H"], width=c["W"],
                          imageL=torch.zeros(1, 3, c["H"], c["W"]), imageR=torch.zeros(1, 3, c["H"], c["W"]))

    for name in fc.ICP_CASES:
        c = fc.icp_inputs(name)
        H, W, ew = c["H"], c["W"], c["edge_width"]
        frame0, frame1 = stereo(c, c["intr0"]), stereo(c, c["intr1"])
        covm = MatchCovariance(NS(device="cpu", kernel_size=c["kernel_size"], min_flow_cov=c["min_flow_cov"],
                                  min_depth_cov=c["min_depth_cov"], match_cov_default=c["match_cov_default"]))
        rp = IFrontend.retrieve_pixels
        kp0 = c["kp0"]
        kp1 = kp0 + rp(kp0, c["flow"]).T
        inb = filterPointsInRange(kp1, (ew, W - ew), (ew, H - ew))
        rows = torch.nonzero(inb).reshape(-1)
        kp0_i, kp1_i = kp0[inb], kp1[inb]
        n = kp0_i.size(0)
        half = c["kernel_size"] // 2
        for kp in (kp0_i, kp1_i.long()):
            assert bool(((kp + half < torch.tensor([W, H])).all())), f"{name}: a covariance window leaves the image"
        kp0_d = rp(kp0_i, c["depth0"]).squeeze(0)
        kp1_d = rp(kp1_i, c["depth1"]).squeeze(0)
        kp0_sigma_dd = rp(kp0_i, c["depth_cov0"]).squeeze(0)
        kp1_sigma_dd = rp(kp1_i, c["depth_cov1"]).squeeze(0)
        kp0_sigma_uv = torch.ones((n, 3)) * c["match_cov_default"]
        kp0_sigma_uv[..., 2] = 0.
        kp1_sigma_uv = rp(kp0_i, c["match_cov"]).T
        clamped = kp1_sigma_uv.clone()
        clamped[..., :2].clamp_(min=c["min_flow_cov"] ** 2)
        fin = torch.isfinite(clamped).all(-1)
        pos0_Tc = pixel2point_NED(kp0_i, kp0_d, frame0.frame_K)
        # the flow-covariance branch of MatchCovariance.estimate (MACVO.py passes kp*_sigma_dd, unused on that branch)
        cov0 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
        cov1 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
        cov0[fin] = covm.estimate(frame0, kp0_i[fin], IStereoDepth.Output(depth=c["depth0"]), kp0_sigma_dd[fin],
                                  kp0_sigma_uv[fin])
        cov1[fin] = covm.estimate(frame1, kp1_i[fin], IStereoDepth.Output(depth=c["depth1"]), kp1_sigma_dd[fin],
                                  clamped[fin])
        match_obs = Bundle({"pixel1_uv": kp0_i, "pixel2_uv": kp1_i, "pixel1_d": kp0_d.unsqueeze(-1),
                            "pixel2_d": kp1_d.unsqueeze(-1), "pixel1_d_cov": kp0_sigma_dd.unsqueeze(-1),
                            "pixel2_d_cov": kp1_sigma_dd.unsqueeze(-1), "obs1_covTc": cov0, "obs2_covTc": cov1})
        chain = FilterCompose(NS(filter_args=[
            NS(type="CovarianceSanityFilter", args=None),
            NS(type="SimpleDepthFilter", args=NS(min_depth=c["min_depth"], max_depth=c["max_depth"])),
            NS(type="LikelyFrontOfCamFilter", args=None)]))
        chain.set_meta(frame0)
        keep_i = chain.filter(match_obs, torch.device("cpu"))
        prev_pose = pp.SE3(c["prev_pose"].float())
        prev_rot = prev_pose.rotation().matrix().repeat((n, 1, 1)).to(torch.float64)
        cov_Tw = torch.bmm(torch.bmm(prev_rot, cov0), prev_rot.transpose(1, 2))
        obs = NS(data={k: v[keep_i] for k, v in match_obs.data.items()})
        pts = NS(data={"pos_Tw": torch.as_tensor(pp.SE3_type.Act(prev_pose, pos0_Tc)[..., :3]).as_subclass(torch.Tensor)[keep_i],
                       "cov_Tw": cov_Tw[keep_i]})
        m = int(keep_i.sum())
        graph = ICP_TwoframePGO(GraphInput(frame_idx=torch.tensor([1]), from_idx=torch.tensor([0]),
                                           init_motion=pp.SE3(c["prev_pose"].float().unsqueeze(0)),
                                           baseline=torch.tensor([0.25]), observations=obs, points=pts,
                                           images_intrinsic=frame1.frame_K, edges_index=torch.zeros(m, dtype=torch.long),
                                           device="cpu"))
        keep = torch.zeros(kp0.size(0), dtype=torch.bool)
        keep[rows[keep_i]] = True
        out = {"case": name, "input_sha": fc.icp_sha(c), "keep": keep, "n_obs": m, "n_inbound": n, "k": kp0.size(0),
               "pixel1_uv": kp0_i[keep_i], "pixel2_uv": kp1_i[keep_i], "pixel1_d": kp0_d[keep_i], "pixel2_d": kp1_d[keep_i],
               "pixel1_d_cov": kp0_sigma_dd[keep_i], "pixel2_d_cov": kp1_sigma_dd[keep_i],
               "obs1_covTc": cov0[keep_i], "obs2_covTc": cov1[keep_i],
               "points_Tc": torch.as_tensor(graph.points_Tc).as_subclass(torch.Tensor).double().clone(),
               "cov_Tw": torch.as_tensor(graph.pts_covTw).as_subclass(torch.Tensor).clone()}
        path = os.path.join(REPO, "tests", "golden", f"observe_icp_{name}.pt")
        torch.save(out, path)
        print(f"wrote {path}: k {out['k']}, in range {n}, kept {m}, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
