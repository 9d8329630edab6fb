"""Generate tests/golden/mixture_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_mixture.py

mixture_standalone.pt: per case of mixture_cases.CASES, the reference GaussianMixtureCovariance (instantiated from the
README's YAML with the case's kernel_size) on the case's keypoints: its (K,3,3) result, the flow covariance after its
in-place clamp, and the tolerance scale S of oracle.mixture.mixture_bound.

mixture_observe_<case>.pt: the calls of Odometry/MACVO.py:198-283 as make_golden_ablation.py makes them, with
GaussianMixtureCovariance as ObsCovModel (depth_est.cov = depth_cov0 / depth_cov1) plain and under each modifier
(mixture_cases.MODELS): keep mask, the MatchObs columns, the FilterCompose chain, cov_Tw and the ICP_TwoframePGO
constructor's buffers, plus S of each kept row's covariances before the modifiers.

Refuses any input where a reference filter weight lies within 1e-5 relative of the 1e-3 threshold."""
import os
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from oracle import mixture as omix  # noqa: E402
from tests.golden import mixture_cases as mc, refharness  # noqa: E402


class Bundle:
    def __init__(self, data):
        self.data = data

    def __len__(self):
        return next(iter(self.data.values())).shape[0]


def main() -> None:
    refharness.install()
    import pypose as pp
    from DataLoader import StereoData
    from Module.Covariance.Project2to3 import ICovariance2to3
    from Module.Frontend.Frontend import IFrontend
    from Module.Frontend.StereoDepth import IStereoDepth
    from Module.OutlierFilter import FilterCompose
    from Module.Optimization.TwoFramePGO.Graphs import GraphInput, ICP_TwoframePGO
    from Utility.Math import gaussain_full_kernels
    from Utility.Point import filterPointsInRange, pixel2point_NED

    def refuse_ties(flow_cov, n, ks, what):
        """the reference's own weights, from the flow covariance the model used (clamped, or the default)"""
        if flow_cov is None:
            flow_cov = torch.ones((n, 3)) * mc.REF_ARGS["match_cov_default"]
            flow_cov[..., 2] = 0.
        cov2 = torch.stack([torch.stack([flow_cov[:, 0], flow_cov[:, 2]], -1), torch.stack([flow_cov[:, 2], flow_cov[:, 1]], -1)], 1)
        p = gaussain_full_kernels(cov2, kernel_size=ks)
        tie = ((p - omix.PROB_THRESHOLD).abs() <= mc.TIE_RTOL * omix.PROB_THRESHOLD)
        assert not bool(tie.any()), f"{what}: a reference weight lies within 1e-5 relative of the 1e-3 threshold"

    def stereo(H, W, intr):
        fx, fy, cx, cy = intr
        return StereoData(T_BS=None, K=torch.tensor([[[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]]),
                          baseline=torch.tensor([0.25]), time_ns=[0], height=H, width=W,
                          imageL=torch.zeros(1, 3, H, W), imageR=torch.zeros(1, 3, H, W))

    out = {}
    for case in mc.CASES:
        c = mc.inputs(case)
        cfg = NS(**dict(mc.REF_ARGS, kernel_size=c["kernel_size"]))
        ICovariance2to3.is_valid_config(NS(type="GaussianMixtureCovariance", args=cfg))
        model = ICovariance2to3.instantiate("GaussianMixtureCovariance", cfg)
        fc = None if c["flow_cov"] is None else c["flow_cov"].clone()
        cov = model.estimate(stereo(mc.H, mc.W, c["intr"]), c["kp"],
                             IStereoDepth.Output(depth=c["depth"], cov=c["depth_cov_map"]), c["depth_cov"], fc)
        refuse_ties(fc, c["kp"].shape[0], c["kernel_size"], case)
        out[case] = {"input_sha": mc.input_sha(c), "cov": cov, "flow_cov_clamped": fc,
                     "bound": omix.mixture_bound(**mc.oracle_call(c))}
        print(f"{case:18s} NaN rows {int(cov.isnan().any(dim=(1, 2)).sum())}")
    path = os.path.join(REPO, "tests", "golden", "mixture_standalone.pt")
    torch.save(out, path)
    print(f"wrote {path}: {os.path.getsize(path) / 1024:.0f} KiB")

    rp = IFrontend.retrieve_pixels
    for case in mc.OBSERVE_CASES:
        c = mc.observe_inputs(case)
        H, W, ew = c["H"], c["W"], c["edge_width"]
        frame0, frame1 = stereo(H, W, c["intr0"]), stereo(H, W, c["intr1"])
        kp0 = c["kp0"]
        kp1 = kp0 + rp(kp0, c["flow"]).T
        inb = filterPointsInRange(kp1, (ew, W - ew), (ew, H - ew))
        rows = torch.nonzero(inb).reshape(-1)
        kp0_i, kp1_i = kp0[inb], kp1[inb]
        n = kp0_i.size(0)
        kp0_d, kp1_d = rp(kp0_i, c["depth0"]).squeeze(0), rp(kp1_i, c["depth1"]).squeeze(0)
        kp0_sigma_dd, kp1_sigma_dd = rp(kp0_i, c["depth_cov0"]).squeeze(0), rp(kp1_i, c["depth_cov1"]).squeeze(0)
        pos0_Tc = pixel2point_NED(kp0_i, kp0_d, frame0.frame_K)
        depth0 = IStereoDepth.Output(depth=c["depth0"], cov=c["depth_cov0"])
        depth1 = IStereoDepth.Output(depth=c["depth1"], cov=c["depth_cov1"])
        fixture = {"case": case, "input_sha": mc.ac.input_sha(c), "n_inbound": n, "k": kp0.size(0)}
        half = c["kernel_size"] // 2
        for kp in (kp0_i, kp1_i.long()):
            assert bool(((kp + half < torch.tensor([W, H])).all())), f"{case}: a window leaves the image"
        for name in mc.MODELS:
            cfg = mc.model_config(name)
            ICovariance2to3.is_valid_config(cfg)
            model = ICovariance2to3.instantiate(cfg.type, cfg.args)
            kp0_sigma_uv = torch.ones((n, 3)) * c["match_cov_default"]
            kp0_sigma_uv[..., 2] = 0.
            kp1_sigma_uv = rp(kp0_i, c["match_cov"]).T           # the MatchObs column pixel2_uv_cov
            clamped = kp1_sigma_uv.clone()
            clamped[..., :2].clamp_(min=c["min_flow_cov"] ** 2)
            fin = torch.isfinite(clamped).all(-1)
            refuse_ties(None, n, c["kernel_size"], f"{case} kp0")
            refuse_ties(clamped[fin], int(fin.sum()), c["kernel_size"], f"{case} kp1")
            sub_uv = kp1_sigma_uv[fin].clone()
            cov0 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
            cov1 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
            cov0[fin] = model.estimate(frame0, kp0_i[fin], depth0, kp0_sigma_dd[fin], kp0_sigma_uv[fin])
            cov1[fin] = model.estimate(frame1, kp1_i[fin], depth1, kp1_sigma_dd[fin], sub_uv)
            kp1_sigma_uv[fin] = sub_uv                            # the in-place clamp reaches the column
            match_obs = Bundle({"pixel1_uv": kp0_i, "pixel2_uv": kp1_i, "pixel1_d": kp0_d.unsqueeze(-1),
                                "pixel2_d": kp1_d.unsqueeze(-1), "pixel1_d_cov": kp0_sigma_dd.unsqueeze(-1),
                                "pixel2_d_cov": kp1_sigma_dd.unsqueeze(-1), "obs1_covTc": cov0, "obs2_covTc": cov1,
                                "pixel2_uv_cov": kp1_sigma_uv})
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
            b0 = omix.mixture_bound(kp0_i[keep_i], c["depth0"], c["depth_cov0"], kp0_sigma_uv[keep_i], *c["intr0"],
                                    c["kernel_size"], c["min_flow_cov"], c["match_cov_default"])
            b1 = omix.mixture_bound(kp1_i[keep_i], c["depth1"], c["depth_cov1"], kp1_sigma_uv[keep_i], *c["intr1"],
                                    c["kernel_size"], c["min_flow_cov"], c["match_cov_default"])
            fixture[name] = {"keep": keep, "n_obs": m, "pixel1_uv": kp0_i[keep_i], "pixel2_uv": kp1_i[keep_i],
                             "pixel2_uv_cov": kp1_sigma_uv[keep_i], "pixel2_d": kp1_d[keep_i], "obs1_covTc": cov0[keep_i],
                             "obs2_covTc": cov1[keep_i], "bound0": b0, "bound1": b1,
                             "points_Tc": torch.as_tensor(graph.points_Tc).as_subclass(torch.Tensor).float().clone(),
                             "cov_Tw": torch.as_tensor(graph.pts_covTw).as_subclass(torch.Tensor).clone()}
            print(f"{case:9s} {name:12s} in range {n}, kept {m}")
        path = os.path.join(REPO, "tests", "golden", f"mixture_observe_{case}.pt")
        torch.save(fixture, path)
        print(f"wrote {path}: {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
