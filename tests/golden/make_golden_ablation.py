"""Generate tests/golden/ablation_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_ablation.py

ablation_modifiers.pt: the reference Modifier_Diagonalize / Modifier_Normalize and both nestings, instantiated through
`ICovariance2to3.instantiate` around a fixed-output model, on tests/golden/ablation_cases.modifier_set().

ablation_observe_<case>.pt: for every covariance model of the ablation configs (ablation_cases.MODELS, built from the YAML
shape by `ICovariance2to3.instantiate`), the calls of Odometry/MACVO.py:198-283 as make_golden_observe_icp.py makes them: the
same `kp1_sigma_uv` tensor goes to `ObsCovModel.estimate` (MatchCovariance clamps it in place, NoCovariance does not), the
FilterCompose(CovarianceSanityFilter, SimpleDepthFilter, LikelyFrontOfCamFilter) chain on the MatchObs columns, cov_Tw and
the ICP_TwoframePGO constructor's buffers. Rows whose clamped 2x2 flow covariance is not finite are taken out of a
MatchCovariance estimate (the reference's pinverse raises there) and get NaN covariances, before the modifiers.

For the "planted" rows the generator reports what the reference's MatchCovariance gives for an indefinite flow covariance
(`planted` in the fixture): whether sigma_xy overflows with a finite diagonal, or every entry is NaN."""
import os
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import ablation_cases as ac, refharness  # noqa: E402


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
    from Utility.Point import filterPointsInRange, pixel2point_NED

    class FixedCovariance(ICovariance2to3):           # the modifiers' submodule for the direct set
        def estimate(self, frame, kp, depth_est, depth_cov, flow_cov):
            return self.config.covs.clone()

        @classmethod
        def is_valid_config(cls, config):
            return

    covs = ac.modifier_set()
    out = {"input_sha": ac.sha(covs), "input": covs}
    for name, (_, ops) in ac.MODELS.items():
        if name == "nocov":
            continue
        cfg = NS(type="FixedCovariance", args=NS(covs=covs))
        for op in ops:
            cfg = NS(type={"diagonalize": "Modifier_Diagonalize", "normalize": "Modifier_Normalize"}[op], args=cfg)
        out[name] = ICovariance2to3.instantiate(cfg.type, cfg.args).estimate(None, covs[:, 0], None, None, None)
    path = os.path.join(REPO, "tests", "golden", "ablation_modifiers.pt")
    torch.save(out, path)
    print(f"wrote {path}: {covs.shape[0]} matrices")

    def stereo(c, intr):
        fx, fy, cx, cy = intr
        return StereoData(T_BS=None, K=torch.tensor([[[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]]),
                          baseline=torch.tensor([0.25]), time_ns=[0], height=c["H"], width=c["W"],
                          imageL=torch.zeros(1, 3, c["H"], c["W"]), imageR=torch.zeros(1, 3, c["H"], c["W"]))

    rp = IFrontend.retrieve_pixels
    for case in ac.CASES:
        c = ac.observe_inputs(case)
        H, W, ew = c["H"], c["W"], c["edge_width"]
        frame0, frame1 = stereo(c, c["intr0"]), stereo(c, c["intr1"])
        kp0 = c["kp0"]
        kp1 = kp0 + rp(kp0, c["flow"]).T
        inb = filterPointsInRange(kp1, (ew, W - ew), (ew, H - ew))
        rows = torch.nonzero(inb).reshape(-1)
        kp0_i, kp1_i = kp0[inb], kp1[inb]
        n = kp0_i.size(0)
        kp0_d, kp1_d = rp(kp0_i, c["depth0"]).squeeze(0), rp(kp1_i, c["depth1"]).squeeze(0)
        kp0_sigma_dd, kp1_sigma_dd = rp(kp0_i, c["depth_cov0"]).squeeze(0), rp(kp1_i, c["depth_cov1"]).squeeze(0)
        pos0_Tc = pixel2point_NED(kp0_i, kp0_d, frame0.frame_K)
        fixture = {"case": case, "input_sha": ac.input_sha(c), "n_inbound": n, "k": kp0.size(0)}
        for name in ac.case_models(case):
            cov_model, ops = ac.MODELS[name]
            cfg = ac.model_config(name)
            ICovariance2to3.is_valid_config(cfg)
            model = ICovariance2to3.instantiate(cfg.type, cfg.args)
            kp0_sigma_uv = torch.ones((n, 3)) * c["match_cov_default"]
            kp0_sigma_uv[..., 2] = 0.
            kp1_sigma_uv = rp(kp0_i, c["match_cov"]).T           # the MatchObs column pixel2_uv_cov
            if cov_model == "identity":
                fin = torch.ones(n, dtype=torch.bool)
            else:
                half = c["kernel_size"] // 2
                for kp in (kp0_i, kp1_i.long()):
                    assert bool(((kp + half < torch.tensor([W, H])).all())), f"{case}: a window leaves the image"
                clamped = kp1_sigma_uv.clone()
                clamped[..., :2].clamp_(min=c["min_flow_cov"] ** 2)
                fin = torch.isfinite(clamped).all(-1)
            if bool(fin.all()):
                cov0 = model.estimate(frame0, kp0_i, IStereoDepth.Output(depth=c["depth0"]), kp0_sigma_dd, kp0_sigma_uv)
                cov1 = model.estimate(frame1, kp1_i, IStereoDepth.Output(depth=c["depth1"]), kp1_sigma_dd, kp1_sigma_uv)
            else:        # the rows the reference's pinverse would raise on: NaN covariances, then the modifiers
                sub_uv = kp1_sigma_uv[fin].clone()
                cov0 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
                cov1 = torch.full((n, 3, 3), float("nan"), dtype=torch.float64)
                cov0[fin] = model.estimate(frame0, kp0_i[fin], IStereoDepth.Output(depth=c["depth0"]), kp0_sigma_dd[fin],
                                           kp0_sigma_uv[fin])
                cov1[fin] = model.estimate(frame1, kp1_i[fin], IStereoDepth.Output(depth=c["depth1"]), kp1_sigma_dd[fin],
                                           sub_uv)
                kp1_sigma_uv[fin] = sub_uv                        # MatchCovariance's in-place clamp reaches the column
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
            sanity = FilterCompose(NS(filter_args=[NS(type="CovarianceSanityFilter", args=None)]))
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
            sane = torch.zeros(kp0.size(0), dtype=torch.bool)
            sane[rows[sanity.filter(match_obs, torch.device("cpu"))]] = True
            fixture[name] = {"keep": keep, "sanity_keep": sane, "n_obs": m,
                             "pixel1_uv": kp0_i[keep_i], "pixel2_uv": kp1_i[keep_i], "pixel2_uv_cov": kp1_sigma_uv[keep_i],
                             "pixel2_d": kp1_d[keep_i], "obs1_covTc": cov0[keep_i], "obs2_covTc": cov1[keep_i],
                             "points_Tc": torch.as_tensor(graph.points_Tc).as_subclass(torch.Tensor).float().clone(),
                             "cov_Tw": torch.as_tensor(graph.pts_covTw).as_subclass(torch.Tensor).clone()}
            if name not in ("nocov", "norm"):     # (cov_Tw of the other models: R obs1_covTc R^T, checked from obs1_covTc)
                del fixture[name]["cov_Tw"]
            if case == "planted":
                at = {int(r): i for i, r in enumerate(rows.tolist())}
                fixture[name]["planted"] = {r: (cov1[at[r]].clone() if r in at else None) for r in ac.PLANTED}
            print(f"{case:9s} {name:8s} in range {n}, kept {m}")
        if case == "planted":
            for r, cv in fixture["diag"]["planted"].items():
                raw = fixture_raw(c, rows, r, frame1)
                print(f"planted row {r}: MatchCovariance gives {raw}")
            fixture["planted_match"] = {r: fixture_raw(c, rows, r, frame1, as_tensor=True) for r in ac.PLANTED}
        path = os.path.join(REPO, "tests", "golden", f"ablation_observe_{case}.pt")
        torch.save(fixture, path)
        print(f"wrote {path}: {os.path.getsize(path) / 1024:.0f} KiB")


def fixture_raw(c, rows, r, frame1, as_tensor=False):
    """the reference MatchCovariance's frame-1 covariance of planted row r, no modifier"""
    from Module.Covariance.Project2to3 import MatchCovariance
    from Module.Frontend.Frontend import IFrontend
    from Module.Frontend.StereoDepth import IStereoDepth
    kp0 = c["kp0"][r:r + 1]
    kp1 = kp0 + IFrontend.retrieve_pixels(kp0, c["flow"]).T
    uv = IFrontend.retrieve_pixels(kp0, c["match_cov"]).T.clone()
    covm = MatchCovariance(NS(device="cpu", **ac.MATCH_ARGS))
    cov = covm.estimate(frame1, kp1, IStereoDepth.Output(depth=c["depth1"]), None, uv)[0]
    if as_tensor:
        return cov
    off = cov[[0, 0, 1, 1, 2, 2], [1, 2, 0, 2, 0, 1]]
    return (f"diagonal finite: {bool(torch.isfinite(cov.diagonal()).all())}, off-diagonal finite: "
            f"{bool(torch.isfinite(off).all())}, sigma_xy {float(cov[1, 2])}")


if __name__ == "__main__":
    main()
