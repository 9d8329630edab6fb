"""Generate tests/golden/observe_*.pt by running the MAC-VO tree itself (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_observe.py

For each case of tests/golden/observe_cases.py, the reference functions in Odometry/MACVO.py:198-283's order:
IFrontend.retrieve_pixels, filterPointsInRange, MatchCovariance.estimate (frame 0 with the constant quantisation
covariance, frame 1 with the retrieved match covariance), pixel2point_NED, CovarianceSanityFilter.filter and
pp.SE3_type.Act on the pypose shim. Where every row is finite, frame 1's call gets the retrieved covariance itself and
the stored pixel2_uv_cov is that tensor after the reference's in-place clamp. Rows whose (clamped) 2x2 flow covariance
is not finite are taken out of the estimate calls, where the reference's `pinverse` would raise, and recorded as
dropped; there pixel2_uv_cov is the same clamp applied by this script. No case has a covariance window
that leaves the image (asserted). Stored: the keep mask, the kept rows' MatchObs columns, pos_Tw, the counts and the
inputs' sha256."""
import os
import sys
from types import SimpleNamespace

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import observe_cases, refharness  # noqa: E402


def main() -> None:
    refharness.install()
    import pypose as pp
    from DataLoader import StereoData
    from Module.Covariance.Project2to3 import MatchCovariance
    from Module.Frontend.Frontend import IFrontend
    from Module.Frontend.StereoDepth import IStereoDepth
    from Module.OutlierFilter import CovarianceSanityFilter
    from Utility.Point import filterPointsInRange, pixel2point_NED

    def stereo(c, intr):
        fx, fy, cx, cy = intr
        return StereoData(T_BS=None, K=torch.tensor([[[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]]),
                          baseline=torch.tensor([0.25]), time_ns=[0], height=c["H"], width=c["W"],
                          imageL=torch.zeros(1, 3, c["H"], c["W"]), imageR=torch.zeros(1, 3, c["H"], c["W"]))

    for name in observe_cases.CASES:
        c = observe_cases.observe_inputs(name)
        H, W, ew = c["H"], c["W"], c["edge_width"]
        frame0, frame1 = stereo(c, c["intr0"]), stereo(c, c["intr1"])
        covm = MatchCovariance(SimpleNamespace(device="cpu", kernel_size=c["kernel_size"], min_flow_cov=c["min_flow_cov"],
                                               min_depth_cov=c["min_depth_cov"], match_cov_default=c["match_cov_default"]))
        kp0 = c["kp0"]
        kp1 = kp0 + IFrontend.retrieve_pixels(kp0, c["flow"]).T
        inb = filterPointsInRange(kp1, (ew, W - ew), (ew, H - ew))
        rows = torch.nonzero(inb).reshape(-1)
        kp0_i, kp1_i = kp0[inb], kp1[inb]
        n = kp0_i.size(0)
        half = c["kernel_size"] // 2
        for kp in (kp0_i, kp1_i.long()):
            assert bool(((kp + half < torch.tensor([W, H])).all())), f"{name}: a covariance window leaves the image"
        kp0_d = IFrontend.retrieve_pixels(kp0_i, c["depth0"]).squeeze(0)
        kp1_disparity = IFrontend.retrieve_pixels(kp1_i, c["disparity1"])
        kp1_sigma_disparity = IFrontend.retrieve_pixels(kp1_i, c["disp_unc1"])
        kp0_sigma_uv = torch.ones((n, 3)) * c["match_cov_default"]
        kp0_sigma_uv[..., 2] = 0.
        kp1_sigma_uv = IFrontend.retrieve_pixels(kp0_i, c["match_cov"]).T
        # estimate() clamps the diagonal in place before anything else; the same clamp on a copy tells which rows its
        # pinverse could not take
        clamped = kp1_sigma_uv.clone()
        clamped[..., :2].clamp_(min=c["min_flow_cov"] ** 2)
        fin = torch.isfinite(clamped).all(-1)
        pos0_Tc = pixel2point_NED(kp0_i, kp0_d, frame0.frame_K)
        cov0 = covm.estimate(frame0, kp0_i[fin], IStereoDepth.Output(depth=c["depth0"]), None, kp0_sigma_uv[fin])
        if bool(fin.all()):
            # MACVO.py's call: pixel2_uv_cov is the caller's tensor as estimate() left it
            cov1 = covm.estimate(frame1, kp1_i, IStereoDepth.Output(depth=c["depth1"]), None, kp1_sigma_uv)
        else:
            # rows with a non-finite 2x2 covariance taken out: pixel2_uv_cov is the copy clamped above
            kp1_sigma_uv = clamped
            cov1 = covm.estimate(frame1, kp1_i[fin], IStereoDepth.Output(depth=c["depth1"]), None, kp1_sigma_uv[fin])
        good = CovarianceSanityFilter(SimpleNamespace()).filter(
            SimpleNamespace(data={"obs1_covTc": cov0, "obs2_covTc": cov1}), torch.device("cpu"))
        keep_i = torch.zeros(n, dtype=torch.bool)
        keep_i[torch.nonzero(fin).reshape(-1)[good]] = True
        prev_pose = pp.SE3(c["prev_pose"].float())
        pos_Tw = pp.SE3_type.Act(prev_pose, pos0_Tc)[..., :3]
        keep = torch.zeros(kp0.size(0), dtype=torch.bool)
        keep[rows[keep_i]] = True
        out = {"case": name, "input_sha": observe_cases.input_sha(c), "keep": keep, "n_obs": int(keep.sum()),
               "n_inbound": n, "k": kp0.size(0), "pixel1_uv": kp0_i[keep_i], "pixel2_uv": kp1_i[keep_i],
               "pixel1_d": kp0_d[keep_i], "pixel2_disp": kp1_disparity.T[keep_i].reshape(-1),
               "pixel2_disp_cov": kp1_sigma_disparity.T[keep_i].reshape(-1), "pixel2_uv_cov": kp1_sigma_uv[keep_i],
               "obs1_covTc": cov0[good], "obs2_covTc": cov1[good],
               "pos_Tw": torch.as_tensor(pos_Tw).as_subclass(torch.Tensor)[keep_i].clone()}
        path = os.path.join(REPO, "tests", "golden", f"observe_{name}.pt")
        torch.save(out, path)
        print(f"wrote {path}: k {out['k']}, in range {n}, kept {out['n_obs']}, {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
