"""Frames/s of the ablation back ends at 640x480, and the device time of `macvo_observe_pack` per covariance model.

End to end: the pipelined `FusedTwoFrameOdometry` with the Full (MatchCovariance, CovAwareSelector), CovKP (NoCovariance),
CovOpt (RandomSelector: no host synchronisation per frame) and ScaleNorm (Modifier_Normalize) back ends, and the plugin-API
`TwoFrameOdometry` with the Full back end, alternated `--repeats` times each in one process. FilterCompose(CovarianceSanity,
SimpleDepth(0.05, auto), LikelyFrontOfCam), graph icp, B200_TartanMotionNet, num_point 200, mapping off, synthetic frontend
weights and a seeded synthetic sequence: with these weights the filter chain leaves no observation, so the LM solve does not
run and the rates do not include it.

Kernel time: observe_pack (observe_kernel + pack_kernel) under MATCH, IDENTITY and MATCH + Normalize, CUDA events over
`--launches` launches, at k = 200 and 4096.

    python tools/bench_ablation.py [--steps 60] [--warmup 10] [--repeats 3] [--launches 500]

Prints one JSON line with the card name and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from tools.bench_paper_reproduce import H, SEQ, W, card  # noqa: E402

COV = {"Full": NS(type="B200_MatchCovariance", args=None), "CovKP": NS(type="B200_NoCovariance", args=None),
       "CovOpt": NS(type="B200_MatchCovariance", args=None),
       "ScaleNorm": NS(type="B200_Modifier_Normalize", args=NS(type="B200_MatchCovariance", args=None))}


def build(name: str, fused: bool, device: str):
    from macvo_b200 import plugins as P
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    match = NS(device=device, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)
    cfg = COV[name]
    if cfg.type == "B200_MatchCovariance":
        cfg = NS(type=cfg.type, args=match)
    elif cfg.args is not None:
        cfg = NS(type=cfg.type, args=NS(type=cfg.args.type, args=match))
    fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=device, enc_dtype="fp32", dec_dtype="fp32",
                                         decoder_depth=12, enforce_positive_disparity=False, cuda_graph=True))
    sel = (P.B200_RandomSelector(NS(mask_width=32, device=device)) if name == "CovOpt" else
           P.B200_CovAwareSelector(NS(device=device, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0,
                                      max_match_cov=100.0)))
    pgo = P.B200_TwoFrame_PGO(NS(graph_type="icp", device=device, vectorize=True, parallel=False, autodiff=False))
    outlier = P.B200_FilterCompose(NS(filter_args=[
        NS(type="B200_CovarianceSanityFilter", args=None),
        NS(type="B200_SimpleDepthFilter", args=NS(min_depth=0.05, max_depth="auto")),
        NS(type="B200_LikelyFrontOfCamFilter", args=None)]))
    motion = P.B200_TartanMotionNet(NS(weight="synthetic", device=device))
    cls = FusedTwoFrameOdometry if fused else TwoFrameOdometry
    return cls(fe, sel, P.ICovariance2to3.instantiate(cfg.type, cfg.args), pgo, num_point=200, mapping=False,
               motion_model=motion, outlier_filter=outlier)


def run(name: str, fused: bool, frames, steps: int, warmup: int, device: str) -> dict:
    odo = build(name, fused, device)
    torch.manual_seed(5)
    odo.initialize(frames[0])
    period = 2 * SEQ - 2
    pp = lambda i: (i % period) if (i % period) < SEQ else period - (i % period)
    seq = [frames[pp(i)] for i in range(1, warmup + steps + 1)]
    obs = []

    def step(i):
        if fused:
            odo.run_pair(seq[i], next_frame=seq[i + 1] if i + 1 < len(seq) and i != warmup - 1 else None)
        else:
            obs.append(odo.run_pair(seq[i]).num_obs)
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    obs.clear()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(warmup, len(seq)):
        step(i)
        if fused:
            odo.latest_pose()
    odo.finish()
    e.record()
    e.synchronize()
    out = {"fps": steps / (s.elapsed_time(e) * 1e-3)}
    if fused:
        out["mean_obs"] = odo.observations()["num_obs"]
        out["host_waits_per_frame"] = statistics.mean(odo.host_waits[warmup:])
    else:
        out["mean_obs"] = statistics.mean(obs) if obs else 0.0
    return out


def kernel_times(launches: int, device: str) -> dict:
    """observe_pack device time per launch pair (ms), median of 3 blocks of `launches`"""
    from macvo_b200 import ops
    from tests.golden import observe_cases as oc
    res = {}
    for k in (200, 4096):
        c = oc.solve_inputs(k, seed=77)
        args, kw = oc.oracle_args(c)
        kp0, maps, (ew, i0, i1, prev) = args[0], [m.to(device) for m in args[1:7]], args[7:]
        kp0, prev = kp0.to(device), prev.to(device)
        buf = ops.ObservationBuffers(k, device)
        nxt = torch.empty((7,), dtype=torch.float64, device=device)
        for spec, ext in (("MATCH", None), ("IDENTITY", {"cov_model": "identity"}),
                          ("MATCH+Normalize", {"cov_model": "match", "cov_ops": ["normalize"]})):
            call = lambda: ops.observe_pack(buf, kp0, *maps, ew, i0, i1, prev, nxt, ext=ext, **kw)
            for _ in range(20):
                call()
            blocks = []
            for _ in range(3):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(launches):
                    call()
                e.record()
                e.synchronize()
                blocks.append(s.elapsed_time(e) / launches)
            res[f"k{k}_{spec}_ms"] = round(statistics.median(blocks), 5)
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=500)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    device = "cuda:0"
    from macvo_b200 import build as mbuild, synthetic
    mbuild.build(verbose=False)
    frames = synthetic.make_sequence(SEQ, H, W, pin=True)
    legs = [("Full", True), ("CovKP", True), ("CovOpt", True), ("ScaleNorm", True), ("Full", False)]
    res: dict = {f"{n}_{'fused' if f else 'plugin_api'}": [] for n, f in legs}
    for _ in range(args.repeats):
        for n, f in legs:
            res[f"{n}_{'fused' if f else 'plugin_api'}"].append(run(n, f, frames, args.steps, args.warmup, device))
    out = {"workload": f"ablation back ends, {W}x{H}, num_point 200, mapping off, synthetic weights and frames",
           **card(), "steps": args.steps, "warmup": args.warmup}
    for key, rs in res.items():
        fps = [r["fps"] for r in rs]
        out[key] = {"fps_runs": [round(f, 2) for f in fps], "fps_median": round(statistics.median(fps), 2),
                    "fps_spread": round(max(fps) - min(fps), 2), "mean_obs_last": rs[-1]["mean_obs"],
                    **({"host_waits_per_frame": rs[-1]["host_waits_per_frame"]} if "host_waits_per_frame" in rs[-1] else {})}
    out["observe_pack"] = kernel_times(args.launches, device)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
