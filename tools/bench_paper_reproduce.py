"""Frames/s of the Paper_Reproduce back end at 640x480: the pipelined `FusedTwoFrameOdometry` (one host synchronisation per
frame) against the plugin-API `TwoFrameOdometry`, alternated three times each in one process.

Back end (Config/Experiment/MACVO/Paper_Reproduce.yaml): B200_CovAwareSelector (max_depth auto), B200_MatchCovariance,
B200_FilterCompose(CovarianceSanityFilter, SimpleDepthFilter(0.05, auto), LikelyFrontOfCamFilter), B200_TwoFrame_PGO
graph_type icp, B200_TartanMotionNet; num_point 200, mapping off. Synthetic frontend weights and a seeded synthetic
sequence (no checkpoint or dataset offline): with these weights LikelyFrontOfCamFilter can drop most rows, so the mean
observation count per frame is printed with the rates.

    python tools/bench_paper_reproduce.py [--steps 60] [--warmup 10]

Prints the card name and its power limit with the numbers."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

H, W, SEQ = 480, 640, 8


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
    except Exception:           # no nvidia-smi: the name from torch, the limit unknown
        name, limit = torch.cuda.get_device_name(), "unknown"
    return {"gpu": name, "power_limit": limit}


def build(fused: bool, device: str):
    from macvo_b200 import plugins as P
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=device, enc_dtype="fp32", dec_dtype="fp32",
                                         decoder_depth=12, enforce_positive_disparity=False, cuda_graph=True))
    sel = P.B200_CovAwareSelector(NS(device=device, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0,
                                     max_match_cov=100.0))
    cov = P.B200_MatchCovariance(NS(device=device, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05,
                                    min_flow_cov=0.25))
    pgo = P.B200_TwoFrame_PGO(NS(graph_type="icp", device=device, vectorize=True, parallel=False, autodiff=False))
    outlier = P.B200_FilterCompose(NS(filter_args=[
        NS(type="B200_CovarianceSanityFilter", args=None),
        NS(type="B200_SimpleDepthFilter", args=NS(min_depth=0.05, max_depth="auto")),
        NS(type="B200_LikelyFrontOfCamFilter", args=None)]))
    motion = P.B200_TartanMotionNet(NS(weight="synthetic", device=device))
    cls = FusedTwoFrameOdometry if fused else TwoFrameOdometry
    return cls(fe, sel, cov, pgo, num_point=200, mapping=False, motion_model=motion, outlier_filter=outlier)


def run(fused: bool, frames, steps: int, warmup: int, device: str) -> dict:
    odo = build(fused, device)
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
            odo.latest_pose()                     # the frame's pose on the host, as a caller would read it
    odo.finish()
    e.record()
    e.synchronize()
    if fused:
        obs.append(odo.observations()["num_obs"])
    return {"fps": steps / (s.elapsed_time(e) * 1e-3), "mean_obs": statistics.mean(obs) if obs else 0.0}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    device = "cuda:0"
    from macvo_b200 import build as mbuild, synthetic
    mbuild.build(verbose=False)
    frames = synthetic.make_sequence(SEQ, H, W, pin=True)
    res = {"fused": [], "plugin_api": []}
    for _ in range(args.repeats):
        for name, fused in (("fused", True), ("plugin_api", False)):
            res[name].append(run(fused, frames, args.steps, args.warmup, device))
    out = {"workload": f"Paper_Reproduce back end, {W}x{H}, num_point 200, mapping off, synthetic weights and frames",
           **card(), "steps": args.steps, "warmup": args.warmup}
    for name, rs in res.items():
        fps = [r["fps"] for r in rs]
        out[name] = {"fps_runs": [round(f, 2) for f in fps], "fps_median": round(statistics.median(fps), 2),
                     "mean_obs_last": rs[-1]["mean_obs"]}
    out["speedup"] = round(out["fused"]["fps_median"] / out["plugin_api"]["fps_median"], 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
