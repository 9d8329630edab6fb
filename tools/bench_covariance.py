"""Device time of the observation-covariance kernels, and frames/s of the fused driver with each covariance model.

Kernels: `ops.match_covariance` without (MatchCovariance) and with a depth-variance map (GaussianMixtureCovariance), kernel
size 31, int64 keypoints with a (K,3) flow covariance on a seeded 640x480 depth / depth-variance map, at K = 200 (a frame's
keypoints), 2048 (mapping points) and 4096; CUDA events over `--launches` launches, median of 3 blocks.

Frames: the pipelined `FusedTwoFrameOdometry` at 640x480 with the MatchCovariance and the GaussianMixtureCovariance models,
mapping on (B200_MappingPointSelector with thresholds that keep every candidate, 2000 points), CovAwareSelector,
CovarianceSanityFilter, graph icp, num_point 200, synthetic frontend weights and a seeded synthetic sequence; the two
models alternate `--repeats` times in one process.

    python tools/bench_covariance.py [--steps 60] [--warmup 10] [--repeats 3] [--launches 500]

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

ARGS = dict(kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)
MODELS = {"match": "B200_MatchCovariance", "mixture": "B200_GaussianMixtureCovariance"}


def kernel_times(launches: int, device: str) -> dict:
    from macvo_b200 import ops
    from tests.golden.cases import _lognormal_like
    g = torch.Generator().manual_seed(11)
    depth = _lognormal_like((1, 1, H, W), g, 2.0).to(device)
    dcov = _lognormal_like((1, 1, H, W), g, 0.25).to(device)
    fx, fy, cx, cy = 320.0, 320.0, 319.5, 239.5
    res = {}
    for k in (200, 2048, 4096):
        kp = torch.stack([torch.randint(16, W - 16, (k,), generator=g), torch.randint(16, H - 16, (k,), generator=g)], 1)
        kp = kp.to(device)
        flow = (_lognormal_like((k, 3), g, 0.125) * torch.tensor([1.0, 1.0, 0.0])).to(device)
        out = torch.empty((k, 3, 3), dtype=torch.float64, device=device)
        calls = {
            "match": lambda: ops.match_covariance(kp, depth, flow, fx, fy, cx, cy, out_cov=out, **ARGS),
            "mixture": lambda: ops.match_covariance(kp, depth, flow, fx, fy, cx, cy, out_cov=out, depth_cov_map=dcov, **ARGS)}
        for name, call in calls.items():
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
                blocks.append(s.elapsed_time(e) * 1e3 / launches)
            res[f"k{k}_{name}_us"] = round(statistics.median(blocks), 2)
    return res


def build(model: str, device: str):
    from macvo_b200 import plugins as P
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=device, enc_dtype="fp32", dec_dtype="fp32",
                                         decoder_depth=12, enforce_positive_disparity=False, cuda_graph=True))
    sel = P.B200_CovAwareSelector(NS(device=device, kernel_size=7, mask_width=32, max_depth="auto", max_depth_cov=250.0,
                                     max_match_cov=100.0))
    pgo = P.B200_TwoFrame_PGO(NS(graph_type="icp", device=device, vectorize=True, parallel=False, autodiff=False))
    outlier = P.B200_CovarianceSanityFilter(None)
    cov = P.ICovariance2to3.instantiate(MODELS[model], NS(device=device, **ARGS))
    msel = P.B200_MappingPointSelector(NS(max_depth=1e4, max_depth_cov=1e4, mask_width=32))
    return FusedTwoFrameOdometry(fe, sel, cov, pgo, num_point=200, mapping=True, map_selector=msel, outlier_filter=outlier)


def frame_rate(model: str, frames, steps: int, warmup: int, device: str) -> dict:
    odo = build(model, device)
    torch.manual_seed(5)
    odo.initialize(frames[0])
    period = 2 * SEQ - 2
    pp = lambda i: (i % period) if (i % period) < SEQ else period - (i % period)
    seq = [frames[pp(i)] for i in range(1, warmup + steps + 1)]

    def step(i):
        odo.run_pair(seq[i], next_frame=seq[i + 1] if i + 1 < len(seq) and i != warmup - 1 else None)
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(warmup, len(seq)):
        step(i)
        odo.latest_pose()
    odo.finish()
    e.record()
    e.synchronize()
    o = odo.observations()
    return {"fps": steps / (s.elapsed_time(e) * 1e-3), "num_obs": o["num_obs"], "map_points": int(o["map_cov"].shape[0])}


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
    out = {"workload": f"covariance models, {W}x{H}, kernel_size 31", **card(), "steps": args.steps, "warmup": args.warmup,
           "kernels": kernel_times(args.launches, device)}
    frames = synthetic.make_sequence(SEQ, H, W, pin=True)
    runs = {m: [] for m in MODELS}
    for _ in range(args.repeats):
        for m in MODELS:
            runs[m].append(frame_rate(m, frames, args.steps, args.warmup, device))
    for m, rs in runs.items():
        fps = [r["fps"] for r in rs]
        out[f"fused_{m}"] = {"fps_runs": [round(f, 2) for f in fps], "fps_median": round(statistics.median(fps), 2),
                             "num_obs_last": rs[-1]["num_obs"], "map_points_last": rs[-1]["map_points"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
