"""Frames/s of the Vanilla ablation at 640x480, and the frontend replay time of B200_FlowFormerFrontend against
B200_FlowFormerCovFrontend's.

End to end: the Vanilla configuration (B200_FlowFormerFrontend, B200_NoCovariance, B200_RandomSelector,
FilterCompose[SimpleDepthFilter(0.05, auto)], graph icp, B200_TartanMotionNet, num_point 200, mapping off) through the
pipelined `FusedTwoFrameOdometry` and the plugin-API `TwoFrameOdometry`, alternated `--repeats` times each in one process;
synthetic weights and a seeded synthetic sequence. The frontend runs under torch's default flags (TF32 off), as the
reference's FlowFormerDepth / FlowFormerMatcher do.

Frontend: one `estimate_pair` CUDA-graph replay, CUDA events over `--replays` replays (median of 3 blocks), of the plain and
the Cov frontend at decoder depth 12, under the default flags (strict fp32 loop) and with TF32 allowed (TF32 loop).

    python tools/bench_vanilla.py [--steps 60] [--warmup 10] [--repeats 3] [--replays 50]

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


def set_tf32(on: bool) -> None:
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = on
    torch.set_float32_matmul_precision("medium" if on else "highest")


def build(fused: bool, device: str):
    from macvo_b200 import plugins as P
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    cls = FusedTwoFrameOdometry if fused else TwoFrameOdometry
    return cls(P.B200_FlowFormerFrontend(NS(weight="synthetic:0", device=device)),
               P.B200_RandomSelector(NS(mask_width=32, device=device)), P.B200_NoCovariance(None),
               P.B200_TwoFrame_PGO(NS(graph_type="icp", device=device, vectorize=True, parallel=False, autodiff=False)),
               num_point=200, mapping=False, motion_model=P.B200_TartanMotionNet(NS(weight="synthetic", device=device)),
               outlier_filter=P.B200_FilterCompose(NS(filter_args=[
                   NS(type="B200_SimpleDepthFilter", args=NS(min_depth=0.05, max_depth="auto"))])))


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
            odo.latest_pose()
    odo.finish()
    e.record()
    e.synchronize()
    out = {"fps": steps / (s.elapsed_time(e) * 1e-3)}
    if fused:
        out["obs_last"] = odo.observations()["num_obs"]
        out["host_waits_per_frame"] = statistics.mean(odo.host_waits[warmup:])
    else:
        out["obs_mean"] = statistics.mean(obs) if obs else 0.0
    return out


def replay_ms(fe, frames, replays: int) -> tuple[float, int]:
    """median ms of one estimate_pair replay over 3 blocks, and the macvo_b200 launches inside it"""
    fe.estimate_pair(frames[0], frames[1])            # capture
    for _ in range(5):
        fe.estimate_pair(frames[1], frames[2])
    blocks = []
    for _ in range(3):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(replays):
            fe._graph.replay()
        e.record()
        e.synchronize()
        blocks.append(s.elapsed_time(e) / replays)
    return statistics.median(blocks), fe._static["launches"]


def frontend_times(frames, replays: int, device: str) -> dict:
    from macvo_b200 import plugins as P
    res = {}
    for tf32 in (False, True):
        mode = "tf32" if tf32 else "default_flags"
        for name in ("plain", "cov"):
            set_tf32(tf32)
            if name == "plain":
                fe = P.B200_FlowFormerFrontend(NS(weight="synthetic:0", device=device))
            else:
                fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=device, enc_dtype="fp32", dec_dtype="fp32",
                                                     decoder_depth=12, enforce_positive_disparity=False, cuda_graph=True))
                set_tf32(tf32)         # (its constructor turns TF32 on)
            ms, launches = replay_ms(fe, frames, replays)
            res[f"{mode}_{name}"] = {"replay_ms": round(ms, 3), "launches": launches}
            del fe
            torch.cuda.empty_cache()
        res[f"{mode}_plain_over_cov"] = round(res[f"{mode}_plain"]["replay_ms"] / res[f"{mode}_cov"]["replay_ms"], 4)
    set_tf32(False)
    return res


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--replays", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    device = "cuda:0"
    from macvo_b200 import build as mbuild, synthetic
    mbuild.build(verbose=False)
    frames = synthetic.make_sequence(SEQ, H, W, pin=True)
    set_tf32(False)
    res: dict = {"fused": [], "plugin_api": []}
    for _ in range(args.repeats):
        for fused in (True, False):
            res["fused" if fused else "plugin_api"].append(run(fused, frames, args.steps, args.warmup, device))
    out = {"workload": f"Vanilla ablation, {W}x{H}, num_point 200, mapping off, synthetic weights and frames, default flags",
           **card(), "steps": args.steps, "warmup": args.warmup}
    for key, rs in res.items():
        fps = [r["fps"] for r in rs]
        out[key] = {"fps_runs": [round(f, 2) for f in fps], "fps_median": round(statistics.median(fps), 2),
                    "fps_spread": round(max(fps) - min(fps), 2),
                    **{k: v for k, v in rs[-1].items() if k != "fps"}}
    out["frontend"] = frontend_times(frames, args.replays, device)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
