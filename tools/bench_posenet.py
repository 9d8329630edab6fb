"""Timing of the TartanMotionNet pose network on one GPU at 640x480 (synthetic weights and maps):

    python tools/bench_posenet.py [--iters 200] [--frames 40] [--out DIR]

  predict_us           steady-state B200_TartanMotionNet.predict (graph replay + head), CUDA events
  kernels              per-kernel device time from a separate torch.profiler run
  conv_GBps            packed weight + activation bytes of every macvo_posenet_conv launch over their summed kernel time,
                       with the share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)
  torch_conv_us        the same layers through torch.nn.functional.conv2d, summed device kernel time from the profiler
                       like conv_us (comparison only)
  fused_fps            FusedTwoFrameOdometry frames/s without / with the motion model (pipelined, frontend CUDA graph)
The card name and power limit are part of the result."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

HBM_TBPS = 3.35


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # the number is still reported, with the reason the card could not be read
        q = f"{torch.cuda.get_device_name(0)}, unknown power limit ({e})"
    return {"gpu": q}


def device_layers(net):
    """(cin, hi, wi, cout, k, stride, pad, packed, bias) of every macvo_posenet_conv launch, in network order"""
    out, c, h, w = [], 128, 14, 20
    for _, on_dev, blocks in net.stages:
        if not on_dev:
            continue
        for b, layers in enumerate(blocks):
            s = 2 if b == 0 else 1
            cout = layers["conv1"][1].numel()
            ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
            if "downsample" in layers:
                out.append((c, h, w, cout, 1, 2, 0, *layers["downsample"][:2]))
            out.append((c, h, w, cout, 3, s, 1, *layers["conv1"][:2]))
            out.append((cout, ho, wo, cout, 3, 1, 1, *layers["conv2"][:2]))
            c, h, w = cout, ho, wo
    out.append((c * h * w, 1, 1, 256, 1, 1, 0, *net.fc1[:2]))
    return out


def events(fn, iters: int) -> float:
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_posenet needs a GPU"
    from macvo_b200 import build, ops, plugins as P, synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    build.build(verbose=False)
    res = card()
    dev = "cuda"
    H, W = 480, 640
    frames = synthetic.make_sequence(args.frames + 1, H, W, pin=True)
    g = torch.Generator().manual_seed(0)
    flow = (torch.randn(1, 2, H, W, generator=g) * 4).to(dev)
    depth = (torch.rand(1, 1, H, W, generator=g) * 20 + 0.5).to(dev)
    mm = P.B200_TartanMotionNet(NS(weight="synthetic:0", device=dev))
    mm.predict(frames[0], None, None)
    res["predict_us"] = events(lambda: mm.predict(frames[1], flow, depth), args.iters)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            mm.predict(frames[1], flow, depth)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and getattr(e, "device_time_total", 0) > 0:
            kern[e.key] = {"calls_per_predict": e.count / 20, "us_per_predict": e.device_time_total / 20}
    res["kernels"] = dict(sorted(kern.items(), key=lambda kv: -kv[1]["us_per_predict"]))
    conv_us = sum(v["us_per_predict"] for k, v in kern.items() if "posenet_conv" in k)

    layers = device_layers(mm.net)
    nbytes = 0
    for cin, hi, wi, cout, k, s, p, packed, bias in layers:
        ho, wo = (hi + 2 * p - k) // s + 1, (wi + 2 * p - k) // s + 1
        nbytes += 4 * (packed.numel() + bias.numel() + cin * hi * wi + cout * ho * wo)
    res["conv_layers"] = len(layers)
    res["conv_bytes"] = nbytes
    res["conv_us"] = conv_us
    res["conv_GBps"] = nbytes / (conv_us * 1e-6) / 1e9 if conv_us else None
    res["conv_share_of_hbm_peak"] = res["conv_GBps"] / (HBM_TBPS * 1e3) if conv_us else None

    torch_layers = []
    for cin, hi, wi, cout, k, s, p, packed, bias in layers:
        wt = torch.randn(cout, cin, k, k, device=dev)
        torch_layers.append((torch.randn(1, cin, hi, wi, device=dev), wt, bias, s, p))
    run_torch = lambda: [F.conv2d(x, wt, b, stride=s, padding=p) for x, wt, b, s, p in torch_layers]
    for _ in range(10):
        run_torch()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:      # device time, like conv_us (no host launch overhead)
        for _ in range(20):
            run_torch()
        torch.cuda.synchronize()
    res["torch_conv_us"] = sum(e.device_time_total for e in prof.key_averages()
                               if e.device_type.name == "CUDA" and getattr(e, "device_time_total", 0) > 0) / 20

    def fused_fps(with_motion: bool) -> float:
        fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=dev, enc_dtype="fp32", dec_dtype="fp32",
                                             decoder_depth=12, enforce_positive_disparity=False, cuda_graph=True))
        odo = FusedTwoFrameOdometry(
            fe, P.B200_CovAwareSelector_NoDepth(NS(device=dev, kernel_size=7, mask_width=32, max_match_cov=100.0)),
            P.B200_MatchCovariance(NS(device=dev, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)),
            P.B200_TwoFrame_PGO(NS(graph_type="disp", device=dev, vectorize=True, parallel=False, autodiff=False)),
            num_point=200, map_selector=None,
            motion_model=P.B200_TartanMotionNet(NS(weight="synthetic:0", device=dev)) if with_motion else None)
        odo.initialize(frames[0])
        warm = 5
        for i in range(1, args.frames + 1):
            if i == warm + 1:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
            odo.run_pair(frames[i], next_frame=frames[i + 1] if i + 1 <= args.frames else None)
        odo.finish()
        return (args.frames - warm) / (time.perf_counter() - t0)

    res["fused_fps"] = {"without_motion_model": fused_fps(False), "with_motion_model": fused_fps(True)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_posenet.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
