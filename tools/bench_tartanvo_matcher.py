"""Timing of B200_TartanVOMatcher (TartanVO's PWC-Net) on one GPU (synthetic weights, images already on the device):

    python tools/bench_tartanvo_matcher.py [--iters 300] [--rounds 5] [--out DIR]

  estimate_us      steady-state `estimate` (CUDA graph replay + the output copies), CUDA events, at 480x640, 640x640 and
                   376x780, under torch's default flags (cuDNN in TF32) and under strict fp32: median over --rounds windows
                   of --iters calls each (about 1 s per window at default flags), with the min and max of the windows
  torch_ops_us     the same network with the warp + correlation restated in torch ops (grid_sample warp, padded-shift
                   correlation) in place of macvo_pwc_warp_corr, same graph, timed in windows alternating with the kernel
                   path's in the same process; max |flow| difference to the kernel path
  levels           from a separate torch.profiler run at 480x640 (default flags): device time of macvo_pwc_warp_corr per
                   level, with its cost-volume FLOPs and output bytes computed from the shapes, against the summed device
                   time of every other kernel (cuDNN convolutions and the small torch ops)
The card name and power limit are part of the result."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

SHAPES = ((480, 640), (640, 640), (376, 780))


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # the number is still reported, with the reason the card could not be read
        q = f"{torch.cuda.get_device_name(0)}, unknown power limit ({e})"
    return {"gpu": q}


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


def torch_warp_corr(f1, f2, flow, scale, out, out_offset):
    """the reference's warp (pwc_model_tartanvo.py:176-212) and correlation in torch ops on the device"""
    B, C, H, W = f2.shape
    g = f2
    if flow is not None:
        ys, xs = torch.meshgrid(torch.arange(H, device=f2.device), torch.arange(W, device=f2.device), indexing="ij")
        v = torch.stack((xs, ys)).float().unsqueeze(0) + flow * scale
        v = torch.stack((2.0 * v[:, 0] / max(W - 1, 1) - 1.0, 2.0 * v[:, 1] / max(H - 1, 1) - 1.0), dim=-1)
        g = F.grid_sample(f2, v, align_corners=True)
        m = F.grid_sample(torch.ones_like(f2[:, :1]), v, align_corners=True)
        m = torch.where(m < 0.9999, 0.0, torch.where(m > 0, 1.0, m))
        g = g * m
    pad = F.pad(g, (4, 4, 4, 4))
    for k in range(81):
        dy, dx = k // 9, k % 9
        out[:, out_offset + k] = (f1 * pad[:, :, dy:dy + H, dx:dx + W]).sum(1) / C
    F.leaky_relu(out[:, out_offset:out_offset + 81], 0.1, inplace=True)
    return out


def set_flags(mode: str) -> None:
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = mode == "default"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tartanvo_matcher needs a GPU"
    from macvo_b200 import build, ops, plugins as P, pwcnet
    from tests.golden import tartanvo_cases
    build.build(verbose=False)
    res = card()
    dev = "cuda"
    kernel_op = ops.pwc_warp_corr

    def frames(H, W):
        f1, f2 = tartanvo_cases.frame(torch.rand(1, 3, H, W)), tartanvo_cases.frame(torch.rand(1, 3, H, W))
        f1.imageL, f2.imageL = f1.imageL.to(dev), f2.imageL.to(dev)
        return f1, f2

    res["estimate_us"], res["torch_ops_us"], res["torch_ops_max_abs_diff"] = {}, {}, {}
    summary = lambda xs: {"median": sorted(xs)[len(xs) // 2], "min": min(xs), "max": max(xs)}
    for H, W in SHAPES:
        f1, f2 = frames(H, W)
        for mode in ("default", "strict_fp32"):
            set_flags(mode)
            key = f"{H}x{W}/{mode}"
            m = P.B200_TartanVOMatcher(NS(weight="synthetic:0", device=dev))
            ref = m.estimate(f1, f2).flow                 # captures the kernel path's graph
            ops.pwc_warp_corr = torch_warp_corr
            try:
                mt = P.B200_TartanVOMatcher(NS(weight="synthetic:0", device=dev))
                alt = mt.estimate(f1, f2).flow            # captures the torch-ops path's graph
            finally:
                ops.pwc_warp_corr = kernel_op
            res["torch_ops_max_abs_diff"][key] = (ref - alt).nan_to_num().abs().max().item()
            ours, theirs = [], []
            for _ in range(args.rounds):                  # alternate the two paths, window by window
                ours.append(events(lambda: m.estimate(f1, f2), args.iters))
                theirs.append(events(lambda: mt.estimate(f1, f2), args.iters))
            res["estimate_us"][key], res["torch_ops_us"][key] = summary(ours), summary(theirs)

    set_flags("default")
    H, W = SHAPES[0]
    f1, f2 = frames(H, W)
    m = P.B200_TartanVOMatcher(NS(weight="synthetic:0", device=dev, cuda_graph=False))    # kernels listed one by one
    for _ in range(5):
        m.estimate(f1, f2)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    reps = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            m.estimate(f1, f2)
        torch.cuda.synchronize()
    corr = [e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "pwc_warp_corr" in e.name]
    other = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "pwc_warp_corr" not in e.name)
    assert len(corr) == 5 * reps, f"expected 5 macvo_pwc_warp_corr launches per call, found {len(corr) / reps}"
    h64, w64 = H // 64 * 64, W // 64 * 64
    levels = {}
    for i, level in enumerate((6, 5, 4, 3, 2)):
        us = sum(corr[i::5]) / reps
        C, h, w = pwcnet.FEAT_CH[level], h64 >> level, w64 >> level
        flops, nbytes = 2 * 81 * C * h * w, 4 * 81 * h * w
        levels[f"level{level}"] = {"shape": [C, h, w], "us": us, "GFLOP": flops / 1e9, "out_MB": nbytes / 1e6,
                                   "GFLOPs": flops / (us * 1e-6) / 1e9 if us else None}
    res["levels_480x640_default"] = levels
    res["pwc_warp_corr_us_per_call"] = sum(corr) / reps
    res["other_kernels_us_per_call"] = other / reps
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_tartanvo_matcher.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
