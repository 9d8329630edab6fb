"""Timing of B200_TartanVODepth (TartanVO's StereoCovNet) on one GPU (synthetic weights, images already on the device):

    python tools/bench_tartanvo_depth.py [--iters 100] [--rounds 5] [--out DIR]

  estimate_us      steady-state `estimate` (CUDA graph replay + the output copies), cov_mode Est, CUDA events, at 480x640,
                   376x780 and 480x752, under torch's default flags (cuDNN in TF32: the head runs in macvo_stereo_head) and
                   under strict fp32 (the head runs as torch ops): median over --rounds windows of --iters calls, with the
                   min and max of the windows
  torch_head_us    default flags, the same network with macvo_stereo_head replaced by the torch ops it fuses (cat,
                   deconv_c11, ReLU, conv_c12, ReLU, conv_c13, ReLU, / 0.02 and the depth arithmetic, crop copy), same
                   graph, windows alternating with the kernel path's in the same process; max disparity difference
  profile          from a separate torch.profiler run at 480x640 (default flags, no graph): device time of macvo_stereo_head
                   against the kernels of the torch-op head it replaces, its TF32 FLOP/s and bytes/s (computed from the
                   shapes) against the H100 SXM data sheet (495 TFLOP/s dense TF32, 3.35 TB/s), and per-stage device time
                   (encoder / the two decoders / head) from CUDA events
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

SHAPES = ((480, 640), (376, 780), (480, 752))


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # the number is still reported, with the reason the card could not be read
        q = f"{torch.cuda.get_device_name(0)}, unknown power limit ({e})"
    return {"gpu": q}


def events(fn, iters: int) -> float:
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def set_flags(mode: str) -> None:
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = mode == "default"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tartanvo_depth needs a GPU"
    from macvo_b200 import build, ops, plugins as P, stereonet
    from tests.golden import tartanvo_cases
    build.build(verbose=False)
    res = card()
    dev = "cuda"
    kernel_op = ops.stereo_head

    def frame(H, W):
        f = tartanvo_cases.frame(torch.rand(1, 3, H, W).to(dev))
        f.imageR = torch.rand(1, 3, H, W).to(dev)
        return f

    def plugin(**kw):
        return P.B200_TartanVODepth(NS(weight="synthetic:0", device=dev, cov_mode="Est", **kw))

    def torch_head_for(net):
        def head(xd, xc, cat0, w11_d, small_d, w11_c, small_c, bf, margin, depth, var):
            d, v = stereonet.depth_torch(net.head_torch(stereonet.DISP, xd, cat0),
                                         net.head_torch(stereonet.COV, xc, cat0) if xc is not None else None, bf)
            my, mx = margin
            depth[..., my:my + d.shape[-2], mx:mx + d.shape[-1]].copy_(d)
            if var is not None:
                var[..., my:my + d.shape[-2], mx:mx + d.shape[-1]].copy_(v)
        return head

    summary = lambda xs: {"median": sorted(xs)[len(xs) // 2], "min": min(xs), "max": max(xs)}
    res["estimate_us"], res["torch_head_us"], res["torch_head_max_disp_diff"] = {}, {}, {}
    for H, W in SHAPES:
        f = frame(H, W)
        set_flags("strict_fp32")
        m = plugin()
        m.estimate(f)
        res["estimate_us"][f"{H}x{W}/strict_fp32"] = summary([events(lambda: m.estimate(f), args.iters)
                                                              for _ in range(args.rounds)])
        set_flags("default")
        m = plugin()
        ref = m.estimate(f).depth                               # captures the kernel path's graph
        mt = plugin()
        ops.stereo_head = torch_head_for(mt.net)
        try:
            alt = mt.estimate(f).depth                          # captures the torch-head path's graph
        finally:
            ops.stereo_head = kernel_op
        fin = torch.isfinite(ref) & torch.isfinite(alt)
        res["torch_head_max_disp_diff"][f"{H}x{W}"] = (80.0 / ref[fin] - 80.0 / alt[fin]).abs().max().item()
        ours, theirs = [], []
        for _ in range(args.rounds):                            # alternate the two paths, window by window
            ours.append(events(lambda: m.estimate(f), args.iters))
            theirs.append(events(lambda: mt.estimate(f), args.iters))
        res["estimate_us"][f"{H}x{W}/default"], res["torch_head_us"][f"{H}x{W}"] = summary(ours), summary(theirs)

    # per-stage device time (CUDA events, no graph) and the head kernel in a profiler run of its own, at 480x640
    set_flags("default")
    H, W = SHAPES[0]
    f = frame(H, W)
    m = plugin(cuda_graph=False)
    net = m.net
    (my, mx), (h64, w64) = m.geometry(H, W)
    ims = torch.rand(2, 3, h64, w64, device=dev)
    depth = torch.full((1, 1, H, W), float("nan"), device=dev)
    var = depth.clone()
    wd, sd = net.head[stereonet.DISP]
    wc, sc = net.head[stereonet.COV]
    with torch.inference_mode(), torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True,
                                                             allow_tf32=True):
        ctx, cats = net.encode(ims)
        xd, xc = net.decode(stereonet.DISP, ctx, cats), net.decode(stereonet.COV, ctx, cats)
        stages = {
            "encoder": lambda: net.encode(ims),
            "decoder_disparity": lambda: net.decode(stereonet.DISP, ctx, cats),
            "decoder_covariance": lambda: net.decode(stereonet.COV, ctx, cats),
            "head_kernel": lambda: kernel_op(xd, xc, cats[0], wd, sd, wc, sc, 80.0, (my, mx), depth, var),
            "head_torch_ops": lambda: torch_head_for(net)(xd, xc, cats[0], wd, sd, wc, sc, 80.0, (my, mx), depth, var),
        }
        res["stage_us_480x640"] = {k: events(fn, 20) for k, fn in stages.items()}
        from torch.profiler import ProfilerActivity, profile
        reps = 10
        for name, fn in (("kernel", stages["head_kernel"]), ("torch_ops", stages["head_torch_ops"])):
            fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    fn()
                torch.cuda.synchronize()
            kern = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    kern[e.name[:80]] = kern.get(e.name[:80], 0.0) + e.device_time / reps
            res[f"profile_head_{name}_us"] = kern
    h2, w2 = h64 // 2, w64 // 2
    flops = 2 * (2 * (h64 * w64) * 64 * 128 * 4 + 2 * h64 * w64 * (64 * 16 + 16))     # both heads: deconv + 1x1 convs
    nbytes = 3 * 64 * h2 * w2 * 4 + 2 * h64 * w64 * 4 + 2 * 4 * 4 * 4 * 64 * 32 * 4
    us = sum(v for k, v in res["profile_head_kernel_us"].items() if "stereo_head" in k)
    res["head_kernel"] = {"device_us": us, "GFLOP": flops / 1e9, "MB": nbytes / 1e6,
                          "TFLOPs": flops / (us * 1e-6) / 1e12 if us else None,
                          "TBs": nbytes / (us * 1e-6) / 1e12 if us else None,
                          "share_of_tf32_peak": flops / (us * 1e-6) / 495e12 if us else None}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_tartanvo_depth.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
