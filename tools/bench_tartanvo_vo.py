"""Frames per second of the TartanVO baseline on one GPU (synthetic weights, every frame a keyframe, images in pinned host
memory):

    python tools/bench_tartanvo_vo.py [--frames 40] [--windows 5] [--out DIR]

  fused_fps     pipeline.FusedTartanVO (one CUDA graph per keyframe: PWC-Net on a side stream next to the depth network
                without its covariance decoder, then the pose network and its head; no host wait per frame)
  eager_fps     the same driver with cuda_graph=False
  plugins_fps   B200_TartanVOMatcher.estimate, B200_TartanVODepth.estimate (cov_mode Est) and B200_TartanMotionNet.predict /
                update in BaselineTartanVO.run's order, each plugin on its own CUDA graph
Each arm runs --frames frames per window, timed by the host clock around the window and a device synchronise; the windows of
the three arms alternate in one process, and the median (with min and max) of --windows windows is reported, at 480x640,
376x780 and 480x752, under torch's default flags and under strict fp32.

  overlap       from a separate torch.profiler run of 6 fused frames at each shape (default flags): per keyframe, device
                time of the kernels on each stream and the time during which kernels of both streams run at once
The card name and power limit are part of the result."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
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


def set_flags(mode: str) -> None:
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = mode == "default"
    torch.set_float32_matmul_precision("highest")


def plugins(cov_mode: str, cuda_graph: bool = True):
    from macvo_b200 import plugins as P
    return (P.B200_TartanVOMatcher(NS(weight="synthetic:0", device="cuda", cuda_graph=cuda_graph)),
            P.B200_TartanVODepth(NS(weight="synthetic:0", device="cuda", cov_mode=cov_mode, cuda_graph=cuda_graph)),
            P.B200_TartanMotionNet(NS(weight="synthetic:0", device="cuda")))


class Frames:
    """an endless stream of StereoFrames cycling over 8 pinned synthetic frames, with increasing frame_idx"""

    def __init__(self, H: int, W: int):
        from macvo_b200 import synthetic
        self.data = synthetic.make_sequence(8, H, W, pin=True)
        for sd in self.data:
            sd.T_BS = torch.tensor([[0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]])
        self.i = 0

    def next(self):
        from macvo_b200.interfaces import StereoFrame
        sd = self.data[self.i % len(self.data)]
        f = StereoFrame(idx=[self.i], time_ns=sd.time_ns, stereo=sd)
        self.i += 1
        return f


class Fused:
    def __init__(self, H, W, cuda_graph=True):
        from macvo_b200.pipeline import FusedTartanVO
        self.vo = FusedTartanVO(*plugins("None", cuda_graph), keyframe_freq=1, cuda_graph=cuda_graph)
        self.frames = Frames(H, W)

    def step(self):
        self.vo.run(self.frames.next())


class PluginSequence:
    def __init__(self, H, W):
        self.matcher, self.depth, self.motion = plugins("Est")
        self.frames = Frames(H, W)
        self.prev = None

    def step(self):
        f = self.frames.next()
        flow = self.matcher.estimate(self.prev.stereo, f.stereo).flow if self.prev is not None else None
        pose = self.motion.predict(f, flow, self.depth.estimate(f.stereo).depth)
        self.motion.update(pose)
        self.prev = f


def window(arm, n: int) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        arm.step()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def overlap(H: int, W: int, out_dir: str) -> dict:
    """kernel intervals per stream from a torch.profiler trace of 6 fused keyframes after 3 warm-up frames"""
    from torch.profiler import ProfilerActivity, profile
    set_flags("default")
    arm = Fused(H, W)
    for _ in range(3):
        arm.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(6):
            arm.step()
        torch.cuda.synchronize()
    path = os.path.join(out_dir, f"tartanvo_vo_{H}x{W}.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        ev = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    streams: dict = {}
    for e in ev:
        streams.setdefault(e["args"].get("stream"), []).append((e["ts"], e["ts"] + e["dur"]))
    busy = {str(s): sum(b - a for a, b in iv) / 6e3 for s, iv in streams.items()}
    both = 0.0
    if len(streams) >= 2:
        (s1, i1), (s2, i2) = sorted(streams.items(), key=lambda kv: -sum(b - a for a, b in kv[1]))[:2]
        # union of each stream's intervals, then the length of their intersection
        def union(iv):
            out = []
            for a, b in sorted(iv):
                if out and a <= out[-1][1]:
                    out[-1][1] = max(out[-1][1], b)
                else:
                    out.append([a, b])
            return out
        u1, u2 = union(i1), union(i2)
        j = 0
        for a, b in u1:
            while j < len(u2) and u2[j][1] <= a:
                j += 1
            k = j
            while k < len(u2) and u2[k][0] < b:
                both += min(b, u2[k][1]) - max(a, u2[k][0])
                k += 1
    span = (max(e["ts"] + e["dur"] for e in ev) - min(e["ts"] for e in ev)) / 6e3 if ev else 0.0
    return {"shape": f"{H}x{W}", "kernels": len(ev), "ms_per_keyframe_span": round(span, 3),
            "busy_ms_per_keyframe_by_stream": {k: round(v, 3) for k, v in busy.items()},
            "concurrent_ms_per_keyframe": round(both / 6e3, 3)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the JSON result and the profiler traces")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark measures the GPU; no CUDA device found"
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    out_dir = args.out or tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    result = {"card": card(), "frames_per_window": args.frames, "windows": args.windows, "runs": []}
    with torch.inference_mode():
        for mode in ("default", "strict"):
            set_flags(mode)
            for H, W in SHAPES:
                arms = {"fused": Fused(H, W), "eager": Fused(H, W, cuda_graph=False), "plugins": PluginSequence(H, W)}
                for arm in arms.values():
                    window(arm, 5)                      # set-up, graph capture, cuDNN algorithm choice
                fps = {k: [] for k in arms}
                for _ in range(args.windows):
                    for k, arm in arms.items():
                        fps[k].append(window(arm, args.frames))
                row = {"mode": mode, "shape": f"{H}x{W}"}
                for k, v in fps.items():
                    row[f"{k}_fps"] = {"median": round(statistics.median(v), 2), "min": round(min(v), 2),
                                       "max": round(max(v), 2)}
                row["fused_over_plugins"] = round(row["fused_fps"]["median"] / row["plugins_fps"]["median"], 3)
                result["runs"].append(row)
                print(json.dumps(row), flush=True)
                del arms
                torch.cuda.empty_cache()
        result["overlap"] = [overlap(H, W, out_dir) for H, W in SHAPES]
    for o in result["overlap"]:
        print(json.dumps(o), flush=True)
    print(json.dumps(result["card"]))
    with open(os.path.join(out_dir, "bench_tartanvo_vo.json"), "w") as fh:
        json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
