"""Time the fused transformer MLP (csrc/mlp_tc.cu) against the four-op sequence it replaces (cuBLAS TF32 fc1, GELU, cuBLAS
TF32 fc2, residual add) at the 640x480 call sites, with CUDA events. Needs a GPU.

    python tools/bench_mlp.py [--iters N]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TF32_DATASHEET_TFLOPS = 495.0      # H100 SXM data sheet, dense TF32 at 700 W: a ceiling, not a measured rate
# (call site, rows M, hidden size, calls per frame) at 640x480, B = 2
SITES = [("vert_block mlp (perceiver)", 16 * 4800, 512, 6),
         ("latent / input-layer ffn", 9600 * 8, 128, 4),
         ("svt stage 0, context (2 images)", 2 * 19200, 512, 2),
         ("svt stage 0, features (3 images)", 3 * 19200, 512, 2)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200, help="timed launches per shape and variant")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        sys.exit("bench_mlp: no CUDA device")
    from macvo_b200 import build, ops
    build.build(verbose=False)
    torch.backends.cuda.matmul.allow_tf32 = True
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card or torch.cuda.get_device_name(0)}")

    def timed(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters * 1e3          # us per call

    total = [0.0, 0.0]
    for name, m, hd, calls in SITES:
        g = torch.Generator().manual_seed(m + hd)
        xn = torch.randn(m, 128, generator=g).to(dev)
        x = torch.randn(m, 128, generator=g).to(dev)
        w1, b1 = (torch.randn(hd, 128, generator=g) / 128 ** 0.5).to(dev), torch.randn(hd, generator=g).to(dev) * 0.1
        w2, b2 = (torch.randn(128, hd, generator=g) / hd ** 0.5).to(dev), torch.randn(128, generator=g).to(dev) * 0.1
        w1t, w2t = ops.round_tf32(w1), ops.round_tf32(w2)
        us_torch = timed(lambda: x + F.linear(F.gelu(F.linear(xn, w1, b1)), w2, b2))
        us_fused = timed(lambda: ops.mlp_tc(xn, x, w1t, b1, w2t, b2))
        flop = 4.0 * m * 128 * hd
        tf = flop / us_fused * 1e-6
        total[0] += calls * us_torch
        total[1] += calls * us_fused
        print(f"{name:34s} M {m:6d} 128->{hd:3d}: torch 4-op {us_torch:8.1f} us   fused {us_fused:8.1f} us   "
              f"x{us_torch / us_fused:4.2f}   fused {tf:6.1f} TFLOP/s = {100 * tf / TF32_DATASHEET_TFLOPS:4.1f} % of the "
              f"{TF32_DATASHEET_TFLOPS:.0f} TFLOP/s TF32 data-sheet rate")
    print(f"per frame (x calls): torch 4-op {total[0] / 1e3:.3f} ms, fused {total[1] / 1e3:.3f} ms")


if __name__ == "__main__":
    main()
