"""Time PatchEmbed's fused token head (csrc/patch_tokens_tc.cu) against the four-op sequence it replaces (cuBLAS TF32
linear 64 -> 128, add_rows_relu_, cuBLAS TF32 linear 128 -> 128, layer_norm) at the 640x480 frame's shape, with CUDA events.
Needs a GPU.

    python tools/bench_patch_tokens.py [--iters N] [--blocks B]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_DATASHEET_TBS = 3.35           # H100 SXM data sheet, HBM3: a ceiling, not a measured rate
TF32_DATASHEET_TFLOPS = 495.0      # H100 SXM data sheet, dense TF32 at 700 W
PERIOD, MAPS = 80, 9600            # 8 x 10 tokens per cost map, 2 x 4800 cost maps per frame at 640x480


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200, help="timed launches per block")
    ap.add_argument("--blocks", type=int, default=3, help="timed blocks per variant; the median is reported")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        sys.exit("bench_patch_tokens: no CUDA device")
    from macvo_b200 import build, ops
    from macvo_b200.flowformer_cov import synthetic_state_dict
    build.build(verbose=False)
    torch.backends.cuda.matmul.allow_tf32 = True
    dev = "cuda:0"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card (name, power limit, max SM clock): {card or torch.cuda.get_device_name(0)}")

    sd = synthetic_state_dict(0)
    p = "memory_encoder.cost_perceiver_encoder.patch_embed."
    w0 = sd[p + "ffn_with_coord.0.weight"].to(dev, torch.float32)[:, :64, 0, 0]
    w2 = sd[p + "ffn_with_coord.2.weight"].to(dev, torch.float32)[:, :, 0, 0]
    b2 = sd[p + "ffn_with_coord.2.bias"].to(dev, torch.float32)
    lw, lb = sd[p + "norm.weight"].to(dev, torch.float32), sd[p + "norm.bias"].to(dev, torch.float32)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(MAPS, PERIOD, 64, generator=g).to(dev)
    term = (torch.randn(PERIOD, 128, generator=g) * 0.25).to(dev)
    w0t, w2t = ops.round_tf32(w0), ops.round_tf32(w2)

    def four_ops():
        t = ops.add_rows_relu_(F.linear(x, w0), term)
        return ops.layer_norm(F.linear(t, w2, b2), lw, lb)

    def fused():
        return ops.patch_tokens_tc(x, w0t, term, w2t, b2, lw, lb)

    assert torch.equal(fused(), four_ops()), "the fused kernel must return the four-op sequence's bits"

    def timed(fn):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        blocks = []
        for _ in range(args.blocks):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            blocks.append(a.elapsed_time(b) / args.iters * 1e3)     # us per call
        return statistics.median(blocks), blocks

    rows = MAPS * PERIOD
    flop = 2.0 * rows * 128 * (64 + 128)
    # algorithmic bytes: the fused kernel reads x and writes the tokens once; the four ops also write and read back the
    # hidden activation (linear, add_rows_relu_ in place) and the pre-norm rows
    fused_bytes = 4.0 * rows * (64 + 128)
    four_bytes = 4.0 * rows * (64 + 128) + 4.0 * rows * 128 * (2 + 2 + 2)
    for name, fn, nbytes in (("four ops (cuBLAS TF32 + add_rows_relu_ + cuBLAS TF32 + layer_norm)", four_ops, four_bytes),
                             ("fused patch_tokens_tc", fused, fused_bytes)):
        us, blocks = timed(fn)
        bound_us = max(nbytes / (HBM_DATASHEET_TBS * 1e12), flop / (TF32_DATASHEET_TFLOPS * 1e12)) * 1e6
        print(f"{name}: {us:8.1f} us (blocks {', '.join(f'{b:.1f}' for b in blocks)})  {nbytes / 1e9:.3f} GB -> "
              f"{nbytes / us * 1e-6:.2f} TB/s, {flop / us * 1e-6:.1f} TFLOP/s; the data-sheet bound ({HBM_DATASHEET_TBS} TB/s HBM, "
              f"{TF32_DATASHEET_TFLOPS:.0f} TFLOP/s TF32) is {bound_us:.1f} us = {100 * bound_us / us:.1f} % of this time")
        if fn is four_ops:
            t_four = us
    print(f"speed-up x{t_four / us:.2f} at {rows} rows (period {PERIOD})")


if __name__ == "__main__":
    main()
