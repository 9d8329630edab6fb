"""Graph timing of one tensor-core (wgmma) convolution (csrc/conv_tc.cu) at the decoder's shapes (B = 2, 60 x 80)."""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from macvo_b200 import ops

DEV = "cuda:0"
torch.backends.cudnn.allow_tf32 = True
B, H, W = 2, 60, 80
shape = (B, H, W)
g = torch.Generator().manual_seed(0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)


def graphed(fn, reps=10):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            for _ in range(reps):
                fn()
    ts = []
    for _ in range(10):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); gr.replay(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2]


for cin, cout, k in ((256, 192, 3), (256, 126, 3), (128, 256, 3), (192, 256, 1), (256, 2, 3)):
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    w = (torch.randn(cout, cin, k, k, generator=g) * 0.05).to(DEV)
    b = torch.randn(cout, generator=g).to(DEV)
    wp, bp, n = ops.pack_conv_filter(w, b)
    rows = torch.zeros(ops.rows_count(B, H, W), cin, dtype=torch.float16, device=DEV)
    ops.pack_rows(x.permute(0, 2, 3, 1).reshape(B * H * W, cin).contiguous(), rows, 0, shape)
    out16 = torch.zeros(ops.rows_count(B, H, W), 256, dtype=torch.float16, device=DEV)
    xl, wl = x.contiguous(memory_format=torch.channels_last), w.contiguous(memory_format=torch.channels_last)
    res = {"conv": [cin, cout, k],
           "tc_us": graphed(lambda: ops.conv_tc(rows, wp, bp, n, k, True, shape, out16=out16)),
           "cudnn_relu_us": graphed(lambda: torch.cudnn_convolution_relu(xl, wl, b, (1, 1), (k // 2, k // 2), (1, 1), 1))}
    print(json.dumps(res))
