"""Device time of the 12-iteration decoder alone (captured into a CUDA graph) at 640x480, under the numerics flags the
frontend sets (TF32 matmuls and convolutions allowed)."""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from types import SimpleNamespace as NS
import torch
from macvo_b200 import plugins as P, synthetic

dev = "cuda"
frames = synthetic.make_sequence(3, 480, 640, pin=True)
fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=dev, enc_dtype="fp32", dec_dtype="fp32", decoder_depth=12,
                                     enforce_positive_disparity=False, cuda_graph=False))
net = fe.net
A = torch.cat([frames[2].imageL, frames[1].imageL]).to(dev)
B = torch.cat([frames[2].imageR, frames[2].imageL]).to(dev)
with torch.inference_mode():
    i1, i2 = ((2 * A) - 1.0), ((2 * B) - 1.0)
    ctx = net.svt(i1, "context_encoder")
    feats = net._conv(net.svt(torch.cat([i1, i2]), "memory_encoder.feat_encoder"), "memory_encoder.channel_convertor")
    cv = net.corr_fn(feats[:2], feats[2:]).to(feats.dtype)
    cm, cmaps = net.cost_perceiver(cv, ctx)
    ctx, cmaps = ctx.float(), cmaps.float()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(2):
            net.memory_decoder(cm, ctx, cmaps)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            net.memory_decoder(cm, ctx, cmaps)
    ts = []
    for _ in range(10):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); g.replay(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
print(json.dumps({"decoder_ms": ts[len(ts) // 2], "device": torch.cuda.get_device_name(0)}))
