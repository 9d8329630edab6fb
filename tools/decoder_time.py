"""Device time of the 12-iteration decoder alone (captured into a CUDA graph): tensor-core convolutions + GRU vs GRU only vs cuDNN."""
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
out = {}
with torch.inference_mode():
    i1, i2 = ((2 * A) - 1.0), ((2 * B) - 1.0)
    ctx = net.svt(i1, "context_encoder")
    feats = net._conv(net.svt(torch.cat([i1, i2]), "memory_encoder.feat_encoder"), "memory_encoder.channel_convertor")
    cv = net.corr_fn(feats[:2], feats[2:]).to(feats.dtype)
    cm, cmaps = net.cost_perceiver(cv, ctx)
    ctx, cmaps = ctx.float(), cmaps.float()
    ref = None
    modes = sys.argv[1].split(",") if len(sys.argv) > 1 else ("conv_tc+gru_tc", "gru_tc", "cudnn")
    for mode in modes:
        net.gru_tensor_cores, net.conv_tensor_cores = mode != "cudnn", mode.startswith("conv_tc+gru_tc")
        net.gru_split_units = mode.endswith("+split")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for _ in range(2):
                res = net.memory_decoder(cm, ctx, cmaps)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                res = net.memory_decoder(cm, ctx, cmaps)
        ts = []
        for _ in range(10):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); g.replay(); b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ts.sort()
        out["decoder_ms_" + mode] = ts[len(ts) // 2]
        if ref is None:
            ref = [r.clone() for r in res]
        else:
            out["flow_diff_rel_vs_" + mode] = ((res[0] - ref[0]).abs().max() / ref[0].abs().max()).item()
            out["logcov_diff_abs_vs_" + mode] = (res[1] - ref[1]).abs().max().item()
print(json.dumps(out))
