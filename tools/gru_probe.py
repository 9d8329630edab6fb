"""Timing of one SepConvGRU update of both decoder units at 60x80: tensor-core (wgmma) kernel path vs cuDNN + glue kernels."""
import json
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from macvo_b200 import ops

DEV = "cuda:0"
torch.backends.cuda.matmul.allow_tf32 = True
torch.backends.cudnn.allow_tf32 = True
B, H, W = 1, int(os.environ.get("GRU_H", 60)), int(os.environ.get("GRU_W", 80))
P = B * H * W
g = torch.Generator().manual_seed(0)
rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(DEV)
names = {"convzr1": (256, 512, 1, 5), "convq1": (128, 512, 1, 5), "convzr2": (256, 512, 5, 1), "convq2": (128, 512, 5, 1)}
ws = [{n: rnd(*sh, scale=0.03) for n, sh in names.items()} for _ in range(2)]
bs = [{n: rnd(sh[0], scale=0.3) for n, sh in names.items()} for _ in range(2)]
gru = ops.SepConvGruTC(ws, bs, B, H, W, DEV)
inp, h0 = rnd(P, 128).relu(), torch.tanh(rnd(P, 128))
mf, agg, gamma = rnd(P, 128).relu(), rnd(P, 128), torch.tensor([0.6], device=DEV)
gru.set_context(inp)
gru.set_state(0, h0)
gru.set_state(1, h0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)


def timed(fn, n=30):
    for _ in range(5):
        fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


# the path it replaces: cuDNN convolutions over channels_last [h|x] maps + gate / blend kernels, two units back to back
bufs = [torch.randn(P, 512, device=DEV) for _ in range(4)]
zb = [torch.empty(P, 128, device=DEV) for _ in range(2)]
hd = [torch.empty(P, 128, device=DEV) for _ in range(2)]
wl = [{k: v.contiguous(memory_format=torch.channels_last) for k, v in w.items()} for w in ws]


def old_step():
    ops.gru_input(mf, agg, gamma, bufs)
    for u in range(2):
        hx, rhx = bufs[2 * u], bufs[2 * u + 1]
        hx_map, rhx_map = (t.view(B, H, W, 512).permute(0, 3, 1, 2) for t in (hx, rhx))
        for o, pad in (("1", (0, 2)), ("2", (2, 0))):
            zr = F.conv2d(hx_map, wl[u]["convzr" + o], None, padding=pad)
            ops.gru_gates(zr.permute(0, 2, 3, 1), hx, zb[u], rhx, bs[u]["convzr" + o])
            q = F.conv2d(rhx_map, wl[u]["convq" + o], None, padding=pad)
            ops.gru_blend(q.permute(0, 2, 3, 1), zb[u], hx, hd[u] if o == "2" else None, bs[u]["convq" + o])


def graphed(fn, reps=10):
    """device time per call with the host out of the picture: `reps` calls captured into one CUDA graph"""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            for _ in range(reps):
                fn()
    return timed(gr.replay, 20) / reps


def tc_step():
    torch.cuda.current_stream().wait_event(gru.step(mf, agg, gamma))


out = {"shape": [B, H, W], "tc_step_us": timed(tc_step), "cudnn_glue_step_us": timed(old_step),
       "tc_step_graph_us": graphed(tc_step), "cudnn_glue_step_graph_us": graphed(old_step)}
lib = ops.load_library()
out["pack_motion_graph_us"] = graphed(lambda: lib.macvo_gru_tc_pack_motion(mf.data_ptr(), agg.data_ptr(), gamma.data_ptr(), gru.x[0].data_ptr(),
                                                                           gru.x[1].data_ptr(), B, H, W, torch.cuda.current_stream().cuda_stream))
flops = 2 * 2 * P * 384 * 2560 * 2          # both passes, both units
out["tc_tflops"] = flops / out["tc_step_graph_us"] / 1e6
print(json.dumps(out))
