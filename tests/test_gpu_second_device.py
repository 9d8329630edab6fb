"""Every launcher whose kernel needs more than 48 KB of dynamic shared memory, first on cuda:0 and then on cuda:1 in the same
process. The shared-memory attribute (and, for patch_tokens_tc, the SM count) belongs to the current device, so a launcher
that configured it once per process would refuse its first launch on the second device. Each device gets its own copies of
the inputs and runs with itself as the current device; the two results must be bit-identical."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")]


def _inputs():
    g = torch.Generator().manual_seed(2)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    B, H, W = 1, 12, 16
    gru_names = {"convzr1": (256, 512, 1, 5), "convq1": (128, 512, 1, 5), "convzr2": (256, 512, 5, 1), "convq2": (128, 512, 5, 1)}
    return dict(
        shape=(B, H, W),
        conv_x=r(B * H * W, 64), conv_w=r(64, 64, 3, 3, scale=0.05), conv_b=r(64),
        gru_w=[{n: r(*s, scale=0.03) for n, s in gru_names.items()} for _ in range(2)],
        gru_b=[{n: r(s[0], scale=0.3) for n, s in gru_names.items()} for _ in range(2)],
        gru_in=r(B * H * W, 128).relu(), gru_h=[torch.tanh(r(B * H * W, 128)) for _ in range(2)],
        gru_mf=r(B * H * W, 128).relu(), gru_agg=r(B * H * W, 128), gru_gamma=torch.tensor([0.6]),
        mlp=[r(300, 128), r(300, 128), r(512, 128, scale=0.09), r(512, scale=0.09), r(128, 512, scale=0.04), r(128, scale=0.04)],
        corr=[r(2, 256, 12, 16), r(2, 256, 12, 16)],
        pt=[r(200, 64, scale=0.5), r(128, 64, scale=0.09), r(80, 128, scale=0.25), r(128, 128, scale=0.09), r(128, scale=0.09),
            1 + r(128, scale=0.1), r(128, scale=0.1)],
        sh=[r(1, 64, 5, 9) for _ in range(3)],
    )


def _run_every_launcher(ops, dev, inp):
    """each launcher once, with `dev` the current device and every operand on it"""
    from macvo_b200 import stereonet
    d = lambda t: t.to(dev)
    out = {}
    B, H, W = shape = inp["shape"]
    rows = torch.zeros(ops.rows_count(B, H, W), 64, dtype=torch.float16, device=dev)
    ops.pack_rows(d(inp["conv_x"]), rows, 0, shape)
    wp, bp, n = ops.pack_conv_filter(d(inp["conv_w"]), d(inp["conv_b"]))
    out["conv_tc"] = torch.zeros(B * H * W, 64, device=dev)
    ops.conv_tc(rows, wp, bp, n, 3, True, shape, out32=out["conv_tc"])

    gru = ops.SepConvGruTC([{k: d(v) for k, v in w.items()} for w in inp["gru_w"]],
                           [{k: d(v) for k, v in b.items()} for b in inp["gru_b"]], B, H, W, dev)
    gru.set_context(d(inp["gru_in"]))
    for u in range(2):
        gru.set_state(u, d(inp["gru_h"][u]))
    torch.cuda.current_stream().wait_event(gru.step(d(inp["gru_mf"]), d(inp["gru_agg"]), d(inp["gru_gamma"])))
    out["gru_h0"], out["gru_h1"] = gru.h[0], gru.h[1]

    xn, resid, w1, b1, w2, b2 = map(d, inp["mlp"])
    out["mlp_tc"] = ops.mlp_tc(xn, resid, ops.round_tf32(w1), b1, ops.round_tf32(w2), b2)

    f1, f2 = map(d, inp["corr"])
    out["corr_3xf16"] = ops.corr_build(f1, f2, mode=ops.CORR_TC_3XF16)
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    out["corr_tf32"] = ops.corr_build(cl(f1), cl(f2), mode=ops.CORR_TC_TF32)

    x, w0, term, w2, b2, lw, lb = map(d, inp["pt"])
    out["patch_tokens_tc"] = ops.patch_tokens_tc(x, ops.round_tf32(w0), term, ops.round_tf32(w2), b2, lw, lb)

    net = stereonet.StereoCovNetDevice(stereonet.synthetic_stereo_state_dict(0), dev)
    xd, xc, c0 = map(d, inp["sh"])
    out["stereo_depth"] = torch.full((1, 1, 12, 20), float("nan"), device=dev)
    out["stereo_var"] = torch.full((1, 1, 12, 20), float("nan"), device=dev)
    ops.stereo_head(xd, xc, c0, *net.head[stereonet.DISP], *net.head[stereonet.COV], 80.0, (1, 1), out["stereo_depth"],
                    out["stereo_var"])
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def test_launchers_run_on_a_second_device_in_the_same_process():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    inp = _inputs()
    prev_tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True                 # stereo_head's deconvolution is a TF32 one
    try:
        results = []
        for i in (0, 1):
            with torch.cuda.device(i):
                results.append(_run_every_launcher(ops, f"cuda:{i}", inp))
    finally:
        torch.backends.cudnn.allow_tf32 = prev_tf32
    for name, first in results[0].items():
        assert torch.equal(first.nan_to_num(123.0), results[1][name].nan_to_num(123.0)), f"{name} differs on cuda:1"
