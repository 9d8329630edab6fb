"""The fused transformer MLP (csrc/mlp_tc.cu): out = resid + W2 GELU_erf(W1 xn + b1) + b2 on TF32 tensor cores, checked against
float64 on tf32 inputs, against today's cuBLAS TF32 path, for row independence, masking, determinism, graph capture, the
torch fallback and the whole frontend with the kernel on and off."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    return ops


def _inputs(m, hd, seed):
    """LayerNorm-scaled rows and weights / biases on the synthetic checkpoint's U(+-1/sqrt(fan_in)) scale"""
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, fan: (torch.rand(shape, generator=g) * 2 - 1) / fan ** 0.5
    xn = F.layer_norm(torch.randn(m, 128, generator=g) * 2 + 0.5, (128,))
    resid = torch.randn(m, 128, generator=g)
    w1, b1, w2, b2 = u((hd, 128), 128), u((hd,), 128), u((128, hd), hd), u((128,), hd)
    return [t.to(DEV) for t in (xn, resid, w1, b1, w2, b2)]


def _ref64(xn, resid, w1, b1, w2, b2, round_tf32):
    """float64 evaluation of the same function on the tf32 values the tensor cores see: xn rounded to tf32 by the kernel,
    the weights as packed (already tf32)"""
    d = lambda t: t.double()
    return d(resid) + F.linear(F.gelu(F.linear(d(round_tf32(xn)), d(w1), d(b1))), d(w2), d(b2))


def _cublas_tf32(xn, resid, w1, b1, w2, b2):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        return resid + F.linear(F.gelu(F.linear(xn, w1, b1)), w2, b2)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("hd", [128, 512])
@pytest.mark.parametrize("m", [1, 127, 128, 129, 4097, 76800])
def test_mlp_tc_accuracy(ops, m, hd):
    xn, resid, w1, b1, w2, b2 = _inputs(m, hd, 17 * m + hd)
    packed = (xn, resid, ops.round_tf32(w1), b1, ops.round_tf32(w2), b2)      # the weights as the network packs them
    got = ops.mlp_tc(*packed)
    ref = _ref64(*packed, ops.round_tf32)
    scale = (ref - resid.double()).abs().max().item()   # the MLP's own contribution sets the scale
    err = (got.double() - ref).abs().max().item()
    err_cublas = (_cublas_tf32(xn, resid, w1, b1, w2, b2).double() - ref).abs().max().item()
    assert err <= 1e-3 * scale, f"err {err:.3e} vs scale {scale:.3e}"
    assert err <= 1.5 * err_cublas, f"fused {err:.3e} vs cuBLAS TF32 {err_cublas:.3e}"


@pytest.mark.parametrize("m,hd", [(76800, 512), (76800, 128), (38400, 512), (57600, 512)])
def test_mlp_tc_matches_cublas_tf32_bits(ops, m, hd):
    """at the frame's call sites the kernel rounds like cuBLAS's TF32 GEMMs (nearest-even tf32 operands and hidden
    activation) and accumulates in the same K order, so it returns the four-op sequence's bits: switching the fused path on
    leaves the frontend's results as they were"""
    xn, resid, w1, b1, w2, b2 = _inputs(m, hd, m + hd)
    got = ops.mlp_tc(xn, resid, ops.round_tf32(w1), b1, ops.round_tf32(w2), b2)
    assert torch.equal(got, _cublas_tf32(xn, resid, w1, b1, w2, b2))


@pytest.mark.parametrize("hd", [128, 512])
def test_mlp_tc_zero_weights_exact_residual(ops, hd):
    xn, resid, w1, b1, w2, b2 = _inputs(1000, hd, 3)
    z1, zb1, z2 = torch.zeros_like(w1), torch.zeros_like(b1), torch.zeros_like(w2)
    assert torch.equal(ops.mlp_tc(xn, resid, z1, zb1, z2, b2), resid + b2)


def test_mlp_tc_rows_independent_and_masked(ops):
    m, hd = 300, 512
    xn, resid, w1, b1, w2, b2 = _inputs(m, hd, 5)
    clean = ops.mlp_tc(xn, resid, w1, b1, w2, b2)
    xn[137, 11] = float("nan")
    dirty = ops.mlp_tc(xn, resid, w1, b1, w2, b2)
    bad = torch.isnan(dirty).any(dim=1)
    assert bad[137].item() and bad.sum().item() == 1
    keep = torch.arange(m, device=DEV) != 137
    assert torch.equal(dirty[keep], clean[keep])


def test_mlp_tc_out_of_range_rows_untouched(ops, monkeypatch):
    """the output is the first M rows of a larger NaN-filled buffer: the last tile's rows past M stay NaN"""
    m, hd = 129, 128
    xn, resid, w1, b1, w2, b2 = _inputs(m, hd, 9)
    buf = torch.full((m + 127, 128), float("nan"), device=DEV)
    real_empty = torch.empty_like
    monkeypatch.setattr(torch, "empty_like", lambda t, **kw: buf[:m] if t is resid else real_empty(t, **kw))
    out = ops.mlp_tc(xn, resid, w1, b1, w2, b2)
    monkeypatch.undo()
    assert out.data_ptr() == buf.data_ptr() and torch.isfinite(buf[:m]).all() and torch.isnan(buf[m:]).all()


def test_mlp_tc_deterministic_and_graph_capturable(ops):
    args = _inputs(76800, 512, 11)
    a, b = ops.mlp_tc(*args), ops.mlp_tc(*args)
    assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.mlp_tc(*args)                                 # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.mlp_tc(*args)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_mlp_tc_rejects_unsupported_shapes(ops):
    xn, resid, w1, b1, w2, b2 = _inputs(64, 256, 1)
    with pytest.raises(ops.MacvoB200Error):
        ops.mlp_tc(xn, resid, w1, b1, w2, b2)             # hidden 256
    with pytest.raises(ops.MacvoB200Error):
        ops.mlp_tc(xn[:, :64].contiguous(), resid[:, :64].contiguous(), w1[:, :64].contiguous(), b1, w2[:64].contiguous(), b2[:64])


def _net(monkeypatch, flag):
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    monkeypatch.setenv("MACVO_B200_MLP_TC", flag)
    return FlowFormerCovNet(synthetic_state_dict(0), DEV)


def test_mlp_residual_fallbacks(ops, monkeypatch):
    """C = 256, a non-contiguous input, strict fp32 or MACVO_B200_MLP_TC=0 keep the torch ops"""
    calls = []
    real = ops.mlp_tc
    monkeypatch.setattr(ops, "mlp_tc", lambda *a: calls.append(1) or real(*a))
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        net = _net(monkeypatch, "1")
        p = "memory_encoder.cost_perceiver_encoder.vertical_encoder_layers.0.local_block.mlp."
        x, xn = torch.randn(2, 500, 128, device=DEV), torch.randn(2, 500, 128, device=DEV)
        fused = net._mlp_residual(x, xn, p, "fc1", "fc2")
        assert len(calls) == 1
        ref = x + F.linear(F.gelu(F.linear(xn, net.W[p + "fc1.weight"], net.W[p + "fc1.bias"])), net.W[p + "fc2.weight"], net.W[p + "fc2.bias"])
        assert (fused - ref).abs().max().item() <= 1e-2 * (ref - x).abs().max().item()
        net._mlp_residual(x, xn.transpose(0, 1).contiguous().transpose(0, 1), p, "fc1", "fc2")   # non-contiguous xn
        p256 = "context_encoder.svt.blocks.1.0.mlp."                                            # SVT stage 1: C = 256
        x2 = torch.randn(1, 300, 256, device=DEV)
        net._mlp_residual(x2, x2.clone(), p256, "fc1", "fc2")
        assert len(calls) == 1
        torch.backends.cuda.matmul.allow_tf32 = False
        net._mlp_residual(x, xn, p, "fc1", "fc2")
        torch.backends.cuda.matmul.allow_tf32 = True
        assert len(calls) == 1
        off = _net(monkeypatch, "0")
        assert not off.mlp_tensor_cores
        off._mlp_residual(x, xn, p, "fc1", "fc2")
        assert len(calls) == 1
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def test_frontend_with_and_without_fused_mlp():
    """640x480, depth 12: flow and covariance are bit-identical with the switch on and off, in TF32 mode because the kernel
    computes cuBLAS's TF32 bits at these shapes, in strict fp32 because the fused path does not engage there"""
    from types import SimpleNamespace as NS
    from macvo_b200 import build, plugins, synthetic
    build.build(verbose=False)
    fr = synthetic.make_sequence(2, 480, 640)
    fe = plugins.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp32", dec_dtype="fp32", decoder_depth=12,
                                               enforce_positive_disparity=False, cuda_graph=False))
    A = torch.cat([fr[1].imageL, fr[0].imageL]).to(DEV)
    B = torch.cat([fr[1].imageR, fr[1].imageL]).to(DEV)
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)

    def run(flag):
        fe.net.mlp_tensor_cores = flag
        with torch.inference_mode():
            flow, cov = fe.net.inference(A, B, shared=(0, 1))
        return flow.double(), cov.double()
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        (f1, c1), (f0, c0) = run(True), run(False)
        assert torch.equal(f1, f0) and torch.equal(c1, c0)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        (f1, c1), (f0, c0) = run(True), run(False)
        assert torch.equal(f1, f0) and torch.equal(c1, c0)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
