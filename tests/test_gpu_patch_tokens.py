"""PatchEmbed's fused token head (csrc/patch_tokens_tc.cu): LayerNorm(W2 relu(W0a x + term[row % 80]) + b2) on TF32 tensor
cores, checked bit for bit against the four-op sequence it replaces (cuBLAS TF32 linear, add_rows_relu_, cuBLAS TF32 linear,
layer_norm), against float64 on tf32 inputs, for masking, determinism, graph capture, shape checks, the strict-fp32 path and
the whole frontend."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PERIOD = 80                      # 8 x 10 tokens per 60 x 80 cost map at 640x480
FRAME_ROWS = 9600 * PERIOD       # 2 x 4800 cost maps per frame
P = "memory_encoder.cost_perceiver_encoder.patch_embed."


@pytest.fixture(scope="module")
def ops():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    return ops


@pytest.fixture
def tf32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _inputs(rows, seed):
    """x, the full ffn_with_coord.0 filter (its first 64 input channels act on x), term, W2, b2, LayerNorm weight and bias,
    from rand / randn and exactly rounded arithmetic only, on the synthetic checkpoint's U(+-1/sqrt(fan_in)) scale"""
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, fan: (torch.rand(shape, generator=g) * 2 - 1) / fan ** 0.5
    x = torch.randn(rows, 64, generator=g) * 0.5
    w0 = u((128, 128), 128)
    term = torch.randn(PERIOD, 128, generator=g) * 0.25
    w2, b2 = u((128, 128), 128), u((128,), 128)
    lw, lb = 1 + torch.randn(128, generator=g) * 0.1, torch.randn(128, generator=g) * 0.1
    return [t.to(DEV) for t in (x, w0, term, w2, b2, lw, lb)]


def _four_ops(ops, x, w0, term, w2, b2, lw, lb):
    """the sequence FlowFormerCovNet.patch_embed runs without the fused kernel; w0 is the (128, 128) filter, sliced as there"""
    t = F.linear(x, w0[:, :64])
    t = ops.add_rows_relu_(t, term)
    return ops.layer_norm(F.linear(t, w2, b2), lw, lb)


def _fused(ops, x, w0, term, w2, b2, lw, lb):
    return ops.patch_tokens_tc(x, ops.round_tf32(w0[:, :64]), term, ops.round_tf32(w2), b2, lw, lb)


def test_patch_tokens_tc_matches_four_ops_at_frame_shape(ops, tf32):
    """(9600, 80, 64) tokens, as the network passes them: the kernel returns the unfused sequence's bits"""
    x, *w = _inputs(FRAME_ROWS, 1)
    x = x.view(9600, PERIOD, 64)
    got = _fused(ops, x, *w)
    assert got.shape == (9600, PERIOD, 128)
    assert torch.equal(got, _four_ops(ops, x, *w))


@pytest.mark.parametrize("rows", [1, 79, 127, 129, PERIOD * 1601])
def test_patch_tokens_tc_matches_four_ops_partial_tiles(ops, tf32, rows):
    """row counts that end inside a 128-row tile and inside an 80-token map. Every output row depends on its own input row
    only, so the reference is the four-op sequence over 80 x 1601 rows, cut to the first `rows`: for a few hundred rows
    cuBLAS picks other GEMM algorithms (another K order) than at the network's row counts, and no kernel returns both."""
    x, *w = _inputs(PERIOD * 1601, 5)
    assert torch.equal(_fused(ops, x[:rows], *w), _four_ops(ops, x, *w)[:rows])


def _ref64(ops, x, w0, term, w2, b2, lw, lb):
    """float64 evaluation on the tf32 values the tensor cores see: x rounded by the kernel, the weights as packed"""
    d = lambda t: t.double()
    rows = x.shape[0]
    h = F.relu(F.linear(d(ops.round_tf32(x)), d(ops.round_tf32(w0[:, :64]))) + d(term).repeat(-(-rows // PERIOD), 1)[:rows])
    return F.layer_norm(F.linear(h, d(ops.round_tf32(w2)), d(b2)), (128,), d(lw), d(lb), 1e-5)


@pytest.mark.parametrize("rows", [129, PERIOD * 1601])
def test_patch_tokens_tc_accuracy(ops, tf32, rows):
    args = _inputs(rows, 7 * rows)
    ref = _ref64(ops, *args)
    scale = ref.abs().max().item()
    err = (_fused(ops, *args).double() - ref).abs().max().item()
    err_cublas = (_four_ops(ops, *args).double() - ref).abs().max().item()
    assert err <= 1e-3 * scale, f"err {err:.3e} vs scale {scale:.3e}"
    assert err <= 1.5 * err_cublas, f"fused {err:.3e} vs cuBLAS TF32 sequence {err_cublas:.3e}"


def test_patch_tokens_tc_out_of_range_rows_untouched(ops, monkeypatch):
    """the output is the first rows of a larger NaN-filled buffer: the last tile's rows past `rows` stay NaN"""
    rows = 129
    x, w0, term, w2, b2, lw, lb = _inputs(rows, 9)
    w0t, w2t = ops.round_tf32(w0[:, :64]), ops.round_tf32(w2)
    buf = torch.full((rows + 127, 128), float("nan"), device=DEV)
    monkeypatch.setattr(torch, "empty", lambda *a, **kw: buf[:rows])
    out = ops.patch_tokens_tc(x, w0t, term, w2t, b2, lw, lb)
    monkeypatch.undo()
    assert out.data_ptr() == buf.data_ptr() and torch.isfinite(buf[:rows]).all() and torch.isnan(buf[rows:]).all()


def test_patch_tokens_tc_deterministic_and_graph_capturable(ops):
    x, w0, term, w2, b2, lw, lb = _inputs(FRAME_ROWS, 11)
    args = (x, ops.round_tf32(w0[:, :64]), term, ops.round_tf32(w2), b2, lw, lb)
    a, b = ops.patch_tokens_tc(*args), ops.patch_tokens_tc(*args)
    assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.patch_tokens_tc(*args)                        # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.patch_tokens_tc(*args)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_patch_tokens_tc_rejects_unsupported_shapes(ops):
    x, w0, term, w2, b2, lw, lb = _inputs(256, 3)
    w0a = w0[:, :64].contiguous()
    with pytest.raises(ops.MacvoB200Error):
        ops.patch_tokens_tc(torch.zeros(256, 128, device=DEV), w0, term, w2, b2, lw, lb)     # 128 input channels
    with pytest.raises(ops.MacvoB200Error):
        ops.patch_tokens_tc(x, w0a[:96], term, w2[:96, :96].contiguous(), b2[:96], lw[:96], lb[:96])   # 96 outputs
    with pytest.raises(ops.MacvoB200Error):
        ops.patch_tokens_tc(x, w0a, term[:, :64].contiguous(), w2, b2, lw, lb)                  # term of 64 channels
    with pytest.raises(ops.MacvoB200Error):
        ops.patch_tokens_tc(x.cpu(), w0a, term, w2, b2, lw, lb)


def _net():
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    return FlowFormerCovNet(synthetic_state_dict(0), DEV)


def test_patch_embed_takes_fused_head_in_tf32_mode_only(ops, monkeypatch):
    """TF32 mode runs the fused kernel; strict fp32 keeps the four ops"""
    calls = []
    real = ops.patch_tokens_tc
    monkeypatch.setattr(ops, "patch_tokens_tc", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    net = _net()
    maps = torch.randn(6, 1, 60, 80, device=DEV)
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        with torch.inference_mode():
            assert net.patch_embed(maps).shape == (6, PERIOD, 128)
        assert len(calls) == 1
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        with torch.inference_mode():
            assert net.patch_embed(maps).shape == (6, PERIOD, 128)
        assert len(calls) == 1
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def test_frontend_with_and_without_fused_patch_tokens(ops, monkeypatch):
    """640x480, depth 12, TF32 mode: flow and covariance are bit-identical with the token head fused and with it forced
    through the old linear / add_rows_relu_ / linear / layer_norm sequence"""
    from types import SimpleNamespace as NS
    from macvo_b200 import plugins, synthetic
    fr = synthetic.make_sequence(2, 480, 640)
    fe = plugins.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp32", dec_dtype="fp32", decoder_depth=12,
                                               enforce_positive_disparity=False, cuda_graph=False))
    A = torch.cat([fr[1].imageL, fr[0].imageL]).to(DEV)
    B = torch.cat([fr[1].imageR, fr[1].imageL]).to(DEV)
    W = fe.net.W

    def old_sequence(t, w0t, term, w2t, b2, lw, lb):
        t = F.linear(t, W[P + "ffn_with_coord.0.weight"][:, :64, 0, 0])
        t = ops.add_rows_relu_(t, term)
        t = F.linear(t, W[P + "ffn_with_coord.2.weight"][:, :, 0, 0], b2)
        return ops.layer_norm(t, lw, lb)

    def run():
        with torch.inference_mode():
            flow, cov = fe.net.inference(A, B, shared=(0, 1))
        return flow.double(), cov.double()
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        f1, c1 = run()
        monkeypatch.setattr(ops, "patch_tokens_tc", old_sequence)
        f0, c0 = run()
        assert torch.equal(f1, f0) and torch.equal(c1, c0)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
