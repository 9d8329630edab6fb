"""Parity of the perceiver-layer kernels (csrc/nn_kernels.cu) against the torch fp32 ops they replace
(Module/Network/FlowFormer/core/encoder.py:12-55, core/attention.py:6-29, core/twins.py:103-114,173-183).
Floating point: tolerance 1e-5 relative to the output scale (different summation order, __expf)."""
import pytest
import torch
import torch.nn.functional as F

from tests.kernel_inventory import expect_variants

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    from macvo_b200 import ops
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    return ops


LAYER_NORM_VARIANT = {64: "layer_norm64_kernel", 128: "layer_norm_kernel<4>", 256: "layer_norm_kernel<8>", 512: "layer_norm_kernel<16>"}


@pytest.mark.parametrize("rows,c", [(1, 128), (7, 128), (4801, 128), (300, 256), (65, 512), (9600 * 8, 128), (9601, 64)])
def test_layer_norm(ops, rows, c):
    g = torch.Generator().manual_seed(rows + c)
    x = (torch.randn(rows, c, generator=g) * 3 + 1.5).to(DEV)
    w, b = torch.randn(c, generator=g).to(DEV), torch.randn(c, generator=g).to(DEV)
    for eps in (1e-5, 1e-6):
        ref = F.layer_norm(x.double(), (c,), w.double(), b.double(), eps)
        got = expect_variants(lambda: ops.layer_norm(x, w, b, eps), LAYER_NORM_VARIANT[c])
        assert (got.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    with pytest.raises(ops.MacvoB200Error):
        ops.layer_norm(x[:, :32].contiguous(), w[:32], b[:32])


@pytest.mark.parametrize("m,h,w", [(3, 8, 8), (5, 12, 16), (4, 60, 80), (2, 13, 17), (2, 90, 160)])
def test_patch_embed_conv1(ops, m, h, w):
    g = torch.Generator().manual_seed(m * h + w)
    maps = torch.randn(m, 1, h, w, generator=g).to(DEV)
    wt, b = (torch.randn(16, 1, 6, 6, generator=g) * 0.2).to(DEV), torch.randn(16, generator=g).to(DEV)
    x = F.pad(maps, (0, (8 - w % 8) % 8, 0, (8 - h % 8) % 8))
    ref = F.relu(F.conv2d(x.double(), wt.double(), b.double(), stride=2, padding=2))
    got = ops.patch_embed_conv1(maps, wt, b, allow_tf32=False)
    assert got.shape == ref.shape and got.is_contiguous(memory_format=torch.channels_last)
    assert (got.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    got = ops.patch_embed_conv1(maps, wt, b, allow_tf32=True)          # TF32 operands, fp32 accumulate (cuDNN's TF32 class)
    assert (got.double() - ref).abs().max().item() <= 3e-3 * ref.abs().max().item()
    # space-to-depth output: same bits, channel block (y & 1) * 2 + (x & 1) of the (ho/2, wo/2, 64) tensor
    s2d = ops.patch_embed_conv1(maps, wt, b, allow_tf32=True, s2d=True)
    ho, wo = got.shape[-2:]
    expect = got.reshape(m, 16, ho // 2, 2, wo // 2, 2).permute(0, 3, 5, 1, 2, 4).reshape(m, 64, ho // 2, wo // 2)
    assert s2d.shape == expect.shape and s2d.is_contiguous(memory_format=torch.channels_last) and torch.equal(s2d, expect)
    w2 = torch.randn(32, 16, 6, 6, generator=g).to(DEV)
    a = F.conv2d(got.double(), w2.double(), None, stride=2, padding=2)
    bb = F.conv2d(s2d.double(), ops.space_to_depth_filter(w2).double(), None, stride=1, padding=1)
    assert (a - bb).abs().max().item() <= 1e-9 * a.abs().max().item()


def _ref_attention(q, k, v, heads):
    B, J, C = k.shape
    d = C // heads
    qh = q.double().reshape(q.shape[0], -1, heads, d).permute(0, 2, 1, 3).expand(B, -1, -1, -1)
    kh, vh = (t.double().reshape(B, J, heads, d).permute(0, 2, 1, 3) for t in (k, v))
    a = (qh @ kh.transpose(-1, -2) * d ** -0.5).softmax(-1)
    return (a @ vh).permute(0, 2, 1, 3).reshape(B, -1, C)


# (batch, nq, nk, heads, head_dim, broadcast q): perceiver input layer / latent self-attention / decoder cross
# attention (few-queries kernel), windowed 7x7, vertical + SVT global attention (shared-K/V kernel)
ATTN_CASES = [(37, 8, 80, 8, 16, True), (50, 8, 8, 8, 16, False), (33, 1, 8, 8, 16, False),
              (12, 49, 49, 8, 16, False), (9, 49, 49, 4, 32, False), (3, 1000, 300, 8, 16, False),
              (2, 700, 300, 4, 32, False), (2, 130, 75, 8, 32, False), (1, 5, 513, 8, 16, False),
              (5, 6, 21, 4, 32, False), (7, 3, 10, 8, 16, False), (2, 9, 30, 8, 16, False),
              (41, 1, 8, 8, 8, False), (6, 8, 20, 8, 8, True), (77, 1, 8, 4, 16, False), (300, 1, 5, 8, 8, False)]


def _attn_variant(b, nq, heads, d, bc, tf32):
    """macvo_small_attention_ex's choice for plain (B, N, C) operands (csrc/nn_kernels.cu): one query, up to 8 queries of 8
    heads (4 slots x 2), the tensor-core kernel for 16+ queries in TF32 mode, else the shared-K/V kernel"""
    if nq == 1 and not bc and d <= 16:
        return f"attn_single_query_kernel<{d}>"
    if nq <= 8 and heads == 8 and d <= 16:
        return f"attn_few_queries_kernel<{d}>"
    return f"attn_tc_kernel<{d}>" if tf32 and nq >= 16 else f"attn_shared_kv_kernel<{d}>"


@pytest.mark.parametrize("case", ATTN_CASES)
def test_small_attention(ops, case):
    b, nq, nk, heads, d, bc = case
    g = torch.Generator().manual_seed(sum(case[:5]))
    q = (torch.randn(1 if bc else b, nq, heads * d, generator=g) * 1.5).to(DEV)
    k = (torch.randn(b, nk, heads * d, generator=g) * 1.5).to(DEV)
    v = torch.randn(b, nk, heads * d, generator=g).to(DEV)
    ref = _ref_attention(q, k, v, heads)
    got = expect_variants(lambda: ops.small_attention(q, k, v, heads, allow_tf32=False), _attn_variant(b, nq, heads, d, bc, False))
    assert got.shape == ref.shape
    assert (got.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    # tensor-core path (TF32 operands, fp32 accumulate): the tolerance of a TF32 bmm-softmax-bmm
    got = expect_variants(lambda: ops.small_attention(q, k, v, heads, allow_tf32=True), _attn_variant(b, nq, heads, d, bc, True))
    assert (got.double() - ref).abs().max().item() <= 4e-3 * ref.abs().max().item()


def test_network_native_layers_match_torch_layers(ops):
    """the whole network with csrc/nn_kernels.cu vs the same network on the torch ops (fp32, TF32 off)"""
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    g = torch.Generator().manual_seed(3)
    i1, i2 = torch.rand(1, 3, 96, 128, generator=g).to(DEV), torch.rand(1, 3, 96, 128, generator=g).to(DEV)
    net = FlowFormerCovNet(synthetic_state_dict(0), DEV, decoder_depth=4)
    f1, c1 = net.inference(i1, i2)
    net._ops = None
    f0, c0 = net.inference(i1, i2)
    assert (f1 - f0).abs().max().item() <= 2e-4 * max(1.0, f0.abs().max().item())
    assert ((c1 - c0).abs() / c0.abs().clamp_min(1e-6)).max().item() <= 1e-3


def test_gru_fused_kernels(ops):
    """csrc/decoder_fused.cu vs the SepConvGRU elementwise ops of core/gru.py:22-43 (torch fp32)."""
    g = torch.Generator().manual_seed(11)
    P = 1237
    mf, agg = torch.randn(P, 128, generator=g).to(DEV), torch.randn(P, 128, generator=g).to(DEV)
    gamma = torch.tensor([0.37], device=DEV)
    bufs = [torch.randn(P, 512, generator=g).to(DEV) for _ in range(4)]
    before = [b.clone() for b in bufs]
    ops.gru_input(mf, agg, gamma, bufs)
    for b, b0 in zip(bufs, before):
        assert torch.equal(b[:, :256], b0[:, :256]) and torch.equal(b[:, 256:384], mf)
        torch.testing.assert_close(b[:, 384:], mf + gamma * agg, rtol=1e-6, atol=1e-6)
    zr, q = torch.randn(P, 256, generator=g).to(DEV) * 3, torch.randn(P, 128, generator=g).to(DEV) * 3
    hx, rhx, z = bufs[0], bufs[1], torch.empty(P, 128, device=DEV)
    h0 = hx[:, :128].clone()
    bzr, bq = torch.randn(256, generator=g).to(DEV), torch.randn(128, generator=g).to(DEV)
    ops.gru_gates(zr, hx, z, rhx, bzr)
    torch.testing.assert_close(z, torch.sigmoid(zr[:, :128] + bzr[:128]), rtol=2e-6, atol=2e-7)
    torch.testing.assert_close(rhx[:, :128], torch.sigmoid(zr[:, 128:] + bzr[128:]) * h0, rtol=2e-6, atol=2e-7)
    dense = torch.empty(P, 128, device=DEV)
    ops.gru_blend(q, z, hx, dense, bq)
    ref = (1 - z) * h0 + z * torch.tanh(q + bq)
    torch.testing.assert_close(hx[:, :128], ref, rtol=2e-6, atol=2e-6)
    assert torch.equal(dense, hx[:, :128])
    with pytest.raises(ops.MacvoB200Error):
        ops.gru_gates(zr.t(), hx, z, rhx)


@pytest.mark.parametrize("shape", [(1, 60, 80), (1, 12, 16), (2, 13, 17), (1, 90, 160)])
def test_sepconv_gru_wgmma(ops, shape):
    """csrc/gru_conv_tc.cu (wgmma implicit GEMM, fp16 operands, fp32 state) vs SepConvGRU (core/gru.py:22-43) in float64:
    (a) against the same arithmetic with the convolution inputs / filters rounded to fp16 (what the kernel computes): 1e-3,
    (b) against the unrounded float64 GRU: 4e-3 (fp16 operand rounding, the TF32-class bound of this mode). Two steps, two units,
    so the layout ping-pong between the 1x5 and the 5x1 pass and the state hand-over to the next iteration are covered."""
    B, H, W = shape
    P = B * H * W
    g = torch.Generator().manual_seed(H * 1000 + W)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(DEV)
    names = {"convzr1": (256, 512, 1, 5), "convq1": (128, 512, 1, 5), "convzr2": (256, 512, 5, 1), "convq2": (128, 512, 5, 1)}
    ws = [{n: rnd(*sh, scale=0.03) for n, sh in names.items()} for _ in range(2)]
    bs = [{n: rnd(sh[0], scale=0.3) for n, sh in names.items()} for _ in range(2)]
    gru = ops.SepConvGruTC(ws, bs, B, H, W, DEV)
    inp = rnd(P, 128).relu()
    h0 = [torch.tanh(rnd(P, 128)) for _ in range(2)]
    gamma = torch.tensor([0.6], device=DEV)
    gru.set_context(inp)
    for u in range(2):
        gru.set_state(u, h0[u])

    def to_map(rows):
        return rows.view(B, H, W, -1).permute(0, 3, 1, 2).double()

    def ref_gru(h, x, w, b, rounded):
        q16 = (lambda t: t.half().double()) if rounded else (lambda t: t)
        for o, pad in (("1", (0, 2)), ("2", (2, 0))):
            hx = torch.cat([q16(h), q16(x)], 1)
            zr = torch.sigmoid(F.conv2d(hx, q16(w["convzr" + o].double()), b["convzr" + o].double(), padding=pad))
            z, r = zr[:, :128], zr[:, 128:]
            q = torch.tanh(F.conv2d(torch.cat([q16(r * h), q16(x)], 1), q16(w["convq" + o].double()), b["convq" + o].double(), padding=pad))
            h = (1 - z) * h + z * q
        return h

    # launch probe on a throwaway step, then back to the initial state (set_state rebuilds every operand a step reads):
    # every step runs both stages, the z / r convolution and then the q convolution
    zeros = torch.zeros(P, 128, device=DEV)
    expect_variants(lambda: torch.cuda.current_stream().wait_event(gru.step(zeros, zeros, gamma)), "gru_conv_tc_kernel<0>",
                    "gru_conv_tc_kernel<1>", "pack_motion_kernel")
    for u in range(2):
        gru.set_state(u, h0[u])
    ref_r, ref_t = [to_map(h) for h in h0], [to_map(h) for h in h0]
    for it in range(2):
        mf, agg = rnd(P, 128).relu(), rnd(P, 128)
        torch.cuda.current_stream().wait_event(gru.step(mf, agg, gamma))     # unit 1's chain runs on a side stream
        xs = torch.cat([inp, mf, mf + gamma * agg], 1)
        for u in range(2):
            # the fp16 rounding of x happens on the fp32 values the pack kernel forms
            ref_r[u] = ref_gru(ref_r[u], to_map(xs), ws[u], bs[u], True)
            ref_t[u] = ref_gru(ref_t[u], to_map(xs), ws[u], bs[u], False)
            got = to_map(gru.h[u])
            assert torch.isfinite(got).all()
            assert (got - ref_r[u]).abs().max().item() <= 1e-3, (it, u)
            assert (got - ref_t[u]).abs().max().item() <= 4e-3, (it, u)
    # pad rows of every operand buffer are still zero (the kernels only write pixel rows): layout U for the 1x5 pass, V for 5x1
    for buf in [gru.x[0]] + gru.h_rows[0] + gru.rh_rows[0]:
        n = B * (H + 4) * (W + 4)
        body = buf[2:2 + n].view(B, H + 4, W + 4, -1).clone()
        body[:, 2:H + 2, 2:W + 2] = 0
        assert not body.any() and not buf[:2].any() and not buf[2 + n:].any()
    for buf in [gru.x[1]] + gru.h_rows[1] + gru.rh_rows[1]:
        n = B * W * (H + 4)
        body = buf[2:2 + n].view(B * W, H + 4, -1)
        assert not body[:, :2].any() and not body[:, -2:].any() and not buf[:2].any() and not buf[2 + n:].any()


@pytest.mark.parametrize("rows,cols", [(3, 4), (17, 4800), (9, 8192), (5, 1236)])
def test_softmax_rows_f16(ops, rows, cols):
    """fused row softmax -> fp16 (the GMA attention matrix, gma.py:39-82) vs float64 softmax: half an fp16 ulp of the result + 1e-7"""
    g = torch.Generator().manual_seed(rows * cols)
    x = (torch.randn(2, rows, cols, generator=g) * 6).to(DEV)
    x[0, 0, : min(cols, 7)] = 40.0                                  # a dominant block: exp of the rest underflows gracefully
    got = ops.softmax_rows_f16(x)
    ref = torch.softmax(x.double(), dim=-1)
    assert got.dtype == torch.float16 and got.shape == x.shape
    assert ((got.double() - ref).abs() <= ref * 2.0 ** -10 + 1e-7).all()
    assert (got.double().sum(-1) - 1).abs().max().item() <= 2e-3
    with pytest.raises(ops.MacvoB200Error):
        ops.softmax_rows_f16(x.cpu())


@pytest.mark.parametrize("b,h,w", [(1, 5, 7), (2, 60, 80), (1, 13, 17)])
def test_convex_upsample(ops, b, h, w):
    """csrc/decoder_fused.cu convex_upsample_kernel vs `upsample_flow` (core/decoder.py:131-139) in float64"""
    from macvo_b200.flowformer_cov import FlowFormerCovNet
    g = torch.Generator().manual_seed(h * w)
    flow = (torch.randn(b, 2, h, w, generator=g) * 10).to(DEV)
    logits = (torch.randn(b, 576, h, w, generator=g) * 8).to(DEV).contiguous(memory_format=torch.channels_last)
    ref = FlowFormerCovNet.convex_upsample(flow.double(), 0.25 * logits.double())
    for m in (logits, logits.contiguous()):                     # channels_last (a conv output) and NCHW (copied once) inputs
        got = ops.convex_upsample(flow, m, 0.25)
        assert got.shape == (b, 2, 8 * h, 8 * w)
        assert (got.double() - ref).abs().max().item() <= 2e-6 * ref.abs().max().item()


def _to_rows_u(ops, x_map, shape):
    """(B, C, H, W) fp32 map -> zero-initialised layout-U fp16 rows via the pack kernel"""
    B, H, W = shape
    C = x_map.shape[1]
    rows = torch.zeros(ops.rows_count(B, H, W), C, dtype=torch.float16, device=DEV)
    ops.pack_rows(x_map.permute(0, 2, 3, 1).reshape(B * H * W, C).contiguous(), rows, 0, shape)
    return rows


def _from_rows_u(rows, shape):
    B, H, W = shape
    body = rows[2:2 + B * (H + 4) * (W + 4)].view(B, H + 4, W + 4, -1)
    pad = body.clone()
    pad[:, 2:H + 2, 2:W + 2] = 0
    assert not pad.any() and not rows[:2].any() and not rows[2 + B * (H + 4) * (W + 4):].any()     # padding untouched
    return body[:, 2:H + 2, 2:W + 2].permute(0, 3, 1, 2).double()


def _conv_tiles(b, h, w):
    """128-row tiles over the layout-U padded pixels of a (b, h, w) map"""
    return -(-(b * (h + 4) * (w + 4)) // 128)


def _conv_n_cta(n_pad, tiles, sms):
    """macvo_conv_tc's output-channel slicing (csrc/conv_tc.cu): as many slices as fit one wave of CTAs, each a multiple of 32
    columns and at most 256 wide (a wider single slice forces the slicing past one wave)"""
    slices = 1
    for s in range(1, 9):
        if n_pad % (32 * s) == 0 and n_pad // s <= 256 and (tiles * s <= sms or n_pad // slices > 256):
            slices = s
    return n_pad // slices


@pytest.mark.parametrize("shape", [(1, 60, 80), (2, 13, 17), (1, 90, 160)])
@pytest.mark.parametrize("cin,cout,k,relu", [(256, 192, 3, True), (128, 256, 3, True), (256, 2, 3, False), (192, 256, 1, True),
                                             (128, 126, 3, True), (64, 2, 3, False), (128, 64, 3, True)])
def test_conv_tc(ops, shape, cin, cout, k, relu):
    """csrc/conv_tc.cu vs F.conv2d in float64 on the same fp16-rounded operands: 1e-3 of the output scale (fp32 accumulation
    order; fp16 re-rounding of the fp16 output where one is written)."""
    B, H, W = shape
    P = B * H * W
    g = torch.Generator().manual_seed(cin * 7 + cout + k + H)
    x = (torch.randn(B, cin, H, W, generator=g)).to(DEV)
    w = (torch.randn(cout, cin, k, k, generator=g) * (cin * k * k) ** -0.5).to(DEV)
    b = torch.randn(cout, generator=g).to(DEV)
    ref = F.conv2d(x.half().double(), w.half().double(), b.double(), padding=k // 2)
    if relu:
        ref = ref.relu()
    scale = ref.abs().max().item()
    wp, bp, n = ops.pack_conv_filter(w, b)
    rows = _to_rows_u(ops, x, shape)
    out16 = torch.zeros(ops.rows_count(B, H, W), 256, dtype=torch.float16, device=DEV)
    o32 = 4 if H % 2 == 0 else 1                                # vector-store path | scalar path
    out32 = torch.full((P, cout + 8), 7.0, device=DEV)
    n_cta = _conv_n_cta(wp.shape[0], _conv_tiles(B, H, W), torch.cuda.get_device_properties(0).multi_processor_count)
    expect_variants(lambda: ops.conv_tc(rows, wp, bp, n, k, relu, shape, out16=out16, out16_offset=64 if cout <= 192 else 0,
                                        out32=out32, out32_offset=o32), f"conv_tc_kernel<{n_cta}>")
    got32 = out32[:, o32:o32 + cout].view(B, H, W, cout).permute(0, 3, 1, 2).double()
    assert (got32 - ref).abs().max().item() <= 1e-3 * scale
    assert (out32[:, :o32] == 7.0).all() and (out32[:, o32 + cout:] == 7.0).all()                   # neighbours untouched
    off = 64 if cout <= 192 else 0
    got16 = _from_rows_u(out16, shape)
    assert (got16[:, off:off + cout] - ref).abs().max().item() <= 2e-3 * scale
    assert not got16[:, :off].any() and not got16[:, off + cout:].any()
    if cout == 2:   # the heads' form: the result is added in place to a (B, 2, H, W) coordinate map
        cmap = torch.randn(B, 2, H, W, generator=g).to(DEV) * 30
        want = cmap.double() + ref
        ops.conv_tc(rows, wp, bp, n, k, relu, shape, add_to_map=cmap)
        assert (cmap.double() - want).abs().max().item() <= 1e-3 * scale + 1e-5 * 30
    if k == 1:      # dense rows in, dense fp16 rows out (the value projection's shape)
        dense_in = x.permute(0, 2, 3, 1).reshape(P, cin).half().contiguous()
        o16 = torch.zeros(P, cout, dtype=torch.float16, device=DEV)
        ops.conv_tc(dense_in, wp, None, n, 1, False, shape, in_dense=True, out16=o16, out16_dense=True)
        ref2 = F.conv2d(x.half().double(), w.half().double())
        assert (o16.view(B, H, W, cout).permute(0, 3, 1, 2).double() - ref2).abs().max().item() <= 2e-3 * ref2.abs().max().item()
    with pytest.raises(ops.MacvoB200Error):
        ops.conv_tc(rows[:-1], wp, bp, n, k, relu, shape, out32=out32)


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("cout,n_cta", [(192, 96), (150, 160), (224, 224), (320, 160)])
def test_conv_tc_slice_widths(ops, cout, n_cta, k):
    """the slice widths only some shapes select: 96 columns (a 7-slot operand ring), 160 (5 slots; cout 150 also leaves 10
    padded columns unstored), 224 (4 slots), and cout 320, which is cut into two 160-column slices even when that takes more
    than one wave. The width W is chosen from the SM count S with a copy of macvo_conv_tc's rule; the probe proves the choice.
    Enough K steps (64-channel blocks x taps) for the ring to wrap: 18 for 3x3 over 128 channels, 8 for 1x1 over 512.
    float64 reference on the fp16-rounded operands: 1e-3 (fp32 rows) / 2e-3 (fp16 rows) of the output scale."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_pad = -(-cout // 32) * 32
    if cout == 320:
        B, H, W = 1, 90, 160
        assert 2 * _conv_tiles(B, H, W) > sms                   # two slices are more than one wave: the 256-column limit forces them
    else:
        B, H = 1, 60
        W = next(w for w in range(60, 400) if _conv_n_cta(n_pad, _conv_tiles(B, H, w), sms) == n_cta)
    tiles = _conv_tiles(B, H, W)
    assert _conv_n_cta(n_pad, tiles, sms) == n_cta
    print(f"conv_tc: S = {sms}, {B} x {H} x {W}, cout {cout} (n_pad {n_pad}), {tiles} tiles -> {n_pad // n_cta} slices of {n_cta}")
    shape, P, cin, relu = (B, H, W), B * H * W, (128 if k == 3 else 512), k == 3
    g = torch.Generator().manual_seed(cout * 10 + k)
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    w = (torch.randn(cout, cin, k, k, generator=g) * (cin * k * k) ** -0.5).to(DEV)
    b = torch.randn(cout, generator=g).to(DEV)
    ref = F.conv2d(x.half().double(), w.half().double(), b.double(), padding=k // 2)
    if relu:
        ref = ref.relu()
    scale = ref.abs().max().item()
    wp, bp, n = ops.pack_conv_filter(w, b)
    rows = _to_rows_u(ops, x, shape)
    out16 = torch.zeros(ops.rows_count(B, H, W), n_pad, dtype=torch.float16, device=DEV)
    out32 = torch.full((P, cout), 7.0, device=DEV)
    expect_variants(lambda: ops.conv_tc(rows, wp, bp, n, k, relu, shape, out16=out16, out32=out32), f"conv_tc_kernel<{n_cta}>")
    got32 = out32.view(B, H, W, cout).permute(0, 3, 1, 2).double()
    assert (got32 - ref).abs().max().item() <= 1e-3 * scale
    got16 = _from_rows_u(out16, shape)
    assert (got16[:, :cout] - ref).abs().max().item() <= 2e-3 * scale
    assert not got16[:, cout:].any()                                 # padded filter columns are never stored


def test_conv_tc_rejects_unsliceable_width(ops):
    """352 output columns: no slice width (a multiple of 32, at most 256) divides them, so the call is refused and writes nothing"""
    B, H, W = 1, 12, 16
    shape, P = (B, H, W), B * H * W
    g = torch.Generator().manual_seed(352)
    x = torch.randn(B, 64, H, W, generator=g).to(DEV)
    wp, bp, n = ops.pack_conv_filter((torch.randn(352, 64, 3, 3, generator=g) * 0.05).to(DEV), torch.randn(352, generator=g).to(DEV))
    assert wp.shape[0] == 352
    rows = _to_rows_u(ops, x, shape)
    out16 = torch.full((ops.rows_count(B, H, W), 352), 3.0, dtype=torch.float16, device=DEV)
    out32 = torch.full((P, 352), 7.0, device=DEV)
    with pytest.raises(ops.MacvoB200Error):
        ops.conv_tc(rows, wp, bp, n, 3, True, shape, out16=out16, out32=out32)
    torch.cuda.synchronize()
    assert (out16 == 3.0).all() and (out32 == 7.0).all()


def test_flow_im2col(ops):
    """the 7x7 flow convolution as im2col rows + a 1x1 tensor-core convolution vs F.conv2d(flow, w, padding=3)"""
    B, H, W = 2, 13, 17
    P = B * H * W
    g = torch.Generator().manual_seed(5)
    c0, c1 = (torch.randn(B, 2, H, W, generator=g) * 20).to(DEV), (torch.randn(B, 2, H, W, generator=g) * 20).to(DEV)
    w, b = (torch.randn(128, 2, 7, 7, generator=g) * 0.1).to(DEV), torch.randn(128, generator=g).to(DEV)
    rows = torch.zeros(P, 128, dtype=torch.float16, device=DEV)
    mf32 = torch.zeros(P, 128, device=DEV)
    mf16 = torch.zeros(ops.rows_count(B, H, W), 128, dtype=torch.float16, device=DEV)
    ops.flow_im2col(c1, c0, rows, mf32, mf16)
    flow = c1 - c0
    assert torch.equal(mf32[:, 126:], flow.permute(0, 2, 3, 1).reshape(P, 2)) and not mf32[:, :126].any()
    assert torch.equal(_from_rows_u(mf16, (B, H, W))[:, 126:], flow.half().double())
    wp, bp, n = ops.pack_conv_filter(w.permute(0, 2, 3, 1).reshape(128, 98, 1, 1), b, in_channels=128)   # 1x1 over the im2col columns
    out = torch.zeros(P, 128, device=DEV)
    ops.conv_tc(rows, wp, bp, n, 1, True, (B, H, W), in_dense=True, out32=out)
    ref = F.conv2d(flow.half().double(), w.half().double(), b.double(), padding=3).relu()
    got = out.view(B, H, W, 128).permute(0, 3, 1, 2).double()
    assert (got - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


def test_lookup_rows_equals_lookup_map(ops):
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import cases
    cm, co = cases.lookup_inputs(2, 12, 16)
    cm, co = cm.to(DEV), co.to(DEV)
    a = expect_variants(lambda: ops.corr_lookup(cm, co), "corr_lookup_kernel<false>")
    b = expect_variants(lambda: ops.corr_lookup(cm, co, rows=True), "corr_lookup_kernel<true>")
    assert b.shape == (2 * 12 * 16, 81)
    assert torch.equal(a.permute(0, 2, 3, 1).reshape(-1, 81), b)          # same arithmetic, other layout: bit-exact


@pytest.mark.parametrize("tf32", [False, True])
def test_fused_qkv_attention_with_additive_terms(ops, tf32):
    """[q|k|v] consumed in place + q_add / k_add slices (b % period) == plain attention on the summed operands"""
    g = torch.Generator().manual_seed(21)
    B, N, heads, d, period = 12, 49, 8, 16, 4
    C = heads * d
    qkv = torch.randn(B, N, 3 * C, generator=g).to(DEV)
    qa, ka = torch.randn(period, N, C, generator=g).to(DEV), torch.randn(period, N, C, generator=g).to(DEV)
    idx = torch.arange(B, device=DEV) % period
    ref = _ref_attention(qkv[..., :C] + qa[idx], qkv[..., C:2 * C] + ka[idx], qkv[..., 2 * C:], heads)
    got = ops.fused_qkv_attention(qkv, heads, qa, ka, allow_tf32=tf32)
    assert (got.double() - ref).abs().max().item() <= (4e-3 if tf32 else 2e-5) * ref.abs().max().item()
    q, k, v = torch.randn(6, 200, C, generator=g).to(DEV), torch.randn(6, 75, C, generator=g).to(DEV), torch.randn(6, 75, C, generator=g).to(DEV)
    qa2 = torch.randn(2, 200, C, generator=g).to(DEV)
    ref = _ref_attention(q + qa2[torch.arange(6, device=DEV) % 2], k, v, heads)
    got = ops.attention_with_terms(q, k, v, heads, qa2, allow_tf32=tf32)
    assert (got.double() - ref).abs().max().item() <= (4e-3 if tf32 else 2e-5) * ref.abs().max().item()


@pytest.mark.parametrize("m,nk", [(5, 80), (3, 35), (2, 96), (7, 1)])
def test_latent_pool_equals_cross_attention(ops, m, nk):
    """fused perceiver input layer (no K / V tensors) vs the explicit MultiHeadAttention of core/attention.py:32-68,
    including the key bias that the fused form drops (softmax-invariant). TF32 tolerance."""
    g = torch.Generator().manual_seed(m * 100 + nk)
    tokens = torch.randn(m, nk, 128, generator=g).to(DEV)
    q = torch.randn(1, 8, 128, generator=g).to(DEV)
    wk, wv = (torch.randn(128, 128, generator=g) * 0.15).to(DEV), (torch.randn(128, 128, generator=g) * 0.15).to(DEV)
    bk, bv = torch.randn(128, generator=g).to(DEV), torch.randn(128, generator=g).to(DEV)
    k = F.linear(tokens.double(), wk.double(), bk.double())
    v = F.linear(tokens.double(), wv.double(), bv.double())
    ref = _ref_attention(q.double(), k, v, 8)
    got = ops.latent_pool(tokens, q[0], wk, wv, bv)
    assert got.shape == (m, 8, 128)
    assert (got.double() - ref).abs().max().item() <= 4e-3 * ref.abs().max().item()


def _token_tile(pixels, sms):
    """macvo_decoder_token's tile choice (csrc/decoder_token.cu): 72-pixel tiles when, at one CTA per SM, they need fewer
    pixel slots over all waves than 64-pixel tiles"""
    cost = lambda tp: -(-(-(-pixels // tp)) // sms) * tp
    return 72 if cost(72) < cost(64) else 64


# the last case takes its width from the SM count S: a pixel count in (64 S, 72 S] selects 72-pixel tiles
@pytest.mark.parametrize("b,h,w", [(1, 5, 7), (2, 12, 16), (2, 60, 80), (1, 33, 47), pytest.param(2, 55, None, id="tile72")])
def test_decoder_token_kernel(ops, b, h, w):
    """csrc/decoder_token.cu vs a float64 torch evaluation of the chain it replaces (decoder.py:20-76,112-116) with the
    network's own weights: token MLP, LayerNorm + sine embedding, q projection, 8-head attention over the pixel's 8
    cost-memory tokens, output projection, FFN; out = [cost_global | cost_forward | 0]. fp32 FMA kernel -> 1e-5.
    Both tile widths run, each with fp32 rows and fp16 layout-U rows out; the 72-pixel case has a ragged last tile and the
    batch boundary inside a tile."""
    from macvo_b200.flowformer_cov import synthetic_state_dict, sine_embed
    sd = {k: v.to(DEV) for k, v in synthetic_state_dict(0).items() if k.startswith("memory_decoder.")}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if w is None:
        w = next(w for w in range(1, 4096) if _token_tile(b * h * w, sms) == 72 and (b * h * w) % 72 and (h * w) % 72)
    P = b * h * w
    tile = _token_tile(P, sms)
    print(f"decoder_token: S = {sms}, B x H x W = {b} x {h} x {w} = {P} pixels -> {tile}-pixel tiles")
    g = torch.Generator().manual_seed(P)
    cf = torch.randn(P, 81, generator=g).to(DEV) * 2
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    coords = (torch.stack([xs, ys], 0).unsqueeze(0).repeat(b, 1, 1, 1) + torch.randn(b, 2, h, w, generator=g) * 5).to(DEV)
    key, value = torch.randn(P, 8, 64, generator=g).to(DEV), torch.randn(P, 8, 64, generator=g).to(DEV)
    blob = ops.decoder_token_blob(sd)
    variant = f"decoder_token_kernel<{tile}>"
    got = expect_variants(lambda: ops.decoder_token(cf, coords, key, value, blob), variant)
    assert got.shape == (P, 160) and torch.equal(got[:, 64:145], cf) and not got[:, 145:].any()
    # the fp16 layout-U variant (the tensor-core motion encoder's input) holds the same rows, rounded once
    rows16 = torch.zeros(ops.rows_count(b, h, w), 192, dtype=torch.float16, device=DEV)
    assert expect_variants(lambda: ops.decoder_token(cf, coords, key, value, blob, out16_rows=rows16), variant) is rows16
    body = _from_rows_u(rows16, (b, h, w))                                      # (B, 192, H, W); asserts the padding stayed zero
    assert torch.equal(body[:, :160].permute(0, 2, 3, 1).reshape(P, 160), got.half().double()) and not body[:, 160:].any()

    m, ca = "memory_decoder.", "memory_decoder.decoder_layer.cross_attend."
    W = {k: v.double() for k, v in sd.items()}
    lin = lambda x, p: F.linear(x, W[p + ".weight"].flatten(1), W[p + ".bias"])
    x = cf.double()
    query = lin(F.gelu(lin(x, m + "flow_token_encoder.0")), m + "flow_token_encoder.2")
    enc = sine_embed(coords.double().permute(0, 2, 3, 1).reshape(P, 2), 64)
    qin = F.layer_norm(query, (64,), W[ca + "norm1.weight"], W[ca + "norm1.bias"], 1e-5) + enc
    q = lin(qin, ca + "q").view(P, 8, 1, 8)                                   # (P, heads, 1, d)
    kh, vh = key.double().view(P, 8, 8, 8).transpose(1, 2), value.double().view(P, 8, 8, 8).transpose(1, 2)   # (P, heads, tokens, d)
    a = (torch.matmul(q, kh.transpose(-1, -2)) * 8 ** -0.5).softmax(-1) @ vh
    a = a.reshape(P, 64)
    gl = query + lin(torch.cat([a, query], 1), ca + "proj")
    gl = gl + lin(F.gelu(lin(F.layer_norm(gl, (64,), W[ca + "norm2.weight"], W[ca + "norm2.bias"], 1e-5), ca + "ffn.0")), ca + "ffn.3")
    err = (got[:, :64].double() - gl).abs().max().item()
    assert err <= 1e-5 * gl.abs().max().item(), err / gl.abs().max().item()


@pytest.mark.parametrize("rows,c", [(7, 128), (76800, 128), (4801, 256), (65, 512)])
def test_add_layer_norm(ops, rows, c):
    g = torch.Generator().manual_seed(rows + c)
    x, r = (torch.randn(rows, c, generator=g) * 2).to(DEV), torch.randn(rows, c, generator=g).to(DEV)
    w, b = torch.randn(c, generator=g).to(DEV), torch.randn(c, generator=g).to(DEV)
    s, y = ops.add_layer_norm(x, r, w, b, 1e-6)
    assert torch.equal(s, x + r)
    ref = F.layer_norm((x + r).double(), (c,), w.double(), b.double(), 1e-6)
    assert (y.double() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
