"""B200_TartanVODepth on the H100: macvo_stereo_head against the float64 oracle (oracle/stereo.py) and against the torch
epilogue, the network against the reference fixtures (tests/golden/tartanvo_depth_*.pt), and the plugin's outputs, CUDA
graph, cov_mode and errors."""
import pytest
import torch

from tests.golden import make_golden_tartanvo_depth as gen

DEV = "cuda"
pytestmark = pytest.mark.gpu
TF32_UNIT = 2.0 ** -11          # unit roundoff of tf32 (10 explicit mantissa bits, round to nearest)


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    from macvo_b200 import build, ops
    build.build(verbose=False)
    ops.load_library()
    return ops


@pytest.fixture(autouse=True)
def _restore_precision_flags():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev[:2]
        torch.set_float32_matmul_precision(prev[2])


def _strict_fp32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")


def _default_flags():
    torch.backends.cuda.matmul.allow_tf32 = False         # torch's defaults
    torch.backends.cudnn.allow_tf32 = True


@pytest.fixture(scope="module")
def net(lib):
    from macvo_b200 import stereonet
    return stereonet.StereoCovNetDevice(stereonet.synthetic_stereo_state_dict(0), DEV)


def _run_kernel(lib, net, xd, xc, cat0, bf, H, W, margin, fill=float("nan")):
    from macvo_b200 import stereonet
    depth = torch.full((1, 1, H, W), fill, device=DEV)
    var = torch.full((1, 1, H, W), fill, device=DEV) if xc is not None else None
    wd, sd = net.head[stereonet.DISP]
    wc, sc = net.head[stereonet.COV] if xc is not None else (None, None)
    lib.stereo_head(xd.to(DEV), xc.to(DEV) if xc is not None else None, cat0.to(DEV), wd, sd, wc, sc, bf, margin, depth, var)
    torch.cuda.synchronize()
    return depth.cpu(), (var.cpu() if var is not None else None)


# ---------------------------------------------------------------------------------------------------------------------------
# kernel vs the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------------
def _check_head(sd, xd, xc, cat0, bf, depth, var):
    """Each head's conv_c13 output is recovered from the kernel's depth / variance and compared with the float64 oracle
    within 4 u S, u the tf32 unit roundoff and S the oracle with every term by its magnitude (two operand roundings per
    product of K = 512 terms, plus fp32 accumulation and the fp32 tail, all far below u)."""
    from oracle import stereo as ost
    d_ref = ost.head_out(sd, "feature.stereo.", xd.double(), cat0.double(), False)
    d_abs = ost.head_out(sd, "feature.stereo.", xd.double(), cat0.double(), False, absolute=True)
    d_got = bf / depth.double() * 0.02
    err = (d_got - d_ref).abs()
    bound = 4 * TF32_UNIT * d_abs + 1e-6 * d_ref.abs()
    assert (err <= bound).all(), f"disparity head: max err {err.max().item():.3g}, worst ratio {(err / bound).max().item():.3g}"
    if xc is None:
        return
    c_ref = ost.head_out(sd, "decoder.", xc.double(), cat0.double(), True)
    c_abs = ost.head_out(sd, "decoder.", xc.double(), cat0.double(), True, absolute=True)
    disp = d_got / 0.02
    c_got = var.double() * disp.pow(4) / bf ** 2
    err = (c_got - c_ref).abs()
    bound = 4 * TF32_UNIT * c_abs + 1e-5 * c_ref.abs() + 1e-30
    assert (err <= bound).all(), f"covariance head: max err {err.max().item():.3g}, worst ratio {(err / bound).max().item():.3g}"


HEAD_SHAPES = [(16, 24), (13, 21), (1, 1), (5, 9), (112, 160), (224, 320)]


@pytest.mark.parametrize("mode", ["Est", "None"])
@pytest.mark.parametrize("h2,w2", HEAD_SHAPES)
def test_kernel_matches_float64_oracle(lib, net, h2, w2, mode):
    _default_flags()
    from macvo_b200 import stereonet
    g = torch.Generator().manual_seed(h2 * 100 + w2)
    # inputs at the scale of the synthetic network's conv_c10 outputs and cat0
    xd, xc, cat0 = (torch.randn(1, 64, h2, w2, generator=g) for _ in range(3))
    est = mode == "Est"
    H, W = 2 * h2 + 10, 2 * w2 + 6
    depth, var = _run_kernel(lib, net, xd, xc if est else None, cat0, 80.0, H, W, (5, 3))
    sd = stereonet.synthetic_stereo_state_dict(0)
    crop = (..., slice(5, 5 + 2 * h2), slice(3, 3 + 2 * w2))
    _check_head(sd, xd, xc if est else None, cat0, 80.0, depth[crop], var[crop] if est else None)
    inside = torch.zeros((H, W), dtype=torch.bool)
    inside[5:5 + 2 * h2, 3:3 + 2 * w2] = True
    assert torch.isnan(depth[0, 0][~inside]).all()
    if est:
        assert torch.isnan(var[0, 0][~inside]).all()


def test_kernel_on_the_reference_head_inputs(lib, net, golden):
    """the reference's own conv_c10 outputs and cat0 (the `small` fixture's window): the kernel against the oracle bound,
    and the reference's depth / variance within the same order"""
    _default_flags()
    from macvo_b200 import stereonet
    g = golden("tartanvo_depth_small.pt")["head"]
    h2, w2 = g["xd"].shape[-2:]
    depth, var = _run_kernel(lib, net, g["xd"], g["xc"], g["cat0"], 80.0, 2 * h2, 2 * w2, (0, 0))
    _check_head(stereonet.synthetic_stereo_state_dict(0), g["xd"], g["xc"], g["cat0"], 80.0, depth, var)
    h, w = g["depth"].shape[-2:]
    ref_disp = 80.0 / g["depth"]
    rel = ((80.0 / depth[..., :h, :w] - ref_disp).abs().max() / ref_disp.abs().max()).item()
    print(f"stereo_head vs reference fixture window: disparity deviation {rel:.3g} of its scale")
    assert rel <= 1e-3


@pytest.mark.parametrize("b_disp,b_cov", [(0.0, 0.0), (0.0, 0.05), (-0.0731, 0.0), (0.1234, -0.2), (0.1234, 0.0371)])
def test_degenerate_heads_match_the_torch_epilogue_exactly(lib, b_disp, b_cov):
    """conv_c13 with zero weights: each head's output is exactly its bias, so the kernel's epilogue (/ 0.02, depth and
    variance) must equal torch's on the device bit for bit, including inf, NaN, negative depth and zero variance"""
    _default_flags()
    from macvo_b200 import stereonet
    n = stereonet.StereoCovNetDevice(stereonet.synthetic_stereo_state_dict(0), DEV)
    for p, b in ((stereonet.DISP, b_disp), (stereonet.COV, b_cov)):
        small = n.head[p][1]
        small[-17:-1] = 0.0
        small[-1] = b
    g = torch.Generator().manual_seed(5)
    xd, xc, cat0 = (torch.randn(1, 64, 9, 11, generator=g) for _ in range(3))
    bf = 0.31 * 412.7
    depth, var = _run_kernel(lib, n, xd, xc, cat0, bf, 18, 22, (0, 0))
    out_d = torch.full((1, 1, 18, 22), b_disp, device=DEV)
    out_c = torch.relu(torch.full((1, 1, 18, 22), b_cov, device=DEV))
    ref_d, ref_v = stereonet.depth_torch(out_d, out_c, bf)
    same = lambda a, b: torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert same(depth, ref_d.cpu()), (depth[0, 0, 0, 0].item(), ref_d[0, 0, 0, 0].item())
    assert same(var, ref_v.cpu()), (var[0, 0, 0, 0].item(), ref_v[0, 0, 0, 0].item())


def test_kernel_writes_only_the_crop_and_checks_arguments(lib, net):
    _default_flags()
    from macvo_b200 import stereonet
    g = torch.Generator().manual_seed(3)
    xd, xc, cat0 = (torch.randn(1, 64, 10, 12, generator=g) for _ in range(3))
    depth, var = _run_kernel(lib, net, xd, xc, cat0, 50.0, 27, 31, (3, 4), fill=12345.0)
    inside = torch.zeros((27, 31), dtype=torch.bool)
    inside[3:23, 4:28] = True
    for t in (depth, var):
        assert (t[0, 0][~inside] == 12345.0).all() and (t[0, 0][inside] != 12345.0).all()
    wd, sd = net.head[stereonet.DISP]
    wc, sc = net.head[stereonet.COV]
    a, c, k = xd.to(DEV), xc.to(DEV), cat0.to(DEV)
    out = torch.zeros(1, 1, 20, 24, device=DEV)
    ok = dict(xd=a, xc=c, cat0=k, w11_d=wd, small_d=sd, w11_c=wc, small_c=sc, bf=1.0, margin=(0, 0), depth=out,
              var=out.clone())
    lib.stereo_head(**ok)
    for bad in (dict(xd=a[:, :32].contiguous()), dict(cat0=k[..., :5].contiguous()), dict(xc=None),
                dict(w11_d=wd[:2].contiguous()), dict(small_c=sc[:10].contiguous()), dict(margin=(1, 0)),
                dict(depth=torch.zeros(1, 1, 19, 24, device=DEV)), dict(xd=xd), dict(var=out[..., :10].contiguous()),
                dict(depth=torch.zeros(1, 1, 20, 24, device=DEV, dtype=torch.float64))):
        with pytest.raises(lib.MacvoB200Error):
            lib.stereo_head(**dict(ok, **bad))
    _strict_fp32()
    with pytest.raises(lib.MacvoB200Error, match="allow_tf32"):
        lib.stereo_head(**ok)
    raw = lib.load_library().macvo_stereo_head
    args = [a.data_ptr(), c.data_ptr(), k.data_ptr(), 10, 12, wd.data_ptr(), sd.data_ptr(), wc.data_ptr(), sc.data_ptr(),
            1.0, 1.0, 0, 0, 20, 24, out.data_ptr(), out.data_ptr(), None]
    for i, v in ((0, None), (2, None), (3, 0), (4, -1), (5, None), (7, None), (11, -1), (13, 19), (14, 23), (15, None),
                 (16, None)):
        bad = list(args)
        bad[i] = v
        assert raw(*bad) == -1, i


# ---------------------------------------------------------------------------------------------------------------------------
# network and plugin
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def P(lib):
    from macvo_b200 import plugins
    return plugins


def _plugin(P, **kw):
    from types import SimpleNamespace as NS
    return P.B200_TartanVODepth(NS(**dict(dict(weight="synthetic:0", device="cuda:0", cov_mode="Est"), **kw)))


def _to_dev(f):
    from types import SimpleNamespace as NS
    return NS(**dict(vars(f), imageL=f.imageL.to(DEV), imageR=f.imageR.to(DEV)))


# deviation from the reference fixture: disparity (bf / depth) over its scale, and the 99th percentile of the variance's
# per-pixel relative error (the variance divides by disparity^4, so near-zero disparities amplify any rounding); measured on
# an H100 80GB HBM3 at a 700 W power limit over the four fixture shapes
STRICT_FP32_TOL = (1e-5, 1e-4)       # at most 1.3e-6 / 7.6e-6 measured
DEFAULT_FLAGS_TOL = (3e-3, 3e-2)     # at most 7.4e-4 / 7.3e-3 measured (cuDNN in TF32, head in macvo_stereo_head)


@pytest.mark.parametrize("flags", ["strict_fp32", "default"])
@pytest.mark.parametrize("name", list(gen.CASES))
def test_network_matches_reference_fixture(P, golden, name, flags):
    g = golden(f"tartanvo_depth_{name}.pt")
    (_strict_fp32 if flags == "strict_fp32" else _default_flags)()
    out = _plugin(P, cuda_graph=False).estimate(_to_dev(gen.frame(name)))
    s = g["stride"]
    depth, cov = out.depth[..., ::s, ::s].cpu(), out.cov[..., ::s, ::s].cpu()
    assert torch.equal(torch.isnan(depth), torch.isnan(g["depth"]))
    fin = torch.isfinite(g["depth"])
    disp, ref = 80.0 / depth[fin].double(), 80.0 / g["depth"][fin].double()
    rel_d = ((disp - ref).abs().max() / ref.abs().max()).item()
    rel_v = ((cov[fin].double() - g["cov"][fin]).abs() / g["cov"][fin].double().abs().clamp_min(1e-30)).quantile(0.99).item()
    print(f"tartanvo depth {name} {flags}: disparity deviation {rel_d:.3g} of its scale, variance p99 relative {rel_v:.3g}")
    tol = STRICT_FP32_TOL if flags == "strict_fp32" else DEFAULT_FLAGS_TOL
    assert rel_d <= tol[0] and rel_v <= tol[1], (rel_d, rel_v)


def test_kernel_path_against_torch_head_path_at_480x640(P, lib, monkeypatch):
    """default flags: the plugin with macvo_stereo_head against the same plugin with the head as torch ops (cuDNN TF32)"""
    _default_flags()
    from macvo_b200 import stereonet
    f = _to_dev(gen.frame("tartanair"))
    a = _plugin(P, cuda_graph=False).estimate(f)

    def torch_head(xd, xc, cat0, w11_d, small_d, w11_c, small_c, bf, margin, depth, var):
        n = P_net[0]
        d, v = stereonet.depth_torch(n.head_torch(stereonet.DISP, xd, cat0),
                                     n.head_torch(stereonet.COV, xc, cat0) if xc is not None else None, bf)
        my, mx = margin
        depth[..., my:my + d.shape[-2], mx:mx + d.shape[-1]].copy_(d)
        if var is not None:
            var[..., my:my + d.shape[-2], mx:mx + d.shape[-1]].copy_(v)
    m = _plugin(P, cuda_graph=False)
    P_net = [m.net]
    monkeypatch.setattr(lib, "stereo_head", torch_head)
    b = m.estimate(f)
    assert torch.equal(torch.isnan(a.depth), torch.isnan(b.depth))
    fin = torch.isfinite(b.depth)
    da, db = 80.0 / a.depth[fin].double(), 80.0 / b.depth[fin].double()
    rel = ((da - db).abs().max() / db.abs().max()).item()
    print(f"480x640 kernel path vs torch-head path (default flags): disparity deviation {rel:.3g} of its scale")
    assert rel <= 3e-3                   # 4.6e-4 measured


@pytest.mark.parametrize("flags", ["strict_fp32", "default"])
@pytest.mark.parametrize("name", ["small", "kitti"])
def test_plugin_outputs_graph_replay_and_cov_mode(P, name, flags):
    (_strict_fp32 if flags == "strict_fp32" else _default_flags)()
    f = _to_dev(gen.frame(name))
    H, W = gen.CASES[name]
    (my, mx), (h64, w64) = P.B200_TartanVODepth.geometry(H, W)
    graphed, eager, none = _plugin(P), _plugin(P, cuda_graph=False), _plugin(P, cov_mode="None")
    a, b, c, n = graphed.estimate(f), graphed.estimate(f), eager.estimate(f), none.estimate(f)
    same = lambda x, y: torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))
    for o in (a, b, c):
        assert o.depth.shape == o.cov.shape == (1, 1, H, W) and o.depth.device == torch.device("cuda:0")
    assert same(a.depth, b.depth) and same(a.cov, b.cov), "graph replay differs from the first call"
    assert same(a.depth, c.depth) and same(a.cov, c.cov), "graph replay differs from cuda_graph: false"
    assert n.cov is None and none.provide_cov is False and graphed.provide_cov is True
    assert same(n.depth, a.depth), "cov_mode None changes the depth"
    inside = torch.zeros((H, W), dtype=torch.bool)
    inside[my:my + h64, mx:mx + w64] = True
    assert torch.equal(torch.isnan(a.depth[0, 0]).cpu(), ~inside)
    assert a.depth.data_ptr() != b.depth.data_ptr() and a.cov.data_ptr() != b.cov.data_ptr()
    keep = b.depth.clone()
    with torch.inference_mode():
        a.depth.zero_()
    graphed.estimate(f)
    assert same(b.depth, keep)


def test_plugin_guards_and_flags(P):
    _default_flags()
    m = _plugin(P)
    m.estimate(_to_dev(gen.frame("small")))
    assert torch.backends.cudnn.allow_tf32 is True and torch.backends.cuda.matmul.allow_tf32 is False
    with pytest.raises(AssertionError, match="shape changed"):
        m.estimate(_to_dev(gen.frame("euroc")))
    f = _to_dev(gen.frame("small"))
    f.baseline = f.baseline * 2
    f.frame_baseline = f.frame_baseline * 2
    with pytest.raises(AssertionError, match="baseline"):
        m.estimate(f)
    from tests.golden import tartanvo_cases
    small = tartanvo_cases.frame(f.imageL[..., :255, :])
    small.imageR = f.imageR[..., :255, :]
    with pytest.raises(ValueError, match="64x64 average pooling"):
        _plugin(P).estimate(small)
