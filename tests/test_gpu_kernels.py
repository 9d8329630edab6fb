"""GPU parity tests (H100): every CUDA kernel, called through the C ABI (macvo_b200.ops -> ctypes),
against the CPU oracle on the same seeded inputs and against the committed golden fixtures.

Tolerances (written next to each assert):
  * keypoint indices, dense maps of (a7), NMS / threshold: BIT-EXACT
  * correlation volume: |err| <= 2e-6 * |f1_i| * |f2_j|  (fp32-class; SIMT and 3xfp16 tensor-core modes)
  * window lookup: 1e-5 relative to the map scale
  * covariance: 1e-5 relative (north_star: 1e-4)
  * PGO pose: 1e-8 against the fp64 oracle (north_star: 1e-4)
"""
import numpy as np
import pytest
import torch

from oracle import covariance as ocov
from oracle import frontend as ofe
from oracle import keypoint as okp
from oracle import pgo as opgo
from tests.golden import cases
from tests.kernel_inventory import expect_variants

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from macvo_b200 import build, ops as _ops
    build.build(verbose=False)
    _ops.load_library()
    torch.backends.cuda.matmul.allow_tf32 = False        # default corr mode = the fp32-class 3 x fp16 split
    torch.backends.cudnn.allow_tf32 = False
    return _ops


DEV = "cuda"


def test_golden_inputs_reproduce_on_this_host(golden):
    """(runs first) the seeded inputs regenerated on the GPU host equal, bit for bit, the ones the fixtures were made from"""
    for name, digest in cases.golden_input_shas().items():
        assert golden(name)["input_sha"] == digest, f"{name}: inputs generated on this host differ from the fixture's"


# ---- (a3) correlation volume --------------------------------------------------------------------------
def _corr_check(out, f1, f2, tol):
    B, D, H, W = f1.shape
    ref = ofe.corr_volume(f1.double(), f2.double()).reshape(B, H * W, H * W)
    scale = f1.reshape(B, D, -1).double().norm(dim=1).unsqueeze(2) * f2.reshape(B, D, -1).double().norm(dim=1).unsqueeze(1)
    err = ((out.reshape(B, H * W, H * W).double().cpu() - ref).abs() / scale).max().item()
    assert tol is None or err <= tol, f"max scaled error {err:.3e} > {tol:.1e}"
    return err


@pytest.mark.parametrize("name", list(cases.CORR_CASES))
def test_corr_simt_matches_oracle_and_golden(ops, golden, name):
    g = golden(f"corr_{name}.pt")
    B, H1, W1 = g["shape"]
    f1, f2 = cases.corr_inputs(B, H1, W1)
    out = ops.corr_build(f1.to(DEV), f2.to(DEV), mode=ops.CORR_SIMT)
    assert out.shape == (B, 1, H1, W1, H1, W1) and out.dtype == torch.float32
    _corr_check(out, f1, f2, 2e-6)
    rows, cols = cases.corr_sample_index(H1 * W1)
    sample = out.reshape(B, H1 * W1, H1 * W1).cpu()[:, rows][:, :, cols]
    torch.testing.assert_close(sample, g["sample"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("shape", [(2, 12, 16), (1, 30, 40), (2, 60, 80), (1, 80, 80), (1, 9, 13)])
def test_corr_tensor_core_3xf16(ops, shape):
    """wgmma kernel, fp32-class accuracy via the fp16 hi/lo split; incl. ragged M/N tile edges."""
    B, H1, W1 = shape
    f1, f2 = cases.corr_inputs(B, H1, W1)
    if (H1 * W1) % 8:
        with pytest.raises(ops.MacvoB200Error):
            ops.corr_build(f1.to(DEV), f2.to(DEV), mode=ops.CORR_TC_3XF16)
        return
    d1, d2 = f1.to(DEV), f2.to(DEV)
    out = expect_variants(lambda: ops.corr_build(d1, d2, mode=ops.CORR_TC_3XF16), "corr_tc_kernel<3>", "split_transpose_kernel")
    _corr_check(out, f1, f2, 2e-6)
    simt = ops.corr_build(f1.to(DEV), f2.to(DEV), mode=ops.CORR_SIMT)
    torch.testing.assert_close(out, simt, rtol=1e-4, atol=2e-4)


@pytest.mark.parametrize("shape", [(2, 12, 16), (1, 30, 40), (2, 60, 80), (1, 80, 80), (1, 9, 13), (1, 90, 160)])
@pytest.mark.parametrize("layout", ["channels_last", "nchw"])
def test_corr_tensor_core_tf32(ops, shape, layout):
    """wgmma tf32, one pass straight over the fp32 K-major features (the mode used when TF32 matmuls are allowed,
    like the reference's own torch.matmul under Frontend.py:275-277). Operands are truncated to 10 mantissa bits by the
    tensor core: |err| <= 2^-9 |f1_i| |f2_j| worst case; asserted at 6e-4 (measured ~2e-4 over 23 M entries), and the
    result must equal an fp64 product of the TRUNCATED operands to fp32 accumulation accuracy (2e-6): that pins the
    arithmetic itself, not just its error class. Incl. ragged tile edges and the 1280x720 size (N = 14400)."""
    B, H1, W1 = shape
    f1, f2 = cases.corr_inputs(B, H1, W1)
    d1, d2 = f1.to(DEV), f2.to(DEV)
    if layout == "channels_last":
        d1, d2 = d1.contiguous(memory_format=torch.channels_last), d2.contiguous(memory_format=torch.channels_last)
    if (H1 * W1) % 8:
        with pytest.raises(ops.MacvoB200Error):
            ops.corr_build(d1, d2, mode=ops.CORR_TC_TF32)
        return
    out = expect_variants(lambda: ops.corr_build(d1, d2, mode=ops.CORR_TC_TF32), "corr_tc_kernel<2>")
    n = H1 * W1
    if n <= 6400:
        _corr_check(out, f1, f2, 6e-4)
        trunc = lambda t: (t.view(torch.int32) & -8192).view(torch.float32)          # keep sign, exponent, 10 mantissa bits
        rna = lambda t: ((t.view(torch.int32) + 4096) & -8192).view(torch.float32)   # round to nearest, ties away
        e_trunc = _corr_check(out, trunc(f1.clone()), trunc(f2.clone()), None)
        e_rna = _corr_check(out, rna(f1.clone()), rna(f2.clone()), None)
        assert e_trunc <= 2e-6, f"not the truncated-operand product: trunc {e_trunc:.2e}, round-to-nearest {e_rna:.2e}"
    else:   # N = 14400: sampled rows against the truncated-operand fp64 product (no O(N^2) CPU work)
        trunc = lambda t: (t.view(torch.int32) & -8192).view(torch.float32)
        a, b = trunc(f1.clone()).reshape(B, 256, n).double(), trunc(f2.clone()).reshape(B, 256, n).double()
        rows = torch.arange(0, n, 997)
        ref = torch.einsum("bdi,bdj->bij", a[:, :, rows], b)
        got = out.reshape(B, n, n)[:, rows].double().cpu()
        scale = a[:, :, rows].norm(dim=1).unsqueeze(2) * b.norm(dim=1).unsqueeze(1)
        assert ((got - ref).abs() / scale).max().item() <= 2e-6


def test_corr_default_mode_follows_allow_tf32(ops):
    f1, f2 = cases.corr_inputs(2, 12, 16)
    d1, d2 = f1.to(DEV), f2.to(DEV)
    try:
        torch.backends.cuda.matmul.allow_tf32 = True
        a = ops.corr_build(d1, d2)
        assert torch.equal(a, ops.corr_build(d1, d2, mode=ops.CORR_TC_TF32))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    assert torch.equal(ops.corr_build(d1, d2), ops.corr_build(d1, d2, mode=ops.CORR_TC_3XF16))


def test_corr_tensor_core_1xf16_exact_for_fp16_features(ops):
    """MACVO_Fast: features are already fp16 -> one tensor-core pass is exact (fp32 accumulate)."""
    f1, f2 = cases.corr_inputs(2, 30, 40)
    f1h, f2h = f1.half(), f2.half()
    d1, d2 = f1h.to(DEV), f2h.to(DEV)
    out = expect_variants(lambda: ops.corr_build(d1, d2), "corr_tc_kernel<1>")     # dispatches to the 1-pass mode
    _corr_check(out, f1h.float(), f2h.float(), 5e-7)


def test_corr_full_size_properties(ops):
    """640x480 size (N = 4800, B = 2): linearity in f1, symmetry corr(f1,f2)[i,j] == corr(f2,f1)[j,i],
    and a column checksum against a fp64 matrix-vector product (no O(N^2) CPU work)."""
    B, H1, W1 = 2, 60, 80
    f1, f2 = cases.corr_inputs(B, H1, W1)
    d1, d2 = f1.to(DEV), f2.to(DEV)
    c12 = ops.corr_build(d1, d2).reshape(B, 4800, 4800)
    c21 = ops.corr_build(d2, d1).reshape(B, 4800, 4800)
    torch.testing.assert_close(c12, c21.transpose(1, 2), rtol=1e-5, atol=2e-5)
    c_scaled = ops.corr_build(2 * d1, d2).reshape(B, 4800, 4800)
    torch.testing.assert_close(c_scaled, 2 * c12, rtol=1e-5, atol=3e-5)           # power-of-two scaling (up to fp16-subnormal rounding of lo)
    colsum = c12.double().sum(dim=2).cpu()                                         # sum_j C[i,j] = f1[:,i] . sum_j f2[:,j]
    ref = torch.einsum("bdi,bd->bi", f1.reshape(B, 256, -1).double(), f2.reshape(B, 256, -1).double().sum(-1))
    torch.testing.assert_close(colsum, ref, rtol=1e-5, atol=2e-3)


# ---- (a5) window lookup -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(cases.LOOKUP_CASES))
def test_lookup_golden(ops, golden, name):
    g = golden(f"lookup_{name}.pt")
    B, H1, W1 = g["shape"]
    cost_maps, coords = cases.lookup_inputs(B, H1, W1)
    keep = coords.clone()
    dcoords = coords.to(DEV)
    out = ops.corr_lookup(cost_maps.to(DEV), dcoords)
    assert torch.equal(dcoords.cpu(), keep)
    torch.testing.assert_close(out.cpu(), g["out"], rtol=1e-5, atol=1e-5 * cost_maps.abs().max().item())


@pytest.mark.parametrize("shape", [(2, 60, 80), (1, 33, 47)])
def test_lookup_full_size_vs_oracle(ops, shape):
    B, H1, W1 = shape
    cost_maps, coords = cases.lookup_inputs(B, H1, W1)
    out = ops.corr_lookup(cost_maps.to(DEV), coords.to(DEV)).cpu()
    ref = ofe.window_lookup(cost_maps, coords)
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5 * cost_maps.abs().max().item())


def test_lookup_integer_coords_first_iteration(ops):
    """iteration 0 of the decoder looks up at exact integer grid coordinates"""
    B, H1, W1 = 1, 20, 24
    cost_maps, _ = cases.lookup_inputs(B, H1, W1)
    ys, xs = torch.meshgrid(torch.arange(H1, dtype=torch.float32), torch.arange(W1, dtype=torch.float32), indexing="ij")
    coords = torch.stack([xs, ys], 0).unsqueeze(0)
    out = ops.corr_lookup(cost_maps.to(DEV), coords.to(DEV)).cpu()
    torch.testing.assert_close(out, ofe.window_lookup(cost_maps, coords), rtol=1e-5, atol=1e-4)


# ---- (a7) dense post-processing: bit exact ----------------------------------------------------------------
@pytest.mark.parametrize("name", list(cases.DENSE_CASES))
@pytest.mark.parametrize("epd", [0, 1])
def test_dense_postproc_bit_exact(ops, golden, epd, name):
    g = golden(f"dense_{name}_{epd}.pt")
    H, W = g["shape"]
    flow, cov = cases.dense_inputs(H, W)
    out = ops.dense_postproc(flow.to(DEV), cov.to(DEV), 0.25 * 320.0, bool(epd))
    for k in ("depth", "disparity", "depth_cov", "disparity_uncertainty", "flow", "flow_cov"):
        a, b = out[k].cpu(), g[k]
        assert a.shape == b.shape and a.dtype == torch.float32, k
        if not torch.equal(a.nan_to_num(123.0), b.nan_to_num(123.0)):
            # round-1 flake (2 of ~60 fresh-process runs): classify the next occurrence — is it the read-back, the kernel
            # run, the uploaded inputs, or the host-side input generation that differs?
            bad = a.nan_to_num(123.0) != b.nan_to_num(123.0)
            idx = bad.nonzero()[:4].tolist()
            again = out[k].cpu()
            rerun = ops.dense_postproc(flow.to(DEV), cov.to(DEV), 0.25 * 320.0, bool(epd))[k].cpu()
            import hashlib
            sha = lambda t: hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()[:12]
            raise AssertionError(
                f"{k}: {int(bad.sum())} mismatches at {idx}: got {a[bad][:4].tolist()} want {b[bad][:4].tolist()}; "
                f"second read-back equal to first: {torch.equal(again.nan_to_num(123.0), a.nan_to_num(123.0))}; "
                f"re-run equals golden: {torch.equal(rerun.nan_to_num(123.0), b.nan_to_num(123.0))}; "
                f"inputs sha {cases.sha(flow, cov)[:16]} (fixture: {g['input_sha'][:16]}); "
                f"upload round trip exact: {torch.equal(flow.to(DEV).cpu(), flow) and torch.equal(cov.to(DEV).cpu(), cov)}; "
                f"cpu capability {torch.backends.cpu.get_cpu_capability()} threads {torch.get_num_threads()}")
    if epd:
        assert out["depth_mask"].dtype == torch.bool and torch.equal(out["depth_mask"].cpu(), g["depth_mask"])
    else:
        assert out["depth_mask"] is None


# ---- (a8) selectors: bit exact indices ----------------------------------------------------------------------
@pytest.mark.parametrize("name", list(cases.SELECTOR_CASES))
def test_selectors_bit_exact(ops, golden, name):
    g = golden(f"selector_{name}.pt")
    H, W = g["shape"]
    flow, cov = cases.selector_inputs(H, W, g["variant"])
    score = ops.ScoreBuffers(H, W, DEV, 7)
    d = ops.dense_postproc(flow.to(DEV), cov.to(DEV), 0.25 * 320.0, False, score=score)   # fused scoring
    cand = ops.CandidateList(H, W, DEV)
    mm = cases.selector_match_mask(H, W).to(DEV) if g["variant"] == "masked" else None
    mw = cases.selector_mask_width(name)
    expect_variants(lambda: ops.select_candidates(score, mw, 100.0, mm, cand), "flag_count_kernel<0>")
    torch.manual_seed(cases.SELECTOR_RNG_SEED)
    kp = ops.sample_candidates(cand, g["num"])
    mcand = ops.CandidateList(H, W, DEV)
    expect_variants(lambda: ops.select_mapping_candidates(d["depth"], d["depth_cov"], mw, 5.0, 0.005, mcand), "flag_count_kernel<1>")
    mp = ops.sample_candidates(mcand, 2000)
    assert kp.dtype == torch.int64 and kp.is_cuda
    assert torch.equal(kp.cpu(), g["kp"]), "keypoint indices must be bit-exact"
    assert torch.equal(mp.cpu(), g["map_kp"]), "mapping-point indices must be bit-exact"
    # the deterministic half against the oracle: identical candidate mask and threshold
    mask, thr = okp.candidate_mask_nodepth(ofe.dense_postproc(flow, cov, 0.25, 320.0)["flow_cov"], 7, mw, 100.0,
                                           cases.selector_match_mask(H, W) if g["variant"] == "masked" else None)
    n = int(cand.n.item())
    assert n == int(mask.sum())
    assert torch.equal(cand.idx[:n].cpu().long(), torch.nonzero(mask.view(-1)).view(-1))
    assert cand.thresh.item() == np.float32(thr)


def test_selector_standalone_scoring_equals_fused(ops):
    H, W = 160, 224
    flow, cov = cases.selector_inputs(H, W, "plain")
    fused = ops.ScoreBuffers(H, W, DEV, 7)
    d = ops.dense_postproc(flow.to(DEV), cov.to(DEV), 80.0, False, score=fused)
    alone = ops.ScoreBuffers(H, W, DEV, 7)
    ops.score_only(d["flow_cov"], alone)
    assert torch.equal(fused.quality, alone.quality) and torch.equal(fused.nms, alone.nms)
    assert int(fused.n_cand.item()) == int(alone.n_cand.item()) == int(alone.nms.sum().item())


def test_selector_empty_nms_set_gives_no_keypoints(ops):
    """all-NaN covariance map: no NMS survivor -> threshold = max_match_cov, 0 keypoints, no error (like the reference)"""
    H, W = 96, 128
    cov = torch.full((1, 3, H, W), float("nan"))
    score = ops.ScoreBuffers(H, W, DEV, 7)
    ops.score_only(cov.to(DEV), score)
    cand = ops.CandidateList(H, W, DEV)
    ops.select_candidates(score, 32, 100.0, None, cand)
    kp = ops.sample_candidates(cand, 10)
    assert kp.shape == (0, 2) and kp.dtype == torch.int64
    assert cand.thresh[0].item() == 100.0 and int(cand.status.item()) == 1


@pytest.mark.parametrize("name", list(cases.SELECTOR_DEPTH_CASES))
def test_depth_aware_selector_bit_exact(ops, golden, name):
    """(a8') CovAwareSelector: quality = (depth_cov0 + depth_cov1) * flow quality, two medians, depth gates"""
    g = golden(f"selector_{name}.pt")
    H, W = g["shape"]
    (f0, c0), (f1, c1) = cases.selector_depth_inputs(H, W, g["variant"])
    d0 = ops.dense_postproc(f0.to(DEV), c0.to(DEV), 0.25 * 320.0, g["variant"] == "masked")
    d1 = ops.dense_postproc(f1.to(DEV), c1.to(DEV), 0.25 * 320.0, False)
    m0 = ~d0["depth_mask"] if g["variant"] == "masked" else None
    mm = cases.selector_match_mask(H, W).to(DEV) if g["variant"] == "masked" else None
    score, cand = ops.ScoreBuffers(H, W, DEV, 7), ops.CandidateList(H, W, DEV)
    ops.score_depth_aware(d1["flow_cov"], d0["depth_cov"], d1["depth_cov"], score)
    mw = cases.selector_mask_width(name)
    expect_variants(lambda: ops.select_candidates_depth(score, d0["depth"], d1["depth"], d0["depth_cov"], mw, 320.0 * 0.25, 250.0,
                                                        100.0, m0, mm, cand), "flag_count_kernel<2>")
    torch.manual_seed(cases.SELECTOR_RNG_SEED)
    kp = ops.sample_candidates(cand, g["num"])
    assert torch.equal(kp.cpu(), g["kp"]), "depth-aware keypoint indices must be bit-exact"


# ---- (a9) retrieve_pixels ---------------------------------------------------------------------------------------
def test_retrieve_pixels(ops):
    g = torch.Generator().manual_seed(0)
    m = torch.randn(1, 3, 50, 70, generator=g)
    kp_i = torch.stack([torch.randint(0, 70, (40,), generator=g), torch.randint(0, 50, (40,), generator=g)], -1)
    kp_f = kp_i.float() + torch.rand(40, 2, generator=g) * 0.99
    dm = m.to(DEV)
    for kp, variant in ((kp_i, "retrieve_pixels_kernel<long>"), (kp_f, "retrieve_pixels_kernel<float>")):
        dkp = kp.to(DEV)
        out = expect_variants(lambda: ops.retrieve_pixels(dkp, dm), variant).cpu()
        assert torch.equal(out, ofe.retrieve_pixels(kp, m))


# ---- (a10) covariance -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(cases.COV_CASES))
def test_match_covariance(ops, golden, name):
    g = golden(f"covariance_{name}.pt")
    H, W, K = g["shape"]
    kp, depth, flow_cov = cases.cov_inputs(H, W, K, g["kind"])
    fc = None if flow_cov is None else flow_cov.to(DEV)
    dkp, dd = kp.to(DEV), depth.to(DEV)
    variant = "match_cov_kernel<long>" if kp.dtype == torch.int64 else "match_cov_kernel<float>"
    cov, pt, status = expect_variants(lambda: ops.match_covariance(dkp, dd, fc, 320.0, 320.0, W / 2, H / 2, want_point=True), variant)
    assert cov.dtype == torch.float64 and cov.shape == (K, 3, 3) and int(status.item()) == 0
    # 1e-5 relative to each matrix' scale (north_star tolerance: 1e-4)
    ref = g["out"]
    scale = ref.abs().amax(dim=(1, 2), keepdim=True)
    assert ((cov.cpu() - ref).abs() / scale).max().item() < 1e-5
    if fc is not None:
        assert torch.equal(fc.cpu(), g["flow_cov_after"]), "in-place clamp of the caller's flow_cov"
    d = depth[0, 0, kp[:, 1].long(), kp[:, 0].long()]
    K3 = torch.tensor([[320.0, 0, W / 2], [0, 320.0, H / 2], [0, 0, 1]])
    torch.testing.assert_close(pt.cpu(), ocov.pixel2point_ned(kp.float() if kp.dtype != torch.float32 else kp, d, K3),
                               rtol=1e-5, atol=1e-5)


def test_match_covariance_axis_quirk(ops):
    """depth = u ramp: the sigma_uu-weighted kernel axis runs along image rows (SURVEY.md §7.3)."""
    H, W = 128, 160
    depth = torch.arange(W, dtype=torch.float32).view(1, 1, 1, W).expand(1, 1, H, W).contiguous()
    kp = torch.tensor([[80, 64]])
    for fc, expect_big in ((torch.tensor([[25.0, 0.0625, 0.0]]), False), (torch.tensor([[0.0625, 25.0, 0.0]]), True)):
        ref = ocov.match_covariance(kp, depth, fc.clone(), 320.0, 320.0, 80.0, 64.0)
        cov, _, _ = ops.match_covariance(kp.to(DEV), depth.to(DEV), fc.clone().to(DEV), 320.0, 320.0, 80.0, 64.0)
        torch.testing.assert_close(cov.cpu(), ref, rtol=1e-5, atol=1e-7)
        assert (cov[0, 0, 0].item() > 1.0) == expect_big


# ---- (a14)+(a15) pose-graph optimisation ----------------------------------------------------------------------------
def _pgo_device_args(c):
    f64 = lambda t: t.double().to(DEV)
    K = c["K"].double()
    intr = (K[0, 0].item(), K[1, 1].item(), K[0, 2].item(), K[1, 2].item(), float(torch.tensor([c["baseline"]]).double()))
    return (f64(c["pos_Tw"]), f64(c["kp2_uv"]), f64(c["kp2_disp"]), f64(c["uv_cov"]), f64(c["disp_cov"]), intr,
            f64(c["init_pose"]))


@pytest.mark.parametrize("name", list(cases.PGO_CASES))
@pytest.mark.parametrize("cluster", [1, 2, 8])
def test_pgo_solve_matches_oracle(ops, golden, name, cluster):
    g = golden(f"pgo_{name}.pt")
    c = cases.pgo_inputs(g["K"], g["seed"])
    pose, stats = ops.pgo_solve(*_pgo_device_args(c), cluster=cluster)
    torch.cuda.synchronize()
    trace = opgo.LMTrace()
    ref = opgo.lm_solve(cases.pgo_graph(c), trace=trace)
    np.testing.assert_allclose(pose.cpu().numpy(), ref, rtol=1e-8, atol=1e-9)       # vs the numpy oracle
    np.testing.assert_allclose(pose.cpu().numpy(), g["pose"].double().numpy(), rtol=1e-8, atol=1e-9)  # vs reference LM
    s = stats.cpu().numpy()
    assert int(s[0]) == trace.steps and int(s[1]) == trace.evaluations, "same accept / reject sequence"
    np.testing.assert_allclose(s[2], trace.losses[-1], rtol=1e-9)


@pytest.mark.parametrize("K", [2048, 4096])
def test_pgo_solve_large(ops, K):
    c = cases.pgo_inputs(K, 6)
    ref = opgo.lm_solve(cases.pgo_graph(c))
    poses = []
    for cluster in (1, 3, 5, 6, 7, 8):
        pose, _ = ops.pgo_solve(*_pgo_device_args(c), cluster=cluster)
        poses.append(pose.cpu().numpy())
        np.testing.assert_allclose(poses[-1], ref, rtol=1e-8, atol=1e-9)
    for p in poses[1:]:
        np.testing.assert_allclose(p, poses[0], rtol=1e-12, atol=1e-13)


def test_pgo_accumulate_packed(ops):
    c = cases.pgo_inputs(512, 6)
    g = cases.pgo_graph(c)
    pose = opgo.se3_exp(np.array([0.02, -0.01, 0.03, 0.004, -0.003, 0.002]))
    args = _pgo_device_args(c)
    acc = ops.pgo_accumulate(*args[:6], torch.tensor(pose).to(DEV)).cpu().numpy()
    W = np.stack([np.linalg.pinv(cb) for cb in g.cov_blocks()])
    A, b, Js, Rs = opgo.normal_equations(g, pose, W, 0.1)
    iu = np.triu_indices(6)
    np.testing.assert_allclose(acc[:21], A[:6, :6][iu], rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(acc[21:27], b[:6], rtol=1e-10, atol=1e-9)
    G = np.einsum("kai,kaj->ij", Js, Js)
    np.testing.assert_allclose(acc[27:48], G[:6, :6][iu], rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(acc[48:54], np.einsum("kai,ka->i", Js, Rs)[:6], rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(acc[54], opgo.robust_loss(g, pose, 0.1), rtol=1e-12)


def test_corr_build_channels_last_inputs_bit_identical(ops):
    """K-major (channels_last) features take the elementwise operand split; same operands -> same bits as the NCHW path"""
    f1, f2 = cases.corr_inputs(2, 12, 16)
    a = ops.corr_build(f1.to(DEV), f2.to(DEV))
    c1, c2 = (t.to(DEV).contiguous(memory_format=torch.channels_last) for t in (f1, f2))
    b = expect_variants(lambda: ops.corr_build(c1, c2), "corr_tc_kernel<3>", "split_kmajor_kernel")
    assert torch.equal(a, b)
    c = ops.corr_build(f1.to(DEV).contiguous(memory_format=torch.channels_last),
                       f2.to(DEV).contiguous(memory_format=torch.channels_last), mode=ops.CORR_TC_1XF16)
    assert torch.equal(c, ops.corr_build(f1.to(DEV), f2.to(DEV), mode=ops.CORR_TC_1XF16))


def test_pgo_rank_deficient_blocks_take_pseudo_inverse_weight(ops):
    """The reference weights every block with torch.pinverse(cov) (Graphs.py:139-148): a zero disparity variance or a
    singular 2x2 pixel covariance must get its Moore-Penrose weight (finite pose), not inf / NaN, and be flagged."""
    c = cases.pgo_inputs(64, 6)
    c["disp_cov"][3] = 0.0
    c["uv_cov"][5] = torch.tensor([1.0, 1.0, 1.0])          # det = 0, rank 1
    c["uv_cov"][9] = torch.tensor([0.0, 0.0, 0.0])          # zero block
    pose, stats = ops.pgo_solve(*_pgo_device_args(c))
    ref = opgo.lm_solve(cases.pgo_graph(c))                  # oracle: np.linalg.pinv per block
    assert np.isfinite(pose.cpu().numpy()).all()
    np.testing.assert_allclose(pose.cpu().numpy(), ref, rtol=1e-8, atol=1e-9)
    assert stats[7].item() == 1.0
    c2 = cases.pgo_inputs(64, 6)
    _, stats2 = ops.pgo_solve(*_pgo_device_args(c2))
    assert stats2[7].item() == 0.0


def test_pgo_solve_counted_reads_block_count_on_device(ops):
    """macvo_pgo_solve_counted: k = min(*k_dev, capacity) read on the device; fewer than min_k blocks leave the pose alone."""
    c = cases.pgo_inputs(64, 6)
    a = _pgo_device_args(c)
    cap = 96
    buf = ops.ObservationBuffers(cap, DEV)
    for name, t in (("pos_Tw", a[0]), ("pixel2_uv", a[1]), ("pixel2_disp", a[2]), ("pixel2_uv_cov", a[3]), ("pixel2_disp_cov", a[4])):
        buf.section(name)[:64] = t
    buf.n_obs.fill_(64)
    pose = a[6].clone()
    stats = torch.zeros(8, dtype=torch.float64, device=DEV)
    ops.pgo_solve_counted(buf, a[5], pose, stats, min_k=10)
    ref, _ = ops.pgo_solve(*a, cluster=1)
    np.testing.assert_allclose(pose.cpu().numpy(), ref.cpu().numpy(), rtol=1e-12, atol=1e-13)
    buf.n_obs.fill_(7)
    pose2 = a[6].clone()
    stats.zero_()
    ops.pgo_solve_counted(buf, a[5], pose2, stats, min_k=10)
    assert torch.equal(pose2, a[6]) and stats[6].item() == 1.0


# ---- (f4) trajectory post-process ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(cases.MOTION_CASES))
def test_motion_interpolate_kernel(ops, golden, name):
    """csrc/motion_interp.cu vs the reference's MotionInterpolate (golden) and the fp64 oracle: fp32 output of fp64
    arithmetic -> 2e-6 of the trajectory extent (blocked scan vs sequential fold differ at fp64 rounding only)."""
    from oracle import map_processor as omp
    g = golden(f"motion_{name}.pt")
    poses, need = cases.motion_inputs(g["F"], g["seed"], g["flagged"])
    d = poses.to(DEV).contiguous()
    count = ops.motion_interpolate_(d, need.to(DEV))
    tol = 2e-6 * max(1.0, float(g["out"].abs().max()))
    np.testing.assert_allclose(d.cpu().numpy(), g["out"].numpy(), rtol=0, atol=tol)
    ref, idx = omp.motion_interpolate(poses.numpy(), need.numpy())
    np.testing.assert_allclose(d.cpu().numpy(), ref, rtol=0, atol=tol)
    assert int(count.item()) == len(idx) and torch.equal(d[0].cpu(), poses[0])


def test_motion_interpolate_long_sequence_blocked_scan(ops):
    """F = 5000 (chunks of 5 motions per thread): the blocked scan must equal the sequential fold of the oracle"""
    from oracle import map_processor as omp
    poses, need = cases.motion_inputs(5000, 11, tuple(range(50, 4900, 13)))
    d = poses.to(DEV).contiguous()
    ops.motion_interpolate_(d, need.to(DEV))
    ref, _ = omp.motion_interpolate(poses.numpy(), need.numpy())
    np.testing.assert_allclose(d.cpu().numpy(), ref, rtol=0, atol=3e-6 * float(np.abs(ref).max()))


def test_cov_sanity_filter_kernel(ops):
    g = torch.Generator().manual_seed(1)
    c1, c2 = torch.randn(300, 3, 3, generator=g).double(), torch.randn(300, 3, 3, generator=g).double()
    c1[5, 1, 2] = float("nan"); c2[17, 0, 0] = float("inf"); c1[200, 2, 2] = -float("inf"); c2[299, 1, 1] = float("nan")
    good = ops.cov_sanity_filter(c1.to(DEV), c2.to(DEV)).cpu()
    bad = c1.isnan().any(dim=(-1, -2)) | c1.isinf().any(dim=(-1, -2)) | c2.isnan().any(dim=(-1, -2)) | c2.isinf().any(dim=(-1, -2))
    assert torch.equal(good, ~bad) and int((~good).sum()) == 4


@pytest.mark.parametrize("name", ["depth_small", "depth_masked", "depth_nan", "depth_euroc", "depth_kitti", "depth_kitti00",
                                  "depth_kitti00_nan", "depth_ragged", "depth_ragged_ties"])
def test_depth_aware_selector_plugin_class(ops, golden, name):
    """the PLUGIN class `B200_CovAwareSelector` (not just the ops): constructed from a YAML-shaped config with
    `max_depth: auto`, fed `IStereoDepth.Output` / `IMatcher.Output`-shaped objects like MACVO.py does"""
    from types import SimpleNamespace as NS
    from macvo_b200 import plugins as P
    g = golden(f"selector_{name}.pt")
    H, W = g["shape"]
    (f0, c0), (f1, c1) = cases.selector_depth_inputs(H, W, g["variant"])
    d0 = ops.dense_postproc(f0.to(DEV), c0.to(DEV), 0.25 * 320.0, g["variant"] == "masked")
    d1 = ops.dense_postproc(f1.to(DEV), c1.to(DEV), 0.25 * 320.0, False)
    cfg = NS(device=DEV, mask_width=cases.selector_mask_width(name), max_depth="auto", kernel_size=7, max_depth_cov=250.0,
             max_match_cov=100.0)
    P.B200_CovAwareSelector.is_valid_config(cfg)
    sel = P.B200_CovAwareSelector(cfg)
    depth0 = NS(depth=d0["depth"], cov=d0["depth_cov"], mask=(~d0["depth_mask"] if g["variant"] == "masked" else None))
    depth1 = NS(depth=d1["depth"], cov=d1["depth_cov"], mask=None)
    match = NS(flow=d1["flow"], cov=d1["flow_cov"], mask=(cases.selector_match_mask(H, W).to(DEV) if g["variant"] == "masked" else None))
    frame = NS(fx=320.0, frame_baseline=0.25)
    torch.manual_seed(cases.SELECTOR_RNG_SEED)
    kp = sel.select_point(frame, g["num"], depth0, depth1, match)
    assert torch.equal(kp.cpu(), g["kp"]) and sel.config.max_depth == 80.0


@pytest.mark.parametrize("name", list(cases.PGO_TYPE_CASES))
def test_pgo_other_graph_types(ops, golden, name):
    """graph types "icp" / "reproj" of TwoFrame_PGO (Optimizer.py:51-68) in the same persistent kernel: pose 1e-8 vs the
    fp64 oracle and vs the reference's LM_analytic run (golden), same accept / reject sequence; through the plugin adapter."""
    from types import SimpleNamespace as NS
    from macvo_b200 import plugins as P
    g = golden(f"pgo_{name}.pt")
    c = cases.pgo_inputs_typed(g["graph_type"], g["K"], g["seed"])
    trace = opgo.LMTrace()
    ref = opgo.lm_solve(cases.pgo_graph(c), trace=trace)
    inp = P.PGOInput(pos_Tw=c["pos_Tw"], kp2_uv=c["kp2_uv"], kp2_disp=c["kp2_disp"], uv_cov=c["uv_cov"], disp_cov=c["disp_cov"],
                     K=c["K"], baseline=c["baseline"], init_pose=c["init_pose"], kp2_d=c["kp2_d"], obs_cov=c["obs_cov"],
                     pts_cov=c["pts_cov"])
    for cluster in (1, 2, 3, 5, 6, 7):
        pose, stats = P.solve_two_frame_pgo(inp, DEV, cluster, g["graph_type"])
        np.testing.assert_allclose(pose.cpu().numpy(), ref, rtol=1e-8, atol=1e-9)
        np.testing.assert_allclose(pose.cpu().numpy(), g["pose"].double().numpy(), rtol=1e-8, atol=1e-9)
        s = stats.cpu().numpy()
        assert int(s[0]) == trace.steps and int(s[1]) == trace.evaluations
    ctx = P.B200_TwoFrame_PGO.init_context(NS(device=DEV, graph_type=g["graph_type"], autodiff=False, vectorize=True, parallel=False))
    _, out = P.B200_TwoFrame_PGO._optimize(ctx, inp)
    np.testing.assert_allclose(out.motion.reshape(-1).cpu().numpy(), ref, rtol=1e-8, atol=1e-9)
