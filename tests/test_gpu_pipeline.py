"""GPU end-to-end parity: the B200 plugins (network with the CUDA correlation / lookup kernels, fused
post-processing + selection, covariance, PGO) against the golden fixtures and against the CPU oracle
pipeline on the same seeded synthetic sequence."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests.golden import cases

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def plugins():
    assert torch.cuda.is_available()
    from macvo_b200 import build, plugins as P
    build.build(verbose=False)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    return P


def _strict_fp32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")


@pytest.mark.parametrize("name", list(cases.NET_CASES))
def test_network_with_cuda_kernels_matches_reference_golden(plugins, golden, name):
    """FlowFormerCov with the sm_90a corr + lookup kernels vs the REFERENCE network's CPU output (golden).
    fp32, TF32 off. The reference's own fp32 result sits ~1e-6 (flow) / ~2e-5 (covariance) from exact arithmetic at these
    sizes (tests/golden/make_golden_cfgA.py measures the same floor at 640x480); asserted: 2e-5 of the flow scale and 3e-4
    relative on the covariance. The 640x480 / depth-12 ladder in both precision modes is tests/test_gpu_parity_ladder.py."""
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    _strict_fp32()
    g = golden(f"net_{name}.pt")
    B, H, W = g["shape"]
    img1, img2 = cases.net_inputs(B, H, W)
    net = FlowFormerCovNet(synthetic_state_dict(0), DEV)
    flow, cov = net.inference(img1.to(DEV), img2.to(DEV))
    flow, cov = flow.cpu(), cov.cpu()
    fscale = g["flow"].abs().mean().item()
    assert (flow - g["flow"]).abs().max().item() <= 2e-5 * max(fscale, 1.0), (flow - g["flow"]).abs().max().item() / fscale
    rel = ((cov - g["cov"]).abs() / g["cov"].abs().clamp_min(1e-6)).max().item()
    assert rel <= 3e-4, rel


def _frontend(P, cuda_graph, depth=12):
    return P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp32", dec_dtype="fp32",
                                           decoder_depth=depth, enforce_positive_disparity=False, cuda_graph=cuda_graph))


def test_frontend_cuda_graph_equals_eager(plugins):
    from macvo_b200 import synthetic
    frames = synthetic.make_sequence(3, 96, 128)
    fe_g, fe_e = _frontend(plugins, True, 4), _frontend(plugins, False, 4)
    _strict_fp32()
    for t in (1, 2):
        dg, mg = fe_g.estimate_pair(frames[t - 1], frames[t])
        de, me = fe_e.estimate_pair(frames[t - 1], frames[t])
        assert dg.depth.shape == (1, 1, 96, 128) and mg.cov.shape == (1, 3, 96, 128) and mg.flow.dtype == torch.float32
        torch.testing.assert_close(mg.flow, me.flow, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(dg.depth, de.depth, rtol=1e-3, atol=1e-4)


def test_pipeline_gpu_vs_cpu_oracle(plugins):
    """Whole hot path on a 3-frame 192x256 synthetic sequence, B200 plugins vs the CPU oracle plugins.
    Dense maps agree to 1e-3 relative (fp32 network on two different BLAS back-ends); given IDENTICAL dense
    maps the selection is bit-exact (tested in test_gpu_kernels); here we check the end-to-end pose stays
    within 2e-3 and that keypoint sets overlap (a single flipped NMS tie changes the randperm draw)."""
    from macvo_b200 import synthetic
    from macvo_b200.flowformer_cov import synthetic_state_dict
    from macvo_b200.pipeline import TwoFrameOdometry
    from oracle import pipeline_cpu as pc
    _strict_fp32()
    H, W = 192, 256
    frames = synthetic.make_sequence(3, H, W)
    P = plugins
    fe = _frontend(P, False, 4)
    gpu = TwoFrameOdometry(
        fe, P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=7, mask_width=32, max_match_cov=100.0)),
        P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)),
        P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
        num_point=64, map_selector=P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)),
        keep_debug=True)
    cpu = TwoFrameOdometry(pc.CpuFrontend(synthetic_state_dict(0), decoder_depth=4), pc.CpuSelector(), pc.CpuCovariance(),
                           pc.CpuPGO(), num_point=64, map_selector=pc.CpuMapSelector(), keep_debug=True)
    torch.manual_seed(5)
    gpu.initialize(frames[0])
    rg = [gpu.run_pair(f) for f in frames[1:]]
    pg = gpu.finish()
    torch.manual_seed(5)
    cpu.initialize(frames[0])
    rc = [cpu.run_pair(f) for f in frames[1:]]
    pcpu = cpu.finish()
    for a, b in zip(rg, rc):
        fa, fb = a.extras["match01"].flow.cpu(), b.extras["match01"].flow
        assert (fa - fb).abs().max().item() <= 3e-3 * max(1.0, fb.abs().mean().item())
        da, db = a.extras["depth1"].depth.cpu(), b.extras["depth1"].depth
        assert ((da - db).abs() / db.abs().clamp_min(1e-3)).median().item() < 2e-2      # depth = bl*fx / |flow_x|, |flow_x| ~ 1 px
        assert abs(a.num_kp - b.num_kp) <= 8
    # pose: when both sides drew the SAME keypoints the poses must agree tightly. One flipped NMS tie (the dense maps
    # differ by ~1e-3 between cuDNN and MKL) shifts the whole randperm draw; with this random-weight network the flow is
    # not a consistent motion field, so poses from different keypoint subsets are unrelated -> only finiteness is checked
    # then. The exact chain (identical dense maps in, bit-exact keypoints, 1e-6 pose) is the next test.
    same = all(a.kp0_uv.shape == b.kp0_uv.shape and bool((a.kp0_uv.cpu() == b.kp0_uv.cpu()).all())
               for a, b in zip(rg, rc))
    assert torch.isfinite(pg).all() and torch.isfinite(pcpu).all()
    if same:
        np.testing.assert_allclose(pg.numpy(), pcpu.numpy(), rtol=0, atol=5e-2 * max(1.0, float(pcpu.abs().max())))


def test_pipeline_on_identical_dense_maps_is_exact(plugins):
    """Feed the GPU selector / covariance / PGO chain the CPU frontend's dense maps: keypoints bit-exact,
    covariances 1e-5, pose 1e-6 (north_star: 1e-4)."""
    from macvo_b200 import synthetic
    from macvo_b200.flowformer_cov import synthetic_state_dict
    from macvo_b200.pipeline import TwoFrameOdometry
    from oracle import pipeline_cpu as pc
    P = plugins
    _strict_fp32()      # a B200 frontend built by an earlier test switches matmul precision to "medium" process-wide
                        # (like the reference frontend does); on CPUs with bf16 units that degrades the ORACLE's einsum

    class UploadFrontend(pc.CpuFrontend):           # CPU network, outputs moved to the GPU as-is
        def _post(self, flow, cov, frame):
            d, m = super()._post(flow, cov, frame)
            up = lambda t: None if t is None else t.to(DEV).contiguous()
            return (NS(depth=up(d.depth), cov=up(d.cov), disparity=up(d.disparity),
                       disparity_uncertainty=up(d.disparity_uncertainty), mask=up(d.mask)),
                    NS(flow=up(m.flow), cov=up(m.cov), mask=None))
        retrieve_pixels = staticmethod(P.B200_FlowFormerCovFrontend.retrieve_pixels)

    H, W = 192, 256
    frames = synthetic.make_sequence(3, H, W)
    sd = synthetic_state_dict(0)
    gpu = TwoFrameOdometry(
        UploadFrontend(sd, decoder_depth=4),
        P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=7, mask_width=32, max_match_cov=100.0)),
        P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)),
        P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
        num_point=64, map_selector=P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)),
        keep_debug=True)
    cpu = TwoFrameOdometry(pc.CpuFrontend(sd, decoder_depth=4), pc.CpuSelector(), pc.CpuCovariance(), pc.CpuPGO(),
                           num_point=64, map_selector=pc.CpuMapSelector(), keep_debug=True)
    torch.manual_seed(5)
    gpu.initialize(frames[0])
    rg = [gpu.run_pair(f) for f in frames[1:]]
    pg = gpu.finish()
    torch.manual_seed(5)
    cpu.initialize(frames[0])
    rc = [cpu.run_pair(f) for f in frames[1:]]
    pcpu = cpu.finish()
    for a, b in zip(rg, rc):
        assert torch.equal(a.kp0_uv.cpu(), b.kp0_uv), "keypoint indices must be bit-exact"
        torch.testing.assert_close(a.kp1_uv.cpu(), b.kp1_uv, rtol=0, atol=0)
        ca, cb = a.extras["pos1_cov"], b.extras["pos1_cov"]
        rel = ((ca - cb).abs() / cb.abs().amax(dim=(1, 2), keepdim=True)).amax(dim=(1, 2))
        worst = int(rel.argmax())
        assert rel.max().item() < 1e-5, (rel.max().item(), worst, a.kp1_uv[worst].tolist(), ca[worst], cb[worst],
                                         (a.extras["depth1"].depth.cpu() - b.extras["depth1"].depth).abs().max().item())
        assert a.num_obs == b.num_obs and a.map_points == b.map_points
    np.testing.assert_allclose(pg.numpy(), pcpu.numpy(), rtol=1e-5, atol=1e-6)


def _upload_frontend_cls(P):
    from oracle import pipeline_cpu as pc

    class UploadFrontend(pc.CpuFrontend):           # CPU network, outputs moved to the GPU as-is
        def _post(self, flow, cov, frame):
            d, m = super()._post(flow, cov, frame)
            up = lambda t: None if t is None else t.to(DEV).contiguous()
            return (NS(depth=up(d.depth), cov=up(d.cov), disparity=up(d.disparity),
                       disparity_uncertainty=up(d.disparity_uncertainty), mask=up(d.mask)),
                    NS(flow=up(m.flow), cov=up(m.cov), mask=None))
        retrieve_pixels = staticmethod(P.B200_FlowFormerCovFrontend.retrieve_pixels)
    return UploadFrontend


def test_fused_tail_matches_cpu_oracle_chain(plugins):
    """(f3) device-side observation building + sanity filter + MatchObs packing + counted LM solve
    (`FusedTwoFrameOdometry`: one host sync per frame) against the CPU oracle chain on IDENTICAL dense maps:
    keypoints bit-exact, pixel2_uv bit-exact, observation covariances 1e-5 relative, survivor counts equal,
    poses 1e-6 (north_star: 1e-4)."""
    from macvo_b200 import synthetic
    from macvo_b200.flowformer_cov import synthetic_state_dict
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    from oracle import pipeline_cpu as pc
    P = plugins
    _strict_fp32()
    H, W = 192, 256
    frames = synthetic.make_sequence(4, H, W)
    sd = synthetic_state_dict(0)
    gpu = FusedTwoFrameOdometry(
        _upload_frontend_cls(P)(sd, decoder_depth=4),
        P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=7, mask_width=32, max_match_cov=100.0)),
        P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)),
        P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
        num_point=64, map_selector=P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)),
        keep_debug=True)
    cpu = TwoFrameOdometry(pc.CpuFrontend(sd, decoder_depth=4), pc.CpuSelector(), pc.CpuCovariance(), pc.CpuPGO(),
                           num_point=64, map_selector=pc.CpuMapSelector(), keep_debug=True)
    torch.manual_seed(5)
    gpu.initialize(frames[0])
    got = []
    for f in frames[1:]:
        r = gpu.run_pair(f)
        got.append((r, gpu.observations(), gpu.latest_pose()))
    pg = gpu.finish()
    torch.manual_seed(5)
    cpu.initialize(frames[0])
    rc = [cpu.run_pair(f) for f in frames[1:]]
    pcpu = cpu.finish()
    for (r, o, pose), b in zip(got, rc):
        assert o["status"] == 0
        keep = b.extras["keep"]
        assert o["num_kp"] == b.num_kp and o["num_obs"] == b.num_obs and r.map_points == b.map_points
        assert torch.equal(o["pixel1_uv"].long(), b.kp0_uv[keep]), "keypoint indices must be bit-exact"
        assert torch.equal(o["pixel2_uv"].float(), b.kp1_uv[keep]), "kp1 = kp0 + flow must be bit-exact"
        for name, ref in (("obs1_covTc", b.extras["pos0_cov"][keep]), ("obs2_covTc", b.extras["pos1_cov"][keep])):
            rel = ((o[name] - ref).abs() / ref.abs().amax(dim=(1, 2), keepdim=True)).amax()
            assert rel.item() < 1e-5, (name, rel.item())
        torch.testing.assert_close(o["pos_Tw"].float(), b.extras["pos_Tw"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(pg.numpy(), pcpu.numpy(), rtol=1e-5, atol=1e-6)


def test_fused_tail_equals_plugin_api_path(plugins):
    """Same frames through the plugin-API driver (`TwoFrameOdometry`, the calls MACVO.run_pair makes) and the fused
    device tail, both on the real B200 frontend: identical keypoints, poses within 1e-6."""
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    P = plugins
    _strict_fp32()
    frames = synthetic.make_sequence(4, 192, 256)

    def build(cls):
        return cls(_frontend(P, False, 4),
                   P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=7, mask_width=32, max_match_cov=100.0)),
                   P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)),
                   P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
                   num_point=64, map_selector=P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)),
                   keep_debug=True)
    a, b = build(TwoFrameOdometry), build(FusedTwoFrameOdometry)
    _strict_fp32()
    torch.manual_seed(5)
    a.initialize(frames[0])
    ra = [a.run_pair(f) for f in frames[1:]]
    pa = a.finish()
    torch.manual_seed(5)
    b.initialize(frames[0])
    for f, x in zip(frames[1:], ra):
        b.run_pair(f)
        o = b.observations()
        assert torch.equal(o["pixel1_uv"].long(), x.kp0_uv.cpu()[x.extras["keep"].cpu()])
        assert o["num_obs"] == x.num_obs
    pb = b.finish()
    np.testing.assert_allclose(pb.numpy(), pa.numpy(), rtol=1e-5, atol=1e-6)


def test_shared_image_is_encoded_once(plugins):
    """The frontend batches [t2.L, t1.L] against [t2.R, t2.L] (Frontend.py:284-285): t2.L appears on both sides, so the feature
    encoder sees 3 images instead of 4 (`shared=(0, 1)`). Same result as encoding it twice (batch-size dependent library kernel
    selection only: 1e-5 of the flow scale, 1e-4 relative on the covariance, strict fp32)."""
    from macvo_b200 import synthetic
    fe = _frontend(plugins, False, 4)
    _strict_fp32()
    fr = synthetic.make_sequence(3, 192, 256)
    A = torch.cat([fr[2].imageL, fr[1].imageL]).to(DEV)
    B = torch.cat([fr[2].imageR, fr[2].imageL]).to(DEV)
    f0, c0 = fe.net.inference(A, B)
    f1, c1 = fe.net.inference(A, B, shared=(0, 1))
    assert (f1 - f0).abs().max().item() <= 1e-5 * max(1.0, f0.abs().max().item())
    assert ((c1 - c0).abs() / c0.abs().clamp_min(1e-6)).max().item() <= 1e-4
    with pytest.raises(ValueError):
        fe.net.inference(A, B, shared=(0, 5))


@pytest.mark.parametrize("graph", [False, True])
def test_software_pipelined_frames_equal_sequential(plugins, graph):
    """`run_pair(frame, next_frame=...)` (next frontend launched ahead, this frame's tail on a second stream) returns exactly what
    the sequential driver returns: keypoints, observation buffers and poses bit-identical over 7 frames, eager and CUDA-graph
    frontend (the graph's static buffers are overwritten by the prefetched frame while the tail still runs)."""
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry
    P = plugins
    frames = synthetic.make_sequence(8, 192, 256, pin=True)

    def build():
        return FusedTwoFrameOdometry(
            _frontend(P, graph, 4),
            P.B200_CovAwareSelector_NoDepth(NS(device=DEV, kernel_size=7, mask_width=32, max_match_cov=100.0)),
            P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25)),
            P.B200_TwoFrame_PGO(NS(graph_type="disp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
            num_point=64, map_selector=P.B200_MappingPointSelector(NS(max_depth=5.0, max_depth_cov=0.005, mask_width=32)))

    runs = []
    for pipelined in (False, True):
        odo = build()
        torch.manual_seed(5)
        odo.initialize(frames[0])
        obs = []
        for i in range(1, len(frames)):
            nxt = frames[i + 1] if pipelined and i + 1 < len(frames) and i != 4 else None      # one sequential frame in between
            odo.run_pair(frames[i], next_frame=nxt)
            obs.append(odo.observations())
        runs.append((obs, odo.finish()))
    _strict_fp32()
    (oa, pa), (ob, pb) = runs
    assert torch.equal(pa, pb)
    for x, y in zip(oa, ob):
        assert x["num_obs"] == y["num_obs"] and x["num_kp"] == y["num_kp"]
        for k in ("pixel1_uv", "pixel2_uv", "pos_Tw", "obs1_covTc", "obs2_covTc", "map_cov", "map_pos_Tc"):
            assert torch.equal(x[k], y[k]), k


def test_match_covariance_accepts_macvo_transposed_view(plugins):
    """Odometry/MACVO.py:231-243 passes `retrieve_pixels(kp0_uv, match01.cov).T` — a NON-contiguous (K,3) view — and
    relies on the in-place clamp reaching that storage (it later becomes pixel2_uv_cov)."""
    from oracle import covariance as ocov
    P = plugins
    _strict_fp32()     # a frontend built by an earlier test leaves float32 matmul precision "medium", which also lowers the CPU oracle's
    H, W, K = 160, 224, 96
    kp, depth, flow_cov = cases.cov_inputs(H, W, K, "float_cov")
    frame = NS(fx=320.0, fy=320.0, cx=112.0, cy=80.0)
    model = P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25))
    base = flow_cov.T.contiguous().to(DEV)                 # (3,K) like retrieve_pixels returns
    view = base.T                                          # what MACVO.py hands to estimate()
    assert not view.is_contiguous()
    out = model.estimate(frame, kp.to(DEV), NS(depth=depth.to(DEV)), None, view)
    ref_fc = flow_cov.clone()
    ref = ocov.match_covariance(kp, depth, ref_fc, 320.0, 320.0, 112.0, 80.0)
    assert out.device.type == "cpu" and out.dtype == torch.float64
    rel = ((out - ref).abs() / ref.abs().amax(dim=(1, 2), keepdim=True)).amax().item()
    assert rel < 1e-5, rel
    assert torch.equal(base.T.cpu(), ref_fc), "the clamp must land in the caller's (3,K) storage"
    # a CPU flow_cov (foreign frontend) is staged and written back
    cpu_fc = flow_cov.clone()
    out2 = model.estimate(frame, kp.to(DEV), NS(depth=depth.to(DEV)), None, cpu_fc)
    assert torch.equal(cpu_fc, ref_fc) and torch.equal(out2, out)


def test_match_covariance_depth_cov_branch(plugins):
    """flow_cov None + depth_cov given: `wvar_depth = depth_cov` (Project2to3.py:163-171)."""
    from oracle import covariance as ocov
    P = plugins
    H, W, K = 160, 224, 32
    kp, depth, _ = cases.cov_inputs(H, W, K, "none")
    dcov = torch.rand(K, generator=torch.Generator().manual_seed(3)) * 0.5 + 0.01
    frame = NS(fx=320.0, fy=320.0, cx=112.0, cy=80.0)
    model = P.B200_MatchCovariance(NS(device=DEV, kernel_size=31, match_cov_default=0.25, min_depth_cov=0.05, min_flow_cov=0.25))
    out = model.estimate(frame, kp.to(DEV), NS(depth=depth.to(DEV)), dcov.to(DEV), None)
    ref = ocov.match_covariance(kp, depth, None, 320.0, 320.0, 112.0, 80.0, depth_cov=dcov)
    rel = ((out - ref).abs() / ref.abs().amax(dim=(1, 2), keepdim=True)).amax().item()
    assert rel < 1e-5, rel
    ref_patch = ocov.match_covariance(kp, depth, None, 320.0, 320.0, 112.0, 80.0)
    assert not torch.allclose(ref, ref_patch), "the branch must actually change the result"


def test_fast_config_served_by_tf32_pipeline_beats_reference_fast_numerics(plugins, golden):
    """BASELINE configs[2] (MACVO_Fast: enc fp16 / dec bf16). The plugin serves half-precision requests with its TF32
    pipeline (`half_precision: tf32`, the default). Yardstick = the REFERENCE's own fp16/bf16 run on the same input
    (net_fast_small.pt): it sits `floor` away from float64 truth (flow 3.3e-3 of its scale, covariance 6e-2). Asserted: our
    output is CLOSER to the truth than the reference's fast path is, hence within ~2x floor of the reference-fast output."""
    P = plugins
    g = golden("net_fast_small.pt")
    B, H, W = g["shape"]
    img1, img2 = cases.net_inputs(B, H, W)
    fe = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp16", dec_dtype="bf16", decoder_depth=12,
                                         enforce_positive_disparity=False, cuda_graph=False))
    assert fe.half_precision == "tf32" and fe.net.enc_dtype == torch.float32
    try:
        flow, cov = fe.net.inference(img1.to(DEV), img2.to(DEV))          # the frontend switched TF32 on, like the reference's
        flow, cov = flow.double().cpu(), cov.double().cpu()
    finally:
        _strict_fp32()
    scale = g["truth_flow"].abs().mean().item()
    ours_flow = ((flow - g["truth_flow"]).abs().max() / scale).item()
    ours_cov = ((cov - g["truth_cov"]).abs() / g["truth_cov"].abs()).max().item()
    assert ours_flow <= g["floor"]["flow_rel"] and ours_cov <= g["floor"]["cov_rel_max"], (ours_flow, ours_cov, g["floor"])
    assert ((flow - g["flow"].double()).abs().max() / scale).item() <= 2 * g["floor"]["flow_rel"]
    # literal dtypes stay available
    fe2 = P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp16", dec_dtype="bf16", decoder_depth=2,
                                          enforce_positive_disparity=False, cuda_graph=False, half_precision="native"))
    assert fe2.net.enc_dtype == torch.float16 and fe2.net.dec_dtype == torch.bfloat16
    _strict_fp32()
