"""The Vanilla ablation's covariance-free frontend and back end on the device (B200_FlowFormerFrontend, macvo_dense_postproc /
macvo_observe_pack with NULL covariance maps, the fused driver). Tolerances:
  flow-only network vs the reference (frontend_plain_*.pt), strict fp32: 2e-5 of the flow scale (the Cov network's bound)
  flow-only flow vs FlowFormerCovNet's flow on the same weights, both loops: bit-identical (same launches on the flow track)
  depth / disparity vs the oracle arithmetic on the kernel's own flow, graph vs eager: bit-exact
  observe_pack without covariance maps: keep mask, counts, gathers and -1 columns bit-exact; MatchCovariance 1e-5 of each
  matrix's largest entry (tests/test_observe.py), identity bit-exact; icp points_Tc bit-exact, cov_Tw 1e-12
  fused driver vs TwoFrameOdometry: equal counts, poses 1e-6 absolute / 1e-5 relative; pipelined == sequential"""
from contextlib import contextmanager
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests.golden import filter_cases as fc
from tests.golden.plain_cases import PLAIN_CASES, observe_pack_no_cov, plain_frontend_inputs

DEV = "cuda"
NAN = float("nan")
ROWS = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
        "pixel1_uv", "pixel1_d")
EXT = ("pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc", "cov_Tw")
EXACT = ("pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "pixel1_uv", "pixel1_d", "pixel2_d",
         "pixel1_d_cov", "pixel2_d_cov", "points_Tc")


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from macvo_b200 import build, ops as _ops
    build.build(verbose=False)
    _ops.load_library()
    return _ops


@contextmanager
def flags(tf32: bool):
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    torch.set_float32_matmul_precision("medium" if tf32 else "highest")
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev[:2]
        torch.set_float32_matmul_precision(prev[2])


def _nets(depth=12):
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    return (FlowFormerCovNet(synthetic_state_dict(0, covariance=False), DEV, decoder_depth=depth, covariance=False),
            FlowFormerCovNet(synthetic_state_dict(0), DEV, decoder_depth=depth))


def _bits(got, ref, what):
    assert torch.equal(got.view(torch.int64 if got.dtype == torch.float64 else torch.int32),
                       ref.view(torch.int64 if ref.dtype == torch.float64 else torch.int32)), what


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PLAIN_CASES))
def test_plain_network_matches_reference_strict(ops, golden, name):
    g = golden(f"frontend_plain_{name}.pt")
    t1l, l2, r2 = (t.to(DEV) for t in plain_frontend_inputs(*g["shape"]))
    plain, _ = _nets()
    with flags(False):
        stereo, none = plain.inference(l2, r2)
        match, _ = plain.inference(t1l, l2)
    assert none is None
    want = g["pair"]["flow"]
    assert (match.cpu() - want).abs().max().item() <= 2e-5 * want.abs().mean().item()
    d = g["pair"]["disparity"]
    assert (stereo[:, :1].abs().cpu() - d).abs().max().item() <= 2e-5 * d.abs().mean().item()


def _frames_640(n=3):
    from macvo_b200 import synthetic
    return synthetic.make_sequence(n, 480, 640)


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["strict", "tf32"])
def test_plain_flow_equals_cov_flow_640x480(ops, tf32):
    """B = 2 shared at 640x480: the flow-only network's flow IS FlowFormerCovNet's flow, in both refinement loops"""
    fr = _frames_640(2)
    A = torch.cat([fr[1].imageL, fr[0].imageL]).to(DEV)
    B = torch.cat([fr[1].imageR, fr[1].imageL]).to(DEV)
    plain, cov = _nets()
    with flags(tf32):
        assert plain._decoder_mode(torch.zeros(1, device=DEV)) == ("tf32" if tf32 else "strict")
        fp, none = plain.inference(A, B, shared=(0, 1))
        fc_, c = cov.inference(A, B, shared=(0, 1))
        torch.cuda.synchronize()
    assert none is None and c is not None
    _bits(fp, fc_, f"flow ({'tf32' if tf32 else 'strict'})")


def _cov_frontend(P, depth=12, cuda_graph=True):
    return P.B200_FlowFormerCovFrontend(NS(weight="synthetic:0", device=DEV, enc_dtype="fp32", dec_dtype="fp32",
                                           decoder_depth=depth, enforce_positive_disparity=False, cuda_graph=cuda_graph))


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True], ids=["strict", "tf32"])
def test_skipped_work_is_skipped(ops, tf32):
    """per replay the plain frontend launches the Cov frontend's kernels minus the covariance branch: per iteration the
    covariance GRU unit (tf32: its 4-stage tensor-core chain; strict: gates + blend per pass) and the 4 covariance-head
    convolutions (own kernels in tf32 mode only), once the covariance upsampling, and in tf32 mode its state packing"""
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    frames = synthetic.make_sequence(3, 192, 256)
    depth = P.B200_FlowFormerFrontend.DECODER_DEPTH
    with flags(tf32):
        cov = _cov_frontend(P, depth)
        plain = P.B200_FlowFormerFrontend(NS(weight="synthetic:0", device=DEV))
    with flags(tf32):                  # (the Cov frontend's constructor turns TF32 on)
        for fe in (cov, plain):
            fe.estimate_pair(frames[0], frames[1])
            fe.estimate_pair(frames[1], frames[2])
    per_iter = ops.SepConvGruTC.LAUNCHES_PER_UNIT + 4 if tf32 else 2 * 2
    once = 1 + (1 if tf32 else 0)
    assert plain._static["launches"] == cov._static["launches"] - (depth * per_iter + once), \
        (plain._static["launches"], cov._static["launches"])


@pytest.mark.gpu
def test_plain_frontend_outputs(ops):
    """estimate_pair / estimate_depth: shapes, None fields, depth / disparity bit-exact against the oracle's arithmetic on the
    kernel's own flow, CUDA graph == eager, and the same flow / depth / disparity as B200_FlowFormerCovFrontend's"""
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    frames = synthetic.make_sequence(3, 192, 256)
    with flags(True):                 # what the Cov frontend's constructor sets; the plain frontend then runs under them
        _check_plain_frontend_outputs(P, frames)


def _check_plain_frontend_outputs(P, frames):
    cov = _cov_frontend(P)
    g_plain = P.B200_FlowFormerFrontend(NS(weight="synthetic:0", device=DEV))
    e_plain = P.B200_FlowFormerFrontend(NS(weight="synthetic:0", device=DEV, cuda_graph=False))
    assert g_plain.provide_cov == (False, False)
    for f0, f1 in ((frames[0], frames[1]), (frames[1], frames[2])):
        dg, mg = g_plain.estimate_pair(f0, f1)
        de, me = e_plain.estimate_pair(f0, f1)
        dc, mc = cov.estimate_pair(f0, f1)
        torch.cuda.synchronize()
        for d, m in ((dg, mg), (de, me)):
            assert d.cov is None and d.mask is None and d.disparity_uncertainty is None and m.cov is None and m.mask is None
            assert d.depth.shape == d.disparity.shape == (1, 1, 192, 256) and m.flow.shape == (1, 2, 192, 256)
        for k in ("depth", "disparity"):
            _bits(getattr(dg, k), getattr(de, k), f"graph vs eager {k}")
            _bits(getattr(dg, k), getattr(dc, k), f"plain vs Cov frontend {k}")
        _bits(mg.flow, me.flow, "graph vs eager flow")
        _bits(mg.flow, mc.flow, "plain vs Cov frontend flow")
        # the oracle's arithmetic on the kernel's own stereo flow (FlowFormerDepth.estimate, StereoDepth.py:122-128)
        A = torch.cat([f1.imageL, f0.imageL]).to(DEV)
        B = torch.cat([f1.imageR, f1.imageL]).to(DEV)
        flow, _ = e_plain.net.inference(A, B, shared=(0, 1))
        disp = flow[0:1, :1].abs().cpu()
        _bits(de.disparity.cpu(), disp, "disparity")
        _bits(de.depth.cpu(), (f1.frame_baseline * f1.fx) * disp.reciprocal(), "depth")
    d = e_plain.estimate_depth(frames[2])
    dc = cov.estimate_depth(frames[2])
    assert d.cov is None and d.mask is None and d.disparity_uncertainty is None
    flow, _ = e_plain.net.inference(frames[2].imageL.to(DEV), frames[2].imageR.to(DEV))
    disp = flow[:, :1].abs().cpu()
    _bits(d.disparity.cpu(), disp, "estimate_depth disparity")
    _bits(d.depth.cpu(), (frames[2].frame_baseline * frames[2].fx) * disp.reciprocal(), "estimate_depth depth")
    _bits(d.depth, dc.depth, "estimate_depth plain vs Cov")


@pytest.mark.gpu
def test_dense_postproc_argument_rules(ops):
    from macvo_b200.ops import MacvoB200Error
    f = torch.randn(2, 2, 8, 8, device=DEV)
    ops.dense_postproc(f, None, 80.0)
    with pytest.raises(MacvoB200Error):
        ops.dense_postproc(f, None, 80.0, enforce_positive_disparity=True)
    lib = ops.load_library()
    d = torch.empty(64, device=DEV)
    assert lib.macvo_dense_postproc(f.data_ptr(), None, 8, 8, 80.0, 6400.0, d.data_ptr(), None, d.data_ptr(), None, None,
                                    None, None) != 0           # depth_cov without est_cov
    assert lib.macvo_dense_postproc(f.data_ptr(), None, 8, 8, 80.0, 6400.0, None, None, None, None, None, None, None) != 0


CASES = {"identity": dict(cov_model="identity"), "match": dict(cov_model="match"),
         "match_unclamped": dict(cov_model="match", match_cov_default=0.05)}


@pytest.mark.gpu
@pytest.mark.parametrize("icp", [False, True], ids=["plain", "icp"])
@pytest.mark.parametrize("case", list(CASES))
def test_observe_pack_without_covariance_maps(ops, case, icp):
    c = fc.icp_solve_inputs(512, seed=682)
    kw = dict(kernel_size=c["kernel_size"], min_flow_cov=c["min_flow_cov"], min_depth_cov=c["min_depth_cov"],
              match_cov_default=c["match_cov_default"])
    kw.update({k: v for k, v in CASES[case].items() if k != "cov_model"})
    if case == "match_unclamped":
        assert kw["match_cov_default"] < kw["min_flow_cov"] ** 2
    model = CASES[case]["cov_model"]
    lo, hi = c["min_depth"], 9.0                 # the depth filter keeps about half of the rows
    ref = observe_pack_no_cov(c["kp0"], c["flow"], c["depth0"], c["depth1"], c["disparity1"], c["edge_width"], c["intr0"],
                              c["intr1"], c["prev_pose"], cov_model=model, depth_range=(lo, hi), icp=icp, **kw)
    buf = ops.ObservationBuffers(512, DEV, extended=icp)
    buf.packed.fill_(NAN)
    nxt = torch.full((7,), NAN, dtype=torch.float64, device=DEV)
    ext = {"simple_depth": True, "min_depth": lo, "max_depth": hi, "icp": icp, "cov_model": model,
           "cov_ops": []}
    ops.observe_pack(buf, c["kp0"].to(DEV), c["flow"].to(DEV), None, c["depth0"].to(DEV), c["depth1"].to(DEV),
                     c["disparity1"].to(DEV), None, c["edge_width"], c["intr0"], c["intr1"], c["prev_pose"].to(DEV), nxt,
                     ext=ext, **kw)
    torch.cuda.synchronize()
    n = ref["n_obs"]
    assert 10 < n < ref["n_inbound"]
    hdr = buf.section("header").cpu().tolist()
    assert hdr == [n, ref["n_inbound"], ref["k"], ref["status"]], hdr
    assert torch.equal(nxt.cpu(), ref["next_pose"])
    names = ROWS + (EXT if icp else ())
    got = {k: buf.section(k)[:n].cpu() for k in names}
    for k in EXACT:
        if k in got:
            _bits(got[k], ref[k].double(), f"{case} {k}")
    for k in ("pixel2_uv_cov", "pixel2_disp_cov") + (("pixel1_d_cov", "pixel2_d_cov") if icp else ()):
        assert bool((got[k] == -1).all()), k
    for k in ("obs1_covTc", "obs2_covTc"):
        if model == "identity":
            _bits(got[k], torch.eye(3, dtype=torch.float64).expand(n, 3, 3).contiguous(), k)
        else:
            scale = ref[k].abs().amax(dim=(-1, -2), keepdim=True)
            assert ((got[k] - ref[k]).abs() / scale).max().item() <= 1e-5, (case, k)
    torch.testing.assert_close(got["pos_Tw"], ref["pos_Tw"].double(), rtol=1e-6, atol=1e-6)
    if icp:
        from oracle import ablation as oab
        R = oab.ofil.quat_matrix_f32(ref["next_pose"][3:7]).double().expand(n, 3, 3)
        want = torch.bmm(torch.bmm(R, got["obs1_covTc"]), R.transpose(1, 2))
        assert ((got["cov_Tw"] - want).abs() / want.abs().amax(dim=(-1, -2), keepdim=True)).max().item() <= 1e-12
    for k in names:
        tail = buf.section(k)[n:].cpu()
        _bits(tail, torch.full_like(tail, NAN), f"{k}[{n}:]")
    with pytest.raises(ops.MacvoB200Error):        # only one of the two maps missing
        ops.observe_pack(buf, c["kp0"].to(DEV), c["flow"].to(DEV), None, c["depth0"].to(DEV), c["depth1"].to(DEV),
                         c["disparity1"].to(DEV), c["disparity1"].to(DEV), c["edge_width"], c["intr0"], c["intr1"],
                         c["prev_pose"].to(DEV), nxt, ext=ext, **kw)


class _PlainMapFrontend:
    """seeded dense maps per frame without covariance (what B200_FlowFormerFrontend hands the back end), uploaded once"""

    def __init__(self, frames):
        from macvo_b200 import plugins as P
        self.retrieve_pixels = staticmethod(P.B200_FlowFormerFrontend.retrieve_pixels)
        self.maps = []
        for i, f in enumerate(frames):
            m = fc.dense_frame_maps(f.height, f.width, seed=300 + i)
            self.maps.append((f, NS(depth=m["depth1"].to(DEV), cov=None, disparity=m["disparity1"].to(DEV),
                                    disparity_uncertainty=None, mask=None), NS(flow=m["flow"].to(DEV), cov=None, mask=None)))

    def _get(self, frame):
        return next(x for x in self.maps if x[0] is frame)

    def estimate_depth(self, frame):
        return self._get(frame)[1]

    def estimate_pair(self, f0, f1):
        return self._get(f1)[1:]


def _vanilla(P, cls, frontend, motion, lo, hi):
    """Vanilla's back end: NoCovariance, RandomSelector, FilterCompose[SimpleDepthFilter], icp, mapping off"""
    return cls(frontend, P.B200_RandomSelector(NS(mask_width=32, device=DEV)), P.B200_NoCovariance(None),
               P.B200_TwoFrame_PGO(NS(graph_type="icp", device=DEV, vectorize=True, parallel=False, autodiff=False)),
               num_point=200, mapping=False,
               motion_model=P.B200_TartanMotionNet(NS(weight="synthetic", device=DEV)) if motion else None,
               outlier_filter=P.B200_FilterCompose(NS(filter_args=[
                   NS(type="B200_SimpleDepthFilter", args=NS(min_depth=lo, max_depth=hi))])),
               keep_debug=True)


@pytest.mark.gpu
@pytest.mark.parametrize("motion", [False, True], ids=["static", "motionnet"])
def test_vanilla_fused_equals_plugin_api_path(ops, motion):
    from macvo_b200 import plugins as P
    from macvo_b200 import synthetic
    from macvo_b200.pipeline import FusedTwoFrameOdometry, TwoFrameOdometry
    frames = synthetic.make_sequence(6, 192, 256)
    lo, hi = fc.MIN_DEPTH, 16.0                  # rows kept and dropped on every frame
    a = _vanilla(P, TwoFrameOdometry, _PlainMapFrontend(frames), motion, lo, hi)
    torch.manual_seed(5)
    a.initialize(frames[0])
    ra = [a.run_pair(f) for f in frames[1:]]
    pa = a.finish()
    runs = []
    for pipelined in (False, True):
        b = _vanilla(P, FusedTwoFrameOdometry, _PlainMapFrontend(frames), motion, lo, hi)
        torch.manual_seed(5)
        b.initialize(frames[0])
        obs = []
        for i in range(1, len(frames)):
            nxt = frames[i + 1] if pipelined and i + 1 < len(frames) and i != 3 else None
            b.run_pair(frames[i], next_frame=nxt)
            obs.append(b.observations())
        runs.append((obs, b.finish(), b.host_waits))
    (oa, pb, wa), (ob, pc, wb) = runs
    assert torch.equal(pb, pc)
    assert wa == wb == [0] * (len(frames) - 1)
    for x, y in zip(oa, ob):
        assert x["num_obs"] == y["num_obs"]
        for k in ROWS + EXT:
            assert torch.equal(x[k], y[k]), k
    for o, r in zip(oa, ra):
        assert o["num_kp"] == r.num_kp and o["num_obs"] == r.num_obs
        assert 10 <= r.num_obs < r.num_kp
        for k in ("pixel2_uv_cov", "pixel2_disp_cov", "pixel1_d_cov", "pixel2_d_cov"):
            assert bool((o[k] == -1).all()), k
        eye = torch.eye(3, dtype=torch.float64)
        assert torch.equal(o["obs1_covTc"], eye.expand_as(o["obs1_covTc"]))
        assert torch.equal(o["obs2_covTc"], eye.expand_as(o["obs2_covTc"]))
    np.testing.assert_allclose(pb.numpy(), pa.numpy(), rtol=1e-5, atol=1e-6)
