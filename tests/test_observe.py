"""macvo_observe_pack (csrc/observe.cu): observation building, covariance sanity filter, point registration and the
order-preserving compaction into the packed float64 buffer, followed by the counted LM solve (macvo_pgo_solve_counted).

CPU: the seeded inputs (tests/golden/observe_cases.py) regenerate bit for bit, the oracle (oracle/observe.py) equals the
reference fixtures (tests/golden/observe_*.pt, written by tests/golden/make_golden_observe.py from the reference
functions) and the plugin-API driver `TwoFrameOdometry`.
GPU: the kernels against the oracle on the same inputs. Tolerances:
  pixel1_uv, pixel2_uv, pixel1_d, pixel2_disp, pixel2_disp_cov, clamped pixel2_uv_cov: bit-exact (NaN == NaN)
  obs1_covTc / obs2_covTc: 1e-5 of each matrix's largest entry (closed-form 2x2 inverse vs the reference's pinverse,
                           fused sums)
  pos_Tw: rtol / atol 1e-6 against the fp32 oracle
  header, n_obs, kept rows and their order, status, next_pose = (double)(float)prev_pose: exact
  counted LM: pose rtol 1e-8 / atol 1e-9 against oracle.pgo.lm_solve on the kernel's own rows, same steps / evaluations
"""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import frontend as ofe
from oracle import observe as oobs
from oracle import pgo as opgo
from tests.golden import observe_cases as oc

DEV = "cuda"
CASES = list(oc.CASES)
NAN = float("nan")
ROWS = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
        "pixel1_uv", "pixel1_d")
EXACT = ("pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "pixel1_uv", "pixel1_d")


def _oracle(c: dict) -> dict:
    args, kw = oc.oracle_args(c)
    return oobs.observe_pack(*args, **kw)


def _bits(got: torch.Tensor, ref: torch.Tensor, what: str) -> None:
    torch.testing.assert_close(got, ref, rtol=0, atol=0, equal_nan=True, msg=lambda m: f"{what}: {m}")


# ---------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_fixture_inputs_reproduce(golden, name):
    assert oc.input_sha(oc.observe_inputs(name)) == golden(f"observe_{name}.pt")["input_sha"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_fixture(golden, name):
    """keep mask, gathers, counts and the clamped flow covariance bit-exact, covariances bit-identical (same torch CPU
    operations), pos_Tw within fp32 rounding of pypose's Act (other operation order); float64 Act as a second check"""
    g = golden(f"observe_{name}.pt")
    c = oc.observe_inputs(name)
    ref = _oracle(c)
    assert torch.equal(ref["keep"], g["keep"])
    assert (ref["n_obs"], ref["n_inbound"], ref["k"], ref["status"]) == (g["n_obs"], g["n_inbound"], g["k"], 0)
    assert not ref["unspecified"].any()
    for name_ in EXACT + ("obs1_covTc", "obs2_covTc"):
        assert ref[name_].dtype == g[name_].dtype, name_
        _bits(ref[name_], g[name_], name_)
    torch.testing.assert_close(ref["pos_Tw"], g["pos_Tw"], rtol=1e-6, atol=1e-6)
    pw64 = opgo.se3_act(c["prev_pose"].float().double().numpy(), ref["pos_Tc"].double().numpy())
    np.testing.assert_allclose(ref["pos_Tw"].double().numpy(), pw64, rtol=1e-6, atol=1e-5)
    assert torch.equal(ref["next_pose"], c["prev_pose"].float().double())


def test_cases_pin_what_they_claim():
    """the boundary rows fall on the side of the strict in-range test they were built for; the non-finite rows are dropped
    except where the reference keeps them (-Inf on the clamped diagonal; NaN disparity / Inf uncertainty pass through)"""
    c = oc.observe_inputs("boundary")
    ref = _oracle(c)
    for row, axis, target, inside in c["rows"]:
        assert bool(ref["keep"][row]) == inside, (row, axis, target)
    c = oc.observe_inputs("nonfinite")
    ref = _oracle(c)
    rows = c["rows"]
    keep = ref["keep"]
    # NaN, +-Inf and 2^100 (its square overflows fp32) anywhere in a window drop the row; 0 and -2 need not
    assert not any(keep[r] for r, (_, v, _) in zip(rows["depth"], oc.DEPTH_SPECIALS) if v not in (0.0, -2.0))
    kept_cov = [r for r, s in zip(rows["cov"], oc.COV_SPECIALS) if s[0] == -oc.INF]
    assert keep[kept_cov].all() and keep[rows["cov"]].sum() == len(kept_cov)
    for key, col in (("disp_nan", "pixel2_disp"), ("unc_inf", "pixel2_disp_cov")):
        r = rows[key][0]
        assert keep[r]
        j = int(keep[:r].sum())
        assert not torch.isfinite(ref[col][j])
    c = oc.observe_inputs("ksize31")          # the clamp of frame 0's constant covariance is active
    assert c["match_cov_default"] < c["min_flow_cov"] ** 2


def test_oracle_matches_plugin_api_driver():
    """TwoFrameOdometry with the CPU plugins (oracle/pipeline_cpu.py) on one frame pair: the optimiser input and the
    covariances equal the oracle's; ties the oracle to the path tests/test_macvo_integration.py runs under MACVO.py"""
    from macvo_b200.pipeline import TwoFrameOdometry
    from oracle.pipeline_cpu import CpuCovariance
    c = oc.observe_inputs("basic")
    ref = _oracle(c)
    zeros = torch.zeros_like(c["depth0"])

    class Frontend:
        retrieve_pixels = staticmethod(lambda uv, m, interpolate=False: ofe.retrieve_pixels(uv, m))

        def estimate_depth(self, frame):
            return NS(depth=c["depth0"], cov=zeros, disparity=zeros, disparity_uncertainty=zeros)

        def estimate_pair(self, f0, f1):
            return (NS(depth=c["depth1"], cov=zeros, disparity=c["disparity1"], disparity_uncertainty=c["disp_unc1"]),
                    NS(flow=c["flow"], cov=c["match_cov"].clone(), mask=None))

    class Selector:
        def select_point(self, *a):
            return c["kp0"].clone()

    class Capture:
        def start_optimize(self, inp):
            self.inp = inp

    def frame(intr):
        fx, fy, cx, cy = intr
        return NS(width=c["W"], height=c["H"], fx=fx, fy=fy, cx=cx, cy=cy, frame_baseline=0.25,
                  frame_K=torch.tensor([[fx, 0., cx], [0., fy, cy], [0., 0., 1.]]))
    opt = Capture()
    odo = TwoFrameOdometry(Frontend(), Selector(), CpuCovariance(c["kernel_size"], c["min_flow_cov"], c["min_depth_cov"],
                                                                 c["match_cov_default"]),
                           opt, num_point=c["kp0"].shape[0], edgewidth=c["edge_width"],
                           match_cov_default=c["match_cov_default"], mapping=False, min_num_point=1, keep_debug=True)
    odo.initialize(frame(c["intr0"]))
    odo.poses = [c["prev_pose"].float()]
    res = odo.run_pair(frame(c["intr1"]))
    assert (res.num_kp, res.num_obs) == (ref["n_inbound"], ref["n_obs"])
    keep = res.extras["keep"]
    _bits(res.kp0_uv[keep], ref["pixel1_uv"], "pixel1_uv")
    _bits(opt.inp.kp2_uv, ref["pixel2_uv"], "pixel2_uv")
    _bits(opt.inp.kp2_disp.reshape(-1), ref["pixel2_disp"], "pixel2_disp")
    _bits(opt.inp.uv_cov, ref["pixel2_uv_cov"], "pixel2_uv_cov")
    _bits(opt.inp.disp_cov.reshape(-1), ref["pixel2_disp_cov"], "pixel2_disp_cov")
    _bits(res.extras["pos0_cov"][keep], ref["obs1_covTc"], "obs1_covTc")
    _bits(res.extras["pos1_cov"][keep], ref["obs2_covTc"], "obs2_covTc")
    torch.testing.assert_close(opt.inp.pos_Tw, ref["pos_Tw"], rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from macvo_b200 import build, ops as _ops
    build.build(verbose=False)
    _ops.load_library()
    return _ops


def _observe(ops, c: dict, buf=None, poison: bool = True):
    """macvo_observe_pack on case `c`; -> (buffers, next_pose on the host)"""
    args, kw = oc.oracle_args(c)
    kp0, maps, (ew, i0, i1, prev) = args[0], args[1:7], args[7:]
    if buf is None:
        buf = ops.ObservationBuffers(max(kp0.shape[0], 1), DEV)
    if poison:
        buf.packed.fill_(NAN)
    next_pose = torch.full((7,), NAN, dtype=torch.float64, device=DEV)
    ops.observe_pack(buf, kp0.to(DEV), *(m.to(DEV) for m in maps), ew, i0, i1, prev.to(DEV), next_pose, **kw)
    torch.cuda.synchronize()
    return buf, next_pose.cpu()


def _rows(buf, n: int) -> dict:
    return {name: buf.section(name)[:n].cpu() for name in ROWS}


def _assert_matches(buf, next_pose, ref: dict, rows_only: bool = False) -> dict:
    n = ref["n_obs"]
    if not rows_only:
        assert buf.section("header").cpu().tolist() == [n, ref["n_inbound"], ref["k"], ref["status"]]
        assert int(buf.n_obs.item()) == n and int(buf.status.item()) == ref["status"]
        assert torch.equal(next_pose, ref["next_pose"])
    got = _rows(buf, n)
    _assert_rows(got, ref)
    return got


def _assert_rows(got: dict, ref: dict) -> None:
    """the kept rows `got` (device) against the oracle's, with the tolerances of the module docstring"""
    for name in EXACT:
        _bits(got[name], ref[name].double(), name)
    for name in ("obs1_covTc", "obs2_covTc"):
        # kept rows passed the sanity filter: a non-finite entry is a row the kernel did not write (NaN poison) or got wrong
        assert torch.isfinite(got[name]).all(), f"{name}: non-finite entries in kept rows"
        r = ref[name]
        if r.shape[0]:
            err = ((got[name] - r).abs() / r.abs().amax(dim=(-1, -2), keepdim=True)).max().item()
            assert err <= 1e-5, f"{name}: {err:.3e}"
    torch.testing.assert_close(got["pos_Tw"], ref["pos_Tw"].double(), rtol=1e-6, atol=1e-6)


def _assert_untouched_past(buf, n: int, before: torch.Tensor | None = None) -> None:
    """every section past row n still holds what was there before the call (NaN poison by default)"""
    for name in ROWS:
        tail = buf.section(name)[n:].cpu()
        prev = torch.full_like(tail, NAN) if before is None else before[name][n:]
        _bits(tail, prev, f"{name}[{n}:]")


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_observe_pack_matches_oracle(ops, name):
    """a. every case: basic (k 700, intr0 != intr1, rotated prev_pose), chunks (k 2500), boundary, nonfinite, ksize"""
    c = oc.observe_inputs(name)
    ref = _oracle(c)
    buf, nxt = _observe(ops, c)
    _assert_matches(buf, nxt, ref)
    _assert_untouched_past(buf, ref["n_obs"])


COMPACTION_K = [1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 3000, 4096]


def _drop_patterns(k: int) -> dict:
    return {"none": [], "all": list(range(k)), "chunk0": list(range(min(k, 1024))),
            "last_warp_chunk0": list(range(992, min(k, 1024))), "every_other": list(range(0, k, 2)), "last": [k - 1]}


@pytest.mark.gpu
@pytest.mark.parametrize("k", COMPACTION_K)
def test_compaction_keeps_order_across_warps_and_chunks(ops, k):
    """b. rows dropped by a NaN match covariance: the survivors keep their order across warp and 1024-record chunk
    boundaries, at capacity k and above it; nothing is written past n_obs"""
    base = oc.compaction_inputs(k)
    for pattern, rows in _drop_patterns(k).items():
        c = oc.drop_rows(base, rows)
        ref = _oracle(c)
        assert ref["n_obs"] == k - len(rows) and ref["n_inbound"] == k, pattern
        for cap in (k, k + 96):
            buf, nxt = _observe(ops, c, ops.ObservationBuffers(cap, DEV))
            got = _assert_matches(buf, nxt, ref)
            _bits(got["pixel1_uv"], ref["pixel1_uv"].double(), f"{pattern} cap {cap}")
            _assert_untouched_past(buf, ref["n_obs"])


@pytest.mark.gpu
def test_zero_keypoints(ops):
    """c. k = 0: header [0, 0, 0, 0], n_obs 0, the motion-model prediction still written"""
    c = oc.compaction_inputs(1)
    c["kp0"] = c["kp0"][:0]
    buf, nxt = _observe(ops, c, ops.ObservationBuffers(64, DEV))
    assert buf.section("header").cpu().tolist() == [0, 0, 0, 0] and int(buf.n_obs.item()) == 0
    assert torch.equal(nxt, c["prev_pose"].float().double())
    _assert_untouched_past(buf, 0)


def _status_case(rows: list[tuple[int, int]]) -> dict:
    """64 x 96 frame, edge_width 2, kernel_size 7, flow (0.5, 0.5) everywhere"""
    c = oc.compaction_inputs(1)
    H, W = 64, 96
    g = torch.Generator().manual_seed(60)
    c.update(H=H, W=W, **oc.dense_maps(H, W, g), **oc._scalars(7, edge_width=2))
    c["flow"] = torch.full((1, 2, H, W), 0.5)
    c["kp0"] = torch.tensor(rows, dtype=torch.int64)
    return c


TOP_LEFT = [(2, 2), (3, 5), (5, 3), (2, 10), (10, 2), (20, 20), (40, 30)]    # windows of the first five wrap
BOTTOM_RIGHT = [(93, 30)]                                                    # u0 + 3 = W: the 7 x 7 window leaves the image
OUTSIDE = [(-1, 5), (96, 10)]                                                # kp0 outside the image


@pytest.mark.gpu
def test_status_bits(ops):
    """d. status is a bitmask: top-left windows wrap like python indices (0, rows equal the oracle), a window crossing the
    bottom-right edge sets 1, a keypoint outside the image 2, both 3"""
    for rows, status in ((TOP_LEFT, 0), (TOP_LEFT + OUTSIDE, 2), (BOTTOM_RIGHT + TOP_LEFT, 1),
                         (OUTSIDE[:1] + BOTTOM_RIGHT + TOP_LEFT + OUTSIDE[1:], 3)):
        c = _status_case(rows)
        ref = _oracle(c)
        assert ref["status"] == status
        buf, nxt = _observe(ops, c)
        hdr = buf.section("header").cpu().tolist()
        assert hdr[1:] == [ref["n_inbound"], ref["k"], status] and int(buf.status.item()) == status
        assert torch.equal(nxt, ref["next_pose"])
        if status & 1 == 0:
            _assert_matches(buf, nxt, ref)
            continue
        # the rows whose window left the image have unspecified covariances; the others keep their values and order
        n = int(hdr[0])
        got = _rows(buf, n)
        spec = torch.tensor([tuple(p) not in BOTTOM_RIGHT for p in got["pixel1_uv"].long().tolist()])
        assert int(spec.sum()) == ref["n_obs"]
        _assert_rows({k: v[spec] for k, v in got.items()}, ref)


@pytest.mark.gpu
def test_buffer_reuse_leaves_rows_past_n_obs_untouched(ops):
    """e. a NaN-poisoned buffer, k = 1500 then k = 300 on the same buffer: each header reflects its own call only and no
    section is written past that call's n_obs"""
    buf = ops.ObservationBuffers(2048, DEV)
    c1 = oc.drop_rows(oc.compaction_inputs(1500), range(0, 1500, 3))
    ref1 = _oracle(c1)
    _, nxt = _observe(ops, c1, buf)
    _assert_matches(buf, nxt, ref1)
    _assert_untouched_past(buf, ref1["n_obs"])
    before = _rows(buf, buf.capacity)
    c2 = oc.drop_rows(oc.compaction_inputs(300, seed=51), [0, 5, 299])
    ref2 = _oracle(c2)
    _, nxt = _observe(ops, c2, buf, poison=False)
    _assert_matches(buf, nxt, ref2)
    _assert_untouched_past(buf, ref2["n_obs"], before)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [2048, 4096])
def test_observe_then_counted_solve(ops, cap):
    """f. the bench shapes: about 35 % of the rows dropped, buffer poisoned with NaN; the counted LM with the automatic
    cluster size (8 at these capacities) and 1, 2, 4 CTAs equals the oracle LM on the kernel's own first n_obs rows"""
    c = oc.solve_inputs(cap, seed=70 + cap)
    ref = _oracle(c)
    assert 0.55 * cap < ref["n_obs"] < 0.75 * cap
    buf, init = _observe(ops, c, ops.ObservationBuffers(cap, DEV))
    _assert_matches(buf, init, ref)
    n = int(buf.n_obs.item())
    got = _rows(buf, n)
    fx, fy, cx, cy = c["intr1"]
    bl = float(torch.tensor(c["baseline"], dtype=torch.float32))
    graph = opgo.GraphData(pos_Tw=got["pos_Tw"].numpy(), kp2_uv=got["pixel2_uv"].numpy(),
                           kp2_disp=got["pixel2_disp"].numpy(), uv_cov=got["pixel2_uv_cov"].numpy(),
                           disp_cov=got["pixel2_disp_cov"].numpy(), fx=fx, fy=fy, cx=cx, cy=cy, baseline=bl,
                           init_pose=init.numpy())
    trace = opgo.LMTrace()
    pose_ref = opgo.lm_solve(graph, trace=trace)
    truth = c["truth"].numpy()
    assert np.linalg.norm(pose_ref[:3] - truth[:3]) < 0.5 * np.linalg.norm(init.numpy()[:3] - truth[:3])
    for cluster in (0, 1, 2, 4):
        pose = init.to(DEV)
        stats = torch.zeros(8, dtype=torch.float64, device=DEV)
        ops.pgo_solve_counted(buf, (fx, fy, cx, cy, bl), pose, stats, min_k=10, cluster=cluster)
        p, s = pose.cpu().numpy(), stats.cpu().numpy()
        assert np.isfinite(p).all(), f"cluster {cluster}: a row past n_obs was read"
        np.testing.assert_allclose(p, pose_ref, rtol=1e-8, atol=1e-9, err_msg=f"cluster {cluster}")
        assert (int(s[0]), int(s[1]), s[6]) == (trace.steps, trace.evaluations, 0.0), f"cluster {cluster}"
    pose = init.to(DEV)
    stats = torch.zeros(8, dtype=torch.float64, device=DEV)
    ops.pgo_solve_counted(buf, (fx, fy, cx, cy, bl), pose, stats, min_k=n + 1)
    assert torch.equal(pose.cpu(), init) and stats[6].item() == 1.0
