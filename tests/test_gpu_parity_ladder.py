"""Frontend parity at the benched shape (640x480) and at the shipped dataset frame sizes (EuRoC 752x480, KITTI 1241x376
and 1226x370): decoder_depth 12, the `estimate_pair` batch of the bench sequence at that size, in BOTH precision modes,
stage by stage, against the float64 ground truth of tests/golden/net_<case>.pt (generated next to the reference's own
fp32 run by tests/golden/make_golden_cfgA.py / make_golden_datasets.py).

Every size is held to the 640x480 bounds and strict floor rule below. The dataset sizes exist because the network picks
its paths from the 1/8-resolution grid H1 x W1 (N = H1 W1), and each takes branches 640x480 never does (asserted in
`test_frontend_parity_ladder` by wrapping the dispatch points):

  case     padded frame  H1 x W1  N     correlation (tf32 / strict)    GMA softmax (tf32)   vertical global attention
  cfgA     640x480       60x80    4800  corr_tc_kernel<2> / <3>        softmax_rows_f16     native
  euroc    752x480       60x94    5640  corr_tc_kernel<2> / <3>        softmax_rows_f16     padded (94 % 4 != 0)
  kitti    1248x376      47x156   7332  corr_simt_kernel (N % 8 = 4)   softmax_rows_f16     padded
  kitti00  1232x376      47x154   7238  corr_simt_kernel               torch + fp16 cast    padded
                                                                       (N % 4 = 2)

Yardstick: the REFERENCE's fp32 CPU result is itself 2.6e-6 (flow, relative to the mean |flow|) and 1.3e-4 (covariance,
relative) away from exact arithmetic on the 640x480 input (`floor`). north_star's "within 1e-4 relative" is therefore met
for the flow by any faithful fp32 implementation and is AT the fp32 noise floor for the covariance.

  strict   allow_tf32 = False: every layer fp32 (our kernels fp32 FMA, cuDNN / cuBLAS fp32, correlation volume 3 x fp16
           split). Asserted: final flow and covariance within 2x the reference's own distance from the truth, within
           1e-5 / 2e-4 of the reference's fp32 output, every stage within a few 1e-5.
  tf32     what bench.py times = the reference GPU frontend's own setting (Frontend.py:275-277: TF32 matmuls and
           convolutions): cuDNN / cuBLAS TF32, our attention / PatchEmbed kernels with TF32 operands, tf32
           correlation volume, fp16 GMA attention matrix. TF32 keeps 10 mantissa bits (2^-11 = 4.9e-4 per operand):
           the encoders already differ by 3.5e-3 of their scale, the refinement contracts that to 6e-4 on the flow.
           Bounds = 1.5 x the measured ladder (tools/parity_ladder.py), so that one dropped mantissa bit
           (2 x the error) fails the test.

sharp, sharp_kitti00: the sharpened checkpoint (tests/golden/cases.py::sharp_state_dict) on the cfgA and kitti00 frames
and branches. With the synthetic checkpoint every softmax is close to uniform, so an error in the plumbing around the
attention kernels (a scale, which keys go with which values, a position term) shrinks by one to two orders of magnitude
before it reaches the flow; with the sharpened one every family's median logit std is 2 - 4 (recorded in the fixture).
Sharper softmaxes also amplify rounding, so these cases are held to their own yardsticks where those are looser:
  strict   every stage within max(BOUNDS strict, 3 x the fixture's fp32 noise floor of that stage: the same class in fp32
           on the CPU against the float64 truth), plus the 2.5 x floor rule on the final flow and covariance;
  tf32     every stage within max(BOUNDS tf32, 1.5 x the library-op path's error at that stage, measured in the same
           test: the same class with none of our kernels, torch / cuDNN / cuBLAS ops under the same TF32 flags, as the
           reference runs on a GPU); 2 x for the full-resolution outputs. The convex upsampling's 64x sharper mask
           amplifies the rounding of the last state, so the two faithful TF32 runs differ more there than anywhere on the
           1/8 grid: on an H100 80GB HBM3 (700 W) our flow error was 0.84x (sharp) and 1.59x (sharp_kitti00) the library
           path's while every 1/8-grid iterate stayed within 1.12x; a GMA temperature error still exceeds the bound 20x.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

pytestmark = pytest.mark.gpu

BOUNDS = {
    # stage: (strict, tf32)   error = max |x - truth| / mean |truth| over the fixture's strided sample
    "context": (2e-5, 6e-3), "feats": (2e-5, 6e-3), "corr_rows": (1e-5, 3e-3), "cost_memory": (1e-5, 2.5e-3),
    "flow_iter": (6e-5, 3.2e-3), "cov_iter": (1e-4, 1.6e-3),
    "flow": (6e-6, 1.35e-3),           # strict: 2.3 x the reference's own 2.6e-6; tf32: 1.5 x the measured 9.0e-4
    "cov_rel_max": (3e-4, 1.8e-2),     # strict: 2.3 x the reference's own 1.3e-4; tf32: 1.5 x the measured 1.2e-2
    "flow_vs_ref32": (1e-5, 1.35e-3), "cov_rel_vs_ref32": (2e-4, 1.8e-2),
}
# Every size is held to these bounds. At the KITTI sizes the REFERENCE's own fp32 output is already close to the strict
# flow and covariance bounds (net_<case>.pt, on the fixture's sample: kitti 4.9e-6 / 2.6e-4, kitti00 4.7e-6 / 2.7e-4,
# against 2.6e-6 / 1.3e-4 at 640x480), so a strict failure there is first to be compared with that distance and with
# flow_vs_ref32 / cov_rel_vs_ref32 (the distance to the reference's fp32 output).


LADDER_CASES = ("cfgA", "euroc", "kitti", "kitti00", "sharp", "sharp_kitti00")
SHARP_CASES = ("sharp", "sharp_kitti00")
FULL_RESOLUTION = ("flow", "cov_rel_max", "flow_vs_ref32", "cov_rel_vs_ref32")      # after the convex upsampling
# which branch each dispatch point takes, per case (the table above): correlation mode in TF32 mode (strict: the fp32-class
# 3 x fp16 split wherever TF32 takes the tensor cores), whether the fp16 GMA softmax kernel runs, native vertical attention
BRANCHES = {"cfgA": ("tf32", True, True), "euroc": ("tf32", True, False), "kitti": ("simt", True, False),
            "kitti00": ("simt", False, False), "sharp": ("tf32", True, True), "sharp_kitti00": ("simt", False, False)}


@pytest.fixture(scope="module")
def ladder_fn():
    assert torch.cuda.is_available()
    from macvo_b200 import build
    build.build(verbose=False)
    import parity_ladder
    return parity_ladder


def _record_branches(monkeypatch) -> dict:
    """wrap the shape-dependent dispatch points of the network and record which branch each call took"""
    from macvo_b200 import ops
    from macvo_b200.flowformer_cov import FlowFormerCovNet
    rec = {"corr": [], "softmax_f16": 0, "vglobal": 0, "vglobal_native": 0}
    corr_mode, softmax_f16 = ops.default_corr_mode, ops.softmax_rows_f16
    vglobal, vglobal_native = FlowFormerCovNet._vert_global_attn, FlowFormerCovNet._vert_global_attn_native
    names = {ops.CORR_SIMT: "simt", ops.CORR_TC_3XF16: "tc3", ops.CORR_TC_1XF16: "tc1", ops.CORR_TC_TF32: "tf32"}

    def corr_mode_rec(*a, **k):
        m = corr_mode(*a, **k)
        rec["corr"].append(names[m])
        return m

    def softmax_rec(*a, **k):
        rec["softmax_f16"] += 1
        return softmax_f16(*a, **k)

    def vglobal_rec(self, *a, **k):
        rec["vglobal"] += 1
        return vglobal(self, *a, **k)

    def vglobal_native_rec(self, *a, **k):
        rec["vglobal_native"] += 1
        return vglobal_native(self, *a, **k)

    monkeypatch.setattr(ops, "default_corr_mode", corr_mode_rec)
    monkeypatch.setattr(ops, "softmax_rows_f16", softmax_rec)
    monkeypatch.setattr(FlowFormerCovNet, "_vert_global_attn", vglobal_rec)
    monkeypatch.setattr(FlowFormerCovNet, "_vert_global_attn_native", vglobal_native_rec)
    return rec


@pytest.mark.parametrize("case", LADDER_CASES)
@pytest.mark.parametrize("mode", ["strict", "tf32"])
def test_frontend_parity_ladder(ladder_fn, golden, monkeypatch, mode, case):
    g = golden(f"net_{case}.pt")
    rec = _record_branches(monkeypatch)
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    lib = None
    try:
        if case in SHARP_CASES and mode == "tf32":
            lib = ladder_fn.ladder(mode, g, case, library_ops=True)
            rec.update(corr=[], softmax_f16=0, vglobal=0, vglobal_native=0)
        res = ladder_fn.ladder(mode, g, case)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev[0], prev[1]
        torch.set_float32_matmul_precision(prev[2])
    col = 0 if mode == "strict" else 1
    # per stage (per iteration for the iterates): the fixed bound, or for the sharp cases the larger of it and the case's
    # own yardstick (module docstring)
    yard, mult = (g.get("floor_stages"), 3.0) if mode == "strict" else (lib, 1.5)
    as_list = lambda v: v if isinstance(v, list) else [v]
    bound = {}
    for name, b in BOUNDS.items():
        n = len(as_list(res[name]))
        m = 2.0 if mode == "tf32" and name in FULL_RESOLUTION else mult
        bound[name] = [max(b[col], m * y) for y in as_list(yard[name])] if case in SHARP_CASES else [b[col]] * n
        assert len(bound[name]) == n, (name, n)
    report = [f"{name} {max(as_list(res[name])):.3e} (bound {max(bound[name]):.2e})" for name in BOUNDS]
    print(f"[{case} {mode}] " + "; ".join(report))
    if lib is not None:
        print(f"[{case} {mode} library ops] " + "; ".join(f"{name} {max(as_list(lib[name])):.3e}" for name in BOUNDS))
    for name in BOUNDS:
        for i, (val, b) in enumerate(zip(as_list(res[name]), bound[name])):
            assert val <= b, f"{case} {mode}: stage {name}[{i}]: {val:.3e} > {b:.2e}  | full ladder: {report}"
    if mode == "strict":
        floor = g["floor"]
        assert res["flow_abs_max"] <= 2.5 * floor["flow_abs_max"] and res["cov_rel_max"] <= 2.5 * floor["cov_rel_max"]
    # the branches this size exists to cover were the ones taken
    corr, softmax_f16, native = BRANCHES[case]
    if mode == "strict" and corr == "tf32":
        corr = "tc3"
    assert rec["corr"] == [corr], rec
    assert rec["softmax_f16"] == (1 if softmax_f16 and mode == "tf32" else 0), rec
    assert rec["vglobal"] > 0 and rec["vglobal_native"] == (rec["vglobal"] if native else 0), rec
