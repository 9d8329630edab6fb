"""Frontend parity at the benched shape: 640x480, decoder_depth 12, the `estimate_pair` batch of the bench sequence, in
BOTH precision modes, stage by stage, against the float64 ground truth of tests/golden/net_cfgA.pt (generated next to the
reference's own fp32 run by tests/golden/make_golden_cfgA.py).

Yardstick: the REFERENCE's fp32 CPU result is itself 2.6e-6 (flow, relative to the mean |flow|) and 1.3e-4 (covariance,
relative) away from exact arithmetic on this input (`floor`). north_star's "within 1e-4 relative" is therefore met for
the flow by any faithful fp32 implementation and is AT the fp32 noise floor for the covariance.

  strict   allow_tf32 = False: every layer fp32 (our kernels fp32 FMA, cuDNN / cuBLAS fp32, correlation volume 3 x fp16
           split). Asserted: final flow and covariance within 2x the reference's own distance from the truth, within
           1e-5 / 2e-4 of the reference's fp32 output, every stage within a few 1e-5.
  tf32     what bench.py times = the reference GPU frontend's own setting (Frontend.py:275-277: TF32 matmuls and
           convolutions): cuDNN / cuBLAS TF32, our attention / PatchEmbed kernels with TF32 operands, tf32
           correlation volume, fp16 GMA attention matrix. TF32 keeps 10 mantissa bits (2^-11 = 4.9e-4 per operand):
           the encoders already differ by 3.5e-3 of their scale, the refinement contracts that to 6e-4 on the flow.
           Bounds = 1.5 x the measured ladder (tools/parity_ladder.py), so that one dropped mantissa bit
           (2 x the error) fails the test.
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


@pytest.fixture(scope="module")
def ladder_fn():
    assert torch.cuda.is_available()
    from macvo_b200 import build
    build.build(verbose=False)
    import parity_ladder
    return parity_ladder


@pytest.mark.parametrize("mode", ["strict", "tf32"])
def test_frontend_parity_ladder_cfgA(ladder_fn, golden, mode):
    g = golden("net_cfgA.pt")
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    try:
        res = ladder_fn.ladder(mode, g)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev[0], prev[1]
        torch.set_float32_matmul_precision(prev[2])
    col = 0 if mode == "strict" else 1
    report = []
    for name, bounds in BOUNDS.items():
        val = max(res[name]) if isinstance(res[name], list) else res[name]
        report.append(f"{name} {val:.3e} (bound {bounds[col]:.1e})")
    print(f"[{mode}] " + "; ".join(report))
    for name, bounds in BOUNDS.items():
        val = max(res[name]) if isinstance(res[name], list) else res[name]
        assert val <= bounds[col], f"{mode}: stage {name}: {val:.3e} > {bounds[col]:.1e}  | full ladder: {report}"
    if mode == "strict":
        floor = g["floor"]
        assert res["flow_abs_max"] <= 2.5 * floor["flow_abs_max"] and res["cov_rel_max"] <= 2.5 * floor["cov_rel_max"]
