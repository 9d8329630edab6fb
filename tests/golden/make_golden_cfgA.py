"""Generate tests/golden/net_cfgA.pt: the 640x480, decoder_depth 12 parity fixture (BASELINE configs[1] shape).

Needs a MAC-VO checkout (~2.5 min):  MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_cfgA.py

Contents (strided samples, tests/golden/cases.py::ladder_sample):
  ref32   flow / cov of the UNMODIFIED reference network (`FlowFormerCov.inference`, flownet.py:37-44) in fp32 on the CPU;
  truth   flow / cov and per-stage intermediates (encoder features, context, correlation rows, cost memory, the flow /
          covariance iterate after each of the 12 refinements) of `FlowFormerCovNet` run in FLOAT64 on the CPU with the
          oracle's correlation / lookup. The reference hard-casts to fp32 at its module interfaces (flownet.py:28-29,
          covhead.py:121-131), so it cannot run in float64 itself; the float64 class is tied to it through the fp32
          comparison below (the two fp32 runs agree to the fp32 noise floor recorded in `floor`).
  floor   |ref32 - truth|: how far the reference's own fp32 arithmetic is from exact arithmetic on this input —
          the yardstick the GPU parity bounds are multiples of (tests/test_gpu_parity_ladder.py).

`generate(case)` writes the same contents for any frame size of cases.LADDER_CASES (make_golden_datasets.py).
"""
from __future__ import annotations

import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import cases, refharness  # noqa: E402


def generate(case: str) -> None:
    refharness.install()
    torch.set_num_threads(8)
    from Module.Network.FlowFormer.configs.submission import get_cfg
    from Module.Network.FlowFormerCov import build_flowformer
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    from oracle import frontend as ofe

    sd = synthetic_state_dict(0)
    A, B = cases.ladder_inputs(case)
    model = build_flowformer(get_cfg(), torch.float32, torch.float32).eval()
    model.load_state_dict(sd)
    t0 = time.time()
    rf, rc = model.inference(A, B)
    print(f"{case} reference fp32: {time.time() - t0:.1f} s")
    del model
    net64 = FlowFormerCovNet(sd, "cpu", torch.float64, torch.float64, corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup)
    net64.taps = {}
    t0 = time.time()
    tf, tc = net64.inference(A.double(), B.double())
    print(f"{case} float64 truth: {time.time() - t0:.1f} s")
    taps = net64.taps
    del net64
    net32 = FlowFormerCovNet(sd, "cpu", corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup)
    of, oc = net32.inference(A, B)

    S = lambda name, t: cases.ladder_sample(case, name, t)
    truth = {"flow": S("flow", tf).clone(), "cov": S("cov", tc).clone()}
    for name, lst in taps.items():
        truth[name] = [S(name, t).clone() for t in lst] if name.endswith("_iter") else S(name, lst[0]).clone()
    floor = {
        "flow_abs_max": (rf.double() - tf).abs().max().item(), "flow_scale": tf.abs().mean().item(),
        "cov_rel_max": ((rc.double() - tc).abs() / tc.abs()).max().item(),
        "class_fp32_vs_ref32_flow_abs_max": (of - rf).abs().max().item(),
        "class_fp32_vs_ref32_cov_rel_max": ((oc - rc).abs() / rc.abs()).max().item(),
    }
    print(case, floor)
    out = {"shape": (2, *cases.LADDER_CASES[case]), "decoder_depth": 12,
           "ref32": {"flow": S("flow", rf).clone(), "cov": S("cov", rc).clone()}, "truth": truth, "floor": floor,
           "input_sum": (float(A.double().sum()), float(B.double().sum()))}
    path = os.path.join(HERE, f"net_{case}.pt")
    torch.save(out, path)
    print(f"wrote net_{case}.pt: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    generate("cfgA")
