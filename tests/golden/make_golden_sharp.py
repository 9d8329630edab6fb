"""Generate tests/golden/net_sharp.pt (640x480, the cfgA frames and branches) and net_sharp_kitti00.pt (1226x370, the
kitti00 branches): the parity fixtures of the sharpened checkpoint (cases.sharp_state_dict), with the contents of
net_cfgA.pt (make_golden_cfgA.py) plus the fp32 noise floor of every ladder stage and the softmax regime reached.

With the synthetic checkpoint every softmax of the frontend is close to uniform (median logit std 0.02 - 0.6), so a
wrong scale, a key paired with the wrong value or a misplaced position term barely moves the flow. The sharpened
checkpoint brings every family's median logit std into cases.SHARP_TARGET; this script asserts that it does on each
fixture's own frames, and that the reference's fp32 distance from the float64 truth (flow, covariance) stays within 10x
of net_cfgA.pt's, so that the sharper network is still one that fp32 computes faithfully.

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_sharp.py [sharp|sharp_kitti00 ...]
    python tests/golden/make_golden_sharp.py --calibrate      (choose cases.SHARP_GAINS; no reference needed)
"""
from __future__ import annotations

import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from make_golden_cfgA import FAMILIES, REPO, generate, softmax_regime  # noqa: E402
from tests.golden import cases  # noqa: E402

SHARP_CASES = ("sharp", "sharp_kitti00")


def regime(gains: dict, case: str = "sharp", depth: int = 3) -> dict:
    """softmax statistics of every family: float64 CPU network at decoder_depth `depth` on a sharp case's frames"""
    from macvo_b200.flowformer_cov import FlowFormerCovNet
    from oracle import frontend as ofe
    A, B = cases.ladder_inputs(case)
    net = FlowFormerCovNet(cases.sharp_state_dict(gains), "cpu", torch.float64, torch.float64, decoder_depth=depth,
                           corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup)
    out: dict = {}
    with softmax_regime(net, out):
        net.inference(A.double(), B.double())
    return out


def calibrate(rounds: int = 6) -> dict:
    """power-of-two gains that bring every family's median logit std into cases.SHARP_TARGET on the 640x480 frames (the
    key counts, and with them the statistics, depend on the frame size: 4 perceiver tokens per pixel at 96x128, 80 at
    640x480). The logits are linear in the product of the query and key gains (in the mask gain), so each round moves a
    family's exponent by the rounded log2 of (target centre / achieved std), split between query and key; downstream
    families see the upstream change through their inputs, hence the rounds. Starts from cases.SHARP_GAINS."""
    lo, hi = cases.SHARP_TARGET
    centre = math.sqrt(lo * hi)
    exps = {f: round(math.log2(cases.sharp_gain(cases.SHARP_GAINS, f, 0) * (cases.sharp_gain(cases.SHARP_GAINS, f, 1)
                                                                          if not f.startswith("mask") else 1.0)))
            for f in FAMILIES}
    to_gains = lambda e: {f: (2.0 ** ((n + 1) // 2), 2.0 ** (n // 2)) if not f.startswith("mask") else 2.0 ** n
                          for f, n in e.items()}
    for r in range(rounds):
        stats = regime(to_gains(exps))
        print(f"round {r}: " + ", ".join(f"{f} 2^{exps[f]} -> {stats[f]['logit_std_median']:.3f}" for f in FAMILIES),
              flush=True)
        if all(lo <= stats[f]["logit_std_median"] <= hi for f in FAMILIES):
            break
        for f in FAMILIES:
            s = stats[f]["logit_std_median"]
            if not lo <= s <= hi:
                exps[f] += max(-4, min(4, round(math.log2(centre / s))))
    else:
        raise SystemExit("calibration did not converge")
    gains = to_gains(exps)
    print("SHARP_GAINS =", gains)
    return gains


def check(case: str, out: dict) -> None:
    lo, hi = cases.SHARP_TARGET
    for f in FAMILIES:
        s = out["regime"][f]["logit_std_median"]
        assert lo <= s <= hi, f"{case}: family {f} reached median logit std {s:.3f}, outside {cases.SHARP_TARGET}"
    base = torch.load(os.path.join(HERE, "net_cfgA.pt"), weights_only=False)["floor"]
    fl = out["floor"]
    assert fl["flow_abs_max"] / fl["flow_scale"] <= 10 * base["flow_abs_max"] / base["flow_scale"], (case, fl, base)
    assert fl["cov_rel_max"] <= 10 * base["cov_rel_max"], (case, fl, base)


if __name__ == "__main__":
    args = sys.argv[1:]
    if args == ["--calibrate"]:
        sys.path.insert(0, REPO)
        calibrate()
        raise SystemExit(0)
    for case in args or SHARP_CASES:
        if case not in SHARP_CASES:
            raise SystemExit(f"unknown case {case!r}: one of {SHARP_CASES}")
        check(case, generate(case, cases.LADDER_WEIGHTS[case]))
