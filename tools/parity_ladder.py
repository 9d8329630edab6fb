"""Per-stage error ladder of the FlowFormerCov frontend at decoder_depth 12: GPU network (strict fp32, and the TF32 /
fp16-GMA mode bench.py times) against the float64 ground truth of tests/golden/net_<case>.pt, next to the reference's own
fp32 distance from that truth (the noise floor). Cases (tests/golden/cases.py::LADDER_CASES): cfgA (640x480, BASELINE
configs[1] shape), euroc (752x480), kitti (1241x376), kitti00 (1226x370), and sharp / sharp_kitti00 (the sharpened
checkpoint, cases.sharp_state_dict, on the cfgA / kitti00 frames). The network is built from the fixture's `weights`.

`library_ops=True` runs the library-op path instead: the same class with none of our kernels (`_ops = None`: torch /
cuDNN / cuBLAS ops, the oracle's correlation and window lookup) on the device under the same precision flags — what the
reference itself runs on a GPU, and the yardstick of the sharp cases in TF32 mode.

    python tools/parity_ladder.py [--out gpurun_out/parity_ladder.json]
    python tools/parity_ladder.py --case kitti --out <file>.json      (another frame size)

Error measure per stage: max |x - truth| / mean |truth|  (relative to the stage's scale); covariance: max relative.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from tests.golden import cases  # noqa: E402

STAGES = ("context", "feats", "corr_rows", "cost_memory")


def set_mode(mode: str) -> None:
    tf32 = mode != "strict"
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.allow_tf32 = tf32
    torch.set_float32_matmul_precision("medium" if tf32 else "highest")


def ladder(mode: str, golden: dict, case: str = "cfgA", device: str = "cuda", library_ops: bool = False) -> dict:
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    from oracle import frontend as ofe
    set_mode(mode)
    A, B = cases.ladder_inputs(case)
    assert golden["shape"] == (2, *cases.LADDER_CASES[case]), (golden["shape"], case)
    weights = golden.get("weights", "synthetic:0")          # fixtures without the entry were made from synthetic:0
    sd = synthetic_state_dict(0) if weights == "synthetic:0" else cases.ladder_state_dict(weights)
    net = FlowFormerCovNet(sd, device, decoder_depth=golden["decoder_depth"])
    if library_ops:
        net._ops, net.corr_fn, net.lookup_fn = None, ofe.corr_volume, ofe.window_lookup
    net.taps = {}
    flow, cov = net.inference(A.to(device), B.to(device))
    torch.cuda.synchronize()
    T, S = golden["truth"], (lambda name, t: cases.ladder_sample(case, name, t))
    rel = lambda x, t: ((x.double().cpu() - t).abs().max() / t.abs().mean()).item()
    out = {}
    for name in STAGES:
        out[name] = rel(S(name, net.taps[name][0]), T[name])
    for name in ("flow_iter", "cov_iter"):
        out[name] = [rel(S(name, x), t) for x, t in zip(net.taps[name], T[name])]
    fs, cs = S("flow", flow).double().cpu(), S("cov", cov).double().cpu()
    out["flow"] = rel(fs, T["flow"])
    out["flow_abs_max"] = (fs - T["flow"]).abs().max().item()
    out["cov_rel_max"] = ((cs - T["cov"]).abs() / T["cov"].abs()).max().item()
    out["cov_rel_p99"] = ((cs - T["cov"]).abs() / T["cov"].abs()).flatten().quantile(0.99).item()
    r = golden["ref32"]
    out["flow_vs_ref32"] = ((fs - r["flow"].double()).abs().max() / T["flow"].abs().mean()).item()
    out["cov_rel_vs_ref32"] = ((cs - r["cov"].double()).abs() / r["cov"].double().abs()).max().item()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default="cfgA", choices=list(cases.LADDER_CASES))
    ap.add_argument("--out", default=os.path.join(REPO, "gpurun_out", "parity_ladder.json"))
    a = ap.parse_args()
    g = torch.load(os.path.join(REPO, "tests", "golden", f"net_{a.case}.pt"), weights_only=False)
    T, r = g["truth"], g["ref32"]
    floor = {"flow": ((r["flow"].double() - T["flow"]).abs().max() / T["flow"].abs().mean()).item(),
             "cov_rel_max": ((r["cov"].double() - T["cov"]).abs() / T["cov"].abs()).max().item()}
    res = {"case": a.case, "floor_ref32_vs_truth": floor, "floor_full_tensor": g["floor"]}
    cols = ("strict", "tf32", "lib_tf32")
    for mode in ("strict", "tf32"):
        res[mode] = ladder(mode, g, a.case)
    res["lib_tf32"] = ladder("tf32", g, a.case, library_ops=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)
    print(f"{'stage':<18}" + "".join(f"{c:>12}" for c in cols))
    for name in STAGES:
        print(f"{name:<18}" + "".join(f"{res[c][name]:>12.3e}" for c in cols))
    for it in ("flow_iter", "cov_iter"):
        for i in range(len(res["strict"][it])):
            print(f"{it} {i + 1:<8}" + "".join(f"{res[c][it][i]:>12.3e}" for c in cols))
    for name in ("flow", "flow_abs_max", "cov_rel_max", "cov_rel_p99", "flow_vs_ref32", "cov_rel_vs_ref32"):
        print(f"{name:<18}" + "".join(f"{res[c][name]:>12.3e}" for c in cols))
    print("reference fp32 vs truth (noise floor):", floor)


if __name__ == "__main__":
    main()
