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
`generate(case, weights="sharp:0")` runs the sharpened checkpoint (cases.sharp_state_dict, make_golden_sharp.py) and
also records `weights`, the fp32 noise floor of every ladder stage (`floor_stages`: the fp32 run of the same class
against the truth, on the ladder's error measure) and the softmax regime each family reached (`regime`).
"""
from __future__ import annotations

import contextlib
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import cases, refharness  # noqa: E402

# every softmax of the frontend, by the weights that set its logits (cases.sharp_rows)
FAMILIES = ("svt_local", "svt_global", "perceiver_input", "latent", "vert_local", "vert_global", "cross_attend", "gma",
            "mask_flow", "mask_cov")


@contextlib.contextmanager
def softmax_regime(net, out: dict):
    """Record, for every softmax a CPU `FlowFormerCovNet` evaluates, the std of each row's logits and its largest weight;
    on exit out[family] = {"logit_std_median", "max_weight_median", "keys", "rows"}. The network's methods are wrapped on
    the instance, its arithmetic is unchanged."""
    rows = {f: ([], []) for f in FAMILIES}
    keys = {}
    stack: list[str] = []

    def add(fam: str, logits: torch.Tensor, dim: int = -1) -> None:
        rows[fam][0].append(logits.std(dim=dim, unbiased=False).flatten().float())
        rows[fam][1].append(logits.softmax(dim=dim).amax(dim=dim).flatten().float())
        keys[fam] = logits.shape[dim]

    attn = net._attn

    def attn_rec(q, k, v, heads):
        B, J, C = k.shape
        d = C // heads
        qh = q.reshape(q.shape[0], q.shape[1], heads, d).permute(0, 2, 1, 3)
        kh = k.reshape(B, J, heads, d).permute(0, 2, 1, 3)
        for b0 in range(0, B, 512):
            add(stack[-1], (qh if qh.shape[0] == 1 else qh[b0:b0 + 512]) @ kh[b0:b0 + 512].transpose(-1, -2) * d ** -0.5)
        return attn(q, k, v, heads)

    def scoped(fam, fn):
        def run(*a, **k):
            stack.append(fam)
            try:
                return fn(*a, **k)
            finally:
                stack.pop()
        return run

    conv = net._conv

    def conv_rec(x, p, *a, **k):
        y = conv(x, p, *a, **k)
        if p == "memory_decoder.att.to_qk":          # GMA scores (gma.py:39-82), as memory_decoder forms them
            qv = (y[:, :128] * (128 ** -0.5)).flatten(2).transpose(1, 2)
            for r0 in range(0, qv.shape[1], 1024):
                add("gma", torch.matmul(qv[:, r0:r0 + 1024], y[:, 128:].flatten(2)))
        return y

    upsample, masks = net.convex_upsample, iter(("mask_flow", "mask_cov"))

    def upsample_rec(flow, mask):
        N, _, H, W = flow.shape
        add(next(masks), mask.reshape(N, 9, 8, 8, H, W), dim=1)
        return upsample(flow, mask)

    wrapped = {"_attn": attn_rec, "_conv": conv_rec, "convex_upsample": upsample_rec,
               "cost_perceiver": scoped("perceiver_input", net.cost_perceiver),
               "_svt_local_attn": scoped("svt_local", net._svt_local_attn),
               "_svt_global_attn": scoped("svt_global", net._svt_global_attn),
               "_latent_layer": scoped("latent", net._latent_layer),
               "_vert_local_attn": scoped("vert_local", net._vert_local_attn),
               "_vert_global_attn": scoped("vert_global", net._vert_global_attn),
               "_refine_torch": scoped("cross_attend", net._refine_torch)}
    for name, fn in wrapped.items():
        setattr(net, name, fn)
    try:
        yield out
    finally:
        for name in wrapped:
            delattr(net, name)
    for fam, (std, w) in rows.items():
        std, w = torch.cat(std), torch.cat(w)
        out[fam] = {"logit_std_median": std.median().item(), "max_weight_median": w.median().item(),
                    "keys": keys[fam], "rows": std.numel()}


def stage_errors(case: str, taps: dict, flow, cov, truth: dict, ref32: dict) -> dict:
    """the parity ladder's error of every stage (tools/parity_ladder.py: max |x - truth| / mean |truth| on the fixture's
    sample; covariance: max relative) for a run's taps and outputs"""
    S = lambda name, t: cases.ladder_sample(case, name, t)
    rel = lambda x, t: ((x.double().cpu() - t).abs().max() / t.abs().mean()).item()
    out = {name: rel(S(name, taps[name][0]), truth[name]) for name in ("context", "feats", "corr_rows", "cost_memory")}
    for name in ("flow_iter", "cov_iter"):
        out[name] = [rel(S(name, x), t) for x, t in zip(taps[name], truth[name])]
    fs, cs = S("flow", flow).double(), S("cov", cov).double()
    out["flow"] = rel(fs, truth["flow"])
    out["cov_rel_max"] = ((cs - truth["cov"]).abs() / truth["cov"].abs()).max().item()
    out["flow_vs_ref32"] = ((fs - ref32["flow"].double()).abs().max() / truth["flow"].abs().mean()).item()
    out["cov_rel_vs_ref32"] = ((cs - ref32["cov"].double()).abs() / ref32["cov"].double().abs()).max().item()
    return out


def generate(case: str, weights: str = "synthetic:0") -> dict:
    refharness.install()
    torch.set_num_threads(8)
    from Module.Network.FlowFormer.configs.submission import get_cfg
    from Module.Network.FlowFormerCov import build_flowformer
    from macvo_b200.flowformer_cov import FlowFormerCovNet
    from oracle import frontend as ofe

    sharp = weights != "synthetic:0"
    sd = cases.ladder_state_dict(weights)
    A, B = cases.ladder_inputs(case)
    model = build_flowformer(get_cfg(), torch.float32, torch.float32).eval()
    model.load_state_dict(sd)
    t0 = time.time()
    rf, rc = model.inference(A, B)
    print(f"{case} reference fp32: {time.time() - t0:.1f} s")
    del model
    net64 = FlowFormerCovNet(sd, "cpu", torch.float64, torch.float64, corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup)
    net64.taps = {}
    regime: dict = {}
    t0 = time.time()
    with softmax_regime(net64, regime) if sharp else contextlib.nullcontext():
        tf, tc = net64.inference(A.double(), B.double())
    print(f"{case} float64 truth: {time.time() - t0:.1f} s")
    taps = net64.taps
    del net64
    net32 = FlowFormerCovNet(sd, "cpu", corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup)
    net32.taps = {} if sharp else None
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
    if sharp:
        out["weights"] = weights
        out["floor_stages"] = stage_errors(case, net32.taps, of, oc, truth, out["ref32"])
        out["regime"] = regime
        print(case, "fp32 floor per stage:", out["floor_stages"])
        print(case, "regime:", regime)
    path = os.path.join(HERE, f"net_{case}.pt")
    torch.save(out, path)
    print(f"wrote net_{case}.pt: {os.path.getsize(path) / 1024:.1f} KiB")
    return out


if __name__ == "__main__":
    generate("cfgA")
