"""Generate the golden fixtures under tests/golden/ by running the REFERENCE ITSELF on CPU.

Needs a MAC-VO checkout:  MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden.py
The fixtures are small `.pt` files holding seeded inputs + the reference's outputs; the tests
(which never need the MAC-VO tree) only read them. Everything is seeded -> re-running reproduces
the files bit-for-bit on the same torch build.

What executes here is the unmodified reference code:
  corr      MemoryEncoder.corr                         Module/Network/FlowFormer/core/encoder.py:256
  lookup    MemoryDecoder.encode_flow_token            Module/Network/FlowFormer/core/decoder.py:141
  network   FlowFormerCov.inference (synthetic weights) Module/Network/FlowFormerCov/flownet.py:37
  postproc  FlowFormerCovFrontend.inference_2_depth/_match  Module/Frontend/Frontend.py:184-200
  selector  CovAwareSelector_NoDepth / MappingPointSelector Module/KeypointSelector.py:362,87
  cov       MatchCovariance.estimate                   Module/Covariance/Project2to3.py:124
  pgo       TwoFrame_PGO._optimize (LM_analytic + Analytic_ReprojDisp_TwoFramePGO) on top of the
            restated pypose (oracle/pypose_shim) — the only non-reference code in the loop.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from tests.golden import refharness  # noqa: E402
from tests.golden import cases  # noqa: E402


def save(name: str, obj: dict) -> None:
    path = os.path.join(HERE, name)
    torch.save(obj, path)
    print(f"wrote {name}: {os.path.getsize(path) / 1024:.1f} KiB")


def main() -> None:
    only = sys.argv[1] if len(sys.argv) > 1 else None      # e.g. `make_golden.py motion` regenerates one family
    global save
    if only:
        _save = save
        save = lambda name, obj: _save(name, obj) if name.startswith(only) else None
    refharness.install()
    torch.set_num_threads(8)
    import Module  # noqa: F401  (registers every plugin class)
    from DataLoader import StereoData
    from Module.Network.FlowFormer.configs.submission import get_cfg
    from Module.Network.FlowFormerCov import build_flowformer
    from Module.Frontend.Frontend import FlowFormerCovFrontend, IFrontend
    from Module.Frontend.StereoDepth import IStereoDepth
    from Module.Frontend.Matching import IMatcher
    from Module.KeypointSelector import CovAwareSelector_NoDepth, MappingPointSelector, CovAwareSelector
    from Module.Covariance.Project2to3 import MatchCovariance
    from Module.Optimization.TwoFramePGO.Optimizer import TwoFrame_PGO
    from Module.Optimization.TwoFramePGO.Graphs import GraphInput
    from Module.Map import MatchObs, PointNode
    import pypose as pp
    from macvo_b200.flowformer_cov import synthetic_state_dict

    cfg = get_cfg()
    model = build_flowformer(cfg, torch.float32, torch.float32).eval()
    model.load_state_dict(synthetic_state_dict(0))

    # ---- corr (a3) ------------------------------------------------------------------------
    for name, (B, H1, W1) in cases.CORR_CASES.items():
        f1, f2 = cases.corr_inputs(B, H1, W1)
        out = model.memory_encoder.corr(f1, f2)
        # keep fixtures small: store a strided sample of the volume + its full checksum
        rows, cols = cases.corr_sample_index(H1 * W1)
        save(f"corr_{name}.pt", {"shape": (B, H1, W1), "input_sha": cases.sha(f1, f2), "sample": out.reshape(B, H1 * W1, H1 * W1)[:, rows][:, :, cols].clone(),
                                 "sum": out.double().sum(), "abs_sum": out.double().abs().sum()})

    # ---- lookup (a5) ----------------------------------------------------------------------
    for name, (B, H1, W1) in cases.LOOKUP_CASES.items():
        cost_maps, coords = cases.lookup_inputs(B, H1, W1)
        out = model.memory_decoder.encode_flow_token(cost_maps, coords.clone())
        save(f"lookup_{name}.pt", {"shape": (B, H1, W1), "out": out.clone(), "input_sha": cases.sha(cost_maps, coords)})

    # ---- network end to end (a2), synthetic weights -----------------------------------------
    for name, (B, H, W) in cases.NET_CASES.items():
        img1, img2 = cases.net_inputs(B, H, W)
        flow, cov = model.inference(img1, img2)
        save(f"net_{name}.pt", {"shape": (B, H, W), "flow": flow.clone(), "cov": cov.clone(), "input_sha": cases.sha(img1, img2)})

    # ---- MACVO_Fast numerics (enc fp16 / dec bf16) of the reference + float64 truth of the same input ----------------
    from oracle import frontend as _ofe
    from macvo_b200.flowformer_cov import FlowFormerCovNet as _Net
    fast = build_flowformer(cfg, torch.float16, torch.bfloat16).eval()
    fast.load_state_dict(synthetic_state_dict(0))
    B, H, W = cases.NET_CASES["small"]
    img1, img2 = cases.net_inputs(B, H, W)
    ff, fc = fast.inference(img1, img2)
    net64 = _Net(synthetic_state_dict(0), "cpu", torch.float64, torch.float64, corr_fn=_ofe.corr_volume, lookup_fn=_ofe.window_lookup)
    tf, tc = net64.inference(img1.double(), img2.double())
    save("net_fast_small.pt", {"shape": (B, H, W), "flow": ff.float().clone(), "cov": fc.float().clone(), "truth_flow": tf.clone(),
                               "truth_cov": tc.clone(), "input_sha": cases.sha(img1, img2),
                               "floor": {"flow_rel": ((ff.double() - tf).abs().max() / tf.abs().mean()).item(),
                                         "cov_rel_max": ((fc.double() - tc).abs() / tc.abs()).max().item()}})

    # ---- dense post-processing (a7) ---------------------------------------------------------
    def stereo(H, W, fx, bl):
        return StereoData(T_BS=None, K=torch.tensor([[[fx, 0., W / 2], [0., fx, H / 2], [0., 0., 1.]]]),
                          baseline=torch.tensor([bl]), time_ns=[0], height=H, width=W,
                          imageL=torch.zeros(1, 3, H, W), imageR=torch.zeros(1, 3, H, W))

    for name, (H, W) in cases.DENSE_CASES.items():
        est_flow, est_cov = cases.dense_inputs(H, W)
        frame = stereo(H, W, 320.0, 0.25)
        for epd in (False, True):
            d = FlowFormerCovFrontend.inference_2_depth(est_flow[0:1], est_cov[0:1], frame, epd)
            m = FlowFormerCovFrontend.inference_2_match(est_flow[1:2], est_cov[1:2])
            save(f"dense_{name}_{int(epd)}.pt", {
                "shape": (H, W), "input_sha": cases.sha(est_flow, est_cov), "depth": d.depth, "disparity": d.disparity, "depth_cov": d.cov,
                "disparity_uncertainty": d.disparity_uncertainty, "depth_mask": d.mask,
                "flow": m.flow, "flow_cov": m.cov})

    # ---- selectors (a8, a8'') ---------------------------------------------------------------
    sel = CovAwareSelector_NoDepth(SimpleNamespace(device="cpu", kernel_size=7, mask_width=32, max_match_cov=100.0))
    mapsel = MappingPointSelector(SimpleNamespace(max_depth=5.0, max_depth_cov=0.005, mask_width=32))
    for name, (H, W, num, variant) in cases.SELECTOR_CASES.items():
        est_flow, est_cov = cases.selector_inputs(H, W, variant)
        frame = stereo(H, W, 320.0, 0.25)
        depth = FlowFormerCovFrontend.inference_2_depth(est_flow[0:1], est_cov[0:1], frame, False)
        match = FlowFormerCovFrontend.inference_2_match(est_flow[1:2], est_cov[1:2])
        if variant == "masked":
            match.mask = cases.selector_match_mask(H, W)
        torch.manual_seed(cases.SELECTOR_RNG_SEED)
        kp = sel.select_point(frame, num, depth, depth, match)
        mp = mapsel.select_point(frame, 2000, depth, depth, match)      # second randperm of the frame
        save(f"selector_{name}.pt", {"shape": (H, W), "num": num, "variant": variant, "kp": kp, "map_kp": mp,
                                     "input_sha": cases.sha(est_flow, est_cov)})

    dsel = CovAwareSelector(SimpleNamespace(device="cpu", kernel_size=7, mask_width=32, max_depth="auto",
                                            max_depth_cov=250.0, max_match_cov=100.0))
    for name, (H, W, num, variant) in cases.SELECTOR_DEPTH_CASES.items():
        (f0, c0), (f1, c1) = cases.selector_depth_inputs(H, W, variant)
        frame = stereo(H, W, 320.0, 0.25)
        depth0 = FlowFormerCovFrontend.inference_2_depth(f0[0:1], c0[0:1], frame, variant == "masked")
        depth1 = FlowFormerCovFrontend.inference_2_depth(f1[0:1], c1[0:1], frame, False)
        match = FlowFormerCovFrontend.inference_2_match(f1[1:2], c1[1:2])
        if variant == "masked":
            match.mask = cases.selector_match_mask(H, W)
            depth0.mask = ~depth0.mask          # reference contract: True = valid (StereoDepth.py:28-30)
        torch.manual_seed(cases.SELECTOR_RNG_SEED)
        kp = dsel.select_point(frame, num, depth0, depth1, match)
        save(f"selector_{name}.pt", {"shape": (H, W), "num": num, "variant": variant, "kp": kp,
                                     "input_sha": cases.sha(f0, c0, f1, c1)})

    # ---- covariance model (a10) ---------------------------------------------------------------
    covm = MatchCovariance(SimpleNamespace(device="cpu", kernel_size=31, match_cov_default=0.25,
                                           min_depth_cov=0.05, min_flow_cov=0.25))
    for name, (H, W, K, kind) in cases.COV_CASES.items():
        kp, depth_map, flow_cov = cases.cov_inputs(H, W, K, kind)
        frame = stereo(H, W, 320.0, 0.25)
        dest = IStereoDepth.Output(depth=depth_map)
        fc = None if flow_cov is None else flow_cov.clone()
        out = covm.estimate(frame, kp, dest, None, fc)
        save(f"covariance_{name}.pt", {"shape": (H, W, K), "kind": kind, "out": out,
                                       "flow_cov_after": fc, "input_sha": cases.sha(kp, depth_map, flow_cov)})

    # ---- two-frame PGO (a13-a16): the three graph types ------------------------------------------
    def run_pgo(c, graph_type):
        K = c["pos_Tw"].shape[0]
        obs = MatchObs.init({
            "pixel1_uv": torch.zeros(K, 2), "pixel2_uv": c["kp2_uv"],
            "pixel1_d": torch.zeros(K, 1), "pixel2_d": c.get("kp2_d", torch.zeros(K)).unsqueeze(-1),
            "pixel1_disp": torch.zeros(K, 1), "pixel2_disp": c["kp2_disp"].unsqueeze(-1),
            "pixel1_disp_cov": torch.zeros(K, 1), "pixel2_disp_cov": c["disp_cov"].unsqueeze(-1),
            "pixel1_d_cov": torch.zeros(K, 1), "pixel2_d_cov": torch.zeros(K, 1),
            "pixel1_uv_cov": torch.zeros(K, 3), "pixel2_uv_cov": c["uv_cov"],
            "obs1_covTc": torch.zeros(K, 3, 3, dtype=torch.double),
            "obs2_covTc": c.get("obs_cov", torch.zeros(K, 3, 3, dtype=torch.double))})
        pts = PointNode.init({"pos_Tw": c["pos_Tw"], "cov_Tw": c.get("pts_cov", torch.zeros(K, 3, 3, dtype=torch.double)),
                              "color": torch.zeros(K, 3, dtype=torch.uint8)})
        gi = GraphInput(torch.tensor([1]), torch.tensor([0]), pp.SE3(c["init_pose"].unsqueeze(0)),
                        torch.tensor([c["baseline"]]), obs, pts, c["K"], torch.zeros(K, dtype=torch.long), "cpu")
        ctx = TwoFrame_PGO.init_context(SimpleNamespace(autodiff=False, graph_type=graph_type, device="cpu",
                                                        vectorize=True, parallel=False))
        # `_optimize` asks for torch.cuda.current_stream() only to hand it to an inactive Timer
        # (Optimizer.py:83-84); this container has no CUDA driver, so give it a placeholder.
        _cs, torch.cuda.current_stream = torch.cuda.current_stream, (lambda *a, **k: None)
        try:
            _, out = TwoFrame_PGO._optimize(ctx, gi)
        finally:
            torch.cuda.current_stream = _cs
        return out.motion.detach().as_subclass(torch.Tensor).clone().reshape(7)

    for name, (K, seed) in cases.PGO_CASES.items():
        c = cases.pgo_inputs(K, seed)
        save(f"pgo_{name}.pt", {"K": K, "seed": seed, "input_sha": cases.sha(*[c[k] for k in ("pos_Tw", "kp2_uv", "kp2_disp", "uv_cov", "disp_cov")]),
                                "pose": run_pgo(c, "disp")})
    for name, (gt, K, seed) in cases.PGO_TYPE_CASES.items():
        c = cases.pgo_inputs_typed(gt, K, seed)
        save(f"pgo_{name}.pt", {"K": K, "seed": seed, "graph_type": gt, "pose": run_pgo(c, gt),
                                "input_sha": cases.sha(*[c[k] for k in ("pos_Tw", "kp2_uv", "kp2_disp", "uv_cov", "disp_cov", "kp2_d", "obs_cov", "pts_cov")])})

    # ---- trajectory post-process at terminate() (f4) --------------------------------------------
    from Module.MapProcessor import MotionInterpolate
    from Module.Map import VisualMap, FrameNode
    for name, (F, seed, flagged) in cases.MOTION_CASES.items():
        poses, need = cases.motion_inputs(F, seed, flagged)
        m = VisualMap()
        for i in range(F):
            m.frames.push(FrameNode.init({"pose": poses[i:i + 1].clone(), "T_BS": pp.identity_SE3(1), "need_interp": need[i:i + 1].clone(),
                                          "time_ns": torch.tensor([i]), "K": torch.eye(3).unsqueeze(0), "baseline": torch.tensor([0.25])}))
        _, idx = MotionInterpolate(SimpleNamespace()).elaborate_map(m.frames)
        save(f"motion_{name}.pt", {"F": F, "seed": seed, "flagged": flagged, "out": m.frames.data["pose"].tensor.clone(),
                                   "interp_idx": idx.clone(), "input_sha": cases.sha(poses, need.to(torch.uint8))})


if __name__ == "__main__":
    main()
