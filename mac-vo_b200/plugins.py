"""B200 plugin classes for MAC-VO's `Module` interfaces (the drop-in boundary, SURVEY.md §8b).

    B200_FlowFormerCovFrontend       IFrontend          replaces CUDAGraph_FlowFormerCovFrontend (Frontend.py:264-353)
    B200_FlowFormerFrontend          IFrontend          replaces FrontendCompose(FlowFormerDepth, FlowFormerMatcher)
                                                        (Frontend.py:131-155, StereoDepth.py:99-135, Matching.py:120-154)
    B200_CovAwareSelector_NoDepth    IKeypointSelector  replaces CovAwareSelector_NoDepth (KeypointSelector.py:349-407)
    B200_CovAwareSelector            IKeypointSelector  replaces CovAwareSelector (KeypointSelector.py:250-347)
    B200_MappingPointSelector        IKeypointSelector  replaces MappingPointSelector (KeypointSelector.py:78-100)
    B200_RandomSelector              IKeypointSelector  replaces RandomSelector (KeypointSelector.py:103-118)
    B200_MatchCovariance             ICovariance2to3    replaces MatchCovariance (Covariance/Project2to3.py:114-182)
    B200_NoCovariance                ICovariance2to3    replaces NoCovariance (Covariance/Project2to3.py:48-57)
    B200_Modifier_Diagonalize        ICovariance2to3    replaces Modifier_Diagonalize (Covariance/Project2to3.py:281-302)
    B200_Modifier_Normalize          ICovariance2to3    replaces Modifier_Normalize (Covariance/Project2to3.py:305-323)
    B200_CovarianceSanityFilter      IObservationFilter replaces CovarianceSanityFilter (OutlierFilter.py:91-100)
    B200_SimpleDepthFilter           IObservationFilter replaces SimpleDepthFilter (OutlierFilter.py:103-124)
    B200_LikelyFrontOfCamFilter      IObservationFilter replaces LikelyFrontOfCamFilter (OutlierFilter.py:127-141)
    B200_FilterCompose               IObservationFilter replaces FilterCompose (OutlierFilter.py:44-75)
    B200_MotionInterpolate           IMapProcessor      replaces MotionInterpolate (MapProcessor.py:52-79)
    B200_TwoFrame_PGO                IOptimizer         replaces TwoFrame_PGO (Optimization/TwoFramePGO/Optimizer.py:23-108)
    B200_TartanMotionNet             IMotionModel       replaces TartanMotionNet (MotionModel.py:89-116)
    B200_TartanVOMatcher             IMatcher           replaces TartanVOMatcher (Frontend/Matching.py:199-230)
    B200_TartanVODepth               IStereoDepth       replaces TartanVODepth (Frontend/StereoDepth.py:186-229)
    B200_TartanVO                    IOdometry          replaces TartanVO (Odometry/BaselineTartanVO.py:12-80)

Same constructor signature (`__init__(config: SimpleNamespace)`), same `is_valid_config` contract
(unknown keys are an error), same argument meaning and return types as the classes they replace; class
names are new because the registry forbids duplicates. With MAC-VO importable they subclass MAC-VO's own
interfaces (see `interfaces.py`); YAML selects them with `type: B200_...` — see INTEGRATION.md.

All compute goes through `ops` (ctypes -> libmacvo_b200.so). No CPU fallback: constructing a plugin with a
non-CUDA device raises.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace

import torch

from . import interfaces as _local
from . import ops
from . import posenet
from . import pwcnet
from . import stereonet
from .flowformer_cov import FlowFormerCovNet, synthetic_state_dict

_REF = _local.reference_available()
if _REF:   # subclass MAC-VO's own interfaces so that importing this module registers the plugins there
    from DataLoader import StereoData  # type: ignore
    from Module.Frontend.Frontend import IFrontend  # type: ignore
    from Module.Frontend.StereoDepth import IStereoDepth  # type: ignore
    from Module.Frontend.Matching import IMatcher  # type: ignore
    from Module.KeypointSelector import IKeypointSelector  # type: ignore
    from Module.Covariance.Project2to3 import ICovariance2to3  # type: ignore
    from Module.OutlierFilter import IObservationFilter  # type: ignore
    from Module.MapProcessor import IMapProcessor  # type: ignore
    from Module.Optimization.TwoFramePGO.Optimizer import TwoFrame_PGO as _PGOBase  # type: ignore
    from Module.Optimization.TwoFramePGO.Graphs import GraphOutput as _RefGraphOutput  # type: ignore
    from Module.MotionModel import IMotionModel  # type: ignore
    import pypose as _pp  # type: ignore
else:
    StereoData = _local.StereoData
    IFrontend, IStereoDepth, IMatcher = _local.IFrontend, _local.IStereoDepth, _local.IMatcher
    IKeypointSelector, ICovariance2to3 = _local.IKeypointSelector, _local.ICovariance2to3
    IObservationFilter, IMapProcessor = _local.IObservationFilter, _local.IMapProcessor
    _PGOBase = _local.IOptimizer
    IMotionModel = _local.IMotionModel
    _pp = None

_DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def _require_cuda(device: str, who: str) -> torch.device:
    if "cuda" not in str(device):
        raise ValueError(f"{who}: the B200 plugins only run on a CUDA device (got device={device!r}); "
                         "use the reference classes for CPU")
    return torch.device(device)


# ================================================================================================
# Frontend
# ================================================================================================
def _load_weights(w, covariance: bool) -> dict:
    """checkpoint path, or "synthetic[:seed]" for the deterministic stand-in"""
    if isinstance(w, str) and w.startswith("synthetic"):
        return synthetic_state_dict(int(w.split(":")[1]) if ":" in w else 0, covariance=covariance)
    return torch.load(w, map_location="cpu", weights_only=True)


class _B200_GraphedPairFrontend(IFrontend):
    """What both FlowFormer frontends share: `estimate_pair` as ONE B = 2 network pass, [t2.L, t1.L] against [t2.R, t2.L]
    (Frontend.py:284-285) with t2.L encoded once, plus the dense post-processing, replayed as a CUDA graph after the first
    call (like CUDAGraph_FlowFormerCovFrontend, Frontend.py:301-353). Subclasses give `_run` (device images -> the
    post-processed dict of `ops.dense_postproc`) and `_outputs` (that dict -> the interface's output pair)."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self._graph = None
        self._static: dict = {}

    def _run(self, input_A, input_B, bl_fx: float) -> dict:
        raise NotImplementedError

    def _outputs(self, d: dict, clone: bool):
        raise NotImplementedError

    @torch.inference_mode()
    def estimate_pair(self, frame_t1: StereoData, frame_t2: StereoData):
        """-> (IStereoDepth.Output of t2, IMatcher.Output t1 -> t2); batches [t2.L, t1.L] vs [t2.R, t2.L]
        exactly like the reference (Frontend.py:284-285)."""
        bl_fx = frame_t2.frame_baseline * frame_t2.fx
        if self._graph is not None:
            # steady state: the four images go straight into the graph's static input buffers (no host-side concatenation;
            # from pinned host memory these are asynchronous copies that overlap the previous frame's tail)
            st = self._static
            shape = (2,) + tuple(frame_t2.imageL.shape[1:])
            assert shape == st["shape"], f"Input shape mismatch for CUDAGraph replay: {shape} != {st['shape']}"
            assert bl_fx == st["bl_fx"], "camera baseline * fx changed since the CUDA graph was captured"
            # each image crosses PCIe once: t1.L is last call's t2.L and already sits in A[0] (device->device move), and
            # B[1] = t2.L is copied from A[0] after the upload
            if st.get("last_t2L") is frame_t1.imageL:
                st["A"][1:2].copy_(st["A"][0:1])
            else:
                st["A"][1:2].copy_(frame_t1.imageL, non_blocking=True)
            st["A"][0:1].copy_(frame_t2.imageL, non_blocking=True)
            st["B"][0:1].copy_(frame_t2.imageR, non_blocking=True)
            st["B"][1:2].copy_(st["A"][0:1])
            st["last_t2L"] = frame_t2.imageL
            self._graph.replay()
            ops.LAUNCHES[0] += st["launches"]
            return self._outputs(st["out"], clone=True)
        input_A = torch.cat([frame_t2.imageL, frame_t1.imageL], dim=0)
        input_B = torch.cat([frame_t2.imageR, frame_t2.imageL], dim=0)
        if not getattr(self.config, "cuda_graph", True):
            out = self._run(input_A.to(self.device, non_blocking=True), input_B.to(self.device, non_blocking=True), bl_fx)
            return self._outputs(out, clone=False)
        # first call: warm up (cuDNN autotune, workspace growth) on a side stream, then capture one frame
        sA = torch.empty(input_A.shape, dtype=torch.float32, device=self.device)
        sB = torch.empty_like(sA)
        sA.copy_(input_A)
        sB.copy_(input_B)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                self._run(sA, sB, bl_fx)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES[0]
        with torch.cuda.graph(graph):
            out = self._run(sA, sB, bl_fx)
        self._graph = graph
        self._static = {"A": sA, "B": sB, "out": out, "shape": tuple(input_A.shape), "bl_fx": bl_fx,
                        "launches": ops.LAUNCHES[0] - n0,     # macvo_b200 kernels inside one replay
                        "last_t2L": frame_t2.imageL}
        graph.replay()                             # (the reference returns its warm-up result here)
        return self._outputs(out, clone=True)

    @staticmethod
    def retrieve_pixels(pixel_uv: torch.Tensor, scalar_map: torch.Tensor | None, interpolate: bool = False):
        """(a9) gather kernel; same contract as IFrontend.retrieve_pixels (Frontend.py:104-118)."""
        if scalar_map is None:
            return None
        if interpolate:
            raise NotImplementedError("Not implemented yet")
        if scalar_map.is_cuda and scalar_map.dtype == torch.float32 and pixel_uv.dtype in (torch.int64, torch.float32):
            return ops.retrieve_pixels(pixel_uv.to(scalar_map.device), scalar_map)
        return scalar_map[0, ..., pixel_uv[..., 1].long(), pixel_uv[..., 0].long()]   # e.g. the CPU colour image


class B200_FlowFormerCovFrontend(_B200_GraphedPairFrontend):
    """FlowFormerCov stereo + flow frontend: correlation volume and window lookup on sm_90a kernels,
    dense post-processing + keypoint scoring fused into one pass, the whole `estimate_pair` replayed as a
    CUDA graph (like CUDAGraph_FlowFormerCovFrontend, Frontend.py:301-353).

    config: weight (checkpoint path, or "synthetic[:seed]" for the deterministic stand-in), device,
    enc_dtype / dec_dtype in {fp32, fp16, bf16}, decoder_depth, enforce_positive_disparity,
    cuda_graph (bool), score_kernel_size (odd int; NMS window of the fused keypoint scoring, 7 in the
    reference configs)."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_FlowFormerCovFrontend")
        sd = _load_weights(config.weight, covariance=True)
        enc, dec = _DTYPES[config.enc_dtype], _DTYPES[config.dec_dtype]
        # MACVO_Fast (enc fp16 / dec bf16, Config/Experiment/MACVO/MACVO_Fast.yaml:8-9) exists because half-precision tensor
        # cores are the fast path on the GPUs MAC-VO targets. The TF32 pipeline of this class (own kernels + TF32
        # cuDNN / cuBLAS) is ~4x closer to exact arithmetic than the
        # reference's own fp16 / bf16 run (flow 9e-4 vs 3.3e-3 of its scale, tests/test_gpu_pipeline.py::test_fast_config_*),
        # so half-precision configs are served by it unless `half_precision: native` asks for the literal dtypes.
        self.half_precision = getattr(config, "half_precision", "tf32")
        if self.half_precision == "tf32":
            enc = dec = torch.float32
        self.net = FlowFormerCovNet(sd, self.device, enc, dec, decoder_depth=config.decoder_depth)
        # the reference frontend enables TF32 tensor cores for the dense layers (Frontend.py:275-277)
        torch.backends.cuda.matmul.allow_tf32 = True
        torch.backends.cudnn.allow_tf32 = True
        torch.set_float32_matmul_precision("medium")
        self._score: ops.ScoreBuffers | None = None

    @property
    def provide_cov(self) -> tuple[bool, bool]:
        return True, True

    # ---- (a7) + fused (a8) scoring ---------------------------------------------------------------
    def _postprocess(self, est_flow, est_cov, bl_fx: float):
        H, W = est_flow.shape[-2:]
        if self._score is None or (self._score.h, self._score.w) != (H, W):
            self._score = ops.ScoreBuffers(H, W, self.device, int(getattr(self.config, "score_kernel_size", 7)))
        return ops.dense_postproc(est_flow, est_cov, bl_fx, self.config.enforce_positive_disparity, score=self._score)

    def _run(self, input_A, input_B, bl_fx: float):
        # input_A = [t2.L, t1.L], input_B = [t2.R, t2.L]: B[1] is A[0], which the feature encoder then sees once
        est_flow, est_cov = self.net.inference(input_A, input_B, shared=(0, 1))
        return self._postprocess(est_flow.float(), est_cov.float(), bl_fx)

    def _outputs(self, d: dict, clone: bool):
        c = (lambda t: t.clone() if t is not None else None) if clone else (lambda t: t)
        depth = IStereoDepth.Output(depth=c(d["depth"]), cov=c(d["depth_cov"]), disparity=c(d["disparity"]),
                                    disparity_uncertainty=c(d["disparity_uncertainty"]), mask=c(d["depth_mask"]))
        match = IMatcher.Output(flow=c(d["flow"]), cov=c(d["flow_cov"]), mask=None)
        # let the selector plugin reuse the fused scores instead of re-reading the covariance map
        self._score.generation += 1
        # (the token is keyed by buffer generation + map address; the covariance map must not be edited in place between
        # estimate_pair and select_point — inference tensors carry no version counter that could detect it)
        match._b200_score = (self._score, self._score.generation, match.cov.data_ptr())  # type: ignore[attr-defined]
        return depth, match

    @torch.inference_mode()
    def estimate_depth(self, frame: StereoData):
        A = frame.imageL.to(self.device, non_blocking=True)
        B = frame.imageR.to(self.device, non_blocking=True)
        est_flow, est_cov = self.net.inference(A, B)
        est_flow, est_cov = est_flow.float(), est_cov.float()
        # B = 1 call: reuse the pair kernel by duplicating the slot (slot 1 outputs are ignored)
        d = ops.dense_postproc(torch.cat([est_flow, est_flow]), torch.cat([est_cov, est_cov]),
                               frame.frame_baseline * frame.fx, self.config.enforce_positive_disparity, score=None)
        return IStereoDepth.Output(depth=d["depth"], cov=d["depth_cov"], disparity=d["disparity"],
                                   disparity_uncertainty=est_cov[0:1, :1], mask=d["depth_mask"])

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        spec = {
            "weight": lambda s: isinstance(s, str),
            "device": lambda s: isinstance(s, str) and "cuda" in s,
            "dec_dtype": lambda b: b in ("fp32", "fp16", "bf16"),
            "enc_dtype": lambda b: b in ("fp32", "fp16", "bf16"),
            "enforce_positive_disparity": lambda b: isinstance(b, bool),
            "decoder_depth": lambda v: isinstance(v, int),
        }
        # optional keys (the reference class has none of them): cuda_graph defaults to True, score_kernel_size to 7,
        # half_precision to "tf32" (how fp16 / bf16 enc_dtype / dec_dtype are served, see __init__)
        optional = {"cuda_graph": lambda b: isinstance(b, bool),
                    "half_precision": lambda v: v in ("tf32", "native"),
                    "score_kernel_size": lambda k: isinstance(k, int) and k % 2 == 1 and 1 <= k <= 15}
        if config is not None:
            spec.update({k: v for k, v in optional.items() if hasattr(config, k)})
        cls._enforce_config_spec(config, spec)


class B200_FlowFormerFrontend(_B200_GraphedPairFrontend):
    """The covariance-free frontend of the Vanilla ablation (Config/Experiment/MACVO/Ablation_Study/TartanAirv2_Vanilla.yaml):
    FrontendCompose of FlowFormerDepth + FlowFormerMatcher, which load the same plain FlowFormer checkpoint (fp32, decoder
    depth 12, configs/submission.py:32). One network serves both: `estimate_pair` is one B = 2 pass, graphed like
    B200_FlowFormerCovFrontend's, `estimate_depth` one eager B = 1 pass.

    Outputs as the reference's: depth / disparity (1,1,H,W) with disparity = |flow_x| and depth = (bl * fx) / disparity
    (StereoDepth.py:122-128), flow (1,2,H,W); every covariance, the disparity uncertainty and the masks are None.
    The TF32 flags are left as the process has them (the reference classes do not touch them), so the network runs its
    strict fp32 loop under torch's defaults and its TF32 loop when the caller allows TF32.

    config: weight (plain FlowFormer or FlowFormerCov checkpoint path, or "synthetic[:seed]"), device, cuda_graph (optional
    bool, default True)."""

    DECODER_DEPTH = 12

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_FlowFormerFrontend")
        self.net = FlowFormerCovNet(_load_weights(config.weight, covariance=False), self.device,
                                    decoder_depth=self.DECODER_DEPTH, covariance=False)

    @property
    def provide_cov(self) -> tuple[bool, bool]:
        return False, False

    def _run(self, input_A, input_B, bl_fx: float):
        est_flow, _ = self.net.inference(input_A, input_B, shared=(0, 1))
        return ops.dense_postproc(est_flow, None, bl_fx)

    def _outputs(self, d: dict, clone: bool):
        c = (lambda t: t.clone()) if clone else (lambda t: t)
        return (IStereoDepth.Output(depth=c(d["depth"]), disparity=c(d["disparity"])),
                IMatcher.Output(flow=c(d["flow"])))

    @torch.inference_mode()
    def estimate_depth(self, frame: StereoData):
        A = frame.imageL.to(self.device, non_blocking=True)
        B = frame.imageR.to(self.device, non_blocking=True)
        est_flow, _ = self.net.inference(A, B)
        d = ops.dense_postproc(est_flow, None, frame.frame_baseline * frame.fx)
        return IStereoDepth.Output(depth=d["depth"], disparity=d["disparity"])

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        spec = {
            "weight": lambda s: isinstance(s, str),
            "device": lambda s: isinstance(s, str) and "cuda" in s,
        }
        if config is not None and hasattr(config, "cuda_graph"):
            spec["cuda_graph"] = lambda b: isinstance(b, bool)
        cls._enforce_config_spec(config, spec)


# ================================================================================================
# Keypoint selectors
# ================================================================================================
class B200_CovAwareSelector_NoDepth(IKeypointSelector):
    """Bit-exact replacement of CovAwareSelector_NoDepth.select_point (KeypointSelector.py:362-407).
    One host round trip (the candidate count, needed for the CPU `torch.randperm`) instead of two."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_CovAwareSelector_NoDepth")
        self._score: ops.ScoreBuffers | None = None
        self._cand: ops.CandidateList | None = None

    @torch.inference_mode()
    def enqueue_candidates(self, frame, depth0_est, depth1_est, match_est) -> "ops.CandidateList":
        """Kernels only (median threshold, flags, ordered compaction) — no host synchronisation. Takes `select_point`'s
        arguments (the depth estimates are not read) so that callers drive either CovAware selector the same way."""
        if match_est is None or match_est.cov is None:
            raise ValueError("B200_CovAwareSelector_NoDepth needs match_est.cov (the reference falls back to a grid "
                             "selector here; compose it with GridSelector in the YAML if that is wanted)")
        cov = match_est.cov
        H, W = cov.shape[-2:]
        token = getattr(match_est, "_b200_score", None)
        score = None
        if token is not None:                              # scores fused into the frontend's post-processing pass
            sc, gen, ptr = token
            if (sc.generation == gen and ptr == cov.data_ptr()
                    and sc.ksize == self.config.kernel_size and (sc.h, sc.w) == (H, W)):
                score = sc
        if score is None:                                  # foreign frontend / modified map: score it ourselves
            if self._score is None or (self._score.h, self._score.w) != (H, W):
                self._score = ops.ScoreBuffers(H, W, self.device, self.config.kernel_size)
            score = self._score
            ops.score_only(cov.to(self.device), score)
        if self._cand is None or self._cand.idx.numel() != H * W:
            self._cand = ops.CandidateList(H, W, self.device)
        ops.select_candidates(score, self.config.mask_width, self.config.max_match_cov, match_est.mask, self._cand)
        return self._cand

    @torch.inference_mode()
    def select_point(self, frame, numPoint: int, depth0_est, depth1_est, match_est) -> torch.Tensor:
        return ops.sample_candidates(self.enqueue_candidates(frame, depth0_est, depth1_est, match_est), numPoint)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
            "mask_width": lambda m: isinstance(m, int) and m >= 0,
            "kernel_size": lambda k: isinstance(k, int) and k > 0 and (k % 2 == 1) and k <= 15,
            "max_match_cov": lambda c: isinstance(c, (int, float)) and c > 0.,
        })


class B200_CovAwareSelector(IKeypointSelector):
    """Bit-exact replacement of CovAwareSelector.select_point (KeypointSelector.py:260-334): the depth-aware
    selector of Paper_Reproduce.yaml (quality = (depth_cov0 + depth_cov1) * flow quality, depth and depth-cov gates)."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_CovAwareSelector")
        self._score: ops.ScoreBuffers | None = None
        self._cand: ops.CandidateList | None = None

    @torch.inference_mode()
    def enqueue_candidates(self, frame, depth0_est, depth1_est, match_est) -> "ops.CandidateList":
        """Kernels only (scores, median thresholds, flags, ordered compaction) — no host synchronisation."""
        assert depth0_est.cov is not None
        assert depth1_est.cov is not None
        if match_est is None or match_est.cov is None:
            raise ValueError("B200_CovAwareSelector needs match_est.cov")
        if self.config.max_depth == "auto":
            self.config.max_depth = frame.fx * frame.frame_baseline
        H, W = match_est.cov.shape[-2:]
        if self._score is None or (self._score.h, self._score.w) != (H, W):
            self._score = ops.ScoreBuffers(H, W, self.device, self.config.kernel_size)
            self._cand = ops.CandidateList(H, W, self.device)
        dev = self.device
        ops.score_depth_aware(match_est.cov.to(dev), depth0_est.cov.to(dev), depth1_est.cov.to(dev), self._score)
        ops.select_candidates_depth(self._score, depth0_est.depth.to(dev), depth1_est.depth.to(dev), depth0_est.cov.to(dev),
                                    self.config.mask_width, self.config.max_depth, self.config.max_depth_cov,
                                    self.config.max_match_cov, depth0_est.mask, match_est.mask, self._cand)
        return self._cand

    @torch.inference_mode()
    def select_point(self, frame, numPoint: int, depth0_est, depth1_est, match_est) -> torch.Tensor:
        return ops.sample_candidates(self.enqueue_candidates(frame, depth0_est, depth1_est, match_est), numPoint)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
            "mask_width": lambda m: isinstance(m, int) and m >= 0,
            "max_depth": lambda dist: (dist == "auto") or (isinstance(dist, (int, float)) and dist > 0.),
            "kernel_size": lambda k: isinstance(k, int) and k > 0 and (k % 2 == 1) and k <= 15,
            "max_depth_cov": lambda c: isinstance(c, (int, float)) and c > 0.,
            "max_match_cov": lambda c: isinstance(c, (int, float)) and c > 0.,
        })


class B200_RandomSelector(IKeypointSelector):
    """Replacement of RandomSelector.select_point (KeypointSelector.py:103-118), the selector of the CovOpt ablation:
    `numPoint` uniform (u, v) in [mask_width, size - mask_width), duplicates possible, drawn by the reference's two
    `torch.randint` calls (rows, then columns) on the configured CUDA device's generator — the same Philox stream, so the
    same keypoints from the same generator state. No candidate list and no host synchronisation."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_RandomSelector")

    def select_device(self, frame, numPoint: int) -> torch.Tensor:
        """(numPoint, 2) int64 on the device; kernels only (what the fused driver calls)"""
        mw = self.config.mask_width
        h_indices = torch.randint(mw, frame.height - mw, (numPoint, 1), device=self.device)
        w_indices = torch.randint(mw, frame.width - mw, (numPoint, 1), device=self.device)
        return torch.cat([w_indices, h_indices], dim=1)

    @torch.inference_mode()
    def select_point(self, frame, numPoint: int, depth0_est, depth1_est, match_est) -> torch.Tensor:
        return self.select_device(frame, numPoint)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {
            "mask_width": lambda m: isinstance(m, int) and m >= 0,
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
        })


class B200_MappingPointSelector(IKeypointSelector):
    """Bit-exact replacement of MappingPointSelector.select_point (KeypointSelector.py:87-100)."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self._cand: ops.CandidateList | None = None

    @torch.inference_mode()
    def enqueue_candidates(self, depth0_est) -> "ops.CandidateList":
        assert depth0_est.cov is not None
        H, W = depth0_est.depth.shape[-2:]
        if self._cand is None or self._cand.idx.numel() != H * W or self._cand.idx.device != depth0_est.depth.device:
            self._cand = ops.CandidateList(H, W, depth0_est.depth.device)
        ops.select_mapping_candidates(depth0_est.depth, depth0_est.cov, self.config.mask_width, self.config.max_depth,
                                      self.config.max_depth_cov, self._cand)
        return self._cand

    @torch.inference_mode()
    def select_point(self, frame, numPoint: int, depth0_est, depth1_est, match_est) -> torch.Tensor:
        return ops.sample_candidates(self.enqueue_candidates(depth0_est), numPoint)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {
            "max_depth": lambda v: isinstance(v, float),
            "max_depth_cov": lambda v: isinstance(v, float),
            "mask_width": lambda v: isinstance(v, int),
        })


# ================================================================================================
# Covariance model
# ================================================================================================
class B200_MatchCovariance(ICovariance2to3):
    """Replacement of MatchCovariance.estimate (Project2to3.py:124-182). Returns a CPU float64 (K,3,3)
    tensor like the reference (its `create_3x3_matrix` assembles the result on the CPU, and
    Odometry/MACVO.py multiplies it with CPU rotations) — filled by ONE device->host copy instead of nine."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_MatchCovariance")
        self.last_status: torch.Tensor | None = None
        self._status_host: torch.Tensor | None = None

    def estimate_device(self, frame, kp, depth_est, depth_cov, flow_cov, want_point: bool = False):
        """Device-resident variant: (cov (K,3,3) fp64 CUDA, point (K,3) fp32 CUDA or None).

        flow_cov may be ANY (K,3) view — Odometry/MACVO.py:231-232 passes `retrieve_pixels(kp, match.cov).T`, a
        transposed view of a (3,K) tensor — the kernel addresses it through its strides, so the reference's in-place
        clamp (Project2to3.py:130-133) lands in the caller's storage (that tensor later becomes `pixel2_uv_cov`).
        A tensor on another device / of another dtype is staged and copied back after the clamp."""
        fc = flow_cov
        staged = None
        if fc is not None and not (fc.is_cuda and fc.device == self.device and fc.dtype == torch.float32):
            staged = fc.to(device=self.device, dtype=torch.float32).contiguous()
            fc = staged
        cov, pt, status = ops.match_covariance(
            kp.to(self.device), depth_est.depth, fc, frame.fx, frame.fy, frame.cx, frame.cy,
            kernel_size=self.config.kernel_size, min_flow_cov=self.config.min_flow_cov,
            min_depth_cov=self.config.min_depth_cov, match_cov_default=self.config.match_cov_default,
            want_point=want_point, depth_cov=depth_cov.to(self.device) if (fc is None and depth_cov is not None) else None)
        if staged is not None:
            flow_cov.copy_(staged)
        self.last_status = status
        return cov, pt

    @torch.inference_mode()
    def estimate(self, frame, kp, depth_est, depth_cov, flow_cov) -> torch.Tensor:
        cov, _ = self.estimate_device(frame, kp, depth_est, depth_cov, flow_cov)
        return self.download(cov)

    def download(self, cov: torch.Tensor) -> torch.Tensor:
        """the CPU float64 copy of `estimate_device`'s covariances (or of a modified version of them); raises the
        reference's IndexError when the last estimate's depth patch left the image"""
        if self._status_host is None:
            self._status_host = torch.zeros((1,), dtype=self.last_status.dtype).pin_memory()
        self._status_host.copy_(self.last_status, non_blocking=True)      # rides in front of the blocking copy below
        out = cov.cpu()                                                     # ONE synchronising device->host copy
        if int(self._status_host[0]) != 0:
            raise IndexError("MatchCovariance: a keypoint's depth patch leaves the image")
        return out

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
            "kernel_size": lambda k: isinstance(k, int) and k % 2 == 1 and 1 <= k <= 31,
            "match_cov_default": lambda c: isinstance(c, (int, float)) and c > 0,
            "min_depth_cov": lambda c: isinstance(c, (int, float)) and c > 0,
            "min_flow_cov": lambda c: isinstance(c, (int, float)) and c > 0,
        })


class B200_NoCovariance(ICovariance2to3):
    """Replacement of NoCovariance (Project2to3.py:48-57), the covariance model of the CovKP ablation: identity
    covariances. Like the reference it reads no depth patch and leaves `flow_cov` alone, so the MatchObs column
    `pixel2_uv_cov` keeps the network's unclamped values. config: none."""

    def estimate(self, frame, kp, depth_est, depth_cov, flow_cov) -> torch.Tensor:
        return torch.eye(3).unsqueeze(0).repeat(kp.size(0), 1, 1).double()       # CPU float64, as the reference

    def estimate_device(self, frame, kp, depth_est, depth_cov, flow_cov, want_point: bool = False):
        """(identity (K,3,3) float64 on the keypoints' / depth map's device, None). The fused driver does not call this:
        observe_pack and its mapping branch build the identity themselves."""
        if want_point:
            raise ValueError("B200_NoCovariance.estimate_device computes no points")
        dev = kp.device if kp.is_cuda else depth_est.depth.device
        return torch.eye(3, dtype=torch.float64, device=dev).repeat(kp.size(0), 1, 1), None

    def download(self, cov: torch.Tensor) -> torch.Tensor:
        return cov.cpu()

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        return


class _B200_CovModifier(ICovariance2to3):
    """A modifier wrapping another B200 covariance model (config: `type` / `args` of the nested model), applied on the
    device by `macvo_cov_modify`."""
    OP = ""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        _require_b200_cov(config.type, type(self).__name__)
        self.submodule = ICovariance2to3.instantiate(config.type, config.args)

    def estimate_device(self, frame, kp, depth_est, depth_cov, flow_cov, want_point: bool = False):
        cov, pt = self.submodule.estimate_device(frame, kp, depth_est, depth_cov, flow_cov, want_point=want_point)
        return ops.cov_modify(cov, [self.OP]), pt

    @torch.inference_mode()
    def estimate(self, frame, kp, depth_est, depth_cov, flow_cov) -> torch.Tensor:
        cov, _ = self.estimate_device(frame, kp, depth_est, depth_cov, flow_cov)
        return self.download(cov)

    def download(self, cov: torch.Tensor) -> torch.Tensor:
        return self.submodule.download(cov)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        assert config is not None
        _require_b200_cov(getattr(config, "type", None), cls.__name__)
        ICovariance2to3.is_valid_config(config)


class B200_Modifier_Diagonalize(_B200_CovModifier):
    """Replacement of Modifier_Diagonalize (Project2to3.py:281-302): the nested model's covariances with their six
    off-diagonal entries set to 0 (a NaN / Inf there disappears before CovarianceSanityFilter sees it)."""
    OP = "diagonalize"


class B200_Modifier_Normalize(_B200_CovModifier):
    """Replacement of Modifier_Normalize (Project2to3.py:305-323): each covariance divided by its OWN determinant (3x3 LU
    with partial pivoting in float64; det 0 gives +-Inf / NaN, which the sanity filter drops, a negative det flips the
    matrix's sign)."""
    OP = "normalize"


def _require_b200_cov(name, who: str) -> None:
    try:
        cls = ICovariance2to3.get_class(name)
    except (KeyError, TypeError):
        cls = None
    if not (isinstance(cls, type) and issubclass(cls, (B200_MatchCovariance, B200_NoCovariance, _B200_CovModifier))):
        raise ValueError(f"{who}: the nested covariance model must be a B200 model (B200_MatchCovariance, "
                         f"B200_NoCovariance or another B200 modifier), got {name!r}")


def cov_spec(cov_model) -> tuple[ICovariance2to3, list[str], dict | None]:
    """(base model, modifiers innermost first, the base model's kernel parameters or None for B200_NoCovariance) of a
    B200 covariance model: what `macvo_observe_pack` and the fused driver's mapping branch need."""
    ops_: list[str] = []
    m = cov_model
    while isinstance(m, _B200_CovModifier):
        ops_.insert(0, m.OP)
        m = m.submodule
    if isinstance(m, B200_NoCovariance):
        return m, ops_, None
    if isinstance(m, B200_MatchCovariance):
        c = m.config
        return m, ops_, dict(kernel_size=c.kernel_size, min_flow_cov=c.min_flow_cov, min_depth_cov=c.min_depth_cov)
    raise ValueError(f"{type(m).__name__} has no device implementation in the fused driver")


# ================================================================================================
# Observation filter
# ================================================================================================
class B200_CovarianceSanityFilter(IObservationFilter):
    """Replacement of CovarianceSanityFilter (Module/OutlierFilter.py:91-100): drops observations whose 3x3 covariances
    hold a NaN / Inf. Device-resident covariances (a caller that keeps MatchObs on the GPU, e.g.
    `pipeline.FusedTwoFrameOdometry`, where the same test runs inside `observe_kernel`) go through
    `macvo_cov_sanity_filter`; the CPU float64 tensors `Odometry/MACVO.py:246-270` builds are tested where they live —
    uploading 2 x K x 72 bytes to test them would cost more than the test."""

    @property
    def required_keys(self) -> set:
        return {"obs1_covTc", "obs2_covTc"}

    @torch.inference_mode()
    def filter(self, values, device: torch.device) -> torch.Tensor:
        c1, c2 = values.data["obs1_covTc"], values.data["obs2_covTc"]
        c1 = c1.tensor if hasattr(c1, "tensor") and not isinstance(c1, torch.Tensor) else c1
        c2 = c2.tensor if hasattr(c2, "tensor") and not isinstance(c2, torch.Tensor) else c2
        if c1.is_cuda and c2.is_cuda and c1.dtype == torch.float64 and c2.dtype == torch.float64:
            return ops.cov_sanity_filter(c1, c2).to(device)
        bad = c1.isnan().any(dim=(-1, -2)) | c1.isinf().any(dim=(-1, -2)) | c2.isnan().any(dim=(-1, -2)) | c2.isinf().any(dim=(-1, -2))
        return (~bad).to(device)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        return

    def observe_ext(self) -> dict:
        """what `macvo_observe_pack` needs to run this filter: nothing, observe_kernel always applies it"""
        return {}


def _column(values, key: str) -> torch.Tensor:
    t = values.data[key]
    return t.tensor if hasattr(t, "tensor") and not isinstance(t, torch.Tensor) else t


class B200_SimpleDepthFilter(IObservationFilter):
    """Replacement of SimpleDepthFilter (Module/OutlierFilter.py:103-124): drops observations whose depth lies below
    min_depth or above max_depth on either frame (a NaN depth passes). `max_depth: auto` becomes fx * baseline in
    `set_meta`. On the device the test runs inside observe_kernel (`observe_ext`)."""

    def set_meta(self, meta) -> None:
        if self.config.max_depth == "auto":
            self.config.max_depth = meta.fx * meta.frame_baseline

    @property
    def required_keys(self) -> set:
        return {"pixel1_d", "pixel2_d"}

    def filter(self, values, device: torch.device) -> torch.Tensor:
        d1, d2 = _column(values, "pixel1_d"), _column(values, "pixel2_d")
        lo, hi = self.config.min_depth, self.config.max_depth
        return (~((d1 < lo) | (d1 > hi) | (d2 < lo) | (d2 > hi)).squeeze(-1)).to(device)

    def observe_ext(self) -> dict:
        if self.config.max_depth == "auto":
            raise ValueError("B200_SimpleDepthFilter: max_depth 'auto' is resolved by set_meta(); call it first")
        # the reference compares fp32 tensors with python floats: the thresholds act rounded to fp32
        return {"simple_depth": True, "min_depth": float(self.config.min_depth), "max_depth": float(self.config.max_depth)}

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        assert config is not None
        if isinstance(config.max_depth, (float, int)):
            assert config.max_depth > config.min_depth
        cls._enforce_config_spec(config, {
            "min_depth": lambda dist: isinstance(dist, (int, float)) and dist > 0.,
            "max_depth": lambda dist: (dist == "auto") or (isinstance(dist, (int, float)) and dist > 0.),
        })


class B200_LikelyFrontOfCamFilter(IObservationFilter):
    """Replacement of LikelyFrontOfCamFilter (Module/OutlierFilter.py:127-141): keeps observations with
    d - 2 sqrt(d_cov) > 0 on both frames; passes everything when any pixel1_d_cov is the -1 placeholder of a frontend
    without depth covariance. On the device: observe_kernel / pack_kernel (`observe_ext`)."""

    @property
    def required_keys(self) -> set:
        return {"pixel1_d", "pixel1_d_cov", "pixel2_d", "pixel2_d_cov"}

    def filter(self, values, device: torch.device) -> torch.Tensor:
        d1, c1 = _column(values, "pixel1_d"), _column(values, "pixel1_d_cov")
        d2, c2 = _column(values, "pixel2_d"), _column(values, "pixel2_d_cov")
        if (c1 == -1).any():
            return torch.ones((d1.shape[0],), dtype=torch.bool, device=device)
        return (((d1 - (c1.sqrt() * 2)) > 0.) & ((d2 - (c2.sqrt() * 2)) > 0.)).squeeze(-1).to(device)

    def observe_ext(self) -> dict:
        return {"front_of_cam": True}

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        return


class B200_FilterCompose(IObservationFilter):
    """Replacement of FilterCompose (Module/OutlierFilter.py:44-75): the AND of its filters' masks. `filter_args` may
    name B200 filters only. The fused driver runs the whole chain inside `macvo_observe_pack` (`observe_ext`)."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.filters = [IObservationFilter.instantiate(a.type, a.args) for a in self.config.filter_args]

    @property
    def required_keys(self) -> set:
        return {k for f in self.filters for k in f.required_keys}

    def set_meta(self, meta) -> None:
        for f in self.filters:
            f.set_meta(meta)

    def filter(self, values, device: torch.device) -> torch.Tensor:
        mask = torch.ones((len(values),), dtype=torch.bool, device=device)
        for f in self.filters:
            mask = torch.logical_and(mask, f.filter(values, device))
        return mask

    def observe_ext(self) -> dict:
        ext: dict = {}
        for f in self.filters:
            if not hasattr(f, "observe_ext"):
                raise ValueError(f"B200_FilterCompose: {type(f).__name__} has no device implementation")
            ext.update(f.observe_ext())
        return ext

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        assert config is not None
        assert isinstance(config.filter_args, list)
        for filter_arg in config.filter_args:
            IObservationFilter.is_valid_config(filter_arg)


def check_sanity_chain(outlier_filter, covariance_finite: bool = False) -> None:
    """The device observation path always applies CovarianceSanityFilter, so the outlier filter must contain
    B200_CovarianceSanityFilter; raises otherwise. covariance_finite: the covariance model only produces finite
    covariances (B200_NoCovariance: identities, finite under any modifier), so the always-on filter cannot drop a row and
    a chain without it (the Vanilla ablation's [SimpleDepthFilter]) means the same thing on the device."""
    if outlier_filter is None or covariance_finite:
        return
    chain = outlier_filter.filters if isinstance(outlier_filter, B200_FilterCompose) else [outlier_filter]
    if not any(isinstance(f, B200_CovarianceSanityFilter) for f in chain):
        raise ValueError("the device observation path always applies CovarianceSanityFilter: the outlier filter must "
                         "contain B200_CovarianceSanityFilter")


def observe_ext(outlier_filter, covariance_finite: bool = False) -> dict | None:
    """`macvo_observe_pack`'s extension for an outlier filter (None: CovarianceSanityFilter alone, which observe_kernel
    always applies). Raises for a filter the device path cannot run, or a chain without the sanity filter (unless
    `covariance_finite`, see `check_sanity_chain`)."""
    if outlier_filter is None:
        return None
    check_sanity_chain(outlier_filter, covariance_finite)
    if not hasattr(outlier_filter, "observe_ext"):
        raise ValueError(f"{type(outlier_filter).__name__} has no device implementation")
    return outlier_filter.observe_ext()


# ================================================================================================
# Map post-processing
# ================================================================================================
class B200_MotionInterpolate(IMapProcessor):
    """Replacement of MotionInterpolate.elaborate_map (Module/MapProcessor.py:52-79), run once at `MACVO.terminate()`:
    relative motions, se3-linear interpolation of the `need_interp` ones, re-integration with quaternion renormalisation —
    one kernel launch (csrc/motion_interp.cu) instead of a Python loop of F pypose compositions. config: {device}."""

    def __init__(self, config: SimpleNamespace | None):
        super().__init__(config)
        self.device = _require_cuda(getattr(config, "device", "cuda"), "B200_MotionInterpolate")

    @torch.inference_mode()
    def elaborate_map(self, frames):
        pose_store, flag_store = frames.data["pose"], frames.data["need_interp"]
        poses = pose_store.tensor if hasattr(pose_store, "tensor") and not isinstance(pose_store, torch.Tensor) else pose_store
        flags = flag_store.tensor if hasattr(flag_store, "tensor") and not isinstance(flag_store, torch.Tensor) else flag_store
        n = poses.shape[0]
        bad = flags[1:].bool().clone()
        bad[:2] = False
        bad[-2:] = False
        interp_idx = torch.nonzero(bad).flatten()
        if n >= 2:
            dev_poses = poses.to(device=self.device, dtype=torch.float32).contiguous()
            ops.motion_interpolate_(dev_poses, flags.to(self.device))
            frames.data["pose"][1:] = dev_poses[1:].to(poses.device)
        return frames, interp_idx

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {"device": lambda d: isinstance(d, str) and "cuda" in d})


# ================================================================================================
# Two-frame pose-graph optimisation
# ================================================================================================
@dataclass
class PGOInput:
    """What Analytic_ReprojDisp_TwoFramePGO reads out of GraphInput (Graphs.py:76-134), as plain tensors."""
    pos_Tw: torch.Tensor        # (K,3)  NED world points
    kp2_uv: torch.Tensor        # (K,2)
    kp2_disp: torch.Tensor      # (K,) or (K,1)
    uv_cov: torch.Tensor        # (K,3)  sigma_uu, sigma_vv, sigma_uv
    disp_cov: torch.Tensor      # (K,) or (K,1)
    K: torch.Tensor             # (3,3)
    baseline: float
    init_pose: torch.Tensor     # (7,) [t, q_xyzw]
    frame_idx: torch.Tensor | None = None
    from_idx: torch.Tensor | None = None
    # graph type "icp" (Graphs.py:33-73) additionally reads:
    kp2_d: torch.Tensor | None = None       # (K,) or (K,1) pixel2_d
    obs_cov: torch.Tensor | None = None     # (K,3,3) float64 obs2_covTc
    pts_cov: torch.Tensor | None = None     # (K,3,3) float64 cov_Tw


@dataclass
class PGOOutput:
    motion: torch.Tensor        # (1,7) float64 on the device (synchronise by reading it)
    frame_idx: torch.Tensor | None
    from_idx: torch.Tensor | None
    stats: torch.Tensor | None = None


def solve_two_frame_pgo(inp: PGOInput, device, cluster: int = 0, graph_type: str = "disp") -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 map values -> float64 (the reference's `.to(dtype=torch.double)`, Optimizer.py:85) -> one launch."""
    f64 = lambda t: t.detach().to(device=device, dtype=torch.float64, non_blocking=True).contiguous()
    K = inp.K.detach().double().cpu()
    intr = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]),
            float(torch.as_tensor(inp.baseline, dtype=torch.float32).double().reshape(-1)[0]))
    if graph_type == "disp":
        return ops.pgo_solve(f64(inp.pos_Tw), f64(inp.kp2_uv), f64(inp.kp2_disp).reshape(-1), f64(inp.uv_cov),
                             f64(inp.disp_cov).reshape(-1), intr, f64(inp.init_pose).reshape(7), cluster=cluster)
    if graph_type == "reproj":
        return ops.pgo_solve_graph("reproj", f64(inp.pos_Tw), intr, f64(inp.init_pose).reshape(7), kp2_uv=f64(inp.kp2_uv),
                                   uv_cov=f64(inp.uv_cov), cluster=cluster)
    # icp: points_Tc = pixel2point_NED(pixel2_uv, pixel2_d, K) is a registered fp32 buffer of the reference graph (Graphs.py:49-51)
    uv = inp.kp2_uv.detach().to(device=device, dtype=torch.float32)
    d = inp.kp2_d.detach().to(device=device, dtype=torch.float32).reshape(-1)
    Kf = inp.K.detach().to(device=device, dtype=torch.float32)
    pc = torch.stack([d, (uv[:, 0] - Kf[0, 2]) / Kf[0, 0] * d, (uv[:, 1] - Kf[1, 2]) / Kf[1, 1] * d], dim=-1)
    return ops.pgo_solve_graph("icp", f64(inp.pos_Tw), intr, f64(inp.init_pose).reshape(7), pc_obs=pc.double().contiguous(),
                               obs_cov=f64(inp.obs_cov), pts_cov=f64(inp.pts_cov), cluster=cluster)


class B200_TwoFrame_PGO(_PGOBase):
    """Replacement of TwoFrame_PGO (graph types "disp" / "reproj" / "icp", analytic Jacobians): the whole Levenberg-Marquardt loop is
    one persistent kernel launch; `start_optimize` returns immediately and `write_map` synchronises on the
    result, which preserves the frontend / optimiser overlap MAC-VO gets from its spawned CPU process."""

    @staticmethod
    def init_context(config) -> dict:
        gt = getattr(config, "graph_type", "disp")
        if gt not in ("disp", "reproj", "icp") or getattr(config, "autodiff", False):
            raise ValueError("B200_TwoFrame_PGO implements graph_type 'disp' / 'reproj' / 'icp' with the analytic Jacobians "
                             "(autodiff: false)")
        return {"device": _require_cuda(config.device, "B200_TwoFrame_PGO"), "cluster": int(getattr(config, "cluster", 0)),
                "graph_type": gt}

    @staticmethod
    def _optimize(context: dict, graph_data):
        if isinstance(graph_data, PGOInput):
            inp = graph_data
        else:   # MAC-VO's GraphInput (Graphs.py:11-22)
            obs, pts = graph_data.observations.data, graph_data.points.data
            inp = PGOInput(pos_Tw=pts["pos_Tw"], kp2_uv=obs["pixel2_uv"], kp2_disp=obs["pixel2_disp"],
                           uv_cov=obs["pixel2_uv_cov"], disp_cov=obs["pixel2_disp_cov"], K=graph_data.images_intrinsic,
                           baseline=graph_data.baseline, init_pose=torch.as_tensor(graph_data.init_motion).reshape(-1)[:7],
                           frame_idx=graph_data.frame_idx, from_idx=graph_data.from_idx)
            if context.get("graph_type") == "icp":
                inp.kp2_d, inp.obs_cov, inp.pts_cov = obs["pixel2_d"], obs["obs2_covTc"], pts["cov_Tw"]
        pose, stats = solve_two_frame_pgo(inp, context["device"], context["cluster"], context.get("graph_type", "disp"))
        if _REF and not isinstance(graph_data, PGOInput):
            return context, _RefGraphOutput(motion=pose.reshape(1, 7), frame_idx=inp.frame_idx, from_idx=inp.from_idx)
        return context, PGOOutput(motion=pose.reshape(1, 7), frame_idx=inp.frame_idx, from_idx=inp.from_idx, stats=stats)

    if not _REF:
        @classmethod
        def is_valid_config(cls, config: SimpleNamespace | None) -> None:
            cls._enforce_config_spec(config, {
                "graph_type": lambda s: s in {"icp", "reproj", "disp"},
                "device": lambda v: isinstance(v, str) and "cuda" in v,
                "vectorize": lambda b: isinstance(b, bool),
                "parallel": lambda b: b is False,
                "autodiff": lambda b: isinstance(b, bool),
            })


# ================================================================================================
# Motion model
# ================================================================================================
class B200_TartanMotionNet(IMotionModel):
    """Replacement of TartanMotionNet (Module/MotionModel.py:89-116) that builds only the pose network `predict` runs
    (no PWC-Net, no stereo net, no cupy / cv2). Everything from the flow and depth maps up to fc1 is one CUDA graph,
    captured on the first prediction and replayed after; the head kernel (fc2 / fc3, pose composition) runs after the
    replay because it reads the previous pose.

    config: weight (checkpoint path — only its `module.flowPoseNet.*` tensors are used — or "synthetic[:seed]"), device.
    `predict` returns identity on its first call, then prev_pose @ se3(motion).Exp() on the device: a pp.SE3 when MAC-VO
    (and pypose) is importable, else a (7,) tensor [t, q_xyzw]."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_TartanMotionNet")
        w = config.weight
        if isinstance(w, str) and w.startswith("synthetic"):
            sd = posenet.synthetic_posenet_state_dict(int(w.split(":")[1]) if ":" in w else 0)
        else:
            sd = posenet.load_checkpoint(w)
        self.net = posenet.PoseNet(sd, self.device)
        self.prev_pose: torch.Tensor | None = None       # (7,) fp32 on the device
        self.motion = torch.zeros((6,), dtype=torch.float32, device=self.device)   # last predicted se3 motion
        self._replay = None
        self._static: dict = {}

    @staticmethod
    def _camera(frame):
        meta = getattr(frame, "stereo", frame)
        return meta, (float(meta.fx), float(meta.fy), float(meta.cx), float(meta.cy)), meta.frame_baseline * meta.fx

    @torch.inference_mode()
    def enqueue(self, frame, flow: torch.Tensor, depth: torch.Tensor) -> torch.Tensor:
        """Replay the graph (input builder .. fc1) for this frame's flow (1,2,H,W) and depth (1,1,H,W); returns the graph's
        static fc1 output (256,), valid until the next call. Kernels only, no host synchronisation."""
        meta, K, bl_fx = self._camera(frame)
        st = self._static
        if self._replay is not None:
            assert tuple(flow.shape) == st["flow"].shape and tuple(depth.shape) == st["depth"].shape, \
                f"map shape changed since the CUDA graph was captured: {tuple(flow.shape)} != {tuple(st['flow'].shape)}"
            assert K == st["K"], "camera intrinsics changed since the CUDA graph was captured"
            assert bl_fx == st["bl_fx"], "camera baseline * fx changed since the CUDA graph was captured"
            st["flow"].copy_(flow, non_blocking=True)
            st["depth"].copy_(depth, non_blocking=True)
            return self._replay()
        sflow = flow.to(device=self.device, dtype=torch.float32).contiguous().clone()
        sdepth = depth.to(device=self.device, dtype=torch.float32).contiguous().clone()
        inp = torch.empty((1, 5, ops.POSENET_H, ops.POSENET_W), dtype=torch.float32, device=self.device)
        inp[:, 3:5] = posenet.intrinsic_layer(meta.height, meta.width, *K[:2], *K[2:], self.device)

        def run():
            ops.posenet_input(sflow, sdepth, bl_fx, inp)
            return self.net.body(inp)
        self._static = {"flow": sflow, "depth": sdepth, "inp": inp, "K": K, "bl_fx": bl_fx}
        self._replay = self._capture(run)
        return self._replay()

    def _capture(self, run):
        """capture `run` (input builder .. fc1) as a CUDA graph; returns a callable that replays it and returns fc1"""
        side = torch.cuda.Stream(self.device)      # warm-up (cuDNN algorithm choice) outside the capture
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES[0]
        with torch.cuda.graph(graph):
            fc1 = run()
        launches = ops.LAUNCHES[0] - n0

        def replay():
            graph.replay()
            ops.LAUNCHES[0] += launches
            return fc1
        return replay

    def head(self, fc1: torch.Tensor, prev_pose: torch.Tensor, next_pose: torch.Tensor) -> None:
        """fc2 / fc3 / pose_norm of fc1 -> self.motion, and next_pose (7,) float64 = prev_pose (7,) float64 @ Exp(motion)"""
        ops.posenet_head(fc1, self.net.head_blob, prev_pose, self.motion, next_pose)

    @staticmethod
    def _tensor(pose) -> torch.Tensor:
        return (pose.tensor() if hasattr(pose, "ltype") else pose).reshape(-1)[:7]

    def _wrap(self, pose: torch.Tensor):
        return _pp.SE3(pose) if _pp is not None else pose

    @torch.inference_mode()
    def predict(self, frame, flow: torch.Tensor | None, depth: torch.Tensor | None):
        if self.prev_pose is None:
            self.prev_pose = torch.tensor([0., 0., 0., 0., 0., 0., 1.], device=self.device)
            return self._wrap(self.prev_pose.clone())
        assert flow is not None and depth is not None, "Motion model requires flow and depth to predict motion"
        fc1 = self.enqueue(frame, flow, depth)
        nxt = torch.empty((7,), dtype=torch.float64, device=self.device)
        self.head(fc1, self.prev_pose.double(), nxt)
        self.prev_pose = nxt.float()
        return self._wrap(self.prev_pose.clone())

    def update(self, pose) -> None:
        self.prev_pose = self._tensor(pose).detach().to(device=self.device, dtype=torch.float32)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        cls._enforce_config_spec(config, {
            "weight": lambda f: isinstance(f, str),
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
        })


# ================================================================================================
# Matcher
# ================================================================================================
class B200_TartanVOMatcher(IMatcher):
    """Replacement of TartanVOMatcher (Module/Frontend/Matching.py:199-230), the optical flow of the TartanVO baseline
    (Config/Experiment/Baseline/TartanVO/TartanVOStereo.yaml): TartanVO's PWC-Net (pwcnet.PWCFlowNet) with its warp +
    correlation in macvo_pwc_warp_corr and its convolutions on cuDNN; no cupy, cv2 or host round trip.

    config: weight (checkpoint path — only its `module.flowNet.*` tensors are used — or "synthetic[:seed]"), device (CUDA),
    optional cuda_graph (default true: crop, network and output shaping are captured as one CUDA graph on the first call
    and replayed after; the image shape must then stay the same).

    `forward` returns what the reference returns (TartanStereoVOMatch.inference, StereoVO_Interface.py:124-151, and
    Matching.py:213-223), as fresh tensors on config.device:
      * flow (1,2,H,W) fp32: both left images centre-cropped to (H//64*64, W//64*64), raw (not normalised), the network's
        flow2 / 0.05, nearest-upsampled x4 and NaN-padded to the frame size;
      * mask (1,1,h64,w64) bool, built like the reference's from the *cropped* flow before padding: True on
        [ph:-ph, pw:-pw] with ph, pw the crop margins — all False when H or W is a multiple of 64 (INTEGRATION.md);
      * a batch other than 1, or an odd total margin, raises AssertionError like the reference."""

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_TartanVOMatcher")
        w = config.weight
        if isinstance(w, str) and w.startswith("synthetic"):
            sd = pwcnet.synthetic_pwc_state_dict(int(w.split(":")[1]) if ":" in w else 0)
        else:
            sd = pwcnet.load_checkpoint(w)
        self.net = pwcnet.PWCFlowNet(sd, self.device)
        self.use_graph = bool(getattr(config, "cuda_graph", True))
        self._replay = None
        self._static: dict = {}

    @property
    def provide_cov(self) -> bool:
        return False

    @staticmethod
    def geometry(H: int, W: int) -> tuple[tuple[int, int], tuple[int, int]]:
        """((crop margin y, x), (h64, w64)) of getCropMargin (StereoVO_Interface.py:107-115), checked like padTo"""
        h64, w64 = H // 64 * 64, W // 64 * 64
        if h64 == 0 or w64 == 0:
            raise ValueError(f"B200_TartanVOMatcher: a {H}x{W} image is smaller than PWC-Net's 64x64 input granule")
        for size, crop, dim in ((H, h64, -2), (W, w64, -1)):
            assert (size - crop) % 2 == 0, \
                f"Can only handle even padding. Target_size={size}, Actual_size={crop} on dim {dim}."
        return ((H - h64) // 2, (W - w64) // 2), (h64, w64)

    def _run(self, images: torch.Tensor, flow_out: torch.Tensor, margin, crop) -> None:
        """images (2,3,H,W) -> flow_out (1,2,H,W): crop, network, / 0.05, nearest x4 into the NaN-padded frame"""
        (my, mx), (h64, w64) = margin, crop
        flow2 = self.net.flow2(images[:, :, my:my + h64, mx:mx + w64].contiguous())
        up = (flow2 / pwcnet.FLOW_NORM).repeat_interleave(4, dim=-2).repeat_interleave(4, dim=-1)
        flow_out[:, :, my:my + h64, mx:mx + w64].copy_(up)

    def _capture(self, run):
        """capture `run` as a CUDA graph (after a warm-up run outside the capture, for cuDNN's algorithm choice); returns a
        callable that replays it"""
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES[0]
        with torch.cuda.graph(graph):
            run()
        launches = ops.LAUNCHES[0] - n0

        def replay():
            graph.replay()
            ops.LAUNCHES[0] += launches
        return replay

    def forward(self, frame_t1: StereoData, frame_t2: StereoData) -> IMatcher.Output:
        img1, img2 = frame_t1.imageL, frame_t2.imageL
        assert img1.size(0) == 1 and img2.size(0) == 1, "The interface will not handle batch dimension correctly."
        H, W = img1.shape[-2:]
        assert tuple(img2.shape[-2:]) == (H, W), "both frames must have the same image size"
        st = self._static
        if self._replay is not None:
            assert (H, W) == st["shape"], f"image shape changed since the CUDA graph was captured: {(H, W)} != {st['shape']}"
        else:
            margin, crop = self.geometry(H, W)
            mask = torch.zeros((1, 1) + crop, dtype=torch.bool, device=self.device)
            ph, pw = margin                              # (frame size - flow size) // 2 of Matching.py:217-218
            mask[..., ph:-ph, pw:-pw] = True             # the reference's slice: empty when a margin is 0
            st = self._static = {"shape": (H, W), "margin": margin, "crop": crop, "mask": mask,
                                 "images": torch.empty((2, 3, H, W), dtype=torch.float32, device=self.device),
                                 "flow": torch.full((1, 2, H, W), float("nan"), dtype=torch.float32, device=self.device)}
        st["images"][0:1].copy_(img1, non_blocking=True)
        st["images"][1:2].copy_(img2, non_blocking=True)
        run = lambda: self._run(st["images"], st["flow"], st["margin"], st["crop"])
        # deterministic cuDNN algorithms (the transposed convolutions would otherwise be free to accumulate with atomics), so
        # that a graph replay, the first call and cuda_graph: false give the same bits; TF32 and the other flags as they are
        with torch.backends.cudnn.flags(enabled=torch.backends.cudnn.enabled, benchmark=torch.backends.cudnn.benchmark,
                                        benchmark_limit=torch.backends.cudnn.benchmark_limit, deterministic=True,
                                        allow_tf32=torch.backends.cudnn.allow_tf32):
            if not self.use_graph:
                run()
            elif self._replay is None:
                self._replay = self._capture(run)
                self._replay()
            else:
                self._replay()
        return IMatcher.Output(flow=st["flow"].clone(), mask=st["mask"].clone())

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        spec = {
            "weight": lambda f: isinstance(f, str),
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
        }
        if config is not None and "cuda_graph" in vars(config):
            spec["cuda_graph"] = lambda b: isinstance(b, bool)
        cls._enforce_config_spec(config, spec)



# ================================================================================================
# Stereo depth
# ================================================================================================
class B200_TartanVODepth(IStereoDepth):
    """Replacement of TartanVODepth (Module/Frontend/StereoDepth.py:186-229), the stereo depth and covariance of the TartanVO
    baseline (Config/Experiment/Baseline/TartanVO/TartanVOStereo.yaml): StereoCovNet(exp=False, decoder="hourglass")
    (stereonet.StereoCovNetDevice) with its convolutions on cuDNN and both full-resolution heads plus the depth conversion
    in macvo_stereo_head.

    config: weight (a TartanVO_depth_cov.pth-style checkpoint, `module.` prefix optional, or "synthetic[:seed]"), device
    (CUDA), cov_mode ("Est" or "None"), optional cuda_graph (default true: crop, normalisation, network and heads are
    captured as one CUDA graph per image shape on the first call and replayed after; the image shape and baseline * fx
    must then stay the same).

    `estimate` returns what the reference returns, as fresh tensors on config.device: depth (1,1,H,W) and, under "Est", cov
    (the depth variance, (1,1,H,W)), computed on the centre crop (H//64*64, W//64*64) and NaN outside it. Under "None" the
    covariance decoder is not run at all (the reference computes it and discards it; the depth is the same).
    The heads run in macvo_stereo_head when torch.backends.cudnn.allow_tf32 is set (torch's default, under which cuDNN runs
    the reference's deconvolution in TF32 too), else as torch ops; the flag is read, never changed."""

    MEAN = stereonet.IMG_MEAN
    STD = stereonet.IMG_STD

    def __init__(self, config: SimpleNamespace):
        super().__init__(config)
        self.device = _require_cuda(config.device, "B200_TartanVODepth")
        w = config.weight
        if isinstance(w, str) and w.startswith("synthetic"):
            sd = stereonet.synthetic_stereo_state_dict(int(w.split(":")[1]) if ":" in w else 0)
        else:
            sd = stereonet.load_checkpoint(w)
        self.net = stereonet.StereoCovNetDevice(sd, self.device)
        self.est_cov = config.cov_mode == "Est"
        self.use_graph = bool(getattr(config, "cuda_graph", True))
        self._mean = torch.tensor(self.MEAN, dtype=torch.float32, device=self.device).view(1, 3, 1, 1)
        self._std = torch.tensor(self.STD, dtype=torch.float32, device=self.device).view(1, 3, 1, 1)
        self._replay = None
        self._static: dict = {}

    @property
    def provide_cov(self) -> bool:
        return self.config.cov_mode == "Est"

    @staticmethod
    def geometry(H: int, W: int) -> tuple[tuple[int, int], tuple[int, int]]:
        """((crop margin y, x), (h64, w64)) of StereoFeature.getCropMargin (network.py:22-31), checked like padTo"""
        h64, w64 = H // 64 * 64, W // 64 * 64
        if h64 < stereonet.MIN_CROP or w64 < stereonet.MIN_CROP:
            raise ValueError(f"B200_TartanVODepth: a {H}x{W} image gives a {h64}x{w64} crop; StereoNet7's 64x64 average "
                             f"pooling at 1/4 resolution needs a crop of at least {stereonet.MIN_CROP}x{stereonet.MIN_CROP}")
        for size, crop, dim in ((H, h64, -2), (W, w64, -1)):
            assert (size - crop) % 2 == 0, \
                f"Can only handle even padding. Target_size={size}, Actual_size={crop} on dim {dim}."
        return ((H - h64) // 2, (W - w64) // 2), (h64, w64)

    def _run(self, st: dict) -> None:
        """images (2,3,H,W) -> depth / var (1,1,H,W) inside the crop: crop, normalise, encoder, decoders, heads"""
        (my, mx), (h64, w64) = st["margin"], st["crop"]
        net, bf = self.net, st["bf"]
        ims = (st["images"][:, :, my:my + h64, mx:mx + w64] - self._mean) / self._std
        ctx, cats = net.encode(ims)
        xd = net.decode(stereonet.DISP, ctx, cats)
        xc = net.decode(stereonet.COV, ctx, cats) if self.est_cov else None
        if st["kernel"]:
            wd, sd_ = net.head[stereonet.DISP]
            wc, sc = net.head[stereonet.COV] if self.est_cov else (None, None)
            ops.stereo_head(xd, xc, cats[0], wd, sd_, wc, sc, bf, (my, mx), st["depth"], st["var"])
            return
        out_d = net.head_torch(stereonet.DISP, xd, cats[0])
        out_c = net.head_torch(stereonet.COV, xc, cats[0]) if self.est_cov else None
        depth, var = stereonet.depth_torch(out_d, out_c, bf)
        st["depth"][..., my:my + h64, mx:mx + w64].copy_(depth)
        if var is not None:
            st["var"][..., my:my + h64, mx:mx + w64].copy_(var)

    def _capture(self, run):
        """capture `run` as a CUDA graph (after a warm-up run outside the capture, for cuDNN's algorithm choice); returns a
        callable that replays it"""
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES[0]
        with torch.cuda.graph(graph):
            run()
        launches = ops.LAUNCHES[0] - n0

        def replay():
            graph.replay()
            ops.LAUNCHES[0] += launches
        return replay

    def estimate(self, frame: StereoData) -> IStereoDepth.Output:
        with torch.inference_mode():
            imgL, imgR = frame.imageL, frame.imageR
            assert imgL.size(0) == 1 and imgR.size(0) == 1, "The interface will not handle batch dimension correctly."
            H, W = imgL.shape[-2:]
            assert tuple(imgR.shape[-2:]) == (H, W), "both images must have the same size"
            bf = frame.frame_baseline * frame.fx
            kernel = self.device.type == "cuda" and bool(torch.backends.cudnn.allow_tf32)
            st = self._static
            if self._replay is not None:
                assert (H, W) == st["shape"], f"image shape changed since the CUDA graph was captured: {(H, W)} != {st['shape']}"
                assert bf == st["bf"], "camera baseline * fx changed since the CUDA graph was captured"
                if kernel != st["kernel"]:          # the TF32 flag changed: the other head path needs its own graph
                    self._replay = None
            if self._replay is None:
                margin, crop = self.geometry(H, W)
                nan = lambda: torch.full((1, 1, H, W), float("nan"), dtype=torch.float32, device=self.device)
                st = self._static = {"shape": (H, W), "margin": margin, "crop": crop, "bf": bf, "kernel": kernel,
                                     "images": torch.empty((2, 3, H, W), dtype=torch.float32, device=self.device),
                                     "depth": nan(), "var": nan() if self.est_cov else None}
            st["images"][0:1].copy_(imgL, non_blocking=True)
            st["images"][1:2].copy_(imgR, non_blocking=True)
            run = lambda: self._run(st)
            # deterministic cuDNN algorithms (the transposed convolutions would otherwise be free to accumulate with atomics),
            # so that a graph replay, the first call and cuda_graph: false give the same bits; TF32 and the other flags as
            # they are
            with torch.backends.cudnn.flags(enabled=torch.backends.cudnn.enabled, benchmark=torch.backends.cudnn.benchmark,
                                            benchmark_limit=torch.backends.cudnn.benchmark_limit, deterministic=True,
                                            allow_tf32=torch.backends.cudnn.allow_tf32):
                if not self.use_graph:
                    run()
                elif self._replay is None:
                    self._replay = self._capture(run)
                    self._replay()
                else:
                    self._replay()
            if self.est_cov:
                return IStereoDepth.Output(depth=st["depth"].clone(), cov=st["var"].clone())
            return IStereoDepth.Output(depth=st["depth"].clone())

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        spec = {
            "weight": lambda f: isinstance(f, str),
            "device": lambda dev: isinstance(dev, str) and "cuda" in dev,
            "cov_mode": lambda m: m in {"Est", "None"},
        }
        if config is not None and "cuda_graph" in vars(config):
            spec["cuda_graph"] = lambda b: isinstance(b, bool)
        cls._enforce_config_spec(config, spec)


# ================================================================================================
# TartanVO baseline driver
# ================================================================================================
_IOdometry = object
if _REF:
    try:    # receive_frames (poses.npy, tensor_map.npz) comes from MAC-VO's own IOdometry
        from Odometry.Interface import IOdometry as _IOdometry  # type: ignore
        from Module.Map import VisualMap as _VisualMap, FrameNode as _FrameNode  # type: ignore
    except ImportError:
        _IOdometry = object


class B200_TartanVO(_IOdometry):
    """Drop-in for the TartanVO baseline's driver (Odometry/BaselineTartanVO.TartanVO): the same Odometry section, the same
    per-frame poses and map, with every network on the device through `pipeline.FusedTartanVO` (see there for what runs
    where). This class only builds the driver from the config and writes its trajectory in MAC-VO's map format.

    It differs from the reference driver in what it does not do: it names no "Naive" map processor (the reference's, which
    MAC-VO does not define; `terminate()` leaves the trajectory as a no-op processor would), its first pose has the map's
    leading dimension, it runs neither the depth network's covariance decoder (whatever `depth.args.cov_mode` says) nor
    the first frame's depth, and all frames must keep one image shape and camera."""

    MATCH, DEPTH = "B200_TartanVOMatcher", "B200_TartanVODepth"

    def __init__(self, match_estimator: "B200_TartanVOMatcher", depth_estimator: "B200_TartanVODepth",
                 keyframe_freq: int, motion: "B200_TartanMotionNet", cuda_graph: bool = True):
        if _IOdometry is not object:
            super().__init__()
        from .pipeline import FusedTartanVO
        self.fused = FusedTartanVO(match_estimator, depth_estimator, motion, keyframe_freq, cuda_graph)
        self._map = None

    @classmethod
    def from_config(cls, cfg: SimpleNamespace, seq=None) -> "B200_TartanVO":
        """`cfg` is the Odometry section (or a whole experiment config holding one); `seq` is not read"""
        cfg = getattr(cfg, "Odometry", cfg)
        cls.is_valid_config(cfg)
        depth_args = SimpleNamespace(**dict(vars(cfg.depth.args), cov_mode="None"))
        freq = cfg.keyframe.args.keyframe_freq if cfg.keyframe.type == "UniformKeyframe" else 1
        graph = bool(getattr(cfg.match.args, "cuda_graph", True)) and bool(getattr(cfg.depth.args, "cuda_graph", True))
        return cls(B200_TartanVOMatcher(cfg.match.args), B200_TartanVODepth(depth_args), freq,
                   B200_TartanMotionNet(cfg.tartanvo), cuda_graph=graph)

    @torch.inference_mode()
    def run(self, frame) -> None:
        self._map = None
        self.fused.run(frame)

    def get_map(self):
        """MAC-VO's VisualMap (a namespace with the same `frames.data` columns without MAC-VO), built once from the device
        trajectory: per frame K, baseline, need_interp, time_ns, pose (fp32 [t, q_xyzw]) and T_BS"""
        if self._map is None:
            poses, interp = self.fused.finish()
            fr = self.fused.frames
            as7 = lambda t: (t.tensor() if hasattr(t, "ltype") else torch.as_tensor(t)).reshape(-1, 7).float().cpu()
            data = {
                "K": torch.cat([f["K"].reshape(-1, 3, 3).float().cpu() for f in fr]),
                "baseline": torch.cat([torch.as_tensor(f["baseline"]).reshape(-1).float().cpu() for f in fr]),
                "need_interp": interp,
                "time_ns": torch.cat([torch.as_tensor(f["time_ns"], dtype=torch.long).reshape(-1) for f in fr]),
                "pose": poses,
                "T_BS": torch.cat([as7(f["T_BS"]) for f in fr]),
            }
            if _IOdometry is not object:
                self._map = _VisualMap()
                self._map.frames.push(_FrameNode.init(data))
            else:
                self._map = SimpleNamespace(frames=SimpleNamespace(
                    data={k: SimpleNamespace(tensor=v) for k, v in data.items()}))
        return self._map

    def terminate(self) -> None:
        if _IOdometry is not object:
            super().terminate()

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        assert config is not None
        for key, want, plugin in (("match", cls.MATCH, B200_TartanVOMatcher), ("depth", cls.DEPTH, B200_TartanVODepth)):
            sec = getattr(config, key, None)
            if sec is None or getattr(sec, "type", None) != want:
                raise ValueError(f"B200_TartanVO: Odometry.{key}.type must be {want}, got "
                                 f"{getattr(sec, 'type', None)!r}")
            plugin.is_valid_config(sec.args)
        B200_TartanMotionNet.is_valid_config(config.tartanvo)
        kf = config.keyframe
        if kf.type == "UniformKeyframe":
            _local._Registry._enforce_config_spec(kf.args, {"keyframe_freq": lambda f: isinstance(f, int) and f >= 1})
        elif kf.type == "AllKeyframe":
            _local._Registry._enforce_config_spec(kf.args, {})
        else:
            raise ValueError(f"B200_TartanVO: Odometry.keyframe.type must be UniformKeyframe or AllKeyframe, got "
                             f"{kf.type!r}")
        spec = {k: (lambda v: True) for k in ("match", "depth", "tartanvo", "keyframe")}
        if "name" in vars(config):
            spec["name"] = lambda n: isinstance(n, str)
        _local._Registry._enforce_config_spec(config, spec)


PLUGINS = {
    "frontend": B200_FlowFormerCovFrontend,
    "frontend_plain": B200_FlowFormerFrontend,
    "keypoint": B200_CovAwareSelector_NoDepth,
    "keypoint_depth": B200_CovAwareSelector,
    "mappoint": B200_MappingPointSelector,
    "cov": B200_MatchCovariance,
    "cov_none": B200_NoCovariance,
    "cov_diagonalize": B200_Modifier_Diagonalize,
    "cov_normalize": B200_Modifier_Normalize,
    "keypoint_random": B200_RandomSelector,
    "outlier": B200_CovarianceSanityFilter,
    "postprocess": B200_MotionInterpolate,
    "optimizer": B200_TwoFrame_PGO,
    "motion": B200_TartanMotionNet,
    "matcher_tartanvo": B200_TartanVOMatcher,
    "depth_tartanvo": B200_TartanVODepth,
    "odometry_tartanvo": B200_TartanVO,
}
