"""Plugin interfaces of the hot path.

MAC-VO instantiates its modules by class name through a registry (`Module.I<X>.instantiate(type, args)`,
Utility/Extensions/SubclassRegistry.py:25-48). When the MAC-VO tree is importable (`import Module` works)
the B200 plugins subclass MAC-VO's OWN interfaces, so importing `macvo_b200.plugins` registers them and a
YAML `type: B200_...` selects them — `Odometry/MACVO.py` stays unchanged.

When MAC-VO is not importable (no MAC-VO tree on the path) the minimal mirrors below
provide the same names, signatures and error behaviour for the methods the hot path uses:

    IFrontend            Module/Frontend/Frontend.py:38-118
    IStereoDepth         Module/Frontend/StereoDepth.py:18-50 (Output, provide_cov, estimate)
    IMatcher             Module/Frontend/Matching.py:20-70 (Output, provide_cov, forward, estimate)
    IKeypointSelector    Module/KeypointSelector.py:17-48
    ICovariance2to3      Module/Covariance/Project2to3.py:16-44
    IMotionModel         Module/MotionModel.py:15-41
    IOptimizer           Module/Optimization/Interface.py:40-242 (sequential mode only)
    StereoData           DataLoader/Interface.py:57-113
    StereoFrame          DataLoader/Interface.py:168-195
    ConfigTestable._enforce_config_spec  Utility/Extensions/Testable.py:23-42
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from dataclasses import dataclass
from types import SimpleNamespace

import torch


def reference_available() -> bool:
    try:
        import Module  # noqa: F401  (MAC-VO's package)
        from Module.Frontend.Frontend import IFrontend  # noqa: F401
        return True
    except Exception:
        return False


# ------------------------------------------------------------------------------------------------
# registry + config checking (mirrors SubclassRegistry / ConfigTestable)
# ------------------------------------------------------------------------------------------------
class _Registry:
    _HIERARCHY: dict[str, type]

    def __init_subclass__(cls, **kwargs) -> None:
        super().__init_subclass__(**kwargs)
        cls._HIERARCHY = {"": cls}
        for parent in cls.mro()[1:]:
            table = parent.__dict__.get("_HIERARCHY")
            if table is None:
                continue
            if cls.__name__ in table:
                raise NameError(f"SubclassRegistry Error: There more than one descendent of class "
                                f"'{parent.__name__}' with name of {cls.__name__}.")
            table[cls.__name__] = cls

    @classmethod
    def get_class(cls, type: str):
        if type in cls._HIERARCHY:
            return cls._HIERARCHY[type]
        raise KeyError(f"Get '{type}' from class {cls.__name__}, expect to be one of {list(cls._HIERARCHY.keys())}")

    @classmethod
    def instantiate(cls, type: str, *args, **kwargs):
        return cls.get_class(type)(*args, **kwargs)

    @classmethod
    def is_valid_config(cls, config: SimpleNamespace | None) -> None:
        if cls.__dict__.get("_IS_INTERFACE", False):
            assert config is not None
            cls.get_class(config.type).is_valid_config(config.args)

    @staticmethod
    def _enforce_config_spec(config, spec, allow_excessive_cfg: bool = False) -> None:
        if not isinstance(spec, dict):
            if not spec(config):
                raise ValueError(f"Config does not match specification! ({config} does not pass test)")
            return
        assert isinstance(config, SimpleNamespace), f"Config does not have same shape as the spec! got {config}"
        for key, test in spec.items():
            if key not in config.__dict__:
                raise KeyError(f"Config does not match specification! (expect to have key {key} but did not found)")
            _Registry._enforce_config_spec(config.__dict__[key], test)
        if not allow_excessive_cfg and len(spec) != len(vars(config)):
            raise KeyError(f"Excessive Keys: {set(vars(config)) - set(spec)} from {list(spec)}")


@dataclass(kw_only=True)
class StereoData:
    T_BS: object
    K: torch.Tensor            # (1,3,3) fp32
    baseline: torch.Tensor     # (1,)
    time_ns: list
    height: int
    width: int
    imageL: torch.Tensor       # (1,3,H,W) fp32 in [0,1]
    imageR: torch.Tensor
    gt_flow: torch.Tensor | None = None
    flow_mask: torch.Tensor | None = None
    gt_depth: torch.Tensor | None = None

    @property
    def frame_baseline(self) -> float:
        assert self.baseline.size(0) == 1, "Can only use frame_baseline on unbatched data"
        return self.baseline.item()

    @property
    def frame_K(self) -> torch.Tensor:
        assert self.K.size(0) == 1
        return self.K[0]

    @property
    def fx(self) -> float: return self.K[0, 0, 0].item()
    @property
    def fy(self) -> float: return self.K[0, 1, 1].item()
    @property
    def cx(self) -> float: return self.K[0, 0, 2].item()
    @property
    def cy(self) -> float: return self.K[0, 1, 2].item()


@dataclass(kw_only=True)
class StereoFrame:
    """DataLoader/Interface.py:168-195 (DataFrame + StereoFrame): what a per-frame odometry driver reads"""
    idx: list
    time_ns: list
    stereo: StereoData
    gt_pose: object = None

    @property
    def frame_idx(self) -> int:
        assert len(self.idx) == 1, "frame_idx property is only valid on unbatched data"
        return self.idx[0]


class IStereoDepth(ABC, _Registry):
    """Module/Frontend/StereoDepth.py:18-50"""
    _IS_INTERFACE = True

    @dataclass
    class Output:
        depth: torch.Tensor
        disparity: torch.Tensor | None = None
        cov: torch.Tensor | None = None
        mask: torch.Tensor | None = None
        disparity_uncertainty: torch.Tensor | None = None

    def __init__(self, config: SimpleNamespace):
        self.config = config

    @property
    @abstractmethod
    def provide_cov(self) -> bool: ...

    @abstractmethod
    def estimate(self, frame: StereoData) -> "IStereoDepth.Output": ...


class IMatcher(ABC, _Registry):
    """Module/Frontend/Matching.py:20-70"""
    _IS_INTERFACE = True

    @dataclass
    class Output:
        flow: torch.Tensor
        cov: torch.Tensor | None = None
        mask: torch.Tensor | None = None

    def __init__(self, config: SimpleNamespace):
        self.config = config

    @property
    @abstractmethod
    def provide_cov(self) -> bool: ...

    @abstractmethod
    def forward(self, frame_t1: StereoData, frame_t2: StereoData) -> "IMatcher.Output": ...

    def estimate(self, frame_t1: StereoData, frame_t2: StereoData) -> "IMatcher.Output":
        with torch.no_grad(), torch.inference_mode():
            return self.forward(frame_t1, frame_t2)


class IFrontend(ABC, _Registry):
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace):
        self.config = config

    @property
    @abstractmethod
    def provide_cov(self) -> tuple[bool, bool]: ...

    @abstractmethod
    def estimate_pair(self, frame_t1: StereoData, frame_t2: StereoData): ...

    @abstractmethod
    def estimate_depth(self, frame: StereoData): ...

    @staticmethod
    def retrieve_pixels(pixel_uv: torch.Tensor, scalar_map: torch.Tensor | None, interpolate: bool = False):
        if scalar_map is None:
            return None
        if interpolate:
            raise NotImplementedError("Not implemented yet")
        return scalar_map[0, ..., pixel_uv[..., 1].long(), pixel_uv[..., 0].long()]


class IKeypointSelector(ABC, _Registry):
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace):
        self.config = config

    @abstractmethod
    def select_point(self, frame: StereoData, numPoint: int, depth0_est, depth1_est, match_est) -> torch.Tensor: ...


class ICovariance2to3(ABC, _Registry):
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace):
        self.config = config

    @abstractmethod
    def estimate(self, frame: StereoData, kp: torch.Tensor, depth_est, depth_cov, flow_cov) -> torch.Tensor: ...


class IObservationFilter(ABC, _Registry):
    """Module/OutlierFilter.py:13-41"""
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace) -> None:
        self.config = config

    def verify_shape(self, value) -> bool:
        return all(k in value.data.keys() for k in self.required_keys)

    def set_meta(self, meta) -> None:
        return None

    @abstractmethod
    def filter(self, values, device: torch.device) -> torch.Tensor: ...


class IMapProcessor(ABC, _Registry):
    """Module/MapProcessor.py:12-25"""
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace | None) -> None:
        self.config = config

    @abstractmethod
    def elaborate_map(self, frames): ...


class IMotionModel(ABC, _Registry):
    """Module/MotionModel.py:15-41: `predict` returns the pose of the incoming frame in world coordinates, `update`
    receives the optimised pose of the previous frame."""
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace) -> None:
        self.config = config

    @abstractmethod
    def predict(self, frame, flow: torch.Tensor | None, depth: torch.Tensor | None) -> torch.Tensor: ...

    @abstractmethod
    def update(self, pose: torch.Tensor) -> None: ...


class IOptimizer(ABC, _Registry):
    """Sequential-mode subset of Module/Optimization/Interface.py (a GPU optimiser runs `parallel: false`:
    its asynchrony is the CUDA stream, not a spawned process)."""
    _IS_INTERFACE = True

    def __init__(self, config: SimpleNamespace) -> None:
        self.config = config
        self.is_parallel_mode = config.parallel
        assert not self.is_parallel_mode, "B200 optimizers run with parallel: false"
        self.context = self.init_context(config)
        self.optimize_res = None
        self.has_opt_job = False

    @staticmethod
    @abstractmethod
    def init_context(config): ...

    @staticmethod
    @abstractmethod
    def _optimize(context, graph_data): ...

    def start_optimize(self, graph_data) -> None:
        self.has_opt_job = True
        self.context, self.optimize_res = self._optimize(self.context, graph_data)

    def get_result(self):
        return self.optimize_res

    def terminate(self) -> None:
        return None
