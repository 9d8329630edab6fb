"""TEST INFRASTRUCTURE — restatement of the parts of `pypose` (pinned by the reference at
pypose==0.6.8, `static_analysis_requirements.txt:1`; source NOT in the MAC-VO tree, not
installed, no network) that MAC-VO's two-frame pose-graph path touches.

Only `tests/`, `tests/golden/make_golden.py`, `__graft_entry__.smoke()` and `bench.py`'s CPU legs
may import this. It exists so that the reference's OWN optimizer code
(`Module/Optimization/PyposeOptimizers.py:136-194`, `TwoFramePGO/Graphs.py:76-230`,
`TwoFramePGO/Optimizer.py:82-102`) can execute in this container and pin the fp64 oracle
(`oracle/pgo.py`). PARITY UNPINNED for what lives in here: no reference test pins pypose's
arithmetic, the semantics below are restated from the published pypose 0.6.8 behaviour:

* SE3 storage `[tx, ty, tz, qx, qy, qz, qw]`; tangent `[tau(3), phi(3)]`.
* `Exp(tau, phi) = (J_l(phi) tau, quat(phi))`; `Inv`, `Act` (R p + t), group product.
* `LieTensor.add_(delta)` on a group element is the LEFT retraction `x <- Exp(delta[..., :6]) * x`
  (the 7th entry of a 7-wide step is ignored; matches "last column is useless",
  `TwoFramePGO/Graphs.py:194,225`).
* `pixel2point` / `point2pixel` (EDN camera convention), `vec2skew`.
"""
from __future__ import annotations

import math
import types
import torch
from torch import nn

__version__ = "0.6.8-restated"


# --------------------------------------------------------------------------------------
# Lie types
# --------------------------------------------------------------------------------------
class _LieType:
    def __init__(self, name: str, dim: int, manifold: int, on_manifold: bool):
        self.name, self.dim, self.manifold, self.on_manifold = name, dim, manifold, on_manifold

    def __repr__(self):
        return self.name

    # pp.SE3_type.Act(pose, pts) is used as an unbound helper by Odometry/MACVO.py:276
    def Act(self, x, p):
        return LieTensor(_raw(x), ltype=self).Act(p)


SE3_type = _LieType("SE3_type", 7, 6, False)
se3_type = _LieType("se3_type", 6, 6, True)
SO3_type = _LieType("SO3_type", 4, 3, False)
so3_type = _LieType("so3_type", 3, 3, True)


def _raw(x) -> torch.Tensor:
    return x.as_subclass(torch.Tensor) if isinstance(x, torch.Tensor) else torch.as_tensor(x)


# --------------------------------------------------------------------------------------
# plain-tensor math
# --------------------------------------------------------------------------------------
def vec2skew(v: torch.Tensor) -> torch.Tensor:
    v = _raw(v)
    O = torch.zeros_like(v[..., 0])
    return torch.stack([
        torch.stack([O, -v[..., 2], v[..., 1]], dim=-1),
        torch.stack([v[..., 2], O, -v[..., 0]], dim=-1),
        torch.stack([-v[..., 1], v[..., 0], O], dim=-1),
    ], dim=-2)


def _quat_mul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by - ax * bz + ay * bw + az * bx,
        aw * bz + ax * by - ay * bx + az * bw,
        aw * bw - ax * bx - ay * by - az * bz,
    ], dim=-1)


def _quat_rot(q: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """R(q) p  via  p + 2 w (v x p) + 2 v x (v x p)."""
    v, w = q[..., :3], q[..., 3:4]
    uv = torch.linalg.cross(v.expand(torch.broadcast_shapes(v.shape, p.shape)),
                            p.expand(torch.broadcast_shapes(v.shape, p.shape)), dim=-1)
    uv = uv * 2
    return p + w * uv + torch.linalg.cross(v.expand_as(uv), uv, dim=-1)


def _quat_matrix(q: torch.Tensor) -> torch.Tensor:
    x, y, z, w = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], dim=-1),
        torch.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], dim=-1),
        torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], dim=-1),
    ], dim=-2)


def _so3_exp(phi: torch.Tensor) -> torch.Tensor:
    theta = phi.norm(dim=-1, keepdim=True)
    t2 = theta * theta
    t4 = t2 * t2
    eps = torch.finfo(phi.dtype).eps
    small = theta <= eps
    safe = torch.where(small, torch.ones_like(theta), theta)
    imag = torch.where(small, 0.5 - t2 / 48 + t4 / 3840, torch.sin(0.5 * safe) / safe)
    real = torch.where(small, 1 - t2 / 8 + t4 / 384, torch.cos(0.5 * theta))
    return torch.cat([phi * imag, real], dim=-1)


def _so3_jl(phi: torch.Tensor) -> torch.Tensor:
    """Left Jacobian of SO(3): I + (1-cos t)/t^2 K + (t - sin t)/t^3 K^2."""
    theta = phi.norm(dim=-1, keepdim=True).unsqueeze(-1)
    t2 = theta * theta
    eps = torch.finfo(phi.dtype).eps
    small = theta <= eps
    safe = torch.where(small, torch.ones_like(theta), theta)
    c1 = torch.where(small, 0.5 - t2 / 24 + t2 * t2 / 720, (1 - torch.cos(safe)) / (safe * safe))
    c2 = torch.where(small, 1.0 / 6 - t2 / 120 + t2 * t2 / 5040, (safe - torch.sin(safe)) / (safe * safe * safe))
    K = vec2skew(phi)
    I = torch.eye(3, dtype=phi.dtype, device=phi.device).expand_as(K)
    return I + c1 * K + c2 * (K @ K)


def _so3_log(q: torch.Tensor) -> torch.Tensor:
    """SO3 Log as pypose computes it: phi = v * 2 atan(|v| / w) / |v| (series 2/w - 2|v|^2 / (3 w^3) near |v| = 0)."""
    v, w = q[..., :3], q[..., 3:4]
    n = v.norm(dim=-1, keepdim=True)
    eps = torch.finfo(q.dtype).eps
    small = n <= eps
    safe = torch.where(small, torch.ones_like(n), n)
    factor = torch.where(small, 2.0 / w - 2.0 * n * n / (3.0 * w * w * w), 2.0 * torch.atan(safe / w) / safe)
    return v * factor


def _so3_jl_inv(phi: torch.Tensor) -> torch.Tensor:
    """Inverse left Jacobian of SO(3): I - K/2 + (1/t^2 - (1 + cos t) / (2 t sin t)) K^2."""
    theta = phi.norm(dim=-1, keepdim=True).unsqueeze(-1)
    t2 = theta * theta
    eps = torch.finfo(phi.dtype).eps
    small = theta <= eps
    safe = torch.where(small, torch.ones_like(theta), theta)
    coef = torch.where(small, 1.0 / 12 + t2 / 720 + t2 * t2 / 30240,
                       1.0 / (safe * safe) - (1 + torch.cos(safe)) / (2 * safe * torch.sin(safe)))
    K = vec2skew(phi)
    I = torch.eye(3, dtype=phi.dtype, device=phi.device).expand_as(K)
    return I - 0.5 * K + coef * (K @ K)


def _se3_log(x: torch.Tensor) -> torch.Tensor:
    phi = _so3_log(x[..., 3:7])
    tau = (_so3_jl_inv(phi) @ x[..., :3].unsqueeze(-1)).squeeze(-1)
    return torch.cat([tau, phi], dim=-1)


def _se3_exp(x: torch.Tensor) -> torch.Tensor:
    tau, phi = x[..., :3], x[..., 3:6]
    t = (_so3_jl(phi) @ tau.unsqueeze(-1)).squeeze(-1)
    return torch.cat([t, _so3_exp(phi)], dim=-1)


# --------------------------------------------------------------------------------------
# LieTensor
# --------------------------------------------------------------------------------------
class LieTensor(torch.Tensor):
    ltype: _LieType

    @staticmethod
    def __new__(cls, data, ltype: _LieType | None = None, requires_grad: bool = False):
        data = _raw(data) if isinstance(data, torch.Tensor) else torch.as_tensor(data)
        obj = torch.Tensor._make_subclass(cls, data.detach() if data.requires_grad and not requires_grad else data,
                                          requires_grad)
        return obj

    def __init__(self, data, ltype: _LieType | None = None, requires_grad: bool = False):
        if ltype is None:
            ltype = getattr(data, "ltype", None)
        assert ltype is not None, "LieTensor needs an ltype"
        assert self.shape[-1] == ltype.dim, f"{ltype} expects last dim {ltype.dim}, got {tuple(self.shape)}"
        self.ltype = ltype

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        out = super().__torch_function__(func, types, args, kwargs or {})
        src = next((a for a in args if isinstance(a, LieTensor) and hasattr(a, "ltype")), None)
        if src is not None:
            def tag(o):
                if isinstance(o, LieTensor) and not hasattr(o, "ltype"):
                    if o.dim() > 0 and o.shape[-1] == src.ltype.dim and o.dtype.is_floating_point:
                        o.ltype = src.ltype
                    else:  # no longer a Lie element (slice / reduction / bool): hand back a plain tensor
                        return o.as_subclass(torch.Tensor)
                return o
            if isinstance(out, (tuple, list)):
                out = type(out)(tag(o) for o in out)
            else:
                out = tag(out)
            # indexing a pp.Parameter (nn.Parameter disables subclass propagation) must still give a Lie element:
            # `self.pose2opt[self.edges_index]` in the ICP graph (TwoFramePGO/Graphs.py:57,64,156)
            if (func is torch.Tensor.__getitem__ and type(out) is torch.Tensor and out.dim() > 0
                    and out.shape[-1] == src.ltype.dim and out.dtype.is_floating_point):
                out = LieTensor(out, ltype=src.ltype)
        return out

    def __repr__(self):
        return f"{getattr(self, 'ltype', '?')} LieTensor:\n{_raw(self)}"

    # ---- group ops --------------------------------------------------------------------
    def tensor(self) -> torch.Tensor:
        return _raw(self)

    def translation(self) -> torch.Tensor:
        assert self.ltype is SE3_type
        return _raw(self)[..., :3]

    def rotation(self) -> "LieTensor":
        if self.ltype is SE3_type:
            return LieTensor(_raw(self)[..., 3:7], ltype=SO3_type)
        assert self.ltype is SO3_type
        return self

    def matrix(self) -> torch.Tensor:
        d = _raw(self)
        if self.ltype is SO3_type:
            return _quat_matrix(d)
        assert self.ltype is SE3_type
        R = _quat_matrix(d[..., 3:7])
        top = torch.cat([R, d[..., :3].unsqueeze(-1)], dim=-1)
        bot = torch.zeros_like(top[..., :1, :])
        bot[..., 0, 3] = 1
        return torch.cat([top, bot], dim=-2)

    def Inv(self) -> "LieTensor":
        d = _raw(self)
        if self.ltype is SO3_type:
            return LieTensor(d * d.new_tensor([-1, -1, -1, 1]), ltype=SO3_type)
        assert self.ltype is SE3_type
        qi = d[..., 3:7] * d.new_tensor([-1, -1, -1, 1])
        ti = -_quat_rot(qi, d[..., :3])
        return LieTensor(torch.cat([ti, qi], dim=-1), ltype=SE3_type)

    def Act(self, p: torch.Tensor) -> torch.Tensor:
        d, p = _raw(self), _raw(p)
        if self.ltype is SO3_type:
            return _quat_rot(d, p)
        assert self.ltype is SE3_type
        return _quat_rot(d[..., 3:7], p) + d[..., :3]

    def Exp(self) -> "LieTensor":
        d = _raw(self)
        if self.ltype is se3_type:
            return LieTensor(_se3_exp(d), ltype=SE3_type)
        assert self.ltype is so3_type
        return LieTensor(_so3_exp(d), ltype=SO3_type)

    def Log(self) -> "LieTensor":
        d = _raw(self)
        if self.ltype is SE3_type:
            return LieTensor(_se3_log(d), ltype=se3_type)
        assert self.ltype is SO3_type
        return LieTensor(_so3_log(d), ltype=so3_type)

    def _compose(self, other: "LieTensor") -> "LieTensor":
        a, b = _raw(self), _raw(other)
        if self.ltype is SO3_type:
            return LieTensor(_quat_mul(a, b), ltype=SO3_type)
        assert self.ltype is SE3_type and other.ltype is SE3_type
        t = _quat_rot(a[..., 3:7], b[..., :3]) + a[..., :3]
        return LieTensor(torch.cat([t, _quat_mul(a[..., 3:7], b[..., 3:7])], dim=-1), ltype=SE3_type)

    def __mul__(self, other):
        if isinstance(other, LieTensor) and hasattr(other, "ltype") and not other.ltype.on_manifold:
            return self._compose(other)
        if isinstance(other, torch.Tensor):
            return self.Act(other)
        return NotImplemented

    def __matmul__(self, other):
        return self.__mul__(other)

    def add_(self, other, alpha=1):
        """In-place retraction.  Group element: x <- Exp(alpha * other[..., :m]) * x."""
        other = _raw(other)
        if self.ltype.on_manifold:
            _raw(self).add_(other, alpha=alpha)
            return self
        delta = LieTensor(alpha * other[..., :self.ltype.manifold], ltype=se3_type if self.ltype is SE3_type else so3_type)
        new = delta.Exp()._compose(self)
        _raw(self).copy_(_raw(new))
        return self


class Parameter(LieTensor, nn.Parameter):
    @staticmethod
    def __new__(cls, data=None, requires_grad: bool = True):
        return torch.Tensor._make_subclass(cls, _raw(data), requires_grad)

    def __init__(self, data=None, requires_grad: bool = True):
        self.ltype = data.ltype

    def __deepcopy__(self, memo):
        out = Parameter(LieTensor(_raw(self).clone(), ltype=self.ltype), self.requires_grad)
        memo[id(self)] = out
        return out


def SE3(data) -> LieTensor:
    return LieTensor(_raw(data) if isinstance(data, torch.Tensor) else torch.as_tensor(data), ltype=SE3_type)


def se3(data) -> LieTensor:
    return LieTensor(_raw(data) if isinstance(data, torch.Tensor) else torch.as_tensor(data), ltype=se3_type)


def SO3(data) -> LieTensor:
    return LieTensor(_raw(data) if isinstance(data, torch.Tensor) else torch.as_tensor(data), ltype=SO3_type)


def identity_SE3(*size, **kwargs) -> LieTensor:
    d = torch.zeros(*size, 7, **kwargs)
    d[..., 6] = 1
    return LieTensor(d, ltype=SE3_type)


def Act(x: LieTensor, p: torch.Tensor) -> torch.Tensor:
    return x.Act(p)


def pixel2point(pixels: torch.Tensor, depth: torch.Tensor, intrinsics: torch.Tensor) -> torch.Tensor:
    """[(u-cx)/fx*d, (v-cy)/fy*d, d] (EDN)."""
    pixels, depth, K = _raw(pixels), _raw(depth), _raw(intrinsics)
    fx, fy, cx, cy = K[..., 0, 0], K[..., 1, 1], K[..., 0, 2], K[..., 1, 2]
    x = (pixels[..., 0] - cx) / fx * depth
    y = (pixels[..., 1] - cy) / fy * depth
    return torch.stack([x, y, depth.expand_as(x)], dim=-1)


def point2pixel(points: torch.Tensor, intrinsics: torch.Tensor, extrinsics=None) -> torch.Tensor:
    """[fx X/Z + cx, fy Y/Z + cy]."""
    points, K = _raw(points), _raw(intrinsics)
    fx, fy, cx, cy = K[..., 0, 0], K[..., 1, 1], K[..., 0, 2], K[..., 1, 2]
    return torch.stack([fx * points[..., 0] / points[..., 2] + cx,
                        fy * points[..., 1] / points[..., 2] + cy], dim=-1)


def _unavailable(name):
    def f(*a, **k):
        raise NotImplementedError(f"pypose.{name} is not restated (not on MAC-VO's two-frame PGO path)")
    f.__name__ = name
    return f


def cumops(input, dim, ops):
    """Inclusive left fold along `dim`: y_0 = x_0, y_i = ops(y_{i-1}, x_i) (pypose 0.6.8 `cumops`; the library evaluates it
    as a doubling scan, which gives the same result for an associative `ops`). Only dim = 0 is needed
    (Module/MapProcessor.py:75)."""
    assert dim == 0
    if input.shape[0] == 0:
        return input
    out = [input[0:1]]
    for i in range(1, input.shape[0]):
        out.append(ops(out[-1], input[i:i + 1]))
    raw = torch.cat([_raw(o) for o in out], dim=0)
    return LieTensor(raw, ltype=input.ltype) if isinstance(input, LieTensor) else raw


def _mat2quat(R: torch.Tensor) -> torch.Tensor:
    """Rotation matrix (..., 3, 3) -> unit quaternion [x, y, z, w] (import-time constants only)."""
    m = R.reshape(-1, 3, 3).double()
    out = []
    for M in m:
        tr = float(M[0, 0] + M[1, 1] + M[2, 2])
        if tr > 0:
            s = math.sqrt(tr + 1.0) * 2
            q = [(M[2, 1] - M[1, 2]) / s, (M[0, 2] - M[2, 0]) / s, (M[1, 0] - M[0, 1]) / s, 0.25 * s]
        elif M[0, 0] > M[1, 1] and M[0, 0] > M[2, 2]:
            s = math.sqrt(1.0 + float(M[0, 0] - M[1, 1] - M[2, 2])) * 2
            q = [0.25 * s, (M[0, 1] + M[1, 0]) / s, (M[0, 2] + M[2, 0]) / s, (M[2, 1] - M[1, 2]) / s]
        elif M[1, 1] > M[2, 2]:
            s = math.sqrt(1.0 + float(M[1, 1] - M[0, 0] - M[2, 2])) * 2
            q = [(M[0, 1] + M[1, 0]) / s, 0.25 * s, (M[1, 2] + M[2, 1]) / s, (M[0, 2] - M[2, 0]) / s]
        else:
            s = math.sqrt(1.0 + float(M[2, 2] - M[0, 0] - M[1, 1])) * 2
            q = [(M[0, 2] + M[2, 0]) / s, (M[1, 2] + M[2, 1]) / s, 0.25 * s, (M[1, 0] - M[0, 1]) / s]
        out.append(torch.tensor([float(v) for v in q], dtype=torch.float64))
    return torch.stack(out).reshape(*R.shape[:-2], 4).to(R.dtype if R.dtype.is_floating_point else torch.float32)


def from_matrix(mat: torch.Tensor, ltype: _LieType, check: bool = True, rtol=1e-5, atol=1e-5) -> LieTensor:
    mat = _raw(mat)
    if ltype is SO3_type:
        return LieTensor(_mat2quat(mat[..., :3, :3]), ltype=SO3_type)
    assert ltype is SE3_type
    q = _mat2quat(mat[..., :3, :3])
    return LieTensor(torch.cat([mat[..., :3, 3].to(q.dtype), q], dim=-1), ltype=SE3_type)


euler2SO3 = _unavailable("euler2SO3")
randn_SE3 = _unavailable("randn_SE3")
module = types.ModuleType("pypose.module")
import sys as _sys
_sys.modules.setdefault("pypose.module", module)
