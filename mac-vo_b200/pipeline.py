"""Per-frame driver of the hot path, for benchmarking / smoke tests without the MAC-VO tree.

It is a restatement of the data flow of `MACVO.run_pair` (Odometry/MACVO.py:173-311) restricted to what the
two-frame pose graph consumes — frontend -> keypoint selection -> in-bound filter -> per-keypoint gathers ->
observation covariances -> sanity filter -> point registration -> two-frame PGO — with the map / factor-graph
bookkeeping (Module/Map, CPU) left out: inside MAC-VO that part is unchanged and it is the CALLER of the
plugins (SURVEY.md §8b), here the optimiser input is assembled directly.

The plugin objects are whatever implements the interfaces: the B200 plugins (`plugins.py`) on the GPU, or
the CPU oracle stand-ins (`oracle/pipeline_cpu.py`) for the CPU baseline — same driver, same order of
calls, same RNG consumption (`select_point` is called for keypoints, then for mapping points).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch

from .plugins import PGOInput


def quat_rotate(q: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """R(q) p for q = [x,y,z,w] (7-vector pose layout of pypose SE3)."""
    v, w = q[..., :3], q[..., 3:4]
    uv = 2 * torch.linalg.cross(v.expand_as(p), p, dim=-1)
    return p + w * uv + torch.linalg.cross(v.expand_as(p), uv, dim=-1)


def se3_act(pose: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    return quat_rotate(pose[3:7].to(p), p) + pose[:3].to(p)


def quat_matrix(q: torch.Tensor) -> torch.Tensor:
    """rotation matrix of q = [x,y,z,w] in q's dtype (pypose `SO3.matrix()`)"""
    x, y, z, w = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], dim=-1),
        torch.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], dim=-1),
        torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], dim=-1),
    ], dim=-2)


class MatchBundle:
    """the `MatchObs` TensorBundle Odometry/MACVO.py:246-270 hands to the outlier filter: `.data` columns, `len()` rows"""

    def __init__(self, data: dict):
        self.data = data

    def __len__(self) -> int:
        return next(iter(self.data.values())).shape[0]


@dataclass
class FrameResult:
    num_kp: int
    num_obs: int
    pose_init: torch.Tensor
    optimizer_output: object
    kp0_uv: torch.Tensor | None = None
    kp1_uv: torch.Tensor | None = None
    map_points: int = 0
    extras: dict = field(default_factory=dict)


class TwoFrameOdometry:
    """args mirror `Odometry.args` of the MAC-VO YAML: num_point, edgewidth, match_cov_default, mapping."""

    def __init__(self, frontend, kp_selector, cov_model, optimizer, num_point: int = 200, edgewidth: int = 32,
                 match_cov_default: float = 0.25, mapping: bool = True, map_selector=None, min_num_point: int = 10,
                 keep_debug: bool = False, motion_model=None, outlier_filter=None):
        self.frontend, self.kp_selector, self.cov_model, self.optimizer = frontend, kp_selector, cov_model, optimizer
        self.motion_model = motion_model            # None: StaticMotionModel (the prediction is the previous pose)
        self.outlier_filter = outlier_filter        # None: CovarianceSanityFilter
        self.graph_type = (getattr(optimizer, "context", None) or {}).get("graph_type", "disp")
        self.map_selector = map_selector
        self.num_point, self.edgewidth, self.match_cov_default = num_point, edgewidth, match_cov_default
        self.mapping, self.min_num_point, self.keep_debug = mapping, min_num_point, keep_debug
        self.prev = None            # (frame, depth output)
        self.poses: list[torch.Tensor] = []
        self._pending = False

    # --- Odometry/MACVO.py:158-171 ---------------------------------------------------------------
    def initialize(self, frame0) -> None:
        depth0 = self.frontend.estimate_depth(frame0)
        self.prev = (frame0, depth0)
        self.poses = [torch.tensor([0., 0., 0., 0., 0., 0., 1.])]
        if self.outlier_filter is not None:
            self.outlier_filter.set_meta(frame0)
        if self.motion_model is not None:         # the first prediction is the identity (MACVO.initialize)
            self.motion_model.predict(frame0, None, depth0.depth)

    def _write_back(self) -> None:
        """Optimizer.write_map (Odometry/MACVO.py:187): blocks on the previous frame's result."""
        if self._pending:
            res = self.optimizer.get_result()
            self.poses[-1] = res.motion.reshape(-1)[:7].detach().double().cpu().float()
            self._pending = False

    # --- Odometry/MACVO.py:173-311 ---------------------------------------------------------------
    def run_pair(self, frame1) -> FrameResult:
        frame0, depth0 = self.prev
        fe = self.frontend
        depth1, match01 = fe.estimate_pair(frame0, frame1)
        self._write_back()
        prev_pose = self.poses[-1]
        if self.motion_model is None:
            est_pose = prev_pose.clone()                               # StaticMotionModel.predict (MotionModel.py:133-137)
        else:                                                          # Odometry/MACVO.py:193-194
            self.motion_model.update(prev_pose)
            pred = self.motion_model.predict(frame1, match01.flow, depth1.depth)
            est_pose = (pred.tensor() if hasattr(pred, "ltype") else pred).reshape(7).detach().cpu().float()

        kp0_uv = self.kp_selector.select_point(frame0, self.num_point, depth0, depth1, match01)
        kp1_uv = kp0_uv + fe.retrieve_pixels(kp0_uv, match01.flow).T
        ew = self.edgewidth
        inb = ((kp1_uv[..., 0] < frame1.width - ew) & (kp1_uv[..., 0] > ew)
               & (kp1_uv[..., 1] < frame1.height - ew) & (kp1_uv[..., 1] > ew))
        kp0_uv, kp1_uv = kp0_uv[inb], kp1_uv[inb]
        num_kp = kp0_uv.size(0)

        # a frontend without covariance maps (B200_FlowFormerFrontend) gives None here, like MACVO.py:212-232
        squeeze = lambda t: None if t is None else t.squeeze(0)
        kp0_d = fe.retrieve_pixels(kp0_uv, depth0.depth).squeeze(0)
        kp0_sigma_dd = squeeze(fe.retrieve_pixels(kp0_uv, depth0.cov))
        kp1_disparity = fe.retrieve_pixels(kp1_uv, depth1.disparity)
        kp1_sigma_disparity = fe.retrieve_pixels(kp1_uv, depth1.disparity_uncertainty)
        kp1_sigma_dd = squeeze(fe.retrieve_pixels(kp1_uv, depth1.cov))

        dev = kp0_uv.device
        kp0_sigma_uv = torch.ones((num_kp, 3), device=dev) * self.match_cov_default
        kp0_sigma_uv[..., 2] = 0.
        kp1_sigma_uv = fe.retrieve_pixels(kp0_uv, match01.cov)
        kp1_sigma_uv = None if kp1_sigma_uv is None else kp1_sigma_uv.T.contiguous()

        K = frame0.frame_K.to(dev)
        fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
        pos0_Tc = torch.stack([kp0_d, (kp0_uv[:, 0] - cx) / fx * kp0_d, (kp0_uv[:, 1] - cy) / fy * kp0_d], dim=-1)  # NED
        pos0_cov = self.cov_model.estimate(frame0, kp0_uv, depth0, kp0_sigma_dd, kp0_sigma_uv)
        pos1_cov = self.cov_model.estimate(frame1, kp1_uv, depth1, kp1_sigma_dd, kp1_sigma_uv)

        kp1_d = None
        if self.outlier_filter is not None or self.graph_type == "icp":
            kp1_d = fe.retrieve_pixels(kp1_uv, depth1.depth).squeeze(0)
        if self.outlier_filter is None:
            # CovarianceSanityFilter (Module/OutlierFilter.py:91-100)
            bad = (pos0_cov.isnan().any(dim=(-1, -2)) | pos0_cov.isinf().any(dim=(-1, -2))
                   | pos1_cov.isnan().any(dim=(-1, -2)) | pos1_cov.isinf().any(dim=(-1, -2)))
            good = ~bad                                                # lives on the host like the covariances: no sync
        else:                                                          # Odometry/MACVO.py:246-272
            placeholder = lambda t: torch.empty((num_kp, 1)).fill_(-1) if t is None else t.unsqueeze(-1).cpu()
            match_obs = MatchBundle({
                "pixel1_uv": kp0_uv.cpu(), "pixel2_uv": kp1_uv.cpu(),
                "pixel1_d": kp0_d.unsqueeze(-1).cpu(), "pixel2_d": kp1_d.unsqueeze(-1).cpu(),
                "pixel1_d_cov": placeholder(kp0_sigma_dd), "pixel2_d_cov": placeholder(kp1_sigma_dd),
                "obs1_covTc": pos0_cov, "obs2_covTc": pos1_cov})
            good = self.outlier_filter.filter(match_obs, torch.device("cpu"))
        num_obs = int(good.sum())
        keep = good.to(dev)
        pos_Tw = se3_act(prev_pose.to(dev), pos0_Tc.float())[keep]

        self.poses.append(est_pose)
        out = None
        if num_obs >= self.min_num_point:
            # MatchObs' -1 placeholders of the missing covariance columns (MACVO.py:250-264)
            if kp1_sigma_uv is None:
                kp1_sigma_uv = torch.full((num_kp, 3), -1.0, device=dev)
            if kp1_sigma_disparity is None:
                kp1_sigma_disparity = torch.full((1, num_kp), -1.0, device=dev)
            inp = PGOInput(pos_Tw=pos_Tw, kp2_uv=kp1_uv[keep].float(), kp2_disp=kp1_disparity.T[keep],
                           uv_cov=kp1_sigma_uv[keep], disp_cov=kp1_sigma_disparity.T[keep], K=frame1.frame_K,
                           baseline=frame1.frame_baseline, init_pose=est_pose)
            if self.graph_type == "icp":                               # MACVO.py:274-280, Graphs.py:49-55
                R = quat_matrix(prev_pose.float()[3:7]).repeat((num_kp, 1, 1)).double()
                cov_Tw = torch.bmm(torch.bmm(R, pos0_cov), R.transpose(1, 2))
                good_h = good.cpu()
                inp.kp2_d, inp.obs_cov, inp.pts_cov = kp1_d[keep], pos1_cov[good_h], cov_Tw[good_h]
            self.optimizer.start_optimize(inp)
            self._pending = True
            out = self.optimizer.get_result() if hasattr(self.optimizer, "optimize_res") else None

        n_map = 0
        if self.mapping and self.map_selector is not None:            # Odometry/MACVO.py:314-337
            map0_uv = self.map_selector.select_point(frame0, 2000, depth0, depth1, match01)
            n_map = map0_uv.size(0)
            if n_map:
                map0_sigma_dd = squeeze(fe.retrieve_pixels(map0_uv, depth0.cov))
                map0_sigma_uv = torch.ones((n_map, 3), device=map0_uv.device) * self.match_cov_default
                map0_sigma_uv[..., 2] = 0.
                self.cov_model.estimate(frame0, map0_uv, depth0, map0_sigma_dd, map0_sigma_uv)

        self.prev = (frame1, depth1)
        res = FrameResult(num_kp=num_kp, num_obs=num_obs, pose_init=est_pose, optimizer_output=out, map_points=n_map)
        if self.keep_debug:
            res.kp0_uv, res.kp1_uv = kp0_uv, kp1_uv
            res.extras = {"depth1": depth1, "match01": match01, "pos0_cov": pos0_cov, "pos1_cov": pos1_cov,
                          "pos_Tw": pos_Tw, "keep": keep, "kp1_d": kp1_d}
        return res

    def finish(self) -> torch.Tensor:
        """Synchronise on the last optimisation and return all poses (F, 7)."""
        self._write_back()
        return torch.stack(self.poses)


class FusedTwoFrameOdometry:
    """Same per-frame data flow as `TwoFrameOdometry`, with everything between the frontend and the optimiser result kept
    on the device (SURVEY.md §8f-3): observation building, CovarianceSanityFilter and MatchObs packing are two launches
    (`ops.observe_pack`, csrc/observe.cu), the LM kernel reads the survivor count on the device
    (`ops.pgo_solve_counted`), the optimised pose of frame t is consumed by frame t+1 without visiting the host, and a
    frame's observations / mapping points / pose travel to pinned host memory in asynchronous copies.

    Host synchronisations per frame: ONE — the two candidate counts that `torch.randperm` needs on the CPU default
    generator (kept for bit-exact keypoints; drawn in MAC-VO's order: keypoints, then mapping points). `TwoFrameOdometry`
    with the plugin-API calls has >= 7 (candidate counts x2, boolean indexing x2, covariance `.cpu()` x3).

    Requires the B200 plugins (uses their device buffers); keypoints and poses equal `TwoFrameOdometry`'s
    (tests/test_gpu_pipeline.py::test_fused_tail_matches_plugin_path).

    `motion_model` (a `plugins.B200_TartanMotionNet`, or None for the previous pose): its graph up to fc1 is enqueued right
    after each frame's frontend, the prefetched next frame's included — it reads only that frame's flow and depth — and
    its head kernel runs in the tail after observe_pack, overwriting the LM's initial pose with the prediction. No extra
    host synchronisation.

    `outlier_filter` (None: CovarianceSanityFilter alone): a B200 observation filter or `B200_FilterCompose` chain that
    contains `B200_CovarianceSanityFilter`; the whole chain runs inside observe_pack (`plugins.observe_ext`). The graph
    type comes from `optimizer.context["graph_type"]`; "icp" packs its extra columns into the same buffer and the counted
    LM reads them there. Either `kp_selector` (B200_CovAwareSelector or its _NoDepth variant) is driven through
    `enqueue_candidates`.

    The ablation back ends: `kp_selector` may be a B200_RandomSelector, whose keypoints are drawn on the device with no
    candidate count, so that with mapping off a frame has NO host synchronisation (`host_waits` records each frame's
    count). `cov_model` may be B200_NoCovariance or B200_Modifier_Diagonalize / _Normalize around a B200 model
    (`plugins.cov_spec`): observe_pack applies the model, and the mapping branch gets the same covariances. With
    B200_NoCovariance the chain may leave out B200_CovarianceSanityFilter (`plugins.check_sanity_chain`).

    A frontend without covariance maps (B200_FlowFormerFrontend, the Vanilla ablation) hands observe_pack NULL maps: the
    packed pixel2_uv_cov / pixel2_disp_cov columns hold MatchObs' -1 placeholder."""

    def __init__(self, frontend, kp_selector, cov_model, optimizer, num_point: int = 200, edgewidth: int = 32,
                 match_cov_default: float = 0.25, mapping: bool = True, map_selector=None, min_num_point: int = 10,
                 num_map_point: int = 2000, keep_debug: bool = False, solver=None, motion_model=None,
                 outlier_filter=None):
        from . import ops
        self.ops = ops
        self.motion_model = motion_model
        self.outlier_filter = outlier_filter
        ctx = getattr(optimizer, "context", None) or {}
        self.graph_type = ctx.get("graph_type", "disp")
        if solver is not None and self.graph_type != "disp":
            raise ValueError(f"a custom solver runs the 'disp' graph only (optimizer graph_type {self.graph_type!r})")
        # solver(obs, intr5, pose_io, stats, min_k): the LM solve on the packed observation buffer; default = one persistent
        # launch on this GPU. bench.py --config sharded plugs in the multi-GPU solve (broadcast + sharded_pgo.FusedShardedPGO)
        self.solver = solver
        self.frontend, self.kp_selector, self.cov_model, self.optimizer = frontend, kp_selector, cov_model, optimizer
        self.map_selector = map_selector
        self.num_point, self.edgewidth, self.match_cov_default = num_point, edgewidth, match_cov_default
        self.mapping, self.min_num_point, self.num_map_point = mapping and map_selector is not None, min_num_point, num_map_point
        self.keep_debug = keep_debug
        from .plugins import B200_RandomSelector, check_sanity_chain, cov_spec
        _, self.cov_ops, params = cov_spec(cov_model)
        self.cov_identity = params is None
        check_sanity_chain(outlier_filter, covariance_finite=self.cov_identity)
        self.device = kp_selector.device
        self.random_kp = isinstance(kp_selector, B200_RandomSelector)   # drawn on the device: no candidate count to wait for
        # B200_NoCovariance has no kernel parameters: observe_pack reads none of them then, and kernel_size 1 reduces the
        # mapping branch's covariance kernel to the point gather at the centre pixel
        self.cov_args = params or dict(kernel_size=1, min_flow_cov=0.25, min_depth_cov=0.05)
        self.cov_ext = {}
        if self.cov_identity or self.cov_ops:
            self.cov_ext = {"cov_model": "identity" if self.cov_identity else "match", "cov_ops": list(self.cov_ops)}
        self.cluster = int(getattr(optimizer, "context", {}).get("cluster", 0)) if hasattr(optimizer, "context") else 0
        icp = self.graph_type == "icp"
        self.obs = [ops.ObservationBuffers(num_point, self.device, extended=icp) for _ in range(2)]      # double buffered
        # filled by initialize (set_meta resolves "auto")
        self.ext = None if outlier_filter is None and not icp and not self.cov_ext else {}
        self.host_waits: list[int] = []     # host synchronisations of each run_pair (0 or 1)
        self.stats = [torch.zeros((8,), dtype=torch.float64, device=self.device) for _ in range(2)]
        if self.mapping:
            self.map_cov = [torch.empty((num_map_point, 3, 3), dtype=torch.float64, device=self.device) for _ in range(2)]
            self.map_cov_host = [torch.empty((num_map_point, 3, 3), dtype=torch.float64).pin_memory() for _ in range(2)]
            self.map_pt_host = [torch.empty((num_map_point, 3), dtype=torch.float32).pin_memory() for _ in range(2)]
            self._eye = torch.eye(3, dtype=torch.float64, device=self.device)
        self.pose_dev: list[torch.Tensor] = []          # (7,) float64 per frame, on the device
        self.pose_host = torch.zeros((2, 7), dtype=torch.float64).pin_memory()
        self.pose_ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.n_map = [0, 0]
        self.frame_no = 0
        self.prev = None
        self.last: FrameResult | None = None
        self._prefetched = None         # (frame, depth, match) of a frontend launched ahead by run_pair(..., next_frame=)
        self._tail_stream = None
        self._tail_done = None

    def initialize(self, frame0) -> None:
        depth0 = self.frontend.estimate_depth(frame0)
        self.prev = (frame0, depth0)
        self.pose_dev = [torch.tensor([0., 0., 0., 0., 0., 0., 1.], dtype=torch.float64, device=self.device)]
        if self.ext is not None:
            from .plugins import observe_ext
            if self.outlier_filter is not None:
                self.outlier_filter.set_meta(frame0)
            self.ext = dict(observe_ext(self.outlier_filter, covariance_finite=self.cov_identity) or {},
                            icp=self.graph_type == "icp", **self.cov_ext)

    @staticmethod
    def _intr(frame) -> tuple[float, float, float, float]:
        K = frame.frame_K if hasattr(frame, "frame_K") else frame.K[0]
        return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])

    @torch.inference_mode()
    def run_pair(self, frame1, next_frame=None) -> FrameResult:
        """One frame. With `next_frame` (the frame the NEXT call will pass) the frames are software-pipelined: its frontend —
        which depends on images only, not on this frame's pose — is enqueued before the host waits for this frame's candidate
        counts, and this frame's tail (sampling gathers, observation building, LM, mapping covariances, result copies) runs on
        a second stream next to it, so neither the tail nor the host round trip of the one synchronisation leaves the GPU idle.
        Results are identical (same kernels, same `randperm` order)."""
        ops = self.ops
        frame0, depth0 = self.prev
        slot = self.frame_no & 1
        if self._prefetched is not None and self._prefetched[0] is frame1:
            depth1, match01, fc1 = self._prefetched[1:]
        else:
            depth1, match01 = self.frontend.estimate_pair(frame0, frame1)
            fc1 = self._enqueue_motion(frame1, depth1, match01)
        self._prefetched = None
        main = torch.cuda.current_stream()
        if self._tail_done is not None:            # the previous frame's tail read the candidate lists the selectors now overwrite
            main.wait_event(self._tail_done)
        # selection kernels for keypoints AND mapping points first, then a single synchronisation for both counts
        # (B200_RandomSelector draws its keypoints right here, in frame order, and needs no count)
        reqs, kp_random = [], None
        if self.random_kp:
            kp_random = self.kp_selector.select_device(frame0, self.num_point)
        else:
            reqs.append((self.kp_selector.enqueue_candidates(frame0, depth0, depth1, match01), self.num_point))
        if self.mapping:
            reqs.append((self.map_selector.enqueue_candidates(depth0), self.num_map_point))
        counts = ops.request_candidate_counts(reqs)
        self.host_waits.append(1 if reqs else 0)
        if next_frame is None:
            if reqs:
                counts.synchronize()
            return self._tail(frame0, frame1, depth0, depth1, match01, reqs, slot, fc1, kp_random)
        d_next, m_next = self.frontend.estimate_pair(frame1, next_frame)
        self._prefetched = (next_frame, d_next, m_next, self._enqueue_motion(next_frame, d_next, m_next))
        if reqs:
            counts.synchronize()
        if self._tail_stream is None:
            self._tail_stream = torch.cuda.Stream(self.device)
        tail = self._tail_stream
        tail.wait_event(counts)
        for t in (match01.flow, match01.cov, depth0.depth, depth1.depth, depth1.disparity, depth1.disparity_uncertainty, fc1,
                  depth0.cov, depth1.cov, kp_random):
            if t is not None:
                t.record_stream(tail)          # allocated on the main stream, consumed on the tail stream
        with torch.cuda.stream(tail):
            res = self._tail(frame0, frame1, depth0, depth1, match01, reqs, slot, fc1, kp_random)
            self._tail_done = torch.cuda.Event()
            self._tail_done.record(tail)
        return res

    def _enqueue_motion(self, frame1, depth1, match01):
        """the motion model's graph (input builder .. fc1) for this frame; its fc1 output copied out of the graph's static
        buffer, which the prefetched next frame's replay overwrites before this frame's tail reads it"""
        if self.motion_model is None:
            return None
        return self.motion_model.enqueue(frame1, match01.flow, depth1.depth).clone()

    def _tail(self, frame0, frame1, depth0, depth1, match01, reqs, slot, fc1=None, kp_random=None) -> FrameResult:
        """everything after the candidate counts reached the host, on the current stream"""
        ops = self.ops
        picks = ops.sample_from_counts(reqs)
        if kp_random is not None:
            picks.insert(0, kp_random)
        kp0_uv = picks[0]
        obs, stats = self.obs[slot], self.stats[slot]
        next_pose = torch.empty((7,), dtype=torch.float64, device=self.device)
        i0, i1 = self._intr(frame0), self._intr(frame1)
        ext = None if self.ext is None else dict(self.ext, depth_cov0=depth0.cov, depth_cov1=depth1.cov)
        ops.observe_pack(obs, kp0_uv, match01.flow, match01.cov, depth0.depth, depth1.depth, depth1.disparity,
                         depth1.disparity_uncertainty, self.edgewidth, i0, i1, self.pose_dev[-1], next_pose,
                         match_cov_default=self.match_cov_default, ext=ext, **self.cov_args)
        if fc1 is not None:     # the motion model's prediction replaces observe_pack's previous-pose prior
            self.motion_model.head(fc1, self.pose_dev[-1], next_pose)
        pose_init = next_pose.clone() if self.keep_debug else None      # the LM's initial pose, before the solve
        bl = float(torch.as_tensor(frame1.frame_baseline, dtype=torch.float32).double().reshape(-1)[0])
        stats.zero_()
        if self.solver is not None:
            self.solver(obs, (*i1, bl), next_pose, stats, self.min_num_point)
        else:
            ops.pgo_solve_counted(obs, (*i1, bl), next_pose, stats, min_k=self.min_num_point, cluster=self.cluster,
                                  graph_type=self.graph_type)
        self.pose_dev.append(next_pose)
        n_map = 0
        if self.mapping:
            map0_uv = picks[1]
            n_map = map0_uv.size(0)
            if n_map:   # constant quantisation covariance for manually selected pixels, clamped like any flow_cov
                sig = max(float(torch.tensor(self.match_cov_default, dtype=torch.float32)),
                          float(torch.tensor(self.cov_args["min_flow_cov"], dtype=torch.float32) ** 2))
                _, pt, _ = ops.match_covariance(map0_uv, depth0.depth, None, *i0, kernel_size=self.cov_args["kernel_size"],
                                                min_flow_cov=self.cov_args["min_flow_cov"],
                                                min_depth_cov=self.cov_args["min_depth_cov"], match_cov_default=sig,
                                                want_point=True, out_cov=self.map_cov[slot][:n_map])
                if self.cov_identity:   # NoCovariance: the covariances are the identity, the points as above
                    self.map_cov[slot][:n_map].copy_(self._eye.expand(n_map, 3, 3))
                if self.cov_ops:
                    ops.cov_modify(self.map_cov[slot][:n_map], self.cov_ops)
                self.map_cov_host[slot][:n_map].copy_(self.map_cov[slot][:n_map], non_blocking=True)
                self.map_pt_host[slot][:n_map].copy_(pt, non_blocking=True)
        self.n_map[slot] = n_map
        # one asynchronous copy ships the frame's MatchObs columns; the pose follows; nothing waits here
        obs.download_async()
        self.pose_host[slot].copy_(next_pose, non_blocking=True)
        self.pose_ready[slot].record()
        self.prev = (frame1, depth1)
        self.frame_no += 1
        res = FrameResult(num_kp=-1, num_obs=-1, pose_init=None, optimizer_output=None, map_points=n_map)
        if self.keep_debug:
            res.kp0_uv = kp0_uv
            res.extras = {"depth1": depth1, "match01": match01, "slot": slot, "pose_init": pose_init}
        self.last = res
        return res

    def latest_pose(self) -> torch.Tensor:
        """Optimised pose of the newest frame on the HOST (float64 (7,)); waits for that frame's pose copy only."""
        slot = (self.frame_no - 1) & 1
        self.pose_ready[slot].synchronize()
        return self.pose_host[slot].clone()

    def observations(self) -> dict:
        """The newest frame's packed observations from pinned host memory (waits for its copy)."""
        slot = (self.frame_no - 1) & 1
        obs = self.obs[slot]
        obs.ready.synchronize()
        hdr = obs.section("header", host=True)
        n = int(hdr[0])
        names = ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov", "pixel2_disp_cov", "obs1_covTc", "obs2_covTc",
                 "pixel1_uv", "pixel1_d")
        if obs.extended:
            names += ("pixel2_d", "pixel1_d_cov", "pixel2_d_cov", "points_Tc", "cov_Tw")
        out = {k: obs.section(k, host=True)[:n].clone() for k in names}
        out.update(num_obs=n, num_kp=int(hdr[1]), num_selected=int(hdr[2]), status=int(hdr[3]))
        if self.mapping:
            self.pose_ready[slot].synchronize()
            m = self.n_map[slot]
            out.update(map_cov=self.map_cov_host[slot][:m].clone(), map_pos_Tc=self.map_pt_host[slot][:m].clone())
        return out

    def finish(self) -> torch.Tensor:
        """All poses (F, 7) float32 like `TwoFrameOdometry.finish` (the map stores fp32 poses)."""
        if self._tail_done is not None:
            self._tail_done.synchronize()
        torch.cuda.current_stream().synchronize()
        return torch.stack([p.cpu().float() for p in self.pose_dev])


def _deterministic_cudnn():
    """the flags B200_TartanVOMatcher / B200_TartanVODepth run their networks under: deterministic cuDNN algorithms, every
    other flag (TF32 included) as the caller set it"""
    cudnn = torch.backends.cudnn
    return cudnn.flags(enabled=cudnn.enabled, benchmark=cudnn.benchmark, benchmark_limit=cudnn.benchmark_limit,
                       deterministic=True, allow_tf32=cudnn.allow_tf32)


class FusedTartanVO:
    """The data flow of the TartanVO baseline's driver (Odometry/BaselineTartanVO.py:35-60) on the device, built from the
    three B200 plugins: `matcher` (B200_TartanVOMatcher), `depth` (B200_TartanVODepth with cov_mode "None": the covariance
    decoder the baseline discards is not run) and `motion` (B200_TartanMotionNet). Their networks run as the plugins run
    them (`_run`, `net.body`, `head`), into buffers this driver owns.

    A frame is a keyframe when frame.frame_idx % keyframe_freq == 0 (UniformKeyframe; 1 for AllKeyframe). A non-keyframe
    enqueues nothing: it carries the previous frame's pose and T_BS, with need_interp True. Per keyframe after the first:
      * L(t) and R(t) cross PCIe once (from the frame's pinned memory, else through double-buffered pinned staging);
        L(t-1) stays on the device from the previous keyframe;
      * PWC-Net on (L(t-1), L(t)) on a side stream, next to the depth network on (L(t), R(t)) on the current stream;
      * after the join, the pose network up to fc1 and its head on the previous pose, which stays on the device: an fp32
        (7,) pose widened to float64 for the head and rounded back, exactly as B200_TartanMotionNet.predict carries it;
      * the pose is written into a device-side trajectory.
    The first keyframe gets the identity; its depth, which the baseline computes and never reads, is not computed.

    cuda_graph (default True): a keyframe's work (both branches, the pose network and its head) is one CUDA graph, captured
    at the second keyframe under the flags the plugins use and replayed after; the image shape, intrinsics and
    baseline * fx must then stay the same. cuda_graph=False runs the same work eagerly.

    Nothing in `run` waits on the device (`host_waits` records, per frame, whether the host had to wait for a staging
    buffer, which only happens for frames in pageable memory), so frame t+1's networks are enqueued while frame t's still
    run. `finish()` synchronises once and returns the (F, 7) fp32 poses and the (F,) need_interp flags; `frames` holds
    what the map stores per frame (K, baseline, T_BS, time_ns)."""

    def __init__(self, matcher, depth, motion, keyframe_freq: int = 1, cuda_graph: bool = True):
        if depth.est_cov:
            raise ValueError("FusedTartanVO runs the depth network without its covariance decoder: build "
                             "B200_TartanVODepth with cov_mode 'None'")
        if not (isinstance(keyframe_freq, int) and keyframe_freq >= 1):
            raise ValueError(f"keyframe_freq must be an integer >= 1, got {keyframe_freq!r}")
        from . import ops
        self.ops = ops
        self.matcher, self.depth, self.motion = matcher, depth, motion
        self.device = motion.device
        self.keyframe_freq, self.cuda_graph = keyframe_freq, cuda_graph
        self.side = torch.cuda.Stream(self.device)
        self.host_waits: list[int] = []
        self.frames: list[dict] = []        # per frame: K, baseline, T_BS, time_ns, need_interp, row (of the trajectory)
        self.traj = torch.empty((256, 7), dtype=torch.float32, device=self.device)    # one row per keyframe, grows x2
        self.num_keyframes = 0
        self._st: dict | None = None
        self._graph = None
        self._staging = None                # two pinned (2,3,H,W) buffers, for frames in pageable memory
        self._staged = [None, None]         # the event after each staging buffer's upload

    def _setup(self, stereo, H: int, W: int) -> None:
        """static buffers for one image shape and camera"""
        from . import posenet
        dev, ops = self.device, self.ops
        meta, K, bl_fx = self.motion._camera(stereo)
        mmargin, mcrop = self.matcher.geometry(H, W)
        dmargin, dcrop = self.depth.geometry(H, W)
        nan = lambda c: torch.full((1, c, H, W), float("nan"), dtype=torch.float32, device=dev)
        inp = torch.empty((1, 5, ops.POSENET_H, ops.POSENET_W), dtype=torch.float32, device=dev)
        inp[:, 3:5] = posenet.intrinsic_layer(meta.height, meta.width, *K[:2], *K[2:], dev)
        dimg = torch.empty((2, 3, H, W), dtype=torch.float32, device=dev)          # [L(t), R(t)]
        self._st = {
            "shape": (H, W), "K": K, "bl_fx": bl_fx, "dimg": dimg,
            "mimg": torch.empty((2, 3, H, W), dtype=torch.float32, device=dev),    # [L(t-1), L(t)]
            "mmargin": mmargin, "mcrop": mcrop, "flow": nan(2), "inp": inp,
            "dst": {"margin": dmargin, "crop": dcrop, "bf": bl_fx, "kernel": None, "images": dimg, "depth": nan(1),
                    "var": None},
            "prev": torch.empty((7,), dtype=torch.float64, device=dev),             # the previous pose, widened
            "next": torch.empty((7,), dtype=torch.float64, device=dev),             # the head's output
            "pose": torch.empty((7,), dtype=torch.float32, device=dev),             # the head's output, rounded to fp32
        }

    def _check(self, H: int, W: int, K, bl_fx: float) -> None:
        st = self._st
        assert (H, W) == st["shape"], f"image shape changed since the CUDA graph was captured: {(H, W)} != {st['shape']}"
        assert K == st["K"], "camera intrinsics changed since the CUDA graph was captured"
        assert bl_fx == st["bl_fx"], "camera baseline * fx changed since the CUDA graph was captured"

    def _upload(self, stereo) -> int:
        """L(t), R(t) -> dimg on the current stream; returns 1 if the host waited for a staging buffer"""
        st, dimg = self._st, self._st["dimg"]
        imgs = (stereo.imageL, stereo.imageR)
        if all(t.is_cuda or t.is_pinned() for t in imgs):
            for i, t in enumerate(imgs):
                dimg[i:i + 1].copy_(t, non_blocking=True)
            return 0
        if self._staging is None:
            self._staging = [torch.empty(dimg.shape, dtype=torch.float32).pin_memory() for _ in range(2)]
        slot = self.num_keyframes & 1
        waited = 0
        ev = self._staged[slot]
        if ev is not None and not ev.query():       # the upload two keyframes ago still reads this buffer
            ev.synchronize()
            waited = 1
        buf = self._staging[slot]
        for i, t in enumerate(imgs):
            buf[i:i + 1].copy_(t)
        dimg.copy_(buf, non_blocking=True)
        ev = self._staged[slot] = torch.cuda.Event()
        ev.record()
        return waited

    def _networks(self) -> torch.Tensor:
        """both branches, joined, and the pose network up to fc1 (returned); on the current stream"""
        st, ops = self._st, self.ops
        main = torch.cuda.current_stream()
        self.side.wait_stream(main)
        with _deterministic_cudnn():
            with torch.cuda.stream(self.side):
                self.matcher._run(st["mimg"], st["flow"], st["mmargin"], st["mcrop"])
            self.depth._run(st["dst"])
        main.wait_stream(self.side)
        ops.posenet_input(st["flow"], st["dst"]["depth"], st["bl_fx"], st["inp"])
        return self.motion.net.body(st["inp"])

    def _keyframe(self) -> None:
        """one keyframe's work after the upload: L(t-1), L(t) into the matcher's input, the networks, the head"""
        st = self._st
        st["mimg"][0].copy_(st["mimg"][1])
        st["mimg"][1].copy_(st["dimg"][0])
        fc1 = self._networks()
        self.motion.head(fc1, st["prev"], st["next"])
        st["pose"].copy_(st["next"])
        st["prev"].copy_(st["pose"])

    def _capture(self):
        """warm up the networks (cuDNN's algorithm choice) outside the capture, then capture `_keyframe`; returns a
        callable that replays it"""
        ops = self.ops
        warm = torch.cuda.Stream(self.device)
        warm.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(warm):
            self._networks()
        torch.cuda.current_stream().wait_stream(warm)
        graph = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES[0]
        with torch.cuda.graph(graph):
            self._keyframe()
        launches = ops.LAUNCHES[0] - n0

        def replay():
            graph.replay()
            ops.LAUNCHES[0] += launches
        return replay

    @torch.inference_mode()
    def run(self, frame) -> None:
        stereo = frame.stereo
        record = {"K": stereo.K, "baseline": stereo.baseline, "time_ns": stereo.time_ns}
        if frame.frame_idx % self.keyframe_freq != 0:
            assert self.frames, "the first frame must be a keyframe"
            prev = self.frames[-1]
            self.frames.append(dict(record, T_BS=prev["T_BS"], need_interp=True, row=prev["row"]))
            self.host_waits.append(0)
            return
        H, W = stereo.imageL.shape[-2:]
        assert stereo.imageL.size(0) == 1 and stereo.imageR.size(0) == 1, \
            "The interface will not handle batch dimension correctly."
        assert tuple(stereo.imageR.shape[-2:]) == (H, W), "both images must have the same size"
        first = self._st is None
        if first:
            self._setup(stereo, H, W)
        else:
            _, K, bl_fx = self.motion._camera(stereo)
            self._check(H, W, K, bl_fx)
        st, k = self._st, self.num_keyframes
        if k == self.traj.size(0):
            grown = torch.empty((2 * k, 7), dtype=torch.float32, device=self.device)
            grown[:k].copy_(self.traj)
            self.traj = grown
        waited = self._upload(stereo)
        if first:
            st["mimg"][1].copy_(st["dimg"][0])
            st["pose"].zero_()[6].fill_(1.0)                  # the identity, [t, q_xyzw]
            st["prev"].copy_(st["pose"])
        else:
            kernel = bool(torch.backends.cudnn.allow_tf32)        # B200_TartanVODepth's head path for this flag
            if kernel != st["dst"]["kernel"]:
                st["dst"]["kernel"], self._graph = kernel, None
            if not self.cuda_graph:
                self._keyframe()
            else:
                if self._graph is None:
                    self._graph = self._capture()
                self._graph()
        self.traj[k].copy_(st["pose"])
        self.frames.append(dict(record, T_BS=stereo.T_BS, need_interp=False, row=k))
        self.num_keyframes = k + 1
        self.host_waits.append(waited)

    def finish(self) -> tuple[torch.Tensor, torch.Tensor]:
        """(F, 7) fp32 poses [t, q_xyzw] and (F,) bool need_interp, on the host; waits for the device once"""
        torch.cuda.current_stream().synchronize()
        traj = self.traj[:self.num_keyframes].cpu()
        rows = torch.tensor([f["row"] for f in self.frames], dtype=torch.long)
        interp = torch.tensor([f["need_interp"] for f in self.frames], dtype=torch.bool)
        return traj[rows], interp
