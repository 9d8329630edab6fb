"""ctypes binding of libmacvo_b200.so (the C ABI in include/macvo_b200.h) for torch CUDA tensors.

PyTorch only supplies device memory and the current stream here; every operator below is a
hand-written sm_90a kernel. There is NO CPU / eager fallback: if the library is missing or the
tensors are not on a CUDA device the call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

from .build import LIB_PATH

Tensor = torch.Tensor

CORR_SIMT, CORR_TC_3XF16, CORR_TC_1XF16, CORR_TC_TF32 = 0, 1, 2, 3
CORR_MODE_NAMES = {0: "simt", 1: "tc3", 2: "tc1", 3: "tf32"}
CORR_KMAJOR_INPUT = 16      # OR-ed into the mode: operands given K-major (channels_last features)
PGO_ACC = 55

_lib = None
_lock = threading.Lock()
LAUNCHES = [0]      # number of macvo_b200 kernels enqueued through this module (bench.py's `gpu_launches`)


class MacvoB200Error(RuntimeError):
    pass


class _ScoreT(C.Structure):
    _fields_ = [("score_cov", C.c_void_p), ("quality", C.c_void_p), ("nms", C.c_void_p),
                ("cand_vals", C.c_void_p), ("n_cand", C.c_void_p), ("ksize", C.c_int),
                ("depth_cov0", C.c_void_p), ("depth_cov1", C.c_void_p), ("flow_quality", C.c_void_p),
                ("cand_vals2", C.c_void_p)]


class _ObserveExt(C.Structure):
    _fields_ = [("depth_cov0", C.c_void_p), ("depth_cov1", C.c_void_p), ("simple_depth", C.c_int),
                ("min_depth", C.c_float), ("max_depth", C.c_float), ("front_of_cam", C.c_int), ("icp", C.c_int),
                ("cov_model", C.c_int), ("cov_ops", C.c_int * 2), ("n_cov_ops", C.c_int)]


class _PgoParams(C.Structure):
    _fields_ = [("max_steps", C.c_int), ("patience", C.c_int), ("max_reject", C.c_int), ("cluster", C.c_int),
                ("decreasing", C.c_double), ("huber_delta", C.c_double), ("radius", C.c_double),
                ("diag_min", C.c_double), ("diag_max", C.c_double)]


EXPORTS = {
    "macvo_b200_version": (C.c_char_p, []),
    "macvo_corr_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "macvo_corr_build": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 4 + [C.c_void_p, C.c_size_t, C.c_void_p]),
    "macvo_corr_lookup": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 5 + [C.c_void_p]),
    "macvo_corr_lookup_rows": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 5 + [C.c_void_p]),
    "macvo_dense_postproc": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_double] * 2 + [C.c_void_p] * 5
                             + [C.POINTER(_ScoreT), C.c_void_p]),
    "macvo_select_workspace_bytes": (C.c_size_t, [C.c_int] * 2),
    "macvo_select_candidates": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_double] + [C.c_void_p] * 5
                                + [C.c_size_t, C.c_void_p]),
    "macvo_select_candidates_depth": (C.c_int, [C.c_void_p] * 10 + [C.c_int] * 3 + [C.c_double] * 3 + [C.c_void_p] * 5
                                      + [C.c_size_t, C.c_void_p]),
    "macvo_select_mapping_candidates": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 3 + [C.c_float] * 2
                                        + [C.c_void_p] * 3 + [C.c_size_t, C.c_void_p]),
    "macvo_gather_pixels": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p] * 2),
    "macvo_retrieve_pixels": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p] + [C.c_int] * 3 + [C.c_void_p] * 2),
    "macvo_match_covariance": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                         C.c_longlong, C.c_longlong, C.c_void_p]
                               + [C.c_float] * 4 + [C.c_int] + [C.c_float] * 3 + [C.c_void_p] * 4),
    "macvo_pgo_solve": (C.c_int, [C.c_void_p] * 5 + [C.c_int] + [C.c_void_p] * 2 + [C.POINTER(_PgoParams)]
                        + [C.c_void_p] * 2),
    "macvo_pgo_solve_graph": (C.c_int, [C.c_int] + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 2 + [C.POINTER(_PgoParams)]
                              + [C.c_void_p] * 2),
    "macvo_pgo_solve_counted": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 2
                                + [C.POINTER(_PgoParams)] + [C.c_void_p] * 2 + [C.c_int] + [C.c_void_p] * 3),
    "macvo_motion_interpolate_workspace_bytes": (C.c_size_t, [C.c_int]),
    "macvo_motion_interpolate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "macvo_cov_sanity_filter": (C.c_int, [C.c_void_p] * 2 + [C.c_int] + [C.c_void_p] * 2),
    "macvo_cov_modify": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "macvo_observe_workspace_bytes": (C.c_size_t, [C.c_int]),
    "macvo_observe_packed_doubles": (C.c_size_t, [C.c_int, C.c_int]),
    "macvo_observe_pack": (C.c_int, [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int] * 3 + [C.c_void_p] * 2
                           + [C.c_int] + [C.c_float] * 3 + [C.c_void_p] * 6 + [C.c_size_t, C.c_void_p]
                           + [C.POINTER(_ObserveExt)]),
    "macvo_pgo_exchange_bytes": (C.c_size_t, [C.c_int]),
    "macvo_p2p_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p), C.c_char_p]),
    "macvo_p2p_open": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "macvo_p2p_close": (C.c_int, [C.c_void_p]),
    "macvo_p2p_free": (C.c_int, [C.c_void_p]),
    "macvo_pgo_solve_sharded": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 2
                                + [C.POINTER(_PgoParams)] + [C.c_void_p] * 2 + [C.c_int, C.c_int, C.c_void_p]),
    "macvo_pgo_accumulate": (C.c_int, [C.c_void_p] * 5 + [C.c_int] + [C.c_void_p] * 2 + [C.c_double]
                             + [C.c_void_p] * 2),
    "macvo_layer_norm": (C.c_int, [C.c_void_p] * 4 + [C.c_longlong, C.c_int, C.c_float, C.c_void_p]),
    "macvo_add_layer_norm": (C.c_int, [C.c_void_p] * 6 + [C.c_longlong, C.c_int, C.c_float, C.c_void_p]),
    "macvo_mlp_tc": (C.c_int, [C.c_void_p] * 7 + [C.c_int] * 3 + [C.c_void_p]),
    "macvo_patch_tokens_tc": (C.c_int, [C.c_void_p] * 8 + [C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "macvo_patch_embed_conv1": (C.c_int, [C.c_void_p] * 4 + [C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "macvo_add_rows_relu": (C.c_int, [C.c_void_p] * 2 + [C.c_longlong, C.c_int, C.c_int, C.c_void_p]),
    "macvo_small_attention": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 7 + [C.c_void_p]),
    "macvo_small_attention_ex": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 10 + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]),
    "macvo_latent_pool": (C.c_int, [C.c_void_p] * 5 + [C.c_longlong, C.c_int, C.c_void_p]),
    "macvo_decoder_token_blob_floats": (C.c_size_t, []),
    "macvo_decoder_token": (C.c_int, [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "macvo_decoder_token_rows": (C.c_int, [C.c_void_p] * 6 + [C.c_int] * 3 + [C.c_float, C.c_void_p]),
    "macvo_gru_input": (C.c_int, [C.c_void_p] * 7 + [C.c_longlong, C.c_void_p]),
    "macvo_gru_gates": (C.c_int, [C.c_void_p] * 5 + [C.c_longlong, C.c_void_p]),
    "macvo_gru_blend": (C.c_int, [C.c_void_p] * 5 + [C.c_longlong, C.c_void_p]),
    "macvo_softmax_rows_f16": (C.c_int, [C.c_void_p] * 2 + [C.c_longlong, C.c_int, C.c_void_p]),
    "macvo_convex_upsample": (C.c_int, [C.c_void_p] * 3 + [C.c_float] + [C.c_int] * 3 + [C.c_void_p]),
    "macvo_rows_count": (C.c_size_t, [C.c_int] * 4),
    "macvo_conv_tc": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p] + [C.c_int] * 7
                      + [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p]),
    "macvo_flow_im2col": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_void_p]),
    "macvo_gru_tc_operand_rows": (C.c_size_t, [C.c_int] * 4),
    "macvo_gru_tc_stage": (C.c_int, [C.c_int] * 5 + [C.c_void_p] * 8),
    "macvo_gru_tc_pack": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p] + [C.c_int] * 6 + [C.c_void_p]),
    "macvo_gru_tc_pack_motion": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_void_p]),
    "macvo_posenet_input": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_double, C.c_void_p, C.c_void_p]),
    "macvo_posenet_conv": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 2 + [C.c_int] * 5
                           + [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "macvo_posenet_head_floats": (C.c_size_t, []),
    "macvo_posenet_head": (C.c_int, [C.c_void_p] * 6),
    "macvo_pwc_warp_corr": (C.c_int, [C.c_void_p] * 3 + [C.c_float] + [C.c_int] * 4 + [C.c_void_p] + [C.c_int] * 2
                            + [C.c_void_p]),
    "macvo_stereo_head": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 2 + [C.c_void_p] * 4 + [C.c_float] * 2 + [C.c_int] * 4
                          + [C.c_void_p] * 3),
}


def load_library(path: str | None = None):
    """dlopen the C-ABI library (no CUDA call is made) and bind every symbol of include/macvo_b200.h."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = path or os.environ.get("MACVO_B200_LIB", LIB_PATH)
        if not os.path.exists(path):
            raise MacvoB200Error(f"{path} not found: build it first with `python -m macvo_b200.build` "
                                 "(or __graft_entry__.build()); there is no CPU fallback")
        lib = C.CDLL(path)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(lib, name)       # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = lib
        return lib


def version() -> str:
    return load_library().macvo_b200_version().decode()


def _check(rc: int, what: str) -> None:
    if rc == 0:
        return
    names = {-1: "MACVO_E_ARG", -2: "MACVO_E_WORKSPACE", -3: "MACVO_E_UNSUPPORTED", -4: "MACVO_E_DRIVER"}
    raise MacvoB200Error(f"{what} failed: {names.get(rc, f'cudaError {rc}')}")


def _dev(t: Tensor, dtype, what: str) -> Tensor:
    if not isinstance(t, Tensor) or not t.is_cuda:
        raise MacvoB200Error(f"{what}: expected a CUDA tensor (the B200 path has no CPU fallback), got "
                             f"{getattr(t, 'device', type(t))}")
    if t.dtype != dtype:
        raise MacvoB200Error(f"{what}: expected {dtype}, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _stream() -> int:
    # raw cudaStream_t of torch's current stream; the public torch.cuda.current_stream() costs ~20 us of Python per call
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def _workspace(key, nbytes: int, device) -> Tensor:
    """Per-call scratch from torch's caching allocator (1024-B aligned view). Never a process-global buffer: inside a
    CUDA-graph capture the allocation comes from the graph's private pool and lives as long as the graph does, so a
    replay can never touch memory that a later, larger call re-allocated (kernel arguments and TMA tensor maps bake
    the address in); outside a capture, stream-ordered reuse by the allocator is safe for these same-stream kernels."""
    buf = torch.empty(max(nbytes, 1024) + 1024, dtype=torch.uint8, device=device)
    off = (-buf.data_ptr()) % 1024
    return buf[off:off + max(nbytes, 1)]


# ------------------------------------------------------------------------------------------------
# (a3) correlation volume
# ------------------------------------------------------------------------------------------------
def default_corr_mode(dim: int, n: int) -> int:
    """Strict fp32 (allow_tf32 off): the fp32-class 3 x fp16 split. With TF32 matmuls allowed — the reference frontend's
    own setting (Frontend.py:275-277), under which ITS `torch.matmul` for this product runs on TF32 tensor cores — one
    tf32 pass straight over the fp32 features (no operand pre-pass)."""
    env = os.environ.get("MACVO_B200_CORR_MODE")
    if env is not None:
        return {"simt": CORR_SIMT, "tc3": CORR_TC_3XF16, "tc1": CORR_TC_1XF16, "tf32": CORR_TC_TF32}[env]
    if not (dim % 64 == 0 and dim <= 256 and n % 8 == 0):
        return CORR_SIMT
    return CORR_TC_TF32 if torch.backends.cuda.matmul.allow_tf32 else CORR_TC_3XF16


def corr_build(fmap1: Tensor, fmap2: Tensor, mode: int | None = None) -> Tensor:
    """(B,D,H,W) x2 -> (B,1,H,W,H,W) fp32, `MemoryEncoder.corr` (encoder.py:256-275).

    fp16 feature maps (MACVO_Fast) use the single-pass fp16 tensor-core mode, which is exact for them."""
    lib = load_library()
    B, D, H, W = fmap1.shape
    n = H * W
    if mode is None:
        mode = default_corr_mode(D, n)
        if fmap1.dtype == torch.float16 and mode in (CORR_TC_3XF16, CORR_TC_TF32):
            mode = CORR_TC_1XF16
    f1 = fmap1.float() if fmap1.dtype != torch.float32 else fmap1
    f2 = fmap2.float() if fmap2.dtype != torch.float32 else fmap2
    cl = torch.channels_last
    kmajor = (mode != CORR_SIMT and f1.is_cuda and f2.is_cuda and not f1.is_contiguous() and not f2.is_contiguous()
              and f1.is_contiguous(memory_format=cl) and f2.is_contiguous(memory_format=cl))
    if mode == CORR_TC_TF32 and not kmajor:     # the tf32 kernel reads K-major rows in place: make them (one copy each)
        f1, f2 = f1.contiguous(memory_format=cl), f2.contiguous(memory_format=cl)
        kmajor = True
    if kmajor:      # channels_last features are already K-major (B, N, D) rows: elementwise operand split, no transpose
        f1, f2 = f1.permute(0, 2, 3, 1), f2.permute(0, 2, 3, 1)
    f1 = _dev(f1, torch.float32, "corr_build fmap1")
    f2 = _dev(f2, torch.float32, "corr_build fmap2")
    out = torch.empty((B, 1, H, W, H, W), dtype=torch.float32, device=f1.device)
    nbytes = lib.macvo_corr_workspace_bytes(B, D, n, mode)
    ws = _workspace("corr", nbytes, f1.device) if nbytes else None
    rc = lib.macvo_corr_build(f1.data_ptr(), f2.data_ptr(), out.data_ptr(), B, D, n, mode | (CORR_KMAJOR_INPUT if kmajor else 0),
                              ws.data_ptr() if ws is not None else None, nbytes, _stream())
    _check(rc, "macvo_corr_build")
    LAUNCHES[0] += {CORR_SIMT: 1, CORR_TC_TF32: 1}.get(mode, 2)
    return out


# ------------------------------------------------------------------------------------------------
# (a5) window lookup
# ------------------------------------------------------------------------------------------------
def corr_lookup(cost_maps: Tensor, coords: Tensor, rows: bool = False) -> Tensor:
    """cost_maps (B*H1*W1, 1, H2, W2) fp32, coords (B,2,H1,W1) fp32 -> (B,81,H1,W1) fp32 (decoder.py:141-153);
    rows=True: the same values as (B*H1*W1, 81) pixels-major rows (the NHWC view)."""
    lib = load_library()
    cm = _dev(cost_maps, torch.float32, "corr_lookup cost_maps")
    co = _dev(coords, torch.float32, "corr_lookup coords")
    B, _, H1, W1 = co.shape
    H2, W2 = cm.shape[-2:]
    assert cm.shape[0] == B * H1 * W1, "one cost map per query pixel"
    out = torch.empty((B * H1 * W1, 81) if rows else (B, 81, H1, W1), dtype=torch.float32, device=cm.device)
    fn = lib.macvo_corr_lookup_rows if rows else lib.macvo_corr_lookup
    _check(fn(cm.data_ptr(), co.data_ptr(), out.data_ptr(), B, H1, W1, H2, W2, _stream()), "macvo_corr_lookup")
    LAUNCHES[0] += 1
    return out


# ------------------------------------------------------------------------------------------------
# (a7) + (a8)
# ------------------------------------------------------------------------------------------------
class ScoreBuffers:
    """Device buffers filled by the fused scoring pass; consumed by `select_candidates`."""

    def __init__(self, h: int, w: int, device, ksize: int):
        self.h, self.w, self.ksize = h, w, ksize
        self.quality = torch.empty((h, w), dtype=torch.float32, device=device)
        self.nms = torch.empty((h, w), dtype=torch.uint8, device=device)
        self.cand_vals = torch.empty((h * w,), dtype=torch.float32, device=device)
        self.n_cand = torch.zeros((1,), dtype=torch.int32, device=device)
        self.generation = 0        # bumped by whoever refills the buffers (host-side bookkeeping)

        self.flow_quality = None   # depth-aware variant only (allocated on first use)
        self.cand_vals2 = None

    def struct(self, score_cov_ptr, dcov0=None, dcov1=None) -> _ScoreT:
        if dcov0 is not None and self.flow_quality is None:
            self.flow_quality = torch.empty_like(self.quality)
            self.cand_vals2 = torch.empty_like(self.cand_vals)
        return _ScoreT(score_cov_ptr, self.quality.data_ptr(), self.nms.data_ptr(), self.cand_vals.data_ptr(),
                       self.n_cand.data_ptr(), self.ksize,
                       dcov0.data_ptr() if dcov0 is not None else None, dcov1.data_ptr() if dcov1 is not None else None,
                       self.flow_quality.data_ptr() if dcov0 is not None else None,
                       self.cand_vals2.data_ptr() if dcov0 is not None else None)


def dense_postproc(est_flow: Tensor, est_cov: Tensor | None, bl_fx: float, enforce_positive_disparity: bool = False,
                   score: ScoreBuffers | None = None) -> dict:
    """One `estimate_pair` of dense maps (Frontend.py:184-200, 291-299) + optional fused keypoint scoring.

    est_flow / est_cov: (2,2,H,W) fp32. bl_fx = baseline*fx as a python float (double), like the reference.
    est_cov None (a frontend without covariance, FlowFormerDepth / FlowFormerMatcher): est_flow (1|2,2,H,W); depth and
    disparity of slot 0, the flow of slot 1 (None for one slot); every covariance / mask output is None."""
    lib = load_library()
    fl = _dev(est_flow, torch.float32, "dense_postproc est_flow")
    if est_cov is None:
        if enforce_positive_disparity or score is not None or fl.dim() != 4 or fl.shape[0] not in (1, 2) or fl.shape[1] != 2:
            raise MacvoB200Error("dense_postproc without est_cov: expects est_flow (1|2,2,H,W) and no mask or scoring")
        H, W = fl.shape[-2:]
        depth = torch.empty((1, 1, H, W), dtype=torch.float32, device=fl.device)
        disparity = torch.empty_like(depth)
        _check(lib.macvo_dense_postproc(fl.data_ptr(), None, H, W, float(bl_fx), float(bl_fx) ** 2, depth.data_ptr(),
                                        disparity.data_ptr(), None, None, None, None, _stream()), "macvo_dense_postproc")
        LAUNCHES[0] += 1
        return {"depth": depth, "disparity": disparity, "depth_cov": None, "disparity_uncertainty": None, "depth_mask": None,
                "flow": fl[1:2] if fl.shape[0] == 2 else None, "flow_cov": None}
    cv = _dev(est_cov, torch.float32, "dense_postproc est_cov")
    assert fl.shape[:2] == (2, 2) and cv.shape == fl.shape
    H, W = fl.shape[-2:]
    dev = fl.device
    depth = torch.empty((1, 1, H, W), dtype=torch.float32, device=dev)
    disparity = torch.empty_like(depth)
    depth_cov = torch.empty_like(depth)
    mask = torch.empty((1, 1, H, W), dtype=torch.uint8, device=dev) if enforce_positive_disparity else None
    flow_cov = torch.empty((1, 3, H, W), dtype=torch.float32, device=dev)
    st = None
    if score is not None:
        score.n_cand.zero_()
        st = score.struct(None)
    rc = lib.macvo_dense_postproc(fl.data_ptr(), cv.data_ptr(), H, W, float(bl_fx), float(bl_fx) ** 2,
                                  depth.data_ptr(), disparity.data_ptr(), depth_cov.data_ptr(),
                                  mask.data_ptr() if mask is not None else None, flow_cov.data_ptr(),
                                  C.byref(st) if st is not None else None, _stream())
    _check(rc, "macvo_dense_postproc")
    LAUNCHES[0] += 1
    return {"depth": depth, "disparity": disparity, "depth_cov": depth_cov,
            "disparity_uncertainty": cv[0:1, :1], "depth_mask": mask.bool() if mask is not None else None,
            "flow": fl[1:2], "flow_cov": flow_cov}


def score_only(match_cov: Tensor, score: ScoreBuffers) -> None:
    """Quality / NMS scoring of an arbitrary (1,3,H,W) covariance map (standalone selector plugin)."""
    lib = load_library()
    mc = _dev(match_cov, torch.float32, "score_only match_cov")
    H, W = mc.shape[-2:]
    score.n_cand.zero_()
    st = score.struct(mc.data_ptr())
    rc = lib.macvo_dense_postproc(None, None, H, W, 0.0, 0.0, None, None, None, None, None, C.byref(st), _stream())
    _check(rc, "macvo_dense_postproc(score)")
    LAUNCHES[0] += 1
    score.generation += 1


def score_depth_aware(match_cov: Tensor, depth_cov0: Tensor, depth_cov1: Tensor, score: ScoreBuffers) -> None:
    """Scoring of the depth-aware selector: quality = (depth_cov0 + depth_cov1) * (uu + vv - 2 uv) + NMS."""
    lib = load_library()
    mc = _dev(match_cov, torch.float32, "score_depth_aware match_cov")
    d0 = _dev(depth_cov0, torch.float32, "score_depth_aware depth_cov0")
    d1 = _dev(depth_cov1, torch.float32, "score_depth_aware depth_cov1")
    H, W = mc.shape[-2:]
    score.n_cand.zero_()
    st = score.struct(mc.data_ptr(), d0, d1)
    rc = lib.macvo_dense_postproc(None, None, H, W, 0.0, 0.0, None, None, None, None, None, C.byref(st), _stream())
    _check(rc, "macvo_dense_postproc(score, depth-aware)")
    LAUNCHES[0] += 1
    score.generation += 1


def select_candidates_depth(score: ScoreBuffers, depth0: Tensor, depth1: Tensor, depth_cov0: Tensor, mask_width: int,
                            max_depth: float, max_depth_cov: float, max_match_cov: float, mask_a: Tensor | None,
                            mask_b: Tensor | None, out: "CandidateList") -> None:
    lib = load_library()
    h, w = score.h, score.w
    nbytes = lib.macvo_select_workspace_bytes(h, w)
    ws = _workspace("select", nbytes, score.quality.device)
    u8 = lambda m: None if m is None else _dev(m.to(torch.uint8) if m.dtype != torch.uint8 else m, torch.uint8, "mask")
    ma, mb = u8(mask_a), u8(mask_b)
    d0, d1 = _dev(depth0, torch.float32, "depth0"), _dev(depth1, torch.float32, "depth1")
    dc0 = _dev(depth_cov0, torch.float32, "depth_cov0")
    if out.thresh.numel() < 2:
        out.thresh = torch.zeros((2,), dtype=torch.float32, device=out.thresh.device)
    rc = lib.macvo_select_candidates_depth(score.flow_quality.data_ptr(), d0.data_ptr(), d1.data_ptr(), dc0.data_ptr(),
                                           score.nms.data_ptr(), score.cand_vals.data_ptr(), score.cand_vals2.data_ptr(),
                                           score.n_cand.data_ptr(), ma.data_ptr() if ma is not None else None,
                                           mb.data_ptr() if mb is not None else None, h, w, int(mask_width),
                                           float(max_depth), float(max_depth_cov), float(max_match_cov),
                                           out.idx.data_ptr(), out.n.data_ptr(), out.thresh.data_ptr(),
                                           out.status.data_ptr(), ws.data_ptr(), nbytes, _stream())
    _check(rc, "macvo_select_candidates_depth")
    LAUNCHES[0] += 4


class CandidateList:
    def __init__(self, h: int, w: int, device):
        self.idx = torch.empty((h * w,), dtype=torch.int32, device=device)
        self.n = torch.zeros((1,), dtype=torch.int32, device=device)
        self.thresh = torch.zeros((1,), dtype=torch.float32, device=device)
        self.status = torch.zeros((1,), dtype=torch.int32, device=device)
        self.host = torch.zeros((2,), dtype=torch.int32).pin_memory()      # [n, status]
        self.perm_host = torch.empty((4096,), dtype=torch.int64).pin_memory()   # staging for the sampled permutation
        self.w = w


def select_candidates(score: ScoreBuffers, mask_width: int, max_match_cov: float, extra_mask: Tensor | None,
                      out: CandidateList) -> None:
    lib = load_library()
    h, w = score.h, score.w
    nbytes = lib.macvo_select_workspace_bytes(h, w)
    ws = _workspace("select", nbytes, score.quality.device)
    em = None
    if extra_mask is not None:
        em = _dev(extra_mask.to(torch.uint8) if extra_mask.dtype != torch.uint8 else extra_mask, torch.uint8, "extra_mask")
    rc = lib.macvo_select_candidates(score.quality.data_ptr(), score.nms.data_ptr(), score.cand_vals.data_ptr(),
                                     score.n_cand.data_ptr(), em.data_ptr() if em is not None else None, h, w,
                                     int(mask_width), float(max_match_cov), out.idx.data_ptr(), out.n.data_ptr(),
                                     out.thresh.data_ptr(), out.status.data_ptr(), ws.data_ptr(), nbytes, _stream())
    _check(rc, "macvo_select_candidates")
    LAUNCHES[0] += 3


def select_mapping_candidates(depth: Tensor, depth_cov: Tensor, mask_width: int, max_depth: float,
                              max_depth_cov: float, out: CandidateList) -> None:
    lib = load_library()
    d = _dev(depth, torch.float32, "mapping depth")
    dc = _dev(depth_cov, torch.float32, "mapping depth_cov")
    h, w = d.shape[-2:]
    nbytes = lib.macvo_select_workspace_bytes(h, w)
    ws = _workspace("select", nbytes, d.device)
    out.status.zero_()
    rc = lib.macvo_select_mapping_candidates(d.data_ptr(), dc.data_ptr(), h, w, int(mask_width), float(max_depth),
                                             float(max_depth_cov), out.idx.data_ptr(), out.n.data_ptr(),
                                             ws.data_ptr(), nbytes, _stream())
    _check(rc, "macvo_select_mapping_candidates")
    LAUNCHES[0] += 2


def sample_candidates(cand: CandidateList, num_point: int) -> Tensor:
    """`perm = torch.randperm(n)[:numPoint]` on the CPU default generator (KeypointSelector.py:404) — the one
    host round trip of the selector (the reference has two: `.item()` and `nonzero`)."""
    return sample_candidates_many([(cand, num_point)])[0]


def request_candidate_counts(requests: list[tuple[CandidateList, int]]) -> torch.cuda.Event:
    """enqueue the device->host copies of every list's count / status; the returned event fires when they have landed"""
    for cand, _ in requests:
        cand.host[0:1].copy_(cand.n, non_blocking=True)
        cand.host[1:2].copy_(cand.status, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    return ev


def sample_from_counts(requests: list[tuple[CandidateList, int]]) -> list[Tensor]:
    """after the event of `request_candidate_counts` fired: `torch.randperm(n)[:numPoint]` per list IN THE GIVEN ORDER from the
    CPU default generator (the order MAC-VO consumes it: keypoints, then mapping points — Odometry/MACVO.py:197,315) and the
    gathers of the drawn candidates on the current stream"""
    lib = load_library()
    outs = []
    for cand, num_point in requests:
        dev = cand.idx.device
        n = int(cand.host[0])   # host[1] = 1 flags "no NMS survivor" (then n == 0, like the reference: median([]) = nan)
        perm = torch.randperm(n)[:num_point]
        k = perm.numel()
        out = torch.empty((k, 2), dtype=torch.int64, device=dev)
        if k:
            if k > cand.perm_host.numel():                           # (pinning per call costs ~0.1 ms: keep a buffer)
                cand.perm_host = torch.empty((k,), dtype=torch.int64).pin_memory()
            cand.perm_host[:k].copy_(perm)
            perm_d = cand.perm_host[:k].to(dev, non_blocking=True)
            _check(lib.macvo_gather_pixels(cand.idx.data_ptr(), perm_d.data_ptr(), k, cand.w, out.data_ptr(), _stream()),
                   "macvo_gather_pixels")
            LAUNCHES[0] += 1
        outs.append(out)
    return outs


def sample_candidates_many(requests: list[tuple[CandidateList, int]]) -> list[Tensor]:
    """Sampling for several candidate lists behind ONE host synchronisation: the counts of all lists are fetched
    together, then drawn per list in the given order (see `sample_from_counts`)."""
    request_candidate_counts(requests).synchronize()
    return sample_from_counts(requests)


# ------------------------------------------------------------------------------------------------
# (a9) retrieve_pixels
# ------------------------------------------------------------------------------------------------
def retrieve_pixels(pixel_uv: Tensor, scalar_map: Tensor) -> Tensor:
    lib = load_library()
    sm = _dev(scalar_map, torch.float32, "retrieve_pixels map")
    if pixel_uv.dtype not in (torch.int64, torch.float32):
        pixel_uv = pixel_uv.float()
    kp = _dev(pixel_uv, pixel_uv.dtype, "retrieve_pixels kp")
    Cc, H, W = sm.shape[-3:]
    K = kp.shape[0]
    out = torch.empty((Cc, K), dtype=torch.float32, device=sm.device)
    _check(lib.macvo_retrieve_pixels(kp.data_ptr(), int(kp.dtype == torch.int64), K, sm.data_ptr(), Cc, H, W,
                                     out.data_ptr(), _stream()), "macvo_retrieve_pixels")
    LAUNCHES[0] += 1
    return out


# ------------------------------------------------------------------------------------------------
# (a10)
# ------------------------------------------------------------------------------------------------
def match_covariance(kp: Tensor, depth_map: Tensor, flow_cov: Tensor | None, fx: float, fy: float, cx: float,
                     cy: float, kernel_size: int = 31, min_flow_cov: float = 0.25, min_depth_cov: float = 0.05,
                     match_cov_default: float = 0.25, want_point: bool = False, depth_cov: Tensor | None = None,
                     out_cov: Tensor | None = None):
    """-> (cov (K,3,3) float64 on the device, point (K,3) fp32 or None, status int32 tensor).

    flow_cov: (K,3) fp32 CUDA tensor with ANY strides (MAC-VO passes the transposed view of a (3,K) gather,
    Odometry/MACVO.py:231-232); its first two columns are clamped in place in the caller's storage like the reference.
    depth_cov: (K,) per-keypoint depth variance, only used when flow_cov is None (Project2to3.py:163-171).
    out_cov: optional preallocated (K,3,3) float64 CUDA view to fill (e.g. a slice of a packed buffer)."""
    lib = load_library()
    dm = _dev(depth_map, torch.float32, "match_covariance depth")
    if kp.dtype not in (torch.int64, torch.float32):
        kp = kp.float()
    kpd = _dev(kp, kp.dtype, "match_covariance kp")
    K = kpd.shape[0]
    H, W = dm.shape[-2:]
    fc, rs, cs = None, 0, 0
    if flow_cov is not None:
        if not (flow_cov.is_cuda and flow_cov.dtype == torch.float32 and flow_cov.dim() == 2 and flow_cov.shape == (K, 3)):
            raise MacvoB200Error("match_covariance: flow_cov must be a (K,3) fp32 CUDA tensor (clamped in place)")
        fc = flow_cov
        rs, cs = (fc.stride(0), fc.stride(1)) if K > 0 else (3, 1)
        if K > 0 and (rs == 0 or cs == 0):
            raise MacvoB200Error("match_covariance: flow_cov is an expanded (stride-0) view; the in-place clamp needs real storage")
    dv = None
    if fc is None and depth_cov is not None:
        dv = _dev(depth_cov.reshape(-1), torch.float32, "match_covariance depth_cov")
        if dv.numel() != K:
            raise MacvoB200Error("match_covariance: depth_cov must have one value per keypoint")
    if out_cov is None:
        cov = torch.empty((K, 3, 3), dtype=torch.float64, device=dm.device)
    else:
        cov = out_cov
        if not (cov.is_cuda and cov.dtype == torch.float64 and cov.is_contiguous() and cov.shape == (K, 3, 3)):
            raise MacvoB200Error("match_covariance: out_cov must be a contiguous (K,3,3) float64 CUDA tensor")
    pt = torch.empty((K, 3), dtype=torch.float32, device=dm.device) if want_point else None
    status = torch.zeros((1,), dtype=torch.int32, device=dm.device)
    rc = lib.macvo_match_covariance(kpd.data_ptr(), int(kpd.dtype == torch.int64), K, dm.data_ptr(), H, W,
                                    fc.data_ptr() if fc is not None else None, rs, cs,
                                    dv.data_ptr() if dv is not None else None, fx, fy, cx, cy, kernel_size,
                                    min_flow_cov, min_depth_cov, match_cov_default, cov.data_ptr(),
                                    pt.data_ptr() if pt is not None else None, status.data_ptr(), _stream())
    _check(rc, "macvo_match_covariance")
    LAUNCHES[0] += 1
    return cov, pt, status


# ------------------------------------------------------------------------------------------------
# (a14) + (a15)
# ------------------------------------------------------------------------------------------------
def _pgo_params(max_steps=10, patience=2, max_reject=16, cluster=0, decreasing=1e-5, huber_delta=0.1, radius=1e3,
                diag_min=1e-6, diag_max=1e32) -> _PgoParams:
    return _PgoParams(max_steps, patience, max_reject, cluster, decreasing, huber_delta, radius, diag_min, diag_max)


def pgo_solve(pos_Tw: Tensor, kp2_uv: Tensor, kp2_disp: Tensor, uv_cov: Tensor, disp_cov: Tensor,
              intr: tuple[float, float, float, float, float], init_pose: Tensor, cluster: int = 0, **kw):
    """All inputs CUDA float64. Returns (pose (7,) float64 CUDA, stats (8,) float64 CUDA); asynchronous."""
    lib = load_library()
    P = [_dev(t, torch.float64, f"pgo_solve arg{i}") for i, t in enumerate((pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov))]
    K = P[0].shape[0]
    pose = _dev(init_pose, torch.float64, "pgo_solve init_pose").reshape(7).clone()
    stats = torch.zeros((8,), dtype=torch.float64, device=pose.device)
    intr_c = (C.c_double * 5)(*[float(v) for v in intr])
    prm = _pgo_params(cluster=cluster, **kw)
    rc = lib.macvo_pgo_solve(*(t.data_ptr() for t in P), K, C.cast(intr_c, C.c_void_p), pose.data_ptr(),
                             C.byref(prm), stats.data_ptr(), _stream())
    _check(rc, "macvo_pgo_solve")
    LAUNCHES[0] += 1
    return pose, stats


PGO_GRAPH_TYPES = {"disp": 0, "reproj": 1, "icp": 2}


def pgo_solve_graph(graph_type: str, pos_Tw: Tensor, intr: tuple[float, float, float, float, float], init_pose: Tensor,
                    kp2_uv: Tensor | None = None, kp2_disp: Tensor | None = None, uv_cov: Tensor | None = None,
                    disp_cov: Tensor | None = None, pc_obs: Tensor | None = None, obs_cov: Tensor | None = None,
                    pts_cov: Tensor | None = None, cluster: int = 0, **kw):
    """TwoFrame_PGO for any of its graph types ("disp" | "reproj" | "icp", Optimizer.py:51-68); CUDA float64 inputs."""
    lib = load_library()
    gt = PGO_GRAPH_TYPES[graph_type]
    d = lambda t, w: None if t is None else _dev(t, torch.float64, f"pgo_solve_graph {w}")
    pos = d(pos_Tw, "pos_Tw")
    arrs = [d(kp2_uv, "kp2_uv"), d(kp2_disp, "kp2_disp"), d(uv_cov, "uv_cov"), d(disp_cov, "disp_cov"), d(pc_obs, "pc_obs"),
            d(obs_cov, "obs_cov"), d(pts_cov, "pts_cov")]
    K = pos.shape[0]
    pose = _dev(init_pose, torch.float64, "pgo_solve_graph init_pose").reshape(7).clone()
    stats = torch.zeros((8,), dtype=torch.float64, device=pose.device)
    intr_c = (C.c_double * 5)(*[float(v) for v in intr])
    prm = _pgo_params(cluster=cluster, **kw)
    rc = lib.macvo_pgo_solve_graph(gt, pos.data_ptr(), *(None if a is None else a.data_ptr() for a in arrs), K,
                                   C.cast(intr_c, C.c_void_p), pose.data_ptr(), C.byref(prm), stats.data_ptr(), _stream())
    _check(rc, "macvo_pgo_solve_graph")
    LAUNCHES[0] += 1
    return pose, stats


def pgo_accumulate(pos_Tw: Tensor, kp2_uv: Tensor, kp2_disp: Tensor, uv_cov: Tensor, disp_cov: Tensor,
                   intr: tuple[float, float, float, float, float], pose: Tensor, huber_delta: float = 0.1) -> Tensor:
    lib = load_library()
    P = [_dev(t, torch.float64, f"pgo_accumulate arg{i}") for i, t in enumerate((pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov))]
    K = P[0].shape[0]
    ps = _dev(pose, torch.float64, "pgo_accumulate pose").reshape(7)
    acc = torch.empty((PGO_ACC,), dtype=torch.float64, device=ps.device)
    intr_c = (C.c_double * 5)(*[float(v) for v in intr])
    rc = lib.macvo_pgo_accumulate(*(t.data_ptr() for t in P), K, C.cast(intr_c, C.c_void_p), ps.data_ptr(),
                                  float(huber_delta), acc.data_ptr(), _stream())
    _check(rc, "macvo_pgo_accumulate")
    LAUNCHES[0] += 1
    return acc


# ------------------------------------------------------------------------------------------------
# (f3) device-side observation building / sanity filter / MatchObs packing + counted PGO solve
# ------------------------------------------------------------------------------------------------
class ObservationBuffers:
    """Device + pinned-host buffers of one frame's observations (layout: include/macvo_b200.h, macvo_observe_pack).
    `extended`: room for the columns the "icp" graph reads (pixel2_d .. cov_Tw, after the header)."""

    def __init__(self, capacity: int, device, extended: bool = False):
        lib = load_library()
        self.capacity = int(capacity)
        self.extended = bool(extended)
        self.n_doubles = int(lib.macvo_observe_packed_doubles(self.capacity, int(self.extended)))
        self.packed = torch.zeros((self.n_doubles,), dtype=torch.float64, device=device)
        self.n_obs = torch.zeros((1,), dtype=torch.int32, device=device)
        self.status = torch.zeros((1,), dtype=torch.int32, device=device)
        self.ws_bytes = int(lib.macvo_observe_workspace_bytes(self.capacity))
        self.ws = torch.empty((self.ws_bytes,), dtype=torch.uint8, device=device)
        self.host = torch.zeros((self.n_doubles,), dtype=torch.float64).pin_memory()
        self.ready = torch.cuda.Event()

    def section(self, name: str, host: bool = False) -> Tensor:
        c = self.capacity
        lo, hi, shape = {"pos_Tw": (0, 3 * c, (c, 3)), "pixel2_uv": (3 * c, 5 * c, (c, 2)), "pixel2_disp": (5 * c, 6 * c, (c,)),
                         "pixel2_uv_cov": (6 * c, 9 * c, (c, 3)), "pixel2_disp_cov": (9 * c, 10 * c, (c,)),
                         "obs1_covTc": (10 * c, 19 * c, (c, 3, 3)), "obs2_covTc": (19 * c, 28 * c, (c, 3, 3)),
                         "pixel1_uv": (28 * c, 30 * c, (c, 2)), "pixel1_d": (30 * c, 31 * c, (c,)),
                         "header": (31 * c, 31 * c + 4, (4,))}.get(name, (None, None, None))
        if lo is None and self.extended:
            e = 31 * c + 4
            lo, hi, shape = {"pixel2_d": (e, e + c, (c,)), "pixel1_d_cov": (e + c, e + 2 * c, (c,)),
                             "pixel2_d_cov": (e + 2 * c, e + 3 * c, (c,)), "points_Tc": (e + 3 * c, e + 6 * c, (c, 3)),
                             "cov_Tw": (e + 6 * c, e + 15 * c, (c, 3, 3))}.get(name, (None, None, None))
        if lo is None:
            raise KeyError(f"ObservationBuffers: no section {name!r}" + ("" if self.extended else " (not extended)"))
        return (self.host if host else self.packed)[lo:hi].view(shape)

    def download_async(self) -> None:
        """ONE asynchronous device->host copy of the whole frame's observations; `self.ready` fires when it landed."""
        self.host.copy_(self.packed, non_blocking=True)
        self.ready.record()


def motion_interpolate_(poses: Tensor, need_interp: Tensor) -> Tensor:
    """MotionInterpolate.elaborate_map (Module/MapProcessor.py:52-79) in place on (F,7) fp32 CUDA poses; need_interp (F,)
    bool / uint8. Returns the device int32 count of interpolated motions."""
    lib = load_library()
    p = poses
    if not (p.is_cuda and p.dtype == torch.float32 and p.dim() == 2 and p.shape[1] == 7 and p.is_contiguous()):
        raise MacvoB200Error("motion_interpolate_: poses must be a contiguous (F,7) fp32 CUDA tensor")
    ni = _dev(need_interp.to(torch.uint8) if need_interp.dtype != torch.uint8 else need_interp, torch.uint8, "need_interp")
    F_ = p.shape[0]
    if ni.numel() != F_:
        raise MacvoB200Error("motion_interpolate_: need_interp must have one flag per frame")
    count = torch.zeros((1,), dtype=torch.int32, device=p.device)
    nbytes = lib.macvo_motion_interpolate_workspace_bytes(F_)
    ws = _workspace("motion", nbytes, p.device) if nbytes else None
    _check(lib.macvo_motion_interpolate(p.data_ptr(), ni.data_ptr(), F_, count.data_ptr(),
                                        ws.data_ptr() if ws is not None else None, nbytes, _stream()), "macvo_motion_interpolate")
    LAUNCHES[0] += 1
    return count


def cov_sanity_filter(obs1_cov: Tensor, obs2_cov: Tensor) -> Tensor:
    """(K,3,3) float64 CUDA x2 -> bool (K,) mask of observations whose covariances are finite (OutlierFilter.py:91-100)"""
    a, b = _dev(obs1_cov, torch.float64, "cov_sanity_filter obs1"), _dev(obs2_cov, torch.float64, "cov_sanity_filter obs2")
    k = a.shape[0]
    good = torch.empty((k,), dtype=torch.uint8, device=a.device)
    _check(load_library().macvo_cov_sanity_filter(a.data_ptr(), b.data_ptr(), k, good.data_ptr(), _stream()),
           "macvo_cov_sanity_filter")
    LAUNCHES[0] += 1
    return good.bool()


COV_MODELS = {"match": 0, "identity": 1}              # macvo_observe_ext_t.cov_model (MACVO_COV_MATCH / _IDENTITY)
COV_OPS = {"diagonalize": 1, "normalize": 2}          # MACVO_COV_DIAGONALIZE / MACVO_COV_NORMALIZE


def _cov_ops(ops: list[str] | tuple[str, ...], what: str):
    bad = [o for o in ops if o not in COV_OPS]
    if bad or len(ops) > 2:
        raise MacvoB200Error(f"{what}: covariance modifiers must be at most two of {sorted(COV_OPS)}, got {list(ops)}")
    return (C.c_int * 2)(*([COV_OPS[o] for o in ops] + [0] * (2 - len(ops))))


def cov_modify(cov: Tensor, ops: list[str] | tuple[str, ...]) -> Tensor:
    """Modifier_Diagonalize / Modifier_Normalize (Project2to3.py:281-323) in place on a contiguous (K,3,3) float64 CUDA
    tensor; `ops` in the order they apply (the innermost wrapper first). Returns `cov`."""
    arr = _cov_ops(ops, "cov_modify")
    if not (isinstance(cov, Tensor) and cov.is_cuda and cov.dtype == torch.float64 and cov.is_contiguous()
            and cov.dim() == 3 and cov.shape[1:] == (3, 3)):
        raise MacvoB200Error("cov_modify: expects a contiguous (K,3,3) float64 CUDA tensor (modified in place)")
    k = cov.shape[0]
    if k and ops:
        _check(load_library().macvo_cov_modify(cov.data_ptr(), k, C.cast(arr, C.c_void_p), len(ops), _stream()),
               "macvo_cov_modify")
        LAUNCHES[0] += 1
    return cov


def observe_pack(buf: ObservationBuffers, kp0_uv: Tensor, flow: Tensor, match_cov: Tensor | None, depth0: Tensor, depth1: Tensor,
                 disparity1: Tensor, disp_unc1: Tensor | None, edge_width: int, intr0, intr1, prev_pose: Tensor, next_pose: Tensor,
                 kernel_size: int = 31, min_flow_cov: float = 0.25, min_depth_cov: float = 0.05,
                 match_cov_default: float = 0.25, ext: dict | None = None) -> None:
    """Odometry/MACVO.py:198-283 for the two-frame graph as two launches (csrc/observe.cu); everything stays on the device.

    ext (None: CovarianceSanityFilter only) = macvo_observe_ext_t as a dict: depth_cov0 / depth_cov1 ((1,1,H,W) fp32 CUDA
    or None), simple_depth (bool), min_depth / max_depth (floats, rounded to fp32 like the reference's comparisons),
    front_of_cam (bool), icp (bool: pack the "icp" graph's columns; needs an extended buffer), cov_model ("match" or
    "identity", the NoCovariance model) and cov_ops (modifier names of COV_OPS, innermost first).

    match_cov and disp_unc1 both None: a frontend without covariance maps (pixel2_uv_cov / pixel2_disp_cov hold -1, kp1's
    MatchCovariance uses match_cov_default unclamped; include/macvo_b200.h)."""
    lib = load_library()
    kp = _dev(kp0_uv, torch.int64, "observe_pack kp0_uv")
    k = kp.shape[0]
    fl = _dev(flow, torch.float32, "observe_pack flow")
    if (match_cov is None) != (disp_unc1 is None):
        raise MacvoB200Error("observe_pack: match_cov and disp_unc1 are None together (no frontend covariance) or not at all")
    mc = None if match_cov is None else _dev(match_cov, torch.float32, "observe_pack match_cov")
    maps = [None if t is None else _dev(t, torch.float32, "observe_pack map") for t in (depth0, depth1, disparity1, disp_unc1)]
    H, W = fl.shape[-2:]
    if (fl.numel() != 2 * H * W or (mc is not None and mc.numel() != 3 * H * W)
            or any(m is not None and m.numel() != H * W for m in maps)):
        raise MacvoB200Error("observe_pack: expects flow (1,2,H,W), match_cov (1,3,H,W) and (1,1,H,W) maps")
    if k > buf.capacity:
        raise MacvoB200Error(f"observe_pack: {k} keypoints exceed the buffer capacity {buf.capacity}")
    pp = _dev(prev_pose, torch.float64, "observe_pack prev_pose")
    if not (next_pose.is_cuda and next_pose.dtype == torch.float64 and next_pose.is_contiguous() and next_pose.numel() == 7):
        raise MacvoB200Error("observe_pack: next_pose must be a contiguous (7,) float64 CUDA tensor")
    i0 = (C.c_float * 4)(*[float(v) for v in intr0])
    i1 = (C.c_float * 4)(*[float(v) for v in intr1])
    xs = None
    if ext is not None:
        unknown = set(ext) - {"depth_cov0", "depth_cov1", "simple_depth", "min_depth", "max_depth", "front_of_cam", "icp",
                              "cov_model", "cov_ops"}
        if unknown:
            raise MacvoB200Error(f"observe_pack: unknown ext keys {sorted(unknown)}")
        if ext.get("icp") and not buf.extended:
            raise MacvoB200Error("observe_pack: the icp columns need ObservationBuffers(..., extended=True)")
        dc = [None if ext.get(n) is None else _dev(ext[n], torch.float32, f"observe_pack {n}") for n in ("depth_cov0", "depth_cov1")]
        if any(m is not None and m.numel() != H * W for m in dc):
            raise MacvoB200Error("observe_pack: depth_cov0 / depth_cov1 must be (1,1,H,W) maps")
        xs = _ObserveExt(None if dc[0] is None else dc[0].data_ptr(), None if dc[1] is None else dc[1].data_ptr(),
                         int(bool(ext.get("simple_depth"))), float(ext.get("min_depth", 0.0)), float(ext.get("max_depth", 0.0)),
                         int(bool(ext.get("front_of_cam"))), int(bool(ext.get("icp"))))
        model = ext.get("cov_model", "match")
        if model not in COV_MODELS:
            raise MacvoB200Error(f"observe_pack: cov_model must be one of {sorted(COV_MODELS)}, got {model!r}")
        ops_ = tuple(ext.get("cov_ops", ()))
        xs.cov_model, xs.cov_ops, xs.n_cov_ops = COV_MODELS[model], _cov_ops(ops_, "observe_pack"), len(ops_)
    buf.status.zero_()
    rc = lib.macvo_observe_pack(kp.data_ptr() if k else None, k, buf.capacity, fl.data_ptr(), None if mc is None else mc.data_ptr(),
                                *(None if m is None else m.data_ptr() for m in maps), H, W, int(edge_width), C.cast(i0, C.c_void_p),
                                C.cast(i1, C.c_void_p), int(kernel_size), float(min_flow_cov), float(min_depth_cov),
                                float(match_cov_default), pp.data_ptr(), next_pose.data_ptr(), buf.packed.data_ptr(),
                                buf.n_obs.data_ptr(), buf.status.data_ptr(), buf.ws.data_ptr(), buf.ws_bytes, _stream(),
                                None if xs is None else C.byref(xs))
    _check(rc, "macvo_observe_pack")
    LAUNCHES[0] += 2


def pgo_solve_counted(buf: ObservationBuffers, intr: tuple[float, float, float, float, float], pose_io: Tensor,
                      stats: Tensor, min_k: int = 10, cluster: int = 0, graph_type: str = "disp", **kw) -> None:
    """LM solve on the packed observation arrays, block count read from buf.n_obs on the device; pose_io (7,) float64
    CUDA holds the initial pose and receives the result (untouched when fewer than min_k observations survive).
    graph_type "icp" reads points_Tc / obs2_covTc / cov_Tw of an extended buffer that observe_pack filled with icp on."""
    lib = load_library()
    c = buf.capacity
    base = buf.packed.data_ptr()
    gt = PGO_GRAPH_TYPES[graph_type]
    icp = (None, None, None)
    if gt == PGO_GRAPH_TYPES["icp"]:
        if not buf.extended:
            raise MacvoB200Error("pgo_solve_counted: graph type 'icp' needs ObservationBuffers(..., extended=True)")
        icp = tuple(buf.section(n).data_ptr() for n in ("points_Tc", "obs2_covTc", "cov_Tw"))
    intr_c = (C.c_double * 5)(*[float(v) for v in intr])
    prm = _pgo_params(cluster=cluster, **kw)       # 0: cluster size chosen from the capacity
    rc = lib.macvo_pgo_solve_counted(base, base + 8 * 3 * c, base + 8 * 5 * c, base + 8 * 6 * c, base + 8 * 9 * c, c,
                                     buf.n_obs.data_ptr(), int(min_k), C.cast(intr_c, C.c_void_p), pose_io.data_ptr(),
                                     C.byref(prm), stats.data_ptr(), _stream(), gt, *icp)
    _check(rc, "macvo_pgo_solve_counted")
    LAUNCHES[0] += 1


class PeerExchange:
    """This rank's exchange buffer for the sharded LM kernel + the peers' buffers mapped through CUDA IPC.

    `handle` (64 bytes) must be all-gathered across the ranks (any transport: torch.distributed object / tensor gather),
    then `connect(handles)` maps every peer. One process per GPU; all ranks of one node (NVLink / NVSwitch peer access)."""

    def __init__(self, world: int, rank: int):
        lib = load_library()
        self.world, self.rank = int(world), int(rank)
        self.nbytes = int(lib.macvo_pgo_exchange_bytes(self.world))
        if self.nbytes == 0:
            raise MacvoB200Error(f"PeerExchange: world size {world} not in [1, 8]")
        ptr = C.c_void_p()
        hbuf = C.create_string_buffer(64)
        _check(lib.macvo_p2p_alloc(self.nbytes, C.byref(ptr), hbuf), "macvo_p2p_alloc")
        self.own, self.handle = ptr.value, hbuf.raw
        self.ptrs = None
        self._opened: list[int] = []

    def connect(self, handles: list[bytes]) -> None:
        lib = load_library()
        arr = (C.c_void_p * self.world)()
        for r, h in enumerate(handles):
            if r == self.rank:
                arr[r] = self.own
                continue
            p = C.c_void_p()
            _check(lib.macvo_p2p_open(C.create_string_buffer(bytes(h), 64), C.byref(p)), "macvo_p2p_open")
            arr[r] = p.value
            self._opened.append(p.value)
        self.ptrs = arr

    def close(self) -> None:
        lib = load_library()
        for p in self._opened:
            lib.macvo_p2p_close(p)
        self._opened = []
        if self.own:
            lib.macvo_p2p_free(self.own)
            self.own = None


def pgo_solve_sharded(shard: list[Tensor], intr: tuple[float, float, float, float, float], init_pose: Tensor,
                      exchange: PeerExchange, cluster: int = 0, k_total: Tensor | None = None, k_offset: int = 0,
                      min_k: int = 0, pose_io: Tensor | None = None, stats: Tensor | None = None, **kw):
    """This rank's part of the multi-GPU solve (csrc/pgo.cu: all-reduce fused into the persistent kernel over peer
    memory). shard = this rank's [pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov] CUDA float64 slices; every rank must call
    this with the same init_pose / parameters. Returns (pose (7,) float64 CUDA, stats (8,)); identical on all ranks."""
    lib = load_library()
    if exchange.ptrs is None:
        raise MacvoB200Error("pgo_solve_sharded: PeerExchange.connect() has not been called")
    P = [_dev(t, torch.float64, f"pgo_solve_sharded arg{i}") for i, t in enumerate(shard)]
    K = P[0].shape[0]
    pose = pose_io if pose_io is not None else _dev(init_pose, torch.float64, "pgo_solve_sharded init_pose").reshape(7).clone()
    if stats is None:
        stats = torch.zeros((8,), dtype=torch.float64, device=pose.device)
    intr_c = (C.c_double * 5)(*[float(v) for v in intr])
    prm = _pgo_params(cluster=cluster, **kw)
    rc = lib.macvo_pgo_solve_sharded(*(t.data_ptr() for t in P), K, None if k_total is None else k_total.data_ptr(),
                                     int(k_offset), int(min_k), C.cast(intr_c, C.c_void_p), pose.data_ptr(),
                                     C.byref(prm), stats.data_ptr(), C.cast(exchange.ptrs, C.c_void_p), exchange.world,
                                     exchange.rank, _stream())
    _check(rc, "macvo_pgo_solve_sharded")
    LAUNCHES[0] += 1
    return pose, stats


# ---- frontend "next" rows: memory-bound perceiver layers (csrc/nn_kernels.cu) ------------------------------
LAYER_NORM_CHANNELS = (64, 128, 256, 512)


def layer_norm(x: Tensor, weight: Tensor, bias: Tensor, eps: float = 1e-5) -> Tensor:
    """nn.LayerNorm over the last dim of a contiguous fp32 CUDA tensor (warp-per-row kernel)."""
    x = _dev(x, torch.float32, "layer_norm x")
    c = x.shape[-1]
    if c not in LAYER_NORM_CHANNELS:
        raise MacvoB200Error(f"layer_norm: channels {c} not in {LAYER_NORM_CHANNELS}")
    y = torch.empty_like(x)
    rc = load_library().macvo_layer_norm(x.data_ptr(), _dev(weight, torch.float32, "ln weight").data_ptr(),
                                         _dev(bias, torch.float32, "ln bias").data_ptr(), y.data_ptr(),
                                         x.numel() // c, c, float(eps), _stream())
    _check(rc, "macvo_layer_norm")
    LAUNCHES[0] += 1
    return y


def add_layer_norm(x: Tensor, resid: Tensor, weight: Tensor, bias: Tensor, eps: float = 1e-5) -> tuple[Tensor, Tensor]:
    """(x + resid, LayerNorm(x + resid)) in one pass over contiguous fp32 CUDA tensors of C in {128, 256, 512} channels."""
    x, resid = _dev(x, torch.float32, "add_layer_norm x"), _dev(resid, torch.float32, "add_layer_norm resid")
    c = x.shape[-1]
    if c not in (128, 256, 512) or x.shape != resid.shape:
        raise MacvoB200Error(f"add_layer_norm: channels {c} / shapes {tuple(x.shape)} vs {tuple(resid.shape)} unsupported")
    s, y = torch.empty_like(x), torch.empty_like(x)
    rc = load_library().macvo_add_layer_norm(x.data_ptr(), resid.data_ptr(), _dev(weight, torch.float32, "ln weight").data_ptr(),
                                             _dev(bias, torch.float32, "ln bias").data_ptr(), s.data_ptr(), y.data_ptr(),
                                             x.numel() // c, c, float(eps), _stream())
    _check(rc, "macvo_add_layer_norm")
    LAUNCHES[0] += 1
    return s, y


MLP_TC_HIDDEN = (128, 512)


def round_tf32(w: Tensor) -> Tensor:
    """fp32 -> the nearest tf32 value (ties to even, like cvt.rn and like cuBLAS's TF32 GEMMs round their operands), still
    stored as fp32: an MLP weight packed once for `mlp_tc`, whose tensor cores would otherwise truncate the low 13 mantissa
    bits."""
    i = w.detach().to(torch.float32).contiguous().view(torch.int32)
    return ((i + 0xFFF + ((i >> 13) & 1)) & -0x2000).view(torch.float32)


def mlp_tc(xn: Tensor, resid: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor) -> Tensor:
    """resid + w2 GELU_erf(w1 xn + b1) + b2 over the last dim (128 channels, hidden size in MLP_TC_HIDDEN) in one TF32
    tensor-core kernel (csrc/mlp_tc.cu); the hidden activation never reaches device memory."""
    xn, resid = _dev(xn, torch.float32, "mlp_tc xn"), _dev(resid, torch.float32, "mlp_tc resid")
    w1, w2 = _dev(w1, torch.float32, "mlp_tc w1"), _dev(w2, torch.float32, "mlp_tc w2")
    b1, b2 = _dev(b1, torch.float32, "mlp_tc b1"), _dev(b2, torch.float32, "mlp_tc b2")
    c, hd = xn.shape[-1], w1.shape[0]
    if (c != 128 or hd not in MLP_TC_HIDDEN or xn.shape != resid.shape or tuple(w1.shape) != (hd, c)
            or tuple(w2.shape) != (c, hd) or b1.numel() != hd or b2.numel() != c):
        raise MacvoB200Error(f"mlp_tc: unsupported shapes xn {tuple(xn.shape)}, resid {tuple(resid.shape)}, "
                             f"w1 {tuple(w1.shape)}, w2 {tuple(w2.shape)}")
    out = torch.empty_like(resid)
    rc = load_library().macvo_mlp_tc(xn.data_ptr(), resid.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                      b2.data_ptr(), out.data_ptr(), xn.numel() // c, c, hd, _stream())
    _check(rc, "macvo_mlp_tc")
    LAUNCHES[0] += 1
    return out


def patch_tokens_tc(x: Tensor, w0: Tensor, term: Tensor, w2: Tensor, b2: Tensor, ln_w: Tensor, ln_b: Tensor,
                    eps: float = 1e-5) -> Tensor:
    """LayerNorm(w2 relu(w0 x + term[row % period]) + b2) over the last dim of x (..., 64) -> (..., 128) in one TF32
    tensor-core kernel (csrc/patch_tokens_tc.cu): PatchEmbed's token head. With w0 / w2 from `round_tf32` it returns the
    bits of cuBLAS TF32 linear, add_rows_relu_, cuBLAS TF32 linear + bias and layer_norm."""
    x, term = _dev(x, torch.float32, "patch_tokens_tc x"), _dev(term, torch.float32, "patch_tokens_tc term")
    w0, w2 = _dev(w0, torch.float32, "patch_tokens_tc w0"), _dev(w2, torch.float32, "patch_tokens_tc w2")
    b2 = _dev(b2, torch.float32, "patch_tokens_tc b2")
    ln_w, ln_b = _dev(ln_w, torch.float32, "patch_tokens_tc ln_w"), _dev(ln_b, torch.float32, "patch_tokens_tc ln_b")
    cin, c = x.shape[-1], w0.shape[0]
    if (cin != 64 or c != 128 or tuple(w0.shape) != (c, cin) or tuple(w2.shape) != (c, c) or term.dim() != 2
            or term.shape[1] != c or term.shape[0] == 0 or any(t.numel() != c for t in (b2, ln_w, ln_b))):
        raise MacvoB200Error(f"patch_tokens_tc: unsupported shapes x {tuple(x.shape)}, w0 {tuple(w0.shape)}, "
                             f"term {tuple(term.shape)}, w2 {tuple(w2.shape)}")
    out = torch.empty(*x.shape[:-1], c, dtype=torch.float32, device=x.device)
    rc = load_library().macvo_patch_tokens_tc(x.data_ptr(), w0.data_ptr(), term.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                              ln_w.data_ptr(), ln_b.data_ptr(), out.data_ptr(), x.numel() // cin, cin, c,
                                              term.shape[0], float(eps), _stream())
    _check(rc, "macvo_patch_tokens_tc")
    LAUNCHES[0] += 1
    return out


def patch_embed_conv1(maps: Tensor, weight: Tensor, bias: Tensor, allow_tf32: bool | None = None, s2d: bool = False) -> Tensor:
    """(M,1,H,W) cost maps -> ReLU(conv 6x6/2 (+ pad to x8)) as a logical (M,16,Ho,Wo) channels_last tensor; s2d=True (TF32
    variant only): the same values space-to-depth, a logical (M,64,Ho/2,Wo/2) channels_last tensor with channel
    ((y & 1) * 2 + (x & 1)) * 16 + c (see `space_to_depth_filter` for the matching 3x3 filter of the next convolution)."""
    maps = _dev(maps, torch.float32, "patch_embed maps")
    m, one, h, w = maps.shape
    if one != 1 or tuple(weight.shape) != (16, 1, 6, 6):
        raise MacvoB200Error("patch_embed_conv1: expects (M,1,H,W) maps and a (16,1,6,6) weight")
    ho, wo = (h + 7) // 8 * 4, (w + 7) // 8 * 4
    tf32 = bool(torch.backends.cudnn.allow_tf32 if allow_tf32 is None else allow_tf32)
    if s2d and not tf32:
        raise MacvoB200Error("patch_embed_conv1: the space-to-depth output exists for the TF32 tensor-core variant only")
    out = torch.empty((m, ho // 2, wo // 2, 64) if s2d else (m, ho, wo, 16), dtype=torch.float32, device=maps.device)
    rc = load_library().macvo_patch_embed_conv1(maps.data_ptr(), _dev(weight, torch.float32, "w").data_ptr(),
                                                _dev(bias, torch.float32, "b").data_ptr(), out.data_ptr(),
                                                m, h, w, int(tf32) | (2 if s2d else 0), _stream())
    _check(rc, "macvo_patch_embed_conv1")
    LAUNCHES[0] += 1
    return out.permute(0, 3, 1, 2)


def space_to_depth_filter(weight: Tensor) -> Tensor:
    """(O, C, 6, 6) stride-2 / padding-2 filter -> the (O, 4C, 3, 3) stride-1 / padding-1 filter that gives the same output on
    the space-to-depth input: W'[o, (dy*2+dx)*C + c, a, b] = W[o, c, 2a+dy, 2b+dx]."""
    o, c, kh, kw = weight.shape
    if (kh, kw) != (6, 6):
        raise MacvoB200Error("space_to_depth_filter: expects a 6x6 filter")
    return weight.reshape(o, c, 3, 2, 3, 2).permute(0, 3, 5, 1, 2, 4).reshape(o, 4 * c, 3, 3)


def small_attention(q: Tensor, k: Tensor, v: Tensor, heads: int, allow_tf32: bool | None = None) -> Tensor:
    """softmax(q k^T / sqrt(d)) v with q (B|1, Nq, heads*d), k/v (B, Nk, heads*d) -> (B, Nq, heads*d); d in {8, 16, 32}.
    allow_tf32=None follows torch.backends.cuda.matmul.allow_tf32 (what the torch bmm it replaces would do)."""
    if allow_tf32 is None:
        allow_tf32 = bool(torch.backends.cuda.matmul.allow_tf32)
    q, k, v = (_dev(t, torch.float32, "attention operand") for t in (q, k, v))
    b, nk, c = k.shape
    d = c // heads
    nq = q.shape[1]
    if q.shape[0] not in (1, b) or q.shape[2] != c or v.shape != k.shape or d * heads != c:
        raise MacvoB200Error(f"small_attention: bad shapes q{tuple(q.shape)} k{tuple(k.shape)} v{tuple(v.shape)}")
    out = torch.empty(b, nq, c, dtype=torch.float32, device=k.device)
    rc = load_library().macvo_small_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), b, nq, nk,
                                              heads, d, int(q.shape[0] == 1 and b > 1), int(allow_tf32), _stream())
    _check(rc, "macvo_small_attention")
    LAUNCHES[0] += 1
    return out


# ---- decoder iteration glue (csrc/decoder_fused.cu) -----------------------------------------------------------
GRU_HID, GRU_IN = 128, 512


def _gru_buf(t: Tensor, what: str) -> Tensor:
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == GRU_IN and t.is_contiguous()):
        raise MacvoB200Error(f"{what}: expected a contiguous fp32 CUDA (pixels, {GRU_IN}) buffer")
    return t


def gru_input(mf: Tensor, agg: Tensor, gamma: Tensor, bufs: list[Tensor]) -> None:
    """write x-part channels 256..511 = [mf | mf + gamma * agg] of up to 4 (pixels, 512) GRU input buffers"""
    mf, agg = _dense(mf, GRU_HID, "gru_input mf"), _dense(agg, GRU_HID, "gru_input agg")
    pixels = mf.numel() // GRU_HID
    ptrs = [_gru_buf(b, "gru_input buffer").data_ptr() for b in bufs] + [None] * (4 - len(bufs))
    rc = load_library().macvo_gru_input(mf.data_ptr(), agg.data_ptr(), _dev(gamma, torch.float32, "gamma").data_ptr(),
                                        *ptrs, pixels, _stream())
    _check(rc, "macvo_gru_input")
    LAUNCHES[0] += 1


def _dense(t: Tensor, cols: int, what: str) -> Tensor:
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() % cols == 0):
        raise MacvoB200Error(f"{what}: expected a contiguous fp32 CUDA pixels-major (.., {cols}) tensor "
                             f"(pass conv outputs as x.permute(0, 2, 3, 1) of a channels_last map)")
    return t


def _bias_ptr(bias, n: int, what: str):
    if bias is None:
        return None
    if not (bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == n):
        raise MacvoB200Error(f"{what}: expected a contiguous fp32 CUDA bias of {n} elements")
    return bias.data_ptr()


def gru_gates(zr: Tensor, hx: Tensor, z_out: Tensor, rhx: Tensor, bias: Tensor | None = None) -> None:
    zr, z_out = _dense(zr, 2 * GRU_HID, "gru_gates zr"), _dense(z_out, GRU_HID, "gru_gates z_out")
    rc = load_library().macvo_gru_gates(zr.data_ptr(), _bias_ptr(bias, 2 * GRU_HID, "gru_gates bias"),
                                        _gru_buf(hx, "hx").data_ptr(), z_out.data_ptr(),
                                        _gru_buf(rhx, "rhx").data_ptr(), hx.shape[0], _stream())
    _check(rc, "macvo_gru_gates")
    LAUNCHES[0] += 1


def gru_blend(q: Tensor, z: Tensor, hx: Tensor, h_dense: Tensor | None, bias: Tensor | None = None) -> None:
    q, z = _dense(q, GRU_HID, "gru_blend q"), _dense(z, GRU_HID, "gru_blend z")
    if h_dense is not None:
        _dense(h_dense, GRU_HID, "gru_blend h_dense")
    rc = load_library().macvo_gru_blend(q.data_ptr(), _bias_ptr(bias, GRU_HID, "gru_blend bias"), z.data_ptr(),
                                        _gru_buf(hx, "hx").data_ptr(),
                                        None if h_dense is None else h_dense.data_ptr(), hx.shape[0], _stream())
    _check(rc, "macvo_gru_blend")
    LAUNCHES[0] += 1


def rows_count(batch: int, height: int, width: int, vertical: int = 0) -> int:
    """rows of a zero-initialised padded pixel-row buffer (layout U, or the GRU's layout V): csrc/rows_layout.cuh"""
    return int(load_library().macvo_rows_count(batch, height, width, vertical))


def pack_conv_filter(weight: Tensor, bias: Tensor | None, in_channels: int | None = None, device=None) -> tuple[Tensor, Tensor | None, int]:
    """(N, C, k, k) fp32 filter -> (n_pad, k*k*c_pad) fp16 GEMM operand of macvo_conv_tc (K index = (ky*k + kx)*c_pad + c), zero
    padded to n_pad % 32 == 0 rows / c_pad % 64 == 0 channels; bias -> (n_pad) fp32. Returns (weights, bias, N)."""
    w = weight.detach().to(device=device or weight.device, dtype=torch.float32)
    n, c, kh, kw = w.shape
    c_pad = in_channels or -(-c // 64) * 64
    n_pad = -(-n // 32) * 32
    wp = torch.zeros(n_pad, kh * kw, c_pad, dtype=torch.float32, device=w.device)
    wp[:n, :, :c] = w.permute(0, 2, 3, 1).reshape(n, kh * kw, c)
    bp = None
    if bias is not None:
        bp = torch.zeros(n_pad, dtype=torch.float32, device=w.device)
        bp[:n] = bias.detach().to(device=w.device, dtype=torch.float32)
    return wp.reshape(n_pad, kh * kw * c_pad).to(torch.float16).contiguous(), bp, n


def conv_tc(in_rows: Tensor, weights: Tensor, bias: Tensor | None, n_valid: int, ksize: int, relu: bool, shape: tuple[int, int, int],
            in_dense: bool = False, out16: Tensor | None = None, out16_offset: int = 0, out16_dense: bool = False,
            out32: Tensor | None = None, out32_offset: int = 0, add_to_map: Tensor | None = None) -> None:
    """3x3 / 1x1 convolution on the tensor-core path (csrc/conv_tc.cu): fp16 pixel rows in, fp16 rows and / or fp32 dense rows out;
    `add_to_map` (B, n_valid, H, W) fp32 instead of out32: the result is added to that map in place"""
    B, H, W = shape
    for t, dt, what in ((in_rows, torch.float16, "in_rows"), (weights, torch.float16, "weights"), (out16, torch.float16, "out16"),
                        (out32, torch.float32, "out32"), (bias, torch.float32, "bias")):
        if t is not None and not (t.is_cuda and t.dtype == dt and t.is_contiguous()):
            raise MacvoB200Error(f"conv_tc: {what} must be a contiguous CUDA {dt} tensor")
    c_in = in_rows.shape[1]
    if weights.shape[1] != ksize * ksize * c_in or (bias is not None and bias.numel() != weights.shape[0]):
        raise MacvoB200Error("conv_tc: filter / bias shape does not match the input rows")
    need = B * H * W if in_dense else rows_count(B, H, W)
    if in_rows.shape[0] != need:
        raise MacvoB200Error(f"conv_tc: expected {need} input rows, got {in_rows.shape[0]}")
    planes = add_to_map is not None
    if planes:
        if out32 is not None or not (add_to_map.is_cuda and add_to_map.dtype == torch.float32 and add_to_map.is_contiguous()
                                     and tuple(add_to_map.shape) == (B, n_valid, H, W)):
            raise MacvoB200Error("conv_tc: add_to_map must be a contiguous fp32 (B, n_valid, H, W) CUDA tensor (and excludes out32)")
        out32 = add_to_map
    for t, dense, off in ((out16, out16_dense, out16_offset), (None if planes else out32, True, out32_offset)):
        if t is not None and (t.shape[0] != (B * H * W if dense else rows_count(B, H, W)) or off + n_valid > t.shape[1]):
            raise MacvoB200Error("conv_tc: output rows / channel range do not fit")
    rc = load_library().macvo_conv_tc(in_rows.data_ptr(), c_in, int(in_dense), weights.data_ptr(), None if bias is None else bias.data_ptr(),
                                      weights.shape[0], n_valid, ksize, int(relu), B, H, W,
                                      None if out16 is None else out16.data_ptr(), 0 if out16 is None else out16.shape[1], out16_offset,
                                      int(out16_dense), None if out32 is None else out32.data_ptr(),
                                      0 if out32 is None else out32.shape[1], out32_offset, int(planes), _stream())
    _check(rc, "macvo_conv_tc")
    LAUNCHES[0] += 1


def flow_im2col(coords1: Tensor, coords0: Tensor, rows: Tensor, mf32: Tensor | None, mf16_rows: Tensor | None) -> None:
    """7x7 neighbourhoods of flow = coords1 - coords0 as (pixels, 128) fp16 GEMM rows; flow -> channels 126, 127 of the mf rows"""
    c1, c0 = _dev(coords1, torch.float32, "coords1"), _dev(coords0, torch.float32, "coords0")
    B, _, H, W = c1.shape
    rc = load_library().macvo_flow_im2col(c1.data_ptr(), c0.data_ptr(), rows.data_ptr(), None if mf32 is None else mf32.data_ptr(),
                                          None if mf16_rows is None else mf16_rows.data_ptr(), B, H, W, _stream())
    _check(rc, "macvo_flow_im2col")
    LAUNCHES[0] += 1


def pack_rows(src: Tensor, dst: Tensor, offset: int, shape: tuple[int, int, int], vertical: int = 0) -> None:
    """fp32 dense pixel rows (pixels, C) -> fp16 padded rows dst[:, offset : offset + C] (layout U, or V when `vertical`)"""
    B, H, W = shape
    if not (src.is_cuda and src.dtype == torch.float32 and src.is_contiguous() and src.dim() == 2 and src.shape[0] == B * H * W):
        raise MacvoB200Error("pack_rows: expected contiguous fp32 (pixels, C) rows")
    _check(load_library().macvo_gru_tc_pack(src.data_ptr(), src.shape[1], src.shape[1], dst.data_ptr(), dst.shape[1], offset, B, H, W,
                                            vertical, _stream()), "macvo_gru_tc_pack")
    LAUNCHES[0] += 1


class SepConvGruTC:
    """The decoder's SepConvGRU units (gru.py:22-43; flow, and covariance for FlowFormerCov, covhead.py:95-131) on the
    tensor-core path (csrc/gru_conv_tc.cu): fp32 recurrent state `h[u]` (pixels, 128) in dense pixel order, fp16 padded operand
    rows for the two passes, one `step` = pack the motion features + one 4-launch chain per unit.

    weights[u]: {"convzr1": (256,512,1,5), "convq1": (128,512,1,5), "convzr2": (256,512,5,1), "convq2": (128,512,5,1)} fp32
    filters with the z | r filters concatenated, biases[u]: the matching (N,) vectors; u = 0 flow, 1 covariance (one unit:
    the plain FlowFormer's flow unit alone)."""

    LAUNCHES_PER_UNIT = 4

    def __init__(self, weights: list[dict], biases: list[dict], batch: int, height: int, width: int, device):
        lib = load_library()
        self.shape, self.device = (int(batch), int(height), int(width)), device
        self.units = len(weights)
        if self.units not in (1, 2) or len(biases) != self.units:
            raise MacvoB200Error("SepConvGruTC: expects the decoder's flow unit, optionally followed by its covariance unit")
        P = batch * height * width
        rows = [int(lib.macvo_gru_tc_operand_rows(batch, height, width, o)) for o in (0, 1)]
        f16 = dict(dtype=torch.float16, device=device)
        self.x = [torch.zeros(r, 3 * GRU_HID, **f16) for r in rows]
        self.h_rows = [[torch.zeros(r, GRU_HID, **f16) for _ in range(self.units)] for r in rows]     # [pass][unit]
        self.rh_rows = [[torch.zeros(r, GRU_HID, **f16) for _ in range(self.units)] for r in rows]
        self.h = [torch.zeros(P, GRU_HID, dtype=torch.float32, device=device) for _ in range(self.units)]
        self.z = [torch.zeros(P, GRU_HID, dtype=torch.float32, device=device) for _ in range(self.units)]
        self.w, self.b = {}, {}
        for u in range(self.units):
            for o in (0, 1):
                for st, name in ((0, f"convzr{o + 1}"), (1, f"convq{o + 1}")):
                    w = weights[u][name].detach().to(device=device, dtype=torch.float32)
                    n = w.shape[0]
                    if tuple(w.shape) != ((n, GRU_IN, 1, 5) if o == 0 else (n, GRU_IN, 5, 1)) or n != (256, 128)[st]:
                        raise MacvoB200Error(f"SepConvGruTC: unexpected filter shape {tuple(w.shape)} for {name}")
                    self.w[u, o, st] = w.reshape(n, GRU_IN, 5).permute(0, 2, 1).reshape(n, 5 * GRU_IN).to(torch.float16).contiguous()
                    self.b[u, o, st] = biases[u][name].detach().to(device=device, dtype=torch.float32).contiguous()
        # device pointers of every (unit, pass, stage) launch: h | r*h rows in, x rows, filters, bias, state, z, rows out
        self._stage_args = {(u, o, st): ((self.h_rows[o] if st == 0 else self.rh_rows[o])[u].data_ptr(), self.x[o].data_ptr(),
                                         self.w[u, o, st].data_ptr(), self.b[u, o, st].data_ptr(), self.h[u].data_ptr(),
                                         self.z[u].data_ptr(), (self.rh_rows[o] if st == 0 else self.h_rows[1 - o])[u].data_ptr())
                            for u in range(self.units) for o in (0, 1) for st in (0, 1)}
        self._side = torch.cuda.Stream(device) if self.units == 2 else None

    def _pack(self, src: Tensor, dst: Tensor, offset: int, vertical: int) -> None:
        B, H, W = self.shape
        src = _dense(src, GRU_HID, "SepConvGruTC rows")
        if src.numel() != B * H * W * GRU_HID:
            raise MacvoB200Error("SepConvGruTC: expected (pixels, 128) rows")
        _check(load_library().macvo_gru_tc_pack(src.data_ptr(), GRU_HID, GRU_HID, dst.data_ptr(), dst.shape[1], offset, B, H, W,
                                                vertical, _stream()), "macvo_gru_tc_pack")
        LAUNCHES[0] += 1

    def set_context(self, inp_rows: Tensor) -> None:
        """x channels [0, 128) = the context features `inp` (constant over the refinement iterations)"""
        for o in (0, 1):
            self._pack(inp_rows, self.x[o], 0, o)

    def set_state(self, unit: int, h_rows: Tensor) -> None:
        self.h[unit].copy_(_dense(h_rows, GRU_HID, "SepConvGruTC state").view(-1, GRU_HID))
        self._pack(self.h[unit], self.h_rows[0][unit], 0, 0)

    def step(self, mf: Tensor, agg: Tensor, gamma: Tensor) -> torch.cuda.Event | None:
        """one SepConvGRU update of every unit with x = [inp | mf | mf + gamma * agg]; new state in `self.h[u]`.
        One 4-launch chain per unit: with 84 CTA tiles per unit (640x480: two 60x80 maps) a launch covering both units would be
        168 CTAs = two waves on 132 SMs per stage, two independent chains of 84-CTA launches keep the SMs filled across the stage
        boundaries. Unit 0's chain runs on the current stream, unit 1's on a side stream; the returned event marks the end of
        unit 1's chain, and whatever reads unit 1's state must make its stream wait on it. With one unit there is no side
        stream and no event (None)."""
        B, H, W = self.shape
        lib = load_library()
        mf, agg = _dense(mf, GRU_HID, "SepConvGruTC mf"), _dense(agg, GRU_HID, "SepConvGruTC agg")
        if mf.numel() != B * H * W * GRU_HID or agg.numel() != mf.numel():
            raise MacvoB200Error("SepConvGruTC.step: expected (pixels, 128) rows")
        main = torch.cuda.current_stream()
        _check(lib.macvo_gru_tc_pack_motion(mf.data_ptr(), agg.data_ptr(), _dev(gamma, torch.float32, "gamma").data_ptr(),
                                            self.x[0].data_ptr(), self.x[1].data_ptr(), B, H, W, main.cuda_stream),
               "macvo_gru_tc_pack_motion")
        unit1_done = None
        if self.units == 2:
            fork = torch.cuda.Event()
            fork.record(main)
            self._side.wait_event(fork)
            self._chain(1, self._side)
            unit1_done = torch.cuda.Event()
            unit1_done.record(self._side)
        self._chain(0, main)
        LAUNCHES[0] += 1 + self.LAUNCHES_PER_UNIT * self.units
        return unit1_done

    def _chain(self, unit: int, stream: torch.cuda.Stream) -> None:
        """the 1x5 pass, then the 5x1 pass, of one unit: stage 0 (z | r) and stage 1 (q + blend) each"""
        B, H, W = self.shape
        lib = load_library()
        for o in (0, 1):
            for stage in (0, 1):
                _check(lib.macvo_gru_tc_stage(stage, o, B, H, W, *self._stage_args[unit, o, stage], stream.cuda_stream),
                       "macvo_gru_tc_stage")


def convex_upsample(flow: Tensor, mask_logits: Tensor, scale: float = 1.0) -> Tensor:
    """`upsample_flow` (core/decoder.py:131-139) in one kernel: flow (B,2,H,W), mask_logits (B,576,H,W) -> (B,2,8H,8W); the
    softmax runs over scale * mask_logits"""
    f = _dev(flow, torch.float32, "convex_upsample flow")
    B, c, H, W = f.shape
    if c != 2 or tuple(mask_logits.shape) != (B, 576, H, W) or not mask_logits.is_cuda or mask_logits.dtype != torch.float32:
        raise MacvoB200Error("convex_upsample: expects flow (B,2,H,W) and fp32 CUDA mask logits (B,576,H,W)")
    m = mask_logits.permute(0, 2, 3, 1)
    if not m.is_contiguous():
        m = m.contiguous()
    out = torch.empty((B, 2, 8 * H, 8 * W), dtype=torch.float32, device=f.device)
    rc = load_library().macvo_convex_upsample(f.data_ptr(), m.data_ptr(), out.data_ptr(), float(scale), B, H, W, _stream())
    _check(rc, "macvo_convex_upsample")
    LAUNCHES[0] += 1
    return out


def softmax_rows_f16(scores: Tensor) -> Tensor:
    """softmax over the last dimension of fp32 scores, written as fp16 (the GMA attention matrix under TF32; gma.py:39-82)"""
    x = _dev(scores, torch.float32, "softmax_rows_f16 scores")
    cols = x.shape[-1]
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    rc = load_library().macvo_softmax_rows_f16(x.data_ptr(), out.data_ptr(), x.numel() // cols, cols, _stream())
    _check(rc, "macvo_softmax_rows_f16")
    LAUNCHES[0] += 1
    return out


def decoder_token_blob(w: dict, prefix: str = "memory_decoder.") -> Tensor:
    """Pack the token-path weights (checkpoint names) into the blob layout of macvo_decoder_token."""
    ca = prefix + "decoder_layer.cross_attend."
    mats = [w[prefix + "flow_token_encoder.0.weight"].flatten(1), w[prefix + "flow_token_encoder.2.weight"].flatten(1),
            w[ca + "q.weight"], w[ca + "proj.weight"], w[ca + "ffn.0.weight"], w[ca + "ffn.3.weight"]]
    vecs = [w[prefix + "flow_token_encoder.0.bias"], w[prefix + "flow_token_encoder.2.bias"], w[ca + "norm1.weight"],
            w[ca + "norm1.bias"], w[ca + "q.bias"], w[ca + "proj.bias"], w[ca + "norm2.weight"], w[ca + "norm2.bias"],
            w[ca + "ffn.0.bias"], w[ca + "ffn.3.bias"]]
    dev = mats[0].device
    freq = torch.arange(16, device=dev, dtype=torch.float32) * (1 / 200) * torch.pi      # as sine_embed builds it
    blob = torch.cat([m.float().t().contiguous().flatten() for m in mats] + [v.float().flatten() for v in vecs] + [freq])
    if blob.numel() != load_library().macvo_decoder_token_blob_floats():
        raise MacvoB200Error(f"decoder_token_blob: {blob.numel()} floats, kernel expects "
                             f"{load_library().macvo_decoder_token_blob_floats()}")
    return blob.contiguous()


def decoder_token(cost_forward: Tensor, coords: Tensor, key: Tensor, value: Tensor, blob: Tensor, eps: float = 1e-5,
                  out16_rows: Tensor | None = None) -> Tensor:
    """one refinement iteration's token path: lookup rows (P,81) + coords (B,2,H,W) + per-pixel keys / values (P,8,64)
    -> (P,160) rows [cost_global | cost_forward | 0] (decoder.py:20-76,112-116; csrc/decoder_token.cu); with `out16_rows` (a
    layout-U fp16 buffer of 192 channels, csrc/rows_layout.cuh) the rows are written there instead (and returned)"""
    cf = _dense(cost_forward, 81, "decoder_token cost_forward")
    co = _dev(coords, torch.float32, "decoder_token coords")
    B, _, H, W = co.shape
    P = B * H * W
    k, v = _dense(key, 64, "decoder_token key"), _dense(value, 64, "decoder_token value")
    if cf.numel() != P * 81 or k.numel() != P * 512 or v.numel() != P * 512:
        raise MacvoB200Error("decoder_token: expects cost_forward (P,81), key / value (P,8,64) with P = B*H*W")
    if out16_rows is not None:
        if not (out16_rows.is_cuda and out16_rows.dtype == torch.float16 and out16_rows.is_contiguous()
                and tuple(out16_rows.shape) == (rows_count(B, H, W), 192)):
            raise MacvoB200Error("decoder_token: out16_rows must be a contiguous fp16 (rows_count(B, H, W), 192) CUDA tensor")
        rc = load_library().macvo_decoder_token_rows(cf.data_ptr(), co.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                     _dense(blob, 1, "decoder_token blob").data_ptr(), out16_rows.data_ptr(), B, H, W,
                                                     float(eps), _stream())
        _check(rc, "macvo_decoder_token_rows")
        LAUNCHES[0] += 1
        return out16_rows
    out = torch.empty((P, 160), dtype=torch.float32, device=cf.device)
    rc = load_library().macvo_decoder_token(cf.data_ptr(), co.data_ptr(), k.data_ptr(), v.data_ptr(),
                                            _dense(blob, 1, "decoder_token blob").data_ptr(), out.data_ptr(), B, H * W,
                                            float(eps), _stream())
    _check(rc, "macvo_decoder_token")
    LAUNCHES[0] += 1
    return out


def add_rows_relu_(x: Tensor, term: Tensor) -> Tensor:
    """in place relu(x + term[row % period]) on x (rows, C) / (M, period, C) with term (period, C)"""
    c = x.shape[-1]
    _dense(x, c, "add_rows_relu x")
    term = _dense(term, c, "add_rows_relu term")
    rc = load_library().macvo_add_rows_relu(x.data_ptr(), term.data_ptr(), x.numel() // c, term.numel() // c, c, _stream())
    _check(rc, "macvo_add_rows_relu")
    LAUNCHES[0] += 1
    return x


def fused_qkv_attention(qkv: Tensor, heads: int, q_add: Tensor | None = None, k_add: Tensor | None = None,
                        allow_tf32: bool | None = None) -> Tensor:
    """attention on a fused projection output qkv (B, N, 3*C) = [q | k | v] consumed in place (self-attention, Nq = Nk = N);
    q_add / k_add (period, N, C): additive terms, batch b uses slice b % period. -> (B, N, C)"""
    qkv = _dev(qkv, torch.float32, "fused_qkv_attention qkv")
    b, n, c3 = qkv.shape
    c = c3 // 3
    if allow_tf32 is None:
        allow_tf32 = bool(torch.backends.cuda.matmul.allow_tf32)
    period = 0
    for t in (q_add, k_add):
        if t is not None:
            _dense(t, c, "fused_qkv_attention additive term")
            if t.shape[-2] != n:
                raise MacvoB200Error("fused_qkv_attention: additive terms must be (period, N, C)")
            period = t.numel() // (n * c)
    out = torch.empty(b, n, c, dtype=torch.float32, device=qkv.device)
    base = qkv.data_ptr()                       # q | k | v start c floats (4 c bytes) apart inside every 3c-float row
    rc = load_library().macvo_small_attention_ex(base, base + 4 * c, base + 8 * c, out.data_ptr(), b, n, n, heads, c // heads,
                                                 0, int(allow_tf32), c3, c3, c3,
                                                 None if q_add is None else q_add.data_ptr(),
                                                 None if k_add is None else k_add.data_ptr(), period, _stream())
    _check(rc, "macvo_small_attention_ex")
    LAUNCHES[0] += 1
    return out


def attention_with_terms(q: Tensor, k: Tensor, v: Tensor, heads: int, q_add: Tensor | None = None,
                         allow_tf32: bool | None = None) -> Tensor:
    """small_attention with q_add (period, Nq, C) added to q on load (batch b uses slice b % period)"""
    q, k, v = (_dev(t, torch.float32, "attention operand") for t in (q, k, v))
    b, nk, c = k.shape
    nq = q.shape[1]
    if allow_tf32 is None:
        allow_tf32 = bool(torch.backends.cuda.matmul.allow_tf32)
    period = 0
    if q_add is not None:
        _dense(q_add, c, "attention_with_terms q_add")
        period = q_add.numel() // (nq * c)
    out = torch.empty(b, nq, c, dtype=torch.float32, device=k.device)
    rc = load_library().macvo_small_attention_ex(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), b, nq, nk, heads,
                                                 c // heads, 0, int(allow_tf32), 0, 0, 0,
                                                 None if q_add is None else q_add.data_ptr(), None, period, _stream())
    _check(rc, "macvo_small_attention_ex")
    LAUNCHES[0] += 1
    return out


def latent_pool(tokens: Tensor, q: Tensor, wk: Tensor, wv: Tensor, bv: Tensor) -> Tensor:
    """Perceiver input-layer attention without K / V: tokens (M, nk, 128), q (8, 128) shared latent queries (already
    projected), wk / wv (128, 128), bv (128) -> (M, 8, 128). TF32 tensor cores (see macvo_latent_pool)."""
    tokens = _dense(tokens, 128, "latent_pool tokens")
    m, nk, c = tokens.shape
    if c != 128 or tuple(q.shape[-2:]) != (8, 128):
        raise MacvoB200Error("latent_pool: expects tokens (M, nk, 128) and q (8, 128)")
    # U^T[h*8 + i, :] = Wk[h*16:(h+1)*16, :]^T q[i, h*16:(h+1)*16] / sqrt(16)
    ut = torch.einsum("ihd,hdc->hic", q.reshape(8, 8, 16), wk.reshape(8, 16, 128)).reshape(64, 128).mul_(0.25).contiguous()
    out = torch.empty(m, 8, 128, dtype=torch.float32, device=tokens.device)
    rc = load_library().macvo_latent_pool(tokens.data_ptr(), ut.data_ptr(), _dense(wv, 128, "wv").data_ptr(),
                                          _bias_ptr(bv, 128, "bv"), out.data_ptr(), m, nk, _stream())
    _check(rc, "macvo_latent_pool")
    LAUNCHES[0] += 1
    return out


# ------------------------------------------------------------------------------------------------
# (f5) TartanMotionNet pose network (csrc/posenet.cu)
# ------------------------------------------------------------------------------------------------
POSENET_H, POSENET_W = 112, 160
POSENET_SPLIT = 8           # K split of macvo_posenet_conv = its thread-block cluster size


def posenet_co_tile(cout: int) -> int:
    """output channels per CTA: cout / 32 tiles x 8 K-splits = 256 CTAs for every layer (two per SM on an H100)"""
    return max(1, cout // 32)


def pack_posenet_conv(weight: Tensor) -> tuple[Tensor, int]:
    """(cout, cin, k, k) (or (cout, cin) for a linear layer) -> the per-CTA weight slabs macvo_posenet_conv streams:
    [cout/co_tile][8][co_tile][cin/8 * k * k], each slab contiguous. Done once, at construction."""
    w = weight.detach().float()
    cout, cin = w.shape[:2]
    if cin % POSENET_SPLIT:
        raise MacvoB200Error(f"pack_posenet_conv: cin {cin} is not a multiple of {POSENET_SPLIT}")
    ct = posenet_co_tile(cout)
    kc = w[0].numel() // POSENET_SPLIT
    packed = (w.reshape(cout // ct, ct, POSENET_SPLIT, kc).permute(0, 2, 1, 3).contiguous().reshape(-1))
    return packed, ct


def posenet_input(flow: Tensor, depth: Tensor, bl_fx: float, out: Tensor) -> None:
    """channels 0..2 of the (1,5,112,160) pose-network input from flow (1,2,H,W) and depth (1,1,H,W)"""
    fl = _dev(flow, torch.float32, "posenet_input flow")
    dp = _dev(depth, torch.float32, "posenet_input depth")
    H, W = fl.shape[-2:]
    if fl.numel() != 2 * H * W or dp.numel() != H * W:
        raise MacvoB200Error("posenet_input: expects flow (1,2,H,W) and depth (1,1,H,W)")
    if H < POSENET_H or W < POSENET_W:
        raise MacvoB200Error(f"posenet_input: maps of {H}x{W} are smaller than the network input {POSENET_H}x{POSENET_W}")
    if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == 5 * POSENET_H * POSENET_W):
        raise MacvoB200Error("posenet_input: out must be a contiguous (1,5,112,160) fp32 CUDA tensor")
    _check(load_library().macvo_posenet_input(fl.data_ptr(), dp.data_ptr(), H, W, float(bl_fx), out.data_ptr(), _stream()),
           "macvo_posenet_input")
    LAUNCHES[0] += 1


def posenet_conv(x: Tensor, packed: Tensor, co_tile: int, bias: Tensor, ksize: int, stride: int, pad: int,
                 resid: Tensor | None = None, relu: bool = False, out: Tensor | None = None) -> Tensor:
    """epilogue(conv2d(x, W, bias, stride, pad) [+ resid]) for one image x (cin,hi,wi) (a leading batch of 1 is accepted);
    W given as pack_posenet_conv's slabs. Returns (1, cout, ho, wo)."""
    x = _dev(x, torch.float32, "posenet_conv x")
    cin, hi, wi = x.shape[-3:]
    if x.numel() != cin * hi * wi:
        raise MacvoB200Error("posenet_conv: x must hold one image")
    b = _dev(bias, torch.float32, "posenet_conv bias")
    cout = b.numel()
    pk = _dev(packed, torch.float32, "posenet_conv weights")
    if pk.numel() != cout * cin * ksize * ksize:
        raise MacvoB200Error(f"posenet_conv: {pk.numel()} packed weights for cout {cout}, cin {cin}, k {ksize}")
    ho, wo = (hi + 2 * pad - ksize) // stride + 1, (wi + 2 * pad - ksize) // stride + 1
    if out is None:
        out = torch.empty((1, cout, ho, wo), dtype=torch.float32, device=x.device)
    elif not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == cout * ho * wo):
        raise MacvoB200Error("posenet_conv: out has the wrong shape")
    r = None
    if resid is not None:
        r = _dev(resid, torch.float32, "posenet_conv resid")
        if r.numel() != cout * ho * wo:
            raise MacvoB200Error("posenet_conv: resid must have the output's shape")
    rc = load_library().macvo_posenet_conv(x.data_ptr(), cin, hi, wi, pk.data_ptr(), b.data_ptr(), cout, ksize, stride, pad,
                                           int(co_tile), r.data_ptr() if r is not None else None, int(bool(relu)),
                                           out.data_ptr(), _stream())
    _check(rc, "macvo_posenet_conv")
    LAUNCHES[0] += 1
    return out


def posenet_head_floats() -> int:
    return int(load_library().macvo_posenet_head_floats())


def posenet_head(fc1_out: Tensor, head_blob: Tensor, prev_pose: Tensor, motion: Tensor, next_pose: Tensor) -> None:
    """fc2 / fc3 of both heads x pose_norm -> motion (6,) fp32, and next_pose (7,) float64 = prev_pose @ se3(motion).Exp()"""
    h = _dev(fc1_out, torch.float32, "posenet_head fc1_out")
    blob = _dev(head_blob, torch.float32, "posenet_head blob")
    pp = _dev(prev_pose, torch.float64, "posenet_head prev_pose")
    if h.numel() != 256 or blob.numel() != posenet_head_floats() or pp.numel() != 7:
        raise MacvoB200Error("posenet_head: expects fc1_out (256,), the head blob and prev_pose (7,)")
    for t, dt, n, what in ((motion, torch.float32, 6, "motion"), (next_pose, torch.float64, 7, "next_pose")):
        if not (t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n):
            raise MacvoB200Error(f"posenet_head: {what} must be a contiguous ({n},) {dt} CUDA tensor")
    _check(load_library().macvo_posenet_head(h.data_ptr(), blob.data_ptr(), pp.data_ptr(), motion.data_ptr(),
                                             next_pose.data_ptr(), _stream()), "macvo_posenet_head")
    LAUNCHES[0] += 1


# ------------------------------------------------------------------------------------------------
# (f6) TartanVOMatcher's PWC-Net: warp + correlation + LeakyReLU of one level (csrc/pwc_corr.cu)
# ------------------------------------------------------------------------------------------------
PWC_DISPLACEMENTS = 81


def pwc_warp_corr(f1: Tensor, f2: Tensor, flow: Tensor | None, scale: float, out: Tensor, out_offset: int) -> Tensor:
    """LeakyReLU_0.1(correlation(f1, warp(f2, scale * flow))) of PWCDCNet_Adapted (no warp when flow is None) written into
    channels [out_offset, out_offset + 81) of out (B, C_out, H, W); f1, f2 (B, C, H, W), flow (B, 2, H, W). Returns out."""
    a = _dev(f1, torch.float32, "pwc_warp_corr f1")
    b = _dev(f2, torch.float32, "pwc_warp_corr f2")
    if a.dim() != 4 or b.shape != a.shape:
        raise MacvoB200Error(f"pwc_warp_corr: f1 {tuple(a.shape)} and f2 {tuple(b.shape)} must be the same (B,C,H,W)")
    B, Cc, H, W = a.shape
    fl = None
    if flow is not None:
        fl = _dev(flow, torch.float32, "pwc_warp_corr flow")
        if tuple(fl.shape) != (B, 2, H, W):
            raise MacvoB200Error(f"pwc_warp_corr: flow {tuple(fl.shape)} must be ({B},2,{H},{W})")
    if not (isinstance(out, Tensor) and out.is_cuda and out.dtype == torch.float32 and out.is_contiguous()
            and out.dim() == 4 and out.shape[0] == B and tuple(out.shape[2:]) == (H, W)):
        raise MacvoB200Error(f"pwc_warp_corr: out must be a contiguous ({B},C_out,{H},{W}) fp32 CUDA tensor")
    if not 0 <= out_offset <= out.shape[1] - PWC_DISPLACEMENTS:
        raise MacvoB200Error(f"pwc_warp_corr: channels [{out_offset}, {out_offset + PWC_DISPLACEMENTS}) exceed out's {out.shape[1]}")
    if b.device != a.device or out.device != a.device or (fl is not None and fl.device != a.device):
        raise MacvoB200Error("pwc_warp_corr: all tensors must be on one device")
    rc = load_library().macvo_pwc_warp_corr(a.data_ptr(), b.data_ptr(), fl.data_ptr() if fl is not None else None,
                                            float(scale), B, Cc, H, W, out.data_ptr(), out.shape[1], int(out_offset),
                                            _stream())
    _check(rc, "macvo_pwc_warp_corr")
    LAUNCHES[0] += 1
    return out


# ------------------------------------------------------------------------------------------------
# (f7) TartanVODepth: both full-resolution heads + the depth conversion (csrc/stereo_head.cu)
# ------------------------------------------------------------------------------------------------
STEREO_HEAD_SMALL = 64 + 16 * 64 + 16 + 16 + 1          # b11 | w12 (16 x 64) | b12 | w13 | b13


def stereo_head(xd: Tensor, xc: Tensor | None, cat0: Tensor, w11_d: Tensor, small_d: Tensor, w11_c: Tensor | None,
                small_c: Tensor | None, bf: float, margin: tuple[int, int], depth: Tensor, var: Tensor | None) -> None:
    """TartanVODepth's heads from the conv_c10 outputs xd (disparity decoder) and xc (covariance decoder, or None) and cat0,
    all (1, 64, h2, w2), into the crop region [my, my + 2 h2) x [mx, mx + 2 w2) of depth / var (1, 1, H, W): deconv_c11 on
    TF32 tensor cores (w11_* from stereonet.arrange_head), conv_c12, conv_c13, / 0.02 and StereoCovNet.inference. The
    deconvolution is a TF32 one, so the call is refused unless torch.backends.cudnn.allow_tf32 is set (the flag under which
    cuDNN would run it in TF32 too)."""
    if not torch.backends.cudnn.allow_tf32:
        raise MacvoB200Error("stereo_head: runs deconv_c11 in TF32, but torch.backends.cudnn.allow_tf32 is False")
    if (xc is None) != (var is None) or (xc is None) != (w11_c is None) or (xc is None) != (small_c is None):
        raise MacvoB200Error("stereo_head: xc, w11_c, small_c and var go together (all or none)")
    a = _dev(xd, torch.float32, "stereo_head xd")
    k = _dev(cat0, torch.float32, "stereo_head cat0")
    if a.dim() != 4 or a.shape[:2] != (1, 64) or k.shape != a.shape:
        raise MacvoB200Error(f"stereo_head: xd {tuple(a.shape)} and cat0 {tuple(k.shape)} must both be (1,64,h2,w2)")
    h2, w2 = a.shape[-2:]
    heads = [(a, w11_d, small_d)]
    if xc is not None:
        c = _dev(xc, torch.float32, "stereo_head xc")
        if c.shape != a.shape:
            raise MacvoB200Error(f"stereo_head: xc {tuple(c.shape)} must be {tuple(a.shape)}")
        heads.append((c, w11_c, small_c))
    for _, w, sm in heads:
        if not (isinstance(w, Tensor) and w.is_cuda and w.dtype == torch.float32 and w.is_contiguous()
                and tuple(w.shape) == (4, 4, 4, 64, 32)):
            raise MacvoB200Error("stereo_head: w11 must be a contiguous (4,4,4,64,32) fp32 CUDA tensor (arrange_head)")
        if not (isinstance(sm, Tensor) and sm.is_cuda and sm.dtype == torch.float32 and sm.is_contiguous()
                and sm.numel() == STEREO_HEAD_SMALL):
            raise MacvoB200Error(f"stereo_head: small must be a contiguous fp32 CUDA tensor of {STEREO_HEAD_SMALL} floats")
    outs = [depth] + ([var] if var is not None else [])
    for o in outs:
        if not (isinstance(o, Tensor) and o.is_cuda and o.dtype == torch.float32 and o.is_contiguous() and o.dim() == 4
                and o.shape[:2] == (1, 1)):
            raise MacvoB200Error("stereo_head: depth / var must be contiguous (1,1,H,W) fp32 CUDA tensors")
    H, W = depth.shape[-2:]
    if var is not None and var.shape != depth.shape:
        raise MacvoB200Error(f"stereo_head: var {tuple(var.shape)} must be {tuple(depth.shape)}")
    my, mx = int(margin[0]), int(margin[1])
    if my < 0 or mx < 0 or my + 2 * h2 > H or mx + 2 * w2 > W:
        raise MacvoB200Error(f"stereo_head: a {2 * h2}x{2 * w2} crop at ({my}, {mx}) does not fit a {H}x{W} frame")
    devs = {t.device for t in [a, k, *outs] + [x for _, w, s in heads for x in (w, s)] + ([heads[1][0]] if xc is not None else [])}
    if len(devs) != 1:
        raise MacvoB200Error("stereo_head: all tensors must be on one device")
    bf = float(bf)
    ptr = lambda t: t.data_ptr() if t is not None else None
    rc = load_library().macvo_stereo_head(a.data_ptr(), ptr(heads[1][0]) if xc is not None else None, k.data_ptr(), h2, w2,
                                          w11_d.data_ptr(), small_d.data_ptr(), ptr(w11_c), ptr(small_c), bf, bf * bf,
                                          my, mx, H, W, depth.data_ptr(), ptr(var), _stream())
    _check(rc, "macvo_stereo_head")
    LAUNCHES[0] += 1
