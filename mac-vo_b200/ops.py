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
F32, F64 = torch.float32, torch.float64

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
    "macvo_gaussian_mixture_covariance": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                    C.c_void_p, C.c_longlong, C.c_longlong, C.c_void_p]
                                          + [C.c_float] * 4 + [C.c_int] + [C.c_float] * 2 + [C.c_void_p] * 4),
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


_ERRORS = {-1: "MACVO_E_ARG", -2: "MACVO_E_WORKSPACE", -3: "MACVO_E_UNSUPPORTED", -4: "MACVO_E_DRIVER"}
_STREAM = object()      # stands for the current stream in `_launch`'s arguments, for entry points that do not take it last


def _call(name: str, *args) -> None:
    rc = getattr(load_library(), name)(*args)
    if rc != 0:
        raise MacvoB200Error(f"{name} failed: {_ERRORS.get(rc, f'cudaError {rc}')}")


def _device() -> int:
    return torch._C._cuda_getDevice()


def _ptr(t: Tensor | None, what: str, dev: int | None = None, arg: int | None = None):
    """Device pointer of a kernel operand: None -> NULL; a tensor must be a CUDA tensor on the current device `dev`,
    because the kernel is enqueued on that device's stream."""
    if t is None:
        return None
    if isinstance(t, Tensor) and t.is_cuda:
        if dev is None:
            dev = _device()
        if t.get_device() == dev:
            return t.data_ptr()
        problem = f"tensor on {t.device}, but the current device is cuda:{dev}"
    else:
        problem = f"expected a CUDA tensor (the B200 path has no CPU fallback), got {getattr(t, 'device', type(t))}"
    raise MacvoB200Error(f"{what}{'' if arg is None else f' argument {arg}'}: {problem}")


def _arg(t: Tensor | None, dtype, what: str, shape: tuple | None = None, numel: int | None = None, cols: int | None = None,
         copy: bool = False, any_strides: bool = False, optional: bool = False) -> Tensor | None:
    """Check one tensor operand and return it: a CUDA tensor of `dtype` with `shape` (None entries match any size),
    `numel` elements, or a multiple of `cols` elements (pixels-major rows). A non-contiguous tensor is copied when `copy`
    (read-only inputs), kept when `any_strides` (the kernel takes the strides), and refused otherwise (every buffer a
    kernel writes, and operands whose layout the caller must provide). None is accepted only when `optional`."""
    if t is None and optional:
        return None
    if not isinstance(t, Tensor) or not t.is_cuda:
        raise MacvoB200Error(f"{what}: expected a CUDA tensor (the B200 path has no CPU fallback), got "
                             f"{getattr(t, 'device', type(t))}")
    if t.dtype != dtype:
        raise MacvoB200Error(f"{what}: expected {dtype}, got {t.dtype}")
    if not (any_strides or t.is_contiguous()):
        if not copy:
            raise MacvoB200Error(f"{what}: expected a contiguous tensor" + (
                f" of pixels-major (.., {cols}) rows (pass conv outputs as x.permute(0, 2, 3, 1) of a channels_last map)"
                if cols else ""))
        t = t.contiguous()
    if shape is not None and (t.dim() != len(shape) or any(s is not None and s != n for s, n in zip(shape, t.shape))):
        raise MacvoB200Error(f"{what}: expected shape {tuple('*' if s is None else s for s in shape)}, got {tuple(t.shape)}")
    if numel is not None and t.numel() != numel:
        raise MacvoB200Error(f"{what}: expected {numel} elements, got {t.numel()}")
    if cols is not None and t.numel() % cols:
        raise MacvoB200Error(f"{what}: expected pixels-major (.., {cols}) rows, got {tuple(t.shape)}")
    return t


def _launch(name: str, *args, launches: int = 1) -> None:
    """Enqueue the library entry point `name` on the current stream of the current device. Tensor arguments become device
    pointers (each must live on the current device); the stream goes last, or where `_STREAM` stands; a non-zero return
    code raises; `launches` kernels are added to LAUNCHES."""
    dev = _device()
    call = [_ptr(a, name, dev, i) if isinstance(a, Tensor) else a for i, a in enumerate(args)]
    # raw cudaStream_t of torch's current stream, asked for only once every operand passed its device check (the public
    # torch.cuda.current_stream() costs ~20 us of Python per call)
    stream = torch._C._cuda_getCurrentRawStream(dev)
    if _STREAM in call:
        call[call.index(_STREAM)] = stream
    else:
        call.append(stream)
    _call(name, *call)
    LAUNCHES[0] += launches


def _mask(m: Tensor | None, what: str) -> Tensor | None:
    """optional bool / uint8 flags -> the uint8 operand the kernels read"""
    if m is None:
        return None
    return _arg(m.to(torch.uint8) if m.dtype != torch.uint8 else m, torch.uint8, what, copy=True)


def _workspace(nbytes: int, device) -> Tensor:
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
    f1 = _arg(f1, F32, "corr_build fmap1", copy=True)
    f2 = _arg(f2, F32, "corr_build fmap2", copy=True)
    out = torch.empty((B, 1, H, W, H, W), dtype=torch.float32, device=f1.device)
    nbytes = load_library().macvo_corr_workspace_bytes(B, D, n, mode)
    ws = _workspace(nbytes, f1.device) if nbytes else None
    _launch("macvo_corr_build", f1, f2, out, B, D, n, mode | (CORR_KMAJOR_INPUT if kmajor else 0), ws, nbytes,
            launches={CORR_SIMT: 1, CORR_TC_TF32: 1}.get(mode, 2))
    return out


# ------------------------------------------------------------------------------------------------
# (a5) window lookup
# ------------------------------------------------------------------------------------------------
def corr_lookup(cost_maps: Tensor, coords: Tensor, rows: bool = False) -> Tensor:
    """cost_maps (B*H1*W1, 1, H2, W2) fp32, coords (B,2,H1,W1) fp32 -> (B,81,H1,W1) fp32 (decoder.py:141-153);
    rows=True: the same values as (B*H1*W1, 81) pixels-major rows (the NHWC view)."""
    cm = _arg(cost_maps, F32, "corr_lookup cost_maps", copy=True)
    co = _arg(coords, F32, "corr_lookup coords", copy=True)
    B, _, H1, W1 = co.shape
    H2, W2 = cm.shape[-2:]
    assert cm.shape[0] == B * H1 * W1, "one cost map per query pixel"
    out = torch.empty((B * H1 * W1, 81) if rows else (B, 81, H1, W1), dtype=torch.float32, device=cm.device)
    _launch("macvo_corr_lookup_rows" if rows else "macvo_corr_lookup", cm, co, out, B, H1, W1, H2, W2)
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

    def struct(self, score_cov: Tensor | None, dcov0: Tensor | None = None, dcov1: Tensor | None = None) -> _ScoreT:
        if dcov0 is not None and self.flow_quality is None:
            self.flow_quality = torch.empty_like(self.quality)
            self.cand_vals2 = torch.empty_like(self.cand_vals)
        aware = dcov0 is not None
        dev = _device()
        p = lambda t: _ptr(t, "ScoreBuffers", dev)
        return _ScoreT(p(score_cov), p(self.quality), p(self.nms), p(self.cand_vals), p(self.n_cand), self.ksize, p(dcov0),
                       p(dcov1), p(self.flow_quality if aware else None), p(self.cand_vals2 if aware else None))


def dense_postproc(est_flow: Tensor, est_cov: Tensor | None, bl_fx: float, enforce_positive_disparity: bool = False,
                   score: ScoreBuffers | None = None) -> dict:
    """One `estimate_pair` of dense maps (Frontend.py:184-200, 291-299) + optional fused keypoint scoring.

    est_flow / est_cov: (2,2,H,W) fp32. bl_fx = baseline*fx as a python float (double), like the reference.
    est_cov None (a frontend without covariance, FlowFormerDepth / FlowFormerMatcher): est_flow (1|2,2,H,W); depth and
    disparity of slot 0, the flow of slot 1 (None for one slot); every covariance / mask output is None."""
    fl = _arg(est_flow, F32, "dense_postproc est_flow", copy=True)
    if est_cov is None:
        if enforce_positive_disparity or score is not None or fl.dim() != 4 or fl.shape[0] not in (1, 2) or fl.shape[1] != 2:
            raise MacvoB200Error("dense_postproc without est_cov: expects est_flow (1|2,2,H,W) and no mask or scoring")
        H, W = fl.shape[-2:]
        depth = torch.empty((1, 1, H, W), dtype=torch.float32, device=fl.device)
        disparity = torch.empty_like(depth)
        _launch("macvo_dense_postproc", fl, None, H, W, float(bl_fx), float(bl_fx) ** 2, depth, disparity, None, None, None, None)
        return {"depth": depth, "disparity": disparity, "depth_cov": None, "disparity_uncertainty": None, "depth_mask": None,
                "flow": fl[1:2] if fl.shape[0] == 2 else None, "flow_cov": None}
    cv = _arg(est_cov, F32, "dense_postproc est_cov", copy=True)
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
    _launch("macvo_dense_postproc", fl, cv, H, W, float(bl_fx), float(bl_fx) ** 2, depth, disparity, depth_cov, mask, flow_cov,
            C.byref(st) if st is not None else None)
    return {"depth": depth, "disparity": disparity, "depth_cov": depth_cov,
            "disparity_uncertainty": cv[0:1, :1], "depth_mask": mask.bool() if mask is not None else None,
            "flow": fl[1:2], "flow_cov": flow_cov}


def _score(match_cov: Tensor, score: ScoreBuffers, depth_cov0: Tensor | None = None, depth_cov1: Tensor | None = None) -> None:
    """the scoring pass of macvo_dense_postproc alone; with the depth covariance maps, the depth-aware quality"""
    H, W = match_cov.shape[-2:]
    score.n_cand.zero_()
    st = score.struct(match_cov, depth_cov0, depth_cov1)
    _launch("macvo_dense_postproc", None, None, H, W, 0.0, 0.0, None, None, None, None, None, C.byref(st))
    score.generation += 1


def score_only(match_cov: Tensor, score: ScoreBuffers) -> None:
    """Quality / NMS scoring of an arbitrary (1,3,H,W) covariance map (standalone selector plugin)."""
    _score(_arg(match_cov, F32, "score_only match_cov", copy=True), score)


def score_depth_aware(match_cov: Tensor, depth_cov0: Tensor, depth_cov1: Tensor, score: ScoreBuffers) -> None:
    """Scoring of the depth-aware selector: quality = (depth_cov0 + depth_cov1) * (uu + vv - 2 uv) + NMS."""
    _score(_arg(match_cov, F32, "score_depth_aware match_cov", copy=True), score,
           _arg(depth_cov0, F32, "score_depth_aware depth_cov0", copy=True),
           _arg(depth_cov1, F32, "score_depth_aware depth_cov1", copy=True))


def select_candidates_depth(score: ScoreBuffers, depth0: Tensor, depth1: Tensor, depth_cov0: Tensor, mask_width: int,
                            max_depth: float, max_depth_cov: float, max_match_cov: float, mask_a: Tensor | None,
                            mask_b: Tensor | None, out: "CandidateList") -> None:
    h, w = score.h, score.w
    if score.flow_quality is None:
        raise MacvoB200Error("select_candidates_depth: the score buffers were not filled by score_depth_aware")
    nbytes = load_library().macvo_select_workspace_bytes(h, w)
    ws = _workspace(nbytes, score.quality.device)
    ma, mb = _mask(mask_a, "select_candidates_depth mask_a"), _mask(mask_b, "select_candidates_depth mask_b")
    d0 = _arg(depth0, F32, "select_candidates_depth depth0", copy=True)
    d1 = _arg(depth1, F32, "select_candidates_depth depth1", copy=True)
    dc0 = _arg(depth_cov0, F32, "select_candidates_depth depth_cov0", copy=True)
    if out.thresh.numel() < 2:
        out.thresh = torch.zeros((2,), dtype=torch.float32, device=out.thresh.device)
    _launch("macvo_select_candidates_depth", score.flow_quality, d0, d1, dc0, score.nms, score.cand_vals, score.cand_vals2,
            score.n_cand, ma, mb, h, w, int(mask_width), float(max_depth), float(max_depth_cov), float(max_match_cov),
            out.idx, out.n, out.thresh, out.status, ws, nbytes, launches=4)


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
    h, w = score.h, score.w
    nbytes = load_library().macvo_select_workspace_bytes(h, w)
    ws = _workspace(nbytes, score.quality.device)
    _launch("macvo_select_candidates", score.quality, score.nms, score.cand_vals, score.n_cand,
            _mask(extra_mask, "select_candidates extra_mask"), h, w, int(mask_width), float(max_match_cov), out.idx, out.n,
            out.thresh, out.status, ws, nbytes, launches=3)


def select_mapping_candidates(depth: Tensor, depth_cov: Tensor, mask_width: int, max_depth: float,
                              max_depth_cov: float, out: CandidateList) -> None:
    d = _arg(depth, F32, "select_mapping_candidates depth", copy=True)
    dc = _arg(depth_cov, F32, "select_mapping_candidates depth_cov", copy=True)
    h, w = d.shape[-2:]
    nbytes = load_library().macvo_select_workspace_bytes(h, w)
    ws = _workspace(nbytes, d.device)
    out.status.zero_()
    _launch("macvo_select_mapping_candidates", d, dc, h, w, int(mask_width), float(max_depth), float(max_depth_cov), out.idx,
            out.n, ws, nbytes, launches=2)


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
            _launch("macvo_gather_pixels", cand.idx, perm_d, k, cand.w, out)
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
    sm = _arg(scalar_map, F32, "retrieve_pixels map", copy=True)
    if pixel_uv.dtype not in (torch.int64, torch.float32):
        pixel_uv = pixel_uv.float()
    kp = _arg(pixel_uv, pixel_uv.dtype, "retrieve_pixels kp", copy=True)
    Cc, H, W = sm.shape[-3:]
    K = kp.shape[0]
    out = torch.empty((Cc, K), dtype=torch.float32, device=sm.device)
    _launch("macvo_retrieve_pixels", kp, int(kp.dtype == torch.int64), K, sm, Cc, H, W, out)
    return out


# ------------------------------------------------------------------------------------------------
# (a10)
# ------------------------------------------------------------------------------------------------
def match_covariance(kp: Tensor, depth_map: Tensor, flow_cov: Tensor | None, fx: float, fy: float, cx: float,
                     cy: float, kernel_size: int = 31, min_flow_cov: float = 0.25, min_depth_cov: float = 0.05,
                     match_cov_default: float = 0.25, want_point: bool = False, depth_cov: Tensor | None = None,
                     out_cov: Tensor | None = None, depth_cov_map: Tensor | None = None):
    """-> (cov (K,3,3) float64 on the device, point (K,3) fp32 or None, status int32 tensor).

    flow_cov: (K,3) fp32 CUDA tensor with ANY strides (MAC-VO passes the transposed view of a (3,K) gather,
    Odometry/MACVO.py:231-232); its first two columns are clamped in place in the caller's storage like the reference.
    depth_cov: (K,) per-keypoint depth variance, only used when flow_cov is None (Project2to3.py:163-171).
    out_cov: optional preallocated (K,3,3) float64 CUDA view to fill (e.g. a slice of a packed buffer).
    depth_cov_map: the (1,1,H,W) per-pixel depth variance of the stereo network (`depth_est.cov`). Given, the model is
    GaussianMixtureCovariance (Project2to3.py:194-272, macvo_gaussian_mixture_covariance) instead of MatchCovariance:
    each tap a Gaussian with its own variance, the mixture's mean and halved variance, which is not clamped (the
    reference never reads min_depth_cov)."""
    dm = _arg(depth_map, F32, "match_covariance depth", copy=True)
    if kp.dtype not in (torch.int64, torch.float32):
        kp = kp.float()
    kpd = _arg(kp, kp.dtype, "match_covariance kp", copy=True)
    K = kpd.shape[0]
    H, W = dm.shape[-2:]
    fc = _arg(flow_cov, F32, "match_covariance flow_cov (clamped in place)", shape=(K, 3), any_strides=True, optional=True)
    rs, cs = 0, 0
    if fc is not None:
        rs, cs = (fc.stride(0), fc.stride(1)) if K > 0 else (3, 1)
        if K > 0 and (rs == 0 or cs == 0):
            raise MacvoB200Error("match_covariance: flow_cov is an expanded (stride-0) view; the in-place clamp needs real storage")
    dv = None
    if fc is None and depth_cov is not None:
        dv = _arg(depth_cov.reshape(-1), F32, "match_covariance depth_cov (one value per keypoint)", numel=K, copy=True)
    vm = _arg(depth_cov_map, F32, "match_covariance depth_cov_map", numel=H * W, copy=True, optional=True)
    if out_cov is None:
        cov = torch.empty((K, 3, 3), dtype=torch.float64, device=dm.device)
    else:
        cov = _arg(out_cov, F64, "match_covariance out_cov", shape=(K, 3, 3))
    pt = torch.empty((K, 3), dtype=torch.float32, device=dm.device) if want_point else None
    status = torch.zeros((1,), dtype=torch.int32, device=dm.device)
    if vm is None:
        _launch("macvo_match_covariance", kpd, int(kpd.dtype == torch.int64), K, dm, H, W, fc, rs, cs, dv, fx, fy, cx, cy,
                kernel_size, min_flow_cov, min_depth_cov, match_cov_default, cov, pt, status)
    else:
        _launch("macvo_gaussian_mixture_covariance", kpd, int(kpd.dtype == torch.int64), K, dm, vm, H, W, fc, rs, cs, dv, fx,
                fy, cx, cy, kernel_size, min_flow_cov, match_cov_default, cov, pt, status)
    return cov, pt, status


# ------------------------------------------------------------------------------------------------
# (a14) + (a15)
# ------------------------------------------------------------------------------------------------
def _pgo_params(max_steps=10, patience=2, max_reject=16, cluster=0, decreasing=1e-5, huber_delta=0.1, radius=1e3,
                diag_min=1e-6, diag_max=1e32) -> _PgoParams:
    return _PgoParams(max_steps, patience, max_reject, cluster, decreasing, huber_delta, radius, diag_min, diag_max)


def _intr(intr: tuple[float, float, float, float, float]):
    """host double[5] {fx, fy, cx, cy, baseline} of the PGO entry points"""
    return C.cast((C.c_double * 5)(*[float(v) for v in intr]), C.c_void_p)


def _pgo_solve_args(what: str, intr, init_pose: Tensor | None, pose_io: Tensor | None, stats: Tensor | None, cluster: int,
                    **kw) -> list:
    """[intr, pose_io, params, stats], which every LM solve entry point takes in this order: the pose is pose_io (7,) float64,
    solved in place, or else a copy of init_pose; stats (8,) float64 is the given buffer or else zeros"""
    if pose_io is not None:
        pose = _arg(pose_io, F64, f"{what} pose_io", numel=7)
    else:
        pose = _arg(init_pose, F64, f"{what} init_pose", copy=True).reshape(7).clone()
    if stats is None:
        stats = torch.zeros((8,), dtype=torch.float64, device=pose.device)
    else:
        stats = _arg(stats, F64, f"{what} stats", numel=8)
    return [_intr(intr), pose, C.byref(_pgo_params(cluster=cluster, **kw)), stats]


def pgo_solve(pos_Tw: Tensor, kp2_uv: Tensor, kp2_disp: Tensor, uv_cov: Tensor, disp_cov: Tensor,
              intr: tuple[float, float, float, float, float], init_pose: Tensor, cluster: int = 0, **kw):
    """All inputs CUDA float64. Returns (pose (7,) float64 CUDA, stats (8,) float64 CUDA); asynchronous."""
    P = [_arg(t, F64, f"pgo_solve arg{i}", copy=True) for i, t in enumerate((pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov))]
    solve = _pgo_solve_args("pgo_solve", intr, init_pose, None, None, cluster, **kw)
    _launch("macvo_pgo_solve", *P, P[0].shape[0], *solve)
    return solve[1], solve[3]


PGO_GRAPH_TYPES = {"disp": 0, "reproj": 1, "icp": 2}


def pgo_solve_graph(graph_type: str, pos_Tw: Tensor, intr: tuple[float, float, float, float, float], init_pose: Tensor,
                    kp2_uv: Tensor | None = None, kp2_disp: Tensor | None = None, uv_cov: Tensor | None = None,
                    disp_cov: Tensor | None = None, pc_obs: Tensor | None = None, obs_cov: Tensor | None = None,
                    pts_cov: Tensor | None = None, cluster: int = 0, **kw):
    """TwoFrame_PGO for any of its graph types ("disp" | "reproj" | "icp", Optimizer.py:51-68); CUDA float64 inputs."""
    gt = PGO_GRAPH_TYPES[graph_type]
    pos = _arg(pos_Tw, F64, "pgo_solve_graph pos_Tw", copy=True)
    arrs = [_arg(t, F64, f"pgo_solve_graph {w}", copy=True, optional=True) for t, w in
            ((kp2_uv, "kp2_uv"), (kp2_disp, "kp2_disp"), (uv_cov, "uv_cov"), (disp_cov, "disp_cov"), (pc_obs, "pc_obs"),
             (obs_cov, "obs_cov"), (pts_cov, "pts_cov"))]
    solve = _pgo_solve_args("pgo_solve_graph", intr, init_pose, None, None, cluster, **kw)
    _launch("macvo_pgo_solve_graph", gt, pos, *arrs, pos.shape[0], *solve)
    return solve[1], solve[3]


def pgo_accumulate(pos_Tw: Tensor, kp2_uv: Tensor, kp2_disp: Tensor, uv_cov: Tensor, disp_cov: Tensor,
                   intr: tuple[float, float, float, float, float], pose: Tensor, huber_delta: float = 0.1) -> Tensor:
    P = [_arg(t, F64, f"pgo_accumulate arg{i}", copy=True) for i, t in enumerate((pos_Tw, kp2_uv, kp2_disp, uv_cov, disp_cov))]
    ps = _arg(pose, F64, "pgo_accumulate pose", copy=True).reshape(7)
    acc = torch.empty((PGO_ACC,), dtype=torch.float64, device=ps.device)
    _launch("macvo_pgo_accumulate", *P, P[0].shape[0], _intr(intr), ps, float(huber_delta), acc)
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
    p = _arg(poses, F32, "motion_interpolate_ poses", shape=(None, 7))
    ni = _mask(need_interp, "motion_interpolate_ need_interp")
    F_ = p.shape[0]
    if ni.numel() != F_:
        raise MacvoB200Error("motion_interpolate_: need_interp must have one flag per frame")
    count = torch.zeros((1,), dtype=torch.int32, device=p.device)
    nbytes = load_library().macvo_motion_interpolate_workspace_bytes(F_)
    ws = _workspace(nbytes, p.device) if nbytes else None
    _launch("macvo_motion_interpolate", p, ni, F_, count, ws, nbytes)
    return count


def cov_sanity_filter(obs1_cov: Tensor, obs2_cov: Tensor) -> Tensor:
    """(K,3,3) float64 CUDA x2 -> bool (K,) mask of observations whose covariances are finite (OutlierFilter.py:91-100)"""
    a = _arg(obs1_cov, F64, "cov_sanity_filter obs1", copy=True)
    b = _arg(obs2_cov, F64, "cov_sanity_filter obs2", copy=True)
    k = a.shape[0]
    good = torch.empty((k,), dtype=torch.uint8, device=a.device)
    _launch("macvo_cov_sanity_filter", a, b, k, good)
    return good.bool()


COV_MODELS = {"match": 0, "identity": 1, "mixture": 2}   # macvo_observe_ext_t.cov_model (MACVO_COV_MATCH / _IDENTITY /
                                                         # _GAUSSIAN_MIXTURE)
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
    k = _arg(cov, F64, "cov_modify cov (modified in place)", shape=(None, 3, 3)).shape[0]
    if k and ops:
        _launch("macvo_cov_modify", cov, k, C.cast(arr, C.c_void_p), len(ops))
    return cov


def observe_pack(buf: ObservationBuffers, kp0_uv: Tensor, flow: Tensor, match_cov: Tensor | None, depth0: Tensor, depth1: Tensor,
                 disparity1: Tensor, disp_unc1: Tensor | None, edge_width: int, intr0, intr1, prev_pose: Tensor, next_pose: Tensor,
                 kernel_size: int = 31, min_flow_cov: float = 0.25, min_depth_cov: float = 0.05,
                 match_cov_default: float = 0.25, ext: dict | None = None) -> None:
    """Odometry/MACVO.py:198-283 for the two-frame graph as two launches (csrc/observe.cu); everything stays on the device.

    ext (None: CovarianceSanityFilter only) = macvo_observe_ext_t as a dict: depth_cov0 / depth_cov1 ((1,1,H,W) fp32 CUDA
    or None), simple_depth (bool), min_depth / max_depth (floats, rounded to fp32 like the reference's comparisons),
    front_of_cam (bool), icp (bool: pack the "icp" graph's columns; needs an extended buffer), cov_model ("match",
    "identity", the NoCovariance model, or "mixture", GaussianMixtureCovariance on depth_cov0 / depth_cov1, which it then
    requires) and cov_ops (modifier names of COV_OPS, innermost first).

    match_cov and disp_unc1 both None: a frontend without covariance maps (pixel2_uv_cov / pixel2_disp_cov hold -1, kp1's
    MatchCovariance uses match_cov_default unclamped; include/macvo_b200.h)."""
    kp = _arg(kp0_uv, torch.int64, "observe_pack kp0_uv", copy=True)
    k = kp.shape[0]
    fl = _arg(flow, F32, "observe_pack flow", copy=True)
    if (match_cov is None) != (disp_unc1 is None):
        raise MacvoB200Error("observe_pack: match_cov and disp_unc1 are None together (no frontend covariance) or not at all")
    mc = _arg(match_cov, F32, "observe_pack match_cov", copy=True, optional=True)
    maps = [_arg(t, F32, "observe_pack map", copy=True, optional=True) for t in (depth0, depth1, disparity1, disp_unc1)]
    H, W = fl.shape[-2:]
    if (fl.numel() != 2 * H * W or (mc is not None and mc.numel() != 3 * H * W)
            or any(m is not None and m.numel() != H * W for m in maps)):
        raise MacvoB200Error("observe_pack: expects flow (1,2,H,W), match_cov (1,3,H,W) and (1,1,H,W) maps")
    if k > buf.capacity:
        raise MacvoB200Error(f"observe_pack: {k} keypoints exceed the buffer capacity {buf.capacity}")
    pp = _arg(prev_pose, F64, "observe_pack prev_pose", copy=True)
    next_pose = _arg(next_pose, F64, "observe_pack next_pose", numel=7)
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
        dc = [_arg(ext.get(n), F32, f"observe_pack {n} ((1,1,H,W) map)", numel=H * W, copy=True, optional=True)
              for n in ("depth_cov0", "depth_cov1")]
        xs = _ObserveExt(_ptr(dc[0], "observe_pack depth_cov0"), _ptr(dc[1], "observe_pack depth_cov1"),
                         int(bool(ext.get("simple_depth"))), float(ext.get("min_depth", 0.0)), float(ext.get("max_depth", 0.0)),
                         int(bool(ext.get("front_of_cam"))), int(bool(ext.get("icp"))))
        model = ext.get("cov_model", "match")
        if model not in COV_MODELS:
            raise MacvoB200Error(f"observe_pack: cov_model must be one of {sorted(COV_MODELS)}, got {model!r}")
        if model == "mixture" and (dc[0] is None or dc[1] is None):
            raise MacvoB200Error("observe_pack: cov_model 'mixture' needs the depth-covariance maps depth_cov0 and depth_cov1")
        ops_ = tuple(ext.get("cov_ops", ()))
        xs.cov_model, xs.cov_ops, xs.n_cov_ops = COV_MODELS[model], _cov_ops(ops_, "observe_pack"), len(ops_)
    buf.status.zero_()
    _launch("macvo_observe_pack", kp if k else None, k, buf.capacity, fl, mc, *maps, H, W, int(edge_width), C.cast(i0, C.c_void_p),
            C.cast(i1, C.c_void_p), int(kernel_size), float(min_flow_cov), float(min_depth_cov), float(match_cov_default), pp,
            next_pose, buf.packed, buf.n_obs, buf.status, buf.ws, buf.ws_bytes, _STREAM, None if xs is None else C.byref(xs),
            launches=2)


def pgo_solve_counted(buf: ObservationBuffers, intr: tuple[float, float, float, float, float], pose_io: Tensor,
                      stats: Tensor, min_k: int = 10, cluster: int = 0, graph_type: str = "disp", **kw) -> None:
    """LM solve on the packed observation arrays, block count read from buf.n_obs on the device; pose_io (7,) float64
    CUDA holds the initial pose and receives the result (untouched when fewer than min_k observations survive).
    graph_type "icp" reads points_Tc / obs2_covTc / cov_Tw of an extended buffer that observe_pack filled with icp on."""
    gt = PGO_GRAPH_TYPES[graph_type]
    icp = (None, None, None)
    if gt == PGO_GRAPH_TYPES["icp"]:
        if not buf.extended:
            raise MacvoB200Error("pgo_solve_counted: graph type 'icp' needs ObservationBuffers(..., extended=True)")
        icp = tuple(buf.section(n) for n in ("points_Tc", "obs2_covTc", "cov_Tw"))
    # 0: cluster size chosen from the capacity
    intr_c, pose, prm, stats = _pgo_solve_args("pgo_solve_counted", intr, None, pose_io, stats, cluster, **kw)
    _launch("macvo_pgo_solve_counted", *(buf.section(n) for n in ("pos_Tw", "pixel2_uv", "pixel2_disp", "pixel2_uv_cov",
                                                                   "pixel2_disp_cov")),
            buf.capacity, buf.n_obs, int(min_k), intr_c, pose, prm, stats, _STREAM, gt, *icp)


class PeerExchange:
    """This rank's exchange buffer for the sharded LM kernel + the peers' buffers mapped through CUDA IPC.

    `handle` (64 bytes) must be all-gathered across the ranks (any transport: torch.distributed object / tensor gather),
    then `connect(handles)` maps every peer. One process per GPU; all ranks of one node (NVLink / NVSwitch peer access)."""

    def __init__(self, world: int, rank: int):
        self.world, self.rank = int(world), int(rank)
        self.nbytes = int(load_library().macvo_pgo_exchange_bytes(self.world))
        if self.nbytes == 0:
            raise MacvoB200Error(f"PeerExchange: world size {world} not in [1, 8]")
        ptr = C.c_void_p()
        hbuf = C.create_string_buffer(64)
        _call("macvo_p2p_alloc", self.nbytes, C.byref(ptr), hbuf)
        self.own, self.handle = ptr.value, hbuf.raw
        self.ptrs = None
        self._opened: list[int] = []

    def connect(self, handles: list[bytes]) -> None:
        arr = (C.c_void_p * self.world)()
        for r, h in enumerate(handles):
            if r == self.rank:
                arr[r] = self.own
                continue
            p = C.c_void_p()
            _call("macvo_p2p_open", C.create_string_buffer(bytes(h), 64), C.byref(p))
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
    if exchange.ptrs is None:
        raise MacvoB200Error("pgo_solve_sharded: PeerExchange.connect() has not been called")
    P = [_arg(t, F64, f"pgo_solve_sharded arg{i}", copy=True) for i, t in enumerate(shard)]
    kt = _arg(k_total, torch.int32, "pgo_solve_sharded k_total", numel=1, optional=True)
    solve = _pgo_solve_args("pgo_solve_sharded", intr, init_pose, pose_io, stats, cluster, **kw)
    _launch("macvo_pgo_solve_sharded", *P, P[0].shape[0], kt, int(k_offset), int(min_k), *solve,
            C.cast(exchange.ptrs, C.c_void_p), exchange.world, exchange.rank)
    return solve[1], solve[3]


# ---- frontend "next" rows: memory-bound perceiver layers (csrc/nn_kernels.cu) ------------------------------
LAYER_NORM_CHANNELS = (64, 128, 256, 512)


def layer_norm(x: Tensor, weight: Tensor, bias: Tensor, eps: float = 1e-5) -> Tensor:
    """nn.LayerNorm over the last dim of a contiguous fp32 CUDA tensor (warp-per-row kernel)."""
    x = _arg(x, F32, "layer_norm x", copy=True)
    c = x.shape[-1]
    if c not in LAYER_NORM_CHANNELS:
        raise MacvoB200Error(f"layer_norm: channels {c} not in {LAYER_NORM_CHANNELS}")
    y = torch.empty_like(x)
    _launch("macvo_layer_norm", x, _arg(weight, F32, "layer_norm weight", copy=True), _arg(bias, F32, "layer_norm bias", copy=True),
            y, x.numel() // c, c, float(eps))
    return y


def add_layer_norm(x: Tensor, resid: Tensor, weight: Tensor, bias: Tensor, eps: float = 1e-5) -> tuple[Tensor, Tensor]:
    """(x + resid, LayerNorm(x + resid)) in one pass over contiguous fp32 CUDA tensors of C in {128, 256, 512} channels."""
    x, resid = _arg(x, F32, "add_layer_norm x", copy=True), _arg(resid, F32, "add_layer_norm resid", copy=True)
    c = x.shape[-1]
    if c not in (128, 256, 512) or x.shape != resid.shape:
        raise MacvoB200Error(f"add_layer_norm: channels {c} / shapes {tuple(x.shape)} vs {tuple(resid.shape)} unsupported")
    s, y = torch.empty_like(x), torch.empty_like(x)
    _launch("macvo_add_layer_norm", x, resid, _arg(weight, F32, "add_layer_norm weight", copy=True),
            _arg(bias, F32, "add_layer_norm bias", copy=True), s, y, x.numel() // c, c, float(eps))
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
    xn, resid, w1, b1, w2, b2 = (_arg(t, F32, f"mlp_tc {n}", copy=True) for t, n in
                                 ((xn, "xn"), (resid, "resid"), (w1, "w1"), (b1, "b1"), (w2, "w2"), (b2, "b2")))
    c, hd = xn.shape[-1], w1.shape[0]
    if (c != 128 or hd not in MLP_TC_HIDDEN or xn.shape != resid.shape or tuple(w1.shape) != (hd, c)
            or tuple(w2.shape) != (c, hd) or b1.numel() != hd or b2.numel() != c):
        raise MacvoB200Error(f"mlp_tc: unsupported shapes xn {tuple(xn.shape)}, resid {tuple(resid.shape)}, "
                             f"w1 {tuple(w1.shape)}, w2 {tuple(w2.shape)}")
    out = torch.empty_like(resid)
    _launch("macvo_mlp_tc", xn, resid, w1, b1, w2, b2, out, xn.numel() // c, c, hd)
    return out


def patch_tokens_tc(x: Tensor, w0: Tensor, term: Tensor, w2: Tensor, b2: Tensor, ln_w: Tensor, ln_b: Tensor,
                    eps: float = 1e-5) -> Tensor:
    """LayerNorm(w2 relu(w0 x + term[row % period]) + b2) over the last dim of x (..., 64) -> (..., 128) in one TF32
    tensor-core kernel (csrc/patch_tokens_tc.cu): PatchEmbed's token head. With w0 / w2 from `round_tf32` it returns the
    bits of cuBLAS TF32 linear, add_rows_relu_, cuBLAS TF32 linear + bias and layer_norm."""
    x, w0, term, w2, b2, ln_w, ln_b = (_arg(t, F32, f"patch_tokens_tc {n}", copy=True) for t, n in
                                       ((x, "x"), (w0, "w0"), (term, "term"), (w2, "w2"), (b2, "b2"), (ln_w, "ln_w"),
                                        (ln_b, "ln_b")))
    cin, c = x.shape[-1], w0.shape[0]
    if (cin != 64 or c != 128 or tuple(w0.shape) != (c, cin) or tuple(w2.shape) != (c, c) or term.dim() != 2
            or term.shape[1] != c or term.shape[0] == 0 or any(t.numel() != c for t in (b2, ln_w, ln_b))):
        raise MacvoB200Error(f"patch_tokens_tc: unsupported shapes x {tuple(x.shape)}, w0 {tuple(w0.shape)}, "
                             f"term {tuple(term.shape)}, w2 {tuple(w2.shape)}")
    out = torch.empty(*x.shape[:-1], c, dtype=torch.float32, device=x.device)
    _launch("macvo_patch_tokens_tc", x, w0, term, w2, b2, ln_w, ln_b, out, x.numel() // cin, cin, c, term.shape[0], float(eps))
    return out


def patch_embed_conv1(maps: Tensor, weight: Tensor, bias: Tensor, allow_tf32: bool | None = None, s2d: bool = False) -> Tensor:
    """(M,1,H,W) cost maps -> ReLU(conv 6x6/2 (+ pad to x8)) as a logical (M,16,Ho,Wo) channels_last tensor; s2d=True (TF32
    variant only): the same values space-to-depth, a logical (M,64,Ho/2,Wo/2) channels_last tensor with channel
    ((y & 1) * 2 + (x & 1)) * 16 + c (see `space_to_depth_filter` for the matching 3x3 filter of the next convolution)."""
    maps = _arg(maps, F32, "patch_embed_conv1 maps", copy=True)
    m, one, h, w = maps.shape
    if one != 1 or tuple(weight.shape) != (16, 1, 6, 6):
        raise MacvoB200Error("patch_embed_conv1: expects (M,1,H,W) maps and a (16,1,6,6) weight")
    ho, wo = (h + 7) // 8 * 4, (w + 7) // 8 * 4
    tf32 = bool(torch.backends.cudnn.allow_tf32 if allow_tf32 is None else allow_tf32)
    if s2d and not tf32:
        raise MacvoB200Error("patch_embed_conv1: the space-to-depth output exists for the TF32 tensor-core variant only")
    out = torch.empty((m, ho // 2, wo // 2, 64) if s2d else (m, ho, wo, 16), dtype=torch.float32, device=maps.device)
    _launch("macvo_patch_embed_conv1", maps, _arg(weight, F32, "patch_embed_conv1 weight", copy=True),
            _arg(bias, F32, "patch_embed_conv1 bias", copy=True), out, m, h, w, int(tf32) | (2 if s2d else 0))
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
    q, k, v = (_arg(t, F32, f"small_attention {n}", copy=True) for t, n in ((q, "q"), (k, "k"), (v, "v")))
    b, nk, c = k.shape
    d = c // heads
    nq = q.shape[1]
    if q.shape[0] not in (1, b) or q.shape[2] != c or v.shape != k.shape or d * heads != c:
        raise MacvoB200Error(f"small_attention: bad shapes q{tuple(q.shape)} k{tuple(k.shape)} v{tuple(v.shape)}")
    out = torch.empty(b, nq, c, dtype=torch.float32, device=k.device)
    _launch("macvo_small_attention", q, k, v, out, b, nq, nk, heads, d, int(q.shape[0] == 1 and b > 1), int(allow_tf32))
    return out


# ---- decoder iteration glue (csrc/decoder_fused.cu) -----------------------------------------------------------
GRU_HID, GRU_IN = 128, 512


def gru_input(mf: Tensor, agg: Tensor, gamma: Tensor, bufs: list[Tensor]) -> None:
    """write x-part channels 256..511 = [mf | mf + gamma * agg] of up to 4 (pixels, 512) GRU input buffers"""
    mf, agg = _arg(mf, F32, "gru_input mf", cols=GRU_HID), _arg(agg, F32, "gru_input agg", cols=GRU_HID)
    bufs = [_arg(b, F32, "gru_input buffer", shape=(None, GRU_IN)) for b in bufs] + [None] * (4 - len(bufs))
    _launch("macvo_gru_input", mf, agg, _arg(gamma, F32, "gru_input gamma", copy=True), *bufs, mf.numel() // GRU_HID)


def gru_gates(zr: Tensor, hx: Tensor, z_out: Tensor, rhx: Tensor, bias: Tensor | None = None) -> None:
    _launch("macvo_gru_gates", _arg(zr, F32, "gru_gates zr", cols=2 * GRU_HID),
            _arg(bias, F32, "gru_gates bias", numel=2 * GRU_HID, optional=True),
            _arg(hx, F32, "gru_gates hx", shape=(None, GRU_IN)), _arg(z_out, F32, "gru_gates z_out", cols=GRU_HID),
            _arg(rhx, F32, "gru_gates rhx", shape=(None, GRU_IN)), hx.shape[0])


def gru_blend(q: Tensor, z: Tensor, hx: Tensor, h_dense: Tensor | None, bias: Tensor | None = None) -> None:
    _launch("macvo_gru_blend", _arg(q, F32, "gru_blend q", cols=GRU_HID),
            _arg(bias, F32, "gru_blend bias", numel=GRU_HID, optional=True), _arg(z, F32, "gru_blend z", cols=GRU_HID),
            _arg(hx, F32, "gru_blend hx", shape=(None, GRU_IN)),
            _arg(h_dense, F32, "gru_blend h_dense", cols=GRU_HID, optional=True), hx.shape[0])


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
    in_rows, weights = _arg(in_rows, torch.float16, "conv_tc in_rows"), _arg(weights, torch.float16, "conv_tc weights")
    out16 = _arg(out16, torch.float16, "conv_tc out16", optional=True)
    out32 = _arg(out32, F32, "conv_tc out32", optional=True)
    bias = _arg(bias, F32, "conv_tc bias", optional=True)
    c_in = in_rows.shape[1]
    if weights.shape[1] != ksize * ksize * c_in or (bias is not None and bias.numel() != weights.shape[0]):
        raise MacvoB200Error("conv_tc: filter / bias shape does not match the input rows")
    need = B * H * W if in_dense else rows_count(B, H, W)
    if in_rows.shape[0] != need:
        raise MacvoB200Error(f"conv_tc: expected {need} input rows, got {in_rows.shape[0]}")
    planes = add_to_map is not None
    if planes:
        if out32 is not None:
            raise MacvoB200Error("conv_tc: add_to_map excludes out32")
        out32 = _arg(add_to_map, F32, "conv_tc add_to_map", shape=(B, n_valid, H, W))
    for t, dense, off in ((out16, out16_dense, out16_offset), (None if planes else out32, True, out32_offset)):
        if t is not None and (t.shape[0] != (B * H * W if dense else rows_count(B, H, W)) or off + n_valid > t.shape[1]):
            raise MacvoB200Error("conv_tc: output rows / channel range do not fit")
    _launch("macvo_conv_tc", in_rows, c_in, int(in_dense), weights, bias, weights.shape[0], n_valid, ksize, int(relu), B, H, W,
            out16, 0 if out16 is None else out16.shape[1], out16_offset, int(out16_dense),
            out32, 0 if out32 is None else out32.shape[1], out32_offset, int(planes))


def flow_im2col(coords1: Tensor, coords0: Tensor, rows: Tensor, mf32: Tensor | None, mf16_rows: Tensor | None) -> None:
    """7x7 neighbourhoods of flow = coords1 - coords0 as (pixels, 128) fp16 GEMM rows; flow -> channels 126, 127 of the mf rows"""
    c1, c0 = _arg(coords1, F32, "flow_im2col coords1", copy=True), _arg(coords0, F32, "flow_im2col coords0", copy=True)
    B, _, H, W = c1.shape
    _launch("macvo_flow_im2col", c1, c0, _arg(rows, torch.float16, "flow_im2col rows"),
            _arg(mf32, F32, "flow_im2col mf32", shape=(B * H * W, 128), optional=True),
            _arg(mf16_rows, torch.float16, "flow_im2col mf16_rows", optional=True), B, H, W)


def pack_rows(src: Tensor, dst: Tensor, offset: int, shape: tuple[int, int, int], vertical: int = 0) -> None:
    """fp32 dense pixel rows (pixels, C), or any contiguous (.., C) tensor of B*H*W rows -> fp16 padded rows
    dst[:, offset : offset + C] (layout U, or V when `vertical`)"""
    B, H, W = shape
    src = _arg(src, F32, "pack_rows src")
    if src.dim() == 0 or src.numel() != B * H * W * src.shape[-1]:
        raise MacvoB200Error("pack_rows: expected contiguous fp32 (pixels, C) rows")
    dst = _arg(dst, torch.float16, "pack_rows dst")
    _launch("macvo_gru_tc_pack", src, src.shape[-1], src.shape[-1], dst, dst.shape[1], offset, B, H, W, vertical)


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
        self._device_index = self.h[0].get_device()
        self._side = torch.cuda.Stream(device) if self.units == 2 else None

    def set_context(self, inp_rows: Tensor) -> None:
        """x channels [0, 128) = the context features `inp` (constant over the refinement iterations)"""
        inp_rows = _arg(inp_rows, F32, "SepConvGruTC context", cols=GRU_HID).view(-1, GRU_HID)
        for o in (0, 1):
            pack_rows(inp_rows, self.x[o], 0, self.shape, o)

    def set_state(self, unit: int, h_rows: Tensor) -> None:
        self.h[unit].copy_(_arg(h_rows, F32, "SepConvGruTC state", cols=GRU_HID).view(-1, GRU_HID))
        pack_rows(self.h[unit], self.h_rows[0][unit], 0, self.shape, 0)

    def step(self, mf: Tensor, agg: Tensor, gamma: Tensor) -> torch.cuda.Event | None:
        """one SepConvGRU update of every unit with x = [inp | mf | mf + gamma * agg]; new state in `self.h[u]`.
        One 4-launch chain per unit: with 84 CTA tiles per unit (640x480: two 60x80 maps) a launch covering both units would be
        168 CTAs = two waves on 132 SMs per stage, two independent chains of 84-CTA launches keep the SMs filled across the stage
        boundaries. Unit 0's chain runs on the current stream, unit 1's on a side stream; the returned event marks the end of
        unit 1's chain, and whatever reads unit 1's state must make its stream wait on it. With one unit there is no side
        stream and no event (None)."""
        B, H, W = self.shape
        if self._device_index != _device():     # the chains below launch with the pointers taken at construction
            raise MacvoB200Error(f"SepConvGruTC.step: the unit lives on cuda:{self._device_index}, but the current device is "
                                 f"cuda:{_device()}")
        mf, agg = _arg(mf, F32, "SepConvGruTC mf", cols=GRU_HID), _arg(agg, F32, "SepConvGruTC agg", cols=GRU_HID)
        if mf.numel() != B * H * W * GRU_HID or agg.numel() != mf.numel():
            raise MacvoB200Error("SepConvGruTC.step: expected (pixels, 128) rows")
        main = torch.cuda.current_stream()
        # the count covers the pack and every unit's chain
        _launch("macvo_gru_tc_pack_motion", mf, agg, _arg(gamma, F32, "SepConvGruTC gamma", copy=True), self.x[0], self.x[1],
                B, H, W, launches=1 + self.LAUNCHES_PER_UNIT * self.units)
        unit1_done = None
        if self.units == 2:
            fork = torch.cuda.Event()
            fork.record(main)
            self._side.wait_event(fork)
            self._chain(1, self._side)
            unit1_done = torch.cuda.Event()
            unit1_done.record(self._side)
        self._chain(0, main)
        return unit1_done

    def _chain(self, unit: int, stream: torch.cuda.Stream) -> None:
        """the 1x5 pass, then the 5x1 pass, of one unit: stage 0 (z | r) and stage 1 (q + blend) each"""
        B, H, W = self.shape
        for o in (0, 1):
            for stage in (0, 1):
                _call("macvo_gru_tc_stage", stage, o, B, H, W, *self._stage_args[unit, o, stage], stream.cuda_stream)


def convex_upsample(flow: Tensor, mask_logits: Tensor, scale: float = 1.0) -> Tensor:
    """`upsample_flow` (core/decoder.py:131-139) in one kernel: flow (B,2,H,W), mask_logits (B,576,H,W) -> (B,2,8H,8W); the
    softmax runs over scale * mask_logits"""
    f = _arg(flow, F32, "convex_upsample flow", copy=True)
    B, c, H, W = f.shape
    if c != 2:
        raise MacvoB200Error("convex_upsample: expects flow (B,2,H,W)")
    m = _arg(mask_logits, F32, "convex_upsample mask_logits", shape=(B, 576, H, W), any_strides=True)
    out = torch.empty((B, 2, 8 * H, 8 * W), dtype=torch.float32, device=f.device)
    _launch("macvo_convex_upsample", f, m.permute(0, 2, 3, 1).contiguous(), out, float(scale), B, H, W)
    return out


def softmax_rows_f16(scores: Tensor) -> Tensor:
    """softmax over the last dimension of fp32 scores, written as fp16 (the GMA attention matrix under TF32; gma.py:39-82)"""
    x = _arg(scores, F32, "softmax_rows_f16 scores", copy=True)
    cols = x.shape[-1]
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _launch("macvo_softmax_rows_f16", x, out, x.numel() // cols, cols)
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
    cf = _arg(cost_forward, F32, "decoder_token cost_forward", cols=81)
    co = _arg(coords, F32, "decoder_token coords", copy=True)
    B, _, H, W = co.shape
    P = B * H * W
    k, v = _arg(key, F32, "decoder_token key", cols=64), _arg(value, F32, "decoder_token value", cols=64)
    if cf.numel() != P * 81 or k.numel() != P * 512 or v.numel() != P * 512:
        raise MacvoB200Error("decoder_token: expects cost_forward (P,81), key / value (P,8,64) with P = B*H*W")
    blob = _arg(blob, F32, "decoder_token blob")
    if out16_rows is not None:
        _launch("macvo_decoder_token_rows", cf, co, k, v, blob,
                _arg(out16_rows, torch.float16, "decoder_token out16_rows", shape=(rows_count(B, H, W), 192)), B, H, W, float(eps))
        return out16_rows
    out = torch.empty((P, 160), dtype=torch.float32, device=cf.device)
    _launch("macvo_decoder_token", cf, co, k, v, blob, out, B, H * W, float(eps))
    return out


def add_rows_relu_(x: Tensor, term: Tensor) -> Tensor:
    """in place relu(x + term[row % period]) on x (rows, C) / (M, period, C) with term (period, C)"""
    c = x.shape[-1]
    _arg(x, F32, "add_rows_relu_ x", cols=c)
    term = _arg(term, F32, "add_rows_relu_ term", cols=c)
    _launch("macvo_add_rows_relu", x, term, x.numel() // c, term.numel() // c, c)
    return x


def fused_qkv_attention(qkv: Tensor, heads: int, q_add: Tensor | None = None, k_add: Tensor | None = None,
                        allow_tf32: bool | None = None) -> Tensor:
    """attention on a fused projection output qkv (B, N, 3*C) = [q | k | v] consumed in place (self-attention, Nq = Nk = N);
    q_add / k_add (period, N, C): additive terms, batch b uses slice b % period. -> (B, N, C)"""
    qkv = _arg(qkv, F32, "fused_qkv_attention qkv", copy=True)
    b, n, c3 = qkv.shape
    c = c3 // 3
    if allow_tf32 is None:
        allow_tf32 = bool(torch.backends.cuda.matmul.allow_tf32)
    period = 0
    for t in (q_add, k_add):
        if t is not None:
            _arg(t, F32, "fused_qkv_attention additive term", cols=c)
            if t.shape[-2] != n:
                raise MacvoB200Error("fused_qkv_attention: additive terms must be (period, N, C)")
            period = t.numel() // (n * c)
    out = torch.empty(b, n, c, dtype=torch.float32, device=qkv.device)
    q, k, v = qkv.split(c, dim=-1)      # column slices of every 3c-float row, read with the row pitch c3
    _launch("macvo_small_attention_ex", q, k, v, out, b, n, n, heads, c // heads, 0, int(allow_tf32), c3, c3, c3, q_add, k_add,
            period)
    return out


def attention_with_terms(q: Tensor, k: Tensor, v: Tensor, heads: int, q_add: Tensor | None = None,
                         allow_tf32: bool | None = None) -> Tensor:
    """small_attention with q_add (period, Nq, C) added to q on load (batch b uses slice b % period)"""
    q, k, v = (_arg(t, F32, f"attention_with_terms {n}", copy=True) for t, n in ((q, "q"), (k, "k"), (v, "v")))
    b, nk, c = k.shape
    nq = q.shape[1]
    if allow_tf32 is None:
        allow_tf32 = bool(torch.backends.cuda.matmul.allow_tf32)
    q_add = _arg(q_add, F32, "attention_with_terms q_add", cols=c, optional=True)
    period = 0 if q_add is None else q_add.numel() // (nq * c)
    out = torch.empty(b, nq, c, dtype=torch.float32, device=k.device)
    _launch("macvo_small_attention_ex", q, k, v, out, b, nq, nk, heads, c // heads, 0, int(allow_tf32), 0, 0, 0, q_add, None,
            period)
    return out


def latent_pool(tokens: Tensor, q: Tensor, wk: Tensor, wv: Tensor, bv: Tensor) -> Tensor:
    """Perceiver input-layer attention without K / V: tokens (M, nk, 128), q (8, 128) shared latent queries (already
    projected), wk / wv (128, 128), bv (128) -> (M, 8, 128). TF32 tensor cores (see macvo_latent_pool)."""
    tokens = _arg(tokens, F32, "latent_pool tokens", cols=128)
    m, nk, c = tokens.shape
    if c != 128 or tuple(q.shape[-2:]) != (8, 128):
        raise MacvoB200Error("latent_pool: expects tokens (M, nk, 128) and q (8, 128)")
    # U^T[h*8 + i, :] = Wk[h*16:(h+1)*16, :]^T q[i, h*16:(h+1)*16] / sqrt(16)
    ut = torch.einsum("ihd,hdc->hic", q.reshape(8, 8, 16), wk.reshape(8, 16, 128)).reshape(64, 128).mul_(0.25).contiguous()
    out = torch.empty(m, 8, 128, dtype=torch.float32, device=tokens.device)
    _launch("macvo_latent_pool", tokens, ut, _arg(wv, F32, "latent_pool wv", cols=128),
            _arg(bv, F32, "latent_pool bv", numel=128, optional=True), out, m, nk)
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
    fl = _arg(flow, F32, "posenet_input flow", copy=True)
    dp = _arg(depth, F32, "posenet_input depth", copy=True)
    H, W = fl.shape[-2:]
    if fl.numel() != 2 * H * W or dp.numel() != H * W:
        raise MacvoB200Error("posenet_input: expects flow (1,2,H,W) and depth (1,1,H,W)")
    if H < POSENET_H or W < POSENET_W:
        raise MacvoB200Error(f"posenet_input: maps of {H}x{W} are smaller than the network input {POSENET_H}x{POSENET_W}")
    _launch("macvo_posenet_input", fl, dp, H, W, float(bl_fx),
            _arg(out, F32, "posenet_input out (1,5,112,160)", numel=5 * POSENET_H * POSENET_W))


def posenet_conv(x: Tensor, packed: Tensor, co_tile: int, bias: Tensor, ksize: int, stride: int, pad: int,
                 resid: Tensor | None = None, relu: bool = False, out: Tensor | None = None) -> Tensor:
    """epilogue(conv2d(x, W, bias, stride, pad) [+ resid]) for one image x (cin,hi,wi) (a leading batch of 1 is accepted);
    W given as pack_posenet_conv's slabs. Returns (1, cout, ho, wo)."""
    x = _arg(x, F32, "posenet_conv x", copy=True)
    cin, hi, wi = x.shape[-3:]
    if x.numel() != cin * hi * wi:
        raise MacvoB200Error("posenet_conv: x must hold one image")
    b = _arg(bias, F32, "posenet_conv bias", copy=True)
    cout = b.numel()
    pk = _arg(packed, F32, "posenet_conv weights", copy=True)
    if pk.numel() != cout * cin * ksize * ksize:
        raise MacvoB200Error(f"posenet_conv: {pk.numel()} packed weights for cout {cout}, cin {cin}, k {ksize}")
    ho, wo = (hi + 2 * pad - ksize) // stride + 1, (wi + 2 * pad - ksize) // stride + 1
    if out is None:
        out = torch.empty((1, cout, ho, wo), dtype=torch.float32, device=x.device)
    else:
        _arg(out, F32, "posenet_conv out", numel=cout * ho * wo)
    r = _arg(resid, F32, "posenet_conv resid (the output's shape)", numel=cout * ho * wo, copy=True, optional=True)
    _launch("macvo_posenet_conv", x, cin, hi, wi, pk, b, cout, ksize, stride, pad, int(co_tile), r, int(bool(relu)), out)
    return out


def posenet_head_floats() -> int:
    return int(load_library().macvo_posenet_head_floats())


def posenet_head(fc1_out: Tensor, head_blob: Tensor, prev_pose: Tensor, motion: Tensor, next_pose: Tensor) -> None:
    """fc2 / fc3 of both heads x pose_norm -> motion (6,) fp32, and next_pose (7,) float64 = prev_pose @ se3(motion).Exp()"""
    h = _arg(fc1_out, F32, "posenet_head fc1_out", copy=True)
    blob = _arg(head_blob, F32, "posenet_head blob", copy=True)
    pp = _arg(prev_pose, F64, "posenet_head prev_pose", copy=True)
    if h.numel() != 256 or blob.numel() != posenet_head_floats() or pp.numel() != 7:
        raise MacvoB200Error("posenet_head: expects fc1_out (256,), the head blob and prev_pose (7,)")
    _launch("macvo_posenet_head", h, blob, pp, _arg(motion, F32, "posenet_head motion", numel=6),
            _arg(next_pose, F64, "posenet_head next_pose", numel=7))


# ------------------------------------------------------------------------------------------------
# (f6) TartanVOMatcher's PWC-Net: warp + correlation + LeakyReLU of one level (csrc/pwc_corr.cu)
# ------------------------------------------------------------------------------------------------
PWC_DISPLACEMENTS = 81


def pwc_warp_corr(f1: Tensor, f2: Tensor, flow: Tensor | None, scale: float, out: Tensor, out_offset: int) -> Tensor:
    """LeakyReLU_0.1(correlation(f1, warp(f2, scale * flow))) of PWCDCNet_Adapted (no warp when flow is None) written into
    channels [out_offset, out_offset + 81) of out (B, C_out, H, W); f1, f2 (B, C, H, W), flow (B, 2, H, W). Returns out."""
    a = _arg(f1, F32, "pwc_warp_corr f1", copy=True)
    b = _arg(f2, F32, "pwc_warp_corr f2", copy=True)
    if a.dim() != 4 or b.shape != a.shape:
        raise MacvoB200Error(f"pwc_warp_corr: f1 {tuple(a.shape)} and f2 {tuple(b.shape)} must be the same (B,C,H,W)")
    B, Cc, H, W = a.shape
    fl = _arg(flow, F32, "pwc_warp_corr flow", shape=(B, 2, H, W), copy=True, optional=True)
    _arg(out, F32, "pwc_warp_corr out", shape=(B, None, H, W))
    if not 0 <= out_offset <= out.shape[1] - PWC_DISPLACEMENTS:
        raise MacvoB200Error(f"pwc_warp_corr: channels [{out_offset}, {out_offset + PWC_DISPLACEMENTS}) exceed out's {out.shape[1]}")
    _launch("macvo_pwc_warp_corr", a, b, fl, float(scale), B, Cc, H, W, out, out.shape[1], int(out_offset))
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
    a = _arg(xd, F32, "stereo_head xd", copy=True)
    k = _arg(cat0, F32, "stereo_head cat0", copy=True)
    if a.dim() != 4 or a.shape[:2] != (1, 64) or k.shape != a.shape:
        raise MacvoB200Error(f"stereo_head: xd {tuple(a.shape)} and cat0 {tuple(k.shape)} must both be (1,64,h2,w2)")
    h2, w2 = a.shape[-2:]
    # the covariance head's operands are None exactly when xc is (checked above)
    c = _arg(xc, F32, "stereo_head xc", shape=tuple(a.shape), copy=True, optional=True)
    for w, s, head, optional in ((w11_d, small_d, "d", False), (w11_c, small_c, "c", True)):
        _arg(w, F32, f"stereo_head w11_{head} (arrange_head)", shape=(4, 4, 4, 64, 32), optional=optional)
        _arg(s, F32, f"stereo_head small_{head}", numel=STEREO_HEAD_SMALL, optional=optional)
    _arg(depth, F32, "stereo_head depth", shape=(1, 1, None, None))
    H, W = depth.shape[-2:]
    _arg(var, F32, "stereo_head var", shape=tuple(depth.shape), optional=True)
    my, mx = int(margin[0]), int(margin[1])
    if my < 0 or mx < 0 or my + 2 * h2 > H or mx + 2 * w2 > W:
        raise MacvoB200Error(f"stereo_head: a {2 * h2}x{2 * w2} crop at ({my}, {mx}) does not fit a {H}x{W} frame")
    bf = float(bf)
    _launch("macvo_stereo_head", a, c, k, h2, w2, w11_d, small_d, w11_c, small_c, bf, bf * bf, my, mx, H, W, depth, var)
