"""Recipe: compile the MAC-VO tree's own PWC-Net correlation kernels (Module/Network/PWCNet/pwc/correlation.py:
kernel_Correlation_rearrange and kernel_Correlation_updateOutput) for sm_90a into oracle/_ref/, so that the GPU tests can pin
macvo_pwc_warp_corr to the reference kernel itself rather than to a restatement of it.

correlation.py holds the kernels as source strings whose SIZE_* macros cupy expands per call (`cupy_kernel`). This recipe
reads the file from the MAC-VO tree at build time (MACVO_REFERENCE_ROOT, default /root/reference), loads it with a stub
`cupy` module, expands the macros with the file's own `cupy_kernel` for each shape in SHAPES (the per-level shapes of the
tests/golden/tartanvo_flow_* cases) and compiles the result with nvcc, together with host launchers written here that
issue the launches of _FunctionCorrelation.forward (correlation.py:290-321). Nothing of the reference enters the
repository: the expanded source and the library live under oracle/_ref/, which git ignores. Without a MAC-VO tree the
recipe does nothing and leaves an existing oracle/_ref/ alone.

    ref_corr_<C>_<H>_<W>(f1, f2, out, rbot0, rbot1, stream): out (1,81,H,W) = correlation(f1, f2) (before LeakyReLU);
    rbot0 / rbot1 are zero-filled (1,H+8,W+8,C) fp32 scratch tensors, as the reference allocates them.
"""
from __future__ import annotations

import importlib.util
import os
import subprocess
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
LIB_PATH = os.path.join(OUT_DIR, "libref_correlation.so")
SRC_REL = os.path.join("Module", "Network", "PWCNet", "pwc", "correlation.py")
FEAT_CH = {2: 32, 3: 64, 4: 96, 5: 128, 6: 196}
CASE_SIZES = ((200, 264), (376, 780), (480, 640), (480, 752))     # tests/golden/tartanvo_cases.CASES


def _shapes() -> list[tuple[int, int, int]]:
    out = []
    for H, W in CASE_SIZES:
        h64, w64 = H // 64 * 64, W // 64 * 64
        for level, C in FEAT_CH.items():
            s = (C, h64 >> level, w64 >> level)
            if s not in out:
                out.append(s)
    return out


SHAPES = _shapes()


def symbol(C: int, H: int, W: int) -> str:
    return f"ref_corr_{C}_{H}_{W}"


def _reference_root() -> str:
    return os.environ.get("MACVO_REFERENCE_ROOT", "/root/reference")


def _load_correlation_module(path: str):
    stub = types.ModuleType("cupy")
    stub.memoize = lambda **kw: (lambda f: f)
    saved = sys.modules.get("cupy")
    sys.modules["cupy"] = stub
    try:
        spec = importlib.util.spec_from_file_location("_macvo_ref_correlation", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            sys.modules.pop("cupy", None)
        else:
            sys.modules["cupy"] = saved
    return mod


def generate_source(path: str) -> str:
    import torch
    mod = _load_correlation_module(path)
    parts = ["#include <cuda_runtime.h>\n"]
    for C, H, W in SHAPES:
        tag = f"{C}_{H}_{W}"
        first = torch.empty((1, C, H, W), device="meta")
        rbot = torch.empty((1, H + 8, W + 8, C), device="meta")
        top = torch.empty((1, 81, H, W), device="meta")
        rearr = mod.cupy_kernel("kernel_Correlation_rearrange", {"input": first, "output": rbot})
        upd = mod.cupy_kernel("kernel_Correlation_updateOutput", {"rbot0": rbot, "rbot1": rbot, "top": top})
        parts.append(rearr.replace("kernel_Correlation_rearrange(", f"kernel_Correlation_rearrange_{tag}("))
        parts.append(upd.replace("kernel_Correlation_updateOutput(", f"kernel_Correlation_updateOutput_{tag}("))
        parts.append(f"""
extern "C" int {symbol(C, H, W)}(const float* f1, const float* f2, float* out, float* rbot0, float* rbot1, void* stream) {{
    cudaStream_t s = (cudaStream_t)stream;
    const int n = {H * W};
    kernel_Correlation_rearrange_{tag}<<<dim3((n + 15) / 16, {C}, 1), dim3(16, 1, 1), 0, s>>>(n, f1, rbot0);
    kernel_Correlation_rearrange_{tag}<<<dim3((n + 15) / 16, {C}, 1), dim3(16, 1, 1), 0, s>>>(n, f2, rbot1);
    kernel_Correlation_updateOutput_{tag}<<<dim3({W}, {H}, 1), dim3(32, 1, 1), {C} * 4, s>>>({81 * H * W}, rbot0, rbot1, out);
    return (int)cudaGetLastError();
}}
""")
    return "\n".join(parts)


def build(verbose: bool = True) -> str | None:
    """compile oracle/_ref/libref_correlation.so from the MAC-VO tree; None (and no change) when the tree is absent"""
    src_py = os.path.join(_reference_root(), SRC_REL)
    if not os.path.isfile(src_py):
        if verbose:
            print(f"[ref_correlation] {src_py} not found: reference correlation kernels not built", file=sys.stderr)
        return None
    source = generate_source(src_py)
    os.makedirs(OUT_DIR, exist_ok=True)
    cu = os.path.join(OUT_DIR, "ref_correlation.cu")
    if os.path.exists(LIB_PATH) and os.path.exists(cu) and open(cu).read() == source:
        return LIB_PATH
    with open(cu, "w") as f:
        f.write(source)
    from macvo_b200.build import _nvcc
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC", "-o", LIB_PATH, cu]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        os.remove(cu)
        raise RuntimeError(f"nvcc failed on the reference correlation kernels:\n{r.stdout}")
    if verbose:
        print(f"[ref_correlation] built {LIB_PATH} ({len(SHAPES)} shapes)", file=sys.stderr)
    return LIB_PATH


if __name__ == "__main__":
    build()
