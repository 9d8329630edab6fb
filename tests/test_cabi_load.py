"""No-GPU checks of the C-ABI boundary: the library builds for sm_90a, loads, and exports every
symbol include/macvo_b200.h declares (no compute call is made)."""
import os
import re
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from macvo_b200 import build, ops
    build.build(verbose=False)
    return ops.load_library()


def _header_symbols():
    text = open(os.path.join(REPO, "include", "macvo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(macvo_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(lib):
    from macvo_b200 import ops
    declared = _header_symbols()
    assert len(declared) >= 13
    assert sorted(ops.EXPORTS) == declared, "ops.EXPORTS must bind exactly what the header declares"
    for name in declared:
        assert hasattr(lib, name), name


def test_version_string(lib):
    from macvo_b200 import ops
    assert ops.version().startswith("macvo_b200") and "sm_90a" in ops.version()


def test_host_only_queries(lib):
    """workspace-size functions are pure host arithmetic"""
    assert lib.macvo_corr_workspace_bytes(2, 256, 4800, 0) == 0
    assert lib.macvo_corr_workspace_bytes(2, 256, 4800, 1) == 4 * 2 * 4800 * 256 * 2
    assert lib.macvo_corr_workspace_bytes(2, 256, 4800, 2) == 2 * 2 * 4800 * 256 * 2
    assert lib.macvo_select_workspace_bytes(480, 640) >= 480 * 640
    # padded pixel-row layouts of the decoder's tensor-core kernels (csrc/rows_layout.cuh): multiples of 256 rows + guards
    for b, h, w in ((1, 60, 80), (2, 60, 80), (2, 13, 17), (1, 90, 160)):
        for vertical, padded in ((0, b * (h + 4) * (w + 4)), (1, b * w * (h + 4))):
            rows = lib.macvo_rows_count(b, h, w, vertical)
            assert rows == -(-padded // 256) * 256 + 32 and rows == lib.macvo_gru_tc_operand_rows(b, h, w, vertical)
    assert lib.macvo_rows_count(0, 60, 80, 0) == 0


def test_tensor_core_decoder_ops_refuse_bad_arguments(lib):
    """argument validation of the decoder's tensor-core wrappers happens on the host, before any launch"""
    import torch
    from macvo_b200 import ops
    with pytest.raises(ops.MacvoB200Error):
        ops.conv_tc(torch.zeros(8, 64, dtype=torch.float16), torch.zeros(32, 64, dtype=torch.float16), None, 32, 1, False, (1, 2, 2))
    with pytest.raises(ops.MacvoB200Error):
        ops.softmax_rows_f16(torch.zeros(4, 8))
    with pytest.raises(ops.MacvoB200Error):
        ops.convex_upsample(torch.zeros(1, 2, 4, 4), torch.zeros(1, 576, 4, 4))
    w, b, n = ops.pack_conv_filter(torch.arange(2 * 3 * 9, dtype=torch.float32).reshape(2, 3, 3, 3), torch.tensor([1.0, 2.0]))
    assert tuple(w.shape) == (32, 9 * 64) and w.dtype == torch.float16 and n == 2 and tuple(b.shape) == (32,)
    assert w[1, 4 * 64 + 2].item() == float(27 + 2 * 9 + 4) and not w[2:].any() and not w[:, 3:64].any()      # K index = tap * C_pad + c


def test_sass_is_hopper_native():
    """the tensor-core kernels must contain wgmma / TMA / mbarrier SASS (HGMMA, UTMALDG, SYNCS)"""
    from macvo_b200 import build
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", build.LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "SYNCS"):
        assert mnemonic in sass, mnemonic
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", build.LIB_PATH], capture_output=True, text=True).stdout


def test_ops_refuse_cpu_tensors(lib):
    import torch
    from macvo_b200 import ops
    with pytest.raises(ops.MacvoB200Error):
        ops.corr_build(torch.zeros(1, 64, 4, 4), torch.zeros(1, 64, 4, 4))
    with pytest.raises(ops.MacvoB200Error):
        ops.corr_lookup(torch.zeros(16, 1, 4, 4), torch.zeros(1, 2, 4, 4))


def test_layer_ops_refuse_cpu_tensors(lib):
    """the perceiver / decoder layer kernels have no CPU fallback either (the network class keeps the torch ops for
    CPU tensors itself; the wrappers must fail loudly)"""
    import torch
    from macvo_b200 import ops
    z = torch.zeros
    calls = [
        lambda: ops.layer_norm(z(4, 128), z(128), z(128)),
        lambda: ops.patch_embed_conv1(z(2, 1, 8, 8), z(16, 1, 6, 6), z(16)),
        lambda: ops.small_attention(z(2, 4, 128), z(2, 4, 128), z(2, 4, 128), 8),
        lambda: ops.fused_qkv_attention(z(2, 49, 384), 8),
        lambda: ops.latent_pool(z(2, 80, 128), z(8, 128), z(128, 128), z(128, 128), z(128)),
        lambda: ops.add_rows_relu_(z(2, 80, 128), z(80, 128)),
        lambda: ops.gru_gates(z(8, 256), z(8, 512), z(8, 128), z(8, 512)),
        lambda: ops.gru_blend(z(8, 128), z(8, 128), z(8, 512), None),
        lambda: ops.gru_input(z(8, 128), z(8, 128), z(1), [z(8, 512)]),
    ]
    for call in calls:
        with pytest.raises(ops.MacvoB200Error):
            call()


def test_network_on_cpu_keeps_torch_layers():
    """FlowFormerCovNet on a CPU device never touches the CUDA library (golden-parity runs of the oracle use it)"""
    import torch
    from macvo_b200.flowformer_cov import FlowFormerCovNet, synthetic_state_dict
    from oracle import frontend as ofe
    net = FlowFormerCovNet(synthetic_state_dict(0), "cpu", corr_fn=ofe.corr_volume, lookup_fn=ofe.window_lookup, decoder_depth=1)
    assert net._ops is None
    g = torch.Generator().manual_seed(0)
    flow, cov = net.inference(torch.rand(1, 3, 64, 96, generator=g), torch.rand(1, 3, 64, 96, generator=g))
    assert flow.shape == (1, 2, 64, 96) and cov.shape == (1, 2, 64, 96) and torch.isfinite(flow).all() and (cov > 0).all()
