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


# public functions of ops that take no device operand: host arithmetic, size queries and weight packing
HOST_ONLY = {"version", "load_library", "default_corr_mode", "round_tf32", "space_to_depth_filter", "rows_count",
             "pack_conv_filter", "decoder_token_blob", "posenet_co_tile", "pack_posenet_conv", "posenet_head_floats",
             "request_candidate_counts"}
# wrappers whose buffer objects (CandidateList, ObservationBuffers: pinned memory, events) need a CUDA driver to construct;
# tests/test_gpu_ops_args.py checks them
NEEDS_CUDA_BUFFERS = {"select_candidates", "select_candidates_depth", "sample_candidates", "sample_candidates_many",
                      "sample_from_counts", "observe_pack", "pgo_solve_counted"}


def _cpu_calls():
    """one call per public wrapper with CPU tensors where the kernel needs device memory"""
    import types
    import torch
    from macvo_b200 import ops
    z = torch.zeros
    f64 = lambda *s: z(*s, dtype=torch.float64)
    pgo = [f64(5, 3), f64(5, 2), f64(5), f64(5, 3), f64(5)]
    intr = (1.0, 1.0, 1.0, 1.0, 1.0)
    return {
        "corr_build": lambda: ops.corr_build(z(1, 64, 4, 4), z(1, 64, 4, 4)),
        "corr_lookup": lambda: ops.corr_lookup(z(16, 1, 4, 4), z(1, 2, 4, 4)),
        "dense_postproc": lambda: ops.dense_postproc(z(2, 2, 4, 4), z(2, 2, 4, 4), 80.0),
        "score_only": lambda: ops.score_only(z(1, 3, 4, 4), ops.ScoreBuffers(4, 4, "cpu", 5)),
        "score_depth_aware": lambda: ops.score_depth_aware(z(1, 3, 4, 4), z(1, 1, 4, 4), z(1, 1, 4, 4),
                                                           ops.ScoreBuffers(4, 4, "cpu", 5)),
        "select_mapping_candidates": lambda: ops.select_mapping_candidates(z(1, 1, 4, 4), z(1, 1, 4, 4), 4, 10.0, 1.0, None),
        "retrieve_pixels": lambda: ops.retrieve_pixels(z(5, 2, dtype=torch.int64), z(1, 1, 4, 4)),
        "match_covariance": lambda: ops.match_covariance(z(5, 2, dtype=torch.int64), z(1, 1, 4, 4), z(5, 3), 1.0, 1.0, 1.0, 1.0),
        "pgo_solve": lambda: ops.pgo_solve(*pgo, intr, f64(7)),
        "pgo_solve_graph": lambda: ops.pgo_solve_graph("disp", pgo[0], intr, f64(7), *pgo[1:]),
        "pgo_accumulate": lambda: ops.pgo_accumulate(*pgo, intr, f64(7)),
        "pgo_solve_sharded": lambda: ops.pgo_solve_sharded(pgo, intr, f64(7), types.SimpleNamespace(ptrs=1, world=1, rank=0)),
        "motion_interpolate_": lambda: ops.motion_interpolate_(z(3, 7), z(3, dtype=torch.bool)),
        "cov_sanity_filter": lambda: ops.cov_sanity_filter(f64(3, 3, 3), f64(3, 3, 3)),
        "cov_modify": lambda: ops.cov_modify(f64(3, 3, 3), ["diagonalize"]),
        "layer_norm": lambda: ops.layer_norm(z(4, 128), z(128), z(128)),
        "add_layer_norm": lambda: ops.add_layer_norm(z(4, 128), z(4, 128), z(128), z(128)),
        "mlp_tc": lambda: ops.mlp_tc(z(4, 128), z(4, 128), z(128, 128), z(128), z(128, 128), z(128)),
        "patch_tokens_tc": lambda: ops.patch_tokens_tc(z(4, 64), z(128, 64), z(2, 128), z(128, 128), z(128), z(128), z(128)),
        "patch_embed_conv1": lambda: ops.patch_embed_conv1(z(2, 1, 8, 8), z(16, 1, 6, 6), z(16)),
        "small_attention": lambda: ops.small_attention(z(2, 4, 128), z(2, 4, 128), z(2, 4, 128), 8),
        "gru_input": lambda: ops.gru_input(z(8, 128), z(8, 128), z(1), [z(8, 512)]),
        "gru_gates": lambda: ops.gru_gates(z(8, 256), z(8, 512), z(8, 128), z(8, 512)),
        "gru_blend": lambda: ops.gru_blend(z(8, 128), z(8, 128), z(8, 512), None),
        "conv_tc": lambda: ops.conv_tc(z(8, 64, dtype=torch.float16), z(32, 64, dtype=torch.float16), None, 32, 1, False,
                                       (1, 2, 2)),
        "flow_im2col": lambda: ops.flow_im2col(z(1, 2, 2, 2), z(1, 2, 2, 2), z(4, 128, dtype=torch.float16), z(4, 128), None),
        "pack_rows": lambda: ops.pack_rows(z(4, 64), z(8, 64, dtype=torch.float16), 0, (1, 2, 2)),
        "convex_upsample": lambda: ops.convex_upsample(z(1, 2, 4, 4), z(1, 576, 4, 4)),
        "softmax_rows_f16": lambda: ops.softmax_rows_f16(z(4, 8)),
        "decoder_token": lambda: ops.decoder_token(z(4, 81), z(1, 2, 2, 2), z(4, 8, 64), z(4, 8, 64), z(10)),
        "add_rows_relu_": lambda: ops.add_rows_relu_(z(2, 80, 128), z(80, 128)),
        "fused_qkv_attention": lambda: ops.fused_qkv_attention(z(2, 49, 384), 8),
        "attention_with_terms": lambda: ops.attention_with_terms(z(2, 4, 128), z(2, 4, 128), z(2, 4, 128), 8),
        "latent_pool": lambda: ops.latent_pool(z(2, 80, 128), z(8, 128), z(128, 128), z(128, 128), z(128)),
        "posenet_input": lambda: ops.posenet_input(z(1, 2, 112, 160), z(1, 1, 112, 160), 1.0, z(1, 5, 112, 160)),
        "posenet_conv": lambda: ops.posenet_conv(z(8, 4, 4), z(32 * 8 * 9), 1, z(32), 3, 1, 1),
        "posenet_head": lambda: ops.posenet_head(z(256), z(16), f64(7), z(6), f64(7)),
        "pwc_warp_corr": lambda: ops.pwc_warp_corr(z(1, 4, 4, 4), z(1, 4, 4, 4), None, 1.0, z(1, 81, 4, 4), 0),
        "stereo_head": lambda: ops.stereo_head(z(1, 64, 2, 3), None, z(1, 64, 2, 3), z(4, 4, 4, 64, 32),
                                               z(ops.STEREO_HEAD_SMALL), None, None, 1.0, (0, 0), z(1, 1, 4, 6), None),
    }


def test_layer_ops_refuse_cpu_tensors(lib):
    """no wrapper has a CPU fallback (the network classes keep the torch ops for CPU tensors themselves; the wrappers must
    fail loudly), and nothing is counted as launched"""
    from macvo_b200 import ops
    for name, call in _cpu_calls().items():
        n0 = ops.LAUNCHES[0]
        with pytest.raises(ops.MacvoB200Error, match="expected a CUDA tensor"):
            call()
        assert ops.LAUNCHES[0] == n0, name


def test_pgo_accumulate_refuses_cpu_tensors_for_every_graph_type(lib):
    """pgo_accumulate's other graph types (graph_type=, the icp columns) refuse CPU operands too, and a graph type's
    missing column before any operand is looked at"""
    import torch
    from macvo_b200 import ops
    f64 = lambda *s: torch.zeros(*s, dtype=torch.float64)
    pos, uv, uvc, intr = f64(5, 3), f64(5, 2), f64(5, 3), (1.0,) * 5
    icp = dict(pc_obs=f64(5, 3), obs_cov=f64(5, 3, 3), pts_cov=f64(5, 3, 3))
    for call in (lambda: ops.pgo_accumulate(pos, uv, None, uvc, None, intr, f64(7), graph_type="reproj", cluster=2),
                 lambda: ops.pgo_accumulate(pos, None, None, None, None, intr, f64(7), graph_type="icp", cluster=8, **icp)):
        with pytest.raises(ops.MacvoB200Error, match="expected a CUDA tensor"):
            call()
    with pytest.raises(ops.MacvoB200Error, match="needs pts_cov"):
        ops.pgo_accumulate(pos, None, None, None, None, intr, f64(7), graph_type="icp", **dict(icp, pts_cov=None))


def test_every_public_wrapper_is_checked():
    """a new public function of ops is either host-only or gets a CPU-tensor case above (and a device case in
    tests/test_gpu_ops_args.py)"""
    import inspect
    from macvo_b200 import ops
    public = {n for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith("_")}
    cases = set(_cpu_calls())
    assert not cases & (HOST_ONLY | NEEDS_CUDA_BUFFERS) and not HOST_ONLY & NEEDS_CUDA_BUFFERS
    assert public == cases | HOST_ONLY | NEEDS_CUDA_BUFFERS, "unlisted: " + ", ".join(sorted(public ^ (cases | HOST_ONLY |
                                                                                                     NEEDS_CUDA_BUFFERS)))


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
