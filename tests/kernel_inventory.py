"""Which kernel variants libmacvo_b200.so holds, which test launches each one, and which variants a call actually launched.

Several launchers pick a template instantiation or a launch shape at run time from the problem size and the device's SM
count, so a suite that checks every kernel at the shapes it happens to use can leave compiled variants that never run.
KERNEL_VARIANTS names, for every kernel entry of the library (as `name<args>`), the test that launches it;
tests/test_kernel_inventory.py holds that table against the binary. FAMILIES groups the instantiations a launcher chooses
between: the test listed for such a variant runs it through `expect_variants`, which proves with torch.profiler that the
variant ran and that no sibling of its family did."""
from __future__ import annotations

import os
import re
import subprocess

NN = "tests/test_gpu_nn_kernels.py::"
KER = "tests/test_gpu_kernels.py::"

KERNEL_VARIANTS = {
    # decoder token path: 64- or 72-pixel tiles, whichever needs fewer pixel slots over all waves
    "decoder_token_kernel<64>": NN + "test_decoder_token_kernel",
    "decoder_token_kernel<72>": NN + "test_decoder_token_kernel",
    # decoder convolutions: output channels per CTA
    "conv_tc_kernel<32>": NN + "test_conv_tc",
    "conv_tc_kernel<64>": NN + "test_conv_tc",
    "conv_tc_kernel<96>": NN + "test_conv_tc_slice_widths",
    "conv_tc_kernel<128>": NN + "test_conv_tc",
    "conv_tc_kernel<160>": NN + "test_conv_tc_slice_widths",
    "conv_tc_kernel<192>": NN + "test_conv_tc",
    "conv_tc_kernel<224>": NN + "test_conv_tc_slice_widths",
    "conv_tc_kernel<256>": NN + "test_conv_tc",
    "flow_im2col_kernel": NN + "test_flow_im2col",
    "pack_rows_kernel": NN + "test_conv_tc",
    # SepConvGRU: stage 0 = the z / r convolution (256 outputs), stage 1 = the q convolution (128 outputs)
    "gru_conv_tc_kernel<0>": NN + "test_sepconv_gru_wgmma",
    "gru_conv_tc_kernel<1>": NN + "test_sepconv_gru_wgmma",
    "pack_motion_kernel": NN + "test_sepconv_gru_wgmma",
    "gru_input_kernel": NN + "test_gru_fused_kernels",
    "gru_gates_kernel": NN + "test_gru_fused_kernels",
    "gru_blend_kernel": NN + "test_gru_fused_kernels",
    "softmax_rows_f16_kernel": NN + "test_softmax_rows_f16",
    "convex_upsample_kernel": NN + "test_convex_upsample",
    # LayerNorm by channel count
    "layer_norm64_kernel": NN + "test_layer_norm",
    "layer_norm_kernel<4>": NN + "test_layer_norm",
    "layer_norm_kernel<8>": NN + "test_layer_norm",
    "layer_norm_kernel<16>": NN + "test_layer_norm",
    # attention by query count, head count, head width and precision mode
    "attn_single_query_kernel<8>": NN + "test_small_attention",
    "attn_single_query_kernel<16>": NN + "test_small_attention",
    "attn_few_queries_kernel<8>": NN + "test_small_attention",
    "attn_few_queries_kernel<16>": NN + "test_small_attention",
    "attn_tc_kernel<16>": NN + "test_small_attention",
    "attn_tc_kernel<32>": NN + "test_small_attention",
    "attn_shared_kv_kernel<16>": NN + "test_small_attention",
    "attn_shared_kv_kernel<32>": NN + "test_small_attention",
    "latent_pool_kernel": NN + "test_latent_pool_equals_cross_attention",
    "patch_conv1_kernel": NN + "test_patch_embed_conv1",
    "patch_conv1_tc_kernel": NN + "test_patch_embed_conv1",
    "pe_pack_weights_kernel": NN + "test_patch_embed_conv1",
    # correlation volume: tensor-core passes (1 = fp16, 2 = tf32, 3 = fp16 hi / lo split) and the operand pre-passes
    "corr_tc_kernel<1>": KER + "test_corr_tensor_core_1xf16_exact_for_fp16_features",
    "corr_tc_kernel<2>": KER + "test_corr_tensor_core_tf32",
    "corr_tc_kernel<3>": KER + "test_corr_tensor_core_3xf16",
    "split_kmajor_kernel": KER + "test_corr_build_channels_last_inputs_bit_identical",
    "split_transpose_kernel": KER + "test_corr_tensor_core_3xf16",
    "corr_simt_kernel": KER + "test_corr_simt_matches_oracle_and_golden",
    # window lookup: (B, 81, H, W) maps or (pixels, 81) rows
    "corr_lookup_kernel<false>": NN + "test_lookup_rows_equals_lookup_map",
    "corr_lookup_kernel<true>": NN + "test_lookup_rows_equals_lookup_map",
    # dense post-processing and keypoint selection; flag_count: 0 = match selector, 1 = mapping points, 2 = depth aware
    "dense_score_kernel": KER + "test_dense_postproc_bit_exact",
    "median_threshold_kernel": KER + "test_selectors_bit_exact",
    "ordered_write_kernel": KER + "test_selectors_bit_exact",
    "gather_pixels_kernel": KER + "test_selectors_bit_exact",
    "flag_count_kernel<0>": KER + "test_selectors_bit_exact",
    "flag_count_kernel<1>": KER + "test_selectors_bit_exact",
    "flag_count_kernel<2>": KER + "test_depth_aware_selector_bit_exact",
    # keypoint gathers by coordinate type
    "retrieve_pixels_kernel<long>": KER + "test_retrieve_pixels",
    "retrieve_pixels_kernel<float>": KER + "test_retrieve_pixels",
    "match_cov_kernel<long>": KER + "test_match_covariance",
    "match_cov_kernel<float>": KER + "test_match_covariance",
    "pgo_lm_kernel": KER + "test_pgo_solve_matches_oracle",
    "pgo_accumulate_kernel": KER + "test_pgo_accumulate_packed",
    "motion_interpolate_kernel": KER + "test_motion_interpolate_kernel",
    "cov_sanity_kernel": KER + "test_cov_sanity_filter_kernel",
    "observe_kernel": "tests/test_observe.py::test_observe_pack_matches_oracle",
    "pack_kernel": "tests/test_observe.py::test_observe_pack_matches_oracle",
    "cov_modify_kernel": "tests/test_ablation_backends.py::test_cov_modify_matches_oracle",
    "mlp_tc_kernel": "tests/test_gpu_mlp_tc.py::test_mlp_tc_accuracy",
    "patch_tokens_tc_kernel": "tests/test_gpu_patch_tokens.py::test_patch_tokens_tc_accuracy",
    "add_rows_relu_kernel": "tests/test_gpu_patch_tokens.py::test_patch_tokens_tc_matches_four_ops_at_frame_shape",
    "posenet_input_kernel": "tests/test_posenet.py::test_gpu_input_builder_matches_reference",
    "posenet_conv_kernel": "tests/test_posenet.py::test_gpu_posenet_conv_matches_float64",
    "posenet_head_kernel": "tests/test_posenet.py::test_gpu_head_matches_shim",
    "pwc_warp_corr_kernel": "tests/test_gpu_tartanvo_matcher.py::test_kernel_matches_float64_oracle",
    "stereo_head_kernel": "tests/test_gpu_tartanvo_depth.py::test_kernel_matches_float64_oracle",
}

FAMILIES = (
    frozenset({"decoder_token_kernel<64>", "decoder_token_kernel<72>"}),
    frozenset(f"conv_tc_kernel<{n}>" for n in range(32, 257, 32)),
    frozenset(f"corr_tc_kernel<{p}>" for p in (1, 2, 3)),
    frozenset({"split_kmajor_kernel", "split_transpose_kernel"}),
    frozenset({"layer_norm64_kernel", "layer_norm_kernel<4>", "layer_norm_kernel<8>", "layer_norm_kernel<16>"}),
    frozenset(f"attn_{k}_kernel<{d}>" for k, ds in (("single_query", (8, 16)), ("few_queries", (8, 16)), ("tc", (16, 32)),
                                                    ("shared_kv", (16, 32))) for d in ds),
    frozenset({"corr_lookup_kernel<false>", "corr_lookup_kernel<true>"}),
    frozenset(f"flag_count_kernel<{m}>" for m in (0, 1, 2)),
    frozenset({"retrieve_pixels_kernel<long>", "retrieve_pixels_kernel<float>"}),
    frozenset({"match_cov_kernel<long>", "match_cov_kernel<float>"}),
    frozenset({"gru_conv_tc_kernel<0>", "gru_conv_tc_kernel<1>"}),
)


def _template_arg(a: str) -> str:
    """`(int)72` (cu++filt) and `72` (the C++ ABI demangler torch.profiler uses) -> `72`; `(bool)0` and `false` -> `false`"""
    a = a.strip()
    m = re.fullmatch(r"\((\w+)\)(-?\d+)", a)
    if not m:
        return a
    return ("false", "true")[int(m.group(2))] if m.group(1) == "bool" else m.group(2)


def normalise(name: str) -> str:
    """a demangled kernel name -> `name<args>`: return type, namespaces and parameter list dropped"""
    s = name.replace("(anonymous namespace)::", "").replace("<unnamed>::", "").strip()
    m = re.match(r"(?:void\s+)?(?:[\w:]+::)?(\w+)(?:<([^<>]*)>)?", s)
    if not m:
        return s
    if m.group(2) is None:
        return m.group(1)
    return m.group(1) + "<" + ",".join(_template_arg(a) for a in m.group(2).split(",")) + ">"


def binary_kernels(lib_path: str) -> set[str]:
    """the kernel entries (`STO_ENTRY` symbols) of a library, demangled by cu++filt and normalised"""
    from macvo_b200 import build
    bin_dir = os.path.dirname(build._nvcc())
    dump = subprocess.run([os.path.join(bin_dir, "cuobjdump"), "-symbols", lib_path], capture_output=True, text=True, check=True)
    mangled = [line.split()[-1] for line in dump.stdout.splitlines() if "STO_ENTRY" in line]
    if not mangled:
        raise AssertionError(f"cuobjdump lists no kernel entry in {lib_path}")
    plain = subprocess.run([os.path.join(bin_dir, "cu++filt")], input="\n".join(mangled) + "\n", capture_output=True, text=True,
                           check=True).stdout.split("\n")
    return {normalise(n) for n in plain if n.strip()}


def family_of(variant: str) -> frozenset:
    for fam in FAMILIES:
        if variant in fam:
            return fam
    return frozenset({variant})


def _profile(fn):
    """fn() under the profiler -> (its result, kernel names), read from the raw activity records. A session of a few
    microseconds of GPU work sometimes delivered no GPU record at all on an H100, so the session is padded by a few
    milliseconds on both sides of the work, and a session with no kernel record runs fn() once more under a new one (every
    probed call is repeatable: same inputs, same outputs). A second empty record fails."""
    import time

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            time.sleep(0.005)
            result = fn()
            torch.cuda.synchronize()
            time.sleep(0.005)
        events = prof.profiler.kineto_results.events()
        names = [normalise(e.name()) for e in events if e.device_type() == DeviceType.CUDA]
        kernels = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
        if kernels:
            return result, kernels
    raise AssertionError("torch.profiler recorded no CUDA kernel in two sessions: the launch probe cannot tell what ran")


def launched(fn) -> list[str]:
    """run fn() under torch.profiler with CUDA activities and return the normalised names of the kernels it launched"""
    return _profile(fn)[1]


def expect_variants(fn, *variants: str):
    """run fn() under the probe; every listed variant must have run and no other member of its family; returns fn()'s result"""
    result, names = _profile(fn)
    ran = set(names)
    for v in variants:
        assert v in KERNEL_VARIANTS, f"{v} is not a kernel of the library"
        assert v in ran, f"expected {v} to run; launched {sorted(ran)}"
        siblings = (family_of(v) - set(variants)) & ran
        assert not siblings, f"expected {v}, but its sibling(s) {sorted(siblings)} ran too"
    return result
