"""Every kernel entry compiled into libmacvo_b200.so is listed in tests/kernel_inventory.py with the test that launches it, and
the table lists nothing the library lacks. A new template instantiation or kernel fails here until a test runs it. CPU only:
cuobjdump and cu++filt read the sm_90a binary without a device."""
import ast
import os

import pytest

from tests import kernel_inventory as inv

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def kernels():
    from macvo_b200 import build
    return inv.binary_kernels(build.build(verbose=False))


def test_every_kernel_in_the_library_is_listed(kernels):
    unlisted = sorted(kernels - set(inv.KERNEL_VARIANTS))
    assert not unlisted, f"kernel entries no test is listed for (add them to KERNEL_VARIANTS with the test that runs them): {unlisted}"


def test_every_listed_kernel_is_in_the_library(kernels):
    stale = sorted(set(inv.KERNEL_VARIANTS) - kernels)
    assert not stale, f"KERNEL_VARIANTS lists kernels the library does not contain: {stale}"


def test_families_hold_listed_variants_only():
    for fam in inv.FAMILIES:
        assert fam <= set(inv.KERNEL_VARIANTS), sorted(fam - set(inv.KERNEL_VARIANTS))
    seen = [v for fam in inv.FAMILIES for v in fam]
    assert len(seen) == len(set(seen)), "a variant belongs to two families"


def test_every_listed_test_exists():
    defined = {}
    for target in set(inv.KERNEL_VARIANTS.values()):
        path, func = target.split("::")
        if path not in defined:
            with open(os.path.join(REPO, path)) as f:
                tree = ast.parse(f.read(), filename=path)
            defined[path] = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
        assert func in defined[path], f"{target} is not a test function"


@pytest.mark.parametrize("raw,want", [
    ("void <unnamed>::decoder_token_kernel<(int)72>(const float *, const float *, float *, long long)", "decoder_token_kernel<72>"),
    ("void (anonymous namespace)::decoder_token_kernel<72>(float const*, float const*, float*, long long)", "decoder_token_kernel<72>"),
    ("void <unnamed>::corr_lookup_kernel<(bool)1>(const float *, float *, int)", "corr_lookup_kernel<true>"),
    ("void (anonymous namespace)::corr_lookup_kernel<false>(float const*, float*, int)", "corr_lookup_kernel<false>"),
    ("void <unnamed>::match_cov_kernel<long>(const T1 *, int, const float *)", "match_cov_kernel<long>"),
    ("<unnamed>::layer_norm64_kernel(const float *, const float *, float *, long long, float)", "layer_norm64_kernel"),
    ("(anonymous namespace)::pgo_lm_kernel((anonymous namespace)::Problem, double*)", "pgo_lm_kernel"),
])
def test_normalise_reads_both_demangler_styles(raw, want):
    """cu++filt (the binary listing) and the C++ ABI demangler (torch.profiler's kernel names) name a variant alike"""
    assert inv.normalise(raw) == want
