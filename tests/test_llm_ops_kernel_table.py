"""Every kernel entry point of libmnn_b200_llm.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; the core library gains no kernel from the LLM ops (CPU)."""
import os
import re

from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_llm_ops.py"
# layernorm_f32_kernel<V, VEC>: V float4 units of a row per thread, VEC the 16-byte path (test_layernorm_against_float64's sweep
# reaches every pair: inner 1024 / 2048 / 4096 / 5504 / 8192 / 16384 / 32768, aligned and 4 bytes off, and inner % 4 != 0)
LLM_KERNEL_TESTS = {
    **{("layernorm_f32_kernel", (v, vec)): f"{HERE}::test_layernorm_against_float64" for v in (1, 2, 4, 8, 16) for vec in (0, 1)},
    ("rope_f32_kernel", ()): f"{HERE}::test_rope_against_restatement",
}


def test_llm_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.LLM_LIB)
    assert entries == set(LLM_KERNEL_TESTS), entries ^ set(LLM_KERNEL_TESTS)
    assert not set(LLM_KERNEL_TESTS) & set(KERNEL_TESTS)
    assert not set(LLM_KERNEL_TESTS) & library_kernels(B.LIB)


def test_llm_kernel_table_names_existing_tests():
    for key, node in LLM_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
