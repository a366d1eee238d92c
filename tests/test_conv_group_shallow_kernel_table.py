"""Every kernel entry point of libmnn_b200_shallow.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so, and no other library holds it (CPU)."""
import os
import re

from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHALLOW_KERNEL_TESTS = {("conv_group_shallow_wgmma_kernel", ()): "tests/test_gpu_conv_group_shallow_wg.py::test_every_width_and_k_block"}


def test_shallow_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    assert library_kernels(B.SHALLOW_LIB) == set(SHALLOW_KERNEL_TESTS)
    assert not set(SHALLOW_KERNEL_TESTS) & (library_kernels(B.LIB) | set(KERNEL_TESTS))


def test_shallow_kernel_table_names_existing_tests():
    for key, node in SHALLOW_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
