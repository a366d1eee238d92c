"""Every kernel entry point of libmnn_b200_gather.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; the core library gains no kernel from the gathers (CPU)."""
import os
import re

from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels
from tests.test_interp_kernel_table import INTERP_KERNEL_TESTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_gather.py"
# gather_slices_kernel<VEC>: the store-path test runs both paths of every slice length
GATHER_KERNEL_TESTS = {
    ("gather_slices_kernel", (0,)): f"{HERE}::test_gather_store_paths",
    ("gather_slices_kernel", (1,)): f"{HERE}::test_gather_store_paths",
    ("gather_elements_kernel", ()): f"{HERE}::test_golden_gathers_bit_exact",
    ("cast_i32_f32_kernel", ()): f"{HERE}::test_casts_bit_exact",
    ("cast_f32_i32_kernel", ()): f"{HERE}::test_casts_bit_exact",
}


def test_gather_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.GATHER_LIB)
    assert entries == set(GATHER_KERNEL_TESTS), entries ^ set(GATHER_KERNEL_TESTS)
    assert not set(GATHER_KERNEL_TESTS) & library_kernels(B.LIB)
    assert not set(GATHER_KERNEL_TESTS) & (set(INTERP_KERNEL_TESTS) | set(KERNEL_TESTS))


def test_gather_kernel_table_names_existing_tests():
    for key, node in GATHER_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
