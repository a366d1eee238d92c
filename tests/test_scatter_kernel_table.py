"""Every kernel entry point of libmnn_b200_scatter.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; no other library's table holds one of them (CPU)."""
import os
import re

from tests.test_gather_kernel_table import GATHER_KERNEL_TESTS
from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels
from tests.test_interp_kernel_table import INTERP_KERNEL_TESTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_scatter.py"
SCATTER_KERNEL_TESTS = {
    ("scatter_init_kernel", (0,)): f"{HERE}::test_copy_paths",
    ("scatter_init_kernel", (1,)): f"{HERE}::test_copy_paths",
    ("scatter_owner_kernel", ()): f"{HERE}::test_golden_scatters_bit_exact",
    ("scatter_copy_kernel", (0,)): f"{HERE}::test_copy_paths",
    ("scatter_copy_kernel", (1,)): f"{HERE}::test_copy_paths",
    ("scatter_keys_kernel", ()): f"{HERE}::test_golden_scatters_bit_exact",
    ("scatter_hist_kernel", ()): f"{HERE}::test_sort_pass_counts",
    ("scatter_scan_kernel", ()): f"{HERE}::test_sort_pass_counts",
    ("scatter_sort_kernel", ()): f"{HERE}::test_sort_pass_counts",
    ("scatter_fold_kernel", (0,)): f"{HERE}::test_golden_scatters_bit_exact",
    ("scatter_fold_kernel", (1,)): f"{HERE}::test_golden_scatters_bit_exact",
    ("scatter_fold_kernel", (2,)): f"{HERE}::test_golden_scatters_bit_exact",
}


def test_scatter_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.SCATTER_LIB)
    assert entries == set(SCATTER_KERNEL_TESTS), entries ^ set(SCATTER_KERNEL_TESTS)
    for lib in (B.LIB, B.GATHER_LIB, B.INTERP_LIB):
        assert not set(SCATTER_KERNEL_TESTS) & library_kernels(lib)
    assert not set(SCATTER_KERNEL_TESTS) & (set(GATHER_KERNEL_TESTS) | set(INTERP_KERNEL_TESTS) | set(KERNEL_TESTS))


def test_scatter_kernel_table_names_existing_tests():
    for key, node in SCATTER_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
