"""Every kernel entry point of libmnn_b200_interp.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; the core library gains no kernel from the Interp (CPU)."""
import os
import re

from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels
from tests.test_deconv_kernel_table import DECONV_KERNEL_TESTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_interp_f32.py"
# interp_f32_kernel<TAPS, VEC>: every case runs both store paths of its resize type
INTERP_KERNEL_TESTS = {("interp_f32_kernel", (taps, vec)): f"{HERE}::test_interp_f32_vector_and_scalar_paths"
                       for taps in (1, 2, 4) for vec in (0, 1)}


def test_interp_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.INTERP_LIB)
    assert entries == set(INTERP_KERNEL_TESTS), entries ^ set(INTERP_KERNEL_TESTS)
    assert not set(INTERP_KERNEL_TESTS) & set(KERNEL_TESTS)
    assert not set(INTERP_KERNEL_TESTS) & set(DECONV_KERNEL_TESTS)
    assert not set(INTERP_KERNEL_TESTS) & library_kernels(B.LIB)


def test_interp_kernel_table_names_existing_tests():
    for key, node in INTERP_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
