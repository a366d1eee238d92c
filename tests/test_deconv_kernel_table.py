"""Every kernel entry point of libmnn_b200_deconv.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; the core library gains no kernel from the Deconvolution (CPU)."""
import os
import re

from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_deconv_f32.py"
# deconv_f32_wgmma_kernel<BN>: the cell matrix plans every tile width
DECONV_KERNEL_TESTS = {
    **{("deconv_f32_wgmma_kernel", (bn,)): f"{HERE}::test_deconv_f32_cell_matrix" for bn in (32, 64, 128)},
    ("pack_deconv_w_f32_kernel", ()): f"{HERE}::test_deconv_f32_matches_float64",
    ("dwdeconv_f32_kernel", ()): f"{HERE}::test_dwdeconv_f32_matches_float64",
}


def test_deconv_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.DECONV_LIB)
    assert entries == set(DECONV_KERNEL_TESTS), entries ^ set(DECONV_KERNEL_TESTS)
    assert not set(DECONV_KERNEL_TESTS) & set(KERNEL_TESTS)
    assert not set(DECONV_KERNEL_TESTS) & library_kernels(B.LIB)


def test_deconv_kernel_table_names_existing_tests():
    for key, node in DECONV_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
