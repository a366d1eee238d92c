"""Every kernel entry point of libmnn_b200_grid_sample.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; no other library's table holds one of them, and the core library gains none (CPU)."""
import os
import re

from tests.test_gather_kernel_table import GATHER_KERNEL_TESTS
from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels
from tests.test_interp_kernel_table import INTERP_KERNEL_TESTS
from tests.test_rnn_kernel_table import RNN_KERNEL_TESTS
from tests.test_scatter_kernel_table import SCATTER_KERNEL_TESTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_grid_sample_f32.py"
# grid_sample_f32_kernel<3-D, nearest, zeros>: each launched on both sides of the channel-group choice
GRID_SAMPLE_KERNEL_TESTS = {("grid_sample_f32_kernel", (d3, nearest, zeros)): f"{HERE}::test_every_instantiation_both_channel_groupings"
                            for d3 in (0, 1) for nearest in (0, 1) for zeros in (0, 1)}


def test_grid_sample_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.GRID_SAMPLE_LIB)
    assert entries == set(GRID_SAMPLE_KERNEL_TESTS), entries ^ set(GRID_SAMPLE_KERNEL_TESTS)
    for lib in (B.LIB, B.GATHER_LIB, B.INTERP_LIB, B.SCATTER_LIB, B.RNN_LIB):
        assert not set(GRID_SAMPLE_KERNEL_TESTS) & library_kernels(lib)
    assert not set(GRID_SAMPLE_KERNEL_TESTS) & (set(GATHER_KERNEL_TESTS) | set(INTERP_KERNEL_TESTS) | set(SCATTER_KERNEL_TESTS) |
                                                set(RNN_KERNEL_TESTS) | set(KERNEL_TESTS))


def test_grid_sample_kernel_table_names_existing_tests():
    for key, node in GRID_SAMPLE_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"
