"""Every kernel entry point of libmnn_b200_rnn.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; no other library's table holds one of them (CPU)."""
import os
import re

from tests.test_gather_kernel_table import GATHER_KERNEL_TESTS
from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels
from tests.test_interp_kernel_table import INTERP_KERNEL_TESTS
from tests.test_scatter_kernel_table import SCATTER_KERNEL_TESTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_rnn.py"
# rnn_recur_f32_kernel<cell (0 LSTM, 1 RNN), R resident, threads per dot product>: each reached by a launch cell (an RNN
# slice small enough for 8 threads per item always fits in shared memory, so <1, 0, 8> does not exist)
RNN_KERNEL_TESTS = {("rnn_recur_f32_kernel", (cell, resident, ks)): f"{HERE}::test_every_launch_cell"
                    for cell in (0, 1) for resident in (0, 1) for ks in (1, 2, 4, 8) if (cell, resident, ks) != (1, 0, 8)}


def test_rnn_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.RNN_LIB)
    assert entries == set(RNN_KERNEL_TESTS), entries ^ set(RNN_KERNEL_TESTS)
    for lib in (B.LIB, B.GATHER_LIB, B.INTERP_LIB, B.SCATTER_LIB):
        assert not set(RNN_KERNEL_TESTS) & library_kernels(lib)
    assert not set(RNN_KERNEL_TESTS) & (set(GATHER_KERNEL_TESTS) | set(INTERP_KERNEL_TESTS) | set(SCATTER_KERNEL_TESTS) |
                                        set(KERNEL_TESTS))


def test_rnn_kernel_table_names_existing_tests():
    for key, node in RNN_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"


def test_every_kernel_is_reached_by_a_launch_cell():
    from oracle import rnn_oracle as R
    for sms in (114, 132):
        reached = {("rnn_recur_f32_kernel", (k[0], k[2], k[6])) for k in R.census(sms)}
        assert reached == set(RNN_KERNEL_TESTS), (sms, reached ^ set(RNN_KERNEL_TESTS))
