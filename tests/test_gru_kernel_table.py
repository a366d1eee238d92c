"""Every kernel entry point of libmnn_b200_gru.so is named with the test that launches it, as tests/test_gpu_dispatch.py's
KERNEL_TESTS does for libmnn_b200.so; no other library's table holds one of them, and the plan census reaches every
instantiation of the recurrence (CPU)."""
import os
import re

from tests.test_gather_kernel_table import GATHER_KERNEL_TESTS
from tests.test_gpu_dispatch import KERNEL_TESTS, library_kernels
from tests.test_grid_sample_kernel_table import GRID_SAMPLE_KERNEL_TESTS
from tests.test_interp_kernel_table import INTERP_KERNEL_TESTS
from tests.test_rnn_kernel_table import RNN_KERNEL_TESTS
from tests.test_scatter_kernel_table import SCATTER_KERNEL_TESTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = "tests/test_gpu_gru.py"
# gru_recur_f32_kernel<linear_before_reset, R resident, threads per dot product>: each reached by a launch cell (a streamed
# slice always has more than 32 items per CTA, so <LBR, 0, 8> does not exist); the repack runs in every execute
GRU_KERNEL_TESTS = {("gru_recur_f32_kernel", (lbr, resident, ks)): f"{HERE}::test_every_launch_cell"
                    for lbr in (0, 1) for resident in (0, 1) for ks in (1, 2, 4, 8) if (resident, ks) != (0, 8)}
GRU_KERNEL_TESTS[("gru_repack_f32_kernel", ())] = f"{HERE}::test_every_launch_cell"


def test_gru_kernel_table_matches_library():
    from mnn_b200 import build as B
    B.build()
    entries = library_kernels(B.GRU_LIB)
    assert entries == set(GRU_KERNEL_TESTS), entries ^ set(GRU_KERNEL_TESTS)
    for lib in (B.LIB, B.GATHER_LIB, B.INTERP_LIB, B.SCATTER_LIB, B.RNN_LIB, B.GRID_SAMPLE_LIB):
        assert not set(GRU_KERNEL_TESTS) & library_kernels(lib)
    assert not set(GRU_KERNEL_TESTS) & (set(GATHER_KERNEL_TESTS) | set(INTERP_KERNEL_TESTS) | set(SCATTER_KERNEL_TESTS) |
                                        set(RNN_KERNEL_TESTS) | set(GRID_SAMPLE_KERNEL_TESTS) | set(KERNEL_TESTS))


def test_gru_kernel_table_names_existing_tests():
    for key, node in GRU_KERNEL_TESTS.items():
        path, func = node.split("::")
        with open(os.path.join(ROOT, path)) as f:
            assert re.search(rf"^def {func}\(", f.read(), re.M), f"{key}: {node} does not exist"


def test_every_kernel_is_reached_by_a_launch_cell():
    from oracle import gru_oracle as G
    recur = {k for k in GRU_KERNEL_TESTS if k[0] == "gru_recur_f32_kernel"}
    for sms in (114, 132):
        reached = {("gru_recur_f32_kernel", (k[0], k[2], k[6])) for k in G.census(sms)}
        assert reached == recur, (sms, reached ^ recur)
