"""CPU checks of the small-batch solve (one thread block per problem, include/LBFGSSmallBatch.h): the shared-memory budget that
lbfgs_b200_small_max_n reports is the formula documented in include/lbfgs_b200.h, and the C++ front compiles on its own."""
import os
import subprocess

import pytest

import lbfgspp_b200 as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIMIT = 232448   # largest dynamic shared memory of one thread block on sm_90 (227 KB)


def a16(b):
    return (b + 15) // 16 * 16


def documented_bytes(n, m, e, objective):
    """Shared memory of one block as include/lbfgs_b200.h states it."""
    M, N = m + 1, (n + 3) // 4 * 4
    p = (max(6 * m, 8) + 7) // 8 * 8
    stored = objective in (lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG)
    data = objective == lb.OBJ_QUAD_TRIDIAG
    vectors = e * N * (5 + 2 * M + 2 * stored + 2 * data)
    return vectors + 2048 + 8 * 5 * p + a16(e * (2 * M + 4 + 6 * M * M)) + a16(e * (2 * m * m + 6 * m + 2))


def documented_max_n(m, e, objective):
    if documented_bytes(0, m, e, objective) >= LIMIT:
        return 0
    n = 4
    while documented_bytes(n, m, e, objective) <= LIMIT:
        n += 4
    return n - 4


@pytest.mark.parametrize("objective", [lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG])
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_max_n_is_the_documented_formula(objective, dtype):
    lb.build_all()
    e = 8 if dtype == "float64" else 4
    prev = None
    for m in range(1, 65):
        got = lb.small_max_n(m, objective, dtype)
        assert got == documented_max_n(m, e, objective), (m, got)
        assert got % 4 == 0
        if got:
            assert documented_bytes(got, m, e, objective) <= LIMIT < documented_bytes(got + 4, m, e, objective)
        if prev is not None:
            assert got <= prev                      # falls as m grows
        prev = got
    if e == 8:
        assert lb.small_max_n(64, objective, dtype) == 0   # the Gram matrices alone exceed one block's shared memory


def test_max_n_at_the_documented_points():
    # fp64 paired Rosenbrock: 152 bytes per coordinate at m = 6, 216 at m = 10
    assert documented_bytes(1004, 6, 8, 0) - documented_bytes(1000, 6, 8, 0) == 4 * 152
    assert documented_bytes(1004, 10, 8, 0) - documented_bytes(1000, 10, 8, 0) == 4 * 216
    assert lb.small_max_n(6, lb.OBJ_ROSENBROCK_PAIRED) == 1480
    assert lb.small_max_n(10, lb.OBJ_ROSENBROCK_PAIRED) == 1016


def test_max_n_refuses_what_it_cannot_size():
    assert lb.small_max_n(0, lb.OBJ_ROSENBROCK_PAIRED) == 0
    assert lb.small_max_n(65, lb.OBJ_ROSENBROCK_PAIRED) == 0
    assert lb.small_max_n(6, 17) == 0
    assert lb.abi().lbfgs_b200_small_max_n(6, 2, 0) == 0


def test_front_header_compiles_standalone(tmp_path):
    """include/LBFGSSmallBatch.h in a translation unit of its own, -Wall -Werror, with every member instantiated."""
    src = tmp_path / "small_batch_tu.cpp"
    src.write_text("""
#include <LBFGSSmallBatch.h>
template class LBFGSpp::LBFGSSmallBatchSolver<double, LBFGSpp::LineSearchMoreThuente>;
template class LBFGSpp::LBFGSSmallBatchSolver<float, LBFGSpp::LineSearchBacktracking>;
template class LBFGSpp::LBFGSSmallBatchSolver<double>;
int main() { return int(LBFGSpp::LBFGSSmallBatchSolver<double>::max_n(6, LBFGS_B200_OBJ_ROSENBROCK_PAIRED) < 0); }
""")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src),
                    "-o", str(tmp_path / "small_batch_tu.o")], check=True)
