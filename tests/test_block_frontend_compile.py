"""Compile-time behaviour of block values in the C++ front end (include/vexcl): `Y = A * X`, `Y += A * X` and
`Y -= A * X` compile; every other expression with block vectors or a block product stops at a static_assert that
says what is allowed, not at an incomplete dtype_of.  Syntax checks only: no device, no link."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

PRELUDE = """
#include <vexcl/vexcl.hpp>
#include <vexcl/sparse/matrix.hpp>
#include <vexcl/sparse/distributed.hpp>
typedef std::array<std::array<double, 3>, 3> M3;
typedef std::array<double, 3> V3;
void f(const std::vector<vex::backend::command_queue> &q, const std::vector<int> &ptr, const std::vector<int> &col,
       const std::vector<M3> &val) {
    vex::sparse::matrix<M3> A(q, 4, 4, ptr, col, val);
    vex::sparse::csr<M3> Ac(q, 4, 4, ptr, col, val);
    vex::sparse::ell<M3> Ae(q, 4, 4, ptr, col, val);
    vex::vector<V3> X(q, 4), Y(q, 4);
    vex::vector<double> x(q, 12);
    %s
}
"""


def _compile(body: str):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not found")
    r = subprocess.run([gxx, "-std=c++17", "-fsyntax-only", "-I", str(ROOT / "include"), "-x", "c++", "-"],
                       input=PRELUDE % body, capture_output=True, text=True, timeout=300)
    return r.returncode, r.stderr


def test_block_assignments_compile():
    code, err = _compile("Y = A * X; Y += A * X; Y -= A * X; Y = Ac * X; Y = Ae * X; "
                         "std::vector<V3> h(4); vex::copy(h, Y); vex::copy(Y, h); V3 e = Y[1]; (void)e;")
    assert code == 0, err


@pytest.mark.parametrize("body, message", [
    ("Y = X + X;", "holds block vectors"),
    ("Y = 2 * X;", "holds block vectors"),
    ("Y = A * X + X;", "holds block vectors"),
    ("Y = 2 * (A * X);", "holds block vectors"),
    ("Y *= A * X;", "holds block vectors"),
    ("x = 2 * (A * X);", "only assigned"),
    ("x = A * X;", "only assigned"),
    ("Y = A * (X + X);", "of its own T and B only"),
    ("vex::sparse::distributed<vex::sparse::matrix<M3>> D(q, 4, 4, ptr, col, val);", "does not take block values"),
])
def test_other_uses_stop_at_a_static_assert(body, message):
    code, err = _compile(body)
    assert code != 0
    assert "static assertion failed" in err and message in err, err[-3000:]
    assert "incomplete type" not in err, err[-3000:]
