"""Compile-time behaviour of complex values in the C++ front end (include/vexcl): `Y = A * X`, `Y += A * X`, `Y -= A * X`,
vex::copy and element reads compile for vex::vector<std::complex<T>>; every other expression with complex vectors or a
complex product, a Reductor of them and vex::sparse::distributed of a complex matrix stop at a static_assert that says
what is allowed, not at an incomplete dtype_of.  Syntax checks only: no device, no link."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

PRELUDE = """
#include <complex>
#include <vexcl/vexcl.hpp>
#include <vexcl/sparse/matrix.hpp>
#include <vexcl/sparse/distributed.hpp>
typedef std::complex<double> Z;
typedef std::complex<float> Zf;
void f(const std::vector<vex::backend::command_queue> &q, const std::vector<int> &ptr, const std::vector<int> &col,
       const std::vector<Z> &val, const std::vector<Zf> &valf) {
    vex::sparse::matrix<Z> A(q, 4, 4, ptr, col, val);
    vex::sparse::csr<Z> Ac(q, 4, 4, ptr, col, val);
    vex::sparse::ell<Z> Ae(q, 4, 4, ptr, col, val);
    vex::sparse::matrix<Zf, long, long> Af(q, 4, 4, ptr, col, valf);
    vex::vector<Z> X(q, 4), Y(q, 4);
    vex::vector<Zf> Xf(q, 4), Yf(q, 4);
    vex::vector<double> x(q, 8);
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


def test_complex_assignments_compile():
    code, err = _compile("Y = A * X; Y += A * X; Y -= A * X; Y = Ac * X; Y = Ae * X; Yf = Af * Xf; Yf -= Af * Xf; "
                         "std::vector<Z> h(4); vex::copy(h, Y); vex::copy(Y, h); Z e = Y[1]; (void)e; "
                         "Y[2] = Z(1, 2); vex::vector<Z> W(q, h); std::cout << W;")
    assert code == 0, err


@pytest.mark.parametrize("body, message", [
    ("Y = X + X;", "holds complex vectors"),
    ("Y = 2 * X;", "holds complex vectors"),
    ("Y = A * X + X;", "holds complex vectors"),
    ("Y = 2 * (A * X);", "holds complex vectors"),
    ("Y *= A * X;", "holds complex vectors"),
    ("x = 2 * (A * X);", "only assigned"),
    ("x = A * X;", "only assigned"),
    ("Y = A * (X + X);", "of its own T only"),
    ("Yf = Af * X;", "of its own T only"),
    ("vex::Reductor<Z, vex::SUM> sum(q); Z s = sum(X); (void)s;", "holds complex vectors"),
    ("vex::Reductor<double, vex::SUM> sum(q); double s = sum(X); (void)s;", "holds complex vectors"),
    ("vex::sparse::distributed<vex::sparse::matrix<Z>> D(q, 4, 4, ptr, col, val);", "does not take complex values"),
])
def test_other_uses_stop_at_a_static_assert(body, message):
    code, err = _compile(body)
    assert code != 0
    assert "static assertion failed" in err and message in err, err[-3000:]
    assert "incomplete type" not in err, err[-3000:]
