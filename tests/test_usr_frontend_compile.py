"""Compile-time behaviour of user value types in the C++ front end (include/vexcl): a type declared with is_cl_native,
type_name_impl, rhs_of and spmv_ops_impl builds vex::sparse::{csr, ell, matrix} and `Y = A * X`, `Y += A * X`, vex::copy
and element reads compile; a missing spmv_ops_impl or type_name_impl, `Y -= A * X`, a scaled product, any other expression
and vex::sparse::distributed stop at a static_assert that says what is missing or allowed.  Syntax checks only: no
device, no link."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

PRELUDE = """
#include <vexcl/vexcl.hpp>
#include <vexcl/sparse/matrix.hpp>
#include <vexcl/sparse/distributed.hpp>
struct blk { double a00, a01, a10, a11; };      // a 2 x 2 block, device double4
struct pair2 { double p, q; };                   // its vector element, device double2
struct zc { double re, im; };                    // a complex number, device double2
struct nops { float f[2]; };                     // declared native, but no spmv_ops_impl
namespace vex {
template <> struct is_cl_native<blk> : std::true_type {};
template <> struct is_cl_native<pair2> : std::true_type {};
template <> struct is_cl_native<zc> : std::true_type {};
template <> struct is_cl_native<nops> : std::true_type {};
template <> struct type_name_impl<blk> { static std::string get() { return "double4"; } };
template <> struct type_name_impl<pair2> { static std::string get() { return "double2"; } };
template <> struct type_name_impl<zc> { static std::string get() { return "double2"; } };
namespace sparse {
template <> struct rhs_of<blk> { typedef pair2 type; };
template <> struct spmv_ops_impl<blk, pair2> {
    static void decl_accum_var(backend::source_generator &src, const std::string &name) {
        src.new_line() << "double2 " << name << " = {0, 0};";
    }
    static void append(backend::source_generator &src, const std::string &sum, const std::string &val) {
        src.new_line() << sum << ".x = " << sum << ".x + " << val << ".x; " << sum << ".y = " << sum << ".y + " << val << ".y;";
    }
    static void append_product(backend::source_generator &src, const std::string &sum, const std::string &m, const std::string &v) {
        src.open("{");
        src.new_line() << "double r0 = " << m << ".x * " << v << ".x + " << m << ".y * " << v << ".y;";
        src.new_line() << "double r1 = " << m << ".z * " << v << ".x + " << m << ".w * " << v << ".y;";
        src.new_line() << sum << ".x = " << sum << ".x + r0; " << sum << ".y = " << sum << ".y + r1;";
        src.close("}");
    }
};
template <> struct spmv_ops_impl<zc, zc> {
    static void decl_accum_var(backend::source_generator &src, const std::string &name) {
        src.new_line() << "double2 " << name << " = {" << 0 << ", " << 0.0 << "};";
    }
    static void append(backend::source_generator &src, const std::string &sum, const std::string &val) {
        src.new_line() << sum << ".x = " << sum << ".x + " << val << ".x; " << sum << ".y = " << sum << ".y + " << val << ".y;";
    }
    static void append_product(backend::source_generator &src, const std::string &sum, const std::string &m, const std::string &v) {
        src.new_line() << sum << ".x = " << sum << ".x + (" << m << ".x * " << v << ".x - " << m << ".y * " << v << ".y);";
        src.new_line() << sum << ".y = " << sum << ".y + (" << m << ".x * " << v << ".y + " << m << ".y * " << v << ".x);";
    }
};
} }
void f(const std::vector<vex::backend::command_queue> &q, const std::vector<int> &ptr, const std::vector<int> &col,
       const std::vector<blk> &val, const std::vector<zc> &zval, const std::vector<nops> &nval) {
    vex::sparse::matrix<blk> A(q, 4, 4, ptr, col, val);
    vex::sparse::csr<blk> Ac(q, 4, 4, ptr, col, val);
    vex::sparse::ell<blk, long, long> Ae(q, 4, 4, ptr, col, val);
    vex::sparse::matrix<zc> Z(q, 4, 4, ptr, col, zval);
    vex::sparse::csr<zc> Zc(q, 4, 4, ptr, col, zval);
    vex::sparse::ell<zc> Ze(q, 4, 4, ptr, col, zval);
    vex::vector<pair2> X(q, 4), Y(q, 4);
    vex::vector<zc> U(q, 4), W(q, 4);
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


def test_user_value_assignments_compile():
    code, err = _compile("Y = A * X; Y += A * X; Y = Ac * X; Y += Ae * X; W = Z * U; W += Zc * U; W = Ze * U; "
                         "std::vector<pair2> h(4); vex::copy(h, Y); vex::copy(Y, h); pair2 e = Y[1]; (void)e; "
                         "Y[2] = pair2{1, 2}; vex::vector<pair2> V(q, h); "
                         "std::vector<zc> hz(4); vex::vector<zc> Uz(q, hz); vex::copy(Uz, hz); zc ez = Uz[0]; (void)ez; "
                         "static_assert(vex::is_user_value<blk>::value && !vex::is_user_value<double>::value, \"trait\"); "
                         "static_assert(std::is_same<decltype(A)::rhs_type, pair2>::value, \"rhs\");")
    assert code == 0, err


def test_built_in_types_keep_their_names():
    code, err = _compile('if (vex::type_name<double>() != "double" || vex::type_name<float>() != "float" || '
                         'vex::type_name<int>() != "int" || vex::type_name<unsigned int>() != "uint" || '
                         'vex::type_name<long>() != "long" || vex::type_name<const double&>() != "double") throw 0; '
                         'vex::backend::source_generator g; g.new_line() << 1 << " " << 0.1; (void)g.str();')
    assert code == 0, err


@pytest.mark.parametrize("body, message", [
    ("vex::sparse::matrix<nops> N(q, 4, 4, ptr, col, nval);", "needs a specialisation of vex::sparse::spmv_ops_impl"),
    ("Y -= A * X;", "is not negated"),
    ("W -= Z * U;", "is not negated"),
    ("Y = 2 * (A * X);", "user value type"),
    ("x = 2 * (A * X);", "only assigned"),
    ("x = A * X;", "only assigned"),
    ("Y = X + X;", "user value type"),
    ("Y *= A * X;", "user value type"),
    ("Y = A * (X + X);", "multiplies a vex::vector<rhs_of<V>::type> only"),
    ("vex::Reductor<double, vex::SUM> sum(q); double s = sum(X); (void)s;", "user value type"),
    ("vex::sparse::distributed<vex::sparse::matrix<blk>> D(q, 4, 4, ptr, col, val);", "does not take user value types"),
    ("vex::sparse::distributed<vex::sparse::matrix<zc>> D(q, 4, 4, ptr, col, zval);", "does not take user value types"),
])
def test_other_uses_stop_at_a_static_assert(body, message):
    code, err = _compile(body)
    assert code != 0
    assert "static assertion failed" in err and message in err, err[-3000:]
    assert "incomplete type" not in err, err[-3000:]


def test_missing_type_name_stops_at_a_static_assert():
    code, err = _compile("std::string s = vex::type_name<nops>(); (void)s;")
    assert code != 0
    assert "static assertion failed" in err and "vex::type_name_impl<T>" in err, err[-3000:]
