"""Compile-time behaviour of the scans and reduce_by_key in the C++ front end (include/vexcl/scan.hpp,
scan_by_key.hpp, reduce_by_key.hpp): every reference spelling with the default operators compiles for the six element
types, and any other operator or comparator -- a plain functor, a VEX_FUNCTION, vex::plus over another type -- and
tuples of keys stop at a static_assert that names what is supported.  Syntax checks only: no device, no link."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
MESSAGE = "support only vex::plus<T> on the values and == on the keys"

PRELUDE = """
#include <vexcl/vexcl.hpp>
#include <vexcl/scan.hpp>
#include <vexcl/scan_by_key.hpp>
#include <vexcl/reduce_by_key.hpp>
#include <tuple>
void f(const std::vector<vex::backend::command_queue> &q) {
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


TYPES = ["double", "float", "int", "unsigned", "long long", "unsigned long long", "int64_t", "uint64_t"]


@pytest.mark.parametrize("T", TYPES)
def test_scan_spellings_compile(T):
    body = (f"vex::vector<{T}> x(q, 4), y(q, 4); const vex::vector<{T}> &cx = x; "
            f"vex::inclusive_scan(x, y); vex::inclusive_scan(cx, x, static_cast<{T}>(1)); vex::inclusive_scan(x, x, static_cast<{T}>(1), vex::plus<{T}>()); "
            f"vex::exclusive_scan(x, y); vex::exclusive_scan(x, x, static_cast<{T}>(2)); vex::exclusive_scan(cx, y, static_cast<{T}>(3), vex::plus<{T}>()); "
            f"static_assert(std::is_base_of<std::plus<{T}>, vex::plus<{T}>>::value, \"plus\");")
    code, err = _compile(body)
    assert code == 0, err[-3000:]


@pytest.mark.parametrize("K", TYPES)
@pytest.mark.parametrize("V", ["double", "float", "int", "unsigned long long"])
def test_by_key_spellings_compile(K, V):
    body = (f"vex::vector<{K}> k(q, 4), ok; vex::vector<{V}> v(q, 4), o(q, 4), ov; const vex::vector<{K}> &ck = k; "
            f"vex::inclusive_scan_by_key(k, v, o); vex::inclusive_scan_by_key(ck, v, v, static_cast<{V}>(1)); "
            f"vex::exclusive_scan_by_key(k, v, o); vex::exclusive_scan_by_key(k, v, v, static_cast<{V}>(2)); "
            f"int n = vex::reduce_by_key(k, v, ok, ov); (void)n; n = vex::reduce_by_key(ck, v, ok, ov);")
    code, err = _compile(body)
    assert code == 0, err[-3000:]


@pytest.mark.parametrize("body", [
    "vex::vector<int> x(q, 4); struct P { int operator()(int a, int b) const { return a + b; } }; vex::inclusive_scan(x, x, 0, P());",
    "vex::vector<double> x(q, 4); vex::exclusive_scan(x, x, 0.0, vex::plus<float>());",
    "vex::vector<double> x(q, 4); VEX_FUNCTION(double, mx, (double, a)(double, b), return a > b ? a : b;); "
    "vex::exclusive_scan(x, x, 0.0, mx);",
    "vex::vector<int> k(q, 4); vex::vector<double> v(q, 4); VEX_FUNCTION(bool, eq, (int, a)(int, b), return a == b;); "
    "VEX_FUNCTION(double, pl, (double, a)(double, b), return a + b;); vex::inclusive_scan_by_key(k, v, v, eq, pl);",
    "vex::vector<int> k(q, 4); vex::vector<double> v(q, 4); VEX_FUNCTION(bool, eq, (int, a)(int, b), return a == b;); "
    "VEX_FUNCTION(double, pl, (double, a)(double, b), return a + b;); vex::exclusive_scan_by_key(k, v, v, eq, pl, 1.0);",
    "vex::vector<int> k(q, 4), ok; vex::vector<double> v(q, 4), ov; VEX_FUNCTION(bool, eq, (int, a)(int, b), return a == b;); "
    "VEX_FUNCTION(double, pl, (double, a)(double, b), return a + b;); vex::reduce_by_key(k, v, ok, ov, eq, pl);",
    "vex::vector<int> k1(q, 4), k2(q, 4); vex::vector<double> v(q, 4); vex::inclusive_scan_by_key(std::tie(k1, k2), v, v);",
    "vex::vector<int> k1(q, 4), k2(q, 4); vex::vector<double> v(q, 4); vex::exclusive_scan_by_key(std::tie(k1, k2), v, v);",
    "vex::vector<int> k1(q, 4), k2(q, 4), o1, o2; vex::vector<double> v(q, 4), ov; "
    "vex::reduce_by_key(std::tie(k1, k2), v, std::tie(o1, o2), ov);",
])
def test_other_operators_and_tuples_stop_at_a_static_assert(body):
    code, err = _compile(body)
    assert code != 0
    assert "static assertion failed" in err and MESSAGE in err, err[-3000:]
