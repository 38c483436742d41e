"""Compile-time behaviour of vex::sort and vex::sort_by_key in the C++ front end (include/vexcl/sort.hpp): the four
built-in comparators compile for the six key types, and any other comparator -- a plain functor, one with a
VEX_FUNCTION device part, one over another type -- and tuples of keys stop at a static_assert that names what is
supported.  Syntax checks only: no device, no link."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
MESSAGE = "support only vex::less<K>, vex::less_equal<K>, vex::greater<K> and vex::greater_equal<K>"

PRELUDE = """
#include <vexcl/vexcl.hpp>
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


@pytest.mark.parametrize("T", ["double", "float", "int", "unsigned", "long long", "unsigned long long", "int64_t", "uint64_t"])
def test_built_in_comparators_compile(T):
    body = (f"vex::vector<{T}> k(q, 4); vex::vector<double> v(q, 4); vex::vector<unsigned> u(q, 4); "
            f"vex::sort(k); vex::sort(k, vex::less<{T}>()); vex::sort(k, vex::less_equal<{T}>()); "
            f"vex::sort(k, vex::greater<{T}>()); vex::sort(k, vex::greater_equal<{T}>()); "
            f"vex::sort_by_key(k, v); vex::sort_by_key(k, u, vex::greater_equal<{T}>()); "
            f"static_assert(std::is_base_of<std::less<{T}>, vex::less<{T}>>::value, \"less\"); "
            f"static_assert(std::is_base_of<std::greater_equal<{T}>, vex::greater_equal<{T}>>::value, \"greater_equal\");")
    code, err = _compile(body)
    assert code == 0, err[-3000:]


@pytest.mark.parametrize("body", [
    "vex::vector<int> k(q, 4); struct C { bool operator()(int a, int b) const { return a < b; } }; vex::sort(k, C());",
    "vex::vector<int> k(q, 4); vex::vector<float> v(q, 4); "
    "struct C { typedef bool result_type; VEX_FUNCTION(bool, device, (int, a)(int, b), return a < b;); C() {} }; "
    "vex::sort_by_key(k, v, C());",
    "vex::vector<int> k(q, 4); vex::sort(k, vex::less<long long>());",
    "vex::vector<double> k(q, 4); vex::vector<int> v(q, 4); vex::sort_by_key(k, v, vex::greater<float>());",
    "vex::vector<int> k1(q, 4); vex::vector<float> k2(q, 4); vex::sort(std::tie(k1, k2), vex::less<int>());",
    "vex::vector<int> k(q, 4); vex::vector<float> v1(q, 4), v2(q, 4); vex::sort_by_key(k, std::tie(v1, v2), vex::less<int>());",
])
def test_other_comparators_and_tuples_stop_at_a_static_assert(body):
    code, err = _compile(body)
    assert code != 0
    assert "static assertion failed" in err and MESSAGE in err, err[-3000:]
