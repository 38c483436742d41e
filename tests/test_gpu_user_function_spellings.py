"""User functions with dependencies and preambles, and program headers, from Python on the GPU (the spellings of the
reference's vexcl/function.hpp:46-225 and backend/common.hpp:120-206).  Every dependency form is compared bit for bit
with one function whose body inlines the same operations: NVRTC compiles both with --fmad=false, so both round op by op
and the bits must be equal.  Reductions and multi-expressions give the bits of the same expression on a temporary, and
each call is one launch per slot."""
import numpy as np
import pytest

import oracle
import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200.api import UserFunction

pytestmark = pytest.mark.gpu

N = 20011
CT = {np.float64: "double", np.float32: "float"}


def _funcs(dtype):
    """The dependency forms and their hand-inlined twins, all in `dtype` (integer literals only, so no promotion)."""
    t, ct = np.dtype(dtype).name, CT[dtype]
    a1, a2 = [(dtype, "x")], [(dtype, "x"), (dtype, "y")]
    f = {}
    f["sq"] = UserFunction(dtype, "sq_" + t, a1, "return x * x;")
    f["lvl2"] = UserFunction(dtype, "lvl2_" + t, a1, f"return sq_{t}(x) + x;", deps=[f["sq"]])
    f["lvl3"] = UserFunction(dtype, "lvl3_" + t, a2, f"return lvl2_{t}(x) * y - sq_{t}(y);", deps=[f["lvl2"], f["sq"]])
    f["lvl3_inl"] = UserFunction(dtype, "lvl3_inl_" + t, a2, f"{ct} s = x * x; {ct} l = s + x; return l * y - y * y;")
    f["twice"] = UserFunction(dtype, "twice_" + t, a1, f"return 2 * sq_{t}(x);", deps=[f["sq"]])
    f["twice_inl"] = UserFunction(dtype, "twice_inl_" + t, a1, "return 2 * (x * x);")
    f["sq_inl"] = UserFunction(dtype, "sq_inl_" + t, a1, "return x * x;")
    f["pre"] = UserFunction(dtype, "pre_" + t, a1, f"return pre_helper_{t}(x) - x;",
                            preamble=f"{ct} pre_helper_{t}({ct} v) {{ return v * v + v; }}\n")
    f["pre_inl"] = UserFunction(dtype, "pre_inl_" + t, a1, f"{ct} h = x * x + x; return h - x;")
    f["hdr"] = UserFunction(dtype, "hdr_" + t, a1, "return x * HDR_K + HDR_C;")
    return f


def _vectors(ctx, dtype, k=2):
    return [vx.vector(ctx, oracle.uniform_real(11 + s, N).astype(dtype)) for s in range(k)]


def _same_bits(a, b):
    assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_dependency_forms_match_their_inlined_twins(ctx, dtype):
    f = _funcs(dtype)
    x, y = _vectors(ctx, dtype)
    z, w = vx.vector(ctx, N, dtype), vx.vector(ctx, N, dtype)
    cases = [
        (f["lvl3"](x, y), f["lvl3_inl"](x, y)),                                    # three levels
        (f["sq"](x) + f["lvl3"](x, y), f["sq_inl"](x) + f["lvl3_inl"](x, y)),      # a dependency also called directly
        (f["twice"](x) - f["lvl2"](y), f["twice_inl"](x) - (f["sq_inl"](y) + y)),  # one dependency shared by two functions
        (f["pre"](x) * y, f["pre_inl"](x) * y),                                    # a preamble
    ]
    for dep, inl in cases:
        z.assign(dep)
        w.assign(inl)
        _same_bits(z.read(), w.read())


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reductions_and_multiexpressions_give_the_bits_of_a_temporary(ctx, dtype):
    f = _funcs(dtype)
    x, y = _vectors(ctx, dtype)
    t, a, b = (vx.vector(ctx, N, dtype) for _ in range(3))
    r = vx.Reductor(ctx, dtype, L.SUM)
    m = vx.Reductor(ctx, dtype, L.MAX)
    t.assign(f["lvl3"](x, y) + f["sq"](x))
    expr = lambda: f["lvl3"](x, y) + f["sq"](x)
    assert r(expr()) == r(t)
    assert m(expr()) == m(t)
    vx.assign_multi([a, b], [f["lvl3"](x, y), f["twice"](y) + x])
    t.assign(f["lvl3"](x, y))
    _same_bits(a.read(), t.read())
    t.assign(f["twice"](y) + x)
    _same_bits(b.read(), t.read())


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_program_headers_push_pop_push(ctx, dtype):
    f = _funcs(dtype)
    (x,) = _vectors(ctx, dtype, 1)
    z, w = vx.vector(ctx, N, dtype), vx.vector(ctx, N, dtype)
    r = vx.Reductor(ctx, dtype, L.SUM)

    def check(k, c):
        inl = UserFunction(dtype, f"hdr_inl_{k}_{c}_{np.dtype(dtype).name}", [(dtype, "x")], f"return x * {k} + {c};")
        z.assign(f["hdr"](x))
        w.assign(inl(x))
        _same_bits(z.read(), w.read())
        assert r(f["hdr"](x)) == r(w)                       # a reduction of a call carries the header too
        a, b = vx.vector(ctx, N, dtype), vx.vector(ctx, N, dtype)
        vx.assign_multi([a, b], [f["hdr"](x), x + 1])       # and so does a multi-expression
        _same_bits(a.read(), w.read())

    vx.push_program_header(ctx, "#define HDR_K 3\n#define HDR_C 1\n")
    try:
        check(3, 1)
        vx.push_program_header(ctx, "#define HDR_K 5\n#define HDR_C 2\n")     # a push replaces the header
        try:
            check(5, 2)
        finally:
            vx.pop_program_header(ctx)
        check(3, 1)                                                         # a pop restores the one before
    finally:
        vx.pop_program_header(ctx)
    vx.push_program_header(ctx, "#define HDR_K 7\n#define HDR_C 4")
    try:
        check(7, 4)
    finally:
        vx.pop_program_header(ctx)
    assert vx.program_header(0) == ""


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_one_launch_per_slot(ctx, dtype):
    f = _funcs(dtype)
    x, y = _vectors(ctx, dtype)
    z = vx.vector(ctx, N, dtype)
    r = vx.Reductor(ctx, dtype, L.SUM)
    for e in (lambda: f["lvl3"](x, y), lambda: f["pre"](x) + f["twice"](y)):
        z.assign(e())                                       # compiled at first use
        ctx.finish()
        n0 = vx.launch_count()
        z.assign(e())
        ctx.finish()
        assert vx.launch_count() - n0 == len(ctx.local)
    r(f["lvl3"](x, y))
    n0 = vx.launch_count()
    r(f["lvl3"](x, y))
    ctx.finish()
    reduce_launches = vx.launch_count() - n0
    r(z)
    n0 = vx.launch_count()
    r(z)
    ctx.finish()
    assert reduce_launches == vx.launch_count() - n0       # as many launches as the reduction of a stored vector
