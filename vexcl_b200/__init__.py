"""vexcl_b200 -- Hopper (sm_90a) back end for the VexCL hot paths.

  include/vexb200.h          C ABI (the drop-in boundary)
  include/vexcl/*.hpp        C++ header front end with the reference's spellings
  vexcl_b200/csrc/           CUDA kernels + C ABI implementation -> libvexb200.so
  vexcl_b200/api.py          Python mirror of the front end over the same C ABI (tests, bench)
"""
from . import _lib
from ._lib import (F64, F32, I32, U32, I64, U64, SET, ADD, SUB, MUL, DIV, MOD, AND, OR, XOR, LSH, RSH,
                   SUM, SUM_KAHAN, MAX, MIN, MINMAX, FMT_AUTO, FMT_CSR, FMT_HELL, FMT_PATTERNS, FMT_SELL, FMT_VALUES_F32, VexbError)
from .api import (Context, vector, Reductor, SpMat, SpMatCCSR, BlockMatrix, ComplexMatrix, UserValueMatrix, stencil, partition, ElementIndex, Scalar, if_else,
                  sin, cos, tan, asin, acos, atan, sinh, cosh, tanh, exp, exp2, log, log2, log10, sqrt, rsqrt,
                  cbrt, fabs, floor, ceil, round_, trunc, pow_, atan2, fmod, hypot, fmin, fmax, fma, make_inline, InlineSpMV, assign_multi,
                  UserFunction, push_program_header, pop_program_header, program_header, make_temp, Temp,
                  raw_pointer, deref, ptr, Pointer, Load, sort, sort_by_key,
                  inclusive_scan, exclusive_scan, inclusive_scan_by_key, exclusive_scan_by_key, reduce_by_key)


def set_param(name: str, value: int):
    _lib.check(_lib.lib().vexb_set_param(name.encode(), int(value)))


def launch_count() -> int:
    import ctypes
    n = ctypes.c_uint64()
    _lib.check(_lib.lib().vexb_launch_count(ctypes.byref(n)))
    return n.value
