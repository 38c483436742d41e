"""spmv_ops_impl snippets of three user value types, written with the fixed names sum, v, xv and t, and a numpy restatement
of the third.  Shared by the CPU and GPU tests of vexb_usr_spmv.

  block(T)   : a 2 x 2 block (T4: a00, a01, a10, a11) times a pair (T2), the arithmetic of the reference's custom_values
               test: r = a_r0 x_0 + a_r1 x_1, then sum_r = sum_r + r.  Same bits as vexb_bspmv with B = 2.
  complex(T) : a + bi (T2) times a complex x (T2), the arithmetic of the reference's examples/complex_spmv.cpp:
               s_re = s_re + (a xr - b xi), s_im = s_im + (a xi + b xr).  Same bits as vexb_zspmv.
  triple     : double3 values times double3 x, a made-up product that mixes components:
               s_x = s_x + v_x x_x, s_y = s_y + (v_y x_y - v_x x_z), s_z = s_z + v_z x_z.
"""
import numpy as np

NAMES = {np.float64: "double", np.float32: "float"}


def block(dt):
    T = NAMES[dt]
    return dict(val_type=T + "4", rhs_type=T + "2", rhs_bytes=2 * np.dtype(dt).itemsize,
                decl=f"{T}2 sum = {{0, 0}};",
                product=f"{{ {T} r = v.x * xv.x + v.y * xv.y; sum.x = sum.x + r; r = v.z * xv.x + v.w * xv.y; sum.y = sum.y + r; }}",
                append="t.x = t.x + sum.x; t.y = t.y + sum.y;")


def complex_(dt):
    T = NAMES[dt]
    return dict(val_type=T + "2", rhs_type=T + "2", rhs_bytes=2 * np.dtype(dt).itemsize,
                decl=f"{T}2 sum = {{0, 0}};",
                product="sum.x = sum.x + (v.x * xv.x - v.y * xv.y);\nsum.y = sum.y + (v.x * xv.y + v.y * xv.x);",
                append="t.x = t.x + sum.x; t.y = t.y + sum.y;")


TRIPLE = dict(val_type="double3", rhs_type="double3", rhs_bytes=24,
              decl="double3 sum = make_double3(0, 0, 0);",
              product="sum.x = sum.x + v.x * xv.x;\nsum.y = sum.y + (v.y * xv.y - v.x * xv.z);\nsum.z = sum.z + v.z * xv.z;",
              append="t.x = t.x + sum.x;\nt.y = t.y + sum.y;\nt.z = t.z + sum.z;")


def triple_spmv(ptr, col, val, x, y0=None):
    """The triple product, one rounding per operation and the row's values in storage order.  val: (nnz, 3), x: (m, 3)
    float64; returns (n, 3): the sums, or y0 + sums when y0 is given."""
    ptr = np.asarray(ptr, np.int64)
    col = np.asarray(col, np.int64)
    n = ptr.size - 1
    w = np.diff(ptr)
    s = np.zeros((n, 3), np.float64)
    for k in range(int(w.max()) if n else 0):
        rows = np.nonzero(w > k)[0]
        j = ptr[rows] + k
        v, xv = val[j], x[col[j]]
        s[rows, 0] = s[rows, 0] + v[:, 0] * xv[:, 0]
        s[rows, 1] = s[rows, 1] + (v[:, 1] * xv[:, 1] - v[:, 0] * xv[:, 2])
        s[rows, 2] = s[rows, 2] + v[:, 2] * xv[:, 2]
    return s if y0 is None else y0 + s
