#!/usr/bin/env python
"""Sparse products of user value types (vexb_usr_spmv, the kernel generated from spmv_ops_impl snippets, opaque values
one per slot) against the built-in kernels of the same matrix: a user 2 x 2 block type against vexb_bspmv with B = 2
(bsell_kernel, planar values), and a user complex type against vexb_zspmv (zsell_kernel, planar re / im).

    python scripts/usr_spmv_probe.py [--nx 128] [--reps 200] [--rounds 5] [--cases z,c] > out.json

Matrix: the complex 7-point stencil on nx^3 rows (128^3: 2 097 152 rows, 14 581 760 entries) with seeded random values
(tests/complex_oracle.py complex_stencil), in double (z) and float (c); the block case uses its [[a, -b], [b, a]]
expansion.  The snippets are those of tests/usr_ops.py, which spell the built-in kernels' arithmetic.  Each pair is timed
with CUDA events over `reps` back-to-back launches, alternating `rounds` times.  Per case it prints the median ms per
product of each kernel, GB/s by format bytes (info().device_bytes of the matrix plus x and y), the time ratios, and
whether the user product's y is bit-identical to the built-in one.  One JSON object, with the card's name and power limit
read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import vexcl_b200 as vx                                    # noqa: E402
from vexcl_b200 import _lib as L                           # noqa: E402
from vexcl_b200.api import Event                           # noqa: E402
from complex_oracle import as_blocks, complex_stencil      # noqa: E402
import usr_ops                                             # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:                                  # the timings stand without it
        return {"gpu": None, "error": str(e)}


def timed(ctx, fn, reps):
    e0, e1 = Event(ctx), Event(ctx)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); e1.sync()
    return e0.elapsed_ms(e1) / reps


def user_matrix(ctx, n, ptr, col, val, ops):
    return vx.UserValueMatrix(ctx, n, n, ptr, col, val, ops["val_type"], ops["rhs_type"], ops["rhs_bytes"],
                              ops["decl"], ops["product"], ops["append"])


def pair(ctx, name, user, builtin, user_info, builtin_info, vec_bytes, reps, rounds):
    lib, k = L.lib(), ctx.local[0]
    dev, st = ctx.devs[k], ctx.streams[k]
    U, B, X, Yu, Yb = user, builtin, *vec_bytes[1:]
    kernels = {
        "user": lambda: lib.vexb_usr_spmv(dev, st, U.h, C.byref(U.ops), X.bufs[k], Yu.bufs[k], 0),
        name: (lambda: lib.vexb_bspmv(dev, st, B.h, X.bufs[k], Yb.bufs[k], 1.0, 0)) if name == "block"
              else (lambda: lib.vexb_zspmv(dev, st, B.h, X.bufs[k], Yb.bufs[k], 1.0, 0)),
    }
    for f in kernels.values():                             # warm-up: NVRTC build, module loads, first touches
        L.check(f()); L.check(f())
    ctx.finish()
    t = {kn: [] for kn in kernels}
    for _ in range(rounds):
        for kn, f in kernels.items():
            t[kn].append(timed(ctx, f, reps))
    med = {kn: statistics.median(v) for kn, v in t.items()}
    fmt = {"user": user_info.device_bytes, name: builtin_info.device_bytes}
    out = {}
    for kn in kernels:
        out[f"{kn}_ms"] = med[kn]
        out[f"{kn}_ms_all"] = t[kn]
        out[f"{kn}_bytes"] = fmt[kn] + vec_bytes[0]
        out[f"{kn}_GBps"] = (fmt[kn] + vec_bytes[0]) / med[kn] / 1e6
    out[f"user_over_{name}_time"] = med["user"] / med[name]
    out[f"user_over_{name}_matrix_bytes"] = user_info.device_bytes / builtin_info.device_bytes
    out[f"user_bit_identical_to_{name}"] = bool(Yu.read().tobytes() == Yb.read().tobytes())
    return out


def case(ctx, nx, dtype, reps, rounds):
    cdtype = np.complex128 if dtype == np.float64 else np.complex64
    ptr, col, val = complex_stencil(nx, cdtype, seed=1)
    n = nx ** 3
    es = np.dtype(dtype).itemsize
    x = np.random.default_rng(42).uniform(-1.0, 1.0, 2 * n).astype(dtype)
    X = vx.vector(ctx, x)
    vec_bytes = 2 * (2 * n * es)
    out = {"dtype": np.dtype(dtype).name, "rows": n, "entries": int(ptr[-1])}

    Uz = user_matrix(ctx, n, ptr, col, val.view(dtype).reshape(-1, 2), usr_ops.complex_(dtype))
    Z = vx.ComplexMatrix(ctx, n, n, ptr, col, val)
    Yu, Yz = vx.vector(ctx, 2 * n, dtype), vx.vector(ctx, 2 * n, dtype)
    out["complex"] = pair(ctx, "complex", Uz, Z, Uz.info(), Z.info(), (vec_bytes, X, Yu, Yz), reps, rounds)
    del Uz, Z

    blocks = as_blocks(val)
    Ub = user_matrix(ctx, n, ptr, col, blocks.reshape(-1, 4), usr_ops.block(dtype))
    Bm = vx.BlockMatrix(ctx, n, n, ptr, col, blocks)
    del blocks
    Yu, Yb = vx.vector(ctx, 2 * n, dtype), vx.vector(ctx, 2 * n, dtype)
    out["block"] = pair(ctx, "block", Ub, Bm, Ub.info(), Bm.info(), (vec_bytes, X, Yu, Yb), reps, rounds)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nx", type=int, default=128)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default="z,c")
    a = ap.parse_args()
    ctx = vx.Context([0])
    out = {"card": card(), "nx": a.nx, "reps": a.reps, "rounds": a.rounds, "cases": []}
    for c in a.cases.split(","):
        out["cases"].append(case(ctx, a.nx, np.float64 if c == "z" else np.float32, a.reps, a.rounds))
        print(json.dumps(out["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
