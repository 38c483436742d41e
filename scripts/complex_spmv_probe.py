#!/usr/bin/env python
"""Complex sparse product (vexb_zspmv) against the same matrix as 2x2 real blocks [[a, -b], [b, a]] (vexb_bspmv) and as
2n x 2n real CSR (vexb_spmv, VEXB_FMT_AUTO).

    python scripts/complex_spmv_probe.py [--nx 128] [--reps 200] [--rounds 5] [--cases z,c] > out.json

Matrix: a complex 7-point stencil on nx^3 rows (128^3: 2 097 152 rows, 14 581 760 entries) with seeded random values
(tests/complex_oracle.py complex_stencil), in complex<double> (z) and complex<float> (c).  The three products are timed
with CUDA events over `reps` back-to-back launches, alternating `rounds` times.  Per case it prints the median ms per
product of each kernel, GB/s by format bytes (info().device_bytes of the matrix plus x and y), the time ratios, and
whether the complex y is bit-identical to the block product and to tests/complex_oracle.py.  One JSON object, with the
card's name and power limit read in the same run."""
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
from block_oracle import expand                            # noqa: E402
from complex_oracle import as_blocks, complex_stencil, zsr_spmv   # noqa: E402


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


def case(ctx, nx, cdtype, reps, rounds):
    lib, k = L.lib(), ctx.local[0]
    dev, st = ctx.devs[k], ctx.streams[k]
    dtype = np.float64 if cdtype == np.complex128 else np.float32
    ptr, col, val = complex_stencil(nx, cdtype, seed=1)
    n = nx ** 3
    es = np.dtype(dtype).itemsize
    rng = np.random.default_rng(42)
    x = rng.uniform(-1.0, 1.0, 2 * n).astype(dtype)
    X = vx.vector(ctx, x)
    Yz, Yb, Ys = (vx.vector(ctx, 2 * n, dtype) for _ in range(3))

    A = vx.ComplexMatrix(ctx, n, n, ptr, col, val)
    blocks = as_blocks(val)
    Ab = vx.BlockMatrix(ctx, n, n, ptr, col, blocks)
    row, ecol, evals = expand(ptr, col, blocks)
    del blocks
    h = C.c_void_p()
    L.check(lib.vexb_csr_create(dev, st, 2 * n, 2 * n, row.ctypes.data, 8, ecol.ctypes.data, 4, evals.ctypes.data,
                                L.F64 if dtype == np.float64 else L.F32, L.FMT_AUTO, C.byref(h)))
    del row, ecol, evals
    sinfo = L.SpmatInfo()
    L.check(lib.vexb_spmat_get_info(h, C.byref(sinfo)))
    zinfo, binfo = A.info(), Ab.info()

    kernels = {
        "complex": lambda: lib.vexb_zspmv(dev, st, A.h, X.bufs[k], Yz.bufs[k], 1.0, 0),
        "block": lambda: lib.vexb_bspmv(dev, st, Ab.h, X.bufs[k], Yb.bufs[k], 1.0, 0),
        "scalar": lambda: lib.vexb_spmv(dev, st, h, X.bufs[k], Ys.bufs[k], 1.0, 0),
    }
    for f in kernels.values():                             # warm-up: module loads, first touches
        L.check(f()); L.check(f())
    ctx.finish()
    t = {name: [] for name in kernels}
    for _ in range(rounds):
        for name, f in kernels.items():
            t[name].append(timed(ctx, f, reps))
    med = {name: statistics.median(v) for name, v in t.items()}

    yz, yb = Yz.read(), Yb.read()
    want = zsr_spmv(ptr, col, val, x)
    lib.vexb_spmat_destroy(h)
    vec_bytes = 2 * (2 * n * es)
    fmt_bytes = {"complex": zinfo.device_bytes, "block": binfo.device_bytes, "scalar": sinfo.device_bytes}
    out = {"dtype": np.dtype(cdtype).name, "rows": n, "entries": int(ptr[-1]),
           "scalar_format": {L.FMT_CSR: "csr", L.FMT_HELL: "hell", L.FMT_SELL: "sell", L.FMT_PATTERNS: "patterns"}.get(sinfo.fmt, sinfo.fmt)}
    for name in kernels:
        out[f"{name}_ms"] = med[name]
        out[f"{name}_ms_all"] = t[name]
        out[f"{name}_bytes"] = fmt_bytes[name] + vec_bytes
        out[f"{name}_GBps"] = (fmt_bytes[name] + vec_bytes) / med[name] / 1e6
    out["complex_over_block_time"] = med["complex"] / med["block"]
    out["complex_over_scalar_time"] = med["complex"] / med["scalar"]
    out["complex_over_block_matrix_bytes"] = zinfo.device_bytes / binfo.device_bytes
    out["complex_bit_identical_to_block"] = bool(yz.tobytes() == yb.tobytes())
    out["complex_bit_identical_to_oracle"] = bool(yz.tobytes() == want.tobytes())
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
        out["cases"].append(case(ctx, a.nx, np.complex128 if c == "z" else np.complex64, a.reps, a.rounds))
        print(json.dumps(out["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
