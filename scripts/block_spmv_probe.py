#!/usr/bin/env python
"""Block sparse product (vexb_bspmv) against the scalar product (vexb_spmv, VEXB_FMT_AUTO) of the same matrix expanded
into scalar CSR.

    python scripts/block_spmv_probe.py [--nx 128] [--reps 200] [--rounds 5] [--cases d2,d3,d4,f3] > out.json

Matrix: a 7-point block stencil on nx^3 block rows (128^3: 2 097 152 block rows, 14 581 760 blocks), diagonally dominant
diagonal blocks and seeded random off-diagonal ones (tests/block_oracle.py block_stencil), for B = 2, 3, 4 in double and
B = 3 in float.  The two products are timed with CUDA events over `reps` back-to-back launches, alternating `rounds`
times.  Per case it prints the median ms per product of each kernel, GB/s by format bytes (info().device_bytes of the
matrix plus x and y), the block / scalar time ratio, whether the block y is bit-identical to tests/block_oracle.py, and
the largest ratio of |y_block - y_scalar| to the bound 2 (w + 2) u |A| |x| of its row (the two sum in different orders).
One JSON object, with the card's name and power limit read in the same run."""
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
from block_oracle import bsr_spmv, block_stencil, expand   # noqa: E402


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


def case(ctx, nx, B, dtype, reps, rounds):
    lib, k = L.lib(), ctx.local[0]
    dev, st = ctx.devs[k], ctx.streams[k]
    ptr, col, val = block_stencil(nx, B, dtype, seed=B)
    n = nx ** 3
    es = np.dtype(dtype).itemsize
    rng = np.random.default_rng(42)
    x = rng.uniform(-1.0, 1.0, n * B).astype(dtype)
    X, Yb, Ys = vx.vector(ctx, x), vx.vector(ctx, n * B, dtype), vx.vector(ctx, n * B, dtype)

    A = vx.BlockMatrix(ctx, n, n, ptr, col, val)
    row, ecol, evals = expand(ptr, col, val)
    h = C.c_void_p()
    L.check(lib.vexb_csr_create(dev, st, n * B, n * B, row.ctypes.data, 8, ecol.ctypes.data, 4, evals.ctypes.data,
                                L.F64 if dtype == np.float64 else L.F32, L.FMT_AUTO, C.byref(h)))
    sinfo = L.SpmatInfo()
    L.check(lib.vexb_spmat_get_info(h, C.byref(sinfo)))
    binfo = A.info()

    block = lambda: lib.vexb_bspmv(dev, st, A.h, X.bufs[k], Yb.bufs[k], 1.0, 0)
    scalar = lambda: lib.vexb_spmv(dev, st, h, X.bufs[k], Ys.bufs[k], 1.0, 0)
    for f in (block, scalar):                              # warm-up: module loads, first touches
        L.check(f()); L.check(f())
    ctx.finish()
    tb, ts = [], []
    for _ in range(rounds):
        tb.append(timed(ctx, block, reps))
        ts.append(timed(ctx, scalar, reps))
    mb, ms = statistics.median(tb), statistics.median(ts)

    yb, ys = Yb.read(), Ys.read()
    want = bsr_spmv(ptr, col, val, x)
    absrow = bsr_spmv(ptr, col, np.abs(val.astype(np.float64)), np.abs(x.astype(np.float64)))    # |A| |x| per row
    w = np.diff(row)
    u = np.finfo(dtype).eps / 2
    bound = 2 * (w + 2) * u * absrow
    err = np.abs(yb.astype(np.float64) - ys.astype(np.float64))
    lib.vexb_spmat_destroy(h)
    vec_bytes = 2 * n * B * es
    return {
        "B": B, "dtype": np.dtype(dtype).name, "block_rows": n, "blocks": int(ptr[-1]),
        "scalar_format": {L.FMT_CSR: "csr", L.FMT_HELL: "hell", L.FMT_SELL: "sell", L.FMT_PATTERNS: "patterns"}.get(sinfo.fmt, sinfo.fmt),
        "block_ms": mb, "scalar_ms": ms, "block_over_scalar": mb / ms,
        "block_ms_all": tb, "scalar_ms_all": ts,
        "block_bytes": binfo.device_bytes + vec_bytes, "scalar_bytes": sinfo.device_bytes + vec_bytes,
        "block_GBps": (binfo.device_bytes + vec_bytes) / mb / 1e6, "scalar_GBps": (sinfo.device_bytes + vec_bytes) / ms / 1e6,
        "block_bit_identical_to_oracle": bool(yb.tobytes() == want.tobytes()),
        "max_err_over_bound": float(np.max(err / np.where(bound > 0, bound, 1))),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nx", type=int, default=128)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default="d2,d3,d4,f3")
    a = ap.parse_args()
    ctx = vx.Context([0])
    out = {"card": card(), "nx": a.nx, "reps": a.reps, "rounds": a.rounds, "cases": []}
    for c in a.cases.split(","):
        dtype = np.float64 if c[0] == "d" else np.float32
        out["cases"].append(case(ctx, a.nx, int(c[1:]), dtype, a.reps, a.rounds))
        print(json.dumps(out["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
