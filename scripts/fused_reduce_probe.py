#!/usr/bin/env python
"""Reductions with an inlined sparse product or a user function: the one-kernel path against the temporary it replaces.

    python scripts/fused_reduce_probe.py [--reps 100] [--rounds 5] [--cases classes,csr,function] > out.json

Cases:
  classes   sum(f - A*x) on the 2-D 5-point Poisson matrix on 3162^2 = 9 998 244 rows (configs[2]), in the hybrid-ELL
            strip the library picks for it (row classes: one class byte per row);
  csr       the same matrix with CSR forced;
  function  sum(plus(x, y)) over two double vectors of 1e8 elements, plus a VEX_FUNCTION.
Each case times, with CUDA events over `reps` back-to-back reductions left in device memory (Reductor.device), the fused
request and the explicit temporary (tmp = expr; Reductor(tmp)), alternating the two `rounds` times in one run.  It
prints the median ms of each, the bytes each path moves by count (matrix bytes from info().device_bytes, 8 bytes per
vector element read or written), GB/s by that count, the time ratio, and whether the two results have the same bits.
One JSON object, with the card's name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import vexcl_b200 as vx                                    # noqa: E402
from vexcl_b200 import _lib as L                           # noqa: E402
from vexcl_b200 import gen                                 # noqa: E402
from vexcl_b200.api import DeviceScalar, Event, UserFunction   # noqa: E402

FMT = {vx.FMT_CSR: "csr", vx.FMT_HELL: "hybrid ell", vx.FMT_SELL: "sliced ell", vx.FMT_PATTERNS: "patterns"}


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


def setup(ctx, name):
    """(expression, n, bytes read by the expression, layout)"""
    rng = np.random.default_rng(42)
    if name == "function":
        n = 100_000_000
        x, y = vx.vector(ctx, rng.uniform(-1.0, 1.0, n)), vx.vector(ctx, rng.uniform(-1.0, 1.0, n))
        plus = UserFunction(np.float64, "plus", [(np.float64, "a"), (np.float64, "b")], "return a + b;")
        return (lambda: plus(x, y)), n, 16 * n, {}, (x, y)
    row, col, val = gen.poisson_strip(2, 3162)
    n = row.size - 1
    A = vx.SpMat(ctx, n, n, row, col, val, vx.FMT_CSR if name == "csr" else vx.FMT_AUTO)
    del row, col, val
    x, f = vx.vector(ctx, rng.uniform(-1.0, 1.0, n)), vx.vector(ctx, rng.uniform(-1.0, 1.0, n))
    s = A.info().loc
    lay = {"fmt": FMT.get(int(s.fmt), int(s.fmt)), "ell_width": int(s.ell_width), "ell_classes": int(s.ell_classes),
           "device_bytes": int(s.device_bytes)}
    return (lambda: f - vx.make_inline(A * x)), n, int(s.device_bytes) + 16 * n, lay, (A, x, f)


def case(ctx, name, reps, rounds):
    mk, n, read_bytes, lay, keep = setup(ctx, name)
    red = vx.Reductor(ctx, np.float64, L.SUM)
    out_f, out_t = DeviceScalar(ctx, np.float64), DeviceScalar(ctx, np.float64)
    tmp = vx.vector(ctx, n)
    expr = mk()

    def fused():
        red.device(expr, out_f)

    def temporary():
        tmp.assign(expr)
        red.device(tmp, out_t)

    runs = {"fused": fused, "temporary": temporary}
    for fn in runs.values():                               # warm-up: compilation, module loads, first touches
        fn(); fn()
    ctx.finish()
    l0 = vx.launch_count(); fused(); launches = {"fused": vx.launch_count() - l0}
    l0 = vx.launch_count(); temporary(); launches["temporary"] = vx.launch_count() - l0
    ctx.finish()
    t = {k: [] for k in runs}
    for _ in range(rounds):
        for k, fn in runs.items():
            t[k].append(timed(ctx, fn, reps))
    med = {k: statistics.median(v) for k, v in t.items()}
    moved = {"fused": read_bytes, "temporary": read_bytes + 16 * n}        # + the temporary written and read back
    res = {"case": name, "rows": n, "layout": lay, "launches": launches,
           "bit_identical": bool(np.asarray(out_f.get()).tobytes() == np.asarray(out_t.get()).tobytes())}
    for k in runs:
        res[f"{k}_ms"] = med[k]
        res[f"{k}_ms_all"] = t[k]
        res[f"{k}_bytes_per_row"] = moved[k] / n
        res[f"{k}_GBps"] = moved[k] / med[k] / 1e6
    res["fused_over_temporary_time"] = med["fused"] / med["temporary"]
    del keep
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default="classes,csr,function")
    a = ap.parse_args()
    ctx = vx.Context([0])
    out = {"card": card(), "reps": a.reps, "rounds": a.rounds, "cases": []}
    for c in a.cases.split(","):
        out["cases"].append(case(ctx, c, a.reps, a.rounds))
        print(json.dumps(out["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
