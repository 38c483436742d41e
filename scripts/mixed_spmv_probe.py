#!/usr/bin/env python
"""Double vex::SpMat products from float-stored values (VEXB_FMT_VALUES_F32) against the double strip of the same
rounded values.

    python scripts/mixed_spmv_probe.py [--reps 200] [--rounds 5] [--cases irregular,poisson] > out.json

Matrices:
  irregular  the bench's irregular matrix: 4M rows, widths U[0,32) (vexcl_b200.gen.irregular_rows, seed 1): sliced ELL;
  poisson    the 2-D 5-point Poisson pattern on 3162^2 = 9 998 244 rows (configs[2]) with seeded random coefficients, so
             no two rows share values and no row classes form: hybrid ELL with slot masks.
For each, the float-valued SpMat and the double SpMat built from val.astype(float32).astype(float64) are timed with CUDA
events over `reps` back-to-back y = A*x, alternating `rounds` times.  It prints the median ms per product of each, GB/s
by format bytes (info().device_bytes plus x and y), the time ratio, the layouts, and whether the two y are bit-identical.
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
from vexcl_b200 import gen                                 # noqa: E402
from vexcl_b200.api import Event                           # noqa: E402

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


def matrix(name):
    if name == "irregular":
        return gen.irregular_rows(4_000_000, 0, 32, seed=1)
    row, col, _ = gen.poisson_strip(2, 3162)
    val = np.random.default_rng(7).uniform(0.5, 1.5, col.size)
    return row, col, val


def layout(info):
    s = info.loc
    return {"fmt": FMT.get(int(s.fmt), int(s.fmt)), "ell_width": int(s.ell_width), "ell_col_bytes": int(s.ell_col_bytes),
            "ell_classes": int(s.ell_classes), "csr_tail_nnz": int(s.csr_tail_nnz), "val_bytes": int(s.val_bytes),
            "device_bytes": int(s.device_bytes)}


def case(ctx, name, reps, rounds):
    row, col, val = matrix(name)
    n = row.size - 1
    A = vx.SpMat(ctx, n, n, row, col, val, vx.FMT_AUTO | vx.FMT_VALUES_F32)
    D = vx.SpMat(ctx, n, n, row, col, val.astype(np.float32).astype(np.float64), vx.FMT_AUTO)
    del col
    x = vx.vector(ctx, np.random.default_rng(42).uniform(-1.0, 1.0, n))
    ya, yd = vx.vector(ctx, n), vx.vector(ctx, n)
    runs = {"float_values": lambda: A.apply(x, ya), "double_values": lambda: D.apply(x, yd)}
    for f in runs.values():                                # warm-up: module loads, first touches
        f(); f()
    ctx.finish()
    t = {k: [] for k in runs}
    for _ in range(rounds):
        for k, f in runs.items():
            t[k].append(timed(ctx, f, reps))
    med = {k: statistics.median(v) for k, v in t.items()}
    la, ld = layout(A.info()), layout(D.info())
    vec = 2 * 8 * n
    out = {"matrix": name, "rows": n, "entries": int(row[-1]), "layout_float_values": la, "layout_double_values": ld,
           "same_layout": {k: v for k, v in la.items() if k not in ("val_bytes", "device_bytes")} ==
                          {k: v for k, v in ld.items() if k not in ("val_bytes", "device_bytes")},
           "bit_identical": bool(ya.read().tobytes() == yd.read().tobytes())}
    for k, dev_bytes in (("float_values", la["device_bytes"]), ("double_values", ld["device_bytes"])):
        out[f"{k}_ms"] = med[k]
        out[f"{k}_ms_all"] = t[k]
        out[f"{k}_bytes_per_entry"] = dev_bytes / int(row[-1])
        out[f"{k}_GBps"] = (dev_bytes + vec) / med[k] / 1e6
    out["float_over_double_time"] = med["float_values"] / med["double_values"]
    out["float_over_double_bytes"] = (la["device_bytes"] + vec) / (ld["device_bytes"] + vec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default="irregular,poisson")
    a = ap.parse_args()
    ctx = vx.Context([0])
    out = {"card": card(), "reps": a.reps, "rounds": a.rounds, "cases": []}
    for c in a.cases.split(","):
        out["cases"].append(case(ctx, c, a.reps, a.rounds))
        print(json.dumps(out["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
