#!/usr/bin/env python
"""Sliced ELL beyond the plain product: four right-hand sides in one pass over the strip, and the product inlined into an
assignment kernel.

    python scripts/sell_fused_probe.py [--reps 200] [--rounds 5] [--rows 4000000] > out.json

Matrix: the bench's irregular matrix, 4M rows of U[0,32) entries (vexcl_b200.gen.irregular_rows, seed 1), which
VEXB_FMT_AUTO stores as sliced ELL.  Timed with CUDA events over `reps` back-to-back calls, alternating the variants
`rounds` times, medians reported:
  multi4        SpMat.apply_multi on 4 vectors (sell_multi_kernel, one launch)
  four_products the same four products one by one ("spmv.no_multi" = 1)
  one_product   y = A*x
  inline        y = z + A*x as one generated kernel sweeping in the strip's storage order
  composed      the same with "spmv.sell_inline" = 0: y = z, then y += A*x
GB/s by format bytes: the strip (info().device_bytes) plus the vectors each variant has to move once.  The results of the
variants that compute the same thing are compared on bits in the same run.  One JSON object, with the card's name, power
limit and clocks read in the same run."""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, cmax, csm, cmem = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": cmax, "sm_clock_after_run": csm, "mem_clock_after_run": cmem}
    except Exception as e:                                  # the timings stand without it
        return {"gpu": None, "error": str(e)}


def timed(ctx, fn, reps):
    e0, e1 = Event(ctx), Event(ctx)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); e1.sync()
    return e0.elapsed_ms(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rows", type=int, default=4_000_000)
    a = ap.parse_args()
    ctx = vx.Context([0])
    row, col, val = gen.irregular_rows(a.rows, 0, 32, seed=1)
    n = row.size - 1
    A = vx.SpMat(ctx, n, n, row, col, val, vx.FMT_AUTO)
    assert A.info().loc.fmt == vx.FMT_SELL, "the probe is about sliced ELL"
    entries, strip = int(row[-1]), int(A.info().loc.device_bytes)
    del col, val
    rng = np.random.default_rng(42)
    xs = [vx.vector(ctx, rng.uniform(-1.0, 1.0, n)) for _ in range(4)]
    ym, y4 = [vx.vector(ctx, n) for _ in range(4)], [vx.vector(ctx, n) for _ in range(4)]
    z, yi, yc, y1 = vx.vector(ctx, rng.uniform(-1.0, 1.0, n)), vx.vector(ctx, n), vx.vector(ctx, n), vx.vector(ctx, n)

    def with_param(name, value, fn):
        def run():
            vx.set_param(name, value)
            fn()
            vx.set_param(name, 1 - value)
        return run

    runs = {
        "multi4": lambda: A.apply_multi(xs, ym),
        "four_products": with_param("spmv.no_multi", 1, lambda: A.apply_multi(xs, y4)),
        "one_product": lambda: A.apply(xs[0], y1),
        "inline": lambda: yi.assign(z + A * xs[0]),
        "composed": with_param("spmv.sell_inline", 0, lambda: yc.assign(z + A * xs[0])),
    }
    launches = {}
    for k, f in runs.items():                              # warm-up: kernel generation, module loads, first touches
        f(); f()
        ctx.finish()
        l0 = vx.launch_count()
        f()
        launches[k] = vx.launch_count() - l0
    ctx.finish()
    t = {k: [] for k in runs}
    for _ in range(a.rounds):
        for k, f in runs.items():
            t[k].append(timed(ctx, f, a.reps))
    med = {k: statistics.median(v) for k, v in t.items()}
    vec = 8 * n
    moved = {"multi4": strip + 8 * vec, "four_products": 4 * (strip + 2 * vec), "one_product": strip + 2 * vec,
             "inline": strip + 3 * vec, "composed": strip + 5 * vec}          # composed: z -> y, then y read and written again
    out = {"card": card(), "reps": a.reps, "rounds": a.rounds, "rows": n, "entries": entries, "strip_bytes": strip,
           "launches": launches,
           "bit_identical_multi": all(a_.read().tobytes() == b_.read().tobytes() for a_, b_ in zip(ym, y4)),
           "bit_identical_inline": yi.read().tobytes() == yc.read().tobytes()}
    for k in runs:
        out[f"{k}_ms"] = med[k]
        out[f"{k}_ms_all"] = t[k]
        out[f"{k}_GBps"] = moved[k] / med[k] / 1e6
    out["multi4_over_four_products_time"] = med["multi4"] / med["four_products"]
    out["multi4_over_one_product_time"] = med["multi4"] / med["one_product"]
    out["inline_over_composed_time"] = med["inline"] / med["composed"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
