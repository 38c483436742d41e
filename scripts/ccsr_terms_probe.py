#!/usr/bin/env python
"""vex::SpMatCCSR products as expression terminals (VEXB_TERM_CCSR) against their composition: the product into a
temporary by the hand-written CCSR kernel, then the rest of the expression.

    python scripts/ccsr_terms_probe.py [--reps 200] [--rounds 5] [--sizes 128,256] > out.json

Matrices: the 3-D Poisson matrix of the reference's benchmark in CCSR form (vexcl_b200.gen.poisson_ccsr, 2 unique rows,
1-byte idx on the device), float64, x uniform in [-1, 1).  For each expression the fused form (one generated kernel) and
its composition (A.apply into t, then the expression with t) are timed with CUDA events over `reps` back-to-back calls,
alternated `rounds` times, medians reported:
  xax       y = x * (A*x)
  sin       y = sin(A*x)
  energy    s = sum(x * (A*x)), left in device memory (Reductor.device), so no call waits for the host
  product   t = A*x alone, for scale
Bytes per row of each form, by the data it has to move once (idx 1 B, each double 8 B): product 17; xax fused 17,
composed 17 + 24; sin fused 17, composed 17 + 16; energy fused 9, composed 17 + 16.  The results of the two forms are
compared on their bits in the same run.  One JSON object, with the card's name, power limit and clocks read in the same
run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import vexcl_b200 as vx                                    # noqa: E402
from vexcl_b200 import _lib as L, api, gen                 # noqa: E402
from vexcl_b200.api import Event                           # noqa: E402

BYTES = {"product": 17, "xax_fused": 17, "xax_composed": 41, "sin_fused": 17, "sin_composed": 33,
         "energy_fused": 9, "energy_composed": 33}


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


def wait_for_background_kernels():
    """Kernels of new expression shapes are generated on a background thread; the interpreter serves until then."""
    pending = C.c_int(1)
    while pending.value:
        L.check(L.lib().vexb_jit_pending(C.byref(pending)))
        time.sleep(0.05)


def probe(ctx, n, reps, rounds):
    N = n ** 3
    idx, row, col, val = gen.poisson_ccsr(n)
    A = vx.SpMatCCSR(ctx, N, idx, row, col, val)
    del idx
    rng = np.random.default_rng(42)
    x = vx.vector(ctx, rng.uniform(-1.0, 1.0, N))
    t, yf, yc = vx.vector(ctx, N), vx.vector(ctx, N), vx.vector(ctx, N)
    red = vx.Reductor(ctx, np.float64, L.SUM)
    sf, sc = api.DeviceScalar(ctx), api.DeviceScalar(ctx)

    def composed(rest):
        def run():
            A.apply(x, t)
            rest()
        return run

    runs = {
        "product": lambda: A.apply(x, t),
        "xax_fused": lambda: yf.assign(x * (A * x)),
        "xax_composed": composed(lambda: yc.assign(x * t)),
        "sin_fused": lambda: yf.assign(vx.sin(A * x)),
        "sin_composed": composed(lambda: yc.assign(vx.sin(t))),
        "energy_fused": lambda: red.device(x * (A * x), sf),
        "energy_composed": composed(lambda: red.device(x * t, sc)),
    }
    launches, same = {}, {}
    for k, f in runs.items():                              # warm-up: kernel generation, module loads, first touches
        f(); f()
        ctx.finish()
        l0 = vx.launch_count()
        f()
        launches[k] = vx.launch_count() - l0
        if k.endswith("_composed"):                        # bits of the two forms of one expression, same run
            e = k[:-len("_composed")]
            runs[e + "_fused"]()
            ctx.finish()
            same[e] = (np.float64(sf.get()).tobytes() == np.float64(sc.get()).tobytes()) if e == "energy" \
                else yf.read().tobytes() == yc.read().tobytes()
    ctx.finish()
    wait_for_background_kernels()
    for f in runs.values():                                # the composed sweeps now take their generated kernels
        f()
    ctx.finish()
    tm = {k: [] for k in runs}
    for _ in range(rounds):
        for k, f in runs.items():
            tm[k].append(timed(ctx, f, reps))
    med = {k: statistics.median(v) for k, v in tm.items()}
    out = {"n": n, "rows": N, "launches": launches, "bit_identical": same}
    for k in runs:
        out[f"{k}_ms"] = med[k]
        out[f"{k}_ms_all"] = tm[k]
        out[f"{k}_bytes_per_row"] = BYTES[k]
        out[f"{k}_GBps"] = BYTES[k] * N / med[k] / 1e6
    for e in ("xax", "sin", "energy"):
        out[f"{e}_fused_over_composed_time"] = med[e + "_fused"] / med[e + "_composed"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", default="128,256")
    a = ap.parse_args()
    ctx = vx.Context([0])
    res = [probe(ctx, int(s), a.reps, a.rounds) for s in a.sizes.split(",")]
    print(json.dumps({"card": card(), "reps": a.reps, "rounds": a.rounds, "dtype": "float64", "results": res}))


if __name__ == "__main__":
    main()
