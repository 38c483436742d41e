#!/usr/bin/env python
"""vex::make_temp against its written-out twin (the same expression with the temporary's definition at every use).

    python scripts/temp_probe.py [--reps 50] [--rounds 5] > out.json

Cases, float64:
  (a) y = (t1 - t2) * (t1 + t2), t1 = sin(x), t2 = cos(x), N = 1e8 -- the docs' example -- on the interpreter
      (eval.jit = 0) and on the NVRTC kernel (eval.jit = 1)
  (b) y = t * t + t, t = make_inline(A*x), on the 10M-row 2-D Poisson matrix (3162 x 3162, hybrid ELL) and on the
      4M-row irregular matrix (widths U[0, 32), sliced ELL)
  (c) vex::tie(a, b) = std::tie(t, sqrt(1 - t*t)), t = sin(x), N = 1e8, the multi-expression kernel
Each form is timed with CUDA events over `reps` back-to-back calls after warm-up, the two forms alternated `rounds`
times, medians reported; the results of both forms are compared on their bits in the same run.  One JSON object, with
the card's name, power limit and clocks read in the same run."""
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


def wait_jit():
    pending = C.c_int(1)
    while pending.value:
        L.check(L.lib().vexb_jit_pending(C.byref(pending)))
        time.sleep(0.05)


class written_out:
    """Within the block every temporary is lowered as its definition written out at each use."""
    def __enter__(self):
        self.saved = api._Lowering.temp
        api._Lowering.temp = lambda low, n: (low.lower(n.a), low.cvt(n.a.dtype, n.dtype))
    def __exit__(self, *a):
        api._Lowering.temp = self.saved


def compare(ctx, reps, rounds, temp, twin, outs):
    """Warm both forms, check their bits, time them alternately.  outs: the vectors both forms write (read after each)."""
    temp(); temp(); wait_jit(); temp()
    got = [o.read().tobytes() for o in outs]
    twin(); twin(); wait_jit(); twin()
    same = got == [o.read().tobytes() for o in outs]
    ctx.finish()
    l0 = vx.launch_count(); temp(); ctx.finish(); lt = vx.launch_count() - l0
    l0 = vx.launch_count(); twin(); ctx.finish(); lw = vx.launch_count() - l0
    tt, tw = [], []
    for _ in range(rounds):
        tt.append(timed(ctx, temp, reps))
        tw.append(timed(ctx, twin, reps))
    mt, mw = statistics.median(tt), statistics.median(tw)
    return {"bit_identical": same, "launches_temp": lt, "launches_written_out": lw, "temp_ms": mt, "written_out_ms": mw,
            "temp_over_written_out": mt / mw, "temp_ms_all": tt, "written_out_ms_all": tw}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--n", type=int, default=100_000_000)
    a = ap.parse_args()
    ctx = vx.Context([0])
    out = {"reps": a.reps, "rounds": a.rounds, "dtype": "float64"}
    rng = np.random.default_rng(42)

    # (a) the docs' example
    x = vx.vector(ctx, rng.uniform(-1.0, 1.0, a.n))
    y = vx.vector(ctx, a.n)
    t1, t2 = vx.make_temp(1, vx.sin(x)), vx.make_temp(2, vx.cos(x))
    docs = lambda: (t1 - t2) * (t1 + t2)

    def twin_of(fn):
        def run():
            with written_out():
                fn()
        return run
    for name, jit in (("docs_interp", 0), ("docs_nvrtc", 1)):
        vx.set_param("eval.jit", jit)
        try:
            out[name] = compare(ctx, a.reps, a.rounds, lambda: y.assign(docs()), twin_of(lambda: y.assign(docs())), [y])
        finally:
            vx.set_param("eval.jit", 2)

    # (c) vex::tie(a, b) = std::tie(t, sqrt(1 - t*t))
    b = vx.vector(ctx, a.n)
    t = vx.make_temp(1, vx.sin(x))
    tie = lambda: vx.assign_multi([y, b], [t, vx.sqrt(1.0 - t * t)])
    out["tie"] = compare(ctx, a.reps, a.rounds, tie, twin_of(tie), [y, b])
    del x, y, b
    ctx.finish()

    # (b) y = t * t + t, t = make_inline(A*x)
    for name, mat, fmt in (("poisson2d_hell", lambda: gen.poisson_strip(2, 3162), vx.FMT_HELL),
                           ("irregular_sell", lambda: gen.irregular_rows(4_000_000, 0, 32), vx.FMT_SELL)):
        row, col, val = mat()
        N = row.size - 1
        A = vx.SpMat(ctx, N, N, row, col, val, fmt)
        del row, col, val
        xs, ys = vx.vector(ctx, rng.uniform(-1.0, 1.0, N)), vx.vector(ctx, N)
        tp = vx.make_temp(1, vx.make_inline(A * xs))
        prod = lambda: ys.assign(tp * tp + tp)
        out[name] = compare(ctx, a.reps, a.rounds, prod, twin_of(prod), [ys])
        out[name]["rows"] = N
        del A, xs, ys
        ctx.finish()
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
