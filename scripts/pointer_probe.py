#!/usr/bin/env python
"""vex::raw_pointer on the device: what a pointer expression costs next to the kernels it stands in for.

    python scripts/pointer_probe.py [--n 100000000] [--reps 20] [--rounds 5] > out.json

Cases, float64:
  (a) the manual stencil y = 2*p[i] - p[left] - p[right] (clamped ends) at N = 1e8, on the interpreter (eval.jit = 0)
      and on the NVRTC kernel (eval.jit = 1), against the 3-point vex::stencil {-1, 2, -1} and the copy y = x;
      the stencil's result is compared with the pointer expression's (same bits: the same three products, added in
      the same order, with clamped ends)
  (b) the N-body user function of the reference (a loop over all n elements per element) at n = 16384 and 65536
Each form is timed with CUDA events over `reps` back-to-back calls after warm-up, the forms alternated `rounds` times,
medians reported.  One JSON object, with the card's name, power limit and clocks read in the same run."""
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


def alternate(ctx, forms, reps, rounds):
    """forms: {name: (fn, params)}; every form warmed, then timed in turn `rounds` times.  Median ms per call."""
    def under(prm, fn):
        for k, v in prm.items():
            vx.set_param(k, v)
        try:
            return fn()
        finally:
            vx.set_param("eval.jit", 2)
    for name, (fn, prm) in forms.items():
        under(prm, lambda: (fn(), fn(), fn()))
    ctx.finish()
    times = {name: [] for name in forms}
    for _ in range(rounds):
        for name, (fn, prm) in forms.items():
            times[name].append(under(prm, lambda: timed(ctx, fn, reps)))
    return {name: statistics.median(t) for name, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--nbody", type=int, nargs="*", default=[16384, 65536])
    a = ap.parse_args()
    ctx = vx.Context([0])
    out = {"card": card(), "n": a.n}

    n = a.n
    X = np.random.default_rng(1).random(n)
    x, y, z, w = vx.vector(ctx, X), vx.vector(ctx, n), vx.vector(ctx, n), vx.vector(ctx, n)
    p, i = vx.raw_pointer(x), vx.ElementIndex()
    left, right = vx.if_else(i > 0, i - 1, i), vx.if_else(i + 1 < n, i + 1, i)
    S = vx.stencil(ctx, [-1.0, 2.0, -1.0], 1)
    manual = lambda: y.assign(2.0 * p[i] - p[left] - p[right])
    forms = {
        "pointer_interp": (manual, {"eval.jit": 0}),
        "pointer_jit": (manual, {"eval.jit": 1}),
        "stencil": (lambda: z.assign(x * S), {}),
        "copy": (lambda: w.assign(x), {}),
    }
    ms = alternate(ctx, forms, a.reps, a.rounds)
    moved = 2 * 8 * n                                       # one read of x, one write of y: what every form must move
    out["stencil_1d"] = {k: {"ms": v, "GBps_min_traffic": moved / v / 1e6} for k, v in ms.items()}
    Y, Z = y.read(), z.read()
    out["stencil_1d"]["pointer_equals_stencil_bits"] = bool(np.array_equal(Y.view(np.uint64), Z.view(np.uint64)))
    out["stencil_1d"]["pointer_max_abs_diff_vs_stencil"] = float(np.max(np.abs(Y - Z)))
    del x, y, z, w

    nbody = vx.UserFunction(np.float64, "nbody", [(np.uint64, "n"), (np.uint64, "j"), (vx.ptr(np.float64), "x")],
                            "double sum = 0; for (size_t i = 0; i < n; ++i) if (i != j) sum += x[i]; return sum;")
    out["nbody"] = {}
    for m in a.nbody:
        Xm = np.random.default_rng(m).random(m)
        xm, ym = vx.vector(ctx, Xm), vx.vector(ctx, m)
        q = vx.raw_pointer(xm)
        ms = alternate(ctx, {"nbody": (lambda: ym.assign(nbody(np.uint64(m), vx.ElementIndex(), q)), {})}, max(2, a.reps // 4), a.rounds)
        got = ym.read()
        ref = Xm.sum() - Xm                                 # closeness only: the body adds in its own order
        out["nbody"][str(m)] = {"ms": ms["nbody"], "Gpairs_per_s": m * m / ms["nbody"] / 1e6,
                                "max_rel_diff_vs_numpy": float(np.max(np.abs(got - ref) / np.abs(ref)))}
    out["card_after"] = card()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
