#!/usr/bin/env python
"""A/B of row classes against slot masks for hybrid-ELL strips in one process: spmv.ell_classes = 1 (the default; 2
below the L2-size floor) against spmv.ell_classes = 0.

    python scripts/ell_class_probe.py [--reps 200] [--rounds 5] [--copy-only] > out.json

First times A.apply on configs[2] against a copy y = x of the same two vectors, alternating (key "copy of the same x
and y"): the copy moves the 16 bytes of x and y per row that the product cannot avoid, so it is the product's ceiling.
Then times, with CUDA events over `reps` back-to-back launches and the two encodings alternating `rounds` times:
A.apply on configs[2] (2-D 5-point, 3162^2) and configs[3] (3-D 7-point, 256^3), SpMat * multivector<4> on configs[2],
one fused CG iteration (product + dot, two sweeps; CUDA graphs) on the 256^3 SPD Laplacian, and A.apply on a 2-D
5-point strip of 1000^2 rows, whose 40 MB of values fit the 50 MB L2 (the size floor).  The results of the two
encodings are compared bit for bit.  Prints one JSON object with the medians, the card's name and its power limit."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import vexcl_b200 as vx                                    # noqa: E402
from vexcl_b200 import gen                                 # noqa: E402
from vexcl_b200 import _lib as L                           # noqa: E402
from vexcl_b200.api import Event                           # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:                                  # the timings stand without it
        return {"gpu": None, "error": str(e)}


def timed(ctx, fn, reps):
    fn(); fn(); ctx.finish()
    e0, e1 = Event(ctx), Event(ctx)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); e1.sync()
    return e0.elapsed_ms(e1) / reps


def build_pair(ctx, row, col, val, n, on=1):
    mats = {}
    for cls in (1, 0):
        vx.set_param("spmv.ell_classes", on if cls else 0)
        try:
            A = vx.SpMat(ctx, n, n, row, col, val)
        finally:
            vx.set_param("spmv.ell_classes", 1)
        info = A.info().loc
        assert info.fmt == vx.FMT_HELL and info.ell_col_bytes == 0 and (info.ell_classes > 0) == bool(cls), \
            (cls, info.fmt, info.ell_col_bytes, info.ell_classes)
        mats[cls] = A
    return mats


def ab(ctx, fns, reps, rounds):
    t = {1: [], 0: []}
    for _ in range(rounds):
        for cls in (1, 0):
            t[cls].append(timed(ctx, fns[cls], reps))
    m1, m0 = statistics.median(t[1]), statistics.median(t[0])
    return {"ms_row_classes": m1, "ms_slot_masks": m0, "ratio": m1 / m0, "all_ms_row_classes": t[1], "all_ms_slot_masks": t[0]}


def products(ctx, key, dim, nx, reps, rounds, out, on=1, multi=False):
    row, col, val = gen.poisson_strip(dim, nx)
    n = row.size - 1
    mats = build_pair(ctx, row, col, val, n, on)
    del row, col, val
    x = vx.vector(ctx, n)
    x.assign(vx.ElementIndex() * (1.0 / n) + 0.25)
    ys = {c: vx.vector(ctx, n) for c in (1, 0)}
    res = ab(ctx, {c: (lambda c=c: mats[c].apply(x, ys[c])) for c in (1, 0)}, reps, rounds)
    res["y_bit_identical"] = bool(np.array_equal(ys[1].read(), ys[0].read()))
    res["device_bytes"] = {c: int(mats[c].info().loc.device_bytes) for c in (1, 0)}
    res["rows"], res["ell_width"], res["classes"] = n, int(mats[1].info().loc.ell_width), int(mats[1].info().loc.ell_classes)
    out[key] = res
    if multi:
        xs = [vx.vector(ctx, n) for _ in range(4)]
        for r, v in enumerate(xs):
            v.assign(vx.ElementIndex() * (1.0 / n) + 0.25 * r)
        ym = {c: [vx.vector(ctx, n) for _ in range(4)] for c in (1, 0)}
        res = ab(ctx, {c: (lambda c=c: mats[c].apply_multi(xs, ym[c])) for c in (1, 0)}, reps, rounds)
        res["y_bit_identical"] = all(np.array_equal(ym[1][r].read(), ym[0][r].read()) for r in range(4))
        out[key + " SpMat * multivector<4>"] = res


def copy_ceiling(ctx, reps, rounds, out):
    """A.apply on configs[2] against y = x on the same two vectors, which moves the same x and y bytes: the ceiling of
    a kernel with this 1:1 read/write mix.  The copy runs both as the generated elementwise kernel (y.assign(x)) and
    as cudaMemcpyAsync device to device."""
    row, col, val = gen.poisson_strip(2, 3162)
    n = row.size - 1
    A = vx.SpMat(ctx, n, n, row, col, val)
    del row, col, val
    assert A.info().loc.ell_classes > 0
    x, y = vx.vector(ctx, n), vx.vector(ctx, n)
    x.assign(vx.ElementIndex() * (1.0 / n) + 0.25)
    k = ctx.local[0]
    fns = {"apply": lambda: A.apply(x, y), "copy": lambda: y.assign(x),
           "memcpy": lambda: L.check(L.lib().vexb_d2d(ctx.devs[k], y.bufs[k], x.bufs[k], 8 * n, ctx.streams[k]))}
    t = {f: [] for f in fns}
    for _ in range(rounds):
        for f, fn in fns.items():
            t[f].append(timed(ctx, fn, reps))
    med = {f: statistics.median(v) for f, v in t.items()}
    out["copy of the same x and y"] = {
        "rows": n, "ms_apply": med["apply"], "ms_copy": med["copy"], "ms_memcpy": med["memcpy"],
        "apply_over_copy": med["apply"] / med["copy"], "apply_over_memcpy": med["apply"] / med["memcpy"],
        "copy_TBps": 16 * n / (med["copy"] * 1e-3) / 1e12, "memcpy_TBps": 16 * n / (med["memcpy"] * 1e-3) / 1e12,
        "apply_TBps_of_x_and_y": 16 * n / (med["apply"] * 1e-3) / 1e12,
        "all_ms_apply": t["apply"], "all_ms_copy": t["copy"], "all_ms_memcpy": t["memcpy"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--copy-only", action="store_true", help="time only A.apply on configs[2] against the copy y = x")
    args = ap.parse_args()
    ctx = vx.Context([0])
    out = {"card": card(), "reps": args.reps, "rounds": args.rounds}

    copy_ceiling(ctx, args.reps, args.rounds, out)
    if args.copy_only:
        print(json.dumps(out))
        return

    products(ctx, "configs[2] 2-D 5-pt 3162^2", 2, 3162, args.reps, args.rounds, out, multi=True)
    products(ctx, "configs[3] 3-D 7-pt 256^3", 3, 256, args.reps, args.rounds, out)
    products(ctx, "below the floor: 2-D 5-pt 1000^2 (40 MB of values)", 2, 1000, args.reps, args.rounds, out, on=2)

    from vexcl_b200.solvers import CGFused
    row, col, val = gen.poisson_strip(3, 256, spd=True)
    n = row.size - 1
    mats = build_pair(ctx, row, col, val, n)
    del row, col, val
    cgs = {}
    for c in (1, 0):
        b, x = vx.vector(ctx, n), vx.vector(ctx, n)
        b.assign(((vx.ElementIndex() * 2654435761) % 1000003) * (1.0 / 1000003) - 0.5)
        x.assign(0.0)
        cgs[c] = (CGFused(mats[c], b, x).capture(), b, x)
        assert cgs[c][0].fused_product
    res = ab(ctx, {c: (lambda c=c: cgs[c][0].run(1)) for c in (1, 0)}, args.reps, args.rounds)
    ctx.finish()
    res["x_bit_identical"] = bool(np.array_equal(cgs[1][2].read(), cgs[0][2].read()))
    res["classes"] = int(mats[1].info().loc.ell_classes)
    out["CG iteration 256^3 SPD, fused, CUDA graphs"] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
