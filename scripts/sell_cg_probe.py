#!/usr/bin/env python
"""The fused product + dot and CGFused on a sliced-ELL matrix, against their compositions.

    python scripts/sell_cg_probe.py [--reps 200] [--rounds 5] [--rows 4000000] > out.json

Matrix: vexcl_b200.gen.irregular_spd (seed 1), symmetric, strictly diagonally dominant, rows of 1 to about 32 entries,
which VEXB_FMT_AUTO stores as sliced ELL.  Timed with CUDA events over `reps` back-to-back calls, alternating the variants
`rounds` times, medians reported:
  apply_dot       SpMat.apply_dot(p, q, pq): dist_apply_kernel with the dot partials + dot_fold_kernel (2 launches)
  apply_reduce    A.apply(p, q) then Reductor.device(p * q, pq), which reads p and q once more
  cg_fused        one CGFused iteration, replayed from its CUDA graphs (4 launches)
  cg_device       one CGDevice iteration, replayed from its CUDA graph
  peer_halo       y = A x on two GPUs with the peer-memory halo (one launch per GPU), against
  copies          the same product with peer_halo=False; only with two devices
The compared results are checked on bits in the same run (y, and the fused dot against nothing: its order differs from
the reduction's, so it is reported with its relative difference).  CG iterations run on from one solve to the next; the
iteration's kernels and bytes do not depend on the values.  One JSON object, with the card's name, power limit and
clocks read in the same run."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import vexcl_b200 as vx                                    # noqa: E402
from vexcl_b200 import _lib as L                           # noqa: E402
from vexcl_b200 import gen                                 # noqa: E402
from vexcl_b200.api import DeviceScalar, Reductor          # noqa: E402
from vexcl_b200.solvers import CGDevice, CGFused           # noqa: E402
from sell_fused_probe import card, timed                   # noqa: E402


def device_count() -> int:
    import torch
    return torch.cuda.device_count()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rows", type=int, default=4_000_000)
    a = ap.parse_args()
    ctx = vx.Context([0])
    row, col, val = gen.irregular_spd(a.rows, seed=1)
    n = row.size - 1
    A = vx.SpMat(ctx, n, n, row, col, val, vx.FMT_AUTO)
    assert A.info().loc.fmt == vx.FMT_SELL, "the probe is about sliced ELL"
    entries = int(row[-1])
    rng = np.random.default_rng(42)
    P = rng.uniform(-1.0, 1.0, n)
    p, q1, q2 = vx.vector(ctx, P), vx.vector(ctx, n), vx.vector(ctx, n)
    d1, d2 = DeviceScalar(ctx), DeviceScalar(ctx)
    red = Reductor(ctx, np.float64, L.SUM)
    b = vx.vector(ctx, rng.uniform(-1.0, 1.0, n))
    xf, xd = vx.vector(ctx, n), vx.vector(ctx, n)
    xf.assign(0.0); xd.assign(0.0)
    cgf, cgd = CGFused(A, b, xf).capture(), CGDevice(A, b, xd).capture()

    def apply_reduce():
        A.apply(p, q2)
        red.device(p * q2, d2)

    runs = {
        "apply_dot": lambda: A.apply_dot(p, q1, d1),
        "apply_reduce": apply_reduce,
        "cg_fused": lambda: cgf.run(1),
        "cg_device": lambda: cgd.run(1),
    }
    out = {"card": card(), "reps": a.reps, "rounds": a.rounds, "rows": n, "entries": entries,
           "strip_bytes": int(A.info().loc.device_bytes), "devices": device_count()}
    launches = {}
    for k, f in runs.items():                              # warm-up: module loads, first touches, graph uploads
        f(); f()
        ctx.finish()
        l0 = vx.launch_count()
        f()
        launches[k] = vx.launch_count() - l0
    ctx.finish()
    out["fused_dot_is_fused"] = bool(A.apply_dot(p, q1, d1))
    out["bit_identical_y"] = q1.read().tobytes() == q2.read().tobytes()
    out["dot_rel_diff"] = abs(d1.get() - d2.get()) / abs(d2.get())

    two = None
    if device_count() >= 2:
        c2, r2 = vx.Context([0, 1], peer_halo=True), vx.Context([0, 1], peer_halo=False)
        B, R = vx.SpMat(c2, n, n, row, col, val), vx.SpMat(r2, n, n, row, col, val)
        out["peer_halo_connected"] = bool(B.peer_halo)
        out["peer_interior_fmt"] = [int(B.info(k).loc.fmt) for k in c2.local]
        xb, yb, xr, yr = vx.vector(c2, P), vx.vector(c2, n), vx.vector(r2, P), vx.vector(r2, n)
        two = {"peer_halo": (c2, lambda: B.apply(xb, yb)), "copies": (r2, lambda: R.apply(xr, yr))}
        for k, (c, f) in two.items():
            f(); f()
            c.finish()
            l0 = vx.launch_count()
            f()
            launches[k] = vx.launch_count() - l0
            c.finish()
        out["bit_identical_two_gpus"] = yb.read().tobytes() == yr.read().tobytes()
    else:
        out["peer_halo"] = "not measured: one device"
    out["launches"] = launches

    t = {k: [] for k in runs}
    if two:
        t.update({k: [] for k in two})
    for _ in range(a.rounds):
        for k, f in runs.items():
            t[k].append(timed(ctx, f, a.reps))
        if two:
            for k, (c, f) in two.items():
                t[k].append(timed(c, f, a.reps))
    med = {k: statistics.median(v) for k, v in t.items()}
    for k in t:
        out[f"{k}_ms"] = med[k]
        out[f"{k}_ms_all"] = t[k]
    out["apply_dot_over_apply_reduce_time"] = med["apply_dot"] / med["apply_reduce"]
    out["cg_fused_over_cg_device_time"] = med["cg_fused"] / med["cg_device"]
    if two:
        out["peer_halo_over_copies_time"] = med["peer_halo"] / med["copies"]
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
