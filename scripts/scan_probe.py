#!/usr/bin/env python
"""vexb_scan and vexb_reduce_by_key_* (one part) next to torch on the same card and data.

    python scripts/scan_probe.py [--sizes 24,27] [--reps 10] [--rounds 3] > out.json

Workloads: n = 2^24 and 2^27 elements of F32, F64 and I64: an inclusive scan against torch.cumsum, an exclusive scan,
and reduce_by_key of sorted I64 keys (runs of about 16) against torch.unique_consecutive(return_counts=True) plus a
segment sum (index_add_ over the inverse).  Each call is timed alone with CUDA events on torch's current stream; ours
get a preallocated workspace.  The two sides alternate `rounds` times, `reps` calls each; medians are reported.
Algorithmic bytes: 3 n s for a scan of s-byte elements (phase 1 reads the input, phase 3 reads it again and writes the
output); for reduce_by_key 2 n (k + s) plus the runs written, k = 8 key bytes.  Shares are of the data sheet's
3.35 TB/s.  Parity: I64 exact against torch, floats within a tolerance (the orders of additions differ).  A
torch.profiler run apart from the timings splits one 2^27 scan and one reduce_by_key per phase.  One JSON object, with
the card's name and power limit read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from vexcl_b200 import _lib as L                           # noqa: E402

PEAK = 3.35e12
VALS = {"F32": (L.F32, torch.float32, 4), "F64": (L.F64, torch.float64, 8), "I64": (L.I64, torch.int64, 8)}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def time_one(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def alternate(ours, theirs, reps, rounds):
    for _ in range(2):
        time_one(ours)
        time_one(theirs)
    t_ours, t_theirs = [], []
    for _ in range(rounds):
        t_ours += [time_one(ours) for _ in range(reps)]
        t_theirs += [time_one(theirs) for _ in range(reps)]
    return statistics.median(t_ours), statistics.median(t_theirs)


def make_vals(name, n, gen):
    dt, tt, s = VALS[name]
    if name == "I64":
        return torch.randint(-(1 << 40), 1 << 40, (n,), dtype=torch.int64, device="cuda", generator=gen)
    return torch.randn(n, dtype=tt, device="cuda", generator=gen)


def close(a, b, name):
    if name == "I64":
        return bool(torch.equal(a, b))
    a, b = a.double(), b.double()
    scale = torch.cumsum(torch.ones_like(a), 0).sqrt().max().item()
    tol = (1e-12 if name == "F64" else 2e-4) * scale * 4
    return bool(((a - b).abs() <= tol * (1 + b.abs())).all().item())


def workspace(n, dt):
    nb = C.c_size_t()
    L.check(L.lib().vexb_scan_workspace_bytes(n, dt, C.byref(nb)))
    return torch.empty(max(nb.value, 1), dtype=torch.uint8, device="cuda"), nb.value


def scan_workload(name, n, exclusive, reps, rounds, gen):
    lib = L.lib()
    dt, tt, s = VALS[name]
    x = make_vals(name, n, gen)
    y = torch.empty_like(x)
    ws, nb = workspace(n, dt)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    dev = torch.cuda.current_device()
    init = torch.zeros(1, dtype=tt).numpy()

    def ours():
        L.check(lib.vexb_scan(dev, stream, x.data_ptr(), y.data_ptr(), dt, n, int(exclusive), init.ctypes.data,
                              ws.data_ptr(), nb))
    out = {}

    def theirs():
        out["r"] = torch.cumsum(x, 0)

    mo, mt = alternate(ours, theirs, reps, rounds)
    ours()
    theirs()
    torch.cuda.synchronize()
    want = out["r"]
    if exclusive:
        want = torch.cat([torch.zeros(1, dtype=tt, device="cuda"), want[:-1]])
    algo = 3 * n * s
    return {"op": "exclusive_scan" if exclusive else "inclusive_scan", "values": name, "n": n,
            "ms_vexb": round(mo, 4), "ms_torch_cumsum": round(mt, 4), "ratio": round(mo / mt, 3),
            "algorithmic_GB": round(algo / 1e9, 3), "GB_per_s": round(algo / mo / 1e6, 1),
            "share_of_3.35TB_s": round(algo / mo / 1e-3 / PEAK, 3), "parity": close(y, want, name)}


def sorted_keys(n, gen):
    return torch.sort(torch.randint(0, max(1, n // 16), (n,), dtype=torch.int64, device="cuda", generator=gen)).values


def rbk_workload(name, n, reps, rounds, gen):
    lib = L.lib()
    dt, tt, s = VALS[name]
    keys, x = sorted_keys(n, gen), make_vals(name, n, gen)
    ws, nb = workspace(n, dt)
    okeys, ovals = torch.empty_like(keys), torch.empty_like(x)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    dev = torch.cuda.current_device()
    runs = C.c_size_t()

    def ours():
        L.check(lib.vexb_reduce_by_key_count(dev, stream, keys.data_ptr(), L.I64, x.data_ptr(), dt, n, ws.data_ptr(), nb,
                                             C.byref(runs)))
        L.check(lib.vexb_reduce_by_key_write(dev, stream, keys.data_ptr(), L.I64, x.data_ptr(), dt, n, okeys.data_ptr(),
                                             ovals.data_ptr(), ws.data_ptr(), nb))
    out = {}

    def theirs():
        u, inv, cnt = torch.unique_consecutive(keys, return_inverse=True, return_counts=True)
        out["r"] = (u, torch.zeros(u.numel(), dtype=tt, device="cuda").index_add_(0, inv, x))

    mo, mt = alternate(ours, theirs, reps, rounds)
    ours()
    theirs()
    torch.cuda.synchronize()
    u, sums = out["r"]
    m = runs.value
    parity = m == u.numel() and bool(torch.equal(okeys[:m], u)) and close(ovals[:m], sums, name)
    algo = 2 * n * (8 + s) + m * (8 + s)
    return {"op": "reduce_by_key", "keys": "I64 sorted, runs of ~16", "values": name, "n": n, "runs": m,
            "ms_vexb": round(mo, 4), "ms_torch_unique_index_add": round(mt, 4), "ratio": round(mo / mt, 3),
            "algorithmic_GB": round(algo / 1e9, 3), "GB_per_s": round(algo / mo / 1e6, 1),
            "share_of_3.35TB_s": round(algo / mo / 1e-3 / PEAK, 3), "parity": parity}


def profile(n, gen):
    """CUDA time per kernel from torch.profiler, over 5 calls each of an F32 inclusive scan and an F64 reduce_by_key."""
    from torch.profiler import ProfilerActivity, profile as prof
    lib = L.lib()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    dev = torch.cuda.current_device()
    res = {}
    x = make_vals("F32", n, gen)
    y = torch.empty_like(x)
    ws, nb = workspace(n, L.F32)
    keys, v = sorted_keys(n, gen), make_vals("F64", n, gen)
    ws2, nb2 = workspace(n, L.F64)
    ok, ov = torch.empty_like(keys), torch.empty_like(v)
    runs = C.c_size_t()
    calls = {
        "inclusive_scan F32": lambda: L.check(lib.vexb_scan(dev, stream, x.data_ptr(), y.data_ptr(), L.F32, n, 0, None,
                                                            ws.data_ptr(), nb)),
        "reduce_by_key I64 keys, F64 values": lambda: (
            L.check(lib.vexb_reduce_by_key_count(dev, stream, keys.data_ptr(), L.I64, v.data_ptr(), L.F64, n,
                                                 ws2.data_ptr(), nb2, C.byref(runs))),
            L.check(lib.vexb_reduce_by_key_write(dev, stream, keys.data_ptr(), L.I64, v.data_ptr(), L.F64, n,
                                                 ok.data_ptr(), ov.data_ptr(), ws2.data_ptr(), nb2))),
    }
    for label, fn in calls.items():
        fn()
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
        per = {}
        for e in p.key_averages():
            if "scan_" in e.key and "_kernel" in e.key:
                k = e.key.split("scan_")[1].split("_kernel")[0]
                per[k] = per.get(k, 0.0) + e.device_time_total / 5 / 1e3
        res[label] = {k: round(t, 4) for k, t in per.items()}
    return {"n": n, "ms_per_call_by_kernel": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="24,27")
    ap.add_argument("--vals", default="F32,F64,I64")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", type=int, default=27, help="log2 n of the profiled calls (0: none)")
    a = ap.parse_args()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    L.check(L.lib().vexb_init())
    res = {"card": card(), "workloads": []}
    for e in (int(s) for s in a.sizes.split(",")):
        for name in a.vals.split(","):
            for w in (lambda: scan_workload(name, 1 << e, False, a.reps, a.rounds, gen),
                      lambda: scan_workload(name, 1 << e, True, a.reps, a.rounds, gen),
                      lambda: rbk_workload(name, 1 << e, a.reps, a.rounds, gen)):
                res["workloads"].append(w())
                print(json.dumps(res["workloads"][-1]), file=sys.stderr, flush=True)
                torch.cuda.empty_cache()
    if a.profile:
        res["profile"] = profile(1 << a.profile, gen)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
