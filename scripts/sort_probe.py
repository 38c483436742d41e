#!/usr/bin/env python
"""vexb_sort (vex::sort / vex::sort_by_key on one part) next to torch.sort(stable=True) on the same card and data.

    python scripts/sort_probe.py [--sizes 24,27] [--reps 10] [--rounds 3] > out.json

Workloads: n = 2^24 and 2^27 keys of U32, F32, I64 and F64, (a) keys only and (b) by key with I64 values = arange,
the like-for-like case, since torch.sort returns int64 indices.  Each call is timed alone with CUDA events on torch's
current stream, the input restored by a copy outside the timed window; vexb_sort gets a preallocated workspace.  The two
sorts alternate `rounds` times, `reps` calls each; medians are reported.  Algorithmic bytes are passes x n (3k + 2v) for
key bytes k and value bytes v (the count and scatter reads of the keys, the scatter write; values read and written once
per pass), over the median time, and as a share of the data sheet's 3.35 TB/s.  Parity: our keys equal torch's bitwise
and our values equal torch's indices, on keys without NaN or -0.0.  A torch.profiler run apart from the timings splits
one U32 sort_by_key into its count, scan and scatter kernels.  One JSON object, with the card's name and power limit
read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from vexcl_b200 import _lib as L                           # noqa: E402

PEAK = 3.35e12
KEYS = {"U32": (L.U32, torch.uint32, 4), "F32": (L.F32, torch.float32, 4), "I64": (L.I64, torch.int64, 8),
        "F64": (L.F64, torch.float64, 8)}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return {"gpu": name, "power_limit": power}


def make_keys(name, n, gen):
    dt, tt, kb = KEYS[name]
    if name.startswith("F"):
        return torch.randn(n, dtype=tt, device="cuda", generator=gen)
    hi = 1 << 62 if kb == 8 else 1 << 31
    k = torch.randint(-hi if name == "I64" else 0, hi, (n,), dtype=torch.int64, device="cuda", generator=gen)
    return k.to(torch.uint32) if name == "U32" else k


def time_one(fn, restore):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    restore()
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def workload(name, n, with_vals, reps, rounds, gen):
    lib = L.lib()
    dt, tt, kb = KEYS[name]
    vb = 8 if with_vals else 0
    src = make_keys(name, n, gen)
    keys = src.clone()
    vals = torch.empty(n, dtype=torch.int64, device="cuda") if with_vals else None
    arange = torch.arange(n, dtype=torch.int64, device="cuda")
    vdt = L.I64 if with_vals else -1
    nb = C.c_size_t()
    L.check(lib.vexb_sort_workspace_bytes(n, dt, vdt, C.byref(nb)))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    dev = torch.cuda.current_device()

    def ours():
        L.check(lib.vexb_sort(dev, stream, keys.data_ptr(), dt, vals.data_ptr() if with_vals else None, vdt, n, 0,
                              ws.data_ptr(), nb.value))

    def restore():
        keys.copy_(src)
        if with_vals:
            vals.copy_(arange)

    torch_src = src
    try:
        torch.sort(src[:16], stable=True)
    except RuntimeError:                            # no CUDA sort for this dtype in torch: the same bits as int32
        torch_src = src.view(torch.int32)
    out = {}

    def theirs():
        out["r"] = torch.sort(torch_src, stable=True)

    for _ in range(2):
        time_one(ours, restore)
        time_one(theirs, lambda: None)
    t_ours, t_torch = [], []
    for _ in range(rounds):
        t_ours += [time_one(ours, restore) for _ in range(reps)]
        t_torch += [time_one(theirs, lambda: None) for _ in range(reps)]
    mo, mt = statistics.median(t_ours), statistics.median(t_torch)
    restore()
    ours()
    theirs()
    torch.cuda.synchronize()
    tv, ti = out["r"]
    parity = None
    if torch_src is src:
        parity = bool(torch.equal(keys.view(torch.uint8), tv.contiguous().view(torch.uint8)))
        if with_vals:
            parity = parity and bool(torch.equal(vals, ti))
    else:
        want = torch.from_numpy(np.sort(src.cpu().numpy(), kind="stable")).cuda()
        parity = bool(torch.equal(keys, want))
    passes = kb
    algo = passes * n * (3 * kb + 2 * vb)
    return {"keys": name, "n": n, "values": "I64 arange" if with_vals else None, "ms_vexb_sort": round(mo, 4),
            "ms_torch_sort": round(mt, 4), "ratio": round(mo / mt, 3), "torch_dtype": str(torch_src.dtype),
            "algorithmic_GB": round(algo / 1e9, 3), "GB_per_s": round(algo / mo / 1e6, 1),
            "share_of_3.35TB_s": round(algo / mo / 1e-3 / PEAK, 3), "parity": parity}


def profile(n, gen):
    """Where the time of one vexb_sort goes: CUDA time per kernel, from torch.profiler over 5 calls of U32 keys with I64
    values (run apart from the timings)."""
    from torch.profiler import ProfilerActivity, profile as prof
    lib = L.lib()
    keys, vals = make_keys("U32", n, gen), torch.arange(n, dtype=torch.int64, device="cuda")
    nb = C.c_size_t()
    L.check(lib.vexb_sort_workspace_bytes(n, L.U32, L.I64, C.byref(nb)))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def ours():
        L.check(lib.vexb_sort(torch.cuda.current_device(), stream, keys.data_ptr(), L.U32, vals.data_ptr(), L.I64, n, 0,
                              ws.data_ptr(), nb.value))
    ours()
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(5):
            ours()
        torch.cuda.synchronize()
    per = {}
    for e in p.key_averages():
        if "sort_" in e.key:
            name = e.key.split("sort_")[1].split("_kernel")[0]
            per[name] = per.get(name, 0.0) + e.device_time_total / 5 / 1e3
    return {"keys": "U32", "values": "I64", "n": n, "ms_per_sort_by_kernel": {k: round(v, 3) for k, v in per.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="24,27")
    ap.add_argument("--keys", default="U32,F32,I64,F64")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", type=int, default=27, help="log2 n of the profiled U32 sort_by_key (0: none)")
    a = ap.parse_args()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    L.check(L.lib().vexb_init())
    res = {"card": card(), "workloads": []}
    for e in (int(s) for s in a.sizes.split(",")):
        for name in a.keys.split(","):
            for with_vals in (False, True):
                res["workloads"].append(workload(name, 1 << e, with_vals, a.reps, a.rounds, gen))
                print(json.dumps(res["workloads"][-1]), file=sys.stderr, flush=True)
                torch.cuda.empty_cache()
    if a.profile:
        res["profile"] = profile(1 << a.profile, gen)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
