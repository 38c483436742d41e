"""Conjugate gradient built from the three hot paths (BASELINE.json configs[4]: "CG step = SpMV + 2 axpy + 2 dot").

The reference has no in-tree solver; its ViennaCL shim composes CG from exactly these pieces
(vexcl/external/viennacl.hpp:36-64: inner_prod -> Reductor, prod -> SpMat, vector expressions).

  cg_host_scalars   the reference-equivalent composition: every dot product returns to the host
                    (two synchronising reductions per iteration), alpha / beta are host scalars.
  CGDevice          same arithmetic, but dot products stay on the device (Reductor.device), alpha and
                    beta are DeviceScalars, so an iteration is 7 asynchronous launches (+ halo) and can
                    be replayed as one CUDA graph.
"""
from __future__ import annotations

import numpy as np

from . import _lib as L
from .api import Context, DeviceScalar, Graph, Reductor, SpMat, vector


def cg_host_scalars(A: SpMat, b: vector, x: vector, iters: int):
    """x is the start vector (updated in place).  Returns the list of rho = r.r after each iteration."""
    ctx = A.ctx
    dot = Reductor(ctx, np.float64, L.SUM)
    r, p, q = vector(ctx, b.n), vector(ctx, b.n), vector(ctx, b.n)
    r.assign(b - A * x)
    p.assign(r)
    rho = dot(r * r)
    hist = []
    for _ in range(iters):
        q.assign(A * p)                       # SpMV
        alpha = rho / dot(p * q)              # dot 1 (host round trip)
        x += alpha * p                        # axpy 1
        r -= alpha * q                        # axpy 2
        rho_new = dot(r * r)                  # dot 2 (host round trip)
        p.assign(r + (rho_new / rho) * p)
        rho = rho_new
        hist.append(float(rho))
    return hist


class CGDevice:
    """CG with device-resident scalars.  step() issues one iteration asynchronously; capture() turns it into a
    CUDA graph (one launch per iteration)."""

    def __init__(self, A: SpMat, b: vector, x: vector):
        ctx = self.ctx = A.ctx
        self.A, self.x = A, x
        self.dot = Reductor(ctx, np.float64, L.SUM)
        self.r, self.p, self.q = vector(ctx, b.n), vector(ctx, b.n), vector(ctx, b.n)
        self.rho, self.rho_new, self.pq, self.alpha, self.beta = (DeviceScalar(ctx) for _ in range(5))
        self.r.assign(b - A * x)
        self.p.assign(self.r)
        self.dot.device(self.r * self.r, self.rho)
        self.graph = None

    def step(self):
        A, x, r, p, q = self.A, self.x, self.r, self.p, self.q
        q.assign(A * p)                                   # SpMV (halo overlapped)
        self.dot.device(p * q, self.pq)                   # dot 1, result stays on the device (+ ncclAllReduce)
        self.alpha.assign(self.rho / self.pq)
        x += self.alpha * p                               # axpy 1
        r -= self.alpha * q                               # axpy 2
        self.dot.device(r * r, self.rho_new)              # dot 2
        self.beta.assign(self.rho_new / self.rho)
        p.assign(r + self.beta * p)
        self.rho.assign(self.rho_new)

    def capture(self):
        self.step()                                       # warm up (allocations, lazy init) outside the capture
        self.ctx.finish()
        self.graph = Graph(self.ctx, self.step)
        return self

    def run(self, iters: int):
        for _ in range(iters):
            if self.graph is not None:
                self.graph.launch()
            else:
                self.step()

    def residual2(self) -> float:
        return float(self.rho.get())


class CGFused:
    """The same iteration in four launches per GPU (BASELINE configs[4], "fused CG step"):

        q = A p  and  (p, q)                                   SpMat.apply_dot: the product kernel (halo pushed over NVLink peer
                                                               memory) leaves per-block partials of (p, q); a one-block kernel
                                                               folds them and combines across the GPUs
        alpha = rho/(p,q); r -= alpha q; rho' = (r, r)         one sweep (vexb_cg_update_r), combine in the kernel
        beta = rho'/rho; x += alpha p; p = r + beta p          one sweep (vexb_cg_update_xp)

    against 7 vector kernels + 3 scalar kernels (+ pack, NCCL, boundary kernels) for CGDevice: 64 instead of 96 bytes
    of vector traffic per row and iteration besides the product.  rho and rho' swap roles every iteration (no copy),
    so two CUDA graphs (even / odd) replay the solver.  Per-element arithmetic is the unfused composition's.
    The product step is fused on matrices whose interior strips are hybrid ELL or sliced ELL (VEXB_FMT_AUTO's choice for
    uneven rows); on CSR or float-valued strips, and on several slots without a peer group, apply_dot composes the
    product and a reduction (fused_product is then False)."""

    def __init__(self, A: SpMat, b: vector, x: vector):
        ctx = self.ctx = A.ctx
        self.A, self.x = A, x
        self.r, self.p, self.q = vector(ctx, b.n), vector(ctx, b.n), vector(ctx, b.n)
        self.rho2 = [DeviceScalar(ctx), DeviceScalar(ctx)]
        self.pq = DeviceScalar(ctx)
        self.r.assign(b - A * x)
        self.p.assign(self.r)
        Reductor(ctx, np.float64, L.SUM).device(self.r * self.r, self.rho2[0])
        self.it = 0
        self.graphs = None
        self.fused_product = None

    def step(self):
        import ctypes as C
        lib, ctx = L.lib(), self.ctx
        A, x, r, p, q = self.A, self.x, self.r, self.p, self.q
        rho, rho_new = self.rho2[self.it & 1], self.rho2[(self.it + 1) & 1]
        self.fused_product = A.apply_dot(p, q, self.pq)                       # q = A p; pq = (p, q)
        peers_ok = ctx.peers is not None and ctx.use_peer_reduce and ctx.nparts > 1
        for k in ctx.local:
            ws, _ = ctx.workspace(k)
            L.check(lib.vexb_cg_update_r(ctx.devs[k], ctx.streams[k], x.dtype, x.part_size(k), r.bufs[k], q.bufs[k],
                                         rho.bufs[k], self.pq.bufs[k], rho_new.bufs[k], ws, ctx.peers[k] if peers_ok else None))
        if ctx.nparts > 1 and not peers_ok:
            if ctx.comms is None:
                raise RuntimeError("CG over several slots needs a peer group or a communicator")
            L.check(lib.vexb_comm_allreduce(len(ctx.local), ctx._arr(ctx.comms), ctx._arr(rho_new.bufs), ctx._arr(ctx.streams), 1, x.dtype, L.SUM))
        for k in ctx.local:
            L.check(lib.vexb_cg_update_xp(ctx.devs[k], ctx.streams[k], x.dtype, x.part_size(k), x.bufs[k], p.bufs[k], r.bufs[k],
                                          rho.bufs[k], self.pq.bufs[k], rho_new.bufs[k]))
        self.it += 1

    def capture(self):
        self.step(); self.step()                          # warm up both parities outside the capture
        self.ctx.finish()
        g = []
        for _ in range(2):
            g.append(Graph(self.ctx, self.step))          # capturing does not execute: `it` advances, the vectors do not
        self.it -= 2
        self.graphs = {self.it & 1: g[0], (self.it + 1) & 1: g[1]}
        return self

    def run(self, iters: int):
        for _ in range(iters):
            if self.graphs is not None:
                self.graphs[self.it & 1].launch()
                self.it += 1
            else:
                self.step()

    def residual2(self) -> float:
        return float(self.rho2[self.it & 1].get())


def cg_fused_bytes_per_iteration(n: int, spmv_bytes: int) -> int:
    """Compulsory traffic of CGFused: the product (which already reads p and writes q) + r sweep 24N + x/p sweep 40N."""
    return spmv_bytes + 64 * n


def cg_bytes_per_iteration(n: int, spmv_bytes: int, count_p_update: bool = True) -> int:
    """Unfused reference-equivalent traffic (BASELINE.md section 3): SpMV + dot(p,q) 16N + axpy 24N + axpy 24N +
    dot(r,r) 8N (+ p = r + beta p, 24N)."""
    return spmv_bytes + (72 + (24 if count_p_update else 0)) * n
