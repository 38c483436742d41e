"""Synthetic workloads of the named configurations, generated strip by strip.

Matrix convention = the reference benchmark's (examples/benchmark.cpp:357-415): a regular
grid, rows on the domain boundary are identity (col = idx, val = 1), interior rows carry the
full 5-point (2-D) / 7-point (3-D) stencil with h2i = (n-1)^2 off-diagonal weight -h2i and
diagonal 4*h2i / 6*h2i, columns in ascending order.  `poisson_strip` produces rows
[r0, r1) only (global column ids, row offsets starting at 0), so that a rank never
materialises more than its own slab.  Grids may be anisotropic (nx, ny, nz) for the weak
scaling runs; h2i is always (nx-1)^2.
"""
from __future__ import annotations

import numpy as np


def poisson_dims(dim: int, nx: int, ny: int | None = None, nz: int | None = None):
    ny = nx if ny is None else ny
    nz = (nx if nz is None else nz) if dim == 3 else 1
    return nx, ny, nz


def poisson_strip(dim: int, nx: int, ny: int | None = None, nz: int | None = None, r0: int = 0, r1: int | None = None,
                  index_dtype=np.int64, spd: bool = False):
    """Rows [r0, r1) of the Poisson matrix on an nx*ny(*nz) grid.  Returns (row, col, val).
    spd=True: the symmetric positive definite form instead of the benchmark's (every row carries the stencil, neighbours
    outside the grid are dropped -- homogeneous Dirichlet conditions eliminated), entries scaled to O(1): what a CG
    iteration needs to converge (the benchmark's identity boundary rows make the matrix non-symmetric)."""
    nx, ny, nz = poisson_dims(dim, nx, ny, nz)
    N = nx * ny * nz
    r1 = N if r1 is None else r1
    idx = np.arange(r0, r1, dtype=np.int64)
    i = idx % nx
    j = (idx // nx) % ny
    k = idx // (nx * ny)
    if spd:
        if dim == 2:
            offs = [-nx, -1, 0, 1, nx]
            ok = [j > 0, i > 0, np.ones(idx.size, bool), i < nx - 1, j < ny - 1]
            vals = [-1.0, -1.0, 4.0, -1.0, -1.0]
        else:
            offs = [-nx * ny, -nx, -1, 0, 1, nx, nx * ny]
            ok = [k > 0, j > 0, i > 0, np.ones(idx.size, bool), i < nx - 1, j < ny - 1, k < nz - 1]
            vals = [-1.0, -1.0, -1.0, 6.0, -1.0, -1.0, -1.0]
        keep = np.stack(ok, axis=1)                              # (rows, w) in ascending column order
        width = keep.sum(axis=1)
        row = np.zeros(idx.size + 1, dtype=np.int64)
        np.cumsum(width, out=row[1:])
        cols = idx[:, None] + np.asarray(offs, dtype=np.int64)[None, :]
        valm = np.broadcast_to(np.asarray(vals)[None, :], keep.shape)
        return row.astype(index_dtype), cols[keep].astype(index_dtype), np.ascontiguousarray(valm[keep])
    bnd = (i == 0) | (i == nx - 1) | (j == 0) | (j == ny - 1)
    if dim == 3:
        bnd |= (k == 0) | (k == nz - 1)
    h2i = float((nx - 1) * (nx - 1))
    if dim == 2:
        offs = np.array([-nx, -1, 0, 1, nx], dtype=np.int64)
        vals = np.array([-h2i, -h2i, 4 * h2i, -h2i, -h2i])
    else:
        offs = np.array([-nx * ny, -nx, -1, 0, 1, nx, nx * ny], dtype=np.int64)
        vals = np.array([-h2i, -h2i, -h2i, 6 * h2i, -h2i, -h2i, -h2i])
    w = offs.size
    width = np.where(bnd, 1, w).astype(np.int64)
    row = np.zeros(idx.size + 1, dtype=np.int64)
    np.cumsum(width, out=row[1:])
    nnz = int(row[-1])
    col = np.empty(nnz, dtype=np.int64)
    val = np.empty(nnz, dtype=np.float64)
    # boundary rows
    b_at = row[:-1][bnd]
    col[b_at] = idx[bnd]
    val[b_at] = 1.0
    # interior rows
    inner = ~bnd
    i_at = row[:-1][inner]
    i_idx = idx[inner]
    for t in range(w):
        col[i_at + t] = i_idx + offs[t]
        val[i_at + t] = vals[t]
    return row.astype(index_dtype), col.astype(index_dtype), val


def poisson_ccsr(n: int, index_dtype=np.uint64, col_dtype=np.int32):
    """The 3-D Poisson matrix on an n^3 grid in CCSR form, as the reference builds it (examples/benchmark.cpp:493-545,
    tests/spmv.cpp:150-197): unique row 0 = boundary (identity), unique row 1 = 7-point stencil.
    Returns (idx, row, col, val)."""
    h2i = float((n - 1) * (n - 1))
    row = np.array([0, 1, 8], dtype=index_dtype)
    col = np.array([0, -n * n, -n, -1, 0, 1, n, n * n], dtype=col_dtype)
    val = np.array([1.0, -h2i, -h2i, -h2i, 6 * h2i, -h2i, -h2i, -h2i])
    g = np.arange(n)
    edge = (g == 0) | (g == n - 1)
    bnd = edge[:, None, None] | edge[None, :, None] | edge[None, None, :]
    idx = np.where(bnd, 0, 1).astype(index_dtype).ravel()
    return idx, row, col, val


def irregular_rows(n: int, lo: int = 0, hi: int = 32, seed: int = 1, index_dtype=np.int64, max_gap: int = 64):
    """An irregular square matrix: row widths U[lo, hi), columns ascending within a row (random gaps of 1..max_gap-1
    starting about half a row's span left of the diagonal, clipped to the matrix), values U[-0.5, 0.5).  max_gap = 64:
    every nonzero's x value in its own 128-byte line (scattered); max_gap = 8: a few per line (clustered, FEM-like).
    Returns (row, col, val)."""
    rng = np.random.default_rng(seed)
    w = rng.integers(lo, hi, n)
    row = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(w, out=row[1:])
    nnz = int(row[-1])
    gaps = rng.integers(1, max_gap, nnz)
    run = np.cumsum(gaps)
    start = np.repeat(run[row[:-1].clip(max=max(nnz - 1, 0))] - gaps[row[:-1].clip(max=max(nnz - 1, 0))], w) if nnz else np.empty(0, np.int64)
    base = np.repeat(np.arange(n, dtype=np.int64) - (max_gap // 4) * w, w)
    col = np.clip(base + (run - start), 0, n - 1)
    return row.astype(index_dtype), col.astype(index_dtype), rng.random(nnz) - 0.5


def irregular_spd(n: int, hi: int = 32, seed: int = 1, max_gap: int = 64):
    """A symmetric positive definite matrix with irregular rows, for CG: the entries of irregular_rows(n, 0, hi, seed)
    below the diagonal, without those clipping sent to column 0 (they would pile up in row 0 and give the spectrum an
    outlier) and one per column where clipping repeated a column, mirrored above the diagonal; on the diagonal 1 + the
    row's sum of |off-diagonal| (strictly diagonally dominant).  Rows hold 1 to about hi entries, about hi / 2 on average.
    Returns int64 row, col and float64 val, columns ascending."""
    row, col, val = irregular_rows(n, 0, hi, seed, np.int64, max_gap)
    r = np.repeat(np.arange(n, dtype=np.int64), np.diff(row))
    low = (col < r) & (col > 0)
    _, first = np.unique(r[low] * n + col[low], return_index=True)
    i, j, v = r[low][first], col[low][first], val[low][first]
    d = np.arange(n, dtype=np.int64)
    rr, cc = np.concatenate([i, j, d]), np.concatenate([j, i, d])
    vv = np.concatenate([v, v, 1.0 + np.bincount(i, np.abs(v), n) + np.bincount(j, np.abs(v), n)])
    order = np.argsort(rr * n + cc, kind="stable")
    out = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rr, minlength=n), out=out[1:])
    return out, cc[order], vv[order]


def ccsr_bytes(nrows: int, idx_bytes: int = 8) -> int:
    """Algorithmic bytes of y = A*x for a CCSR matrix: idx as the reference stores it (size_t), x and y once; the
    unique-row table is negligible."""
    return nrows * (idx_bytes + 16)


def poisson_nnz(dim: int, nx: int, ny: int | None = None, nz: int | None = None) -> tuple[int, int]:
    nx, ny, nz = poisson_dims(dim, nx, ny, nz)
    N = nx * ny * nz
    if dim == 2:
        inner = max(nx - 2, 0) * max(ny - 2, 0)
        return N, inner * 5 + (N - inner)
    inner = max(nx - 2, 0) * max(ny - 2, 0) * max(nz - 2, 0)
    return N, inner * 7 + (N - inner)


def spmv_bytes(nrows: int, ncols: int, nnz: int, append: bool = False) -> int:
    """Algorithmic bytes of y = A*x (BASELINE.md section 3): double values, 32-bit columns and row
    pointers, x and y touched once; + nrows*8 for y += A*x."""
    return nnz * 12 + (nrows + 1) * 4 + ncols * 8 + nrows * 8 + (nrows * 8 if append else 0)
