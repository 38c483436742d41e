"""The order of additions of csrc/scan.cu (vexb_scan, vexb_scan_by_key, vexb_reduce_by_key_*) restated in numpy.

Every add is rounded in the value dtype (numpy rounds each operation on float32 / float64 arrays on its own; integer
arrays wrap), vectorised over tiles and threads.  The identity is -0.0 for floats (-0.0 + x == x exactly) and 0 for
integers.  Segmented pairs (f, s) combine as (fa, sa) . (fb, sb) = (fa | fb, fb ? sb : sa + sb).

  heads   element i heads a run when i == 0 or keys[i] != keys[i - 1] (float ==); without keys only element 0 does
  reduce  tiles of 4096 = 256 threads x 16 consecutive elements; thread j folds its elements in order from the identity
          (s = head ? x : s + x); Kogge-Stone over the 32 lanes of each warp (offsets 1..16), exclusive by a shift of
          one lane; Kogge-Stone over the 8 warp totals (offsets 1, 2, 4); the tile's pair is warp 7's inclusive value
  carry   1024 threads; thread p folds tiles [p P, (p + 1) P), P = ceil(T / 1024), in order from the identity; the same
          Kogge-Stone over lanes and over the 32 warp totals; each thread walks its tiles from its exclusive prefix,
          writing the running value as the tile's carry, then combining the tile's pair
  apply   thread j starts at r = xf ? xs : carry + xs, with (xf, xs) = (warp prefix) . (lane prefix); inclusive:
          r = head ? x : r + x, written; exclusive: r = init + r, then per element r = init on a head, write r, r = r + x
"""
from __future__ import annotations

import numpy as np

TILE, THREADS, ITEMS, WARPS = 4096, 256, 16, 8
CARRY_THREADS = 1024


def identity(dtype):
    dtype = np.dtype(dtype)
    return dtype.type(-0.0) if dtype.kind == "f" else dtype.type(0)


def heads_of(n: int, keys=None) -> np.ndarray:
    h = np.zeros(n, dtype=bool)
    if n == 0:
        return h
    if keys is None:
        h[0] = True
    else:
        keys = np.asarray(keys)
        h[0] = True
        h[1:] = ~(keys[1:] == keys[:-1])
    return h


def _seg(fa, sa, fb, sb):
    return fa | fb, np.where(fb, sb, sa + sb)


def _kogge_stone(f, s, width, ident):
    """Inclusive segmented Kogge-Stone over the last axis (lanes), offsets 1, 2, ... < width."""
    o = 1
    while o < width:
        fu = np.concatenate([np.zeros_like(f[..., :o]), f[..., :-o]], axis=-1)
        su = np.concatenate([np.full_like(s[..., :o], ident), s[..., :-o]], axis=-1)
        lane = np.arange(f.shape[-1]) >= o
        ns = np.where(f, s, su + s)
        f, s = np.where(lane, f | fu, f), np.where(lane, ns, s)
        o <<= 1
    return f, s


def _shift1(f, s, ident):
    return (np.concatenate([np.zeros_like(f[..., :1]), f[..., :-1]], axis=-1),
            np.concatenate([np.full_like(s[..., :1], ident), s[..., :-1]], axis=-1))


def _block_scan(f, s, nwarps, ident):
    """Exclusive prefix per thread and the block's pair; f, s: (..., nwarps * 32)."""
    shp = f.shape[:-1]
    f = f.reshape(*shp, nwarps, 32)
    s = s.reshape(*shp, nwarps, 32)
    fi, si = _kogge_stone(f, s, 32, ident)
    fe, se = _shift1(fi, si, ident)
    wfi, wsi = _kogge_stone(fi[..., 31], si[..., 31], nwarps, ident)
    pf, ps = _shift1(wfi, wsi, ident)
    xf, xs = _seg(pf[..., None], ps[..., None], fe, se)
    return xf.reshape(*shp, nwarps * 32), xs.reshape(*shp, nwarps * 32), wfi[..., -1], wsi[..., -1]


def _threads(x, h, ident):
    """Per thread of every tile: values and heads (T, 256, 16), and the thread's folded pair."""
    n = x.size
    T = -(-n // TILE)
    xp = np.full(T * TILE, ident, dtype=x.dtype)
    xp[:n] = x
    hp = np.zeros(T * TILE, dtype=bool)
    hp[:n] = h
    xp, hp = xp.reshape(T, THREADS, ITEMS), hp.reshape(T, THREADS, ITEMS)
    f = np.zeros((T, THREADS), dtype=bool)
    s = np.full((T, THREADS), ident, dtype=x.dtype)
    for k in range(ITEMS):
        s = np.where(hp[..., k], xp[..., k], s + xp[..., k])
        f = f | hp[..., k]
    return xp, hp, f, s


def carries(af, asum, ident):
    """Phase 2: the carry into every tile from the tiles' pairs."""
    T = asum.size
    per = -(-T // CARRY_THREADS)
    fp = np.zeros(CARRY_THREADS * per, dtype=bool)
    sp = np.full(CARRY_THREADS * per, ident, dtype=asum.dtype)
    fp[:T], sp[:T] = af, asum
    fp, sp = fp.reshape(CARRY_THREADS, per), sp.reshape(CARRY_THREADS, per)
    f = np.zeros(CARRY_THREADS, dtype=bool)
    s = np.full(CARRY_THREADS, ident, dtype=asum.dtype)
    for m in range(per):
        s = np.where(fp[:, m], sp[:, m], s + sp[:, m])
        f = f | fp[:, m]
    _, xs, _, _ = _block_scan(f, s, CARRY_THREADS // 32, ident)
    out = np.empty((CARRY_THREADS, per), dtype=asum.dtype)
    run = xs
    for m in range(per):
        out[:, m] = run
        run = np.where(fp[:, m], sp[:, m], run + sp[:, m])
    return out.reshape(-1)[:T]


def _scan(x, h, exclusive: bool, init):
    x = np.asarray(x)
    dt = x.dtype
    ident = identity(dt)
    n = x.size
    with np.errstate(over="ignore", invalid="ignore"):
        xp, hp, f, s = _threads(x, h, ident)
        xf, xs, af, asum = _block_scan(f, s, WARPS, ident)
        c = carries(af, asum, ident)
        r = np.where(xf, xs, c[:, None] + xs)
        out = np.empty_like(xp)
        if exclusive:
            init = np.asarray(init).astype(dt)
            r = init + r
            for k in range(ITEMS):
                r = np.where(hp[..., k], init, r)
                out[..., k] = r
                r = r + xp[..., k]
        else:
            for k in range(ITEMS):
                r = np.where(hp[..., k], xp[..., k], r + xp[..., k])
                out[..., k] = r
    return out.reshape(-1)[:n]


def scan(x, exclusive: bool = False, init=0):
    """vexb_scan of one slice."""
    x = np.asarray(x)
    return _scan(x, heads_of(x.size), exclusive, init)


def scan_by_key(keys, x, exclusive: bool = False, init=0):
    """vexb_scan_by_key."""
    x = np.asarray(x)
    return _scan(x, heads_of(x.size, keys), exclusive, init)


def reduce_by_key(keys, x):
    """vexb_reduce_by_key_*: (okeys, ovals), the last key and the inclusive value at the end of every run."""
    keys, x = np.asarray(keys), np.asarray(x)
    h = heads_of(x.size, keys)
    incl = _scan(x, h, False, 0)
    ends = np.append(h[1:], True) if x.size else h
    return keys[ends], incl[ends]


def scan_parts(x, sizes, exclusive: bool = False, init=0):
    """The front ends on several parts: the first non-empty part starts at init, the others at the identity; the local
    totals are folded in the element type and each carry is added to its part."""
    x = np.asarray(x)
    dt = x.dtype
    ident = identity(dt)
    outs, totals, started, o = [], [], False, 0
    with np.errstate(over="ignore", invalid="ignore"):
        for m in sizes:
            p = x[o:o + m]
            o += m
            if m == 0:
                outs.append(p.copy())
                totals.append(None)
                continue
            out = scan(p, exclusive, init if not started else ident)
            started = True
            totals.append(dt.type(out[-1] + p[-1]) if exclusive else out[-1])
            outs.append(out)
        carry = None
        for i, m in enumerate(sizes):
            if m == 0:
                continue
            if carry is None:
                carry = totals[i]
            else:
                outs[i] = outs[i] + carry
                carry = dt.type(carry + totals[i])
    return np.concatenate(outs) if outs else x.copy()
