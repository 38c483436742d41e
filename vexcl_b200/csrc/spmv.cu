// Sparse strips on one device: y (=|+=) alpha * A * x.
//
// Replaces SpMatCSR / SpMatHELL (vexcl/spmat/csr.inl:45-209,
// vexcl/spmat/hybrid_ell.inl:53-330): one thread per row, 8-byte indices,
// row-strided (uncoalesced) val/col reads in the CSR case.
//
// CSR here is a row-block *stream* kernel:
//   * rows are cut on the host into tiles of <= tile_nnz nonzeros / <= tile_rows rows;
//   * one CTA per tile; an elected thread issues three TMA bulk copies
//     (cp.async.bulk.shared.global -> UBLKCP) that stage the tile's row_ptr, col
//     and val slices in shared memory and complete on an mbarrier;
//   * phase A: all threads walk the staged nonzeros (coalesced), gather x[col]
//     through L1/L2 and overwrite val in place with the product;
//   * phase B: one thread per row adds its products in storage order -- the same
//     sequential order as the reference kernel (csr.inl:163-170) -- or, for
//     tiles with long rows, one warp per row with a shuffle tree;
//   * rows longer than a tile are handled by a whole CTA straight from HBM.
// Indices are 32-bit on the device (always lossless after the per-strip
// renumbering, csr.inl:92-107), halving index traffic against SpMat<double>'s
// default size_t (spmat.hpp:56).
//
// HELL keeps the reference layout (column-major ELL with pitch alignup(n,16),
// sentinel column -1, CSR tail; hybrid_ell.inl:60,139-144,252-268) with 32-bit
// columns, and unrolls the ELL loop for the common small widths.
#include "spmat.hpp"
#include "ccsr.hpp"
#include "spmv_dev.cuh"
#include <cstring>
#include <string>
#include <unordered_map>
#include <algorithm>


namespace vexb {

// Phase A of the stream kernels: val_s[j] *= x[col_s[j]] for j in [lo, lo+cnt), all threads.
// The gathers of a batch are issued before any product is stored, so a thread keeps UA
// independent L1/L2 requests in flight (a plain loop would serialise on the in-place store).
template <class T, int UA>
__device__ __forceinline__ void phase_a_products(T *val_s, const int *col_s, const T *__restrict__ x,
                                                 int lo, int cnt, int tid, int nthreads) {
    const uint64_t keep = l2_policy_keep();
    const int hi = lo + cnt;
    for (int j = lo + tid; j < hi; j += nthreads * UA) {
        T xv[UA];
#pragma unroll
        for (int u = 0; u < UA; ++u) {
            const int jj = j + u * nthreads;
            xv[u] = (jj < hi) ? ldg_keep(x + col_s[jj], keep) : T(0);
        }
#pragma unroll
        for (int u = 0; u < UA; ++u) {
            const int jj = j + u * nthreads;
            if (jj < hi) val_s[jj] = t_mul<T>(val_s[jj], xv[u]);
        }
    }
}

__device__ __forceinline__ void mbar_wait_fwd(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}

// Shared-memory carve-up (dynamic): [val: (tile_nnz+8)*sizeof(T)] [col: (tile_nnz+8)*4] [rp: (tile_rows+12)*4] [mbarrier]
template <class T>
__global__ void __launch_bounds__(256) csr_stream_kernel(const int2 *__restrict__ tile, const int *__restrict__ rowptr,
                                                          const int *__restrict__ col, const T *__restrict__ val,
                                                          const T *__restrict__ x, T *y, T alpha, int append,
                                                          int tile_nnz, int tile_rows, const int *__restrict__ row_ids) {
    extern __shared__ __align__(128) unsigned char smem[];
    T *val_s = reinterpret_cast<T *>(smem);
    int *col_s = reinterpret_cast<int *>(smem + (size_t)(tile_nnz + 8) * sizeof(T));
    int *rp_s = col_s + (tile_nnz + 8);
    uint64_t *bar = reinterpret_cast<uint64_t *>(rp_s + (tile_rows + 12));

    const int2 t0 = tile[blockIdx.x], t1 = tile[blockIdx.x + 1];
    const int r0 = t0.x, nr = t1.x - t0.x;
    const int j0 = t0.y, cnt = t1.y - t0.y;
    if (nr <= 0) return;

    if (cnt > tile_nnz) {
        // one long row: the whole CTA strides over it straight from global memory
        T s = T(0);
        for (int j = j0 + threadIdx.x; j < j0 + cnt; j += blockDim.x) s = t_add<T>(s, t_mul<T>(val[j], x[col[j]]));
        __shared__ T red[8];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            T tot = red[0];
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w) tot = t_add<T>(tot, red[w]);
            store_y<T>(y, row_ids ? (size_t)row_ids[r0] : (size_t)r0, tot, alpha, append);
        }
        return;
    }

    // aligned windows for the bulk copies (16-byte granularity)
    const int j0a = j0 & ~3, j1a = (j0 + cnt + 3) & ~3;
    const int r0a = r0 & ~3, r1a = (r0 + nr + 1 + 3) & ~3;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(bar)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t bv = (uint32_t)(j1a - j0a) * (uint32_t)sizeof(T);
        const uint32_t bc = (uint32_t)(j1a - j0a) * 4u;
        const uint32_t br = (uint32_t)(r1a - r0a) * 4u;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bv + bc + br) : "memory");
        const uint64_t stream = l2_policy_stream();
        if (bv) { bulk_g2s(val_s, val + j0a, bv, bar, stream); bulk_g2s(col_s, col + j0a, bc, bar, stream); }
        bulk_g2s(rp_s, rowptr + r0a, br, bar, stream);
    }
    __syncthreads();   // barrier init visible to all waiters
    {
        uint32_t done = 0;
        while (!done) {
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(done) : "r"(smem_u32(bar)), "r"(0u) : "memory");
        }
    }
    // phase A: products in place
    const int lo = j0 - j0a;
    phase_a_products<T, 8>(val_s, col_s, x, lo, cnt, (int)threadIdx.x, (int)blockDim.x);
    __syncthreads();
    // phase B
    const int *rp = rp_s + (r0 - r0a);
    if (cnt <= 12 * nr) {
        for (int r = threadIdx.x; r < nr; r += blockDim.x) {
            const int a = rp[r] - j0a, b = rp[r + 1] - j0a;
            T s = T(0);
            for (int j = a; j < b; ++j) s = t_add<T>(s, val_s[j]);
            store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
        }
    } else {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
        for (int r = warp; r < nr; r += nw) {
            const int a = rp[r] - j0a, b = rp[r + 1] - j0a;
            T s = T(0);
            for (int j = a + lane; j < b; j += 32) s = t_add<T>(s, val_s[j]);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
            if (lane == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
        }
    }
}

// ---- CTA tiles with a staged x window (spmv.kernel = 6) ----------------------------------------------------------
// On matrices whose rows scatter over a band (every nonzero in its own 128-byte line of x) the gathers, not HBM, bound
// every kernel above: the L1 tag stage takes one line per cycle per SM, a warp-wide gather 32 of them.  Here the tile's
// slice of x -- columns
// [cmin, cmax] of its nonzeros, found on the host -- is one more TMA bulk copy into shared memory, and phase A gathers
// from there: a handful of bank conflicts instead of 32 tag lookups.  The window is read from L2 (x stays resident),
// HBM traffic is unchanged.  Tiles whose window would not fit (tile_x.y == 0) gather from global memory as before.
// Everything else is csr_stream_kernel: row-block tiles, val/col/row_ptr staged by TMA, products in place, rows added
// in storage order.
template <class T>
__global__ void __launch_bounds__(256) csr_window_kernel(const int2 *__restrict__ tile, const int2 *__restrict__ tile_x,
                                                         const int *__restrict__ rowptr, const int *__restrict__ col,
                                                         const T *__restrict__ val, const T *__restrict__ x, T *y, T alpha,
                                                         int append, int tile_nnz, int tile_rows, int xwin,
                                                         const int *__restrict__ row_ids) {
    extern __shared__ __align__(128) unsigned char smem[];
    T *val_s = reinterpret_cast<T *>(smem);
    T *x_s = val_s + (tile_nnz + 8);
    int *col_s = reinterpret_cast<int *>(x_s + (xwin + 4));
    int *rp_s = col_s + (tile_nnz + 8);
    uint64_t *bar = reinterpret_cast<uint64_t *>(rp_s + (tile_rows + 12));

    const int2 t0 = tile[blockIdx.x], t1 = tile[blockIdx.x + 1];
    const int2 tx = tile_x[blockIdx.x];                  // {first column of the window (even), its length (0: no window)}
    const int r0 = t0.x, nr = t1.x - t0.x;
    const int j0 = t0.y, cnt = t1.y - t0.y;
    if (nr <= 0) return;

    if (cnt > tile_nnz) {
        // one long row: the whole CTA strides over it straight from global memory
        T s = T(0);
        for (int j = j0 + threadIdx.x; j < j0 + cnt; j += blockDim.x) s = t_add<T>(s, t_mul<T>(val[j], x[col[j]]));
        __shared__ T red[8];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            T tot = red[0];
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w) tot = t_add<T>(tot, red[w]);
            store_y<T>(y, row_ids ? (size_t)row_ids[r0] : (size_t)r0, tot, alpha, append);
        }
        return;
    }

    const int j0a = j0 & ~3, j1a = (j0 + cnt + 3) & ~3;
    const int r0a = r0 & ~3, r1a = (r0 + nr + 1 + 3) & ~3;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(bar)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t bv = (uint32_t)(j1a - j0a) * (uint32_t)sizeof(T);
        const uint32_t bc = (uint32_t)(j1a - j0a) * 4u;
        const uint32_t br = (uint32_t)(r1a - r0a) * 4u;
        const uint32_t bx = (uint32_t)tx.y * (uint32_t)sizeof(T);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bv + bc + br + bx) : "memory");
        const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
        if (bx) bulk_g2s(x_s, x + tx.x, bx, bar, keep);
        if (bv) { bulk_g2s(val_s, val + j0a, bv, bar, stream); bulk_g2s(col_s, col + j0a, bc, bar, stream); }
        bulk_g2s(rp_s, rowptr + r0a, br, bar, stream);
    }
    __syncthreads();
    mbar_wait_fwd(bar, 0u);
    const int lo = j0 - j0a;
    if (tx.y) {
        // phase A from the window: val_s[j] *= x_s[col_s[j] - first column]
        const int hi = lo + cnt, cb = tx.x, nt = (int)blockDim.x;
        for (int j = lo + (int)threadIdx.x; j < hi; j += nt * 8) {
            int c[8]; T xv[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int jj = j + u * nt; c[u] = jj < hi ? col_s[jj] - cb : 0; }
#pragma unroll
            for (int u = 0; u < 8; ++u) xv[u] = x_s[c[u]];
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int jj = j + u * nt; if (jj < hi) val_s[jj] = t_mul<T>(val_s[jj], xv[u]); }
        }
    } else {
        phase_a_products<T, 8>(val_s, col_s, x, lo, cnt, (int)threadIdx.x, (int)blockDim.x);
    }
    __syncthreads();
    const int *rp = rp_s + (r0 - r0a);
    if (cnt <= 12 * nr) {
        for (int r = threadIdx.x; r < nr; r += blockDim.x) {
            const int a = rp[r] - j0a, b = rp[r + 1] - j0a;
            T s = T(0);
            for (int j = a; j < b; ++j) s = t_add<T>(s, val_s[j]);
            store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
        }
    } else {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
        for (int r = warp; r < nr; r += nw) {
            const int a = rp[r] - j0a, b = rp[r + 1] - j0a;
            T s = T(0);
            for (int j = a + lane; j < b; j += 32) s = t_add<T>(s, val_s[j]);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
            if (lane == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
        }
    }
}

// ---- register-staged version of the stream kernel ------------------------------------------------
// Same tiles, same two phases, but val / col go from HBM straight into registers (coalesced 8-byte
// and 4-byte loads, L1 no-allocate), and only the products pass through shared memory.  Shared memory
// per CTA drops from 26.8 KB to 16 KB, so L1 keeps ~150 KB for the x gathers (the TMA version leaves it
// ~14 KB), and the bytes in flight live in the register file instead of the staging buffers.
constexpr int kDirectThreads = 256;
constexpr int kDirectPerThread = 8;                   // tile_nnz <= 2048

template <class T>
__global__ void __launch_bounds__(kDirectThreads, 5) csr_direct_kernel(const int2 *__restrict__ tile, const int *__restrict__ rowptr,
                                                                        const int *__restrict__ col, const T *__restrict__ val,
                                                                        const T *__restrict__ x, T *y, T alpha, int append,
                                                                        int tile_nnz, const int *__restrict__ row_ids) {
    extern __shared__ __align__(16) unsigned char smem[];
    T *prod = reinterpret_cast<T *>(smem);
    const int tid = threadIdx.x;
    const int2 t0 = __ldg(tile + blockIdx.x), t1 = __ldg(tile + blockIdx.x + 1);
    const int r0 = t0.x, nr = t1.x - t0.x;
    const int j0 = t0.y, cnt = t1.y - t0.y;
    if (nr <= 0) return;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();

    if (cnt > tile_nnz) {
        // one long row (build() gives a row longer than tile_nnz a tile of its own; prod holds only tile_nnz
        // products): the whole CTA strides over it
        T s = T(0);
        for (int j = j0 + tid; j < j0 + cnt; j += kDirectThreads) s = t_add<T>(s, t_mul<T>(ldg_stream(val + j, stream), ldg_keep(x + ldg_stream(col + j, stream), keep)));
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
        if ((tid & 31) == 0) prod[tid >> 5] = s;
        __syncthreads();
        if (tid == 0) {
            T tot = prod[0];
            for (int w = 1; w < kDirectThreads / 32; ++w) tot = t_add<T>(tot, prod[w]);
            store_y<T>(y, row_ids ? (size_t)row_ids[r0] : (size_t)r0, tot, alpha, append);
        }
        return;
    }

    // row pointers of the (up to two) rows this thread will sum in phase B: issued first, needed last
    int ra[2] = {0, 0}, rb[2] = {0, 0};
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const int r = tid + p * kDirectThreads;
        if (r < nr) { ra[p] = __ldg(rowptr + r0 + r); rb[p] = __ldg(rowptr + r0 + r + 1); }
    }
    // this thread's nonzeros j0 + tid + k*256: all loads issued back to back
    int c[kDirectPerThread]; T v[kDirectPerThread]; T xv[kDirectPerThread];
#pragma unroll
    for (int k = 0; k < kDirectPerThread; ++k) {
        const int j = tid + k * kDirectThreads;
        if (j < cnt) { c[k] = ldg_stream(col + j0 + j, stream); v[k] = ldg_stream(val + j0 + j, stream); }
    }
#pragma unroll
    for (int k = 0; k < kDirectPerThread; ++k) {
        const int j = tid + k * kDirectThreads;
        xv[k] = (j < cnt) ? ldg_keep(x + c[k], keep) : T(0);
    }
#pragma unroll
    for (int k = 0; k < kDirectPerThread; ++k) {
        const int j = tid + k * kDirectThreads;
        if (j < cnt) prod[j] = t_mul<T>(v[k], xv[k]);
    }
    __syncthreads();
    // phase B: row sums in storage order
    if (cnt <= 12 * nr) {
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int r = tid + p * kDirectThreads;
            if (r < nr) {
                T s = T(0);
                for (int j = ra[p] - j0; j < rb[p] - j0; ++j) s = t_add<T>(s, prod[j]);
                store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
            }
        }
        for (int r = tid + 2 * kDirectThreads; r < nr; r += kDirectThreads) {
            const int a = __ldg(rowptr + r0 + r) - j0, b = __ldg(rowptr + r0 + r + 1) - j0;
            T s = T(0);
            for (int j = a; j < b; ++j) s = t_add<T>(s, prod[j]);
            store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
        }
    } else {
        const int lane = tid & 31, warp = tid >> 5;
        for (int r = warp; r < nr; r += kDirectThreads / 32) {
            const int a = __ldg(rowptr + r0 + r) - j0, b = __ldg(rowptr + r0 + r + 1) - j0;
            T s = T(0);
            for (int j = a + lane; j < b; j += 32) s = t_add<T>(s, prod[j]);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
            if (lane == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
        }
    }
}

// ---- persistent, warp-specialised, multi-stage version of the stream kernel ---------------------
// One producer warp keeps up to `stages` tiles in flight with TMA bulk copies (full/empty
// mbarrier ring); eight consumer warps do phase A / phase B of the oldest tile meanwhile, so
// HBM never waits for the gather or the row sums.  Grid = resident CTAs only; tiles are dealt
// round-robin (tile = blockIdx.x + it * gridDim.x).
constexpr int kPipeConsumers = 256;
constexpr int kPipeThreads = kPipeConsumers + 32;

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}

template <class T>
__global__ void __launch_bounds__(kPipeThreads) csr_pipe_kernel(const int2 *__restrict__ tile, int n_tiles,
                                                                 const int *__restrict__ rowptr, const int *__restrict__ col,
                                                                 const T *__restrict__ val, const T *__restrict__ x, T *y,
                                                                 T alpha, int append, int tile_nnz, int tile_rows, int stages,
                                                                 const int *__restrict__ row_ids) {
    extern __shared__ __align__(128) unsigned char smem[];
    const size_t val_bytes = (size_t)(tile_nnz + 8) * sizeof(T);
    const size_t col_bytes = (size_t)(tile_nnz + 8) * 4;
    const size_t rp_bytes = (size_t)(tile_rows + 12) * 4;
    const size_t stage_bytes = (val_bytes + col_bytes + rp_bytes + 127) & ~(size_t)127;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + stage_bytes * stages);
    uint64_t *empty = full + stages;
    int4 *meta = reinterpret_cast<int4 *>(empty + stages);          // per stage: {r0, nr, j0, cnt}

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(full + s)) : "memory");
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(empty + s)), "r"(kPipeConsumers / 32) : "memory");
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kPipeConsumers / 32) {
        // ===== producer warp (one elected lane) =====
        if (lane == 0) {
            const uint64_t stream = l2_policy_stream();
            int it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
                const int s = it % stages;
                const uint32_t ph = (uint32_t)(it / stages) & 1u;
                mbar_wait(empty + s, ph ^ 1u);                       // slot free (passes at once on the first lap)
                const int2 t0 = __ldg(tile + t), t1 = __ldg(tile + t + 1);
                const int r0 = t0.x, nr = t1.x - t0.x, j0 = t0.y, cnt = t1.y - t0.y;
                meta[s] = make_int4(r0, nr, j0, cnt);
                unsigned char *base = smem + stage_bytes * s;
                if (cnt > tile_nnz || nr <= 0) {
                    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(full + s)) : "memory");
                    continue;
                }
                const int j0a = j0 & ~3, j1a = (j0 + cnt + 3) & ~3;
                const int r0a = r0 & ~3, r1a = (r0 + nr + 1 + 3) & ~3;
                const uint32_t bv = (uint32_t)(j1a - j0a) * (uint32_t)sizeof(T);
                const uint32_t bc = (uint32_t)(j1a - j0a) * 4u;
                const uint32_t br = (uint32_t)(r1a - r0a) * 4u;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(full + s)), "r"(bv + bc + br) : "memory");
                if (bv) { bulk_g2s(base, val + j0a, bv, full + s, stream); bulk_g2s(base + val_bytes, col + j0a, bc, full + s, stream); }
                bulk_g2s(base + val_bytes + col_bytes, rowptr + r0a, br, full + s, stream);
            }
        }
        return;
    }

    // ===== consumer warps =====
    const int tid = threadIdx.x;                                      // 0 .. 255
    int it = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
        const int s = it % stages;
        const uint32_t ph = (uint32_t)(it / stages) & 1u;
        mbar_wait(full + s, ph);
        const int4 m = meta[s];
        const int r0 = m.x, nr = m.y, j0 = m.z, cnt = m.w;
        unsigned char *base = smem + stage_bytes * s;
        T *val_s = reinterpret_cast<T *>(base);
        const int *col_s = reinterpret_cast<const int *>(base + val_bytes);
        const int *rp_s = reinterpret_cast<const int *>(base + val_bytes + col_bytes);
        if (nr > 0 && cnt > tile_nnz) {
            // one long row, straight from global memory, reduced across the consumer warps
            T sacc = T(0);
            for (int j = j0 + tid; j < j0 + cnt; j += kPipeConsumers) sacc = t_add<T>(sacc, t_mul<T>(val[j], __ldg(x + col[j])));
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) sacc = t_add<T>(sacc, __shfl_down_sync(0xffffffffu, sacc, off));
            T *red = val_s;                                           // the stage is unused for this tile
            if (lane == 0) red[warp] = sacc;
            asm volatile("bar.sync 1, %0;" :: "n"(kPipeConsumers) : "memory");
            if (tid == 0) {
                T tot = red[0];
                for (int w = 1; w < kPipeConsumers / 32; ++w) tot = t_add<T>(tot, red[w]);
                store_y<T>(y, row_ids ? (size_t)row_ids[r0] : (size_t)r0, tot, alpha, append);
            }
            asm volatile("bar.sync 1, %0;" :: "n"(kPipeConsumers) : "memory");
        } else if (nr > 0) {
            const int j0a = j0 & ~3, r0a = r0 & ~3;
            const int lo = j0 - j0a;
            // phase A: products in place (coalesced walk over the staged nonzeros, x gathered through L1/L2)
            phase_a_products<T, 8>(val_s, col_s, x, lo, cnt, tid, kPipeConsumers);
            asm volatile("bar.sync 1, %0;" :: "n"(kPipeConsumers) : "memory");
            // phase B: row sums in storage order
            const int *rp = rp_s + (r0 - r0a);
            if (cnt <= 12 * nr) {
                for (int r = tid; r < nr; r += kPipeConsumers) {
                    const int a = rp[r] - j0a, b = rp[r + 1] - j0a;
                    T sacc = T(0);
                    for (int j = a; j < b; ++j) sacc = t_add<T>(sacc, val_s[j]);
                    store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, sacc, alpha, append);
                }
            } else {
                for (int r = warp; r < nr; r += kPipeConsumers / 32) {
                    const int a = rp[r] - j0a, b = rp[r + 1] - j0a;
                    T sacc = T(0);
                    for (int j = a + lane; j < b; j += 32) sacc = t_add<T>(sacc, val_s[j]);
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1) sacc = t_add<T>(sacc, __shfl_down_sync(0xffffffffu, sacc, off));
                    if (lane == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, sacc, alpha, append);
                }
            }
        }
        // release the stage: generic-proxy accesses ordered before the next TMA write into it
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(empty + s)) : "memory");
    }
}

// Rows per thread of hell_kernel on row-class strips.  Measured on configs[2] / configs[3] (H100 80GB HBM3, 400 W):
// 1 row 0.080 / 0.137 ms, 2 rows 0.077 / 0.126 ms, 4 rows 0.083 / 0.140 ms.
constexpr int kEllClassRows = 2;
// How many blocks ahead hell_kernel prefetches into L2 on row-class strips.  Measured on configs[2] / configs[3]
// (H100 80GB HBM3, 700 W), ms per product: none 0.0776 / 0.126, 132 0.0695 / 0.117, 264 and 528 0.0693 / 0.117,
// 792 0.0695 / 0.117, 1584 0.0703 / 0.118, 3168 0.0912 / 0.152 (prefetched lines evicted before their rows run).
// In bench.py (400 W card) 132 blocks cost configs[3] less than 528 (+1.4 % against +3.9 %) for the same gain on configs[2].
constexpr int kEllClassPrefetchBlocks = 132;

// V: stored value type (hell_row_sum); float under double vectors for VEXB_FMT_VALUES_F32 strips, which never use row classes.
template <class T, int W, class C, class V = T>
__global__ void __launch_bounds__(256) hell_kernel(size_t n, size_t pitch, int w_dyn, const C *__restrict__ ell_col, const EllShifts shift,
                                                    const V *__restrict__ ell_val, const int *__restrict__ tail_ptr,
                                                    const int *__restrict__ tail_col, const V *__restrict__ tail_val,
                                                    const T *__restrict__ x, T *y, T alpha, int append,
                                                    const int *__restrict__ row_ids, int prefetch_blocks) {
    if constexpr (std::is_same<C, EllClass>::value) {
        static_assert(std::is_same<T, V>::value, "row classes keep their table in the vector type");
        // Row classes: a row moves 17 bytes (class, x, y), too few for one row per thread to keep enough bytes in flight.
        // A thread takes kEllClassRows rows, a block apart, so at every sub-step a warp's lanes hold consecutive rows
        // (coalesced class bytes and y stores); rows past the end repeat row n-1 and store nothing.
        constexpr int R = kEllClassRows;
        const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
        if (threadIdx.x == 0 && prefetch_blocks > 0) {
            // The rows of the block prefetch_blocks ahead: their class bytes and the x window of the largest shift, the
            // first touch of its lines (the other slots read them again later, from L2).  HBM then streams while this
            // block's threads wait on their own loads.
            const long long f0 = ((long long)blockIdx.x + prefetch_blocks) * blockDim.x * R;
            if (f0 < (long long)n) {
                const long long f1 = min(f0 + (long long)blockDim.x * R, (long long)n);
                int dmax = shift.s[0];
#pragma unroll
                for (int j = 1; j < W; ++j) dmax = max(dmax, shift.s[j]);
                prefetch_l2(x, f0 + dmax, f1 + dmax, (long long)shift.x_max + 1, keep);
                prefetch_l2(ell_col, f0, f1, (long long)n, stream);
            }
        }
        const size_t i0 = (size_t)blockIdx.x * blockDim.x * R + threadIdx.x;
        if (i0 >= n) return;
        size_t rows[R]; T sum[R];
#pragma unroll
        for (int r = 0; r < R; ++r) rows[r] = min(i0 + (size_t)r * blockDim.x, n - 1);
        hell_class_rows<T, W, R>(rows, ell_col, shift, ell_val, tail_ptr, tail_col, tail_val, x, stream, keep, sum);
#pragma unroll
        for (int r = 0; r < R; ++r)
            if (i0 + (size_t)r * blockDim.x < n) store_y<T>(y, row_ids ? (size_t)row_ids[rows[r]] : rows[r], sum[r], alpha, append);
    } else {
        (void)prefetch_blocks;
        const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n) return;
        const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
        const T sum = hell_row_sum<T, W, C, V>(i, pitch, w_dyn, ell_col, shift, ell_val, tail_ptr, tail_col, tail_val, x, stream, keep);
        store_y<T>(y, row_ids ? (size_t)row_ids[i] : i, sum, alpha, append);
    }
}

// ---- several right-hand sides at once: SpMat * multivector (vexcl/multivector.hpp, operations.hpp:861-881) ------------
// The reference multiplies component by component and streams the matrix K times.  Here a row's columns and values are
// loaded once and used for K gathers / K sums: for configs[2] with K = 4 that is 41 (values + slot mask) + 4*16 = 105
// bytes per row instead of 4 * 57.  Per component the products are added in the same order as in hell_kernel (same bits).
template <int K> struct MultiPtr { const void *x[K]; void *y[K]; };

// Schedule: ptxas's default (about 40 registers, 6 blocks per SM) rather than a 64-register plan that issues all K*W
// gathers before the first product -- the bound here is occupancy, not instruction order.  Not re-measured on H100.
template <class T, int W, class C, int K>
__global__ void __launch_bounds__(256) hell_multi_kernel(size_t n, size_t pitch, int w_dyn, const C *__restrict__ ell_col, const EllShifts shift,
                                                          const T *__restrict__ ell_val, const int *__restrict__ tail_ptr,
                                                          const int *__restrict__ tail_col, const T *__restrict__ tail_val,
                                                          MultiPtr<K> mp, T alpha, int append, const int *__restrict__ row_ids, size_t y_offset) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    T sum[K];
#pragma unroll
    for (int k = 0; k < K; ++k) sum[k] = T(0);
    static_assert(W > 0 || !std::is_same<C, EllDiag>::value, "the diagonal encoding needs one shift per slot: unrolled widths only");
    if constexpr (std::is_same<C, EllClass>::value) {
        // row classes (hell_class_rows): the first component's gathers go out before the class byte is back; the
        // row's mask and values are then looked up once for all K components
        static_assert(W > 0 && W <= (int)kEllDiagMaxWidth, "row classes hold one slot mask byte: unrolled widths up to 8 only");
        const unsigned id = ldg_stream(ell_col + i, stream);
        T xv[W];
#pragma unroll
        for (int j = 0; j < W; ++j) xv[j] = ldg_keep(static_cast<const T *>(mp.x[0]) + ell_class_column(i, shift, j), keep);
        const unsigned m = ldg_table(reinterpret_cast<const unsigned char *>(ell_val) + id);
        T v[W];
#pragma unroll
        for (int j = 0; j < W; ++j) v[j] = ldg_table(ell_val + kEllClassHeader / sizeof(T) + id * W + j);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            if (k > 0) {
                const T *x = static_cast<const T *>(mp.x[k]);
#pragma unroll
                for (int j = 0; j < W; ++j) xv[j] = ldg_keep(x + ell_class_column(i, shift, j), keep);
            }
#pragma unroll
            for (int j = 0; j < W; ++j) if ((m >> j) & 1u) sum[k] = t_add<T>(sum[k], t_mul<T>(v[j], xv[j]));
        }
    } else {
        const unsigned mask = ell_row_mask(ell_col, i, stream);
        if (W > 0) {
            int c[W > 0 ? W : 1]; T v[W > 0 ? W : 1];
#pragma unroll
            for (int j = 0; j < W; ++j) { c[j] = ell_slot_column(ell_col, i, pitch, j, ell_shift_of(shift, j), mask, stream); v[j] = ldg_stream(ell_val + i + (size_t)j * pitch, stream); }
            // one component at a time (W gathers in flight, then that component's products), the order chosen over issuing
            // all K*W gathers first
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const T *x = static_cast<const T *>(mp.x[k]);
                T xv[W > 0 ? W : 1];
#pragma unroll
                for (int j = 0; j < W; ++j) xv[j] = (c[j] != -1) ? ldg_keep(x + c[j], keep) : T(0);
#pragma unroll
                for (int j = 0; j < W; ++j) if (c[j] != -1) sum[k] = t_add<T>(sum[k], t_mul<T>(v[j], xv[j]));
            }
        } else {
            for (int j = 0; j < w_dyn; ++j) {
                const int c = ell_slot_column(ell_col, i, pitch, j, shift.s[0], mask, stream);   // run-time widths: one shift for all slots (build())
                if (c != -1) {
                    const T v = ldg_stream(ell_val + i + (size_t)j * pitch, stream);
#pragma unroll
                    for (int k = 0; k < K; ++k) sum[k] = t_add<T>(sum[k], t_mul<T>(v, ldg_keep(static_cast<const T *>(mp.x[k]) + c, keep)));
                }
            }
        }
    }
    if (tail_ptr) {
        for (int j = tail_ptr[i], e = tail_ptr[i + 1]; j < e; ++j) {
            const T v = tail_val[j]; const int c = tail_col[j];
#pragma unroll
            for (int k = 0; k < K; ++k) sum[k] = t_add<T>(sum[k], t_mul<T>(v, __ldg(static_cast<const T *>(mp.x[k]) + c)));
        }
    }
    const size_t r = row_ids ? (size_t)row_ids[i] : i + y_offset;
#pragma unroll
    for (int k = 0; k < K; ++k) store_y<T>(static_cast<T *>(mp.y[k]), r, sum[k], alpha, append);
}

// spmv.kernel = 3: one thread per row straight from the CSR arrays ("CSR-scalar").  Neighbouring lanes read
// neighbouring rows, i.e. addresses a row length apart: not coalesced per instruction, but every 32-byte sector a warp
// touches is consumed completely by it over the row loop, so with L1 allocation (plain loads, no streaming hint) DRAM
// traffic stays at the algorithmic figure.  No shared memory, no barrier, no tile descriptor: every thread always has
// loads in flight, like hell_kernel.  V: stored value type, as in hell_kernel.
template <class T, class V = T>
__global__ void __launch_bounds__(256) csr_scalar_kernel(size_t n, const int *__restrict__ rowptr, const int *__restrict__ col,
                                                          const V *__restrict__ val, const T *__restrict__ x, T *y, T alpha,
                                                          int append, const int *__restrict__ row_ids) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    int j = rowptr[r];
    const int e = rowptr[r + 1];
    T sum = T(0);
    for (; j + 4 <= e; j += 4) {                                       // four gathers in flight, products in storage order
        const int c0 = col[j], c1 = col[j + 1], c2 = col[j + 2], c3 = col[j + 3];
        const T v0 = val[j], v1 = val[j + 1], v2 = val[j + 2], v3 = val[j + 3];
        const T x0 = __ldg(x + c0), x1 = __ldg(x + c1), x2 = __ldg(x + c2), x3 = __ldg(x + c3);
        sum = t_add<T>(sum, t_mul<T>(v0, x0)); sum = t_add<T>(sum, t_mul<T>(v1, x1));
        sum = t_add<T>(sum, t_mul<T>(v2, x2)); sum = t_add<T>(sum, t_mul<T>(v3, x3));
    }
    for (; j < e; ++j) sum = t_add<T>(sum, t_mul<T>(T(val[j]), __ldg(x + col[j])));
    store_y<T>(y, row_ids ? (size_t)row_ids[r] : r, sum, alpha, append);
}

// ---- warp tiles (spmv.kernel = 4) --------------------------------------------------------------------------------
// The row-block stream kernel again, but the unit of work is a WARP, not a CTA: rows are cut on the host into tiles of
// <= 256 nonzeros (8 per lane) and <= 256 rows; a warp loads its tile's col/val with coalesced 4/8-byte loads straight
// into registers (L1 no-allocate, L2 evict-first), gathers x (L2 evict-last), parks the products in its private 2 KB of
// shared memory and sums rows from there -- in storage order by one lane per row (short rows: same bits as the reference
// loop, csr.inl:163-170) or by groups of 4 / 8 / 32 lanes with a shuffle tree (longer rows).  There is no CTA-wide
// barrier and no mbarrier: warps drift apart, so the loads of one overlap the gathers and row sums of the others (the
// one-shot CTA kernel serialises load -> wait -> gather -> sum per CTA).  Warps are persistent and fetch the NEXT tile's
// descriptor while working on the
// current one, so the col/val loads never wait on a dependent descriptor load.
constexpr int kWarpTileNnz = 256;
constexpr int kWarpTileRows = 256;
constexpr int kWarpPer = kWarpTileNnz / 32;

// Row sums of one warp tile from the products parked in shared memory.  G lanes share a row (G = 1: one lane per row,
// storage order); pass p covers rows p*(32/G) .. ; the row pointers of the first two passes arrive preloaded (pa/pb), the
// rest are fetched here.
template <class T, int G>
__device__ __forceinline__ void warp_rows(const T *prod, const int *__restrict__ rowptr, int r0, int nr, int j0, int lane,
                                          const int (&pa)[2], const int (&pb)[2], T *y, T alpha, int append,
                                          const int *__restrict__ row_ids) {
    constexpr int RPW = 32 / G;                       // rows per warp pass
    const int sub = lane % G, grp = lane / G;
    int pass = 0;
    for (int rb = 0; rb < nr; rb += RPW, ++pass) {
        const int r = rb + grp;
        T s = T(0);
        if (r < nr) {
            int a, b;
            if (pass == 0) { a = pa[0]; b = pb[0]; } else if (pass == 1) { a = pa[1]; b = pb[1]; }
            else { a = __ldg(rowptr + r0 + r); b = __ldg(rowptr + r0 + r + 1); }
            a -= j0; b -= j0;
            for (int j = a + sub; j < b; j += G) s = t_add<T>(s, prod[j]);
        }
        if (G > 1) {
#pragma unroll
            for (int off = G / 2; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off, G));
        }
        if (r < nr && sub == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
    }
}

// lanes per row for a tile of cnt nonzeros in nr rows
__device__ __forceinline__ int warp_tile_group(int cnt, int nr) { return cnt <= 6 * nr ? 1 : cnt <= 24 * nr ? 4 : cnt <= 64 * nr ? 8 : 32; }

// V: stored value type, as in hell_kernel.  Float values under double vectors need more than the 64 registers of 4 CTAs
// per SM (88 bytes of spills): that instantiation runs 3.
template <class T, class V = T>
__global__ void __launch_bounds__(256, std::is_same<T, V>::value ? 4 : 3) csr_warp_kernel(const int2 *__restrict__ tile, int n_tiles, const int *__restrict__ rowptr,
                                                           const int *__restrict__ col, const V *__restrict__ val,
                                                           const T *__restrict__ x, T *y, T alpha, int append,
                                                           const int *__restrict__ row_ids) {
    __shared__ T prod_all[8][kWarpTileNnz];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T *prod = prod_all[warp];
    const int total_warps = gridDim.x * 8;
    int t = blockIdx.x * 8 + warp;
    if (t >= n_tiles) return;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();

    // Software pipeline over the tiles t, t + W, t + 2W, ... of this warp.  While the row sums of tile i are computed from
    // shared memory, the col/val/row-pointer loads of tile i+1 are already in flight (their registers are free again once
    // the products of tile i are parked), and the descriptor of tile i+2 is on its way.
    int2 d0 = __ldg(tile + t), d1 = __ldg(tile + t + 1);                 // current
    int2 n0 = d0, n1 = d1;                                               // next
    { const int tn = t + total_warps; if (tn < n_tiles) { n0 = __ldg(tile + tn); n1 = __ldg(tile + tn + 1); } }
    int c[kWarpPer]; V v[kWarpPer]; int pa[2], pb[2];
    auto issue = [&](const int2 &e0, const int2 &e1) {
        const int r0 = e0.x, nr = e1.x - e0.x, j0 = e0.y, cnt = e1.y - e0.y;
        if (cnt > kWarpTileNnz || nr <= 0) return;
#pragma unroll
        for (int k = 0; k < kWarpPer; ++k) {
            const int j = lane + 32 * k;
            if (j < cnt) { c[k] = ldg_stream(col + j0 + j, stream); v[k] = ldg_stream(val + j0 + j, stream); }
        }
        const int G = warp_tile_group(cnt, nr), rpw = 32 / G, grp = lane / G;
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int r = p * rpw + grp;
            if (r < nr) { pa[p] = __ldg(rowptr + r0 + r); pb[p] = __ldg(rowptr + r0 + r + 1); }
        }
    };
    issue(d0, d1);
    while (true) {
        const int tn = t + total_warps, tnn = tn + total_warps;
        const int r0 = d0.x, nr = d1.x - d0.x, j0 = d0.y, cnt = d1.y - d0.y;
        int2 m0 = n0, m1 = n1;                                           // descriptor after next
        if (tnn < n_tiles) { m0 = __ldg(tile + tnn); m1 = __ldg(tile + tnn + 1); }
        if (cnt > kWarpTileNnz) {
            // one long row: the warp strides over it
            T s = T(0);
            for (int j = j0 + lane; j < j0 + cnt; j += 32) s = t_add<T>(s, t_mul<T>(T(ldg_stream(val + j, stream)), ldg_keep(x + ldg_stream(col + j, stream), keep)));
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off));
            if (lane == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0] : (size_t)r0, s, alpha, append);
            if (tn < n_tiles) issue(n0, n1);
        } else if (nr > 0) {
            if constexpr (std::is_same<T, V>::value) {
#pragma unroll
                for (int k = 0; k < kWarpPer; ++k) {
                    const int j = lane + 32 * k;
                    if (j < cnt) v[k] = t_mul<T>(v[k], ldg_keep(x + c[k], keep));
                }
#pragma unroll
                for (int k = 0; k < kWarpPer; ++k) {
                    const int j = lane + 32 * k;
                    if (j < cnt) prod[j] = v[k];
                }
            } else {
                // float values under double vectors: the products cannot go back over the values, they go straight to
                // shared memory once all gathers are out (a third register array would spill)
                T xv[kWarpPer];
#pragma unroll
                for (int k = 0; k < kWarpPer; ++k) {
                    const int j = lane + 32 * k;
                    if (j < cnt) xv[k] = ldg_keep(x + c[k], keep);
                }
#pragma unroll
                for (int k = 0; k < kWarpPer; ++k) {
                    const int j = lane + 32 * k;
                    if (j < cnt) prod[j] = t_mul<T>(T(v[k]), xv[k]);
                }
            }
            const int qa[2] = {pa[0], pa[1]}, qb[2] = {pb[0], pb[1]};
            __syncwarp();
            if (tn < n_tiles) issue(n0, n1);                             // next tile's loads fly during the row sums below
            switch (warp_tile_group(cnt, nr)) {
                case 1:  warp_rows<T, 1>(prod, rowptr, r0, nr, j0, lane, qa, qb, y, alpha, append, row_ids); break;
                case 4:  warp_rows<T, 4>(prod, rowptr, r0, nr, j0, lane, qa, qb, y, alpha, append, row_ids); break;
                case 8:  warp_rows<T, 8>(prod, rowptr, r0, nr, j0, lane, qa, qb, y, alpha, append, row_ids); break;
                default: warp_rows<T, 32>(prod, rowptr, r0, nr, j0, lane, qa, qb, y, alpha, append, row_ids); break;
            }
            __syncwarp();
        } else if (tn < n_tiles) issue(n0, n1);
        if (tn >= n_tiles) break;
        t = tn; d0 = n0; d1 = n1; n0 = m0; n1 = m1;
    }
}

// ---- warp rings (spmv.kernel = 5) --------------------------------------------------------------------------------
// The warp-tile kernel with the matrix stream taken off the warps' critical path.  Each warp is a persistent worker with a
// private ring of `stages` shared-memory slots; lane 0 keeps stages-1 tiles ahead of the one being multiplied with TMA
// bulk copies (cp.async.bulk -> UBLKCP) of the tile's val, col and row-pointer slices, each ring slot completing on its
// own mbarrier.  While a warp waits for x gathers or adds up rows, its next tiles are already in flight -- the HBM stream
// no longer stops when a warp does (the register-staged warp tiles reach 0.57 of the roofline on the irregular matrix:
// a warp's loads are only in flight while that warp has nothing else to do).  There is no CTA-wide barrier anywhere:
// warps drift apart freely.  Products are parked in place (over the staged values), rows are added from there by 1 / 4 /
// 8 / 32 lanes per row exactly as in csr_warp_kernel, so the bits are the same.
constexpr int kRingSlots = kWarpTileNnz + 8;             // aligned window of a tile: <= 256 + 3 + 3 entries
constexpr int kRingRp = kWarpTileRows + 8;               // aligned window of its row pointers: <= 257 + 3 + 3 entries
template <class T> struct RingStage {
    static constexpr size_t val_bytes = (size_t)kRingSlots * sizeof(T);
    static constexpr size_t col_bytes = (size_t)kRingSlots * 4;
    static constexpr size_t rp_bytes = (size_t)kRingRp * 4;
    static constexpr size_t bytes = (val_bytes + col_bytes + rp_bytes + 127) & ~(size_t)127;
};

template <class T, int G>
__device__ __forceinline__ void ring_rows(const T *prod, const int *rp, int r0, int nr, int ja, int lane, T *y, T alpha,
                                          int append, const int *__restrict__ row_ids) {
    constexpr int RPW = 32 / G;
    const int sub = lane % G, grp = lane / G;
    for (int rb = 0; rb < nr; rb += RPW) {
        const int r = rb + grp;
        T s = T(0);
        if (r < nr) {
            const int a = rp[r] - ja, b = rp[r + 1] - ja;
            for (int j = a + sub; j < b; j += G) s = t_add<T>(s, prod[j]);
        }
        if (G > 1) {
#pragma unroll
            for (int off = G / 2; off > 0; off >>= 1) s = t_add<T>(s, __shfl_down_sync(0xffffffffu, s, off, G));
        }
        if (r < nr && sub == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, s, alpha, append);
    }
}

template <class T>
__global__ void __launch_bounds__(256, 3) csr_ring_kernel(const int2 *__restrict__ tile, int n_tiles, const int *__restrict__ rowptr,
                                                       const int *__restrict__ col, const T *__restrict__ val,
                                                       const T *__restrict__ x, T *y, T alpha, int append,
                                                       const int *__restrict__ row_ids, int stages) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    unsigned char *ring = smem + (size_t)warp * stages * RingStage<T>::bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + (size_t)nwarps * stages * RingStage<T>::bytes) + warp * stages;
    const int total_warps = gridDim.x * nwarps;
    const int t0 = blockIdx.x * nwarps + warp;
    if (t0 >= n_tiles) return;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    if (lane == 0) {
        for (int s = 0; s < stages; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(bars + s)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();

    // lane 0: start the copies of one tile into ring slot s (nothing to copy for a row longer than a tile)
    auto issue = [&](int2 e0, int2 e1, int s) {
        const int r0 = e0.x, nr = e1.x - e0.x, j0 = e0.y, cnt = e1.y - e0.y;
        if (cnt > kWarpTileNnz || nr <= 0 || cnt <= 0) return;
        const int ja = j0 & ~3, je = (j0 + cnt + 3) & ~3;
        const int ra = r0 & ~3, re = (r0 + nr + 1 + 3) & ~3;
        unsigned char *base = ring + (size_t)s * RingStage<T>::bytes;
        const uint32_t bv = (uint32_t)(je - ja) * (uint32_t)sizeof(T), bc = (uint32_t)(je - ja) * 4u, br = (uint32_t)(re - ra) * 4u;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bars + s)), "r"(bv + bc + br) : "memory");
        bulk_g2s(base, val + ja, bv, bars + s, stream);
        bulk_g2s(base + RingStage<T>::val_bytes, col + ja, bc, bars + s, stream);
        bulk_g2s(base + RingStage<T>::val_bytes + RingStage<T>::col_bytes, rowptr + ra, br, bars + s, stream);
    };
    auto desc = [&](int t, int2 &e0, int2 &e1) {
        if (t < n_tiles) { e0 = __ldg(tile + t); e1 = __ldg(tile + t + 1); } else { e0 = make_int2(0, 0); e1 = e0; }
    };

    // prologue: tiles 0 .. stages-2 of this warp go out; the descriptor of the tile to issue next is kept in registers
    int2 c0, c1, q0, q1;
    desc(t0, c0, c1);                                                   // current tile
    {
        int2 e0 = c0, e1 = c1;
        for (int k = 0; k < stages - 1; ++k) {
            const int t = t0 + k * total_warps;
            if (t >= n_tiles) break;
            if (k > 0) desc(t, e0, e1);
            if (lane == 0) issue(e0, e1, k);
        }
    }
    desc(t0 + (stages - 1) * total_warps, q0, q1);                      // next tile to issue
    unsigned phase = 0;                                                  // bit s: parity to wait for on ring slot s
    int it = 0;
    for (int t = t0; t < n_tiles; t += total_warps, ++it) {
        const int s = it % stages;
        // keep the ring full: the slot tile `it-1` just left takes tile `it + stages-1`
        {
            const int tq = t + (stages - 1) * total_warps;
            if (tq < n_tiles && lane == 0) issue(q0, q1, (it + stages - 1) % stages);
        }
        int2 n0, n1;
        desc(t + total_warps, n0, n1);                                  // next tile to multiply (already in flight)
        int2 m0, m1;
        desc(t + stages * total_warps, m0, m1);                         // tile to issue in the next iteration
        const int r0 = c0.x, nr = c1.x - c0.x, j0 = c0.y, cnt = c1.y - c0.y;
        if (cnt > kWarpTileNnz) {
            // one long row: the warp strides over it straight from global memory
            T sacc = T(0);
            for (int j = j0 + lane; j < j0 + cnt; j += 32) sacc = t_add<T>(sacc, t_mul<T>(ldg_stream(val + j, stream), ldg_keep(x + ldg_stream(col + j, stream), keep)));
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) sacc = t_add<T>(sacc, __shfl_down_sync(0xffffffffu, sacc, off));
            if (lane == 0) store_y<T>(y, row_ids ? (size_t)row_ids[r0] : (size_t)r0, sacc, alpha, append);
        } else if (nr > 0 && cnt <= 0) {
            // empty rows only
            for (int r = lane; r < nr; r += 32) store_y<T>(y, row_ids ? (size_t)row_ids[r0 + r] : (size_t)r0 + r, T(0), alpha, append);
        } else if (nr > 0) {
            mbar_wait(bars + s, (phase >> s) & 1u);
            phase ^= 1u << s;
            unsigned char *base = ring + (size_t)s * RingStage<T>::bytes;
            T *val_s = reinterpret_cast<T *>(base);
            const int *col_s = reinterpret_cast<const int *>(base + RingStage<T>::val_bytes);
            const int *rp_s = reinterpret_cast<const int *>(base + RingStage<T>::val_bytes + RingStage<T>::col_bytes);
            const int ja = j0 & ~3, lo = j0 - ja;
            T xv[kWarpPer];
#pragma unroll
            for (int k = 0; k < kWarpPer; ++k) {
                const int j = lane + 32 * k;
                xv[k] = (j < cnt) ? ldg_keep(x + col_s[lo + j], keep) : T(0);
            }
#pragma unroll
            for (int k = 0; k < kWarpPer; ++k) {
                const int j = lane + 32 * k;
                if (j < cnt) val_s[lo + j] = t_mul<T>(val_s[lo + j], xv[k]);
            }
            __syncwarp();
            const int *rp = rp_s + (r0 - (r0 & ~3));
            switch (warp_tile_group(cnt, nr)) {
                case 1:  ring_rows<T, 1>(val_s, rp, r0, nr, ja, lane, y, alpha, append, row_ids); break;
                case 4:  ring_rows<T, 4>(val_s, rp, r0, nr, ja, lane, y, alpha, append, row_ids); break;
                case 8:  ring_rows<T, 8>(val_s, rp, r0, nr, ja, lane, y, alpha, append, row_ids); break;
                default: ring_rows<T, 32>(val_s, rp, r0, nr, ja, lane, y, alpha, append, row_ids); break;
            }
            // the slot is reused by a bulk copy in the next iteration: order this warp's generic-proxy accesses before it
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        __syncwarp();
        c0 = n0; c1 = n1; q0 = m0; q1 = m1;
    }
}

// ---- sliced ELL (VEXB_FMT_SELL) ------------------------------------------------------------------------------------
// Irregular rows: hybrid ELL pads (or spills into its CSR tail), and every CSR kernel above either reads col/val
// uncoalesced (thread per row) or stages products through shared memory, which shares the L1 data pipe with the x
// gathers, so on irregular matrices that pipe, not DRAM, is the limit.  SELL-32-sigma keeps hybrid ELL's access pattern
// (a warp's loads of a slot are 32
// consecutive entries; one lane per row, sum in a register, no shared memory) without its padding: slices of 32 rows are
// as wide as THEIR longest row, and rows are sorted by length inside windows of sigma rows first, so a slice's rows are
// nearly equally long.  Products are added in storage order: same bits as the reference loop (csr.inl:163-170).
// C = short: a stored column is its distance from (the lane's row + shift), -32768 = padding (banded strips: 10 instead
// of 12 bytes per slot); C = int: the column itself, -1 = padding.  V: stored value type, as in hell_kernel.
template <class T, class C, class V = T>
__global__ void __launch_bounds__(256) sell_kernel(size_t n_slices, const int *__restrict__ slice_ptr, const int *__restrict__ perm,
                                                   const C *__restrict__ col, int shift, const V *__restrict__ val,
                                                   const T *__restrict__ x, T *y, T alpha, int append,
                                                   const int *__restrict__ row_ids, size_t y_offset) {
    const size_t s = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (s >= n_slices) return;
    const int lane = threadIdx.x & 31;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    const int base = __ldg(slice_ptr + s), w = (__ldg(slice_ptr + s + 1) - base) >> 5;
    const int r = ldg_stream(perm + s * 32 + lane, stream);
    const C *cp = col + base + lane;
    const V *vp = val + base + lane;
    const size_t rr = r >= 0 ? (size_t)r : 0;
    T sum = T(0);
    int k = 0;
    for (; k + 4 <= w; k += 4) {                          // 4 slots: 8 coalesced loads, then 4 gathers, in flight together
        int c[4]; V v[4]; T xv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { c[u] = ell_column(ldg_stream(cp + (k + u) * 32, stream), rr, shift); v[u] = ldg_stream(vp + (k + u) * 32, stream); }
#pragma unroll
        for (int u = 0; u < 4; ++u) xv[u] = c[u] != -1 ? ldg_keep(x + c[u], keep) : T(0);
#pragma unroll
        for (int u = 0; u < 4; ++u) if (c[u] != -1) sum = t_add<T>(sum, t_mul<T>(T(v[u]), xv[u]));
    }
    for (; k < w; ++k) {
        const int c = ell_column(ldg_stream(cp + k * 32, stream), rr, shift);
        const T v = ldg_stream(vp + k * 32, stream);
        if (c != -1) sum = t_add<T>(sum, t_mul<T>(v, ldg_keep(x + c, keep)));
    }
    if (r >= 0) store_y<T>(y, row_ids ? (size_t)row_ids[r] : (size_t)r + y_offset, sum, alpha, append);
}

// K right-hand sides in one pass over a sliced-ELL strip (SpMat * multivector): sell_kernel's decomposition, a slot's
// column and value loaded once and used for K gathers and K sums.  Per component the products are added in storage
// order, as in sell_kernel on that component alone (same bits).
template <class T, class C, int K>
__global__ void __launch_bounds__(256) sell_multi_kernel(size_t n_slices, const int *__restrict__ slice_ptr, const int *__restrict__ perm,
                                                         const C *__restrict__ col, int shift, const T *__restrict__ val,
                                                         MultiPtr<K> mp, T alpha, int append,
                                                         const int *__restrict__ row_ids, size_t y_offset) {
    const size_t s = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (s >= n_slices) return;
    const int lane = threadIdx.x & 31;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    const int base = __ldg(slice_ptr + s), w = (__ldg(slice_ptr + s + 1) - base) >> 5;
    const int r = ldg_stream(perm + s * 32 + lane, stream);
    const C *cp = col + base + lane;
    const T *vp = val + base + lane;
    const size_t rr = r >= 0 ? (size_t)r : 0;
    T sum[K];
#pragma unroll
    for (int q = 0; q < K; ++q) sum[q] = T(0);
    int k = 0;
    for (; k + 4 <= w; k += 4) {                          // 4 slots: 8 coalesced loads, then 4 K gathers
        int c[4]; T v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { c[u] = ell_column(ldg_stream(cp + (k + u) * 32, stream), rr, shift); v[u] = ldg_stream(vp + (k + u) * 32, stream); }
        T xv[K][4];
#pragma unroll
        for (int q = 0; q < K; ++q)
#pragma unroll
            for (int u = 0; u < 4; ++u) xv[q][u] = c[u] != -1 ? ldg_keep(static_cast<const T *>(mp.x[q]) + c[u], keep) : T(0);
#pragma unroll
        for (int q = 0; q < K; ++q)
#pragma unroll
            for (int u = 0; u < 4; ++u) if (c[u] != -1) sum[q] = t_add<T>(sum[q], t_mul<T>(v[u], xv[q][u]));
    }
    for (; k < w; ++k) {
        const int c = ell_column(ldg_stream(cp + k * 32, stream), rr, shift);
        const T v = ldg_stream(vp + k * 32, stream);
        if (c != -1) {
#pragma unroll
            for (int q = 0; q < K; ++q) sum[q] = t_add<T>(sum[q], t_mul<T>(v, ldg_keep(static_cast<const T *>(mp.x[q]) + c, keep)));
        }
    }
    if (r < 0) return;
    const size_t yr = row_ids ? (size_t)row_ids[r] : (size_t)r + y_offset;
#pragma unroll
    for (int q = 0; q < K; ++q) store_y<T>(static_cast<T *>(mp.y[q]), yr, sum[q], alpha, append);
}

template <class T>
__global__ void zero_rows_kernel(T *y, size_t n, const int *__restrict__ row_ids) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[row_ids ? (size_t)row_ids[i] : i] = T(0);
}

template <class T>
static int upload(std::vector<T> &h, size_t pad, void **d, size_t *bytes_acc) {
    const size_t n = h.size() + pad;
    *d = nullptr;
    if (n == 0) return VEXB_OK;
    VEXB_CUDA(cudaMalloc(d, n * sizeof(T)));
    if (pad) VEXB_CUDA(cudaMemset((char *)*d + h.size() * sizeof(T), 0, pad * sizeof(T)));
    if (!h.empty()) VEXB_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    *bytes_acc += n * sizeof(T);
    return VEXB_OK;
}

// A per-entry value array of the strip: as built, or as float on VEXB_FMT_VALUES_F32 strips (exact: the values were
// rounded to float by check_fmt_flags).
template <class T>
static int upload_values(vexb_spmat *A, std::vector<T> &h, size_t pad, void **d) {
    if (!A->val_f32) return upload(h, pad, d, &A->device_bytes);
    std::vector<float> f(h.begin(), h.end());
    return upload(f, pad, d, &A->device_bytes);
}

// Width of the ELL part: smallest w such that the rows wider than w are fewer
// than n/3 (ELL assumed 3x faster than CSR; hybrid_ell.inl:66-113).
static size_t hell_width(const std::vector<int> &rowptr, size_t n) {
    size_t maxw = 0;
    for (size_t i = 0; i < n; ++i) maxw = std::max(maxw, (size_t)(rowptr[i + 1] - rowptr[i]));
    std::vector<size_t> hist(maxw + 1, 0);
    for (size_t i = 0; i < n; ++i) ++hist[rowptr[i + 1] - rowptr[i]];
    size_t rows = n;
    for (size_t w = 0; w < maxw; ++w) {
        rows -= hist[w];                 // rows wider than w
        if (3.0 * rows < n) return w;
    }
    return maxw;
}

// Row patterns: many PDE matrices repeat a handful of rows (same column offsets from the diagonal, same values).  Such
// a strip is stored as the unique rows plus ONE BYTE per row naming its pattern -- the reference's CCSR format
// (spmat/ccsr.hpp), found automatically -- and multiplied by ccsr_kernel: 17 B/row of compulsory traffic for a 5-point
// stencil instead of 76 B/row in hybrid ELL.  Values are compared bit for bit and rows are accumulated in storage
// order, so the product has the same bits as the ELL / CSR kernels.  Returns false when the strip has more than
// `max_patterns` distinct rows.
template <class T>
static bool find_row_patterns(size_t n, const std::vector<int> &rowptr, const std::vector<int> &col, const std::vector<T> &val,
                              size_t max_patterns, std::vector<int> &idx, std::vector<int> &prow, std::vector<int> &pcol,
                              std::vector<T> &pval) {
    idx.assign(n, 0); prow.assign(1, 0); pcol.clear(); pval.clear();
    std::unordered_map<std::string, int> seen;
    std::string key;
    int last = -1;
    for (size_t i = 0; i < n; ++i) {
        const int b = rowptr[i], w = rowptr[i + 1] - b;
        if (last >= 0 && prow[last + 1] - prow[last] == w) {           // most rows repeat the previous row's pattern
            const int q = prow[last];
            bool same = true;
            for (int j = 0; j < w && same; ++j)
                same = (col[b + j] - (int)i == pcol[q + j]) && std::memcmp(&val[b + j], &pval[q + j], sizeof(T)) == 0;
            if (same) { idx[i] = last; continue; }
        }
        key.resize((size_t)w * (sizeof(int) + sizeof(T)));
        for (int j = 0; j < w; ++j) {
            const int rel = col[b + j] - (int)i;
            std::memcpy(&key[(size_t)j * sizeof(int)], &rel, sizeof(int));
            std::memcpy(&key[(size_t)w * sizeof(int) + (size_t)j * sizeof(T)], &val[b + j], sizeof(T));
        }
        auto it = seen.find(key);
        if (it == seen.end()) {
            if (prow.size() - 1 >= max_patterns) return false;
            const int id = (int)prow.size() - 1;
            for (int j = 0; j < w; ++j) { pcol.push_back(col[b + j] - (int)i); pval.push_back(val[b + j]); }
            prow.push_back((int)pcol.size());
            it = seen.emplace(key, id).first;
        }
        idx[i] = last = it->second;
    }
    return true;
}

// Row classes of a slot-mask strip (spmv.ell_classes): the distinct (slot mask, W slot values) tuples of its `pitch`
// stored rows -- padding rows included, which give the mask-0 tuple -- numbered in order of first appearance.  Fills
// id (one class per row) and the class table as the kernels read it (kEllClassHeader bytes of masks, then W values per
// class), and returns the number of classes; 0 when there are more than kEllMaxClasses.  Values are compared bit for bit.
template <class T>
static size_t ell_row_classes(size_t pitch, size_t w, const std::vector<EllDiag> &mask, const std::vector<T> &eval,
                              std::vector<unsigned char> &id, std::vector<unsigned char> &table) {
    const size_t tb = w * sizeof(T);
    id.assign(pitch, 0); table.assign(kEllClassHeader, 0);
    std::unordered_map<std::string, int> seen;
    std::string key(1 + tb, '\0');
    int last = -1;
    for (size_t i = 0; i < pitch; ++i) {
        key[0] = (char)mask[i].mask;
        for (size_t k = 0; k < w; ++k) std::memcpy(&key[1 + k * sizeof(T)], &eval[i + pitch * k], sizeof(T));
        if (last >= 0 && table[last] == (unsigned char)key[0] &&                      // most rows repeat the previous row's class
            std::memcmp(&table[kEllClassHeader + (size_t)last * tb], &key[1], tb) == 0) { id[i] = (unsigned char)last; continue; }
        auto it = seen.find(key);
        if (it == seen.end()) {
            if (seen.size() == kEllMaxClasses) return 0;
            const int c = (int)seen.size();
            table[c] = (unsigned char)key[0];
            table.insert(table.end(), key.begin() + 1, key.end());
            it = seen.emplace(key, c).first;
        }
        id[i] = (unsigned char)(last = it->second);
    }
    return seen.size();
}

template <class T>
static int build(vexb_spmat *A, std::vector<int> &rowptr, std::vector<int> &col, std::vector<T> &val, int fmt, bool plain) {
    const size_t n = A->nrows_stored;
    if (fmt == VEXB_FMT_AUTO && param("spmv.auto_patterns", 0)) fmt = VEXB_FMT_PATTERNS;   // off until measured (DESIGN.md section 7)
    if (fmt == VEXB_FMT_PATTERNS) {
        // only for strips whose stored row r is row r of y (no row map) and that are worth it; otherwise as AUTO
        std::vector<int> idx, prow, pcol; std::vector<T> pval;
        const size_t limit = (size_t)std::max(1l, std::min(param("spmv.max_patterns", 256), 65536l));
        if (plain && n > 0 && A->nnz > 0 && find_row_patterns<T>(n, rowptr, col, val, limit, idx, prow, pcol, pval)) {
            // a strip the CCSR kernel cannot take (e.g. too many entries in the unique-row table) is simply not compressed
            if (ccsr_create_ex(A->dev, n, A->ncols, prow.size() - 1, idx.data(), 4, prow.data(), 4, pcol.data(), 4, pval.data(),
                               A->val_dtype, &A->patterns) == VEXB_OK) {
                A->fmt = VEXB_FMT_PATTERNS;
                A->n_patterns = prow.size() - 1;
                A->val_f32 = false;                                     // the unique-row table stays double
                return VEXB_OK;
            }
            A->patterns = nullptr;
        }
        fmt = VEXB_FMT_AUTO;
    }
    if (fmt == VEXB_FMT_AUTO) {
        // As the reference does on GPUs (spmat.hpp:98-103): hybrid ELL, which streams coalesced slots where the CSR
        // kernels stage or read uncoalesced, so it is kept even with some padding; only when the
        // padded storage would exceed 3x the nonzeros (a few very long rows among many short ones are
        // already caught by the CSR tail) does the CSR stream kernel take over.
        const size_t w = hell_width(rowptr, n);
        size_t tail = 0;
        for (size_t i = 0; i < n; ++i) { const size_t rw = rowptr[i + 1] - rowptr[i]; if (rw > w) tail += rw - w; }
        const double padded = (double)w * (double)((n + 15) / 16 * 16) + (double)tail;
        // regular rows: hybrid ELL; rows too uneven for it (more than a quarter of the stored slots would be padding or
        // tail): sliced ELL, which keeps the access pattern and drops the padding (spmv.auto_sell = 0: round-1 rule)
        if (A->nnz == 0) fmt = VEXB_FMT_CSR;
        else if (padded <= 1.25 * (double)A->nnz && tail * 20 <= A->nnz) fmt = VEXB_FMT_HELL;
        else if (param("spmv.auto_sell", 1)) fmt = VEXB_FMT_SELL;
        else fmt = padded <= 3.0 * (double)A->nnz ? VEXB_FMT_HELL : VEXB_FMT_CSR;
    }
    A->fmt = fmt;
    if (fmt == VEXB_FMT_SELL) {
        std::vector<int> perm, sptr;
        size_t slots = 0;
        if (!sell_layout(n, rowptr.data(), param("spmv.sell_sigma", 1024), perm, sptr, &slots)) {
            set_error(__FILE__, __LINE__, "strip too large for sliced ELL");
            return VEXB_ERR_UNSUPPORTED;
        }
        const size_t ns = sptr.size() - 1;
        std::vector<int> scol(slots, -1);
        std::vector<T> sval(slots, T(0));
        for (size_t sl = 0; sl < ns; ++sl)
            for (int l = 0; l < 32; ++l) {
                const int r = perm[sl * 32 + l];
                if (r < 0) continue;
                for (int j = rowptr[r], k = 0; j < rowptr[r + 1]; ++j, ++k) {
                    scol[(size_t)sptr[sl] + (size_t)k * 32 + l] = col[j];
                    sval[(size_t)sptr[sl] + (size_t)k * 32 + l] = val[j];
                }
            }
        A->n_slices = ns; A->sell_slots = slots;
        VEXB_TRY(upload(sptr, 0, (void **)&A->sell_ptr, &A->device_bytes));
        VEXB_TRY(upload(perm, 0, (void **)&A->sell_perm, &A->device_bytes));
        bool narrow = false;
        if (param("spmv.col16", 1) && A->nnz > 0) {
            // banded strips: every column within +-32767 of (its row + one shift) -> 16-bit columns, as for hybrid ELL
            long long lo = 0, hi = 0; bool any = false;
            for (size_t i = 0; i < n; ++i)
                for (int j = rowptr[i]; j < rowptr[i + 1]; ++j) {
                    const long long d = (long long)col[j] - (long long)i;
                    if (!any) { lo = hi = d; any = true; } else { lo = std::min(lo, d); hi = std::max(hi, d); }
                }
            if (any && hi - lo <= 65534) {
                const long long shift = lo + 32767;
                std::vector<short> s16(slots, (short)-32768);
                for (size_t sl = 0; sl < ns; ++sl)
                    for (int l = 0; l < 32; ++l) {
                        const int r = perm[sl * 32 + l];
                        if (r < 0) continue;
                        for (int j = rowptr[r], k = 0; j < rowptr[r + 1]; ++j, ++k)
                            s16[(size_t)sptr[sl] + (size_t)k * 32 + l] = (short)((long long)col[j] - (long long)r - shift);
                    }
                A->sell_shift = (int)shift;
                VEXB_TRY(upload(s16, 32, (void **)&A->sell_col16, &A->device_bytes));
                narrow = true;
            }
        }
        if (!narrow) VEXB_TRY(upload(scol, 32, (void **)&A->sell_col, &A->device_bytes));
        VEXB_TRY(upload_values(A, sval, 32, &A->sell_val));
        return VEXB_OK;
    }
    if (fmt == VEXB_FMT_CSR) {
        long tn = param("spmv.tile_nnz", 2048), tr = param("spmv.tile_rows", 512);
        tn = std::max(64l, std::min(tn, 8192l)) & ~3l;
        tr = std::max(32l, std::min(tr, 4096l)) & ~3l;
        A->tile_nnz = tn; A->tile_rows = tr;
        std::vector<int2> tiles;
        size_t r = 0;
        while (r < n) {
            size_t e = r; const int j0 = rowptr[r];
            while (e < n && e - r < (size_t)tr && rowptr[e + 1] - j0 <= tn) ++e;
            if (e == r) e = r + 1;        // a single row longer than a tile
            tiles.push_back(make_int2((int)r, j0));
            r = e;
        }
        tiles.push_back(make_int2((int)n, rowptr[n]));
        A->n_tiles = tiles.size() - 1;
        VEXB_TRY(upload(tiles, 0, (void **)&A->tile, &A->device_bytes));
        // x window of every tile for csr_window_kernel: columns [cmin, cmax] of its nonzeros, start aligned down to 16
        // bytes (bulk copy), length rounded up likewise; {0, 0} when it exceeds spmv.xwin entries or would pass the end of x
        {
            long xw = param("spmv.xwin", 2048);
            xw = std::max(64l, std::min(xw, 8192l)) & ~3l;
            A->xwin = (size_t)xw;
            std::vector<int2> tx(A->n_tiles, make_int2(0, 0));
            size_t windowed = 0;
            for (size_t t = 0; t < A->n_tiles; ++t) {
                const int a = tiles[t].y, b = tiles[t + 1].y;
                if (b <= a || b - a > tn) continue;
                int cmin = col[a], cmax = col[a];
                for (int j = a + 1; j < b; ++j) { cmin = std::min(cmin, col[j]); cmax = std::max(cmax, col[j]); }
                const int G = (int)(16 / sizeof(T));                   // bulk copies move multiples of 16 bytes from 16-byte aligned addresses
                const int c0 = cmin & ~(G - 1);
                const int len = (cmax - c0 + 1 + G - 1) & ~(G - 1);
                if (len <= xw && (size_t)c0 + (size_t)len <= A->ncols) { tx[t] = make_int2(c0, len); ++windowed; }   // never past the end of x
            }
            A->n_windowed_tiles = windowed;
            VEXB_TRY(upload(tx, 0, (void **)&A->tile_x, &A->device_bytes));
        }
        // warp tiles for csr_warp_kernel: <= 256 nnz and <= 256 rows, cut at row boundaries; a longer row is its own tile
        std::vector<int2> wt;
        size_t maxw = 0;
        for (r = 0; r < n;) {
            size_t e = r; const int j0 = rowptr[r];
            while (e < n && e - r < (size_t)kWarpTileRows && rowptr[e + 1] - j0 <= kWarpTileNnz) ++e;
            if (e == r) e = r + 1;
            wt.push_back(make_int2((int)r, j0));
            r = e;
        }
        wt.push_back(make_int2((int)n, rowptr[n]));
        for (size_t i = 0; i < n; ++i) maxw = std::max(maxw, (size_t)(rowptr[i + 1] - rowptr[i]));
        A->n_wtiles = wt.size() - 1; A->max_row_nnz = maxw;
        VEXB_TRY(upload(wt, 0, (void **)&A->wtile, &A->device_bytes));
        // Kernel for this strip unless spmv.kernel says otherwise.  Short, even rows (max <= 2 x mean, mean <= 8): one
        // thread per row straight from the CSR arrays (csr_scalar_kernel) -- every lane always has loads in flight and the
        // sectors a warp touches are used up within a few iterations.  Anything else: warp tiles, which keep col/val
        // coalesced where thread per row would not.
        const double mean = n ? (double)A->nnz / (double)n : 0.0;
        A->csr_variant = (mean <= 8.0 && (double)maxw <= 2.0 * mean + 2.0) ? 3 : 4;
        // CTA tiles with the x window in shared memory stay opt-in (spmv.kernel = 6 or spmv.auto_window = 1): the
        // one-shot CTA (copy, wait, multiply, add up) costs more than the L1 tag lookups it saves
        // (float-valued strips: 3 and 4 only)
        if (A->csr_variant == 4 && !A->val_f32 && param("spmv.auto_window", 0) && A->n_windowed_tiles * 10 >= A->n_tiles * 9) A->csr_variant = 6;
        VEXB_TRY(upload(rowptr, 16, (void **)&A->rowptr, &A->device_bytes));
        VEXB_TRY(upload(col, 16, (void **)&A->col, &A->device_bytes));
        VEXB_TRY(upload_values(A, val, 16, &A->val));
    } else {
        const size_t w = hell_width(rowptr, n);
        const size_t pitch = (n + 15) / 16 * 16;            // alignup(n, 16): hybrid_ell.inl:60
        A->ell_width = w; A->ell_pitch = pitch;
        std::vector<int> ecol(pitch * w, -1);               // sentinel (col_t)(-1): hybrid_ell.inl:139
        std::vector<T> eval(pitch * w, T(0));
        std::vector<int> tptr(n + 1, 0), tcol; std::vector<T> tval;
        // Slot alignment.  The reference packs a row's entries into slots 0, 1, ... (hybrid_ell.inl:139-144).  A row with
        // fewer than w entries may keep them in ANY increasing sequence of slots -- the kernels walk the slots in order and
        // skip padding, so the products are still added in storage order and y has the same bits.  Short rows (grid
        // boundaries: an identity row, a stencil with a neighbour missing) are therefore placed so that each entry
        // lands in the slot where full rows keep the entry at the same distance from the diagonal.  Every slot then
        // holds ONE distance on a structured grid, whatever the grid size, which is what lets the 16-bit column
        // encoding below (one shift per slot) cover 7-point stencils on 256^3 and 512^3 points: 10 instead of 12 bytes per
        // stored entry.  vexb_spmat_hell_download compacts rows to the left again (the reference's packing).
        std::vector<long long> ref(w, 0);
        bool have_ref = false;
        if (param("spmv.slot_align", 1)) {
            for (size_t i = 0; i < n && !have_ref; ++i)
                if ((size_t)(rowptr[i + 1] - rowptr[i]) >= w && w > 0) {
                    for (size_t k = 0; k < w; ++k) ref[k] = (long long)col[rowptr[i] + k] - (long long)i;
                    have_ref = true;
                }
        }
        for (size_t i = 0; i < n; ++i) {
            const int b = rowptr[i], cnt = rowptr[i + 1] - b;
            if (have_ref && cnt > 0 && (size_t)cnt < w) {
                size_t s0 = 0;
                for (int q = 0; q < cnt; ++q) {
                    const long long d = (long long)col[b + q] - (long long)i;
                    const size_t last = w - (size_t)(cnt - q);        // latest slot that leaves room for the entries after this one
                    size_t t = s0;
                    bool found = false;
                    for (size_t c = s0; c <= last && !found; ++c) if (ref[c] == d) { t = c; found = true; }
                    for (size_t c = s0; c <= last && !found; ++c) if (std::llabs(ref[c] - d) <= 16384) { t = c; found = true; }
                    ecol[i + pitch * t] = col[b + q]; eval[i + pitch * t] = val[b + q];
                    s0 = t + 1;
                }
            } else {
                size_t cntw = 0;
                for (int j = b; j < rowptr[i + 1]; ++j) {
                    if (cntw < w) { ecol[i + pitch * cntw] = col[j]; eval[i + pitch * cntw] = val[j]; ++cntw; }
                    else { tcol.push_back(col[j]); tval.push_back(val[j]); }
                }
            }
            tptr[i + 1] = (int)tcol.size();
        }
        A->tail_nnz = tcol.size();
        if (param("spmv.col16", 1) && w > 0) {
            // Banded matrices: the stored columns of ELL slot k lie within +-32767 of (row + shift[k]) for one shift per
            // slot, so the ELL columns fit 16 bits.  The kernel then streams 10 instead of 12 bytes per stored entry; same
            // bits in y, only the index encoding differs.  One shift per slot (not per strip) is what admits stencils
            // on 3-D grids: the k-th neighbour of every row is the same distance away (+-n*n for a 7-point stencil on
            // n^3 points), whatever that distance is.  Strips wider than kEllShiftSlots share the last shift among the
            // remaining slots.  spmv.col16 = 0 keeps 32-bit columns (and no slot masks either).
            std::vector<long long> lo(kEllShiftSlots, 0), hi(kEllShiftSlots, 0);
            std::vector<char> any(kEllShiftSlots, 0);
            // Widths without an unrolled instantiation in every kernel run the kernels' run-time loop over the slots, which
            // cannot index the by-value shift table without spilling it to local memory: such strips use ONE shift for
            // all slots (g = 0 for every slot).
            const bool per_slot = ell_width_is_unrolled_everywhere(w);
            for (size_t k = 0; k < w; ++k) {
                const size_t g = per_slot ? std::min<size_t>(k, kEllShiftSlots - 1) : 0;
                for (size_t i = 0; i < n; ++i) {
                    const int c = ecol[i + pitch * k];
                    if (c < 0) continue;
                    const long long d = (long long)c - (long long)i;
                    if (!any[g]) { lo[g] = hi[g] = d; any[g] = 1; } else { lo[g] = std::min(lo[g], d); hi[g] = std::max(hi[g], d); }
                }
            }
            bool fits = false, ok = true, diag = per_slot && w <= kEllDiagMaxWidth && param("spmv.ell_diag", 1);
            for (int g = 0; g < kEllShiftSlots; ++g) if (any[g]) { fits = true; if (hi[g] - lo[g] > 65534) ok = false; if (hi[g] != lo[g]) diag = false; }
            if (fits && diag) {
                // Every entry of slot k is exactly lo[k] from its row (a structured grid after slot alignment): the column
                // array carries no information beyond which slots are padding.  Store that as one mask byte per row and
                // the distances themselves as the shifts: 8 + 1/w instead of 10 bytes per stored entry, same bits in y.
                // spmv.ell_diag = 0 stops at 16-bit columns.
                EllShifts sh{};
                for (int g = 0; g < kEllShiftSlots; ++g) sh.s[g] = any[g] ? (int)lo[g] : 0;
                std::vector<EllDiag> mask(pitch, EllDiag{0});
                for (size_t k = 0; k < w; ++k)
                    for (size_t i = 0; i < n; ++i)
                        if (ecol[i + pitch * k] >= 0) mask[i].mask |= (unsigned char)(1u << k);
                A->ell_shifts = sh;
                // Row classes: a constant-coefficient stencil has a handful of distinct rows (2 on a 5-point Laplacian:
                // interior and identity), so one class byte per row and a small table of masks and values replace the
                // masks and the W values per row -- 17 instead of 57 bytes per row of configs[2] moved by a product.
                // spmv.ell_classes: 0 = never, 1 (default) = when the values would exceed the L2, 2 = at any size.
                // Smaller strips keep slot masks and their stored layout (DESIGN.md section 3 has the measurement
                // below the floor).
                const long classes = param("spmv.ell_classes", 1);
                int l2 = 0;
                if (classes == 1) VEXB_CUDA(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, A->dev));
                std::vector<unsigned char> cid, ctab;
                if ((classes == 2 || (classes == 1 && eval.size() * sizeof(T) > (size_t)l2)) &&
                    (A->ell_nclass = ell_row_classes(pitch, w, mask, eval, cid, ctab)) > 0) {
                    // padding slots gather x at a column clamped to the strip's largest one (ell_class_column)
                    A->ell_shifts.x_max = *std::max_element(ecol.begin(), ecol.end());
                    A->val_f32 = false;                         // the class table and the CSR tail stay double
                    VEXB_TRY(upload(cid, 0, (void **)&A->ell_class, &A->device_bytes));
                    VEXB_TRY(upload(ctab, 0, &A->ell_ctab, &A->device_bytes));
                } else {
                    VEXB_TRY(upload(mask, 0, (void **)&A->ell_mask, &A->device_bytes));
                }
            } else if (fits && ok) {
                EllShifts sh{};
                for (int g = 0; g < kEllShiftSlots; ++g) sh.s[g] = any[per_slot ? g : 0] ? (int)(lo[per_slot ? g : 0] + 32767) : 0;
                std::vector<short> e16(pitch * w, (short)-32768);
                for (size_t k = 0; k < w; ++k) {
                    const long long shift = sh.s[std::min<size_t>(k, kEllShiftSlots - 1)];
                    for (size_t i = 0; i < n; ++i) {
                        const int c = ecol[i + pitch * k];
                        if (c >= 0) e16[i + pitch * k] = (short)((long long)c - (long long)i - shift);
                    }
                }
                A->ell_shifts = sh;
                VEXB_TRY(upload(e16, 0, (void **)&A->ell_col16, &A->device_bytes));
            }
        }
        if (!A->ell_col16 && !A->ell_mask && !A->ell_class) VEXB_TRY(upload(ecol, 0, (void **)&A->ell_col, &A->device_bytes));
        if (!A->ell_class) VEXB_TRY(upload_values(A, eval, 0, &A->ell_val));
        if (A->tail_nnz) {
            VEXB_TRY(upload(tptr, 0, (void **)&A->tail_ptr, &A->device_bytes));
            VEXB_TRY(upload(tcol, 0, (void **)&A->tail_col, &A->device_bytes));
            VEXB_TRY(upload_values(A, tval, 0, &A->tail_val));
        }
    }
    return VEXB_OK;
}

// V: stored value type of the per-entry value arrays (float on VEXB_FMT_VALUES_F32 strips under double vectors).  Such
// strips are sliced ELL, hybrid ELL without row classes, or CSR run by variant 3 or 4: the other kernels are only ever
// launched with V = T.
template <class T, class V = T>
static int spmv_launch(const vexb_spmat *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    // A strip touches exactly its stored rows: all of y[0, nrows) normally, y[row_ids[r]] for a
    // row-compressed strip, y[y_offset + r] for a strip that covers a contiguous sub-range.
    const size_t n = A->nrows_stored;
    if (n == 0) return VEXB_OK;
    y += A->y_offset;
    if (A->nnz == 0) {
        // y = A*x with an empty strip must still zero y (csr.inl:195-200)
        if (!append) { zero_rows_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(y, n, A->row_ids); VEXB_LAUNCHED(); }
        return VEXB_OK;
    }
    if (A->fmt == VEXB_FMT_PATTERNS) return vexb_ccsr_spmv(A->dev, (void *)st, A->patterns, x, y, (double)alpha, append);
    if (A->fmt == VEXB_FMT_SELL) {
        // y was advanced by y_offset above; the kernel adds nothing more
        const unsigned sb = (unsigned)((A->n_slices + 7) / 8);
        if (A->sell_col16) sell_kernel<T, short, V><<<sb, 256, 0, st>>>(A->n_slices, A->sell_ptr, A->sell_perm, A->sell_col16, A->sell_shift, (const V *)A->sell_val,
                                                                      x, y, alpha, append, A->row_ids, 0);
        else sell_kernel<T, int, V><<<sb, 256, 0, st>>>(A->n_slices, A->sell_ptr, A->sell_perm, A->sell_col, 0, (const V *)A->sell_val,
                                                      x, y, alpha, append, A->row_ids, 0);
        VEXB_LAUNCHED();
        return VEXB_OK;
    }
    // spmv.kernel: 0 = TMA-staged one-shot CTA tiles, 1 = persistent TMA pipeline, 2 = register-staged CTA tiles, 3 = thread per row,
    //              4 = warp tiles, 5 = warp rings (TMA), 6 = CTA tiles with the x window in shared memory; unset (-1) = the strip's own choice (build(): 3 for short even rows, else 4)
    long variant = param("spmv.kernel", param("spmv.pipeline", 0) ? 1 : -1);
    if (variant < 0) variant = A->csr_variant;
    if (!std::is_same<T, V>::value && A->fmt == VEXB_FMT_CSR && variant != 3 && variant != 4)
        VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "spmv.kernel = %ld has no float-valued instantiation: CSR strips with float values run 3 and 4", variant);
    if (A->fmt == VEXB_FMT_CSR && variant == 6 && (reinterpret_cast<uintptr_t>(x) & 15) != 0) variant = 4;   // the window copy needs a 16-byte aligned x
    if (A->fmt == VEXB_FMT_CSR && variant == 6) {
        const size_t smem = (A->tile_nnz + 8) * sizeof(T) + (A->xwin + 4) * sizeof(T) + (A->tile_nnz + 8) * 4 + (A->tile_rows + 12) * 4 + 16;
        static std::atomic<unsigned long long> attr_set[2];
        const int ti = sizeof(T) == 8 ? 0 : 1;
        const unsigned long long bit = 1ull << (A->dev & 63);
        if (smem > 48 * 1024 && !(attr_set[ti].load() & bit)) {
            VEXB_CUDA(cudaFuncSetAttribute(csr_window_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            attr_set[ti].fetch_or(bit);
        }
        csr_window_kernel<T><<<(unsigned)A->n_tiles, 256, smem, st>>>(A->tile, A->tile_x, A->rowptr, A->col, (const T *)A->val, x, y, alpha, append,
                                                                     (int)A->tile_nnz, (int)A->tile_rows, (int)A->xwin, A->row_ids);
        VEXB_LAUNCHED();
    } else if (A->fmt == VEXB_FMT_CSR && variant == 5) {
        long stages = std::max(2l, std::min(param("spmv.ring_stages", 3), 8l));
        long warps = std::max(1l, std::min(param("spmv.ring_warps", 8), 8l));
        const size_t smem = (size_t)warps * stages * RingStage<T>::bytes + (size_t)warps * stages * 8;
        static std::atomic<unsigned long long> attr_set[2];
        const int ti = sizeof(T) == 8 ? 0 : 1;
        const unsigned long long bit = 1ull << (A->dev & 63);
        if (!(attr_set[ti].load() & bit)) {
            VEXB_CUDA(cudaFuncSetAttribute(csr_ring_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
            attr_set[ti].fetch_or(bit);
        }
        VEXB_CHECK(smem <= 224 * 1024, "spmv.ring_stages x spmv.ring_warps needs %zu bytes of shared memory", smem);
        int per_sm = 0;
        VEXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, csr_ring_kernel<T>, (int)warps * 32, smem));
        if (per_sm < 1) per_sm = 1;
        const long cap = param("spmv.ctas_per_sm", 0);
        if (cap > 0 && per_sm > cap) per_sm = (int)cap;
        const size_t grid = std::min((A->n_wtiles + warps - 1) / warps, (size_t)per_sm * (size_t)sm_count(A->dev));
        csr_ring_kernel<T><<<(unsigned)grid, (unsigned)warps * 32, smem, st>>>(A->wtile, (int)A->n_wtiles, A->rowptr, A->col, (const T *)A->val, x, y,
                                                                             alpha, append, A->row_ids, (int)stages);
        VEXB_LAUNCHED();
    } else if (A->fmt == VEXB_FMT_CSR && variant == 4) {
        static std::atomic<int> per_sm[2];
        const int ti = sizeof(T) == 8 ? 0 : 1;
        if (!per_sm[ti].load()) {
            int v = 0;
            VEXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, csr_warp_kernel<T, V>, 256, 0));
            per_sm[ti].store(v > 0 ? v : 1);
        }
        const long cap = param("spmv.ctas_per_sm", 0);
        const size_t resident = (size_t)(cap > 0 && cap < per_sm[ti].load() ? cap : per_sm[ti].load()) * (size_t)sm_count(A->dev);
        const size_t grid = std::min((A->n_wtiles + 7) / 8, resident);
        csr_warp_kernel<T, V><<<(unsigned)grid, 256, 0, st>>>(A->wtile, (int)A->n_wtiles, A->rowptr, A->col, (const V *)A->val, x, y, alpha, append, A->row_ids);
        VEXB_LAUNCHED();
    } else if (A->fmt == VEXB_FMT_CSR && variant == 3) {
        csr_scalar_kernel<T, V><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, A->rowptr, A->col, (const V *)A->val, x, y, alpha, append, A->row_ids);
        VEXB_LAUNCHED();
    } else if (A->fmt == VEXB_FMT_CSR && variant == 2 && A->tile_nnz <= (size_t)kDirectThreads * kDirectPerThread) {
        const size_t smem = std::max<size_t>(A->tile_nnz, 64) * sizeof(T);
        csr_direct_kernel<T><<<(unsigned)A->n_tiles, kDirectThreads, smem, st>>>(A->tile, A->rowptr, A->col, (const T *)A->val, x, y,
                                                                                alpha, append, (int)A->tile_nnz, A->row_ids);
        VEXB_LAUNCHED();
    } else if (A->fmt == VEXB_FMT_CSR && variant == 1) {
        long stages = param("spmv.stages", 4);
        stages = std::max(2l, std::min(stages, 16l));
        const size_t stage_bytes = ((A->tile_nnz + 8) * sizeof(T) + (A->tile_nnz + 8) * 4 + (A->tile_rows + 12) * 4 + 127) & ~(size_t)127;
        size_t smem = stage_bytes * stages + 16 * stages + 16 * stages + 16;
        while (smem > 220 * 1024 && stages > 2) { --stages; smem = stage_bytes * stages + 32 * stages + 16; }
        // the opt-in shared-memory limit is a per-device function attribute: set it on every device once
        static std::atomic<unsigned long long> attr_set[2];
        const int ti = sizeof(T) == 8 ? 0 : 1;
        const unsigned long long bit = 1ull << (A->dev & 63);
        if (!(attr_set[ti].load() & bit)) {
            VEXB_CUDA(cudaFuncSetAttribute(csr_pipe_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
            attr_set[ti].fetch_or(bit);
        }
        int per_sm = 0;
        VEXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, csr_pipe_kernel<T>, kPipeThreads, smem));
        if (per_sm < 1) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "CSR tile of %zu nnz does not fit in shared memory", A->tile_nnz);
        const long cap = param("spmv.ctas_per_sm", 0);
        if (cap > 0 && per_sm > cap) per_sm = (int)cap;
        const size_t grid = std::min(A->n_tiles, (size_t)per_sm * (size_t)sm_count(A->dev));
        csr_pipe_kernel<T><<<(unsigned)grid, kPipeThreads, smem, st>>>(A->tile, (int)A->n_tiles, A->rowptr, A->col, (const T *)A->val, x, y,
                                                                     alpha, append, (int)A->tile_nnz, (int)A->tile_rows, (int)stages, A->row_ids);
        VEXB_LAUNCHED();
    } else if (A->fmt == VEXB_FMT_CSR) {
        const size_t smem = (A->tile_nnz + 8) * sizeof(T) + (A->tile_nnz + 8) * 4 + (A->tile_rows + 12) * 4 + 16;
        static std::atomic<unsigned long long> attr_set[2];
        const int ti = sizeof(T) == 8 ? 0 : 1;
        const unsigned long long bit = 1ull << (A->dev & 63);
        if (smem > 48 * 1024 && !(attr_set[ti].load() & bit)) {
            VEXB_CUDA(cudaFuncSetAttribute(csr_stream_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            attr_set[ti].fetch_or(bit);
        }
        csr_stream_kernel<T><<<(unsigned)A->n_tiles, 256, smem, st>>>(A->tile, A->rowptr, A->col, (const T *)A->val, x, y, alpha, append,
                                                                     (int)A->tile_nnz, (int)A->tile_rows, A->row_ids);
        VEXB_LAUNCHED();
    } else {
        const unsigned blocks = (unsigned)((n + 255) / 256);
#define HL(W) do { \
            if (A->ell_col16) hell_kernel<T, W, short, V><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_col16, A->ell_shifts, \
                  (const V *)A->ell_val, A->tail_ptr, A->tail_col, (const V *)A->tail_val, x, y, alpha, append, A->row_ids, 0); \
            else hell_kernel<T, W, int, V><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_col, EllShifts{}, \
                  (const V *)A->ell_val, A->tail_ptr, A->tail_col, (const V *)A->tail_val, x, y, alpha, append, A->row_ids, 0); } while (0)
#define HD(W) hell_kernel<T, W, EllDiag, V><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_mask, A->ell_shifts, \
                  (const V *)A->ell_val, A->tail_ptr, A->tail_col, (const V *)A->tail_val, x, y, alpha, append, A->row_ids, 0)
#define HC(W) hell_kernel<T, W, EllClass><<<(unsigned)((n + 256 * kEllClassRows - 1) / (256 * kEllClassRows)), 256, 0, st>>>( \
                  n, A->ell_pitch, (int)A->ell_width, A->ell_class, A->ell_shifts, (const T *)A->ell_ctab, A->tail_ptr, A->tail_col, \
                  (const T *)A->tail_val, x, y, alpha, append, A->row_ids, kEllClassPrefetchBlocks)
        if (A->ell_class) {
            switch (A->ell_width) {   // = the widths build() gives row classes: those of slot masks (never float-valued)
                case 3: HC(3); break; case 5: HC(5); break; case 7: HC(7); break;
                default: VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no hell_kernel for row classes of width %zu", A->ell_width);
            }
        } else if (A->ell_mask) {
            switch (A->ell_width) {   // = the widths build() gives slot masks: ell_width_is_unrolled_everywhere and <= kEllDiagMaxWidth
                case 3: HD(3); break; case 5: HD(5); break; case 7: HD(7); break;
                default: VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no hell_kernel for slot masks of width %zu", A->ell_width);
            }
        } else switch (A->ell_width) {
            case 1: HL(1); break; case 2: HL(2); break; case 3: HL(3); break; case 4: HL(4); break;
            case 5: HL(5); break; case 6: HL(6); break; case 7: HL(7); break; case 8: HL(8); break;
            case 9: HL(9); break;
            default: HL(0); break;
        }
#undef HC
#undef HD
#undef HL
        VEXB_LAUNCHED();
    }
    return VEXB_OK;
}

template <class T, int K>
static int spmv_multi_launch(const vexb_spmat *A, cudaStream_t st, const void *const *x, void *const *y, T alpha, int append) {
    const size_t n = A->nrows_stored;
    MultiPtr<K> mp;
    for (int k = 0; k < K; ++k) { mp.x[k] = x[k]; mp.y[k] = y[k]; }
    if (A->fmt == VEXB_FMT_SELL) {
        const unsigned sb = (unsigned)((A->n_slices + 7) / 8);
        if (A->sell_col16) sell_multi_kernel<T, short, K><<<sb, 256, 0, st>>>(A->n_slices, A->sell_ptr, A->sell_perm, A->sell_col16, A->sell_shift,
                                                                             (const T *)A->sell_val, mp, alpha, append, A->row_ids, A->y_offset);
        else sell_multi_kernel<T, int, K><<<sb, 256, 0, st>>>(A->n_slices, A->sell_ptr, A->sell_perm, A->sell_col, 0,
                                                             (const T *)A->sell_val, mp, alpha, append, A->row_ids, A->y_offset);
        VEXB_LAUNCHED();
        return VEXB_OK;
    }
    const unsigned blocks = (unsigned)((n + 255) / 256);
#define HM(W) do { \
        if (A->ell_col16) hell_multi_kernel<T, W, short, K><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_col16, A->ell_shifts, \
              (const T *)A->ell_val, A->tail_ptr, A->tail_col, (const T *)A->tail_val, mp, alpha, append, A->row_ids, A->y_offset); \
        else hell_multi_kernel<T, W, int, K><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_col, EllShifts{}, \
              (const T *)A->ell_val, A->tail_ptr, A->tail_col, (const T *)A->tail_val, mp, alpha, append, A->row_ids, A->y_offset); } while (0)
#define HD(W) hell_multi_kernel<T, W, EllDiag, K><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_mask, A->ell_shifts, \
              (const T *)A->ell_val, A->tail_ptr, A->tail_col, (const T *)A->tail_val, mp, alpha, append, A->row_ids, A->y_offset)
#define HC(W) hell_multi_kernel<T, W, EllClass, K><<<blocks, 256, 0, st>>>(n, A->ell_pitch, (int)A->ell_width, A->ell_class, A->ell_shifts, \
              (const T *)A->ell_ctab, A->tail_ptr, A->tail_col, (const T *)A->tail_val, mp, alpha, append, A->row_ids, A->y_offset)
    if (A->ell_class) {
        switch (A->ell_width) {   // = the widths build() gives row classes
            case 3: HC(3); break; case 5: HC(5); break; case 7: HC(7); break;
            default: VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no hell_multi_kernel for row classes of width %zu", A->ell_width);
        }
    } else if (A->ell_mask) {
        switch (A->ell_width) {   // = the widths build() gives slot masks
            case 3: HD(3); break; case 5: HD(5); break; case 7: HD(7); break;
            default: VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no hell_multi_kernel for slot masks of width %zu", A->ell_width);
        }
    } else switch (A->ell_width) {
        case 3: HM(3); break; case 5: HM(5); break; case 7: HM(7); break; case 9: HM(9); break;   // = ell_width_is_unrolled_everywhere
        default: HM(0); break;
    }
#undef HC
#undef HD
#undef HM
    VEXB_LAUNCHED();
    return VEXB_OK;
}

} // namespace vexb

int vexb::spmat_from_csr(int dev, size_t nrows, size_t ncols, std::vector<int> &rowptr, std::vector<int> &col,
                         const void *val, int val_dtype, int fmt, const std::vector<int> *row_ids, vexb_spmat **out) {
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    auto *A = new vexb_spmat();
    A->dev = dev; A->val_dtype = val_dtype; A->nrows = nrows; A->ncols = ncols;
    A->nrows_stored = rowptr.size() - 1; A->nnz = (size_t)rowptr.back();
    A->val_f32 = (fmt & VEXB_FMT_VALUES_F32) != 0;      // build() clears it where the values go to a table
    fmt &= ~VEXB_FMT_VALUES_F32;
    const size_t nnz = A->nnz;
    int st = VEXB_OK;
    if (val_dtype == VEXB_F64) { std::vector<double> v((const double *)val, (const double *)val + nnz); st = build<double>(A, rowptr, col, v, fmt, row_ids == nullptr); }
    else { std::vector<float> v((const float *)val, (const float *)val + nnz); st = build<float>(A, rowptr, col, v, fmt, row_ids == nullptr); }
    if (st == VEXB_OK && row_ids) {
        std::vector<int> ids(*row_ids);
        st = upload(ids, 0, (void **)&A->row_ids, &A->device_bytes);
    }
    if (st == VEXB_OK && (A->fmt == VEXB_FMT_CSR || A->fmt == VEXB_FMT_HELL || A->fmt == VEXB_FMT_SELL)) {
        SpmvDesc d; memset(&d, 0, sizeof(d));
        d.ell_col = A->ell_col_any(); d.ell_val = A->ell_val_any();
        d.tail_ptr = A->tail_ptr; d.tail_col = A->tail_col; d.tail_val = A->tail_val;
        d.rowptr = A->rowptr; d.col = A->col; d.val = A->val;
        d.pitch = A->ell_pitch; d.width = (int)A->ell_width;
        for (int g = 0; g < kEllShiftSlots; ++g) d.shifts[g] = A->ell_shifts.s[g];
        d.x_max = A->ell_shifts.x_max;
        d.slice_ptr = A->sell_ptr; d.perm = A->sell_perm; d.sell_val = A->sell_val; d.sell_shift = A->sell_shift; d.n_slices = A->n_slices;
        d.sell_col = A->sell_col16 ? (const void *)A->sell_col16 : (const void *)A->sell_col;
        cudaError_t e = cudaMalloc(&A->d_desc, sizeof(d));
        if (e == cudaSuccess) e = cudaMemcpy(A->d_desc, &d, sizeof(d), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { set_error(__FILE__, __LINE__, "strip descriptor upload failed: %s", cudaGetErrorString(e)); st = VEXB_ERR_CUDA; }
    }
    if (st != VEXB_OK) { vexb_spmat_destroy(A); return st; }
    *out = A;
    return VEXB_OK;
}

int vexb::check_fmt_flags(int fmt, int val_dtype, const void *val, size_t n, std::vector<double> &rounded) {
    const int base = fmt & ~VEXB_FMT_VALUES_F32;
    VEXB_CHECK(base >= VEXB_FMT_AUTO && base <= VEXB_FMT_SELL, "bad format %d", fmt);
    if (!(fmt & VEXB_FMT_VALUES_F32)) return VEXB_OK;
    VEXB_CHECK(val_dtype == VEXB_F64, "VEXB_FMT_VALUES_F32 needs double values");
    rounded.resize(n);
    for (size_t j = 0; j < n; ++j) {
        const double v = static_cast<const double *>(val)[j];
        const float f = (float)v;                                     // round to nearest even
        VEXB_CHECK(!std::isinf(f) || std::isinf(v), "value %g at entry %zu overflows float (VEXB_FMT_VALUES_F32)", v, j);
        rounded[j] = (double)f;
    }
    return VEXB_OK;
}

using namespace vexb;

// Host-only: the sliced-ELL layout VEXB_FMT_SELL would use for these row pointers (tests/test_hostlogic.py).
extern "C" int vexb_csr_sell_layout(size_t nrows, const void *ptr, int ptr_bytes, long sigma, size_t *n_slices, size_t *n_slots,
                                    int32_t *perm, int32_t *slice_ptr) {
    VEXB_CHECK(ptr_bytes == 4 || ptr_bytes == 8, "ptr_bytes must be 4 or 8");
    VEXB_CHECK((nrows == 0 || ptr) && n_slices && n_slots, "NULL argument");
    std::vector<int> rp(nrows + 1, 0);
    const int64_t p0 = nrows ? read_index(ptr, ptr_bytes, 0) : 0;
    for (size_t i = 0; i <= nrows && nrows; ++i) {
        const int64_t v = read_index(ptr, ptr_bytes, i) - p0;
        VEXB_CHECK(v >= 0 && v < (int64_t)INT32_MAX && (i == 0 || v >= rp[i - 1]), "row pointers decrease or overflow at row %zu", i);
        rp[i] = (int)v;
    }
    std::vector<int> pm, sp;
    size_t slots = 0;
    if (!sell_layout(nrows, rp.data(), sigma, pm, sp, &slots)) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "strip too large for sliced ELL");
    *n_slices = sp.size() - 1; *n_slots = slots;
    if (perm) std::copy(pm.begin(), pm.end(), perm);
    if (slice_ptr) std::copy(sp.begin(), sp.end(), slice_ptr);
    return VEXB_OK;
}

extern "C" int vexb_csr_create(int dev, void *stream, size_t nrows, size_t ncols,
                               const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                               const void *val, int val_dtype, int fmt, vexb_spmat **out) {
    (void)stream;
    VEXB_CHECK(out, "out is NULL");
    VEXB_CHECK(ptr_bytes == 4 || ptr_bytes == 8, "ptr_bytes must be 4 or 8");
    VEXB_CHECK(col_bytes == 4 || col_bytes == 8, "col_bytes must be 4 or 8");
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "values must be f64 or f32");
    VEXB_CHECK(nrows == 0 || ptr, "ptr is NULL");
    VEXB_CHECK(nrows < (size_t)INT32_MAX && ncols < (size_t)INT32_MAX, "strip dimensions exceed 32-bit local indices");

    const int64_t p0 = nrows ? read_index(ptr, ptr_bytes, 0) : 0;
    const int64_t nnz = nrows ? read_index(ptr, ptr_bytes, nrows) - p0 : 0;
    VEXB_CHECK(nnz >= 0 && nnz < (int64_t)INT32_MAX - 64, "strip nnz=%lld does not fit 32-bit row pointers", (long long)nnz);
    VEXB_CHECK(nnz == 0 || (col && val), "col/val is NULL");
    std::vector<double> rounded;                                       // format, flag, and values under the flag
    VEXB_TRY(check_fmt_flags(fmt, val_dtype, val, (size_t)nnz, rounded));
    if (fmt & VEXB_FMT_VALUES_F32) val = rounded.data();

    std::vector<int> rp(nrows + 1), c((size_t)nnz);
    for (size_t i = 0; i <= nrows; ++i) {
        rp[i] = nrows ? (int)(read_index(ptr, ptr_bytes, i) - p0) : 0;
        VEXB_CHECK(i == 0 || rp[i] >= rp[i - 1], "row pointers decrease at row %zu", i);
    }
    for (size_t j = 0; j < (size_t)nnz; ++j) {
        const int64_t cj = read_index(col, col_bytes, j);
        VEXB_CHECK(cj >= 0 && (size_t)cj < ncols, "column %lld out of range at nnz %zu", (long long)cj, j);
        c[j] = (int)cj;
    }
    // every argument is checked before a device is touched
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    return spmat_from_csr(dev, nrows, ncols, rp, c, val, val_dtype, fmt, nullptr, out);
}

extern "C" int vexb_spmat_destroy(vexb_spmat *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    cudaFree(A->val); cudaFree(A->col); cudaFree(A->rowptr); cudaFree(A->tile); cudaFree(A->tile_x); cudaFree(A->wtile); cudaFree(A->d_desc);
    vexb_ccsr_destroy(A->patterns);
    cudaFree(A->sell_ptr); cudaFree(A->sell_perm); cudaFree(A->sell_col); cudaFree(A->sell_col16); cudaFree(A->sell_val);
    cudaFree(A->row_ids); cudaFree(A->ell_col); cudaFree(A->ell_col16); cudaFree(A->ell_mask); cudaFree(A->ell_class); cudaFree(A->ell_ctab); cudaFree(A->ell_val); cudaFree(A->tail_ptr); cudaFree(A->tail_col); cudaFree(A->tail_val);
    delete A;
    return VEXB_OK;
}

extern "C" int vexb_spmat_get_info(const vexb_spmat *A, vexb_spmat_info *info) {
    VEXB_CHECK(A && info, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->nrows = A->nrows; info->ncols = A->ncols; info->nnz = A->nnz;
    info->fmt = A->fmt; info->val_dtype = A->val_dtype;
    info->ell_width = A->ell_width; info->ell_pitch = A->ell_pitch; info->csr_tail_nnz = A->tail_nnz;
    info->n_tiles = A->n_tiles; info->tile_nnz = A->tile_nnz;
    info->device_bytes = A->device_bytes;
    info->ell_col_bytes = A->ell_mask || A->ell_class ? 0 : A->ell_col16 ? 2 : A->ell_col ? 4 : 0;
    info->ell_classes = (int32_t)A->ell_nclass;
    info->val_bytes = A->patterns || A->ell_class ? 0 : A->val_f32 ? 4 : (int32_t)dtype_size(A->val_dtype);
    if (A->patterns) {
        vexb_ccsr_info ci;
        VEXB_TRY(vexb_ccsr_get_info(A->patterns, &ci));
        info->n_tiles = A->n_patterns;                   // PATTERNS: number of unique rows
        info->tile_nnz = ci.nnz;                         //           entries in the unique-row table
        info->device_bytes += ci.device_bytes;
    }
    return VEXB_OK;
}

extern "C" int vexb_csr_row_patterns(size_t nrows, const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                                     const void *val, int val_dtype, size_t max_patterns, size_t *n_patterns, int32_t *idx) {
    VEXB_CHECK(n_patterns && (ptr || !nrows), "null argument");
    VEXB_CHECK((ptr_bytes == 4 || ptr_bytes == 8) && (col_bytes == 4 || col_bytes == 8), "ptr/col must be 32- or 64-bit integers");
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "values must be f64 or f32");
    VEXB_CHECK(nrows < (size_t)INT32_MAX, "too many rows");
    const int64_t p0 = nrows ? read_index(ptr, ptr_bytes, 0) : 0;
    const int64_t nnz = nrows ? read_index(ptr, ptr_bytes, nrows) - p0 : 0;
    VEXB_CHECK(nnz >= 0 && nnz < (int64_t)INT32_MAX, "nnz does not fit 32 bits");
    std::vector<int> rp(nrows + 1, 0), c((size_t)nnz), id, prow, pcol;
    for (size_t i = 0; i <= nrows && nrows; ++i) rp[i] = (int)(read_index(ptr, ptr_bytes, i) - p0);
    for (size_t j = 0; j < (size_t)nnz; ++j) c[j] = (int)read_index(col, col_bytes, j);
    bool ok;
    if (val_dtype == VEXB_F64) {
        std::vector<double> v((const double *)val, (const double *)val + nnz), pv;
        ok = find_row_patterns<double>(nrows, rp, c, v, max_patterns, id, prow, pcol, pv);
    } else {
        std::vector<float> v((const float *)val, (const float *)val + nnz), pv;
        ok = find_row_patterns<float>(nrows, rp, c, v, max_patterns, id, prow, pcol, pv);
    }
    *n_patterns = ok ? prow.size() - 1 : 0;
    if (ok && idx) std::memcpy(idx, id.data(), nrows * sizeof(int32_t));
    return ok ? VEXB_OK : VEXB_ERR_UNSUPPORTED;
}

// n values of a per-entry value array to the host in the strip's value type (float-valued strips: widened to double)
static int download_values(const vexb_spmat *A, void *dst, const void *src, size_t n) {
    if (!A->val_f32) { VEXB_CUDA(cudaMemcpy(dst, src, n * dtype_size(A->val_dtype), cudaMemcpyDeviceToHost)); return VEXB_OK; }
    std::vector<float> f(n);
    VEXB_CUDA(cudaMemcpy(f.data(), src, n * sizeof(float), cudaMemcpyDeviceToHost));
    std::copy(f.begin(), f.end(), static_cast<double *>(dst));
    return VEXB_OK;
}

extern "C" int vexb_spmat_hell_download(const vexb_spmat *A, int32_t *ell_col, void *ell_val,
                                        int64_t *csr_ptr, int32_t *csr_col, void *csr_val) {
    VEXB_CHECK(A && A->fmt == VEXB_FMT_HELL, "not a HELL matrix");
    DeviceGuard g(A->dev);
    const size_t vs = dtype_size(A->val_dtype), ne = A->ell_pitch * A->ell_width;
    if (ell_col && ne && A->ell_col) VEXB_CUDA(cudaMemcpy(ell_col, A->ell_col, ne * 4, cudaMemcpyDeviceToHost));
    // row classes: each row's mask and values are its class's entry in the table
    std::vector<unsigned char> cid, ctab;
    if ((ell_col || ell_val) && ne && A->ell_class) {
        cid.resize(A->ell_pitch); ctab.resize(kEllClassHeader + A->ell_nclass * A->ell_width * vs);
        VEXB_CUDA(cudaMemcpy(cid.data(), A->ell_class, cid.size(), cudaMemcpyDeviceToHost));
        VEXB_CUDA(cudaMemcpy(ctab.data(), A->ell_ctab, ctab.size(), cudaMemcpyDeviceToHost));
    }
    if (ell_col && ne && (A->ell_mask || A->ell_class)) {
        // slot masks: column of slot k = row + shift of slot k where the row's mask has bit k, else -1
        std::vector<EllDiag> mask(A->ell_pitch);
        if (A->ell_mask) VEXB_CUDA(cudaMemcpy(mask.data(), A->ell_mask, A->ell_pitch * sizeof(EllDiag), cudaMemcpyDeviceToHost));
        else for (size_t i = 0; i < A->ell_pitch; ++i) mask[i].mask = ctab[cid[i]];
        for (size_t k = 0; k < A->ell_width; ++k)
            for (size_t i = 0; i < A->ell_pitch; ++i)
                ell_col[i + A->ell_pitch * k] = (mask[i].mask >> k) & 1u ? (int32_t)((long long)i + A->ell_shifts.s[k]) : -1;
    }
    if (ell_col && ne && A->ell_col16) {
        // 16-bit storage: decode back to the reference's layout (column, or -1 for padding)
        std::vector<short> e16(ne);
        VEXB_CUDA(cudaMemcpy(e16.data(), A->ell_col16, ne * 2, cudaMemcpyDeviceToHost));
        for (size_t k = 0; k < A->ell_width; ++k)
            for (size_t i = 0; i < A->ell_pitch; ++i) {
                const short raw = e16[i + A->ell_pitch * k];
                ell_col[i + A->ell_pitch * k] = raw == (short)-32768 ? -1 : (int32_t)((long long)i + A->ell_shifts.s[std::min<size_t>(k, vexb::kEllShiftSlots - 1)] + raw);
            }
    }
    if (ell_val && ne && A->ell_class) {
        for (size_t k = 0; k < A->ell_width; ++k)
            for (size_t i = 0; i < A->ell_pitch; ++i)
                memcpy((char *)ell_val + (i + A->ell_pitch * k) * vs, &ctab[kEllClassHeader + ((size_t)cid[i] * A->ell_width + k) * vs], vs);
    } else if (ell_val && ne) VEXB_TRY(download_values(A, ell_val, A->ell_val, ne));
    if (ell_col && ell_val && ne) {
        // the reference's packing: a row's entries in slots 0, 1, ... (the device layout may leave gaps, see build())
        for (size_t i = 0; i < A->nrows_stored; ++i) {
            size_t dst = 0;
            for (size_t k = 0; k < A->ell_width; ++k) {
                const size_t at = i + A->ell_pitch * k;
                if (ell_col[at] == -1) continue;
                const size_t to = i + A->ell_pitch * dst;
                if (to != at) {
                    ell_col[to] = ell_col[at]; ell_col[at] = -1;
                    memcpy((char *)ell_val + to * vs, (char *)ell_val + at * vs, vs);
                    memset((char *)ell_val + at * vs, 0, vs);
                }
                ++dst;
            }
        }
    }
    if (csr_ptr) {
        if (A->tail_nnz) {
            std::vector<int> tp(A->nrows_stored + 1);
            VEXB_CUDA(cudaMemcpy(tp.data(), A->tail_ptr, tp.size() * 4, cudaMemcpyDeviceToHost));
            for (size_t i = 0; i <= A->nrows_stored; ++i) csr_ptr[i] = tp[i];
        } else for (size_t i = 0; i <= A->nrows_stored; ++i) csr_ptr[i] = 0;
    }
    if (csr_col && A->tail_nnz) VEXB_CUDA(cudaMemcpy(csr_col, A->tail_col, A->tail_nnz * 4, cudaMemcpyDeviceToHost));
    if (csr_val && A->tail_nnz) VEXB_TRY(download_values(A, csr_val, A->tail_val, A->tail_nnz));
    return VEXB_OK;
}

extern "C" int vexb_spmv(int dev, void *stream, const vexb_spmat *A, const void *x, void *y, double alpha, int append) {
    VEXB_CHECK(A, "matrix is NULL");
    VEXB_CHECK(dev == A->dev, "matrix lives on device %d, not %d", A->dev, dev);
    VEXB_CHECK(A->nrows == 0 || y, "y is NULL");
    VEXB_CHECK(A->nnz == 0 || x, "x is NULL");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    if (A->val_dtype == VEXB_F64 && A->val_f32) return spmv_launch<double, float>(A, (cudaStream_t)stream, (const double *)x, (double *)y, alpha, append);
    if (A->val_dtype == VEXB_F64) return spmv_launch<double>(A, (cudaStream_t)stream, (const double *)x, (double *)y, alpha, append);
    return spmv_launch<float>(A, (cudaStream_t)stream, (const float *)x, (float *)y, (float)alpha, append);
}

// y_k (=|+=) alpha * A x_k for k < nrhs, the matrix streamed once per group of up to 4 right-hand sides (hybrid-ELL and
// sliced-ELL strips); other formats, float-valued strips (VEXB_FMT_VALUES_F32) and single vectors go through vexb_spmv one by one.
// vex::SpMat * vex::multivector.
extern "C" int vexb_spmv_multi(int dev, void *stream, const vexb_spmat *A, int nrhs, const void *const *x, void *const *y,
                               double alpha, int append) {
    VEXB_CHECK(A && nrhs >= 1 && x && y, "bad arguments");
    VEXB_CHECK(dev == A->dev, "matrix lives on device %d, not %d", A->dev, dev);
    for (int k = 0; k < nrhs; ++k) VEXB_CHECK((A->nrows == 0 || y[k]) && (A->nnz == 0 || x[k]), "vector %d is NULL", k);
    const bool fused = (A->fmt == VEXB_FMT_HELL || A->fmt == VEXB_FMT_SELL) && !A->val_f32 && A->nnz > 0 && A->nrows_stored > 0 && nrhs > 1 && !param("spmv.no_multi", 0);
    if (!fused) {
        for (int k = 0; k < nrhs; ++k) VEXB_TRY(vexb_spmv(dev, stream, A, x[k], y[k], alpha, append));
        return VEXB_OK;
    }
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    cudaStream_t st = (cudaStream_t)stream;
    for (int k0 = 0; k0 < nrhs;) {
        const int rest = nrhs - k0;
        const int K = rest >= 4 ? 4 : rest;                  // groups of 4, then 3 / 2 / 1
        if (K == 1) { VEXB_TRY(vexb_spmv(dev, stream, A, x[k0], y[k0], alpha, append)); break; }
#define GO(T, KK) VEXB_TRY((spmv_multi_launch<T, KK>(A, st, x + k0, y + k0, (T)alpha, append)))
        if (A->val_dtype == VEXB_F64) { if (K == 4) GO(double, 4); else if (K == 3) GO(double, 3); else GO(double, 2); }
        else { if (K == 4) GO(float, 4); else if (K == 3) GO(float, 3); else GO(float, 2); }
#undef GO
        k0 += K;
    }
    return VEXB_OK;
}
