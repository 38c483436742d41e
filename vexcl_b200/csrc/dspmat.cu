// The slice of a multi-device vex::SpMat owned by ONE device, and SpMat::apply.
//
//   vexb_dspmat_create  <- SpMat ctor body for device d (vexcl/spmat.hpp:86-105) and the
//                          local/remote split with ghost renumbering of
//                          SpMatCSR / SpMatHELL (vexcl/spmat/csr.inl:70-112,
//                          vexcl/spmat/hybrid_ell.inl:132-193)
//   vexb_dspmat_pack    <- vals = permutation(cols)(xloc)     (spmat.hpp:127-135)
//   vexb_halo_exchange  <- D2H, host shuffle, H2D             (spmat.hpp:149-176), now grouped
//                          ncclSend/ncclRecv straight between device buffers over NVLink
//   vexb_dspmat_apply   <- SpMat::apply                       (spmat.hpp:120-185)
//
// The remote strip stores only rows that have remote entries (row-compressed),
// so mul_remote touches y only where a ghost contributes; rows without ghosts
// are left alone where the reference adds alpha*0.
#include "dspmat.hpp"
#include "comm.hpp"
#include "peer.cuh"
#define VEXB_MAX_HALO_PARTS VEXB_MAX_PEERS
#include <algorithm>

namespace vexb {

template <class T>
__global__ void pack_kernel(const int *__restrict__ cols, const T *__restrict__ x, T *__restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __ldg(x + cols[i]);
}

} // namespace vexb

using namespace vexb;

#define VEXB_NCCL(expr) do { ncclResult_t r_ = (expr); if (r_ != ncclSuccess) { \
    ::vexb::set_error(__FILE__, __LINE__, "%s failed: %s", #expr, g_nccl.ncclGetErrorString(r_)); \
    return VEXB_ERR_NCCL; } } while (0)

extern "C" int vexb_dspmat_destroy(vexb_dspmat *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    vexb_spmat_destroy(A->loc); vexb_spmat_destroy(A->bnd); vexb_spmat_destroy(A->rem);
    cudaFree(A->send_cols); cudaFree(A->send_buf); cudaFree(A->ghost_buf);
    halo_link_destroy(A->halo);
    if (A->side) cudaStreamDestroy(A->side);
    if (A->ev_pack) cudaEventDestroy(A->ev_pack);
    if (A->ev_halo) cudaEventDestroy(A->ev_halo);
    if (A->ev_x) cudaEventDestroy(A->ev_x);
    delete A;
    return VEXB_OK;
}

extern "C" int vexb_dspmat_create(int dev, void *stream, int part, const vexb_halo_plan *plan,
                                  size_t nrows, const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                                  const void *val, int val_dtype, int fmt, vexb_dspmat **out) {
    (void)stream;
    VEXB_CHECK(out && plan, "NULL argument");
    VEXB_CHECK(part >= 0 && part < plan->nparts, "part %d out of range", part);
    VEXB_CHECK(ptr_bytes == 4 || ptr_bytes == 8, "ptr_bytes must be 4 or 8");
    VEXB_CHECK(col_bytes == 4 || col_bytes == 8, "col_bytes must be 4 or 8");
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "values must be f64 or f32");
    VEXB_CHECK(nrows == 0 || ptr, "ptr is NULL");

    const size_t col_begin = plan->col_part[part], col_end = plan->col_part[part + 1];
    const std::vector<int64_t> &ghost = plan->ghost[part];
    const size_t vs = dtype_size(val_dtype);
    const int64_t p0 = nrows ? read_index(ptr, ptr_bytes, 0) : 0;
    const int64_t nnz = nrows ? read_index(ptr, ptr_bytes, nrows) - p0 : 0;
    VEXB_CHECK(nnz == 0 || (col && val), "col/val is NULL");
    VEXB_CHECK(nnz < (int64_t)INT32_MAX - 64, "strip nnz does not fit 32-bit row pointers");
    // format, flag, and values under the flag, before a device is touched; every strip below gets the rounded values
    std::vector<double> rounded;
    VEXB_TRY(check_fmt_flags(fmt, val_dtype, val, nnz > 0 ? (size_t)nnz : 0, rounded));
    if (fmt & VEXB_FMT_VALUES_F32) val = rounded.data();
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);

    auto *A = new vexb_dspmat();
    A->dev = dev; A->part = part; A->nparts = plan->nparts; A->val_dtype = val_dtype;
    A->values_f32 = (fmt & VEXB_FMT_VALUES_F32) != 0;
    A->nrows = nrows; A->ncols_local = col_end - col_begin; A->n_ghost = ghost.size();
    A->send_counts = plan->send_counts[part]; A->recv_counts = plan->recv_counts[part];
    A->ghost_counts.resize(plan->nparts); A->land_off.assign(plan->nparts, 0);
    for (int p = 0; p < plan->nparts; ++p) {
        A->ghost_counts[p] = plan->ghost[p].size();
        for (int q = 0; q < part; ++q) A->land_off[p] += plan->recv_counts[p][q];   // receives land in ascending source order
    }

    // Split each row into local and remote entries, keeping storage order (csr.inl:92-112).
    std::vector<int> lrow(nrows + 1, 0), lcol; lcol.reserve((size_t)nnz);
    std::vector<char> lval; lval.reserve((size_t)nnz * vs);
    std::vector<int> rrow_full(nrows + 1, 0), rcol; std::vector<char> rval;
    for (size_t i = 0; i < nrows; ++i) {
        const int64_t a = read_index(ptr, ptr_bytes, i) - p0, b = read_index(ptr, ptr_bytes, i + 1) - p0;
        if (b < a) { vexb_dspmat_destroy(A); VEXB_FAIL(VEXB_ERR_INVALID, "row pointers decrease at row %zu", i); }
        for (int64_t j = a; j < b; ++j) {
            const int64_t c = read_index(col, col_bytes, (size_t)j);
            const char *vj = (const char *)val + (size_t)j * vs;
            if ((size_t)c >= col_begin && (size_t)c < col_end) {
                lcol.push_back((int)(c - (int64_t)col_begin));
                lval.insert(lval.end(), vj, vj + vs);
            } else {
                const auto it = std::lower_bound(ghost.begin(), ghost.end(), c);
                if (it == ghost.end() || *it != c) { vexb_dspmat_destroy(A); VEXB_FAIL(VEXB_ERR_INVALID, "column %lld of row %zu is not in the halo plan", (long long)c, i); }
                rcol.push_back((int)(it - ghost.begin()));
                rval.insert(rval.end(), vj, vj + vs);
            }
        }
        lrow[i + 1] = (int)lcol.size();
        rrow_full[i + 1] = (int)rcol.size();
    }
    A->loc_nnz = lcol.size(); A->rem_nnz = rcol.size();
    if (nnz <= param("dspmat.keep_split_max_nnz", 20000000)) {   // host copy of the split, for parity checks only
        A->loc_ptr.assign(lrow.begin(), lrow.end()); A->loc_col.assign(lcol.begin(), lcol.end()); A->loc_val = lval;
        A->rem_ptr.assign(rrow_full.begin(), rrow_full.end()); A->rem_col.assign(rcol.begin(), rcol.end()); A->rem_val = rval;
        A->split_kept = true;
    }

    int st = VEXB_OK;
    if (rcol.empty()) {
        st = spmat_from_csr(dev, nrows, A->ncols_local, lrow, lcol, lval.data(), val_dtype, fmt, nullptr, &A->loc);
    } else {
        // Rows that own a ghost entry ("boundary" rows) are split off: the interior strip does not
        // depend on the halo and runs on the main stream while the halo is in flight; the boundary rows
        // (local entries, then ghost entries) follow the halo on the side stream.  Disjoint rows, no race on y.
        // Interior = the longest run of consecutive rows without ghost entries (for slab partitions that is
        // everything but a grid line or two at the ends): stored as a plain strip with a row offset, no row
        // map.  If ghosts are scattered all over (longest run < 80 % of the rows) the interior is instead every
        // ghost-free row, row-compressed.
        size_t best_lo = 0, best_hi = 0, run_lo = 0;
        for (size_t i = 0; i <= nrows; ++i) {
            const bool boundary = i == nrows || rrow_full[i + 1] > rrow_full[i];
            if (boundary) { if (i - run_lo > best_hi - best_lo) { best_lo = run_lo; best_hi = i; } run_lo = i + 1; }
        }
        const bool contiguous = (best_hi - best_lo) * 5 >= nrows * 4;
        std::vector<int> bids, rids, irids, brow(1, 0), rrow(1, 0), irow(1, 0), bcol, icol;
        std::vector<char> bval, ival;
        for (size_t i = 0; i < nrows; ++i) {
            const bool has_ghost = rrow_full[i + 1] > rrow_full[i];
            const bool interior = contiguous ? (i >= best_lo && i < best_hi) : !has_ghost;
            std::vector<int> &dc = interior ? icol : bcol;
            std::vector<char> &dv = interior ? ival : bval;
            dc.insert(dc.end(), lcol.begin() + lrow[i], lcol.begin() + lrow[i + 1]);
            dv.insert(dv.end(), lval.begin() + (size_t)lrow[i] * vs, lval.begin() + (size_t)lrow[i + 1] * vs);
            if (interior) { irids.push_back((int)i); irow.push_back((int)icol.size()); }
            else { bids.push_back((int)i); brow.push_back((int)bcol.size()); }
            if (has_ghost) { rids.push_back((int)i); rrow.push_back(rrow_full[i + 1]); }
        }
        if (contiguous) {
            st = spmat_from_csr(dev, irids.size(), A->ncols_local, irow, icol, ival.data(), val_dtype, fmt, nullptr, &A->loc);
            if (st == VEXB_OK) A->loc->y_offset = best_lo;
        } else {
            st = spmat_from_csr(dev, nrows, A->ncols_local, irow, icol, ival.data(), val_dtype, fmt, &irids, &A->loc);
        }
        if (st == VEXB_OK && plan->nparts <= VEXB_MAX_HALO_PARTS) {
            // the same boundary rows once more, local and ghost entries together in storage order (column-major, one
            // thread per row): what the fused peer-memory apply reads (distapply.cu).  col >= 0: local x index,
            // col <= -2: ghost index -(col+2), -1: padding.
            int wb = 0;
            for (int i : bids) wb = std::max(wb, (lrow[i + 1] - lrow[i]) + (rrow_full[i + 1] - rrow_full[i]));
            const size_t bp = (bids.size() + 15) / 16 * 16;
            std::vector<int> mcol(bp * (size_t)wb, -1);
            std::vector<char> mval(bp * (size_t)wb * vs, 0);
            for (size_t k = 0; k < bids.size(); ++k) {
                const size_t i = (size_t)bids[k];
                const int64_t a = read_index(ptr, ptr_bytes, i) - p0, b = read_index(ptr, ptr_bytes, i + 1) - p0;
                int jl = lrow[i], jr = rrow_full[i], slot = 0;
                for (int64_t j = a; j < b; ++j, ++slot) {
                    const int64_t c = read_index(col, col_bytes, (size_t)j);
                    const bool local = (size_t)c >= col_begin && (size_t)c < col_end;
                    mcol[k + bp * (size_t)slot] = local ? lcol[jl++] : -(rcol[jr++] + 2);
                    memcpy(&mval[(k + bp * (size_t)slot) * vs], (const char *)val + (size_t)j * vs, vs);
                }
            }
            st = halo_set_boundary(A, bids, wb, mcol, mval.data());
        }
        const int bfmt = VEXB_FMT_CSR | (fmt & VEXB_FMT_VALUES_F32);
        if (st == VEXB_OK) st = spmat_from_csr(dev, nrows, A->ncols_local, brow, bcol, bval.data(), val_dtype, bfmt, &bids, &A->bnd);
        if (st == VEXB_OK) st = spmat_from_csr(dev, nrows, A->n_ghost, rrow, rcol, rval.data(), val_dtype, bfmt, &rids, &A->rem);
    }
    if (st == VEXB_OK && plan->nparts <= VEXB_MAX_HALO_PARTS) st = halo_prepare(A);
    if (st != VEXB_OK) { vexb_dspmat_destroy(A); return st; }

    const std::vector<int64_t> &sc = plan->send_cols[part];
    A->n_send = sc.size();
    auto fail = [&](cudaError_t e, const char *what) { set_error(__FILE__, __LINE__, "%s failed: %s", what, cudaGetErrorString(e)); vexb_dspmat_destroy(A); return VEXB_ERR_CUDA; };
    cudaError_t e;
    if (A->n_send) {
        std::vector<int> sc32(sc.begin(), sc.end());
        if ((e = cudaMalloc((void **)&A->send_cols, A->n_send * 4)) != cudaSuccess) return fail(e, "cudaMalloc");
        if ((e = cudaMemcpy(A->send_cols, sc32.data(), A->n_send * 4, cudaMemcpyHostToDevice)) != cudaSuccess) return fail(e, "cudaMemcpy");
        if ((e = cudaMalloc(&A->send_buf, A->n_send * vs)) != cudaSuccess) return fail(e, "cudaMalloc");
    }
    if (A->n_ghost) {
        if ((e = cudaMalloc(&A->ghost_buf, A->n_ghost * vs)) != cudaSuccess) return fail(e, "cudaMalloc");
        if ((e = cudaMemset(A->ghost_buf, 0, A->n_ghost * vs)) != cudaSuccess) return fail(e, "cudaMemset");
    }
    // The halo stream gets the highest priority so that its small transfer kernels are scheduled
    // ahead of the thousands of CTAs of the local product they overlap with.
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if ((e = cudaStreamCreateWithPriority(&A->side, cudaStreamNonBlocking, prio_hi)) != cudaSuccess) return fail(e, "cudaStreamCreate");
    if ((e = cudaEventCreateWithFlags(&A->ev_pack, cudaEventDisableTiming)) != cudaSuccess) return fail(e, "cudaEventCreate");
    if ((e = cudaEventCreateWithFlags(&A->ev_halo, cudaEventDisableTiming)) != cudaSuccess) return fail(e, "cudaEventCreate");
    if ((e = cudaEventCreateWithFlags(&A->ev_x, cudaEventDisableTiming)) != cudaSuccess) return fail(e, "cudaEventCreate");
    *out = A;
    return VEXB_OK;
}

extern "C" int vexb_dspmat_get_info(const vexb_dspmat *A, vexb_dspmat_info *info) {
    VEXB_CHECK(A && info, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->nrows = A->nrows; info->ncols_local = A->ncols_local; info->n_ghost = A->n_ghost; info->n_send = A->n_send;
    info->loc_nnz = A->loc_nnz; info->rem_nnz = A->rem_nnz;
    if (A->loc) vexb_spmat_get_info(A->loc, &info->loc);
    if (A->rem) vexb_spmat_get_info(A->rem, &info->rem);
    return VEXB_OK;
}

extern "C" int vexb_dspmat_download_split(const vexb_dspmat *A, int64_t *loc_ptr, int64_t *loc_col, void *loc_val,
                                          int64_t *rem_ptr, int64_t *rem_col, void *rem_val) {
    VEXB_CHECK(A, "matrix is NULL");
    if (!A->split_kept) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "split tables were not kept for this strip (nnz above dspmat.keep_split_max_nnz)");
    if (loc_ptr) std::copy(A->loc_ptr.begin(), A->loc_ptr.end(), loc_ptr);
    if (loc_col) std::copy(A->loc_col.begin(), A->loc_col.end(), loc_col);
    if (loc_val) memcpy(loc_val, A->loc_val.data(), A->loc_val.size());
    if (rem_ptr) std::copy(A->rem_ptr.begin(), A->rem_ptr.end(), rem_ptr);
    if (rem_col) std::copy(A->rem_col.begin(), A->rem_col.end(), rem_col);
    if (rem_val) memcpy(rem_val, A->rem_val.data(), A->rem_val.size());
    return VEXB_OK;
}

extern "C" int vexb_dspmat_inline_strip(const vexb_dspmat *A, const vexb_spmat **strip) {
    VEXB_CHECK(A && strip, "NULL argument");
    const vexb_spmat *S = A->loc;
    // the generated row loop reads values of the vector type: float-valued strips are multiplied into a temporary instead
    const bool ok = S && !A->n_ghost && !A->bnd && !A->rem && !S->row_ids && S->y_offset == 0 && S->nrows_stored == A->nrows &&
                    (S->fmt == VEXB_FMT_CSR || S->fmt == VEXB_FMT_HELL) && !S->val_f32 && S->d_desc && !param("spmv.no_inline", 0);
    *strip = ok ? S : nullptr;
    return VEXB_OK;
}

extern "C" int vexb_dspmat_sweep_strip(const vexb_dspmat *A, const vexb_spmat **strip) {
    VEXB_CHECK(A && strip, "NULL argument");
    const vexb_spmat *S = A->loc;
    const bool ok = S && !A->n_ghost && !A->bnd && !A->rem && !S->row_ids && S->y_offset == 0 && S->nrows_stored == A->nrows &&
                    S->fmt == VEXB_FMT_SELL && !S->val_f32 && S->d_desc && param("spmv.sell_inline", 1) && !param("spmv.no_inline", 0);
    *strip = ok ? S : nullptr;
    return VEXB_OK;
}

extern "C" void *vexb_dspmat_send_buffer(const vexb_dspmat *A) { return A ? A->send_buf : nullptr; }
extern "C" void *vexb_dspmat_ghost_buffer(const vexb_dspmat *A) { return A ? A->ghost_buf : nullptr; }

extern "C" int vexb_dspmat_pack(const vexb_dspmat *A, void *stream, const void *x) {
    VEXB_CHECK(A, "matrix is NULL");
    if (!A->n_send) return VEXB_OK;
    VEXB_CHECK(x, "x is NULL");
    DeviceGuard g(A->dev); VEXB_CHECK(g.ok, "cannot select device %d", A->dev);
    const unsigned blocks = (unsigned)((A->n_send + 255) / 256);
    if (A->val_dtype == VEXB_F64) pack_kernel<double><<<blocks, 256, 0, (cudaStream_t)stream>>>(A->send_cols, (const double *)x, (double *)A->send_buf, A->n_send);
    else pack_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(A->send_cols, (const float *)x, (float *)A->send_buf, A->n_send);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

extern "C" int vexb_dspmat_mul_local(const vexb_dspmat *A, void *stream, const void *x, void *y, double alpha, int append) {
    VEXB_CHECK(A && A->loc, "matrix is NULL");
    VEXB_TRY(vexb_spmv(A->dev, stream, A->loc, x, y, alpha, append));
    if (A->bnd) VEXB_TRY(vexb_spmv(A->dev, stream, A->bnd, x, y, alpha, append));
    return VEXB_OK;
}

extern "C" int vexb_dspmat_mul_remote(const vexb_dspmat *A, void *stream, void *y, double alpha) {
    VEXB_CHECK(A, "matrix is NULL");
    if (!A->rem) return VEXB_OK;
    return vexb_spmv(A->dev, stream, A->rem, A->ghost_buf, y, alpha, 1);
}

// Copy-engine exchange for a single process that owns every part: peer (or same-device)
// cudaMemcpyAsync from each owner's send buffer into the requester's ghost buffer.
static int halo_exchange_copies(int nlocal, vexb_dspmat *const *parts, void *const *streams) {
    const int np = parts[0]->nparts;
    VEXB_CHECK(nlocal == np, "without a communicator every part must be local (%d of %d given)", nlocal, np);
    for (int k = 0; k < nlocal; ++k) VEXB_CHECK(parts[k]->part == k, "parts must be passed in order");
    for (int d = 0; d < np; ++d) {
        const vexb_dspmat *D = parts[d];
        cudaStream_t st = streams ? (cudaStream_t)streams[d] : nullptr;
        const size_t vs = dtype_size(D->val_dtype);
        DeviceGuard g(D->dev);
        size_t ro = 0;
        for (int p = 0; p < np; ++p) {
            const size_t cnt = D->recv_counts[p];
            if (!cnt) continue;
            const vexb_dspmat *P = parts[p];
            size_t so = 0;
            for (int q = 0; q < d; ++q) so += P->send_counts[q];
            VEXB_CHECK(P->send_counts[d] == cnt, "plan mismatch between parts %d and %d", p, d);
            VEXB_CUDA(cudaStreamWaitEvent(st, P->ev_pack, 0));            // owner's pack must have run
            VEXB_CUDA(cudaMemcpyPeerAsync((char *)D->ghost_buf + ro * vs, D->dev, (const char *)P->send_buf + so * vs, P->dev, cnt * vs, st));
            ro += cnt;
        }
    }
    return VEXB_OK;
}

extern "C" int vexb_halo_exchange(int nlocal, vexb_comm *const *comms, vexb_dspmat *const *parts, void *const *streams) {
    VEXB_CHECK(nlocal >= 1 && parts, "bad arguments");
    bool any = false;
    for (int k = 0; k < nlocal; ++k) any = any || parts[k]->n_send || parts[k]->n_ghost;
    if (!any) return VEXB_OK;
    if (!comms) return halo_exchange_copies(nlocal, parts, streams);
    VEXB_TRY(nccl_load());
    for (int k = 0; k < nlocal; ++k) {
        VEXB_CHECK(comms[k] && comms[k]->rank == parts[k]->part && comms[k]->nranks == parts[k]->nparts,
                   "communicator rank/size does not match matrix part %d", parts[k]->part);
    }
    VEXB_NCCL(g_nccl.ncclGroupStart());
    for (int k = 0; k < nlocal; ++k) {
        const vexb_dspmat *A = parts[k];
        cudaStream_t st = streams ? (cudaStream_t)streams[k] : nullptr;
        const size_t vs = dtype_size(A->val_dtype);
        const ncclDataType_t dt = nccl_dtype(A->val_dtype);
        size_t so = 0, ro = 0;
        for (int p = 0; p < A->nparts; ++p) {
            ncclResult_t r = ncclSuccess;
            if (A->send_counts[p]) r = g_nccl.ncclSend((const char *)A->send_buf + so * vs, A->send_counts[p], dt, p, comms[k]->comm, st);
            if (r == ncclSuccess && A->recv_counts[p]) r = g_nccl.ncclRecv((char *)A->ghost_buf + ro * vs, A->recv_counts[p], dt, p, comms[k]->comm, st);
            if (r != ncclSuccess) { g_nccl.ncclGroupEnd(); VEXB_FAIL(VEXB_ERR_NCCL, "ncclSend/Recv failed: %s", g_nccl.ncclGetErrorString(r)); }
            so += A->send_counts[p]; ro += A->recv_counts[p];
        }
    }
    VEXB_NCCL(g_nccl.ncclGroupEnd());
    return VEXB_OK;
}

extern "C" int vexb_dspmat_apply(int nlocal, vexb_comm *const *comms, vexb_dspmat *const *parts, void *const *streams,
                                 const void *const *x, void *const *y, double alpha, int append) {
    VEXB_CHECK(nlocal >= 1 && parts && x && y, "bad arguments");
    bool halo = false;
    for (int k = 0; k < nlocal; ++k) { VEXB_CHECK(parts[k], "part %d is NULL", k); halo = halo || parts[k]->n_send || parts[k]->n_ghost; }
    if (!halo) {
        for (int k = 0; k < nlocal; ++k)
            VEXB_TRY(vexb_dspmat_mul_local(parts[k], streams ? streams[k] : nullptr, x[k], y[k], alpha, append));
        return VEXB_OK;
    }
    // Peer-memory halo connected on every part (vexb_dspmat_halo_connect*): one fused launch per part, no NCCL, no copies.
    bool peer_halo = !param("dspmat.no_peer_halo", 0);
    for (int k = 0; peer_halo && k < nlocal; ++k) { int c = 0; vexb_dspmat_halo_connected(parts[k], &c); peer_halo = c != 0; }
    if (peer_halo) {
        for (int k = 0; k < nlocal; ++k)
            VEXB_TRY(dist_apply(parts[k], (cudaStream_t)(streams ? streams[k] : nullptr), x[k], y[k], alpha, append, nullptr, nullptr, nullptr));
        return VEXB_OK;
    }
    std::vector<void *> side(nlocal);
    // 1. side stream (high priority): wait for x, gather what the neighbours need (spmat.hpp:127-135)
    for (int k = 0; k < nlocal; ++k) {
        const vexb_dspmat *A = parts[k];
        cudaStream_t st = streams ? (cudaStream_t)streams[k] : nullptr;
        DeviceGuard g(A->dev);
        VEXB_CUDA(cudaEventRecord(A->ev_x, st));
        VEXB_CUDA(cudaStreamWaitEvent(A->side, A->ev_x, 0));
        if (!comms)   // copy path: the previous apply's readers of my send buffer must be done
            for (int d = 0; d < nlocal; ++d) if (d != k && A->send_counts[d]) VEXB_CUDA(cudaStreamWaitEvent(A->side, parts[d]->ev_halo, 0));
        VEXB_TRY(vexb_dspmat_pack(A, A->side, x[k]));
        VEXB_CUDA(cudaEventRecord(A->ev_pack, A->side));
        side[k] = (void *)A->side;
    }
    // 2. main stream: rows that need no ghosts (spmat.hpp:142-146), concurrently with ...
    for (int k = 0; k < nlocal; ++k)
        VEXB_TRY(vexb_spmv(parts[k]->dev, streams ? streams[k] : nullptr, parts[k]->loc, x[k], y[k], alpha, append));
    // 3. ... the halo over NVLink on the side streams (replaces spmat.hpp:149-176), then the boundary rows
    VEXB_TRY(vexb_halo_exchange(nlocal, comms, parts, side.data()));
    for (int k = 0; k < nlocal; ++k) {
        const vexb_dspmat *A = parts[k];
        cudaStream_t st = streams ? (cudaStream_t)streams[k] : nullptr;
        if (A->bnd) VEXB_TRY(vexb_spmv(A->dev, A->side, A->bnd, x[k], y[k], alpha, append));
        VEXB_TRY(vexb_dspmat_mul_remote(A, A->side, y[k], alpha));                 // spmat.hpp:178-183
        DeviceGuard g(A->dev);
        VEXB_CUDA(cudaEventRecord(A->ev_halo, A->side));
        VEXB_CUDA(cudaStreamWaitEvent(st, A->ev_halo, 0));
    }
    return VEXB_OK;
}

// y (=|+=) alpha*A*x with the partials of dot_with . y_new computed in the product kernel's epilogue, then a one-block
// fold that also combines across the GPUs of `peers` (every GPU ends with the same bits).  This is q = A p; (p, q) of a CG
// iteration without re-reading p and q (the reference fuses the product into a consumer kernel on one device: sparse/product.hpp:45-130,
// spmat/inline_spmv.hpp:68-76; its multi-device SpMat needs a separate reduction).  Needs the peer-memory halo on every
// part (or a single part) and a hybrid- or sliced-ELL interior strip with entries and values of the vector type: otherwise
// VEXB_ERR_UNSUPPORTED and the caller composes it.
extern "C" int vexb_dspmat_apply_dot(int nlocal, vexb_dspmat *const *parts, void *const *streams, const void *const *x,
                                     void *const *y, double alpha, int append, const void *const *dot_with,
                                     void *const *d_result, vexb_peer *const *peers) {
    VEXB_CHECK(nlocal >= 1 && parts && x && y && dot_with && d_result, "bad arguments");
    for (int k = 0; k < nlocal; ++k) {
        VEXB_CHECK(parts[k] && dot_with[k] && d_result[k], "part %d: NULL argument", k);
        int c = 0;
        VEXB_TRY(vexb_dspmat_halo_connected(parts[k], &c));
        const vexb_spmat *S = parts[k]->loc;
        if (!c || !S || (S->fmt != VEXB_FMT_HELL && S->fmt != VEXB_FMT_SELL) || S->nnz == 0 || param("dspmat.no_peer_halo", 0) ||
            param("dspmat.no_fused_dot", 0))
            VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "fused product + dot needs the peer-memory halo and a hybrid- or sliced-ELL interior strip on every part");
        if (parts[k]->values_f32) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no fused product + dot for float values (VEXB_FMT_VALUES_F32)");
        VEXB_CHECK(parts[k]->nparts == 1 || (peers && peers[k]), "part %d: a peer group is needed to combine the dot across GPUs", k);
    }
    for (int k = 0; k < nlocal; ++k)
        VEXB_TRY(dist_apply(parts[k], (cudaStream_t)(streams ? streams[k] : nullptr), x[k], y[k], alpha, append, dot_with[k], d_result[k],
                            parts[k]->nparts > 1 ? peers[k] : nullptr));
    return VEXB_OK;
}

// SpMat::apply for nrhs vectors at once (vex::SpMat * vex::multivector): x[k * nrhs + r], y[k * nrhs + r] are part k's slices
// of component r.  Parts without a halo multiply all components in one pass over the matrix (vexb_spmv_multi); with a halo
// the components go through vexb_dspmat_apply one after the other, as the reference does (operations.hpp:876-880).
extern "C" int vexb_dspmat_apply_multi(int nlocal, vexb_comm *const *comms, vexb_dspmat *const *parts, void *const *streams,
                                       int nrhs, const void *const *x, void *const *y, double alpha, int append) {
    VEXB_CHECK(nlocal >= 1 && nrhs >= 1 && parts && x && y, "bad arguments");
    bool halo = false;
    for (int k = 0; k < nlocal; ++k) { VEXB_CHECK(parts[k], "part %d is NULL", k); halo = halo || parts[k]->n_send || parts[k]->n_ghost; }
    if (!halo) {
        for (int k = 0; k < nlocal; ++k)
            VEXB_TRY(vexb_spmv_multi(parts[k]->dev, streams ? streams[k] : nullptr, parts[k]->loc, nrhs, x + (size_t)k * nrhs, y + (size_t)k * nrhs, alpha, append));
        return VEXB_OK;
    }
    std::vector<const void *> xs(nlocal); std::vector<void *> ys(nlocal);
    for (int r = 0; r < nrhs; ++r) {
        for (int k = 0; k < nlocal; ++k) { xs[k] = x[(size_t)k * nrhs + r]; ys[k] = y[(size_t)k * nrhs + r]; }
        VEXB_TRY(vexb_dspmat_apply(nlocal, comms, parts, streams, xs.data(), ys.data(), alpha, append));
    }
    return VEXB_OK;
}
