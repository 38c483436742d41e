// vexb_reduce: fold an expression over one device slice into ONE device value.
//
// Replaces `vexcl_reductor_kernel` (vexcl/reductor.hpp:343-385, :511-564): a
// per-thread grid-stride fold, a shared-memory tree with 11 barriers, 8*SM
// partials copied to the host and folded there (:412-436).
//
// Here: per-thread fold with several independent accumulators fed by 32-byte
// (two 128-bit) loads -> warp shuffle tree -> one partial per block -> the last block to
// finish (atomic ticket) folds the partials in a fixed order, so the value for
// a given launch configuration is deterministic and stays on the device, ready
// for vexb_comm_allreduce or a single 8-byte D2H.
#include "expr_eval.cuh"
#include "shapes.cuh"
#include "peer.cuh"      // fold.cuh: Fold, RtFold, block_finish, the peer exchange

namespace vexb {

int jit_reduce(int dev, cudaStream_t st, const vexb_expr &e, int dtype, size_t n, size_t index_offset, int nops, const int *ops,
               bool multi, size_t cap, void *d_result, void *d_workspace, const PeerArgs &pa);

template <int SH, int OP, class T, int U>
__global__ void __launch_bounds__(256) reduce_sweep_kernel(SweepArgs a, size_t n, void *ws, T *result, PeerArgs pa) {
    typedef Shape<SH> S;
    typedef Lanes<T> L;
    constexpr int E = L::E;
    constexpr int K = S::K;
    const T sc[2] = {sweep_scalar<T>(a, 0), sweep_scalar<T>(a, 1)};
    Fold<OP, T> acc[U][E];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < E; ++j) acc[u][j].init();
    const size_t nvec = n / E;
    const size_t stride = (size_t)gridDim.x * blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; base < nvec; base += stride) {
        Vec256 in[K][U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) {
#pragma unroll
                for (int k = 0; k < K; ++k) in[k][u] = ldg256((const char *)a.v[k] + iv * 32);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) {
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    T v[K];
#pragma unroll
                    for (int k = 0; k < K; ++k) v[k] = L::get(in[k][u], j);
                    acc[u][j].take(S::template f<T>(v, sc));
                }
            }
        }
    }
    const size_t i = nvec * E + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        T v[K];
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = ((const T *)a.v[k])[i];
        acc[0][0].take(S::template f<T>(v, sc));
    }
    Fold<OP, T> f = acc[0][0];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < E; ++j) if (u || j) f.merge(acc[u][j]);
    block_finish<OP, T>(f, ws, result, pa);
}

// ---- CG vector updates (BASELINE configs[4]: "fused CG step = SpMV + 2 axpy + 2 dot") ---------------------------------
// After q = A p and (p, q) (one launch: vexb_dspmat_apply_dot) an iteration needs
//     alpha = rho / (p, q);  r -= alpha q;  rho' = (r, r)                       <- cg_update_r_kernel, one sweep, 24 B/row
//     beta = rho' / rho;     x += alpha p;  p = r + beta p                      <- cg_update_xp_kernel, one sweep, 40 B/row
// The scalars stay in device memory (the divisions happen in the kernels), rho' is folded like any Reductor sum and
// combined across GPUs through the peer mailboxes in the same kernel.  Same unfused arithmetic per element as the
// composition x += alpha*p; r -= alpha*q; sum(r*r); p = r + beta*p through vexb_eval / vexb_reduce, 64 bytes per row
// instead of 96 (x += alpha p is deferred to the sweep that rewrites p anyway: it needs the OLD p, which that sweep reads).
template <class T, int U>
__global__ void __launch_bounds__(256) cg_update_r_kernel(size_t n, T *r, const T *q, const T *rho, const T *pq,
                                                           void *ws, T *rho_new, PeerArgs pa) {
    typedef Lanes<T> L;
    constexpr int E = L::E;
    const T alpha = Arith<T>::div(*rho, *pq);
    Fold<VEXB_SUM, T> acc[U][E];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < E; ++j) acc[u][j].init();
    const size_t nvec = n / E;
    const size_t stride = (size_t)gridDim.x * blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; base < nvec; base += stride) {
        Vec256 vr[U], vq[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) { vr[u] = ldg256((const char *)r + iv * 32); vq[u] = ldg256((const char *)q + iv * 32); }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) {
                Vec256 orr;
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    const T rn = Arith<T>::sub(L::get(vr[u], j), Arith<T>::mul(alpha, L::get(vq[u], j)));
                    L::set(orr, j, rn);
                    acc[u][j].take(Arith<T>::mul(rn, rn));
                }
                stg256((char *)r + iv * 32, orr);
            }
        }
    }
    const size_t i = nvec * E + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const T rn = Arith<T>::sub(r[i], Arith<T>::mul(alpha, q[i]));
        r[i] = rn;
        acc[0][0].take(Arith<T>::mul(rn, rn));
    }
    Fold<VEXB_SUM, T> f = acc[0][0];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < E; ++j) if (u || j) f.merge(acc[u][j]);
    block_finish<VEXB_SUM, T>(f, ws, rho_new, pa);
}

template <class T, int U>
__global__ void __launch_bounds__(256) cg_update_xp_kernel(size_t n, T *x, T *p, const T *r, const T *rho, const T *pq, const T *rho_new) {
    typedef Lanes<T> L;
    constexpr int E = L::E;
    const T alpha = Arith<T>::div(*rho, *pq);
    const T beta = Arith<T>::div(*rho_new, *rho);
    const size_t nvec = n / E;
    const size_t stride = (size_t)gridDim.x * blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; base < nvec; base += stride) {
        Vec256 vx[U], vr[U], vp[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) { vx[u] = ldg256((const char *)x + iv * 32); vr[u] = ldg256((const char *)r + iv * 32); vp[u] = ldg256((const char *)p + iv * 32); }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) {
                Vec256 ox, op;
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    const T pj = L::get(vp[u], j);
                    L::set(ox, j, Arith<T>::add(L::get(vx[u], j), Arith<T>::mul(alpha, pj)));
                    L::set(op, j, Arith<T>::add(L::get(vr[u], j), Arith<T>::mul(beta, pj)));
                }
                stg256((char *)x + iv * 32, ox); stg256((char *)p + iv * 32, op);
            }
        }
    }
    const size_t i = nvec * E + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const T pj = p[i];
        x[i] = Arith<T>::add(x[i], Arith<T>::mul(alpha, pj));
        p[i] = Arith<T>::add(r[i], Arith<T>::mul(beta, pj));
    }
}

template <class T> __device__ __forceinline__ T v_as(V v);
template <> __device__ __forceinline__ double v_as<double>(V v) { return v.f; }
template <> __device__ __forceinline__ float v_as<float>(V v) { return (float)v.f; }
template <> __device__ __forceinline__ int v_as<int>(V v) { return (int)v.i; }
template <> __device__ __forceinline__ unsigned v_as<unsigned>(V v) { return (unsigned)v.u; }
template <> __device__ __forceinline__ long long v_as<long long>(V v) { return v.i; }
template <> __device__ __forceinline__ unsigned long long v_as<unsigned long long>(V v) { return v.u; }

template <int OP, class T, int U, bool EXT>
__global__ void __launch_bounds__(256) reduce_interp_kernel(const __grid_constant__ vexb_expr e, int dtype, size_t n,
                                                             size_t index_offset, void *ws, T *result, PeerArgs pa) {
    const int rt = program_result_type(e);
    Fold<OP, T> acc[U];
#pragma unroll
    for (int k = 0; k < U; ++k) acc[k].init();
    const size_t chunk = (size_t)blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * chunk; base < n; base += (size_t)gridDim.x * chunk) {
        size_t idx[U]; bool active[U]; V out[U];
#pragma unroll
        for (int k = 0; k < U; ++k) { idx[k] = base + (size_t)k * blockDim.x + threadIdx.x; active[k] = idx[k] < n; }
        eval_expr<U, EXT>(e, idx, active, index_offset, out);
#pragma unroll
        for (int k = 0; k < U; ++k) if (active[k]) acc[k].take(v_as<T>(convert(out[k], rt, dtype)));
    }
    Fold<OP, T> f = acc[0];
#pragma unroll
    for (int k = 1; k < U; ++k) f.merge(acc[k]);
    block_finish<OP, T>(f, ws, result, pa);
}

// ---- several reductions of ONE expression in one pass: vex::CombineReductors<R...> (reductor.hpp:132-280) ------------
// The expression is evaluated once per element and fed to up to VEXB_MAX_COMBINED folds (RtFold, fold.cuh); every fold then
// finishes like a single reduction (its own partials and ticket in its own slice of the workspace, its own combine across
// the GPUs).
struct MultiOps { int n; int op[VEXB_MAX_COMBINED]; };

template <class T, int U, bool EXT>
__global__ void __launch_bounds__(256) reduce_multi_kernel(const __grid_constant__ vexb_expr e, int dtype, size_t n, size_t index_offset,
                                                            MultiOps ops, void *ws, size_t ws_stride, T *result, PeerArgs pa) {
    const int rt = program_result_type(e);
    RtFold<T> acc[VEXB_MAX_COMBINED];
    for (int k = 0; k < ops.n; ++k) acc[k].init(ops.op[k]);
    const size_t chunk = (size_t)blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * chunk; base < n; base += (size_t)gridDim.x * chunk) {
        size_t idx[U]; bool active[U]; V out[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { idx[u] = base + (size_t)u * blockDim.x + threadIdx.x; active[u] = idx[u] < n; }
        eval_expr<U, EXT>(e, idx, active, index_offset, out);
#pragma unroll
        for (int u = 0; u < U; ++u) if (active[u]) {
            const T v = v_as<T>(convert(out[u], rt, dtype));
            for (int k = 0; k < ops.n; ++k) acc[k].take(ops.op[k], v);
        }
    }
    for (int k = 0; k < ops.n; ++k) {
        void *wk = reinterpret_cast<char *>(ws) + (size_t)k * ws_stride;
        switch (ops.op[k]) {          // uniform across the block: the barriers inside block_finish are safe
            case VEXB_MAX: { Fold<VEXB_MAX, T> f; f.x = acc[k].x; f.y = T(0); block_finish<VEXB_MAX, T>(f, wk, result + k, pa); break; }
            case VEXB_MIN: { Fold<VEXB_MIN, T> f; f.x = acc[k].x; f.y = T(0); block_finish<VEXB_MIN, T>(f, wk, result + k, pa); break; }
            default:       { Fold<VEXB_SUM, T> f; f.x = acc[k].x; f.y = T(0); block_finish<VEXB_SUM, T>(f, wk, result + k, pa); break; }
        }
        __syncthreads();
    }
}

template <int OP, class T>
__global__ void identity_kernel(T *result) {
    Fold<OP, T> f; f.init();
    result[0] = f.x;
    if (OP == VEXB_MINMAX) result[1] = f.y;
}

static const int kMaxBlocksPerSm = 16;

// eval.jit != 0 (with eval.force_interp = 1 its default is 0): generated kernels may serve expressions that have no
// hand-written form
static bool jit_enabled() { return (param("eval.force_interp", 0) ? param("eval.jit", 0) : param("eval.jit", 2)) != 0; }

template <int SH, class T>
static void launch_rsweep(int op, int blocks, cudaStream_t st, const SweepArgs &a, size_t n, void *ws, void *res, const PeerArgs &pa) {
    switch (op) {
#define C(OP) case OP: reduce_sweep_kernel<SH, OP, T, 2><<<blocks, 256, 0, st>>>(a, n, ws, (T *)res, pa); break;
        C(VEXB_SUM) C(VEXB_SUM_KAHAN) C(VEXB_MAX) C(VEXB_MIN) C(VEXB_MINMAX)
#undef C
    }
}

template <class T>
static bool launch_rsweep_shape(int sh, int op, int blocks, cudaStream_t st, const SweepArgs &a, size_t n, void *ws, void *res, const PeerArgs &pa) {
    switch (sh) {
#define C(ID) case ID: launch_rsweep<ID, T>(op, blocks, st, a, n, ws, res, pa); return true;
        C(SH_COPY) C(SH_MUL) C(SH_SQR) C(SH_SUB) C(SH_ABSDIFF)
#undef C
        default: return false;
    }
}

template <class T>
static void launch_rinterp(int op, int blocks, cudaStream_t st, const vexb_expr &e, int dtype, size_t n, size_t off, void *ws, void *res, const PeerArgs &pa) {
    switch (op) {
#define C(OP) case OP: \
        if (expr_extended(e))  reduce_interp_kernel<OP, T, 4, true><<<blocks, 256, 0, st>>>(e, dtype, n, off, ws, (T *)res, pa); \
        else                   reduce_interp_kernel<OP, T, 4, false><<<blocks, 256, 0, st>>>(e, dtype, n, off, ws, (T *)res, pa); \
        break;
        C(VEXB_SUM) C(VEXB_SUM_KAHAN) C(VEXB_MAX) C(VEXB_MIN) C(VEXB_MINMAX)
#undef C
    }
}

template <class T>
static void launch_identity(int op, cudaStream_t st, void *res) {
    switch (op) {
#define C(OP) case OP: identity_kernel<OP, T><<<1, 1, 0, st>>>((T *)res); break;
        C(VEXB_SUM) C(VEXB_SUM_KAHAN) C(VEXB_MAX) C(VEXB_MIN) C(VEXB_MINMAX)
#undef C
    }
}

} // namespace vexb

using namespace vexb;

extern "C" int vexb_reduce_workspace_bytes(int dev, size_t *bytes) {
    VEXB_CHECK(bytes, "bytes is NULL");
    *bytes = sizeof(ReduceWs) + (size_t)16 * kMaxBlocksPerSm * (size_t)sm_count(dev);
    return VEXB_OK;
}

extern "C" int vexb_reduce_identity(int dev, void *stream, int dtype, int op, void *d_result) {
    VEXB_CHECK(d_result, "d_result is NULL");
    VEXB_CHECK(op >= VEXB_SUM && op <= VEXB_MINMAX, "bad reduce op %d", op);
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case VEXB_F64: launch_identity<double>(op, st, d_result); break;
        case VEXB_F32: launch_identity<float>(op, st, d_result); break;
        case VEXB_I32: launch_identity<int>(op, st, d_result); break;
        case VEXB_U32: launch_identity<unsigned>(op, st, d_result); break;
        case VEXB_I64: launch_identity<long long>(op, st, d_result); break;
        case VEXB_U64: launch_identity<unsigned long long>(op, st, d_result); break;
        default: VEXB_FAIL(VEXB_ERR_INVALID, "bad dtype %d", dtype);
    }
    VEXB_LAUNCHED();
    return VEXB_OK;
}

extern "C" int vexb_reduce(int dev, void *stream, const vexb_expr *expr, int dtype, size_t n,
                           size_t index_offset, int op, void *d_result, void *d_workspace) {
    return vexb_reduce_all(dev, stream, expr, dtype, n, index_offset, op, d_result, d_workspace, nullptr);
}

extern "C" int vexb_reduce_all(int dev, void *stream, const vexb_expr *expr, int dtype, size_t n,
                               size_t index_offset, int op, void *d_result, void *d_workspace, vexb_peer *peer) {
    PeerArgs pa; memset(&pa, 0, sizeof(pa));
    if (peer && peer->nranks > 1) {
        VEXB_CHECK(peer->dev == dev, "peer group lives on device %d, not %d", peer->dev, dev);
        pa = peer->args();
    }
    VEXB_CHECK(dtype >= VEXB_F64 && dtype <= VEXB_U64, "bad dtype %d", dtype);
    VEXB_CHECK(op >= VEXB_SUM && op <= VEXB_MINMAX, "bad reduce op %d", op);
    VEXB_CHECK(d_result && d_workspace, "d_result / d_workspace is NULL");
    if (op == VEXB_SUM_KAHAN && !dtype_is_float(dtype)) op = VEXB_SUM;
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, n != 0));
    if (n == 0) {                                                               // reductor.hpp:318-321
        VEXB_TRY(vexb_reduce_identity(dev, stream, dtype, op, d_result));
        return pa.nranks > 1 ? vexb_peer_allreduce(peer, stream, d_result, dtype, op) : VEXB_OK;
    }
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    cudaStream_t st = (cudaStream_t)stream;
    const int sms = sm_count(dev);
    long bps = param("reduce.blocks_per_sm", 8);
    if (bps < 1) bps = 1; if (bps > kMaxBlocksPerSm) bps = kMaxBlocksPerSm;
    const size_t cap = (size_t)sms * (size_t)bps;
    // user functions and inlined sparse products have no pre-compiled form: one kernel generated for the request (jit.cu)
    if (expr_has_call(e) || expr_has_product(e)) return jit_reduce(dev, st, e, dtype, n, index_offset, 1, &op, false, cap, d_result, d_workspace, pa);
    // loads through raw pointers: the generated kernel too unless eval.jit = 0 (its fold has the bits of reducing the
    // expression's temporary), the interpreter when NVRTC cannot be loaded
    if (expr_has_load(e) && jit_enabled()) {
        const int s = jit_reduce(dev, st, e, dtype, n, index_offset, 1, &op, false, cap, d_result, d_workspace, pa);
        if (s != VEXB_ERR_UNSUPPORTED) return s;
    }

    if ((dtype == VEXB_F64 || dtype == VEXB_F32) && !param("eval.force_interp", 0)) {
        ShapeMatch m = match_shape(e, dtype);
        SweepArgs a; memset(&a, 0, sizeof(a));
        bool ok = m.shape != SH_NONE;
        for (int j = 0; ok && j < 3; ++j) if (m.vslot[j] >= 0) { a.v[j] = e.term[m.vslot[j]].v.ptr; ok = aligned32(a.v[j]); }
        for (int j = 0; ok && j < 2; ++j) if (m.sslot[j] >= 0) ok = false; // reduce shapes take no scalars
        if (ok) {
            const size_t E = dtype == VEXB_F64 ? 4 : 8;
            size_t want = (n / E + 511) / 512; if (want < 1) want = 1;
            const int blocks = (int)(want < cap ? want : cap);
            bool launched = dtype == VEXB_F64 ? launch_rsweep_shape<double>(m.shape, op, blocks, st, a, n, d_workspace, d_result, pa)
                                              : launch_rsweep_shape<float>(m.shape, op, blocks, st, a, n, d_workspace, d_result, pa);
            if (launched) { VEXB_LAUNCHED(); return VEXB_OK; }
        }
    }
    size_t want = (n + 1023) / 1024;
    const int blocks = (int)(want < cap ? want : cap);
    switch (dtype) {
        case VEXB_F64: launch_rinterp<double>(op, blocks, st, e, dtype, n, index_offset, d_workspace, d_result, pa); break;
        case VEXB_F32: launch_rinterp<float>(op, blocks, st, e, dtype, n, index_offset, d_workspace, d_result, pa); break;
        case VEXB_I32: launch_rinterp<int>(op, blocks, st, e, dtype, n, index_offset, d_workspace, d_result, pa); break;
        case VEXB_U32: launch_rinterp<unsigned>(op, blocks, st, e, dtype, n, index_offset, d_workspace, d_result, pa); break;
        case VEXB_I64: launch_rinterp<long long>(op, blocks, st, e, dtype, n, index_offset, d_workspace, d_result, pa); break;
        default:       launch_rinterp<unsigned long long>(op, blocks, st, e, dtype, n, index_offset, d_workspace, d_result, pa); break;
    }
    VEXB_LAUNCHED();
    return VEXB_OK;
}

extern "C" int vexb_reduce_fetch(int dev, void *stream, const void *d_result, int dtype, int count, void *host_out) {
    VEXB_CHECK(d_result && host_out && count > 0, "bad arguments");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    VEXB_CUDA(cudaMemcpyAsync(host_out, d_result, dtype_size(dtype) * (size_t)count, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    VEXB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    // a kernel that gave up waiting for a peer GPU (fused combine, peer-memory halo) poisons its result and raises the
    // process-wide fault: report it here instead of handing back a poisoned value as if it were a sum
    unsigned long long fault = 0;
    vexb_peer_fault(&fault, 0);
    if (fault) VEXB_FAIL(VEXB_ERR_PEER, "a peer GPU did not arrive within the time limit (first seen at epoch %llu); results that needed it are NaN / all-ones", fault);
    return VEXB_OK;
}

extern "C" int vexb_cg_update_r(int dev, void *stream, int dtype, size_t n, void *r, const void *q,
                                const void *d_rho, const void *d_pq, void *d_rho_new, void *d_workspace, vexb_peer *peer) {
    VEXB_CHECK(dtype == VEXB_F64 || dtype == VEXB_F32, "CG updates are defined for f64 / f32");
    VEXB_CHECK(d_rho && d_pq && d_rho_new && d_workspace, "NULL scalar / workspace");
    PeerArgs pa; memset(&pa, 0, sizeof(pa));
    if (peer && peer->nranks > 1) { VEXB_CHECK(peer->dev == dev, "peer group lives on device %d, not %d", peer->dev, dev); pa = peer->args(); }
    if (n == 0) {
        VEXB_TRY(vexb_reduce_identity(dev, stream, dtype, VEXB_SUM, d_rho_new));
        return pa.nranks > 1 ? vexb_peer_allreduce(peer, stream, d_rho_new, dtype, VEXB_SUM) : VEXB_OK;
    }
    VEXB_CHECK(r && q && aligned32(r) && aligned32(q), "vectors must be non-NULL and 32-byte aligned");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    long bps = param("reduce.blocks_per_sm", 8);
    if (bps < 1) bps = 1; if (bps > kMaxBlocksPerSm) bps = kMaxBlocksPerSm;
    const size_t cap = (size_t)sm_count(dev) * (size_t)bps;
    const size_t E = dtype == VEXB_F64 ? 4 : 8;
    size_t want = (n / E + 511) / 512; if (want < 1) want = 1;
    const int blocks = (int)(want < cap ? want : cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == VEXB_F64) cg_update_r_kernel<double, 2><<<blocks, 256, 0, st>>>(n, (double *)r, (const double *)q, (const double *)d_rho,
                                (const double *)d_pq, d_workspace, (double *)d_rho_new, pa);
    else cg_update_r_kernel<float, 2><<<blocks, 256, 0, st>>>(n, (float *)r, (const float *)q, (const float *)d_rho,
                                (const float *)d_pq, d_workspace, (float *)d_rho_new, pa);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

extern "C" int vexb_cg_update_xp(int dev, void *stream, int dtype, size_t n, void *x, void *p, const void *r,
                                 const void *d_rho, const void *d_pq, const void *d_rho_new) {
    VEXB_CHECK(dtype == VEXB_F64 || dtype == VEXB_F32, "CG updates are defined for f64 / f32");
    VEXB_CHECK(d_rho && d_pq && d_rho_new, "NULL scalar");
    if (n == 0) return VEXB_OK;
    VEXB_CHECK(x && p && r && aligned32(x) && aligned32(p) && aligned32(r), "vectors must be non-NULL and 32-byte aligned");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    const size_t E = dtype == VEXB_F64 ? 4 : 8;
    size_t want = (n / E + 255) / 256; if (want < 1) want = 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == VEXB_F64) cg_update_xp_kernel<double, 1><<<(unsigned)want, 256, 0, st>>>(n, (double *)x, (double *)p, (const double *)r,
                                (const double *)d_rho, (const double *)d_pq, (const double *)d_rho_new);
    else cg_update_xp_kernel<float, 1><<<(unsigned)want, 256, 0, st>>>(n, (float *)x, (float *)p, (const float *)r,
                                (const float *)d_rho, (const float *)d_pq, (const float *)d_rho_new);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

template <class T>
static void launch_rmulti(int blocks, cudaStream_t st, const vexb_expr &e, int dtype, size_t n, size_t off, const vexb::MultiOps &ops,
                          void *ws, size_t stride, void *res, const PeerArgs &pa) {
    if (vexb::expr_extended(e))  vexb::reduce_multi_kernel<T, 4, true><<<blocks, 256, 0, st>>>(e, dtype, n, off, ops, ws, stride, (T *)res, pa);
    else                         vexb::reduce_multi_kernel<T, 4, false><<<blocks, 256, 0, st>>>(e, dtype, n, off, ops, ws, stride, (T *)res, pa);
}

extern "C" int vexb_reduce_multi(int dev, void *stream, const vexb_expr *expr, int dtype, size_t n, size_t index_offset,
                                 int nops, const int *ops, void *d_result, void *d_workspace, vexb_peer *peer) {
    VEXB_CHECK(nops >= 1 && nops <= VEXB_MAX_COMBINED && ops, "between 1 and %d reductions can be combined", VEXB_MAX_COMBINED);
    VEXB_CHECK(dtype >= VEXB_F64 && dtype <= VEXB_U64, "bad dtype %d", dtype);
    VEXB_CHECK(d_result && d_workspace, "d_result / d_workspace is NULL");
    MultiOps mo; mo.n = nops;
    for (int k = 0; k < nops; ++k) {
        VEXB_CHECK(ops[k] >= VEXB_SUM && ops[k] <= VEXB_MIN, "reduction %d: only SUM, SUM_Kahan, MAX and MIN combine", k);
        mo.op[k] = (ops[k] == VEXB_SUM_KAHAN && !dtype_is_float(dtype)) ? VEXB_SUM : ops[k];
    }
    PeerArgs pa; memset(&pa, 0, sizeof(pa));
    if (peer && peer->nranks > 1) { VEXB_CHECK(peer->dev == dev, "peer group lives on device %d, not %d", peer->dev, dev); pa = peer->args(); }
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, n != 0));
    const size_t es = dtype_size(dtype);
    if (n == 0) {
        for (int k = 0; k < nops; ++k) {
            VEXB_TRY(vexb_reduce_identity(dev, stream, dtype, mo.op[k], (char *)d_result + (size_t)k * es));
            if (pa.nranks > 1) VEXB_TRY(vexb_peer_allreduce(peer, stream, (char *)d_result + (size_t)k * es, dtype, mo.op[k]));
        }
        return VEXB_OK;
    }
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    size_t stride = 0;
    VEXB_TRY(vexb_reduce_workspace_bytes(dev, &stride));
    long bps = param("reduce.blocks_per_sm", 8);
    if (bps < 1) bps = 1; if (bps > kMaxBlocksPerSm) bps = kMaxBlocksPerSm;
    const size_t cap = (size_t)sm_count(dev) * (size_t)bps;
    size_t want = (n + 1023) / 1024;
    const int blocks = (int)(want < cap ? want : cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (expr_has_call(e) || expr_has_product(e)) return jit_reduce(dev, st, e, dtype, n, index_offset, nops, mo.op, true, cap, d_result, d_workspace, pa);
    if (expr_has_load(e) && jit_enabled()) {
        const int s = jit_reduce(dev, st, e, dtype, n, index_offset, nops, mo.op, true, cap, d_result, d_workspace, pa);
        if (s != VEXB_ERR_UNSUPPORTED) return s;
    }
    switch (dtype) {
        case VEXB_F64: launch_rmulti<double>(blocks, st, e, dtype, n, index_offset, mo, d_workspace, stride, d_result, pa); break;
        case VEXB_F32: launch_rmulti<float>(blocks, st, e, dtype, n, index_offset, mo, d_workspace, stride, d_result, pa); break;
        case VEXB_I32: launch_rmulti<int>(blocks, st, e, dtype, n, index_offset, mo, d_workspace, stride, d_result, pa); break;
        case VEXB_U32: launch_rmulti<unsigned>(blocks, st, e, dtype, n, index_offset, mo, d_workspace, stride, d_result, pa); break;
        case VEXB_I64: launch_rmulti<long long>(blocks, st, e, dtype, n, index_offset, mo, d_workspace, stride, d_result, pa); break;
        default:       launch_rmulti<unsigned long long>(blocks, st, e, dtype, n, index_offset, mo, d_workspace, stride, d_result, pa); break;
    }
    VEXB_LAUNCHED();
    return VEXB_OK;
}
