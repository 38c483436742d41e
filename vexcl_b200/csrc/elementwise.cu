// vexb_eval: lhs[i] OP= expr(i) over one device slice.
//
// Replaces the generated `vexcl_vector_kernel` and its launch
// (vexcl/operations.hpp:1856-1895): a scalar 8-byte-per-thread grid-stride
// loop on 8*SM blocks of 512 threads (vexcl/backend/cuda/kernel.hpp:164-193).
//
// Here:  (1) recognised shapes run a hand-written sweep -- 32 bytes per operand
//            per thread as two 128-bit loads (LDG.E.128), U vectors in flight
//            per thread, 128-bit stores, L1 no-allocate (every byte is touched once);
//        (2) everything else runs the IR interpreter (expr_eval.cuh).
// Both are pure HBM streams; neither contracts mul+add into FMA.
#include "expr_eval.cuh"
#include <vector>
#include "shapes.cuh"

namespace vexb {

int jit_eval_multi(int dev, cudaStream_t st, int ncomp, void *const *lhs, int lhs_dtype, int aop, const vexb_expr *const *es,
                   size_t n, size_t index_offset, int mode, bool *done);
int jit_eval(int dev, cudaStream_t st, void *lhs, int lhs_dtype, int aop, const vexb_expr &e, size_t n, size_t index_offset,
             int mode, bool *done);

template <int SH, int AOP, class T, int U>
__global__ void __launch_bounds__(256) sweep_kernel(T *lhs, SweepArgs a, size_t n) {
    typedef Shape<SH> S;
    typedef Lanes<T> L;
    constexpr int E = L::E;
    constexpr int K = S::K;
    const T sc[2] = {sweep_scalar<T>(a, 0), sweep_scalar<T>(a, 1)};
    const size_t nvec = n / E;
    const size_t stride = (size_t)gridDim.x * blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; base < nvec; base += stride) {
        Vec256 in[K > 0 ? K : 1][U];
        Vec256 acc[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) {
#pragma unroll
                for (int k = 0; k < K; ++k) in[k][u] = ldg256((const char *)a.v[k] + iv * 32);
                if (AOP != VEXB_SET) acc[u] = ldg256((const char *)lhs + iv * 32);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t iv = base + (size_t)u * blockDim.x;
            if (iv < nvec) {
                Vec256 out;
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    T v[K > 0 ? K : 1];
#pragma unroll
                    for (int k = 0; k < K; ++k) v[k] = L::get(in[k][u], j);
                    T r = S::template f<T>(v, sc);
                    if (AOP == VEXB_ADD) r = Arith<T>::add(L::get(acc[u], j), r);
                    if (AOP == VEXB_SUB) r = Arith<T>::sub(L::get(acc[u], j), r);
                    L::set(out, j, r);
                }
                stg256((char *)lhs + iv * 32, out);
            }
        }
    }
    // tail: fewer than E elements
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t i = nvec * E + g;
    if (i < n) {
        T v[K > 0 ? K : 1];
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] = ((const T *)a.v[k])[i];
        T r = S::template f<T>(v, sc);
        if (AOP == VEXB_ADD) r = Arith<T>::add(lhs[i], r);
        if (AOP == VEXB_SUB) r = Arith<T>::sub(lhs[i], r);
        lhs[i] = r;
    }
}

template <int U, bool EXT>
__global__ void __launch_bounds__(256) interp_kernel(const __grid_constant__ vexb_expr e, void *lhs, int lhs_dtype,
                                                      size_t n, size_t index_offset) {
    const int rt = program_result_type(e);
    const size_t chunk = (size_t)blockDim.x * U;
    for (size_t base = (size_t)blockIdx.x * chunk; base < n; base += (size_t)gridDim.x * chunk) {
        size_t idx[U]; bool active[U]; V out[U];
#pragma unroll
        for (int k = 0; k < U; ++k) { idx[k] = base + (size_t)k * blockDim.x + threadIdx.x; active[k] = idx[k] < n; }
        eval_expr<U, EXT>(e, idx, active, index_offset, out);
#pragma unroll
        for (int k = 0; k < U; ++k)
            if (active[k]) store_as(lhs, idx[k], convert(out[k], rt, lhs_dtype), lhs_dtype);
    }
}

typedef void (*sweep_fn)(void *, SweepArgs, size_t);

template <int SH, int AOP, class T>
static void launch_sweep(int blocks, cudaStream_t st, void *lhs, const SweepArgs &a, size_t n) {
    sweep_kernel<SH, AOP, T, 2><<<blocks, 256, 0, st>>>((T *)lhs, a, n);
}

template <int SH, class T>
static void launch_sweep_aop(int aop, int blocks, cudaStream_t st, void *lhs, const SweepArgs &a, size_t n) {
    switch (aop) {
        case VEXB_SET: launch_sweep<SH, VEXB_SET, T>(blocks, st, lhs, a, n); break;
        case VEXB_ADD: launch_sweep<SH, VEXB_ADD, T>(blocks, st, lhs, a, n); break;
        default:       launch_sweep<SH, VEXB_SUB, T>(blocks, st, lhs, a, n); break;
    }
}

template <class T>
static void launch_sweep_shape(int sh, int aop, int blocks, cudaStream_t st, void *lhs, const SweepArgs &a, size_t n) {
    switch (sh) {
#define C(ID) case ID: launch_sweep_aop<ID, T>(aop, blocks, st, lhs, a, n); break;
        C(SH_COPY) C(SH_FILL) C(SH_ADD) C(SH_SUB) C(SH_MUL) C(SH_DIV) C(SH_SQR) C(SH_SCALE)
        C(SH_MULADD) C(SH_AXPY) C(SH_XPAY) C(SH_XMAY) C(SH_AXPBY) C(SH_ABSDIFF)
#undef C
        default: break;
    }
}

static bool scalar_as_double(const vexb_term &t, double *out) {
    switch (t.dtype) {
        case VEXB_F64: *out = t.v.f64; return true;
        case VEXB_F32: *out = (double)t.v.f32; return true;
        default: return false;
    }
}

// Decide whether (lhs, aop, e) can take a sweep kernel; fills args on success.
static bool plan_sweep(const void *lhs, int lhs_dtype, int aop, const vexb_expr &e, ShapeMatch *mm, SweepArgs *args) {
    if (!(lhs_dtype == VEXB_F64 || lhs_dtype == VEXB_F32)) return false;
    if (!(aop == VEXB_SET || aop == VEXB_ADD || aop == VEXB_SUB)) return false;
    if (param("eval.force_interp", 0)) return false;
    ShapeMatch m = match_shape(e, lhs_dtype);
    if (m.shape == SH_NONE) return false;
    if (lhs && !aligned32(lhs)) return false;
    SweepArgs a; memset(&a, 0, sizeof(a));
    for (int j = 0; j < 3; ++j) if (m.vslot[j] >= 0) {
        a.v[j] = e.term[m.vslot[j]].v.ptr;
        if (!aligned32(a.v[j])) return false;
    }
    for (int j = 0; j < 2; ++j) if (m.sslot[j] >= 0) {
        const vexb_term &t = e.term[m.sslot[j]];
        if (t.kind == VEXB_TERM_DSCALAR) a.sp[j] = t.v.ptr;          // dtype == lhs dtype (checked by the signature)
        else if (!scalar_as_double(t, &a.s[j])) return false;
    }
    *mm = m; *args = a;
    return true;
}

// A raw pointer that addresses a target slice: threads would read elements that others overwrite (the reference races
// there).  VEXB_ERR_UNSUPPORTED before any launch; the front ends then redirect the pointer to a device copy.
static int check_pointer_targets(const vexb_expr &e, void *const *lhs, int ncomp) {
    for (int k = 0; k < e.n_terms; ++k)
        for (int c = 0; c < ncomp; ++c)
            if (e.term[k].kind == VEXB_TERM_PTR && e.term[k].v.ptr == lhs[c])
                VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "term %d: a raw pointer addresses target %d of the assignment; read a copy of that vector instead", k, c);
    return VEXB_OK;
}

// Rewrite `lhs OP= rhs` (OP != SET) as a plain program: lhs = (L)((C)lhs OP (C)rhs),
// C = common type of lhs and rhs, as C/C++ compound assignment does.
static int fold_compound(const vexb_expr &e, const void *lhs, int lhs_dtype, int aop, vexb_expr *out) {
    static const int opmap[] = {-1, VEXB_OP_ADD, VEXB_OP_SUB, VEXB_OP_MUL, VEXB_OP_DIV, VEXB_OP_MOD,
                                VEXB_OP_BAND, VEXB_OP_BOR, VEXB_OP_BXOR, VEXB_OP_SHL, VEXB_OP_SHR};
    VEXB_CHECK(aop > VEXB_SET && aop <= VEXB_RSH, "bad assign op %d", aop);
    const int R = host_result_type(e);
    // shifts keep the (promoted) type of the LEFT operand, only the count comes from the right: `a >>= b` on a signed a
    // is an arithmetic shift whatever the type of b (C/C++ [expr.shift]; the reference emits `lhs[i] >>= rhs`)
    const bool shift = aop == VEXB_LSH || aop == VEXB_RSH;
    const int C = shift ? lhs_dtype : common_dtype(lhs_dtype, R);
    if (aop >= VEXB_MOD && (dtype_is_float(C) || (shift && dtype_is_float(R))))
        VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "compound assignment %d is not defined for floating operands", aop);
    VEXB_CHECK(e.n_terms < VEXB_MAX_TERMS, "too many terminals for compound assignment");
    VEXB_CHECK(e.n_code + 4 <= VEXB_MAX_CODE, "program too long for compound assignment");
    memset(out, 0, sizeof(*out));
    out->n_terms = e.n_terms + 1;
    for (int k = 0; k < e.n_terms; ++k) out->term[k] = e.term[k];
    vexb_term &lt = out->term[e.n_terms];
    lt.kind = VEXB_TERM_VEC; lt.dtype = (uint8_t)lhs_dtype; lt.v.ptr = lhs;
    int n = 0;
    const int defs = temp_prefix_length(e);                 // temporaries are defined on an empty stack: before lhs[i]
    for (int pc = 0; pc < defs; ++pc) out->code[n++] = e.code[pc];
    out->code[n++] = vexb_instr{VEXB_OP_TERM, (uint8_t)lhs_dtype, (uint16_t)e.n_terms};
    if (lhs_dtype != C) out->code[n++] = vexb_instr{VEXB_OP_CVT, (uint8_t)C, (uint16_t)lhs_dtype};
    for (int pc = defs; pc < e.n_code; ++pc) out->code[n++] = e.code[pc];
    if (R != C) out->code[n++] = vexb_instr{VEXB_OP_CVT, (uint8_t)C, (uint16_t)R};
    out->code[n++] = vexb_instr{(uint8_t)opmap[aop], (uint8_t)C, 0};
    out->n_code = n;
    return VEXB_OK;
}

} // namespace vexb

using namespace vexb;

extern "C" int vexb_eval_path(int lhs_dtype, int assign_op, const vexb_expr *expr, char *buf, size_t buflen) {
    VEXB_CHECK(buf && buflen > 0, "bad buffer");
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, false));
    ShapeMatch m; SweepArgs a;
    // alignment is checked on the real pointers too: a 32-byte aligned dummy lhs stands in here
    alignas(32) static char dummy[32];
    if (expr_has_call(e) || expr_has_product(e)) snprintf(buf, buflen, "jit");
    else if (plan_sweep(dummy, lhs_dtype, assign_op, e, &m, &a)) snprintf(buf, buflen, "sweep:%s", shape_name(m.shape));
    else snprintf(buf, buflen, param("eval.jit", 0) == 1 ? "jit" : "interp");
    return VEXB_OK;
}

extern "C" int vexb_eval(int dev, void *stream, void *lhs, int lhs_dtype, int assign_op,
                         const vexb_expr *expr, size_t n, size_t index_offset) {
    VEXB_CHECK(lhs_dtype >= VEXB_F64 && lhs_dtype <= VEXB_U64, "bad lhs dtype %d", lhs_dtype);
    VEXB_CHECK(assign_op >= VEXB_SET && assign_op <= VEXB_RSH, "bad assign op %d", assign_op);
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, n != 0));
    if (n == 0) return VEXB_OK;                    // empty partitions are legal (operations.hpp:1886)
    VEXB_CHECK(lhs != nullptr, "lhs is NULL");
    VEXB_TRY(check_pointer_targets(e, &lhs, 1));
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    cudaStream_t st = (cudaStream_t)stream;
    const int sms = sm_count(dev);

    // user functions have no pre-compiled form: NVRTC side path (csrc/jit.cu)
    // ... and neither have sparse products used as terminals: their row loops are generated into the kernel
    if (expr_has_call(e) || expr_has_product(e)) { bool done = false; return jit_eval(dev, st, lhs, lhs_dtype, assign_op, e, n, index_offset, 1, &done); }

    ShapeMatch m; SweepArgs a;
    if (plan_sweep(lhs, lhs_dtype, assign_op, e, &m, &a)) {
        const size_t E = lhs_dtype == VEXB_F64 ? 4 : 8;
        const size_t nvec = n / E;
        const size_t per_block = 256 * 2;
        size_t want = (nvec + per_block - 1) / per_block;
        if (want < 1) want = 1;
        const long bps = param("sweep.blocks_per_sm", 8);
        size_t cap = param("sweep.persistent", 0) ? (size_t)sms * (size_t)bps : want;
        int blocks = (int)(want < cap ? want : cap);
        if (lhs_dtype == VEXB_F64) launch_sweep_shape<double>(m.shape, assign_op, blocks, st, lhs, a, n);
        else                       launch_sweep_shape<float>(m.shape, assign_op, blocks, st, lhs, a, n);
        VEXB_LAUNCHED();
        return VEXB_OK;
    }

    // No hand-written sweep for this shape.  eval.jit: 0 = always the interpreter, 1 = always the NVRTC-specialised
    // kernel, 2 (default) = interpreter for the first uses of a shape, specialised kernel once it is hot.
    const long jit_mode = param("eval.force_interp", 0) ? param("eval.jit", 0) : param("eval.jit", 2);
    if (jit_mode) {
        bool done = false;
        VEXB_TRY(jit_eval(dev, st, lhs, lhs_dtype, assign_op, e, n, index_offset, (int)jit_mode, &done));
        if (done) return VEXB_OK;
    }

    vexb_expr prog;
    if (assign_op != VEXB_SET) { VEXB_TRY(fold_compound(e, lhs, lhs_dtype, assign_op, &prog)); }
    else prog = e;
    const size_t per_block = 256 * 4;
    size_t want = (n + per_block - 1) / per_block;
    const size_t cap = (size_t)sms * (size_t)param("interp.blocks_per_sm", 4);
    const int blocks = (int)(want < cap ? want : cap);
    if (expr_extended(prog)) interp_kernel<4, true><<<blocks, 256, 0, st>>>(prog, lhs, lhs_dtype, n, index_offset);
    else                      interp_kernel<4, false><<<blocks, 256, 0, st>>>(prog, lhs, lhs_dtype, n, index_offset);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

// All components of a multi-expression assignment in one launch (assign_multiexpression, vexcl/operations.hpp:2081-2185):
// lhs[k][i] OP= expr_k(i) for k < ncomp, every right-hand side of element i evaluated before any left-hand side of
// element i is written (so components may read what other components write, as in vex::tie(x, y) = (x + y, y - x)).
// Served by a kernel generated for the tuple of expressions (NVRTC, compiled in the background at first use like any
// other new shape).  *handled = 0: not served (NVRTC absent, still compiling, a sparse product among the terminals, more
// than 8 components) -- the caller evaluates component by component, staging through temporaries where needed.
extern "C" int vexb_eval_multi(int dev, void *stream, int ncomp, void *const *lhs, int lhs_dtype, int assign_op,
                               const vexb_expr *const *exprs, size_t n, size_t index_offset, int *handled) {
    VEXB_CHECK(handled, "handled is NULL");
    *handled = 0;
    VEXB_CHECK(ncomp >= 1 && lhs && exprs, "bad arguments");
    VEXB_CHECK(lhs_dtype >= VEXB_F64 && lhs_dtype <= VEXB_U64, "bad lhs dtype %d", lhs_dtype);
    VEXB_CHECK(assign_op >= VEXB_SET && assign_op <= VEXB_RSH, "bad assign op %d", assign_op);
    if (ncomp < 2 || ncomp > 8) return VEXB_OK;
    std::vector<vexb_expr> es((size_t)ncomp);
    std::vector<const vexb_expr *> ps((size_t)ncomp);
    for (int c = 0; c < ncomp; ++c) {
        VEXB_CHECK(exprs[c], "expression %d is NULL", c);
        VEXB_TRY(normalize_expr(exprs[c], &es[(size_t)c], n != 0));
        ps[(size_t)c] = &es[(size_t)c];
    }
    if (n == 0) { *handled = 1; return VEXB_OK; }
    for (int c = 0; c < ncomp; ++c) VEXB_CHECK(lhs[c] != nullptr, "lhs %d is NULL", c);
    for (int c = 0; c < ncomp; ++c) VEXB_TRY(check_pointer_targets(es[(size_t)c], lhs, ncomp));   // before any fall-back
    const long jit_mode = param("eval.force_interp", 0) ? param("eval.jit", 0) : param("eval.jit", 2);
    if (!jit_mode || !param("eval.fuse_multi", 1)) return VEXB_OK;
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    bool done = false;
    VEXB_TRY(jit_eval_multi(dev, (cudaStream_t)stream, ncomp, lhs, lhs_dtype, assign_op, ps.data(), n, index_offset, (int)jit_mode, &done));
    *handled = done ? 1 : 0;
    return VEXB_OK;
}
