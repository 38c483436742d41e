// Device-side evaluator for the postfix expression IR (include/vexb200.h).
//
// This replaces the *generated source text* of the reference
// (vexcl/operations.hpp:1209-1353: binary/unary/ternary/function emitters):
// instead of compiling a string per expression type, one pre-compiled kernel
// walks the program, which sits in the kernel parameter (constant) bank so
// every fetch of an instruction is a uniform load shared by the warp.
//
// Arithmetic never contracts a*b+c into an FMA (explicit _rn intrinsics), so
// results are bit-identical to the unfused CPU restatement in oracle/.
#pragma once
#include "common.cuh"

namespace vexb {

union V {
    double f;             // F64, and F32 (held exactly as a double)
    long long i;          // I32 (sign-extended), I64
    unsigned long long u; // U32 (zero-extended), U64
};

__device__ __forceinline__ bool is_float(int t) { return t <= VEXB_F32; }

// Wrap an integer result to the width/signedness of type t.
__device__ __forceinline__ V wrap_int(long long x, int t) {
    V r;
    switch (t) {
        case VEXB_I32: r.i = (long long)(int)x; break;
        case VEXB_U32: r.u = (unsigned long long)(unsigned)x; break;
        default: r.i = x; break;
    }
    return r;
}

__device__ __forceinline__ V load_term(const vexb_term &t, size_t idx, size_t index_offset, bool active) {
    V r; r.u = 0;
    if (t.kind == VEXB_TERM_VEC) {
        if (active) {
            switch (t.dtype) {
                case VEXB_F64: r.f = ((const double *)t.v.ptr)[idx]; break;
                case VEXB_F32: r.f = (double)((const float *)t.v.ptr)[idx]; break;
                case VEXB_I32: r.i = (long long)((const int *)t.v.ptr)[idx]; break;
                case VEXB_U32: r.u = (unsigned long long)((const unsigned *)t.v.ptr)[idx]; break;
                case VEXB_I64: r.i = ((const long long *)t.v.ptr)[idx]; break;
                default:       r.u = ((const unsigned long long *)t.v.ptr)[idx]; break;
            }
        }
    } else if (t.kind == VEXB_TERM_SCALAR) {
        switch (t.dtype) {
            case VEXB_F64: r.f = t.v.f64; break;
            case VEXB_F32: r.f = (double)t.v.f32; break;
            case VEXB_I32: r.i = (long long)t.v.i32; break;
            case VEXB_U32: r.u = (unsigned long long)t.v.u32; break;
            case VEXB_I64: r.i = t.v.i64; break;
            default:       r.u = t.v.u64; break;
        }
    } else if (t.kind == VEXB_TERM_DSCALAR) {   // one device-resident value, same for every element
        switch (t.dtype) {
            case VEXB_F64: r.f = *(const double *)t.v.ptr; break;
            case VEXB_F32: r.f = (double)*(const float *)t.v.ptr; break;
            case VEXB_I32: r.i = (long long)*(const int *)t.v.ptr; break;
            case VEXB_U32: r.u = (unsigned long long)*(const unsigned *)t.v.ptr; break;
            case VEXB_I64: r.i = *(const long long *)t.v.ptr; break;
            default:       r.u = *(const unsigned long long *)t.v.ptr; break;
        }
    } else { // VEXB_TERM_INDEX
        r.u = (unsigned long long)(index_offset + idx) + (unsigned long long)t.v.i64;
    }
    return r;
}

// Element idx of the array of a VEXB_TERM_PTR terminal (VEXB_OP_LOAD), 0 outside [0, count).  The back end never lets a
// kernel write an array it reads this way (a pointer into the target is refused), so the read-only path is safe.
__device__ __forceinline__ V load_elem(const vexb_term &t, int dtype, long long idx) {
    V r; r.u = 0;
    unsigned long long count = 0;
#pragma unroll
    for (int b = 5; b >= 0; --b) count = count << 8 | t.pad[b];
    if ((unsigned long long)idx >= count) return r;
    const void *p = t.v.ptr;
    switch (dtype) {
        case VEXB_F64: r.f = __ldg((const double *)p + idx); break;
        case VEXB_F32: r.f = (double)__ldg((const float *)p + idx); break;
        case VEXB_I32: r.i = (long long)__ldg((const int *)p + idx); break;
        case VEXB_U32: r.u = (unsigned long long)__ldg((const unsigned *)p + idx); break;
        case VEXB_I64: r.i = __ldg((const long long *)p + idx); break;
        default:       r.u = __ldg((const unsigned long long *)p + idx); break;
    }
    return r;
}

__device__ __forceinline__ V convert(V a, int from, int to) {
    if (from == to) return a;
    V r;
    if (is_float(from)) {
        if (to == VEXB_F64) return a;
        if (to == VEXB_F32) { r.f = (double)(float)a.f; return r; }
        switch (to) {
            case VEXB_I32: r.i = (long long)(int)a.f; break;
            case VEXB_U32: r.u = (unsigned long long)(unsigned)a.f; break;
            case VEXB_I64: r.i = (long long)a.f; break;
            default:       r.u = (unsigned long long)a.f; break;
        }
        return r;
    }
    // integer source
    if (to == VEXB_F64) { r.f = (from == VEXB_U64) ? (double)a.u : (double)a.i; return r; }
    if (to == VEXB_F32) { r.f = (from == VEXB_U64) ? (double)(float)a.u : (double)(float)a.i; return r; }
    return wrap_int(a.i, to);
}

__device__ __forceinline__ bool truthy(V a, int t) { return is_float(t) ? (a.f != 0.0) : (a.i != 0); }

__device__ __forceinline__ V binary_op(int op, int t, V a, V b) {
    V r; r.u = 0;
    if (t == VEXB_F64) {
        switch (op) {
            case VEXB_OP_ADD: r.f = __dadd_rn(a.f, b.f); break;
            case VEXB_OP_SUB: r.f = __dsub_rn(a.f, b.f); break;
            case VEXB_OP_MUL: r.f = __dmul_rn(a.f, b.f); break;
            case VEXB_OP_DIV: r.f = __ddiv_rn(a.f, b.f); break;
            case VEXB_OP_MOD: case VEXB_OP_FMOD: r.f = fmod(a.f, b.f); break;
            case VEXB_OP_POW:   r.f = pow(a.f, b.f); break;
            case VEXB_OP_ATAN2: r.f = atan2(a.f, b.f); break;
            case VEXB_OP_HYPOT: r.f = hypot(a.f, b.f); break;
            case VEXB_OP_FMIN:  r.f = fmin(a.f, b.f); break;
            case VEXB_OP_FMAX:  r.f = fmax(a.f, b.f); break;
            case VEXB_OP_LT: r.i = a.f <  b.f; break;
            case VEXB_OP_GT: r.i = a.f >  b.f; break;
            case VEXB_OP_LE: r.i = a.f <= b.f; break;
            case VEXB_OP_GE: r.i = a.f >= b.f; break;
            case VEXB_OP_EQ: r.i = a.f == b.f; break;
            case VEXB_OP_NE: r.i = a.f != b.f; break;
            case VEXB_OP_LAND: r.i = (a.f != 0.0) && (b.f != 0.0); break;
            case VEXB_OP_LOR:  r.i = (a.f != 0.0) || (b.f != 0.0); break;
            default: break;
        }
    } else if (t == VEXB_F32) {
        const float x = (float)a.f, y = (float)b.f;
        switch (op) {
            case VEXB_OP_ADD: r.f = (double)__fadd_rn(x, y); break;
            case VEXB_OP_SUB: r.f = (double)__fsub_rn(x, y); break;
            case VEXB_OP_MUL: r.f = (double)__fmul_rn(x, y); break;
            case VEXB_OP_DIV: r.f = (double)__fdiv_rn(x, y); break;
            case VEXB_OP_MOD: case VEXB_OP_FMOD: r.f = (double)fmodf(x, y); break;
            case VEXB_OP_POW:   r.f = (double)powf(x, y); break;
            case VEXB_OP_ATAN2: r.f = (double)atan2f(x, y); break;
            case VEXB_OP_HYPOT: r.f = (double)hypotf(x, y); break;
            case VEXB_OP_FMIN:  r.f = (double)fminf(x, y); break;
            case VEXB_OP_FMAX:  r.f = (double)fmaxf(x, y); break;
            case VEXB_OP_LT: r.i = x <  y; break;
            case VEXB_OP_GT: r.i = x >  y; break;
            case VEXB_OP_LE: r.i = x <= y; break;
            case VEXB_OP_GE: r.i = x >= y; break;
            case VEXB_OP_EQ: r.i = x == y; break;
            case VEXB_OP_NE: r.i = x != y; break;
            case VEXB_OP_LAND: r.i = (x != 0.f) && (y != 0.f); break;
            case VEXB_OP_LOR:  r.i = (x != 0.f) || (y != 0.f); break;
            default: break;
        }
    } else {
        const bool sgn = (t == VEXB_I32 || t == VEXB_I64);
        const int bits = (t == VEXB_I32 || t == VEXB_U32) ? 32 : 64;
        switch (op) {
            case VEXB_OP_ADD: return wrap_int((long long)(a.u + b.u), t);
            case VEXB_OP_SUB: return wrap_int((long long)(a.u - b.u), t);
            case VEXB_OP_MUL: return wrap_int((long long)(a.u * b.u), t);
            case VEXB_OP_DIV:
                if (b.u == 0) return r;
                return sgn ? wrap_int((b.i == -1) ? (long long)(0ull - a.u) : a.i / b.i, t) : wrap_int((long long)(a.u / b.u), t);
            case VEXB_OP_MOD: case VEXB_OP_FMOD:
                if (b.u == 0) return r;
                return sgn ? wrap_int((b.i == -1) ? 0 : a.i % b.i, t) : wrap_int((long long)(a.u % b.u), t);
            case VEXB_OP_BAND: return wrap_int(a.i & b.i, t);
            case VEXB_OP_BOR:  return wrap_int(a.i | b.i, t);
            case VEXB_OP_BXOR: return wrap_int(a.i ^ b.i, t);
            case VEXB_OP_SHL:  return wrap_int((long long)(a.u << (b.u & (bits - 1))), t);
            case VEXB_OP_SHR:  return sgn ? wrap_int(a.i >> (b.u & (bits - 1)), t) : wrap_int((long long)(a.u >> (b.u & (bits - 1))), t);
            case VEXB_OP_FMIN: return sgn ? wrap_int(a.i < b.i ? a.i : b.i, t) : wrap_int((long long)(a.u < b.u ? a.u : b.u), t);
            case VEXB_OP_FMAX: return sgn ? wrap_int(a.i > b.i ? a.i : b.i, t) : wrap_int((long long)(a.u > b.u ? a.u : b.u), t);
            case VEXB_OP_LT: r.i = sgn ? (a.i <  b.i) : (a.u <  b.u); break;
            case VEXB_OP_GT: r.i = sgn ? (a.i >  b.i) : (a.u >  b.u); break;
            case VEXB_OP_LE: r.i = sgn ? (a.i <= b.i) : (a.u <= b.u); break;
            case VEXB_OP_GE: r.i = sgn ? (a.i >= b.i) : (a.u >= b.u); break;
            case VEXB_OP_EQ: r.i = a.u == b.u; break;
            case VEXB_OP_NE: r.i = a.u != b.u; break;
            case VEXB_OP_LAND: r.i = (a.u != 0) && (b.u != 0); break;
            case VEXB_OP_LOR:  r.i = (a.u != 0) || (b.u != 0); break;
            default: break;
        }
    }
    return r;
}

__device__ __forceinline__ V unary_op(int op, int t, V a) {
    V r; r.u = 0;
    if (op == VEXB_OP_LNOT) { r.i = !truthy(a, t); return r; }
    if (t == VEXB_F64) {
        const double x = a.f;
        switch (op) {
            case VEXB_OP_NEG: r.f = -x; break;
            case VEXB_OP_SIN: r.f = sin(x); break;     case VEXB_OP_COS: r.f = cos(x); break;
            case VEXB_OP_TAN: r.f = tan(x); break;     case VEXB_OP_ASIN: r.f = asin(x); break;
            case VEXB_OP_ACOS: r.f = acos(x); break;   case VEXB_OP_ATAN: r.f = atan(x); break;
            case VEXB_OP_SINH: r.f = sinh(x); break;   case VEXB_OP_COSH: r.f = cosh(x); break;
            case VEXB_OP_TANH: r.f = tanh(x); break;   case VEXB_OP_EXP: r.f = exp(x); break;
            case VEXB_OP_EXP2: r.f = exp2(x); break;   case VEXB_OP_LOG: r.f = log(x); break;
            case VEXB_OP_LOG2: r.f = log2(x); break;   case VEXB_OP_LOG10: r.f = log10(x); break;
            case VEXB_OP_SQRT: r.f = __dsqrt_rn(x); break; case VEXB_OP_RSQRT: r.f = rsqrt(x); break;
            case VEXB_OP_CBRT: r.f = cbrt(x); break;   case VEXB_OP_FABS: r.f = fabs(x); break;
            case VEXB_OP_FLOOR: r.f = floor(x); break; case VEXB_OP_CEIL: r.f = ceil(x); break;
            case VEXB_OP_ROUND: r.f = round(x); break; case VEXB_OP_TRUNC: r.f = trunc(x); break;
            default: break;
        }
    } else if (t == VEXB_F32) {
        const float x = (float)a.f; float y = 0.f;
        switch (op) {
            case VEXB_OP_NEG: y = -x; break;
            case VEXB_OP_SIN: y = sinf(x); break;     case VEXB_OP_COS: y = cosf(x); break;
            case VEXB_OP_TAN: y = tanf(x); break;     case VEXB_OP_ASIN: y = asinf(x); break;
            case VEXB_OP_ACOS: y = acosf(x); break;   case VEXB_OP_ATAN: y = atanf(x); break;
            case VEXB_OP_SINH: y = sinhf(x); break;   case VEXB_OP_COSH: y = coshf(x); break;
            case VEXB_OP_TANH: y = tanhf(x); break;   case VEXB_OP_EXP: y = expf(x); break;
            case VEXB_OP_EXP2: y = exp2f(x); break;   case VEXB_OP_LOG: y = logf(x); break;
            case VEXB_OP_LOG2: y = log2f(x); break;   case VEXB_OP_LOG10: y = log10f(x); break;
            case VEXB_OP_SQRT: y = __fsqrt_rn(x); break; case VEXB_OP_RSQRT: y = rsqrtf(x); break;
            case VEXB_OP_CBRT: y = cbrtf(x); break;   case VEXB_OP_FABS: y = fabsf(x); break;
            case VEXB_OP_FLOOR: y = floorf(x); break; case VEXB_OP_CEIL: y = ceilf(x); break;
            case VEXB_OP_ROUND: y = roundf(x); break; case VEXB_OP_TRUNC: y = truncf(x); break;
            default: break;
        }
        r.f = (double)y;
    } else {
        switch (op) {
            case VEXB_OP_NEG: return wrap_int((long long)(0ull - a.u), t);
            case VEXB_OP_FABS: return (t == VEXB_I32 || t == VEXB_I64) ? wrap_int(a.i < 0 ? (long long)(0ull - a.u) : a.i, t) : a;
            default: return a;
        }
    }
    return r;
}

// Result dtype of a program (type of its last node).
__host__ __device__ inline int program_result_type(const vexb_expr &e) {
    if (e.n_code <= 0) return VEXB_F64;
    const vexb_instr &in = e.code[e.n_code - 1];
    if (in.op == VEXB_OP_TERM) {
        const vexb_term &t = e.term[in.arg];
        return t.kind == VEXB_TERM_INDEX ? VEXB_U64 : t.dtype;
    }
    if ((in.op >= VEXB_OP_LT && in.op <= VEXB_OP_LOR) || in.op == VEXB_OP_LNOT) return VEXB_I32;
    return in.type;
}

// Evaluate the program for U element indices at once (U independent lanes give
// the memory system U loads in flight per terminal).  The top of the stack is
// kept in registers; deeper entries spill to a small per-thread array.
// EXT: the program may use the extended opcodes -- temporaries (VEXB_OP_TDEF / VEXB_OP_TREF),
// kept in a per-lane file beside the stack, and loads through raw pointers (VEXB_OP_LOAD).
// Programs without them take the EXT = false instantiation, which is exactly the evaluator
// without those arms: two more arms in the one switch cost the 32-bit reductions register
// spills they did not have.
template <int U, bool EXT = false>
__device__ __forceinline__ void eval_expr(const vexb_expr &e, const size_t (&idx)[U], const bool (&active)[U],
                                          size_t index_offset, V (&out)[U]) {
    V st[VEXB_MAX_STACK][U];
    V tmp[EXT ? VEXB_MAX_TEMPS : 1][U];
    V tos[U];
    int d = 0;
#pragma unroll
    for (int k = 0; k < U; ++k) tos[k].u = 0;
    const int n_code = e.n_code;
    // The dispatch is outside the lane loops, and double-precision arithmetic on double vectors -- the
    // common case -- has its own arms, so the cost of decoding an instruction is shared by U elements.
#define VEXB_LANES _Pragma("unroll") for (int k = 0; k < U; ++k)
    for (int pc = 0; pc < n_code; ++pc) {
        const vexb_instr in = e.code[pc];
        const int op = in.op, t = in.type;
        if constexpr (EXT) {
            if (op == VEXB_OP_TDEF) {           // the host admits it at depth 1 only: the stack is empty after it
                VEXB_LANES tmp[in.arg][k] = tos[k];
                d = 0;
                continue;
            }
            if (op == VEXB_OP_TREF) {
                if (d > 0) { VEXB_LANES st[d - 1][k] = tos[k]; }
                VEXB_LANES tos[k] = tmp[in.arg][k];
                ++d;
                continue;
            }
            if (op == VEXB_OP_LOAD) {           // pops the I64 index, pushes the element; lanes past the end read nothing
                const vexb_term &tm = e.term[in.arg];
                VEXB_LANES tos[k] = active[k] ? load_elem(tm, t, tos[k].i) : V{0};
                continue;
            }
        }
        switch (op) {
            case VEXB_OP_TERM: {
                if (d > 0) { VEXB_LANES st[d - 1][k] = tos[k]; }
                const vexb_term &tm = e.term[in.arg];
                if (tm.kind == VEXB_TERM_VEC && tm.dtype == VEXB_F64) {
                    const double *p = (const double *)tm.v.ptr;
                    VEXB_LANES tos[k].f = active[k] ? __ldcs(p + idx[k]) : 0.0;
                } else {
                    VEXB_LANES tos[k] = load_term(tm, idx[k], index_offset, active[k]);
                }
                ++d;
                break;
            }
            case VEXB_OP_CVT:
                VEXB_LANES tos[k] = convert(tos[k], in.arg, t);
                break;
            case VEXB_OP_ADD:
                if (t == VEXB_F64) { VEXB_LANES tos[k].f = __dadd_rn(st[d - 2][k].f, tos[k].f); }
                else { VEXB_LANES tos[k] = binary_op(op, t, st[d - 2][k], tos[k]); }
                --d; break;
            case VEXB_OP_SUB:
                if (t == VEXB_F64) { VEXB_LANES tos[k].f = __dsub_rn(st[d - 2][k].f, tos[k].f); }
                else { VEXB_LANES tos[k] = binary_op(op, t, st[d - 2][k], tos[k]); }
                --d; break;
            case VEXB_OP_MUL:
                if (t == VEXB_F64) { VEXB_LANES tos[k].f = __dmul_rn(st[d - 2][k].f, tos[k].f); }
                else { VEXB_LANES tos[k] = binary_op(op, t, st[d - 2][k], tos[k]); }
                --d; break;
            case VEXB_OP_DIV:
                if (t == VEXB_F64) { VEXB_LANES tos[k].f = __ddiv_rn(st[d - 2][k].f, tos[k].f); }
                else { VEXB_LANES tos[k] = binary_op(op, t, st[d - 2][k], tos[k]); }
                --d; break;
            case VEXB_OP_SELECT:
                VEXB_LANES tos[k] = (st[d - 3][k].i != 0) ? st[d - 2][k] : tos[k];
                d -= 2; break;
            case VEXB_OP_FMA:
                if (t == VEXB_F32) { VEXB_LANES tos[k].f = (double)__fmaf_rn((float)st[d - 3][k].f, (float)st[d - 2][k].f, (float)tos[k].f); }
                else { VEXB_LANES tos[k].f = __fma_rn(st[d - 3][k].f, st[d - 2][k].f, tos[k].f); }
                d -= 2; break;
            default:
                if ((op >= VEXB_OP_MOD && op <= VEXB_OP_LOR) || (op >= VEXB_OP_POW && op <= VEXB_OP_FMAX)) {
                    VEXB_LANES tos[k] = binary_op(op, t, st[d - 2][k], tos[k]);
                    --d;
                } else {
                    VEXB_LANES tos[k] = unary_op(op, t, tos[k]);
                }
                break;
        }
    }
#undef VEXB_LANES
#pragma unroll
    for (int k = 0; k < U; ++k) out[k] = tos[k];
}

__device__ __forceinline__ void store_as(void *p, size_t idx, V v, int dtype) {
    switch (dtype) {
        case VEXB_F64: ((double *)p)[idx] = v.f; break;
        case VEXB_F32: ((float *)p)[idx] = (float)v.f; break;
        case VEXB_I32: ((int *)p)[idx] = (int)v.i; break;
        case VEXB_U32: ((unsigned *)p)[idx] = (unsigned)v.u; break;
        case VEXB_I64: ((long long *)p)[idx] = v.i; break;
        default:       ((unsigned long long *)p)[idx] = v.u; break;
    }
}

} // namespace vexb
