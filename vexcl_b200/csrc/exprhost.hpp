// Host-side handling of the expression IR: validation, normalisation
// (constant-fold conversions of scalars, de-duplicate vector terminals) and
// shape recognition for the hand-written sweep kernels.
#pragma once
#include "common.cuh"
#include <string>
#include <map>

namespace vexb {

// Registry of user functions (jit.cu): argument count / types of function `id`, -1 if unknown.
int function_arity(int id);
int function_arg_dtype(int id, int k);
int function_ret_dtype(int id);

inline int op_arity(int op) {
    if (op == VEXB_OP_TERM) return 0;
    if (op == VEXB_OP_CVT || op == VEXB_OP_NEG || op == VEXB_OP_LNOT) return 1;
    if (op >= VEXB_OP_ADD && op <= VEXB_OP_LOR) return 2;
    if (op == VEXB_OP_SELECT || op == VEXB_OP_FMA) return 3;
    if (op >= VEXB_OP_SIN && op <= VEXB_OP_TRUNC) return 1;
    if (op >= VEXB_OP_POW && op <= VEXB_OP_FMAX) return 2;
    if (op == VEXB_OP_TDEF) return 1;
    if (op == VEXB_OP_TREF) return 0;
    if (op == VEXB_OP_LOAD) return 1;
    return -1;
}

inline bool dtype_is_float(int t) { return t == VEXB_F64 || t == VEXB_F32; }

// Usual arithmetic conversions restricted to the six supported types.
inline int common_dtype(int a, int b) {
    if (a == VEXB_F64 || b == VEXB_F64) return VEXB_F64;
    if (a == VEXB_F32 || b == VEXB_F32) return VEXB_F32;
    if (a == VEXB_U64 || b == VEXB_U64) return VEXB_U64;
    if (a == VEXB_I64 || b == VEXB_I64) return VEXB_I64;
    if (a == VEXB_U32 || b == VEXB_U32) return VEXB_U32;
    return VEXB_I32;
}

// Host mirror of the device `convert` for scalar terminals.
inline void convert_scalar_term(vexb_term &t, int to) {
    const int from = t.dtype;
    if (from == to) return;
    long double x = 0; long long i = 0; unsigned long long u = 0; bool isf = dtype_is_float(from);
    switch (from) {
        case VEXB_F64: x = t.v.f64; break;
        case VEXB_F32: x = t.v.f32; break;
        case VEXB_I32: i = t.v.i32; u = (unsigned long long)i; break;
        case VEXB_U32: u = t.v.u32; i = (long long)u; break;
        case VEXB_I64: i = t.v.i64; u = (unsigned long long)i; break;
        default:       u = t.v.u64; i = (long long)u; break;
    }
    t.v.u64 = 0;
    if (isf) {
        const double d = (double)x;
        switch (to) {
            case VEXB_F64: t.v.f64 = d; break;
            case VEXB_F32: t.v.f32 = (float)d; break;
            case VEXB_I32: t.v.i32 = (int)d; break;
            case VEXB_U32: t.v.u32 = (unsigned)d; break;
            case VEXB_I64: t.v.i64 = (long long)d; break;
            default:       t.v.u64 = (unsigned long long)d; break;
        }
    } else {
        switch (to) {
            case VEXB_F64: t.v.f64 = (from == VEXB_U64) ? (double)u : (double)i; break;
            case VEXB_F32: t.v.f32 = (from == VEXB_U64) ? (float)u : (float)i; break;
            case VEXB_I32: t.v.i32 = (int)i; break;
            case VEXB_U32: t.v.u32 = (unsigned)i; break;
            case VEXB_I64: t.v.i64 = i; break;
            default:       t.v.u64 = u; break;
        }
    }
    t.dtype = (uint8_t)to;
}

inline bool is_product_term(int kind) { return kind == VEXB_TERM_SPMV || kind == VEXB_TERM_CCSR; }

// Sparse products used as terminals (VEXB_TERM_SPMV, VEXB_TERM_CCSR): their row loops are generated into the kernel.
inline bool expr_has_product(const vexb_expr &e) {
    for (int k = 0; k < e.n_terms; ++k) if (is_product_term(e.term[k].kind)) return true;
    return false;
}

inline bool expr_has_call(const vexb_expr &e) {
    for (int pc = 0; pc < e.n_code; ++pc) if (e.code[pc].op == VEXB_OP_CALL) return true;
    return false;
}

inline bool expr_has_temps(const vexb_expr &e) {
    for (int pc = 0; pc < e.n_code; ++pc) if (e.code[pc].op == VEXB_OP_TDEF) return true;
    return false;
}

inline bool expr_has_load(const vexb_expr &e) {
    for (int pc = 0; pc < e.n_code; ++pc) if (e.code[pc].op == VEXB_OP_LOAD) return true;
    return false;
}

// Programs the interpreter serves with its extended opcodes (temporaries, loads through raw pointers): the EXT
// instantiation of eval_expr (expr_eval.cuh).
inline bool expr_extended(const vexb_expr &e) { return expr_has_temps(e) || expr_has_load(e); }

inline bool is_ptr_type(int t) { return (t & VEXB_PTR(0)) != 0; }

// Number of leading instructions that define temporaries: the program up to and including its last TDEF (0 without).
inline int temp_prefix_length(const vexb_expr &e) {
    int n = 0;
    for (int pc = 0; pc < e.n_code; ++pc) if (e.code[pc].op == VEXB_OP_TDEF) n = pc + 1;
    return n;
}

inline int host_result_type(const vexb_expr &e) {
    if (e.n_code <= 0) return VEXB_F64;
    const vexb_instr &in = e.code[e.n_code - 1];
    if (in.op == VEXB_OP_TERM) {
        const vexb_term &t = e.term[in.arg];
        return t.kind == VEXB_TERM_INDEX ? VEXB_U64 : t.dtype;
    }
    if ((in.op >= VEXB_OP_LT && in.op <= VEXB_OP_LOR) || in.op == VEXB_OP_LNOT) return VEXB_I32;
    return in.type;
}

// Validate `in` and write the normalised program to `out`.
inline int normalize_expr(const vexb_expr *in, vexb_expr *out, bool need_ptrs = true) {
    VEXB_CHECK(in && out, "expression is NULL");
    VEXB_CHECK(in->n_terms >= 0 && in->n_terms <= VEXB_MAX_TERMS, "n_terms=%d out of range", in->n_terms);
    VEXB_CHECK(in->n_code >= 1 && in->n_code <= VEXB_MAX_CODE, "n_code=%d out of range", in->n_code);
    for (int k = 0; k < in->n_terms; ++k) {
        const vexb_term &t = in->term[k];
        VEXB_CHECK(t.kind <= VEXB_TERM_PTR, "term %d: bad kind %d", k, (int)t.kind);
        VEXB_CHECK(t.dtype <= VEXB_U64, "term %d: bad dtype %d", k, (int)t.dtype);
        VEXB_CHECK(!need_ptrs || (t.kind != VEXB_TERM_VEC && t.kind != VEXB_TERM_DSCALAR && t.kind != VEXB_TERM_PTR) || t.v.ptr != nullptr,
                   "term %d: NULL device pointer", k);
        if (t.kind == VEXB_TERM_SPMV) {
            VEXB_CHECK(t.v.ptr != nullptr, "term %d: NULL matrix handle", k);
            VEXB_CHECK(t.pad[0] < in->n_terms && in->term[t.pad[0]].kind == VEXB_TERM_VEC && in->term[t.pad[0]].dtype == t.dtype,
                       "term %d: the sparse product's x must be a vector terminal of the matrix's value type", k);
        }
        if (t.kind == VEXB_TERM_CCSR) {
            // the handle is not read here: a source query (vexb_jit_source*) may pass NULL with pad[1] set
            VEXB_CHECK(!need_ptrs || t.v.ptr != nullptr, "term %d: NULL CCSR matrix handle", k);
            VEXB_CHECK(t.dtype == VEXB_F64 || t.dtype == VEXB_F32, "term %d: CCSR values are float or double", k);
            VEXB_CHECK(t.pad[1] == 1 || t.pad[1] == 2 || t.pad[1] == 4, "term %d: CCSR idx width %d is not 1, 2 or 4", k, (int)t.pad[1]);
            VEXB_CHECK(t.pad[0] < in->n_terms && in->term[t.pad[0]].kind == VEXB_TERM_VEC && in->term[t.pad[0]].dtype == t.dtype,
                       "term %d: the CCSR product's x must be a vector terminal of the matrix's value type", k);
        }
    }
    // 1. de-duplicate vector and pointer terminals (same kind, same pointer, same dtype) and drop unused ones.
    int remap[VEXB_MAX_TERMS];
    for (int k = 0; k < VEXB_MAX_TERMS; ++k) remap[k] = -1;
    memset(out, 0, sizeof(*out));
    int depth = 0, maxdepth = 0;
    // temporaries: the type each slot was defined with (-1: not yet), and the type of every value on the stack (the TDEF
    // check needs the top's)
    int temp_type[VEXB_MAX_TEMPS];
    for (int k = 0; k < VEXB_MAX_TEMPS; ++k) temp_type[k] = -1;
    int stype[VEXB_MAX_CODE + 1];
    // the output slot of input terminal `k`: vectors, device scalars and pointers shared by address and type
    auto shared_slot = [&](int k) {
        const vexb_term &t = in->term[k];
        int slot = remap[k];
        if (slot < 0 && (t.kind == VEXB_TERM_VEC || t.kind == VEXB_TERM_DSCALAR || t.kind == VEXB_TERM_PTR)) {
            for (int j = 0; j < out->n_terms; ++j)
                if (out->term[j].kind == t.kind && out->term[j].v.ptr == t.v.ptr && out->term[j].dtype == t.dtype &&
                    (t.kind != VEXB_TERM_PTR || memcmp(out->term[j].pad, t.pad, sizeof(t.pad)) == 0)) { slot = j; break; }
        }
        return slot;
    };
    for (int pc = 0; pc < in->n_code; ++pc) {
        vexb_instr ins = in->code[pc];
        int ar = op_arity(ins.op);
        if (ins.op == VEXB_OP_CALL) {
            ar = function_arity(ins.arg);
            VEXB_CHECK(ar >= 0, "instr %d: call of unregistered function %d", pc, (int)ins.arg);
            VEXB_CHECK(ins.type == function_ret_dtype(ins.arg), "instr %d: call result type does not match the declaration", pc);
        }
        VEXB_CHECK(ar >= 0, "instr %d: unknown opcode %d", pc, (int)ins.op);
        const bool ptr_push = ins.op == VEXB_OP_TERM && ins.arg < in->n_terms && in->term[ins.arg].kind == VEXB_TERM_PTR;
        VEXB_CHECK(ins.type <= VEXB_U64 || (ptr_push && ins.type == VEXB_PTR(in->term[ins.arg].dtype)), "instr %d: bad type %d", pc, (int)ins.type);
        VEXB_CHECK(depth >= ar, "instr %d: stack underflow", pc);
        // a pointer value (VEXB_OP_TERM on a VEXB_TERM_PTR) goes to a call parameter declared with its type, and nowhere else
        for (int q = 0; q < ar; ++q) {
            const int have = stype[depth - ar + q];
            if (ins.op == VEXB_OP_CALL && (is_ptr_type(have) || is_ptr_type(function_arg_dtype(ins.arg, q))))
                VEXB_CHECK(have == function_arg_dtype(ins.arg, q), "instr %d: argument %d of the call is %s, the function declares %s", pc, q,
                           is_ptr_type(have) ? "a pointer" : "a value", is_ptr_type(function_arg_dtype(ins.arg, q)) ? "a pointer of another type" : "a value");
            else VEXB_CHECK(ins.op == VEXB_OP_CALL || !is_ptr_type(have), "instr %d: a raw pointer is only passed to a user function (read an element with VEXB_OP_LOAD)", pc);
        }
        if (ins.op == VEXB_OP_LOAD) {
            VEXB_CHECK(ins.arg < in->n_terms && in->term[ins.arg].kind == VEXB_TERM_PTR, "instr %d: LOAD reads through a pointer terminal", pc);
            VEXB_CHECK(stype[depth - 1] == VEXB_I64, "instr %d: the index of a LOAD is I64, not type %d", pc, stype[depth - 1]);
            VEXB_CHECK(ins.type == in->term[ins.arg].dtype, "instr %d: LOAD of type %d through a pointer of type %d", pc, (int)ins.type, (int)in->term[ins.arg].dtype);
            int slot = shared_slot(ins.arg);
            if (slot < 0) { VEXB_CHECK(out->n_terms < VEXB_MAX_TERMS, "too many terminals"); slot = out->n_terms++; out->term[slot] = in->term[ins.arg]; }   // pad: the count
            remap[ins.arg] = slot;
            ins.arg = (uint16_t)slot;
        }
        if (ins.op == VEXB_OP_TDEF || ins.op == VEXB_OP_TREF) {
            VEXB_CHECK(ins.arg < VEXB_MAX_TEMPS, "instr %d: temporary slot %d out of range (at most %d temporaries)", pc, (int)ins.arg, VEXB_MAX_TEMPS);
            if (ins.op == VEXB_OP_TDEF) {
                VEXB_CHECK(temp_type[ins.arg] < 0, "instr %d: temporary %d is defined twice", pc, (int)ins.arg);
                VEXB_CHECK(depth == 1, "instr %d: a temporary is defined at stack depth %d (definitions come first, at depth 1)", pc, depth);
                VEXB_CHECK(stype[0] == ins.type, "instr %d: temporary %d has type %d, the value it stores type %d", pc, (int)ins.arg, (int)ins.type, stype[0]);
                temp_type[ins.arg] = ins.type;
                depth = 0;
            } else {
                VEXB_CHECK(temp_type[ins.arg] >= 0, "instr %d: temporary %d is read before its definition", pc, (int)ins.arg);
                VEXB_CHECK(temp_type[ins.arg] == ins.type, "instr %d: temporary %d is read as type %d, defined as type %d", pc, (int)ins.arg, (int)ins.type, temp_type[ins.arg]);
                stype[depth++] = ins.type;
                if (depth > maxdepth) maxdepth = depth;
            }
            out->code[out->n_code++] = ins;
            continue;
        }
        if (ins.op == VEXB_OP_TERM) {
            VEXB_CHECK(ins.arg < in->n_terms, "instr %d: term slot %d out of range", pc, (int)ins.arg);
            const vexb_term &t = in->term[ins.arg];
            int slot = shared_slot(ins.arg);
            if (slot < 0 && is_product_term(t.kind)) {
                // the x it multiplies: an ordinary vector terminal (shared with other uses of the same vector)
                const vexb_term &xt = in->term[t.pad[0]];
                int xs = remap[t.pad[0]];
                for (int j = 0; xs < 0 && j < out->n_terms; ++j)
                    if (out->term[j].kind == VEXB_TERM_VEC && out->term[j].v.ptr == xt.v.ptr && out->term[j].dtype == xt.dtype) xs = j;
                if (xs < 0) { VEXB_CHECK(out->n_terms < VEXB_MAX_TERMS, "too many terminals"); xs = out->n_terms++; out->term[xs] = xt; memset(out->term[xs].pad, 0, sizeof(xt.pad)); }
                remap[t.pad[0]] = xs;
                for (int j = 0; j < out->n_terms; ++j)
                    if (out->term[j].kind == t.kind && out->term[j].v.ptr == t.v.ptr && out->term[j].pad[0] == xs &&
                        (t.kind != VEXB_TERM_CCSR || out->term[j].pad[1] == t.pad[1])) { slot = j; break; }
                if (slot < 0) {
                    VEXB_CHECK(out->n_terms < VEXB_MAX_TERMS, "too many terminals");
                    slot = out->n_terms++; out->term[slot] = t; memset(out->term[slot].pad, 0, sizeof(t.pad));
                    out->term[slot].pad[0] = (uint8_t)xs;
                    if (t.kind == VEXB_TERM_CCSR) out->term[slot].pad[1] = t.pad[1];      // idx width
                }
            }
            if (slot < 0) { slot = out->n_terms++; out->term[slot] = t; if (t.kind != VEXB_TERM_PTR) memset(out->term[slot].pad, 0, sizeof(t.pad)); }
            remap[ins.arg] = slot;
            ins.arg = (uint16_t)slot;
            ins.type = (t.kind == VEXB_TERM_INDEX) ? VEXB_U64 : t.kind == VEXB_TERM_PTR ? VEXB_PTR(t.dtype) : t.dtype;
        } else if (ins.op == VEXB_OP_CVT) {
            VEXB_CHECK(ins.arg <= VEXB_U64, "instr %d: bad CVT source type", pc);
            // 2. fold a conversion applied directly to a scalar terminal.
            if (out->n_code > 0) {
                vexb_instr &prev = out->code[out->n_code - 1];
                if (prev.op == VEXB_OP_TERM && out->term[prev.arg].kind == VEXB_TERM_SCALAR) {
                    vexb_term t = out->term[prev.arg];
                    convert_scalar_term(t, ins.type);
                    int refs = 0;                                        // other pushes of the same scalar slot keep its old type
                    for (int q = 0; q < out->n_code; ++q) if (out->code[q].op == VEXB_OP_TERM && out->code[q].arg == prev.arg) ++refs;
                    bool shared = refs > 1;
                    for (int q = 0; !shared && q < VEXB_MAX_TERMS; ++q) if (remap[q] == (int)prev.arg) {
                        // a later instruction of the input may push this input slot again: look ahead
                        for (int r = pc + 1; r < in->n_code; ++r) if (in->code[r].op == VEXB_OP_TERM && in->code[r].arg == q) shared = true;
                    }
                    if (!shared) {
                        out->term[prev.arg] = t;                          // referenced once: fold in place, no new slot
                        for (int q = 0; q < VEXB_MAX_TERMS; ++q) if (remap[q] == (int)prev.arg) remap[q] = -1;
                    } else {
                        VEXB_CHECK(out->n_terms < VEXB_MAX_TERMS, "too many terminals");
                        const int slot = out->n_terms++;
                        out->term[slot] = t;
                        prev.arg = (uint16_t)slot;
                    }
                    prev.type = ins.type;
                    stype[depth - 1] = ins.type;
                    continue;
                }
            }
            if (ins.arg == ins.type) continue; // no-op conversion
        } else if (ins.op >= VEXB_OP_BAND && ins.op <= VEXB_OP_SHR) {
            VEXB_CHECK(!dtype_is_float(ins.type), "instr %d: bitwise op on floating type", pc);
        } else if ((ins.op >= VEXB_OP_SIN && ins.op <= VEXB_OP_TRUNC && ins.op != VEXB_OP_FABS) ||
                   (ins.op >= VEXB_OP_POW && ins.op <= VEXB_OP_HYPOT) || ins.op == VEXB_OP_FMA) {
            VEXB_CHECK(dtype_is_float(ins.type), "instr %d: math function on integer type", pc);
        }
        depth += 1 - ar;
        if (depth > maxdepth) maxdepth = depth;
        stype[depth - 1] = ((ins.op >= VEXB_OP_LT && ins.op <= VEXB_OP_LOR) || ins.op == VEXB_OP_LNOT) ? VEXB_I32 : ins.type;
        out->code[out->n_code++] = ins;
    }
    VEXB_CHECK(depth == 1, "program leaves %d values on the stack (expected 1)", depth);
    VEXB_CHECK(!is_ptr_type(stype[0]), "the result of a program is a value, not a raw pointer");
    VEXB_CHECK(maxdepth <= VEXB_MAX_STACK, "expression too deep (%d > %d)", maxdepth, VEXB_MAX_STACK);
    // 3. compact away scalar slots orphaned by folding
    bool used[VEXB_MAX_TERMS] = {false};
    auto names_term = [](int op) { return op == VEXB_OP_TERM || op == VEXB_OP_LOAD; };
    for (int pc = 0; pc < out->n_code; ++pc) if (names_term(out->code[pc].op)) used[out->code[pc].arg] = true;
    for (int k = 0; k < out->n_terms; ++k) if (used[k] && is_product_term(out->term[k].kind)) used[out->term[k].pad[0]] = true;
    int newslot[VEXB_MAX_TERMS]; int n = 0;
    for (int k = 0; k < out->n_terms; ++k) newslot[k] = used[k] ? n++ : -1;
    for (int k = 0; k < out->n_terms; ++k) if (used[k] && is_product_term(out->term[k].kind)) out->term[k].pad[0] = (uint8_t)newslot[out->term[k].pad[0]];
    for (int k = 0; k < out->n_terms; ++k) if (used[k] && newslot[k] != k) out->term[newslot[k]] = out->term[k];
    for (int k = n; k < out->n_terms; ++k) memset(&out->term[k], 0, sizeof(vexb_term));
    out->n_terms = n;
    for (int pc = 0; pc < out->n_code; ++pc) if (names_term(out->code[pc].op)) out->code[pc].arg = (uint16_t)newslot[out->code[pc].arg];
    return VEXB_OK;
}

// Shapes with a hand-written kernel body.  v* are vector terminals, s* scalars.
enum ShapeId {
    SH_COPY,    // v0
    SH_FILL,    // s0
    SH_ADD,     // v0 + v1
    SH_SUB,     // v0 - v1
    SH_MUL,     // v0 * v1
    SH_DIV,     // v0 / v1
    SH_SQR,     // v0 * v0
    SH_SCALE,   // s0 * v0
    SH_MULADD,  // v0 + v1 * v2         (a = b + c*d, north_star / benchmark.cpp:171-176)
    SH_AXPY,    // s0 * v0 + v1         (SAXPY a = alpha*a + b, benchmark.cpp:102-107)
    SH_XPAY,    // v0 + s0 * v1         (CG update p = r + beta*p)
    SH_XMAY,    // v0 - s0 * v1         (CG update r = r - alpha*q)
    SH_AXPBY,   // s0 * v0 + s1 * v1
    SH_ABSDIFF, // fabs(v0 - v1)        (reductions: max(fabs(x - y)))
    SH_NONE
};

struct ShapeMatch {
    int shape = SH_NONE;
    int vslot[3] = {-1, -1, -1};   // term slot feeding v0..v2
    int sslot[2] = {-1, -1};       // term slot feeding s0..s1
};

// Signature: terminals numbered by first appearance ("V0", "S0"), ops as symbols.
inline std::string expr_signature(const vexb_expr &e, int T, int (&vs)[VEXB_MAX_TERMS], int (&ss)[VEXB_MAX_TERMS], int &nv, int &ns) {
    std::string sig; nv = ns = 0;
    int vnum[VEXB_MAX_TERMS], snum[VEXB_MAX_TERMS];
    for (int k = 0; k < VEXB_MAX_TERMS; ++k) vnum[k] = snum[k] = -1;
    for (int pc = 0; pc < e.n_code; ++pc) {
        const vexb_instr &in = e.code[pc];
        if (in.op == VEXB_OP_TERM) {
            const vexb_term &t = e.term[in.arg];
            if (t.dtype != T) return "";
            if (t.kind == VEXB_TERM_VEC) {
                if (vnum[in.arg] < 0) { vnum[in.arg] = nv; vs[nv++] = in.arg; }
                sig += "V"; sig += char('0' + vnum[in.arg]);
            } else if (t.kind == VEXB_TERM_SCALAR || t.kind == VEXB_TERM_DSCALAR) {
                if (snum[in.arg] < 0) { snum[in.arg] = ns; ss[ns++] = in.arg; }
                sig += "S"; sig += char('0' + snum[in.arg]);
            } else return "";
        } else {
            if (in.type != T) return "";
            switch (in.op) {
                case VEXB_OP_ADD: sig += "+"; break;
                case VEXB_OP_SUB: sig += "-"; break;
                case VEXB_OP_MUL: sig += "*"; break;
                case VEXB_OP_DIV: sig += "/"; break;
                case VEXB_OP_FABS: sig += "|"; break;
                default: return "";
            }
        }
        sig += " ";
    }
    return sig;
}

inline ShapeMatch match_shape(const vexb_expr &e, int T) {
    struct Entry { const char *sig; int shape; int vperm[3]; int sperm[2]; };
    // vperm[j] = which signature vector number feeds shape input v_j.
    static const Entry table[] = {
        {"V0 ",                 SH_COPY,   {0, -1, -1}, {-1, -1}},
        {"S0 ",                 SH_FILL,   {-1, -1, -1}, {0, -1}},
        {"V0 V1 + ",            SH_ADD,    {0, 1, -1}, {-1, -1}},
        {"V0 V1 - ",            SH_SUB,    {0, 1, -1}, {-1, -1}},
        {"V0 V1 * ",            SH_MUL,    {0, 1, -1}, {-1, -1}},
        {"V0 V1 / ",            SH_DIV,    {0, 1, -1}, {-1, -1}},
        {"V0 V0 * ",            SH_SQR,    {0, -1, -1}, {-1, -1}},
        {"S0 V0 * ",            SH_SCALE,  {0, -1, -1}, {0, -1}},
        {"V0 S0 * ",            SH_SCALE,  {0, -1, -1}, {0, -1}},
        {"V0 V1 V2 * + ",       SH_MULADD, {0, 1, 2}, {-1, -1}},   // b + c*d
        {"V0 V1 * V2 + ",       SH_MULADD, {2, 0, 1}, {-1, -1}},   // c*d + b
        {"S0 V0 * V1 + ",       SH_AXPY,   {0, 1, -1}, {0, -1}},   // alpha*a + b
        {"V0 S0 * V1 + ",       SH_AXPY,   {0, 1, -1}, {0, -1}},   // a*alpha + b
        {"V0 S0 V1 * + ",       SH_XPAY,   {0, 1, -1}, {0, -1}},   // r + beta*p
        {"V0 V1 S0 * + ",       SH_XPAY,   {0, 1, -1}, {0, -1}},   // r + p*beta
        {"V0 S0 V1 * - ",       SH_XMAY,   {0, 1, -1}, {0, -1}},   // r - alpha*q
        {"V0 V1 S0 * - ",       SH_XMAY,   {0, 1, -1}, {0, -1}},
        {"S0 V0 * S1 V1 * + ",  SH_AXPBY,  {0, 1, -1}, {0, 1}},
        {"V0 V1 - | ",          SH_ABSDIFF,{0, 1, -1}, {-1, -1}},
    };
    ShapeMatch m;
    int vs[VEXB_MAX_TERMS], ss[VEXB_MAX_TERMS], nv, ns;
    const std::string sig = expr_signature(e, T, vs, ss, nv, ns);
    if (sig.empty()) return m;
    for (const Entry &en : table) {
        if (sig == en.sig) {
            m.shape = en.shape;
            for (int j = 0; j < 3; ++j) m.vslot[j] = en.vperm[j] >= 0 ? vs[en.vperm[j]] : -1;
            for (int j = 0; j < 2; ++j) m.sslot[j] = en.sperm[j] >= 0 ? ss[en.sperm[j]] : -1;
            return m;
        }
    }
    return m;
}

inline const char *shape_name(int s) {
    static const char *names[] = {"copy", "fill", "add", "sub", "mul", "div", "sqr", "scale", "muladd",
                                  "axpy", "xpay", "xmay", "axpby", "absdiff", "none"};
    return (s >= 0 && s <= SH_NONE) ? names[s] : "?";
}

} // namespace vexb
