// NVRTC side path: expressions that call user-defined functions (VEX_FUNCTION, vexcl/function.hpp:225)
// cannot be served by pre-compiled kernels, because the function body is C source supplied at run time.
// For those -- and, opt-in through the tunable "eval.jit", for any expression that has no hand-written
// sweep -- the IR is printed as CUDA C (one statement per IR instruction), compiled ONCE with NVRTC for
// sm_90a (--fmad=false, so results stay bit-identical to the interpreter and the unfused CPU loop),
// kept in the program cache that every run-time kernel shares (jit_program), and launched through the
// driver API on the caller's stream.  This is the only place where the build resembles the reference's
// run-time code generation (vexcl/operations.hpp:1841-1884, vexcl/backend/cuda/compiler.hpp:53-115); it
// needs libnvrtc and libcuda at run time, both dlopen()ed.
#include "exprhost.hpp"
#include "jit.hpp"
#include "spmat.hpp"
#include "ccsr.hpp"
#include "peer.cuh"
#include "fold_text.inc"       // kFoldText: csrc/fold.cuh byte for byte, stringified by vexcl_b200/build.py
#include <dlfcn.h>
#include <algorithm>
#include <cctype>
#include <map>
#include <mutex>
#include <condition_variable>
#include <memory>
#include <functional>
#include <thread>
#include <sstream>
#include <vector>

namespace vexb {

// deps: ids of functions registered earlier, which the body calls by their plain names; preamble: file-scope text
// (helpers, macros) that the body may use (VEX_FUNCTION_D / _SD, VEX_FUNCTION_V1_WITH_PREAMBLE, vexcl/function.hpp).
struct UserFunc { std::string name; int ret; std::vector<int> args; std::string body; std::vector<int> deps; std::string preamble; };
static std::mutex g_fmx;
static std::vector<UserFunc> g_funcs;
constexpr int kMaxDeps = 64;                        // entries of one dependency list

// Program headers (vex::push_program_header, backend/common.hpp): a stack per device ordinal.  A push replaces the
// effective header (the top), a pop restores the one before.  It goes at the very top of every program compiled for that
// device that carries user text, and is part of those kernels' cache keys.
constexpr int kMaxHeaderDevices = 1024;
static std::mutex g_hdr_mx;
static std::map<int, std::vector<std::string>> g_headers;

std::string program_header(int dev) {
    std::lock_guard<std::mutex> l(g_hdr_mx);
    auto it = g_headers.find(dev);
    return it == g_headers.end() || it->second.empty() ? std::string() : it->second.back();
}

// `src` with `header` at its very top (on a line of its own); `src` itself when the header is empty.
static std::string with_program_header(const std::string &header, const std::string &src) {
    if (header.empty()) return src;
    return header + (header.back() == '\n' ? "" : "\n") + src;
}

int function_arity(int id) { std::lock_guard<std::mutex> l(g_fmx); return (id >= 0 && id < (int)g_funcs.size()) ? (int)g_funcs[id].args.size() : -1; }
int function_arg_dtype(int id, int k) { std::lock_guard<std::mutex> l(g_fmx); return g_funcs[id].args[k]; }
int function_ret_dtype(int id) { std::lock_guard<std::mutex> l(g_fmx); return (id >= 0 && id < (int)g_funcs.size()) ? g_funcs[id].ret : -1; }

static const char *ctype(int dt) {
    switch (dt) {
        case VEXB_F64: return "double"; case VEXB_F32: return "float"; case VEXB_I32: return "int";
        case VEXB_U32: return "unsigned int"; case VEXB_I64: return "long long"; default: return "unsigned long long";
    }
}
static const char *ufield(int dt) {
    switch (dt) {
        case VEXB_F64: return "f64"; case VEXB_F32: return "f32"; case VEXB_I32: return "i32";
        case VEXB_U32: return "u32"; case VEXB_I64: return "i64"; default: return "u64";
    }
}
// A parameter type of a user function: the value types, and `T *` for VEXB_PTR(T).
static std::string param_ctype(int dt) { return is_ptr_type(dt) ? std::string(ctype(dt & ~VEXB_PTR(0))) + " *" : std::string(ctype(dt)); }
static bool is_f(int t) { return t == VEXB_F64 || t == VEXB_F32; }
static bool is_signed(int t) { return t == VEXB_I32 || t == VEXB_I64; }

static const char *math_name(int op) {
    switch (op) {
        case VEXB_OP_SIN: return "sin"; case VEXB_OP_COS: return "cos"; case VEXB_OP_TAN: return "tan";
        case VEXB_OP_ASIN: return "asin"; case VEXB_OP_ACOS: return "acos"; case VEXB_OP_ATAN: return "atan";
        case VEXB_OP_SINH: return "sinh"; case VEXB_OP_COSH: return "cosh"; case VEXB_OP_TANH: return "tanh";
        case VEXB_OP_EXP: return "exp"; case VEXB_OP_EXP2: return "exp2"; case VEXB_OP_LOG: return "log";
        case VEXB_OP_LOG2: return "log2"; case VEXB_OP_LOG10: return "log10"; case VEXB_OP_SQRT: return "sqrt";
        case VEXB_OP_RSQRT: return "rsqrt"; case VEXB_OP_CBRT: return "cbrt"; case VEXB_OP_FABS: return "fabs";
        case VEXB_OP_FLOOR: return "floor"; case VEXB_OP_CEIL: return "ceil"; case VEXB_OP_ROUND: return "round";
        case VEXB_OP_TRUNC: return "trunc"; case VEXB_OP_POW: return "pow"; case VEXB_OP_ATAN2: return "atan2";
        case VEXB_OP_FMOD: return "fmod"; case VEXB_OP_HYPOT: return "hypot"; case VEXB_OP_FMIN: return "fmin";
        case VEXB_OP_FMAX: return "fmax"; case VEXB_OP_FMA: return "fma";
    }
    return "";
}

// The user functions of a program.  A function the expression calls is emitted as name_<id>, after the closure of its
// dependency lists: post-order over the lists as written, every function of it once and under its plain name, the name
// its dependents' bodies use (so a called function that is also a dependency appears under both names).  A function's
// preamble goes once, before its first definition.  Two distinct functions with one plain name are refused here, before
// NVRTC sees the program.  Without dependencies and preambles the text is that of the called functions alone.
static int emit_user_functions(const vexb_expr *const *es, int ncomp, std::ostream &s) {
    std::lock_guard<std::mutex> l(g_fmx);
    const size_t nf = g_funcs.size();
    std::vector<bool> called(nf, false), plain(nf, false), pre(nf, false);
    std::map<std::string, int> plain_ids;
    auto define = [&](int id, bool as_plain) {
        const UserFunc &f = g_funcs[id];
        if (!f.preamble.empty() && !pre[id]) {
            pre[id] = true;
            s << f.preamble << (f.preamble.back() == '\n' ? "" : "\n");
        }
        s << "__device__ __forceinline__ " << ctype(f.ret) << " " << f.name;
        if (!as_plain) s << "_" << id;
        s << "(";
        for (size_t k = 0; k < f.args.size(); ++k) s << (k ? ", " : "") << param_ctype(f.args[k]) << " prm" << (k + 1);
        s << ") {\n" << f.body << "\n}\n";
    };
    std::function<int(int)> dependency = [&](int id) -> int {
        if (plain[id]) return VEXB_OK;
        plain[id] = true;
        auto ins = plain_ids.emplace(g_funcs[id].name, id);
        if (!ins.second) VEXB_FAIL(VEXB_ERR_INVALID, "user functions %d and %d are both named '%s' among the dependencies of one program",
                                   ins.first->second, id, g_funcs[id].name.c_str());
        for (int d : g_funcs[id].deps) VEXB_TRY(dependency(d));
        define(id, true);
        return VEXB_OK;
    };
    for (int comp = 0; comp < ncomp; ++comp)
        for (int pc = 0; pc < es[comp]->n_code; ++pc) if (es[comp]->code[pc].op == VEXB_OP_CALL && !called[es[comp]->code[pc].arg]) {
            const int id = es[comp]->code[pc].arg; called[id] = true;
            for (int d : g_funcs[id].deps) VEXB_TRY(dependency(d));
            define(id, false);
        }
    return VEXB_OK;
}

// Whether a program needs NVRTC's --device-as-default-execution-space: some function it calls, or one of their
// dependencies, has a preamble, whose helpers are written without __device__ (the reference's own example does so).
static bool program_has_preamble(const vexb_expr *const *es, int ncomp) {
    std::lock_guard<std::mutex> l(g_fmx);
    std::vector<bool> seen(g_funcs.size(), false);
    std::function<bool(int)> walk = [&](int id) {
        if (seen[id]) return false;
        seen[id] = true;
        if (!g_funcs[id].preamble.empty()) return true;
        for (int d : g_funcs[id].deps) if (walk(d)) return true;
        return false;
    };
    for (int comp = 0; comp < ncomp; ++comp)
        for (int pc = 0; pc < es[comp]->n_code; ++pc)
            if (es[comp]->code[pc].op == VEXB_OP_CALL && walk(es[comp]->code[pc].arg)) return true;
    return false;
}

// The header of device `dev` for a program, or "" when the program carries no user text (no call) or dev < 0 (the
// source printers without a device).
static std::string header_for(int dev, const vexb_expr *const *es, int ncomp) {
    if (dev < 0) return std::string();
    for (int comp = 0; comp < ncomp; ++comp) if (expr_has_call(*es[comp])) return program_header(dev);
    return std::string();
}

// A cache key extended by the header it was compiled under; keys of programs without a header stay as they were.
static std::string key_with_header(std::string key, const std::string &header) {
    if (!header.empty()) { key.push_back('\0'); key += "header:"; key += header; }
    return key;
}

// Print a normalised program as CUDA C.  One `const T rK = ...;` per instruction keeps the text linear in
// the program length; the semantics of every operator mirror csrc/expr_eval.cuh.
// ncomp > 1: the components of a multi-expression assignment (vex::tie(a, b) = std::tie(e0, e1), multivector
// arithmetic; assign_multiexpression, vexcl/operations.hpp:2081-2185) in ONE kernel: every right-hand side of element i
// is evaluated -- all its loads done -- before any left-hand side of element i is stored, which is the reference's
// buf_k rule (operations.hpp:2143-2157) and makes temporaries for `tie(x, y) = (x + y, y - x)` unnecessary.
// The part shared by the elementwise and the reduction kernels: terminal table, user functions, sparse row functions and
// one vexb_elem function per component (element i of the right-hand side, converted to the lhs type).
// A request whose products include a sliced-ELL strip is swept in that strip's storage order (generate_source_n), so it
// holds at most one distinct such strip, any number of times.  *term: the first terminal on it, -1 when there is none.
static int sell_sweep_term(const vexb_expr &e, int *term) {
    *term = -1;
    for (int k = 0; k < e.n_terms; ++k) if (e.term[k].kind == VEXB_TERM_SPMV) {
        const vexb_spmat *A = static_cast<const vexb_spmat *>(e.term[k].v.ptr);
        if (!A || A->fmt != VEXB_FMT_SELL) continue;
        if (*term < 0) *term = k;
        else if (e.term[*term].v.ptr != A) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "term %d: a second sliced-ELL strip in one expression (the kernel sweeps in the storage order of one)", k);
    }
    return VEXB_OK;
}

// Whether a kernel passes a raw pointer to a user function (a VEXB_OP_TERM on a VEXB_TERM_PTR), whose body may write
// through it: the kernel's loads then take the plain path, not the read-only one.
static bool passes_pointers(const vexb_expr *const *es, int ncomp) {
    for (int c = 0; c < ncomp; ++c)
        for (int pc = 0; pc < es[c]->n_code; ++pc)
            if (es[c]->code[pc].op == VEXB_OP_TERM && es[c]->term[es[c]->code[pc].arg].kind == VEXB_TERM_PTR) return true;
    return false;
}

// Print instructions [from, to) of a normalised program as CUDA C onto the value stack `st`: one `const T rPC = ...;` per
// instruction, whose semantics mirror csrc/expr_eval.cuh.  A TDEF prints `const T tK = <top>;` and names slot K tK; a
// TREF pushes tnames[K], which is tK or the parameter that carries the value in (multi-expression kernels).  A pointer
// argument pushes `(T *)tt.t[K].v.ptr`; a LOAD reads through the read-only path when `ldg` (nothing in the kernel
// writes the array), else with a plain load.
static void print_code(const vexb_expr &e, int from, int to, std::string (&tnames)[VEXB_MAX_TEMPS], std::ostream &s,
                       std::vector<std::pair<std::string, int>> &st, bool ldg = true) {
    for (int pc = from; pc < to; ++pc) {
        const vexb_instr &in = e.code[pc];
        const int op = in.op, t = in.type;
        std::ostringstream r;
        int rt = t;
        auto pop = [&]() { auto v = st.back(); st.pop_back(); return v; };
        if (op == VEXB_OP_TDEF) {
            tnames[in.arg] = "t" + std::to_string(in.arg);
            s << "    const " << ctype(t) << " " << tnames[in.arg] << " = " << pop().first << ";\n";
            continue;
        }
        if (op == VEXB_OP_TREF) { st.emplace_back(tnames[in.arg], t); continue; }
        if (op == VEXB_OP_TERM && e.term[in.arg].kind == VEXB_TERM_PTR) {
            st.emplace_back(std::string("(") + ctype(e.term[in.arg].dtype) + " *)tt.t[" + std::to_string(in.arg) + "].v.ptr", t);
            continue;
        }
        if (op == VEXB_OP_LOAD) {                       // 0 outside [0, count): a guarded load never touches what its guard excludes
            const std::string k = std::to_string(in.arg), idx = pop().first;
            const std::string p = std::string("(const ") + ctype(t) + " *)tt.t[" + k + "].v.ptr + " + idx;
            r << "(unsigned long long)" << idx << " < vexb_count(tt.t[" << k << "]) ? " << (ldg ? "__ldg(" + p + ")" : "*(" + p + ")")
              << " : (" << ctype(t) << ")0";
        } else if (op == VEXB_OP_TERM) {
            const vexb_term &tm = e.term[in.arg];
            const int k = in.arg;
            rt = tm.kind == VEXB_TERM_INDEX ? VEXB_U64 : tm.dtype;
            if (tm.kind == VEXB_TERM_VEC) r << "__ldcs((const " << ctype(rt) << " *)tt.t[" << k << "].v.ptr + i)";
            else if (tm.kind == VEXB_TERM_DSCALAR) r << "*(const " << ctype(rt) << " *)tt.t[" << k << "].v.ptr";
            else if (tm.kind == VEXB_TERM_SPMV) r << "spmv_" << k << "((const spmv_desc_j *)tt.t[" << k << "].v.ptr, (const " << ctype(rt)
                                                  << " *)tt.t[" << (int)tm.pad[0] << "].v.ptr, i"
                                                  << (static_cast<const vexb_spmat *>(tm.v.ptr)->fmt == VEXB_FMT_SELL ? ", t)" : ")");
            else if (tm.kind == VEXB_TERM_CCSR) r << "ccsr_" << k << "((const ccsr_desc_j *)tt.t[" << k << "].v.ptr, (const " << ctype(rt)
                                                  << " *)tt.t[" << (int)tm.pad[0] << "].v.ptr, i)";
            else if (tm.kind == VEXB_TERM_SCALAR) r << "tt.t[" << k << "].v." << ufield(rt);
            else r << "off + i + (unsigned long long)tt.t[" << k << "].v.i64";
        } else if (op == VEXB_OP_CVT) {
            auto a = pop(); r << "(" << ctype(t) << ")" << a.first;
        } else if (op == VEXB_OP_NEG) {
            auto a = pop(); r << "-" << a.first;
        } else if (op == VEXB_OP_LNOT) {
            auto a = pop(); rt = VEXB_I32; r << "(int)!" << a.first;
        } else if (op == VEXB_OP_SELECT) {
            auto c = pop(), b = pop(), a = pop();
            r << "(" << a.first << " != 0) ? " << b.first << " : " << c.first;
        } else if (op == VEXB_OP_FMA) {
            auto c = pop(), b = pop(), a = pop();
            r << (t == VEXB_F32 ? "fmaf(" : "fma(") << a.first << ", " << b.first << ", " << c.first << ")";
        } else if (op == VEXB_OP_CALL) {
            std::vector<std::string> args(function_arity(in.arg));
            for (int k = (int)args.size() - 1; k >= 0; --k) args[k] = pop().first;
            std::string nm; { std::lock_guard<std::mutex> l(g_fmx); nm = g_funcs[in.arg].name; }
            r << nm << "_" << in.arg << "(";
            for (size_t k = 0; k < args.size(); ++k) r << (k ? ", " : "") << args[k];
            r << ")";
        } else if ((op >= VEXB_OP_ADD && op <= VEXB_OP_LOR) || (op >= VEXB_OP_POW && op <= VEXB_OP_FMAX)) {
            auto b = pop(), a = pop();
            const std::string &x = a.first, &y = b.first;
            const int bits = (t == VEXB_I32 || t == VEXB_U32) ? 31 : 63;
            switch (op) {
                case VEXB_OP_ADD: r << x << " + " << y; break;
                case VEXB_OP_SUB: r << x << " - " << y; break;
                case VEXB_OP_MUL: r << x << " * " << y; break;
                case VEXB_OP_DIV:
                    if (is_f(t)) r << x << " / " << y;
                    else if (is_signed(t)) r << "(" << y << " == 0) ? 0 : (" << y << " == -1 ? (" << ctype(t) << ")(0 - (unsigned " << (t == VEXB_I32 ? "int" : "long long") << ")" << x << ") : " << x << " / " << y << ")";
                    else r << "(" << y << " == 0) ? 0 : " << x << " / " << y;
                    break;
                case VEXB_OP_MOD: case VEXB_OP_FMOD:
                    if (is_f(t)) r << (t == VEXB_F32 ? "fmodf(" : "fmod(") << x << ", " << y << ")";
                    else if (is_signed(t)) r << "(" << y << " == 0 || " << y << " == -1) ? 0 : " << x << " % " << y;
                    else r << "(" << y << " == 0) ? 0 : " << x << " % " << y;
                    break;
                case VEXB_OP_BAND: r << x << " & " << y; break;
                case VEXB_OP_BOR:  r << x << " | " << y; break;
                case VEXB_OP_BXOR: r << x << " ^ " << y; break;
                case VEXB_OP_SHL:  r << x << " << (" << y << " & " << bits << ")"; break;
                case VEXB_OP_SHR:  r << x << " >> (" << y << " & " << bits << ")"; break;
                case VEXB_OP_LT: rt = VEXB_I32; r << "(int)(" << x << " < " << y << ")"; break;
                case VEXB_OP_GT: rt = VEXB_I32; r << "(int)(" << x << " > " << y << ")"; break;
                case VEXB_OP_LE: rt = VEXB_I32; r << "(int)(" << x << " <= " << y << ")"; break;
                case VEXB_OP_GE: rt = VEXB_I32; r << "(int)(" << x << " >= " << y << ")"; break;
                case VEXB_OP_EQ: rt = VEXB_I32; r << "(int)(" << x << " == " << y << ")"; break;
                case VEXB_OP_NE: rt = VEXB_I32; r << "(int)(" << x << " != " << y << ")"; break;
                case VEXB_OP_LAND: rt = VEXB_I32; r << "(int)((" << x << " != 0) && (" << y << " != 0))"; break;
                case VEXB_OP_LOR:  rt = VEXB_I32; r << "(int)((" << x << " != 0) || (" << y << " != 0))"; break;
                case VEXB_OP_FMIN: case VEXB_OP_FMAX:
                    if (is_f(t)) r << math_name(op) << (t == VEXB_F32 ? "f(" : "(") << x << ", " << y << ")";
                    else r << "(" << x << (op == VEXB_OP_FMIN ? " < " : " > ") << y << ") ? " << x << " : " << y;
                    break;
                default: r << math_name(op) << (t == VEXB_F32 ? "f(" : "(") << x << ", " << y << ")"; break;
            }
        } else {    // unary math
            auto a = pop();
            if (op == VEXB_OP_FABS && !is_f(t)) {
                if (is_signed(t)) r << "(" << a.first << " < 0) ? (" << ctype(t) << ")(0 - (unsigned " << (t == VEXB_I32 ? "int" : "long long") << ")" << a.first << ") : " << a.first;
                else r << a.first;
            } else r << math_name(op) << (t == VEXB_F32 ? "f(" : "(") << a.first << ")";
        }
        std::string name = "r" + std::to_string(pc);
        s << "    const " << ctype(rt) << " " << name << " = " << r.str() << ";\n";
        st.emplace_back(name, rt);
    }
}

// The temporaries of a multi-expression assignment.  Each component's slots are its own; a temporary that several
// components define by the same instructions over equal terminals (same kind, dtype and pointer or value) is one class,
// which the kernel computes once per element and hands to every component that reads it (`vex::tie(a, b) =
// std::tie(t, sqrt(1 - t*t))` evaluates t once).  Classes are numbered in the order components define them, so a class
// comes after the classes its definition reads.
struct TempClasses {
    int cls[8][VEXB_MAX_TEMPS];                         // class of component c's slot k, -1 where c does not define k
    std::vector<int> comp, from, to, type;              // class g: defined by instructions [from, to) of component comp
    std::vector<std::vector<int>> reads;                // class g: the classes its definition reads, in order of first use
};

static TempClasses temp_classes(const vexb_expr *const *es, int ncomp) {
    TempClasses tc;
    std::vector<std::string> keys;
    for (int c = 0; c < ncomp; ++c) {
        const vexb_expr &e = *es[c];
        for (int k = 0; k < VEXB_MAX_TEMPS; ++k) tc.cls[c][k] = -1;
        std::string key;                                // the definition of the next TDEF, terminals by content
        int from = 0;
        for (int pc = 0; pc < e.n_code; ++pc) {
            const vexb_instr &in = e.code[pc];
            if (in.op == VEXB_OP_TDEF) {
                key.push_back((char)in.type);
                int g = 0;
                while (g < (int)keys.size() && keys[g] != key) ++g;
                if (g == (int)keys.size()) {
                    keys.push_back(key);
                    tc.comp.push_back(c); tc.from.push_back(from); tc.to.push_back(pc); tc.type.push_back(in.type);
                    std::vector<int> reads;
                    for (int q = from; q < pc; ++q) if (e.code[q].op == VEXB_OP_TREF) {
                        const int j = tc.cls[c][e.code[q].arg];
                        if (std::find(reads.begin(), reads.end(), j) == reads.end()) reads.push_back(j);
                    }
                    tc.reads.push_back(reads);
                }
                tc.cls[c][in.arg] = g;
                key.clear();
                from = pc + 1;
                continue;
            }
            key.push_back((char)in.op); key.push_back((char)in.type);
            if (in.op == VEXB_OP_TERM || in.op == VEXB_OP_LOAD) key.append(reinterpret_cast<const char *>(&e.term[in.arg]), sizeof(vexb_term));
            else if (in.op == VEXB_OP_TREF) key += "#" + std::to_string(tc.cls[c][in.arg]);
            else { key.push_back((char)(in.arg & 0xff)); key.push_back((char)(in.arg >> 8)); }
        }
    }
    return tc;
}

// sell: where the terminal of the request's sliced-ELL strip goes (sell_sweep_term); NULL for the callers that do not
// sweep in storage order (reductions), which refuse such strips.
static int generate_elements(const vexb_expr *const *es, int ncomp, int lhs_dtype, int aop, std::ostringstream &s, bool *spmv, int *sell = nullptr) {
    const vexb_expr &e = *es[0];
    if (sell) VEXB_TRY(sell_sweep_term(e, sell));
    const bool sweep = sell && *sell >= 0 && ncomp == 1;
    s << "// generated by libvexb200 (csrc/jit.cu)\n"
         "struct term_j { unsigned char kind, dtype, pad[6]; union { const void *ptr; double f64; float f32; int i32;"
         " unsigned int u32; long long i64; unsigned long long u64; } v; };\n"
         "struct terms_j { term_j t[" << VEXB_MAX_TERMS << "]; };\n";
    bool loads = false;
    for (int comp = 0; comp < ncomp; ++comp) loads = loads || expr_has_load(*es[comp]);
    if (loads)                                          // the element count of a pointer terminal (pad[0..5], VEXB_TERM_PTR)
        s << "__device__ __forceinline__ unsigned long long vexb_count(const term_j &t) {\n"
             "  unsigned long long c = 0;\n  for (int b = 5; b >= 0; --b) c = c << 8 | t.pad[b];\n  return c;\n}\n";
    VEXB_TRY(emit_user_functions(es, ncomp, s));
    // sparse products used as terminals (VEXB_TERM_SPMV): one row function per terminal, specialised to the strip's format
    // -- hybrid ELL with the width as a literal (fully unrolled: all column/value loads, then all gathers of x, in
    // flight at once, like hell_kernel), 32-bit columns, 16-bit offsets, slot masks or row classes, with or without a CSR tail; or plain CSR, one thread per
    // row.  Products and sums are separate operations (--fmad=false) added in storage order: same bits as vexb_spmv.
    bool any_spmv = false;
    for (int comp = 1; comp < ncomp; ++comp)
        for (int k = 0; k < es[comp]->n_terms; ++k)
            VEXB_CHECK(!is_product_term(es[comp]->term[k].kind), "sparse products are not fused into multi-expression kernels");
    for (int k = 0; k < e.n_terms; ++k) if (e.term[k].kind == VEXB_TERM_SPMV) {
        VEXB_CHECK(ncomp == 1, "sparse products are not fused into multi-expression kernels");
        const vexb_spmat *A = static_cast<const vexb_spmat *>(e.term[k].v.ptr);
        VEXB_CHECK(A && (A->fmt == VEXB_FMT_CSR || A->fmt == VEXB_FMT_HELL || (A->fmt == VEXB_FMT_SELL && sweep)) && !A->row_ids && A->y_offset == 0 && A->d_desc,
                   "term %d: this strip cannot be inlined into an expression (format / row map)", k);
        VEXB_CHECK(A->val_dtype == e.term[k].dtype, "term %d: value type of the matrix differs from the terminal's", k);
        VEXB_CHECK(!A->val_f32, "term %d: a strip with float values (VEXB_FMT_VALUES_F32) cannot be inlined into an expression", k);
        const char *T = ctype(e.term[k].dtype);
        if (!any_spmv) {
            s << "struct spmv_desc_j { const void *ell_col; const void *ell_val; const int *tail_ptr; const int *tail_col; const void *tail_val;\n"
                 "                     const int *rowptr; const int *col; const void *val; unsigned long long pitch; int width; int shifts[" << kEllShiftSlots << "]; int x_max;\n"
                 "                     const int *slice_ptr; const int *perm; const void *sell_col; const void *sell_val; int sell_shift; unsigned long long n_slices; };\n";
            any_spmv = true;
        }
        s << "__device__ __forceinline__ " << T << " spmv_" << k << "(const spmv_desc_j *__restrict__ m, const " << T
          << " *__restrict__ x, unsigned long long i" << (A->fmt == VEXB_FMT_SELL ? ", unsigned long long t" : "") << ") {\n  " << T << " sum = 0;\n";
        if (A->fmt == VEXB_FMT_SELL) {
            // sell_kernel's loop for stored lane t (slice t >> 5, lane t & 31), which holds row i: 4 slots a turn -- their
            // column and value loads, then the gathers -- then the remainder
            const bool c16 = A->sell_col16 != nullptr;
            const char *CT = c16 ? "short" : "int";
            const char *dec = c16 ? "raw == (short)-32768 ? -1 : rs + (int)raw" : "raw";
            s << "  const int base = __ldg(m->slice_ptr + (t >> 5)), w = (__ldg(m->slice_ptr + (t >> 5) + 1) - base) >> 5;\n"
                 "  const " << CT << " *cp = (const " << CT << " *)m->sell_col + base + (t & 31);\n"
                 "  const " << T << " *vp = (const " << T << " *)m->sell_val + base + (t & 31);\n";
            if (c16) s << "  const int rs = (int)i + m->sell_shift;\n";
            s << "  int k = 0;\n"
                 "  for (; k + 4 <= w; k += 4) {\n"
                 "    int c[4]; " << T << " v[4], xv[4];\n"
                 "#pragma unroll\n    for (int u = 0; u < 4; ++u) { const " << CT << " raw = __ldcs(cp + (k + u) * 32); c[u] = " << dec << "; v[u] = __ldcs(vp + (k + u) * 32); }\n"
                 "#pragma unroll\n    for (int u = 0; u < 4; ++u) xv[u] = c[u] != -1 ? __ldg(x + c[u]) : (" << T << ")0;\n"
                 "#pragma unroll\n    for (int u = 0; u < 4; ++u) if (c[u] != -1) sum = sum + v[u] * xv[u];\n"
                 "  }\n"
                 "  for (; k < w; ++k) { const " << CT << " raw = __ldcs(cp + k * 32); const int c = " << dec << "; const " << T
              << " v = __ldcs(vp + k * 32); if (c != -1) sum = sum + v * __ldg(x + c); }\n";
        } else if (A->fmt == VEXB_FMT_HELL) {
            const int W = (int)A->ell_width;
            const bool c16 = A->ell_col16 != nullptr;
            const char *CT = c16 ? "short" : "int";
            if (W > 0 && A->ell_class) {
                // row classes (spmv.ell_classes): the gathers at clamped columns first, then the row's slot mask and
                // values from the class table (masks in its first 256 bytes), the set slots added in order
                s << "  const unsigned cls = __ldcs((const unsigned char *)m->ell_col + i);\n"
                     "  const " << T << " *tv = (const " << T << " *)((const char *)m->ell_val + " << kEllClassHeader << ") + cls * " << W << ";\n"
                     "  " << T << " xv[" << W << "];\n"
                     "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) xv[j] = __ldg(x + min((unsigned)((int)i + m->shifts[j]), (unsigned)m->x_max));\n"
                     "  const unsigned mask = __ldg((const unsigned char *)m->ell_val + cls);\n"
                     "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) if ((mask >> j) & 1u) sum = sum + __ldg(tv + j) * xv[j];\n";
            } else if (W > 0 && A->ell_mask) {
                // slot masks (spmv.ell_diag): column of slot j = i + shifts[j] where bit j of the row's mask is set
                s << "  const unsigned mask = __ldcs((const unsigned char *)m->ell_col + i); const " << T << " *ev = (const " << T << " *)m->ell_val;\n"
                     "  const unsigned long long pitch = m->pitch;\n"
                     "  int c[" << W << "]; " << T << " v[" << W << "], xv[" << W << "];\n"
                     "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) { c[j] = (mask >> j) & 1u ? (int)i + m->shifts[j] : -1; v[j] = __ldcs(ev + i + j * pitch); }\n"
                     "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) xv[j] = c[j] != -1 ? __ldg(x + c[j]) : (" << T << ")0;\n"
                     "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) if (c[j] != -1) sum = sum + v[j] * xv[j];\n";
            } else if (W > 0) {
                s << "  const " << CT << " *ec = (const " << CT << " *)m->ell_col; const " << T << " *ev = (const " << T << " *)m->ell_val;\n"
                     "  const unsigned long long pitch = m->pitch;\n";
                const bool unroll = W <= 16;
                if (unroll) {
                    s << "  int c[" << W << "]; " << T << " v[" << W << "], xv[" << W << "];\n"
                         "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) { const " << CT << " raw = __ldcs(ec + i + j * pitch); c[j] = "
                      << (c16 ? "raw == (short)-32768 ? -1 : (int)i + m->shifts[j] + (int)raw" : "raw") << "; v[j] = __ldcs(ev + i + j * pitch); }\n"
                         "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) xv[j] = c[j] != -1 ? __ldg(x + c[j]) : (" << T << ")0;\n"
                         "#pragma unroll\n  for (int j = 0; j < " << W << "; ++j) if (c[j] != -1) sum = sum + v[j] * xv[j];\n";
                } else {
                    s << "  for (int j = 0; j < " << W << "; ++j) { const " << CT << " raw = __ldcs(ec + i + j * pitch); const int c = "
                      << (c16 ? "raw == (short)-32768 ? -1 : (int)i + m->shifts[j < " + std::to_string(kEllShiftSlots - 1) + " ? j : " + std::to_string(kEllShiftSlots - 1) + "] + (int)raw" : std::string("raw")) << "; if (c != -1) sum = sum + __ldcs(ev + i + j * pitch) * __ldg(x + c); }\n";
                }
            }
            if (A->tail_nnz) s << "  for (int j = m->tail_ptr[i], e = m->tail_ptr[i + 1]; j < e; ++j) sum = sum + ((const " << T
                               << " *)m->tail_val)[j] * __ldg(x + m->tail_col[j]);\n";
        } else {
            s << "  const " << T << " *val = (const " << T << " *)m->val;\n"
                 "  int j = m->rowptr[i]; const int e = m->rowptr[i + 1];\n"
                 "  for (; j + 4 <= e; j += 4) {\n"
                 "    const int c0 = m->col[j], c1 = m->col[j + 1], c2 = m->col[j + 2], c3 = m->col[j + 3];\n"
                 "    const " << T << " v0 = val[j], v1 = val[j + 1], v2 = val[j + 2], v3 = val[j + 3];\n"
                 "    const " << T << " x0 = __ldg(x + c0), x1 = __ldg(x + c1), x2 = __ldg(x + c2), x3 = __ldg(x + c3);\n"
                 "    sum = sum + v0 * x0; sum = sum + v1 * x1; sum = sum + v2 * x2; sum = sum + v3 * x3;\n"
                 "  }\n"
                 "  for (; j < e; ++j) sum = sum + val[j] * __ldg(x + m->col[j]);\n";
        }
        s << "  return sum;\n}\n";
    }
    // CCSR products used as terminals (VEXB_TERM_CCSR): one row function per terminal, specialised to the value type and
    // the idx width (pad[1]) only -- never to the matrix, whose handle is not read here -- so one kernel serves every CCSR
    // matrix of that shape.  The row loop of ccsr_kernel: idx[i], then the unique row's entries through the read-only path
    // (the table is a few dozen bytes, and interior rows of a warp share one unique row), up to 8 gathers in flight, the
    // products added in storage order as separate operations (--fmad=false): the bits of vexb_ccsr_spmv(alpha = 1).
    bool any_ccsr = false;
    for (int k = 0; k < e.n_terms; ++k) if (e.term[k].kind == VEXB_TERM_CCSR) {
        VEXB_CHECK(ncomp == 1, "sparse products are not fused into multi-expression kernels");
        const int w = e.term[k].pad[1];
        VEXB_CHECK(w == 1 || w == 2 || w == 4, "term %d: CCSR idx width %d is not 1, 2 or 4", k, w);
        const char *T = ctype(e.term[k].dtype);
        const char *IT = w == 1 ? "unsigned char" : w == 2 ? "unsigned short" : "int";
        if (!any_ccsr) {
            s << "struct ccsr_desc_j { const void *idx; const int *row; const int *col; const void *val; };\n";
            any_ccsr = true;
        }
        s << "__device__ __forceinline__ " << T << " ccsr_" << k << "(const ccsr_desc_j *__restrict__ m, const " << T
          << " *__restrict__ x, unsigned long long i) {\n"
             "  const int u = (int)__ldg((const " << IT << " *)m->idx + i);\n"
             "  const int *__restrict__ cp = m->col; const " << T << " *__restrict__ vp = (const " << T << " *)m->val;\n"
             "  const " << T << " *xi = x + i;\n"
             "  " << T << " sum = 0;\n"
             "  for (int j = __ldg(m->row + u), e = __ldg(m->row + u + 1); j < e; j += 8) {\n"
             "    " << T << " xv[8];\n"
             "#pragma unroll\n    for (int q = 0; q < 8; ++q) xv[q] = j + q < e ? __ldg(xi + __ldg(cp + j + q)) : (" << T << ")0;\n"
             "#pragma unroll\n    for (int q = 0; q < 8; ++q) if (j + q < e) sum = sum + __ldg(vp + j + q) * xv[q];\n"
             "  }\n  return sum;\n}\n";
    }
    const char *LT = ctype(lhs_dtype);
    const bool ldg = !passes_pointers(es, ncomp);
    // Multi-expression kernels with temporaries: one function per class of temporaries (temp_classes), vexb_temp_g, which
    // takes the classes its definition reads as parameters g<j>; the kernel calls each once per element and passes the
    // values to the components, whose functions then start after their definitions.
    bool multi_temps = false;
    for (int comp = 0; ncomp > 1 && comp < ncomp; ++comp) multi_temps = multi_temps || expr_has_temps(*es[comp]);
    const TempClasses tc = multi_temps ? temp_classes(es, ncomp) : TempClasses();
    for (size_t g = 0; g < tc.comp.size(); ++g) {
        const vexb_expr &e = *es[tc.comp[g]];
        std::string tnames[VEXB_MAX_TEMPS];
        for (int pc = tc.from[g]; pc < tc.to[g]; ++pc)
            if (e.code[pc].op == VEXB_OP_TREF) tnames[e.code[pc].arg] = "g" + std::to_string(tc.cls[tc.comp[g]][e.code[pc].arg]);
        s << "__device__ __forceinline__ " << ctype(tc.type[g]) << " vexb_temp_" << g << "(const terms_j &tt, unsigned long long i, unsigned long long off";
        for (int j : tc.reads[g]) s << ", const " << ctype(tc.type[j]) << " g" << j;
        s << ") {\n";
        std::vector<std::pair<std::string, int>> st;
        print_code(e, tc.from[g], tc.to[g], tnames, s, st, ldg);
        VEXB_CHECK(st.size() == 1, "internal: a temporary did not reduce to one value");
        s << "    return " << st.back().first << ";\n}\n";
    }
    // One element of the assignment as a function; the kernel below evaluates four of them (a grid stride apart) before it
    // stores any, so a thread has 4 x (number of vector operands) loads in flight instead of one round trip per element.
    for (int comp = 0; comp < ncomp; ++comp) {
    const vexb_expr &e = *es[comp];
    s << "__device__ __forceinline__ " << LT << " vexb_elem" << (ncomp > 1 ? "_" + std::to_string(comp) : std::string()) << "(const terms_j &tt, const " << LT
      << " *lhs, unsigned long long i, unsigned long long off" << (sweep ? ", unsigned long long t" : "");
    std::string tnames[VEXB_MAX_TEMPS];
    for (int k = 0; multi_temps && k < VEXB_MAX_TEMPS; ++k) if (tc.cls[comp][k] >= 0) {
        tnames[k] = "t" + std::to_string(k);
        s << ", const " << ctype(tc.type[tc.cls[comp][k]]) << " " << tnames[k];
    }
    s << ") {\n";
    std::vector<std::pair<std::string, int>> st;        // (variable name, dtype)
    print_code(e, multi_temps ? temp_prefix_length(e) : 0, e.n_code, tnames, s, st, ldg);
    VEXB_CHECK(st.size() == 1, "internal: program did not reduce to one value");
    const std::string res = st.back().first; const int R = st.back().second;
    if (aop == VEXB_SET) {
        s << "    return (" << LT << ")" << res << ";\n";
    } else {
        static const char *sym[] = {"", "+", "-", "*", "/", "%", "&", "|", "^", "<<", ">>"};
        // C/C++ compound assignment: lhs = (L)((C)lhs op (C)rhs), C = the common type -- except for shifts, where the
        // result has the (promoted) type of the LEFT operand and only the count comes from the right (a >>= b on a signed
        // a stays an arithmetic shift whatever the type of b).
        const bool shift = aop == VEXB_LSH || aop == VEXB_RSH;
        const int C = shift ? lhs_dtype : common_dtype(lhs_dtype, R);
        if (aop >= VEXB_MOD && (is_f(C) || (shift && is_f(R)))) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "compound assignment %d is not defined for floating operands", aop);
        s << "    return (" << LT << ")((" << ctype(C) << ")lhs[i] " << sym[aop] << " (" << ctype(C) << ")" << res << ");\n";
    }
    s << "}\n";
    }   // components
    *spmv = any_spmv || any_ccsr;
    return VEXB_OK;
}

static int generate_source_n(const vexb_expr *const *es, int ncomp, int lhs_dtype, int aop, std::string *out) {
    std::ostringstream s;
    bool any_spmv = false;
    int sell = -1;
    VEXB_TRY(generate_elements(es, ncomp, lhs_dtype, aop, s, &any_spmv, &sell));
    const char *LT = ctype(lhs_dtype);
    if (sell >= 0) {
        // Storage-order sweep: one thread per stored lane of the sliced-ELL strip, every operand and the target at the
        // lane's row r.  A warp reads the strip's columns and values coalesced, as sell_kernel does, and its accesses to
        // the other operands fall inside one window of sigma rows.  sell_layout puts every row in exactly one lane, so
        // every element is written once.
        s << "extern \"C\" __global__ void __launch_bounds__(256) vexb_jit_kernel(const terms_j tt, " << LT
          << " *lhs, unsigned long long n, unsigned long long off) {\n"
             "  const spmv_desc_j *m = (const spmv_desc_j *)tt.t[" << sell << "].v.ptr;\n"
             "  const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;\n"
             "  if (t >= m->n_slices * 32ull) return;\n"
             "  const int r = __ldcs(m->perm + t);\n"
             "  if (r < 0 || (unsigned long long)r >= n) return;\n"
             "  lhs[r] = vexb_elem(tt, lhs, (unsigned long long)r, off, t);\n}\n";
        *out = s.str();
        return VEXB_OK;
    }
    if (ncomp > 1) {
        s << "struct multi_j { terms_j c[" << ncomp << "]; " << LT << " *lhs[" << ncomp << "]; };\n"
             "extern \"C\" __global__ void __launch_bounds__(256) vexb_jit_kernel(const multi_j mt, unsigned long long n, unsigned long long off) {\n"
             "  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;\n"
             "  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {\n";
        bool temps = false;
        for (int c = 0; c < ncomp; ++c) temps = temps || expr_has_temps(*es[c]);
        const TempClasses tc = temps ? temp_classes(es, ncomp) : TempClasses();
        for (size_t g = 0; g < tc.comp.size(); ++g) {
            s << "    const " << ctype(tc.type[g]) << " g" << g << " = vexb_temp_" << g << "(mt.c[" << tc.comp[g] << "], i, off";
            for (int j : tc.reads[g]) s << ", g" << j;
            s << ");\n";
        }
        for (int c = 0; c < ncomp; ++c) {
            s << "    const " << LT << " a" << c << " = vexb_elem_" << c << "(mt.c[" << c << "], mt.lhs[" << c << "], i, off";
            for (int k = 0; temps && k < VEXB_MAX_TEMPS; ++k) if (tc.cls[c][k] >= 0) s << ", g" << tc.cls[c][k];
            s << ");\n";
        }
        for (int c = 0; c < ncomp; ++c) s << "    mt.lhs[" << c << "][i] = a" << c << ";\n";
        s << "  }\n}\n";
        *out = s.str();
        return VEXB_OK;
    }
    // Four elements per thread, 256 apart inside one contiguous chunk of 1024 per block: 4 x (number of vector operands)
    // loads in flight per thread, and every stream still advances through memory contiguously.  (Four elements a GRID
    // stride apart would make 16 widely separated streams per operand, which cost more in DRAM page locality than the
    // extra loads in flight bring.)
    const int U = any_spmv ? 1 : 4;                    // a row loop per element is its own source of parallel loads
    s << "extern \"C\" __global__ void __launch_bounds__(256) vexb_jit_kernel(const terms_j tt, " << LT
      << " *lhs, unsigned long long n, unsigned long long off) {\n";
    if (U > 1) {
        s << "  const unsigned long long chunk = " << U * 256 << "ull, step = (unsigned long long)gridDim.x * chunk;\n"
             "  for (unsigned long long base = (unsigned long long)blockIdx.x * chunk; base < n; base += step) {\n"
             "    const unsigned long long i = base + threadIdx.x;\n"
             "    if (base + chunk <= n) {\n";
        for (int u = 0; u < U; ++u) s << "      const " << LT << " a" << u << " = vexb_elem(tt, lhs, i + " << u * 256 << "ull, off);\n";
        for (int u = 0; u < U; ++u) s << "      lhs[i + " << u * 256 << "ull] = a" << u << ";\n";
        s << "    } else {\n"
             "      for (unsigned long long k = i; k < n; k += 256) lhs[k] = vexb_elem(tt, lhs, k, off);\n"
             "    }\n  }\n}\n";
    } else {
        s << "  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;\n"
             "  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) lhs[i] = vexb_elem(tt, lhs, i, off);\n}\n";
    }
    *out = s.str();
    return VEXB_OK;
}

static int generate_source(const vexb_expr &e, int lhs_dtype, int aop, std::string *out) {
    const vexb_expr *p = &e;
    return generate_source_n(&p, 1, lhs_dtype, aop, out);
}

// ---- reductions of expressions with user functions or inlined sparse products ----------------------------------------
// Without this, such a reduction is two launches: the expression into a temporary of its own type (vexb_eval, the kernel
// above), then that temporary through vexb_reduce_all / vexb_reduce_multi.  Here one generated kernel does both: element
// i comes from the same vexb_elem text, rounded to the expression's type as the temporary stores it, converted to the
// reduction's type as the pre-compiled reduction reads it (convert, expr_eval.cuh), and folded in the order, by the grid,
// and with the very code (fold.cuh, embedded) that the pre-compiled kernel would apply to the temporary.  So the result
// has the bits of the two-launch path, and A*x, or f(x, y), never goes to memory.
//   RED_SWEEP  : reduce_sweep_kernel<SH_COPY, OP, T, 2> -- one op, dtype F64 / F32 equal to the expression's type, and
//                eval.force_interp = 0 (the temporary would take the hand-written sweep): E = 32 / sizeof(T) consecutive
//                elements per thread and chunk, two chunks in flight, the tail element into acc[0][0]
//   RED_INTERP : reduce_interp_kernel<OP, T, 4> -- every other single op
//   RED_MULTI  : reduce_multi_kernel<T, 4> -- vexb_reduce_multi (CombineReductors), one workspace slice per op
enum { RED_SWEEP = 0, RED_INTERP = 1, RED_MULTI = 2 };

static int reduce_skeleton(const vexb_expr &e, int dtype, bool multi) {
    if (multi) return RED_MULTI;
    if ((dtype == VEXB_F64 || dtype == VEXB_F32) && dtype == host_result_type(e) && !param("eval.force_interp", 0)) return RED_SWEEP;
    return RED_INTERP;
}

static const char *op_name(int op) {
    switch (op) {
        case VEXB_SUM: return "VEXB_SUM"; case VEXB_SUM_KAHAN: return "VEXB_SUM_KAHAN"; case VEXB_MAX: return "VEXB_MAX";
        case VEXB_MIN: return "VEXB_MIN"; default: return "VEXB_MINMAX";
    }
}

// ops: already mapped (SUM_KAHAN -> SUM on integer types), one for RED_SWEEP / RED_INTERP.
static int generate_reduce_source(const vexb_expr &e, int dtype, int nops, const int *ops, int skel, std::string *out) {
    const int R = host_result_type(e);
    const char *T = ctype(dtype), *RT = ctype(R);
    std::ostringstream s;
    s << "// generated by libvexb200 (csrc/jit.cu): reduction\n"
         "enum { VEXB_SUM = " << VEXB_SUM << ", VEXB_SUM_KAHAN = " << VEXB_SUM_KAHAN << ", VEXB_MAX = " << VEXB_MAX
      << ", VEXB_MIN = " << VEXB_MIN << ", VEXB_MINMAX = " << VEXB_MINMAX << " };\n";
    s.write(reinterpret_cast<const char *>(kFoldText), sizeof(kFoldText) - 1);
    s << "// end of fold.cuh\n";
    const vexb_expr *p = &e;
    bool any_spmv = false;
    VEXB_TRY(generate_elements(&p, 1, R, VEXB_SET, s, &any_spmv));
    s << "using namespace vexb;\n"
         "__device__ __forceinline__ " << T << " vexb_red_val(const terms_j &tt, unsigned long long i, unsigned long long off) {\n"
         "  const " << RT << " v = vexb_elem(tt, (const " << RT << " *)0, i, off);\n"
         "  return (" << T << ")v;\n}\n"
         "extern \"C\" __global__ void __launch_bounds__(256) vexb_reduce_kernel(const terms_j tt, unsigned long long n, unsigned long long off,\n"
         "    void *ws, unsigned long long ws_stride, " << T << " *result, PeerArgs pa) {\n";
    if (skel == RED_SWEEP) {
        const std::string F = std::string("Fold<") + op_name(ops[0]) + ", " + T + ">";
        s << "  constexpr int U = 2, E = " << (dtype == VEXB_F64 ? 4 : 8) << ";\n"
             "  " << F << " acc[U][E];\n"
             "#pragma unroll\n  for (int u = 0; u < U; ++u)\n"
             "#pragma unroll\n    for (int j = 0; j < E; ++j) acc[u][j].init();\n"
             "  const unsigned long long nvec = n / E;\n"
             "  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x * U;\n"
             "  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x * U + threadIdx.x; base < nvec; base += stride) {\n"
             "#pragma unroll\n    for (int u = 0; u < U; ++u) {\n"
             "      const unsigned long long iv = base + (unsigned long long)u * blockDim.x;\n"
             "      if (iv < nvec) {\n"
             "#pragma unroll\n        for (int j = 0; j < E; ++j) acc[u][j].take(vexb_red_val(tt, iv * E + j, off));\n"
             "      }\n    }\n  }\n"
             "  const unsigned long long i = nvec * E + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;\n"
             "  if (i < n) acc[0][0].take(vexb_red_val(tt, i, off));\n"
             "  " << F << " f = acc[0][0];\n"
             "#pragma unroll\n  for (int u = 0; u < U; ++u)\n"
             "#pragma unroll\n    for (int j = 0; j < E; ++j) if (u || j) f.merge(acc[u][j]);\n"
             "  block_finish<" << op_name(ops[0]) << ", " << T << ">(f, ws, result, pa);\n}\n";
    } else if (skel == RED_INTERP) {
        const std::string F = std::string("Fold<") + op_name(ops[0]) + ", " + T + ">";
        s << "  constexpr int U = 4;\n"
             "  " << F << " acc[U];\n"
             "#pragma unroll\n  for (int k = 0; k < U; ++k) acc[k].init();\n"
             "  const unsigned long long chunk = (unsigned long long)blockDim.x * U;\n"
             "  for (unsigned long long base = (unsigned long long)blockIdx.x * chunk; base < n; base += (unsigned long long)gridDim.x * chunk) {\n"
             "#pragma unroll\n    for (int k = 0; k < U; ++k) {\n"
             "      const unsigned long long i = base + (unsigned long long)k * blockDim.x + threadIdx.x;\n"
             "      if (i < n) acc[k].take(vexb_red_val(tt, i, off));\n"
             "    }\n  }\n"
             "  " << F << " f = acc[0];\n"
             "#pragma unroll\n  for (int k = 1; k < U; ++k) f.merge(acc[k]);\n"
             "  block_finish<" << op_name(ops[0]) << ", " << T << ">(f, ws, result, pa);\n}\n";
    } else {
        s << "  constexpr int U = 4, NOPS = " << nops << ";\n"
             "  const int ops[NOPS] = {";
        for (int k = 0; k < nops; ++k) s << (k ? ", " : "") << op_name(ops[k]);
        s << "};\n"
             "  RtFold<" << T << "> acc[NOPS];\n"
             "#pragma unroll\n  for (int k = 0; k < NOPS; ++k) acc[k].init(ops[k]);\n"
             "  const unsigned long long chunk = (unsigned long long)blockDim.x * U;\n"
             "  for (unsigned long long base = (unsigned long long)blockIdx.x * chunk; base < n; base += (unsigned long long)gridDim.x * chunk) {\n"
             "#pragma unroll\n    for (int u = 0; u < U; ++u) {\n"
             "      const unsigned long long i = base + (unsigned long long)u * blockDim.x + threadIdx.x;\n"
             "      if (i < n) {\n"
             "        const " << T << " v = vexb_red_val(tt, i, off);\n"
             "#pragma unroll\n        for (int k = 0; k < NOPS; ++k) acc[k].take(ops[k], v);\n"
             "      }\n    }\n  }\n";
        for (int k = 0; k < nops; ++k) {
            // the finish of reduce_multi_kernel: MAX and MIN as themselves, both sums as a plain sum of the partials
            const char *fo = ops[k] == VEXB_MAX ? "VEXB_MAX" : ops[k] == VEXB_MIN ? "VEXB_MIN" : "VEXB_SUM";
            s << "  { Fold<" << fo << ", " << T << "> f; f.x = acc[" << k << "].x; f.y = (" << T << ")0;\n"
                 "    block_finish<" << fo << ", " << T << ">(f, (char *)ws + " << k << "ull * ws_stride, result + " << k << ", pa); }\n"
                 "  __syncthreads();\n";
        }
        s << "}\n";
    }
    *out = s.str();
    return VEXB_OK;
}

// ---- NVRTC + driver API, resolved at first use ---------------------------------------------------
typedef int nvrtcResult; typedef struct _nvrtcProgram *nvrtcProgram;
typedef int CUresult; typedef struct CUmod_st *CUmodule; typedef struct CUfunc_st *CUfunction; typedef struct CUstream_st *CUstream;
struct JitApi {
    void *nvrtc = nullptr, *cuda = nullptr;
    nvrtcResult (*nvrtcCreateProgram)(nvrtcProgram *, const char *, const char *, int, const char *const *, const char *const *) = nullptr;
    nvrtcResult (*nvrtcCompileProgram)(nvrtcProgram, int, const char *const *) = nullptr;
    nvrtcResult (*nvrtcGetCUBINSize)(nvrtcProgram, size_t *) = nullptr;
    nvrtcResult (*nvrtcGetCUBIN)(nvrtcProgram, char *) = nullptr;
    nvrtcResult (*nvrtcGetProgramLogSize)(nvrtcProgram, size_t *) = nullptr;
    nvrtcResult (*nvrtcGetProgramLog)(nvrtcProgram, char *) = nullptr;
    nvrtcResult (*nvrtcDestroyProgram)(nvrtcProgram *) = nullptr;
    const char *(*nvrtcGetErrorString)(nvrtcResult) = nullptr;
    CUresult (*cuModuleLoadData)(CUmodule *, const void *) = nullptr;
    CUresult (*cuModuleGetFunction)(CUfunction *, CUmodule, const char *) = nullptr;
    CUresult (*cuLaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void **, void **) = nullptr;
    CUresult (*cuGetErrorString)(CUresult, const char **) = nullptr;
};
static JitApi g_jit;
static std::mutex g_jmx;

static std::mutex g_load_mx;
static int load_nvrtc() {
    std::lock_guard<std::mutex> lock(g_load_mx);
    if (g_jit.nvrtc) return VEXB_OK;
    const char *names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12"};
    void *h = nullptr;
    for (const char *nm : names) { h = dlopen(nm, RTLD_NOW); if (h) break; }
    if (!h) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "user functions need NVRTC, and libnvrtc.so.12 cannot be loaded: %s", dlerror());
#define L(sym) do { *(void **)(&g_jit.sym) = dlsym(h, #sym); if (!g_jit.sym) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "NVRTC lacks %s", #sym); } while (0)
    L(nvrtcCreateProgram); L(nvrtcCompileProgram); L(nvrtcGetCUBINSize); L(nvrtcGetCUBIN);
    L(nvrtcGetProgramLogSize); L(nvrtcGetProgramLog); L(nvrtcDestroyProgram); L(nvrtcGetErrorString);
#undef L
    g_jit.nvrtc = h;
    return VEXB_OK;
}
static int load_driver() {
    std::lock_guard<std::mutex> lock(g_load_mx);
    if (g_jit.cuda) return VEXB_OK;
    void *h = dlopen("libcuda.so.1", RTLD_NOW);
    if (!h) VEXB_FAIL(VEXB_ERR_CUDA, "cannot load libcuda.so.1: %s", dlerror());
#define L(sym) do { *(void **)(&g_jit.sym) = dlsym(h, #sym); if (!g_jit.sym) VEXB_FAIL(VEXB_ERR_CUDA, "driver lacks %s", #sym); } while (0)
    L(cuModuleLoadData); L(cuModuleGetFunction); L(cuLaunchKernel); L(cuGetErrorString);
#undef L
    g_jit.cuda = h;
    return VEXB_OK;
}

// One NVRTC compilation at a time.  The library is documented as thread safe, but a test binary that starts a dozen
// background compilations within its first second (one per new expression shape) while the main thread compiles a user
// function crashed inside nvrtcCompileProgram on every cold start and never on a warm one:
// compilations are rare and short, serialising them costs nothing that matters.
static std::mutex g_nvrtc_mx;
static std::atomic<bool> g_bg_cancel{false};       // set while the process is leaving: queued compilations give up (see below)
constexpr int VEXB_ERR_CANCELLED = -100;           // internal only, never returned through the ABI

// device_default: --device-as-default-execution-space, for programs with a preamble (program_has_preamble) only.
static int compile_cubin(const std::string &src, std::vector<char> *cubin, std::string *log, bool device_default) {
    VEXB_TRY(load_nvrtc());
    std::lock_guard<std::mutex> nvrtc_lock(g_nvrtc_mx);
    if (g_bg_cancel.load()) return VEXB_ERR_CANCELLED;                 // queued behind another compilation while the process exits
    nvrtcProgram prog = nullptr;
    nvrtcResult r = g_jit.nvrtcCreateProgram(&prog, src.c_str(), "vexb_jit.cu", 0, nullptr, nullptr);
    if (r != 0) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "nvrtcCreateProgram: %s", g_jit.nvrtcGetErrorString(r));
    const char *opts[] = {"--gpu-architecture=sm_90a", "--fmad=false", "--std=c++17", "-lineinfo", "--device-as-default-execution-space"};
    r = g_jit.nvrtcCompileProgram(prog, device_default ? 5 : 4, opts);
    size_t ls = 0;
    g_jit.nvrtcGetProgramLogSize(prog, &ls);
    std::string lg(ls ? ls : 1, '\0');
    if (ls) g_jit.nvrtcGetProgramLog(prog, &lg[0]);
    if (log) *log = lg.c_str();
    if (r != 0) {
        g_jit.nvrtcDestroyProgram(&prog);
        VEXB_FAIL(VEXB_ERR_INVALID, "NVRTC could not compile the expression (%s):\n%.700s", g_jit.nvrtcGetErrorString(r), lg.c_str());
    }
    size_t cs = 0;
    g_jit.nvrtcGetCUBINSize(prog, &cs);
    cubin->resize(cs);
    g_jit.nvrtcGetCUBIN(prog, cubin->data());
    g_jit.nvrtcDestroyProgram(&prog);
    return VEXB_OK;
}

struct terms_host { vexb_term t[VEXB_MAX_TERMS]; };

// The shape of a request without its pointers and scalar values (those travel in the terminal table at launch): the
// instructions, the terminal kinds / types, the lhs type and the assignment, byte for byte.  This string IS the cache key
// (no hashing: two different requests can never share a kernel).
static std::string request_signature(const vexb_expr &e, int lhs_dtype, int aop) {
    std::string k;
    k.reserve(8 + 4 * (size_t)e.n_code + 2 * (size_t)e.n_terms);
    k.push_back((char)lhs_dtype); k.push_back((char)aop); k.push_back((char)e.n_code); k.push_back((char)e.n_terms);
    for (int pc = 0; pc < e.n_code; ++pc) {
        k.push_back((char)e.code[pc].op); k.push_back((char)e.code[pc].type);
        k.push_back((char)(e.code[pc].arg & 0xff)); k.push_back((char)(e.code[pc].arg >> 8));
    }
    for (int t = 0; t < e.n_terms; ++t) {
        k.push_back((char)e.term[t].kind); k.push_back((char)e.term[t].dtype);
        if (e.term[t].kind == VEXB_TERM_SPMV) {          // the generated row loop depends on the strip's format, not on its data
            const vexb_spmat *A = static_cast<const vexb_spmat *>(e.term[t].v.ptr);
            k.push_back((char)e.term[t].pad[0]); k.push_back((char)A->fmt); k.push_back(A->ell_class ? 3 : A->ell_mask ? 2 : A->ell_col16 || A->sell_col16 ? 1 : 0); k.push_back(A->tail_nnz ? 1 : 0);
            const unsigned w = (unsigned)A->ell_width;
            k.push_back((char)(w & 0xff)); k.push_back((char)((w >> 8) & 0xff)); k.push_back((char)((w >> 16) & 0xff)); k.push_back((char)(w >> 24));
        } else if (e.term[t].kind == VEXB_TERM_CCSR) {   // x's slot and the idx width; never the matrix
            k.push_back((char)e.term[t].pad[0]); k.push_back((char)e.term[t].pad[1]);
        }
    }
    return k;
}

// The kernel parameter terms_j of a request: its terminals, with every sparse product's handle replaced by the strip's
// device descriptor.
static int pack_terms(const vexb_expr &e, int dev, size_t n, terms_host *tt) {
    memset(tt, 0, sizeof(*tt));
    for (int k = 0; k < e.n_terms; ++k) {
        tt->t[k] = e.term[k];
        if (e.term[k].kind == VEXB_TERM_SPMV) {
            const vexb_spmat *A = static_cast<const vexb_spmat *>(e.term[k].v.ptr);
            VEXB_CHECK(A->dev == dev, "term %d: the matrix lives on device %d, not %d", k, A->dev, dev);
            VEXB_CHECK(A->nrows_stored >= n, "term %d: the strip has %zu rows, the expression %zu elements", k, A->nrows_stored, n);
            tt->t[k].v.ptr = A->d_desc;
        } else if (e.term[k].kind == VEXB_TERM_CCSR) {
            void *desc = nullptr;
            VEXB_TRY(ccsr_term_desc(static_cast<const vexb_ccsr *>(e.term[k].v.ptr), &desc));
            tt->t[k].v.ptr = desc;
        }
    }
    return VEXB_OK;
}

// The CCSR terminals of a request against their handles, before anything is compiled or launched.  lhs: the assignment's
// target (NULL for reductions); a kernel that writes x[i] while other threads read x[i + col[j]] would race, so an x that
// is the target is VEXB_ERR_UNSUPPORTED (the front ends evaluate the product into a temporary first).
static int check_ccsr_terms(const vexb_expr &e, int dev, const void *lhs, size_t n, size_t index_offset) {
    for (int k = 0; k < e.n_terms; ++k) if (e.term[k].kind == VEXB_TERM_CCSR)
        VEXB_TRY(ccsr_term_check(static_cast<const vexb_ccsr *>(e.term[k].v.ptr), k, dev, e.term[k].dtype, e.term[k].pad[1], n, index_offset));
    for (int k = 0; k < e.n_terms; ++k)
        if (e.term[k].kind == VEXB_TERM_CCSR && lhs && e.term[e.term[k].pad[0]].v.ptr == lhs)
            VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "term %d: the CCSR product's x is the assignment's target; evaluate the product into a temporary first", k);
    return VEXB_OK;
}

// One cache entry per program.  state: 0 new, 1 compiling (a thread owns it), 2 cubin ready, 3 failed.
struct JitEntry {
    std::mutex mx; std::condition_variable cv;
    int state = 0; long uses = 0;
    int status = VEXB_OK; std::string error;           // of a failed compilation (returned to every later request)
    std::vector<char> cubin;
    std::map<int, CUfunction> fn;                       // per device, loaded by the first request on that device
};
static std::map<std::string, std::shared_ptr<JitEntry>> g_entries;

// Background compilations and process exit.  NVRTC registers exit handlers of its own lazily, during its first
// compilation; exit() runs handlers last-registered-first, so a compilation still in flight when the host program
// leaves main() has NVRTC's statics destroyed under it and crashes (a test binary whose checks had all passed ended with
// SIGSEGV inside nvrtcCompileProgram on every cold start; it reproduces without a GPU).
// No atexit handler of ours can be registered late enough.  What does run earlier: exit() destroys the calling thread's
// thread_local objects BEFORE any atexit handler.  So a thread that starts a background compilation arms a thread_local
// guard whose destructor cancels the compilations that have not started and waits for the one that has.  The atexit
// handler stays as a second line (exit() called from a thread that never touched the JIT).
static std::mutex g_bg_mx;
static std::vector<std::thread> g_bg_threads;
static void join_background_compilations() {
    g_bg_cancel.store(true);
    std::vector<std::thread> ts;
    { std::lock_guard<std::mutex> lock(g_bg_mx); ts.swap(g_bg_threads); }
    for (auto &t : ts) if (t.joinable()) t.join();
    g_bg_cancel.store(false);
}
struct BackgroundJoinGuard {
    bool armed = false;
    ~BackgroundJoinGuard() { if (armed) join_background_compilations(); }
};
static thread_local BackgroundJoinGuard tl_bg_guard;

// NVRTC for one entry; runs WITHOUT any lock of the cache (hundreds of milliseconds), on the requesting thread or on a
// background thread.
static void compile_entry(std::shared_ptr<JitEntry> en, std::string src, bool device_default) {
    std::vector<char> cubin;
    const int st = compile_cubin(src, &cubin, nullptr, device_default);
    const std::string err = st == VEXB_OK ? std::string() : std::string(vexb_last_error());
    std::lock_guard<std::mutex> lock(en->mx);
    if (st == VEXB_ERR_CANCELLED) en->state = 0;                       // the process is leaving: back to "never tried"
    else if (st == VEXB_OK) { en->cubin.swap(cubin); en->state = 2; }
    else { en->status = st; en->error = err; en->state = 3; }
    en->cv.notify_all();
}

static void spawn_background(std::shared_ptr<JitEntry> en, std::string src, bool device_default) {
    std::lock_guard<std::mutex> bl(g_bg_mx);
    static bool registered = false;
    if (!registered) { registered = true; atexit(join_background_compilations); }
    g_bg_threads.emplace_back(compile_entry, en, std::move(src), device_default);
    tl_bg_guard.armed = true;
}

int jit_program(int dev, const std::string &key, const char *name, const std::string &header, const JitSource &source,
                bool wait, void **fn) {
    *fn = nullptr;
    std::shared_ptr<JitEntry> en;
    {
        std::lock_guard<std::mutex> lock(g_jmx);                      // short: map lookup only
        auto &slot = g_entries[key_with_header(key, header)];
        if (!slot) slot = std::make_shared<JitEntry>();
        en = slot;
    }
    std::unique_lock<std::mutex> lock(en->mx);
    if (en->state == 0) {
        JitBuild b;
        b.uses = ++en->uses;
        const int st = source(&b);
        if (st != VEXB_OK) { en->state = 3; en->status = st; en->error = vexb_last_error(); }
        else if (b.later) return VEXB_OK;
        else {
            en->state = 1;
            std::string src = with_program_header(header, b.text);
            if (b.background) { spawn_background(en, std::move(src), b.device_default); return VEXB_OK; }
            lock.unlock();
            compile_entry(en, std::move(src), b.device_default);
            lock.lock();
        }
    }
    if (en->state == 1) {
        if (!wait) return VEXB_OK;
        en->cv.wait(lock, [&] { return en->state != 1; });
    }
    if (en->state == 3) { set_error(__FILE__, __LINE__, "%s", en->error.c_str()); return en->status; }
    if (en->state != 2) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "the compilation of %s was cancelled: the process is exiting", name);
    if (dev < 0) return VEXB_OK;
    auto it = en->fn.find(dev);
    if (it == en->fn.end()) {
        VEXB_TRY(load_driver());
        VEXB_CUDA(cudaFree(0));                                       // make sure the primary context is current
        CUmodule mod = nullptr;
        CUfunction f = nullptr;
        const char *what = "cuModuleLoadData";
        CUresult r = g_jit.cuModuleLoadData(&mod, en->cubin.data());
        if (r == 0) { what = "cuModuleGetFunction"; r = g_jit.cuModuleGetFunction(&f, mod, name); }
        if (r != 0) { const char *m = ""; g_jit.cuGetErrorString(r, &m); VEXB_FAIL(VEXB_ERR_CUDA, "%s(%s) failed: %s", what, name, m); }
        it = en->fn.emplace(dev, f).first;
    }
    *fn = it->second;
    return VEXB_OK;
}

int jit_launch(void *fn, unsigned grid, unsigned block, unsigned smem, cudaStream_t st, void **args) {
    CUresult r = g_jit.cuLaunchKernel((CUfunction)fn, grid, 1, 1, block, 1, 1, smem, (CUstream)st, args, nullptr);
    if (r != 0) { const char *m = ""; g_jit.cuGetErrorString(r, &m); VEXB_FAIL(VEXB_ERR_CUDA, "cuLaunchKernel failed: %s", m); }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return VEXB_OK;
}

int jit_print(std::string src, int compile, bool device_default, char *buf, size_t *len) {
    if (compile) {
        std::vector<char> cubin; std::string log;
        VEXB_TRY(compile_cubin(src, &cubin, &log, device_default));
        src += "// NVRTC: ok, cubin " + std::to_string(cubin.size()) + " bytes\n";
        if (!log.empty()) src += "/* log:\n" + log + "*/\n";
    }
    if (buf) {
        VEXB_CHECK(*len > src.size(), "buffer too small (%zu <= %zu)", *len, src.size());
        memcpy(buf, src.c_str(), src.size() + 1);
    }
    *len = src.size() + 1;
    return VEXB_OK;
}

// mode 1: the specialised kernel is mandatory (user functions, eval.jit = 1): compile now if nobody has, wait if somebody
// is, report errors.  mode 2 ("auto", the default for expressions without a sweep): the first use of a new shape starts
// an NVRTC compilation on a background thread and returns at once; the pre-compiled interpreter serves this and the next
// launches (no start-up stall) until the cubin is ready, then every launch takes the specialised kernel.  Both produce the
// same bits, so the switch is invisible.  `eval.jit_after` (0) delays the compilation until a shape has been used that
// often, `eval.jit_sync` (0) compiles on the requesting thread instead.  *done = false means "not handled here" (the
// caller runs the interpreter).
int jit_eval(int dev, cudaStream_t st, void *lhs, int lhs_dtype, int aop, const vexb_expr &e, size_t n, size_t index_offset,
             int mode, bool *done) {
    *done = false;
    int sell = -1;
    VEXB_TRY(sell_sweep_term(e, &sell));                              // before the cache: the signature does not tell strips apart
    VEXB_TRY(check_ccsr_terms(e, dev, lhs, n, index_offset));
    const vexb_expr *pe = &e;
    void *fn = nullptr;
    const int s = jit_program(dev, request_signature(e, lhs_dtype, aop), "vexb_jit_kernel", header_for(dev, &pe, 1), [&](JitBuild *b) -> int {
        if (mode == 2 && b->uses <= param("eval.jit_after", 0)) { b->later = true; return VEXB_OK; }
        b->background = mode == 2 && !param("eval.jit_sync", 0);
        b->device_default = program_has_preamble(&pe, 1);
        return generate_source(e, lhs_dtype, aop, &b->text);
    }, mode != 2, &fn);
    if (mode == 2 && !fn) return VEXB_OK;                             // not ready, or failed: the interpreter serves
    VEXB_TRY(s);
    *done = true;
    terms_host tt;
    VEXB_TRY(pack_terms(e, dev, n, &tt));
    unsigned long long nn = n, off = index_offset;
    void *args[] = {&tt, &lhs, &nn, &off};
    bool any_spmv = false;
    for (int k = 0; k < e.n_terms; ++k) any_spmv = any_spmv || is_product_term(e.term[k].kind);
    const size_t per_block = any_spmv ? 256 : 1024;                    // elements per block and loop trip (generate_source: U = 1 / 4)
    size_t blocks = (n + per_block - 1) / per_block;
    const size_t cap = (size_t)sm_count(dev) * 64;
    if (blocks > cap) blocks = cap;
    if (sell >= 0) blocks = (static_cast<const vexb_spmat *>(e.term[sell].v.ptr)->n_slices + 7) / 8;   // a thread per stored lane, no loop
    return jit_launch(fn, (unsigned)blocks, 256, 0, st, args);
}

// The components of a multi-expression assignment in one kernel (generate_source_n).  Same modes as jit_eval, without
// eval.jit_after; *done = false means "not served here" (NVRTC missing or failed, still compiling in the background, more
// than 8 components, a sparse product among the terminals): the caller evaluates component by component.
int jit_eval_multi(int dev, cudaStream_t st, int ncomp, void *const *lhs, int lhs_dtype, int aop, const vexb_expr *const *es,
                   size_t n, size_t index_offset, int mode, bool *done) {
    *done = false;
    if (ncomp < 2 || ncomp > 8) return VEXB_OK;
    for (int c = 0; c < ncomp; ++c)
        for (int k = 0; k < es[c]->n_terms; ++k) if (is_product_term(es[c]->term[k].kind)) return VEXB_OK;
    std::string key(1, (char)ncomp);
    for (int c = 0; c < ncomp; ++c) { key += request_signature(*es[c], lhs_dtype, aop); key.push_back('|'); }
    bool temps = false;
    for (int c = 0; c < ncomp; ++c) temps = temps || expr_has_temps(*es[c]);
    if (temps) {                                                      // which temporaries the components share: by pointer
        const TempClasses tc = temp_classes(es, ncomp);
        key += "temps:";
        for (int c = 0; c < ncomp; ++c) for (int k = 0; k < VEXB_MAX_TEMPS; ++k) key.push_back((char)tc.cls[c][k]);
    }
    void *fn = nullptr;
    jit_program(dev, "multi:" + key, "vexb_jit_kernel", header_for(dev, es, ncomp), [&](JitBuild *b) {
        b->background = mode == 2 && !param("eval.jit_sync", 0);
        b->device_default = program_has_preamble(es, ncomp);
        return generate_source_n(es, ncomp, lhs_dtype, aop, &b->text);
    }, mode != 2, &fn);
    if (!fn) return VEXB_OK;
    // kernel parameter: struct multi_j { terms_j c[ncomp]; T *lhs[ncomp]; } -- packed for the actual ncomp
    std::vector<unsigned char> prm((size_t)ncomp * sizeof(terms_host) + (size_t)ncomp * sizeof(void *), 0);
    for (int c = 0; c < ncomp; ++c) {
        terms_host tt;
        VEXB_TRY(pack_terms(*es[c], dev, n, &tt));
        memcpy(prm.data() + (size_t)c * sizeof(terms_host), &tt, sizeof(tt));
        memcpy(prm.data() + (size_t)ncomp * sizeof(terms_host) + (size_t)c * sizeof(void *), &lhs[c], sizeof(void *));
    }
    unsigned long long nn = n, off = index_offset;
    void *args[] = {prm.data(), &nn, &off};
    size_t blocks = (n + 255) / 256;
    const size_t cap = (size_t)sm_count(dev) * 32;
    if (blocks > cap) blocks = cap;
    VEXB_TRY(jit_launch(fn, (unsigned)blocks, 256, 0, st, args));
    *done = true;
    return VEXB_OK;
}

int jit_pending();
// 1 while any background compilation is running (tests and benchmarks wait for the specialised kernel with this)
int jit_pending() {
    std::lock_guard<std::mutex> lock(g_jmx);
    for (auto &kv : g_entries) { std::lock_guard<std::mutex> l2(kv.second->mx); if (kv.second->state == 1) return 1; }
    return 0;
}

// One launch per slot for a reduction of an expression with user functions or inlined sparse products (see
// generate_reduce_source).  Compiled synchronously at its first use, then cached per request shape, dtype, ops and
// skeleton, and per device.  VEXB_ERR_UNSUPPORTED only when NVRTC cannot be loaded: the front ends then evaluate the
// expression into a temporary and reduce that.  The caller has selected `dev` and handled n == 0.
int jit_reduce(int dev, cudaStream_t st, const vexb_expr &e, int dtype, size_t n, size_t index_offset, int nops, const int *ops,
               bool multi, size_t cap, void *d_result, void *d_workspace, const PeerArgs &pa) {
    VEXB_TRY(check_ccsr_terms(e, dev, nullptr, n, index_offset));
    const int skel = reduce_skeleton(e, dtype, multi);
    const vexb_expr *pe = &e;
    std::string key = "reduce:" + request_signature(e, host_result_type(e), VEXB_SET);
    key.push_back('|'); key.push_back((char)dtype); key.push_back((char)skel); key.push_back((char)nops);
    for (int k = 0; k < nops; ++k) key.push_back((char)ops[k]);
    void *fn = nullptr;
    VEXB_TRY(jit_program(dev, key, "vexb_reduce_kernel", header_for(dev, &pe, 1), [&](JitBuild *b) {
        b->device_default = program_has_preamble(&pe, 1);
        return generate_reduce_source(e, dtype, nops, ops, skel, &b->text);
    }, true, &fn));
    terms_host tt;
    VEXB_TRY(pack_terms(e, dev, n, &tt));
    size_t blocks;
    if (skel == RED_SWEEP) {
        const size_t E = dtype == VEXB_F64 ? 4 : 8;
        blocks = (n / E + 511) / 512; if (blocks < 1) blocks = 1;
    } else blocks = (n + 1023) / 1024;
    if (blocks > cap) blocks = cap;
    size_t stride = 0;
    VEXB_TRY(vexb_reduce_workspace_bytes(dev, &stride));
    unsigned long long nn = n, off = index_offset, ws_stride = stride;
    PeerArgs peer = pa;
    void *args[] = {&tt, &nn, &off, &d_workspace, &ws_stride, &d_result, &peer};
    return jit_launch(fn, (unsigned)blocks, 256, 0, st, args);
}

} // namespace vexb

using namespace vexb;

extern "C" int vexb_function_register(const char *name, int ret_dtype, int nargs, const int *arg_dtypes,
                                      const char *body, int *id) {
    return vexb_function_register_ex(name, ret_dtype, nargs, arg_dtypes, body, 0, nullptr, nullptr, id);
}

extern "C" int vexb_function_register_ex(const char *name, int ret_dtype, int nargs, const int *arg_dtypes, const char *body,
                                         int ndeps, const int *deps, const char *preamble, int *id) {
    VEXB_CHECK(name && body && id, "NULL argument");
    VEXB_CHECK(ndeps >= 0 && ndeps <= kMaxDeps && (ndeps == 0 || deps), "a user function lists 0..%d dependencies", kMaxDeps);
    VEXB_CHECK(ret_dtype >= VEXB_F64 && ret_dtype <= VEXB_U64, "bad return type %d", ret_dtype);
    VEXB_CHECK(nargs >= 0 && nargs <= 8 && (nargs == 0 || arg_dtypes), "a user function takes 0..8 arguments");
    VEXB_CHECK(*name && (isalpha((unsigned char)*name) || *name == '_'), "'%s' is not an identifier", name);
    for (const char *c = name; *c; ++c) VEXB_CHECK(isalnum((unsigned char)*c) || *c == '_', "'%s' is not an identifier", name);
    UserFunc f; f.name = name; f.ret = ret_dtype; f.body = body;
    for (int k = 0; k < nargs; ++k) {
        // a value type, or VEXB_PTR(value type): a `T *` parameter that takes a VEXB_TERM_PTR terminal
        const int base = is_ptr_type(arg_dtypes[k]) ? arg_dtypes[k] & ~VEXB_PTR(0) : arg_dtypes[k];
        VEXB_CHECK(base >= VEXB_F64 && base <= VEXB_U64 && (arg_dtypes[k] == base || arg_dtypes[k] == VEXB_PTR(base)), "bad type of argument %d", k);
        f.args.push_back(arg_dtypes[k]);
    }
    if (preamble) f.preamble = preamble;
    std::lock_guard<std::mutex> l(g_fmx);
    for (int k = 0; k < ndeps; ++k) {
        VEXB_CHECK(deps[k] >= 0 && (size_t)deps[k] < g_funcs.size(), "dependency %d: %d is not a registered function", k, deps[k]);
        f.deps.push_back(deps[k]);
    }
    for (size_t k = 0; k < g_funcs.size(); ++k) {
        const UserFunc &o = g_funcs[k];
        if (o.name == f.name && o.ret == f.ret && o.args == f.args && o.body == f.body && o.deps == f.deps && o.preamble == f.preamble) {
            *id = (int)k;
            return VEXB_OK;
        }
    }
    VEXB_CHECK(g_funcs.size() < 65535, "too many user functions");
    g_funcs.push_back(f);
    *id = (int)g_funcs.size() - 1;
    return VEXB_OK;
}

// Compile the kernel of a request shape ahead of its first use (background != 0: on a background thread, as the first
// vexb_eval of that shape would).  Needs NVRTC but no device: the module is loaded by the first launch.
extern "C" int vexb_jit_precompile(int lhs_dtype, int assign_op, const vexb_expr *expr, int background) {
    VEXB_CHECK(expr, "expr is NULL");
    VEXB_CHECK(lhs_dtype >= VEXB_F64 && lhs_dtype <= VEXB_U64, "bad lhs dtype %d", lhs_dtype);
    VEXB_CHECK(assign_op >= VEXB_SET && assign_op <= VEXB_RSH, "bad assign op %d", assign_op);
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, false));
    int sell = -1;
    VEXB_TRY(sell_sweep_term(e, &sell));
    void *fn = nullptr;
    const vexb_expr *pe = &e;
    return jit_program(-1, request_signature(e, lhs_dtype, assign_op), "vexb_jit_kernel", std::string(), [&](JitBuild *b) {
        b->background = background != 0;
        b->device_default = program_has_preamble(&pe, 1);
        return generate_source(e, lhs_dtype, assign_op, &b->text);
    }, !background, &fn);
}

extern "C" int vexb_jit_pending(int *pending) {
    VEXB_CHECK(pending, "pending is NULL");
    *pending = jit_pending();
    return VEXB_OK;
}

extern "C" int vexb_program_header_push(int dev, const char *text) {
    VEXB_CHECK(dev >= 0 && dev < kMaxHeaderDevices, "bad device ordinal %d", dev);
    VEXB_CHECK(text, "text is NULL");
    std::lock_guard<std::mutex> l(g_hdr_mx);
    g_headers[dev].push_back(text);
    return VEXB_OK;
}

extern "C" int vexb_program_header_pop(int dev) {
    VEXB_CHECK(dev >= 0 && dev < kMaxHeaderDevices, "bad device ordinal %d", dev);
    std::lock_guard<std::mutex> l(g_hdr_mx);
    auto it = g_headers.find(dev);
    VEXB_CHECK(it != g_headers.end() && !it->second.empty(), "no program header was pushed on device %d", dev);
    it->second.pop_back();
    return VEXB_OK;
}

extern "C" int vexb_program_header_get(int dev, char *buf, size_t *len) {
    VEXB_CHECK(len, "len is NULL");
    VEXB_CHECK(dev >= 0 && dev < kMaxHeaderDevices, "bad device ordinal %d", dev);
    const std::string h = program_header(dev);
    if (buf) {
        VEXB_CHECK(*len > h.size(), "buffer too small (%zu <= %zu)", *len, h.size());
        memcpy(buf, h.c_str(), h.size() + 1);
    }
    *len = h.size() + 1;
    return VEXB_OK;
}

// The kernel vexb_eval_multi would generate for these components, as text (and, with compile != 0, compiled by NVRTC for
// sm_90a without touching a device): lets a CPU-only box check that multi-expression kernels build.
extern "C" int vexb_jit_source_multi(int lhs_dtype, int assign_op, int ncomp, const vexb_expr *const *exprs, char *buf, size_t *len, int compile) {
    return vexb_jit_source_multi_dev(-1, lhs_dtype, assign_op, ncomp, exprs, buf, len, compile);
}

// The printers below with dev >= 0 print what device dev would compile, its program header included; dev = -1: no header.
static int check_print_dev(int dev) {
    VEXB_CHECK(dev >= -1 && dev < kMaxHeaderDevices, "bad device ordinal %d", dev);
    return VEXB_OK;
}

extern "C" int vexb_jit_source_multi_dev(int dev, int lhs_dtype, int assign_op, int ncomp, const vexb_expr *const *exprs, char *buf,
                                         size_t *len, int compile) {
    VEXB_TRY(check_print_dev(dev));
    VEXB_CHECK(len && exprs, "NULL argument");
    VEXB_CHECK(ncomp >= 2 && ncomp <= 8, "a multi-expression kernel takes 2..8 components");
    VEXB_CHECK(lhs_dtype >= VEXB_F64 && lhs_dtype <= VEXB_U64, "bad lhs dtype %d", lhs_dtype);
    VEXB_CHECK(assign_op >= VEXB_SET && assign_op <= VEXB_RSH, "bad assign op %d", assign_op);
    std::vector<vexb_expr> es((size_t)ncomp);
    std::vector<const vexb_expr *> ps((size_t)ncomp);
    for (int c = 0; c < ncomp; ++c) {
        VEXB_CHECK(exprs[c], "expression %d is NULL", c);
        VEXB_TRY(normalize_expr(exprs[c], &es[(size_t)c], false));
        ps[(size_t)c] = &es[(size_t)c];
    }
    std::string src;
    VEXB_TRY(generate_source_n(ps.data(), ncomp, lhs_dtype, assign_op, &src));
    return jit_print(with_program_header(header_for(dev, ps.data(), ncomp), src), compile, program_has_preamble(ps.data(), ncomp), buf, len);
}

extern "C" int vexb_jit_source(int lhs_dtype, int assign_op, const vexb_expr *expr, char *buf, size_t *len, int compile) {
    return vexb_jit_source_dev(-1, lhs_dtype, assign_op, expr, buf, len, compile);
}

extern "C" int vexb_jit_source_dev(int dev, int lhs_dtype, int assign_op, const vexb_expr *expr, char *buf, size_t *len, int compile) {
    VEXB_TRY(check_print_dev(dev));
    VEXB_CHECK(len, "len is NULL");
    VEXB_CHECK(lhs_dtype >= VEXB_F64 && lhs_dtype <= VEXB_U64, "bad lhs dtype %d", lhs_dtype);
    VEXB_CHECK(assign_op >= VEXB_SET && assign_op <= VEXB_RSH, "bad assign op %d", assign_op);
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, false));
    std::string src;
    VEXB_TRY(generate_source(e, lhs_dtype, assign_op, &src));
    const vexb_expr *pe = &e;
    return jit_print(with_program_header(header_for(dev, &pe, 1), src), compile, program_has_preamble(&pe, 1), buf, len);
}

// The kernel vexb_reduce_all (nops == 1) or vexb_reduce_multi (nops > 1) generates for a reduction of this expression in
// `dtype`, as text (and, with compile != 0, compiled by NVRTC for sm_90a without touching a device).  The skeleton follows
// the tunables in force ("eval.force_interp").  Every argument is checked before anything is generated.
extern "C" int vexb_jit_source_reduce(int dtype, int nops, const int *ops, const vexb_expr *expr, char *buf, size_t *len, int compile) {
    return vexb_jit_source_reduce_dev(-1, dtype, nops, ops, expr, buf, len, compile);
}

extern "C" int vexb_jit_source_reduce_dev(int dev, int dtype, int nops, const int *ops, const vexb_expr *expr, char *buf, size_t *len,
                                          int compile) {
    VEXB_TRY(check_print_dev(dev));
    VEXB_CHECK(len, "len is NULL");
    VEXB_CHECK(dtype >= VEXB_F64 && dtype <= VEXB_U64, "bad dtype %d", dtype);
    VEXB_CHECK(nops >= 1 && nops <= VEXB_MAX_COMBINED && ops, "between 1 and %d reductions can be combined", VEXB_MAX_COMBINED);
    int mo[VEXB_MAX_COMBINED];
    for (int k = 0; k < nops; ++k) {
        if (nops == 1) VEXB_CHECK(ops[k] >= VEXB_SUM && ops[k] <= VEXB_MINMAX, "bad reduce op %d", ops[k]);
        else VEXB_CHECK(ops[k] >= VEXB_SUM && ops[k] <= VEXB_MIN, "reduction %d: only SUM, SUM_Kahan, MAX and MIN combine", k);
        mo[k] = (ops[k] == VEXB_SUM_KAHAN && !dtype_is_float(dtype)) ? VEXB_SUM : ops[k];
    }
    vexb_expr e;
    VEXB_TRY(normalize_expr(expr, &e, false));
    std::string src;
    VEXB_TRY(generate_reduce_source(e, dtype, nops, mo, reduce_skeleton(e, dtype, nops > 1), &src));
    const vexb_expr *pe = &e;
    return jit_print(with_program_header(header_for(dev, &pe, 1), src), compile, program_has_preamble(&pe, 1), buf, len);
}
