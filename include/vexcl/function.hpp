#ifndef VEXCL_FUNCTION_HPP
#define VEXCL_FUNCTION_HPP
/*
 * Builtin device functions usable inside vector expressions (vexcl/function.hpp:255-268 and the
 * list that follows :287).  Each maps to one IR opcode evaluated with CUDA's math library.
 * The result type is the common type of the arguments (as the reference assumes,
 * operations.hpp:1750-1764); integer arguments of floating-only functions are promoted to double.
 *
 * User-defined functions (VEX_FUNCTION and friends, function.hpp:46-225) carry a C source body, optionally a list of
 * user functions the body calls by name (VEX_FUNCTION_D / _SD / _DS) or a file-scope preamble
 * (VEX_FUNCTION_V1_WITH_PREAMBLE); expressions that call one are compiled at first use by the library's NVRTC side
 * path (csrc/jit.cu) and cached.
 */
#include <cctype>
#include <string>
#include <type_traits>
#include "operations.hpp"

namespace vex {

template <int OP, bool FloatOnly, class... Args>
struct function_node : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef typename std::common_type<typename detail::value_of<Args>::type...>::type common;
    typedef typename std::conditional<FloatOnly && std::is_integral<common>::value, double,
                                      typename detail::promoted<common>::type>::type value_type;
    static const size_t multi_size = detail::max_ncomp<Args...>::value;
    std::tuple<Args...> args;
    explicit function_node(Args... a) : args(a...) {}

    int lower(detail::ir_builder &b) const {
        lower_args(b, std::index_sequence_for<Args...>());
        b.emit(OP, dtype_of<value_type>::value);
        return dtype_of<value_type>::value;
    }
    void props(detail::expr_props &p) const { props_args(p, std::index_sequence_for<Args...>()); }
    private:
        template <size_t... I> void lower_args(detail::ir_builder &b, std::index_sequence<I...>) const {
            int dummy[] = {0, (b.cvt(std::get<I>(args).lower(b), dtype_of<value_type>::value), 0)...}; (void)dummy;
        }
        template <size_t... I> void props_args(detail::expr_props &p, std::index_sequence<I...>) const {
            int dummy[] = {0, (std::get<I>(args).props(p), 0)...}; (void)dummy;
        }
};

#define VEXCL_BUILTIN_1(name, OP, FLOATONLY) \
    template <class A> \
    const typename std::enable_if<is_vector_expr<A>::value, function_node<OP, FLOATONLY, typename detail::operand<A>::type> >::type \
    name(const A &a) { return function_node<OP, FLOATONLY, typename detail::operand<A>::type>(detail::operand<A>::wrap(a)); }

#define VEXCL_BUILTIN_2(name, OP, FLOATONLY) \
    template <class A, class B> \
    const typename std::enable_if<detail::is_operand<A>::value && detail::is_operand<B>::value && \
                            (is_vector_expr<A>::value || is_vector_expr<B>::value), \
        function_node<OP, FLOATONLY, typename detail::operand<A>::type, typename detail::operand<B>::type> >::type \
    name(const A &a, const B &b) { \
        return function_node<OP, FLOATONLY, typename detail::operand<A>::type, typename detail::operand<B>::type>( \
                detail::operand<A>::wrap(a), detail::operand<B>::wrap(b)); }

#define VEXCL_BUILTIN_3(name, OP, FLOATONLY) \
    template <class A, class B, class C> \
    const typename std::enable_if<detail::is_operand<A>::value && detail::is_operand<B>::value && detail::is_operand<C>::value && \
                            (is_vector_expr<A>::value || is_vector_expr<B>::value || is_vector_expr<C>::value), \
        function_node<OP, FLOATONLY, typename detail::operand<A>::type, typename detail::operand<B>::type, typename detail::operand<C>::type> >::type \
    name(const A &a, const B &b, const C &c) { \
        return function_node<OP, FLOATONLY, typename detail::operand<A>::type, typename detail::operand<B>::type, typename detail::operand<C>::type>( \
                detail::operand<A>::wrap(a), detail::operand<B>::wrap(b), detail::operand<C>::wrap(c)); }

VEXCL_BUILTIN_1(sin, VEXB_OP_SIN, true)     VEXCL_BUILTIN_1(cos, VEXB_OP_COS, true)     VEXCL_BUILTIN_1(tan, VEXB_OP_TAN, true)
VEXCL_BUILTIN_1(asin, VEXB_OP_ASIN, true)   VEXCL_BUILTIN_1(acos, VEXB_OP_ACOS, true)   VEXCL_BUILTIN_1(atan, VEXB_OP_ATAN, true)
VEXCL_BUILTIN_1(sinh, VEXB_OP_SINH, true)   VEXCL_BUILTIN_1(cosh, VEXB_OP_COSH, true)   VEXCL_BUILTIN_1(tanh, VEXB_OP_TANH, true)
VEXCL_BUILTIN_1(exp, VEXB_OP_EXP, true)     VEXCL_BUILTIN_1(exp2, VEXB_OP_EXP2, true)   VEXCL_BUILTIN_1(log, VEXB_OP_LOG, true)
VEXCL_BUILTIN_1(log2, VEXB_OP_LOG2, true)   VEXCL_BUILTIN_1(log10, VEXB_OP_LOG10, true) VEXCL_BUILTIN_1(sqrt, VEXB_OP_SQRT, true)
VEXCL_BUILTIN_1(rsqrt, VEXB_OP_RSQRT, true) VEXCL_BUILTIN_1(cbrt, VEXB_OP_CBRT, true)   VEXCL_BUILTIN_1(fabs, VEXB_OP_FABS, false)
VEXCL_BUILTIN_1(abs, VEXB_OP_FABS, false)   VEXCL_BUILTIN_1(floor, VEXB_OP_FLOOR, true) VEXCL_BUILTIN_1(ceil, VEXB_OP_CEIL, true)
VEXCL_BUILTIN_1(round, VEXB_OP_ROUND, true) VEXCL_BUILTIN_1(trunc, VEXB_OP_TRUNC, true)
VEXCL_BUILTIN_2(pow, VEXB_OP_POW, true)     VEXCL_BUILTIN_2(atan2, VEXB_OP_ATAN2, true) VEXCL_BUILTIN_2(fmod, VEXB_OP_FMOD, true)
VEXCL_BUILTIN_2(hypot, VEXB_OP_HYPOT, true) VEXCL_BUILTIN_2(fmin, VEXB_OP_FMIN, false)  VEXCL_BUILTIN_2(fmax, VEXB_OP_FMAX, false)
VEXCL_BUILTIN_2(min, VEXB_OP_FMIN, false)   VEXCL_BUILTIN_2(max, VEXB_OP_FMAX, false)
VEXCL_BUILTIN_3(fma, VEXB_OP_FMA, true)     VEXCL_BUILTIN_3(mad, VEXB_OP_FMA, true)

#undef VEXCL_BUILTIN_1
#undef VEXCL_BUILTIN_2
#undef VEXCL_BUILTIN_3

// ---- user-defined functions ------------------------------------------------------------------------
namespace detail {

/// The IR type of an argument spelled `t`.  `T*` and `const T*` over the six element types are pointer parameters
/// (VEXB_PTR(T)), which take a vex::raw_pointer (vector_pointer.hpp).
inline int dtype_from_name(std::string t) {
    std::string u;
    for (char c : t) if (!std::isspace(static_cast<unsigned char>(c))) u += c;
    if (!u.empty() && u.back() == '*') {
        std::string e = u.substr(0, u.size() - 1);
        if (e.compare(0, 5, "const") == 0) e = e.substr(5);
        if (e.compare(0, 3, "cl_") == 0) e = e.substr(3);
        // only the six element types: bool, char and short would name arrays of another element size
        if (e == "double") return VEXB_PTR(VEXB_F64);
        if (e == "float") return VEXB_PTR(VEXB_F32);
        if (e == "int") return VEXB_PTR(VEXB_I32);
        if (e == "uint" || e == "unsigned" || e == "unsignedint") return VEXB_PTR(VEXB_U32);
        if (e == "long" || e == "longlong" || e == "ptrdiff_t") return VEXB_PTR(VEXB_I64);
        if (e == "ulong" || e == "size_t" || e == "unsignedlong" || e == "unsignedlonglong") return VEXB_PTR(VEXB_U64);
        throw std::runtime_error("VEX_FUNCTION: unsupported pointer argument type '" + t + "'");
    }
    if (u.compare(0, 3, "cl_") == 0) u = u.substr(3);
    if (u == "double") return VEXB_F64;
    if (u == "float") return VEXB_F32;
    if (u == "int" || u == "bool" || u == "char" || u == "short") return VEXB_I32;
    if (u == "uint" || u == "unsigned" || u == "unsignedint") return VEXB_U32;
    if (u == "long" || u == "longlong" || u == "ptrdiff_t") return VEXB_I64;
    if (u == "ulong" || u == "size_t" || u == "unsignedlong" || u == "unsignedlonglong") return VEXB_U64;
    throw std::runtime_error("VEX_FUNCTION: unsupported argument type '" + t + "'");
}
inline const char* dtype_c_name(int dt) {
    switch (dt) { case VEXB_F64: return "double"; case VEXB_F32: return "float"; case VEXB_I32: return "int";
                  case VEXB_U32: return "unsigned int"; case VEXB_I64: return "long long"; default: return "unsigned long long"; }
}
/// Parse "(double, x)(double, y)" into types and a prologue that names the arguments.
inline void parse_arguments(const std::string &seq, std::vector<int> &types, std::string &prologue) {
    size_t pos = 0;
    while ((pos = seq.find('(', pos)) != std::string::npos) {
        const size_t end = seq.find(')', pos), comma = seq.rfind(',', end);
        precondition(end != std::string::npos && comma != std::string::npos && comma > pos, "VEX_FUNCTION: malformed argument list");
        std::string type = seq.substr(pos + 1, comma - pos - 1), name = seq.substr(comma + 1, end - comma - 1);
        name.erase(0, name.find_first_not_of(" \t")); name.erase(name.find_last_not_of(" \t") + 1);
        types.push_back(dtype_from_name(type));
        if (types.back() & VEXB_PTR(0)) {             // T *name = prmK; (const T *name for a const T* parameter)
            const bool c = type.find("const") != std::string::npos;
            prologue += std::string(c ? "const " : "") + dtype_c_name(types.back() & ~VEXB_PTR(0)) + " *" + name + " = prm" + std::to_string(types.size()) + "; ";
        } else
        prologue += std::string("const ") + dtype_c_name(types.back()) + " " + name + " = prm" + std::to_string(types.size()) + "; ";
        pos = end + 1;
    }
}
/// The IR type of a parameter of a signature: T* and const T* are pointer parameters (VEXB_PTR).
template <class A> struct param_dtype { static const int value = dtype_of<typename promoted<A>::type>::value; };
template <class A> struct param_dtype<A*> { static const int value = VEXB_PTR(dtype_of<typename std::remove_cv<A>::type>::value); };
template <class T> struct signature_types;
template <class R, class... A> struct signature_types<R(A...)> {
    typedef R result;
    static std::vector<int> args() { return std::vector<int>{param_dtype<A>::value...}; }
};

} // namespace detail

template <class Ret, class... Args>
struct call_node : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef typename detail::promoted<Ret>::type value_type;
    static const size_t multi_size = detail::max_ncomp<Args...>::value;
    int id; std::vector<int> arg_types;
    std::tuple<Args...> args;
    call_node(int id, const std::vector<int> &arg_types, Args... a) : id(id), arg_types(arg_types), args(a...) {}
    int lower(detail::ir_builder &b) const {
        lower_args(b, std::index_sequence_for<Args...>());
        b.emit(VEXB_OP_CALL, dtype_of<value_type>::value, id);
        return dtype_of<value_type>::value;
    }
    void props(detail::expr_props &p) const { props_args(p, std::index_sequence_for<Args...>()); }
    private:
        template <size_t... I> void lower_args(detail::ir_builder &b, std::index_sequence<I...>) const {
            int dummy[] = {0, (arg(b, std::get<I>(args).lower(b), arg_types[I]), 0)...}; (void)dummy;
        }
        template <size_t... I> void props_args(detail::expr_props &p, std::index_sequence<I...>) const {
            int dummy[] = {0, (std::get<I>(args).props(p), 0)...}; (void)dummy;
        }
        // a pointer parameter takes a raw_pointer of its element type, and a raw_pointer goes to nothing else
        static void arg(detail::ir_builder &b, int t, int declared) {
            precondition(!((t | declared) & VEXB_PTR(0)) || t == declared,
                         "user function: a T* parameter takes a vex::raw_pointer of a vector<T>, and a raw_pointer goes to nothing else");
            b.cvt(t, declared);
        }
};

/// Base of the objects the VEX_FUNCTION macros define.  Impl supplies fn_name(), fn_types(), fn_deps(), fn_preamble()
/// and fn_body().  Dependencies are registered first (their ids come from their own id()), so a function's id is always
/// larger than those of the functions its body calls.
template <class Impl, class Ret>
struct user_function {
    typedef Ret result_type;
    static int id(std::vector<int> *types_out = nullptr) {
        static std::vector<int> types;
        static const int fid = [] {
            std::string prologue;
            Impl::fn_types(types, prologue);
            std::vector<int> deps;
            Impl::fn_deps(deps);
            const std::string preamble = Impl::fn_preamble();
            int k = -1;
            VEXB_CHECKED(vexb_function_register_ex(Impl::fn_name(), dtype_of<typename detail::promoted<Ret>::type>::value,
                                                   static_cast<int>(types.size()), types.data(), (prologue + Impl::fn_body()).c_str(),
                                                   static_cast<int>(deps.size()), deps.data(), preamble.c_str(), &k));
            return k;
        }();
        if (types_out) *types_out = types;
        return fid;
    }
    template <class... A>
    const call_node<Ret, typename detail::operand<A>::type...> operator()(const A&... a) const {
        std::vector<int> types;
        const int fid = id(&types);
        precondition(types.size() == sizeof...(A), std::string(Impl::fn_name()) + ": wrong number of arguments");
        return call_node<Ret, typename detail::operand<A>::type...>(fid, types, detail::operand<A>::wrap(a)...);
    }
};

} // namespace vex

/// Converts unquoted text into a string literal (function.hpp:46).
#define VEX_STRINGIZE_SOURCE(...) #__VA_ARGS__

// The dependency sequence (f)(g)(h) of VEX_FUNCTION_D / _SD as statements `deps.push_back(<id of f>);`, one per element:
// the two macros call each other through the sequence and the last one left is pasted into an empty *_END.
#define VEXCL_FUNCTION_DEP_0(dep) deps.push_back(std::decay<decltype(dep)>::type::id()); VEXCL_FUNCTION_DEP_1
#define VEXCL_FUNCTION_DEP_1(dep) deps.push_back(std::decay<decltype(dep)>::type::id()); VEXCL_FUNCTION_DEP_0
#define VEXCL_FUNCTION_DEP_0_END
#define VEXCL_FUNCTION_DEP_1_END
#define VEXCL_FUNCTION_CAT(a, b) VEXCL_FUNCTION_CAT_I(a, b)
#define VEXCL_FUNCTION_CAT_I(a, b) a##b
#define VEXCL_FUNCTION_DEPS(seq) VEXCL_FUNCTION_CAT(VEXCL_FUNCTION_DEP_0 seq, _END)

/// The object `fname` of type vex_function_fname, registered under the plain name "fname" (the name dependents call).
#define VEXCL_FUNCTION_SINK(rettype, fname, fargs, dependencies, preamble_str, body_str) \
    struct vex_function_##fname : vex::user_function<vex_function_##fname, rettype> { \
        vex_function_##fname() {} \
        static const char* fn_name() { return #fname; } \
        static void fn_types(std::vector<int> &t, std::string &prologue) { vex::detail::parse_arguments(#fargs, t, prologue); } \
        static void fn_deps(std::vector<int> &deps) { (void)deps; VEXCL_FUNCTION_DEPS(dependencies) } \
        static std::string fn_preamble() { return preamble_str; } \
        static std::string fn_body() { return body_str; } \
    } const fname

/// VEX_FUNCTION_SD(return_type, name, (type1, arg1)..., (dep1)(dep2)..., body_str)   -- function.hpp:194-203
/// A function whose body calls the user functions dep1, dep2, ... by name; they are compiled into every program that
/// calls it.
#define VEX_FUNCTION_SD(rettype, fname, fargs, dependencies, body_str) \
    VEXCL_FUNCTION_SINK(rettype, fname, fargs, dependencies, "", body_str)
#define VEX_FUNCTION_DS VEX_FUNCTION_SD
/// Same with the body as unquoted source.
#define VEX_FUNCTION_D(rettype, fname, fargs, dependencies, ...) \
    VEX_FUNCTION_SD(rettype, fname, fargs, dependencies, #__VA_ARGS__)
/// VEX_FUNCTION(return_type, name, (type1, arg1)(type2, arg2)..., body)      -- function.hpp:225
#define VEX_FUNCTION(rettype, fname, fargs, ...) VEX_FUNCTION_S(rettype, fname, fargs, #__VA_ARGS__)
/// Same with the body given as a string.
#define VEX_FUNCTION_S(rettype, fname, fargs, body_str) VEX_FUNCTION_SD(rettype, fname, fargs, , body_str)

/// Older form, the type only: VEX_FUNCTION_V1_TYPE(name, double(double, double), preamble_str, "return prm1 + prm2;")
/// defines vex_function_name (function.hpp:70-118).  The preamble is file-scope text (helpers, macros) before the body.
#define VEX_FUNCTION_V1_TYPE(fname, signature, preamble_str, body_str) \
    struct vex_function_##fname : vex::user_function<vex_function_##fname, vex::detail::signature_types<signature>::result> { \
        vex_function_##fname() {} \
        static const char* fn_name() { return #fname; } \
        static void fn_types(std::vector<int> &t, std::string&) { t = vex::detail::signature_types<signature>::args(); } \
        static void fn_deps(std::vector<int>&) {} \
        static std::string fn_preamble() { return preamble_str; } \
        static std::string fn_body() { return body_str; } \
    }
/// VEX_FUNCTION_V1(name, double(double, double), "return prm1 + prm2;")
#define VEX_FUNCTION_V1(fname, signature, body_str) VEX_FUNCTION_V1_TYPE(fname, signature, "", body_str) const fname
/// VEX_FUNCTION_V1_WITH_PREAMBLE(name, double(double), "double sq(double x) { return x * x; }\n", "return sq(prm1);")
#define VEX_FUNCTION_V1_WITH_PREAMBLE(fname, signature, preamble_str, body_str) \
    VEX_FUNCTION_V1_TYPE(fname, signature, preamble_str, body_str) const fname

#endif
