#ifndef VEXCL_OPERATIONS_HPP
#define VEXCL_OPERATIONS_HPP
/*
 * Expression front end.  The reference builds Boost.Proto trees and, per expression
 * type, emits and compiles kernel source (vexcl/operations.hpp:455-512 grammar,
 * :1209-1353 emitters, :1818-1897 assign_expression).  Here the trees are plain C++17
 * templates and are lowered, per call, to the postfix IR of include/vexb200.h; the
 * library picks a pre-compiled sm_90a kernel for it (hand-written sweep for the
 * recognised shapes, interpreter otherwise).  No Boost, no run-time compilation.
 *
 * Accepted operators = the reference grammar's (operations.hpp:457-506):
 *   + - * / %   unary + -   < > <= >= == !=   && || !   & | ^ << >>
 * plus builtin functions (function.hpp), if_else, element_index, tagged terminals, and the subscript and
 * dereference of a vex::raw_pointer (vector_pointer.hpp).
 * Arithmetic scalars are by-value terminals (operations.hpp:168-175).  Node value
 * types follow C++'s usual arithmetic conversions; comparisons and logical operators
 * yield int.
 */
#include <algorithm>
#include <cstring>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>
#include "backend.hpp"
#include "types.hpp"
#include "util.hpp"

namespace vex {

template <typename T> class vector;

/// Marker base of every expression node and terminal.
struct vector_expr_tag {};
/// Specialised for operands that are not nodes: vex::SpMatCCSR products (spmat/ccsr.hpp).
template <class T> struct is_vector_expr_type : std::is_base_of<vector_expr_tag, T> {};
template <class T> struct is_vector_expr : is_vector_expr_type<typename std::decay<T>::type> {};

/// Assignment operators, same set as vexcl/operations.hpp:70-80.
namespace assign {
struct SET { static const int op = VEXB_SET; }; struct ADD { static const int op = VEXB_ADD; };
struct SUB { static const int op = VEXB_SUB; }; struct MUL { static const int op = VEXB_MUL; };
struct DIV { static const int op = VEXB_DIV; }; struct MOD { static const int op = VEXB_MOD; };
struct AND { static const int op = VEXB_AND; }; struct OR  { static const int op = VEXB_OR;  };
struct XOR { static const int op = VEXB_XOR; }; struct LSH { static const int op = VEXB_LSH; };
struct RSH { static const int op = VEXB_RSH; };
}

namespace detail {

/// Builds the IR of one expression for one device slice.
struct ir_builder {
    vexb_expr e;
    unsigned part;
    int comp;                       ///< component being lowered when the expression is a multi-expression, else -1
    explicit ir_builder(unsigned part, int comp = -1) : part(part), comp(comp) { std::memset(&e, 0, sizeof(e)); }

    int new_term() {
        precondition(e.n_terms < VEXB_MAX_TERMS, "expression has too many terminals");
        return e.n_terms++;
    }
    void emit(int op, int type, int arg = 0) {
        precondition(e.n_code < VEXB_MAX_CODE, "expression is too long");
        vexb_instr &i = e.code[e.n_code++];
        i.op = static_cast<uint8_t>(op); i.type = static_cast<uint8_t>(type); i.arg = static_cast<uint16_t>(arg);
    }
    void push_vec(const void *ptr, int dtype) {
        int k = new_term();
        e.term[k].kind = VEXB_TERM_VEC; e.term[k].dtype = static_cast<uint8_t>(dtype); e.term[k].v.ptr = ptr;
        emit(VEXB_OP_TERM, dtype, k);
    }
    template <class T> void push_scalar(T v) {
        typedef typename std::conditional<std::is_floating_point<T>::value, T,
                typename std::conditional<(sizeof(T) < 4), int, T>::type>::type P;     // integer promotion
        const int dt = dtype_of<P>::value;
        int k = new_term();
        e.term[k].kind = VEXB_TERM_SCALAR; e.term[k].dtype = static_cast<uint8_t>(dt);
        const P p = static_cast<P>(v);
        std::memcpy(&e.term[k].v, &p, sizeof(P));
        emit(VEXB_OP_TERM, dt, k);
    }
    void push_index(long long offset) {
        int k = new_term();
        e.term[k].kind = VEXB_TERM_INDEX; e.term[k].dtype = VEXB_U64; e.term[k].v.i64 = offset;
        emit(VEXB_OP_TERM, VEXB_U64, k);
    }
    /// Row `i` of `A * x` as a terminal (VEXB_TERM_SPMV): A is a plain strip on this device, xptr its x slice.
    void push_spmv(const vexb_spmat *A, const void *xptr, int dtype) {
        int xs = new_term();
        e.term[xs].kind = VEXB_TERM_VEC; e.term[xs].dtype = static_cast<uint8_t>(dtype); e.term[xs].v.ptr = xptr;
        int k = new_term();
        e.term[k].kind = VEXB_TERM_SPMV; e.term[k].dtype = static_cast<uint8_t>(dtype); e.term[k].v.ptr = A;
        e.term[k].pad[0] = static_cast<uint8_t>(xs);
        emit(VEXB_OP_TERM, dtype, k);
    }
    /// Row `i` of `A * x` for a vex::SpMatCCSR (VEXB_TERM_CCSR); idx_bytes: the matrix's idx width on the device.
    void push_ccsr(const vexb_ccsr *A, int idx_bytes, const void *xptr, int dtype) {
        int xs = new_term();
        e.term[xs].kind = VEXB_TERM_VEC; e.term[xs].dtype = static_cast<uint8_t>(dtype); e.term[xs].v.ptr = xptr;
        int k = new_term();
        e.term[k].kind = VEXB_TERM_CCSR; e.term[k].dtype = static_cast<uint8_t>(dtype); e.term[k].v.ptr = A;
        e.term[k].pad[0] = static_cast<uint8_t>(xs); e.term[k].pad[1] = static_cast<uint8_t>(idx_bytes);
        emit(VEXB_OP_TERM, dtype, k);
    }
    void cvt(int from, int to) { if (from != to) emit(VEXB_OP_CVT, to, from); }
    /// A raw pointer (VEXB_TERM_PTR): the device address of element 0 of an array of `count` elements of `dtype` (a load
    /// outside them reads 0).  Returns its slot, for a VEXB_OP_LOAD or a VEXB_OP_TERM that passes the pointer to a user
    /// function.
    int ptr_term(const void *ptr, int dtype, size_t count) {
        int k = new_term();
        e.term[k].kind = VEXB_TERM_PTR; e.term[k].dtype = static_cast<uint8_t>(dtype); e.term[k].v.ptr = ptr;
        for (int b = 0; b < 6; ++b) e.term[k].pad[b] = static_cast<uint8_t>(static_cast<unsigned long long>(count) >> (8 * b));
        return k;
    }

    // ---- temporaries (vex::make_temp, temporary.hpp) ----
    // The program is code[0, n_prefix), the definitions in post-order (each ends with its VEXB_OP_TDEF), then the
    // expression.  A definition is lowered in place, where its first use is, and then moved to the end of the prefix.
    int n_prefix = 0;
    struct temp_def { size_t tag; int type; std::string def; };
    std::vector<temp_def> temps;                      ///< slot k: temporary make_temp<tag>, with its definition by content

    /// A temporary whose definition was just lowered: code[n_prefix + rel, n_code), with terminals from slot `terms` on.
    /// The first use of `tag` moves it into the prefix; a later one drops it again (when it is the same program) and both
    /// read the one slot.
    void use_temp(size_t tag, int rel, int terms, int type) {
        const int from = n_prefix + rel;              // definitions of nested temporaries have moved into the prefix meanwhile
        const std::string def = definition(from, e.n_code);
        for (size_t k = 0; k < temps.size(); ++k) if (temps[k].tag == tag) {
            if (temps[k].def != def || temps[k].type != type)
                throw backend::error(VEXB_ERR_INVALID, "make_temp<" + std::to_string(tag) + ">: one tag names two different expressions");
            e.n_code = from;                          // the same program: its second lowering (no new temporaries) goes
            for (int j = terms; j < e.n_terms; ++j) std::memset(&e.term[j], 0, sizeof(vexb_term));
            e.n_terms = terms;
            emit(VEXB_OP_TREF, type, static_cast<int>(k));
            return;
        }
        precondition(temps.size() < VEXB_MAX_TEMPS, "expression has too many temporaries");
        emit(VEXB_OP_TDEF, type, static_cast<int>(temps.size()));
        std::rotate(e.code + n_prefix, e.code + from, e.code + e.n_code);
        n_prefix += e.n_code - from;
        temps.push_back(temp_def{tag, type, def});
        emit(VEXB_OP_TREF, type, static_cast<int>(temps.size() - 1));
    }
    private:
        // code[from, to) with every terminal by content (a product's x too), so that two lowerings compare equal
        std::string definition(int from, int to) const {
            std::string d;
            for (int pc = from; pc < to; ++pc) {
                const vexb_instr &in = e.code[pc];
                d.append(reinterpret_cast<const char*>(&in), sizeof(in) - sizeof(in.arg));
                if (in.op != VEXB_OP_TERM && in.op != VEXB_OP_LOAD) { d.append(reinterpret_cast<const char*>(&in.arg), sizeof(in.arg)); continue; }
                vexb_term t = e.term[in.arg];
                const bool product = t.kind == VEXB_TERM_SPMV || t.kind == VEXB_TERM_CCSR;
                if (product) t.pad[0] = 0;
                d.append(reinterpret_cast<const char*>(&t), sizeof(t));
                if (product) d.append(reinterpret_cast<const char*>(&e.term[e.term[in.arg].pad[0]]), sizeof(vexb_term));
            }
            return d;
        }
};

/// Queue list / partition / size of the first vector terminal (get_expression_properties, operations.hpp:1411).
struct expr_props {
    const std::vector<backend::command_queue> *queue = nullptr;
    std::vector<size_t> part;
    size_t size = 0;
    bool sized = false;
    int comp = -1;                  ///< component being prepared (multi-expressions), else -1
    const void *target = nullptr;   ///< assignments: device slice 0 of the left-hand side (a CCSR product of it takes a temporary)
    /// Assignments only (assign_expression): the generated kernel may sweep in the storage order of ONE sliced-ELL strip
    /// (vexb_dspmat_sweep_strip).  The first product that asks claims it; products of other such matrices take a temporary.
    bool sweeps = false;
    const vexb_spmat *swept = nullptr;
    template <class M> bool claim_sweep(const M &A) {
        if (!sweeps || A.queue_list().empty()) return false;
        for (unsigned d = 0; d < A.queue_list().size(); ++d) if (!A.sweep_strip(d)) return false;
        if (swept && swept != A.sweep_strip(0)) return false;
        swept = A.sweep_strip(0);
        return true;
    }

    void see(const std::vector<backend::command_queue> &q, const std::vector<size_t> &p, size_t n) {
        if (!queue) { queue = &q; part = p; }
        see_size(n);
        see_devices(q);
    }
    /// A raw pointer (vector_pointer.hpp): its queue list, but no size or partition (expression_properties of the
    /// reference's vector_pointer).  Every vector of such an expression must have one part, on the pointer's device.
    void see_pointer(const std::vector<backend::command_queue> &q) {
        if (!queue) queue = &q;
        precondition(ptr_dev < 0 || ptr_dev == q[0].ordinal(), "raw pointers of one expression must live on one device");
        ptr_dev = q[0].ordinal();
        see_devices(q);
    }
    void see_size(size_t n) {
        if (!sized) { size = n; sized = true; }
        else precondition(size == n, "Expression terminals have different sizes");   // VEXCL_CHECK_SIZES (operations.hpp:1824-1840)
    }
    size_t part_size(unsigned d) const { return part.empty() ? 0 : part[d + 1] - part[d]; }
    size_t part_start(unsigned d) const { return part.empty() ? 0 : part[d]; }
    private:
        int ptr_dev = -1;           ///< device of the expression's raw pointers, -1 without
        bool several_parts = false; ///< some vector of the expression has more than one part
        std::vector<int> devs;      ///< devices of the one-part vectors
        void see_devices(const std::vector<backend::command_queue> &q) {
            if (q.size() != 1) several_parts = true;
            else devs.push_back(q[0].ordinal());
            if (ptr_dev < 0) return;
            precondition(!several_parts, "raw_pointer: every vector of the expression must have one part");
            for (int d : devs) precondition(d == ptr_dev, "raw_pointer: every vector of the expression must live on the pointer's device");
        }
};

template <class T> struct promoted {
    typedef typename std::conditional<std::is_floating_point<T>::value, T,
            typename std::conditional<(sizeof(T) < 4), int, T>::type>::type type;
};

} // namespace detail

/// By-value arithmetic terminal.
template <class T>
struct scalar_term : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef typename detail::promoted<T>::type value_type;
    T v;
    explicit scalar_term(T v) : v(v) {}
    int lower(detail::ir_builder &b) const { b.push_scalar(v); return dtype_of<value_type>::value; }
    void props(detail::expr_props&) const {}
};

namespace detail {

// How an operand is held inside a node: vectors and other lvalue terminals by reference,
// temporaries (sub-expressions) by value, arithmetic values as scalar terminals.
template <class X, class Enable = void> struct operand;
template <class X>
struct operand<X, typename std::enable_if<std::is_arithmetic<typename std::decay<X>::type>::value>::type> {
    typedef scalar_term<typename std::decay<X>::type> type;
    static type wrap(const X &x) { return type(x); }
};
template <class X>
struct operand<X, typename std::enable_if<is_vector_expr<X>::value && std::decay<X>::type::hold_by_reference>::type> {
    typedef const typename std::decay<X>::type& type;
    static type wrap(const X &x) { return x; }
};
template <class X>
struct operand<X, typename std::enable_if<is_vector_expr<X>::value && !std::decay<X>::type::hold_by_reference>::type> {
    typedef typename std::decay<X>::type type;
    static type wrap(const X &x) { return x; }
};

template <class X> struct is_operand
    : std::integral_constant<bool, is_vector_expr<X>::value || std::is_arithmetic<typename std::decay<X>::type>::value> {};

template <class X> struct value_of { typedef typename std::decay<X>::type::value_type type; };

// Number of components of a multi-expression (multivector.hpp); 0 for ordinary vector expressions.
template <class X, class Enable = void> struct ncomp : std::integral_constant<size_t, 0> {};
template <class X> struct ncomp<X, typename std::enable_if<(std::decay<X>::type::multi_size > 0)>::type>
    : std::integral_constant<size_t, std::decay<X>::type::multi_size> {};
template <class... X> struct max_ncomp : std::integral_constant<size_t, 0> {};
template <class X, class... Y> struct max_ncomp<X, Y...>
    : std::integral_constant<size_t, (ncomp<X>::value > max_ncomp<Y...>::value ? ncomp<X>::value : max_ncomp<Y...>::value)> {};

} // namespace detail

#define VEXCL_NODE_COMMON static const bool hold_by_reference = false;

// ---- operator tags ------------------------------------------------------------------------
namespace op {
#define VEXB_ARITH_TAG(name, code, sym) \
    struct name { static const int opcode = code; static const bool compare = false; \
        template <class A, class B> struct result { typedef decltype(std::declval<A>() sym std::declval<B>()) type; }; };
VEXB_ARITH_TAG(plus, VEXB_OP_ADD, +) VEXB_ARITH_TAG(minus, VEXB_OP_SUB, -) VEXB_ARITH_TAG(multiplies, VEXB_OP_MUL, *)
VEXB_ARITH_TAG(divides, VEXB_OP_DIV, /) VEXB_ARITH_TAG(modulus, VEXB_OP_MOD, %)
VEXB_ARITH_TAG(bit_and, VEXB_OP_BAND, &) VEXB_ARITH_TAG(bit_or, VEXB_OP_BOR, |) VEXB_ARITH_TAG(bit_xor, VEXB_OP_BXOR, ^)
VEXB_ARITH_TAG(shift_left, VEXB_OP_SHL, <<) VEXB_ARITH_TAG(shift_right, VEXB_OP_SHR, >>)
#undef VEXB_ARITH_TAG
#define VEXB_CMP_TAG(name, code) \
    struct name { static const int opcode = code; static const bool compare = true; \
        template <class A, class B> struct result { typedef int type; }; };
VEXB_CMP_TAG(less, VEXB_OP_LT) VEXB_CMP_TAG(greater, VEXB_OP_GT) VEXB_CMP_TAG(less_equal, VEXB_OP_LE)
VEXB_CMP_TAG(greater_equal, VEXB_OP_GE) VEXB_CMP_TAG(equal_to, VEXB_OP_EQ) VEXB_CMP_TAG(not_equal_to, VEXB_OP_NE)
VEXB_CMP_TAG(logical_and, VEXB_OP_LAND) VEXB_CMP_TAG(logical_or, VEXB_OP_LOR)
#undef VEXB_CMP_TAG
} // namespace op

template <class Tag, class L, class R>
struct binary_node : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef typename detail::value_of<L>::type lhs_value;
    typedef typename detail::value_of<R>::type rhs_value;
    typedef typename std::decay<typename Tag::template result<lhs_value, rhs_value>::type>::type raw_value;
    typedef typename detail::promoted<raw_value>::type value_type;
    typedef typename std::common_type<lhs_value, rhs_value>::type operand_type;   // type the operands meet in

    static const size_t multi_size = detail::max_ncomp<L, R>::value;

    L l; R r;
    binary_node(L l, R r) : l(l), r(r) {}

    int lower(detail::ir_builder &b) const {
        const int C = Tag::compare ? dtype_of<typename detail::promoted<operand_type>::type>::value : dtype_of<value_type>::value;
        b.cvt(l.lower(b), C);
        b.cvt(r.lower(b), C);
        b.emit(Tag::opcode, C);
        return dtype_of<value_type>::value;
    }
    void props(detail::expr_props &p) const { l.props(p); r.props(p); }
};

namespace op {
struct negate { static const int opcode = VEXB_OP_NEG; };
struct logical_not { static const int opcode = VEXB_OP_LNOT; };
}

template <class Tag, class A>
struct unary_node : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef typename detail::value_of<A>::type arg_value;
    typedef typename std::conditional<std::is_same<Tag, op::logical_not>::value, int, arg_value>::type value_type;
    static const size_t multi_size = detail::ncomp<A>::value;
    A a;
    explicit unary_node(A a) : a(a) {}
    int lower(detail::ir_builder &b) const {
        const int t = a.lower(b);
        b.emit(Tag::opcode, t);
        return dtype_of<value_type>::value;
    }
    void props(detail::expr_props &p) const { a.props(p); }
};

/// cond ? a : b  (if_else, operations.hpp:1277-1301).
template <class C, class A, class B>
struct select_node : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef typename detail::promoted<typename std::common_type<typename detail::value_of<A>::type,
                                                                 typename detail::value_of<B>::type>::type>::type value_type;
    static const size_t multi_size = detail::max_ncomp<C, A, B>::value;
    C c; A a; B b_;
    select_node(C c, A a, B b) : c(c), a(a), b_(b) {}
    int lower(detail::ir_builder &b) const {
        const int V = dtype_of<value_type>::value;
        const int ct = c.lower(b);
        if (ct != VEXB_I32) {                                   // any arithmetic condition: (c != 0)
            int k = b.new_term();
            b.e.term[k].kind = VEXB_TERM_SCALAR; b.e.term[k].dtype = static_cast<uint8_t>(ct); b.e.term[k].v.u64 = 0;
            b.emit(VEXB_OP_TERM, ct, k);
            b.emit(VEXB_OP_NE, ct);
        }
        b.cvt(a.lower(b), V);
        b.cvt(b_.lower(b), V);
        b.emit(VEXB_OP_SELECT, V);
        return V;
    }
    void props(detail::expr_props &p) const { c.props(p); a.props(p); b_.props(p); }
};

template <class C, class A, class B>
const typename std::enable_if<detail::is_operand<C>::value && detail::is_operand<A>::value && detail::is_operand<B>::value &&
                        (is_vector_expr<C>::value || is_vector_expr<A>::value || is_vector_expr<B>::value),
    select_node<typename detail::operand<C>::type, typename detail::operand<A>::type, typename detail::operand<B>::type> >::type
if_else(const C &c, const A &a, const B &b) {
    return select_node<typename detail::operand<C>::type, typename detail::operand<A>::type, typename detail::operand<B>::type>(
            detail::operand<C>::wrap(c), detail::operand<A>::wrap(a), detail::operand<B>::wrap(b));
}

// ---- operators -------------------------------------------------------------------------------
#define VEXCL_BINARY_OPERATOR(sym, tag) \
    template <class L, class R> \
    const typename std::enable_if<detail::is_operand<L>::value && detail::is_operand<R>::value && \
                            (is_vector_expr<L>::value || is_vector_expr<R>::value), \
        binary_node<op::tag, typename detail::operand<L>::type, typename detail::operand<R>::type> >::type \
    operator sym(const L &l, const R &r) { \
        return binary_node<op::tag, typename detail::operand<L>::type, typename detail::operand<R>::type>( \
                detail::operand<L>::wrap(l), detail::operand<R>::wrap(r)); \
    }
VEXCL_BINARY_OPERATOR(+, plus) VEXCL_BINARY_OPERATOR(-, minus) VEXCL_BINARY_OPERATOR(*, multiplies)
VEXCL_BINARY_OPERATOR(/, divides) VEXCL_BINARY_OPERATOR(%, modulus)
VEXCL_BINARY_OPERATOR(&, bit_and) VEXCL_BINARY_OPERATOR(|, bit_or) VEXCL_BINARY_OPERATOR(^, bit_xor)
VEXCL_BINARY_OPERATOR(<<, shift_left) VEXCL_BINARY_OPERATOR(>>, shift_right)
VEXCL_BINARY_OPERATOR(<, less) VEXCL_BINARY_OPERATOR(>, greater) VEXCL_BINARY_OPERATOR(<=, less_equal)
VEXCL_BINARY_OPERATOR(>=, greater_equal) VEXCL_BINARY_OPERATOR(==, equal_to) VEXCL_BINARY_OPERATOR(!=, not_equal_to)
VEXCL_BINARY_OPERATOR(&&, logical_and) VEXCL_BINARY_OPERATOR(||, logical_or)
#undef VEXCL_BINARY_OPERATOR

template <class A>
const typename std::enable_if<is_vector_expr<A>::value, unary_node<op::negate, typename detail::operand<A>::type> >::type
operator-(const A &a) { return unary_node<op::negate, typename detail::operand<A>::type>(detail::operand<A>::wrap(a)); }

template <class A>
const typename std::enable_if<is_vector_expr<A>::value, unary_node<op::logical_not, typename detail::operand<A>::type> >::type
operator!(const A &a) { return unary_node<op::logical_not, typename detail::operand<A>::type>(detail::operand<A>::wrap(a)); }

template <class A>
typename std::enable_if<is_vector_expr<A>::value, typename detail::operand<A>::type>::type
operator+(const A &a) { return detail::operand<A>::wrap(a); }

// ---- additive operators (SpMat * vector; operations.hpp:425-447, :759-776) ---------------------
/// `M * x`, possibly scaled; M provides apply(x, y, alpha, append).
template <class M, class V>
struct additive_operator {
    const M &A; const V &x;
    typename V::value_type scale;
    additive_operator(const M &A, const V &x, typename V::value_type scale = 1) : A(A), x(x), scale(scale) {}
    void apply(V &y, typename V::value_type sign, bool append) const { A.apply(x, y, sign * scale, append); }
};

namespace detail {
/// The scalar of a direct product's vector element: T of std::array<T, B> and std::complex<T>.  A user value type has none;
/// double stands in for it, so that expression nodes around a misused product still form and stop at a static_assert.
template <class R, class = void> struct direct_scalar { typedef double type; };
template <class R> struct direct_scalar<R, decltype(void(std::declval<typename R::value_type>()))> { typedef typename R::value_type type; };
/// Can M::mul scale its product (alpha != 1)?  Not when M says `static const bool scales = false` (user value types).
template <class M, class = void> struct direct_scales : std::true_type {};
template <class M> struct direct_scales<M, typename std::enable_if<!M::scales>::type> : std::false_type {};
}

/// `M * x` that M writes straight into y with one call, M::mul(x, y, alpha, append): the product of a block, complex or
/// user-value sparse matrix (sparse/matrix.hpp).  vex::vector takes it as y = A*x, y += A*x and, unless M is of a user
/// value type, y -= A*x.  It has no kernel form, so any other expression that holds it stops at the static_assert below.
template <class M, class V>
struct direct_product : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef typename detail::direct_scalar<typename M::rhs_type>::type value_type;   // expression nodes around a misused product still form
    const M &A; const V &x;
    direct_product(const M &A, const V &x) : A(A), x(x) {}
    void props(detail::expr_props&) const { static_assert(sizeof(M) == 0, "a block, complex or user-value matrix product is only assigned: Y = A * X, Y += A * X or (not for user value types) Y -= A * X"); }
    int lower(detail::ir_builder&) const { return -1; }
};

namespace detail {
/// Does M offer `const vexb_spmat* inline_strip(unsigned device) const` (a strip usable as a VEXB_TERM_SPMV terminal)?
template <class M, class = void> struct has_inline_strip : std::false_type {};
template <class M> struct has_inline_strip<M, decltype(void(std::declval<const M&>().inline_strip(0u)))> : std::true_type {};

/// A sum of additive terms, each able to append itself to a vector of value type T -- and, when its operator can be
/// inlined (vex::SpMat strips without a halo), to lower itself as `scale * (row i of A*x)` into the consumer's kernel.
template <class T>
struct additive_terms {
    struct term {
        std::function<void(vex::vector<T>&, T, bool)> apply;       ///< y (=|+=) sign * scale * A * x
        std::function<bool(unsigned)> can_inline;                    ///< on device d
        std::function<const vexb_spmat*(unsigned)> sweep_strip;      ///< device d's sliced-ELL strip for a storage-order sweep, or NULL
        std::function<void(ir_builder&, T)> lower;                   ///< pushes sign * scale * (A*x)_i
        void operator()(vex::vector<T> &y, T sign, bool append) const { apply(y, sign, append); }
    };
    std::vector<term> terms;
    additive_terms() {}
    template <class M> additive_terms(const additive_operator<M, vex::vector<T>> &a) { terms.push_back(make(a)); }
    additive_terms scaled(T s) const {
        additive_terms r;
        for (auto &t : terms) {
            term u;
            u.apply = [t, s](vex::vector<T> &y, T sign, bool append) { t.apply(y, sign * s, append); };
            u.can_inline = t.can_inline;
            u.sweep_strip = t.sweep_strip;
            u.lower = [t, s](ir_builder &b, T sign) { t.lower(b, sign * s); };
            r.terms.push_back(u);
        }
        return r;
    }
    additive_terms& append(const additive_terms &o, T s = 1) {
        for (auto &t : o.scaled(s).terms) terms.push_back(t);
        return *this;
    }
    private:
        template <class M>
        static typename std::enable_if<has_inline_strip<M>::value, term>::type make(const additive_operator<M, vex::vector<T>> &a) {
            term t;
            t.apply = [a](vex::vector<T> &y, T sign, bool append) { a.apply(y, sign, append); };
            t.can_inline = [a](unsigned d) { return a.A.inline_strip(d) != nullptr; };
            t.sweep_strip = [a](unsigned d) { return a.A.sweep_strip(d); };
            t.lower = [a](ir_builder &b, T sign) {
                const int dt = dtype_of<T>::value;
                b.push_scalar(static_cast<T>(sign * a.scale));
                const vexb_spmat *s = a.A.inline_strip(b.part);
                b.push_spmv(s ? s : a.A.sweep_strip(b.part), a.x(b.part).raw(), dt);
                b.emit(VEXB_OP_MUL, dt);
            };
            return t;
        }
        template <class M>
        static typename std::enable_if<!has_inline_strip<M>::value, term>::type make(const additive_operator<M, vex::vector<T>> &a) {
            term t;
            t.apply = [a](vex::vector<T> &y, T sign, bool append) { a.apply(y, sign, append); };
            t.can_inline = [](unsigned) { return false; };
            t.sweep_strip = [](unsigned) { return static_cast<const vexb_spmat*>(nullptr); };
            t.lower = [](ir_builder&, T) {};
            return t;
        }
};

/// `expr + s1*(A1*x1) + s2*(A2*x2) ...` as ONE expression: the vector part followed by the inlined products, added in the
/// order the unfused path applies them (same bits), evaluated by a single generated kernel.
template <class E, class T>
struct fused_mixed : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef T value_type;
    const E &expr; const additive_terms<T> &terms; T sign;
    fused_mixed(const E &e, const additive_terms<T> &t, T sign) : expr(e), terms(t), sign(sign) {}
    void props(expr_props &p) const {
        // the terms' sliced-ELL strip (vector::inlinable admits one) is claimed before the vector part asks
        for (auto &t : terms.terms) if (!t.can_inline(0) && !p.swept) p.swept = t.sweep_strip(0);
        expr.props(p);
    }
    int lower(ir_builder &b) const {
        const int dt = dtype_of<T>::value;
        const int et = expr.lower(b);
        b.cvt(et, dt);
        for (auto &t : terms.terms) { t.lower(b, sign); b.emit(VEXB_OP_ADD, dt); }
        return dt;
    }
};
} // namespace detail

/// vector expression +/- additive terms (the split of vector.hpp:758-763).
template <class Expr, class T>
struct mixed_expression {
    Expr expr;
    detail::additive_terms<T> terms;
    mixed_expression(Expr e, detail::additive_terms<T> t) : expr(e), terms(t) {}
};

// scaling: s * (A*x), (A*x) * s, (A*x) / s, -(A*x)
template <class M, class V, class S>
typename std::enable_if<std::is_arithmetic<S>::value, additive_operator<M, V> >::type
operator*(S s, const additive_operator<M, V> &a) { return additive_operator<M, V>(a.A, a.x, a.scale * static_cast<typename V::value_type>(s)); }
template <class M, class V, class S>
typename std::enable_if<std::is_arithmetic<S>::value, additive_operator<M, V> >::type
operator*(const additive_operator<M, V> &a, S s) { return additive_operator<M, V>(a.A, a.x, a.scale * static_cast<typename V::value_type>(s)); }
template <class M, class V, class S>
typename std::enable_if<std::is_arithmetic<S>::value, additive_operator<M, V> >::type
operator/(const additive_operator<M, V> &a, S s) { return additive_operator<M, V>(a.A, a.x, a.scale / static_cast<typename V::value_type>(s)); }
template <class M, class V>
additive_operator<M, V> operator-(const additive_operator<M, V> &a) { return additive_operator<M, V>(a.A, a.x, -a.scale); }

// sums of additive terms
template <class M1, class M2, class T>
detail::additive_terms<T> operator+(const additive_operator<M1, vector<T>> &a, const additive_operator<M2, vector<T>> &b) {
    return detail::additive_terms<T>(a).append(detail::additive_terms<T>(b));
}
template <class M1, class M2, class T>
detail::additive_terms<T> operator-(const additive_operator<M1, vector<T>> &a, const additive_operator<M2, vector<T>> &b) {
    return detail::additive_terms<T>(a).append(detail::additive_terms<T>(b), T(-1));
}
template <class M, class T>
detail::additive_terms<T> operator+(detail::additive_terms<T> a, const additive_operator<M, vector<T>> &b) { return a.append(detail::additive_terms<T>(b)); }
template <class M, class T>
detail::additive_terms<T> operator-(detail::additive_terms<T> a, const additive_operator<M, vector<T>> &b) { return a.append(detail::additive_terms<T>(b), T(-1)); }

// vector expression +/- additive
template <class E, class M, class T>
typename std::enable_if<detail::is_operand<E>::value, mixed_expression<typename detail::operand<E>::type, T> >::type
operator+(const E &e, const additive_operator<M, vector<T>> &a) {
    return mixed_expression<typename detail::operand<E>::type, T>(detail::operand<E>::wrap(e), detail::additive_terms<T>(a));
}
template <class E, class M, class T>
typename std::enable_if<detail::is_operand<E>::value, mixed_expression<typename detail::operand<E>::type, T> >::type
operator-(const E &e, const additive_operator<M, vector<T>> &a) {
    return mixed_expression<typename detail::operand<E>::type, T>(detail::operand<E>::wrap(e), detail::additive_terms<T>(a).scaled(T(-1)));
}
template <class E, class M, class T>
typename std::enable_if<detail::is_operand<E>::value, mixed_expression<typename detail::operand<E>::type, T> >::type
operator+(const additive_operator<M, vector<T>> &a, const E &e) { return e + a; }
template <class E, class M, class T>
typename std::enable_if<is_vector_expr<E>::value,
    mixed_expression<unary_node<op::negate, typename detail::operand<E>::type>, T> >::type
operator-(const additive_operator<M, vector<T>> &a, const E &e) {
    return mixed_expression<unary_node<op::negate, typename detail::operand<E>::type>, T>(-e, detail::additive_terms<T>(a));
}
// mixed +/- additive, mixed +/- vector expression
template <class E, class M, class T>
mixed_expression<E, T> operator+(mixed_expression<E, T> m, const additive_operator<M, vector<T>> &a) { m.terms.append(detail::additive_terms<T>(a)); return m; }
template <class E, class M, class T>
mixed_expression<E, T> operator-(mixed_expression<E, T> m, const additive_operator<M, vector<T>> &a) { m.terms.append(detail::additive_terms<T>(a), T(-1)); return m; }
template <class E, class T, class X>
typename std::enable_if<detail::is_operand<X>::value,
    mixed_expression<binary_node<op::plus, E, typename detail::operand<X>::type>, T> >::type
operator+(const mixed_expression<E, T> &m, const X &x) {
    typedef binary_node<op::plus, E, typename detail::operand<X>::type> N;
    return mixed_expression<N, T>(N(m.expr, detail::operand<X>::wrap(x)), m.terms);
}
template <class E, class T, class X>
typename std::enable_if<detail::is_operand<X>::value,
    mixed_expression<binary_node<op::minus, E, typename detail::operand<X>::type>, T> >::type
operator-(const mixed_expression<E, T> &m, const X &x) {
    typedef binary_node<op::minus, E, typename detail::operand<X>::type> N;
    return mixed_expression<N, T>(N(m.expr, detail::operand<X>::wrap(x)), m.terms);
}

namespace detail {

/// Point the raw-pointer terminals of `e` that address `target` at a device copy of it (`copy`: made here unless it holds
/// one already; the caller keeps it until the launch is enqueued, and freeing waits for the device).  The back end refuses a pointer into the
/// target (VEXB_ERR_UNSUPPORTED): threads would read elements that others overwrite.  Through the copy, `x = p[(i + 1) %
/// n]` with p = raw_pointer(x) rotates x and every element reads the old values.  False when no terminal addresses it.
template <class T>
bool redirect_pointers(vexb_expr &e, const void *target, int dtype, size_t bytes, const backend::command_queue &q,
                       backend::device_vector<T> &copy) {
    bool hit = false;
    for (int k = 0; k < e.n_terms; ++k) hit = hit || (e.term[k].kind == VEXB_TERM_PTR && e.term[k].v.ptr == target);
    if (!hit) return false;
    precondition(bytes % sizeof(T) == 0, "raw_pointer: bad target size");
    if (!copy.raw()) {
        copy = backend::device_vector<T>(q, bytes / sizeof(T));
        if (bytes) VEXB_CHECKED(vexb_d2d(q.ordinal(), copy.raw(), target, bytes, q.raw()));
    }
    for (int k = 0; k < e.n_terms; ++k)
        if (e.term[k].kind == VEXB_TERM_PTR && e.term[k].v.ptr == target && e.term[k].dtype == dtype) e.term[k].v.ptr = copy.raw();
    return true;
}

/// lhs OP= expr on every device slice (replaces assign_expression, operations.hpp:1818-1897).
template <class OP, class T, class Expr>
void assign_expression(vex::vector<T> &lhs, const Expr &expr, int comp = -1) {
    expr_props p;
    p.comp = comp;
    p.sweeps = comp < 0;
    if (lhs.nparts()) p.target = lhs(0).raw();
    p.see(lhs.queue_list(), lhs.partition(), lhs.size());
    expr.props(p);
    const std::vector<backend::command_queue> &queue = lhs.queue_list();
    for (unsigned d = 0; d < queue.size(); ++d) {
        ir_builder b(d, comp);
        expr.lower(b);
        int st = vexb_eval(queue[d].ordinal(), queue[d].raw(), lhs(d).raw(), dtype_of<T>::value, OP::op,
                           &b.e, lhs.part_size(d), lhs.part_start(d));
        backend::device_vector<T> copy;
        if (st == VEXB_ERR_UNSUPPORTED && redirect_pointers(b.e, lhs(d).raw(), dtype_of<T>::value, lhs.part_size(d) * sizeof(T), queue[d], copy))
            st = vexb_eval(queue[d].ordinal(), queue[d].raw(), lhs(d).raw(), dtype_of<T>::value, OP::op,
                           &b.e, lhs.part_size(d), lhs.part_start(d));
        VEXB_CHECKED(st);
    }
}

} // namespace detail
} // namespace vex
#endif
