#ifndef VEXCL_VECTOR_POINTER_HPP
#define VEXCL_VECTOR_POINTER_HPP
/*
 * vex::raw_pointer(x) (vexcl/vector_pointer.hpp): the device address of element 0 of a one-part vector, so that an
 * expression can read any element, not only element i:
 *     auto p = vex::raw_pointer(x);
 *     y = 2 * p[i] - p[left] - p[right];          // neighbours with boundary formulas
 *     y = p[idx];                                  // a gather through an index vector
 *     y = *(p + i) + (p + i)[-1];                  // pointer arithmetic, as in C
 *     y = nbody(n, vex::element_index(), p);       // VEX_FUNCTION(double, nbody, (size_t, n)(size_t, j)(double*, x), ...)
 *
 * p[e], *(p + e), (p + a)[b], a + p, p - a and *p lower to one VEXB_OP_LOAD (include/vexb200.h): every offset is
 * widened to 64 bits on its own (signed types sign-extended, unsigned zero-extended), then added, as C adds to a
 * pointer.  A read outside the vector gives 0: both branches of an if_else are evaluated, so
 * `if_else(i > 0, p[i - 1], 0)` must not touch element -1.  Offsets are integral expressions or scalars.  A user
 * function takes the pointer itself for a parameter declared `T*` (or `const T*`); the pointer then goes to the
 * function with no arithmetic on it.  Any other use of a pointer -- `p * 2`, `p + 1.5`, `p - q`, `-p` -- stops at a
 * static_assert.
 *
 * A pointer contributes its queue list but no size (the reference's expression_properties), so an expression of
 * pointers alone takes its size from the target.  Every vector of an expression that holds a pointer must have one
 * part, on the pointer's device; otherwise the assignment throws before anything is launched.  When the pointer
 * addresses the assignment's target, the expression reads a device copy of it instead: `x = p[(i + 1) % n]` rotates x
 * and every element reads the old values (the reference races there).
 */
#include "vector.hpp"

namespace vex {

namespace detail {

/// The offset of a pointer with no arithmetic on it.
struct no_offset {
    int lower(ir_builder&) const { return -1; }
    void props(expr_props&) const {}
};

/// prev + e (Neg: prev - e) in 64-bit arithmetic, e widened on its own.
template <class Prev, class E, bool Neg>
struct offset_sum {
    Prev prev; E e;
    offset_sum(Prev p, E e) : prev(p), e(e) {}
    int lower(ir_builder &b) const {
        const bool first = prev.lower(b) < 0;
        b.cvt(e.lower(b), VEXB_I64);
        if (!first) b.emit(Neg ? VEXB_OP_SUB : VEXB_OP_ADD, VEXB_I64);
        else if (Neg) b.emit(VEXB_OP_NEG, VEXB_I64);
        return VEXB_I64;
    }
    void props(expr_props &p) const { prev.props(p); e.props(p); }
};

/// Is E an integral expression or scalar (what may be added to a pointer)?
template <class E, class = void> struct integral_offset : std::false_type {};
template <class E> struct integral_offset<E, typename std::enable_if<is_operand<E>::value>::type>
    : std::is_integral<typename value_of<typename operand<E>::type>::type> {};

/// The operand an offset is held as; a scalar stands in for a refused one, so that only the static_assert speaks.
template <class E, bool Ok = integral_offset<E>::value> struct offset_operand {
    typedef typename operand<E>::type type;
    static type wrap(const E &e) { return operand<E>::wrap(e); }
};
template <class E> struct offset_operand<E, false> {
    typedef scalar_term<long long> type;
    static type wrap(const E&) { return type(0); }
};

template <class X> struct always_false : std::false_type {};

} // namespace detail

/// One element read through a pointer: *(p + offset).
template <class T, class Off>
struct pointer_load : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef T value_type;
    const vector<T> &v; Off off;
    pointer_load(const vector<T> &v, Off off) : v(v), off(off) {}
    int lower(detail::ir_builder &b) const {
        if (off.lower(b) < 0) b.push_scalar(0LL);                 // *p: element 0
        const int dt = dtype_of<T>::value;
        b.emit(VEXB_OP_LOAD, dt, b.ptr_term(v(0).raw(), dt, v.size()));
        return dt;
    }
    void props(detail::expr_props &p) const { p.see_pointer(v.queue_list()); off.props(p); }
};

/// A pointer into a one-part vector, with the integral offsets added to it so far.
template <class T, class Off = detail::no_offset>
struct pointer_expr {
    typedef T value_type;
    typedef Off offset_type;
    const vector<T> &v; Off off;
    explicit pointer_expr(const vector<T> &v, Off off = Off()) : v(v), off(off) {}

    /// p[e]: the element e places from where p points.
    template <class E>
    pointer_load<T, detail::offset_sum<Off, typename detail::offset_operand<E>::type, false>> operator[](const E &e) const {
        static_assert(detail::integral_offset<E>::value, "a raw_pointer is indexed by an integral expression or scalar");
        typedef detail::offset_sum<Off, typename detail::offset_operand<E>::type, false> O;
        return pointer_load<T, O>(v, O(off, detail::offset_operand<E>::wrap(e)));
    }
    /// *p: the element p points to.
    pointer_load<T, Off> operator*() const { return pointer_load<T, Off>(v, off); }

    // The pointer itself, as the argument of a user function's `T*` parameter (VEXB_OP_TERM of a VEXB_TERM_PTR).
    int lower(detail::ir_builder &b) const {
        static_assert(std::is_same<Off, detail::no_offset>::value,
                      "a user function takes a raw_pointer without arithmetic: pass the pointer and the offset separately");
        const int dt = dtype_of<T>::value;
        b.emit(VEXB_OP_TERM, VEXB_PTR(dt), b.ptr_term(v(0).raw(), dt, v.size()));
        return VEXB_PTR(dt);
    }
    void props(detail::expr_props &p) const { p.see_pointer(v.queue_list()); off.props(p); }
};

/// The terminal of the reference's spelling: a pointer with no arithmetic on it.
template <class T> using vector_pointer = pointer_expr<T, detail::no_offset>;

/// Cast vex::vector to a raw pointer; refused, like the reference, for vectors of more than one part.
template <typename T>
inline vector_pointer<T> raw_pointer(const vector<T> &v) {
    precondition(v.nparts() == 1, "raw_pointer is not supported for multi-device contexts");
    return vector_pointer<T>(v);
}

namespace detail {
/// A pointer is held by value where a user function's argument goes (call_node, function.hpp).
template <class T, class Off> struct operand<pointer_expr<T, Off>, void> {
    typedef pointer_expr<T, Off> type;
    static type wrap(const type &p) { return p; }
};
}

// ---- pointer arithmetic: p + e, e + p, p - e -------------------------------------------------------------------
template <class T, class Off, class E>
pointer_expr<T, detail::offset_sum<Off, typename detail::offset_operand<E>::type, false>>
operator+(const pointer_expr<T, Off> &p, const E &e) {
    static_assert(detail::integral_offset<E>::value, "pointer arithmetic takes an integral expression or scalar");
    typedef detail::offset_sum<Off, typename detail::offset_operand<E>::type, false> O;
    return pointer_expr<T, O>(p.v, O(p.off, detail::offset_operand<E>::wrap(e)));
}
template <class E, class T, class Off>
pointer_expr<T, detail::offset_sum<Off, typename detail::offset_operand<E>::type, false>>
operator+(const E &e, const pointer_expr<T, Off> &p) {
    static_assert(detail::integral_offset<E>::value, "pointer arithmetic takes an integral expression or scalar");
    return p + e;
}
template <class T, class Off, class E>
pointer_expr<T, detail::offset_sum<Off, typename detail::offset_operand<E>::type, true>>
operator-(const pointer_expr<T, Off> &p, const E &e) {
    static_assert(detail::integral_offset<E>::value, "pointer arithmetic takes an integral expression or scalar");
    typedef detail::offset_sum<Off, typename detail::offset_operand<E>::type, true> O;
    return pointer_expr<T, O>(p.v, O(p.off, detail::offset_operand<E>::wrap(e)));
}
template <class T, class O1, class U, class O2>
void operator+(const pointer_expr<T, O1>&, const pointer_expr<U, O2>&) {
    static_assert(detail::always_false<T>::value, "two raw pointers are not added");
}
template <class T, class O1, class U, class O2>
void operator-(const pointer_expr<T, O1>&, const pointer_expr<U, O2>&) {
    static_assert(detail::always_false<T>::value, "the difference of two raw pointers is not an expression");
}
template <class E, class T, class Off>
void operator-(const E&, const pointer_expr<T, Off>&) {
    static_assert(detail::always_false<T>::value, "a raw_pointer is not subtracted from a value");
}

// ---- every other operator on a pointer is refused ----------------------------------------------------------------
#define VEXCL_POINTER_REFUSED(sym) \
    template <class T, class Off, class X> void operator sym(const pointer_expr<T, Off>&, const X&) { \
        static_assert(detail::always_false<T>::value, "a raw_pointer is only indexed, dereferenced, offset by an integer " \
                      "or passed to a user function: read an element, p[i] or *(p + i), to compute with it"); } \
    template <class X, class T, class Off> void operator sym(const X&, const pointer_expr<T, Off>&) { \
        static_assert(detail::always_false<T>::value, "a raw_pointer is only indexed, dereferenced, offset by an integer " \
                      "or passed to a user function: read an element, p[i] or *(p + i), to compute with it"); } \
    template <class T, class O1, class U, class O2> void operator sym(const pointer_expr<T, O1>&, const pointer_expr<U, O2>&) { \
        static_assert(detail::always_false<T>::value, "a raw_pointer is only indexed, dereferenced, offset by an integer " \
                      "or passed to a user function: read an element, p[i] or *(p + i), to compute with it"); }
VEXCL_POINTER_REFUSED(*) VEXCL_POINTER_REFUSED(/) VEXCL_POINTER_REFUSED(%)
VEXCL_POINTER_REFUSED(&) VEXCL_POINTER_REFUSED(|) VEXCL_POINTER_REFUSED(^) VEXCL_POINTER_REFUSED(<<) VEXCL_POINTER_REFUSED(>>)
VEXCL_POINTER_REFUSED(<) VEXCL_POINTER_REFUSED(>) VEXCL_POINTER_REFUSED(<=) VEXCL_POINTER_REFUSED(>=)
VEXCL_POINTER_REFUSED(==) VEXCL_POINTER_REFUSED(!=) VEXCL_POINTER_REFUSED(&&) VEXCL_POINTER_REFUSED(||)
#undef VEXCL_POINTER_REFUSED
template <class T, class Off> void operator-(const pointer_expr<T, Off>&) {
    static_assert(detail::always_false<T>::value, "a raw_pointer is not negated: read an element, p[i] or *(p + i), to compute with it");
}
template <class T, class Off> void operator!(const pointer_expr<T, Off>&) {
    static_assert(detail::always_false<T>::value, "a raw_pointer is not a condition: read an element, p[i] or *(p + i), to compute with it");
}

} // namespace vex
#endif
