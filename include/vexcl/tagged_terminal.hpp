#ifndef VEXCL_TAGGED_TERMINAL_HPP
#define VEXCL_TAGGED_TERMINAL_HPP
// vex::tag<N>(x) (vexcl/tagged_terminal.hpp:50-74, :247-266).  In the reference a tag tells the
// kernel generator that two terminals are the same object so it emits one parameter.  The IR
// normaliser of this build already merges vector terminals that point at the same buffer, so a
// tagged terminal is simply an assignable alias of its vector, and a tagged scalar the scalar.
#include "vector.hpp"

namespace vex {

template <size_t Tag, class T>
struct tagged_terminal : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef T value_type;
    vector<T> &term;
    explicit tagged_terminal(vector<T> &v) : term(v) {}
    int lower(detail::ir_builder &b) const { return term.lower(b); }
    void props(detail::expr_props &p) const { term.props(p); }

#define VEXCL_TAGGED_ASSIGN(cop) \
    template <class Expr> const tagged_terminal& operator cop(const Expr &expr) const { term cop expr; return *this; }
    VEXCL_TAGGED_ASSIGN(=) VEXCL_TAGGED_ASSIGN(+=) VEXCL_TAGGED_ASSIGN(-=) VEXCL_TAGGED_ASSIGN(*=) VEXCL_TAGGED_ASSIGN(/=)
    VEXCL_TAGGED_ASSIGN(%=) VEXCL_TAGGED_ASSIGN(&=) VEXCL_TAGGED_ASSIGN(|=) VEXCL_TAGGED_ASSIGN(^=) VEXCL_TAGGED_ASSIGN(<<=) VEXCL_TAGGED_ASSIGN(>>=)
#undef VEXCL_TAGGED_ASSIGN
    const tagged_terminal& operator=(const tagged_terminal &o) const { term = o.term; return *this; }
};

template <size_t Tag, class T>
tagged_terminal<Tag, T> tag(vector<T> &v) { return tagged_terminal<Tag, T>(v); }

/// vex::tag<N>(s) of a scalar (`auto N = vex::tag<1>(x.size())`): one kernel parameter in the reference, the by-value
/// terminal of the scalar here.
template <size_t Tag, class T>
typename std::enable_if<std::is_arithmetic<T>::value, scalar_term<T> >::type tag(const T &v) { return scalar_term<T>(v); }

} // namespace vex
#endif
