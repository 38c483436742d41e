#ifndef VEXCL_TEMPORARY_HPP
#define VEXCL_TEMPORARY_HPP
/*
 * vex::make_temp<Tag>(expr) and vex::make_temp<Tag, T>(expr) (vexcl/temporary.hpp): a subexpression stored in a
 * per-element local variable, evaluated once per element before the expression that uses it, and read by every use.
 *     auto t1 = vex::make_temp<1>(sin(x));
 *     auto t2 = vex::make_temp<2>(cos(x));
 *     y = (t1 - t2) * (t1 + t2);
 * The node lowers to VEXB_OP_TDEF / VEXB_OP_TREF (include/vexb200.h): each definition goes, in post-order, ahead of the
 * expression, so a temporary may use others (nested temporaries).  The value is converted to T, the expression's type
 * unless given, and the result has the bits of the expression with T(expr) written out at every use.
 *
 * One Tag is one temporary within an expression; the same Tag over a different expression is a vex::backend::error
 * (the reference keeps the first).  The expression may hold user functions, vex::make_inline(A * x), vex::sparse and
 * SpMatCCSR products; in a multi-expression each component lowers it on its own (make_temp<1>(tan(mv)) is one
 * temporary per component).  An additive vex::SpMat product needs vex::make_inline, as in the reference.
 */
#include <memory>
#include "operations.hpp"

namespace vex {

template <class T, size_t Tag, class Expr>
struct temporary : vector_expr_tag {
    VEXCL_NODE_COMMON
    typedef T value_type;
    static const size_t multi_size = detail::ncomp<Expr>::value;
    // Every copy of the node (one per use in an expression) shares one inner expression, so that what its props() sets
    // up -- the vector a product that cannot be inlined is evaluated into -- is the same for every use, and the uses
    // lower to one program.
    struct holder { Expr e; };
    std::shared_ptr<const holder> expr;
    explicit temporary(Expr e) : expr(std::make_shared<const holder>(holder{e})) {}
    int lower(detail::ir_builder &b) const {
        const int t = dtype_of<T>::value;
        const int rel = b.e.n_code - b.n_prefix, terms = b.e.n_terms;
        b.cvt(expr->e.lower(b), t);
        b.use_temp(Tag, rel, terms, t);
        return t;
    }
    void props(detail::expr_props &p) const { expr->e.props(p); }
};

namespace detail {
template <class Expr> struct temp_operand {
    static_assert(is_vector_expr<Expr>::value,
                  "vex::make_temp takes a vector expression: write an additive product as vex::make_inline(A * x)");
    typedef typename operand<Expr>::type type;
    typedef typename std::decay<type>::type::value_type value_type;
};
}

// Deduced return types: overload resolution never looks inside temp_operand, whose static_assert is for the call chosen.
/// The value of `expr` as a temporary of type T, one per element (make_temp<Tag, T>).
template <size_t Tag, class T, class Expr>
auto make_temp(const Expr &expr) {
    return temporary<T, Tag, typename detail::temp_operand<Expr>::type>(detail::operand<Expr>::wrap(expr));
}

/// The value of `expr` as a temporary of the expression's type, one per element.
template <size_t Tag, class Expr>
auto make_temp(const Expr &expr) {
    typedef detail::temp_operand<Expr> O;
    return temporary<typename O::value_type, Tag, typename O::type>(detail::operand<Expr>::wrap(expr));
}

} // namespace vex
#endif
