#ifndef VEXCL_SPARSE_PRODUCT_HPP
#define VEXCL_SPARSE_PRODUCT_HPP
/*
 * `A * x` for the vex::sparse classes as a *terminal* of vector expressions
 * (vexcl/sparse/product.hpp:45-130): usable anywhere a vector is, e.g.
 *     y = x + A * x;      s = sum(f - A * x);      y = A * (2 * x + z);
 * As in the reference, the row loop is emitted into the consumer's kernel: the product is a
 * VEXB_TERM_SPMV terminal of the IR, and the expression runs as one NVRTC-generated kernel
 * specialised to the strip's format (CSR, or hybrid ELL with its width unrolled).  `x` may itself
 * be an expression; it is then evaluated into a temporary first (a gather needs all of x).
 * A reduction such as `sum(f - A*x)` is one generated kernel too: the row loop feeds the fold directly.
 * In an assignment a sliced-ELL strip is a terminal too: the kernel then sweeps in the strip's storage order (one such
 * matrix per expression; a reduction of it keeps its temporary).  Row-pattern strips go through a temporary y instead.
 */
#include <memory>
#include "../operations.hpp"
#include "../vector.hpp"

namespace vex {
namespace sparse {

template <class Matrix, class Vector>
struct matrix_vector_product : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef typename Matrix::value_type value_type;

    const Matrix &A;
    typename detail::operand<Vector>::type x;
    mutable std::shared_ptr<vex::vector<value_type>> y, xt;

    matrix_vector_product(const Matrix &A, const Vector &x) : A(A), x(detail::operand<Vector>::wrap(x)) {}

    // Evaluated once per launch of the enclosing expression, before lowering.
    void props(detail::expr_props &p) const {
        xv = &materialize(x);
        fused = std::is_floating_point<value_type>::value;
        for (unsigned d = 0; fused && d < A.queue_list().size(); ++d) fused = A.inline_strip(d) != nullptr;
        if (!fused && std::is_floating_point<value_type>::value) fused = p.claim_sweep(A);     // assignments: a sliced-ELL strip, swept in storage order
        if (fused) { p.see(A.queue_list(), vex::partition(A.rows(), A.queue_list()), A.rows()); return; }   // row loop goes into the consumer's kernel
        if (!y || y->size() != A.rows()) y = std::make_shared<vex::vector<value_type>>(A.queue_list(), A.rows());
        A.mul(*xv, *y);
        y->props(p);
    }
    int lower(detail::ir_builder &b) const {
        if (!fused) return y->lower(b);
        const vexb_spmat *s = A.inline_strip(b.part);
        b.push_spmv(s ? s : A.sweep_strip(b.part), (*xv)(b.part).raw(), dtype_of<value_type>::value);
        return dtype_of<value_type>::value;
    }
    mutable bool fused = false;
    mutable const vex::vector<value_type> *xv = nullptr;
    private:
        const vex::vector<value_type>& materialize(const vex::vector<value_type> &v) const { return v; }
        template <class E>
        const vex::vector<value_type>& materialize(const E &e) const {
            if (!xt || xt->size() != A.cols()) xt = std::make_shared<vex::vector<value_type>>(A.queue_list(), A.cols());
            *xt = e;
            return *xt;
        }
};

} // namespace sparse
} // namespace vex
#endif
