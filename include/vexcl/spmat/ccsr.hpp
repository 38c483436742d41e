#ifndef VEXCL_SPMAT_CCSR_HPP
#define VEXCL_SPMAT_CCSR_HPP
/*
 * vex::SpMatCCSR<val_t, col_t, idx_t> (vexcl/spmat/ccsr.hpp:54-86): "compressed CSR".  Only the unique rows of the
 * matrix are stored, column positions are relative to the diagonal, and idx[i] names the unique row of matrix row i.
 * Single device, like the reference.  The product is libvexb200's ccsr_kernel (csrc/ccsr.cu); `A * x` takes part in
 * `y = A * x`, `y += A * x`, `y = expr + A * x`, ... through the same additive-operator rules as vex::SpMat, for
 * vectors and multivectors.
 * Anywhere else an operand goes -- `sin(A * x)`, `x * (A * x)`, `y *= A * x`, a VEX_FUNCTION argument, if_else,
 * `sum(x * (A * x))`, vex::make_inline(A * x) -- the product of a vector is the reference's ccsr_product terminal
 * (ccsr.hpp:88-270): a VEXB_TERM_CCSR whose row loop is generated into the consumer's kernel, so the product never goes
 * to memory.  Same bits as `t = A * x` followed by the expression with t.
 */
#include <memory>
#include "../vector.hpp"
#include "../multivector.hpp"

namespace vex {

template <typename val_t, typename col_t = ptrdiff_t, typename idx_t = size_t>
struct SpMatCCSR {
    static_assert(std::is_signed<col_t>::value, "Column type for CCSR format has to be signed.");
    static_assert(sizeof(col_t) == 4 || sizeof(col_t) == 8, "column type must be 32 or 64 bit");
    static_assert(sizeof(idx_t) == 4 || sizeof(idx_t) == 8, "index type must be 32 or 64 bit");
    typedef val_t value_type;

    /// n rows, m unique rows; idx: n entries, row: m+1 offsets into col/val (ccsr.hpp:70-78).
    SpMatCCSR(const backend::command_queue &queue, size_t n, size_t m,
              const idx_t *idx, const idx_t *row, const col_t *col, const val_t *val)
        : queue(queue), n(n)
    {
        vexb_ccsr *h = nullptr;
        VEXB_CHECKED(vexb_ccsr_create(queue.ordinal(), queue.raw(), n, m, idx, sizeof(idx_t), row, sizeof(idx_t),
                                      col, sizeof(col_t), val, dtype_of<val_t>::value, &h));
        mtx.reset(h, [](vexb_ccsr *p) { vexb_ccsr_destroy(p); });
        idx_bytes = info().idx_bytes;
    }

    void apply(const vex::vector<val_t> &x, vex::vector<val_t> &y, val_t alpha = 1, bool append = false) const {
        precondition(x.nparts() == 1 && y.nparts() == 1, "SpMatCCSR works with single-device vectors only");
        precondition(x.size() == n && y.size() == n, "SpMatCCSR::apply: vector sizes do not match the matrix");
        precondition(x.queue_list()[0].ordinal() == queue.ordinal(), "SpMatCCSR and its vectors must live on the same device");
        VEXB_CHECKED(vexb_ccsr_spmv(queue.ordinal(), y.queue_list()[0].raw(), mtx.get(), x(0).raw(), y(0).raw(),
                                    static_cast<double>(alpha), append));
    }
    size_t rows() const { return n; }
    size_t cols() const { return n; }
    vexb_ccsr_info info() const { vexb_ccsr_info i; VEXB_CHECKED(vexb_ccsr_get_info(mtx.get(), &i)); return i; }

    backend::command_queue queue;
    size_t n;
    std::shared_ptr<vexb_ccsr> mtx;
    int idx_bytes = 0;              ///< width of idx on the device (1, 2 or 4), part of a terminal's kernel shape
};

template <typename val_t, typename col_t, typename idx_t>
additive_operator<SpMatCCSR<val_t, col_t, idx_t>, vector<val_t>>
operator*(const SpMatCCSR<val_t, col_t, idx_t> &A, const vector<val_t> &x) {
    return additive_operator<SpMatCCSR<val_t, col_t, idx_t>, vector<val_t>>(A, x);
}
/// `A * x` standing where an operand goes (VEXB_TERM_CCSR), scaled inside the expression when it carries a scale.  One
/// slice only, as in the reference.  When x is the assignment's target, the product is evaluated into a temporary first:
/// threads writing x[i] while others read x[i + col[j]] would race.
template <typename val_t, typename col_t, typename idx_t>
struct ccsr_product : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef val_t value_type;
    const SpMatCCSR<val_t, col_t, idx_t> &A; const vector<val_t> &x; val_t scale;
    mutable std::shared_ptr<vector<val_t>> tmp;
    mutable bool aliased = false;
    ccsr_product(const SpMatCCSR<val_t, col_t, idx_t> &A, const vector<val_t> &x, val_t scale) : A(A), x(x), scale(scale) {}
    void props(detail::expr_props &p) const {
        precondition(x.nparts() == 1, "SpMatCCSR works with single-device vectors only");
        precondition(x.size() == A.n, "SpMatCCSR product: vector size does not match the matrix");
        precondition(x.queue_list()[0].ordinal() == A.queue.ordinal(), "SpMatCCSR and its vectors must live on the same device");
        aliased = p.target == x(0).raw();
        if (aliased) {
            if (!tmp) tmp = std::make_shared<vector<val_t>>(x.queue_list(), A.n);
            A.apply(x, *tmp, 1, false);
        }
        p.see(x.queue_list(), x.partition(), A.n);
    }
    int lower(detail::ir_builder &b) const {
        const int dt = dtype_of<val_t>::value;
        if (scale != val_t(1)) b.push_scalar(scale);
        if (aliased) tmp->lower(b);
        else b.push_ccsr(A.mtx.get(), A.idx_bytes, x(b.part).raw(), dt);
        if (scale != val_t(1)) b.emit(VEXB_OP_MUL, dt);
        return dt;
    }
};

template <typename val_t, typename col_t, typename idx_t>
struct is_vector_expr_type<additive_operator<SpMatCCSR<val_t, col_t, idx_t>, vector<val_t>>> : std::true_type {};
namespace detail {
template <typename val_t, typename col_t, typename idx_t>
struct operand<additive_operator<SpMatCCSR<val_t, col_t, idx_t>, vector<val_t>>, void> {
    typedef ccsr_product<val_t, col_t, idx_t> type;
    static type wrap(const additive_operator<SpMatCCSR<val_t, col_t, idx_t>, vector<val_t>> &a) { return type(a.A, a.x, a.scale); }
};
}

/// vex::make_inline(A * x) (spmat/ccsr.hpp:88-270 is the reference's terminal): the unscaled product as a terminal.
template <typename val_t, typename col_t, typename idx_t>
const ccsr_product<val_t, col_t, idx_t>
make_inline(const additive_operator<SpMatCCSR<val_t, col_t, idx_t>, vector<val_t>> &base) {
    precondition(base.scale == 1, "make_inline: scale the inlined product inside the expression instead");
    return ccsr_product<val_t, col_t, idx_t>(base.A, base.x, 1);
}

template <typename val_t, typename col_t, typename idx_t, size_t N>
additive_operator<SpMatCCSR<val_t, col_t, idx_t>, multivector<val_t, N>>
operator*(const SpMatCCSR<val_t, col_t, idx_t> &A, const multivector<val_t, N> &x) {
    return additive_operator<SpMatCCSR<val_t, col_t, idx_t>, multivector<val_t, N>>(A, x);
}

} // namespace vex
#endif
