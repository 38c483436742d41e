#ifndef VEXCL_SPARSE_DISTRIBUTED_HPP
#define VEXCL_SPARSE_DISTRIBUTED_HPP
/*
 * vex::sparse::distributed<Matrix> (vexcl/sparse/distributed.hpp:23-427): the multi-device wrapper of
 * the sparse:: classes.  Same partition, local/remote split and ghost exchange tables as vex::SpMat
 * (the two reference classes build them twice, spmat.hpp:291-378 and distributed.hpp:51-215); here both
 * sit on vexb_dspmat, so the halo goes over NCCL / NVLink instead of through host memory
 * (reference: blocking read per device, host shuffle, write; distributed.hpp:346-426).
 */
#include "../spmat.hpp"
#include "matrix.hpp"

namespace vex {
namespace sparse {

namespace detail_sparse {
template <class M> struct format_of { static const int value = VEXB_FMT_AUTO; };
template <int F, class V, class C, class P> struct format_of<single_device_matrix<F, V, C, P>> { static const int value = F; };
}

template <class Matrix>
class distributed {
    public:
        typedef typename Matrix::value_type value_type;
        typedef typename Matrix::col_type col_type;
        typedef typename Matrix::ptr_type ptr_type;
        static_assert(!detail_sparse::is_block_value<value_type>::value,
                      "vex::sparse::distributed does not take block values: use vex::sparse::matrix on a single device");
        static_assert(!detail_sparse::is_complex_value<value_type>::value,
                      "vex::sparse::distributed does not take complex values: use vex::sparse::matrix on a single device");
        static_assert(!detail_sparse::is_user_value<value_type>::value,
                      "vex::sparse::distributed does not take user value types: use vex::sparse::matrix on a single device");

        template <class PtrRange, class ColRange, class ValRange>
        distributed(const std::vector<backend::command_queue> &q, size_t nrows, size_t ncols,
                    const PtrRange &ptr, const ColRange &col, const ValRange &val, bool /*fast_setup*/ = true)
            : q(q), A(q, nrows, ncols, detail_sparse::range_data(ptr), detail_sparse::range_data(col), detail_sparse::range_data(val),
                      detail_sparse::format_of<Matrix>::value)
        {}

        size_t rows() const { return A.rows(); }
        size_t cols() const { return A.cols(); }
        size_t nonzeros() const { return A.nonzeros(); }
        const std::vector<backend::command_queue>& queue_list() const { return q; }

        void mul(const vex::vector<value_type> &x, vex::vector<value_type> &y, value_type alpha = 1, bool append = false) const {
            A.apply(x, y, alpha, append);
        }

        /// Device d's strip when a generated kernel can walk its rows (no halo on that device), else NULL.
        const vexb_spmat* inline_strip(unsigned d) const { return A.inline_strip(d); }
        const vexb_spmat* sweep_strip(unsigned d) const { return A.sweep_strip(d); }

        template <class Expr>
        friend typename std::enable_if<is_vector_expr<Expr>::value, matrix_vector_product<distributed, Expr> >::type
        operator*(const distributed &A, const Expr &x) { return matrix_vector_product<distributed, Expr>(A, x); }
    private:
        std::vector<backend::command_queue> q;
        vex::SpMat<value_type, col_type, ptr_type> A;
};

} // namespace sparse
} // namespace vex
#endif
