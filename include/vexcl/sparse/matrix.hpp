#ifndef VEXCL_SPARSE_MATRIX_HPP
#define VEXCL_SPARSE_MATRIX_HPP
/*
 * vex::sparse::csr / ell / matrix: single-device sparse matrices (vexcl/sparse/csr.hpp:47-196,
 * vexcl/sparse/ell.hpp:61-508, vexcl/sparse/matrix.hpp:10-150).  Default index types are int.
 * csr -> the TMA-staged CSR row-block kernel, ell -> hybrid ELL (the reference's layout and width
 * rule; its device-side csr2ell conversion, ell.hpp:348-506, happens on the host at upload here),
 * matrix -> libvexb200's own choice (the reference picks csr on CPUs and ell on GPUs).
 * With B x B block values (std::array<std::array<T, B>, B>) all three are the block format below, with
 * std::complex<T> values the complex format below, and with a user value type (vex::is_user_value, a product given
 * by its vex::sparse::spmv_ops_impl) the user-value format below.
 */
#include <array>
#include <complex>
#include <iterator>
#include <memory>
#include "../vector.hpp"
#include "product.hpp"
#include "spmv_ops.hpp"

namespace vex {
namespace sparse {

namespace detail_sparse {
template <class R> inline size_t range_size(const R &r) { return static_cast<size_t>(std::distance(std::begin(r), std::end(r))); }
template <class R> inline auto range_data(const R &r) -> decltype(&*std::begin(r)) { return range_size(r) ? &*std::begin(r) : nullptr; }
}

template <int Format, typename Val, typename Col, typename Ptr, typename Enable = void>
class single_device_matrix {
    public:
        typedef Val value_type; typedef Val val_type; typedef Col col_type; typedef Ptr ptr_type;

        template <class PtrRange, class ColRange, class ValRange>
        single_device_matrix(const std::vector<backend::command_queue> &q, size_t nrows, size_t ncols,
                             const PtrRange &ptr, const ColRange &col, const ValRange &val, bool /*fast_setup*/ = true)
            : q(q), n(nrows), m(ncols), nnz(detail_sparse::range_size(val))
        {
            precondition(q.size() == 1, "sparse matrices of this kind are only supported for single-device contexts");
            static_assert(sizeof(Col) == 4 || sizeof(Col) == 8, "column type must be 32 or 64 bit");
            static_assert(sizeof(Ptr) == 4 || sizeof(Ptr) == 8, "pointer type must be 32 or 64 bit");
            vexb_spmat *h = nullptr;
            VEXB_CHECKED(vexb_csr_create(q[0].ordinal(), q[0].raw(), nrows, ncols, detail_sparse::range_data(ptr), sizeof(Ptr),
                                         detail_sparse::range_data(col), sizeof(Col), detail_sparse::range_data(val),
                                         dtype_of<Val>::value, Format, &h));
            A.reset(h, [](vexb_spmat *p) { vexb_spmat_destroy(p); });
        }
        single_device_matrix() : n(0), m(0), nnz(0) {}

        size_t rows() const { return n; }
        size_t cols() const { return m; }
        size_t nonzeros() const { return nnz; }
        const std::vector<backend::command_queue>& queue_list() const { return q; }

        /// y = A * x
        void mul(const vex::vector<Val> &x, vex::vector<Val> &y, Val alpha = 1, bool append = false) const {
            precondition(x.size() == m && y.size() == n, "sparse product: vector sizes do not match the matrix");
            VEXB_CHECKED(vexb_spmv(q[0].ordinal(), q[0].raw(), A.get(), x(0).raw(), y(0).raw(), static_cast<double>(alpha), append));
        }

        /// The strip when a generated kernel can walk its rows (CSR / hybrid ELL with values of the vector type), else NULL.
        const vexb_spmat* inline_strip(unsigned = 0) const {
            vexb_spmat_info i;
            if (!A || vexb_spmat_get_info(A.get(), &i) != VEXB_OK) return nullptr;
            if (i.val_dtype == VEXB_F64 && i.val_bytes == 4) return nullptr;      // VEXB_FMT_VALUES_F32
            return (i.fmt == VEXB_FMT_CSR || i.fmt == VEXB_FMT_HELL) ? A.get() : nullptr;
        }

        /// The strip when an assignment can take it as a terminal by sweeping in its storage order (sliced ELL with values of
        /// the vector type, "spmv.sell_inline" on and "spmv.no_inline" off), else NULL.
        const vexb_spmat* sweep_strip(unsigned = 0) const {
            vexb_spmat_info i;
            long on = 1, off = 0;
            if (!A || vexb_spmat_get_info(A.get(), &i) != VEXB_OK) return nullptr;
            if (vexb_get_param("spmv.sell_inline", &on) != VEXB_OK) on = 1;       // never set: the default
            if (vexb_get_param("spmv.no_inline", &off) != VEXB_OK) off = 0;
            if (i.val_dtype == VEXB_F64 && i.val_bytes == 4) return nullptr;      // VEXB_FMT_VALUES_F32
            return (i.fmt == VEXB_FMT_SELL && on && !off) ? A.get() : nullptr;
        }

        template <class Expr>
        friend typename std::enable_if<is_vector_expr<Expr>::value, matrix_vector_product<single_device_matrix, Expr> >::type
        operator*(const single_device_matrix &A, const Expr &x) { return matrix_vector_product<single_device_matrix, Expr>(A, x); }
    private:
        std::vector<backend::command_queue> q;
        size_t n, m, nnz;
        std::shared_ptr<vexb_spmat> A;
};

/// Value type of a vector multiplied by a matrix with value type V (vexcl/sparse/distributed.hpp:17-21): V itself, and
/// std::array<T, B> for B x B blocks.
template <class V, class Enable = void> struct rhs_of { typedef V type; };
template <class T, size_t B> struct rhs_of<std::array<std::array<T, B>, B>> { typedef std::array<T, B> type; };

namespace detail_sparse {
template <class V> struct is_block_value : std::false_type {};
template <class T, size_t B> struct is_block_value<std::array<std::array<T, B>, B>> : std::true_type {};
}

/// Block matrices: B x B blocks of double or float as values (B = 2, 3, 4), the reference's custom value types
/// (tests/sparse_matrices.cpp:239-282) for real blocks.  Row and column counts, ptr and col are in blocks; x and y are
/// vex::vector<std::array<T, B>>.  csr, ell and matrix all take the one block format of libvexb200 (sliced ELL over
/// block rows, vexb_bsr_create).  `Y = A * X`, `Y += A * X` and `Y -= A * X` are one vexb_bspmv launch into Y; the
/// product has no kernel form, so it takes part in no other expression.
template <int Format, typename T, size_t B, typename Col, typename Ptr>
class single_device_matrix<Format, std::array<std::array<T, B>, B>, Col, Ptr> {
    public:
        typedef std::array<std::array<T, B>, B> value_type; typedef value_type val_type; typedef Col col_type; typedef Ptr ptr_type;
        typedef typename rhs_of<value_type>::type rhs_type;
        static_assert(std::is_same<T, double>::value || std::is_same<T, float>::value, "block values must be double or float");
        static_assert(B >= 2 && B <= 4, "blocks must be 2x2, 3x3 or 4x4");
        static_assert(sizeof(rhs_type) == B * sizeof(T) && sizeof(value_type) == B * B * sizeof(T),
                      "std::array must hold its elements without padding");

        template <class PtrRange, class ColRange, class ValRange>
        single_device_matrix(const std::vector<backend::command_queue> &q, size_t nrows, size_t ncols,
                             const PtrRange &ptr, const ColRange &col, const ValRange &val, bool /*fast_setup*/ = true)
            : q(q), n(nrows), m(ncols), nnz(detail_sparse::range_size(val))
        {
            precondition(q.size() == 1, "sparse matrices of this kind are only supported for single-device contexts");
            static_assert(sizeof(Col) == 4 || sizeof(Col) == 8, "column type must be 32 or 64 bit");
            static_assert(sizeof(Ptr) == 4 || sizeof(Ptr) == 8, "pointer type must be 32 or 64 bit");
            vexb_bspmat *h = nullptr;
            VEXB_CHECKED(vexb_bsr_create(q[0].ordinal(), q[0].raw(), nrows, ncols, static_cast<int>(B), detail_sparse::range_data(ptr),
                                         sizeof(Ptr), detail_sparse::range_data(col), sizeof(Col), detail_sparse::range_data(val),
                                         dtype_of<T>::value, &h));
            A.reset(h, [](vexb_bspmat *p) { vexb_bspmat_destroy(p); });
        }
        single_device_matrix() : n(0), m(0), nnz(0) {}

        size_t rows() const { return n; }
        size_t cols() const { return m; }
        size_t nonzeros() const { return nnz; }
        const std::vector<backend::command_queue>& queue_list() const { return q; }

        /// y = alpha * A * x   or   y += alpha * A * x
        void mul(const vex::vector<rhs_type> &x, vex::vector<rhs_type> &y, double alpha = 1, bool append = false) const {
            precondition(x.size() == m && y.size() == n, "sparse product: vector sizes do not match the matrix");
            VEXB_CHECKED(vexb_bspmv(q[0].ordinal(), q[0].raw(), A.get(), x(0).raw(), y(0).raw(), alpha, append));
        }

        friend direct_product<single_device_matrix, vex::vector<rhs_type>> operator*(const single_device_matrix &A, const vex::vector<rhs_type> &x) {
            return direct_product<single_device_matrix, vex::vector<rhs_type>>(A, x);
        }
        template <class Expr>
        friend typename std::enable_if<is_vector_expr<Expr>::value && !std::is_same<Expr, vex::vector<rhs_type>>::value,
                                       direct_product<single_device_matrix, Expr>>::type
        operator*(const single_device_matrix &A, const Expr &x) {
            static_assert(sizeof(Expr) == 0, "a block matrix multiplies a vex::vector<std::array<T, B>> of its own T and B only");
            return direct_product<single_device_matrix, Expr>(A, x);
        }
    private:
        std::vector<backend::command_queue> q;
        size_t n, m, nnz;
        std::shared_ptr<vexb_bspmat> A;
};

namespace detail_sparse {
template <class V> struct is_complex_value : std::false_type {};
template <class T> struct is_complex_value<std::complex<T>> : std::true_type {};
template <class V> struct is_user_value
    : std::integral_constant<bool, vex::is_user_value<V>::value && !is_block_value<V>::value && !is_complex_value<V>::value> {};
}

/// Complex matrices: std::complex<double> or std::complex<float> values, the reference's examples/complex_spmv.cpp.  x and
/// y are vex::vector<std::complex<T>>.  csr, ell and matrix all take the one complex format of libvexb200 (sliced ELL,
/// vexb_zsr_create).  `Y = A * X`, `Y += A * X` and `Y -= A * X` are one vexb_zspmv launch into Y; the product has no
/// kernel form, so it takes part in no other expression.
template <int Format, typename T, typename Col, typename Ptr>
class single_device_matrix<Format, std::complex<T>, Col, Ptr> {
    public:
        typedef std::complex<T> value_type; typedef value_type val_type; typedef Col col_type; typedef Ptr ptr_type;
        typedef typename rhs_of<value_type>::type rhs_type;
        static_assert(std::is_same<T, double>::value || std::is_same<T, float>::value, "complex values must be std::complex<double> or std::complex<float>");
        static_assert(sizeof(value_type) == 2 * sizeof(T), "std::complex must hold (re, im) without padding");

        template <class PtrRange, class ColRange, class ValRange>
        single_device_matrix(const std::vector<backend::command_queue> &q, size_t nrows, size_t ncols,
                             const PtrRange &ptr, const ColRange &col, const ValRange &val, bool /*fast_setup*/ = true)
            : q(q), n(nrows), m(ncols), nnz(detail_sparse::range_size(val))
        {
            precondition(q.size() == 1, "sparse matrices of this kind are only supported for single-device contexts");
            static_assert(sizeof(Col) == 4 || sizeof(Col) == 8, "column type must be 32 or 64 bit");
            static_assert(sizeof(Ptr) == 4 || sizeof(Ptr) == 8, "pointer type must be 32 or 64 bit");
            vexb_zspmat *h = nullptr;
            VEXB_CHECKED(vexb_zsr_create(q[0].ordinal(), q[0].raw(), nrows, ncols, detail_sparse::range_data(ptr), sizeof(Ptr),
                                         detail_sparse::range_data(col), sizeof(Col), detail_sparse::range_data(val),
                                         dtype_of<T>::value, &h));
            A.reset(h, [](vexb_zspmat *p) { vexb_zspmat_destroy(p); });
        }
        single_device_matrix() : n(0), m(0), nnz(0) {}

        size_t rows() const { return n; }
        size_t cols() const { return m; }
        size_t nonzeros() const { return nnz; }
        const std::vector<backend::command_queue>& queue_list() const { return q; }

        /// y = alpha * A * x   or   y += alpha * A * x, alpha real
        void mul(const vex::vector<rhs_type> &x, vex::vector<rhs_type> &y, double alpha = 1, bool append = false) const {
            precondition(x.size() == m && y.size() == n, "sparse product: vector sizes do not match the matrix");
            VEXB_CHECKED(vexb_zspmv(q[0].ordinal(), q[0].raw(), A.get(), x(0).raw(), y(0).raw(), alpha, append));
        }

        friend direct_product<single_device_matrix, vex::vector<rhs_type>> operator*(const single_device_matrix &A, const vex::vector<rhs_type> &x) {
            return direct_product<single_device_matrix, vex::vector<rhs_type>>(A, x);
        }
        template <class Expr>
        friend typename std::enable_if<is_vector_expr<Expr>::value && !std::is_same<Expr, vex::vector<rhs_type>>::value,
                                       direct_product<single_device_matrix, Expr>>::type
        operator*(const single_device_matrix &A, const Expr &x) {
            static_assert(sizeof(Expr) == 0, "a complex matrix multiplies a vex::vector<std::complex<T>> of its own T only");
            return direct_product<single_device_matrix, Expr>(A, x);
        }
    private:
        std::vector<backend::command_queue> q;
        size_t n, m, nnz;
        std::shared_ptr<vexb_zspmat> A;
};

/// Matrices of a user value type V (vex::is_user_value: is_cl_native<V> specialised true, V neither arithmetic, nor a
/// block, nor complex), the reference's sparse/spmv_ops.hpp: x and y are vex::vector<rhs_of<V>::type>, and the product is
/// generated from spmv_ops_impl<V, rhs_of<V>::type>, whose snippets are built once, here, and compiled by NVRTC at the
/// first product on a device.  csr, ell and matrix all take the one user-value format of libvexb200 (sliced ELL,
/// vexb_usr_create).  `Y = A * X` and `Y += A * X` are one vexb_usr_spmv launch into Y.  spmv_ops_impl has no hook for
/// negation or scaling, so `Y -= A * X` and scaled products stop at a static_assert, and the product takes part in no
/// other expression.
template <int Format, typename V, typename Col, typename Ptr>
class single_device_matrix<Format, V, Col, Ptr, typename std::enable_if<detail_sparse::is_user_value<V>::value>::type> {
    public:
        typedef V value_type; typedef value_type val_type; typedef Col col_type; typedef Ptr ptr_type;
        typedef typename rhs_of<value_type>::type rhs_type;
        static const bool scales = false;           // direct_product: no Y -= A * X
        static_assert(sizeof(V) % 4 == 0 && sizeof(V) <= 64, "a user value type must be a multiple of 4 bytes, at most 64");

        template <class PtrRange, class ColRange, class ValRange>
        single_device_matrix(const std::vector<backend::command_queue> &q, size_t nrows, size_t ncols,
                             const PtrRange &ptr, const ColRange &col, const ValRange &val, bool /*fast_setup*/ = true)
            : q(q), n(nrows), m(ncols), nnz(detail_sparse::range_size(val))
        {
            precondition(q.size() == 1, "sparse matrices of this kind are only supported for single-device contexts");
            static_assert(sizeof(Col) == 4 || sizeof(Col) == 8, "column type must be 32 or 64 bit");
            static_assert(sizeof(Ptr) == 4 || sizeof(Ptr) == 8, "pointer type must be 32 or 64 bit");
            typedef spmv_ops_impl<value_type, rhs_type> ops;
            backend::source_generator d, p, a;
            ops::decl_accum_var(d, "sum");
            ops::append_product(p, "sum", "v", "xv");
            ops::append(a, "t", "sum");
            src = std::make_shared<std::array<std::string, 5>>(std::array<std::string, 5>{
                {type_name<value_type>(), type_name<rhs_type>(), d.str(), p.str(), a.str()}});
            vexb_usrmat *h = nullptr;
            VEXB_CHECKED(vexb_usr_create(q[0].ordinal(), q[0].raw(), nrows, ncols, detail_sparse::range_data(ptr), sizeof(Ptr),
                                         detail_sparse::range_data(col), sizeof(Col), detail_sparse::range_data(val),
                                         static_cast<int>(sizeof(value_type)), &h));
            A.reset(h, [](vexb_usrmat *p) { vexb_usrmat_destroy(p); });
        }
        single_device_matrix() : n(0), m(0), nnz(0) {}

        size_t rows() const { return n; }
        size_t cols() const { return m; }
        size_t nonzeros() const { return nnz; }
        const std::vector<backend::command_queue>& queue_list() const { return q; }

        /// y = A * x   or   y += A * x; alpha must be 1 (Y -= A * X does not compile)
        void mul(const vex::vector<rhs_type> &x, vex::vector<rhs_type> &y, double alpha = 1, bool append = false) const {
            precondition(alpha == 1, "a product of a user value type is not scaled");
            precondition(x.size() == m && y.size() == n, "sparse product: vector sizes do not match the matrix");
            const std::array<std::string, 5> &s = *src;
            vexb_usr_ops o;
            o.val_type = s[0].c_str(); o.rhs_type = s[1].c_str(); o.rhs_bytes = sizeof(rhs_type);
            o.decl = s[2].c_str(); o.product = s[3].c_str(); o.append = s[4].c_str();
            VEXB_CHECKED(vexb_usr_spmv(q[0].ordinal(), q[0].raw(), A.get(), &o, x(0).raw(), y(0).raw(), append));
        }

        friend direct_product<single_device_matrix, vex::vector<rhs_type>> operator*(const single_device_matrix &A, const vex::vector<rhs_type> &x) {
            return direct_product<single_device_matrix, vex::vector<rhs_type>>(A, x);
        }
        template <class Expr>
        friend typename std::enable_if<is_vector_expr<Expr>::value && !std::is_same<Expr, vex::vector<rhs_type>>::value,
                                       direct_product<single_device_matrix, Expr>>::type
        operator*(const single_device_matrix &A, const Expr &x) {
            static_assert(sizeof(Expr) == 0, "a matrix of a user value type multiplies a vex::vector<rhs_of<V>::type> only");
            return direct_product<single_device_matrix, Expr>(A, x);
        }
    private:
        std::vector<backend::command_queue> q;
        size_t n, m, nnz;
        std::shared_ptr<const std::array<std::string, 5>> src;     // device names of V and X, decl, product, append
        std::shared_ptr<vexb_usrmat> A;
};

template <typename Val, typename Col = int, typename Ptr = Col> using csr   = single_device_matrix<VEXB_FMT_CSR,  Val, Col, Ptr>;
template <typename Val, typename Col = int, typename Ptr = Col> using ell    = single_device_matrix<VEXB_FMT_HELL, Val, Col, Ptr>;
template <typename Val, typename Col = int, typename Ptr = Col> using matrix = single_device_matrix<VEXB_FMT_AUTO, Val, Col, Ptr>;

} // namespace sparse
} // namespace vex
#endif
